// Host tokenizer of the C++ layer: the `tokenizer.json` pipeline the reference runs through the
// HF `tokenizers` crate inside model2vec-rs (encode_with_args -> tokenizer.encode_batch_fast(..,
// add_special_tokens = false), reference call site src/search/mod.rs:69), restated for the subset of
// components a SentencePiece-style static-embedding model uses:
//   normalizer     Sequence | Lowercase | Replace (string pattern, or the regex " {2,}") | Strip |
//                  Prepend | Precompiled (the SentencePiece charsmap carried by tokenizer.json --
//                  nmt_nfkc for the XLM-R family the reference's model uses: double-array trie +
//                  replacement blob, applied grapheme by grapheme exactly as tokenizers'
//                  normalizers/precompiled.rs does, quirks included; extended grapheme clusters per
//                  UAX #29 from generated property tables, grapheme_break.inc) |
//                  NFC/NFD/NFKC/NFKD/Nmt (identity on printable ASCII; a line with other characters
//                  is REFUSED with an error -- those composition tables are not restated here)
//   pre_tokenizer  Metaspace (replacement, prepend_scheme always|first|never, split) | WhitespaceSplit |
//                  Sequence of those
//   added_tokens   split out of the text before the model sees it, as AddedVocabulary::extract_and_normalize does:
//                  normalized = false tokens on the raw text, normalized = true tokens on the normalised
//                  pieces; leftmost-longest, lstrip / rstrip honoured; single_word = true is refused.
//                  (A document line that contains "<s>" or "<mask>" literally gets that token's id.)
//   model          Unigram (vocab [[token, score]...], unk_id, byte_fallback = false): Viterbi over a
//                  byte trie exactly as tokenizers' `encode_optimized` (f64 scores, strict > on ties,
//                  unknown characters at min_score - 10, consecutive unknowns fused into one token)
// Anything else in tokenizer.json fails the constructor with a clear message.  Output ids are
// checked token for token against HF `tokenizers` on synthetic vocabularies (tests/test_host_cpp.py);
// the real model's tokenizer.json is not available offline (SURVEY 8c: parity unpinned for it).
#pragma once

#include <cstdint>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "semtools_host.hpp"
#include "semtools_store.hpp"   // Json

namespace semtools {

class HfTokenizer : public Tokenizer {
 public:
  explicit HfTokenizer(const std::string &tokenizer_json_path);
  // the same from the bytes of a tokenizer.json (stb_tokenizer_load)
  static std::unique_ptr<HfTokenizer> from_json(const std::string &json_text);
  // ids of one line as encode_with_args prepares them: the id of the model's `unk_token` removed -- when the
  // model section NAMES one (WordPiece / BPE style "unk_token": "<tok>"; model2vec-rs reads exactly that key,
  // [UPSTREAM-MEMORY]).  A Unigram section carries `unk_id` instead, so -- as in the Python host and in
  // model2vec itself -- nothing is dropped and an unknown character pools the unk row.
  std::vector<uint32_t> encode(const std::string &text) const override;
  // ids exactly as tokenizer.encode(text, add_special_tokens = false).ids
  std::vector<uint32_t> encode_raw(const std::string &text) const;
  // the normalizer alone (tokenizer.normalizer.normalize_str)
  std::string normalize_str(const std::string &text) const { return normalize(text); }
  size_t median_token_length() const override { return median_len_; }
  size_t vocab_size() const { return tokens_.size(); }
  bool has_unk() const { return has_unk_; }
  uint32_t unk_id() const { return unk_id_; }
  bool drops_unk() const { return drop_unk_; }
  // fnv1a64 of the file: part of the store's model fingerprint
  uint64_t fingerprint() const { return file_hash_; }

  // What the library's GPU tokenizer (stb_embed_text) restates: encode_raw's fast path -- a single Metaspace
  // step with split = true -- on lines of printable ASCII, where every normaliser step is one of the ops below.
  // ok = false: the shape has no GPU form and every line stays on the host.
  enum AsciiOpKind { OP_LOWER = 0, OP_MULTISPACE, OP_STRIP, OP_PREPEND };
  struct AsciiOp { int kind; bool left = true, right = true; std::string text; };
  struct AsciiPlan {
    bool ok = false;
    std::vector<AsciiOp> ops;              // the normaliser on printable ASCII, in order (Precompiled steps are the identity there)
    bool byte_ok[128] = {};                // printable bytes every Precompiled step leaves alone, as they are and lowercased
    size_t grow = 0;                       // bytes the Prepend steps can add to a line
    std::string replacement;               // Metaspace: one non-ASCII character
    int prepend_scheme = 0;                // 0 always, 1 first, 2 never
    std::vector<std::string> added;        // contents of every added token, normalised or not
    bool added_normalized = false;         // some of them are matched in the normalised text
    // a left Strip under prepend scheme "first": HF decides "first" by the original offset of the split, which a
    // stripped leading space moves off 0, so a line that starts with a space is not taken
    bool decline_leading_space = false;
  };
  AsciiPlan ascii_plan() const;
  // What the UTF-8 GPU tokenizer (STB_TOKENIZER_UTF8) restates, for a shape ascii_plan() accepts: the normaliser
  // steps in order, Precompiled included (kind OP_PRECOMPILED, charsmap maps[map]), and the host tables those steps
  // read -- the charsmaps' darts-clone units and replacement blobs, the grapheme-break properties (BMP as one byte
  // per code point: gcb | ext_pict << 4 | incb << 5; supplementary planes through the three range tables) and the
  // per-character lowercase map.  Pointers stay valid for the tokenizer's lifetime.
  enum { OP_PRECOMPILED = OP_PREPEND + 1 };
  struct Utf8Op { int kind; bool left = true, right = true; std::string text; int map = -1; };
  struct CharsmapView { const uint32_t *trie; size_t n_trie; const char *normalized; size_t n_normalized; const bool *ascii_plain; };
  struct PropRange { uint32_t a, b; uint8_t v; };
  struct Utf8View {
    std::vector<Utf8Op> ops;
    std::vector<CharsmapView> maps;
    const uint8_t *gb_bmp;                                   // 0x10000 bytes
    const PropRange *gcb, *ext_pict, *incb;
    size_t n_gcb, n_ext_pict, n_incb;
    const LowerEntry *lower;
    size_t n_lower;
  };
  Utf8View utf8_view() const;
  // The Unigram model as unigram() reads it: root_[256], first_child_[n_nodes + 1], child_byte_ / child_node_
  // [n_edges], terminal_[n_nodes], scores_[vocab]
  struct TrieView {
    const uint32_t *root; const uint32_t *first_child; const uint8_t *child_byte; const uint32_t *child_node;
    const int32_t *terminal; size_t n_nodes, n_edges;
    const double *scores; size_t n_scores; double unk_score;   // min_score - 10
    bool has_unk; uint32_t unk_id; bool drop_unk; uint32_t drop_id;
  };
  TrieView trie() const;

 private:
  HfTokenizer() = default;
  void load(const std::string &json_text);
  struct NormStep { int kind; std::string a, b; bool left = true, right = true; int map = -1; };
  // SentencePiece precompiled charsmap: darts-clone double array + NUL-separated replacement strings
  struct Charsmap {
    std::vector<uint32_t> trie;
    std::string normalized;
    // offset of the replacement of the SHORTEST key that is a prefix of p[0..n), or -1
    // (spm_precompiled: common_prefix_search(...)[0])
    int64_t first_prefix(const char *p, size_t n) const;
    bool ascii_plain[128] = {};   // printable ASCII bytes the map leaves alone when they stand alone
  };
  std::string apply_charsmap(const Charsmap &m, const std::string &s) const;
  struct PreStep { int kind; std::string replacement; int prepend = 0; bool split = true; };
  struct Added { std::string content; uint32_t id = 0; bool lstrip = false, rstrip = false; };
  struct Seg { int64_t id; std::string text; size_t start; };          // id < 0: plain text
  void split_added(const std::string &s, const std::vector<Added> &set, std::vector<Seg> &out) const;
  std::string normalize(const std::string &text) const;
  void pre_tokenize(const std::string &normalized, std::vector<std::string> &pieces, bool at_origin = true) const;
  void unigram(const std::string &piece, std::vector<uint32_t> &out) const;
  void add_norm(const Json &j);
  void add_pre(const Json &j);

  std::vector<NormStep> norm_;
  std::vector<Charsmap> maps_;
  std::vector<Added> added_raw_, added_norm_;                          // normalized = false / true
  std::vector<PreStep> pre_;
  std::vector<std::string> tokens_;
  std::vector<double> scores_;
  double min_score_ = 0.0;
  bool has_unk_ = false;           // Unigram unk_id: what unknown characters are mapped to
  uint32_t unk_id_ = 0;
  bool drop_unk_ = false;          // model.unk_token named and found: encode() removes drop_id_
  uint32_t drop_id_ = 0;
  size_t median_len_ = 1;
  uint64_t file_hash_ = 0;
  // byte trie, flattened after construction: node n's children are child_byte_/child_node_
  // [first_child_[n], first_child_[n + 1]) sorted by byte (the root has a direct 256-entry table);
  // terminal_[node] = token id or -1
  uint32_t step(uint32_t node, unsigned char c) const;      // child or UINT32_MAX
  std::vector<uint32_t> first_child_, child_node_;
  std::vector<uint8_t> child_byte_;
  uint32_t root_[256];
  std::vector<int32_t> terminal_;
};

// Extended grapheme clusters (UAX #29, GB1-GB13 including GB9c and GB11) of a UTF-8 string: the END offset
// of every cluster, in order (what unicode_segmentation::graphemes(true) yields).  Bytes that are not valid
// UTF-8 stand alone.
std::vector<size_t> grapheme_ends(const std::string &s);

}  // namespace semtools

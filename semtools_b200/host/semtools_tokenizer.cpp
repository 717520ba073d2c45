// HfTokenizer: tokenizer.json (Unigram + Metaspace subset) on the host.  See semtools_tokenizer.hpp.
// Semantics follow HF `tokenizers` 0.21/0.22 (the crate model2vec-rs 0.1.3 links; Cargo.lock:4375):
//   normalizers/{utils.rs,replace.rs,strip.rs,prepend.rs,precompiled.rs}, pre_tokenizers/metaspace.rs,
//   models/unigram/model.rs (encode_optimized, fuse_unk = true, K_UNK_PENALTY = 10);
//   Precompiled: crate spm_precompiled 0.1 (darts-clone unit layout, common_prefix_search) over
//   unicode_segmentation's extended grapheme clusters.
#include "semtools_tokenizer.hpp"

#include <algorithm>
#include <fstream>
#include <sstream>
#include <stdexcept>

extern "C" uint64_t stb_fnv1a64(const uint8_t *bytes, uint64_t len);

namespace semtools {

namespace {
enum { N_LOWER = 0, N_REPLACE_STR, N_REPLACE_MULTISPACE, N_STRIP, N_PREPEND, N_UNICODE_ASCII_ONLY, N_PRECOMPILED };
enum { P_METASPACE = 0, P_WHITESPACE_SPLIT };
enum { PREPEND_ALWAYS = 0, PREPEND_FIRST, PREPEND_NEVER };

std::string slurp(const std::string &p) {
  std::ifstream f(p, std::ios::binary);
  if (!f) throw std::runtime_error("cannot read " + p);
  std::stringstream ss; ss << f.rdbuf(); return ss.str();
}
const Json &need(const Json &j, const char *key, const char *where) {
  const Json *v = j.get(key);
  if (!v) throw std::runtime_error(std::string("tokenizer.json: ") + where + " lacks \"" + key + "\"");
  return *v;
}
std::string type_of(const Json &j) {
  const Json *t = j.get("type");
  return (t && t->type == Json::Str) ? t->str : "";
}
inline size_t utf8_len(unsigned char c) { return c < 0x80 ? 1 : (c >> 5) == 6 ? 2 : (c >> 4) == 14 ? 3 : (c >> 3) == 30 ? 4 : 1; }
// Unicode White_Space (what Rust's char::is_whitespace tests)
bool is_space_at(const std::string &s, size_t i, size_t *len) {
  const unsigned char c = (unsigned char)s[i];
  if (c < 0x80) { *len = 1; return c == ' ' || (c >= 9 && c <= 13); }
  const size_t n = utf8_len(c);
  *len = n;
  if (i + n > s.size()) return false;
  uint32_t cp = 0;
  if (n == 2) cp = ((c & 0x1F) << 6) | ((unsigned char)s[i + 1] & 0x3F);
  else if (n == 3) cp = ((c & 0x0F) << 12) | (((unsigned char)s[i + 1] & 0x3F) << 6) | ((unsigned char)s[i + 2] & 0x3F);
  else return false;
  return cp == 0x85 || cp == 0xA0 || cp == 0x1680 || (cp >= 0x2000 && cp <= 0x200A) || cp == 0x2028 || cp == 0x2029 || cp == 0x202F ||
         cp == 0x205F || cp == 0x3000;
}

// ---- extended grapheme clusters (UAX #29) -------------------------------------------------------
using GbRange = HfTokenizer::PropRange;
#include "grapheme_break.inc"
enum { GB_OTHER = 0, GB_CR, GB_LF, GB_CONTROL, GB_EXTEND, GB_ZWJ, GB_RI, GB_PREPEND, GB_SPACINGMARK, GB_L, GB_V, GB_T, GB_LV, GB_LVT };
enum { INCB_NONE = 0, INCB_CONSONANT, INCB_EXTEND, INCB_LINKER };

template <size_t N>
uint8_t gb_lookup(const GbRange (&t)[N], uint32_t cp) {
  size_t lo = 0, hi = N;
  while (lo < hi) { const size_t mid = (lo + hi) >> 1; if (t[mid].b < cp) lo = mid + 1; else hi = mid; }
  return (lo < N && t[lo].a <= cp) ? t[lo].v : 0;
}
inline uint8_t gcb_of(uint32_t cp) {
  if (cp >= 0xAC00 && cp <= 0xD7A3) return (cp - 0xAC00) % 28 == 0 ? GB_LV : GB_LVT;
  return gb_lookup(kGcbRanges, cp);
}
// all three properties of a code point in one byte: gcb | ext_pict << 4 | incb << 5; the BMP is a direct table
// built once (function-local static: thread-safe), supplementary planes go through the range tables
inline uint8_t gb_props_slow(uint32_t cp) {
  return (uint8_t)(gcb_of(cp) | (gb_lookup(kExtPictRanges, cp) ? 0x10 : 0) | (gb_lookup(kInCbRanges, cp) << 5));
}
const std::vector<uint8_t> &gb_bmp() {
  static const std::vector<uint8_t> bmp = [] {
    std::vector<uint8_t> t(0x10000);
    for (uint32_t c = 0; c < 0x10000; ++c) t[c] = gb_props_slow(c);
    return t;
  }();
  return bmp;
}
inline uint8_t gb_props(uint32_t cp) { return cp < 0x10000 ? gb_bmp()[cp] : gb_props_slow(cp); }
// one scalar value at s[i]; malformed sequences yield the single byte as an (unassigned-looking) code point
inline uint32_t decode_at(const std::string &s, size_t i, size_t *len) {
  const unsigned char c = (unsigned char)s[i];
  size_t n = utf8_len(c);
  if (c < 0x80) { *len = 1; return c; }
  if (n == 1 || i + n > s.size()) { *len = 1; return 0xFFFD; }
  uint32_t cp = n == 2 ? (c & 0x1F) : n == 3 ? (c & 0x0F) : (c & 0x07);
  for (size_t k = 1; k < n; ++k) {
    const unsigned char d = (unsigned char)s[i + k];
    if ((d & 0xC0) != 0x80) { *len = 1; return 0xFFFD; }
    cp = (cp << 6) | (d & 0x3F);
  }
  *len = n;
  return cp;
}

std::string b64_decode(const std::string &in) {
  static int8_t T[256]; static bool init = false;
  if (!init) {
    for (int i = 0; i < 256; ++i) T[i] = -1;
    const char *A = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    for (int i = 0; i < 64; ++i) T[(unsigned char)A[i]] = (int8_t)i;
    init = true;
  }
  std::string out;
  out.reserve(in.size() * 3 / 4);
  uint32_t acc = 0; int bits = 0;
  for (unsigned char c : in) {
    if (c == '=') break;
    if (T[c] < 0) { if (c == '\n' || c == '\r' || c == ' ') continue; throw std::runtime_error("tokenizer.json: precompiled_charsmap is not base64"); }
    acc = (acc << 6) | (uint32_t)T[c]; bits += 6;
    if (bits >= 8) { bits -= 8; out.push_back((char)((acc >> bits) & 0xFF)); }
  }
  return out;
}
}  // namespace

std::vector<size_t> grapheme_ends(const std::string &s) {
  std::vector<size_t> ends;
  size_t i = 0, len = 0;
  int prev = -1, ri_run = 0, ep_state = 0, incb_state = 0;   // ep: 1 = ExtPict Extend*, 2 = ... ZWJ; incb: 1 = Consonant [Extend|Linker]*, 2 = with a Linker
  while (i < s.size()) {
    const uint32_t cp = decode_at(s, i, &len);
    const uint8_t props = gb_props(cp);
    const int c = props & 0x0F;
    const bool ep = (props & 0x10) != 0;
    const int incb = props >> 5;
    if (prev >= 0) {
      bool brk;
      if (prev == GB_CR && c == GB_LF) brk = false;                                              // GB3
      else if (prev == GB_CONTROL || prev == GB_CR || prev == GB_LF) brk = true;                 // GB4
      else if (c == GB_CONTROL || c == GB_CR || c == GB_LF) brk = true;                          // GB5
      else if (prev == GB_L && (c == GB_L || c == GB_V || c == GB_LV || c == GB_LVT)) brk = false;   // GB6
      else if ((prev == GB_LV || prev == GB_V) && (c == GB_V || c == GB_T)) brk = false;         // GB7
      else if ((prev == GB_LVT || prev == GB_T) && c == GB_T) brk = false;                       // GB8
      else if (c == GB_EXTEND || c == GB_ZWJ) brk = false;                                       // GB9
      else if (c == GB_SPACINGMARK) brk = false;                                                 // GB9a
      else if (prev == GB_PREPEND) brk = false;                                                  // GB9b
      else if (incb_state == 2 && incb == INCB_CONSONANT) brk = false;                           // GB9c
      else if (ep_state == 2 && ep) brk = false;                                                 // GB11
      else if (prev == GB_RI && c == GB_RI && (ri_run & 1)) brk = false;                         // GB12, GB13
      else brk = true;                                                                           // GB999
      if (brk) ends.push_back(i);
    }
    ri_run = c == GB_RI ? ri_run + 1 : 0;
    if (ep) ep_state = 1;
    else if (ep_state == 1 && c == GB_EXTEND) ep_state = 1;
    else if (ep_state == 1 && c == GB_ZWJ) ep_state = 2;
    else ep_state = 0;
    if (incb == INCB_CONSONANT) incb_state = 1;
    else if (incb_state >= 1 && incb == INCB_EXTEND) { /* keeps its state */ }
    else if (incb_state >= 1 && incb == INCB_LINKER) incb_state = 2;
    else incb_state = 0;
    prev = c;
    i += len;
  }
  if (!s.empty()) ends.push_back(s.size());
  return ends;
}

// darts-clone unit layout (sentencepiece third_party/darts_clone, restated by spm_precompiled)
int64_t HfTokenizer::Charsmap::first_prefix(const char *p, size_t n) const {
  if (trie.empty()) return -1;
  auto has_leaf = [](uint32_t u) { return ((u >> 8) & 1u) == 1u; };
  auto value = [](uint32_t u) { return u & ((1u << 31) - 1u); };
  auto label = [](uint32_t u) { return u & ((1u << 31) | 0xFFu); };
  auto offset = [](uint32_t u) { return (size_t)(u >> 10) << ((u & (1u << 9)) >> 6); };
  size_t node = 0;
  uint32_t unit = trie[0];
  node ^= offset(unit);
  for (size_t i = 0; i < n; ++i) {
    const unsigned char c = (unsigned char)p[i];
    if (c == 0) break;
    node ^= c;
    if (node >= trie.size()) return -1;
    unit = trie[node];
    if (label(unit) != c) return -1;
    node ^= offset(unit);
    if (has_leaf(unit)) {
      if (node >= trie.size()) return -1;
      return (int64_t)value(trie[node]);
    }
  }
  return -1;
}

// normalizers/precompiled.rs: every grapheme shorter than 6 bytes is looked up WHOLE first (the first,
// i.e. shortest, key that is a prefix of it replaces the whole grapheme); otherwise character by character
std::string HfTokenizer::apply_charsmap(const Charsmap &m, const std::string &s) const {
  if (m.trie.empty()) return s;
  std::string o;
  o.reserve(s.size());
  auto emit = [&](int64_t at) { for (size_t k = (size_t)at; k < m.normalized.size() && m.normalized[k] != 0; ++k) o.push_back(m.normalized[k]); };
  auto slow = [&](const std::string &seg) {
    size_t b = 0;
    for (size_t e : grapheme_ends(seg)) {
      bool done = false;
      if (e - b < 6) {
        const int64_t at = m.first_prefix(seg.data() + b, e - b);
        if (at >= 0) { emit(at); done = true; }
      }
      if (!done) {
        size_t i = b, len = 0;
        while (i < e) {
          decode_at(seg, i, &len);
          const int64_t at = m.first_prefix(seg.data() + i, len);
          if (at >= 0) emit(at); else o.append(seg, i, len);
          i += len;
        }
      }
      b = e;
    }
  };
  // Fast path: a printable ASCII character between ASCII neighbours is a grapheme of its own (it is neither
  // Extend / SpacingMark / ZWJ nor preceded by a Prepend character, and no ASCII character is
  // Extended_Pictographic or an Indic consonant), so cluster boundaries on both sides are certain; if the map
  // leaves it alone it is copied.  Everything else goes through the grapheme walk, one maximal segment at a time.
  const size_t n = s.size();
  auto fast = [&](size_t i) {
    const unsigned char c = (unsigned char)s[i];
    return c >= 0x20 && c < 0x7F && m.ascii_plain[c] && (i + 1 == n || (unsigned char)s[i + 1] < 0x80) && (i == 0 || (unsigned char)s[i - 1] < 0x80);
  };
  size_t i = 0;
  while (i < n) {
    if (fast(i)) { o.push_back(s[i]); ++i; continue; }
    size_t j = i + 1;
    while (j < n && !fast(j)) ++j;
    slow(s.substr(i, j - i));
    i = j;
  }
  return o;
}

void HfTokenizer::add_norm(const Json &j) {
  if (j.type == Json::Null) return;
  const std::string t = type_of(j);
  if (t == "Sequence") { for (const auto &n : need(j, "normalizers", "Sequence normalizer").arr) add_norm(n); return; }
  if (t == "Lowercase") { norm_.push_back({N_LOWER, "", ""}); return; }
  if (t == "Replace") {
    const Json &pat = need(j, "pattern", "Replace normalizer");
    const std::string content = need(j, "content", "Replace normalizer").str;
    if (const Json *s = pat.get("String")) { if (!s->str.empty()) norm_.push_back({N_REPLACE_STR, s->str, content}); return; }
    if (const Json *r = pat.get("Regex")) {
      if (r->str == " {2,}") { norm_.push_back({N_REPLACE_MULTISPACE, "", content}); return; }
      throw std::runtime_error("tokenizer.json: Replace normalizer with regex /" + r->str + "/ is not supported by the C++ host (only \" {2,}\")");
    }
    throw std::runtime_error("tokenizer.json: Replace normalizer without pattern");
  }
  if (t == "Strip") {
    NormStep s{N_STRIP, "", ""};
    if (const Json *l = j.get("strip_left")) s.left = l->b;
    if (const Json *r = j.get("strip_right")) s.right = r->b;
    norm_.push_back(s); return;
  }
  if (t == "Prepend") { norm_.push_back({N_PREPEND, need(j, "prepend", "Prepend normalizer").str, ""}); return; }
  if (t == "Precompiled") {
    Charsmap m;
    const Json *c = j.get("precompiled_charsmap");
    if (c && c->type == Json::Str && !c->str.empty()) {
      const std::string blob = b64_decode(c->str);
      if (blob.size() < 4) throw std::runtime_error("tokenizer.json: precompiled_charsmap is truncated");
      auto u32_at = [&](size_t o) { return (uint32_t)(unsigned char)blob[o] | ((uint32_t)(unsigned char)blob[o + 1] << 8) |
                                           ((uint32_t)(unsigned char)blob[o + 2] << 16) | ((uint32_t)(unsigned char)blob[o + 3] << 24); };
      const size_t trie_bytes = u32_at(0);
      if (trie_bytes % 4 != 0 || 4 + trie_bytes > blob.size()) throw std::runtime_error("tokenizer.json: precompiled_charsmap has a bad trie size");
      m.trie.resize(trie_bytes / 4);
      for (size_t k = 0; k < m.trie.size(); ++k) m.trie[k] = u32_at(4 + 4 * k);
      m.normalized = blob.substr(4 + trie_bytes);
      for (int ch = 0x20; ch < 0x7F; ++ch) { const char b1 = (char)ch; m.ascii_plain[ch] = m.first_prefix(&b1, 1) < 0; }
    }                                                        // null / empty charsmap: identity
    NormStep st{N_PRECOMPILED, "", ""};
    st.map = (int)maps_.size();
    maps_.push_back(std::move(m));
    norm_.push_back(st); return;
  }
  if (t == "NFC" || t == "NFD" || t == "NFKC" || t == "NFKD" || t == "Nmt") {
    norm_.push_back({N_UNICODE_ASCII_ONLY, t, ""}); return;
  }
  throw std::runtime_error("tokenizer.json: normalizer \"" + t + "\" is not supported by the C++ host");
}

void HfTokenizer::add_pre(const Json &j) {
  if (j.type == Json::Null) return;
  const std::string t = type_of(j);
  if (t == "Sequence") { for (const auto &n : need(j, "pretokenizers", "Sequence pre_tokenizer").arr) add_pre(n); return; }
  if (t == "Metaspace") {
    PreStep p{P_METASPACE, "\xE2\x96\x81", PREPEND_ALWAYS, true};
    if (const Json *r = j.get("replacement")) p.replacement = r->str;
    if (const Json *s = j.get("prepend_scheme")) p.prepend = s->str == "first" ? PREPEND_FIRST : s->str == "never" ? PREPEND_NEVER : PREPEND_ALWAYS;
    else if (const Json *a = j.get("add_prefix_space")) p.prepend = a->b ? PREPEND_ALWAYS : PREPEND_NEVER;   // pre-0.15 files
    if (const Json *s = j.get("split")) p.split = s->b;
    pre_.push_back(p); return;
  }
  if (t == "WhitespaceSplit") { pre_.push_back({P_WHITESPACE_SPLIT, "", 0, true}); return; }
  throw std::runtime_error("tokenizer.json: pre_tokenizer \"" + t + "\" is not supported by the C++ host");
}

HfTokenizer::HfTokenizer(const std::string &path) { load(slurp(path)); }

std::unique_ptr<HfTokenizer> HfTokenizer::from_json(const std::string &json_text) {
  std::unique_ptr<HfTokenizer> t(new HfTokenizer());
  t->load(json_text);
  return t;
}

void HfTokenizer::load(const std::string &text) {
  file_hash_ = stb_fnv1a64(reinterpret_cast<const uint8_t *>(text.data()), text.size());
  const Json j = Json::parse(text);
  if (const Json *n = j.get("normalizer")) add_norm(*n);
  if (const Json *p = j.get("pre_tokenizer")) add_pre(*p);
  const Json &model = need(j, "model", "the file");
  if (type_of(model) != "Unigram") throw std::runtime_error("tokenizer.json: model \"" + type_of(model) + "\" is not supported by the C++ host (Unigram only)");
  if (const Json *bf = model.get("byte_fallback"); bf && bf->b) throw std::runtime_error("tokenizer.json: Unigram byte_fallback is not supported by the C++ host");
  if (const Json *u = model.get("unk_id"); u && u->type == Json::Num) { has_unk_ = true; unk_id_ = (uint32_t)std::min<uint64_t>(u->as_u64("unk_id"), 0xFFFFFFFFull); }
  const Json &vocab = need(model, "vocab", "Unigram model");
  tokens_.reserve(vocab.arr.size()); scores_.reserve(vocab.arr.size());
  for (const auto &e : vocab.arr) {
    if (e.type != Json::Arr || e.arr.size() != 2) throw std::runtime_error("tokenizer.json: malformed Unigram vocab entry");
    tokens_.push_back(e.arr[0].str);
    scores_.push_back(e.arr[1].num);
  }
  if (tokens_.empty()) throw std::runtime_error("tokenizer.json: empty vocabulary");
  if (has_unk_ && unk_id_ >= tokens_.size()) throw std::runtime_error("tokenizer.json: unk_id outside the vocabulary");
  if (const Json *ut = model.get("unk_token"); ut && ut->type == Json::Str) {      // token_to_id(unk_token): the last id carrying that string
    for (size_t id = tokens_.size(); id-- > 0;)
      if (tokens_[id] == ut->str) { drop_unk_ = true; drop_id_ = (uint32_t)id; break; }
    if (!drop_unk_) throw std::runtime_error("tokenizer.json: unk_token \"" + ut->str + "\" is not in the vocabulary");
  }
  min_score_ = *std::min_element(scores_.begin(), scores_.end());
  // byte trie; a token that occurs twice keeps the LAST id (tokenizers builds token_to_ids by insertion)
  std::unordered_map<uint64_t, uint32_t> edges;             // (node << 8 | byte) -> child, construction only
  terminal_.push_back(-1);
  for (size_t id = 0; id < tokens_.size(); ++id) {
    uint32_t node = 0;
    for (unsigned char c : tokens_[id]) {
      const uint64_t key = ((uint64_t)node << 8) | c;
      auto it = edges.find(key);
      if (it == edges.end()) { it = edges.emplace(key, (uint32_t)terminal_.size()).first; terminal_.push_back(-1); }
      node = it->second;
    }
    if (!tokens_[id].empty()) terminal_[node] = (int32_t)id;
  }
  // flatten: children of a node contiguous and sorted by byte (cache-friendly Viterbi walks)
  std::vector<std::pair<uint64_t, uint32_t>> flat(edges.begin(), edges.end());
  std::sort(flat.begin(), flat.end());
  first_child_.assign(terminal_.size() + 1, 0);
  child_byte_.resize(flat.size()); child_node_.resize(flat.size());
  for (const auto &e : flat) first_child_[(e.first >> 8) + 1]++;
  for (size_t i = 1; i < first_child_.size(); ++i) first_child_[i] += first_child_[i - 1];
  for (size_t i = 0; i < flat.size(); ++i) { child_byte_[i] = (uint8_t)(flat[i].first & 0xff); child_node_[i] = flat[i].second; }
  for (int b = 0; b < 256; ++b) root_[b] = UINT32_MAX;
  for (uint32_t i = first_child_[0]; i < first_child_[1]; ++i) root_[child_byte_[i]] = child_node_[i];
  // added tokens (added_vocabulary.rs): matched before the model; normalized ones are matched in normalised text
  if (const Json *at = j.get("added_tokens"); at && at->type == Json::Arr) {
    for (const auto &e : at->arr) {
      Added a;
      a.content = need(e, "content", "added token").str;
      a.id = (uint32_t)std::min<uint64_t>(need(e, "id", "added token").as_u64("an added token id"), 0xFFFFFFFFull);
      bool normalized = false;
      if (const Json *v = e.get("lstrip")) a.lstrip = v->b;
      if (const Json *v = e.get("rstrip")) a.rstrip = v->b;
      if (const Json *v = e.get("normalized")) normalized = v->b;
      if (const Json *v = e.get("single_word"); v && v->b) throw std::runtime_error("tokenizer.json: added token \"" + a.content + "\" has single_word = true, which the C++ host does not support");
      if (a.content.empty()) continue;
      if (normalized) { a.content = normalize(a.content); if (!a.content.empty()) added_norm_.push_back(a); }
      else added_raw_.push_back(a);
    }
  }
  // median token length in BYTES over the vocabulary (model2vec: `tk.len()` of every vocab key)
  std::vector<size_t> lens;
  lens.reserve(tokens_.size());
  for (const auto &t : tokens_) lens.push_back(t.size());
  std::sort(lens.begin(), lens.end());
  median_len_ = std::max<size_t>(1, lens[lens.size() / 2]);
}

HfTokenizer::AsciiPlan HfTokenizer::ascii_plan() const {
  AsciiPlan p, none;
  if (pre_.size() != 1 || pre_[0].kind != P_METASPACE || !pre_[0].split || !has_unk_) return none;
  const std::string &rep = pre_[0].replacement;
  // one non-ASCII character: it cannot occur in a printable-ASCII line, so only spaces delimit pieces
  if (rep.empty() || (unsigned char)rep[0] < 0x80 || utf8_len((unsigned char)rep[0]) != rep.size()) return none;
  p.replacement = rep;
  p.prepend_scheme = pre_[0].prepend;
  bool lower = false;
  for (const auto &st : norm_) lower = lower || st.kind == N_LOWER;
  for (int c = 0x20; c < 0x7F; ++c) p.byte_ok[c] = true;
  for (const auto &st : norm_) {
    switch (st.kind) {
      case N_LOWER: p.ops.push_back({OP_LOWER, true, true, ""}); break;
      case N_REPLACE_MULTISPACE:
        if (st.b != " ") return none;
        p.ops.push_back({OP_MULTISPACE, true, true, ""}); break;
      case N_STRIP:
        p.ops.push_back({OP_STRIP, st.left, st.right, ""});
        p.decline_leading_space = p.decline_leading_space || (st.left && p.prepend_scheme == PREPEND_FIRST);
        break;
      case N_PREPEND:
        p.ops.push_back({OP_PREPEND, true, true, st.a});
        p.grow += st.a.size(); break;
      case N_PRECOMPILED: {
        const Charsmap &m = maps_[st.map];
        if (m.trie.empty()) break;                           // identity
        for (int c = 0x20; c < 0x7F; ++c) {
          const int l = (lower && c >= 'A' && c <= 'Z') ? c + 32 : c;
          p.byte_ok[c] = p.byte_ok[c] && m.ascii_plain[c] && m.ascii_plain[l];
        }
        break;
      }
      default: return none;                                  // string Replace, the Unicode forms
    }
  }
  for (const auto &op : p.ops)                               // Prepend text goes through the same checks as the line
    for (unsigned char c : op.text)
      if (c < 0x20 || c > 0x7E || !p.byte_ok[c]) return none;
  for (const auto &a : added_raw_) p.added.push_back(a.content);
  for (const auto &a : added_norm_) p.added.push_back(a.content);
  p.added_normalized = !added_norm_.empty();
  p.ok = true;
  return p;
}

HfTokenizer::Utf8View HfTokenizer::utf8_view() const {
  Utf8View v;
  for (const auto &st : norm_) {
    switch (st.kind) {
      case N_LOWER: v.ops.push_back({OP_LOWER, true, true, ""}); break;
      case N_REPLACE_MULTISPACE: v.ops.push_back({OP_MULTISPACE, true, true, ""}); break;
      case N_STRIP: v.ops.push_back({OP_STRIP, st.left, st.right, ""}); break;
      case N_PREPEND: v.ops.push_back({OP_PREPEND, true, true, st.a}); break;
      case N_PRECOMPILED:
        if (!maps_[st.map].trie.empty()) v.ops.push_back({OP_PRECOMPILED, true, true, "", st.map});   // else the identity
        break;
      default: break;                                        // not a shape ascii_plan() accepts
    }
  }
  for (const auto &m : maps_) v.maps.push_back({m.trie.data(), m.trie.size(), m.normalized.data(), m.normalized.size(), m.ascii_plain});
  v.gb_bmp = gb_bmp().data();
  v.gcb = kGcbRanges; v.n_gcb = sizeof(kGcbRanges) / sizeof(kGcbRanges[0]);
  v.ext_pict = kExtPictRanges; v.n_ext_pict = sizeof(kExtPictRanges) / sizeof(kExtPictRanges[0]);
  v.incb = kInCbRanges; v.n_incb = sizeof(kInCbRanges) / sizeof(kInCbRanges[0]);
  v.lower = lower_table().data(); v.n_lower = lower_table().size();
  return v;
}

HfTokenizer::TrieView HfTokenizer::trie() const {
  return {root_, first_child_.data(), child_byte_.data(), child_node_.data(), terminal_.data(), terminal_.size(), child_node_.size(),
          scores_.data(), scores_.size(), min_score_ - 10.0, has_unk_, unk_id_, drop_unk_, drop_id_};
}

std::string HfTokenizer::normalize(const std::string &in) const {
  std::string s = in;
  for (const auto &st : norm_) {
    switch (st.kind) {
      case N_LOWER: s = to_lowercase_per_char(s); break;
      case N_REPLACE_STR: {
        std::string o; size_t pos = 0, f;
        while ((f = s.find(st.a, pos)) != std::string::npos) { o.append(s, pos, f - pos); o += st.b; pos = f + st.a.size(); }
        o.append(s, pos, std::string::npos); s.swap(o); break;
      }
      case N_REPLACE_MULTISPACE: {
        std::string o; size_t i = 0;
        while (i < s.size()) {
          if (s[i] == ' ') { size_t e = i; while (e < s.size() && s[e] == ' ') ++e; if (e - i >= 2) o += st.b; else o += ' '; i = e; }
          else o += s[i++];
        }
        s.swap(o); break;
      }
      case N_STRIP: {
        size_t b = 0, e = s.size(), l;
        if (st.left) while (b < e && is_space_at(s, b, &l)) b += l;
        if (st.right) {
          for (;;) {                                   // step back one UTF-8 character at a time
            if (e <= b) break;
            size_t k = e - 1;
            while (k > b && ((unsigned char)s[k] & 0xC0) == 0x80) --k;
            if (is_space_at(s, k, &l) && k + l == e) e = k; else break;
          }
        }
        s = s.substr(b, e - b); break;
      }
      case N_PREPEND: if (!s.empty()) s = st.a + s; break;
      case N_PRECOMPILED: s = apply_charsmap(maps_[st.map], s); break;
      case N_UNICODE_ASCII_ONLY:
        for (unsigned char c : s)
          if (c >= 0x80 || (c < 0x20 && c != '\t' && c != '\n' && c != '\r'))
            throw std::runtime_error("the C++ host applies the " + st.a + " normalizer to printable ASCII only; this line needs the Python host");
        break;
    }
  }
  return s;
}

// AddedVocabulary::find_matches: leftmost-longest matches of the set's contents, lstrip / rstrip widening
// the match over neighbouring whitespace; the text between matches stays plain (id -1)
void HfTokenizer::split_added(const std::string &s, const std::vector<Added> &set, std::vector<Seg> &out) const {
  out.clear();
  if (set.empty() || s.empty()) { out.push_back({-1, s, 0}); return; }
  size_t pos = 0, start_offset = 0;
  while (pos < s.size()) {
    const Added *best = nullptr;
    for (const auto &a : set)
      if (a.content.size() <= s.size() - pos && (!best || a.content.size() > best->content.size()) && s.compare(pos, a.content.size(), a.content) == 0) best = &a;
    if (!best) { ++pos; continue; }
    size_t start = pos, stop = pos + best->content.size(), l;
    const size_t mat_end = stop;
    if (best->lstrip) {                                      // the run of whitespace that ends at `start`
      size_t k = start;
      for (;;) {
        if (k == 0) break;
        size_t c = k - 1;
        while (c > 0 && ((unsigned char)s[c] & 0xC0) == 0x80) --c;
        if (is_space_at(s, c, &l) && c + l == k) k = c; else break;
      }
      start = std::max(k, start_offset);
    }
    if (best->rstrip) while (stop < s.size() && is_space_at(s, stop, &l)) stop += l;
    if (start_offset < start) out.push_back({-1, s.substr(start_offset, start - start_offset), start_offset});
    out.push_back({(int64_t)best->id, s.substr(start, stop - start), start});
    start_offset = stop;
    pos = mat_end;
  }
  if (start_offset < s.size()) out.push_back({-1, s.substr(start_offset), start_offset});
}

void HfTokenizer::pre_tokenize(const std::string &normalized, std::vector<std::string> &pieces, bool at_origin_in) const {
  pieces.clear();
  pieces.push_back(normalized);
  bool first_step = at_origin_in;
  for (const auto &p : pre_) {
    std::vector<std::string> next;
    size_t piece_no = 0;
    for (const auto &piece : pieces) {
      if (p.kind == P_WHITESPACE_SPLIT) {
        size_t i = 0, l;
        while (i < piece.size()) {
          while (i < piece.size() && is_space_at(piece, i, &l)) i += l;
          size_t b = i;
          while (i < piece.size() && !is_space_at(piece, i, &l)) i += l;
          if (i > b) next.push_back(piece.substr(b, i - b));
        }
      } else {
        // Metaspace: ' ' -> replacement; prepend (always | first: only the piece that starts the
        // original string | never) unless already there; split MergedWithNext on the replacement
        std::string s;
        for (char c : piece) { if (c == ' ') s += p.replacement; else s += c; }
        const bool starts = s.compare(0, p.replacement.size(), p.replacement) == 0;
        const bool at_origin = first_step && piece_no == 0;
        if (!starts && (p.prepend == PREPEND_ALWAYS || (p.prepend == PREPEND_FIRST && at_origin))) s = p.replacement + s;
        if (!p.split) { if (!s.empty()) next.push_back(s); }
        else {
          size_t b = 0, pos = p.replacement.empty() ? std::string::npos : s.find(p.replacement, 0);
          // every delimiter starts a new piece that runs up to the next delimiter
          if (pos != 0 && !s.empty()) { const size_t e = pos == std::string::npos ? s.size() : pos; next.push_back(s.substr(0, e)); b = e; }
          while (b < s.size()) {
            const size_t nxt = s.find(p.replacement, b + p.replacement.size());
            const size_t e = nxt == std::string::npos ? s.size() : nxt;
            next.push_back(s.substr(b, e - b));
            b = e;
          }
        }
      }
      ++piece_no;
    }
    pieces.swap(next);
    first_step = false;
  }
}

uint32_t HfTokenizer::step(uint32_t node, unsigned char c) const {
  if (node == 0) return root_[c];
  uint32_t lo = first_child_[node], hi = first_child_[node + 1];
  if (hi - lo <= 8) { for (; lo < hi; ++lo) if (child_byte_[lo] == c) return child_node_[lo]; return UINT32_MAX; }
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (child_byte_[mid] < c) lo = mid + 1; else hi = mid; }
  return (lo < first_child_[node + 1] && child_byte_[lo] == c) ? child_node_[lo] : UINT32_MAX;
}

// models/unigram/model.rs: encode_optimized + tokenize (string -> id, unknown strings -> unk_id)
void HfTokenizer::unigram(const std::string &s, std::vector<uint32_t> &out) const {
  const size_t size = s.size();
  if (size == 0) return;
  struct Node { uint32_t id = 0; double score = 0.0; int64_t starts_at = -1; };
  static thread_local std::vector<Node> best;           // per-thread scratch: a piece is a few bytes, the allocation was the cost
  best.assign(size + 1, Node());
  const double unk_score = min_score_ - 10.0;
  size_t at = 0;
  while (at < size) {
    const double here = best[at].score;
    bool has_single = false;
    const size_t mblen = std::min(utf8_len((unsigned char)s[at]), size - at);
    uint32_t node = 0;
    for (size_t k = at; k < size; ++k) {
      node = step(node, (unsigned char)s[k]);
      if (node == UINT32_MAX) break;
      const int32_t id = terminal_[node];
      if (id < 0) continue;
      const size_t key_pos = k + 1;
      Node &t = best[key_pos];
      const double cand = scores_[id] + here;
      if (t.starts_at < 0 || cand > t.score) { t.score = cand; t.starts_at = (int64_t)at; t.id = (uint32_t)id; }
      if (!has_single && key_pos - at == mblen) has_single = true;
    }
    if (!has_single) {
      if (!has_unk_) throw std::runtime_error("tokenizer: a character is not in the vocabulary and the model has no unk_id");
      Node &t = best[at + mblen];
      const double cand = unk_score + here;
      if (t.starts_at < 0 || cand > t.score) { t.score = cand; t.starts_at = (int64_t)at; t.id = unk_id_; }
    }
    at += mblen;
  }
  // backtrack; consecutive unknown characters fuse into ONE unk token (fuse_unk)
  static thread_local std::vector<uint32_t> rev;
  rev.clear();
  size_t ends = size;
  bool in_unk = false;
  while (ends > 0) {
    const Node &n = best[ends];
    if (has_unk_ && n.id == unk_id_) { if (!in_unk) { rev.push_back(unk_id_); in_unk = true; } }
    else { rev.push_back(n.id); in_unk = false; }
    ends = (size_t)n.starts_at;
  }
  out.insert(out.end(), rev.rbegin(), rev.rend());
}

std::vector<uint32_t> HfTokenizer::encode_raw(const std::string &text) const {
  std::vector<std::string> pieces;
  std::vector<uint32_t> ids;
  std::vector<Seg> raw, sub;
  split_added(text, added_raw_, raw);                       // 1. non-normalised added tokens, on the text as given
  for (const auto &seg : raw) {
    if (seg.id >= 0) { ids.push_back((uint32_t)seg.id); continue; }
    const std::string normalized = normalize(seg.text);     // 2. normalise what is left, then the normalised added tokens
    if (normalized.empty()) continue;                       // an empty split yields no token
    split_added(normalized, added_norm_, sub);
    for (const auto &part : sub) {
      if (part.id >= 0) { ids.push_back((uint32_t)part.id); continue; }
      if (part.text.empty()) continue;
      const bool origin = seg.start == 0 && part.start == 0;               // Metaspace "first": only the split that starts the input
      if (pre_.size() == 1 && pre_[0].kind == P_METASPACE && pre_[0].split && !pre_[0].replacement.empty()) {
        // the usual pipeline, without materialising the pieces: every space becomes the replacement and starts a piece
        // that runs to the next one; a leading replacement is added per the prepend scheme (same result as pre_tokenize)
        const PreStep &m = pre_[0];
        const std::string &t = part.text, &rep = m.replacement;
        static thread_local std::string piece;
        const bool starts = t[0] == ' ' || t.compare(0, rep.size(), rep) == 0;
        const bool prepend = !starts && (m.prepend == PREPEND_ALWAYS || (m.prepend == PREPEND_FIRST && origin));
        piece.clear();
        if (prepend) piece = rep;
        size_t i = 0;
        const size_t n = t.size();
        while (i < n) {
          const bool at_space = t[i] == ' ';
          const bool at_rep = !at_space && t.compare(i, rep.size(), rep) == 0;
          if (at_space || at_rep) {                                        // a delimiter: close the running piece, start the next with it
            if (!piece.empty()) unigram(piece, ids);
            piece = rep;
            i += at_space ? 1 : rep.size();
          } else piece.push_back(t[i++]);
        }
        if (!piece.empty()) unigram(piece, ids);
        continue;
      }
      pre_tokenize(part.text, pieces, origin);
      for (const auto &p : pieces) unigram(p, ids);
    }
  }
  return ids;
}

std::vector<uint32_t> HfTokenizer::encode(const std::string &text) const {
  std::vector<uint32_t> ids = encode_raw(text);
  if (drop_unk_) ids.erase(std::remove(ids.begin(), ids.end(), drop_id_), ids.end());  // encode_with_args: ids.retain(|id| id != unk_token_id)
  return ids;
}

}  // namespace semtools

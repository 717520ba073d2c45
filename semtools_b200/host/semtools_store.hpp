// C++ mirror of the workspace layer (reference src/workspace/mod.rs, src/workspace/store.rs)
// on the flat store format that semtools_b200/workspace.py defines (`<root>/flat.b200/`:
// store.json + rows.i32 + line_embeddings.f32).  Both implementations read and write the
// same files (tests/test_host_cpp.py round-trips them).  The nearest-neighbour query is the
// GPU's (stb_search with row ranges, STB_MODE_STORE_QUERY); nothing here computes a distance.
#pragma once
#include <cstdint>
#include <stdexcept>
#include <functional>
#include <map>
#include <optional>
#include <set>
#include <string>
#include <unordered_map>
#include <vector>

#include "semtools_host.hpp"

namespace semtools {

constexpr uint32_t CURRENT_EMBEDDING_VERSION = 2;      // store.rs:34
constexpr size_t LINE_EMBEDDING_SIZE = 256;            // store.rs:37

// The one rule for where a store's GPU mirror lives: in HBM, unless creating or uploading it there fails with
// STB_ERR_NOMEM; then its rows stay in host memory and only their q8 copy goes to HBM (stb_corpus_create_host).
// The hits are the same either way.  `create` is the device attempt (a test passes one that fails).  Returns the
// stb status; *out is the mirror holding the n rows, or null.
using CorpusCreateFn = int (*)(stb_ctx *, uint32_t, uint64_t, uint64_t, stb_corpus **);
int upload_mirror(stb_ctx *ctx, const float *rows, uint64_t n, stb_corpus **out, CorpusCreateFn create = stb_corpus_create);

struct WorkspaceConfig {                               // mod.rs:8-25
  std::string name = "default";
  std::string root_dir;
  size_t in_batch_size = 5000;
  size_t oversample_factor = 3;
};

struct Workspace {                                     // mod.rs:27-101
  WorkspaceConfig config;
  static std::string root_path(const std::string &name);
  static std::string config_path_for(const std::string &name);
  static std::string active(const std::optional<std::string> &workspace_name);   // throws "No active workspace..."
  static Workspace open(const std::optional<std::string> &workspace_name);
  void save() const;
};

struct DocMeta {                                       // store.rs:52-58
  std::string path;
  uint64_t size_bytes = 0;
  int64_t mtime = 0;
  uint32_t version = CURRENT_EMBEDDING_VERSION;        // serialised as "_version"
  uint64_t id() const;                                 // fnv1a(path), store.rs:75-80
};

struct LineEmbedding {                                 // store.rs:67-73
  std::string path;
  int32_t line_number = 0;
  std::vector<float> embedding;
  uint64_t id() const;                                 // fnv1a(path || i32 LE), store.rs:82-89
};

struct RankedLine {                                    // store.rs:91-96
  std::string path;
  int32_t line_number = 0;
  float distance = 0.f;
};

struct DocumentState {                                 // store.rs:60-65
  enum Kind { Unchanged, Changed, New } kind = Unchanged;
  std::string filename, content;
  DocMeta meta;
};

struct WorkspaceStats { size_t total_documents = 0; bool has_index = true; std::string index_type = "FLAT"; };

class Store {
 public:
  static Store open(const std::string &workspace_dir);                       // store.rs:113-183
  std::map<std::string, DocMeta> get_existing_docs(const std::vector<std::string> &paths) const;   // :185-233
  std::vector<DocumentState> analyze_document_states(const std::vector<std::string> &paths) const; // :549-611
  void upsert_document_metadata(const std::vector<DocMeta> &metas);          // :373-399
  void upsert_line_embeddings(const std::vector<LineEmbedding> &lines);      // :402-434
  void delete_document_metadata(const std::vector<std::string> &paths);      // :235-296 (current version only)
  void delete_line_embeddings(const std::vector<std::string> &paths);        // :298-357
  void delete_documents(const std::vector<std::string> &paths);              // :360-370
  std::vector<std::string> get_all_document_paths() const;                   // :447-479
  size_t count_documents() const { return docs_.size(); }                    // :613-625
  size_t count_line_embeddings() const { return rows_.size() / 2; }          // :627-637
  WorkspaceStats get_stats() const { return {docs_.size(), true, "FLAT"}; }  // :436-445 (reference hard-codes "HNSW")
  // row ranges (half-open, ascending) of the rows whose path is in `subset_paths`
  std::vector<uint64_t> ranges_for(const std::vector<std::string> &subset_paths) const;
  // Store::search_line_embeddings, store.rs:481-546, on the GPU
  std::vector<RankedLine> search_line_embeddings(const std::vector<float> &query, const std::vector<std::string> &subset_paths,
                                                 size_t top_k, std::optional<float> max_distance, int device = 0);
  const std::vector<float> &matrix() const { return emb_; }

  // fingerprint of the embedder (model + tokenizer) whose vectors this handle writes; recorded in
  // store.json.  A store written with another fingerprint has every document reported Changed.
  std::string model_fingerprint;
  const std::string &stored_model_fingerprint() const { return stored_model_; }

 private:
  // Consistency protocol shared with the Python host (workspace.py: Store): store.json is the
  // commit record ({"rows", "gen", "files", "model"}), replaced atomically after the row files hold
  // the new state; rows beyond the committed count are debris of an interrupted flush; deletions
  // write a new generation of row files; flock(<dir>/.lock) shared while loading, exclusive around
  // every mutation, which first reloads when another process committed in between.
  void load();
  void flush();
  template <class F> void mutate(F &&apply);
  uint64_t disk_gen() const;
  std::string dir_;
  uint64_t gen_ = 0;
  std::string rows_file_ = "rows.i32", emb_file_ = "line_embeddings.f32";
  std::string stored_model_;
  std::vector<std::string> paths_;
  std::unordered_map<std::string, int32_t> path_idx_;
  std::vector<DocMeta> docs_;                       // insertion order, as the Python dict
  std::vector<int32_t> rows_;                       // (path idx, line_number) pairs
  std::vector<float> emb_;                          // N x 256
  std::unordered_map<uint64_t, size_t> id_row_;
  // persistence bookkeeping (same policy as the Python store): rows [0, n_disk_) are on disk and
  // equal to memory except dirty_; rewrite_ forces a full rewrite (first flush, deletions)
  size_t n_disk_ = 0;
  std::set<size_t> dirty_;
  bool rewrite_ = true;
 public:
  unsigned full_rewrites = 0;
};

// search_with_workspace (search/mod.rs:146-216): diff `files` against the store, embed only
// New/Changed documents through `embed_lines` (lines -> N x 256 f32), upsert, filtered query.
using EmbedLinesFn = std::function<std::vector<float>(const std::vector<std::string> &)>;
std::vector<RankedLine> search_with_workspace(const std::vector<std::string> &files, const std::vector<float> &query_embedding,
                                              const EmbedLinesFn &embed_lines, const SearchConfig &cfg,
                                              const std::optional<std::string> &workspace_name,
                                              const std::function<void(const std::string &)> &log = nullptr, int device = 0,
                                              const std::string &model_fingerprint = "");
// print_workspace_search_results (cmds/search.rs:66-110) and the workspace JSON (:208-237)
std::string format_workspace_search_results(const std::vector<RankedLine> &ranked, size_t n_lines, bool is_tty);
std::string workspace_output_json(const std::vector<RankedLine> &ranked, size_t n_lines);

// minimal JSON value (enough for store.json / config.json)
struct Json {
  enum Type { Null, Bool, Num, Str, Arr, Obj } type = Null;
  bool b = false;
  double num = 0;
  std::string raw_num;                              // integer text kept exactly
  std::string str;
  std::vector<Json> arr;
  std::vector<std::pair<std::string, Json>> obj;
  const Json *get(const std::string &key) const;
  // the number as an unsigned integer; throws unless it is a non-negative whole number below 2^63
  // (a double -> integer conversion out of range is undefined behaviour)
  uint64_t as_u64(const char *what) const {
    if (type != Num || !(num >= 0.0 && num < 9.2e18) || num != (double)(uint64_t)num) throw std::runtime_error(std::string("json: ") + what + " is not a non-negative integer");
    return (uint64_t)num;
  }
  static Json parse(const std::string &text);       // throws std::runtime_error
};

}  // namespace semtools

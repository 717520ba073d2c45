#include "semtools_store.hpp"

#include <fcntl.h>
#include <sys/file.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <sstream>
#include <stdexcept>

namespace semtools {

// ------------------------------------------------------------------ tiny JSON ----------
namespace {
struct P {
  const std::string &s;
  size_t i = 0;
  void ws() { while (i < s.size() && (s[i] == ' ' || s[i] == '\n' || s[i] == '\t' || s[i] == '\r')) ++i; }
  [[noreturn]] void fail(const char *m) { throw std::runtime_error(std::string("json: ") + m); }
  Json value() {
    ws();
    if (i >= s.size()) fail("unexpected end");
    Json v;
    char c = s[i];
    if (c == '{') {
      v.type = Json::Obj; ++i; ws();
      if (s[i] == '}') { ++i; return v; }
      for (;;) {
        ws(); Json k = value(); if (k.type != Json::Str) fail("key");
        ws(); if (s[i++] != ':') fail("colon");
        v.obj.emplace_back(k.str, value());
        ws(); if (s[i] == ',') { ++i; continue; }
        if (s[i] == '}') { ++i; return v; }
        fail("object");
      }
    }
    if (c == '[') {
      v.type = Json::Arr; ++i; ws();
      if (s[i] == ']') { ++i; return v; }
      for (;;) {
        v.arr.push_back(value());
        ws(); if (s[i] == ',') { ++i; continue; }
        if (s[i] == ']') { ++i; return v; }
        fail("array");
      }
    }
    if (c == '"') {
      v.type = Json::Str; ++i;
      while (i < s.size() && s[i] != '"') {
        if (s[i] == '\\') {
          char e = s[++i];
          switch (e) {
            case 'n': v.str += '\n'; break; case 't': v.str += '\t'; break; case 'r': v.str += '\r'; break;
            case 'b': v.str += '\b'; break; case 'f': v.str += '\f'; break; case '/': v.str += '/'; break;
            case '\\': v.str += '\\'; break; case '"': v.str += '"'; break;
            case 'u': {
              unsigned cp = (unsigned)std::stoul(s.substr(i + 1, 4), nullptr, 16); i += 4;
              if (cp >= 0xD800 && cp < 0xDC00 && s.compare(i + 1, 2, "\\u") == 0) {   // surrogate pair
                unsigned lo = (unsigned)std::stoul(s.substr(i + 3, 4), nullptr, 16); i += 6;
                cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
              }
              if (cp < 0x80) v.str += (char)cp;
              else if (cp < 0x800) { v.str += (char)(0xC0 | (cp >> 6)); v.str += (char)(0x80 | (cp & 0x3F)); }
              else if (cp < 0x10000) { v.str += (char)(0xE0 | (cp >> 12)); v.str += (char)(0x80 | ((cp >> 6) & 0x3F)); v.str += (char)(0x80 | (cp & 0x3F)); }
              else { v.str += (char)(0xF0 | (cp >> 18)); v.str += (char)(0x80 | ((cp >> 12) & 0x3F)); v.str += (char)(0x80 | ((cp >> 6) & 0x3F)); v.str += (char)(0x80 | (cp & 0x3F)); }
              break;
            }
            default: fail("escape");
          }
          ++i;
        } else v.str += s[i++];
      }
      if (i >= s.size()) fail("string");
      ++i;
      return v;
    }
    if (s.compare(i, 4, "true") == 0) { v.type = Json::Bool; v.b = true; i += 4; return v; }
    if (s.compare(i, 5, "false") == 0) { v.type = Json::Bool; i += 5; return v; }
    if (s.compare(i, 4, "null") == 0) { i += 4; return v; }
    size_t j = i;
    while (j < s.size() && (std::isdigit((unsigned char)s[j]) || s[j] == '-' || s[j] == '+' || s[j] == '.' || s[j] == 'e' || s[j] == 'E')) ++j;
    if (j == i) fail("value");
    v.type = Json::Num; v.raw_num = s.substr(i, j - i); v.num = std::strtod(v.raw_num.c_str(), nullptr); i = j;
    return v;
  }
};
}  // namespace

const Json *Json::get(const std::string &key) const {
  for (const auto &kv : obj) if (kv.first == key) return &kv.second;
  return nullptr;
}
Json Json::parse(const std::string &text) { P p{text}; Json v = p.value(); return v; }

static std::string read_file(const std::string &p) {
  std::ifstream f(p, std::ios::binary);
  if (!f) throw std::runtime_error("cannot read " + p);
  std::stringstream ss; ss << f.rdbuf(); return ss.str();
}
static bool exists(const std::string &p) { struct stat st; return ::stat(p.c_str(), &st) == 0; }
static void mkdirs(const std::string &p) {
  std::string cur;
  for (size_t i = 0; i <= p.size(); ++i) {
    if (i == p.size() || p[i] == '/') { if (!cur.empty()) ::mkdir(cur.c_str(), 0755); }
    if (i < p.size()) cur += p[i];
  }
}
static std::string home() {
  const char *h = std::getenv("HOME");
  if (!h || !*h) throw std::runtime_error("No home dir found?");
  return h;
}

// ------------------------------------------------------------------ Workspace (mod.rs) --
std::string Workspace::root_path(const std::string &name) { return home() + "/.semtools/workspaces/" + name; }
std::string Workspace::config_path_for(const std::string &name) { return root_path(name) + "/config.json"; }
std::string Workspace::active(const std::optional<std::string> &workspace_name) {
  std::string a;
  if (workspace_name) a = *workspace_name;
  else if (const char *e = std::getenv("SEMTOOLS_WORKSPACE")) a = e;
  if (a.empty()) throw std::runtime_error("No active workspace. Run: workspace use <name>");
  return a;
}
Workspace Workspace::open(const std::optional<std::string> &workspace_name) {
  const std::string a = active(workspace_name);
  Workspace ws;
  try {
    Json j = Json::parse(read_file(config_path_for(a)));
    const Json *n = j.get("name"), *r = j.get("root_dir"), *b = j.get("in_batch_size"), *o = j.get("oversample_factor");
    if (!n || !r || !b || !o || n->type != Json::Str || r->type != Json::Str) throw std::runtime_error("cfg");
    ws.config.name = n->str; ws.config.root_dir = r->str;
    ws.config.in_batch_size = (size_t)b->as_u64("in_batch_size"); ws.config.oversample_factor = (size_t)o->as_u64("oversample_factor");
  } catch (const std::exception &) {
    ws.config = WorkspaceConfig();
  }
  if (ws.config.root_dir.empty()) ws.config.root_dir = root_path(a);
  if (ws.config.name.empty() || ws.config.name == "default") ws.config.name = a;
  return ws;
}
void Workspace::save() const {
  const std::string p = config_path_for(config.name);
  mkdirs(p.substr(0, p.rfind('/')));
  std::ofstream f(p);
  f << "{\n  \"name\": " << json_string(config.name) << ",\n  \"root_dir\": " << json_string(config.root_dir)
    << ",\n  \"in_batch_size\": " << config.in_batch_size << ",\n  \"oversample_factor\": " << config.oversample_factor << "\n}";
}

// ------------------------------------------------------------------ ids ------------------
uint64_t DocMeta::id() const { return stb_fnv1a64(reinterpret_cast<const uint8_t *>(path.data()), path.size()); }
uint64_t LineEmbedding::id() const { return stb_line_id(reinterpret_cast<const uint8_t *>(path.data()), path.size(), line_number); }

// ------------------------------------------------------------------ Store ----------------
namespace {
struct DirLock {                                   // flock(<dir>/.lock), released on scope exit
  int fd = -1;
  DirLock(const std::string &dir, bool exclusive) {
    fd = ::open((dir + "/.lock").c_str(), O_RDWR | O_CREAT, 0644);
    if (fd < 0 || ::flock(fd, exclusive ? LOCK_EX : LOCK_SH) != 0) { if (fd >= 0) ::close(fd); fd = -1; throw std::runtime_error("cannot lock workspace store " + dir); }
  }
  ~DirLock() { if (fd >= 0) { ::flock(fd, LOCK_UN); ::close(fd); } }
  DirLock(const DirLock &) = delete;
  DirLock &operator=(const DirLock &) = delete;
};
long long file_size(const std::string &p) { struct stat st; return ::stat(p.c_str(), &st) == 0 ? (long long)st.st_size : -1; }
}  // namespace

Store Store::open(const std::string &workspace_dir) {
  Store s;
  s.dir_ = workspace_dir + "/flat.b200";
  mkdirs(s.dir_);
  DirLock lk(s.dir_, false);
  s.load();
  return s;
}

uint64_t Store::disk_gen() const {
  if (!exists(dir_ + "/GEN")) return 0;
  return std::strtoull(read_file(dir_ + "/GEN").c_str(), nullptr, 10);
}

void Store::load() {
  paths_.clear(); path_idx_.clear(); docs_.clear(); rows_.clear(); emb_.clear(); id_row_.clear(); dirty_.clear();
  gen_ = 0; rows_file_ = "rows.i32"; emb_file_ = "line_embeddings.f32"; stored_model_.clear();
  n_disk_ = 0; rewrite_ = true;
  const std::string meta = dir_ + "/store.json";
  if (!exists(meta)) return;
  Json j = Json::parse(read_file(meta));
  const Json *fmt = j.get("format");
  if (!fmt || fmt->str != "semtools_b200.flat.v1") throw std::runtime_error("unknown store format");
  // a damaged commit record is an error message, never undefined behaviour: every field is checked
  auto corrupt = [&](const char *what) { return std::runtime_error("workspace store " + dir_ + ": store.json is corrupt (" + what + "); delete the directory to rebuild it"); };
  auto field = [&](const Json &o, const char *key, Json::Type t) -> const Json & {
    const Json *v = o.type == Json::Obj ? o.get(key) : nullptr;
    if (!v || v->type != t) throw corrupt(key);
    return *v;
  };
  for (const auto &p : field(j, "paths", Json::Arr).arr) {
    if (p.type != Json::Str) throw corrupt("paths");
    path_idx_[p.str] = (int32_t)paths_.size(); paths_.push_back(p.str);
  }
  for (const auto &d : field(j, "docs", Json::Arr).arr) {
    DocMeta m;
    m.path = field(d, "path", Json::Str).str;
    m.size_bytes = std::strtoull(field(d, "size_bytes", Json::Num).raw_num.c_str(), nullptr, 10);
    m.mtime = std::strtoll(field(d, "mtime", Json::Num).raw_num.c_str(), nullptr, 10);
    m.version = (uint32_t)field(d, "_version", Json::Num).as_u64("_version");
    docs_.push_back(m);
  }
  if (const Json *g = j.get("gen")) { if (g->type != Json::Num) throw corrupt("gen"); gen_ = std::strtoull(g->raw_num.c_str(), nullptr, 10); }
  if (const Json *f = j.get("files"); f && f->type == Json::Obj) {
    auto file_name = [&](const char *key, std::string &dst) {
      if (const Json *v = f->get(key)) {
        if (v->type != Json::Str || v->str.empty() || v->str.find('/') != std::string::npos || v->str[0] == '.') throw corrupt("files");
        dst = v->str;
      }
    };
    file_name("rows", rows_file_);
    file_name("emb", emb_file_);
  }
  if (const Json *m = j.get("model"); m && m->type == Json::Str) stored_model_ = m->str;
  const std::string rows_p = dir_ + "/" + rows_file_, emb_p = dir_ + "/" + emb_file_;
  const long long rs = file_size(rows_p), es = file_size(emb_p);
  const size_t n_rows_file = rs > 0 ? (size_t)rs / 8 : 0, n_emb_file = es > 0 ? (size_t)es / (LINE_EMBEDDING_SIZE * 4) : 0;
  size_t n = std::min(n_rows_file, n_emb_file);
  if (const Json *r = j.get("rows")) { if (r->type != Json::Num) throw corrupt("rows"); n = (size_t)std::strtoull(r->raw_num.c_str(), nullptr, 10); }
  if (n_rows_file < n || n_emb_file < n)
    throw std::runtime_error("workspace store " + dir_ + " is truncated: store.json commits " + std::to_string(n) + " rows, the row files hold " +
                             std::to_string(n_rows_file) + " / " + std::to_string(n_emb_file) + "; delete the directory to rebuild it");
  rows_.resize(2 * n); emb_.resize(n * LINE_EMBEDDING_SIZE);
  if (n) {
    std::ifstream fr(rows_p, std::ios::binary), fe(emb_p, std::ios::binary);
    fr.read(reinterpret_cast<char *>(rows_.data()), (std::streamsize)(rows_.size() * 4));
    fe.read(reinterpret_cast<char *>(emb_.data()), (std::streamsize)(emb_.size() * 4));
    if (!fr || !fe) throw std::runtime_error("workspace store " + dir_ + ": short read");
  }
  for (size_t r = 0; r < n; ++r) {
    const int32_t pi = rows_[2 * r];
    if (pi < 0 || (size_t)pi >= paths_.size())
      throw std::runtime_error("workspace store " + dir_ + " is corrupt: a row refers to path index " + std::to_string(pi) + " but the path table has " +
                               std::to_string(paths_.size()) + " entries; delete the directory to rebuild it");
    LineEmbedding le{paths_[pi], rows_[2 * r + 1], {}};
    id_row_[le.id()] = r;
  }
  n_disk_ = n;
  rewrite_ = false;
}

template <class F>
void Store::mutate(F &&apply) {
  DirLock lk(dir_, true);
  if (disk_gen() != gen_) load();                  // another process committed since this handle loaded
  apply();
  flush();
}

void Store::flush() {                              // caller holds the exclusive lock
  const uint64_t gen = gen_ + 1;
  std::string rows_file = rows_file_, emb_file = emb_file_;
  std::string rows_p = dir_ + "/" + rows_file, emb_p = dir_ + "/" + emb_file;
  const size_t n = rows_.size() / 2;
  std::string old_rows, old_emb;
  const bool have = exists(rows_p) && exists(emb_p);
  const bool damaged = have && (file_size(rows_p) < (long long)(n_disk_ * 8) || file_size(emb_p) < (long long)(n_disk_ * LINE_EMBEDDING_SIZE * 4));
  if (rewrite_ || !have || damaged) {
    if (exists(rows_p) || exists(emb_p)) {         // never overwrite a committed generation in place
      old_rows = rows_p; old_emb = emb_p;
      rows_file = "rows." + std::to_string(gen) + ".i32"; emb_file = "line_embeddings." + std::to_string(gen) + ".f32";
      rows_p = dir_ + "/" + rows_file; emb_p = dir_ + "/" + emb_file;
    }
    { std::ofstream f(rows_p, std::ios::binary); f.write(reinterpret_cast<const char *>(rows_.data()), (std::streamsize)(rows_.size() * 4)); }
    { std::ofstream f(emb_p, std::ios::binary); f.write(reinterpret_cast<const char *>(emb_.data()), (std::streamsize)(emb_.size() * 4)); }
    ++full_rewrites;
  } else {
    // anything beyond the committed rows is the debris of an interrupted flush
    if (::truncate(rows_p.c_str(), (off_t)(n_disk_ * 8)) != 0 || ::truncate(emb_p.c_str(), (off_t)(n_disk_ * LINE_EMBEDDING_SIZE * 4)) != 0)
      throw std::runtime_error("workspace store " + dir_ + ": cannot truncate the row files");
    std::fstream fr(rows_p, std::ios::in | std::ios::out | std::ios::binary), fe(emb_p, std::ios::in | std::ios::out | std::ios::binary);
    for (size_t r : dirty_) {
      if (r >= n_disk_) continue;
      fr.seekp((std::streamoff)(r * 8)); fr.write(reinterpret_cast<const char *>(rows_.data() + 2 * r), 8);
      fe.seekp((std::streamoff)(r * LINE_EMBEDDING_SIZE * 4));
      fe.write(reinterpret_cast<const char *>(emb_.data() + r * LINE_EMBEDDING_SIZE), LINE_EMBEDDING_SIZE * 4);
    }
    if (n > n_disk_) {
      fr.seekp(0, std::ios::end); fr.write(reinterpret_cast<const char *>(rows_.data() + 2 * n_disk_), (std::streamsize)((n - n_disk_) * 8));
      fe.seekp(0, std::ios::end);
      fe.write(reinterpret_cast<const char *>(emb_.data() + n_disk_ * LINE_EMBEDDING_SIZE), (std::streamsize)((n - n_disk_) * LINE_EMBEDDING_SIZE * 4));
    }
  }
  const std::string tmp = dir_ + "/store.json.tmp";
  {
    const std::string &model = model_fingerprint.empty() ? stored_model_ : model_fingerprint;
    std::ofstream f(tmp);
    f << "{\"format\": \"semtools_b200.flat.v1\", \"dim\": 256, \"rows\": " << n << ", \"gen\": " << gen
      << ", \"files\": {\"rows\": " << json_string(rows_file) << ", \"emb\": " << json_string(emb_file) << "}, \"model\": ";
    if (model.empty()) f << "null"; else f << json_string(model);
    f << ", \"paths\": [";
    for (size_t i = 0; i < paths_.size(); ++i) f << (i ? ", " : "") << json_string(paths_[i]);
    f << "], \"docs\": [";
    for (size_t i = 0; i < docs_.size(); ++i)
      f << (i ? ", " : "") << "{\"path\": " << json_string(docs_[i].path) << ", \"size_bytes\": " << docs_[i].size_bytes
        << ", \"mtime\": " << docs_[i].mtime << ", \"_version\": " << docs_[i].version << "}";
    f << "]}";
  }
  std::rename(tmp.c_str(), (dir_ + "/store.json").c_str());        // the commit
  { std::ofstream f(dir_ + "/GEN.tmp"); f << gen; }
  std::rename((dir_ + "/GEN.tmp").c_str(), (dir_ + "/GEN").c_str());
  if (!old_rows.empty()) { ::unlink(old_rows.c_str()); ::unlink(old_emb.c_str()); }
  gen_ = gen; rows_file_ = rows_file; emb_file_ = emb_file;
  if (!model_fingerprint.empty()) stored_model_ = model_fingerprint;
  n_disk_ = n; rewrite_ = false; dirty_.clear();
}

std::map<std::string, DocMeta> Store::get_existing_docs(const std::vector<std::string> &paths) const {
  std::map<std::string, DocMeta> out;
  for (const auto &p : paths)
    for (const auto &d : docs_) if (d.path == p) { out[p] = d; break; }
  return out;
}

std::vector<DocumentState> Store::analyze_document_states(const std::vector<std::string> &paths) const {
  auto existing = get_existing_docs(paths);
  std::vector<DocumentState> states;
  for (const auto &fp : paths) {
    struct stat st;
    if (::stat(fp.c_str(), &st) != 0) continue;                     // :578-581 missing file: skipped
    DocMeta cur{fp, (uint64_t)st.st_size, (int64_t)st.st_mtime, CURRENT_EMBEDDING_VERSION};
    DocumentState ds;
    ds.filename = fp; ds.meta = cur;
    auto it = existing.find(fp);
    // a store written by another embedder (both fingerprints known): everything is re-embedded
    const bool foreign = !model_fingerprint.empty() && !stored_model_.empty() && model_fingerprint != stored_model_;
    if (it != existing.end() && it->second.size_bytes == cur.size_bytes && it->second.mtime == cur.mtime &&
        it->second.version == CURRENT_EMBEDDING_VERSION && !foreign) {
      ds.kind = DocumentState::Unchanged;
    } else {
      ds.kind = it != existing.end() ? DocumentState::Changed : DocumentState::New;
      ds.content = read_file(fp);
    }
    states.push_back(std::move(ds));
  }
  return states;
}

void Store::upsert_document_metadata(const std::vector<DocMeta> &metas) {
  if (metas.empty()) return;
  mutate([&] {
    for (const auto &m : metas) {
      auto it = std::find_if(docs_.begin(), docs_.end(), [&](const DocMeta &d) { return d.path == m.path; });
      if (it != docs_.end()) *it = m; else docs_.push_back(m);
    }
  });
}

void Store::upsert_line_embeddings(const std::vector<LineEmbedding> &lines) {
  if (lines.empty()) return;
  mutate([&] {
  for (const auto &le : lines) {
    if (le.embedding.size() != LINE_EMBEDDING_SIZE) throw std::runtime_error("embedding must have 256 floats");
    int32_t pi;
    auto pit = path_idx_.find(le.path);
    if (pit == path_idx_.end()) { pi = (int32_t)paths_.size(); paths_.push_back(le.path); path_idx_[le.path] = pi; }
    else pi = pit->second;
    const uint64_t rid = le.id();
    auto rit = id_row_.find(rid);
    size_t row;
    if (rit != id_row_.end()) { row = rit->second; dirty_.insert(row); }   // upsert replaces by id
    else { row = rows_.size() / 2; id_row_[rid] = row; rows_.resize(rows_.size() + 2); emb_.resize(emb_.size() + LINE_EMBEDDING_SIZE); }
    rows_[2 * row] = pi; rows_[2 * row + 1] = le.line_number;
    std::memcpy(emb_.data() + row * LINE_EMBEDDING_SIZE, le.embedding.data(), LINE_EMBEDDING_SIZE * 4);
  }
  });
}

void Store::delete_document_metadata(const std::vector<std::string> &paths) {
  if (paths.empty()) return;
  mutate([&] {
    for (const auto &p : paths)
      docs_.erase(std::remove_if(docs_.begin(), docs_.end(), [&](const DocMeta &d) { return d.path == p && d.version == CURRENT_EMBEDDING_VERSION; }), docs_.end());
  });
}

void Store::delete_line_embeddings(const std::vector<std::string> &paths) {
  if (paths.empty()) return;
  mutate([&] {
  std::vector<char> kill(paths_.size(), 0);
  for (const auto &p : paths) { auto it = path_idx_.find(p); if (it != path_idx_.end()) kill[it->second] = 1; }
  size_t w = 0;
  const size_t n = rows_.size() / 2;
  for (size_t r = 0; r < n; ++r) {
    if (kill[rows_[2 * r]]) continue;
    if (w != r) {
      rows_[2 * w] = rows_[2 * r]; rows_[2 * w + 1] = rows_[2 * r + 1];
      std::memmove(emb_.data() + w * LINE_EMBEDDING_SIZE, emb_.data() + r * LINE_EMBEDDING_SIZE, LINE_EMBEDDING_SIZE * 4);
    }
    ++w;
  }
  rows_.resize(2 * w); emb_.resize(w * LINE_EMBEDDING_SIZE);
  if (w != n) rewrite_ = true;                                      // rows moved: the files are rewritten
  id_row_.clear();
  for (size_t r = 0; r < w; ++r) { LineEmbedding le{paths_[rows_[2 * r]], rows_[2 * r + 1], {}}; id_row_[le.id()] = r; }
  });
}

void Store::delete_documents(const std::vector<std::string> &paths) {
  if (paths.empty()) return;
  delete_document_metadata(paths);
  delete_line_embeddings(paths);
}

std::vector<std::string> Store::get_all_document_paths() const {
  std::vector<std::string> out;
  for (const auto &d : docs_) out.push_back(d.path);
  return out;
}

std::vector<uint64_t> Store::ranges_for(const std::vector<std::string> &subset_paths) const {
  std::vector<char> sel(paths_.size(), 0);
  for (const auto &p : subset_paths) { auto it = path_idx_.find(p); if (it != path_idx_.end()) sel[it->second] = 1; }
  std::vector<uint64_t> ranges;
  const size_t n = rows_.size() / 2;
  size_t r = 0;
  while (r < n) {
    if (!sel[rows_[2 * r]]) { ++r; continue; }
    size_t e = r;
    while (e < n && sel[rows_[2 * e]]) ++e;
    ranges.push_back(r); ranges.push_back(e);
    r = e;
  }
  return ranges;
}

int upload_mirror(stb_ctx *ctx, const float *rows, uint64_t n, stb_corpus **out, CorpusCreateFn create) {
  *out = nullptr;
  stb_corpus *c = nullptr;
  int rc = create(ctx, STB_DIM, n, 0, &c);
  if (rc == STB_OK) rc = stb_corpus_append(c, rows, n);
  if (rc == STB_OK) { *out = c; return STB_OK; }
  stb_corpus_destroy(c);
  if (rc != STB_ERR_NOMEM) return rc;
  c = nullptr;
  rc = stb_corpus_create_host(ctx, STB_DIM, n, 0, &c);
  if (rc == STB_OK) rc = stb_corpus_append(c, rows, n);
  if (rc == STB_OK) *out = c;
  else stb_corpus_destroy(c);
  return rc;
}

std::vector<RankedLine> Store::search_line_embeddings(const std::vector<float> &query, const std::vector<std::string> &subset_paths,
                                                      size_t top_k, std::optional<float> max_distance, int device) {
  std::vector<RankedLine> out;
  if (subset_paths.empty() || top_k == 0) return out;               // :489-491
  auto ranges = ranges_for(subset_paths);
  if (ranges.empty() || query.size() != LINE_EMBEDDING_SIZE) return out;
  stb_ctx *ctx = nullptr; stb_corpus *corpus = nullptr;
  auto chk = [&](int rc) { if (rc < 0) { std::string m = stb_last_error(); stb_corpus_destroy(corpus); stb_ctx_destroy(ctx); throw StbError(rc, m); } };
  chk(stb_ctx_create(device, nullptr, &ctx));
  chk(upload_mirror(ctx, emb_.data(), rows_.size() / 2, &corpus));
  std::vector<stb_hit> hits(top_k);
  uint64_t n = 0;
  chk(stb_search(ctx, corpus, query.data(), (uint32_t)top_k, max_distance ? 1 : 0, max_distance ? (double)*max_distance : 0.0,
                 STB_MODE_STORE_QUERY, ranges.data(), (uint32_t)(ranges.size() / 2), hits.data(), top_k, &n));
  for (uint64_t i = 0; i < n; ++i)
    out.push_back({paths_[rows_[2 * hits[i].row]], rows_[2 * hits[i].row + 1], (float)hits[i].distance});   // :531 f32
  stb_corpus_destroy(corpus);
  stb_ctx_destroy(ctx);
  return out;
}

// ------------------------------------------------------------------ search_with_workspace --
std::vector<RankedLine> search_with_workspace(const std::vector<std::string> &files, const std::vector<float> &query_embedding,
                                              const EmbedLinesFn &embed_lines, const SearchConfig &cfg,
                                              const std::optional<std::string> &workspace_name,
                                              const std::function<void(const std::string &)> &log, int device,
                                              const std::string &model_fingerprint) {
  Workspace ws = Workspace::open(workspace_name);
  Store store = Store::open(ws.config.root_dir);
  store.model_fingerprint = model_fingerprint;
  std::vector<LineEmbedding> to_upsert;
  std::vector<DocMeta> docs;
  for (auto &st : store.analyze_document_states(files)) {
    if (st.kind == DocumentState::Unchanged) continue;
    const std::vector<std::string> lines = rust_lines(st.content);
    if (lines.empty()) continue;                                   // create_document_from_content -> None
    const std::vector<float> emb = embed_lines(lines);
    if (emb.size() != lines.size() * LINE_EMBEDDING_SIZE) throw std::runtime_error("embed_lines returned the wrong size");
    for (size_t i = 0; i < lines.size(); ++i)
      to_upsert.push_back({st.filename, (int32_t)i,                 // 0-based line numbers (mod.rs:178)
                           std::vector<float>(emb.begin() + i * LINE_EMBEDDING_SIZE, emb.begin() + (i + 1) * LINE_EMBEDDING_SIZE)});
    docs.push_back(st.meta);
  }
  if (!to_upsert.empty()) {
    if (log) log("Updating workspace with " + std::to_string(to_upsert.size()) + " lines from new/changed docs...");
    store.upsert_line_embeddings(to_upsert);
  }
  if (!docs.empty()) {
    if (log) log("Updating workspace with " + std::to_string(docs.size()) + " new/changed documents...");
    store.upsert_document_metadata(docs);
  }
  std::optional<float> max_d;
  if (cfg.max_distance) max_d = (float)*cfg.max_distance;           // mod.rs:211 `as f32`
  return store.search_line_embeddings(query_embedding, files, cfg.top_k, max_d, device);
}

static bool read_lines(const std::string &path, std::vector<std::string> &lines) {
  std::ifstream f(path, std::ios::binary);
  if (!f) return false;
  std::stringstream ss; ss << f.rdbuf();
  lines = rust_lines(ss.str());
  return true;
}

std::string format_workspace_search_results(const std::vector<RankedLine> &ranked, size_t n_lines, bool is_tty) {
  std::string out;
  char num[32];
  for (const auto &rl : ranked) {
    const size_t m = (size_t)rl.line_number;
    const size_t start = m > n_lines ? m - n_lines : 0;
    const size_t end = m + n_lines + 1;                             // NOT clamped in the header (:77-79)
    out += rl.path + ":" + std::to_string(start) + "::" + std::to_string(end) + " (" + rust_display_f32(rl.distance) + ")\n";
    std::vector<std::string> lines;
    if (read_lines(rl.path, lines)) {
      const size_t actual_end = std::min(end, lines.size());
      if (start > actual_end) throw std::runtime_error("slice index starts past the end (the reference panics here)");
      for (size_t n = start; n < actual_end; ++n) {
        snprintf(num, sizeof(num), "%4zu", n + 1);
        if (n == m && is_tty) out += std::string("\x1b[43m\x1b[30m") + num + ": " + lines[n] + "\x1b[0m\n";
        else out += std::string(num) + ": " + lines[n] + "\n";
      }
    } else {
      out += "    [Error: Could not read file content]\n";
    }
    out += "\n";
  }
  return out;
}

std::string workspace_output_json(const std::vector<RankedLine> &ranked, size_t n_lines) {
  if (ranked.empty()) return "{\n  \"results\": []\n}";
  std::string o = "{\n  \"results\": [\n";
  for (size_t i = 0; i < ranked.size(); ++i) {
    const auto &rl = ranked[i];
    const size_t m = (size_t)rl.line_number;
    const size_t start = m > n_lines ? m - n_lines : 0, end = m + n_lines + 1;
    std::string content;
    std::vector<std::string> lines;
    if (read_lines(rl.path, lines)) {
      for (size_t n = start; n < std::min(end, lines.size()); ++n) { if (n > start) content += "\n"; content += lines[n]; }
    } else {
      content = "[Error: Could not read file content]";
    }
    o += "    {\n";
    o += "      \"filename\": " + json_string(rl.path) + ",\n";
    o += "      \"start_line_number\": " + std::to_string(start) + ",\n";
    o += "      \"end_line_number\": " + std::to_string(end) + ",\n";
    o += "      \"match_line_number\": " + std::to_string(m) + ",\n";
    o += "      \"distance\": " + json_f64((double)rl.distance) + ",\n";   // f32 widened to f64 (:233)
    o += "      \"content\": " + json_string(content) + "\n";
    o += i + 1 < ranked.size() ? "    },\n" : "    }\n";
  }
  o += "  ]\n}";
  return o;
}

}  // namespace semtools

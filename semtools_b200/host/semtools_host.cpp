#include "semtools_host.hpp"
#include "semtools_store.hpp"   // Json

#include <cstring>
#include <fstream>
#include <iterator>

#include <algorithm>
#include <charconv>
#include <cmath>
#include <cstdio>
#include <fstream>
#include <sstream>
#include <thread>

namespace semtools {

static void check(int rc) {
  if (rc < 0) throw StbError(rc, stb_last_error());
}

std::vector<std::string> rust_lines(const std::string &content) {
  std::vector<std::string> out;
  if (content.empty()) return out;
  size_t pos = 0;
  while (pos <= content.size()) {
    size_t nl = content.find('\n', pos);
    if (nl == std::string::npos) {
      if (pos < content.size()) out.emplace_back(content.substr(pos));   // unterminated last line: kept verbatim (a trailing '\r' stays)
      break;
    }
    size_t end = nl;
    if (end > pos && content[end - 1] == '\r') --end;                    // "\r\n" is one terminator
    out.emplace_back(content.substr(pos, end - pos));
    pos = nl + 1;
  }
  return out;
}

std::string to_lowercase_ascii(const std::string &s) {
  std::string r = s;
  for (auto &c : r)
    if (c >= 'A' && c <= 'Z') c = (char)(c - 'A' + 'a');
  return r;
}

// ---- str::to_lowercase (full Unicode mapping + Final_Sigma), mod.rs:63-67 ------------------
namespace {
#include "unicode_lower.inc"

bool in_ranges(const CpRange *r, size_t n, uint32_t cp) {
  size_t lo = 0, hi = n;
  while (lo < hi) {
    const size_t mid = (lo + hi) / 2;
    if (cp > r[mid].hi) lo = mid + 1;
    else if (cp < r[mid].lo) hi = mid;
    else return true;
  }
  return false;
}
bool case_ignorable(uint32_t cp) { return in_ranges(kCaseIgnorable, sizeof(kCaseIgnorable) / sizeof(CpRange), cp); }
bool cased_not_ignorable(uint32_t cp) { return in_ranges(kCasedNotIgn, sizeof(kCasedNotIgn) / sizeof(CpRange), cp); }

// decodes one scalar value; a malformed byte is returned as 0x110000 + byte (passes through)
uint32_t decode(const std::string &s, size_t &i) {
  const unsigned char b0 = (unsigned char)s[i];
  auto cont = [&](size_t k) { return i + k < s.size() && ((unsigned char)s[i + k] & 0xC0) == 0x80; };
  if (b0 < 0x80) { i += 1; return b0; }
  if (b0 >= 0xC2 && b0 <= 0xDF && cont(1)) { uint32_t c = ((b0 & 0x1Fu) << 6) | ((unsigned char)s[i + 1] & 0x3Fu); i += 2; return c; }
  if (b0 >= 0xE0 && b0 <= 0xEF && cont(1) && cont(2)) {
    uint32_t c = ((b0 & 0x0Fu) << 12) | (((unsigned char)s[i + 1] & 0x3Fu) << 6) | ((unsigned char)s[i + 2] & 0x3Fu);
    if (c >= 0x800 && !(c >= 0xD800 && c <= 0xDFFF)) { i += 3; return c; }
  }
  if (b0 >= 0xF0 && b0 <= 0xF4 && cont(1) && cont(2) && cont(3)) {
    uint32_t c = ((b0 & 0x07u) << 18) | (((unsigned char)s[i + 1] & 0x3Fu) << 12) | (((unsigned char)s[i + 2] & 0x3Fu) << 6) |
                 ((unsigned char)s[i + 3] & 0x3Fu);
    if (c >= 0x10000 && c <= 0x10FFFF) { i += 4; return c; }
  }
  i += 1;
  return 0x110000u + b0;
}
void encode(uint32_t c, std::string &out) {
  if (c >= 0x110000u) { out += (char)(c - 0x110000u); return; }      // malformed byte, unchanged
  if (c < 0x80) out += (char)c;
  else if (c < 0x800) { out += (char)(0xC0 | (c >> 6)); out += (char)(0x80 | (c & 0x3F)); }
  else if (c < 0x10000) { out += (char)(0xE0 | (c >> 12)); out += (char)(0x80 | ((c >> 6) & 0x3F)); out += (char)(0x80 | (c & 0x3F)); }
  else { out += (char)(0xF0 | (c >> 18)); out += (char)(0x80 | ((c >> 12) & 0x3F)); out += (char)(0x80 | ((c >> 6) & 0x3F)); out += (char)(0x80 | (c & 0x3F)); }
}
}  // namespace

static std::string to_lowercase_impl(const std::string &s, bool final_sigma);
std::string to_lowercase(const std::string &s) { return to_lowercase_impl(s, true); }
// char::to_lowercase applied per character (what the tokenizers Lowercase normalizer does): the same
// mapping WITHOUT the context-sensitive Final_Sigma rule of str::to_lowercase
std::string to_lowercase_per_char(const std::string &s) { return to_lowercase_impl(s, false); }

const std::vector<LowerEntry> &lower_table() {
  static const std::vector<LowerEntry> t = [] {
    std::vector<LowerEntry> v;
    for (const LowerMap &m : kLower) v.push_back({m.cp, m.n, {m.to[0], m.to[1], m.to[2]}});
    return v;
  }();
  return t;
}

static std::string to_lowercase_impl(const std::string &s, bool final_sigma) {
  std::vector<uint32_t> cps;
  cps.reserve(s.size());
  for (size_t i = 0; i < s.size();) cps.push_back(decode(s, i));
  std::string out;
  out.reserve(s.size());
  const size_t n_map = sizeof(kLower) / sizeof(LowerMap);
  for (size_t i = 0; i < cps.size(); ++i) {
    const uint32_t c = cps[i];
    if (c < 0x80) { out += (char)((c >= 'A' && c <= 'Z') ? c + 32 : c); continue; }
    if (c == 0x3A3 && !final_sigma) { encode(0x3C3, out); continue; }   // char::to_lowercase: always the medial form
    if (c == 0x3A3) {
      // Final_Sigma: preceded by a cased letter (skipping case-ignorables) and not followed by one
      size_t j = i;
      bool before = false;
      while (j > 0) { --j; if (!case_ignorable(cps[j])) { before = cased_not_ignorable(cps[j]); break; } }
      bool after = false;
      for (size_t k = i + 1; k < cps.size(); ++k) if (!case_ignorable(cps[k])) { after = cased_not_ignorable(cps[k]); break; }
      encode(before && !after ? 0x3C2 : 0x3C3, out);
      continue;
    }
    size_t lo = 0, hi = n_map;
    while (lo < hi) { const size_t mid = (lo + hi) / 2; if (kLower[mid].cp < c) lo = mid + 1; else hi = mid; }
    if (lo < n_map && kLower[lo].cp == c) for (int t = 0; t < kLower[lo].n; ++t) encode(kLower[lo].to[t], out);
    else encode(c, out);
  }
  return out;
}

// shortest round-trip decimal digits and exponent: value = 0.d1d2... x 10^exp10
template <class F>
static void shortest_digits(F x, std::string &digits, int &exp10) {
  char buf[64];
  auto r = std::to_chars(buf, buf + sizeof(buf), x, std::chars_format::scientific);
  std::string s(buf, r.ptr);                       // d.ddddde[+-]XX
  size_t e = s.find('e');
  std::string mant = s.substr(0, e);
  int ex = std::stoi(s.substr(e + 1));
  digits.clear();
  for (char c : mant)
    if (c >= '0' && c <= '9') digits.push_back(c);
  while (digits.size() > 1 && digits.back() == '0') digits.pop_back();
  exp10 = ex + 1;                                  // digits as 0.DDDD x 10^exp10
}

template <class F>
static std::string positional(F x, bool keep_point_zero) {
  if (x == 0) return keep_point_zero ? (std::signbit(x) ? "-0.0" : "0.0") : (std::signbit(x) ? "-0" : "0");
  std::string d;
  int e;
  shortest_digits(std::fabs(x), d, e);
  std::string s;
  if (e <= 0) s = "0." + std::string((size_t)(-e), '0') + d;
  else if ((size_t)e >= d.size()) { s = d + std::string((size_t)e - d.size(), '0'); if (keep_point_zero) s += ".0"; }
  else s = d.substr(0, (size_t)e) + "." + d.substr((size_t)e);
  return (x < 0 ? "-" : "") + s;
}

std::string rust_display_f64(double x) {
  if (std::isnan(x)) return "NaN";
  if (std::isinf(x)) return x > 0 ? "inf" : "-inf";
  return positional(x, false);
}

std::string rust_display_f32(float x) {
  if (std::isnan(x)) return "NaN";
  if (std::isinf(x)) return x > 0 ? "inf" : "-inf";
  return positional(x, false);
}

std::string json_f64(double x) {
  if (std::isnan(x) || std::isinf(x)) return "null";
  const double a = std::fabs(x);
  if (x == 0.0 || (a >= 1e-5 && a < 1e16)) return positional(x, true);   // ryu: positional while -5 < kk <= 16
  std::string d;
  int e;
  shortest_digits(a, d, e);
  std::string m = d.substr(0, 1);
  if (d.size() > 1) m += "." + d.substr(1);
  return (x < 0 ? "-" : "") + m + "e" + std::to_string(e - 1);
}

std::string json_string(const std::string &s) {
  std::string o = "\"";
  for (unsigned char c : s) {
    switch (c) {
      case '"': o += "\\\""; break;
      case '\\': o += "\\\\"; break;
      case '\n': o += "\\n"; break;
      case '\r': o += "\\r"; break;
      case '\t': o += "\\t"; break;
      case 8: o += "\\b"; break;
      case 12: o += "\\f"; break;
      default:
        if (c < 0x20) { char b[8]; snprintf(b, sizeof(b), "\\u%04x", c); o += b; }
        else o.push_back((char)c);
    }
  }
  return o + "\"";
}

WordLevelTokenizer::WordLevelTokenizer(const std::string &vocab_path) {
  std::ifstream f(vocab_path);
  if (!f) throw std::runtime_error("cannot open vocabulary " + vocab_path);
  std::string tok;
  uint32_t id = 0;
  while (std::getline(f, tok)) vocab.emplace_back(tok, id++);
  build_index();
}

WordLevelTokenizer::WordLevelTokenizer(std::vector<std::string> tokens) {
  uint32_t id = 0;
  for (auto &t : tokens) vocab.emplace_back(std::move(t), id++);
  build_index();
}

void WordLevelTokenizer::build_index() {
  std::sort(vocab.begin(), vocab.end());
  index_.reserve(vocab.size() * 2);
  for (const auto &kv : vocab) index_.emplace(std::string_view(kv.first), kv.second);   // first id wins on duplicates
}

std::vector<uint32_t> WordLevelTokenizer::encode(const std::string &text) const {
  std::vector<uint32_t> ids;
  auto is_space = [](unsigned char c) { return c == ' ' || (c >= '\t' && c <= '\r'); };   // isspace, "C" locale
  const size_t n = text.size();
  size_t i = 0;
  while (i < n) {
    while (i < n && is_space((unsigned char)text[i])) ++i;
    size_t j = i;
    while (j < n && !is_space((unsigned char)text[j])) ++j;
    if (j > i) {
      auto it = index_.find(std::string_view(text.data() + i, j - i));
      if (it != index_.end()) ids.push_back(it->second);       // unknown words: dropped (unk removal)
    }
    i = j;
  }
  return ids;
}

std::string_view truncate_chars(std::string_view line, size_t max_chars) {
  if (!max_chars || line.size() <= max_chars) return line;        // bytes >= chars: only then can it be too long
  size_t pos = 0, chars = 0;
  while (pos < line.size() && chars < max_chars) {
    const unsigned char c = (unsigned char)line[pos];
    pos += c < 0x80 ? 1 : (c >> 5) == 6 ? 2 : (c >> 4) == 14 ? 3 : (c >> 3) == 30 ? 4 : 1;
    ++chars;
  }
  return line.substr(0, std::min(pos, line.size()));
}

void tokenize_to_csr(const std::vector<std::string> &lines, const Tokenizer &tok, size_t max_len,
                     std::vector<uint64_t> &offsets, std::vector<uint32_t> &ids, unsigned threads) {
  const size_t n = lines.size();
  if (threads == 0) threads = std::max(1u, std::thread::hardware_concurrency());
  threads = (unsigned)std::min<size_t>(threads, std::max<size_t>(1, n / 256));     // no thread for < 256 lines
  offsets.assign(n + 1, 0);
  std::vector<std::vector<uint32_t>> part(threads);
  auto work = [&](unsigned t) {
    const size_t lo = n * t / threads, hi = n * (t + 1) / threads;
    auto &out = part[t];
    const size_t max_chars = tok.median_token_length() ? max_len * tok.median_token_length() : 0;
    for (size_t i = lo; i < hi; ++i) {
      auto v = tok.encode(std::string(truncate_chars(lines[i], max_chars)));
      if (v.size() > max_len) v.resize(max_len);               // truncate(max_length)
      offsets[i + 1] = v.size();                               // per-line count; prefix-summed below
      out.insert(out.end(), v.begin(), v.end());
    }
  };
  if (threads == 1) work(0);
  else {
    std::vector<std::thread> pool;
    for (unsigned t = 0; t < threads; ++t) pool.emplace_back(work, t);
    for (auto &th : pool) th.join();
  }
  for (size_t i = 0; i < n; ++i) offsets[i + 1] += offsets[i];
  ids.clear();
  ids.reserve(offsets[n]);
  for (auto &p : part) ids.insert(ids.end(), p.begin(), p.end());
}

Searcher::Searcher(int device) {
  check(stb_ctx_create(device, nullptr, &ctx_));
  check(stb_corpus_create(ctx_, STB_DIM, 1024, 0, &corpus_));
}

Searcher::~Searcher() {
  stb_tokenizer_destroy(text_tok_);
  stb_corpus_destroy(corpus_);
  stb_table_destroy(table_);
  stb_ctx_destroy(ctx_);
}

void Searcher::load_table(const float *E, uint64_t V, bool normalize, const float *weights, uint64_t n_weights,
                          const uint32_t *mapping, uint64_t n_mapping) {
  if (table_) { stb_table_destroy(table_); table_ = nullptr; }
  check(stb_table_load(ctx_, E, V, STB_DIM, n_weights ? weights : nullptr, n_weights, n_mapping ? mapping : nullptr, n_mapping,
                       normalize ? 1 : 0, &table_));
}

bool Searcher::load_text_tokenizer(const std::string &json, uint32_t flags) {
  if (text_tok_) { stb_tokenizer_destroy(text_tok_); text_tok_ = nullptr; }
  const int rc = stb_tokenizer_load_ex(ctx_, reinterpret_cast<const uint8_t *>(json.data()), json.size(), flags, &text_tok_);
  if (rc == STB_ERR_ARG) { text_tok_ = nullptr; return false; }
  check(rc);
  return true;
}

// ---- model directory (safetensors) ---------------------------------------------------------------
namespace {
float half_to_float(uint16_t h) {
  const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
  uint32_t exp = (h >> 10) & 0x1Fu, man = h & 0x3FFu, bits;
  if (exp == 0) {
    if (man == 0) bits = sign;
    else { int e = -1; do { ++e; man <<= 1; } while (!(man & 0x400u)); bits = sign | ((uint32_t)(127 - 15 - e) << 23) | ((man & 0x3FFu) << 13); }
  } else if (exp == 31) bits = sign | 0x7F800000u | (man << 13);
  else bits = sign | ((exp + 112u) << 23) | (man << 13);
  float f; memcpy(&f, &bits, 4); return f;
}
std::string read_all(const std::string &p) {
  std::ifstream f(p, std::ios::binary);
  if (!f) throw std::runtime_error("cannot read " + p);
  return std::string((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}
struct StTensor { std::string dtype; std::vector<uint64_t> shape; const unsigned char *data = nullptr; uint64_t bytes = 0; uint64_t count = 0; };
bool st_find(const Json &hdr, const std::string &blob, uint64_t base, const char *name, StTensor &t) {
  const Json *e = hdr.get(name);
  if (!e || e->type != Json::Obj) return false;
  const Json *dt = e->get("dtype"), *sh = e->get("shape"), *off = e->get("data_offsets");
  if (!dt || !sh || !off || off->arr.size() != 2) throw std::runtime_error(std::string("model.safetensors: malformed entry for ") + name);
  t.dtype = dt->str;
  t.count = 1;
  for (const auto &d : sh->arr) {
    const uint64_t dim = d.as_u64("a tensor dimension");
    if (dim && t.count > (1ull << 40) / dim) throw std::runtime_error(std::string("model.safetensors: ") + name + " is implausibly large");
    t.shape.push_back(dim); t.count *= dim;
  }
  const uint64_t a = off->arr[0].as_u64("a data offset"), b = off->arr[1].as_u64("a data offset");
  if (b < a || base + b > blob.size()) throw std::runtime_error(std::string("model.safetensors: data of ") + name + " lies outside the file");
  t.data = reinterpret_cast<const unsigned char *>(blob.data()) + base + a;
  t.bytes = b - a;
  return true;
}
template <class T> T load_le(const unsigned char *p) { T v; memcpy(&v, p, sizeof(T)); return v; }
void to_f32(const StTensor &t, const char *name, std::vector<float> &out) {
  const uint64_t w = t.dtype == "F32" ? 4 : t.dtype == "F16" ? 2 : t.dtype == "I8" ? 1 : t.dtype == "F64" ? 8 : 0;
  if (!w || t.bytes != t.count * w) throw std::runtime_error(std::string("model.safetensors: ") + name + " has dtype " + t.dtype + " / a size the host does not read");
  out.resize(t.count);                               // only after the header's element count has been checked against the data it points at
  for (uint64_t i = 0; i < t.count; ++i) {
    const unsigned char *p = t.data + i * w;
    out[i] = w == 4 ? load_le<float>(p) : w == 2 ? half_to_float(load_le<uint16_t>(p)) : w == 1 ? (float)(int8_t)p[0] : (float)load_le<double>(p);
  }
}
}  // namespace

ModelDir load_model_dir(const std::string &dir) {
  ModelDir m;
  m.tokenizer_path = dir + "/tokenizer.json";
  const std::string tok = read_all(m.tokenizer_path);
  const Json cfg = Json::parse(read_all(dir + "/config.json"));
  if (const Json *n = cfg.get("normalize"); n && n->type == Json::Bool) m.normalize = n->b;
  const std::string blob = read_all(dir + "/model.safetensors");
  if (blob.size() < 8) throw std::runtime_error("model.safetensors: truncated");
  const uint64_t hlen = load_le<uint64_t>(reinterpret_cast<const unsigned char *>(blob.data()));
  if (8 + hlen > blob.size()) throw std::runtime_error("model.safetensors: header longer than the file");
  const Json hdr = Json::parse(blob.substr(8, hlen));
  StTensor e, w, mp;
  if (!st_find(hdr, blob, 8 + hlen, "embeddings", e)) throw std::runtime_error("model.safetensors: no \"embeddings\" tensor");
  if (e.shape.size() != 2 || e.shape[1] != STB_DIM) throw std::runtime_error("model.safetensors: the embedding table must be V x 256");
  m.V = e.shape[0];
  to_f32(e, "embeddings", m.E);
  if (st_find(hdr, blob, 8 + hlen, "weights", w)) to_f32(w, "weights", m.weights);
  if (st_find(hdr, blob, 8 + hlen, "mapping", mp)) {
    const uint64_t width = mp.dtype == "I64" || mp.dtype == "U64" ? 8 : mp.dtype == "I32" || mp.dtype == "U32" ? 4 : 0;
    if (!width || mp.bytes != mp.count * width) throw std::runtime_error("model.safetensors: mapping has dtype " + mp.dtype + " / a size the host does not read");
    m.mapping.resize(mp.count);
    for (uint64_t i = 0; i < mp.count; ++i) m.mapping[i] = width == 8 ? (uint32_t)load_le<uint64_t>(mp.data + 8 * i) : load_le<uint32_t>(mp.data + 4 * i);
  }
  // model.py StaticModel.fingerprint: fnv1a64(tokenizer.json bytes) ^ (fnv1a64(first 1 MiB of the f32 table) * golden ratio)
  const uint64_t ht = stb_fnv1a64(reinterpret_cast<const uint8_t *>(tok.data()), tok.size());
  const uint64_t he = stb_fnv1a64(reinterpret_cast<const uint8_t *>(m.E.data()), std::min<uint64_t>(m.E.size() * sizeof(float), 1u << 20));
  char buf[96];
  snprintf(buf, sizeof(buf), "model2vec:%llux%d:n%d:%016llx", (unsigned long long)m.V, STB_DIM, m.normalize ? 1 : 0,
           (unsigned long long)(ht ^ (he * 0x9E3779B97F4A7C15ull)));
  m.fingerprint = buf;
  return m;
}

uint64_t Searcher::rows() const {
  uint64_t n = 0;
  check(stb_corpus_rows(corpus_, &n));
  return n;
}

static void to_csr(const std::vector<std::string> &lines, const Tokenizer &tok, size_t max_len,
                   std::vector<uint64_t> &offsets, std::vector<uint32_t> &ids) {
  tokenize_to_csr(lines, tok, max_len, offsets, ids);
}

// encode_with_args(lines, Some(2048), 16384) (mod.rs:69): batches of 16384 lines.  A producer thread
// tokenises batch i+1 (itself multi-threaded, tokenize_to_csr) while this thread has K3 embed batch i
// (stb_embed: CSR H2D + kernel + optional D2H), so host tokenisation and the GPU overlap; the result is
// identical to one big batch because lines are independent.  `out` (n x 256) and `append_to` may be null.
static const size_t kEmbedBatchLines = 16384;
// With the tokenizer loaded into the library (text_tok), each batch goes to stb_embed_text as text instead, cut by
// truncate_str as tokenize_to_csr cuts it: the library tokenises it, so there is no producer thread to run.
static void embed_batched(stb_ctx *ctx, stb_table *table, const std::vector<std::string> &lines, const Tokenizer &tok,
                          float *out, stb_corpus *append_to, const stb_tokenizer *text_tok) {
  const size_t n = lines.size(), n_batches = (n + kEmbedBatchLines - 1) / kEmbedBatchLines;
  if (text_tok) {
    const size_t max_chars = tok.median_token_length() ? 2048 * tok.median_token_length() : 0;
    std::string text;
    std::vector<uint64_t> offsets;
    for (size_t b = 0; b < n_batches; ++b) {
      const size_t first = b * kEmbedBatchLines, count = std::min(kEmbedBatchLines, n - first);
      text.clear();
      offsets.assign(1, 0);
      for (size_t i = first; i < first + count; ++i) {
        text += truncate_chars(lines[i], max_chars);
        offsets.push_back(text.size());
      }
      check(stb_embed_text(ctx, text_tok, table, reinterpret_cast<const uint8_t *>(text.data()), offsets.data(), count, 2048,
                           out ? out + first * STB_DIM : nullptr, append_to));
    }
    return;
  }
  struct Batch { std::vector<uint64_t> offsets; std::vector<uint32_t> ids; size_t first = 0, count = 0; };
  auto tokenise = [&](size_t b, Batch &dst) {
    dst.first = b * kEmbedBatchLines;
    dst.count = std::min(kEmbedBatchLines, n - dst.first);
    std::vector<std::string> part(lines.begin() + dst.first, lines.begin() + dst.first + dst.count);
    tokenize_to_csr(part, tok, 2048, dst.offsets, dst.ids);
  };
  auto embed = [&](const Batch &b) {
    uint32_t dummy = 0;
    check(stb_embed(ctx, table, b.offsets.data(), b.ids.empty() ? &dummy : b.ids.data(), b.count,
                    out ? out + b.first * STB_DIM : nullptr, append_to));
  };
  Batch cur, nxt;
  tokenise(0, cur);
  for (size_t b = 0; b < n_batches; ++b) {
    std::thread producer;
    std::exception_ptr perr;
    if (b + 1 < n_batches) producer = std::thread([&] { try { tokenise(b + 1, nxt); } catch (...) { perr = std::current_exception(); } });
    try { embed(cur); } catch (...) { if (producer.joinable()) producer.join(); throw; }
    if (producer.joinable()) producer.join();
    if (perr) std::rethrow_exception(perr);
    std::swap(cur, nxt);
  }
}

bool Searcher::add_document(const std::string &filename, const std::string &content, const Tokenizer &tok, bool ignore_case) {
  auto lines = rust_lines(content);
  if (lines.empty()) return false;                             // mod.rs:57-59
  if (!table_) throw std::runtime_error("load_table first");
  std::vector<std::string> emb_lines = lines;
  if (ignore_case) for (auto &l : emb_lines) l = to_lowercase(l);
  Document d{filename, std::move(lines), rows()};
  embed_batched(ctx_, table_, emb_lines, tok, nullptr, corpus_, text_tok_);   // rows go straight into the corpus in HBM
  docs_.push_back(std::move(d));
  return true;
}

std::vector<float> Searcher::embed_lines(const std::vector<std::string> &lines, const Tokenizer &tok, bool ignore_case) const {
  if (!table_) throw std::runtime_error("load_table first");
  std::vector<float> out(lines.size() * STB_DIM);
  if (lines.empty()) return out;
  std::vector<std::string> emb_lines = lines;
  if (ignore_case) for (auto &l : emb_lines) l = to_lowercase(l);
  embed_batched(ctx_, table_, emb_lines, tok, out.data(), nullptr, text_tok_);
  return out;
}

bool Searcher::add_document_embeddings(const std::string &filename, const std::vector<std::string> &lines, const float *emb) {
  if (lines.empty()) return false;
  Document d{filename, lines, rows()};
  check(stb_corpus_append(corpus_, emb, lines.size()));
  docs_.push_back(std::move(d));
  return true;
}

std::vector<float> Searcher::encode_single(const std::string &query, const Tokenizer &tok) const {
  if (!table_) throw std::runtime_error("load_table first");
  std::vector<uint64_t> offsets;
  std::vector<uint32_t> ids;
  to_csr({query}, tok, 512, offsets, ids);                     // encode -> max_length 512
  std::vector<float> out(STB_DIM);
  uint32_t dummy = 0;
  check(stb_embed(ctx_, table_, offsets.data(), ids.empty() ? &dummy : ids.data(), 1, out.data(), nullptr));
  return out;
}

std::vector<SearchResult> Searcher::search_documents(const std::vector<float> &q, const SearchConfig &cfg) const {
  if (q.size() != STB_DIM) return {};                          // cosine -> None: every line skipped (mod.rs:87)
  uint64_t cap = std::max<uint64_t>(cfg.top_k, 1), n = 0;
  if (cfg.max_distance) cap = std::max<uint64_t>(cap, 4096);
  std::vector<stb_hit> hits(cap);
  for (;;) {
    int rc = stb_search(ctx_, corpus_, q.data(), (uint32_t)cfg.top_k, cfg.max_distance ? 1 : 0,
                        cfg.max_distance.value_or(0.0), STB_MODE_SEARCH_DOCUMENTS, nullptr, 0, hits.data(), cap, &n);
    if (rc == STB_ERR_CAPACITY) { cap = n; hits.resize(cap); continue; }
    check(rc);
    break;
  }
  std::vector<SearchResult> out;
  for (uint64_t i = 0; i < n; ++i) {
    // locate (document, line): last document with row_start <= row
    auto it = std::upper_bound(docs_.begin(), docs_.end(), hits[i].row,
                               [](uint64_t r, const Document &d) { return r < d.row_start; });
    const Document &d = *(it - 1);
    const size_t idx = (size_t)(hits[i].row - d.row_start);
    const size_t start = idx > cfg.n_lines ? idx - cfg.n_lines : 0;            // mod.rs:90
    const size_t end = std::min(d.lines.size(), idx + cfg.n_lines + 1);        // mod.rs:91
    SearchResult r;
    r.filename = d.filename;
    r.lines.assign(d.lines.begin() + start, d.lines.begin() + end);
    r.start = start; r.end = end; r.match_line = idx; r.distance = hits[i].distance;
    out.push_back(std::move(r));
  }
  return out;
}

std::string format_search_results(const std::vector<SearchResult> &results, bool is_tty) {
  std::string out;
  char num[32];
  for (const auto &r : results) {
    out += r.filename + ":" + std::to_string(r.start) + "::" + std::to_string(r.end) + " (" + rust_display_f64(r.distance) + ")\n";
    for (size_t i = 0; i < r.lines.size(); ++i) {
      const size_t n = r.start + i;
      snprintf(num, sizeof(num), "%4zu", n + 1);
      if (n == r.match_line && is_tty) out += std::string("\x1b[43m\x1b[30m") + num + ": " + r.lines[i] + "\x1b[0m\n";
      else out += std::string(num) + ": " + r.lines[i] + "\n";
    }
    out += "\n";
  }
  return out;
}

std::string search_output_json(const std::vector<SearchResult> &results) {
  if (results.empty()) return "{\n  \"results\": []\n}";
  std::string o = "{\n  \"results\": [\n";
  for (size_t i = 0; i < results.size(); ++i) {
    const auto &r = results[i];
    std::string content;
    for (size_t j = 0; j < r.lines.size(); ++j) { if (j) content += "\n"; content += r.lines[j]; }
    o += "    {\n";
    o += "      \"filename\": " + json_string(r.filename) + ",\n";
    o += "      \"start_line_number\": " + std::to_string(r.start) + ",\n";
    o += "      \"end_line_number\": " + std::to_string(r.end) + ",\n";
    o += "      \"match_line_number\": " + std::to_string(r.match_line) + ",\n";
    o += "      \"distance\": " + json_f64(r.distance) + ",\n";
    o += "      \"content\": " + json_string(content) + "\n";
    o += i + 1 < results.size() ? "    },\n" : "    }\n";
  }
  o += "  ]\n}";
  return o;
}

}  // namespace semtools

// GPU tokenizer of stb_embed_text: the fast path of HfTokenizer::encode_raw (host/semtools_tokenizer.cpp) --
// a Unigram model behind one Metaspace step with split = true -- on lines of printable ASCII.
//
// Which lines come here is decided by one rule (line_taken, stb_tokenizer_gpu_lines); the others are tokenised
// on host threads by the same HfTokenizer.  Per chunk of lines:
//   stb_tok_normalize_kernel  thread per taken line: the normaliser on printable ASCII, in place in a per-line
//                             region of len + grow + 1 bytes (Prepend adds at most `grow`)
//   stb_tok_unigram_kernel    thread per line: Metaspace pieces (a space starts a piece, the replacement leads
//                             it; the first piece gets it per the prepend scheme), each through the Viterbi of
//                             HfTokenizer::unigram; ids go to the line's region of tok_tmp, the count to tok_cnt
//                             (a declined line's count is its host ids')
//   stb_tok_scan_kernel       one block: exclusive scan of the counts -> K3's CSR offsets
//   stb_tok_write_kernel      warp per line: taken lines' ids from tok_tmp, declined lines' from the host CSR
// A line of k normalised bytes has at most k + 1 tokens (each token covers at least one character, the
// replacement is one character standing for a space or the prepended one), so the region also holds its ids.
#include <algorithm>
#include <exception>
#include <memory>
#include <string>
#include <thread>

#include "common.cuh"
#include "../host/semtools_tokenizer.hpp"

#define STB_TOK_MAX_OPS 8
#define STB_TOK_MAX_PREPEND 16
#define STB_TOK_THREADS 128

using semtools::HfTokenizer;

struct TokPlanDev {
  int n_ops;
  int kind[STB_TOK_MAX_OPS], left[STB_TOK_MAX_OPS], right[STB_TOK_MAX_OPS], pre_len[STB_TOK_MAX_OPS];
  uint8_t pre[STB_TOK_MAX_OPS][STB_TOK_MAX_PREPEND];
  uint8_t rep[4];
  int rep_len;
  int scheme;          // 0 always, 1 first, 2 never
  uint32_t grow;
};

struct TokTrieDev {
  const uint32_t *root, *first_child, *child_node;
  const uint8_t *child_byte;
  const int32_t *terminal;
  const double *scores;
  double unk_score;
  uint32_t unk_id, drop_id;
  int drop_unk;
};

struct stb_tokenizer {
  stb_ctx *ctx = nullptr;
  std::unique_ptr<HfTokenizer> hf;
  HfTokenizer::AsciiPlan plan;         // plan.ok = false: every line is declined
  TokPlanDev dplan{};
  TokTrieDev dtrie{};
  StbBuf<uint32_t> root, first_child, child_node;
  StbBuf<uint8_t> child_byte;
  StbBuf<int32_t> terminal;
  StbBuf<double> scores;
};

// ------------------------------------------------------------------------------------------------ kernels ---
__global__ void __launch_bounds__(STB_TOK_THREADS)
stb_tok_normalize_kernel(const uint8_t *text, const uint64_t *off, const uint8_t *taken, uint64_t m, const TokPlanDev p,
                         uint8_t *norm, uint32_t *nlen) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m || !taken[i]) return;
  const uint64_t b = off[i];
  uint32_t n = (uint32_t)(off[i + 1] - b);
  uint8_t *s = norm + b + i * (p.grow + 1);
  for (uint32_t k = 0; k < n; ++k) s[k] = text[b + k];
  for (int o = 0; o < p.n_ops; ++o) {
    switch (p.kind[o]) {
      case HfTokenizer::OP_LOWER:
        for (uint32_t k = 0; k < n; ++k) if (s[k] >= 'A' && s[k] <= 'Z') s[k] += 32;
        break;
      case HfTokenizer::OP_MULTISPACE: {                   // every run of spaces -> one space
        uint32_t w = 0, r = 0;
        while (r < n) {
          if (s[r] == ' ') { while (r < n && s[r] == ' ') ++r; s[w++] = ' '; }
          else s[w++] = s[r++];
        }
        n = w;
        break;
      }
      case HfTokenizer::OP_STRIP: {
        uint32_t lo = 0, hi = n;
        if (p.left[o]) while (lo < hi && s[lo] == ' ') ++lo;
        if (p.right[o]) while (hi > lo && s[hi - 1] == ' ') --hi;
        for (uint32_t k = lo; k < hi; ++k) s[k - lo] = s[k];
        n = hi - lo;
        break;
      }
      case HfTokenizer::OP_PREPEND: {
        const uint32_t L = (uint32_t)p.pre_len[o];
        if (n == 0 || L == 0) break;
        for (uint32_t k = n; k-- > 0;) s[k + L] = s[k];
        for (uint32_t k = 0; k < L; ++k) s[k] = p.pre[o][k];
        n += L;
        break;
      }
    }
  }
  nlen[i] = n;
}

__device__ __forceinline__ uint32_t tok_step(const TokTrieDev &t, uint32_t node, uint8_t c) {
  if (node == 0) return __ldg(t.root + c);
  uint32_t lo = __ldg(t.first_child + node);
  const uint32_t end = __ldg(t.first_child + node + 1);
  uint32_t hi = end;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(t.child_byte + mid) < c) lo = mid + 1; else hi = mid;
  }
  return (lo < end && __ldg(t.child_byte + lo) == c) ? __ldg(t.child_node + lo) : 0xffffffffu;
}

__device__ __forceinline__ uint32_t tok_utf8_len(uint8_t c) {
  return c < 0x80 ? 1 : (c >> 5) == 6 ? 2 : (c >> 4) == 14 ? 3 : (c >> 3) == 30 ? 4 : 1;
}

struct TokLattice {
  double score[STB_TOKENIZER_PIECE_CAP + 1];
  int32_t id[STB_TOKENIZER_PIECE_CAP + 1];
  int16_t start[STB_TOKENIZER_PIECE_CAP + 1];
};

// One piece -- the replacement (if `rep`) then run[0, len) -- through HfTokenizer::unigram: ids appended at
// ids[*cnt ..] while below `limit`, *cnt counts them all (after the unk fusing and the unk_token drop).
__device__ void tok_piece(const TokPlanDev &p, const TokTrieDev &t, TokLattice &L, bool rep, const uint8_t *run,
                          uint32_t len, uint32_t *ids, uint32_t *cnt, uint32_t limit, int *err) {
  const uint32_t r = rep ? (uint32_t)p.rep_len : 0, size = r + len;
  if (size == 0) return;
  if (size > STB_TOKENIZER_PIECE_CAP) { atomicOr(err, 1); return; }
  auto byte = [&](uint32_t k) -> uint8_t { return k < r ? p.rep[k] : run[k - r]; };
  for (uint32_t k = 0; k <= size; ++k) { L.score[k] = 0.0; L.id[k] = 0; L.start[k] = -1; }
  uint32_t at = 0;
  while (at < size) {
    const double here = L.score[at];
    bool has_single = false;
    const uint32_t mb = min(tok_utf8_len(byte(at)), size - at);
    uint32_t node = 0;
    for (uint32_t k = at; k < size; ++k) {
      node = tok_step(t, node, byte(k));
      if (node == 0xffffffffu) break;
      const int32_t id = __ldg(t.terminal + node);
      if (id < 0) continue;
      const uint32_t kp = k + 1;
      const double cand = __ldg(t.scores + id) + here;
      if (L.start[kp] < 0 || cand > L.score[kp]) { L.score[kp] = cand; L.start[kp] = (int16_t)at; L.id[kp] = id; }
      if (!has_single && kp - at == mb) has_single = true;
    }
    if (!has_single) {
      const uint32_t kp = at + mb;
      const double cand = t.unk_score + here;
      if (L.start[kp] < 0 || cand > L.score[kp]) { L.score[kp] = cand; L.start[kp] = (int16_t)at; L.id[kp] = (int32_t)t.unk_id; }
    }
    at += mb;
  }
  // backtrack twice: count the piece's ids, then write them back to front
  uint32_t k = 0;
  for (int pass = 0; pass < 2; ++pass) {
    uint32_t e = size, j = 0;
    bool in_unk = false;
    while (e > 0) {
      const uint32_t id = (uint32_t)L.id[e];
      bool emit = true;
      if (id == t.unk_id) { emit = !in_unk; in_unk = true; } else in_unk = false;
      if (emit && !(t.drop_unk && id == t.drop_id)) {
        if (pass == 1) { const uint32_t pos = *cnt + k - 1 - j; if (pos < limit) ids[pos] = id; }
        ++j;
      }
      e = (uint32_t)L.start[e];
    }
    k = j;
  }
  *cnt += k;
}

__global__ void __launch_bounds__(STB_TOK_THREADS)
stb_tok_unigram_kernel(const uint8_t *norm, const uint32_t *nlen, const uint64_t *off, const uint8_t *taken,
                       const uint64_t *hoff, uint64_t m, const TokPlanDev p, const TokTrieDev t, uint32_t max_length,
                       uint32_t *tmp, uint32_t *count, int *err) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  if (!taken[i]) { count[i] = (uint32_t)(hoff[i + 1] - hoff[i]); return; }
  TokLattice L;
  const uint64_t base = off[i] + i * (p.grow + 1);
  const uint32_t region = (uint32_t)(off[i + 1] - off[i]) + p.grow + 1, limit = min(region, max_length);
  const uint8_t *s = norm + base;
  const uint32_t n = nlen[i];
  uint32_t *ids = tmp + base, cnt = 0;
  if (n > 0) {
    // encode_raw's Metaspace fast path; a taken line is one split that starts the input (origin)
    const bool prepend = s[0] != ' ' && p.scheme != 2;
    uint32_t q = 0;
    if (s[0] != ' ') {
      while (q < n && s[q] != ' ') ++q;
      tok_piece(p, t, L, prepend, s, q, ids, &cnt, limit, err);
    }
    while (q < n) {                                        // s[q] == ' ': the next piece
      uint32_t e = q + 1;
      while (e < n && s[e] != ' ') ++e;
      tok_piece(p, t, L, true, s + q + 1, e - q - 1, ids, &cnt, limit, err);
      q = e;
    }
  }
  if (cnt > region && region < max_length) atomicOr(err, 2);
  count[i] = min(cnt, max_length);
}

// exclusive scan of m counts into off[0..m] (one block of 1024 threads, a contiguous segment each)
__global__ void __launch_bounds__(1024) stb_tok_scan_kernel(const uint32_t *count, uint64_t m, uint64_t *off) {
  __shared__ uint64_t part[1024];
  const int tid = threadIdx.x;
  const uint64_t per = (m + 1023) / 1024, lo = min(m, tid * per), hi = min(m, lo + per);
  uint64_t s = 0;
  for (uint64_t j = lo; j < hi; ++j) s += count[j];
  part[tid] = s;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {
    const uint64_t v = tid >= d ? part[tid - d] : 0;
    __syncthreads();
    part[tid] += v;
    __syncthreads();
  }
  uint64_t run = tid ? part[tid - 1] : 0;
  for (uint64_t j = lo; j < hi; ++j) { off[j] = run; run += count[j]; }
  if (tid == 1023) off[m] = part[1023];
}

__global__ void __launch_bounds__(256)
stb_tok_write_kernel(const uint64_t *csr_off, const uint32_t *count, const uint8_t *taken, const uint32_t *tmp,
                     const uint64_t *off, uint32_t grow, const uint64_t *hoff, const uint32_t *hids, uint64_t m,
                     uint32_t *ids) {
  const uint64_t line = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (line >= m) return;
  const uint64_t dst = csr_off[line];
  const uint32_t c = count[line];
  const uint32_t *src = taken[line] ? tmp + off[line] + line * (grow + 1) : hids + hoff[line];
  for (uint32_t j = lane; j < c; j += 32) ids[dst + j] = src[j];
}

// ------------------------------------------------------------------------------------------------- host ---
const stb_ctx *stb_tokenizer_ctx(const stb_tokenizer *tok) { return tok->ctx; }

// The one rule for which lines go to the GPU (header: stb_tokenizer_gpu_lines).
static bool line_taken(const stb_tokenizer *tok, const uint8_t *s, uint64_t n) {
  const HfTokenizer::AsciiPlan &p = tok->plan;
  if (!p.ok) return false;
  uint64_t run = 0, longest = 0;
  for (uint64_t k = 0; k < n; ++k) {
    const uint8_t c = s[k];
    if (c < 0x20 || c > 0x7E || !p.byte_ok[c]) return false;
    run = c == ' ' ? 0 : run + 1;
    longest = std::max(longest, run);
  }
  if (p.replacement.size() + p.grow + longest > STB_TOKENIZER_PIECE_CAP) return false;
  if (p.decline_leading_space && n && s[0] == ' ') return false;
  if (p.added.empty()) return true;
  const std::string line(reinterpret_cast<const char *>(s), n);
  for (const auto &a : p.added) if (line.find(a) != std::string::npos) return false;
  if (p.added_normalized) {
    const std::string norm = tok->hf->normalize_str(line);
    for (const auto &a : p.added) if (norm.find(a) != std::string::npos) return false;
  }
  return true;
}

static int check_text(const uint8_t *text, const uint64_t *offsets, uint64_t n_lines, const char *what) {
  if (!offsets) { stb_set_error("%s: text_offsets is null", what); return STB_ERR_ARG; }
  if (offsets[0] != 0) { stb_set_error("%s: text_offsets[0] must be 0", what); return STB_ERR_ARG; }
  for (uint64_t i = 0; i < n_lines; ++i)
    if (offsets[i + 1] < offsets[i]) { stb_set_error("%s: text_offsets not monotone at line %llu", what, (unsigned long long)i); return STB_ERR_ARG; }
  if (offsets[n_lines] && !text) { stb_set_error("%s: text is null", what); return STB_ERR_ARG; }
  return STB_OK;
}

int stb_text_host(const stb_tokenizer *tok, const uint8_t *text, const uint64_t *offsets, uint64_t n_lines,
                  uint32_t max_length, StbTextHost &h) {
  int rc = check_text(text, offsets, n_lines, "embed_text");
  if (rc) return rc;
  h.taken.assign(n_lines, 0);
  h.hoff.assign(n_lines + 1, 0);
  h.hids.clear();
  unsigned threads = std::max(1u, std::thread::hardware_concurrency());
  threads = (unsigned)std::min<uint64_t>(threads, std::max<uint64_t>(1, n_lines / 256));
  std::vector<std::vector<uint32_t>> part(threads);
  std::vector<std::string> fail(threads);
  auto work = [&](unsigned w) {
    const uint64_t lo = n_lines * w / threads, hi = n_lines * (w + 1) / threads;
    try {
      for (uint64_t i = lo; i < hi; ++i) {
        const uint8_t *s = text + offsets[i];
        const uint64_t n = offsets[i + 1] - offsets[i];
        if ((h.taken[i] = line_taken(tok, s, n))) continue;
        std::vector<uint32_t> v = tok->hf->encode(std::string(reinterpret_cast<const char *>(s), n));
        if (v.size() > max_length) v.resize(max_length);
        h.hoff[i + 1] = v.size();
        part[w].insert(part[w].end(), v.begin(), v.end());
      }
    } catch (const std::exception &e) {
      fail[w] = e.what();
    }
  };
  if (threads == 1) work(0);
  else {
    std::vector<std::thread> pool;
    for (unsigned w = 0; w < threads; ++w) pool.emplace_back(work, w);
    for (auto &th : pool) th.join();
  }
  for (const auto &f : fail)
    if (!f.empty()) { stb_set_error("embed_text: %s", f.c_str()); return STB_ERR_ARG; }
  for (uint64_t i = 0; i < n_lines; ++i) h.hoff[i + 1] += h.hoff[i];
  h.hids.reserve(h.hoff[n_lines]);
  for (auto &p : part) h.hids.insert(h.hids.end(), p.begin(), p.end());
  h.chunk_at.clear();
  for (uint64_t l = 0; l < n_lines;) {
    h.chunk_at.push_back(l);
    const uint64_t first = l;
    ++l;
    while (l < n_lines && l - first < STB_TEXT_CHUNK_LINES && offsets[l + 1] - offsets[first] <= STB_TEXT_CHUNK_BYTES) ++l;
  }
  h.chunk_at.push_back(n_lines);
  return STB_OK;
}

// ids of chunk [l0, l0 + m), at most: a taken line's region (capped at max_length), a declined line's host ids
static uint64_t chunk_ids_bound(const stb_tokenizer *tok, const StbTextHost &h, const uint64_t *offsets, uint64_t l0,
                                uint64_t m, uint32_t max_length) {
  uint64_t bound = 0;
  for (uint64_t i = l0; i < l0 + m; ++i)
    bound += h.taken[i] ? std::min<uint64_t>(max_length, offsets[i + 1] - offsets[i] + tok->dplan.grow + 1) : h.hoff[i + 1] - h.hoff[i];
  return bound;
}

int stb_tok_reserve(stb_ctx *ctx, const stb_tokenizer *tok, const StbTextHost &h, const uint64_t *offsets, uint32_t max_length) {
  uint64_t bytes = 1, lines = 1, hids = 1, region = 1, ids = 1;
  for (size_t c = 0; c + 1 < h.chunk_at.size(); ++c) {
    const uint64_t l0 = h.chunk_at[c], m = h.chunk_at[c + 1] - l0, b = offsets[l0 + m] - offsets[l0];
    bytes = std::max(bytes, b);
    lines = std::max(lines, m);
    hids = std::max(hids, h.hoff[l0 + m] - h.hoff[l0]);
    region = std::max(region, b + m * (tok->dplan.grow + 1));
    ids = std::max(ids, chunk_ids_bound(tok, h, offsets, l0, m, max_length));
  }
  int rc;
  if ((rc = ctx->tok_text.reserve(bytes, 1 << 20)) != STB_OK ||
      (rc = ctx->tok_off.reserve(lines + 1, 4096)) != STB_OK || (rc = ctx->tok_hoff.reserve(lines + 1, 4096)) != STB_OK ||
      (rc = ctx->tok_taken.reserve(lines, 4096)) != STB_OK || (rc = ctx->tok_hids.reserve(hids, 4096)) != STB_OK ||
      (rc = ctx->tok_norm.reserve(region, 1 << 20)) != STB_OK || (rc = ctx->tok_tmp.reserve(region, 1 << 20)) != STB_OK ||
      (rc = ctx->tok_nlen.reserve(lines, 4096)) != STB_OK || (rc = ctx->tok_cnt.reserve(lines, 4096)) != STB_OK ||
      (rc = ctx->embed_off_dev.reserve(lines + 1, 4096)) != STB_OK || (rc = ctx->embed_ids_dev.reserve(ids, 65536)) != STB_OK)
    return rc;
  return STB_OK;
}

int stb_tok_chunk(stb_ctx *ctx, const stb_tokenizer *tok, const StbTextHost &h, const uint8_t *text,
                  const uint64_t *offsets, uint64_t l0, uint64_t m, uint32_t max_length) {
  const uint64_t b0 = offsets[l0], bytes = offsets[l0 + m] - b0, h0 = h.hoff[l0], nh = h.hoff[l0 + m] - h0;
  const uint32_t grow = tok->dplan.grow;
  std::vector<uint64_t> off(m + 1), hoff(m + 1);
  for (uint64_t i = 0; i <= m; ++i) { off[i] = offsets[l0 + i] - b0; hoff[i] = h.hoff[l0 + i] - h0; }
  cudaStream_t st = ctx->stream;
  if (bytes) STB_CUDA(cudaMemcpyAsync(ctx->tok_text, text + b0, bytes, cudaMemcpyHostToDevice, st));
  STB_CUDA(cudaMemcpyAsync(ctx->tok_off, off.data(), (m + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  STB_CUDA(cudaMemcpyAsync(ctx->tok_hoff, hoff.data(), (m + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  STB_CUDA(cudaMemcpyAsync(ctx->tok_taken, h.taken.data() + l0, m, cudaMemcpyHostToDevice, st));
  if (nh) STB_CUDA(cudaMemcpyAsync(ctx->tok_hids, h.hids.data() + h0, nh * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  const unsigned blocks = (unsigned)((m + STB_TOK_THREADS - 1) / STB_TOK_THREADS);
  stb_tok_normalize_kernel<<<blocks, STB_TOK_THREADS, 0, st>>>(ctx->tok_text, ctx->tok_off, ctx->tok_taken, m, tok->dplan,
                                                               ctx->tok_norm, ctx->tok_nlen);
  STB_CUDA(cudaGetLastError());
  stb_tok_unigram_kernel<<<blocks, STB_TOK_THREADS, 0, st>>>(ctx->tok_norm, ctx->tok_nlen, ctx->tok_off, ctx->tok_taken,
                                                             ctx->tok_hoff, m, tok->dplan, tok->dtrie, max_length,
                                                             ctx->tok_tmp, ctx->tok_cnt, ctx->tok_flag);
  STB_CUDA(cudaGetLastError());
  stb_tok_scan_kernel<<<1, 1024, 0, st>>>(ctx->tok_cnt, m, ctx->embed_off_dev);
  STB_CUDA(cudaGetLastError());
  stb_tok_write_kernel<<<(unsigned)((m * 32 + 255) / 256), 256, 0, st>>>(ctx->embed_off_dev, ctx->tok_cnt, ctx->tok_taken,
                                                                         ctx->tok_tmp, ctx->tok_off, grow, ctx->tok_hoff,
                                                                         ctx->tok_hids, m, ctx->embed_ids_dev);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches += 4;
  return STB_OK;
}

extern "C" {

int stb_tokenizer_load(stb_ctx *ctx, const uint8_t *json, uint64_t len, stb_tokenizer **out) {
  int rc = stb_ctx_use(ctx);
  if (rc) return rc;
  if (!out || (!json && len)) { stb_set_error("tokenizer_load: null argument"); return STB_ERR_ARG; }
  *out = nullptr;
  std::unique_ptr<stb_tokenizer> t(new (std::nothrow) stb_tokenizer());
  if (!t) { stb_set_error("out of host memory"); return STB_ERR_NOMEM; }
  t->ctx = ctx;
  try {
    t->hf = HfTokenizer::from_json(std::string(reinterpret_cast<const char *>(json), len));
    t->plan = t->hf->ascii_plan();
  } catch (const std::exception &e) {
    stb_set_error("tokenizer_load: %s", e.what());
    return STB_ERR_ARG;
  }
  HfTokenizer::AsciiPlan &p = t->plan;
  if (p.ops.size() > STB_TOK_MAX_OPS) p.ok = false;
  for (const auto &op : p.ops) if (op.text.size() > STB_TOK_MAX_PREPEND) p.ok = false;
  TokPlanDev &d = t->dplan;
  if (p.ok) {
    d.n_ops = (int)p.ops.size();
    for (int o = 0; o < d.n_ops; ++o) {
      d.kind[o] = p.ops[o].kind; d.left[o] = p.ops[o].left; d.right[o] = p.ops[o].right;
      d.pre_len[o] = (int)p.ops[o].text.size();
      memcpy(d.pre[o], p.ops[o].text.data(), p.ops[o].text.size());
    }
    d.rep_len = (int)p.replacement.size();
    memcpy(d.rep, p.replacement.data(), p.replacement.size());
    d.scheme = p.prepend_scheme;
    d.grow = (uint32_t)p.grow;
  }
  const HfTokenizer::TrieView v = t->hf->trie();
  if ((rc = t->root.alloc(256)) != STB_OK || (rc = t->first_child.alloc(v.n_nodes + 1)) != STB_OK ||
      (rc = t->child_node.alloc(std::max<size_t>(v.n_edges, 1))) != STB_OK ||
      (rc = t->child_byte.alloc(std::max<size_t>(v.n_edges, 1))) != STB_OK ||
      (rc = t->terminal.alloc(v.n_nodes)) != STB_OK || (rc = t->scores.alloc(v.n_scores)) != STB_OK)
    return rc;
  cudaError_t e = cudaMemcpy(t->root, v.root, 256 * sizeof(uint32_t), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(t->first_child, v.first_child, (v.n_nodes + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && v.n_edges) e = cudaMemcpy(t->child_node, v.child_node, v.n_edges * sizeof(uint32_t), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && v.n_edges) e = cudaMemcpy(t->child_byte, v.child_byte, v.n_edges, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(t->terminal, v.terminal, v.n_nodes * sizeof(int32_t), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(t->scores, v.scores, v.n_scores * sizeof(double), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) { stb_set_error("tokenizer_load: upload failed: %s", cudaGetErrorString(e)); return STB_ERR_CUDA; }
  t->dtrie = {t->root, t->first_child, t->child_node, t->child_byte, t->terminal, t->scores, v.unk_score, v.unk_id, v.drop_id, v.drop_unk ? 1 : 0};
  if ((rc = ctx->tok_flag.reserve(1)) != STB_OK) return rc;
  *out = t.release();
  return STB_OK;
}

int stb_tokenizer_destroy(stb_tokenizer *t) {
  if (!t) return STB_OK;
  if (t->ctx && stb_ctx_alive(t->ctx)) { cudaSetDevice(t->ctx->device); cudaStreamSynchronize(t->ctx->stream); }
  else cudaDeviceSynchronize();
  cudaGetLastError();
  delete t;
  return STB_OK;
}

int stb_tokenizer_gpu_lines(const stb_tokenizer *tok, const uint8_t *text, const uint64_t *text_offsets, uint64_t n_lines,
                            uint8_t *taken) {
  if (!tok || (n_lines && !taken)) { stb_set_error("tokenizer_gpu_lines: null argument"); return STB_ERR_ARG; }
  if (n_lines == 0) return STB_OK;
  int rc = check_text(text, text_offsets, n_lines, "tokenizer_gpu_lines");
  if (rc) return rc;
  for (uint64_t i = 0; i < n_lines; ++i) taken[i] = line_taken(tok, text + text_offsets[i], text_offsets[i + 1] - text_offsets[i]);
  return STB_OK;
}

int stb_debug_tokenize(stb_ctx *ctx, const stb_tokenizer *tok, const uint8_t *text, const uint64_t *text_offsets,
                       uint64_t n_lines, uint32_t max_length, uint64_t *ids_offsets, uint32_t *ids, uint64_t ids_cap,
                       uint8_t *taken) {
  int rc = stb_ctx_use(ctx);
  if (rc) return rc;
  if (!tok || tok->ctx != ctx || !ids_offsets || (ids_cap && !ids)) { stb_set_error("debug_tokenize: bad argument"); return STB_ERR_ARG; }
  ids_offsets[0] = 0;
  if (n_lines == 0) return STB_OK;
  StbTextHost h;
  if ((rc = stb_text_host(tok, text, text_offsets, n_lines, max_length, h)) != STB_OK) return rc;
  if (taken) memcpy(taken, h.taken.data(), n_lines);
  if ((rc = stb_tok_reserve(ctx, tok, h, text_offsets, max_length)) != STB_OK) return rc;
  STB_CUDA(cudaMemsetAsync(ctx->tok_flag, 0, sizeof(int), ctx->stream));
  bool fits = true;
  for (size_t c = 0; c + 1 < h.chunk_at.size(); ++c) {
    const uint64_t l0 = h.chunk_at[c], m = h.chunk_at[c + 1] - l0;
    if ((rc = stb_tok_chunk(ctx, tok, h, text, text_offsets, l0, m, max_length)) != STB_OK) return rc;
    std::vector<uint64_t> off(m + 1);
    STB_CUDA(cudaMemcpyAsync(off.data(), ctx->embed_off_dev, (m + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
    STB_CUDA(cudaStreamSynchronize(ctx->stream));
    const uint64_t base = ids_offsets[l0];
    for (uint64_t i = 1; i <= m; ++i) ids_offsets[l0 + i] = base + off[i];
    fits = fits && base + off[m] <= ids_cap;
    if (fits && off[m])
      STB_CUDA(cudaMemcpy(ids + base, ctx->embed_ids_dev, off[m] * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  }
  int flag = 0;
  STB_CUDA(cudaMemcpy(&flag, ctx->tok_flag, sizeof(int), cudaMemcpyDeviceToHost));
  if (flag) { stb_set_error("debug_tokenize: a GPU piece overflowed its bound (flag %d)", flag); return STB_ERR_STATE; }
  if (!fits) { stb_set_error("debug_tokenize: %llu ids do not fit ids_cap", (unsigned long long)ids_offsets[n_lines]); return STB_ERR_CAPACITY; }
  return STB_OK;
}

}  // extern "C"

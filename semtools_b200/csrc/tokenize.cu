// GPU tokenizer of stb_embed_text: the fast path of HfTokenizer::encode_raw (host/semtools_tokenizer.cpp) --
// a Unigram model behind one Metaspace step with split = true -- on lines of printable ASCII (a flags-0 handle)
// or of any valid UTF-8 (a STB_TOKENIZER_UTF8 handle).
//
// Which lines come here is decided by one rule (line_taken, stb_tokenizer_gpu_lines); the others are tokenised
// on host threads by the same HfTokenizer.  Per chunk of lines, a flags-0 handle runs:
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
//
// A UTF-8 handle runs, per chunk:
//   stb_tok_utf8_normalize_kernel  thread per candidate line: the normaliser steps in order (Lowercase per
//                             character, Replace(" {2,}"), Strip on White_Space, Prepend, Precompiled cluster by
//                             cluster), between tok_norm and tok_norm2 in a region of STB_TOK_UTF8_R x len +
//                             grow + 1 bytes; a status byte per line: 0, or why the line is given back
//   stb_tok_utf8_unigram_kernel    thread per candidate line with status 0: Metaspace pieces split on spaces and
//                             on the replacement itself, each through the same Viterbi (tok_piece)
//   one copy of the status bytes to the host, which encodes the given-back lines with HfTokenizer and uploads
//   the chunk's host CSR (declined and given-back lines) and which lines' ids came from the GPU; then
//   stb_tok_fill_kernel (host lines' counts), stb_tok_scan_kernel and stb_tok_write_kernel as above.
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
// A UTF-8 line's region is R x len + grow + 1 bytes.  Normalising grows text only where the charsmap expands a
// character (ligatures, squared and circled forms, U+FDFA: 3 bytes -> 33) or Lowercase lengthens one (U+0130:
// 2 bytes -> 3); most scripts keep their length or shrink (full-width forms 3 -> 1).  R = 2 leaves room for
// every line of the multilingual probe and gives back only pathological ones (embed_text_utf8_probe.py reports
// the overflow count).
#define STB_TOK_UTF8_R 2u

// why a UTF-8 candidate line is given back to the host tokenizer (tok_status)
enum { TOK_GPU = 0, TOK_OVERFLOW = 1, TOK_PIECE_CAP = 2, TOK_FIRST = 3 };

using semtools::HfTokenizer;
using semtools::LowerEntry;

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

// The tables of a UTF-8 handle's normaliser: per op, the Precompiled charsmap it applies (darts-clone units,
// replacement blob, the printable ASCII bytes it leaves alone); the grapheme-break properties; the lowercase map
struct TokMapDev {
  const uint32_t *trie;
  const uint8_t *norm;
  uint32_t n_trie, n_norm;
  uint32_t ascii_plain[4];
};
struct TokUtf8Dev {
  TokMapDev map[STB_TOK_MAX_OPS];
  const uint8_t *gb_bmp;
  const HfTokenizer::PropRange *gcb, *ext_pict, *incb;
  uint32_t n_gcb, n_ext_pict, n_incb, n_lower;
  const LowerEntry *lower;
};

struct stb_tokenizer {
  stb_ctx *ctx = nullptr;
  std::unique_ptr<HfTokenizer> hf;
  HfTokenizer::AsciiPlan plan;         // plan.ok = false: every line is declined
  bool utf8 = false;                   // STB_TOKENIZER_UTF8: the rule and the kernels take UTF-8 text
  TokPlanDev dplan{};
  TokTrieDev dtrie{};
  TokUtf8Dev dutf8{};
  StbBuf<uint32_t> root, first_child, child_node;
  StbBuf<uint8_t> child_byte;
  StbBuf<int32_t> terminal;
  StbBuf<double> scores;
  // UTF-8 handles: every charsmap's units and blob back to back, the BMP property bytes, the range tables, kLower
  StbBuf<uint32_t> cm_trie;
  StbBuf<uint8_t> cm_norm, gb_bmp;
  StbBuf<HfTokenizer::PropRange> gb_ranges;
  StbBuf<LowerEntry> lower;
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

// ------------------------------------------------------------------------------------ UTF-8 kernels ---
// The rule hands these kernels valid UTF-8 only, and every step writes valid UTF-8, so decoding needs no checks.
__device__ __forceinline__ uint32_t tok_decode(const uint8_t *s, uint32_t *len) {
  const uint32_t c = s[0];
  if (c < 0x80) { *len = 1; return c; }
  if (c < 0xE0) { *len = 2; return ((c & 0x1F) << 6) | (s[1] & 0x3F); }
  if (c < 0xF0) { *len = 3; return ((c & 0x0F) << 12) | ((s[1] & 0x3F) << 6) | (s[2] & 0x3F); }
  *len = 4;
  return ((c & 0x07) << 18) | ((s[1] & 0x3F) << 12) | ((s[2] & 0x3F) << 6) | (s[3] & 0x3F);
}

// appends cp at d[*w], or returns false when it would pass cap
__device__ __forceinline__ bool tok_encode(uint32_t cp, uint8_t *d, uint32_t *w, uint32_t cap) {
  const uint32_t n = cp < 0x80 ? 1 : cp < 0x800 ? 2 : cp < 0x10000 ? 3 : 4;
  if (*w + n > cap) return false;
  uint8_t *o = d + *w;
  if (n == 1) o[0] = (uint8_t)cp;
  else if (n == 2) { o[0] = (uint8_t)(0xC0 | (cp >> 6)); o[1] = (uint8_t)(0x80 | (cp & 0x3F)); }
  else if (n == 3) { o[0] = (uint8_t)(0xE0 | (cp >> 12)); o[1] = (uint8_t)(0x80 | ((cp >> 6) & 0x3F)); o[2] = (uint8_t)(0x80 | (cp & 0x3F)); }
  else {
    o[0] = (uint8_t)(0xF0 | (cp >> 18)); o[1] = (uint8_t)(0x80 | ((cp >> 12) & 0x3F));
    o[2] = (uint8_t)(0x80 | ((cp >> 6) & 0x3F)); o[3] = (uint8_t)(0x80 | (cp & 0x3F));
  }
  *w += n;
  return true;
}

// Unicode White_Space at s (is_space_at)
__device__ __forceinline__ bool tok_is_space(const uint8_t *s, uint32_t *len) {
  const uint32_t c = s[0];
  if (c < 0x80) { *len = 1; return c == ' ' || (c >= 9 && c <= 13); }
  const uint32_t cp = tok_decode(s, len);
  return cp == 0x85 || cp == 0xA0 || cp == 0x1680 || (cp >= 0x2000 && cp <= 0x200A) || cp == 0x2028 || cp == 0x2029 ||
         cp == 0x202F || cp == 0x205F || cp == 0x3000;
}

__device__ uint8_t tok_range(const HfTokenizer::PropRange *t, uint32_t n, uint32_t cp) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(&t[mid].b) < cp) lo = mid + 1; else hi = mid; }
  return (lo < n && __ldg(&t[lo].a) <= cp) ? __ldg(&t[lo].v) : 0;
}

// gcb | ext_pict << 4 | incb << 5, as the host's gb_props (Hangul syllables are in the BMP table)
__device__ __forceinline__ uint8_t tok_gb_props(const TokUtf8Dev &u, uint32_t cp) {
  if (cp < 0x10000) return __ldg(u.gb_bmp + cp);
  return (uint8_t)(tok_range(u.gcb, u.n_gcb, cp) | (tok_range(u.ext_pict, u.n_ext_pict, cp) ? 0x10 : 0) |
                   (tok_range(u.incb, u.n_incb, cp) << 5));
}

// UAX #29 extended grapheme clusters, the state machine of grapheme_ends: is there a boundary before a character
// with these properties?  (GCB values and InCB values as in semtools_tokenizer.cpp)
struct TokGb { int prev = -1, ri_run = 0, ep_state = 0, incb_state = 0; };
__device__ __forceinline__ bool tok_gb_break(TokGb &g, uint8_t props) {
  enum { OTHER = 0, CR, LF, CONTROL, EXTEND, ZWJ, RI, PREPEND, SPACINGMARK, L, V, T, LV, LVT };
  const int c = props & 0x0F, incb = props >> 5, prev = g.prev;
  const bool ep = (props & 0x10) != 0;
  bool brk = false;
  if (prev >= 0) {
    if (prev == CR && c == LF) brk = false;                                                    // GB3
    else if (prev == CONTROL || prev == CR || prev == LF) brk = true;                          // GB4
    else if (c == CONTROL || c == CR || c == LF) brk = true;                                   // GB5
    else if (prev == L && (c == L || c == V || c == LV || c == LVT)) brk = false;              // GB6
    else if ((prev == LV || prev == V) && (c == V || c == T)) brk = false;                     // GB7
    else if ((prev == LVT || prev == T) && c == T) brk = false;                                // GB8
    else if (c == EXTEND || c == ZWJ) brk = false;                                             // GB9
    else if (c == SPACINGMARK) brk = false;                                                    // GB9a
    else if (prev == PREPEND) brk = false;                                                     // GB9b
    else if (g.incb_state == 2 && incb == 1) brk = false;                                      // GB9c
    else if (g.ep_state == 2 && ep) brk = false;                                               // GB11
    else if (prev == RI && c == RI && (g.ri_run & 1)) brk = false;                             // GB12, GB13
    else brk = true;                                                                           // GB999
  }
  g.ri_run = c == RI ? g.ri_run + 1 : 0;
  if (ep) g.ep_state = 1;
  else if (g.ep_state == 1 && c == EXTEND) g.ep_state = 1;
  else if (g.ep_state == 1 && c == ZWJ) g.ep_state = 2;
  else g.ep_state = 0;
  if (incb == 1) g.incb_state = 1;                                      // Consonant
  else if (g.incb_state >= 1 && incb == 2) {}                           // Extend keeps the state
  else if (g.incb_state >= 1 && incb == 3) g.incb_state = 2;            // Linker
  else g.incb_state = 0;
  g.prev = c;
  return brk;
}

// Charsmap::first_prefix: the darts-clone walk, stopping at NUL; offset of the shortest key's replacement or -1
__device__ int64_t tok_first_prefix(const TokMapDev &m, const uint8_t *p, uint32_t n) {
  if (m.n_trie == 0) return -1;
  auto offset = [](uint32_t u) { return (uint64_t)(u >> 10) << ((u & (1u << 9)) >> 6); };
  uint64_t node = 0;
  uint32_t unit = __ldg(m.trie);
  node ^= offset(unit);
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t c = p[i];
    if (c == 0) break;
    node ^= c;
    if (node >= m.n_trie) return -1;
    unit = __ldg(m.trie + node);
    if ((unit & ((1u << 31) | 0xFFu)) != c) return -1;
    node ^= offset(unit);
    if ((unit >> 8) & 1u) {
      if (node >= m.n_trie) return -1;
      return (int64_t)(__ldg(m.trie + node) & ((1u << 31) - 1u));
    }
  }
  return -1;
}

// apply_charsmap: every cluster shorter than 6 bytes is looked up whole (the shortest key that is a prefix of it
// replaces it), otherwise character by character.  A one-byte cluster of a printable ASCII byte the map leaves
// alone is copied (the lookup would find nothing).  *lead: whether the first output byte comes from the first
// cluster.  Returns false when the output would pass cap.
__device__ bool tok_charsmap(const TokMapDev &m, const TokUtf8Dev &u, const uint8_t *s, uint32_t n, uint8_t *d,
                             uint32_t *out_n, uint32_t cap, bool *lead) {
  uint32_t w = 0;
  auto emit = [&](int64_t at) {
    for (uint32_t k = (uint32_t)at; k < m.n_norm; ++k) {
      const uint8_t b = __ldg(m.norm + k);
      if (b == 0) break;
      if (w >= cap) return false;
      d[w++] = b;
    }
    return true;
  };
  auto copy = [&](uint32_t b, uint32_t e) {
    if (w + (e - b) > cap) return false;
    for (uint32_t k = b; k < e; ++k) d[w++] = s[k];
    return true;
  };
  auto cluster = [&](uint32_t b, uint32_t e) {
    if (e - b == 1 && s[b] >= 0x20 && s[b] < 0x7F && ((m.ascii_plain[s[b] >> 5] >> (s[b] & 31)) & 1u)) return copy(b, e);
    if (e - b < 6) {
      const int64_t at = tok_first_prefix(m, s + b, e - b);
      if (at >= 0) return emit(at);
    }
    uint32_t i = b, len = 0;
    while (i < e) {
      tok_decode(s + i, &len);
      const int64_t at = tok_first_prefix(m, s + i, len);
      if (!(at >= 0 ? emit(at) : copy(i, i + len))) return false;
      i += len;
    }
    return true;
  };
  TokGb g;
  uint32_t b = 0, i = 0, len = 0;
  while (i < n) {
    const uint32_t cp = tok_decode(s + i, &len);
    if (tok_gb_break(g, tok_gb_props(u, cp))) {
      if (!cluster(b, i)) return false;
      if (b == 0 && w == 0) *lead = false;
      b = i;
    }
    i += len;
  }
  if (n && !cluster(b, n)) return false;
  if (b == 0 && w == 0) *lead = false;
  *out_n = w;
  return true;
}

// char::to_lowercase per character (to_lowercase_per_char): ASCII directly, U+03A3 to U+03C3, else kLower
__device__ bool tok_lower(const TokUtf8Dev &u, const uint8_t *s, uint32_t n, uint8_t *d, uint32_t *out_n, uint32_t cap) {
  uint32_t w = 0, i = 0, len = 0;
  while (i < n) {
    const uint8_t c = s[i];
    if (c < 0x80) {
      if (w >= cap) return false;
      d[w++] = (c >= 'A' && c <= 'Z') ? c + 32 : c;
      ++i;
      continue;
    }
    const uint32_t cp = tok_decode(s + i, &len);
    i += len;
    if (cp == 0x3A3) { if (!tok_encode(0x3C3, d, &w, cap)) return false; continue; }
    uint32_t lo = 0, hi = u.n_lower;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(&u.lower[mid].cp) < cp) lo = mid + 1; else hi = mid; }
    if (lo < u.n_lower && __ldg(&u.lower[lo].cp) == cp) {
      const uint32_t k = __ldg(&u.lower[lo].n);
      for (uint32_t t = 0; t < k; ++t) if (!tok_encode(__ldg(&u.lower[lo].to[t]), d, &w, cap)) return false;
    } else if (!tok_encode(cp, d, &w, cap)) return false;
  }
  *out_n = w;
  return true;
}

// Thread per candidate line: the normaliser's steps in order.  The text is copied into the line's region of norm;
// Lowercase and Precompiled write to the same region of norm2 and the two swap; the result ends in norm.
__global__ void __launch_bounds__(STB_TOK_THREADS)
stb_tok_utf8_normalize_kernel(const uint8_t *text, const uint64_t *off, const uint64_t *roff, const uint8_t *taken,
                              uint64_t m, const TokPlanDev p, const TokUtf8Dev u, uint8_t *norm, uint8_t *norm2,
                              uint32_t *nlen, uint8_t *status) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m || !taken[i]) return;
  const uint64_t b = off[i], base = roff[i] + i * (p.grow + 1);
  const uint32_t cap = (uint32_t)(roff[i + 1] - roff[i]) + p.grow;
  uint32_t n = (uint32_t)(off[i + 1] - b);
  uint8_t *s = norm + base, *d = norm2 + base;
  for (uint32_t k = 0; k < n; ++k) s[k] = text[b + k];
  bool lead = true;                                     // the first byte still comes from original offset 0
  uint8_t st = TOK_GPU;
  for (int o = 0; o < p.n_ops && st == TOK_GPU; ++o) {
    switch (p.kind[o]) {
      case HfTokenizer::OP_LOWER:
      case HfTokenizer::OP_PRECOMPILED: {
        uint32_t w = 0;
        const bool ok = p.kind[o] == HfTokenizer::OP_LOWER ? tok_lower(u, s, n, d, &w, cap)
                                                           : tok_charsmap(u.map[o], u, s, n, d, &w, cap, &lead);
        if (!ok) { st = TOK_OVERFLOW; break; }
        uint8_t *t = s; s = d; d = t;
        n = w;
        break;
      }
      case HfTokenizer::OP_MULTISPACE: {                   // every run of U+0020 -> one space
        uint32_t w = 0, r = 0;
        while (r < n) {
          if (s[r] == ' ') { while (r < n && s[r] == ' ') ++r; s[w++] = ' '; }
          else s[w++] = s[r++];
        }
        n = w;
        break;
      }
      case HfTokenizer::OP_STRIP: {
        uint32_t lo = 0, hi = n, len = 0;
        if (p.left[o]) while (lo < hi && tok_is_space(s + lo, &len)) lo += len;
        if (p.right[o]) {
          while (hi > lo) {                                // step back one character at a time
            uint32_t k = hi - 1;
            while (k > lo && (s[k] & 0xC0) == 0x80) --k;
            if (tok_is_space(s + k, &len) && k + len == hi) hi = k; else break;
          }
        }
        if (lo > 0) lead = false;
        for (uint32_t k = lo; k < hi; ++k) s[k - lo] = s[k];
        n = hi - lo;
        break;
      }
      case HfTokenizer::OP_PREPEND: {
        const uint32_t L = (uint32_t)p.pre_len[o];
        if (n == 0 || L == 0) break;
        if (n + L > cap) { st = TOK_OVERFLOW; break; }
        for (uint32_t k = n; k-- > 0;) s[k + L] = s[k];
        for (uint32_t k = 0; k < L; ++k) s[k] = p.pre[o][k];
        n += L;
        break;
      }
    }
  }
  if (st == TOK_GPU && s != norm + base) for (uint32_t k = 0; k < n; ++k) norm[base + k] = s[k];
  // "first": HF prepends to the split whose original offset is 0; a text that starts with a delimiter gets none
  if (st == TOK_GPU && p.scheme == 1 && !lead && n > 0 && s[0] != ' ') {
    bool rep = n >= (uint32_t)p.rep_len;
    for (int k = 0; rep && k < p.rep_len; ++k) rep = s[k] == p.rep[k];
    if (!rep) st = TOK_FIRST;
  }
  nlen[i] = n;
  status[i] = st;
}

// Thread per candidate line of status 0: encode_raw's Metaspace fast path on UTF-8 -- a space or the replacement
// itself closes the running piece and starts the next one with the replacement; the first piece gets it per
// the prepend scheme ("first": this split starts the line, the normaliser checked its offset).  A piece past
// STB_TOKENIZER_PIECE_CAP gives the line back before any Viterbi runs.
__global__ void __launch_bounds__(STB_TOK_THREADS)
stb_tok_utf8_unigram_kernel(const uint8_t *norm, const uint32_t *nlen, const uint64_t *roff, const uint8_t *taken,
                            uint64_t m, const TokPlanDev p, const TokTrieDev t, uint32_t max_length, uint32_t *tmp,
                            uint32_t *count, uint8_t *status, int *err) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m || !taken[i] || status[i] != TOK_GPU) return;
  const uint64_t base = roff[i] + i * (p.grow + 1);
  const uint32_t region = (uint32_t)(roff[i + 1] - roff[i]) + p.grow + 1, limit = min(region, max_length);
  const uint8_t *s = norm + base;
  const uint32_t n = nlen[i], R = (uint32_t)p.rep_len;
  auto delim = [&](uint32_t q) -> uint32_t {            // bytes of the delimiter at q, or 0
    if (s[q] == ' ') return 1;
    if (q + R > n) return 0;
    for (uint32_t k = 0; k < R; ++k) if (s[q + k] != p.rep[k]) return 0;
    return R;
  };
  // pieces(f): f(rep, run, len) for every piece, in order
  auto pieces = [&](auto &&f) {
    if (n == 0) return;
    uint32_t q = 0, dl = delim(0);
    if (dl == 0) {
      uint32_t e = 0;
      while (e < n && delim(e) == 0) e += tok_utf8_len(s[e]);
      f(p.scheme != 2, s, e);
      q = e;
      dl = q < n ? delim(q) : 0;
    }
    while (q < n) {                                      // a delimiter at q: the next piece
      uint32_t e = q + dl, ndl = 0;
      while (e < n && (ndl = delim(e)) == 0) e += tok_utf8_len(s[e]);
      f(true, s + q + dl, e - q - dl);
      q = e;
      dl = ndl;
    }
  };
  bool fits = true;
  pieces([&](bool rep, const uint8_t *, uint32_t len) { if ((rep ? R : 0) + len > STB_TOKENIZER_PIECE_CAP) fits = false; });
  if (!fits) { status[i] = TOK_PIECE_CAP; return; }
  TokLattice L;
  uint32_t *ids = tmp + base, cnt = 0;
  pieces([&](bool rep, const uint8_t *run, uint32_t len) { tok_piece(p, t, L, rep, run, len, ids, &cnt, limit, err); });
  if (cnt > region && region < max_length) atomicOr(err, 2);
  count[i] = min(cnt, max_length);
}

// the counts of the lines whose ids come from the host CSR (declined or given back)
__global__ void stb_tok_fill_kernel(const uint8_t *gpu, const uint64_t *hoff, uint64_t m, uint32_t *count) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m && !gpu[i]) count[i] = (uint32_t)(hoff[i + 1] - hoff[i]);
}

// ------------------------------------------------------------------------------------------------- host ---
const stb_ctx *stb_tokenizer_ctx(const stb_tokenizer *tok) { return tok->ctx; }

// Well-formed UTF-8: shortest form, no surrogates, nothing above U+10FFFF
static bool utf8_valid(const uint8_t *s, uint64_t n) {
  uint64_t i = 0;
  while (i < n) {
    const uint8_t c = s[i];
    if (c < 0x80) { ++i; continue; }
    uint32_t k;
    uint8_t lo = 0x80, hi = 0xBF;                          // range of the second byte
    if (c >= 0xC2 && c <= 0xDF) k = 1;
    else if (c >= 0xE0 && c <= 0xEF) { k = 2; if (c == 0xE0) lo = 0xA0; if (c == 0xED) hi = 0x9F; }
    else if (c >= 0xF0 && c <= 0xF4) { k = 3; if (c == 0xF0) lo = 0x90; if (c == 0xF4) hi = 0x8F; }
    else return false;
    if (n - i <= k) return false;                          // truncated
    if (s[i + 1] < lo || s[i + 1] > hi) return false;
    for (uint32_t j = 2; j <= k; ++j) if ((s[i + j] & 0xC0) != 0x80) return false;
    i += k + 1;
  }
  return true;
}

// The one rule for which lines go to the GPU (header: stb_tokenizer_gpu_lines).
static bool line_taken(const stb_tokenizer *tok, const uint8_t *s, uint64_t n) {
  const HfTokenizer::AsciiPlan &p = tok->plan;
  if (!p.ok) return false;
  if (tok->utf8) {
    if (!utf8_valid(s, n)) return false;
  } else {
    uint64_t run = 0, longest = 0;
    for (uint64_t k = 0; k < n; ++k) {
      const uint8_t c = s[k];
      if (c < 0x20 || c > 0x7E || !p.byte_ok[c]) return false;
      run = c == ' ' ? 0 : run + 1;
      longest = std::max(longest, run);
    }
    if (p.replacement.size() + p.grow + longest > STB_TOKENIZER_PIECE_CAP) return false;
    if (p.decline_leading_space && n && s[0] == ' ') return false;
  }
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

// bytes of a taken line's region per text byte: 1 (printable ASCII), STB_TOK_UTF8_R (UTF-8)
static uint64_t region_factor(const stb_tokenizer *tok) { return tok->utf8 ? STB_TOK_UTF8_R : 1; }

// ids of chunk [l0, l0 + m), at most: a taken line's region (capped at max_length), a declined line's host ids
// (a UTF-8 chunk's given-back lines are added once they are known: tok_chunk_utf8)
static uint64_t chunk_ids_bound(const stb_tokenizer *tok, const StbTextHost &h, const uint64_t *offsets, uint64_t l0,
                                uint64_t m, uint32_t max_length) {
  uint64_t bound = 0;
  const uint64_t r = region_factor(tok);
  for (uint64_t i = l0; i < l0 + m; ++i)
    bound += h.taken[i] ? std::min<uint64_t>(max_length, r * (offsets[i + 1] - offsets[i]) + tok->dplan.grow + 1) : h.hoff[i + 1] - h.hoff[i];
  return bound;
}

int stb_tok_reserve(stb_ctx *ctx, const stb_tokenizer *tok, const StbTextHost &h, const uint64_t *offsets, uint32_t max_length) {
  uint64_t bytes = 1, lines = 1, hids = 1, region = 1, ids = 1;
  for (size_t c = 0; c + 1 < h.chunk_at.size(); ++c) {
    const uint64_t l0 = h.chunk_at[c], m = h.chunk_at[c + 1] - l0, b = offsets[l0 + m] - offsets[l0];
    bytes = std::max(bytes, b);
    lines = std::max(lines, m);
    hids = std::max(hids, h.hoff[l0 + m] - h.hoff[l0]);
    region = std::max(region, region_factor(tok) * b + m * (tok->dplan.grow + 1));
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
  if (tok->utf8 && ((rc = ctx->tok_norm2.reserve(region, 1 << 20)) != STB_OK || (rc = ctx->tok_roff.reserve(lines + 1, 4096)) != STB_OK ||
                    (rc = ctx->tok_status.reserve(lines, 4096)) != STB_OK))
    return rc;
  return STB_OK;
}

// HfTokenizer::encode of each listed line on host threads, truncated to max_length: ids[k] for lines[k]
static int encode_on_host(const stb_tokenizer *tok, const uint8_t *text, const uint64_t *offsets,
                          const std::vector<uint64_t> &lines, uint32_t max_length, std::vector<std::vector<uint32_t>> &ids) {
  ids.assign(lines.size(), {});
  unsigned threads = std::max(1u, std::thread::hardware_concurrency());
  threads = (unsigned)std::min<uint64_t>(threads, std::max<uint64_t>(1, lines.size() / 16));
  std::vector<std::string> fail(threads);
  auto work = [&](unsigned w) {
    try {
      for (uint64_t k = lines.size() * w / threads; k < lines.size() * (w + 1) / threads; ++k) {
        const uint64_t i = lines[k];
        ids[k] = tok->hf->encode(std::string(reinterpret_cast<const char *>(text + offsets[i]), offsets[i + 1] - offsets[i]));
        if (ids[k].size() > max_length) ids[k].resize(max_length);
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
  return STB_OK;
}

// One chunk through a UTF-8 handle: normalise and run the Viterbi on the candidates, read their status bytes,
// encode the given-back lines on the host, then upload the chunk's host CSR and compact as the ASCII flow does.
// h.taken[l] becomes 1 only for the lines whose ids came from the GPU.
static int tok_chunk_utf8(stb_ctx *ctx, const stb_tokenizer *tok, StbTextHost &h, const uint8_t *text,
                          const uint64_t *offsets, uint64_t l0, uint64_t m, uint32_t max_length) {
  const uint64_t b0 = offsets[l0], bytes = offsets[l0 + m] - b0;
  const uint32_t grow = tok->dplan.grow;
  std::vector<uint64_t> off(m + 1), roff(m + 1);
  for (uint64_t i = 0; i <= m; ++i) { off[i] = offsets[l0 + i] - b0; roff[i] = STB_TOK_UTF8_R * off[i]; }
  cudaStream_t st = ctx->stream;
  uint8_t *taken = h.taken.data() + l0;
  const bool any = std::find(taken, taken + m, 1) != taken + m;
  const unsigned blocks = (unsigned)((m + STB_TOK_THREADS - 1) / STB_TOK_THREADS);
  std::vector<uint8_t> status(m, TOK_GPU);
  if (any) {
    if (bytes) STB_CUDA(cudaMemcpyAsync(ctx->tok_text, text + b0, bytes, cudaMemcpyHostToDevice, st));
    STB_CUDA(cudaMemcpyAsync(ctx->tok_off, off.data(), (m + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
    STB_CUDA(cudaMemcpyAsync(ctx->tok_roff, roff.data(), (m + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
    STB_CUDA(cudaMemcpyAsync(ctx->tok_taken, taken, m, cudaMemcpyHostToDevice, st));
    stb_tok_utf8_normalize_kernel<<<blocks, STB_TOK_THREADS, 0, st>>>(ctx->tok_text, ctx->tok_off, ctx->tok_roff, ctx->tok_taken, m,
                                                                      tok->dplan, tok->dutf8, ctx->tok_norm, ctx->tok_norm2,
                                                                      ctx->tok_nlen, ctx->tok_status);
    STB_CUDA(cudaGetLastError());
    stb_tok_utf8_unigram_kernel<<<blocks, STB_TOK_THREADS, 0, st>>>(ctx->tok_norm, ctx->tok_nlen, ctx->tok_roff, ctx->tok_taken, m,
                                                                    tok->dplan, tok->dtrie, max_length, ctx->tok_tmp, ctx->tok_cnt,
                                                                    ctx->tok_status, ctx->tok_flag);
    STB_CUDA(cudaGetLastError());
    STB_CUDA(cudaMemcpyAsync(status.data(), ctx->tok_status, m, cudaMemcpyDeviceToHost, st));
    STB_CUDA(cudaStreamSynchronize(st));
    ctx->kernel_launches += 2;
  }
  // the give-back: candidates the kernels could not finish exactly
  std::vector<uint64_t> back;
  for (uint64_t i = 0; i < m; ++i)
    if (taken[i] && status[i] != TOK_GPU) { back.push_back(l0 + i); taken[i] = 0; }
  std::vector<std::vector<uint32_t>> back_ids;
  int rc;
  if (!back.empty() && (rc = encode_on_host(tok, text, offsets, back, max_length, back_ids)) != STB_OK) return rc;
  // the chunk's host CSR: declined lines from h, given-back lines from back_ids
  std::vector<uint64_t> hoff(m + 1, 0);
  std::vector<uint32_t> hids;
  uint64_t ids_bound = 0;
  for (uint64_t i = 0, k = 0; i < m; ++i) {
    if (k < back.size() && back[k] == l0 + i) {
      hids.insert(hids.end(), back_ids[k].begin(), back_ids[k].end());
      ++k;
    } else if (!taken[i]) hids.insert(hids.end(), h.hids.begin() + h.hoff[l0 + i], h.hids.begin() + h.hoff[l0 + i + 1]);
    else ids_bound += std::min<uint64_t>(max_length, roff[i + 1] - roff[i] + grow + 1);
    hoff[i + 1] = hids.size();
  }
  ids_bound += hids.size();
  // growing frees buffers the previous chunk's kernels may still read: only on an idle stream
  if (hids.size() > ctx->tok_hids.cap || ids_bound > ctx->embed_ids_dev.cap) STB_CUDA(cudaStreamSynchronize(st));
  if ((rc = ctx->tok_hids.reserve(std::max<size_t>(hids.size(), 1), 4096)) != STB_OK ||
      (rc = ctx->embed_ids_dev.reserve(std::max<uint64_t>(ids_bound, 1), 65536)) != STB_OK)
    return rc;
  STB_CUDA(cudaMemcpyAsync(ctx->tok_hoff, hoff.data(), (m + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  if (!hids.empty()) STB_CUDA(cudaMemcpyAsync(ctx->tok_hids, hids.data(), hids.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  if (!back.empty() || !any) STB_CUDA(cudaMemcpyAsync(ctx->tok_taken, taken, m, cudaMemcpyHostToDevice, st));
  if (!any) STB_CUDA(cudaMemcpyAsync(ctx->tok_roff, roff.data(), (m + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  stb_tok_fill_kernel<<<blocks, STB_TOK_THREADS, 0, st>>>(ctx->tok_taken, ctx->tok_hoff, m, ctx->tok_cnt);
  STB_CUDA(cudaGetLastError());
  stb_tok_scan_kernel<<<1, 1024, 0, st>>>(ctx->tok_cnt, m, ctx->embed_off_dev);
  STB_CUDA(cudaGetLastError());
  stb_tok_write_kernel<<<(unsigned)((m * 32 + 255) / 256), 256, 0, st>>>(ctx->embed_off_dev, ctx->tok_cnt, ctx->tok_taken,
                                                                         ctx->tok_tmp, ctx->tok_roff, grow, ctx->tok_hoff,
                                                                         ctx->tok_hids, m, ctx->embed_ids_dev);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches += 3;
  return STB_OK;
}

int stb_tok_chunk(stb_ctx *ctx, const stb_tokenizer *tok, StbTextHost &h, const uint8_t *text,
                  const uint64_t *offsets, uint64_t l0, uint64_t m, uint32_t max_length) {
  if (tok->utf8) return tok_chunk_utf8(ctx, tok, h, text, offsets, l0, m, max_length);
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

// A UTF-8 handle's normaliser tables in HBM, built from the host tokenizer's own arrays (utf8_view)
static int upload_utf8_tables(stb_tokenizer *t, const std::vector<HfTokenizer::Utf8Op> &ops) {
  const HfTokenizer::Utf8View v = t->hf->utf8_view();
  size_t n_trie = 0, n_norm = 0;
  for (const auto &m : v.maps) { n_trie += m.n_trie; n_norm += m.n_normalized; }
  const size_t n_ranges = v.n_gcb + v.n_ext_pict + v.n_incb;
  int rc;
  if ((rc = t->cm_trie.alloc(std::max<size_t>(n_trie, 1))) != STB_OK || (rc = t->cm_norm.alloc(std::max<size_t>(n_norm, 1))) != STB_OK ||
      (rc = t->gb_bmp.alloc(0x10000)) != STB_OK || (rc = t->gb_ranges.alloc(n_ranges)) != STB_OK ||
      (rc = t->lower.alloc(v.n_lower)) != STB_OK)
    return rc;
  std::vector<size_t> trie_at, norm_at;
  size_t ta = 0, na = 0;
  cudaError_t e = cudaSuccess;
  for (const auto &m : v.maps) {
    trie_at.push_back(ta); norm_at.push_back(na);
    if (e == cudaSuccess && m.n_trie) e = cudaMemcpy(t->cm_trie.p + ta, m.trie, m.n_trie * sizeof(uint32_t), cudaMemcpyHostToDevice);
    if (e == cudaSuccess && m.n_normalized) e = cudaMemcpy(t->cm_norm.p + na, m.normalized, m.n_normalized, cudaMemcpyHostToDevice);
    ta += m.n_trie; na += m.n_normalized;
  }
  if (e == cudaSuccess) e = cudaMemcpy(t->gb_bmp, v.gb_bmp, 0x10000, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(t->gb_ranges, v.gcb, v.n_gcb * sizeof(HfTokenizer::PropRange), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(t->gb_ranges.p + v.n_gcb, v.ext_pict, v.n_ext_pict * sizeof(HfTokenizer::PropRange), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(t->gb_ranges.p + v.n_gcb + v.n_ext_pict, v.incb, v.n_incb * sizeof(HfTokenizer::PropRange), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(t->lower, v.lower, v.n_lower * sizeof(LowerEntry), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) { stb_set_error("tokenizer_load: upload failed: %s", cudaGetErrorString(e)); return STB_ERR_CUDA; }
  TokUtf8Dev &u = t->dutf8;
  for (size_t o = 0; o < ops.size(); ++o) {
    if (ops[o].kind != HfTokenizer::OP_PRECOMPILED) continue;
    const auto &m = v.maps[ops[o].map];
    TokMapDev &d = u.map[o];
    d.trie = t->cm_trie.p + trie_at[ops[o].map];
    d.norm = t->cm_norm.p + norm_at[ops[o].map];
    d.n_trie = (uint32_t)m.n_trie;
    d.n_norm = (uint32_t)m.n_normalized;
    for (int c = 0x20; c < 0x7F; ++c) if (m.ascii_plain[c]) d.ascii_plain[c >> 5] |= 1u << (c & 31);
  }
  u.gb_bmp = t->gb_bmp;
  u.gcb = t->gb_ranges; u.n_gcb = (uint32_t)v.n_gcb;
  u.ext_pict = t->gb_ranges.p + v.n_gcb; u.n_ext_pict = (uint32_t)v.n_ext_pict;
  u.incb = t->gb_ranges.p + v.n_gcb + v.n_ext_pict; u.n_incb = (uint32_t)v.n_incb;
  u.lower = t->lower; u.n_lower = (uint32_t)v.n_lower;
  return STB_OK;
}

extern "C" {

int stb_tokenizer_load_ex(stb_ctx *ctx, const uint8_t *json, uint64_t len, uint32_t flags, stb_tokenizer **out) {
  int rc = stb_ctx_use(ctx);
  if (rc) return rc;
  if (!out || (!json && len)) { stb_set_error("tokenizer_load: null argument"); return STB_ERR_ARG; }
  *out = nullptr;
  if (flags & ~STB_TOKENIZER_UTF8) { stb_set_error("tokenizer_load: unknown flags 0x%x", flags); return STB_ERR_ARG; }
  std::unique_ptr<stb_tokenizer> t(new (std::nothrow) stb_tokenizer());
  if (!t) { stb_set_error("out of host memory"); return STB_ERR_NOMEM; }
  t->ctx = ctx;
  t->utf8 = (flags & STB_TOKENIZER_UTF8) != 0;
  try {
    t->hf = HfTokenizer::from_json(std::string(reinterpret_cast<const char *>(json), len));
    t->plan = t->hf->ascii_plan();
  } catch (const std::exception &e) {
    stb_set_error("tokenizer_load: %s", e.what());
    return STB_ERR_ARG;
  }
  HfTokenizer::AsciiPlan &p = t->plan;
  // a UTF-8 handle runs every normaliser step, Precompiled included; a flags-0 handle the printable-ASCII ones
  std::vector<HfTokenizer::Utf8Op> ops;
  if (t->utf8 && p.ok) ops = t->hf->utf8_view().ops;
  else for (const auto &op : p.ops) ops.push_back({op.kind, op.left, op.right, op.text});
  if (ops.size() > STB_TOK_MAX_OPS) p.ok = false;
  for (const auto &op : ops) if (op.text.size() > STB_TOK_MAX_PREPEND) p.ok = false;
  TokPlanDev &d = t->dplan;
  if (p.ok) {
    d.n_ops = (int)ops.size();
    for (int o = 0; o < d.n_ops; ++o) {
      d.kind[o] = ops[o].kind; d.left[o] = ops[o].left; d.right[o] = ops[o].right;
      d.pre_len[o] = (int)ops[o].text.size();
      memcpy(d.pre[o], ops[o].text.data(), ops[o].text.size());
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
  if (t->utf8 && p.ok && (rc = upload_utf8_tables(t.get(), ops)) != STB_OK) return rc;
  if ((rc = ctx->tok_flag.reserve(1)) != STB_OK) return rc;
  *out = t.release();
  return STB_OK;
}

int stb_tokenizer_load(stb_ctx *ctx, const uint8_t *json, uint64_t len, stb_tokenizer **out) {
  return stb_tokenizer_load_ex(ctx, json, len, 0, out);
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
  if (taken) memcpy(taken, h.taken.data(), n_lines);         // after the chunks: a UTF-8 handle's give-back clears lines
  int flag = 0;
  STB_CUDA(cudaMemcpy(&flag, ctx->tok_flag, sizeof(int), cudaMemcpyDeviceToHost));
  if (flag) { stb_set_error("debug_tokenize: a GPU piece overflowed its bound (flag %d)", flag); return STB_ERR_STATE; }
  if (!fits) { stb_set_error("debug_tokenize: %llu ids do not fit ids_cap", (unsigned long long)ids_offsets[n_lines]); return STB_ERR_CAPACITY; }
  return STB_OK;
}

}  // extern "C"

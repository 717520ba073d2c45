// Internal declarations shared by the translation units of libsemtools_b200.so.
// Everything here is sm_90a-only product code; nothing in this directory may
// include, link or call anything under oracle/.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <vector>

#include "../../include/semtools_b200.h"

#define STB_D 256           // floats per row
#define STB_ROW_F4 64       // float4 per row
#define STB_SCAN_THREADS 256
#define STB_SCAN_MINB 2     // CTAs per SM the scan kernels are register-budgeted for
#define STB_SCAN_WARPS (STB_SCAN_THREADS / 32)
#define STB_SORT_CAP 1024   // keys one CTA sorts in shared memory
// Rigorous bound (with ~4x slack) on |approx cosine - exact cosine| for the fp32
// scan arithmetic on rows whose squared norm is a normal fp32 number; derivation
// in DESIGN.md "Candidate completeness".  Rows outside that range are forced
// into the candidate set instead of being scored.
#define STB_SCORE_EPS 1.0e-5
// Element type of the 16-bit L2-normalised corpus shadow (K2 operand; K1's opt-in half-width
// scan): fp16 by default (same wgmma rate as bf16, 8x smaller rounding bound for unit
// rows; validated on hardware in round 2), bf16 with -DSTB_SHADOW_F16=0.
#ifndef STB_SHADOW_F16
#define STB_SHADOW_F16 1
#endif
// |q^ . shadow(x) - exact cosine| when only the ROW is rounded (K1 shadow scan: the query stays
// f32): <= u * ||q^|| * ||x^|| = u (unit roundoff: 2^-8 bf16, 2^-11 fp16; fp16 components below 2^-14 add
// <= 16 * 2^-25 * ||q^||_1 <= 8e-6), plus f32 accumulation and rsqrt (< 2e-5).
#if STB_SHADOW_F16
#define STB_SHADOW_SCAN_EPS 0.00052
#else
#define STB_SHADOW_SCAN_EPS 0.0040
#endif
// K1 candidate tiers (which copy of the corpus the streaming pass reads; the exact f64 re-rank
// and the completeness proof are common to all): f32 rows (1 KiB/row), 16-bit normalised shadow
// (512 B/row, also K2's operand), int8 codes + per-row scale (260 B/row).
#define STB_TIER_F32 0
#define STB_TIER_H16 1
#define STB_TIER_Q8 2
// q8 scores are upper bounds of the exact cosine up to the fp32 evaluation of the bound itself
// and of the two normalisations (< 4e-6, scan_topk.cu: stb_scan_q8); proof slack:
#define STB_Q8_SCAN_EPS 2.0e-5
// the q8 tier always keeps K' = 128 candidates; beyond this top_k the gap between the k-th and
// the 128th best is too small for its ~0.01 per-row error term to prove anything
#define STB_Q8_MAX_K 16
// the q8 tier's top-k scan skips a row whose 4-bit upper bound u4 (>= c - 1e-5) is below the proven
// threshold T (<= c_k - 1e-5) by more than this: then c < c_k strictly (scan_topk.cu: stb_scan_q4)
#define STB_Q4_SKIP_EPS 2.0e-5
#define STB_Q4_WORDS 16     // threshold words per launch slot (>= STB_Q8_MAX_K)

void stb_set_error(const char *fmt, ...);

#define STB_CUDA(call)                                                             \
  do {                                                                             \
    cudaError_t _e = (call);                                                       \
    if (_e != cudaSuccess) {                                                       \
      stb_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call,                  \
                    cudaGetErrorString(_e));                                       \
      return STB_ERR_CUDA;                                                         \
    }                                                                              \
  } while (0)

// The one owner of every device (cudaMalloc) and page-locked host (cudaMallocHost) buffer of the library: cap
// elements of T at p, freed by the destructor.  It converts to T *, so launches, copies and indexing read it as
// the pointer.  alloc(n) frees what it holds, then allocates exactly n elements.  reserve(need, floor) keeps
// the buffer if it holds need elements, else allocates max(need, floor, 1.5 cap) and only then frees the old
// one.  Neither keeps the contents.  A failed allocation returns STB_ERR_NOMEM with the byte count in the
// error message and leaves the buffer as it was (after alloc's free: empty).  Freeing an old buffer that a
// kernel may still read is the caller's to order (stream synchronise).
template <class T, bool PINNED = false>
struct StbBuf {
  T *p = nullptr;
  size_t cap = 0;
  StbBuf() = default;
  StbBuf(const StbBuf &) = delete;
  StbBuf &operator=(const StbBuf &) = delete;
  StbBuf(StbBuf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  StbBuf &operator=(StbBuf &&o) noexcept {
    if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
    return *this;
  }
  ~StbBuf() { release(); }
  operator T *() const { return p; }
  int alloc(size_t n) {
    release();
    return take(n);
  }
  int reserve(size_t need, size_t floor = 0) {
    if (need <= cap && p) return STB_OK;
    size_t n = need > floor ? need : floor;
    if (cap + cap / 2 > n) n = cap + cap / 2;
    return take(n);
  }

 private:
  int take(size_t n) {
    void *np = nullptr;
    const cudaError_t e = PINNED ? cudaMallocHost(&np, n * sizeof(T)) : cudaMalloc(&np, n * sizeof(T));
    if (e != cudaSuccess) {
      cudaGetLastError();
      stb_set_error("%s(%zu bytes) failed: %s", PINNED ? "cudaMallocHost" : "cudaMalloc", n * sizeof(T), cudaGetErrorString(e));
      return STB_ERR_NOMEM;
    }
    release();
    p = static_cast<T *>(np);
    cap = n;
    return STB_OK;
  }
  void release() {
    if (p) {
      if (PINNED) cudaFreeHost(p); else cudaFree(p);
      cudaGetLastError();
    }
    p = nullptr;
    cap = 0;
  }
};
template <class T> using StbPinned = StbBuf<T, true>;

struct stb_ctx {
  int device;
  int sm_count;
  cudaStream_t stream;
  bool own_stream;
  // --- scan scratch (device) ---
  StbBuf<uint64_t> block_keys;     // candidate keys of every tree level
  StbBuf<unsigned int> counters;   // tree arrival counters (zeroed; kernels re-zero)
  // K1 tile-ticket counters (monotonic; scan_topk.cu: stb_for_each_tile).  A ring of STB_TICKET_SLOTS
  // counters, one per launch in turn: with the overlapped launch mode two consecutive scans run
  // concurrently and must not draw from the same counter.
  StbBuf<unsigned long long> tickets;
  unsigned long long ticket_next[8];   // per slot: its value when the next launch using it starts
  unsigned long long topk_launches;    // picks the slot
  bool ticket_ring;                    // set by the first overlapped launch; until then every launch uses slot 0
  // K1 co-scan (scan_topk.cu: stb_coscan_offset): per ticket slot, the tile offset its last co-scan launch
  // chose, as a tagged word (tag << 32 | offset, the tag is the launch count); the host's copy of the tags
  // (0: the slot's last launch did not co-scan) and the last co-scan launch, which the next one may follow
  StbBuf<unsigned long long> coscan_off;
  uint32_t coscan_tag[8];
  struct {
    const void *rows;                  // the scanned corpus's f32 rows; null: no launch to follow
    int src;
    uint64_t n_virtual, tiles, t_bulk;
    unsigned long long t_base;
    int slot;
    uint32_t tag;
  } coscan_prev;
  // q8 tier prefilter (scan_topk.cu: stb_scan_q4): STB_TICKET_SLOTS x STB_Q4_WORDS tagged threshold words,
  // one slot per launch in turn; the launch count is the tag
  StbBuf<unsigned long long> q4_thr;
  unsigned long long q4_launches;
  StbBuf<unsigned long long> q4_refined;   // rows the prefilter passed on to the int8 codes (stb_debug_q4_refined)
  StbBuf<float> q_dev;             // 256 f32 staging for host queries
  StbBuf<stb_hit> hits_dev;        // result hits (top-k path)
  StbBuf<uint32_t> status_dev;     // [0]=n hits, [1]=complete flag, [2..] debug
  StbBuf<uint32_t> collect_rows;   // threshold/fallback compaction: local row ids
  StbBuf<unsigned long long> collect_count;
  StbBuf<stb_hit> collect_hits;    // exact hits of collected rows (sorted in place)
  StbBuf<uint64_t> ranges_dev;     // [3 * n] : begin(local), end(local), vstart
  StbBuf<int> err_flag;            // device int: scratch flag of the copy builders, stb_embed and K2's query shadow; zeroed before each use
  StbBuf<unsigned int> hist_dev;   // 4096-bin score histogram (large-k path)
  // cudaFuncSetAttribute is per DEVICE: remembered per context, never in function statics
  // (one process may hold contexts on several GPUs)
  uint32_t func_attr_mask;
  size_t finish2_smem_set;
  // --- K2 scratch ---
  StbBuf<uint8_t> bq_tiles;     // query shadow tiles
  StbBuf<float> b_submax;       // [n_sub][q_pad]
  StbBuf<float> b_tilemax;     // [n_tiles][q_pad]
  StbBuf<uint64_t> b_cand;        // [q_pad][slices][32]
  StbBuf<float> b_thr;             // v2: [q_pad] emission thresholds
  StbBuf<uint32_t> b_cnt;          // v2: [q_pad] emitted-candidate counters
  StbBuf<uint64_t> b_keys;        // v2: [q_pad][cand_cap] emitted keys
  StbBuf<uint32_t> b_qbad;        // [q_pad] 1: query could not be normalised
  StbBuf<float4> b_q8c;          // route 7: [q_pad] {1/S, h_l1, e_q, S} of each query's q16
  // stb_search_batch_filtered: the clipped ranges (local [begin, end) u32 pairs), the listed tiles and the
  // eligible-row bitmap (8 words per shadow tile), all built from the same clipped ranges
  StbBuf<uint32_t> b_franges;
  StbBuf<uint32_t> b_ftiles;
  StbBuf<uint32_t> b_fbits;
  // stb_search_batch_subsets (route 6; b_franges / b_fbits hold every tensor group's ranges / bitmap): both
  // passes' work lists and the slots' rows in one upload, the queries in slot order, the bad flags per
  // compact row, and (host, malloc) each caller query's slot and compact row for stb_debug_batch_last
  StbBuf<uint32_t> s_work;
  StbBuf<float> s_qslots;
  StbBuf<uint32_t> s_qbad;
  std::vector<uint32_t> s_map;
  // stb_search_batch_threshold (per chunk of queries): per-(query, segment) destinations of the first pass's
  // keys, the re-emission's segment offsets, cursors, queries and thresholds, the compact candidates and their
  // sort buffers (4 x u64 per candidate), per-slot offsets / query / pass count / output position, the hits
  // in output order and the sorts' scratch
  StbBuf<uint64_t> t_dst;
  StbBuf<uint64_t> t_segoff;
  StbBuf<uint32_t> t_cur;
  StbBuf<float> t_rq;
  StbBuf<float> t_rthr;
  StbBuf<uint64_t> t_buf;
  StbBuf<int> t_off;
  StbBuf<uint32_t> t_slot;       // [2][slots]: query of each slot, then its pass count
  StbBuf<uint64_t> t_out_at;
  StbBuf<stb_hit> t_hits;
  StbBuf<uint8_t> t_sort_tmp;
  uint32_t b_last[6];             // the last K2 call's route record (api.cu: k2_record)
  StbBuf<float> bq_dev;           // host-call staging: queries
  StbBuf<stb_hit> bh_dev;         // host-call staging: hits
  StbBuf<uint32_t> bs_dev;        // host-call staging: status
  StbBuf<uint64_t> embed_off_dev;  // K3 staging: CSR offsets
  StbBuf<uint32_t> embed_ids_dev;  // K3 staging: token ids
  StbBuf<float> embed_out_dev;     // K3 output when not appending to a corpus
  // in-place corpus mutations (stb_corpus_update / _remove): row staging (<= STB_MUT_CHUNK_ROWS rows),
  // row ids or kept-segment table, and the q8 / shadow bad-row flags
  StbBuf<float> mut_stage;
  StbBuf<uint64_t> mut_idx;
  StbBuf<int> mut_flags;
  // --- pinned host staging ---
  StbPinned<float> q_pin;
  StbPinned<stb_hit> hits_pin;
  StbPinned<uint32_t> status_pin;
  StbPinned<float> many_q_pin;          // stb_search_many: queries / per-query status (kernels write the latter directly)
  StbPinned<uint32_t> many_status_pin;
  // --- counters ---
  uint64_t kernel_launches;
  uint64_t fallback_searches;
  // --- K3 ---
  StbBuf<int> embed_flag;          // device int: K3's sticky range flag; set only by stb_embed_dev, cleared only by stb_embed_status
};

#define STB_TICKET_SLOTS 8
// Spin-wait bound of the peer-memory exchanges (SM cycles, ~15 s): long enough that ranks entering a sharded
// search a few seconds apart (first-call allocations, a busy host) still meet; a peer that is really gone
// costs one bound, the call reports it (status 0xfffffffe / 2) and the caller must stop using the exchange:
// ranks that disagree on whether an exchange happened no longer issue the same sequence of calls.
#define STB_XCHG_TIMEOUT_CYCLES 30000000000ll
#define STB_XCHG_SLOTS 4
#define STB_XCHG_MAX_WORLD 8
struct StbXchgArgs {
  unsigned char *base[STB_XCHG_MAX_WORLD];   // exchange buffer of every rank (peer-mapped)
  uint32_t world, rank, max_k, slot;
  unsigned long long seq;
};

struct stb_xchg {
  stb_ctx *ctx;
  uint32_t world, rank, max_k;
  StbBuf<unsigned char> local;               // this rank's buffer (plain device memory, which IPC requires)
  size_t bytes;
  unsigned char *peers[STB_XCHG_MAX_WORLD];  // peers[rank] == local
  bool ipc_opened[STB_XCHG_MAX_WORLD];
  bool connected;
  unsigned long long seq;
  // batch area (stb_xchg_create_batch; sharded K2): 2 slots x { flags[world] u64 | status[world][max_nq] u32 |
  // hits[world][max_nq][max_k] } behind the single-query area
  uint32_t max_nq;
  size_t batch_off, batch_slot_bytes;
  unsigned long long batch_seq;
  StbBuf<unsigned int> batch_ticket;         // device: arrival counter of the push kernel
  bool dead;                                 // a synchronous call saw a peer time-out: every later call is refused
};

struct stb_table {
  stb_ctx *ctx;
  StbBuf<float> E;            // V x 256
  uint64_t V;
  StbBuf<float> weights;      // or empty
  uint64_t n_weights;
  StbBuf<uint32_t> mapping;   // or empty
  uint64_t n_mapping;
  int normalize;
};

struct stb_corpus {
  stb_ctx *ctx;
  float *rows;         // capacity x 256: dev_rows, or on a host-rows corpus the device address of rows_host
  StbBuf<float> dev_rows;   // a device corpus's rows
  // stb_corpus_create_host: the rows live in page-locked, device-mapped host memory (kernels read them over
  // the host link through `rows`) and the q8 copy is kept current by every call that writes rows
  float *rows_host;    // null on a device corpus
  int host_rows;
  uint64_t n;
  uint64_t capacity;
  uint64_t row_base;
  uint64_t epoch;            // bumped by every change that is not an append (an IVF-PQ index refuses to extend over it)
  // K2: L2-normalised bf16 copy in wgmma tile layout (built lazily, rebuilt when n changes)
  StbBuf<uint8_t> shadow;    // whole 256-row tiles of 128 KiB
  uint64_t shadow_rows;      // rows covered by `shadow` (== n when valid)
  int shadow_bad;            // 1: some row cannot be normalised in fp32 -> tensor path refused
  // K1 tier q8: int8 codes [capacity][256] + per-row scale, built lazily / by stb_corpus_prepare
  // (q8_scale.cap: the rows all four hold)
  StbBuf<uint8_t> q8;
  StbBuf<float> q8_scale;
  StbBuf<uint8_t> q4;        // ... its nibble plane [capacity][128] and per-row {s, rho} (top-k prefilter)
  StbBuf<float2> q4_sr;
  uint64_t q8_rows;          // rows covered (== n when valid; also the plane's)
  int q8_bad;
  // per-tier bookkeeping: a reduced-width tier is skipped once it proves fewer than half of its
  // results on this corpus (index = STB_TIER_*)
  uint32_t tier_tries[3], tier_proven[3];
  uint32_t searches_since_change;   // lazy builds wait for the second query on an unchanged corpus
  uint32_t ivfpq_live;       // IVF-PQ indexes built on this corpus and not yet destroyed: update / remove refuse
};

// Row ranges as stb_search takes them: n half-open [begin, end) pairs, ascending and disjoint (api.cu).
bool stb_ranges_ordered(const uint64_t *ranges, uint32_t n);

// Validates such ranges (global rows) and clips them to a shard's rows [row_base, row_base + n_rows):
// emit(begin, end) receives each non-empty piece in local rows, in order.  STB_ERR_RANGE, with `what`
// leading the message, when the ranges are not ascending and disjoint.
template <class Emit>
int stb_clip_ranges(const char *what, const uint64_t *ranges, uint32_t n, uint64_t row_base, uint64_t n_rows, Emit &&emit) {
  if (!stb_ranges_ordered(ranges, n)) { stb_set_error("%s: row_ranges must be ascending, disjoint, half-open", what); return STB_ERR_RANGE; }
  const uint64_t hi = row_base + n_rows;
  for (uint32_t i = 0; i < n; ++i) {
    const uint64_t b = ranges[2 * i] > row_base ? ranges[2 * i] : row_base;
    const uint64_t e = ranges[2 * i + 1] < hi ? ranges[2 * i + 1] : hi;
    if (b < e) emit(b - row_base, e - row_base);
  }
  return STB_OK;
}

// stb_clip_ranges appending each local piece to *loc as a [begin, end) u32 pair (a shard holds < 2^32 rows).
inline int stb_clip_ranges_u32(const char *what, const uint64_t *ranges, uint32_t n, uint64_t row_base, uint64_t n_rows,
                               std::vector<uint32_t> *loc) {
  loc->reserve(loc->size() + 2 * (size_t)n);
  return stb_clip_ranges(what, ranges, n, row_base, n_rows,
                         [&](uint64_t b, uint64_t e) { loc->push_back((uint32_t)b); loc->push_back((uint32_t)e); });
}

// hits[n, k) = (+inf, UINT64_MAX): the unused tail of a top-k result, as the kernels pad it.
inline void stb_pad_hits(stb_hit *hits, uint64_t n, uint64_t k) {
  for (uint64_t j = n; j < k; ++j) { hits[j].distance = INFINITY; hits[j].row = UINT64_MAX; }
}

// stb_corpus_update / stb_corpus_remove without their refusal of live IVF-PQ indexes (api.cu).  With a
// hook, an index that follows the change (stb_ivfpq_update / stb_ivfpq_remove) acts at the points where it
// must, all before the first row is written:
//   check()   in place of that refusal, after the null-argument checks;
//   begin()   once the arguments are validated and the corpus's staging buffers are reserved;
//   staged()  update only: rows [i0, i0 + m) of the call, uploaded to the staging buffer, for every chunk
//             that holds one of the call's first `staged_rows` rows (set by begin());
//   ready()   last chance to refuse.
// A non-zero return ends the call with that status and nothing written.
struct StbCorpusHook {
  uint64_t staged_rows = 0;
  virtual int check() = 0;
  virtual int begin() { return STB_OK; }
  virtual int staged(const float *stage_dev, uint64_t i0, uint64_t m) { (void)stage_dev; (void)i0; (void)m; return STB_OK; }
  virtual int ready() { return STB_OK; }
  virtual ~StbCorpusHook() {}
};
int stb_corpus_update_impl(stb_corpus *c, const uint64_t *idx, const float *rows, uint64_t n, const char *what,
                           StbCorpusHook *hook);
int stb_corpus_remove_impl(stb_corpus *c, const uint64_t *ranges, uint32_t n_ranges, const char *what,
                           StbCorpusHook *hook);

// ---- corpus_update.cu -----------------------------------------------------------------------
#define STB_MUT_CHUNK_ROWS 262144   // staging rows of an update / removal chunk: 256 MiB of f32 at most
struct StbCorpusWriteArgs {
  float4 *rows;
  const float4 *stage;        // m staged rows
  const uint64_t *idx;        // local destination of staged row i, or null: first + i
  uint64_t first, m;
  uint8_t *q8; float *q8_scale; uint8_t *q4; float2 *q4_sr;
  uint64_t q8_rows;           // rows the q8 copy covers (0: none)
  uint8_t *shadow;
  uint64_t shadow_rows;       // rows the 16-bit shadow covers (0: none)
  int *flags;                 // [0] a written q8 row cannot be normalised, [1] the same for the shadow
};
int stb_launch_corpus_write(stb_ctx *ctx, const StbCorpusWriteArgs &a);
// staging row i <- the row that lands at local row first + i once the removed rows are gone
int stb_launch_corpus_gather(stb_ctx *ctx, const float *rows, const uint64_t *seg_dev, uint32_t n_seg, uint64_t first,
                             uint64_t m, float *stage);

// ---- scan_topk.cu -------------------------------------------------------------
// Fast path: one kernel = scan + per-warp running top-K' + CTA/tree merge +
// exact f64 re-rank + completeness check.  q_dev: 256 f32 on device.
// n_ranges > 0: ranges_dev holds local [begin,end,vstart] triples.
// tier: STB_TIER_* -- which copy of `c` the streaming pass reads (must exist and be current).
// overlapped: the launch is one of a pipelined single-GPU series (stb_search_topk_dev, stb_search_many
// without an exchange) and takes no exchange or ranges: the grid is sized for ONE CTA per SM and
// releases its dependent at its START, so the next query's scan co-runs with this one instead of
// waiting for it to drain (scan_topk.cu: "overlapped launches").  It co-scans: it starts its pass where
// its predecessor on the same corpus is reading, so the two scans share each tile's read through L2.
int stb_launch_scan_topk(stb_ctx *ctx, const stb_corpus *c, int tier, const float *q_dev, uint32_t top_k,
                         const uint64_t *ranges_dev, uint32_t n_ranges,
                         uint64_t n_virtual, stb_hit *out_hits_dev,
                         uint32_t *out_status_dev, const StbXchgArgs *xchg = nullptr, bool overlapped = false);
// int8 codes + scales, nibble plane + {s, rho} of rows [first_row, n_rows) (q8 tier)
// rows_first: the row rows_dev[0] holds (a staged chunk of a host-rows corpus), 0 for a whole matrix
int stb_launch_q8_build(stb_ctx *ctx, const float *rows_dev, uint64_t first_row, uint64_t n_rows, uint8_t *out,
                        float *scale, uint8_t *plane, float2 *sr, int *bad_flag_dev, uint64_t rows_first = 0);
// Largest top_k the fast path serves.
uint32_t stb_scan_topk_max_k(void);
// Collect path: every row whose approximate cosine >= cos_floor (or that cannot be
// scored safely) is appended to ctx->collect_rows; total count -> collect_count.
// tier: STB_TIER_F32 (approximate cosine of the f32 rows) or STB_TIER_Q8 (upper bounds from the int8 copy)
int stb_launch_scan_collect(stb_ctx *ctx, const stb_corpus *c, int tier,
                            const float *q_dev, float cos_floor,
                            const uint64_t *ranges_dev, uint32_t n_ranges,
                            uint64_t n_virtual);
// Large-k support: 4096-bin histogram of the approximate cosine over the scanned rows
// (bin b: cos in (1-(b+1)/2048, 1-b/2048]).  hist_dev: 4096 u32 on device.
int stb_launch_scan_hist(stb_ctx *ctx, const stb_corpus *c, int tier, const float *q_dev, const uint64_t *ranges_dev,
                         uint32_t n_ranges, uint64_t n_virtual, unsigned int *hist_dev);
// Test hooks (stb_debug_scan_scores, stb_debug_q4_scan): the f32 / h16 / q8 pass, or the q8 tier's prefiltered
// top-k scan, with a sink that stores each scanned local row's score into score[row] and counts it in seen[row].
// The q4 form also stores u4 and T per row and l8 per refined row (pin != 0: T held at -inf); words: top_k
// threshold words (zeroed; tag 1), refined: a zeroed counter.
int stb_launch_debug_scan(stb_ctx *ctx, const stb_corpus *c, int tier, const float *q_dev, const uint64_t *ranges_dev,
                          uint32_t n_ranges, uint64_t n_virtual, float *score, unsigned int *seen);
int stb_launch_debug_q4(stb_ctx *ctx, const stb_corpus *c, const float *q_dev, uint32_t top_k, const uint64_t *ranges_dev,
                        uint32_t n_ranges, uint64_t n_virtual, unsigned long long *words, unsigned long long *refined,
                        int pin, float *u4, float *t, float *l8, float *u8, unsigned int *seen);
// Exact canonical distances of m collected rows -> hits (invalid/failing rows get
// distance=+inf,row=UINT64_MAX); counts passing rows into pass_count.
int stb_launch_exact(stb_ctx *ctx, const float *rows, uint64_t row_base,
                     const float *q_dev, const uint32_t *row_ids, uint64_t m,
                     double limit, stb_hit *hits, uint64_t m_padded,
                     unsigned long long *pass_count);
// In-place ascending sort by (distance,row) of m_padded (power of two) hits.
int stb_launch_sort_hits(stb_ctx *ctx, stb_hit *hits, uint64_t m_padded);

// ---- hits_merge.cu --------------------------------------------------------------
int stb_launch_hits_merge(stb_ctx *ctx, const stb_hit *lists_dev, uint32_t n_lists,
                          uint32_t per_list, uint32_t top_k, stb_hit *out_dev);

int stb_launch_hits_merge_batch(stb_ctx *ctx, const stb_hit *lists_dev, uint32_t n_lists, uint32_t nq,
                                uint32_t per_list, uint32_t top_k, stb_hit *out_dev);
// sharded K2 exchange over peer memory: push this rank's nq x k hits + per-query status into every
// peer's batch slot, then (second launch) wait for all peers and merge per query
struct StbBatchXchgArgs {
  unsigned char *slot[STB_XCHG_MAX_WORLD];   // batch slot of every rank (peer-mapped), this batch's parity
  uint32_t world, rank, max_nq, max_k, nq, top_k;
  unsigned long long seq;
  unsigned int *ticket;
};
int stb_launch_batch_xchg(stb_ctx *ctx, const StbBatchXchgArgs &a, const stb_hit *local_hits, const uint32_t *local_status,
                          stb_hit *out_hits, uint32_t *out_status);

// opt-in to > 48 KiB dynamic shared memory (or another function attribute) once per context
enum { STB_ATTR_GEMM0 = 0, STB_ATTR_GEMM1, STB_ATTR_MERGE, STB_ATTR_IVF_PROBE, STB_ATTR_IVF_V2, STB_ATTR_FINISH2,
       STB_ATTR_IVF_BATCH, STB_ATTR_GEMM0F, STB_ATTR_GEMM1F, STB_ATTR_GEMM2, STB_ATTR_GEMM0W, STB_ATTR_GEMM1W,
       STB_ATTR_Q8GEMM0, STB_ATTR_Q8GEMM1, STB_ATTR_Q8GEMM2, STB_ATTR_THRESH_BIG };
#define STB_ATTR_ONCE(ctx, bit, call)                         \
  do {                                                        \
    if (!((ctx)->func_attr_mask & (1u << (bit)))) {           \
      STB_CUDA(call);                                         \
      (ctx)->func_attr_mask |= 1u << (bit);                   \
    }                                                         \
  } while (0)

// ---- embed_pool.cu --------------------------------------------------------------
int stb_launch_embed(stb_ctx *ctx, const stb_table *t, const uint64_t *offsets_dev,
                     const uint32_t *ids_dev, uint64_t n_lines, float *out_dev,
                     int *err_flag_dev);

// ---- batch_scan.cu (K2) ------------------------------------------------------------------
// rows_first: the row rows_dev[0] holds, as stb_launch_q8_build
int stb_launch_shadow_build(stb_ctx *ctx, const float *rows_dev, uint64_t n_rows, int tile,
                            uint8_t *out, int *bad_flag_dev, uint64_t first_row = 0,
                            uint32_t *row_bad_dev = nullptr, uint64_t rows_first = 0);
int stb_launch_batch_gemm(stb_ctx *ctx, const uint8_t *a_tiles, uint32_t m_tiles,
                          const uint8_t *b_tiles, uint32_t n_tiles, float *submax,
                          float *tilemax, float *full_out);
int stb_launch_batch_gemm_strided(stb_ctx *ctx, const uint8_t *a_tiles, uint32_t m_tiles,
                                  const uint8_t *b_tiles, uint32_t n_tiles, uint32_t tile_stride,
                                  float *submax, float *tilemax, float *full_out);
int stb_launch_batch_gemm_emit(stb_ctx *ctx, const uint8_t *a_tiles, uint32_t m_tiles,
                               const uint8_t *b_tiles, uint32_t n_tiles, uint64_t n_rows,
                               const float *thr, uint32_t *cand_cnt, uint64_t *cand_keys,
                               uint32_t cand_cap);
// the same two passes over the listed tiles tile_ids[0, n_listed), eligible rows (bitmap) only
int stb_launch_batch_gemm_sample_filtered(stb_ctx *ctx, const uint8_t *a_tiles, uint32_t m_tiles,
                                          const uint8_t *b_tiles, const uint32_t *tile_ids,
                                          const uint32_t *bitmap, uint32_t n_sample, uint32_t tile_stride,
                                          float *tilemax);
int stb_launch_batch_gemm_emit_filtered(stb_ctx *ctx, const uint8_t *a_tiles, uint32_t m_tiles,
                                        const uint8_t *b_tiles, const uint32_t *tile_ids,
                                        const uint32_t *bitmap, uint32_t n_listed, uint64_t n_rows,
                                        const float *thr, uint32_t *cand_cnt, uint64_t *cand_keys,
                                        uint32_t cand_cap);
// the same two passes with one filter per 64-query half, over per-corpus-tile work items (batch_scan.cu, GemmArgs)
int stb_launch_batch_gemm_sample_work(stb_ctx *ctx, const uint8_t *a_tiles, const uint8_t *b_tiles,
                                      const uint32_t *tile_ids, uint32_t n_tiles, const uint32_t *cta_tiles,
                                      const uint32_t *item_off, const uint4 *items, const uint32_t *bitmap,
                                      uint32_t tm_cols, float *tilemax);
int stb_launch_batch_gemm_emit_work(stb_ctx *ctx, const uint8_t *a_tiles, const uint8_t *b_tiles,
                                    const uint32_t *tile_ids, uint32_t n_tiles, const uint32_t *cta_tiles,
                                    const uint32_t *item_off, const uint4 *items, const uint32_t *bitmap,
                                    const uint32_t *slot_row, uint64_t n_rows, const float *thr, uint32_t *cand_cnt,
                                    uint64_t *cand_keys, uint32_t cand_cap);
// the query slots of those passes: f32 rows gathered into slot order, then the per-row bad flags scattered
// back and the sampled maxima preset to -inf
int stb_launch_batch_slots_gather(stb_ctx *ctx, const float *rows, const uint32_t *slot_row, uint32_t n_slots, float *out);
int stb_launch_batch_slots_prep(stb_ctx *ctx, const uint32_t *slot_row, const uint32_t *slot_bad, uint32_t n_slots,
                                uint32_t *row_bad, float *tilemax, uint64_t n_tilemax);
// thr[q] = k-th largest of query q's n_sample sampled maxima - slack (negative: the shadow's 2 STB_BATCH_EPS), -inf
// when fewer than k were sampled, +inf for padding queries and where q_skip (may be null) is set
int stb_launch_batch_thresh(stb_ctx *ctx, const float *tilemax, uint32_t n_sample, uint32_t nq,
                            uint32_t q_pad, uint32_t top_k, float *thr, float slack = -1.0f,
                            const uint32_t *q_skip = nullptr);
// candidates live in per-(query, CTA) segments: keys [q_pad][n_seg][seg_cap], counts [q_pad][n_seg];
// n_seg = stb_batch_emit_grid() = the grid the emitting GEMM runs with
uint32_t stb_batch_emit_grid(const stb_ctx *ctx, uint32_t n_tiles);
int stb_launch_batch_finish2(stb_ctx *ctx, const uint64_t *cand_keys, const uint32_t *cand_cnt, uint32_t n_seg,
                             uint32_t seg_cap, uint32_t nq, uint32_t top_k, const float *rows,
                             uint64_t n_rows, uint64_t row_base, const float *queries_dev,
                             const uint32_t *q_bad, stb_hit *out_hits, uint32_t *out_status,
                             const float *q8_scale = nullptr, const float4 *q8_qc = nullptr,
                             const float *thr = nullptr);
// Route 7 (the q8 copy on the int8 tensor cores, batch_scan.cu): the query tiles -- hi / lo bytes of q16 in the
// wgmma layout, m_tiles x 64 KiB -- with per-query {1/S, h_l1, e_q, S} and unusable flags (q16: [nq][256] or null);
// the sampling pass (tile maxima of the lower bound l over tiles 0, stride, ... (n_sample of them)); the emitting
// pass (every row whose upper bound u reaches thr, into the segments as stb_launch_batch_gemm_emit); and the
// debug pass (dot, u and l of every (query, row) into [m_tiles * 128][ceil(n_rows / 256) * 256] matrices)
int stb_launch_q8_query_tiles(stb_ctx *ctx, const float *q_dev, uint32_t nq, uint32_t q_pad, uint8_t *tiles,
                              float4 *qc, uint32_t *q_bad, int16_t *q16);
int stb_launch_batch_q8_gemm_sample(stb_ctx *ctx, const uint8_t *a_tiles, const float4 *qc, uint32_t m_tiles,
                                    const uint8_t *codes, const float *scales, uint64_t n_rows, uint32_t n_sample,
                                    uint32_t tile_stride, float *tilemax);
int stb_launch_batch_q8_gemm_emit(stb_ctx *ctx, const uint8_t *a_tiles, const float4 *qc, uint32_t m_tiles,
                                  const uint8_t *codes, const float *scales, uint64_t n_rows, const float *thr,
                                  uint32_t *cand_cnt, uint64_t *cand_keys, uint32_t cand_cap);
int stb_launch_batch_q8_gemm_debug(stb_ctx *ctx, const uint8_t *a_tiles, const float4 *qc, uint32_t m_tiles,
                                   const uint8_t *codes, const float *scales, uint64_t n_rows, int32_t *dot, float *u,
                                   float *l);
void stb_batch_build_params(int *shadow_is_f16, double *eps);
// threshold mode's re-emission: the emitting pass into exactly sized segments cand_keys[seg_off[i], seg_off[i+1])
// (i = query * grid + CTA), cursors [q_pad][grid] zeroed
int stb_launch_batch_gemm_emit_sized(stb_ctx *ctx, const uint8_t *a_tiles, uint32_t m_tiles,
                                     const uint8_t *b_tiles, uint32_t n_tiles, uint64_t n_rows,
                                     const float *thr, uint32_t *cursors, uint64_t *cand_keys,
                                     const uint64_t *seg_off);

// ---- batch_threshold.cu (K2 threshold mode) -------------------------------------------------------
// thr[i] = t for the queries i < nq that are non-zero and normalisable, +inf for the others and the padding
int stb_launch_batch_thr_dist(stb_ctx *ctx, const float *q_dev, const uint32_t *q_bad, uint32_t nq, uint32_t q_pad,
                              float t, float *thr);
// segment i of the first pass (cnt[i] keys at keys + i * seg_cap) -> out[dst[i] ..]; dst[i] = ~0: skipped
int stb_launch_batch_thr_compact(stb_ctx *ctx, const uint64_t *keys, const uint32_t *cnt, const uint64_t *dst,
                                 uint64_t n_pairs, uint32_t seg_cap, uint64_t *out);
// slot r < n: query src[idx[r]] and thr_src[idx[r]]; slots [n, r_pad): thr +inf
int stb_launch_batch_thr_gather(stb_ctx *ctx, const float *src, const float *thr_src, const uint32_t *idx, uint32_t n,
                                uint32_t r_pad, float *dst, float *thr_dst);
// slot s: keys [off[s], off[s+1]) re-scored against query qidx[s]: (distance bits, global row), or (+inf, ~0)
// when not d < limit; pass[s] = rows kept
int stb_launch_batch_thr_rescore(stb_ctx *ctx, const uint64_t *keys, const int *off, const uint32_t *qidx,
                                 uint32_t n_slots, const float *queries_dev, const float *rows, uint64_t row_base,
                                 double limit, uint64_t *dist_bits, uint64_t *grow, uint32_t *pass);
// slot s: its first pass[s] sorted pairs -> out[dst[s] ..]
int stb_launch_batch_thr_write(stb_ctx *ctx, const uint64_t *dist_bits, const uint64_t *grow, const int *off,
                               const uint32_t *pass, uint32_t n_slots, const uint64_t *dst, stb_hit *out);
// segmented sorts over the slots: keys by row (low 32 bits); (distance bits, row) pairs stably by distance
int stb_batch_thr_sort_bytes(stb_ctx *ctx, int n_items, uint32_t n_slots, const int *off, size_t *bytes);
int stb_batch_thr_sort_rows(stb_ctx *ctx, void *tmp, size_t tmp_bytes, int n_items, uint32_t n_slots, const int *off,
                            const uint64_t *keys_in, uint64_t *keys_out);
int stb_batch_thr_sort_dist(stb_ctx *ctx, void *tmp, size_t tmp_bytes, int n_items, uint32_t n_slots, const int *off,
                            const uint64_t *dist_bits, uint64_t *dist_out, const uint64_t *grow, uint64_t *grow_out);
int stb_launch_batch_select(stb_ctx *ctx, const float *submax, uint32_t n_sub, uint32_t q_pad,
                            uint32_t n_slices, uint64_t *cand);
int stb_launch_batch_finish(stb_ctx *ctx, const uint64_t *cand, uint32_t n_slices, uint32_t n_sub,
                            uint32_t nq, uint32_t top_k, const float *rows, uint64_t n_rows,
                            uint64_t row_base, const float *queries_dev, const uint32_t *q_bad,
                            stb_hit *out_hits, uint32_t *out_status, const float *submax, uint32_t q_pad);

// ---- ivfpq.cu: the eligibility bitmap of a path filter ----------------------------
// bitmap[w] bit j = local row 32w + j lies in one of the n_ranges local [begin, end) u32 pairs of ranges_dev
// (ascending, disjoint), for w < n_words.  With set_off_dev (2 n_sets entries on the device), one launch
// writes n_sets bitmaps: bitmap s at bitmap + s * n_words from the pairs [set_off_dev[2s], set_off_dev[2s+1])
// of ranges_dev, and n_ranges is unused.
int stb_launch_row_bitmap(stb_ctx *ctx, const uint32_t *ranges_dev, uint32_t n_ranges, uint64_t n_words,
                          uint32_t *bitmap, uint32_t n_sets = 1, const uint64_t *set_off_dev = nullptr);

// ---- device helpers ---------------------------------------------------------------
// The distance limit of a search without max_distance: max_distance.unwrap_or(100.0), strict.
#define STB_DEFAULT_MAX_DIST 100.0

#ifdef __CUDACC__
#include <math_constants.h>

// Monotone map float -> uint32 (larger float -> larger uint), total order with
// -inf lowest; NaN never reaches it.
__device__ __forceinline__ uint32_t stb_f2ord(float f) {
  uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float stb_ord2f(uint32_t o) {
  uint32_t b = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
  return __uint_as_float(b);
}
// Candidate key: ascending key order == (score descending, row ascending).
__device__ __forceinline__ uint64_t stb_make_key(float score, uint32_t row) {
  return ((uint64_t)(~stb_f2ord(score)) << 32) | (uint64_t)row;
}
#define STB_KEY_INVALID 0xffffffffffffffffull
__device__ __forceinline__ float stb_key_score(uint64_t k) {
  return stb_ord2f(~(uint32_t)(k >> 32));
}
__device__ __forceinline__ uint32_t stb_key_row(uint64_t k) { return (uint32_t)k; }

__device__ __forceinline__ bool stb_hit_less(double da, uint64_t ra, double db,
                                             uint64_t rb) {
  return (da < db) || (da == db && ra < rb);
}

// ---- the exact re-rank: canonical distance (oracle orc_cosine_f32), hit order, hit output ----
// Every kernel that returns hits scores them with these, so the bits match the oracle's.
// sqd: the query staged in f64 (exact conversion of the f32 components).

// ||q||^2: f64 FMAs in index order.
__device__ __forceinline__ double stb_canon_q2(const double *sqd) {
  double q2 = 0.0;
#pragma unroll 8
  for (int i = 0; i < STB_D; ++i) q2 = fma(sqd[i], sqd[i], q2);
  return q2;
}

// q . row and ||row||^2: f64 FMAs in index order, one rounding per step.  f32 x f32 products are
// exact in f64, so this equals the oracle bit for bit.  LDG: the row is in global memory and read
// through the read-only path; otherwise it is staged in shared memory.
template <bool LDG>
__device__ __forceinline__ void stb_canon_dot(const double *sqd, const float4 *row, double &ab, double &r2) {
  ab = 0.0;
  r2 = 0.0;
#pragma unroll 8
  for (int i = 0; i < STB_ROW_F4; ++i) {
    const float4 v = LDG ? __ldg(row + i) : row[i];
    const double vx = (double)v.x, vy = (double)v.y, vz = (double)v.z, vw = (double)v.w;
    ab = fma(sqd[4 * i + 0], vx, ab); r2 = fma(vx, vx, r2);
    ab = fma(sqd[4 * i + 1], vy, ab); r2 = fma(vy, vy, r2);
    ab = fma(sqd[4 * i + 2], vz, ab); r2 = fma(vz, vz, r2);
    ab = fma(sqd[4 * i + 3], vw, ab); r2 = fma(vw, vw, r2);
  }
}

// Cosine distance: 0 when both vectors are zero, 1 when orthogonal, else max(0, 1 - ab / (|q| |r|)).
// Callers keep a hit iff the result is strictly below their limit.
__device__ __forceinline__ double stb_canon_dist(double ab, double q2, double r2) {
  if (q2 == 0.0 && r2 == 0.0) return 0.0;
  if (ab == 0.0) return 1.0;
  const double t = 1.0 - ab / (sqrt(q2) * sqrt(r2));
  return t > 0.0 ? t : 0.0;
}

// Ascending sort by (distance, row) of n (power of two) pairs in shared memory; any blockDim.x.
__device__ __forceinline__ void stb_cta_sort_hits(double *sd, uint64_t *sr, uint32_t n) {
  for (uint32_t kk = 2; kk <= n; kk <<= 1)
    for (uint32_t j = kk >> 1; j > 0; j >>= 1) {
      for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t ixj = i ^ j;
        if (ixj > i) {
          const bool up = ((i & kk) == 0);
          const bool gt = stb_hit_less(sd[ixj], sr[ixj], sd[i], sr[i]);
          if (gt == up) {
            const double td = sd[i]; const uint64_t tr = sr[i];
            sd[i] = sd[ixj]; sr[i] = sr[ixj]; sd[ixj] = td; sr[ixj] = tr;
          }
        }
      }
      __syncthreads();
    }
}

// Ascending sort of n (power of two) keys in shared memory, thread-strided; any blockDim.x.
__device__ __forceinline__ void stb_cta_sort_keys_strided(uint64_t *keys, uint32_t n) {
  for (uint32_t kk = 2; kk <= n; kk <<= 1)
    for (uint32_t j = kk >> 1; j > 0; j >>= 1) {
      for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t ixj = i ^ j;
        if (ixj > i) {
          const uint64_t x = keys[i], y = keys[ixj];
          const bool up = ((i & kk) == 0);
          if ((x > y) == up) { keys[i] = y; keys[ixj] = x; }
        }
      }
      __syncthreads();
    }
}

// out[0, k): the first n_out sorted pairs, then (+inf, UINT64_MAX) padding, which merges as-is.
__device__ __forceinline__ void stb_write_hits(stb_hit *out, const double *sd, const uint64_t *sr, uint32_t n_out,
                                               uint32_t k) {
  for (uint32_t i = threadIdx.x; i < k; i += blockDim.x) {
    stb_hit h;
    h.distance = (i < n_out) ? sd[i] : CUDART_INF;
    h.row = (i < n_out) ? sr[i] : 0xffffffffffffffffull;
    out[i] = h;
  }
}

// Ascending bitonic sort of n keys (power of two, <= R*256) held in shared memory,
// done in registers: element i = r*256 + tid lives in register k[r] of thread tid, so a
// compare-exchange at distance j is a register swap (j >= 256), a shuffle (j < 32) or a
// shared-memory exchange (32 <= j < 256; the only steps that need __syncthreads).
// Requires blockDim.x == 256.
template <int R>
__device__ __forceinline__ void stb_cta_sort_keys_t(uint64_t *keys, int n) {
  const int tid = threadIdx.x;
  uint64_t k[R];
#pragma unroll
  for (int r = 0; r < R; ++r) k[r] = (r * 256 + tid < n) ? keys[r * 256 + tid] : STB_KEY_INVALID;
  __syncthreads();
  for (int kk = 2; kk <= n; kk <<= 1) {
    for (int j = kk >> 1; j > 0; j >>= 1) {
      if (j >= 256) {
        // in-thread exchange; dr spelled out so k[] stays in registers
#pragma unroll
        for (int dr = 1; dr < R; dr <<= 1) {
          if (j == dr * 256) {
#pragma unroll
            for (int r = 0; r < R; ++r) {
              if ((r & dr) == 0) {
                const bool up = (((r * 256 + tid) & kk) == 0);
                uint64_t x = k[r], y = k[r | dr];
                if ((x > y) == up) { k[r] = y; k[r | dr] = x; }
              }
            }
          }
        }
      } else if (j >= 32) {
#pragma unroll
        for (int r = 0; r < R; ++r) keys[r * 256 + tid] = k[r];
        __syncthreads();
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const int i = r * 256 + tid;
          const uint64_t other = keys[i ^ j];
          const bool keep_min = (((i & j) == 0) == ((i & kk) == 0));
          k[r] = keep_min ? (k[r] < other ? k[r] : other) : (k[r] > other ? k[r] : other);
        }
        __syncthreads();
      } else {
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const int i = r * 256 + tid;
          const uint64_t other = __shfl_xor_sync(0xffffffffu, k[r], j);
          const bool keep_min = (((i & j) == 0) == ((i & kk) == 0));
          k[r] = keep_min ? (k[r] < other ? k[r] : other) : (k[r] > other ? k[r] : other);
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < R; ++r) keys[r * 256 + tid] = k[r];
  __syncthreads();
}

#endif

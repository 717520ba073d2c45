// Internal declarations shared by the translation units of libsemtools_b200.so.
// Everything here is sm_90a-only product code; nothing in this directory may
// include, link or call anything under oracle/.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

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

struct stb_ctx {
  int device;
  int sm_count;
  cudaStream_t stream;
  bool own_stream;
  // --- scan scratch (device) ---
  uint64_t *block_keys;     // candidate keys of every tree level
  size_t block_keys_cap;    // in keys
  unsigned int *counters;   // tree arrival counters (zeroed; kernels re-zero)
  size_t counters_cap;
  // K1 tile-ticket counters (monotonic; scan_topk.cu: stb_for_each_tile).  A ring of STB_TICKET_SLOTS
  // counters, one per launch in turn: with the overlapped launch mode two consecutive scans run
  // concurrently and must not draw from the same counter.
  unsigned long long *tickets;
  unsigned long long ticket_next[8];   // per slot: its value when the next launch using it starts
  unsigned long long topk_launches;    // picks the slot
  bool ticket_ring;                    // set by the first overlapped launch; until then every launch uses slot 0
  // K1 co-scan (scan_topk.cu: stb_coscan_offset): per ticket slot, the tile offset its last co-scan launch
  // chose, as a tagged word (tag << 32 | offset, the tag is the launch count); the host's copy of the tags
  // (0: the slot's last launch did not co-scan) and the last co-scan launch, which the next one may follow
  unsigned long long *coscan_off;
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
  unsigned long long *q4_thr;
  unsigned long long q4_launches;
  unsigned long long *q4_refined;      // rows the prefilter passed on to the int8 codes (stb_debug_q4_refined)
  float *q_dev;             // 256 f32 staging for host queries
  stb_hit *hits_dev;        // result hits (top-k path)
  size_t hits_cap;
  uint32_t *status_dev;     // [0]=n hits, [1]=complete flag, [2..] debug
  uint32_t *collect_rows;   // threshold/fallback compaction: local row ids
  size_t collect_cap;
  unsigned long long *collect_count;
  stb_hit *collect_hits;    // exact hits of collected rows (sorted in place)
  size_t collect_hits_cap;
  uint64_t *ranges_dev;     // [3 * n] : begin(local), end(local), vstart
  size_t ranges_cap;
  int *err_flag;            // device int: scratch flag of the copy builders, stb_embed and K2's query shadow; zeroed before each use
  unsigned int *hist_dev;       // 4096-bin score histogram (large-k path)
  // cudaFuncSetAttribute is per DEVICE: remembered per context, never in function statics
  // (one process may hold contexts on several GPUs)
  uint32_t func_attr_mask;
  size_t finish2_smem_set;
  // --- K2 scratch ---
  uint8_t *bq_tiles; size_t bq_tiles_cap;     // query shadow tiles
  float *b_submax; size_t b_submax_cap;       // [n_sub][q_pad]
  float *b_tilemax; size_t b_tilemax_cap;     // [n_tiles][q_pad]
  uint64_t *b_cand; size_t b_cand_cap;        // [q_pad][slices][32]
  float *b_thr; size_t b_thr_cap;             // v2: [q_pad] emission thresholds
  uint32_t *b_cnt; size_t b_cnt_cap;          // v2: [q_pad] emitted-candidate counters
  uint64_t *b_keys; size_t b_keys_cap;        // v2: [q_pad][cand_cap] emitted keys
  uint32_t *b_qbad; size_t b_qbad_cap;        // [q_pad] 1: query could not be normalised
  // stb_search_batch_filtered: the clipped ranges (local [begin, end) u32 pairs), the listed tiles and the
  // eligible-row bitmap (8 words per shadow tile), all built from the same clipped ranges
  uint32_t *b_franges; size_t b_franges_cap;
  uint32_t *b_ftiles; size_t b_ftiles_cap;
  uint32_t *b_fbits; size_t b_fbits_cap;
  // the last K2 call: route (1 = v1, 2 = v2, 3 = filtered v2, 4 = filtered, nothing on the tensor cores), nq,
  // n_sample, stride, n_seg, seg_cap
  uint32_t b_last[6];
  float *bq_dev; size_t bq_dev_cap;           // host-call staging: queries
  stb_hit *bh_dev; size_t bh_dev_cap;         // host-call staging: hits
  uint32_t *bs_dev; size_t bs_dev_cap;        // host-call staging: status
  uint64_t *embed_off_dev;  // K3 staging: CSR offsets
  size_t embed_off_cap;
  uint32_t *embed_ids_dev;  // K3 staging: token ids
  size_t embed_ids_cap;
  float *embed_out_dev;     // K3 output when not appending to a corpus
  size_t embed_out_cap;
  // in-place corpus mutations (stb_corpus_update / _remove): row staging (<= STB_MUT_CHUNK_ROWS rows),
  // row ids or kept-segment table, and the q8 / shadow bad-row flags
  float *mut_stage; size_t mut_stage_cap;
  uint64_t *mut_idx; size_t mut_idx_cap;
  int *mut_flags; size_t mut_flags_cap;
  // --- pinned host staging ---
  float *q_pin;
  stb_hit *hits_pin;
  size_t hits_pin_cap;
  uint32_t *status_pin;
  float *many_q_pin;          // stb_search_many: queries / per-query status (kernels write the latter directly)
  uint32_t *many_status_pin;
  size_t many_q_pin_cap;      // in floats
  // --- counters ---
  uint64_t kernel_launches;
  uint64_t fallback_searches;
  // --- K3 ---
  int *embed_flag;          // device int: K3's sticky range flag; set only by stb_embed_dev, cleared only by stb_embed_status
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
  unsigned char *local;                      // this rank's buffer (cudaMalloc)
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
  unsigned int *batch_ticket;                // device: arrival counter of the push kernel
  bool dead;                                 // a synchronous call saw a peer time-out: every later call is refused
};

struct stb_table {
  stb_ctx *ctx;
  float *E;            // V x 256
  uint64_t V;
  float *weights;      // or nullptr
  uint64_t n_weights;
  uint32_t *mapping;   // or nullptr
  uint64_t n_mapping;
  int normalize;
};

struct stb_corpus {
  stb_ctx *ctx;
  float *rows;         // capacity x 256
  uint64_t n;
  uint64_t capacity;
  uint64_t row_base;
  uint64_t epoch;            // bumped by every change that is not an append (an IVF-PQ index refuses to extend over it)
  // K2: L2-normalised bf16 copy in wgmma tile layout (built lazily, rebuilt when n changes)
  uint8_t *shadow;
  uint64_t shadow_rows;      // rows covered by `shadow` (== n when valid)
  uint64_t shadow_cap_tiles;
  int shadow_bad;            // 1: some row cannot be normalised in fp32 -> tensor path refused
  // K1 tier q8: int8 codes [capacity][256] + per-row scale, built lazily / by stb_corpus_prepare
  uint8_t *q8;
  float *q8_scale;
  uint8_t *q4;               // ... its nibble plane [capacity][128] and per-row {s, rho} (top-k prefilter)
  float2 *q4_sr;
  uint64_t q8_rows;          // rows covered (== n when valid; also the plane's)
  uint64_t q8_cap_rows;
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
int stb_launch_q8_build(stb_ctx *ctx, const float *rows_dev, uint64_t first_row, uint64_t n_rows, uint8_t *out,
                        float *scale, uint8_t *plane, float2 *sr, int *bad_flag_dev);
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
       STB_ATTR_IVF_BATCH, STB_ATTR_GEMM0F, STB_ATTR_GEMM1F };
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
int stb_launch_shadow_build(stb_ctx *ctx, const float *rows_dev, uint64_t n_rows, int tile,
                            uint8_t *out, int *bad_flag_dev, uint64_t first_row = 0,
                            uint32_t *row_bad_dev = nullptr);
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
int stb_launch_batch_thresh(stb_ctx *ctx, const float *tilemax, uint32_t n_sample, uint32_t nq,
                            uint32_t q_pad, uint32_t top_k, float *thr);
// candidates live in per-(query, CTA) segments: keys [q_pad][n_seg][seg_cap], counts [q_pad][n_seg];
// n_seg = stb_batch_emit_grid() = the grid the emitting GEMM runs with
uint32_t stb_batch_emit_grid(const stb_ctx *ctx, uint32_t n_tiles);
int stb_launch_batch_finish2(stb_ctx *ctx, const uint64_t *cand_keys, const uint32_t *cand_cnt, uint32_t n_seg,
                             uint32_t seg_cap, uint32_t nq, uint32_t top_k, const float *rows,
                             uint64_t n_rows, uint64_t row_base, const float *queries_dev,
                             const uint32_t *q_bad, stb_hit *out_hits, uint32_t *out_status);
void stb_batch_build_params(int *shadow_is_f16, double *eps);
int stb_launch_batch_select(stb_ctx *ctx, const float *submax, uint32_t n_sub, uint32_t q_pad,
                            uint32_t n_slices, uint64_t *cand);
int stb_launch_batch_finish(stb_ctx *ctx, const uint64_t *cand, uint32_t n_slices, uint32_t n_sub,
                            uint32_t nq, uint32_t top_k, const float *rows, uint64_t n_rows,
                            uint64_t row_base, const float *queries_dev, const uint32_t *q_bad,
                            stb_hit *out_hits, uint32_t *out_status, const float *submax, uint32_t q_pad);

// ---- ivfpq.cu: the eligibility bitmap of a path filter ----------------------------
// bitmap[w] bit j = local row 32w + j lies in one of the n_ranges local [begin, end) u32 pairs of ranges_dev
// (ascending, disjoint), for w < n_words
int stb_launch_row_bitmap(stb_ctx *ctx, const uint32_t *ranges_dev, uint32_t n_ranges, uint64_t n_words,
                          uint32_t *bitmap);

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

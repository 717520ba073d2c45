// K5: IVF-PQ index over a corpus shard -- coarse probe + ADC-table code scan + exact re-rank.
//
// The reference snapshot has NO IVF_PQ (its store is qdrant-edge with a plain index and
// quantization_config None, src/workspace/store.rs:129-130,156-157; "IVF_PQ" survives only
// as stale text in README.md:125).  This component is therefore self-specified (BASELINE
// config 5: nlist=4096, nprobe=64) and PARITY-UNPINNED: it is measured by recall@k against
// the exact scan (K1) and by bytes/query; every returned distance is still the canonical
// exact f64 cosine distance of that row, so a returned hit is never wrong, only possibly
// not the global best.
//
// Index (per shard, all in HBM):
//   centroids  [nlist][256] f32, unit norm (spherical k-means on L2-normalised rows)
//   codebooks  [32][256][8]  f32: product quantiser of the residual x^ - c(x), 8 dims/byte
//   codes      [n][32] u8 grouped by list, order[n] = local row of each code, list_off[nlist+1]
//              (within a list, ascending row order: see "adding rows")
// Query: coarse scores q^.c_j (nlist*1 KiB read), top-nprobe lists, LUT[s][code] = q^_s .
// cb[s][code] (32 KiB), ADC score = q^.c_list + sum_s LUT[s][code_s] over the probed
// lists' codes ((nprobe/nlist)*n*32 bytes), running top-R, exact re-rank of R rows.
//
// Forced rows: a row with a non-finite component or an fp32 ||x||^2 outside [1e-30, 1e30] (the
// rows K1 forces into its candidates) has no usable direction, so its PQ code says nothing about
// its cosine.  Such rows are kept out of the inverted lists and out of training; the build records
// them in a side list (at most IVF_FORCED_CAP, usually empty) that every search re-ranks exactly
// in addition to the ADC candidates.
#include <math_constants.h>

#include <algorithm>
#include <cub/device/device_radix_sort.cuh>
#include <vector>

#include "common.cuh"

#define PQ_M 32
#define PQ_DSUB 8
#define PQ_KSUB 256
#define IVF_FORCED_CAP 1024        // forced rows per index; more -> the build or extend fails with STB_ERR_STATE
#define IVF_HOST_TOPK_MAX 4096     // stb_ivfpq_search: top_k and rerank cap of the multi-launch search
#define IVF_NO_LIST 0xffffffffu    // assign[] of a forced row

// batched search (see "batched search" below)
#define IVFB_MAX_NQ 4096           // queries per stb_ivfpq_search_batch_dev call (the host form chunks)
#define IVFB_QTILE 16              // queries per CTA of the coarse kernel
#define IVFB_SCAN_CTAS 8           // scan CTAs per query
#define IVFB_SCAN_THREADS 256
#define IVFB_WARPS (IVFB_SCAN_CTAS * IVFB_SCAN_THREADS / 32)   // 64 scan warps per query
#define IVFB_WARP_KEEP 64          // best keys a scan warp keeps (2 per lane)
#define IVFB_KEPT (IVFB_WARPS * IVFB_WARP_KEEP)                // 4096 kept keys per query
#define IVFB_FIN_THREADS 512
#define IVFB_FIN_SMEM 65536
#define IVFB_RERANK_CAP 1024

struct stb_ivfpq {
  stb_ctx *ctx;
  const stb_corpus *corpus;
  uint64_t corpus_epoch;      // corpus->epoch when the index was built: extend refuses another
  uint32_t nlist;
  uint64_t n;                 // rows indexed (listed + forced): rows [0, n) of the corpus
  float *centroids;           // [nlist][256]
  float *codebooks;           // [32][256][8]
  uint8_t *codes;             // [n_listed][32], grouped by list
  uint32_t *order;            // [n_listed] local row of code i
  uint32_t *list_off;         // [nlist+1] (device); list_off[nlist] = n_listed = n - n_forced
  std::vector<uint32_t> list_off_h;
  uint32_t *forced;           // [n_forced] local rows outside the lists, ascending
  uint32_t n_forced;
  // query scratch
  float *coarse;              // [nlist]
  float *lut;                 // [32][256]
  uint32_t *probe;            // [nprobe_max] list ids, [nprobe_max+1] prefix of lengths
  stb_hit *cand;              // candidate (-score,pos) hits, padded
  size_t cand_cap;
  uint32_t *cand_rows;        // local rows of the R best candidates
  // fused search (v2)
  uint64_t *keys2;            // [ADC2_MAX_CTAS][ADC2_KEEP] per-CTA best candidates (score desc, code position)
  unsigned int *tickets;      // [2] last-CTA tickets of the two fused kernels (kernels re-zero them)
  // batched search scratch (its own buffers: a batch and a single query enqueued back to back do not
  // share any), sized for b_cap queries, grown on demand
  uint32_t b_cap;
  float *b_q;                 // [b_cap][256] queries of the host form
  float *b_coarse;            // [b_cap][nlist]
  uint32_t *b_probe;          // [b_cap][2 * 1024 + 2]: nprobe list ids, the prefix of their lengths (filtered:
                              // and the eligible codes), IVFB_PROBE_STRIDE apart
  float *b_lut;               // [b_cap][32][256]
  uint64_t *b_kept;           // [b_cap][IVFB_KEPT] each warp's best keys
  uint64_t *b_drop;           // [b_cap][IVFB_WARPS] the best key each warp dropped
  stb_hit *b_hits;            // [b_cap][1024] hits of the host form
  uint32_t *b_status;         // [b_cap][2]
  uint32_t last_info[4];      // {nq, nprobe, top_k, rerank} of the last batch launch (nq = 0: none yet)
  bool last_filtered;         // the last batch launch was a filtered search's
  // filtered search scratch (the eligibility pass), grown on demand
  uint32_t *f_bitmap;         // [f_words] eligible local rows; f_words >= ceil(n / 32)
  uint64_t f_words;
  uint32_t *f_elig;           // [nlist] eligible codes per list
  uint32_t *f_ranges;         // [f_ranges_cap][2] clipped local ranges
  uint32_t f_ranges_cap;
};

// ------------------------------------------------------------------ assignment GEMM ---
// best[row] = argmax_j  x_row . c_j   (f32, 64x64 block tile, 4x4 per thread, K chunks of 32)
__global__ void __launch_bounds__(256)
ivf_assign_kernel(const float *__restrict__ X, uint64_t n, const float *__restrict__ C, uint32_t nlist,
                  uint32_t *__restrict__ assign) {
  __shared__ float As[32][64 + 4];
  __shared__ float Bs[32][64 + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const uint64_t row0 = (uint64_t)blockIdx.x * 64;
  float best[4];
  uint32_t bidx[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { best[i] = -CUDART_INF_F; bidx[i] = 0; }
  for (uint32_t c0 = 0; c0 < nlist; c0 += 64) {
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int k0 = 0; k0 < STB_D; k0 += 32) {
      // each thread loads 8 floats of A and of B: element e = tid + 256*u -> (r = e/32, k = e%32)
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int e = tid + 256 * u, r = e >> 5, k = e & 31;
        const uint64_t gr = row0 + r;
        As[k][r] = (gr < n) ? __ldg(X + gr * STB_D + k0 + k) : 0.f;
        const uint32_t gc = c0 + r;
        Bs[k][r] = (gc < nlist) ? __ldg(C + (size_t)gc * STB_D + k0 + k) : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 32; ++k) {
        const float4 a = *reinterpret_cast<const float4 *>(&As[k][ty * 4]);
        const float4 b = *reinterpret_cast<const float4 *>(&Bs[k][tx * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t c = c0 + tx * 4 + j;
        if (c < nlist && acc[i][j] > best[i]) { best[i] = acc[i][j]; bidx[i] = c; }
      }
  }
  // reduce over the 16 tx threads of a row group (consecutive lanes of a half-warp)
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int off = 8; off > 0; off >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best[i], off);
      const uint32_t oi = __shfl_xor_sync(0xffffffffu, bidx[i], off);
      if (ov > best[i] || (ov == best[i] && oi < bidx[i])) { best[i] = ov; bidx[i] = oi; }
    }
    const uint64_t gr = row0 + ty * 4 + i;
    if (tx == 0 && gr < n) assign[gr] = bidx[i];
  }
}

// ---------------------------------------------------------------- k-means updates -----
// K1's forced-candidate rule on the fp32 ||x||^2 (NaN and +inf included: a non-finite component
// makes ss NaN or +inf).
__device__ __forceinline__ bool ivf_forced(float ss) { return !(ss >= 1e-30f && ss <= 1e30f); }

// fp32 ||x||^2 of a row held as 8 floats per lane of a full warp
__device__ __forceinline__ float ivf_warp_ss(float4 v0, float4 v1) {
  float ss = v0.x * v0.x + v0.y * v0.y + v0.z * v0.z + v0.w * v0.w + v1.x * v1.x + v1.y * v1.y + v1.z * v1.z + v1.w * v1.w;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
  return ss;
}

// Loads into (v0, v1) the first row r, r+1, ... (mod n, at most 32 tries) that is not forced and
// leaves its index in r; zeros and false if all of them are forced.  Seeds of centroids and codebook
// entries come from here, so no seed is non-finite.
__device__ __forceinline__ bool ivf_load_seed_row(const float4 *X, uint64_t n, uint64_t stride, uint64_t &r, float4 &v0,
                                                  float4 &v1) {
  const int lane = threadIdx.x & 31;
  for (int t = 0; t < 32; ++t, r = (r + 1) % n) {
    v0 = __ldg(X + r * stride * STB_ROW_F4 + 2 * lane); v1 = __ldg(X + r * stride * STB_ROW_F4 + 2 * lane + 1);
    if (!ivf_forced(ivf_warp_ss(v0, v1))) return true;
  }
  v0 = v1 = make_float4(0.f, 0.f, 0.f, 0.f);
  return false;
}

// sums[c] += x^ (normalised row), counts[c] += 1   (warp per row; forced rows are skipped)
__global__ void ivf_accumulate_kernel(const float4 *__restrict__ X, uint64_t n, uint64_t stride,
                                      const uint32_t *__restrict__ assign, float *sums, uint32_t *counts) {
  const int lane = threadIdx.x & 31;
  const uint64_t i = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= n) return;
  const float4 v0 = __ldg(X + i * stride * STB_ROW_F4 + 2 * lane), v1 = __ldg(X + i * stride * STB_ROW_F4 + 2 * lane + 1);
  const float ss = ivf_warp_ss(v0, v1);
  if (ivf_forced(ss)) return;
  const float inv = rsqrtf(ss);
  float *dst = sums + (size_t)assign[i] * STB_D + 8 * lane;
  atomicAdd(dst + 0, v0.x * inv); atomicAdd(dst + 1, v0.y * inv); atomicAdd(dst + 2, v0.z * inv); atomicAdd(dst + 3, v0.w * inv);
  atomicAdd(dst + 4, v1.x * inv); atomicAdd(dst + 5, v1.y * inv); atomicAdd(dst + 6, v1.z * inv); atomicAdd(dst + 7, v1.w * inv);
  if (lane == 0) atomicAdd(counts + assign[i], 1u);
}

// centroid = normalise(sum); empty cluster -> re-seeded from a sample row that is not forced
__global__ void ivf_finish_centroids_kernel(float *C, const float *sums, const uint32_t *counts, uint32_t nlist,
                                            const float4 *X, uint64_t n, uint64_t stride, uint32_t iter) {
  const int lane = threadIdx.x & 31;
  const uint32_t c = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (c >= nlist) return;
  float4 v0, v1;
  if (counts[c] > 0) {
    v0 = *reinterpret_cast<const float4 *>(sums + (size_t)c * STB_D + 8 * lane);
    v1 = *reinterpret_cast<const float4 *>(sums + (size_t)c * STB_D + 8 * lane + 4);
  } else {
    uint64_t r = ((uint64_t)c * 2654435761ull + (uint64_t)iter * 40503ull) % n;
    ivf_load_seed_row(X, n, stride, r, v0, v1);
  }
  const float ss = ivf_warp_ss(v0, v1);
  const float inv = ss > 0.f ? rsqrtf(ss) : 0.f;
  float *dst = C + (size_t)c * STB_D + 8 * lane;
  dst[0] = v0.x * inv; dst[1] = v0.y * inv; dst[2] = v0.z * inv; dst[3] = v0.w * inv;
  dst[4] = v1.x * inv; dst[5] = v1.y * inv; dst[6] = v1.z * inv; dst[7] = v1.w * inv;
}

// ------------------------------------------------------------------ PQ train / encode --
// Lane s of a warp owns sub-space s (8 dims) of the residual x^ - c(x) of one row.
// mode 0: accumulate into the code's sums/counts (k-means step; forced rows are skipped);
// mode 1: write the code (a forced row's code is never read: the row stays out of the lists).
// The 256 KB of codebooks do not fit in shared memory: a launch handles sub-spaces
// [s0, s0+8) (64 KB), 4 rows per warp step (lane = row_in_group*8 + sub-space).
struct PqArgs {
  const float4 *X; uint64_t n, stride;
  const uint32_t *assign; const float *C; const float *cb;   // cb [32][256][8]
  float *sums; uint32_t *counts;                             // [32][256][8], [32][256]
  uint8_t *codes_out;                                        // [n][32] (row order)
  int s0, mode;
};
__global__ void __launch_bounds__(256)
pq_step_kernel(const PqArgs a) {
  extern __shared__ float s_cb[];   // [8][256][8]
  for (int i = threadIdx.x; i < 8 * PQ_KSUB * PQ_DSUB; i += blockDim.x)
    s_cb[i] = a.cb[(size_t)a.s0 * PQ_KSUB * PQ_DSUB + i];
  __syncthreads();
  const int lane = threadIdx.x & 31, rl = lane >> 3, sl = lane & 7;
  const uint64_t warp = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const uint64_t nwarps = (uint64_t)gridDim.x * (blockDim.x >> 5);
  for (uint64_t g = warp; g * 4 < a.n; g += nwarps) {
    const uint64_t i = g * 4 + rl;
    const bool valid = i < a.n;
    const uint64_t ic = valid ? i : a.n - 1;
    // row norm: every lane of the 8-lane group reads a different eighth of the row
    const float4 *xr = a.X + ic * a.stride * STB_ROW_F4;
    float ss = 0.f;
#pragma unroll
    for (int u = 0; u < 8; ++u) { const float4 v = __ldg(xr + sl * 8 + u); ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w; }
    ss += __shfl_xor_sync(0xffffffffu, ss, 4); ss += __shfl_xor_sync(0xffffffffu, ss, 2); ss += __shfl_xor_sync(0xffffffffu, ss, 1);
    const float inv = (ss > 0.f && ss < CUDART_INF_F) ? rsqrtf(ss) : 0.f;
    const int s = a.s0 + sl;
    const float4 x0 = __ldg(xr + s * 2), x1 = __ldg(xr + s * 2 + 1);
    const float4 *cr = reinterpret_cast<const float4 *>(a.C + (size_t)a.assign[ic] * STB_D);
    const float4 c0 = __ldg(cr + s * 2), c1 = __ldg(cr + s * 2 + 1);
    const float r[8] = {x0.x * inv - c0.x, x0.y * inv - c0.y, x0.z * inv - c0.z, x0.w * inv - c0.w,
                        x1.x * inv - c1.x, x1.y * inv - c1.y, x1.z * inv - c1.z, x1.w * inv - c1.w};
    float bd = CUDART_INF_F;
    int bc = 0;
    const float *cb = s_cb + (size_t)sl * PQ_KSUB * PQ_DSUB;
    for (int code = 0; code < PQ_KSUB; ++code) {
      const float4 e0 = *reinterpret_cast<const float4 *>(cb + code * 8), e1 = *reinterpret_cast<const float4 *>(cb + code * 8 + 4);
      float d = (r[0] - e0.x) * (r[0] - e0.x);
      d = fmaf(r[1] - e0.y, r[1] - e0.y, d); d = fmaf(r[2] - e0.z, r[2] - e0.z, d); d = fmaf(r[3] - e0.w, r[3] - e0.w, d);
      d = fmaf(r[4] - e1.x, r[4] - e1.x, d); d = fmaf(r[5] - e1.y, r[5] - e1.y, d); d = fmaf(r[6] - e1.z, r[6] - e1.z, d);
      d = fmaf(r[7] - e1.w, r[7] - e1.w, d);
      if (d < bd) { bd = d; bc = code; }
    }
    if (!valid) continue;
    if (a.mode == 0) {
      if (ivf_forced(ss)) continue;
      float *dst = a.sums + ((size_t)s * PQ_KSUB + bc) * PQ_DSUB;
#pragma unroll
      for (int d = 0; d < 8; ++d) atomicAdd(dst + d, r[d]);
      atomicAdd(a.counts + s * PQ_KSUB + bc, 1u);
    } else {
      a.codes_out[i * PQ_M + s] = (uint8_t)bc;
    }
  }
}

__global__ void pq_finish_codebooks_kernel(float *cb, const float *sums, const uint32_t *counts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;      // (s, code)
  if (i >= PQ_M * PQ_KSUB) return;
  const uint32_t c = counts[i];
  if (c == 0) return;                                        // keep the previous entry
  for (int d = 0; d < 8; ++d) cb[(size_t)i * 8 + d] = sums[(size_t)i * 8 + d] / (float)c;
}

// seed codebooks from residuals of 256 sample rows that are not forced (a zero entry if none is found)
__global__ void pq_seed_kernel(float *cb, const float4 *X, uint64_t n, uint64_t stride, const uint32_t *assign, const float *C) {
  const int code = blockIdx.x, lane = threadIdx.x;          // 256 blocks x 32 lanes (lane = sub-space)
  uint64_t i = ((uint64_t)code * 7919u) % n;
  float4 x0, x1;
  float *dst = cb + ((size_t)lane * PQ_KSUB + code) * PQ_DSUB;
  if (!ivf_load_seed_row(X, n, stride, i, x0, x1)) {
    for (int d = 0; d < 8; ++d) dst[d] = 0.f;
    return;
  }
  const float inv = rsqrtf(ivf_warp_ss(x0, x1));
  const float4 *cr = reinterpret_cast<const float4 *>(C + (size_t)assign[i] * STB_D);
  const float4 c0 = __ldg(cr + lane * 2), c1 = __ldg(cr + lane * 2 + 1);
  dst[0] = x0.x * inv - c0.x; dst[1] = x0.y * inv - c0.y; dst[2] = x0.z * inv - c0.z; dst[3] = x0.w * inv - c0.w;
  dst[4] = x1.x * inv - c1.x; dst[5] = x1.y * inv - c1.y; dst[6] = x1.z * inv - c1.z; dst[7] = x1.w * inv - c1.w;
}

// ------------------------------------------------------------------ inverted lists ----
// Every change of the lists -- the build's add phase over [0, n), stb_ivfpq_extend, stb_ivfpq_update and
// stb_ivfpq_remove -- is one edit (IvfEdit, host side below): some old entries leave, the others are
// renumbered, and m new entries join their lists.
//   ivf_assign_kernel, pq_step_kernel mode 1   list and code of each new row (each row's arithmetic is
//                                              independent of its place in the launch and of where the row
//                                              is read from: a copy of an indexed row gets that row's list
//                                              and code bit for bit)
//   ivf_flag_forced_kernel                     forced rows: assign = IVF_NO_LIST, counted
//   ivf_hist_kernel                            new rows per list; the sort's values 0..m-1
//   cub::DeviceRadixSort::SortPairs            stable bucketing: keys = list id (the low bits that separate
//                                              0..nlist-1 from IVF_NO_LIST), values = new entry i.  An LSD radix
//                                              sort is stable, so each list's new entries stay ascending and the
//                                              forced rows come last, ascending; no atomic decides a position.
// An edit that drops entries (update, remove) describes the old indexed rows that stay as kept segments
// {[begin, end), dst}: row r of segment k becomes dst_k + r - begin_k (dst_k = begin_k for an update).
//   ivff_bitmap_kernel                         kept-row bitmap from the segments
//   ivff_elig_kernel                           kept entries per list
//   ivf_compact_kernel                         surviving entries of each list, in list order, renumbered
//   ivf_merge_kernel                           the new codes / order: list l = a merge by row of its survivors
//                                              (every old entry for extend and build) and its new entries.
// The forced side list (at most IVF_FORCED_CAP rows) is filtered, renumbered and merged on the host.
// So every list and the forced list are in ascending row order, and the index is a function of the
// quantisers and the rows: any sequence of edits reaching the same rows gives the same arrays.  CUB rather
// than a hand-written counting scatter: it is stable by construction, takes 2 passes for nlist <= 8192
// (14 key bits) and ships header-only with the toolkit.

// forced rows (warp per row): assign[i] = IVF_NO_LIST, counted in *n_forced
__global__ void ivf_flag_forced_kernel(const float4 *__restrict__ X, uint64_t n, uint32_t *assign, uint32_t *n_forced) {
  const int lane = threadIdx.x & 31;
  const uint64_t i = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= n) return;
  const float4 v0 = __ldg(X + i * STB_ROW_F4 + 2 * lane), v1 = __ldg(X + i * STB_ROW_F4 + 2 * lane + 1);
  if (!ivf_forced(ivf_warp_ss(v0, v1)) || lane != 0) return;
  assign[i] = IVF_NO_LIST;
  atomicAdd(n_forced, 1u);
}
// hist[l] = new rows of list l (forced rows not counted); idx[i] = i
__global__ void ivf_hist_kernel(const uint32_t *assign, uint64_t n, uint32_t *hist, uint32_t *idx) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  idx[i] = (uint32_t)i;
  if (assign[i] != IVF_NO_LIST) atomicAdd(hist + assign[i], 1u);
}

// Survivors of an edit that drops entries (warp per list, one pass over the list in order): entry i of
// list l whose row is set in `bitmap` goes to position surv_off[l] + (survivors of l before it), with
// surv_pos = i and surv_row = its renumbered row (binary search of the kept segment holding it).
__global__ void ivf_compact_kernel(const uint32_t *__restrict__ list_off, const uint32_t *__restrict__ order, uint32_t nlist,
                                   const uint32_t *__restrict__ bitmap, const uint32_t *__restrict__ kept,
                                   const uint32_t *__restrict__ kept_dst, uint32_t n_kept,
                                   const uint32_t *__restrict__ surv_off, uint32_t *surv_pos, uint32_t *surv_row) {
  const uint32_t lane = threadIdx.x & 31, l = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (l >= nlist) return;
  const uint32_t b = __ldg(list_off + l), e = __ldg(list_off + l + 1);
  uint32_t out = __ldg(surv_off + l);
  for (uint32_t i0 = b; i0 < e; i0 += 32) {
    const uint32_t i = i0 + lane;
    uint32_t row = 0;
    bool keep = false;
    if (i < e) { row = __ldg(order + i); keep = (__ldg(bitmap + (row >> 5)) >> (row & 31)) & 1u; }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      uint32_t lo = 0, hi = n_kept;   // the last segment with begin <= row (it holds the row: its bit is set)
      while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(kept + 2 * mid) <= row) lo = mid; else hi = mid; }
      const uint32_t p = out + __popc(bal & ((1u << lane) - 1u));
      surv_pos[p] = i;
      surv_row[p] = __ldg(kept_dst + lo) + (row - __ldg(kept + 2 * lo));
    }
    out += __popc(bal);
  }
}

// Thread per entry of the new lists.  Position o < n_out lies in list l (new_off[l] <= o < new_off[l+1]).
// List l merges its ns survivors (positions surv_off[l].. of the survivor arrays; without them, the old
// list itself) with its nn new entries (sorted positions new_off[l] - surv_off[l] ..), both ascending by row
// and disjoint.  A merge-path binary search finds i = survivors among the list's first `within` outputs;
// output `within` is then the smaller of survivor i and new entry within - i.  For an extend every new row
// is larger than every old one: i = min(within, ns), i.e. the old entries, then the new rows.
struct MergeArgs {
  const uint8_t *old_codes; const uint32_t *old_order;
  const uint32_t *surv_off, *new_off; uint32_t nlist;
  const uint32_t *surv_pos, *surv_row;        // survivors (null: every old entry, unrenumbered; surv_off = old offsets)
  const uint8_t *codes_row; const uint32_t *sorted; const uint32_t *new_rows; uint64_t first;   // new entry i: code
                                              // codes_row[i], row new_rows[i] (null: first + i)
  uint32_t n_out;
  uint8_t *codes; uint32_t *order;
};
__device__ __forceinline__ uint32_t ivf_surv_row(const MergeArgs &a, uint32_t s) {
  return a.surv_row ? __ldg(a.surv_row + s) : __ldg(a.old_order + s);
}
__device__ __forceinline__ uint32_t ivf_new_row(const MergeArgs &a, uint32_t i) {
  return a.new_rows ? __ldg(a.new_rows + i) : (uint32_t)(a.first + i);
}
__global__ void __launch_bounds__(256)
ivf_merge_kernel(const MergeArgs a) {
  const uint64_t o = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= a.n_out) return;
  uint32_t lo = 0, hi = a.nlist;      // the list l with new_off[l] <= o < new_off[l+1]
  while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(a.new_off + mid) <= o) lo = mid; else hi = mid; }
  const uint32_t nb0 = __ldg(a.new_off + lo), within = (uint32_t)o - nb0;
  const uint32_t sb = __ldg(a.surv_off + lo), ns = __ldg(a.surv_off + lo + 1) - sb;
  const uint32_t nb = nb0 - sb, nn = __ldg(a.new_off + lo + 1) - nb0 - ns;
  uint32_t i = within > nn ? within - nn : 0, ie = min(within, ns);
  while (i < ie) {
    const uint32_t mid = (i + ie) >> 1;
    if (ivf_surv_row(a, sb + mid) < ivf_new_row(a, __ldg(a.sorted + nb + within - mid - 1))) i = mid + 1; else ie = mid;
  }
  const uint32_t j = within - i;
  const uint4 *src;
  uint32_t row;
  uint32_t nj = 0, nrow = 0;
  if (j < nn) { nj = __ldg(a.sorted + nb + j); nrow = ivf_new_row(a, nj); }
  if (i < ns && (j >= nn || ivf_surv_row(a, sb + i) < nrow)) {
    const uint32_t pos = a.surv_pos ? __ldg(a.surv_pos + sb + i) : sb + i;
    src = reinterpret_cast<const uint4 *>(a.old_codes + (size_t)pos * PQ_M);
    row = ivf_surv_row(a, sb + i);
  } else {
    src = reinterpret_cast<const uint4 *>(a.codes_row + (size_t)nj * PQ_M);
    row = nrow;
  }
  uint4 *dst = reinterpret_cast<uint4 *>(a.codes + o * PQ_M);
  const uint4 c0 = __ldg(src), c1 = __ldg(src + 1);
  dst[0] = c0; dst[1] = c1;
  a.order[o] = row;
}

// ------------------------------------------------------------------ query arithmetic --
// Every query kernel, single and batched, computes the coarse scores, the LUT and the ADC scores
// with these helpers, so a query's values are the same bits whichever path computes them.

// c . q and q . q of a centroid and a query held as 8 floats per lane of a full warp (lane L holds
// dims 8L..8L+7), each reduced over the warp by an xor butterfly; every lane ends with both sums.
__device__ __forceinline__ void ivf_coarse_dot(float4 a0, float4 a1, float4 b0, float4 b1, float &d, float &qq) {
  d = a0.x * b0.x + a0.y * b0.y + a0.z * b0.z + a0.w * b0.w + a1.x * b1.x + a1.y * b1.y + a1.z * b1.z + a1.w * b1.w;
  qq = b0.x * b0.x + b0.y * b0.y + b0.z * b0.z + b0.w * b0.w + b1.x * b1.x + b1.y * b1.y + b1.z * b1.z + b1.w * b1.w;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) { d += __shfl_xor_sync(0xffffffffu, d, off); qq += __shfl_xor_sync(0xffffffffu, qq, off); }
}
// coarse score q^ . c from ivf_coarse_dot's sums (0 for a query whose q . q is not positive)
__device__ __forceinline__ float ivf_coarse_score(float d, float qq) { return qq > 0.f ? d * rsqrtf(qq) : 0.f; }

// 1 / ||q|| of the query in shared memory: serial fp32 sum in index order (one thread)
__device__ __forceinline__ float ivf_query_inv(const float *sq) {
  float s = 0.f;
  for (int i = 0; i < STB_D; ++i) s += sq[i] * sq[i];
  return s > 0.f ? rsqrtf(s) : 0.f;
}

// LUT entry i = (sub-space s = i / 256, code i % 256): FMA chain of q^_s . cb[s][code]
__device__ __forceinline__ float ivf_lut_entry(const float *sq, float inv, const float *cb, int i) {
  const int sub = i / PQ_KSUB;
  const float *e = cb + (size_t)i * PQ_DSUB;
  float d = 0.f;
#pragma unroll
  for (int t = 0; t < 8; ++t) d = fmaf(sq[sub * 8 + t] * inv, e[t], d);
  return d;
}


// ADC score of a code (its 32 bytes in c0, c1): s (its list's coarse score) + LUT[0][c0] + ... +
// LUT[31][c31], in that order.  Only fp32 additions in a fixed order, so the bits are those of any
// such sum (numpy reproduces them).  ivf_adc_kernel and ivf_adc_finish_kernel spell the same sum out
// inline: routed through this helper, the compiler assigns their registers differently.
__device__ __forceinline__ float ivf_adc_sum(const float *s_lut, uint4 c0, uint4 c1, float s) {
  const uint32_t w[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    s += s_lut[(4 * i + 0) * PQ_KSUB + (w[i] & 0xff)];
    s += s_lut[(4 * i + 1) * PQ_KSUB + ((w[i] >> 8) & 0xff)];
    s += s_lut[(4 * i + 2) * PQ_KSUB + ((w[i] >> 16) & 0xff)];
    s += s_lut[(4 * i + 3) * PQ_KSUB + (w[i] >> 24)];
  }
  return s;
}

// ------------------------------------------------------------------ query kernels -----
// coarse[j] = q^ . c_j   (warp per centroid)
__global__ void ivf_coarse_kernel(const float *C, uint32_t nlist, const float *q, float *coarse) {
  const int lane = threadIdx.x & 31;
  const uint32_t c = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (c >= nlist) return;
  const float4 *cr = reinterpret_cast<const float4 *>(C + (size_t)c * STB_D), *q4 = reinterpret_cast<const float4 *>(q);
  const float4 a0 = __ldg(cr + 2 * lane), a1 = __ldg(cr + 2 * lane + 1), b0 = __ldg(q4 + 2 * lane), b1 = __ldg(q4 + 2 * lane + 1);
  float d, qq;
  ivf_coarse_dot(a0, a1, b0, b1, d, qq);
  if (lane == 0) coarse[c] = ivf_coarse_score(d, qq);
}

// one CTA: top-nprobe lists (bitonic sort of <= 8192 keys), prefix of their lengths, LUT
__global__ void __launch_bounds__(1024)
ivf_probe_lut_kernel(const float *coarse, uint32_t nlist, uint32_t nprobe, const uint32_t *list_off, const float *cb,
                     const float *q, uint32_t *probe, float *lut) {
  extern __shared__ uint64_t skeys[];   // npow2 keys
  __shared__ float sq[STB_D];
  __shared__ float s_inv;
  uint32_t npow = 1; while (npow < nlist) npow <<= 1;
  for (uint32_t i = threadIdx.x; i < npow; i += blockDim.x)
    skeys[i] = (i < nlist) ? stb_make_key(coarse[i], i) : STB_KEY_INVALID;
  if (threadIdx.x < STB_D) sq[threadIdx.x] = q[threadIdx.x];
  __syncthreads();
  if (threadIdx.x == 0) s_inv = ivf_query_inv(sq);
  stb_cta_sort_keys_strided(skeys, npow);
  // probe[0..nprobe) = list ids (best first); probe[nprobe_max .. ] = prefix of list lengths
  if (threadIdx.x == 0) {
    uint32_t acc = 0;
    for (uint32_t p = 0; p < nprobe; ++p) {
      const uint32_t l = stb_key_row(skeys[p]);
      probe[p] = l;
      probe[nprobe + p] = acc;
      acc += list_off[l + 1] - list_off[l];
    }
    probe[2 * nprobe] = acc;
  }
  const float inv = s_inv;
  for (int i = threadIdx.x; i < PQ_M * PQ_KSUB; i += blockDim.x) lut[i] = ivf_lut_entry(sq, inv, cb, i);
}

// ADC scan over the probed lists: lane = one code (32 bytes); score = coarse[list] + sum LUT.
// Rows are dealt to warps 32 at a time round-robin (a list's -- i.e. a cluster's -- rows
// spread over all warps); each warp keeps its 64 best in registers (same running top-K'
// structure as K1) and emits them as stb_hit {-score, pos}.
struct AdcArgs {
  const uint8_t *codes; const uint32_t *list_off; const uint32_t *probe; uint32_t nprobe;
  const float *coarse; const float *lut; stb_hit *cand;
};
struct AdcTop {          // 2 entries per lane = 64 per warp
  float ls[2]; uint32_t lr[2]; float thr; int lane;
  __device__ __forceinline__ void init() {
    ls[0] = ls[1] = -CUDART_INF_F; lr[0] = lr[1] = 0xffffffffu; thr = -CUDART_INF_F; lane = threadIdx.x & 31;
  }
  __device__ __forceinline__ void insert(float cs, uint32_t cr) {
    const float m = fminf(ls[0], ls[1]);
    const int mi = ls[1] < ls[0] ? 1 : 0;
    const unsigned owners = __ballot_sync(0xffffffffu, m == thr);
    if (lane == __ffs(owners) - 1) { if (mi == 0) { ls[0] = cs; lr[0] = cr; } else { ls[1] = cs; lr[1] = cr; } }
    float t = fminf(ls[0], ls[1]);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) t = fminf(t, __shfl_xor_sync(0xffffffffu, t, off));
    thr = t;
  }
  __device__ __forceinline__ void push(float s, uint32_t r) {
    unsigned mask = __ballot_sync(0xffffffffu, s > thr);
    while (mask) {
      const int src = __ffs(mask) - 1;
      mask &= mask - 1;
      const float cs = __shfl_sync(0xffffffffu, s, src);
      const uint32_t cr = __shfl_sync(0xffffffffu, r, src);
      if (cs > thr) insert(cs, cr);
    }
  }
};
__global__ void __launch_bounds__(256)
ivf_adc_kernel(const AdcArgs a) {
  __shared__ float s_lut[PQ_M * PQ_KSUB];      // 32 KB
  for (int i = threadIdx.x; i < PQ_M * PQ_KSUB; i += blockDim.x) s_lut[i] = a.lut[i];
  __syncthreads();
  const uint32_t total = a.probe[2 * a.nprobe];
  const int lane = threadIdx.x & 31;
  const uint32_t warp = blockIdx.x * 8 + (threadIdx.x >> 5), n_warps = gridDim.x * 8;
  AdcTop top;
  top.init();
  for (uint64_t g = warp; g * 32 < total; g += n_warps) {
    const uint64_t v = g * 32 + lane;
    float s = -CUDART_INF_F;
    uint32_t pos = 0;
    if (v < total) {
      uint32_t lo = 0, hi = a.nprobe;      // probe p with prefix[p] <= v < prefix[p+1]
      while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (a.probe[a.nprobe + mid] <= v) lo = mid; else hi = mid; }
      const uint32_t l = a.probe[lo];
      pos = a.list_off[l] + (uint32_t)(v - a.probe[a.nprobe + lo]);
      const uint4 *cp = reinterpret_cast<const uint4 *>(a.codes + (size_t)pos * PQ_M);
      const uint4 c0 = __ldg(cp), c1 = __ldg(cp + 1);
      const uint32_t w[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
      s = a.coarse[l];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s += s_lut[(4 * i + 0) * PQ_KSUB + (w[i] & 0xff)];
        s += s_lut[(4 * i + 1) * PQ_KSUB + ((w[i] >> 8) & 0xff)];
        s += s_lut[(4 * i + 2) * PQ_KSUB + ((w[i] >> 16) & 0xff)];
        s += s_lut[(4 * i + 3) * PQ_KSUB + (w[i] >> 24)];
      }
    }
    top.push(s, pos);
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    stb_hit h;
    const bool ok = top.lr[e] != 0xffffffffu || top.ls[e] > -CUDART_INF_F;
    h.distance = ok ? -(double)top.ls[e] : CUDART_INF;
    h.row = ok ? (uint64_t)top.lr[e] : 0xffffffffffffffffull;
    a.cand[(size_t)warp * 64 + e * 32 + lane] = h;
  }
}

// cand_rows[i] = order[pos of the i-th best candidate]
__global__ void ivf_pick_rows_kernel(const stb_hit *cand, uint32_t r, const uint32_t *order, uint32_t *rows, uint32_t *n_valid) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= r) return;
  const uint64_t pos = cand[i].row;
  if (pos != 0xffffffffffffffffull) { rows[i] = order[pos]; atomicAdd(n_valid, 1u); }
  else rows[i] = 0xffffffffu;
}

// ------------------------------------------------------------------ fused search (v2) ---
// Two launches and ONE host synchronisation per query (v1: ~25 launches, 4-5 syncs):
//   ivf_coarse_probe_kernel  coarse scores (warp per centroid); the LAST CTA to finish sorts
//                            them, writes the probe list + prefix sums and the ADC table.
//   ivf_adc_finish_kernel    ADC scan (32-row chunks dealt round-robin over CTAs first, then
//                            warps, so a tight cluster's contiguous codes spread over every
//                            CTA); each warp keeps its 64 best, each CTA its ADC2_KEEP best; the
//                            LAST CTA sorts the 32 x 64 = 2048 survivors, re-scores the best
//                            `rerank` rows and the forced rows exactly (canonical f64, as K1) and
//                            writes the top-k hits.
// The funnel returns the `rerank` best ADC scores exactly when no warp and no CTA of the deal holds
// more than 64 of them (every code is re-ranked when the probed lists hold <= 2048 codes).
// stb_ivfpq_search runs it iff rerank <= ADC2_RERANK_CAP and top_k <= 1024, else the multi-launch search above.
#define ADC2_THREADS 512
#define ADC2_MAX_CTAS 32
#define ADC2_KEEP 64        // per CTA; chunks are dealt round-robin over the 32 CTAs, so each sees a uniform sample: ~16 of the best 512 land in one CTA
#define ADC2_RERANK_CAP 1024
#define ADC2_SMEM 65536

struct Probe2Args {
  const float *C; uint32_t nlist, nprobe; const float *q; float *coarse; const uint32_t *list_off; const float *cb;
  uint32_t *probe; float *lut; unsigned int *ticket;
};

__global__ void __launch_bounds__(1024)
ivf_coarse_probe_kernel(const Probe2Args a) {
  extern __shared__ uint64_t p2_keys[];   // npow2 keys (last CTA only)
  __shared__ float sq[STB_D];
  __shared__ float s_inv;
  __shared__ unsigned s_last;
  const int lane = threadIdx.x & 31;
  const uint32_t c = blockIdx.x * 32 + (threadIdx.x >> 5);
  if (c < a.nlist) {
    const float4 *cr = reinterpret_cast<const float4 *>(a.C + (size_t)c * STB_D), *q4 = reinterpret_cast<const float4 *>(a.q);
    const float4 a0 = __ldg(cr + 2 * lane), a1 = __ldg(cr + 2 * lane + 1), b0 = __ldg(q4 + 2 * lane), b1 = __ldg(q4 + 2 * lane + 1);
    float d, qq;
    ivf_coarse_dot(a0, a1, b0, b1, d, qq);
    if (lane == 0) { a.coarse[c] = ivf_coarse_score(d, qq); __threadfence(); }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = (atomicAdd(a.ticket, 1u) == gridDim.x - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // ---- last CTA: every coarse score is visible (read through L2)
  uint32_t npow = 1; while (npow < a.nlist) npow <<= 1;
  for (uint32_t i = threadIdx.x; i < npow; i += blockDim.x)
    p2_keys[i] = (i < a.nlist) ? stb_make_key(__ldcg(a.coarse + i), i) : STB_KEY_INVALID;
  if (threadIdx.x < STB_D) sq[threadIdx.x] = a.q[threadIdx.x];
  __syncthreads();
  if (threadIdx.x == 0) s_inv = ivf_query_inv(sq);
  stb_cta_sort_keys_strided(p2_keys, npow);
  // list sizes in parallel (one thread per probed list), then a serial prefix over shared memory:
  // a single thread chasing 2 x nprobe dependent global loads cost ~20 us of this kernel's 62
  __shared__ uint32_t s_sz[1024];
  if (threadIdx.x < a.nprobe) {
    const uint32_t l = stb_key_row(p2_keys[threadIdx.x]);
    a.probe[threadIdx.x] = l;
    s_sz[threadIdx.x] = __ldg(a.list_off + l + 1) - __ldg(a.list_off + l);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t acc = 0;
    for (uint32_t p = 0; p < a.nprobe; ++p) { a.probe[a.nprobe + p] = acc; acc += s_sz[p]; }
    a.probe[2 * a.nprobe] = acc;
    *a.ticket = 0;                                   // ready for the next query (stream-ordered)
  }
  const float inv = s_inv;
  for (int i = threadIdx.x; i < PQ_M * PQ_KSUB; i += blockDim.x) a.lut[i] = ivf_lut_entry(sq, inv, a.cb, i);
}

struct Adc2Args {
  const uint8_t *codes; const uint32_t *list_off; const uint32_t *probe; uint32_t nprobe;
  const float *coarse; const float *lut; const uint32_t *order;
  uint64_t *keys2; unsigned int *ticket;
  const float4 *rows; uint64_t row_base; const float *q; uint32_t top_k, rerank;
  const uint32_t *forced; uint32_t n_forced;   // re-ranked in addition to the ADC candidates
  stb_hit *out_hits; uint32_t *out_status;     // status: [0] hits, [1] codes scanned
};

__global__ void __launch_bounds__(ADC2_THREADS, 1)
ivf_adc_finish_kernel(const Adc2Args a) {
  extern __shared__ __align__(16) uint8_t dyn[];          // 64 KiB
  float *s_lut = reinterpret_cast<float *>(dyn);          // [0, 32 KiB) during the scan
  uint64_t *s_keys = reinterpret_cast<uint64_t *>(dyn + 32768);   // 1024 keys during the CTA reduction
  __shared__ double sqd[STB_D];
  __shared__ double s_q2;
  __shared__ unsigned s_last;
  __shared__ int s_pass;
  const uint32_t tid = threadIdx.x;
  const int lane = tid & 31;
  const uint32_t warp_in = tid >> 5, n_ctas = gridDim.x;
  for (uint32_t i = tid; i < PQ_M * PQ_KSUB; i += ADC2_THREADS) s_lut[i] = a.lut[i];
  __syncthreads();
  const uint32_t total = a.probe[2 * a.nprobe];
  AdcTop top;
  top.init();
  // chunk g (32 consecutive codes) -> CTA g % n_ctas, warp (g / n_ctas) % 16
  for (uint64_t g = blockIdx.x + (uint64_t)n_ctas * warp_in; g * 32 < total; g += (uint64_t)n_ctas * (ADC2_THREADS / 32)) {
    const uint64_t v = g * 32 + lane;
    float s = -CUDART_INF_F;
    uint32_t pos = 0;
    if (v < total) {
      uint32_t lo = 0, hi = a.nprobe;
      while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (a.probe[a.nprobe + mid] <= v) lo = mid; else hi = mid; }
      const uint32_t l = a.probe[lo];
      pos = a.list_off[l] + (uint32_t)(v - a.probe[a.nprobe + lo]);
      const uint4 *cp = reinterpret_cast<const uint4 *>(a.codes + (size_t)pos * PQ_M);
      const uint4 c0 = __ldg(cp), c1 = __ldg(cp + 1);
      const uint32_t w[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
      s = a.coarse[l];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s += s_lut[(4 * i + 0) * PQ_KSUB + (w[i] & 0xff)];
        s += s_lut[(4 * i + 1) * PQ_KSUB + ((w[i] >> 8) & 0xff)];
        s += s_lut[(4 * i + 2) * PQ_KSUB + ((w[i] >> 16) & 0xff)];
        s += s_lut[(4 * i + 3) * PQ_KSUB + (w[i] >> 24)];
      }
    }
    top.push(s, pos);
  }
  // CTA reduction: 16 warps x 64 -> the ADC2_KEEP best of this CTA
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const bool ok = top.lr[e] != 0xffffffffu || top.ls[e] > -CUDART_INF_F;
    s_keys[warp_in * 64 + e * 32 + lane] = ok ? stb_make_key(top.ls[e], top.lr[e]) : STB_KEY_INVALID;
  }
  __syncthreads();
  stb_cta_sort_keys_strided(s_keys, (ADC2_THREADS / 32) * 64);
  for (uint32_t i = tid; i < ADC2_KEEP; i += ADC2_THREADS) a.keys2[(size_t)blockIdx.x * ADC2_KEEP + i] = s_keys[i];
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_last = (atomicAdd(a.ticket, 1u) == n_ctas - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // ---- last CTA: global selection + exact re-rank
  uint64_t *fk = reinterpret_cast<uint64_t *>(dyn);       // up to 2048 keys = 16 KiB
  const uint32_t n_all = n_ctas * ADC2_KEEP;
  uint32_t n_sort = 64;
  while (n_sort < n_all) n_sort <<= 1;
  for (uint32_t i = tid; i < n_sort; i += ADC2_THREADS) fk[i] = (i < n_all) ? __ldcg(a.keys2 + i) : STB_KEY_INVALID;
  for (uint32_t i = tid; i < STB_D; i += ADC2_THREADS) sqd[i] = (double)a.q[i];
  if (tid == 0) s_pass = 0;
  __syncthreads();
  stb_cta_sort_keys_strided(fk, n_sort);
  if (tid == 0) s_q2 = stb_canon_q2(sqd);
  __syncthreads();
  const uint32_t r = min(min(a.rerank, (uint32_t)ADC2_RERANK_CAP), n_all);
  uint32_t n2 = 32;
  while (n2 < r + a.n_forced) n2 <<= 1;
  // keys 0..r) live in dyn[0, 8 KiB); the (distance,row) pairs of the r candidates and the forced
  // rows (<= 1024 + IVF_FORCED_CAP) go to dyn[16 KiB, 48 KiB)
  double *sd = reinterpret_cast<double *>(dyn + 16384);
  uint64_t *sr = reinterpret_cast<uint64_t *>(dyn + 16384 + 8 * (ADC2_RERANK_CAP + IVF_FORCED_CAP));
  const double q2 = s_q2;
  for (uint32_t c = tid; c < n2; c += ADC2_THREADS) {
    double d = CUDART_INF;
    uint64_t grow = 0xffffffffffffffffull;
    uint64_t row = 0xffffffffffffffffull;
    if (c < r) {
      const uint64_t key = fk[c];
      if (key != STB_KEY_INVALID) row = a.order[stb_key_row(key)];
    } else if (c < r + a.n_forced) {
      row = a.forced[c - r];
    }
    if (row != 0xffffffffffffffffull) {
      double ab, r2;
      stb_canon_dot<true>(sqd, a.rows + row * STB_ROW_F4, ab, r2);
      const double dist = stb_canon_dist(ab, q2, r2);
      if (dist < STB_DEFAULT_MAX_DIST) { d = dist; grow = a.row_base + row; atomicAdd(&s_pass, 1); }
    }
    sd[c] = d; sr[c] = grow;
  }
  __syncthreads();
  stb_cta_sort_hits(sd, sr, n2);
  const uint32_t n_out = min((uint32_t)s_pass, a.top_k);
  stb_write_hits(a.out_hits, sd, sr, n_out, a.top_k);
  if (tid == 0) { a.out_status[0] = n_out; a.out_status[1] = total; *a.ticket = 0; }
}

// ------------------------------------------------------------------ batched search ------
// nq queries in four launches, each query computed as the single path computes it and selected exactly:
//   ivfb_coarse_kernel     coarse scores [nq][nlist]: a warp per centroid reduces it against a tile of
//                          IVFB_QTILE queries staged in shared memory (ivf_coarse_dot, the single
//                          path's lane split and butterfly, so the same bits).
//   ivfb_probe_lut_kernel  a CTA per query: sort of the coarse keys, probe list + prefix of the list
//                          lengths, LUT [32][256] (ivf_query_inv, ivf_lut_entry).
//   ivfb_scan_kernel       grid (IVFB_SCAN_CTAS, nq): 32-code chunk g of a query's probed codes goes
//                          to CTA g % 8, warp (g / 8) % 8 (a cluster's codes spread over all 64
//                          warps); each warp keeps its IVFB_WARP_KEEP best keys (stb_make_key: ADC
//                          score desc, code position asc) exactly and records the best key it dropped.
//                          Every query reads its own codes: nq x (codes scanned x 32 B).
//   ivfb_finish_kernel     a CTA per query: T = the rerank-th best of the 4096 kept keys.  When no warp
//                          dropped a key better than T, the kept keys hold the `rerank` best codes;
//                          otherwise the query takes the exact slow route: an MSB-first radix select of
//                          the rerank-th best key over all its codes (8 passes of 8 bits, scores
//                          recomputed), then one pass that emits every key at or above it.  The
//                          candidates' rows and the forced rows are re-ranked with the canonical
//                          distance as on every K5 path.
// A code whose ADC score is NaN or -inf (a query with a non-finite component) is no candidate, as on
// the single path.

__global__ void __launch_bounds__(1024)
ivfb_coarse_kernel(const float *C, uint32_t nlist, const float *qs, uint32_t nq, float *coarse) {
  __shared__ float4 sq[IVFB_QTILE][STB_ROW_F4];
  const int lane = threadIdx.x & 31;
  const uint32_t q0 = blockIdx.y * IVFB_QTILE, nt = min((uint32_t)IVFB_QTILE, nq - q0);
  const float4 *q4 = reinterpret_cast<const float4 *>(qs) + (size_t)q0 * STB_ROW_F4;
  for (uint32_t i = threadIdx.x; i < nt * STB_ROW_F4; i += blockDim.x) sq[i / STB_ROW_F4][i % STB_ROW_F4] = __ldg(q4 + i);
  __syncthreads();
  const uint32_t c = blockIdx.x * 32 + (threadIdx.x >> 5);
  if (c >= nlist) return;
  const float4 *cr = reinterpret_cast<const float4 *>(C + (size_t)c * STB_D);
  const float4 a0 = __ldg(cr + 2 * lane), a1 = __ldg(cr + 2 * lane + 1);
  for (uint32_t j = 0; j < nt; ++j) {
    float d, qq;
    ivf_coarse_dot(a0, a1, sq[j][2 * lane], sq[j][2 * lane + 1], d, qq);
    if (lane == 0) coarse[(size_t)(q0 + j) * nlist + c] = ivf_coarse_score(d, qq);
  }
}

// Per query: probe[0, nprobe) list ids, probe[nprobe, 2 nprobe] the prefix of their lengths (the last entry
// is the number of probed codes).  FILTER adds probe[2 nprobe + 1] = the eligible codes of the probed lists.
#define IVFB_PROBE_STRIDE(nprobe, FILTER) (2 * (nprobe) + 1 + (FILTER ? 1 : 0))

// FILTER: only lists with elig[l] > 0 are taken, in the same (coarse score desc, list id asc) order; the
// slots past the min(nprobe, E) lists taken hold IVF_NO_LIST and the total as their prefix, so a search
// of the prefix never lands on them.
template <bool FILTER>
__global__ void __launch_bounds__(1024)
ivfb_probe_lut_kernel(const float *coarse, uint32_t nlist, uint32_t nprobe, const uint32_t *list_off, const float *cb,
                      const float *qs, uint32_t *probe, float *lut, const uint32_t *elig) {
  extern __shared__ uint64_t pb_keys[];   // npow2 keys
  __shared__ float sq[STB_D];
  __shared__ float s_inv;
  __shared__ uint32_t s_sz[1024];
  const uint32_t q = blockIdx.x;
  const float *cq = coarse + (size_t)q * nlist;
  uint32_t *pr = probe + (size_t)q * IVFB_PROBE_STRIDE(nprobe, FILTER);
  uint32_t npow = 1; while (npow < nlist) npow <<= 1;
  for (uint32_t i = threadIdx.x; i < npow; i += blockDim.x) pb_keys[i] = (i < nlist) ? stb_make_key(cq[i], i) : STB_KEY_INVALID;
  if (threadIdx.x < STB_D) sq[threadIdx.x] = qs[(size_t)q * STB_D + threadIdx.x];
  __syncthreads();
  if (threadIdx.x == 0) s_inv = ivf_query_inv(sq);
  stb_cta_sort_keys_strided(pb_keys, npow);
  if (!FILTER) {
    if (threadIdx.x < nprobe) {
      const uint32_t l = stb_key_row(pb_keys[threadIdx.x]);
      pr[threadIdx.x] = l;
      s_sz[threadIdx.x] = __ldg(list_off + l + 1) - __ldg(list_off + l);
    }
  } else {
    // compaction of the sorted lists with an eligible code, 1024 sorted positions per step, until nprobe
    // are taken; s_el[p] = eligible codes of probe slot p
    __shared__ uint32_t s_el[1024], s_wcnt[32], s_taken;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_taken = 0;
    __syncthreads();
    for (uint32_t base = 0; base < nlist; base += blockDim.x) {
      const uint32_t taken = s_taken;
      if (taken >= nprobe) break;                                   // uniform: read after a barrier
      const uint32_t i = base + threadIdx.x;
      const uint32_t l = i < nlist ? stb_key_row(pb_keys[i]) : 0;
      const uint32_t e = i < nlist ? __ldg(elig + l) : 0;
      const unsigned bal = __ballot_sync(0xffffffffu, e > 0);
      if (lane == 0) s_wcnt[warp] = __popc(bal);
      __syncthreads();
      uint32_t rank = taken + __popc(bal & ((1u << lane) - 1));
      for (uint32_t w = 0; w < warp; ++w) rank += s_wcnt[w];
      if (e > 0 && rank < nprobe) {
        pr[rank] = l;
        s_sz[rank] = __ldg(list_off + l + 1) - __ldg(list_off + l);
        s_el[rank] = e;
      }
      __syncthreads();
      if (threadIdx.x == 0) { uint32_t t = 0; for (uint32_t w = 0; w < blockDim.x / 32; ++w) t += s_wcnt[w]; s_taken = taken + t; }
      __syncthreads();
    }
    const uint32_t used = min(s_taken, nprobe);
    for (uint32_t p = used + threadIdx.x; p < nprobe; p += blockDim.x) { pr[p] = IVF_NO_LIST; s_sz[p] = 0; s_el[p] = 0; }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t el = 0;
      for (uint32_t p = 0; p < used; ++p) el += s_el[p];
      pr[2 * nprobe + 1] = el;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t acc = 0;
    for (uint32_t p = 0; p < nprobe; ++p) { pr[nprobe + p] = acc; acc += s_sz[p]; }
    pr[2 * nprobe] = acc;
  }
  const float inv = s_inv;
  float *lq = lut + (size_t)q * PQ_M * PQ_KSUB;
  for (int i = threadIdx.x; i < PQ_M * PQ_KSUB; i += blockDim.x) lq[i] = ivf_lut_entry(sq, inv, cb, i);
}

// The IVFB_WARP_KEEP best keys a warp has seen (2 per lane, exact: keys are distinct), and the best
// (smallest) key it has dropped.  Smaller key = better; STB_KEY_INVALID fills empty slots.
struct IvfbTop {
  uint64_t k[2], thr, drop;   // thr: the worst kept key (warp-uniform)
  int lane;
  // keep < 64: slots keep..63 hold key 0, which no code has (its score would be a NaN) and which is
  // never evicted, so the warp keeps `keep` codes
  __device__ __forceinline__ void init(uint32_t keep) {
    lane = threadIdx.x & 31;
    k[0] = (uint32_t)lane < keep ? STB_KEY_INVALID : 0ull;
    k[1] = (uint32_t)(32 + lane) < keep ? STB_KEY_INVALID : 0ull;
    thr = drop = STB_KEY_INVALID;
  }
  __device__ __forceinline__ void insert(uint64_t ck) {   // warp-uniform ck < thr: replaces the worst kept key
    const uint64_t m = k[0] > k[1] ? k[0] : k[1];
    const unsigned owners = __ballot_sync(0xffffffffu, m == thr);
    if (lane == __ffs(owners) - 1) { if (k[0] == m) k[0] = ck; else k[1] = ck; }
    drop = min(drop, thr);
    uint64_t t = k[0] > k[1] ? k[0] : k[1];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) t = max(t, __shfl_xor_sync(0xffffffffu, t, off));
    thr = t;
  }
  __device__ __forceinline__ void push(uint64_t key) {
    unsigned mask = __ballot_sync(0xffffffffu, key < thr);
    if (!(key < thr)) drop = min(drop, key);
    while (mask) {
      const int src = __ffs(mask) - 1;
      mask &= mask - 1;
      const uint64_t ck = __shfl_sync(0xffffffffu, key, src);
      if (ck < thr) insert(ck); else drop = min(drop, ck);
    }
  }
};

// key of probed code v of a query (STB_KEY_INVALID past the end and for a NaN or -inf score); pref,
// start and pc: per probed list the prefix of lengths, list_off of the list and its coarse score.
// FILTER with a bitmap: a code whose row (order[pos]) is not eligible is STB_KEY_INVALID too, decided
// before its 32 bytes are read.
template <bool FILTER>
__device__ __forceinline__ uint64_t ivfb_code_key(uint64_t v, uint32_t total, uint32_t nprobe, const uint32_t *pref,
                                                  const uint32_t *start, const float *pc, const float *s_lut,
                                                  const uint8_t *codes, const uint32_t *order, const uint32_t *bitmap) {
  if (v >= total) return STB_KEY_INVALID;
  uint32_t lo = 0, hi = nprobe;      // probe p with pref[p] <= v < pref[p+1]
  while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (pref[mid] <= v) lo = mid; else hi = mid; }
  const uint32_t pos = start[lo] + (uint32_t)(v - pref[lo]);
  if (FILTER && bitmap) {
    const uint32_t row = __ldg(order + pos);
    if (!((__ldg(bitmap + (row >> 5)) >> (row & 31)) & 1u)) return STB_KEY_INVALID;
  }
  const uint4 *cp = reinterpret_cast<const uint4 *>(codes + (size_t)pos * PQ_M);
  const float s = ivf_adc_sum(s_lut, __ldg(cp), __ldg(cp + 1), pc[lo]);
  return s > -CUDART_INF_F ? stb_make_key(s, pos) : STB_KEY_INVALID;
}

struct IvfbArgs {
  const float *C; uint32_t nlist, nq, nprobe, top_k, rerank, keep;
  const uint32_t *list_off; const float *cb; const uint8_t *codes; const uint32_t *order;
  const float *qs; float *coarse; uint32_t *probe; float *lut; uint64_t *kept, *drop;
  const float4 *rows; uint64_t row_base; const uint32_t *forced; uint32_t n_forced;
  stb_hit *out_hits; uint32_t *out_status;   // [nq][top_k], [nq][2] = {hits, codes scanned}
  // filtered search only (the FILTER instantiations read them)
  const uint32_t *bitmap;                    // eligible local rows, 1 bit each; NULL: every row
  double max_dist;                           // a hit needs distance < max_dist
};

template <bool FILTER>
__global__ void __launch_bounds__(IVFB_SCAN_THREADS)
ivfb_scan_kernel(const IvfbArgs a) {
  __shared__ float s_lut[PQ_M * PQ_KSUB];      // 32 KiB
  __shared__ uint32_t s_pref[1024], s_start[1024];
  __shared__ float s_pc[1024];
  const uint32_t q = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t *pr = a.probe + (size_t)q * IVFB_PROBE_STRIDE(a.nprobe, FILTER);
  const float *lq = a.lut + (size_t)q * PQ_M * PQ_KSUB;
  for (uint32_t i = tid; i < PQ_M * PQ_KSUB; i += IVFB_SCAN_THREADS) s_lut[i] = lq[i];
  for (uint32_t p = tid; p < a.nprobe; p += IVFB_SCAN_THREADS) {
    const uint32_t l = pr[p];
    if (FILTER && l == IVF_NO_LIST) { s_pref[p] = pr[a.nprobe + p]; s_start[p] = 0; s_pc[p] = 0.f; continue; }
    s_pref[p] = pr[a.nprobe + p]; s_start[p] = __ldg(a.list_off + l); s_pc[p] = a.coarse[(size_t)q * a.nlist + l];
  }
  __syncthreads();
  const uint32_t total = pr[2 * a.nprobe];
  IvfbTop top;
  top.init(a.keep);
  // chunk g (32 consecutive codes) -> CTA g % IVFB_SCAN_CTAS, warp (g / IVFB_SCAN_CTAS) % 8
  for (uint64_t g = blockIdx.x + (uint64_t)IVFB_SCAN_CTAS * warp; g * 32 < total; g += IVFB_WARPS)
    top.push(ivfb_code_key<FILTER>(g * 32 + lane, total, a.nprobe, s_pref, s_start, s_pc, s_lut, a.codes, a.order, a.bitmap));
  uint64_t d = top.drop;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) d = min(d, __shfl_xor_sync(0xffffffffu, d, off));
  const uint32_t w = blockIdx.x * (IVFB_SCAN_THREADS / 32) + warp;   // warp of the query, 0..63
  uint64_t *kq = a.kept + (size_t)q * IVFB_KEPT + w * IVFB_WARP_KEEP;
  kq[lane] = top.k[0] ? top.k[0] : STB_KEY_INVALID; kq[32 + lane] = top.k[1] ? top.k[1] : STB_KEY_INVALID;
  if (lane == 0) a.drop[(size_t)q * IVFB_WARPS + w] = d;
}

// FILTER: the slow route skips the IVF_NO_LIST slots and reads eligibility through ivfb_code_key, only
// the eligible forced rows are re-ranked, a hit needs distance < a.max_dist, and the codes reported
// scanned are the probed lists' eligible codes.
template <bool FILTER>
__global__ void __launch_bounds__(IVFB_FIN_THREADS)
ivfb_finish_kernel(const IvfbArgs a) {
  extern __shared__ __align__(16) uint8_t dyn[];                     // IVFB_FIN_SMEM
  uint64_t *keys = reinterpret_cast<uint64_t *>(dyn);               // [0, 32 KiB): kept keys, then candidates
  __shared__ double sqd[STB_D];
  __shared__ double s_q2;
  __shared__ int s_pass;
  __shared__ unsigned s_slow, s_nc, s_need;
  __shared__ uint32_t s_hist[256];
  __shared__ unsigned long long s_prefix;
  const uint32_t q = blockIdx.x, tid = threadIdx.x;
  const uint32_t *pr = a.probe + (size_t)q * IVFB_PROBE_STRIDE(a.nprobe, FILTER);
  const uint32_t total = pr[2 * a.nprobe];
  const uint32_t r = a.rerank;
  for (uint32_t i = tid; i < IVFB_KEPT; i += IVFB_FIN_THREADS) keys[i] = a.kept[(size_t)q * IVFB_KEPT + i];
  for (uint32_t i = tid; i < STB_D; i += IVFB_FIN_THREADS) sqd[i] = (double)a.qs[(size_t)q * STB_D + i];
  if (tid == 0) { s_pass = 0; s_slow = 0; }
  __syncthreads();
  stb_cta_sort_keys_strided(keys, IVFB_KEPT);
  // every key a warp dropped is >= its recorded drop; the kept keys hold the r best iff each is > T
  const uint64_t T = keys[r - 1];
  if (tid < IVFB_WARPS) {
    const uint64_t d = a.drop[(size_t)q * IVFB_WARPS + tid];
    if (d != STB_KEY_INVALID && d < T) s_slow = 1;
  }
  if (tid == 0) s_q2 = stb_canon_q2(sqd);
  __syncthreads();
  uint32_t nc = r;                                                   // candidates: keys[0, nc)
  if (s_slow) {
    // exact slow route: radix select of the r-th best key over every probed code
    float *s_lut = reinterpret_cast<float *>(dyn + 32768);          // [32 KiB, 64 KiB)
    const float *lq = a.lut + (size_t)q * PQ_M * PQ_KSUB;
    for (uint32_t i = tid; i < PQ_M * PQ_KSUB; i += IVFB_FIN_THREADS) s_lut[i] = lq[i];
    uint32_t *s_pref = reinterpret_cast<uint32_t *>(dyn);           // [0, 12 KiB) during the selection
    uint32_t *s_start = s_pref + 1024;
    float *s_pc = reinterpret_cast<float *>(s_pref + 2048);
    for (uint32_t p = tid; p < a.nprobe; p += IVFB_FIN_THREADS) {
      const uint32_t l = pr[p];
      if (FILTER && l == IVF_NO_LIST) { s_pref[p] = pr[a.nprobe + p]; s_start[p] = 0; s_pc[p] = 0.f; continue; }
      s_pref[p] = pr[a.nprobe + p]; s_start[p] = __ldg(a.list_off + l); s_pc[p] = a.coarse[(size_t)q * a.nlist + l];
    }
    if (tid == 0) { s_prefix = 0; s_need = r; }
    for (int pass = 0; pass < 8; ++pass) {
      const int shift = 56 - 8 * pass;
      const uint64_t hi_mask = pass == 0 ? 0ull : (~0ull << (shift + 8));
      for (uint32_t i = tid; i < 256; i += IVFB_FIN_THREADS) s_hist[i] = 0;
      __syncthreads();
      const uint64_t prefix = s_prefix;
      for (uint64_t v = tid; v < total; v += IVFB_FIN_THREADS) {
        const uint64_t key = ivfb_code_key<FILTER>(v, total, a.nprobe, s_pref, s_start, s_pc, s_lut, a.codes, a.order, a.bitmap);
        if (key != STB_KEY_INVALID && (key & hi_mask) == prefix) atomicAdd(&s_hist[(key >> shift) & 255], 1u);
      }
      __syncthreads();
      if (tid == 0) {
        uint32_t need = s_need;
        if (pass == 0) {                                             // fewer valid codes than r: take them all
          uint32_t valid = 0;
          for (int b = 0; b < 256; ++b) valid += s_hist[b];
          need = min(need, valid);
        }
        if (need > 0) {
          uint32_t cum = 0, b = 0;
          while (cum + s_hist[b] < need) cum += s_hist[b++];
          s_prefix = prefix | ((uint64_t)b << shift);
          need -= cum;
        } else {
          s_prefix = 0;                                              // nothing valid: the emit pass takes nothing
        }
        s_need = need;
      }
      __syncthreads();
    }
    const uint64_t thr = s_prefix;
    const bool none = s_need == 0;
    if (tid == 0) s_nc = 0;
    __syncthreads();
    uint64_t *cand = reinterpret_cast<uint64_t *>(dyn + 16384);     // [16 KiB, 24 KiB): r <= 1024 keys
    if (!none)
      for (uint64_t v = tid; v < total; v += IVFB_FIN_THREADS) {
        const uint64_t key = ivfb_code_key<FILTER>(v, total, a.nprobe, s_pref, s_start, s_pc, s_lut, a.codes, a.order, a.bitmap);
        if (key <= thr) cand[atomicAdd(&s_nc, 1u)] = key;           // exactly min(r, valid) keys
      }
    __syncthreads();
    nc = s_nc;
    for (uint32_t i = tid; i < nc; i += IVFB_FIN_THREADS) keys[i] = cand[i];
    __syncthreads();
  }
  // re-rank: the candidates' rows and the forced rows, canonical distance, (distance, row) order
  uint32_t n2 = 32;
  while (n2 < nc + a.n_forced) n2 <<= 1;
  double *sd = reinterpret_cast<double *>(dyn + 16384);             // [16 KiB, 32 KiB)
  uint64_t *sr = reinterpret_cast<uint64_t *>(dyn + 32768);         // [32 KiB, 48 KiB)
  uint64_t *rows_c = reinterpret_cast<uint64_t *>(dyn + 49152);     // [48 KiB, 64 KiB): local row of entry c
  for (uint32_t c = tid; c < n2; c += IVFB_FIN_THREADS) {
    uint64_t row = 0xffffffffffffffffull;
    if (c < nc) {
      const uint64_t key = keys[c];
      if (key != STB_KEY_INVALID) row = a.order[stb_key_row(key)];
    } else if (c < nc + a.n_forced) {
      row = a.forced[c - nc];
      if (FILTER && a.bitmap && !((__ldg(a.bitmap + (row >> 5)) >> (row & 31)) & 1u)) row = 0xffffffffffffffffull;
    }
    rows_c[c] = row;
  }
  __syncthreads();                                                   // keys are read before sd overwrites them
  const double q2 = s_q2;
  const double limit = FILTER ? a.max_dist : STB_DEFAULT_MAX_DIST;
  for (uint32_t c = tid; c < n2; c += IVFB_FIN_THREADS) {
    double d = CUDART_INF;
    uint64_t grow = 0xffffffffffffffffull;
    const uint64_t row = rows_c[c];
    if (row != 0xffffffffffffffffull) {
      double ab, r2;
      stb_canon_dot<true>(sqd, a.rows + row * STB_ROW_F4, ab, r2);
      const double dist = stb_canon_dist(ab, q2, r2);
      if (dist < limit) { d = dist; grow = a.row_base + row; atomicAdd(&s_pass, 1); }
    }
    sd[c] = d; sr[c] = grow;
  }
  __syncthreads();
  stb_cta_sort_hits(sd, sr, n2);
  const uint32_t n_out = min((uint32_t)s_pass, a.top_k);
  stb_write_hits(a.out_hits + (size_t)q * a.top_k, sd, sr, n_out, a.top_k);
  if (tid == 0) { a.out_status[2 * q] = n_out; a.out_status[2 * q + 1] = FILTER ? pr[2 * a.nprobe + 1] : total; }
}

// ------------------------------------------------------------------ filtered search ------
// The eligibility pass of stb_ivfpq_search_filtered, once per call (every query of the call shares it):
//   ivff_bitmap_kernel  bit r of the bitmap = local row r lies in one of the clipped ranges (thread per
//                       32-row word: a binary search for the first range ending past the word, then the
//                       at most 32 non-empty ranges that touch it); stb_launch_row_bitmap, which
//                       stb_search_batch_filtered uses too
//   ivff_elig_kernel    elig[l] = eligible codes of list l (warp per list, order[] read once: 4 B per
//                       listed row); without a bitmap elig[l] is the list's length
// The batched kernels' FILTER instantiations then probe only lists with elig > 0 and drop every code
// and forced row whose bit is clear.
__global__ void ivff_bitmap_kernel(const uint32_t *ranges, uint32_t n_ranges, uint32_t n_words, uint32_t *bitmap) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;   // ranges: [begin, end) local pairs, ascending
  if (w >= n_words) return;
  const uint64_t w0 = (uint64_t)w * 32, w1 = w0 + 32;
  uint32_t lo = 0, hi = n_ranges;                              // first range with end > w0
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (ranges[2 * mid + 1] <= w0) lo = mid + 1; else hi = mid; }
  uint32_t bits = 0;
  for (uint32_t i = lo; i < n_ranges && ranges[2 * i] < w1; ++i) {
    const uint32_t b = (uint32_t)(max((uint64_t)ranges[2 * i], w0) - w0);
    const uint32_t e = (uint32_t)(min((uint64_t)ranges[2 * i + 1], w1) - w0);   // 0 <= b < e <= 32
    bits |= (e - b == 32 ? 0xffffffffu : ((1u << (e - b)) - 1u)) << b;
  }
  bitmap[w] = bits;
}

int stb_launch_row_bitmap(stb_ctx *ctx, const uint32_t *ranges_dev, uint32_t n_ranges, uint64_t n_words, uint32_t *bitmap) {
  if (n_words == 0) return STB_OK;
  ivff_bitmap_kernel<<<(unsigned)((n_words + 255) / 256), 256, 0, ctx->stream>>>(ranges_dev, n_ranges, (uint32_t)n_words, bitmap);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches += 1;
  return STB_OK;
}

__global__ void ivff_elig_kernel(const uint32_t *list_off, const uint32_t *order, uint32_t nlist, const uint32_t *bitmap,
                                 uint32_t *elig) {
  const uint32_t lane = threadIdx.x & 31, l = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (l >= nlist) return;
  const uint32_t b = __ldg(list_off + l), e = __ldg(list_off + l + 1);
  if (!bitmap) { if (lane == 0) elig[l] = e - b; return; }
  uint32_t cnt = 0;
  for (uint32_t i = b + lane; i < e; i += 32) {
    const uint32_t row = __ldg(order + i);
    cnt += (__ldg(bitmap + (row >> 5)) >> (row & 31)) & 1u;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
  if (lane == 0) elig[l] = cnt;
}

// ------------------------------------------------------------------ host side ---------
// Device buffers of one edit of the lists: freed with it (after a stream synchronise, so no kernel still
// reads them) unless adopted by the index.  A failed allocation is STB_ERR_NOMEM.
struct IvfScratch {
  cudaStream_t st;
  std::vector<void *> p;
  template <class T> int alloc(T **ptr, size_t bytes) {
    *ptr = nullptr;
    const cudaError_t e = cudaMalloc(reinterpret_cast<void **>(ptr), std::max<size_t>(bytes, 16));
    if (e != cudaSuccess) {
      cudaGetLastError();
      stb_set_error("ivfpq: cudaMalloc(%zu bytes) failed: %s", bytes, cudaGetErrorString(e));
      return STB_ERR_NOMEM;
    }
    p.push_back(*ptr);
    return STB_OK;
  }
  void adopt(const void *q) { p.erase(std::find(p.begin(), p.end(), q)); }
  ~IvfScratch() {
    cudaStreamSynchronize(st);
    for (void *q : p) cudaFree(q);
    cudaGetLastError();
  }
};
#define IVF_TRY(call)                      \
  do {                                     \
    const int _rc = (call);                \
    if (_rc != STB_OK) return _rc;         \
  } while (0)

// One edit of the lists (see "inverted lists").  The caller fills in what changes; then
//   ivf_edit_alloc    allocates every buffer the edit needs,
//   ivf_edit_encode   computes the list and code of new entries [i0, i0 + mc) from rows anywhere on the device,
//   ivf_edit_plan     writes the new arrays beside the old ones; an edit that would leave more than
//                     IVF_FORCED_CAP forced rows is refused (STB_ERR_STATE),
//   ivf_edit_swap     installs them.
// Until the swap the index is untouched and searchable, so a caller can still back out.  Peak extra memory:
// the new codes + order (36 B per listed row, old and new), 48 B per new entry (list ids and sort values,
// double-buffered, the codes in entry order, their rows) and, when entries leave, a bitmap of the indexed
// rows, the kept segments and 8 B per old listed entry (survivor positions and rows).
struct IvfEdit {
  IvfScratch t;
  uint64_t m = 0, first = 0;          // new entries: rows first + i (build, extend), or rows_h[i] (update)
  std::vector<uint32_t> rows_h;       //   local rows, ascending
  bool keep_all = true;               // no old entry leaves and none is renumbered (build, extend)
  std::vector<uint32_t> kept, kept_dst;   // otherwise the kept segments: [begin, end) pairs and their dst
  uint32_t n_kept = 0;
  uint64_t n_after = 0;               // indexed rows after the edit
  int key_bits = 0;
  size_t sort_bytes = 0;
  uint32_t *assign = nullptr, *assign_alt = nullptr, *vals = nullptr, *vals_alt = nullptr, *counts = nullptr;
  uint32_t *new_rows = nullptr, *kept_d = nullptr, *bitmap = nullptr, *elig = nullptr, *surv_pos = nullptr;
  uint32_t *surv_row = nullptr, *surv_off_d = nullptr, *new_off_d = nullptr, *order = nullptr, *forced = nullptr;
  uint8_t *codes_row = nullptr, *codes = nullptr;
  void *sort_tmp = nullptr;
  std::vector<uint32_t> new_off, forced_h;
  explicit IvfEdit(cudaStream_t st) : t{st, {}} {}
  IvfEdit(const IvfEdit &) = delete;
  IvfEdit &operator=(const IvfEdit &) = delete;
  // kept segment {[b, e), dst}; segments come in ascending order
  void keep(uint32_t b, uint32_t e, uint32_t dst) {
    kept.push_back(b); kept.push_back(e); kept_dst.push_back(dst);
    ++n_kept;
  }
};

static int ivf_edit_alloc(stb_ivfpq *x, IvfEdit &e) {
  const uint32_t nlist = x->nlist;
  const uint64_t m = e.m, n_old = x->list_off_h[nlist];
  cudaStream_t st = e.t.st;
  e.key_bits = 32 - __builtin_clz(nlist);          // 2^key_bits - 1 >= nlist: IVF_NO_LIST sorts last
  if (m) {
    cub::DoubleBuffer<uint32_t> kb(nullptr, nullptr), vb(nullptr, nullptr);
    STB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, e.sort_bytes, kb, vb, (uint32_t)m, 0, e.key_bits, st));
  }
  IVF_TRY(e.t.alloc(&e.assign, m * 4));
  IVF_TRY(e.t.alloc(&e.assign_alt, m * 4));
  IVF_TRY(e.t.alloc(&e.vals, m * 4));
  IVF_TRY(e.t.alloc(&e.vals_alt, m * 4));
  IVF_TRY(e.t.alloc(&e.codes_row, m * PQ_M));
  IVF_TRY(e.t.alloc(&e.counts, (size_t)(nlist + 1) * 4));
  IVF_TRY(e.t.alloc(&e.sort_tmp, e.sort_bytes));
  IVF_TRY(e.t.alloc(&e.codes, (n_old + m) * PQ_M));
  IVF_TRY(e.t.alloc(&e.order, (n_old + m) * 4));
  IVF_TRY(e.t.alloc(&e.new_off_d, (size_t)(nlist + 1) * 4));
  IVF_TRY(e.t.alloc(&e.forced, IVF_FORCED_CAP * 4));
  if (!e.rows_h.empty()) IVF_TRY(e.t.alloc(&e.new_rows, m * 4));
  if (!e.keep_all) {
    IVF_TRY(e.t.alloc(&e.kept_d, (size_t)e.n_kept * 3 * 4));   // pairs, then dst
    IVF_TRY(e.t.alloc(&e.bitmap, (x->n + 31) / 32 * 4));
    IVF_TRY(e.t.alloc(&e.elig, (size_t)nlist * 4));
    IVF_TRY(e.t.alloc(&e.surv_pos, n_old * 4));
    IVF_TRY(e.t.alloc(&e.surv_row, n_old * 4));
    IVF_TRY(e.t.alloc(&e.surv_off_d, (size_t)(nlist + 1) * 4));
  }
  STB_CUDA(cudaMemsetAsync(e.counts, 0, (size_t)(nlist + 1) * 4, st));
  return STB_OK;
}

// list, code and forced flag of new entries [i0, i0 + mc), rows X[0 .. mc)
static int ivf_edit_encode(stb_ivfpq *x, IvfEdit &e, const float *X, uint64_t i0, uint64_t mc) {
  if (mc == 0) return STB_OK;
  stb_ctx *ctx = x->ctx;
  cudaStream_t st = e.t.st;
  const float4 *X4 = reinterpret_cast<const float4 *>(X);
  ivf_assign_kernel<<<(unsigned)((mc + 63) / 64), 256, 0, st>>>(X, mc, x->centroids, x->nlist, e.assign + i0);
  STB_CUDA(cudaFuncSetAttribute(pq_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * PQ_KSUB * PQ_DSUB * 4));
  PqArgs pa;
  pa.X = X4; pa.n = mc; pa.stride = 1; pa.assign = e.assign + i0; pa.C = x->centroids; pa.cb = x->codebooks;
  pa.sums = nullptr; pa.counts = nullptr; pa.codes_out = e.codes_row + i0 * PQ_M; pa.mode = 1;
  for (int s0 = 0; s0 < PQ_M; s0 += 8) {
    pa.s0 = s0;
    pq_step_kernel<<<ctx->sm_count * 2, 256, 8 * PQ_KSUB * PQ_DSUB * 4, st>>>(pa);
  }
  // forced rows leave the lists; counts[nlist] is their count
  ivf_flag_forced_kernel<<<(unsigned)((mc + 7) / 8), 256, 0, st>>>(X4, mc, e.assign + i0, e.counts + x->nlist);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches += 6;                               // assign, 4 x encode, flag
  return STB_OK;
}

// renumbered row of an old indexed row, or false if it leaves (host form of ivf_compact_kernel's search)
static bool ivf_edit_renumber(const IvfEdit &e, uint32_t row, uint32_t &out) {
  if (e.keep_all) { out = row; return true; }
  uint32_t lo = 0, hi = e.n_kept;                          // first segment with begin > row
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (e.kept[2 * mid] <= row) lo = mid + 1; else hi = mid; }
  if (lo == 0 || row >= e.kept[2 * (lo - 1) + 1]) return false;
  out = e.kept_dst[lo - 1] + (row - e.kept[2 * (lo - 1)]);
  return true;
}

static int ivf_edit_plan(stb_ivfpq *x, IvfEdit &e, const char *who) {
  stb_ctx *ctx = x->ctx;
  cudaStream_t st = e.t.st;
  const uint32_t nlist = x->nlist;
  const uint64_t m = e.m;
  cub::DoubleBuffer<uint32_t> kb(e.assign, e.assign_alt), vb(e.vals, e.vals_alt);
  if (m) {
    ivf_hist_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(e.assign, m, e.counts, e.vals);
    STB_CUDA(cub::DeviceRadixSort::SortPairs(e.sort_tmp, e.sort_bytes, kb, vb, (uint32_t)m, 0, e.key_bits, st));
    if (!e.rows_h.empty())
      STB_CUDA(cudaMemcpyAsync(e.new_rows, e.rows_h.data(), m * 4, cudaMemcpyHostToDevice, st));
    ctx->kernel_launches += 2;                             // hist, sort (as one)
  }
  std::vector<uint32_t> hist(nlist + 1), surv(nlist, 0);
  if (!e.keep_all) {
    const uint64_t words = (x->n + 31) / 32;
    if (e.n_kept) {
      STB_CUDA(cudaMemcpyAsync(e.kept_d, e.kept.data(), (size_t)e.n_kept * 8, cudaMemcpyHostToDevice, st));
      STB_CUDA(cudaMemcpyAsync(e.kept_d + 2 * e.n_kept, e.kept_dst.data(), (size_t)e.n_kept * 4, cudaMemcpyHostToDevice, st));
    }
    if (words) ivff_bitmap_kernel<<<(unsigned)((words + 255) / 256), 256, 0, st>>>(e.kept_d, e.n_kept, (uint32_t)words, e.bitmap);
    ivff_elig_kernel<<<(nlist + 7) / 8, 256, 0, st>>>(x->list_off, x->order, nlist, e.bitmap, e.elig);
    STB_CUDA(cudaMemcpyAsync(surv.data(), e.elig, (size_t)nlist * 4, cudaMemcpyDeviceToHost, st));
    ctx->kernel_launches += 2;
  } else {
    for (uint32_t l = 0; l < nlist; ++l) surv[l] = x->list_off_h[l + 1] - x->list_off_h[l];
  }
  STB_CUDA(cudaMemcpyAsync(hist.data(), e.counts, (size_t)(nlist + 1) * 4, cudaMemcpyDeviceToHost, st));
  STB_CUDA(cudaGetLastError());
  STB_CUDA(cudaStreamSynchronize(st));
  // the forced side list: old forced rows that stay (renumbered), merged with the new ones (the sort's tail)
  const uint32_t nf_new = hist[nlist];
  std::vector<uint32_t> old_f(x->n_forced), tail(nf_new);
  if (x->n_forced) STB_CUDA(cudaMemcpyAsync(old_f.data(), x->forced, (size_t)x->n_forced * 4, cudaMemcpyDeviceToHost, st));
  if (nf_new) STB_CUDA(cudaMemcpyAsync(tail.data(), vb.Current() + (m - nf_new), (size_t)nf_new * 4, cudaMemcpyDeviceToHost, st));
  STB_CUDA(cudaStreamSynchronize(st));
  std::vector<uint32_t> kept_f;
  for (uint32_t r : old_f) { uint32_t nr; if (ivf_edit_renumber(e, r, nr)) kept_f.push_back(nr); }
  for (uint32_t &v : tail) v = e.rows_h.empty() ? (uint32_t)(e.first + v) : e.rows_h[v];
  e.forced_h.resize(kept_f.size() + tail.size());
  std::merge(kept_f.begin(), kept_f.end(), tail.begin(), tail.end(), e.forced_h.begin());
  if (e.forced_h.size() > IVF_FORCED_CAP) {
    stb_set_error("%s: %zu rows are non-finite or have an fp32 squared norm outside [1e-30, 1e30] (at most %u)", who,
                  e.forced_h.size(), (unsigned)IVF_FORCED_CAP);
    return STB_ERR_STATE;
  }
  std::vector<uint32_t> surv_off(nlist + 1, 0);
  e.new_off.assign(nlist + 1, 0);
  for (uint32_t l = 0; l < nlist; ++l) {
    surv_off[l + 1] = surv_off[l] + surv[l];
    e.new_off[l + 1] = e.new_off[l] + surv[l] + hist[l];
  }
  const uint32_t n_out = e.new_off[nlist];
  STB_CUDA(cudaMemcpyAsync(e.new_off_d, e.new_off.data(), (size_t)(nlist + 1) * 4, cudaMemcpyHostToDevice, st));
  if (!e.forced_h.empty())
    STB_CUDA(cudaMemcpyAsync(e.forced, e.forced_h.data(), e.forced_h.size() * 4, cudaMemcpyHostToDevice, st));
  MergeArgs ma;
  ma.old_codes = x->codes; ma.old_order = x->order; ma.new_off = e.new_off_d; ma.nlist = nlist;
  ma.surv_off = x->list_off; ma.surv_pos = nullptr; ma.surv_row = nullptr;
  if (!e.keep_all) {
    STB_CUDA(cudaMemcpyAsync(e.surv_off_d, surv_off.data(), (size_t)(nlist + 1) * 4, cudaMemcpyHostToDevice, st));
    ivf_compact_kernel<<<(nlist + 7) / 8, 256, 0, st>>>(x->list_off, x->order, nlist, e.bitmap, e.kept_d,
                                                         e.kept_d + 2 * e.n_kept, e.n_kept, e.surv_off_d, e.surv_pos,
                                                         e.surv_row);
    ma.surv_off = e.surv_off_d; ma.surv_pos = e.surv_pos; ma.surv_row = e.surv_row;
    ctx->kernel_launches += 1;
  }
  ma.codes_row = e.codes_row; ma.sorted = vb.Current(); ma.new_rows = e.new_rows; ma.first = e.first;
  ma.n_out = n_out; ma.codes = e.codes; ma.order = e.order;
  if (n_out) {
    ivf_merge_kernel<<<(unsigned)(((uint64_t)n_out + 255) / 256), 256, 0, st>>>(ma);
    ctx->kernel_launches += 1;
  }
  STB_CUDA(cudaGetLastError());
  // the host vectors the copies above read die with the caller: the copies must be done
  STB_CUDA(cudaStreamSynchronize(st));
  return STB_OK;
}

// Installs a planned edit.  Searches enqueued before it have finished (the stream is synchronised), so the
// old arrays can go.
static int ivf_edit_swap(stb_ivfpq *x, IvfEdit &e) {
  STB_CUDA(cudaStreamSynchronize(e.t.st));
  e.t.adopt(e.codes); e.t.adopt(e.order); e.t.adopt(e.new_off_d); e.t.adopt(e.forced);
  cudaFree(x->codes); cudaFree(x->order); cudaFree(x->list_off); cudaFree(x->forced);
  x->codes = e.codes; x->order = e.order; x->list_off = e.new_off_d; x->forced = e.forced;
  x->list_off_h.swap(e.new_off);
  x->n_forced = (uint32_t)e.forced_h.size();
  x->n = e.n_after;
  return STB_OK;
}

// Indexes rows [first, first + m) of x's corpus (the build's add phase and stb_ivfpq_extend): on success x
// holds the extended lists and n = first + m; on any error x is unchanged and usable.
static int ivf_add_rows(stb_ivfpq *x, uint64_t first, uint64_t m, const char *who) {
  IvfEdit e(x->ctx->stream);
  e.m = m; e.first = first; e.n_after = first + m;
  IVF_TRY(ivf_edit_alloc(x, e));
  IVF_TRY(ivf_edit_encode(x, e, x->corpus->rows + first * STB_D, 0, m));
  IVF_TRY(ivf_edit_plan(x, e, who));
  return ivf_edit_swap(x, e);
}

extern "C" {

int stb_ivfpq_destroy(stb_ivfpq *x) {
  if (!x) return STB_OK;
  const_cast<stb_corpus *>(x->corpus)->ivfpq_live--;
  cudaFree(x->centroids); cudaFree(x->codebooks); cudaFree(x->codes); cudaFree(x->order); cudaFree(x->list_off);
  cudaFree(x->coarse); cudaFree(x->lut); cudaFree(x->probe); cudaFree(x->cand); cudaFree(x->cand_rows);
  cudaFree(x->keys2); cudaFree(x->tickets); cudaFree(x->forced);
  cudaFree(x->b_q); cudaFree(x->b_coarse); cudaFree(x->b_probe); cudaFree(x->b_lut); cudaFree(x->b_kept);
  cudaFree(x->b_drop); cudaFree(x->b_hits); cudaFree(x->b_status);
  cudaFree(x->f_bitmap); cudaFree(x->f_elig); cudaFree(x->f_ranges);
  cudaGetLastError();
  delete x;
  return STB_OK;
}

#define IVF_CUDA(call)                                                                  \
  do {                                                                                  \
    cudaError_t _e = (call);                                                            \
    if (_e != cudaSuccess) {                                                            \
      stb_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
      cudaGetLastError();                                                               \
      stb_ivfpq_destroy(x);                                                             \
      return STB_ERR_CUDA;                                                              \
    }                                                                                   \
  } while (0)

int stb_ivfpq_build(stb_ctx *ctx, const stb_corpus *corpus, uint32_t nlist, uint32_t train_rows, uint32_t iters,
                    stb_ivfpq **out) {
  if (!ctx || !corpus || !out) { stb_set_error("ivfpq_build: null argument"); return STB_ERR_ARG; }
  if (corpus->ctx != ctx) { stb_set_error("ivfpq_build: corpus belongs to another context"); return STB_ERR_ARG; }
  if (cudaSetDevice(ctx->device) != cudaSuccess) { stb_set_error("cudaSetDevice failed"); return STB_ERR_CUDA; }
  const uint64_t n = corpus->n;
  if (nlist < 1 || nlist > 8192 || n < nlist || n < 256) { stb_set_error("ivfpq_build: need 1 <= nlist <= 8192 <= rows and rows >= 256"); return STB_ERR_ARG; }
  if (iters < 1) iters = 8;
  stb_ivfpq *x = new (std::nothrow) stb_ivfpq();
  if (!x) { stb_set_error("out of host memory"); return STB_ERR_NOMEM; }
  x->ctx = ctx; x->corpus = corpus; x->corpus_epoch = corpus->epoch; x->nlist = nlist; x->n = 0;
  // counted from here: every failure below ends in stb_ivfpq_destroy, which takes the count back, so only a
  // built index holds it (stb_corpus_update / stb_corpus_remove refuse while it does)
  const_cast<stb_corpus *>(corpus)->ivfpq_live++;
  x->centroids = nullptr; x->codebooks = nullptr; x->codes = nullptr; x->order = nullptr; x->list_off = nullptr;
  x->coarse = nullptr; x->lut = nullptr; x->probe = nullptr; x->cand = nullptr; x->cand_cap = 0; x->cand_rows = nullptr;
  x->keys2 = nullptr; x->tickets = nullptr; x->forced = nullptr; x->n_forced = 0;
  x->b_cap = 0; x->b_q = nullptr; x->b_coarse = nullptr; x->b_probe = nullptr; x->b_lut = nullptr; x->b_kept = nullptr;
  x->b_drop = nullptr; x->b_hits = nullptr; x->b_status = nullptr;
  for (int i = 0; i < 4; ++i) x->last_info[i] = 0;
  x->last_filtered = false;
  x->f_bitmap = nullptr; x->f_words = 0; x->f_elig = nullptr; x->f_ranges = nullptr; x->f_ranges_cap = 0;
  cudaStream_t st = ctx->stream;
  // training sample: every `stride`-th row
  uint64_t ns = std::min<uint64_t>(n, std::max<uint32_t>(train_rows, nlist * 32u));
  const uint64_t stride = std::max<uint64_t>(1, n / ns);
  ns = std::min<uint64_t>(ns, (n + stride - 1) / stride);
  const float4 *X4 = reinterpret_cast<const float4 *>(corpus->rows);
  float *sums = nullptr, *pq_sums = nullptr;
  uint32_t *counts = nullptr, *pq_counts = nullptr, *assign = nullptr;
  IVF_CUDA(cudaMalloc(&x->centroids, (size_t)nlist * STB_D * 4));
  IVF_CUDA(cudaMalloc(&x->codebooks, (size_t)PQ_M * PQ_KSUB * PQ_DSUB * 4));
  IVF_CUDA(cudaMalloc(&sums, (size_t)nlist * STB_D * 4));
  IVF_CUDA(cudaMalloc(&counts, (size_t)(nlist + 1) * 4));
  IVF_CUDA(cudaMalloc(&pq_sums, (size_t)PQ_M * PQ_KSUB * PQ_DSUB * 4));
  IVF_CUDA(cudaMalloc(&pq_counts, (size_t)PQ_M * PQ_KSUB * 4));
  IVF_CUDA(cudaMalloc(&assign, ns * 4));
  // ---- coarse k-means on the sample (strided view of the corpus: stride in rows) --------
  // initial centroids: evenly spaced sample rows, normalised
  IVF_CUDA(cudaMemsetAsync(counts, 0, (size_t)nlist * 4, st));
  ivf_finish_centroids_kernel<<<(nlist + 7) / 8, 256, 0, st>>>(x->centroids, sums, counts, nlist, X4, ns, stride, 0);
  // the strided sample is gathered into a dense buffer so the GEMM kernel sees contiguous rows
  float *sample = nullptr;
  IVF_CUDA(cudaMalloc(&sample, ns * STB_D * 4));
  IVF_CUDA(cudaMemcpy2DAsync(sample, STB_D * 4, corpus->rows, stride * STB_D * 4, STB_D * 4, ns, cudaMemcpyDeviceToDevice, st));
  const float4 *S4 = reinterpret_cast<const float4 *>(sample);
  for (uint32_t it = 0; it < iters; ++it) {
    ivf_assign_kernel<<<(unsigned)((ns + 63) / 64), 256, 0, st>>>(sample, ns, x->centroids, nlist, assign);
    IVF_CUDA(cudaMemsetAsync(sums, 0, (size_t)nlist * STB_D * 4, st));
    IVF_CUDA(cudaMemsetAsync(counts, 0, (size_t)nlist * 4, st));
    ivf_accumulate_kernel<<<(unsigned)((ns + 7) / 8), 256, 0, st>>>(S4, ns, 1, assign, sums, counts);
    ivf_finish_centroids_kernel<<<(nlist + 7) / 8, 256, 0, st>>>(x->centroids, sums, counts, nlist, S4, ns, 1, it + 1);
  }
  // ---- PQ codebooks on the sample residuals -------------------------------------------------
  ivf_assign_kernel<<<(unsigned)((ns + 63) / 64), 256, 0, st>>>(sample, ns, x->centroids, nlist, assign);
  pq_seed_kernel<<<PQ_KSUB, 32, 0, st>>>(x->codebooks, S4, ns, 1, assign, x->centroids);
  IVF_CUDA(cudaFuncSetAttribute(pq_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * PQ_KSUB * PQ_DSUB * 4));
  PqArgs pa;
  pa.X = S4; pa.n = ns; pa.stride = 1; pa.assign = assign; pa.C = x->centroids; pa.cb = x->codebooks;
  pa.sums = pq_sums; pa.counts = pq_counts; pa.codes_out = nullptr;
  for (uint32_t it = 0; it < iters; ++it) {
    IVF_CUDA(cudaMemsetAsync(pq_sums, 0, (size_t)PQ_M * PQ_KSUB * PQ_DSUB * 4, st));
    IVF_CUDA(cudaMemsetAsync(pq_counts, 0, (size_t)PQ_M * PQ_KSUB * 4, st));
    for (int s0 = 0; s0 < PQ_M; s0 += 8) {
      pa.s0 = s0; pa.mode = 0;
      pq_step_kernel<<<ctx->sm_count * 2, 256, 8 * PQ_KSUB * PQ_DSUB * 4, st>>>(pa);
    }
    pq_finish_codebooks_kernel<<<(PQ_M * PQ_KSUB + 255) / 256, 256, 0, st>>>(x->codebooks, pq_sums, pq_counts);
  }
  IVF_CUDA(cudaGetLastError());
  // training buffers go before the add phase allocates its own
  IVF_CUDA(cudaStreamSynchronize(st));
  cudaFree(sums); cudaFree(counts); cudaFree(pq_sums); cudaFree(pq_counts); cudaFree(assign); cudaFree(sample);
  // ---- add: rows [0, n) into empty lists, as stb_ivfpq_extend adds its rows ----------------------
  IVF_CUDA(cudaMalloc(&x->list_off, (size_t)(nlist + 1) * 4));
  IVF_CUDA(cudaMemsetAsync(x->list_off, 0, (size_t)(nlist + 1) * 4, st));
  x->list_off_h.assign(nlist + 1, 0);
  int rc = ivf_add_rows(x, 0, n, "ivfpq_build");
  if (rc != STB_OK) { stb_ivfpq_destroy(x); return rc; }
  // query scratch
  IVF_CUDA(cudaMalloc(&x->coarse, (size_t)nlist * 4));
  IVF_CUDA(cudaMalloc(&x->lut, (size_t)PQ_M * PQ_KSUB * 4));
  IVF_CUDA(cudaMalloc(&x->probe, (size_t)(2 * 1024 + 1) * 4));
  IVF_CUDA(cudaMalloc(&x->cand_rows, (IVF_HOST_TOPK_MAX + IVF_FORCED_CAP) * 4 + 16));   // + the valid-row counter
  IVF_CUDA(cudaMalloc(&x->keys2, (size_t)ADC2_MAX_CTAS * ADC2_KEEP * 8));
  IVF_CUDA(cudaMalloc(&x->tickets, 2 * sizeof(unsigned int)));
  IVF_CUDA(cudaMemsetAsync(x->tickets, 0, 2 * sizeof(unsigned int), ctx->stream));
  IVF_CUDA(cudaGetLastError());
  IVF_CUDA(cudaStreamSynchronize(st));
  ctx->kernel_launches += 3 + iters * 8;                   // training (the add phase counts its own)
  *out = x;
  return STB_OK;
}

int stb_ivfpq_stats(const stb_ivfpq *x, uint64_t *rows, uint32_t *nlist, uint32_t *max_list, uint64_t *bytes) {
  if (!x) { stb_set_error("null index"); return STB_ERR_ARG; }
  if (rows) *rows = x->n;
  if (nlist) *nlist = x->nlist;
  if (max_list) { uint32_t m = 0; for (uint32_t l = 0; l < x->nlist; ++l) m = std::max(m, x->list_off_h[l + 1] - x->list_off_h[l]); *max_list = m; }
  if (bytes) *bytes = x->n * (PQ_M + 4) + (uint64_t)x->nlist * 1024 + PQ_M * PQ_KSUB * PQ_DSUB * 4;
  return STB_OK;
}

// Indexes the rows appended to the corpus since the build or the last extend, with the build's quantisers
// (ivf_add_rows).  A corpus that started a new epoch (cleared) no longer holds the rows the index refers to.
int stb_ivfpq_extend(stb_ivfpq *x, uint64_t *out_added) {
  if (out_added) *out_added = 0;
  if (!x) { stb_set_error("ivfpq_extend: null index"); return STB_ERR_ARG; }
  if (cudaSetDevice(x->ctx->device) != cudaSuccess) { stb_set_error("cudaSetDevice failed"); return STB_ERR_CUDA; }
  const stb_corpus *c = x->corpus;
  if (c->epoch != x->corpus_epoch || c->n < x->n) {
    stb_set_error("ivfpq_extend: the corpus was cleared since the index was built (%llu rows, the index holds %llu)",
                  (unsigned long long)c->n, (unsigned long long)x->n);
    return STB_ERR_STATE;
  }
  const uint64_t m = c->n - x->n;
  if (m == 0) return STB_OK;
  const int rc = ivf_add_rows(x, x->n, m, "ivfpq_extend");
  if (rc == STB_OK && out_added) *out_added = m;
  return rc;
}

}  // extern "C"

// ---- stb_ivfpq_update / stb_ivfpq_remove: the corpus call (api.cu) with the index's edit hooked in ----
// The refusals of another live index and of a corpus in another epoch replace the corpus's refusal of live
// indexes; the edit is planned (every buffer allocated, the forced rows counted) before the corpus writes
// anything and installed once the corpus call has succeeded.
struct IvfHook : StbCorpusHook {
  stb_ivfpq *x;
  const char *who;
  IvfEdit e;
  bool checked = false;               // the corpus call got past its argument checks
  bool edit = false;                  // some indexed row changes
  IvfHook(stb_ivfpq *x_, const char *who_) : x(x_), who(who_), e(x_->ctx->stream) {}
  int check() override {
    const stb_corpus *c = x->corpus;
    if (c->ivfpq_live > 1) {
      stb_set_error("%s: %u IVF-PQ indexes on this corpus refer to its rows; destroy the others first", who, c->ivfpq_live);
      return STB_ERR_STATE;
    }
    if (c->epoch != x->corpus_epoch || c->n < x->n) {
      stb_set_error("%s: the corpus was cleared since the index was built (%llu rows, the index holds %llu)", who,
                    (unsigned long long)c->n, (unsigned long long)x->n);
      return STB_ERR_STATE;
    }
    checked = true;
    return STB_OK;
  }
  // after the corpus call: install the edit, follow the corpus into its new epoch
  int finish(int rc) {
    if (rc != STB_OK || !checked) return rc;
    if (edit) IVF_TRY(ivf_edit_swap(x, e));
    x->corpus_epoch = x->corpus->epoch;
    return STB_OK;
  }
};

// Update: the replaced indexed rows leave their lists (or the forced list) and come back as new entries with
// the list and code of their new value, encoded from the staging buffer.  Nothing is renumbered.
struct IvfUpdateHook : IvfHook {
  const uint64_t *idx;
  uint64_t n;
  IvfUpdateHook(stb_ivfpq *x_, const uint64_t *idx_, uint64_t n_) : IvfHook(x_, "ivfpq_update"), idx(idx_), n(n_) {}
  int begin() override {
    const uint64_t base = x->corpus->row_base;
    uint64_t m = 0;                   // idx is validated: ascending, so the indexed rows come first
    while (m < n && idx[m] - base < x->n) ++m;
    if (m == 0) return STB_OK;
    edit = true;
    staged_rows = m;
    e.m = m; e.n_after = x->n; e.keep_all = false;
    e.rows_h.resize(m);
    uint32_t b = 0;
    for (uint64_t i = 0; i < m; ++i) {
      const uint32_t r = (uint32_t)(idx[i] - base);
      if (r > b) e.keep(b, r, b);
      b = r + 1;
      e.rows_h[i] = r;
    }
    if (x->n > b) e.keep(b, (uint32_t)x->n, b);
    return ivf_edit_alloc(x, e);
  }
  int staged(const float *stage, uint64_t i0, uint64_t m) override {
    if (i0 >= e.m) return STB_OK;
    return ivf_edit_encode(x, e, stage, i0, std::min(m, e.m - i0));
  }
  int ready() override { return edit ? ivf_edit_plan(x, e, who) : STB_OK; }
};

// Remove: the removed indexed rows leave; every entry behind them moves down by the removed rows below it.
struct IvfRemoveHook : IvfHook {
  const uint64_t *ranges;
  uint32_t n_ranges;
  IvfRemoveHook(stb_ivfpq *x_, const uint64_t *r, uint32_t nr) : IvfHook(x_, "ivfpq_remove"), ranges(r), n_ranges(nr) {}
  int begin() override {
    const uint64_t base = x->corpus->row_base;
    uint64_t b = 0, dst = 0;          // ranges are validated: ascending, disjoint, inside the corpus
    for (uint32_t i = 0; i < n_ranges; ++i) {
      const uint64_t rb = std::min(ranges[2 * i] - base, x->n), re = std::min(ranges[2 * i + 1] - base, x->n);
      if (rb == re) break;            // past the indexed rows
      if (rb > b) { e.keep((uint32_t)b, (uint32_t)rb, (uint32_t)dst); dst += rb - b; }
      b = re;
    }
    if (b == 0 && e.n_kept == 0) return STB_OK;   // no indexed row is removed
    if (x->n > b) { e.keep((uint32_t)b, (uint32_t)x->n, (uint32_t)dst); dst += x->n - b; }
    edit = true;
    e.keep_all = false; e.n_after = dst;
    IVF_TRY(ivf_edit_alloc(x, e));
    return ivf_edit_plan(x, e, who);
  }
};

extern "C" {

// Replaces rows of the index's corpus (stb_corpus_update) and re-indexes the replaced indexed rows.
int stb_ivfpq_update(stb_ivfpq *x, const uint64_t *idx, const float *rows, uint64_t n) {
  if (!x) { stb_set_error("ivfpq_update: null index"); return STB_ERR_ARG; }
  IvfUpdateHook h(x, idx, n);
  return h.finish(stb_corpus_update_impl(const_cast<stb_corpus *>(x->corpus), idx, rows, n, "ivfpq_update", &h));
}

// Deletes rows of the index's corpus (stb_corpus_remove) and drops and renumbers the index's entries to match.
int stb_ivfpq_remove(stb_ivfpq *x, const uint64_t *ranges, uint32_t n_ranges) {
  if (!x) { stb_set_error("ivfpq_remove: null index"); return STB_ERR_ARG; }
  IvfRemoveHook h(x, ranges, n_ranges);
  return h.finish(stb_corpus_remove_impl(const_cast<stb_corpus *>(x->corpus), ranges, n_ranges, "ivfpq_remove", &h));
}

// Approximate top-k: probe `nprobe` lists, keep the `rerank` best ADC scores, re-score those
// rows exactly (canonical f64 distance on the f32 corpus rows), return the best top_k by
// (distance,row).  q_dev: 256 f32 on device.  Synchronous (returns host hits).
// fused search (coarse probe + ADC/finish), asynchronous: q, hits and status on the device
static int ivf_fused_launch(stb_ivfpq *x, const float *q_dev, uint32_t nprobe, uint32_t top_k, uint32_t rerank,
                            stb_hit *out_hits_dev, uint32_t *out_status_dev) {
  stb_ctx *ctx = x->ctx;
  cudaStream_t st = ctx->stream;
  uint32_t npow2 = 1; while (npow2 < x->nlist) npow2 <<= 1;
  if (!(ctx->func_attr_mask & (1u << STB_ATTR_IVF_V2))) {
    STB_CUDA(cudaFuncSetAttribute(ivf_coarse_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 8));
    STB_CUDA(cudaFuncSetAttribute(ivf_adc_finish_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ADC2_SMEM));
    ctx->func_attr_mask |= 1u << STB_ATTR_IVF_V2;
  }
  Probe2Args pa;
  pa.C = x->centroids; pa.nlist = x->nlist; pa.nprobe = nprobe; pa.q = q_dev; pa.coarse = x->coarse;
  pa.list_off = x->list_off; pa.cb = x->codebooks; pa.probe = x->probe; pa.lut = x->lut; pa.ticket = x->tickets;
  ivf_coarse_probe_kernel<<<(x->nlist + 31) / 32, 1024, npow2 * 8, st>>>(pa);
  STB_CUDA(cudaGetLastError());
  Adc2Args aa;
  aa.codes = x->codes; aa.list_off = x->list_off; aa.probe = x->probe; aa.nprobe = nprobe; aa.coarse = x->coarse;
  aa.lut = x->lut; aa.order = x->order; aa.keys2 = x->keys2; aa.ticket = x->tickets + 1;
  aa.rows = reinterpret_cast<const float4 *>(x->corpus->rows); aa.row_base = x->corpus->row_base; aa.q = q_dev;
  aa.top_k = top_k; aa.rerank = rerank; aa.forced = x->forced; aa.n_forced = x->n_forced;
  aa.out_hits = out_hits_dev; aa.out_status = out_status_dev;
  ivf_adc_finish_kernel<<<ADC2_MAX_CTAS, ADC2_THREADS, ADC2_SMEM, st>>>(aa);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches += 2;
  return STB_OK;
}

// Asynchronous device-resident form (sharded use: per-rank probe -> all-gather of k hits -> stb_hits_merge_dev).
// out_hits_dev receives top_k entries (unused tail: +inf / UINT64_MAX), out_status_dev[0] = hits, [1] = codes scanned.
int stb_ivfpq_search_dev(stb_ivfpq *x, const float *q_dev, uint32_t nprobe, uint32_t top_k, uint32_t rerank,
                         stb_hit *out_hits_dev, uint32_t *out_status_dev) {
  if (!x || !q_dev || !out_hits_dev || !out_status_dev) { stb_set_error("ivfpq_search_dev: null argument"); return STB_ERR_ARG; }
  if (cudaSetDevice(x->ctx->device) != cudaSuccess) { stb_set_error("cudaSetDevice failed"); return STB_ERR_CUDA; }
  if (top_k == 0 || top_k > 1024) { stb_set_error("ivfpq_search_dev: top_k must be 1..1024"); return STB_ERR_ARG; }
  nprobe = std::max(1u, std::min(std::min(nprobe, x->nlist), 1024u));
  rerank = std::max(top_k, std::min(rerank, (uint32_t)ADC2_RERANK_CAP));
  return ivf_fused_launch(x, q_dev, nprobe, top_k, rerank, out_hits_dev, out_status_dev);
}

// ---- batched search ----
// grows the batch scratch to hold nq (<= IVFB_MAX_NQ) queries; cudaFree synchronises, so a batch still
// in flight finishes before its buffers go
static int ivfb_reserve(stb_ivfpq *x, uint32_t nq) {
  if (nq <= x->b_cap) return STB_OK;
  const uint32_t cap = std::min<uint32_t>(IVFB_MAX_NQ, (nq + 63) / 64 * 64);
  cudaFree(x->b_q); cudaFree(x->b_coarse); cudaFree(x->b_probe); cudaFree(x->b_lut); cudaFree(x->b_kept);
  cudaFree(x->b_drop); cudaFree(x->b_hits); cudaFree(x->b_status);
  x->b_q = nullptr; x->b_coarse = nullptr; x->b_probe = nullptr; x->b_lut = nullptr; x->b_kept = nullptr;
  x->b_drop = nullptr; x->b_hits = nullptr; x->b_status = nullptr;
  x->b_cap = 0;
  STB_CUDA(cudaMalloc(&x->b_q, (size_t)cap * STB_D * 4));
  STB_CUDA(cudaMalloc(&x->b_coarse, (size_t)cap * x->nlist * 4));
  STB_CUDA(cudaMalloc(&x->b_probe, (size_t)cap * IVFB_PROBE_STRIDE(1024, true) * 4));
  STB_CUDA(cudaMalloc(&x->b_lut, (size_t)cap * PQ_M * PQ_KSUB * 4));
  STB_CUDA(cudaMalloc(&x->b_kept, (size_t)cap * IVFB_KEPT * 8));
  STB_CUDA(cudaMalloc(&x->b_drop, (size_t)cap * IVFB_WARPS * 8));
  STB_CUDA(cudaMalloc(&x->b_hits, (size_t)cap * 1024 * sizeof(stb_hit)));
  STB_CUDA(cudaMalloc(&x->b_status, (size_t)cap * 2 * 4));
  x->b_cap = cap;
  return STB_OK;
}

// The filter of a filtered launch: the eligibility pass's outputs and the distance limit.
struct IvfbFilter {
  const uint32_t *bitmap;     // NULL: every indexed row is eligible
  const uint32_t *elig;       // [nlist]
  double max_dist;
};

// four launches for 1 <= nq <= IVFB_MAX_NQ queries (arguments already clamped); asynchronous.
// f != NULL: the filtered search's instantiations of the probe, scan and finish kernels.
static int ivfb_launch(stb_ivfpq *x, const float *q_dev, uint32_t nq, uint32_t nprobe, uint32_t top_k, uint32_t rerank,
                       stb_hit *out_hits_dev, uint32_t *out_status_dev, const IvfbFilter *f = nullptr) {
  stb_ctx *ctx = x->ctx;
  cudaStream_t st = ctx->stream;
  int rc = ivfb_reserve(x, nq);
  if (rc != STB_OK) return rc;
  uint32_t npow2 = 1; while (npow2 < x->nlist) npow2 <<= 1;
  if (!(ctx->func_attr_mask & (1u << STB_ATTR_IVF_BATCH))) {
    STB_CUDA(cudaFuncSetAttribute(ivfb_probe_lut_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 8));
    STB_CUDA(cudaFuncSetAttribute(ivfb_finish_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, IVFB_FIN_SMEM));
    STB_CUDA(cudaFuncSetAttribute(ivfb_probe_lut_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 8));
    STB_CUDA(cudaFuncSetAttribute(ivfb_finish_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, IVFB_FIN_SMEM));
    ctx->func_attr_mask |= 1u << STB_ATTR_IVF_BATCH;
  }
  IvfbArgs a;
  // STB_IVFPQ_BATCH_KEEP=k (1..64): each scan warp keeps only k codes (tests drive the exact slow route)
  const char *keep_env = getenv("STB_IVFPQ_BATCH_KEEP");
  a.keep = keep_env ? std::max(1, std::min(atoi(keep_env), IVFB_WARP_KEEP)) : IVFB_WARP_KEEP;
  a.C = x->centroids; a.nlist = x->nlist; a.nq = nq; a.nprobe = nprobe; a.top_k = top_k; a.rerank = rerank;
  a.list_off = x->list_off; a.cb = x->codebooks; a.codes = x->codes; a.order = x->order;
  a.qs = q_dev; a.coarse = x->b_coarse; a.probe = x->b_probe; a.lut = x->b_lut; a.kept = x->b_kept; a.drop = x->b_drop;
  a.rows = reinterpret_cast<const float4 *>(x->corpus->rows); a.row_base = x->corpus->row_base;
  a.forced = x->forced; a.n_forced = x->n_forced; a.out_hits = out_hits_dev; a.out_status = out_status_dev;
  a.bitmap = f ? f->bitmap : nullptr; a.max_dist = f ? f->max_dist : STB_DEFAULT_MAX_DIST;
  ivfb_coarse_kernel<<<dim3((x->nlist + 31) / 32, (nq + IVFB_QTILE - 1) / IVFB_QTILE), 1024, 0, st>>>(x->centroids, x->nlist, q_dev,
                                                                                                   nq, x->b_coarse);
  STB_CUDA(cudaGetLastError());
  if (!f) {
    ivfb_probe_lut_kernel<false><<<nq, 1024, npow2 * 8, st>>>(x->b_coarse, x->nlist, nprobe, x->list_off, x->codebooks, q_dev,
                                                              x->b_probe, x->b_lut, nullptr);
    STB_CUDA(cudaGetLastError());
    ivfb_scan_kernel<false><<<dim3(IVFB_SCAN_CTAS, nq), IVFB_SCAN_THREADS, 0, st>>>(a);
    STB_CUDA(cudaGetLastError());
    ivfb_finish_kernel<false><<<nq, IVFB_FIN_THREADS, IVFB_FIN_SMEM, st>>>(a);
  } else {
    ivfb_probe_lut_kernel<true><<<nq, 1024, npow2 * 8, st>>>(x->b_coarse, x->nlist, nprobe, x->list_off, x->codebooks, q_dev,
                                                             x->b_probe, x->b_lut, f->elig);
    STB_CUDA(cudaGetLastError());
    ivfb_scan_kernel<true><<<dim3(IVFB_SCAN_CTAS, nq), IVFB_SCAN_THREADS, 0, st>>>(a);
    STB_CUDA(cudaGetLastError());
    ivfb_finish_kernel<true><<<nq, IVFB_FIN_THREADS, IVFB_FIN_SMEM, st>>>(a);
  }
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches += 4;
  x->last_info[0] = nq; x->last_info[1] = nprobe; x->last_info[2] = top_k; x->last_info[3] = rerank;
  x->last_filtered = f != nullptr;
  return STB_OK;
}

static void ivfb_clamp(const stb_ivfpq *x, uint32_t top_k, uint32_t &nprobe, uint32_t &rerank) {
  nprobe = std::max(1u, std::min(std::min(nprobe, x->nlist), 1024u));
  rerank = std::max(top_k, std::min(rerank, (uint32_t)IVFB_RERANK_CAP));
}

int stb_ivfpq_search_batch_dev(stb_ivfpq *x, const float *q_dev, uint32_t nq, uint32_t nprobe, uint32_t top_k,
                               uint32_t rerank, stb_hit *out_hits_dev, uint32_t *out_status_dev) {
  if (!x) { stb_set_error("ivfpq_search_batch_dev: null index"); return STB_ERR_ARG; }
  if (nq == 0) return STB_OK;
  if (!q_dev || !out_hits_dev || !out_status_dev) { stb_set_error("ivfpq_search_batch_dev: null argument"); return STB_ERR_ARG; }
  if (top_k == 0 || top_k > 1024) { stb_set_error("ivfpq_search_batch_dev: top_k must be 1..1024"); return STB_ERR_ARG; }
  if (nq > IVFB_MAX_NQ) { stb_set_error("ivfpq_search_batch_dev: nq must be <= %u", (unsigned)IVFB_MAX_NQ); return STB_ERR_ARG; }
  if (cudaSetDevice(x->ctx->device) != cudaSuccess) { stb_set_error("cudaSetDevice failed"); return STB_ERR_CUDA; }
  ivfb_clamp(x, top_k, nprobe, rerank);
  return ivfb_launch(x, q_dev, nq, nprobe, top_k, rerank, out_hits_dev, out_status_dev);
}

// The host forms' chunk loop (arguments checked and clamped, top_k >= 1): chunks of IVFB_MAX_NQ queries,
// one synchronisation each.
static int ivfb_host_chunks(stb_ivfpq *x, const float *q, uint32_t nq, uint32_t nprobe, uint32_t top_k, uint32_t rerank,
                            stb_hit *out_hits, uint32_t *out_n, uint64_t *out_scanned, const IvfbFilter *f) {
  cudaStream_t st = x->ctx->stream;
  std::vector<uint32_t> status;
  for (uint32_t q0 = 0; q0 < nq; q0 += IVFB_MAX_NQ) {   // one synchronisation per chunk
    const uint32_t m = std::min<uint32_t>(IVFB_MAX_NQ, nq - q0);
    int rc = ivfb_reserve(x, m);
    if (rc != STB_OK) return rc;
    STB_CUDA(cudaMemcpyAsync(x->b_q, q + (size_t)q0 * STB_D, (size_t)m * STB_D * 4, cudaMemcpyHostToDevice, st));
    if ((rc = ivfb_launch(x, x->b_q, m, nprobe, top_k, rerank, x->b_hits, x->b_status, f)) != STB_OK) return rc;
    status.resize(2 * (size_t)m);
    STB_CUDA(cudaMemcpyAsync(out_hits + (size_t)q0 * top_k, x->b_hits, (size_t)m * top_k * sizeof(stb_hit),
                             cudaMemcpyDeviceToHost, st));
    STB_CUDA(cudaMemcpyAsync(status.data(), x->b_status, (size_t)m * 2 * 4, cudaMemcpyDeviceToHost, st));
    STB_CUDA(cudaStreamSynchronize(st));
    for (uint32_t i = 0; i < m; ++i) {
      out_n[q0 + i] = status[2 * i];
      if (out_scanned) out_scanned[q0 + i] = status[2 * i + 1];
    }
  }
  return STB_OK;
}

int stb_ivfpq_search_batch(stb_ivfpq *x, const float *q, uint32_t nq, uint32_t nprobe, uint32_t top_k, uint32_t rerank,
                           stb_hit *out_hits, uint32_t *out_n, uint64_t *out_scanned) {
  if (!x) { stb_set_error("ivfpq_search_batch: null index"); return STB_ERR_ARG; }
  if (nq == 0) return STB_OK;
  if (!q || !out_n || (top_k && !out_hits)) { stb_set_error("ivfpq_search_batch: null argument"); return STB_ERR_ARG; }
  if (top_k > 1024) { stb_set_error("ivfpq_search_batch: top_k must be <= 1024"); return STB_ERR_ARG; }
  if (top_k == 0) {
    for (uint32_t i = 0; i < nq; ++i) { out_n[i] = 0; if (out_scanned) out_scanned[i] = 0; }
    return STB_OK;
  }
  if (cudaSetDevice(x->ctx->device) != cudaSuccess) { stb_set_error("cudaSetDevice failed"); return STB_ERR_CUDA; }
  ivfb_clamp(x, top_k, nprobe, rerank);
  return ivfb_host_chunks(x, q, nq, nprobe, top_k, rerank, out_hits, out_n, out_scanned, nullptr);
}

int stb_ivfpq_search_filtered(stb_ivfpq *x, const float *q, uint32_t nq, uint32_t nprobe, uint32_t top_k, uint32_t rerank,
                              int has_max, double max_distance, const uint64_t *row_ranges, uint32_t n_ranges,
                              stb_hit *out_hits, uint32_t *out_n, uint64_t *out_scanned) {
  if (!x) { stb_set_error("ivfpq_search_filtered: null index"); return STB_ERR_ARG; }
  if (nq == 0) return STB_OK;
  if (!q || !out_n || (top_k && !out_hits)) { stb_set_error("ivfpq_search_filtered: null argument"); return STB_ERR_ARG; }
  if (n_ranges && !row_ranges) { stb_set_error("ivfpq_search_filtered: row_ranges is null"); return STB_ERR_ARG; }
  if (top_k > 1024) { stb_set_error("ivfpq_search_filtered: top_k must be <= 1024"); return STB_ERR_ARG; }
  // global ranges -> local [begin, end) pairs clipped to the indexed rows [row_base, row_base + n)
  std::vector<uint32_t> loc;
  if (row_ranges) {
    loc.reserve(2 * (size_t)n_ranges);
    const int rc = stb_clip_ranges("ivfpq_search_filtered", row_ranges, n_ranges, x->corpus->row_base, x->n,
                                   [&](uint64_t b, uint64_t e) { loc.push_back((uint32_t)b); loc.push_back((uint32_t)e); });
    if (rc != STB_OK) return rc;
  }
  if (top_k == 0 || (row_ranges && loc.empty())) {             // nothing can be returned: no launch
    for (uint32_t i = 0; i < nq; ++i) { out_n[i] = 0; if (out_scanned) out_scanned[i] = 0; }
    for (uint64_t i = 0; i < (uint64_t)nq * top_k; ++i) { out_hits[i].distance = INFINITY; out_hits[i].row = UINT64_MAX; }
    return STB_OK;
  }
  stb_ctx *ctx = x->ctx;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { stb_set_error("cudaSetDevice failed"); return STB_ERR_CUDA; }
  ivfb_clamp(x, top_k, nprobe, rerank);
  cudaStream_t st = ctx->stream;
  // eligibility pass: bitmap of the eligible rows, eligible codes per list
  if (!x->f_elig) STB_CUDA(cudaMalloc(&x->f_elig, (size_t)x->nlist * 4));
  const uint32_t *bitmap = nullptr;
  if (row_ranges) {
    const uint64_t words = (x->n + 31) / 32;
    if (words > x->f_words) {
      cudaFree(x->f_bitmap); x->f_bitmap = nullptr; x->f_words = 0;
      STB_CUDA(cudaMalloc(&x->f_bitmap, words * 4));
      x->f_words = words;
    }
    const uint32_t nr = (uint32_t)(loc.size() / 2);
    if (nr > x->f_ranges_cap) {
      const uint32_t cap = std::max<uint32_t>(nr, 1024);
      cudaFree(x->f_ranges); x->f_ranges = nullptr; x->f_ranges_cap = 0;
      STB_CUDA(cudaMalloc(&x->f_ranges, (size_t)cap * 2 * 4));
      x->f_ranges_cap = cap;
    }
    STB_CUDA(cudaMemcpyAsync(x->f_ranges, loc.data(), loc.size() * 4, cudaMemcpyHostToDevice, st));
    const int rc = stb_launch_row_bitmap(ctx, x->f_ranges, nr, words, x->f_bitmap);
    if (rc != STB_OK) return rc;
    bitmap = x->f_bitmap;
  }
  ivff_elig_kernel<<<(x->nlist + 7) / 8, 256, 0, st>>>(x->list_off, x->order, x->nlist, bitmap, x->f_elig);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches += 1;
  IvfbFilter f;
  f.bitmap = bitmap; f.elig = x->f_elig;
  f.max_dist = has_max ? std::min(max_distance, STB_DEFAULT_MAX_DIST) : STB_DEFAULT_MAX_DIST;   // as stb_search
  const int rc = ivfb_host_chunks(x, q, nq, nprobe, top_k, rerank, out_hits, out_n, out_scanned, &f);
  STB_CUDA(cudaStreamSynchronize(st));                         // `loc` is read by the copy above
  return rc;
}

int stb_ivfpq_search(stb_ivfpq *x, const float *q, uint32_t nprobe, uint32_t top_k, uint32_t rerank,
                     stb_hit *out_hits, uint32_t *out_n, uint64_t *out_scanned) {
  if (!x || !q || !out_hits || !out_n) { stb_set_error("ivfpq_search: null argument"); return STB_ERR_ARG; }
  stb_ctx *ctx = x->ctx;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { stb_set_error("cudaSetDevice failed"); return STB_ERR_CUDA; }
  *out_n = 0;
  if (top_k == 0) return STB_OK;
  if (top_k > IVF_HOST_TOPK_MAX) { stb_set_error("ivfpq_search: top_k must be <= %u", (unsigned)IVF_HOST_TOPK_MAX); return STB_ERR_ARG; }
  nprobe = std::max(1u, std::min(std::min(nprobe, x->nlist), 1024u));
  rerank = std::max(top_k, std::min(rerank, (uint32_t)IVF_HOST_TOPK_MAX));
  cudaStream_t st = ctx->stream;
  memcpy(ctx->q_pin, q, STB_D * sizeof(float));
  STB_CUDA(cudaMemcpyAsync(ctx->q_dev, ctx->q_pin, STB_D * sizeof(float), cudaMemcpyHostToDevice, st));
  if (rerank <= ADC2_RERANK_CAP && top_k <= 1024) {
    // fused search: two launches, one synchronisation
    int frc = ivf_fused_launch(x, ctx->q_dev, nprobe, top_k, rerank, ctx->hits_dev, ctx->status_dev);
    if (frc != STB_OK) return frc;
    STB_CUDA(cudaMemcpyAsync(ctx->status_pin, ctx->status_dev, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    STB_CUDA(cudaMemcpyAsync(ctx->hits_pin, ctx->hits_dev, top_k * sizeof(stb_hit), cudaMemcpyDeviceToHost, st));
    STB_CUDA(cudaStreamSynchronize(st));
    const uint32_t n_out = std::min<uint32_t>(ctx->status_pin[0], top_k);
    memcpy(out_hits, ctx->hits_pin, n_out * sizeof(stb_hit));
    *out_n = n_out;
    if (out_scanned) *out_scanned = ctx->status_pin[1];
    return STB_OK;
  }
  ivf_coarse_kernel<<<(x->nlist + 7) / 8, 256, 0, st>>>(x->centroids, x->nlist, ctx->q_dev, x->coarse);
  uint32_t npow = 1; while (npow < x->nlist) npow <<= 1;
  STB_ATTR_ONCE(ctx, STB_ATTR_IVF_PROBE,
                cudaFuncSetAttribute(ivf_probe_lut_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 8));
  ivf_probe_lut_kernel<<<1, 1024, npow * 8, st>>>(x->coarse, x->nlist, nprobe, x->list_off, x->codebooks, ctx->q_dev, x->probe, x->lut);
  ctx->kernel_launches += 2;
  uint32_t total = 0;
  STB_CUDA(cudaMemcpyAsync(&total, x->probe + 2 * nprobe, 4, cudaMemcpyDeviceToHost, st));
  STB_CUDA(cudaStreamSynchronize(st));
  if (out_scanned) *out_scanned = total;
  int rc;
  uint32_t nv = 0;
  if (total > 0) {
    // warps: enough to spread every list over many warps and fill the GPU, at most 512, and enough
    // that the warps' 64-entry lists hold min(rerank, total) candidates.  When total <= rerank no
    // warp sees more than 64 codes, so every scanned code is re-ranked.
    const uint32_t want = std::min(total, rerank);
    const uint32_t ctas = std::max<uint32_t>(1, std::min<uint32_t>(std::max((total + 2047) / 2048, (want + 511) / 512), 64));
    uint64_t m = (uint64_t)ctas * 8 * 64, m_pad = 1024;
    while (m_pad < m) m_pad <<= 1;
    if (m_pad > x->cand_cap) {
      cudaFree(x->cand); x->cand = nullptr; x->cand_cap = 0;
      STB_CUDA(cudaMalloc(&x->cand, m_pad * sizeof(stb_hit)));
      x->cand_cap = m_pad;
    }
    if (m_pad > m) {   // padding entries: +inf
      std::vector<stb_hit> pad(m_pad - m);
      for (auto &h : pad) { h.distance = INFINITY; h.row = 0xffffffffffffffffull; }
      STB_CUDA(cudaMemcpyAsync(x->cand + m, pad.data(), pad.size() * sizeof(stb_hit), cudaMemcpyHostToDevice, st));
      STB_CUDA(cudaStreamSynchronize(st));
    }
    AdcArgs a;
    a.codes = x->codes; a.list_off = x->list_off; a.probe = x->probe; a.nprobe = nprobe; a.coarse = x->coarse; a.lut = x->lut;
    a.cand = x->cand;
    ivf_adc_kernel<<<ctas, 256, 0, st>>>(a);
    STB_CUDA(cudaGetLastError());
    if ((rc = stb_launch_sort_hits(ctx, x->cand, m_pad)) != STB_OK) return rc;
    // r <= rerank <= IVF_HOST_TOPK_MAX entries of cand_rows; the valid ones come first (sorted by -score)
    const uint32_t r = (uint32_t)std::min<uint64_t>(rerank, m);
    uint32_t *n_valid = x->cand_rows + IVF_HOST_TOPK_MAX + IVF_FORCED_CAP;
    STB_CUDA(cudaMemsetAsync(n_valid, 0, 4, st));
    ivf_pick_rows_kernel<<<(r + 255) / 256, 256, 0, st>>>(x->cand, r, x->order, x->cand_rows, n_valid);
    STB_CUDA(cudaMemcpyAsync(&nv, n_valid, 4, cudaMemcpyDeviceToHost, st));
    STB_CUDA(cudaStreamSynchronize(st));
    ctx->kernel_launches += 2;
  }
  // the forced rows follow the ADC candidates
  if (x->n_forced) {
    STB_CUDA(cudaMemcpyAsync(x->cand_rows + nv, x->forced, (size_t)x->n_forced * 4, cudaMemcpyDeviceToDevice, st));
    nv += x->n_forced;
  }
  if (nv == 0) return STB_OK;
  // exact canonical distances of the nv candidate rows, sorted by (distance,row)
  uint64_t e_pad = 1024;
  while (e_pad < nv) e_pad <<= 1;
  if ((size_t)e_pad > ctx->collect_hits_cap) {
    cudaFree(ctx->collect_hits); ctx->collect_hits = nullptr; ctx->collect_hits_cap = 0;
    STB_CUDA(cudaMalloc(&ctx->collect_hits, e_pad * sizeof(stb_hit)));
    ctx->collect_hits_cap = e_pad;
  }
  if ((rc = stb_launch_exact(ctx, x->corpus->rows, x->corpus->row_base, ctx->q_dev, x->cand_rows, nv, STB_DEFAULT_MAX_DIST,
                             ctx->collect_hits, e_pad, ctx->collect_count + 1)) != STB_OK) return rc;
  if ((rc = stb_launch_sort_hits(ctx, ctx->collect_hits, e_pad)) != STB_OK) return rc;
  unsigned long long pass = 0;
  STB_CUDA(cudaMemcpyAsync(&pass, ctx->collect_count + 1, sizeof(pass), cudaMemcpyDeviceToHost, st));
  STB_CUDA(cudaStreamSynchronize(st));
  const uint32_t n_out = (uint32_t)std::min<unsigned long long>(pass, top_k);
  if (n_out) {
    STB_CUDA(cudaMemcpyAsync(out_hits, ctx->collect_hits, n_out * sizeof(stb_hit), cudaMemcpyDeviceToHost, st));
    STB_CUDA(cudaStreamSynchronize(st));
  }
  *out_n = n_out;
  return STB_OK;
}

int stb_debug_ivfpq_export(const stb_ivfpq *x, float *centroids, float *codebooks, uint32_t *list_off, uint32_t *order,
                           uint8_t *codes, uint32_t *forced) {
  if (!x) { stb_set_error("ivfpq_export: null index"); return STB_ERR_ARG; }
  if (cudaSetDevice(x->ctx->device) != cudaSuccess) { stb_set_error("cudaSetDevice failed"); return STB_ERR_CUDA; }
  const uint64_t listed = x->list_off_h[x->nlist];
  STB_CUDA(cudaStreamSynchronize(x->ctx->stream));
  if (centroids) STB_CUDA(cudaMemcpy(centroids, x->centroids, (size_t)x->nlist * STB_D * 4, cudaMemcpyDeviceToHost));
  if (codebooks) STB_CUDA(cudaMemcpy(codebooks, x->codebooks, (size_t)PQ_M * PQ_KSUB * PQ_DSUB * 4, cudaMemcpyDeviceToHost));
  if (list_off) memcpy(list_off, x->list_off_h.data(), (size_t)(x->nlist + 1) * 4);
  if (order && listed) STB_CUDA(cudaMemcpy(order, x->order, listed * 4, cudaMemcpyDeviceToHost));
  if (codes && listed) STB_CUDA(cudaMemcpy(codes, x->codes, listed * PQ_M, cudaMemcpyDeviceToHost));
  if (forced && x->n_forced) STB_CUDA(cudaMemcpy(forced, x->forced, (size_t)x->n_forced * 4, cudaMemcpyDeviceToHost));
  return STB_OK;
}

int stb_debug_ivfpq_batch_last(const stb_ivfpq *x, uint32_t i, uint32_t info[4], float *coarse, uint32_t *probe,
                               float *lut) {
  if (!x) { stb_set_error("ivfpq_batch_last: null index"); return STB_ERR_ARG; }
  if (x->last_info[0] == 0) { stb_set_error("ivfpq_batch_last: no batched search yet"); return STB_ERR_STATE; }
  if (i >= x->last_info[0]) { stb_set_error("ivfpq_batch_last: query %u of %u", i, x->last_info[0]); return STB_ERR_ARG; }
  if (cudaSetDevice(x->ctx->device) != cudaSuccess) { stb_set_error("cudaSetDevice failed"); return STB_ERR_CUDA; }
  STB_CUDA(cudaStreamSynchronize(x->ctx->stream));
  const uint32_t nprobe = x->last_info[1];
  if (info) for (int k = 0; k < 4; ++k) info[k] = x->last_info[k];
  if (coarse) STB_CUDA(cudaMemcpy(coarse, x->b_coarse + (size_t)i * x->nlist, (size_t)x->nlist * 4, cudaMemcpyDeviceToHost));
  const size_t stride = x->last_filtered ? IVFB_PROBE_STRIDE(nprobe, true) : IVFB_PROBE_STRIDE(nprobe, false);
  if (probe) STB_CUDA(cudaMemcpy(probe, x->b_probe + (size_t)i * stride, (size_t)nprobe * 4, cudaMemcpyDeviceToHost));
  if (lut) STB_CUDA(cudaMemcpy(lut, x->b_lut + (size_t)i * PQ_M * PQ_KSUB, (size_t)PQ_M * PQ_KSUB * 4, cudaMemcpyDeviceToHost));
  return STB_OK;
}

}  // extern "C"

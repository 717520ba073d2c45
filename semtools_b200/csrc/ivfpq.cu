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
//   codes      [n][32] u8 sorted by list, order[n] = local row of each code, list_off[nlist+1]
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
#include <vector>

#include "common.cuh"

#define PQ_M 32
#define PQ_DSUB 8
#define PQ_KSUB 256
#define IVF_FORCED_CAP 1024        // forced rows per index; more -> the build fails with STB_ERR_STATE
#define IVF_HOST_TOPK_MAX 4096     // stb_ivfpq_search: top_k and rerank cap of the multi-launch search
#define IVF_NO_LIST 0xffffffffu    // assign[] of a forced row

struct stb_ivfpq {
  stb_ctx *ctx;
  const stb_corpus *corpus;
  uint32_t nlist;
  uint64_t n;                 // rows indexed (listed + forced)
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
// forced rows (warp per row): assign[i] = IVF_NO_LIST, local row appended to forced[] (count in
// *n_forced; entries past `cap` are counted, not written)
__global__ void ivf_flag_forced_kernel(const float4 *__restrict__ X, uint64_t n, uint32_t *assign, uint32_t *forced,
                                       uint32_t cap, uint32_t *n_forced) {
  const int lane = threadIdx.x & 31;
  const uint64_t i = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= n) return;
  const float4 v0 = __ldg(X + i * STB_ROW_F4 + 2 * lane), v1 = __ldg(X + i * STB_ROW_F4 + 2 * lane + 1);
  if (!ivf_forced(ivf_warp_ss(v0, v1)) || lane != 0) return;
  assign[i] = IVF_NO_LIST;
  const uint32_t k = atomicAdd(n_forced, 1u);
  if (k < cap) forced[k] = (uint32_t)i;
}
__global__ void ivf_hist_kernel(const uint32_t *assign, uint64_t n, uint32_t *hist) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && assign[i] != IVF_NO_LIST) atomicAdd(hist + assign[i], 1u);
}
__global__ void ivf_scatter_kernel(const uint32_t *assign, uint64_t n, uint32_t *cursor, const uint8_t *codes_row,
                                   uint8_t *codes, uint32_t *order) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || assign[i] == IVF_NO_LIST) return;
  const uint32_t pos = atomicAdd(cursor + assign[i], 1u);
  order[pos] = (uint32_t)i;
  const uint4 *src = reinterpret_cast<const uint4 *>(codes_row + i * PQ_M);
  uint4 *dst = reinterpret_cast<uint4 *>(codes + (size_t)pos * PQ_M);
  dst[0] = src[0]; dst[1] = src[1];
}

// ------------------------------------------------------------------ query kernels -----
// coarse[j] = q^ . c_j   (warp per centroid)
__global__ void ivf_coarse_kernel(const float *C, uint32_t nlist, const float *q, float *coarse) {
  const int lane = threadIdx.x & 31;
  const uint32_t c = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (c >= nlist) return;
  const float4 *cr = reinterpret_cast<const float4 *>(C + (size_t)c * STB_D), *q4 = reinterpret_cast<const float4 *>(q);
  const float4 a0 = __ldg(cr + 2 * lane), a1 = __ldg(cr + 2 * lane + 1), b0 = __ldg(q4 + 2 * lane), b1 = __ldg(q4 + 2 * lane + 1);
  float d = a0.x * b0.x + a0.y * b0.y + a0.z * b0.z + a0.w * b0.w + a1.x * b1.x + a1.y * b1.y + a1.z * b1.z + a1.w * b1.w;
  float qq = b0.x * b0.x + b0.y * b0.y + b0.z * b0.z + b0.w * b0.w + b1.x * b1.x + b1.y * b1.y + b1.z * b1.z + b1.w * b1.w;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) { d += __shfl_xor_sync(0xffffffffu, d, off); qq += __shfl_xor_sync(0xffffffffu, qq, off); }
  if (lane == 0) coarse[c] = qq > 0.f ? d * rsqrtf(qq) : 0.f;
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
  if (threadIdx.x == 0) { float s = 0.f; for (int i = 0; i < STB_D; ++i) s += sq[i] * sq[i]; s_inv = s > 0.f ? rsqrtf(s) : 0.f; }
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
  for (int i = threadIdx.x; i < PQ_M * PQ_KSUB; i += blockDim.x) {
    const int s = i / PQ_KSUB;
    const float *e = cb + (size_t)i * PQ_DSUB;
    float d = 0.f;
#pragma unroll
    for (int t = 0; t < 8; ++t) d = fmaf(sq[s * 8 + t] * inv, e[t], d);
    lut[i] = d;
  }
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
// Default since round 2 (validated on hardware); STB_IVFPQ_V1=1 selects the multi-launch search above.
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
    float d = a0.x * b0.x + a0.y * b0.y + a0.z * b0.z + a0.w * b0.w + a1.x * b1.x + a1.y * b1.y + a1.z * b1.z + a1.w * b1.w;
    float qq = b0.x * b0.x + b0.y * b0.y + b0.z * b0.z + b0.w * b0.w + b1.x * b1.x + b1.y * b1.y + b1.z * b1.z + b1.w * b1.w;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) { d += __shfl_xor_sync(0xffffffffu, d, off); qq += __shfl_xor_sync(0xffffffffu, qq, off); }
    if (lane == 0) { a.coarse[c] = qq > 0.f ? d * rsqrtf(qq) : 0.f; __threadfence(); }
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
  if (threadIdx.x == 0) { float s = 0.f; for (int i = 0; i < STB_D; ++i) s += sq[i] * sq[i]; s_inv = s > 0.f ? rsqrtf(s) : 0.f; }
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
  for (int i = threadIdx.x; i < PQ_M * PQ_KSUB; i += blockDim.x) {
    const int sub = i / PQ_KSUB;
    const float *e = a.cb + (size_t)i * PQ_DSUB;
    float d = 0.f;
#pragma unroll
    for (int t = 0; t < 8; ++t) d = fmaf(sq[sub * 8 + t] * inv, e[t], d);
    a.lut[i] = d;
  }
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

// ------------------------------------------------------------------ host side ---------
extern "C" {

int stb_ivfpq_destroy(stb_ivfpq *x) {
  if (!x) return STB_OK;
  cudaFree(x->centroids); cudaFree(x->codebooks); cudaFree(x->codes); cudaFree(x->order); cudaFree(x->list_off);
  cudaFree(x->coarse); cudaFree(x->lut); cudaFree(x->probe); cudaFree(x->cand); cudaFree(x->cand_rows);
  cudaFree(x->keys2); cudaFree(x->tickets); cudaFree(x->forced);
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
  x->ctx = ctx; x->corpus = corpus; x->nlist = nlist; x->n = n;
  x->centroids = nullptr; x->codebooks = nullptr; x->codes = nullptr; x->order = nullptr; x->list_off = nullptr;
  x->coarse = nullptr; x->lut = nullptr; x->probe = nullptr; x->cand = nullptr; x->cand_cap = 0; x->cand_rows = nullptr;
  x->keys2 = nullptr; x->tickets = nullptr; x->forced = nullptr; x->n_forced = 0;
  cudaStream_t st = ctx->stream;
  // training sample: every `stride`-th row
  uint64_t ns = std::min<uint64_t>(n, std::max<uint32_t>(train_rows, nlist * 32u));
  const uint64_t stride = std::max<uint64_t>(1, n / ns);
  ns = std::min<uint64_t>(ns, (n + stride - 1) / stride);
  const float4 *X4 = reinterpret_cast<const float4 *>(corpus->rows);
  float *sums = nullptr, *pq_sums = nullptr;
  uint32_t *counts = nullptr, *pq_counts = nullptr, *assign = nullptr, *cursor = nullptr;
  uint8_t *codes_row = nullptr;
  IVF_CUDA(cudaMalloc(&x->centroids, (size_t)nlist * STB_D * 4));
  IVF_CUDA(cudaMalloc(&x->codebooks, (size_t)PQ_M * PQ_KSUB * PQ_DSUB * 4));
  IVF_CUDA(cudaMalloc(&sums, (size_t)nlist * STB_D * 4));
  IVF_CUDA(cudaMalloc(&counts, (size_t)(nlist + 1) * 4));
  IVF_CUDA(cudaMalloc(&pq_sums, (size_t)PQ_M * PQ_KSUB * PQ_DSUB * 4));
  IVF_CUDA(cudaMalloc(&pq_counts, (size_t)PQ_M * PQ_KSUB * 4));
  IVF_CUDA(cudaMalloc(&assign, n * 4));
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
  // ---- add: assign + encode every row, then group by list --------------------------------------
  IVF_CUDA(cudaMalloc(&codes_row, n * PQ_M));
  IVF_CUDA(cudaMalloc(&x->codes, n * PQ_M));
  IVF_CUDA(cudaMalloc(&x->order, n * 4));
  IVF_CUDA(cudaMalloc(&x->list_off, (size_t)(nlist + 1) * 4));
  IVF_CUDA(cudaMalloc(&cursor, (size_t)nlist * 4));
  ivf_assign_kernel<<<(unsigned)((n + 63) / 64), 256, 0, st>>>(corpus->rows, n, x->centroids, nlist, assign);
  pa.X = X4; pa.n = n; pa.stride = 1; pa.codes_out = codes_row;
  for (int s0 = 0; s0 < PQ_M; s0 += 8) {
    pa.s0 = s0; pa.mode = 1;
    pq_step_kernel<<<ctx->sm_count * 2, 256, 8 * PQ_KSUB * PQ_DSUB * 4, st>>>(pa);
  }
  // forced rows leave the lists (assign = IVF_NO_LIST) for the side list; counts[nlist] is their count
  IVF_CUDA(cudaMalloc(&x->forced, IVF_FORCED_CAP * 4));
  IVF_CUDA(cudaMemsetAsync(counts, 0, (size_t)(nlist + 1) * 4, st));
  ivf_flag_forced_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(X4, n, assign, x->forced, IVF_FORCED_CAP, counts + nlist);
  ivf_hist_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(assign, n, counts);
  std::vector<uint32_t> hist(nlist + 1);
  IVF_CUDA(cudaMemcpyAsync(hist.data(), counts, (size_t)(nlist + 1) * 4, cudaMemcpyDeviceToHost, st));
  IVF_CUDA(cudaStreamSynchronize(st));
  if (hist[nlist] > IVF_FORCED_CAP) {
    stb_set_error("ivfpq_build: %u rows are non-finite or have an fp32 squared norm outside [1e-30, 1e30] (at most %u)",
                  hist[nlist], (unsigned)IVF_FORCED_CAP);
    cudaFree(sums); cudaFree(counts); cudaFree(pq_sums); cudaFree(pq_counts); cudaFree(assign); cudaFree(cursor);
    cudaFree(codes_row); cudaFree(sample);
    stb_ivfpq_destroy(x);
    return STB_ERR_STATE;
  }
  x->n_forced = hist[nlist];
  {  // ascending, so the side list does not depend on the order the atomics ran in
    std::vector<uint32_t> f(x->n_forced);
    IVF_CUDA(cudaMemcpyAsync(f.data(), x->forced, (size_t)x->n_forced * 4, cudaMemcpyDeviceToHost, st));
    IVF_CUDA(cudaStreamSynchronize(st));
    std::sort(f.begin(), f.end());
    IVF_CUDA(cudaMemcpyAsync(x->forced, f.data(), (size_t)x->n_forced * 4, cudaMemcpyHostToDevice, st));
    IVF_CUDA(cudaStreamSynchronize(st));
  }
  x->list_off_h.assign(nlist + 1, 0);
  for (uint32_t l = 0; l < nlist; ++l) x->list_off_h[l + 1] = x->list_off_h[l] + hist[l];
  IVF_CUDA(cudaMemcpyAsync(x->list_off, x->list_off_h.data(), (size_t)(nlist + 1) * 4, cudaMemcpyHostToDevice, st));
  IVF_CUDA(cudaMemcpyAsync(cursor, x->list_off_h.data(), (size_t)nlist * 4, cudaMemcpyHostToDevice, st));
  ivf_scatter_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(assign, n, cursor, codes_row, x->codes, x->order);
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
  cudaFree(sums); cudaFree(counts); cudaFree(pq_sums); cudaFree(pq_counts); cudaFree(assign); cudaFree(cursor);
  cudaFree(codes_row); cudaFree(sample);
  ctx->kernel_launches += 8 + iters * 12;
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
  const char *v1_env = getenv("STB_IVFPQ_V1");            // STB_IVFPQ_V1=1: the round-1 multi-launch search
  if (!(v1_env && v1_env[0] == '1') && rerank <= ADC2_RERANK_CAP && top_k <= 1024) {
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

}  // extern "C"

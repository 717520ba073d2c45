// K2 threshold mode: every row under a distance threshold for a batch of queries (stb_search_batch_threshold).
//
// Semantics: Q independent search_documents calls with max_distance set (reference src/search/mod.rs:88-89,
// 115-116): every row with canonical distance < M, ordered by (distance, row).  The tensor-core pass is K2's
// candidate-emitting wgmma GEMM (batch_scan.cu, STB_EPI_EMIT and its exactly sized variant STB_EPI_EMIT_SIZED); this file holds the
// steps around it and the exact finish.
#include <math_constants.h>

#include <algorithm>

#include <cub/device/device_segmented_radix_sort.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include "common.cuh"

// =========================================================================================
// The emission threshold is given, not sampled (api.cu: thr_emission_value, DESIGN §5):
//   thr = RD_f32(((1 - M) - EPS) - delta)  for the queries the tensor path answers, +inf for the rest.
// A row with canonical d < M has exact cosine c > 1 - M - delta, so its score a >= c - EPS >= thr.
// Pipeline: thresholds -> emitting GEMM (STB_EPI_EMIT, 64 keys per (query, CTA)) -> [queries with an overflowed
// segment: STB_EPI_EMIT_SIZED into exactly sized segments] -> compact -> sort by row -> exact re-score, d < M ->
// stable sort by distance -> hits.
// =========================================================================================

// One warp per query of the tile-padded batch: +inf (never emits) for padding queries, queries that cannot be
// normalised and the zero query (canonical distance 0 to a zero row, score 0); t for every other query.
__global__ void __launch_bounds__(256)
stb_batch_thr_dist_kernel(const float4 *__restrict__ q, const uint32_t *__restrict__ q_bad, uint32_t nq,
                          uint32_t q_pad, float t, float *thr) {
  const int lane = threadIdx.x & 31;
  const uint32_t i = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= q_pad) return;
  bool nz = false;
  if (i < nq) {
    const float4 v0 = __ldg(q + (size_t)i * STB_ROW_F4 + 2 * lane), v1 = __ldg(q + (size_t)i * STB_ROW_F4 + 2 * lane + 1);
    nz = (v0.x != 0.f) | (v0.y != 0.f) | (v0.z != 0.f) | (v0.w != 0.f) | (v1.x != 0.f) | (v1.y != 0.f) |
         (v1.z != 0.f) | (v1.w != 0.f);
  }
  nz = __any_sync(0xffffffffu, nz);
  if (lane == 0) thr[i] = (i < nq && nz && !q_bad[i]) ? t : CUDART_INF_F;
}

int stb_launch_batch_thr_dist(stb_ctx *ctx, const float *q_dev, const uint32_t *q_bad, uint32_t nq, uint32_t q_pad,
                              float t, float *thr) {
  stb_batch_thr_dist_kernel<<<(q_pad + 7) / 8, 256, 0, ctx->stream>>>(reinterpret_cast<const float4 *>(q_dev), q_bad,
                                                                      nq, q_pad, t, thr);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// One warp per (query, segment) of the first pass: segment idx's keys (count cnt[idx] <= seg_cap) to
// out[dst[idx] ..]; dst = ~0: the query is not answered from this pass.
__global__ void __launch_bounds__(256)
stb_batch_thr_compact_kernel(const uint64_t *__restrict__ keys, const uint32_t *__restrict__ cnt,
                             const uint64_t *__restrict__ dst, uint64_t n_pairs, uint32_t seg_cap, uint64_t *out) {
  const int lane = threadIdx.x & 31;
  const uint64_t idx = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (idx >= n_pairs) return;
  const uint64_t o = __ldg(dst + idx);
  if (o == ~0ull) return;
  const uint32_t c = __ldg(cnt + idx);
  for (uint32_t j = lane; j < c; j += 32) out[o + j] = __ldg(keys + idx * seg_cap + j);
}

int stb_launch_batch_thr_compact(stb_ctx *ctx, const uint64_t *keys, const uint32_t *cnt, const uint64_t *dst,
                                 uint64_t n_pairs, uint32_t seg_cap, uint64_t *out) {
  if (n_pairs == 0) return STB_OK;
  stb_batch_thr_compact_kernel<<<(unsigned)((n_pairs + 7) / 8), 256, 0, ctx->stream>>>(keys, cnt, dst, n_pairs, seg_cap, out);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// One warp per slot r of the re-emission batch (r < r_pad): the f32 query src[idx[r]] and its threshold, for
// the query shadow builder; padding slots get thr = +inf.
__global__ void __launch_bounds__(256)
stb_batch_thr_gather_kernel(const float4 *__restrict__ src, const float *__restrict__ thr_src,
                            const uint32_t *__restrict__ idx, uint32_t n, uint32_t r_pad, float4 *dst, float *thr_dst) {
  const int lane = threadIdx.x & 31;
  const uint32_t r = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= r_pad) return;
  if (r < n) {
    const uint32_t i = __ldg(idx + r);
    dst[(size_t)r * STB_ROW_F4 + 2 * lane] = __ldg(src + (size_t)i * STB_ROW_F4 + 2 * lane);
    dst[(size_t)r * STB_ROW_F4 + 2 * lane + 1] = __ldg(src + (size_t)i * STB_ROW_F4 + 2 * lane + 1);
  }
  if (lane == 0) thr_dst[r] = (r < n) ? __ldg(thr_src + __ldg(idx + r)) : CUDART_INF_F;
}

int stb_launch_batch_thr_gather(stb_ctx *ctx, const float *src, const float *thr_src, const uint32_t *idx, uint32_t n,
                                uint32_t r_pad, float *dst, float *thr_dst) {
  stb_batch_thr_gather_kernel<<<(r_pad + 7) / 8, 256, 0, ctx->stream>>>(reinterpret_cast<const float4 *>(src), thr_src,
                                                                        idx, n, r_pad, reinterpret_cast<float4 *>(dst), thr_dst);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// One CTA per answered query (slot s): its keys keys[off[s], off[s+1]) (sorted by row) are re-scored with the
// canonical helpers against query qidx[s].  Passing rows (d < limit, strict) -> (distance bits, global row);
// the others -> (+inf bits, UINT64_MAX), which sort after every pass.  pass[s] = rows that pass.  A
// non-negative double's bits order as the double does, so the distance sort can run on the bits.
__global__ void __launch_bounds__(256)
stb_batch_thr_rescore_kernel(const uint64_t *__restrict__ keys, const int *__restrict__ off,
                             const uint32_t *__restrict__ qidx, const float *__restrict__ queries,
                             const float4 *__restrict__ rows, uint64_t row_base, double limit,
                             uint64_t *dist_bits, uint64_t *grow, uint32_t *pass) {
  __shared__ double sqd[STB_D];
  __shared__ double s_q2;
  __shared__ uint32_t s_pass;
  const uint32_t s = blockIdx.x;
  const float *qf = queries + (size_t)__ldg(qidx + s) * STB_D;
  for (int i = threadIdx.x; i < STB_D; i += blockDim.x) sqd[i] = (double)__ldg(qf + i);
  if (threadIdx.x == 0) s_pass = 0;
  __syncthreads();
  if (threadIdx.x == 0) s_q2 = stb_canon_q2(sqd);
  __syncthreads();
  const double q2 = s_q2;
  uint32_t np = 0;
  for (int j = __ldg(off + s) + (int)threadIdx.x; j < __ldg(off + s + 1); j += blockDim.x) {
    const uint32_t row = stb_key_row(keys[j]);
    double ab, r2;
    stb_canon_dot<true>(sqd, rows + (size_t)row * STB_ROW_F4, ab, r2);
    const double dist = stb_canon_dist(ab, q2, r2);
    const bool ok = dist < limit;
    dist_bits[j] = ok ? (uint64_t)__double_as_longlong(dist) : (uint64_t)__double_as_longlong(CUDART_INF);
    grow[j] = ok ? row_base + row : 0xffffffffffffffffull;
    np += ok ? 1u : 0u;
  }
  atomicAdd(&s_pass, np);
  __syncthreads();
  if (threadIdx.x == 0) pass[s] = s_pass;
}

int stb_launch_batch_thr_rescore(stb_ctx *ctx, const uint64_t *keys, const int *off, const uint32_t *qidx,
                                 uint32_t n_slots, const float *queries_dev, const float *rows, uint64_t row_base,
                                 double limit, uint64_t *dist_bits, uint64_t *grow, uint32_t *pass) {
  if (n_slots == 0) return STB_OK;
  stb_batch_thr_rescore_kernel<<<n_slots, 256, 0, ctx->stream>>>(keys, off, qidx, queries_dev,
                                                                 reinterpret_cast<const float4 *>(rows), row_base,
                                                                 limit, dist_bits, grow, pass);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// One CTA per answered query: its first pass[s] sorted pairs -> out[dst[s] ..] as stb_hit.
__global__ void __launch_bounds__(256)
stb_batch_thr_write_kernel(const uint64_t *__restrict__ dist_bits, const uint64_t *__restrict__ grow,
                           const int *__restrict__ off, const uint32_t *__restrict__ pass,
                           const uint64_t *__restrict__ dst, stb_hit *out) {
  const uint32_t s = blockIdx.x;
  const int o = __ldg(off + s);
  const uint32_t n = __ldg(pass + s);
  stb_hit *w = out + __ldg(dst + s);
  for (uint32_t j = threadIdx.x; j < n; j += blockDim.x) {
    stb_hit h;
    h.distance = __longlong_as_double((long long)dist_bits[o + j]);
    h.row = grow[o + j];
    w[j] = h;
  }
}

int stb_launch_batch_thr_write(stb_ctx *ctx, const uint64_t *dist_bits, const uint64_t *grow, const int *off,
                               const uint32_t *pass, uint32_t n_slots, const uint64_t *dst, stb_hit *out) {
  if (n_slots == 0) return STB_OK;
  stb_batch_thr_write_kernel<<<n_slots, 256, 0, ctx->stream>>>(dist_bits, grow, off, pass, dst, out);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// Segmented sorts of the answered queries' candidates, segment s = [off[s], off[s+1]):
//   rows: keys ordered by the row in their low 32 bits (rows are distinct within a segment)
//   dist: (distance bits, global row) pairs stably ordered by distance; the rows already ascend within a
//         segment, so the result is in (distance, row) order, stb_hit_less's
// stb_batch_thr_sort_bytes: the scratch either sort needs for n_items keys in n_slots segments.
int stb_batch_thr_sort_bytes(stb_ctx *ctx, int n_items, uint32_t n_slots, const int *off, size_t *bytes) {
  size_t b1 = 0, b2 = 0;
  STB_CUDA(cub::DeviceSegmentedRadixSort::SortKeys(nullptr, b1, (const uint64_t *)nullptr, (uint64_t *)nullptr, n_items,
                                                   (int)n_slots, off, off + 1, 0, 32, ctx->stream));
  STB_CUDA(cub::DeviceSegmentedSort::StableSortPairs(nullptr, b2, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                                     (const uint64_t *)nullptr, (uint64_t *)nullptr, n_items,
                                                     (int)n_slots, off, off + 1, ctx->stream));
  *bytes = std::max<size_t>(std::max(b1, b2), 1);
  return STB_OK;
}

int stb_batch_thr_sort_rows(stb_ctx *ctx, void *tmp, size_t tmp_bytes, int n_items, uint32_t n_slots, const int *off,
                            const uint64_t *keys_in, uint64_t *keys_out) {
  if (n_items == 0) return STB_OK;
  STB_CUDA(cub::DeviceSegmentedRadixSort::SortKeys(tmp, tmp_bytes, keys_in, keys_out, n_items, (int)n_slots, off, off + 1,
                                                   0, 32, ctx->stream));
  ctx->kernel_launches++;
  return STB_OK;
}

int stb_batch_thr_sort_dist(stb_ctx *ctx, void *tmp, size_t tmp_bytes, int n_items, uint32_t n_slots, const int *off,
                            const uint64_t *dist_bits, uint64_t *dist_out, const uint64_t *grow, uint64_t *grow_out) {
  if (n_items == 0) return STB_OK;
  STB_CUDA(cub::DeviceSegmentedSort::StableSortPairs(tmp, tmp_bytes, dist_bits, dist_out, grow, grow_out, n_items,
                                                     (int)n_slots, off, off + 1, ctx->stream));
  ctx->kernel_launches++;
  return STB_OK;
}

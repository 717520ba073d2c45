// K4: merge per-shard hit lists by (distance,row) -- the final sort_by + take of
// reference src/search/mod.rs:107-119 (and src/workspace/store.rs:538-543) applied
// across row shards.  Latency-bound: n_lists*per_list*16 bytes in, top_k*16 out.
#include <math_constants.h>

#include "common.cuh"

#define STB_MERGE_CAP 4096   // hits one CTA sorts in shared memory (64 KiB)

__global__ void __launch_bounds__(256, 1)
stb_hits_merge_kernel(const stb_hit *lists, uint32_t total, uint32_t n_sort, uint32_t top_k,
                      stb_hit *out) {
  extern __shared__ __align__(16) unsigned char smem[];
  double *sd = reinterpret_cast<double *>(smem);
  uint64_t *sr = reinterpret_cast<uint64_t *>(smem + (size_t)n_sort * sizeof(double));
  for (uint32_t i = threadIdx.x; i < n_sort; i += blockDim.x) {
    if (i < total) {
      stb_hit h = lists[i];
      // NaN distances never leave the scan; treat anything unordered as padding
      bool ok = h.distance == h.distance && h.row != 0xffffffffffffffffull;
      sd[i] = ok ? h.distance : CUDART_INF;
      sr[i] = ok ? h.row : 0xffffffffffffffffull;
    } else {
      sd[i] = CUDART_INF;
      sr[i] = 0xffffffffffffffffull;
    }
  }
  __syncthreads();
  stb_cta_sort_hits(sd, sr, n_sort);
  stb_write_hits(out, sd, sr, min(top_k, n_sort), top_k);
}

// Batched form: lists[n_lists][nq][per_list] -> out[nq][top_k]; one CTA per query.
__global__ void __launch_bounds__(128)
stb_hits_merge_batch_kernel(const stb_hit *lists, uint32_t n_lists, uint32_t nq, uint32_t per_list,
                            uint32_t n_sort, uint32_t top_k, stb_hit *out) {
  extern __shared__ __align__(16) unsigned char smem[];
  double *sd = reinterpret_cast<double *>(smem);
  uint64_t *sr = reinterpret_cast<uint64_t *>(smem + (size_t)n_sort * sizeof(double));
  const uint32_t q = blockIdx.x, total = n_lists * per_list;
  for (uint32_t i = threadIdx.x; i < n_sort; i += blockDim.x) {
    double d = CUDART_INF;
    uint64_t r = 0xffffffffffffffffull;
    if (i < total) {
      const stb_hit h = lists[((size_t)(i / per_list) * nq + q) * per_list + (i % per_list)];
      if (h.distance == h.distance && h.row != 0xffffffffffffffffull) { d = h.distance; r = h.row; }
    }
    sd[i] = d; sr[i] = r;
  }
  __syncthreads();
  stb_cta_sort_hits(sd, sr, n_sort);
  stb_write_hits(out + (size_t)q * top_k, sd, sr, min(top_k, n_sort), top_k);
}

// ---- sharded K2: exchange of the nq x k per-rank hits over NVLink peer memory -------------------
// Slot layout (per rank, per parity): flags[world] u64 | status[world][max_nq] u32 | hits[world][max_nq][max_k].
__device__ __forceinline__ unsigned long long *bx_flags(unsigned char *slot) { return reinterpret_cast<unsigned long long *>(slot); }
__device__ __forceinline__ uint32_t *bx_status(unsigned char *slot, uint32_t world) { return reinterpret_cast<uint32_t *>(slot + (size_t)world * 8); }
__device__ __forceinline__ stb_hit *bx_hits(unsigned char *slot, uint32_t world, uint32_t max_nq) {
  return reinterpret_cast<stb_hit *>(slot + (((size_t)world * 8 + (size_t)world * max_nq * 4 + 15) & ~(size_t)15));
}

// Push: CTA q stores query q's k hits + status into lane `rank` of EVERY rank's slot (its own included);
// the last CTA to finish (device ticket) release-stores the batch sequence number into every rank's flag.
__global__ void __launch_bounds__(128)
stb_batch_xchg_push_kernel(const StbBatchXchgArgs a, const stb_hit *local_hits, const uint32_t *local_status) {
  const uint32_t q = blockIdx.x;
  for (uint32_t idx = threadIdx.x; idx < a.world * a.top_k; idx += blockDim.x) {
    const uint32_t p = idx / a.top_k, i = idx % a.top_k;
    bx_hits(a.slot[p], a.world, a.max_nq)[((size_t)a.rank * a.max_nq + q) * a.max_k + i] = local_hits[(size_t)q * a.top_k + i];
  }
  if (threadIdx.x < a.world) bx_status(a.slot[threadIdx.x], a.world)[(size_t)a.rank * a.max_nq + q] = local_status[2 * q + 1];
  __threadfence_system();
  __syncthreads();
  __shared__ unsigned int s_last;
  if (threadIdx.x == 0) s_last = (atomicAdd(a.ticket, 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (!s_last) return;
  __threadfence_system();
  if (threadIdx.x == 0) *a.ticket = 0u;                               // re-arm for the next batch
  if (threadIdx.x < a.world)
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(bx_flags(a.slot[threadIdx.x]) + a.rank), "l"(a.seq) : "memory");
}

// Merge: CTA q waits until every rank's flag in the LOCAL slot carries this batch's sequence number,
// then merges the world x k hits of query q by (distance,row); status[2q+1] = every rank proved its part.
__global__ void __launch_bounds__(128)
stb_batch_xchg_merge_kernel(const StbBatchXchgArgs a, uint32_t n_sort, stb_hit *out, uint32_t *out_status) {
  extern __shared__ __align__(16) unsigned char smem[];
  double *sd = reinterpret_cast<double *>(smem);
  uint64_t *sr = reinterpret_cast<uint64_t *>(smem + (size_t)n_sort * sizeof(double));
  __shared__ unsigned int s_timeout;
  unsigned char *mine = a.slot[a.rank];
  if (threadIdx.x == 0) s_timeout = 0u;
  __syncthreads();
  if (threadIdx.x < a.world) {
    const unsigned long long *f = bx_flags(mine) + threadIdx.x;
    const long long t0 = clock64();
    for (;;) {
      unsigned long long v;
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(f) : "memory");
      if (v == a.seq) break;
      if (clock64() - t0 > STB_XCHG_TIMEOUT_CYCLES) { s_timeout = 1u; break; }    // a peer is gone
    }
  }
  __syncthreads();
  const uint32_t q = blockIdx.x, total = a.world * a.top_k;
  const stb_hit *lh = bx_hits(mine, a.world, a.max_nq);
  for (uint32_t i = threadIdx.x; i < n_sort; i += blockDim.x) {
    double d = CUDART_INF;
    uint64_t r = 0xffffffffffffffffull;
    if (i < total) {
      const stb_hit *src = lh + ((size_t)(i / a.top_k) * a.max_nq + q) * a.max_k + (i % a.top_k);
      const double dd = __ldcv(&src->distance);
      const uint64_t rr = __ldcv(&src->row);
      if (dd == dd && rr != 0xffffffffffffffffull) { d = dd; r = rr; }
    }
    sd[i] = d; sr[i] = r;
  }
  __syncthreads();
  stb_cta_sort_hits(sd, sr, n_sort);
  stb_write_hits(out + (size_t)q * a.top_k, sd, sr, min(a.top_k, n_sort), a.top_k);
  if (threadIdx.x == 0) {
    uint32_t ok = s_timeout ? 0u : 1u, n = 0;
    const uint32_t *st = bx_status(mine, a.world);
    for (uint32_t p = 0; p < a.world; ++p) ok &= __ldcv(st + (size_t)p * a.max_nq + q) ? 1u : 0u;
    for (uint32_t i = 0; i < a.top_k && i < n_sort; ++i) n += sr[i] != 0xffffffffffffffffull ? 1u : 0u;
    out_status[2 * q] = n;
    out_status[2 * q + 1] = s_timeout ? 2u : ok;                      // 2 = a peer never arrived
  }
}

int stb_launch_batch_xchg(stb_ctx *ctx, const StbBatchXchgArgs &a, const stb_hit *local_hits, const uint32_t *local_status,
                          stb_hit *out_hits, uint32_t *out_status) {
  const uint64_t total = (uint64_t)a.world * a.top_k;
  if (total > 2048) { stb_set_error("batch_xchg: %llu hits per query exceed 2048", (unsigned long long)total); return STB_ERR_ARG; }
  uint32_t n_sort = 2;
  while (n_sort < total) n_sort <<= 1;
  stb_batch_xchg_push_kernel<<<a.nq, 128, 0, ctx->stream>>>(a, local_hits, local_status);
  STB_CUDA(cudaGetLastError());
  stb_batch_xchg_merge_kernel<<<a.nq, 128, (size_t)n_sort * 16, ctx->stream>>>(a, n_sort, out_hits, out_status);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches += 2;
  return STB_OK;
}

int stb_launch_hits_merge_batch(stb_ctx *ctx, const stb_hit *lists_dev, uint32_t n_lists, uint32_t nq,
                                uint32_t per_list, uint32_t top_k, stb_hit *out_dev) {
  const uint64_t total = (uint64_t)n_lists * per_list;
  if (total > 2048) { stb_set_error("hits_merge_batch: %llu hits per query exceed 2048", (unsigned long long)total); return STB_ERR_ARG; }
  uint32_t n_sort = 2;
  while (n_sort < total) n_sort <<= 1;
  stb_hits_merge_batch_kernel<<<nq, 128, (size_t)n_sort * 16, ctx->stream>>>(lists_dev, n_lists, nq, per_list, n_sort, top_k, out_dev);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

int stb_launch_hits_merge(stb_ctx *ctx, const stb_hit *lists_dev, uint32_t n_lists,
                          uint32_t per_list, uint32_t top_k, stb_hit *out_dev) {
  uint64_t total = (uint64_t)n_lists * per_list;
  if (total > STB_MERGE_CAP) {
    stb_set_error("hits_merge: %llu hits exceed the %d-hit merge capacity",
                  (unsigned long long)total, STB_MERGE_CAP);
    return STB_ERR_ARG;
  }
  uint32_t n_sort = 2;
  while (n_sort < total) n_sort <<= 1;
  size_t smem = (size_t)n_sort * 16;
  STB_ATTR_ONCE(ctx, STB_ATTR_MERGE,
                cudaFuncSetAttribute(stb_hits_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     STB_MERGE_CAP * 16));
  stb_hits_merge_kernel<<<1, 256, smem, ctx->stream>>>(lists_dev, (uint32_t)total, n_sort, top_k,
                                                      out_dev);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// K3: token-id gather + mean-pool + L2-normalise (model2vec static embedding).
//
// Replaces StaticModel::pool_ids as reached from encode_with_args / encode_single
// (reference call sites src/search/mod.rs:69,138,153; src/cmds/search.rs:136,154;
// arithmetic in model2vec-rs 0.1.3, restated in oracle/semtools_oracle.c).
//
// Bit-exact contract: per dimension the token rows are accumulated sequentially in
// token order with an UNFUSED f32 multiply (by the token weight) and add; the mean
// is an IEEE f32 divide; the norm is a sequential f32 fold of the squares in
// dimension order, IEEE sqrt, max(.,1e-12), IEEE divide.  Hence the explicit
// __fmul_rn/__fadd_rn/__fdiv_rn/__fsqrt_rn below: nothing here may be contracted.
//
// HBM/L2-bound: T random 1 KiB table-row gathers per line (algorithmic bytes
// 1028*T + 1024 per line).  One warp per line; a lane owns 8 of the 256 dims as
// two float4 (columns 4*lane.. and 128+4*lane..), so each gathered row is two fully
// coalesced 512-byte warp loads, issued 8 tokens deep before the dependent adds.
#include "common.cuh"

#define STB_EMBED_THREADS 256
#define STB_EMBED_WARPS (STB_EMBED_THREADS / 32)
#define STB_EMBED_DEPTH 4     // tokens (2 x 512-byte warp loads each) in flight per warp
#define STB_EMBED_MINB 3      // CTAs per SM the register budget is sized for

struct EmbedArgs {
  const float4 *E;
  uint64_t V;
  const float *weights;
  uint64_t n_weights;
  const uint32_t *mapping;
  uint64_t n_mapping;
  int normalize;
  const uint64_t *offsets;
  const uint32_t *ids;
  uint64_t n_lines;
  float4 *out;
  int *err_flag;
};

__global__ void __launch_bounds__(STB_EMBED_THREADS, STB_EMBED_MINB)
stb_embed_kernel(const EmbedArgs a) {
  __shared__ __align__(16) float s_sq[STB_EMBED_WARPS][STB_D];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint64_t warps_total = (uint64_t)gridDim.x * STB_EMBED_WARPS;
  for (uint64_t line = (uint64_t)blockIdx.x * STB_EMBED_WARPS + warp; line < a.n_lines;
       line += warps_total) {
    const uint64_t beg = __ldg(a.offsets + line), end = __ldg(a.offsets + line + 1);
    float4 acc0 = make_float4(0.f, 0.f, 0.f, 0.f), acc1 = acc0;
    bool bad = false;
    for (uint64_t t0 = beg; t0 < end; t0 += STB_EMBED_DEPTH) {
      const int chunk = (int)min((uint64_t)STB_EMBED_DEPTH, end - t0);
      // lane u < chunk resolves token u: table row and weight
      uint32_t my_row = 0;
      float my_w = 1.0f;
      if (lane < chunk) {
        uint64_t tok = __ldg(a.ids + t0 + lane);
        uint64_t row = (a.mapping && tok < a.n_mapping) ? (uint64_t)__ldg(a.mapping + tok) : tok;
        my_w = (a.weights && tok < a.n_weights) ? __ldg(a.weights + tok) : 1.0f;
        if (row >= a.V) { bad = true; row = 0; }
        my_row = (uint32_t)row;
      }
      float4 v0[STB_EMBED_DEPTH], v1[STB_EMBED_DEPTH];
      float w[STB_EMBED_DEPTH];
#pragma unroll
      for (int u = 0; u < STB_EMBED_DEPTH; ++u) {
        uint32_t row = __shfl_sync(0xffffffffu, my_row, u);
        w[u] = __shfl_sync(0xffffffffu, my_w, u);
        if (u < chunk) {
          const float4 *p = a.E + (size_t)row * STB_ROW_F4;
          v0[u] = __ldg(p + lane);
          v1[u] = __ldg(p + 32 + lane);
        }
      }
#pragma unroll
      for (int u = 0; u < STB_EMBED_DEPTH; ++u) {
        if (u < chunk) {
          acc0.x = __fadd_rn(acc0.x, __fmul_rn(v0[u].x, w[u]));
          acc0.y = __fadd_rn(acc0.y, __fmul_rn(v0[u].y, w[u]));
          acc0.z = __fadd_rn(acc0.z, __fmul_rn(v0[u].z, w[u]));
          acc0.w = __fadd_rn(acc0.w, __fmul_rn(v0[u].w, w[u]));
          acc1.x = __fadd_rn(acc1.x, __fmul_rn(v1[u].x, w[u]));
          acc1.y = __fadd_rn(acc1.y, __fmul_rn(v1[u].y, w[u]));
          acc1.z = __fadd_rn(acc1.z, __fmul_rn(v1[u].z, w[u]));
          acc1.w = __fadd_rn(acc1.w, __fmul_rn(v1[u].w, w[u]));
        }
      }
    }
    if (__any_sync(0xffffffffu, bad)) {
      if (lane == 0) atomicExch(a.err_flag, 1);
    }
    const uint64_t cnt = end - beg;
    const float denom = (float)(cnt > 0 ? cnt : 1);
    acc0.x = __fdiv_rn(acc0.x, denom); acc0.y = __fdiv_rn(acc0.y, denom);
    acc0.z = __fdiv_rn(acc0.z, denom); acc0.w = __fdiv_rn(acc0.w, denom);
    acc1.x = __fdiv_rn(acc1.x, denom); acc1.y = __fdiv_rn(acc1.y, denom);
    acc1.z = __fdiv_rn(acc1.z, denom); acc1.w = __fdiv_rn(acc1.w, denom);
    if (a.normalize) {
      // squares in parallel, then ONE lane folds them in dimension order
      float4 *sq4 = reinterpret_cast<float4 *>(s_sq[warp]);
      sq4[lane] = make_float4(__fmul_rn(acc0.x, acc0.x), __fmul_rn(acc0.y, acc0.y),
                              __fmul_rn(acc0.z, acc0.z), __fmul_rn(acc0.w, acc0.w));
      sq4[32 + lane] = make_float4(__fmul_rn(acc1.x, acc1.x), __fmul_rn(acc1.y, acc1.y),
                                   __fmul_rn(acc1.z, acc1.z), __fmul_rn(acc1.w, acc1.w));
      __syncwarp();
      float ss = 0.0f;
      if (lane == 0) {
#pragma unroll 8
        for (int i = 0; i < STB_ROW_F4; ++i) {
          float4 s = sq4[i];
          ss = __fadd_rn(ss, s.x); ss = __fadd_rn(ss, s.y);
          ss = __fadd_rn(ss, s.z); ss = __fadd_rn(ss, s.w);
        }
      }
      ss = __shfl_sync(0xffffffffu, ss, 0);
      __syncwarp();
      const float norm = fmaxf(__fsqrt_rn(ss), 1e-12f);   // f32::max ignores NaN, as fmaxf
      acc0.x = __fdiv_rn(acc0.x, norm); acc0.y = __fdiv_rn(acc0.y, norm);
      acc0.z = __fdiv_rn(acc0.z, norm); acc0.w = __fdiv_rn(acc0.w, norm);
      acc1.x = __fdiv_rn(acc1.x, norm); acc1.y = __fdiv_rn(acc1.y, norm);
      acc1.z = __fdiv_rn(acc1.z, norm); acc1.w = __fdiv_rn(acc1.w, norm);
    }
    float4 *o = a.out + (size_t)line * STB_ROW_F4;
    o[lane] = acc0;
    o[32 + lane] = acc1;
  }
}

int stb_launch_embed(stb_ctx *ctx, const stb_table *t, const uint64_t *offsets_dev,
                     const uint32_t *ids_dev, uint64_t n_lines, float *out_dev,
                     int *err_flag_dev) {
  if (n_lines == 0) return STB_OK;
  EmbedArgs a;
  a.E = reinterpret_cast<const float4 *>(t->E.p);
  a.V = t->V;
  a.weights = t->weights;
  a.n_weights = t->n_weights;
  a.mapping = t->mapping;
  a.n_mapping = t->n_mapping;
  a.normalize = t->normalize;
  a.offsets = offsets_dev;
  a.ids = ids_dev;
  a.n_lines = n_lines;
  a.out = reinterpret_cast<float4 *>(out_dev);
  a.err_flag = err_flag_dev;
  int occ = 0;
  STB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, stb_embed_kernel,
                                                          STB_EMBED_THREADS, 0));
  if (occ < 1) occ = 1;
  uint64_t want = (n_lines + STB_EMBED_WARPS - 1) / STB_EMBED_WARPS;
  uint64_t grid = (uint64_t)ctx->sm_count * occ;
  if (want < grid) grid = want;
  stb_embed_kernel<<<(unsigned)grid, STB_EMBED_THREADS, 0, ctx->stream>>>(a);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

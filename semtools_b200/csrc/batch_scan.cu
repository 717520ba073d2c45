// K2: batched-query cosine scan on the Hopper tensor cores (wgmma + bulk-TMA + mbarrier).
//
// No reference analogue (the reference handles one query per process,
// src/search/mod.rs:77-120); semantics are those of Q independent search_documents
// calls.  BASELINE config 3: 10M x 256 corpus, 1024 queries, top-k 10.
//
// Pipeline (all on the context's stream):
//   1. stb_shadow_build_kernel  rows/queries f32 -> L2-normalised 16-bit copy, stored in HBM
//                               ALREADY in the wgmma shared-memory tile layout
//                               (K-major, 128-byte swizzle), so a tile is one
//                               contiguous block and is fetched with plain bulk-TMA
//                               copies (cp.async.bulk), no tensor map needed.
//   2. stb_batch_gemm_kernel    D[128 queries x 256 rows] = A . B^T per (query tile,
//                               corpus tile) on wgmma.mma_async m64n256k16 (16-bit in,
//                               f32 register accumulators), one 64-query half per
//                               consumer warpgroup, a producer warpgroup issuing the copies.
//                               The corpus tile (128 KB) stays resident in smem
//                               while the query tiles stream through a 6-slab ring from
//                               L2 (64 KB streamed per 16.8 MFLOP).
//                               Epilogue: max over each 32-row sub-tile of the accumulator
//                               fragments (lane-quad shuffles) -> submax[subtile][query].
//   3. stb_batch_select_kernel  per query: the 32 sub-tiles with the largest maxima.
//   4. stb_batch_finish_kernel  per query: exact canonical f64 re-score of the 32x32
//                               candidate rows, sort by (distance,row), top-k, and the
//                               completeness proof: every unselected row has approximate
//                               cosine <= m* (the smallest selected sub-tile maximum),
//                               hence exact cosine <= m* + EPS2 (bf16 rounding bound).
// Tensor-bound: 2*Q*N*256 FLOP per batch; HBM traffic N*512 B (16-bit shadow) once.
#include <cudaTypedefs.h>   // CUtensorMap, PFN_cuTensorMapEncodeTiled (route 7); no libcuda link
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math_constants.h>

#include <algorithm>

#include "common.cuh"
#include "row_encode.cuh"
#include "q8_query.cuh"

#define STB_B_TILE 256            // corpus rows per tile  (MMA N)
#define STB_A_TILE 128            // queries per tile      (MMA M, two m64 warpgroups)
#define STB_SLAB_K 64             // bf16 per 128-byte swizzled row
#define STB_N_SLABS 4             // 256 / 64
#define STB_B_SLAB_BYTES (STB_B_TILE * 128)     // 32 KiB
#define STB_A_SLAB_BYTES (STB_A_TILE * 128)     // 16 KiB
#define STB_A_RING 6
#define STB_SUB 32                // rows per sub-tile
#define STB_BATCH_KSEL 32         // sub-tiles kept per query
// Shadow element type.  fp16 (default, STB_SHADOW_F16=1 in common.cuh) or bf16
// (-DSTB_SHADOW_F16=0; same wgmma rate).  For L2-normalised rows every element is
// <= 1, so fp16's range suffices and its 10-bit mantissa shrinks the selection margin ~4x:
//   bf16: 8 significand bits -> unit roundoff u = 2^-8; both operands rounded:
//         |approx - exact cosine| <= (2u+u^2) = 0.00783, + f32 accumulation + rsqrt  < 0.0079
//         (attained within 2%: tests/test_batch_v2_model.py builds the adversarial row)
//   fp16: u = 2^-11 for |x| >= 2^-14; smaller elements err by <= 2^-25 absolutely, at most
//         2*256*2^-25 = 1.5e-5 over a row pair; total < 0.00101
#if STB_SHADOW_F16
#define STB_BATCH_EPS 0.0012
#else
#define STB_BATCH_EPS 0.0080
#endif

// ------------------------------------------------------------------ PTX wrappers ---
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  // bounded spin: a protocol bug must trap, never hang the GPU
  for (uint32_t spins = 0;; ++spins) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (done) return;
    if (spins > (1u << 26)) __trap();
  }
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// Warpgroup MMA (sm_90a): D[regs] (+)= A[smem desc] * B[smem desc]^T, 16-bit inputs, f32 accumulators.
#if STB_SHADOW_F16
#define STB_WG_AB "f16.f16"
#else
#define STB_WG_AB "bf16.bf16"
#endif
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching an accumulator across a wgmma fence / wait
__device__ __forceinline__ void wg_reg_fence(float (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void wg_mma_m64n256k16(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32." STB_WG_AB " {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, 0;\n\t}"
      :
        "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// Shared-memory matrix descriptor, K-major operand, 128-byte swizzle (sm_90 wgmma format):
//   [0,14) start address >> 4 | [16,30) leading byte offset >> 4 (unused for swizzled
//   K-major, canonical value 1) | [32,46) stride byte offset >> 4 (8 rows x 128 B = 1024)
//   | [49,52) base offset = 0 (atoms are 1024-byte aligned) | [62,64) layout = 1 (SWIZZLE_128B).
__device__ __forceinline__ uint64_t wg_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3ffffu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// --------------------------------------------------------------- 1. shadow builder ---
// One warp per row; lane l owns k = 8l..8l+7 = one 16-byte chunk (row_encode.cuh: stb_shadow_pack_row,
// stb_shadow_offset).  Rows [n_rows, n_padded) are the zero padding of the last tile.
template <int TILE>
__global__ void __launch_bounds__(256)
stb_shadow_build_kernel(const float4 *__restrict__ rows, uint64_t first_row, uint64_t n_rows, uint64_t n_padded,
                        uint8_t *__restrict__ out, int *bad_flag, uint32_t *row_bad, uint64_t rows_first) {
  const int lane = threadIdx.x & 31;
  const uint64_t row = first_row + (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= n_padded) return;
  float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
  if (row < n_rows) {
    v0 = __ldg(rows + (row - rows_first) * STB_ROW_F4 + 2 * lane);
    v1 = __ldg(rows + (row - rows_first) * STB_ROW_F4 + 2 * lane + 1);
  }
  // per-row record (query tiles): a row that cannot be normalised bounds nothing; the finish kernels mark
  // it unproven
  const uint4 pk = stb_shadow_pack_row(v0, v1, lane, row, bad_flag, row_bad);
  *reinterpret_cast<uint4 *>(out + stb_shadow_offset<TILE>(row, lane)) = pk;
}

// ------------------------------------------------------------------- 2. wgmma GEMM ---
struct GemmArgs {
  const uint8_t *a_tiles;     // query shadow: m_tiles x (4 slabs x 16 KiB)
  const uint8_t *b_tiles;     // corpus shadow: n_tiles x (4 slabs x 32 KiB)
  uint32_t m_tiles;           // ceil(Q / 128)
  uint32_t n_tiles;           // ceil(N / 256)
  // maxima are stored [query tile][sub-tile or tile][128 queries]: the selection pass streams
  // them contiguously
  union {
    float *submax;            // [m_tiles][n_tiles * 8][128]  per-32-row maxima
    const uint4 *items;       // STB_GEMM_WORK (below)
  };
  union {
    float *tilemax;           // [m_tiles][n_tiles][128]      per-256-row maxima (STB_GEMM_WORK: [m_tiles][tile_stride][128])
    const uint32_t *slot_row; // STB_GEMM_WORK, EPI 1 (below)
  };
  union {
    float *full_out;          // debug: full score matrix [m_tiles*128][n_tiles*256] or null
    const uint32_t *item_off; // STB_GEMM_WORK (below)
  };
  uint32_t tile_stride;       // corpus tile t of this launch is shadow tile t * tile_stride (sampling pass)
  // EPI == 1 (candidate-emitting epilogue, pipeline v2):
  const float *thr;           // [q_pad] per-query score threshold (+inf for padding queries)
  uint32_t *cand_cnt;         // [q_pad][grid] candidates emitted per (query, CTA) (> cand_cap: overflow marker)
  uint64_t *cand_keys;        // [q_pad][grid][cand_cap] keys (score desc, local row)
  uint32_t cand_cap;          // per-segment capacity
  uint64_t n_rows;            // real corpus rows (padding rows of the last tile are never emitted)
  // FILTER (stb_search_batch_filtered): tile t of the launch is shadow tile tile_ids[t * tile_stride]
  const uint32_t *tile_ids;   // listed tiles: the shadow tiles holding an eligible row, ascending
  const uint32_t *bitmap;     // eligible local rows, 1 bit each: 8 words per shadow tile
  // EPI == 2 (stb_search_batch_threshold's re-emission): segment (q, CTA) is cand_keys[seg_off[q * grid + CTA],
  // seg_off[q * grid + CTA + 1]), sized by the first pass's exact counts; cand_cnt holds the cursors
  union {
    const uint64_t *seg_off;  // [q_pad * grid + 1]
    const uint32_t *cta_tiles;  // STB_GEMM_WORK (below)
  };
  // STB_GEMM_WORK (stb_search_batch_subsets; the unions keep the layout the other modes compile against): CTA b
  // walks the corpus tiles u in [cta_tiles[b], cta_tiles[b + 1]) (shadow tile tile_ids[u]); tile u's work items
  // are items[item_off[u], item_off[u + 1]), each {query tile, mask slot of half 0, mask slot of half 1, sample
  // columns}: a mask slot is 8 bitmap words at bitmap + 8 * slot; the sample columns (EPI 0: low / high 16
  // bits, 0xffff: none) index tilemax [m_tiles][tile_stride][128].  EPI 1 writes query slot s's keys and count
  // at row slot_row[s] (~0: a padding slot, which never emits).
};

// Filter modes of the GEMM: every tile, the listed tiles of one filter, or a work list of (query tile, masks)
// per corpus tile, one filter per 64-query half
#define STB_GEMM_ALL 0
#define STB_GEMM_LISTED 1
#define STB_GEMM_WORK 2

// warpgroup 0: bulk-copy producer (one thread); warpgroups 1 and 2: wgmma + epilogue, each on
// 64 of the 128 queries of a query tile (m64n256 accumulators, 128 f32 registers per thread)
#define STB_GEMM_THREADS 384
#define STB_GEMM_CONSUMER_WARPS 8
#define STB_GEMM_SMEM (STB_N_SLABS * STB_B_SLAB_BYTES + STB_A_RING * STB_A_SLAB_BYTES + 1024 + 256)
// STB_GEMM_WORK: three 64-byte mask buffers behind the barriers instead of two 32-byte ones
#define STB_GEMM_SMEM_WORK (STB_GEMM_SMEM + 128)
static_assert(STB_GEMM_SMEM_WORK <= 227 * 1024, "GEMM shared memory");

// FILTER == STB_GEMM_WORK (EPI 0 or 1), the body of stb_batch_gemm_kernel below on its shared memory and
// initialised barriers: the same pipeline and epilogues per 64-query half, over each corpus tile's work items
// (GemmArgs) instead of every query tile.  Kept apart from the kernel body so the other modes compile as they
// did.  An item's 2 x 8 mask words arrive with its first query slab; item i of a CTA uses mask buffer i % 3:
// item i + 3's slab 0 reuses the ring slot of item i + 1's slab 2, which every consumer warp releases only
// after the epilogue of item i.
template <int EPI>
__device__ __forceinline__ void stb_batch_gemm_work(const GemmArgs &args, uint8_t *sB, uint8_t *sA, uint64_t *bars) {
  uint64_t *b_full = bars + 0, *b_empty = bars + STB_N_SLABS;
  uint64_t *a_full = bars + 2 * STB_N_SLABS, *a_empty = a_full + STB_A_RING;
  uint32_t *s_mask = reinterpret_cast<uint32_t *>(bars + 24);       // [3][2][8]
  static_assert(24 * 8 + 3 * 16 * 4 <= 256 + (STB_GEMM_SMEM_WORK - STB_GEMM_SMEM), "work-item mask words must fit");
  static_assert(STB_A_RING == 6 && STB_N_SLABS == 4, "the mask buffer rule (item % 3) assumes this ring");
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t t0 = __ldg(args.cta_tiles + blockIdx.x), t1 = __ldg(args.cta_tiles + blockIdx.x + 1);

  if (warp < 4) {
    // ===== bulk-copy producer (one thread) =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      uint32_t a_cnt = 0;
      for (uint32_t u = t0, it = 0; u < t1; ++u, ++it) {
        const uint8_t *src = args.b_tiles + (uint64_t)__ldg(args.tile_ids + u) * (size_t)(STB_N_SLABS * STB_B_SLAB_BYTES);
        for (int s = 0; s < STB_N_SLABS; ++s) {
          mbar_wait(b_empty + s, (it & 1) ^ 1);
          mbar_expect_tx(b_full + s, STB_B_SLAB_BYTES);
          bulk_g2s(sB + s * STB_B_SLAB_BYTES, src + (size_t)s * STB_B_SLAB_BYTES, STB_B_SLAB_BYTES, b_full + s);
        }
        const uint32_t w1 = __ldg(args.item_off + u + 1);
        for (uint32_t w = __ldg(args.item_off + u); w < w1; ++w) {
          const uint4 item = __ldg(args.items + w);
          for (int s = 0; s < STB_N_SLABS; ++s, ++a_cnt) {
            const uint32_t slot = a_cnt % STB_A_RING;
            mbar_wait(a_empty + slot, ((a_cnt / STB_A_RING) & 1) ^ 1);
            if (s == 0) {
              uint32_t *mk = s_mask + ((a_cnt / STB_N_SLABS) % 3) * 16;
              mbar_expect_tx(a_full + slot, STB_A_SLAB_BYTES + 64);
              bulk_g2s(mk, args.bitmap + (size_t)item.y * 8, 32, a_full + slot);
              bulk_g2s(mk + 8, args.bitmap + (size_t)item.z * 8, 32, a_full + slot);
            } else {
              mbar_expect_tx(a_full + slot, STB_A_SLAB_BYTES);
            }
            bulk_g2s(sA + slot * STB_A_SLAB_BYTES, args.a_tiles + ((size_t)item.x * STB_N_SLABS + s) * STB_A_SLAB_BYTES,
                     STB_A_SLAB_BYTES, a_full + slot);
          }
        }
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  // ===== consumers (accumulator layout as in stb_batch_gemm_kernel) =====
  const uint32_t half = (uint32_t)(warp >> 2) - 1u;
  const uint32_t qrow = half * 64 + (warp & 3) * 16 + (lane >> 2);
  const uint32_t quad = lane & 3;
  float d[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) d[i] = 0.f;
  uint32_t a_cnt = 0;
  for (uint32_t u = t0, it = 0; u < t1; ++u, ++it) {
    const uint64_t tile_row0 = (uint64_t)__ldg(args.tile_ids + u) * STB_B_TILE;
    const uint32_t w0 = __ldg(args.item_off + u), w1 = __ldg(args.item_off + u + 1);
    for (uint32_t w = w0; w < w1; ++w, a_cnt += STB_N_SLABS) {
      const uint4 item = __ldg(args.items + w);
      const uint32_t m = item.x;
      const uint32_t *mask = s_mask + ((a_cnt / STB_N_SLABS) % 3) * 16 + half * 8;   // this half's filter
      const uint32_t q0 = m * STB_A_TILE + qrow;
      [[maybe_unused]] float thr[2];
      [[maybe_unused]] uint32_t cnt[2], cnt0[2], qout[2];
      if constexpr (EPI == 1) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          // a padding slot never emits and owns no segment
          const uint32_t r = __ldg(args.slot_row + q0 + 8 * h);
          thr[h] = (r == 0xffffffffu) ? CUDART_INF_F : __ldg(args.thr + q0 + 8 * h);
          qout[h] = (r == 0xffffffffu) ? 0u : r;
          cnt0[h] = args.cand_cnt[(size_t)qout[h] * gridDim.x + blockIdx.x];
          cnt[h] = cnt0[h];
        }
      }
      wg_reg_fence(d);
#pragma unroll
      for (int s = 0; s < STB_N_SLABS; ++s) {
        const uint32_t slot = (a_cnt + s) % STB_A_RING;
        if (w == w0) mbar_wait(b_full + s, it & 1);
        mbar_wait(a_full + slot, ((a_cnt + s) / STB_A_RING) & 1);
        wg_fence();
        const uint32_t a_addr = smem_u32(sA + slot * STB_A_SLAB_BYTES + half * (64 * 128));
        const uint32_t b_addr = smem_u32(sB + s * STB_B_SLAB_BYTES);
#pragma unroll
        for (int k = 0; k < STB_SLAB_K / 16; ++k)
          wg_mma_m64n256k16(d, wg_desc_sw128(a_addr + k * 32), wg_desc_sw128(b_addr + k * 32), (uint32_t)((s | k) != 0));
        wg_commit();
        if (s > 0) {
          wg_wait<1>();
          if (lane == 0) {
            mbar_arrive(a_empty + (a_cnt + s - 1) % STB_A_RING);
            if (w + 1 == w1) mbar_arrive(b_empty + s - 1);
          }
        }
      }
      wg_wait<0>();
      wg_reg_fence(d);
      if (lane == 0) {
        mbar_arrive(a_empty + (a_cnt + STB_N_SLABS - 1) % STB_A_RING);
        if (w + 1 == w1) mbar_arrive(b_empty + STB_N_SLABS - 1);
      }

      if constexpr (EPI == 0) {
        // tile maximum over this half's eligible rows (ineligible scores -inf, as FILTER == STB_GEMM_LISTED),
        // stored at the half's column of its group's sample (0xffff: the tile is not in that sample)
        float tmx[2] = {-CUDART_INF_F, -CUDART_INF_F};
#pragma unroll
        for (int c = 0; c < STB_B_TILE / STB_SUB; ++c) {
          const uint32_t mw = mask[c];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float mx = -CUDART_INF_F;
#pragma unroll
            for (int ii = 0; ii < 4; ++ii)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                mx = fmaxf(mx, ((mw >> (ii * 8 + quad * 2 + e)) & 1u) ? d[16 * c + 4 * ii + 2 * h + e] : -CUDART_INF_F);
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            tmx[h] = fmaxf(tmx[h], mx);
          }
        }
        const uint32_t col = half ? (item.w >> 16) : (item.w & 0xffffu);
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (quad == (uint32_t)(2 + h) && col != 0xffffu)
            args.tilemax[((size_t)m * args.tile_stride + col) * STB_A_TILE + qrow + 8 * h] = tmx[h];
      } else {
        // emission as stb_batch_gemm_kernel's EPI 1, into the segments of row qout
#pragma unroll
        for (int c = 0; c < STB_B_TILE / STB_SUB; ++c) {
          const uint64_t row0 = tile_row0 + (uint64_t)c * STB_SUB;
          const uint32_t mw = mask[c];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint32_t hit = 0u;
#pragma unroll
            for (int ii = 0; ii < 4; ++ii)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                hit |= (d[16 * c + 4 * ii + 2 * h + e] >= thr[h] ? 1u : 0u) << (ii * 8 + quad * 2 + e);
            hit |= __shfl_xor_sync(0xffffffffu, hit, 1);
            hit |= __shfl_xor_sync(0xffffffffu, hit, 2);
            if (row0 + 32 > args.n_rows) hit &= (row0 < args.n_rows) ? ((1u << (uint32_t)(args.n_rows - row0)) - 1u) : 0u;
            hit &= mw;
            uint64_t *seg = args.cand_keys + ((size_t)qout[h] * gridDim.x + blockIdx.x) * args.cand_cap;
#pragma unroll
            for (int ii = 0; ii < 4; ++ii)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const uint32_t b = ii * 8 + quad * 2 + e;
                const uint32_t pos = cnt[h] + __popc(hit & ((1u << b) - 1u));
                const uint64_t key = stb_make_key(d[16 * c + 4 * ii + 2 * h + e], (uint32_t)(row0 + b));
                if (((hit >> b) & 1u) && pos < args.cand_cap) seg[pos] = key;
              }
            cnt[h] += __popc(hit);
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (quad == 0 && cnt[h] != cnt0[h]) args.cand_cnt[(size_t)qout[h] * gridDim.x + blockIdx.x] = cnt[h];
      }
    }
  }
}

// EPI 0: per-sub-tile / per-tile maxima (pipeline v1, and the sampling pass of v2).
// EPI 1: emit every (query,row) whose approximate score reaches the query's threshold.
// EPI 2: the same emission into exactly sized segments at args.seg_off (unfiltered only).
// FILTER == STB_GEMM_LISTED: the CTAs walk the listed tiles (args.tile_ids) and only eligible rows count
// (args.bitmap): EPI 0 takes each tile maximum over its eligible rows, EPI 1 emits eligible rows only.  The
// tile's 8 bitmap words arrive with its first corpus slab, double-buffered behind the mbarriers.
// FILTER == STB_GEMM_WORK: stb_batch_gemm_work above.
template <int EPI, int FILTER>
__global__ void __launch_bounds__(STB_GEMM_THREADS, 1)
stb_batch_gemm_kernel(const GemmArgs args) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment required by the 128-byte swizzle atoms
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t *sB = smem;
  uint8_t *sA = smem + STB_N_SLABS * STB_B_SLAB_BYTES;
  uint64_t *bars = reinterpret_cast<uint64_t *>(sA + STB_A_RING * STB_A_SLAB_BYTES);
  uint64_t *b_full = bars + 0, *b_empty = bars + STB_N_SLABS;      // one pair per K-slab
  uint64_t *a_full = bars + 2 * STB_N_SLABS, *a_empty = a_full + STB_A_RING;
  // FILTER: [2][8] bitmap words, slot it & 1 = the tile of iteration it (the 256 bytes behind the ring hold
  // the 20 barriers, then these 64 bytes)
  [[maybe_unused]] uint32_t *s_mask = reinterpret_cast<uint32_t *>(bars + 24);
  static_assert(24 * 8 + 2 * 8 * 4 <= 256, "mask words must fit behind the barriers");

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < STB_N_SLABS; ++i) { mbar_init(b_full + i, 1); mbar_init(b_empty + i, STB_GEMM_CONSUMER_WARPS); }
    for (int i = 0; i < STB_A_RING; ++i) { mbar_init(a_full + i, 1); mbar_init(a_empty + i, STB_GEMM_CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if constexpr (FILTER == STB_GEMM_WORK) {
    static_assert(EPI == 0 || EPI == 1, "work lists serve v2's two passes");
    stb_batch_gemm_work<EPI>(args, sB, sA, bars);
    return;
  }

  const uint32_t my_tiles = (args.n_tiles > blockIdx.x) ? (args.n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

  if (warp < 4) {
    // ===== bulk-copy producer (one thread) =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      uint32_t a_cnt = 0;
      for (uint32_t it = 0; it < my_tiles; ++it) {
        const uint64_t t = blockIdx.x + (uint64_t)it * gridDim.x;
        // corpus tile, slab by slab: slab s of the previous tile is released as soon as the
        // last query tile's MMAs on it retire, so the refill overlaps the remaining slabs
        if constexpr (FILTER == STB_GEMM_LISTED) {
          const uint64_t tile = __ldg(args.tile_ids + t * args.tile_stride);
          const uint8_t *src = args.b_tiles + tile * (size_t)(STB_N_SLABS * STB_B_SLAB_BYTES);
          for (int s = 0; s < STB_N_SLABS; ++s) {
            mbar_wait(b_empty + s, (it & 1) ^ 1);
            if (s == 0) {
              // the mask slot of iteration it - 2 is free: every consumer warp released slab 0 of the tile
              // of it - 1, which it does only after the epilogues of the tile of it - 2
              mbar_expect_tx(b_full, STB_B_SLAB_BYTES + 32);
              bulk_g2s(s_mask + (it & 1) * 8, args.bitmap + tile * 8, 32, b_full);
            } else {
              mbar_expect_tx(b_full + s, STB_B_SLAB_BYTES);
            }
            bulk_g2s(sB + s * STB_B_SLAB_BYTES, src + (size_t)s * STB_B_SLAB_BYTES, STB_B_SLAB_BYTES, b_full + s);
          }
        } else {
          const uint8_t *src = args.b_tiles + t * args.tile_stride * (size_t)(STB_N_SLABS * STB_B_SLAB_BYTES);
          for (int s = 0; s < STB_N_SLABS; ++s) {
            mbar_wait(b_empty + s, (it & 1) ^ 1);
            mbar_expect_tx(b_full + s, STB_B_SLAB_BYTES);
            bulk_g2s(sB + s * STB_B_SLAB_BYTES, src + (size_t)s * STB_B_SLAB_BYTES, STB_B_SLAB_BYTES, b_full + s);
          }
        }
        for (uint32_t m = 0; m < args.m_tiles; ++m) {
          for (int s = 0; s < STB_N_SLABS; ++s, ++a_cnt) {
            const uint32_t slot = a_cnt % STB_A_RING;
            mbar_wait(a_empty + slot, ((a_cnt / STB_A_RING) & 1) ^ 1);
            mbar_expect_tx(a_full + slot, STB_A_SLAB_BYTES);
            bulk_g2s(sA + slot * STB_A_SLAB_BYTES,
                     args.a_tiles + ((size_t)m * STB_N_SLABS + s) * STB_A_SLAB_BYTES, STB_A_SLAB_BYTES,
                     a_full + slot);
          }
        }
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  // ===== consumers: wgmma over one 64-query half of every query tile, then the epilogue =====
  // Accumulator fragment of m64nN (PTX ISA, wgmma D layout): thread (warp w, lane l) of the
  // warpgroup holds rows r = 16w + l/4 and r + 8; d[4i + e] is (r, 8i + 2(l%4) + e), d[4i + 2 + e]
  // is (r + 8, same column).  A 32-row sub-tile c is d[16c .. 16c + 15], spread over a lane quad.
  const uint32_t half = (uint32_t)(warp >> 2) - 1u;       // which 64 queries of the tile
  const uint32_t qrow = half * 64 + (warp & 3) * 16 + (lane >> 2);   // + 8 for the second row
  const uint32_t quad = lane & 3;
  const uint64_t n_sub = (uint64_t)args.n_tiles * (STB_B_TILE / STB_SUB);
  float d[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) d[i] = 0.f;
  uint32_t a_cnt = 0;
  for (uint32_t it = 0; it < my_tiles; ++it) {
    const uint64_t t = blockIdx.x + (uint64_t)it * gridDim.x;
    [[maybe_unused]] uint64_t tile_row0 = 0;                 // FILTER: first row of the shadow tile
    if constexpr (FILTER == STB_GEMM_LISTED) tile_row0 = (uint64_t)__ldg(args.tile_ids + t * args.tile_stride) * STB_B_TILE;
    for (uint32_t m = 0; m < args.m_tiles; ++m, a_cnt += STB_N_SLABS) {
      const uint32_t q0 = m * STB_A_TILE + qrow;
      [[maybe_unused]] float thr[2];
      [[maybe_unused]] uint32_t cnt[2], cnt0[2];
      [[maybe_unused]] uint64_t seg_base[2];
      [[maybe_unused]] uint32_t seg_len[2];
      if constexpr (EPI >= 1) {       // epilogue state, fetched while the MMAs run
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          thr[h] = __ldg(args.thr + q0 + 8 * h);
          cnt0[h] = args.cand_cnt[(size_t)(q0 + 8 * h) * gridDim.x + blockIdx.x];
          cnt[h] = cnt0[h];
          if constexpr (EPI == 2) {
            const uint64_t *so = args.seg_off + (size_t)(q0 + 8 * h) * gridDim.x + blockIdx.x;
            seg_base[h] = __ldg(so);
            seg_len[h] = (uint32_t)(__ldg(so + 1) - seg_base[h]);
          }
        }
      }
      wg_reg_fence(d);
#pragma unroll
      for (int s = 0; s < STB_N_SLABS; ++s) {
        const uint32_t slot = (a_cnt + s) % STB_A_RING;
        if (m == 0) mbar_wait(b_full + s, it & 1);
        mbar_wait(a_full + slot, ((a_cnt + s) / STB_A_RING) & 1);
        wg_fence();
        const uint32_t a_addr = smem_u32(sA + slot * STB_A_SLAB_BYTES + half * (64 * 128));
        const uint32_t b_addr = smem_u32(sB + s * STB_B_SLAB_BYTES);
#pragma unroll
        for (int k = 0; k < STB_SLAB_K / 16; ++k)   // advancing K by 16 elements = 32 bytes inside the swizzle atom
          wg_mma_m64n256k16(d, wg_desc_sw128(a_addr + k * 32), wg_desc_sw128(b_addr + k * 32), (uint32_t)((s | k) != 0));
        wg_commit();
        if (s > 0) {
          // slab s-1 has been read: free its query slot (and, after the last query tile, its corpus slab)
          wg_wait<1>();
          if (lane == 0) {
            mbar_arrive(a_empty + (a_cnt + s - 1) % STB_A_RING);
            if (m + 1 == args.m_tiles) mbar_arrive(b_empty + s - 1);
          }
        }
      }
      wg_wait<0>();
      wg_reg_fence(d);
      if (lane == 0) {
        mbar_arrive(a_empty + (a_cnt + STB_N_SLABS - 1) % STB_A_RING);
        if (m + 1 == args.m_tiles) mbar_arrive(b_empty + STB_N_SLABS - 1);
      }

      if constexpr (EPI == 0) {
        float tmx[2] = {-CUDART_INF_F, -CUDART_INF_F};
#pragma unroll
        for (int c = 0; c < STB_B_TILE / STB_SUB; ++c) {
          [[maybe_unused]] uint32_t mw = 0;
          if constexpr (FILTER == STB_GEMM_LISTED) mw = s_mask[(it & 1) * 8 + c];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float mx;
            if constexpr (FILTER == STB_GEMM_LISTED) {
              // an ineligible row's score is -inf here (a select, no branch): the maximum is an eligible
              // row's score, which the threshold's sufficiency argument needs
              mx = -CUDART_INF_F;
#pragma unroll
              for (int ii = 0; ii < 4; ++ii)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                  mx = fmaxf(mx, ((mw >> (ii * 8 + quad * 2 + e)) & 1u) ? d[16 * c + 4 * ii + 2 * h + e] : -CUDART_INF_F);
            } else {
              mx = d[16 * c + 2 * h];
#pragma unroll
              for (int ii = 0; ii < 4; ++ii)
                mx = fmaxf(mx, fmaxf(d[16 * c + 4 * ii + 2 * h], d[16 * c + 4 * ii + 2 * h + 1]));
            }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            tmx[h] = fmaxf(tmx[h], mx);
            if (args.submax && quad == (uint32_t)h)
              args.submax[((size_t)m * n_sub + t * (STB_B_TILE / STB_SUB) + c) * STB_A_TILE + qrow + 8 * h] = mx;
          }
          if (args.full_out) {
#pragma unroll
            for (int ii = 0; ii < 4; ++ii)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                float *o = args.full_out + (size_t)(q0 + 8 * h) * ((size_t)args.n_tiles * STB_B_TILE) + t * STB_B_TILE +
                           c * STB_SUB + ii * 8 + quad * 2;
                *reinterpret_cast<float2 *>(o) = make_float2(d[16 * c + 4 * ii + 2 * h], d[16 * c + 4 * ii + 2 * h + 1]);
              }
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (quad == (uint32_t)(2 + h)) args.tilemax[((size_t)m * args.n_tiles + t) * STB_A_TILE + qrow + 8 * h] = tmx[h];
      } else {
        // The threshold is the k-th best score of a ~1.5 % sample minus the rounding margin, so an
        // emission is rare.  Each (query, CTA) pair owns a private segment of the candidate buffer
        // and its own cursor, kept in step by the four lanes of the quad that hold the query's row:
        // no atomics, and keys land in ascending row order within a 32-row sub-tile.
#pragma unroll
        for (int c = 0; c < STB_B_TILE / STB_SUB; ++c) {
          uint64_t row0;
          [[maybe_unused]] uint32_t mw = 0;
          if constexpr (FILTER == STB_GEMM_LISTED) {
            row0 = tile_row0 + (uint64_t)c * STB_SUB;
            mw = s_mask[(it & 1) * 8 + c];
          } else {
            row0 = t * STB_B_TILE + (uint64_t)c * STB_SUB;
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            // Branch-free on purpose: an accumulator read on a divergent path makes the compiler
            // serialise the wgmma of the next query tile behind it.
            uint32_t hit = 0u;
#pragma unroll
            for (int ii = 0; ii < 4; ++ii)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                hit |= (d[16 * c + 4 * ii + 2 * h + e] >= thr[h] ? 1u : 0u) << (ii * 8 + quad * 2 + e);
            hit |= __shfl_xor_sync(0xffffffffu, hit, 1);
            hit |= __shfl_xor_sync(0xffffffffu, hit, 2);
            if (row0 + 32 > args.n_rows) hit &= (row0 < args.n_rows) ? ((1u << (uint32_t)(args.n_rows - row0)) - 1u) : 0u;   // padding rows
            if constexpr (FILTER == STB_GEMM_LISTED) hit &= mw;                                                                                    // ineligible rows
            uint64_t *seg;
            uint32_t seg_cap;
            if constexpr (EPI == 2) {
              seg = args.cand_keys + seg_base[h];
              seg_cap = seg_len[h];
            } else {
              seg = args.cand_keys + ((size_t)(q0 + 8 * h) * gridDim.x + blockIdx.x) * args.cand_cap;
              seg_cap = args.cand_cap;
            }
#pragma unroll
            for (int ii = 0; ii < 4; ++ii)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const uint32_t b = ii * 8 + quad * 2 + e;
                const uint32_t pos = cnt[h] + __popc(hit & ((1u << b) - 1u));
                const uint64_t key = stb_make_key(d[16 * c + 4 * ii + 2 * h + e], (uint32_t)(row0 + b));
                if (((hit >> b) & 1u) && pos < seg_cap) seg[pos] = key;
              }
            cnt[h] += __popc(hit);                       // > cand_cap = overflow marker
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (quad == 0 && cnt[h] != cnt0[h]) args.cand_cnt[(size_t)(q0 + 8 * h) * gridDim.x + blockIdx.x] = cnt[h];
      }
    }
  }
}

void stb_batch_build_params(int *shadow_is_f16, double *eps) {
  if (shadow_is_f16) *shadow_is_f16 = STB_SHADOW_F16;
  if (eps) *eps = STB_BATCH_EPS;
}

// ------------------------------------------------------- host-side: shadow + GEMM ------
int stb_launch_shadow_build(stb_ctx *ctx, const float *rows_dev, uint64_t n_rows, int tile, uint8_t *out,
                            int *bad_flag_dev, uint64_t first_row, uint32_t *row_bad_dev, uint64_t rows_first) {
  // rows [first_row, n_rows) plus the zero padding of the last tile; first_row must be tile-aligned
  const uint64_t n_padded = (n_rows + tile - 1) / tile * tile;
  if (n_padded == 0 || first_row >= n_padded) return STB_OK;
  const unsigned blocks = (unsigned)((n_padded - first_row + 7) / 8);
  if (tile == STB_B_TILE)
    stb_shadow_build_kernel<STB_B_TILE><<<blocks, 256, 0, ctx->stream>>>(reinterpret_cast<const float4 *>(rows_dev), first_row, n_rows, n_padded, out, bad_flag_dev, row_bad_dev, rows_first);
  else
    stb_shadow_build_kernel<STB_A_TILE><<<blocks, 256, 0, ctx->stream>>>(reinterpret_cast<const float4 *>(rows_dev), first_row, n_rows, n_padded, out, bad_flag_dev, row_bad_dev, rows_first);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

template <int EPI, int FILTER = STB_GEMM_ALL>
static int launch_gemm(stb_ctx *ctx, const GemmArgs &a) {
  const int attr = FILTER == STB_GEMM_WORK ? (EPI == 0 ? STB_ATTR_GEMM0W : STB_ATTR_GEMM1W)
                   : FILTER == STB_GEMM_LISTED ? (EPI == 0 ? STB_ATTR_GEMM0F : STB_ATTR_GEMM1F)
                   : (EPI == 0 ? STB_ATTR_GEMM0 : (EPI == 1 ? STB_ATTR_GEMM1 : STB_ATTR_GEMM2));
  const int smem = FILTER == STB_GEMM_WORK ? STB_GEMM_SMEM_WORK : STB_GEMM_SMEM;
  STB_ATTR_ONCE(ctx, attr,
                cudaFuncSetAttribute(stb_batch_gemm_kernel<EPI, FILTER>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  // STB_GEMM_WORK: the same grid as the caller's cta_tiles (stb_batch_emit_grid)
  unsigned grid = (unsigned)std::min<uint32_t>(a.n_tiles, (uint32_t)ctx->sm_count);
  if (grid == 0) return STB_OK;
  stb_batch_gemm_kernel<EPI, FILTER><<<grid, STB_GEMM_THREADS, smem, ctx->stream>>>(a);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

int stb_launch_batch_gemm(stb_ctx *ctx, const uint8_t *a_tiles, uint32_t m_tiles, const uint8_t *b_tiles,
                          uint32_t n_tiles, float *submax, float *tilemax, float *full_out) {
  return stb_launch_batch_gemm_strided(ctx, a_tiles, m_tiles, b_tiles, n_tiles, 1, submax, tilemax, full_out);
}

// maxima epilogue over the tiles 0, stride, 2*stride, ... (n_tiles of them); submax may be null
int stb_launch_batch_gemm_strided(stb_ctx *ctx, const uint8_t *a_tiles, uint32_t m_tiles, const uint8_t *b_tiles,
                                  uint32_t n_tiles, uint32_t tile_stride, float *submax, float *tilemax, float *full_out) {
  GemmArgs a{};
  a.a_tiles = a_tiles; a.b_tiles = b_tiles; a.m_tiles = m_tiles; a.n_tiles = n_tiles;
  a.submax = submax; a.tilemax = tilemax; a.full_out = full_out; a.tile_stride = tile_stride;
  return launch_gemm<0>(ctx, a);
}

// candidate-emitting epilogue over all tiles
int stb_launch_batch_gemm_emit(stb_ctx *ctx, const uint8_t *a_tiles, uint32_t m_tiles, const uint8_t *b_tiles,
                               uint32_t n_tiles, uint64_t n_rows, const float *thr, uint32_t *cand_cnt,
                               uint64_t *cand_keys, uint32_t cand_cap) {
  GemmArgs a{};
  a.a_tiles = a_tiles; a.b_tiles = b_tiles; a.m_tiles = m_tiles; a.n_tiles = n_tiles; a.tile_stride = 1;
  a.thr = thr; a.cand_cnt = cand_cnt; a.cand_keys = cand_keys; a.cand_cap = cand_cap; a.n_rows = n_rows;
  return launch_gemm<1>(ctx, a);
}

// Pipeline v2 on the eligible rows only (stb_search_batch_filtered): the sampling pass over the listed tiles
// 0, stride, 2*stride, ... (n_sample of them), tile maxima over eligible rows ...
int stb_launch_batch_gemm_sample_filtered(stb_ctx *ctx, const uint8_t *a_tiles, uint32_t m_tiles, const uint8_t *b_tiles,
                                          const uint32_t *tile_ids, const uint32_t *bitmap, uint32_t n_sample,
                                          uint32_t tile_stride, float *tilemax) {
  GemmArgs a{};
  a.a_tiles = a_tiles; a.b_tiles = b_tiles; a.m_tiles = m_tiles; a.n_tiles = n_sample; a.tile_stride = tile_stride;
  a.tilemax = tilemax; a.tile_ids = tile_ids; a.bitmap = bitmap;
  return launch_gemm<0, STB_GEMM_LISTED>(ctx, a);
}

// ... and the candidate-emitting pass over all n_listed listed tiles, eligible rows only
int stb_launch_batch_gemm_emit_filtered(stb_ctx *ctx, const uint8_t *a_tiles, uint32_t m_tiles, const uint8_t *b_tiles,
                                        const uint32_t *tile_ids, const uint32_t *bitmap, uint32_t n_listed, uint64_t n_rows,
                                        const float *thr, uint32_t *cand_cnt, uint64_t *cand_keys, uint32_t cand_cap) {
  GemmArgs a{};
  a.a_tiles = a_tiles; a.b_tiles = b_tiles; a.m_tiles = m_tiles; a.n_tiles = n_listed; a.tile_stride = 1;
  a.thr = thr; a.cand_cnt = cand_cnt; a.cand_keys = cand_keys; a.cand_cap = cand_cap; a.n_rows = n_rows;
  a.tile_ids = tile_ids; a.bitmap = bitmap;
  return launch_gemm<1, STB_GEMM_LISTED>(ctx, a);
}

// Pipeline v2 with one filter per 64-query half (stb_search_batch_subsets): the sampling pass and the emitting
// pass over corpus tiles tile_ids[0, n_tiles), each with its work items (GemmArgs, STB_GEMM_WORK); masks are
// 8-word slots of `bitmap`.  The sampling pass writes tilemax [m_tiles][tm_cols][128] at each half's sample
// column; the emitting pass writes slot s's keys and count at row slot_row[s].
int stb_launch_batch_gemm_sample_work(stb_ctx *ctx, const uint8_t *a_tiles, const uint8_t *b_tiles, const uint32_t *tile_ids,
                                      uint32_t n_tiles, const uint32_t *cta_tiles, const uint32_t *item_off, const uint4 *items,
                                      const uint32_t *bitmap, uint32_t tm_cols, float *tilemax) {
  GemmArgs a{};
  a.a_tiles = a_tiles; a.b_tiles = b_tiles; a.tile_ids = tile_ids; a.n_tiles = n_tiles; a.cta_tiles = cta_tiles;
  a.item_off = item_off; a.items = items; a.bitmap = bitmap; a.tile_stride = tm_cols; a.tilemax = tilemax;
  return launch_gemm<0, STB_GEMM_WORK>(ctx, a);
}

int stb_launch_batch_gemm_emit_work(stb_ctx *ctx, const uint8_t *a_tiles, const uint8_t *b_tiles, const uint32_t *tile_ids,
                                    uint32_t n_tiles, const uint32_t *cta_tiles, const uint32_t *item_off, const uint4 *items,
                                    const uint32_t *bitmap, const uint32_t *slot_row, uint64_t n_rows, const float *thr,
                                    uint32_t *cand_cnt, uint64_t *cand_keys, uint32_t cand_cap) {
  GemmArgs a{};
  a.a_tiles = a_tiles; a.b_tiles = b_tiles; a.tile_ids = tile_ids; a.n_tiles = n_tiles; a.cta_tiles = cta_tiles;
  a.item_off = item_off; a.items = items; a.bitmap = bitmap; a.slot_row = slot_row; a.n_rows = n_rows;
  a.thr = thr; a.cand_cnt = cand_cnt; a.cand_keys = cand_keys; a.cand_cap = cand_cap;
  return launch_gemm<1, STB_GEMM_WORK>(ctx, a);
}

// stb_search_batch_subsets's query slots: slot s holds the f32 query row slot_row[s] of `rows` (zeros for a
// padding slot, ~0) ...
__global__ void stb_batch_slots_gather_kernel(const float4 *__restrict__ rows, const uint32_t *__restrict__ slot_row,
                                              uint32_t n_slots, float4 *__restrict__ out) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;       // one float4 each
  if (i >= (uint64_t)n_slots * STB_ROW_F4) return;
  const uint32_t r = __ldg(slot_row + i / STB_ROW_F4);
  out[i] = (r == 0xffffffffu) ? make_float4(0.f, 0.f, 0.f, 0.f) : __ldg(rows + (uint64_t)r * STB_ROW_F4 + i % STB_ROW_F4);
}

// ... and, once the slots' shadow is built: row_bad[slot_row[s]] = slot_bad[s], and every tilemax entry -inf,
// so the columns past a group's own sample never rank above its sampled maxima
__global__ void stb_batch_slots_prep_kernel(const uint32_t *__restrict__ slot_row, const uint32_t *__restrict__ slot_bad,
                                            uint32_t n_slots, uint32_t *__restrict__ row_bad, float *__restrict__ tilemax,
                                            uint64_t n_tilemax) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_slots) {
    const uint32_t r = slot_row[i];
    if (r != 0xffffffffu) row_bad[r] = slot_bad[i];
  }
  if (i < n_tilemax) tilemax[i] = -CUDART_INF_F;
}

int stb_launch_batch_slots_gather(stb_ctx *ctx, const float *rows, const uint32_t *slot_row, uint32_t n_slots, float *out) {
  const uint64_t n = (uint64_t)n_slots * STB_ROW_F4;
  if (n == 0) return STB_OK;
  stb_batch_slots_gather_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(
      reinterpret_cast<const float4 *>(rows), slot_row, n_slots, reinterpret_cast<float4 *>(out));
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

int stb_launch_batch_slots_prep(stb_ctx *ctx, const uint32_t *slot_row, const uint32_t *slot_bad, uint32_t n_slots,
                                uint32_t *row_bad, float *tilemax, uint64_t n_tilemax) {
  const uint64_t n = std::max<uint64_t>(n_slots, n_tilemax);
  if (n == 0) return STB_OK;
  stb_batch_slots_prep_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(slot_row, slot_bad, n_slots, row_bad,
                                                                                     tilemax, n_tilemax);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// Threshold mode's re-emission: the candidate-emitting pass over all tiles into the exactly sized segments
// seg_off[] of cand_keys; cursors [q_pad][grid] zeroed by the caller
int stb_launch_batch_gemm_emit_sized(stb_ctx *ctx, const uint8_t *a_tiles, uint32_t m_tiles, const uint8_t *b_tiles,
                                     uint32_t n_tiles, uint64_t n_rows, const float *thr, uint32_t *cursors,
                                     uint64_t *cand_keys, const uint64_t *seg_off) {
  GemmArgs a{};
  a.a_tiles = a_tiles; a.b_tiles = b_tiles; a.m_tiles = m_tiles; a.n_tiles = n_tiles; a.tile_stride = 1;
  a.thr = thr; a.cand_cnt = cursors; a.cand_keys = cand_keys; a.n_rows = n_rows; a.seg_off = seg_off;
  return launch_gemm<2>(ctx, a);
}


// ------------------------------------------------------------- 3. sub-tile selection ---
// grid (m_tiles, n_slices), 128 threads = the 128 queries of one query tile x one slice of
// sub-tiles; lane keeps the KSEL best (value, sub-tile) of its query in shared memory
// ([entry][lane] layout: conflict-free) with the running minimum in registers.
struct SelectArgs {
  const float *submax;      // [m_tiles][n_sub][128]  (tile maxima when called on tilemax)
  uint32_t n_sub, q_pad, n_slices;
  uint64_t *cand;           // [q_pad][n_slices][KSEL] keys: (~ord(value) << 32) | sub-tile
};

__global__ void __launch_bounds__(128)
stb_batch_select_kernel(const SelectArgs a) {
  __shared__ float s_val[4][STB_BATCH_KSEL * 32];
  __shared__ uint32_t s_idx[4][STB_BATCH_KSEL * 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t slice = blockIdx.y;
  const uint32_t q = blockIdx.x * 128 + threadIdx.x;
  const uint32_t per = (a.n_sub + a.n_slices - 1) / a.n_slices;
  const uint32_t s0 = slice * per, s1 = min(a.n_sub, s0 + per);
  float *val = s_val[warp];
  uint32_t *idx = s_idx[warp];
  int cnt = 0, minpos = 0;
  float thr = -CUDART_INF_F;
  const float *p = a.submax + (size_t)blockIdx.x * a.n_sub * 128 + threadIdx.x;   // CTA reads 512 B rows
  // 16 independent coalesced loads in flight per lane before the (rare) list updates
  // (measured: 64 is slower -- 151 registers, longer serial tail per batch)
  constexpr int UNR = 16;
  for (uint32_t st0 = s0; st0 < s1; st0 += UNR) {
    float vbuf[UNR];
#pragma unroll
    for (int u = 0; u < UNR; ++u)
      vbuf[u] = (st0 + u < s1) ? __ldcs(p + (size_t)(st0 + u) * 128) : -CUDART_INF_F;
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      const float v = vbuf[u];
      const uint32_t st = st0 + u;
      if (st >= s1) break;
      if (cnt < STB_BATCH_KSEL) {
        val[cnt * 32 + lane] = v; idx[cnt * 32 + lane] = st;
        if (++cnt == STB_BATCH_KSEL) {
          thr = CUDART_INF_F;
          for (int e = 0; e < STB_BATCH_KSEL; ++e) { float x = val[e * 32 + lane]; if (x < thr) { thr = x; minpos = e; } }
        }
      } else if (v > thr) {
        val[minpos * 32 + lane] = v; idx[minpos * 32 + lane] = st;
        thr = CUDART_INF_F;
        for (int e = 0; e < STB_BATCH_KSEL; ++e) { float x = val[e * 32 + lane]; if (x < thr) { thr = x; minpos = e; } }
      }
    }
  }
  uint64_t *out = a.cand + ((size_t)q * a.n_slices + slice) * STB_BATCH_KSEL;
  for (int e = 0; e < STB_BATCH_KSEL; ++e)
    out[e] = (e < cnt) ? stb_make_key(val[e * 32 + lane], idx[e * 32 + lane]) : STB_KEY_INVALID;
}

// ------------------------------------------------------------------ 4. exact finish ---
struct FinishArgs {
  const uint64_t *cand;     // [q_pad][n_slices][KSEL]  keys over TILES (value = tile maximum)
  const float *submax;      // [m_tiles][n_tiles * 8][128]
  uint32_t q_pad;
  uint32_t n_slices, n_sub, nq, top_k;
  const float4 *rows;       // corpus f32 rows (local)
  uint64_t n_rows, row_base;
  const float *queries;     // [nq][256] f32 (device)
  const uint32_t *q_bad;    // [nq] 1: the query could not be normalised (never proven)
  stb_hit *out_hits;        // [nq][top_k]
  uint32_t *out_status;     // [nq][2]: hits, complete
};

#define STB_FINISH_KEYS 4096     // candidate tile keys one query can bring (128 slices x 32)

__global__ void __launch_bounds__(256, 3)
stb_batch_finish_kernel(const FinishArgs a) {
  // one 32 KB buffer, reused: [0,4096) tile keys -> [0,256) sub-tile keys, then
  // sd = buf[1024..2048) as doubles and sr = buf[2048..3072) for the (distance,row) pairs
  __shared__ uint64_t buf[STB_FINISH_KEYS];
  uint64_t *skeys = buf;
  double *sd = reinterpret_cast<double *>(buf + 1024);
  uint64_t *sr = buf + 2048;
  __shared__ double sqd[STB_D];
  __shared__ double s_q2;
  __shared__ int s_pass, s_alltiles;
  const uint32_t q = blockIdx.x;
  const int tid = threadIdx.x;
  // launched with 256 threads (one per sub-tile key below); with the stride known the shared-memory
  // sorts fit 64 registers, i.e. 4 CTAs per SM
  __builtin_assume(blockDim.x == 256);
  // 1. merge the per-slice candidate tiles, keep the KSEL best
  const uint32_t n_in = a.n_slices * STB_BATCH_KSEL;     // <= STB_FINISH_KEYS
  int n_sort = 64;
  while ((uint32_t)n_sort < n_in) n_sort <<= 1;
  const uint64_t *src = a.cand + (size_t)q * n_in;
  for (int i = tid; i < n_sort; i += 256) skeys[i] = ((uint32_t)i < n_in) ? src[i] : STB_KEY_INVALID;
  for (int i = tid; i < STB_D; i += 256) sqd[i] = (double)__ldg(a.queries + (size_t)q * STB_D + i);
  if (tid == 0) s_pass = 0;
  __syncthreads();
  stb_cta_sort_keys_strided(skeys, n_sort);      // in place, ascending (best first)
  // 1b. the KSEL best sub-tiles all lie inside the KSEL best tiles (a tile's maximum is the
  //     maximum of its 8 sub-tiles): expand those tiles to their 8 sub-tile maxima, sort
  //     again and keep the KSEL best sub-tiles.
  {
    // <= KSEL tile candidates in total means every slice offered ALL its tiles: nothing unselected
    if (tid == 0) s_alltiles = (skeys[STB_BATCH_KSEL] == STB_KEY_INVALID) ? 1 : 0;
    uint64_t mykey = STB_KEY_INVALID;
    const uint64_t tkey = skeys[tid >> 3];                 // tid < 256 -> tile slot tid/8, sub-tile tid%8
    if (tkey != STB_KEY_INVALID) {
      const uint32_t st = stb_key_row(tkey) * (STB_B_TILE / STB_SUB) + (tid & 7);
      if (st < a.n_sub) mykey = stb_make_key(__ldg(a.submax + ((size_t)(q >> 7) * a.n_sub + st) * 128 + (q & 127)), st);
    }
    __syncthreads();
    skeys[tid] = mykey;                                   // 256 threads -> 256 sub-tile keys
    __syncthreads();
    stb_cta_sort_keys_strided(skeys, 256);
  }
  if (tid == 0) s_q2 = stb_canon_q2(sqd);
  __syncthreads();
  // 2. exact canonical distance of every row of the selected sub-tiles (one thread per row)
  const double q2 = s_q2;
  for (int c = tid; c < STB_BATCH_KSEL * STB_SUB; c += 256) {
    const uint64_t key = skeys[c / STB_SUB];
    double d = CUDART_INF;
    uint64_t grow = 0xffffffffffffffffull;
    if (key != STB_KEY_INVALID) {
      const uint64_t row = (uint64_t)stb_key_row(key) * STB_SUB + (c % STB_SUB);
      if (row < a.n_rows) {
        double ab, r2;
        stb_canon_dot<true>(sqd, a.rows + row * STB_ROW_F4, ab, r2);
        const double dist = stb_canon_dist(ab, q2, r2);
        if (dist < STB_DEFAULT_MAX_DIST) { d = dist; grow = a.row_base + row; atomicAdd(&s_pass, 1); }
      }
    }
    sd[c] = d; sr[c] = grow;
  }
  __syncthreads();
  // 3. sort the 1024 (distance,row) pairs
  stb_cta_sort_hits(sd, sr, STB_BATCH_KSEL * STB_SUB);
  // 4. hits + completeness proof
  const uint32_t k = a.top_k;
  const uint32_t n_out = min((uint32_t)s_pass, k);
  stb_write_hits(a.out_hits + (size_t)q * k, sd, sr, n_out, k);
  if (tid == 0) {
    bool complete;
    if (s_alltiles && skeys[STB_BATCH_KSEL] == STB_KEY_INVALID) complete = true;   // every sub-tile was re-scored
    else if (skeys[STB_BATCH_KSEL - 1] == STB_KEY_INVALID) complete = false;        // (cannot happen: < KSEL sub-tiles but tiles left out)
    else {
      // m* = KSEL-th best selected sub-tile maximum bounds every unselected row's approximate
      // cosine: sub-tiles left out inside the selected tiles rank below it, and a left-out
      // tile's maximum is <= the KSEL-th tile maximum <= m* (each selected tile contributes a
      // sub-tile equal to its maximum).  Hence exact cosine <= m* + EPS for all of them.
      const float m_star = stb_key_score(skeys[STB_BATCH_KSEL - 1]);
      complete = (n_out == k) && ((1.0 - (double)m_star - STB_BATCH_EPS) > sd[k - 1]);
    }
    if (a.q_bad[q]) complete = false;       // unnormalisable query: its scores bound nothing
    a.out_status[2 * q] = n_out;
    a.out_status[2 * q + 1] = complete ? 1u : 0u;
  }
}

int stb_launch_batch_select(stb_ctx *ctx, const float *submax, uint32_t n_sub, uint32_t q_pad,
                            uint32_t n_slices, uint64_t *cand) {
  SelectArgs a;
  a.submax = submax; a.n_sub = n_sub; a.q_pad = q_pad; a.n_slices = n_slices; a.cand = cand;
  dim3 grid(q_pad / 128, n_slices);
  stb_batch_select_kernel<<<grid, 128, 0, ctx->stream>>>(a);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

int stb_launch_batch_finish(stb_ctx *ctx, const uint64_t *cand, uint32_t n_slices, uint32_t n_sub,
                            uint32_t nq, uint32_t top_k, const float *rows, uint64_t n_rows,
                            uint64_t row_base, const float *queries_dev, const uint32_t *q_bad, stb_hit *out_hits,
                            uint32_t *out_status, const float *submax, uint32_t q_pad) {
  FinishArgs a;
  a.cand = cand; a.n_slices = n_slices; a.n_sub = n_sub; a.nq = nq; a.top_k = top_k;
  a.submax = submax; a.q_pad = q_pad;
  a.rows = reinterpret_cast<const float4 *>(rows); a.n_rows = n_rows; a.row_base = row_base;
  a.queries = queries_dev; a.q_bad = q_bad; a.out_hits = out_hits; a.out_status = out_status;
  stb_batch_finish_kernel<<<nq, 256, 0, ctx->stream>>>(a);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// =========================================================================================
// Pipeline v2 (top_k <= 64 where it fits; the maxima/select/finish pipeline above serves the rest):
//   sampling GEMM (maxima epilogue over ~4*SMs strided COMPLETE tiles) -> per-query threshold
//   -> full GEMM whose epilogue emits the rows reaching the threshold -> exact finish.
// Why the candidate set is sufficient, for ANY k (a = approximate score, c = exact cosine,
// |a - c| <= EPS = STB_BATCH_EPS):
//   S_k = k-th largest sampled tile maximum.  Each tile maximum is the score of a real row
//   (only complete tiles are sampled), so k distinct rows have a >= S_k, hence c >= S_k - EPS,
//   hence the k-th largest exact cosine C_k >= S_k - EPS.  A row of the exact top-k has
//   c >= min(C_k, 1) (distance = max(0, 1 - c) is monotone in c and clamps at c >= 1), so
//   a >= min(C_k, 1) - EPS >= S_k - 2 EPS (S_k <= 1 + EPS).  Emitting a >= S_k - 2 EPS loses none.
//   The same argument with "sample" = all rows narrows the emitted set to a >= A_k - 2 EPS
//   (A_k = k-th largest emitted score = k-th largest score overall) before the exact re-score.
//   No further proof obligation: the result is complete unless a capacity overflowed.
// Filtered (FILTER GEMMs): "rows" are the eligible rows.  The sample is taken over listed tiles (each holds an
//   eligible row) with ineligible scores masked to -inf, so each sampled maximum is an eligible row's score and
//   S_k bounds the eligible k-th cosine; an unmasked ineligible row could lift S_k above it, and the eligible
//   top-k would then go unemitted while the finish still reports the query proven.
// =========================================================================================
#define STB_V2_MAX_SAMPLE 608          // 19 values per lane in the threshold kernel
#define STB_V2_MAX_K 64                // threshold kernel extracts k maxima serially

struct ThreshArgs {
  const float *tilemax;     // [m_tiles][n_sample][128]
  uint32_t n_sample, nq, q_pad, top_k;
  float *thr;               // [q_pad]
  float slack;              // thr = k-th largest sampled maximum - slack
  const uint32_t *q_skip;   // [nq] or null: 1 = the query emits nothing (thr +inf)
};

// one warp per query: lane l holds sampled tile maxima l, l+32, ...; k rounds of warp-max
// extraction give the k-th largest.
__global__ void __launch_bounds__(256)
stb_batch_thresh_kernel(const ThreshArgs a) {
  const int lane = threadIdx.x & 31;
  const uint32_t q = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (q >= a.q_pad) return;
  if (q >= a.nq) { if (lane == 0) a.thr[q] = CUDART_INF_F; return; }       // padding query: never emits
  float v[STB_V2_MAX_SAMPLE / 32];
  const float *p = a.tilemax + (size_t)(q >> 7) * a.n_sample * 128 + (q & 127);
#pragma unroll
  for (int j = 0; j < STB_V2_MAX_SAMPLE / 32; ++j) {
    const uint32_t idx = j * 32 + lane;
    v[j] = (idx < a.n_sample) ? __ldg(p + (size_t)idx * 128) : -CUDART_INF_F;
  }
  float kth = -CUDART_INF_F;
  if (a.top_k <= a.n_sample && a.top_k <= STB_V2_MAX_K) {
    for (uint32_t round = 0; round < a.top_k; ++round) {
      float lm = v[0];
#pragma unroll
      for (int j = 1; j < STB_V2_MAX_SAMPLE / 32; ++j) lm = fmaxf(lm, v[j]);
      float wm = lm;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) wm = fmaxf(wm, __shfl_xor_sync(0xffffffffu, wm, off));
      const unsigned owners = __ballot_sync(0xffffffffu, lm == wm);
      if (lane == __ffs(owners) - 1) {                  // remove ONE instance of the maximum
        bool removed = false;
#pragma unroll
        for (int j = 0; j < STB_V2_MAX_SAMPLE / 32; ++j)
          if (!removed && v[j] == wm) { v[j] = -CUDART_INF_F; removed = true; }
      }
      kth = wm;
    }
  }
  // fewer than k sampled tiles (or k too large): -inf = emit everything (tiny corpora fit the cap)
  if (lane == 0) a.thr[q] = (a.q_skip && a.q_skip[q]) ? CUDART_INF_F : (kth == -CUDART_INF_F) ? -CUDART_INF_F : kth - a.slack;
}

// Same result for samples beyond 608 tiles (large shards): CTA per query, the sampled maxima
// staged in shared memory, k rounds of block-max extraction.  Up to 49152 maxima (192 KiB): v2's plans stay
// within 8192 (32 KiB, the default limit); route 7's plan samples up to the full capacity on the largest corpora.
#define STB_V2_BIG_SAMPLE 49152
__global__ void __launch_bounds__(256)
stb_batch_thresh_big_kernel(const ThreshArgs a) {
  extern __shared__ float tb_vals[];          // n_sample floats
  __shared__ float s_wm[8];
  __shared__ int s_wi[8];
  __shared__ float s_kth;
  const uint32_t q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (q >= a.nq) { if (tid == 0) a.thr[q] = CUDART_INF_F; return; }
  const float *p = a.tilemax + (size_t)(q >> 7) * a.n_sample * 128 + (q & 127);
  for (uint32_t i = tid; i < a.n_sample; i += 256) tb_vals[i] = __ldg(p + (size_t)i * 128);
  if (tid == 0) s_kth = -CUDART_INF_F;
  __syncthreads();
  if (a.top_k <= a.n_sample && a.top_k <= STB_V2_MAX_K) {
    for (uint32_t round = 0; round < a.top_k; ++round) {
      float lm = -CUDART_INF_F;
      int li = -1;
      for (uint32_t i = tid; i < a.n_sample; i += 256) {
        const float v = tb_vals[i];
        if (li < 0 || v > lm) { lm = v; li = (int)i; }
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, lm, off);
        const int oi = __shfl_xor_sync(0xffffffffu, li, off);
        if (oi >= 0 && (li < 0 || om > lm || (om == lm && oi < li))) { lm = om; li = oi; }
      }
      if (lane == 0) { s_wm[warp] = lm; s_wi[warp] = li; }
      __syncthreads();
      if (tid == 0) {
        float bm = s_wm[0];
        int bi = s_wi[0];
        for (int w = 1; w < 8; ++w)
          if (s_wi[w] >= 0 && (bi < 0 || s_wm[w] > bm || (s_wm[w] == bm && s_wi[w] < bi))) { bm = s_wm[w]; bi = s_wi[w]; }
        s_kth = bm;
        if (bi >= 0) tb_vals[bi] = -CUDART_INF_F;       // remove ONE instance
      }
      __syncthreads();
    }
  }
  if (tid == 0) {
    const float kth = (a.top_k <= a.n_sample && a.top_k <= STB_V2_MAX_K) ? s_kth : -CUDART_INF_F;
    a.thr[q] = (a.q_skip && a.q_skip[q]) ? CUDART_INF_F : (kth == -CUDART_INF_F) ? -CUDART_INF_F : kth - a.slack;
  }
}

struct Finish2Args {
  const uint64_t *cand_keys;   // [q_pad][n_seg][seg_cap]
  const uint32_t *cand_cnt;    // [q_pad][n_seg]
  uint32_t n_seg, seg_cap, nq, top_k;
  const float4 *rows;
  uint64_t n_rows, row_base;
  const float *queries;        // [nq][256]
  const uint32_t *q_bad;       // [nq] 1: the query could not be normalised (never proven)
  stb_hit *out_hits;           // [nq][top_k]
  uint32_t *out_status;        // [nq][2]: hits, complete
  // route 7 (null on the shadow's routes): the keys hold q8 upper bounds u (stb_batch_q8_gemm_kernel); the q8
  // scales, the queries' {1/S, h_l1, e_q, S} and the emission thresholds the proof is checked against
  const float *q8_scale;
  const float4 *q8_qc;
  const float *thr;
};

#define STB_F2_KEYS 4096         // emitted candidates one query may bring (sum over its segments)
#define STB_F2_RESCORE 1024      // exact re-scores per query after narrowing (dense neighbourhoods)
#define STB_F2_STRIDE 260        // floats per staged row (1 KiB + 16 B: conflict-free LDS.128)

// One CTA (256 threads) per query: gather the query's segments, sort by approximate score
// (register/shuffle bitonic network), narrow to a >= A_k - 2 EPS, re-score those rows exactly
// (rows staged through shared memory with coalesced loads, f64 chains on 4 warps -- K1's re-rank)
// and sort the (distance,row) pairs.  A capacity overflow anywhere marks the query unproven.
__global__ void __launch_bounds__(256)
stb_batch_finish2_kernel(const Finish2Args a) {
  extern __shared__ __align__(16) uint8_t f2_smem[];      // keys[4096] | 32 staged rows
  uint64_t *skeys = reinterpret_cast<uint64_t *>(f2_smem);
  float *srows = reinterpret_cast<float *>(f2_smem + STB_F2_KEYS * sizeof(uint64_t));
  __shared__ double sqd[STB_D];
  __shared__ double sd[STB_F2_RESCORE];
  __shared__ uint64_t sr[STB_F2_RESCORE];
  __shared__ double s_q2;
  __shared__ uint32_t s_off[256 + 1];
  __shared__ int s_pass, s_over;
  __shared__ unsigned s_m2;
  __shared__ unsigned s_sel[3];
  const uint32_t q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t k = a.top_k;
  auto give_up = [&]() {                               // the host answers this query through K1
    stb_write_hits(a.out_hits + (size_t)q * k, sd, sr, 0, k);
    if (tid == 0) { a.out_status[2 * q] = 0; a.out_status[2 * q + 1] = 0; }
  };
  // 1. segment counts -> offsets (n_seg <= 256: one thread per segment, warp scans + 8-entry fix-up)
  if (tid == 0) { s_pass = 0; s_over = 0; s_m2 = 0; s_sel[0] = s_sel[1] = s_sel[2] = 0; }
  __syncthreads();
  uint32_t c = 0;
  if ((uint32_t)tid < a.n_seg) {
    c = a.cand_cnt[(size_t)q * a.n_seg + tid];
    if (c > a.seg_cap) { s_over = 1; c = a.seg_cap; }
  }
  uint32_t incl = c;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += v;
  }
  __shared__ uint32_t s_wsum[8];
  if (lane == 31) s_wsum[warp] = incl;
  __syncthreads();
  uint32_t base = 0;
  for (int w = 0; w < warp; ++w) base += s_wsum[w];
  s_off[tid] = base + incl - c;
  if (tid == 255) s_off[256] = base + incl;
  for (int i = tid; i < STB_D; i += 256) sqd[i] = (double)__ldg(a.queries + (size_t)q * STB_D + i);
  __syncthreads();
  const uint32_t m_all = s_off[256];
  if (s_over || m_all > STB_F2_KEYS) { give_up(); return; }          // uniform per CTA
  // 2. gather (each thread copies its own segment: ~5 keys) and sort best-first
  {
    const uint64_t *src = a.cand_keys + ((size_t)q * a.n_seg + tid) * a.seg_cap;
    const uint32_t o = s_off[tid];
    for (uint32_t i = 0; i < c; ++i) skeys[o + i] = src[i];
  }
  int n_sort = 256;
  while ((uint32_t)n_sort < m_all) n_sort <<= 1;
  const int span = n_sort <= 256 ? 256 : (n_sort <= 1024 ? 1024 : STB_F2_KEYS);   // the register sort writes back its whole span
  __syncthreads();
  for (int i = (int)m_all + tid; i < span; i += 256) skeys[i] = STB_KEY_INVALID;
  __syncthreads();
  if (n_sort <= 256) stb_cta_sort_keys_t<1>(skeys, n_sort);
  else if (n_sort <= 1024) stb_cta_sort_keys_t<4>(skeys, n_sort);
  else stb_cta_sort_keys_t<16>(skeys, n_sort);
  // 3. narrow to a >= A_k - 2 EPS (everything when fewer than k rows were emitted)
  float cut = -CUDART_INF_F;
  if (a.q8_scale) {
    // route 7: the keys are upper bounds u >= c - 1e-5.  l = u - 2 (s h_l1 + e_q) - 2 STB_Q8_SCAN_EPS is a lower bound
    // of c (the q8 bounds' two error terms, plus the fp32 evaluation of u and of this difference), so the k
    // emitted rows with the largest l have c >= L_k, and a row with u < L_k - STB_Q8_SCAN_EPS has c < L_k: it
    // can neither be a result nor tie with one.  Those rows are dropped before any f32 row is read.  L_k: the
    // largest T with #{l >= T} >= k, bit by bit on the ordered l (staged where the rows go later)
    if (m_all >= k) {
      uint32_t *lo = reinterpret_cast<uint32_t *>(srows);
      const float4 qc = __ldg(a.q8_qc + q);
      for (uint32_t i = tid; i < m_all; i += 256) {
        const float w = fmaf(__ldg(a.q8_scale + stb_key_row(skeys[i])), qc.y, qc.z);
        lo[i] = stb_f2ord(stb_key_score(skeys[i]) - 2.0f * w - 2.0f * (float)STB_Q8_SCAN_EPS);
      }
      __syncthreads();
      uint32_t T = 0;
      for (int bit = 31; bit >= 0; --bit) {
        const uint32_t cand = T | (1u << bit);
        uint32_t n_ge = 0;
        for (uint32_t i = tid; i < m_all; i += 256) n_ge += lo[i] >= cand ? 1u : 0u;
        n_ge = __reduce_add_sync(0xffffffffu, n_ge);
        if (lane == 0 && n_ge) atomicAdd(&s_sel[bit % 3], n_ge);
        __syncthreads();
        if (s_sel[bit % 3] >= k) T = cand;
        if (tid == 0) s_sel[(bit + 1) % 3] = 0;     // the counter of round bit - 2, last read before this round's barrier
      }
      cut = stb_ord2f(T) - (float)STB_Q8_SCAN_EPS;
    }
  } else if (m_all >= k) {
    cut = stb_key_score(skeys[k - 1]) - 2.0f * (float)STB_BATCH_EPS;
  }
  for (uint32_t i = tid; i < m_all; i += 256)
    if (stb_key_score(skeys[i]) >= cut) atomicMax(&s_m2, i + 1);
  if (tid == 5 * 32) s_q2 = stb_canon_q2(sqd);
  __syncthreads();
  const uint32_t m2 = s_m2;
  if (m2 > STB_F2_RESCORE) { give_up(); return; }
  // 4. exact canonical distances, 32 rows per pass
  const double q2 = s_q2;
  for (uint32_t c0 = 0; c0 < m2; c0 += 32) {
    {
      constexpr int PER = 32 * STB_ROW_F4 / 256;
      float4 v[PER];
#pragma unroll
      for (int u = 0; u < PER; ++u) {
        const int t = tid + u * 256;
        const uint32_t ci = c0 + (t >> 6);
        v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ci < m2) v[u] = __ldg(a.rows + (size_t)stb_key_row(skeys[ci]) * STB_ROW_F4 + (t & 63));
      }
#pragma unroll
      for (int u = 0; u < PER; ++u) {
        const int t = tid + u * 256;
        *reinterpret_cast<float4 *>(srows + (t >> 6) * STB_F2_STRIDE + (t & 63) * 4) = v[u];
      }
    }
    __syncthreads();
    if (tid < 128 && lane < 8) {
      const int cl = warp * 8 + lane;
      const uint32_t ci = c0 + cl;
      if (ci < m2) {
        double ab, r2;
        stb_canon_dot<false>(sqd, reinterpret_cast<const float4 *>(srows + cl * STB_F2_STRIDE), ab, r2);
        const double dist = stb_canon_dist(ab, q2, r2);
        if (dist < STB_DEFAULT_MAX_DIST) { sd[ci] = dist; sr[ci] = a.row_base + (uint64_t)stb_key_row(skeys[ci]); atomicAdd(&s_pass, 1); }
        else { sd[ci] = CUDART_INF; sr[ci] = 0xffffffffffffffffull; }
      }
    }
    __syncthreads();
  }
  // 5. sort the (distance,row) pairs, write the top-k
  uint32_t n2 = 32;
  while (n2 < m2) n2 <<= 1;
  for (uint32_t i = m2 + tid; i < n2; i += 256) { sd[i] = CUDART_INF; sr[i] = 0xffffffffffffffffull; }
  __syncthreads();
  stb_cta_sort_hits(sd, sr, n2);
  const uint32_t n_out = min((uint32_t)s_pass, k);
  stb_write_hits(a.out_hits + (size_t)q * k, sd, sr, n_out, k);
  if (tid == 0) {
    bool complete = !a.q_bad[q];
    if (a.q8_scale) {
      // route 7: a row that was not emitted has u < thr, hence c <= u + 1e-5 < thr + 1e-5; the query is proven if
      // the k-th re-scored distance beats every such row strictly (the margin also covers the f64 distance's
      // rounding).  thr is finite here: the plan samples at least k tiles, each holding a real row
      complete = complete && n_out == k && sd[k - 1] < 1.0 - (double)a.thr[q] - STB_Q8_SCAN_EPS;
    }
    a.out_status[2 * q] = n_out;
    a.out_status[2 * q + 1] = complete ? 1u : 0u;
  }
}

int stb_launch_batch_thresh(stb_ctx *ctx, const float *tilemax, uint32_t n_sample, uint32_t nq, uint32_t q_pad,
                            uint32_t top_k, float *thr, float slack, const uint32_t *q_skip) {
  if (n_sample > STB_V2_BIG_SAMPLE) { stb_set_error("batch_thresh: sample too large"); return STB_ERR_ARG; }
  ThreshArgs a;
  a.tilemax = tilemax; a.n_sample = n_sample; a.nq = nq; a.q_pad = q_pad; a.top_k = top_k; a.thr = thr;
  a.slack = slack < 0.f ? 2.0f * (float)STB_BATCH_EPS : slack; a.q_skip = q_skip;
  if (n_sample <= STB_V2_MAX_SAMPLE) stb_batch_thresh_kernel<<<(q_pad + 7) / 8, 256, 0, ctx->stream>>>(a);
  else {
    const size_t smem = (size_t)n_sample * sizeof(float);
    if (smem > 48 * 1024)
      STB_ATTR_ONCE(ctx, STB_ATTR_THRESH_BIG, cudaFuncSetAttribute(stb_batch_thresh_big_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                                   STB_V2_BIG_SAMPLE * (int)sizeof(float)));
    stb_batch_thresh_big_kernel<<<q_pad, 256, smem, ctx->stream>>>(a);
  }
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

uint32_t stb_batch_emit_grid(const stb_ctx *ctx, uint32_t n_tiles) {
  return std::min<uint32_t>(n_tiles, (uint32_t)ctx->sm_count);
}

int stb_launch_batch_finish2(stb_ctx *ctx, const uint64_t *cand_keys, const uint32_t *cand_cnt, uint32_t n_seg,
                             uint32_t seg_cap, uint32_t nq, uint32_t top_k, const float *rows, uint64_t n_rows,
                             uint64_t row_base, const float *queries_dev, const uint32_t *q_bad, stb_hit *out_hits,
                             uint32_t *out_status, const float *q8_scale, const float4 *q8_qc, const float *thr) {
  if (top_k > STB_F2_RESCORE || n_seg > 256 || n_seg == 0) { stb_set_error("batch_finish2: bad shape"); return STB_ERR_ARG; }
  Finish2Args a;
  a.cand_keys = cand_keys; a.cand_cnt = cand_cnt; a.n_seg = n_seg; a.seg_cap = seg_cap; a.nq = nq; a.top_k = top_k;
  a.rows = reinterpret_cast<const float4 *>(rows); a.n_rows = n_rows; a.row_base = row_base;
  a.queries = queries_dev; a.q_bad = q_bad; a.out_hits = out_hits; a.out_status = out_status;
  a.q8_scale = q8_scale; a.q8_qc = q8_qc; a.thr = thr;
  constexpr size_t smem = STB_F2_KEYS * sizeof(uint64_t) + 32 * STB_F2_STRIDE * sizeof(float);
  STB_ATTR_ONCE(ctx, STB_ATTR_FINISH2, cudaFuncSetAttribute(stb_batch_finish2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  stb_batch_finish2_kernel<<<nq, 256, smem, ctx->stream>>>(a);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// =========================================================================================
// Route 7: pipeline v2 on the q8 copy and the int8 tensor cores, for corpora whose 16-bit shadow does not fit
// in HBM.  Every row already has int8 codes x8 and a scale s there (K1's q8 tier, 260 B per row); the query is
// quantised exactly as K1 quantises it (q8_query.cuh: q16 = rint(q^ S) = 256 hi + lo, two signed bytes).  Per
// (query, row) the GEMM computes K1's integer dot = 256 (hi . x8) + lo . x8 (exact in int32) and from it K1's
// bounds, bit for bit (scan_topk.cu: stb_scan_q8, stb_scan_q4):
//     u = s (dot / S + h_l1) + e_q  >=  c - 1e-5        l = s (dot / S - h_l1) - e_q - 2e-5  <=  c - 1e-5
// Sufficiency, as v2's with the two bounds in place of the one symmetric EPS: S_k = k-th largest sampled tile
// maximum of l; each is a real row's l (rows past n are masked), so k distinct rows have c >= S_k and C_k >= S_k.
// A row of the exact top-k has c >= min(C_k, 1) >= S_k (l < 1), so u >= S_k - 1e-5: emitting u >= thr = S_k -
// STB_Q8_SCAN_EPS loses none.  The finish (stb_batch_finish2_kernel with the q8 arguments) drops emitted rows
// that cannot win, re-scores the rest exactly and proves the query only if the k-th distance beats thr + eps.
// =========================================================================================

#define STB_Q8_B_SLAB_BYTES (STB_B_TILE * 128)            // 128 code bytes of 256 rows: 32 KiB
#define STB_Q8_GEMM_SMEM (2 * STB_Q8_B_SLAB_BYTES + STB_A_RING * STB_A_SLAB_BYTES + 2 * STB_B_TILE * 4 + 256 + 1024)
static_assert(STB_Q8_GEMM_SMEM <= 227 * 1024, "q8 GEMM shared memory");

// 1. Query tiles.  One warp per query slot (all four lane groups compute the same query, as stb_q8_query's
// reductions require); lane j < 8 writes its 16-byte chunk j of each of the tile's four K-slabs: hi bytes of
// components 0-127, hi 128-255, lo 0-127, lo 128-255, each [128 queries x 128 B] in the 128-byte swizzle.
// Padding slots (>= nq) are zero and flagged.
__global__ void __launch_bounds__(256)
stb_q8_query_tiles_kernel(const float *__restrict__ q, uint32_t nq, uint32_t q_pad, uint8_t *__restrict__ tiles,
                          float4 *__restrict__ qc, uint32_t *__restrict__ q_bad, int16_t *__restrict__ q16) {
  const int lane = threadIdx.x & 31, j = lane & 7;
  const uint32_t qi = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (qi >= q_pad) return;                                  // warp-uniform
  uint32_t hi[8] = {0, 0, 0, 0, 0, 0, 0, 0}, lo[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
  bool bad = true;
  if (qi < nq) {
    const StbQ8Query Q = stb_q8_query(q + (size_t)qi * STB_D, j);
#pragma unroll
    for (int i = 0; i < 8; ++i) { hi[i] = Q.qhi[i]; lo[i] = Q.qlo[i]; }
    c = make_float4(Q.inv_S, Q.h_l1, Q.e_q, Q.S);
    bad = Q.unusable;
  }
  if (lane < 8) {
    const uint32_t r = qi % STB_A_TILE;
    uint8_t *t = tiles + (size_t)(qi / STB_A_TILE) * (4 * STB_A_SLAB_BYTES) + (r >> 3) * 1024 + (r & 7) * 128 +
                 ((j ^ (r & 7)) * 16);
    *reinterpret_cast<uint4 *>(t) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4 *>(t + STB_A_SLAB_BYTES) = make_uint4(hi[4], hi[5], hi[6], hi[7]);
    *reinterpret_cast<uint4 *>(t + 2 * STB_A_SLAB_BYTES) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    *reinterpret_cast<uint4 *>(t + 3 * STB_A_SLAB_BYTES) = make_uint4(lo[4], lo[5], lo[6], lo[7]);
    if (q16 && qi < nq) {
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int k = (i < 4 ? 16 * j + 4 * i : 128 + 16 * j + 4 * (i - 4)) + e;
          q16[(size_t)qi * STB_D + k] = (int16_t)(256 * (int)(int8_t)(hi[i] >> (8 * e)) + (int)(int8_t)(lo[i] >> (8 * e)));
        }
    }
  }
  if (lane == 0) { qc[qi] = c; q_bad[qi] = bad ? 1u : 0u; }
}

int stb_launch_q8_query_tiles(stb_ctx *ctx, const float *q_dev, uint32_t nq, uint32_t q_pad, uint8_t *tiles, float4 *qc,
                              uint32_t *q_bad, int16_t *q16) {
  if (q_pad == 0) return STB_OK;
  stb_q8_query_tiles_kernel<<<(q_pad + 7) / 8, 256, 0, ctx->stream>>>(q_dev, nq, q_pad, tiles, qc, q_bad, q16);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// 2. The GEMM.  Corpus tile = 256 rows: two K-slabs of codes (bytes 0-127 and 128-255 of each row, 32 KiB each)
// loaded with the tensor maps below, which apply the 128-byte swizzle on the way in (the q8 copy stays row-major
// for K1 and zero-fills rows past n), and the tile's 256 scales (1 KiB) with slab 0, double-buffered by tile
// parity: the producer refills buffer (it + 1) & 1 only after every consumer warp released slab 0 of tile it,
// which it does after the epilogues of tile it - 1.  Query tiles stream through the 6-slab ring of
// stb_batch_gemm_kernel.  Per (query tile, corpus tile) a consumer warpgroup runs the hi slabs (K = 256, 8
// wgmma m64n256k32 s8), waits, multiplies its s32 accumulators by 256 and accumulates the lo slabs on top.
__device__ __forceinline__ void wg_reg_fence_s32(int32_t (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+r"(d[i])::"memory");
}
__device__ __forceinline__ void wg_mma_m64n256k32_s8(int32_t (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p;\n\t}"
      :
        "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
        "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
        "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
        "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
        "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
        "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
        "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]),
        "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]),
        "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]),
        "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]),
        "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]),
        "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]),
        "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111]),
        "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]), "+r"(d[118]), "+r"(d[119]),
        "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]), "+r"(d[126]), "+r"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void tma_load_2d(void *dst_smem, const CUtensorMap *map, int x, int y, uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(dst_smem)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const CUtensorMap *map, int x, uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.tensor.1d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2}], [%3];" ::"r"(
          smem_u32(dst_smem)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(smem_u32(bar))
      : "memory");
}

struct Q8GemmArgs {
  const uint8_t *a_tiles;     // m_tiles x 4 slabs x 16 KiB (stb_q8_query_tiles_kernel)
  const float4 *qc;           // [q_pad] {1/S, h_l1, e_q, S}
  uint32_t m_tiles;
  uint32_t n_tiles;           // corpus tiles of this launch: tile t is corpus tile t * tile_stride
  uint32_t tile_stride;
  uint64_t n_rows;            // rows past n (the zero-filled tail of the last tile) never count
  float *tilemax;             // EPI 0: [m_tiles][n_tiles][128] maximum of l per tile
  const float *thr;           // EPI 1: [q_pad] emission thresholds on u ...
  uint32_t *cand_cnt;         //        [q_pad][grid] counts (> cand_cap: overflow marker)
  uint64_t *cand_keys;        //        [q_pad][grid][cand_cap] keys (u desc, local row)
  uint32_t cand_cap;
  int32_t *dot_out;           // EPI 2: [m_tiles * 128][n_tiles * 256] dot, u and l
  float *u_out, *l_out;
};

// EPI 0: sampling (tile maxima of l); EPI 1: emit every row whose u reaches the query's threshold; EPI 2: debug
template <int EPI>
__global__ void __launch_bounds__(STB_GEMM_THREADS, 1)
stb_batch_q8_gemm_kernel(const __grid_constant__ CUtensorMap codes_map, const __grid_constant__ CUtensorMap scale_map,
                         const Q8GemmArgs args) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t *sB = smem;                                          // 2 code slabs
  uint8_t *sA = smem + 2 * STB_Q8_B_SLAB_BYTES;                // query ring
  float *s_scale = reinterpret_cast<float *>(sA + STB_A_RING * STB_A_SLAB_BYTES);   // [2][256]
  uint64_t *bars = reinterpret_cast<uint64_t *>(s_scale + 2 * STB_B_TILE);
  uint64_t *b_full = bars + 0, *b_empty = bars + 2;
  uint64_t *a_full = bars + 4, *a_empty = a_full + STB_A_RING;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) { mbar_init(b_full + i, 1); mbar_init(b_empty + i, STB_GEMM_CONSUMER_WARPS); }
    for (int i = 0; i < STB_A_RING; ++i) { mbar_init(a_full + i, 1); mbar_init(a_empty + i, STB_GEMM_CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const uint32_t my_tiles = (args.n_tiles > blockIdx.x) ? (args.n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

  if (warp < 4) {
    // ===== producer (one thread) =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      uint32_t a_cnt = 0;
      for (uint32_t it = 0; it < my_tiles; ++it) {
        const int row0 = (int)((blockIdx.x + (uint64_t)it * gridDim.x) * args.tile_stride * STB_B_TILE);
        for (int s = 0; s < 2; ++s) {
          mbar_wait(b_empty + s, (it & 1) ^ 1);
          if (s == 0) {
            mbar_expect_tx(b_full, STB_Q8_B_SLAB_BYTES + STB_B_TILE * 4);
            tma_load_1d(s_scale + (it & 1) * STB_B_TILE, &scale_map, row0, b_full);
          } else {
            mbar_expect_tx(b_full + s, STB_Q8_B_SLAB_BYTES);
          }
          tma_load_2d(sB + s * STB_Q8_B_SLAB_BYTES, &codes_map, s * 128, row0, b_full + s);
        }
        for (uint32_t m = 0; m < args.m_tiles; ++m) {
          for (int s = 0; s < 4; ++s, ++a_cnt) {
            const uint32_t slot = a_cnt % STB_A_RING;
            mbar_wait(a_empty + slot, ((a_cnt / STB_A_RING) & 1) ^ 1);
            mbar_expect_tx(a_full + slot, STB_A_SLAB_BYTES);
            bulk_g2s(sA + slot * STB_A_SLAB_BYTES, args.a_tiles + ((size_t)m * 4 + s) * STB_A_SLAB_BYTES, STB_A_SLAB_BYTES,
                     a_full + slot);
          }
        }
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  // ===== consumers (accumulator layout as in stb_batch_gemm_kernel) =====
  const uint32_t half = (uint32_t)(warp >> 2) - 1u;
  const uint32_t qrow = half * 64 + (warp & 3) * 16 + (lane >> 2);
  const uint32_t quad = lane & 3;
  int32_t d[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) d[i] = 0;
  uint32_t a_cnt = 0;
  for (uint32_t it = 0; it < my_tiles; ++it) {
    const uint64_t t = blockIdx.x + (uint64_t)it * gridDim.x;
    const uint64_t row0 = t * args.tile_stride * STB_B_TILE;
    const float *sc = s_scale + (it & 1) * STB_B_TILE;
    for (uint32_t m = 0; m < args.m_tiles; ++m, a_cnt += 4) {
      const uint32_t q0 = m * STB_A_TILE + qrow;
      float4 qc[2];
      [[maybe_unused]] float thr[2];
      [[maybe_unused]] uint32_t cnt[2], cnt0[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        qc[h] = __ldg(args.qc + q0 + 8 * h);
        if constexpr (EPI == 1) {
          thr[h] = __ldg(args.thr + q0 + 8 * h);
          cnt0[h] = args.cand_cnt[(size_t)(q0 + 8 * h) * gridDim.x + blockIdx.x];
          cnt[h] = cnt0[h];
        }
      }
      wg_reg_fence_s32(d);
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        const uint32_t slot = (a_cnt + s) % STB_A_RING;
        if (m == 0 && s < 2) mbar_wait(b_full + s, it & 1);
        mbar_wait(a_full + slot, ((a_cnt + s) / STB_A_RING) & 1);
        if (s == 2) {
          // the hi products are complete: dot = 256 hi.x8 + lo.x8 (|256 hi.x8| <= 256 * 127 * 127 * 256 < 2^31)
          wg_wait<0>();
          wg_reg_fence_s32(d);
#pragma unroll
          for (int i = 0; i < 128; ++i) d[i] *= 256;
          wg_reg_fence_s32(d);
        }
        wg_fence();
        const uint32_t a_addr = smem_u32(sA + slot * STB_A_SLAB_BYTES + half * (64 * 128));
        const uint32_t b_addr = smem_u32(sB + (s & 1) * STB_Q8_B_SLAB_BYTES);
#pragma unroll
        for (int k = 0; k < 4; ++k)   // K by 32 bytes inside the swizzle atom
          wg_mma_m64n256k32_s8(d, wg_desc_sw128(a_addr + k * 32), wg_desc_sw128(b_addr + k * 32), (uint32_t)((s | k) != 0));
        wg_commit();
        if (s > 0) {
          wg_wait<1>();
          if (lane == 0) {
            mbar_arrive(a_empty + (a_cnt + s - 1) % STB_A_RING);
            if (m + 1 == args.m_tiles && s == 3) mbar_arrive(b_empty);    // slab 0's lo pass has retired
          }
        }
      }
      wg_wait<0>();
      wg_reg_fence_s32(d);
      if (lane == 0) {
        mbar_arrive(a_empty + (a_cnt + 3) % STB_A_RING);
        if (m + 1 == args.m_tiles) mbar_arrive(b_empty + 1);
      }

      // d[16c + 4ii + 2h + e]: query qrow + 8h, tile column 32c + 8ii + 2quad + e
      if constexpr (EPI == 0) {
        const uint32_t n_real = args.n_rows > row0 + STB_B_TILE ? STB_B_TILE : (uint32_t)(args.n_rows > row0 ? args.n_rows - row0 : 0);
        float tmx[2] = {-CUDART_INF_F, -CUDART_INF_F};
#pragma unroll
        for (int c = 0; c < STB_B_TILE / STB_SUB; ++c)
#pragma unroll
          for (int ii = 0; ii < 4; ++ii) {
            const uint32_t col = c * STB_SUB + ii * 8 + quad * 2;
            const float2 s2 = *reinterpret_cast<const float2 *>(sc + col);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const bool real = col + e < n_real;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const float l = fmaf(e ? s2.y : s2.x, fmaf((float)d[16 * c + 4 * ii + 2 * h + e], qc[h].x, -qc[h].y), -qc[h].z) -
                                (float)STB_Q8_SCAN_EPS;
                tmx[h] = fmaxf(tmx[h], real ? l : -CUDART_INF_F);
              }
            }
          }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          tmx[h] = fmaxf(tmx[h], __shfl_xor_sync(0xffffffffu, tmx[h], 1));
          tmx[h] = fmaxf(tmx[h], __shfl_xor_sync(0xffffffffu, tmx[h], 2));
          if (quad == (uint32_t)h) args.tilemax[((size_t)m * args.n_tiles + t) * STB_A_TILE + qrow + 8 * h] = tmx[h];
        }
      } else if constexpr (EPI == 1) {
        // as stb_batch_gemm_kernel's EPI 1: a private segment per (query, CTA), branch-free hit masks
#pragma unroll
        for (int c = 0; c < STB_B_TILE / STB_SUB; ++c) {
          const uint64_t r0 = row0 + (uint64_t)c * STB_SUB;
          float u[4][2][2];
#pragma unroll
          for (int ii = 0; ii < 4; ++ii) {
            const float2 s2 = *reinterpret_cast<const float2 *>(sc + c * STB_SUB + ii * 8 + quad * 2);
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                u[ii][h][e] = fmaf(e ? s2.y : s2.x, fmaf((float)d[16 * c + 4 * ii + 2 * h + e], qc[h].x, qc[h].y), qc[h].z);
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint32_t hit = 0u;
#pragma unroll
            for (int ii = 0; ii < 4; ++ii)
#pragma unroll
              for (int e = 0; e < 2; ++e) hit |= (u[ii][h][e] >= thr[h] ? 1u : 0u) << (ii * 8 + quad * 2 + e);
            hit |= __shfl_xor_sync(0xffffffffu, hit, 1);
            hit |= __shfl_xor_sync(0xffffffffu, hit, 2);
            if (r0 + 32 > args.n_rows) hit &= (r0 < args.n_rows) ? ((1u << (uint32_t)(args.n_rows - r0)) - 1u) : 0u;
            uint64_t *seg = args.cand_keys + ((size_t)(q0 + 8 * h) * gridDim.x + blockIdx.x) * args.cand_cap;
#pragma unroll
            for (int ii = 0; ii < 4; ++ii)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const uint32_t b = ii * 8 + quad * 2 + e;
                const uint32_t pos = cnt[h] + __popc(hit & ((1u << b) - 1u));
                if (((hit >> b) & 1u) && pos < args.cand_cap) seg[pos] = stb_make_key(u[ii][h][e], (uint32_t)(r0 + b));
              }
            cnt[h] += __popc(hit);
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (quad == 0 && cnt[h] != cnt0[h]) args.cand_cnt[(size_t)(q0 + 8 * h) * gridDim.x + blockIdx.x] = cnt[h];
      } else {
        const size_t ld = (size_t)args.n_tiles * STB_B_TILE;
#pragma unroll
        for (int c = 0; c < STB_B_TILE / STB_SUB; ++c)
#pragma unroll
          for (int ii = 0; ii < 4; ++ii) {
            const uint32_t col = c * STB_SUB + ii * 8 + quad * 2;
            const float2 s2 = *reinterpret_cast<const float2 *>(sc + col);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const size_t o = (size_t)(q0 + 8 * h) * ld + row0 + col;
              const int32_t d0 = d[16 * c + 4 * ii + 2 * h], d1 = d[16 * c + 4 * ii + 2 * h + 1];
              *reinterpret_cast<int2 *>(args.dot_out + o) = make_int2(d0, d1);
              *reinterpret_cast<float2 *>(args.u_out + o) =
                  make_float2(fmaf(s2.x, fmaf((float)d0, qc[h].x, qc[h].y), qc[h].z), fmaf(s2.y, fmaf((float)d1, qc[h].x, qc[h].y), qc[h].z));
              *reinterpret_cast<float2 *>(args.l_out + o) =
                  make_float2(fmaf(s2.x, fmaf((float)d0, qc[h].x, -qc[h].y), -qc[h].z) - (float)STB_Q8_SCAN_EPS,
                              fmaf(s2.y, fmaf((float)d1, qc[h].x, -qc[h].y), -qc[h].z) - (float)STB_Q8_SCAN_EPS);
            }
          }
      }
    }
  }
}

// The q8 copy's tensor maps, encoded per launch (a map holds the buffer's address, which moves when the copy
// grows): codes as [n_rows][256] u8 in [256 rows][128 B] boxes with the 128-byte swizzle, scales as [n_rows] f32
// in 256-entry boxes.  Rows past n_rows read as zeros.  The driver's encoder is taken through the runtime, so the
// library does not link libcuda.
static int q8_tensor_maps(const uint8_t *codes, const float *scales, uint64_t n_rows, CUtensorMap *codes_map,
                          CUtensorMap *scale_map) {
  // looked up once per process (thread-safe initialisation of the local static); null if unavailable
  static const PFN_cuTensorMapEncodeTiled_v12000 encode = []() -> PFN_cuTensorMapEncodeTiled_v12000 {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    const cudaError_t e = cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &fn, 12000, cudaEnableDefault, &qr);
    if (e != cudaSuccess) cudaGetLastError();
    return (e == cudaSuccess && qr == cudaDriverEntryPointSuccess) ? reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn) : nullptr;
  }();
  if (!encode) { stb_set_error("q8 GEMM: cuTensorMapEncodeTiled unavailable"); return STB_ERR_CUDA; }
  const cuuint64_t cdim[2] = {256, n_rows}, cstride[1] = {256};
  const cuuint32_t cbox[2] = {128, STB_B_TILE}, one[2] = {1, 1};
  CUresult r = encode(codes_map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t *>(codes), cdim, cstride, cbox, one,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { stb_set_error("q8 GEMM: code tensor map (error %d)", (int)r); return STB_ERR_CUDA; }
  const cuuint64_t sdim[1] = {n_rows}, sstride[1] = {4};
  const cuuint32_t sbox[1] = {STB_B_TILE};
  r = encode(scale_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 1, const_cast<float *>(scales), sdim, sstride, sbox, one,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { stb_set_error("q8 GEMM: scale tensor map (error %d)", (int)r); return STB_ERR_CUDA; }
  return STB_OK;
}

template <int EPI>
static int launch_q8_gemm(stb_ctx *ctx, const uint8_t *codes, const float *scales, const Q8GemmArgs &a) {
  if (a.n_rows == 0 || a.n_rows > 0x7fffff00ull) { stb_set_error("q8 GEMM: %llu rows", (unsigned long long)a.n_rows); return STB_ERR_ARG; }
  CUtensorMap cm, sm;
  int rc = q8_tensor_maps(codes, scales, a.n_rows, &cm, &sm);
  if (rc != STB_OK) return rc;
  STB_ATTR_ONCE(ctx, EPI == 0 ? STB_ATTR_Q8GEMM0 : (EPI == 1 ? STB_ATTR_Q8GEMM1 : STB_ATTR_Q8GEMM2),
                cudaFuncSetAttribute(stb_batch_q8_gemm_kernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, STB_Q8_GEMM_SMEM));
  const unsigned grid = (unsigned)std::min<uint32_t>(a.n_tiles, (uint32_t)ctx->sm_count);   // = stb_batch_emit_grid
  if (grid == 0) return STB_OK;
  stb_batch_q8_gemm_kernel<EPI><<<grid, STB_GEMM_THREADS, STB_Q8_GEMM_SMEM, ctx->stream>>>(cm, sm, a);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

int stb_launch_batch_q8_gemm_sample(stb_ctx *ctx, const uint8_t *a_tiles, const float4 *qc, uint32_t m_tiles,
                                    const uint8_t *codes, const float *scales, uint64_t n_rows, uint32_t n_sample,
                                    uint32_t tile_stride, float *tilemax) {
  Q8GemmArgs a{};
  a.a_tiles = a_tiles; a.qc = qc; a.m_tiles = m_tiles; a.n_tiles = n_sample; a.tile_stride = tile_stride;
  a.n_rows = n_rows; a.tilemax = tilemax;
  return launch_q8_gemm<0>(ctx, codes, scales, a);
}

int stb_launch_batch_q8_gemm_emit(stb_ctx *ctx, const uint8_t *a_tiles, const float4 *qc, uint32_t m_tiles,
                                  const uint8_t *codes, const float *scales, uint64_t n_rows, const float *thr,
                                  uint32_t *cand_cnt, uint64_t *cand_keys, uint32_t cand_cap) {
  Q8GemmArgs a{};
  a.a_tiles = a_tiles; a.qc = qc; a.m_tiles = m_tiles; a.n_tiles = (uint32_t)((n_rows + STB_B_TILE - 1) / STB_B_TILE);
  a.tile_stride = 1; a.n_rows = n_rows; a.thr = thr; a.cand_cnt = cand_cnt; a.cand_keys = cand_keys; a.cand_cap = cand_cap;
  return launch_q8_gemm<1>(ctx, codes, scales, a);
}

int stb_launch_batch_q8_gemm_debug(stb_ctx *ctx, const uint8_t *a_tiles, const float4 *qc, uint32_t m_tiles,
                                   const uint8_t *codes, const float *scales, uint64_t n_rows, int32_t *dot, float *u,
                                   float *l) {
  Q8GemmArgs a{};
  a.a_tiles = a_tiles; a.qc = qc; a.m_tiles = m_tiles; a.n_tiles = (uint32_t)((n_rows + STB_B_TILE - 1) / STB_B_TILE);
  a.tile_stride = 1; a.n_rows = n_rows; a.dot_out = dot; a.u_out = u; a.l_out = l;
  return launch_q8_gemm<2>(ctx, codes, scales, a);
}

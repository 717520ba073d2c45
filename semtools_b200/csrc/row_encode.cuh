// Per-row encodings of the reduced-width corpus copies, shared by the builders (stb_q8_build_kernel,
// stb_shadow_build_kernel) and the in-place corpus mutations (corpus_update.cu), so a row re-encoded
// after an update or a move is byte for byte the row a fresh build writes.  One warp per row; lane l
// holds elements 8l .. 8l+7 of the f32 row in v0, v1.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstring>

#include "common.cuh"

// Nibble plane layout: 32-row tiles of 4096 B.  Chunk m (m < 8, 16 B: components 32m .. 32m+31) of row r
// sits at (r / 32) * 4096 + m * 512 + (r % 32) * 16, so one lane per row reading chunk m of a tile makes
// one 512-byte contiguous warp load (stb_scan_q4).  A plane of n rows takes ceil(n / 32) whole tiles.
#define STB_Q4_TILE_ROWS 32
__host__ __device__ __forceinline__ size_t stb_q4_plane_offset(uint64_t row, int m) {
  return (size_t)(row >> 5) * 4096 + (size_t)m * 512 + (size_t)((uint32_t)row & 31u) * 16;
}
__host__ __device__ __forceinline__ size_t stb_q4_plane_bytes(uint64_t rows) { return (size_t)((rows + 31) >> 5) * 4096; }

// rows [first, first + n) in row order (128 B each) from `tiles`, a copy of the plane's tiles from tile
// first / 32 on (stb_debug_corpus_copy)
inline void stb_q4_plane_gather(const uint8_t *tiles, uint64_t first, uint64_t n, uint8_t *out) {
  const size_t base = stb_q4_plane_offset(first & ~(uint64_t)31, 0);
  for (uint64_t i = 0; i < n; ++i)
    for (int m = 0; m < 8; ++m) memcpy(out + i * 128 + m * 16, tiles + (stb_q4_plane_offset(first + i, m) - base), 16);
}

// q8 tier entry of one row: int8 codes, scale, nibble plane and {s, rho} (scan_topk.cu: stb_scan_q8,
// stb_scan_q4).  Rows whose fp32 squared norm is not a normal number set *bad_flag (the tier is then
// refused for this corpus, like the 16-bit shadow); true zero rows get scale 0 and all-zero codes.
__device__ __forceinline__ void stb_q8_encode_row(float4 v0, float4 v1, int lane, uint64_t row, uint8_t *__restrict__ out,
                                                  float *__restrict__ scale, uint8_t *__restrict__ plane,
                                                  float2 *__restrict__ sr, int *bad_flag) {
  float ss = v0.x * v0.x + v0.y * v0.y + v0.z * v0.z + v0.w * v0.w + v1.x * v1.x + v1.y * v1.y + v1.z * v1.z + v1.w * v1.w;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
  float inv = 0.f;
  if (ss != 0.f) {
    if (!(ss >= 1e-30f && ss <= 1e30f)) { if (lane == 0) atomicExch(bad_flag, 1); }   // NaN/inf/extreme
    else inv = rsqrtf(ss);
  } else {
    const bool nz = (v0.x != 0.f) | (v0.y != 0.f) | (v0.z != 0.f) | (v0.w != 0.f) | (v1.x != 0.f) | (v1.y != 0.f) |
                    (v1.z != 0.f) | (v1.w != 0.f);
    if (__any_sync(0xffffffffu, nz) && lane == 0) atomicExch(bad_flag, 1);             // underflowed tiny row
  }
  const float x[8] = {v0.x * inv, v0.y * inv, v0.z * inv, v0.w * inv, v1.x * inv, v1.y * inv, v1.z * inv, v1.w * inv};
  float am = 0.f;
#pragma unroll
  for (int e = 0; e < 8; ++e) am = fmaxf(am, fabsf(x[e]));
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, off));
  const float s = am * (1.0f / 127.0f);
  const float inv_s = am > 0.f ? 127.0f / am : 0.f;
  uint32_t w0 = 0, w1 = 0, n0 = 0, n1 = 0;
  float r2 = 0.f;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int c0 = max(-127, min(127, __float2int_rn(x[e] * inv_s)));
    const int c1 = max(-127, min(127, __float2int_rn(x[4 + e] * inv_s)));
    w0 |= (uint32_t)(c0 & 255) << (8 * e);
    w1 |= (uint32_t)(c1 & 255) << (8 * e);
    const int h0 = (c0 + 128) >> 4, h1 = (c1 + 128) >> 4;      // h + 8 in [0, 15]
    n0 |= (uint32_t)h0 << (8 * e);
    n1 |= (uint32_t)h1 << (8 * e);
    // x^ - s (16 h + 7.5) with h = h0 - 8: the centre 16 h0 - 120.5 = (32 h0 - 241) / 2 is exact in fp32
    const float d0 = x[e] - s * (0.5f * (float)(32 * h0 - 241));
    const float d1 = x[4 + e] - s * (0.5f * (float)(32 * h1 - 241));
    r2 = fmaf(d0, d0, fmaf(d1, d1, r2));
  }
  *reinterpret_cast<uint2 *>(out + row * 256 + (size_t)lane * 8) = make_uint2(w0, w1);
  // plane: lane 4m + t holds components 32m + 8t .. +7; t < 2 are the low nibbles of bytes 8t .. of chunk m,
  // t >= 2 the high nibbles of the same bytes (from lane + 2)
  const uint32_t p0 = __shfl_down_sync(0xffffffffu, n0, 2), p1 = __shfl_down_sync(0xffffffffu, n1, 2);
  if ((lane & 2) == 0)
    *reinterpret_cast<uint2 *>(plane + stb_q4_plane_offset(row, lane >> 2) + (size_t)(lane & 1) * 8) = make_uint2(n0 | (p0 << 4), n1 | (p1 << 4));
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) r2 += __shfl_xor_sync(0xffffffffu, r2, off);
  if (lane == 0) {
    scale[row] = s;
    // rounded up: 1e-4 relative covers the fp32 evaluation of the 256 differences and their sum
    sr[row] = make_float2(s, sqrtf(r2) * 1.0001f + 1e-6f);
  }
}

// 16-bit shadow entry of one row: lane l's 16-byte chunk of the L2-normalised row (slab l/8, chunk l%8).
// A row that cannot be normalised in fp32 sets *bad_flag and is scaled by 0 (NaN where a component is NaN or
// infinite).  row_bad (may be null; query tiles): per-row record of the same, 1 or 0 at row_bad[row].
__device__ __forceinline__ uint4 stb_shadow_pack_row(float4 v0, float4 v1, int lane, uint64_t row, int *bad_flag,
                                                     uint32_t *row_bad) {
  float ss = v0.x * v0.x + v0.y * v0.y + v0.z * v0.z + v0.w * v0.w + v1.x * v1.x + v1.y * v1.y +
             v1.z * v1.z + v1.w * v1.w;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
  float inv = 0.f;
  bool bad = false;
  if (ss != 0.f) {
    if (!(ss >= 1e-30f && ss <= 1e30f)) bad = true;   // NaN/inf/extreme
    else inv = rsqrtf(ss);
  } else {
    // fp32 underflow of a tiny non-zero row: cannot be normalised here -> batch path unusable
    bool nz = (v0.x != 0.f) | (v0.y != 0.f) | (v0.z != 0.f) | (v0.w != 0.f) | (v1.x != 0.f) | (v1.y != 0.f) |
              (v1.z != 0.f) | (v1.w != 0.f);
    bad = __any_sync(0xffffffffu, nz);
  }
  if (bad && lane == 0) atomicExch(bad_flag, 1);
  if (row_bad && lane == 0) row_bad[row] = bad ? 1u : 0u;
#if STB_SHADOW_F16
  __half2 p0 = __floats2half2_rn(v0.x * inv, v0.y * inv);
  __half2 p1 = __floats2half2_rn(v0.z * inv, v0.w * inv);
  __half2 p2 = __floats2half2_rn(v1.x * inv, v1.y * inv);
  __half2 p3 = __floats2half2_rn(v1.z * inv, v1.w * inv);
#else
  __nv_bfloat162 p0 = __floats2bfloat162_rn(v0.x * inv, v0.y * inv);
  __nv_bfloat162 p1 = __floats2bfloat162_rn(v0.z * inv, v0.w * inv);
  __nv_bfloat162 p2 = __floats2bfloat162_rn(v1.x * inv, v1.y * inv);
  __nv_bfloat162 p3 = __floats2bfloat162_rn(v1.z * inv, v1.w * inv);
#endif
  uint4 pk;
  pk.x = *reinterpret_cast<uint32_t *>(&p0); pk.y = *reinterpret_cast<uint32_t *>(&p1);
  pk.z = *reinterpret_cast<uint32_t *>(&p2); pk.w = *reinterpret_cast<uint32_t *>(&p3);
  return pk;
}

// Byte offset of lane l's chunk of `row` in the shadow.  Tile layout: tile t -> 4 slabs -> [TILE rows x 128 B],
// 8-row x 128-B atoms with the 16-byte chunk index XOR-ed by (row % 8)  (the hardware 128B swizzle).
template <int TILE>
__device__ __forceinline__ size_t stb_shadow_offset(uint64_t row, int lane) {
  const uint64_t tile = row / TILE;
  const uint32_t r = (uint32_t)(row % TILE);
  const uint32_t slab = lane >> 3, chunk = lane & 7;
  return tile * (size_t)(TILE * 512) + (size_t)slab * (TILE * 128) + (size_t)(r >> 3) * 1024 +
         (size_t)(r & 7) * 128 + (size_t)((chunk ^ (r & 7)) * 16);
}

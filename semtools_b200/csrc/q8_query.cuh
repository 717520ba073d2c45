// The query as K1's q8 scan and K2's q8 route see it: the fp32 normalisation of a query and its 16-bit
// quantisation, split into a high and a low signed byte (scan_topk.cu: stb_scan_q8 derives the bounds built on
// it).  Both kernels call these, so a query's words, scale and error terms are the same bits in both.
#pragma once

#include "common.cuh"

// fixed-order ||q||^2 of a lane's 8 float4 + 8-lane group reduction; classifies the query
struct StbQueryNorm { float rq; bool q_zero, q_bad; };
__device__ __forceinline__ StbQueryNorm stb_query_norm(const float4 (&q)[8]) {
  float qx = 0.f, qy = 0.f, qz = 0.f, qw = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    qx = fmaf(q[i].x, q[i].x, qx); qy = fmaf(q[i].y, q[i].y, qy);
    qz = fmaf(q[i].z, q[i].z, qz); qw = fmaf(q[i].w, q[i].w, qw);
  }
  float b2 = (qx + qy) + (qz + qw);
  b2 += __shfl_xor_sync(0xffffffffu, b2, 4);
  b2 += __shfl_xor_sync(0xffffffffu, b2, 2);
  b2 += __shfl_xor_sync(0xffffffffu, b2, 1);
  // b2 == 0 in fp32 is either a true zero vector or an underflowed tiny one
  bool q_any = false;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    q_any |= (q[i].x != 0.f) | (q[i].y != 0.f) | (q[i].z != 0.f) | (q[i].w != 0.f);
  q_any = __any_sync(0xffffffffu, q_any);   // all four groups hold the same query
  StbQueryNorm r;
  r.q_zero = (b2 == 0.f) && !q_any;
  r.q_bad = !r.q_zero && !(b2 >= 1e-30f && b2 <= 1e30f);  // NaN/inf/denormal/underflow
  r.rq = r.q_zero ? 0.f : rsqrtf(b2);
  return r;
}

// q16 of four query components (scaled by qs), split into a high and a low signed byte word
__device__ __forceinline__ void stb_q16_words(float4 q, float qs, bool unusable, uint32_t &hw, uint32_t &lw, int &l1, int &sum) {
  const float f[4] = {q.x, q.y, q.z, q.w};
  hw = 0; lw = 0;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    int v = unusable ? 0 : __float2int_rn(f[e] * qs);
    v = max(-32639, min(32639, v));
    l1 += abs(v);
    sum += v;
    const int lo = ((v + 128) & 255) - 128;               // signed low byte
    const int hi = (v - lo) >> 8;                         // exact: v - lo is a multiple of 256
    hw |= (uint32_t)(hi & 255) << (8 * e);
    lw |= (uint32_t)(lo & 255) << (8 * e);
  }
}

// The query as the q8 tier sees it (see stb_scan_q8); lane j holds the components of row bytes
// [16j, 16j+16) and [128+16j, 128+16j+16).
struct StbQ8Query {
  uint32_t qhi[8], qlo[8];
  float S, qs, inv_S, h_l1, e_q;
  bool unusable;
};
__device__ __forceinline__ StbQ8Query stb_q8_query(const float *qf, int j) {
  StbQ8Query Q;
  float4 q[8];
  const float4 *q4 = reinterpret_cast<const float4 *>(qf);
#pragma unroll
  for (int i = 0; i < 4; ++i) { q[i] = __ldg(q4 + 4 * j + i); q[4 + i] = __ldg(q4 + 32 + 4 * j + i); }
  const StbQueryNorm qn = stb_query_norm(q);
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(q[i].x), fabsf(q[i].y)), fmaxf(fabsf(q[i].z), fabsf(q[i].w))));
  }
  amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
  amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
  amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
  amax *= qn.rq;                                            // max |q^_i|
  Q.unusable = qn.q_zero || qn.q_bad || !(amax > 0.f && amax <= 1.0001f);
  Q.S = Q.unusable ? 1.f : 32639.0f / amax;
  Q.qs = qn.rq * Q.S;
  int l1 = 0, sum = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) stb_q16_words(q[i], Q.qs, Q.unusable, Q.qhi[i], Q.qlo[i], l1, sum);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 4);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  Q.inv_S = 1.0f / Q.S;
  Q.h_l1 = 0.50025f * (float)l1 * Q.inv_S;                  // (0.5 + 3e-5 + fp slack) * ||q~||_1
  Q.e_q = 9.7f * Q.inv_S;
  return Q;
}

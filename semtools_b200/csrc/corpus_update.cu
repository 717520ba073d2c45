// In-place corpus mutations (stb_corpus_update, stb_corpus_remove; host side in api.cu).
//
// Both write f32 rows from a bounded device staging buffer and re-encode the reduced-width copies at the
// rows they write, with the builders' own per-row encodings (row_encode.cuh), so every copy keeps covering a
// prefix of the rows and that prefix stays byte for byte what a fresh build writes.
//   stb_corpus_write_kernel   staging row i -> rows[dst_i] (+ q8 codes / scale / plane / {s, rho} when
//                             dst_i < q8_rows, + the 16-bit shadow entry when dst_i < shadow_rows);
//                             dst_i = idx[i] (update) or first + i (a chunk of a removal's moved tail)
//   stb_corpus_gather_kernel  output row first + i of a removal -> staging row i, its source found by a
//                             binary search of the kept-segment table
// One warp per row; lane l holds elements 8l .. 8l+7.
#include "common.cuh"
#include "row_encode.cuh"

__global__ void __launch_bounds__(256) stb_corpus_write_kernel(StbCorpusWriteArgs a) {
  const int lane = threadIdx.x & 31;
  const uint64_t i = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= a.m) return;
  const uint64_t row = a.idx ? a.idx[i] : a.first + i;
  const float4 v0 = a.stage[i * STB_ROW_F4 + 2 * lane];
  const float4 v1 = a.stage[i * STB_ROW_F4 + 2 * lane + 1];
  a.rows[row * STB_ROW_F4 + 2 * lane] = v0;
  a.rows[row * STB_ROW_F4 + 2 * lane + 1] = v1;
  if (row < a.q8_rows) stb_q8_encode_row(v0, v1, lane, row, a.q8, a.q8_scale, a.q4, a.q4_sr, a.flags);
  if (row < a.shadow_rows) {
    const uint4 pk = stb_shadow_pack_row(v0, v1, lane, row, a.flags + 1, nullptr);
    *reinterpret_cast<uint4 *>(a.shadow + stb_shadow_offset<256>(row, lane)) = pk;
  }
}

// seg: n_seg {dst, src} pairs, dst ascending, seg[0].dst <= first: output row d is row src + (d - dst) of
// the last pair with dst <= d.
__global__ void __launch_bounds__(256)
stb_corpus_gather_kernel(const float4 *__restrict__ rows, const uint64_t *__restrict__ seg, uint32_t n_seg,
                         uint64_t first, uint64_t m, float4 *__restrict__ stage) {
  const int lane = threadIdx.x & 31;
  const uint64_t i = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= m) return;
  const uint64_t d = first + i;
  uint32_t lo = 0, hi = n_seg;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(seg + 2 * mid) <= d) lo = mid;
    else hi = mid;
  }
  const uint64_t src = __ldg(seg + 2 * lo + 1) + (d - __ldg(seg + 2 * lo));
  stage[i * STB_ROW_F4 + 2 * lane] = __ldg(rows + src * STB_ROW_F4 + 2 * lane);
  stage[i * STB_ROW_F4 + 2 * lane + 1] = __ldg(rows + src * STB_ROW_F4 + 2 * lane + 1);
}

// Plain launches (no programmatic stream serialisation): an overlapped scan still reading the rows these
// kernels overwrite finishes before they start.
int stb_launch_corpus_write(stb_ctx *ctx, const StbCorpusWriteArgs &a) {
  if (a.m == 0) return STB_OK;
  stb_corpus_write_kernel<<<(unsigned)((a.m + 7) / 8), 256, 0, ctx->stream>>>(a);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

int stb_launch_corpus_gather(stb_ctx *ctx, const float *rows, const uint64_t *seg_dev, uint32_t n_seg, uint64_t first,
                             uint64_t m, float *stage) {
  if (m == 0) return STB_OK;
  stb_corpus_gather_kernel<<<(unsigned)((m + 7) / 8), 256, 0, ctx->stream>>>(
      reinterpret_cast<const float4 *>(rows), seg_dev, n_seg, first, m, reinterpret_cast<float4 *>(stage));
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// K1 (+ in-kernel K4): cosine scan with running top-K', tree merge, exact re-rank.
//
// Replaces the loop/sort/take of search_documents (reference
// src/search/mod.rs:84-119; one simsimd f32::cosine per line at :86) and the
// filtered nearest query of Store::search_line_embeddings
// (src/workspace/store.rs:495-543).
//
// HBM-bound: the only large traffic is the corpus matrix, 1 KiB per row, read
// exactly once with 128-bit coalesced loads (8 lanes cover one 128-byte line of a
// row; a warp instruction touches 4 full lines).  Everything else (query, K'
// candidates per CTA, k results) is bytes.  The narrower candidate tiers read less: the 16-bit
// shadow 512 B per row; the q8 tier's top-k scan a 136 B/row 4-bit plane, plus the 260 B int8 codes
// of the few rows whose 4-bit bound can still reach the k-th best (stb_scan_q4).
//
// Exactness: the streaming pass ranks rows by an fp32 approximate cosine and keeps
// the best K' = 32*E per warp; the surviving K' of the whole grid are re-scored by
// one thread each in the oracle's canonical arithmetic (f64 accumulation in index
// order) and sorted by (distance,row).  The result is accepted only if the worst
// kept approximate score proves that no dropped row can reach the k-th exact
// distance (STB_SCORE_EPS); otherwise status[1]=0 and the host runs the collect
// path below, which is exact for any input.
#include <math_constants.h>

#include <cuda_fp16.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "row_encode.cuh"
#include "q8_query.cuh"

#define STB_SCAN_U 2   // rows per 8-lane group per iteration (loads in flight = 8*U float4)

// streamed once: read through the non-coherent path without allocating in L1
__device__ __forceinline__ float4 stb_ld_stream(const float4 *p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

struct ScanArgs {
  const float4 *rows;        // local row 0
  uint64_t n_virtual;        // rows to scan (== n_rows when no ranges)
  const float *q;            // 256 f32 (device)
  const uint64_t *vstart;    // [n_ranges+1] virtual prefix (ranges mode)
  const uint64_t *rbegin;    // [n_ranges]   local first row of each range
  uint32_t n_ranges;
  // dynamic tile schedule, always used by the top-k kernel; null in the collect and histogram
  // kernels, which keep the static warp-strided schedule:
  unsigned long long *tickets;   // monotonic counter shared by every launch of the context
  unsigned long long t_base;     // its value when this launch starts (host-tracked)
  uint64_t t_bulk;               // tickets [0, t_bulk) cover STB_TICKET_TILES tiles each, later ones one tile
};

// A pass's ScanArgs over row ranges as k1_upload_ranges (api.cu) packs them: vstart[r.n + 1], then rbegin[r.n];
// the only decoder of that layout.  No tickets: the top-k launch sets its own.
static ScanArgs stb_scan_args(const stb_corpus *c, const float *q_dev, const StbRowRanges &r) {
  ScanArgs a;
  a.rows = reinterpret_cast<const float4 *>(c->rows);
  a.n_virtual = r.n_virtual;
  a.q = q_dev;
  a.vstart = r.dev;
  a.rbegin = r.dev ? r.dev + (r.n + 1) : nullptr;
  a.n_ranges = r.n;
  a.tickets = nullptr; a.t_base = 0; a.t_bulk = 0;
  return a;
}

// Grid of the static warp-strided schedule over n_virtual rows, 4 * u rows per tile: one tile per warp, at most
// STB_SCAN_MINB CTAs per SM.
static unsigned stb_scan_grid(const stb_ctx *ctx, uint64_t n_virtual, int u) {
  const uint64_t tiles = (n_virtual + 4 * u - 1) / (4 * u);
  const uint64_t want = (tiles + STB_SCAN_WARPS - 1) / STB_SCAN_WARPS;
  const uint64_t grid = (uint64_t)ctx->sm_count * STB_SCAN_MINB;
  return (unsigned)(want < grid ? (want < 1 ? 1 : want) : grid);
}

// ---- tile schedule + row map shared by the three scans -----------------------------------
// RANGES == 0: whole shard, tiles are warp-strided (the grid streams one contiguous window).
// RANGES == 1: row ranges (workspace path filter).  Blocks of WB consecutive tiles are
// warp-strided and a warp walks each block in order, so the virtual->local row map costs one
// binary search per block per lane and a forward step per row afterwards (the per-row
// 15-step search of round 1 held this mode at 0.52 of the HBM peak).
// Dynamic schedule (args.tickets != null): warps draw tickets from one atomic counter; a ticket is
// STB_TICKET_TILES consecutive tiles, except that the last ~2 tiles per warp are handed out one
// by one so the grid drains evenly.  Tickets are issued in row order, so the grid still streams
// one contiguous window.  Why: the grid fills every CTA slot, and with a static partition a CTA
// that starts late finishes late -- under PDL the next query's last CTA cannot start before this
// query's final (merge) CTA exits, which exposed the whole tail (10 us at K'=32, 77 us at
// K'=128) on every pipelined query.  With tickets a late CTA simply finds less work.
// Every warp makes exactly one failing draw, so a launch advances the counter by
// n_tickets + total_warps -- the host tracks the base of the next launch with that.
// Co-scan (RANGES == 0 only): the tickets count virtual tiles v, and the warp scores tile (v + off) mod
// n_tiles, so the pass starts at tile off and wraps around the end
// (stb_coscan_offset).  Which warp scores which row does not change the
// lists, the drop bounds or the proof, so any offset gives the same result.
// The tiles of ticket t in pass order: with RANGES == 0 shifted by the co-scan offset *off and wrapped at n_tiles.
template <int RANGES, class Body>
__device__ __forceinline__ void stb_ticket_walk(const ScanArgs &args, uint64_t t, uint64_t n_tiles, const uint32_t *off, Body &&body) {
  const uint64_t t0 = stb_ticket_first_tile(t, args.t_bulk);
  const uint64_t t1 = t < args.t_bulk ? t0 + STB_TICKET_TILES : t0 + 1;
  if constexpr (RANGES == 0) {
    // *off: a shared word, read per ticket so that it holds no register across the scoring
    uint32_t tile = (uint32_t)t0 + *reinterpret_cast<const volatile uint32_t *>(off);   // off < n_tiles < 2^32
    if (tile >= n_tiles) tile -= (uint32_t)n_tiles;
    for (uint32_t left = (uint32_t)(t1 - t0); left; --left) {
      body(tile, false);
      if (++tile == n_tiles) tile = 0;
    }
  } else {
    for (uint64_t tile = t0; tile < t1; ++tile) body(tile, tile == t0);
  }
}

template <int RANGES, int WB, class Body>
__device__ __forceinline__ void stb_for_each_tile(const ScanArgs &args, uint64_t n_tiles, const uint32_t *off, Body &&body) {
  if (args.tickets) {
    // The next ticket is drawn BEFORE the current one is processed, so the atomic's L2 round trip
    // (~1 us under load) overlaps a ticket's worth of loads instead of stalling the warp 4-6 times per
    // query (at 1.25M rows per GPU that was ~10 % of the scan).  A warp stops drawing at its first
    // failing draw, so the "exactly one failing draw per warp" bookkeeping holds.
    const int lane = threadIdx.x & 31;
    auto draw = [&]() -> unsigned long long {
      unsigned long long t = 0;
      if (lane == 0) t = atomicAdd(args.tickets, 1ull);
      return __shfl_sync(0xffffffffu, t, 0) - args.t_base;
    };
    unsigned long long cur = draw();
    while (stb_ticket_first_tile(cur, args.t_bulk) < n_tiles) {
      const unsigned long long nxt = draw();
      stb_ticket_walk<RANGES>(args, cur, n_tiles, off, body);
      cur = nxt;
    }
    return;
  }
  const uint64_t warps_total = (uint64_t)gridDim.x * (blockDim.x >> 5);
  const uint64_t warp_id = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if constexpr (RANGES == 0) {
    for (uint64_t tile = warp_id; tile < n_tiles; tile += warps_total) body(tile, false);
  } else {
    const uint64_t n_blocks = (n_tiles + WB - 1) / WB;
    for (uint64_t blk = warp_id; blk < n_blocks; blk += warps_total) {
      const uint64_t t0 = blk * WB;
      const uint64_t t1 = t0 + WB < n_tiles ? t0 + WB : n_tiles;
      for (uint64_t tile = t0; tile < t1; ++tile) body(tile, tile == t0);
    }
  }
}

template <int RANGES>
struct StbRowMap {
  uint32_t rlo;
  bool fresh;
  __device__ __forceinline__ void restart() { fresh = true; }
  // virtual row -> local row: largest idx with vstart[idx] <= v.  A lane's virtual rows only
  // grow inside a block: search once, then step to the next range(s).
  __device__ __forceinline__ uint32_t map(const ScanArgs &a, uint64_t v) {
    if constexpr (RANGES == 0) return (uint32_t)v;
    else {
      if (fresh) {
        uint32_t lo = 0, hi = a.n_ranges;
        while (hi - lo > 1) {
          const uint32_t mid = (lo + hi) >> 1;
          if (__ldg(a.vstart + mid) <= v) lo = mid; else hi = mid;
        }
        rlo = lo;
        fresh = false;
      } else {
        while (rlo + 1 < a.n_ranges && __ldg(a.vstart + rlo + 1) <= v) ++rlo;
      }
      return (uint32_t)(__ldg(a.rbegin + rlo) + (v - __ldg(a.vstart + rlo)));
    }
  }
};

// Approximate-cosine scan over the f32 rows.  Calls sink(score, local_row) once per 4*U-row
// tile with a warp-uniform control flow; lanes that do not represent a row pass -inf.
template <int U, int RANGES, class Sink>
__device__ __forceinline__ void stb_scan_rows(const ScanArgs &args, Sink &sink, const uint32_t *off = nullptr) {
  const int lane = threadIdx.x & 31;
  const int g = lane >> 3;   // row group inside the warp
  const int j = lane & 7;    // 16-byte column slot inside the group
  // query slice of this lane: float4 index j + 8*i
  float4 q[8];
  const float4 *q4 = reinterpret_cast<const float4 *>(args.q);
#pragma unroll
  for (int i = 0; i < 8; ++i) q[i] = __ldg(q4 + j + 8 * i);
  const StbQueryNorm qn = stb_query_norm(q);
  const bool q_zero = qn.q_zero, q_bad = qn.q_bad;
  const float rq = qn.rq;

  constexpr uint64_t tile_rows = 4 * U;
  const uint64_t n_tiles = (args.n_virtual + tile_rows - 1) / tile_rows;
  StbRowMap<RANGES> rmap;
  rmap.restart();
  stb_for_each_tile<RANGES, 64 / (4 * U)>(args, n_tiles, off, [&](uint64_t tile, bool first) {
    if (first) rmap.restart();
    float4 a[U][8];
    uint32_t row[U];
    bool valid[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      uint64_t v = tile * tile_rows + (uint64_t)(u * 4 + g);
      valid[u] = v < args.n_virtual;
      uint64_t vc = valid[u] ? v : (args.n_virtual - 1);
      row[u] = rmap.map(args, vc);
      const float4 *p = args.rows + (size_t)row[u] * STB_ROW_F4 + j;
#pragma unroll
      for (int i = 0; i < 8; ++i) a[u][i] = stb_ld_stream(p + 8 * i);
    }
    float sc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float dx = 0.f, dy = 0.f, dz = 0.f, dw = 0.f;
      float nx = 0.f, ny = 0.f, nz = 0.f, nw = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        dx = fmaf(a[u][i].x, q[i].x, dx); dy = fmaf(a[u][i].y, q[i].y, dy);
        dz = fmaf(a[u][i].z, q[i].z, dz); dw = fmaf(a[u][i].w, q[i].w, dw);
        nx = fmaf(a[u][i].x, a[u][i].x, nx); ny = fmaf(a[u][i].y, a[u][i].y, ny);
        nz = fmaf(a[u][i].z, a[u][i].z, nz); nw = fmaf(a[u][i].w, a[u][i].w, nw);
      }
      float ab = (dx + dy) + (dz + dw);
      float a2 = (nx + ny) + (nz + nw);
      ab += __shfl_xor_sync(0xffffffffu, ab, 4);
      a2 += __shfl_xor_sync(0xffffffffu, a2, 4);
      ab += __shfl_xor_sync(0xffffffffu, ab, 2);
      a2 += __shfl_xor_sync(0xffffffffu, a2, 2);
      ab += __shfl_xor_sync(0xffffffffu, ab, 1);
      a2 += __shfl_xor_sync(0xffffffffu, a2, 1);
      float s;
      if (a2 == 0.f) {
        // rare: a true zero row (simsimd rules: d = 0 vs a zero query, else d = 1) or a
        // row so small that its fp32 squared norm underflowed -> forced candidate.
        // All 8 lanes of the group hold the same a2, so the group votes together.
        bool nz = false;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          nz |= (a[u][i].x != 0.f) | (a[u][i].y != 0.f) | (a[u][i].z != 0.f) | (a[u][i].w != 0.f);
        nz = __any_sync(0xffu << (8 * g), nz);
        s = nz ? CUDART_INF_F : (q_zero ? 1.f : 0.f);
      } else if (q_bad || !(a2 >= 1e-30f && a2 <= 1e30f)) s = CUDART_INF_F;  // forced candidate
      else s = ab * rsqrtf(a2) * rq;
      sc[u] = valid[u] ? s : -CUDART_INF_F;
    }
    float s = -CUDART_INF_F;
    uint32_t r = 0;
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (j == u) { s = sc[u]; r = row[u]; }
    sink.template consume<4 * U>(s, r);
  });
}

// Half-width scan (tier "h16"): the same running top-K' selection, but the scores come from the
// 16-bit L2-normalised shadow that K2 uses (512 B per row instead of 1 KiB), so the HBM-bound
// pass moves half the bytes.  The exact f64 re-rank and the completeness proof are unchanged
// except for the margin (STB_SHADOW_SCAN_EPS: only the row is rounded, the query stays f32).
// Shadow layout (batch_scan.cu): tile t = row / 256 -> 4 K-slabs x [256 rows x 128 B],
// 16-byte chunk index XOR (row % 8).  Lane j of a row's 8-lane group reads PHYSICAL chunk
// j ^ (row % 8) of every slab, i.e. LOGICAL chunk j = elements s*64 + 8j .. +8 (s = 0..3), so
// each lane pairs a fixed 32-element slice of the query with every row; the group still
// covers each 128-byte line completely.
__device__ __forceinline__ float2 stb_shadow_pair(uint32_t w) {
#if STB_SHADOW_F16
  return __half22float2(*reinterpret_cast<const __half2 *>(&w));
#else
  return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
#endif
}

template <int U, int RANGES, class Sink>
__device__ __forceinline__ void stb_scan_shadow(const ScanArgs &args, const uint8_t *shadow, Sink &sink, const uint32_t *off = nullptr) {
  const int lane = threadIdx.x & 31;
  const int g = lane >> 3;   // row group inside the warp
  const int j = lane & 7;    // logical 16-byte chunk of every K-slab
  // query slice: elements s*64 + 8j + e  (s < 4, e < 8) = float4 index s*16 + 2j + {0,1}
  float4 q[8];
  const float4 *q4 = reinterpret_cast<const float4 *>(args.q);
#pragma unroll
  for (int sl = 0; sl < 4; ++sl) { q[2 * sl] = __ldg(q4 + sl * 16 + 2 * j); q[2 * sl + 1] = __ldg(q4 + sl * 16 + 2 * j + 1); }
  const StbQueryNorm qn = stb_query_norm(q);
  const bool q_bad = qn.q_bad;
  const float rq = qn.rq;

  constexpr uint64_t tile_rows = 4 * U;
  const uint64_t n_tiles = (args.n_virtual + tile_rows - 1) / tile_rows;
  StbRowMap<RANGES> rmap;
  rmap.restart();
  stb_for_each_tile<RANGES, 64 / (4 * U)>(args, n_tiles, off, [&](uint64_t tile, bool first) {
    if (first) rmap.restart();
    uint4 a[U][4];
    uint32_t row[U];
    bool valid[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint64_t v = tile * tile_rows + (uint64_t)(u * 4 + g);
      valid[u] = v < args.n_virtual;
      const uint64_t vc = valid[u] ? v : (args.n_virtual - 1);
      row[u] = rmap.map(args, vc);
      const uint32_t rr = row[u] & 255u;
      const uint8_t *p = shadow + (size_t)(row[u] >> 8) * (size_t)(256 * 512) + (size_t)(rr >> 3) * 1024 + (size_t)(rr & 7u) * 128 +
                         (size_t)((j ^ (int)(rr & 7u)) * 16);
#pragma unroll
      for (int sl = 0; sl < 4; ++sl) {
        const float4 t = stb_ld_stream(reinterpret_cast<const float4 *>(p + (size_t)sl * (256 * 128)));
        a[u][sl] = make_uint4(__float_as_uint(t.x), __float_as_uint(t.y), __float_as_uint(t.z), __float_as_uint(t.w));
      }
    }
    float sc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float dx = 0.f, dy = 0.f, dz = 0.f, dw = 0.f;
#pragma unroll
      for (int sl = 0; sl < 4; ++sl) {
        const float2 e0 = stb_shadow_pair(a[u][sl].x), e1 = stb_shadow_pair(a[u][sl].y);
        const float2 e2 = stb_shadow_pair(a[u][sl].z), e3 = stb_shadow_pair(a[u][sl].w);
        dx = fmaf(e0.x, q[2 * sl].x, dx); dy = fmaf(e0.y, q[2 * sl].y, dy);
        dz = fmaf(e1.x, q[2 * sl].z, dz); dw = fmaf(e1.y, q[2 * sl].w, dw);
        dx = fmaf(e2.x, q[2 * sl + 1].x, dx); dy = fmaf(e2.y, q[2 * sl + 1].y, dy);
        dz = fmaf(e3.x, q[2 * sl + 1].z, dz); dw = fmaf(e3.y, q[2 * sl + 1].w, dw);
      }
      float ab = (dx + dy) + (dz + dw);
      ab += __shfl_xor_sync(0xffffffffu, ab, 4);
      ab += __shfl_xor_sync(0xffffffffu, ab, 2);
      ab += __shfl_xor_sync(0xffffffffu, ab, 1);
      // the shadow row is already unit-norm (zero rows stay zero: score 0 = distance 1)
      const float s = q_bad ? CUDART_INF_F : ab * rq;
      sc[u] = valid[u] ? s : -CUDART_INF_F;
    }
    float s = -CUDART_INF_F;
    uint32_t r = 0;
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (j == u) { s = sc[u]; r = row[u]; }
    sink.template consume<4 * U>(s, r);
  });
}

// Quarter-width scan (tier "q8"): candidates come from an 8-bit copy of the corpus -- row x is
// L2-normalised in fp32 (x^), scaled by its own s = max|x^_i| / 127 and rounded to int8
// (stb_q8_build_kernel): 256 B + one f32 scale per row = 260 B instead of 1 KiB.  The query is
// normalised and quantised to 16 bits per component (q16 = rint(q^ * S), S = 32639 / max|q^_i|),
// split into two signed bytes (q16 = 256 * hi + lo) so the dot product is two dp4a chains,
// exact in int32 (|dot| <= 127 * 32639 * 256 < 2^31).  What the list ranks by is not the
// approximate cosine a = s * dot / S but an UPPER BOUND of the exact one:
//     |c - a| <= sum_i |q~_i| |x^_i - s x8_i|  +  sum_i |q^_i - q~_i| |x^_i|
//             <= s * (0.5 + 3e-5) * ||q16||_1 / S   +   (0.6 / S) * ||x^||_1 ,  ||x^||_1 <= 16.001
//     u = s * (dot / S + 0.50025 * ||q16||_1 / S) + 9.7 / S          >=  c - 1e-5
// (||q16||_1 is an exact integer sum).  Every row dropped from the lists has u <= u_min, hence
// exact cosine <= u_min + 1e-5: the completeness proof is the f32 one with the per-row error
// term folded into the score, so rows with a large scale are promoted instead of widening a
// global margin.  A zero or unscorable query makes every score +inf: the proof fails and the
// caller falls through to the f32 tiers.  The query's quantisation (stb_q16_words, stb_q8_query) is in
// q8_query.cuh, shared with K2's q8 route.

// int8 dot products (group-reduced, every lane of the group holds them) and scales of U rows;
// qhi / qlo: this lane's query words (StbQ8Query, or a copy in shared memory)
template <int U>
__device__ __forceinline__ void stb_q8_dots(const uint32_t *qhi, const uint32_t *qlo, const uint8_t *q8, const float *q8_scale,
                                            const uint32_t (&row)[U], int j, int (&dot)[U], float (&sc_row)[U]) {
  uint4 a[U][2];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const uint8_t *p = q8 + (size_t)row[u] * 256 + (size_t)j * 16;
    const float4 t0 = stb_ld_stream(reinterpret_cast<const float4 *>(p));
    const float4 t1 = stb_ld_stream(reinterpret_cast<const float4 *>(p + 128));
    a[u][0] = make_uint4(__float_as_uint(t0.x), __float_as_uint(t0.y), __float_as_uint(t0.z), __float_as_uint(t0.w));
    a[u][1] = make_uint4(__float_as_uint(t1.x), __float_as_uint(t1.y), __float_as_uint(t1.z), __float_as_uint(t1.w));
    sc_row[u] = __ldg(q8_scale + row[u]);                   // 8 lanes, one address
  }
#pragma unroll
  for (int u = 0; u < U; ++u) {
    int dh = 0, dl = 0;
    const uint32_t w[8] = {a[u][0].x, a[u][0].y, a[u][0].z, a[u][0].w, a[u][1].x, a[u][1].y, a[u][1].z, a[u][1].w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      dh = __dp4a((int)w[i], (int)qhi[i], dh);
      dl = __dp4a((int)w[i], (int)qlo[i], dl);
    }
    int d = dh * 256 + dl;
    d += __shfl_xor_sync(0xffffffffu, d, 4);
    d += __shfl_xor_sync(0xffffffffu, d, 2);
    d += __shfl_xor_sync(0xffffffffu, d, 1);
    dot[u] = d;
  }
}

template <int U, int RANGES, class Sink>
__device__ __forceinline__ void stb_scan_q8(const ScanArgs &args, const uint8_t *q8, const float *q8_scale, Sink &sink, const uint32_t *off = nullptr) {
  const int lane = threadIdx.x & 31;
  const int g = lane >> 3;   // row group inside the warp
  const int j = lane & 7;
  const StbQ8Query Q = stb_q8_query(args.q, j);

  constexpr uint64_t tile_rows = 4 * U;
  const uint64_t n_tiles = (args.n_virtual + tile_rows - 1) / tile_rows;
  StbRowMap<RANGES> rmap;
  rmap.restart();
  stb_for_each_tile<RANGES, 2>(args, n_tiles, off, [&](uint64_t tile, bool first) {
    if (first) rmap.restart();
    float sc_row[U];
    int dot[U];
    uint32_t row[U];
    bool valid[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint64_t v = tile * tile_rows + (uint64_t)(u * 4 + g);
      valid[u] = v < args.n_virtual;
      const uint64_t vc = valid[u] ? v : (args.n_virtual - 1);
      row[u] = rmap.map(args, vc);
    }
    stb_q8_dots<U>(Q.qhi, Q.qlo, q8, q8_scale, row, j, dot, sc_row);
    float sc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const float s = Q.unusable ? CUDART_INF_F : fmaf(sc_row[u], fmaf((float)dot[u], Q.inv_S, Q.h_l1), Q.e_q);
      sc[u] = valid[u] ? s : -CUDART_INF_F;
    }
    float s = -CUDART_INF_F;
    uint32_t r = 0;
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (j == u) { s = sc[u]; r = row[u]; }
    sink.template consume<4 * U>(s, r);
  });
}

// ---- the q8 tier's top-k scan: a 4-bit prefilter in front of the int8 codes --------------------
// Beside the int8 codes the builder keeps a nibble plane, h_i = code_i >> 4 in [-8, 7] stored as
// h_i + 8, two per byte (128 B/row), and per row {s, rho} with rho >= ||x^ - s (16 h + 7.5)||_2
// (16 h + 7.5 is the midpoint of the 16 codes a nibble stands for).  Byte r of a row's chunk m
// (m < 8, r < 16) holds component 32m + r in its low nibble and 32m + 16 + r in its high nibble,
// so w & 0x0F0F0F0F and w & 0xF0F0F0F0 (16x the high nibbles) each line up with one query word;
// the chunks of 32 consecutive rows are stored together (row_encode.cuh: stb_q4_plane_offset) and
// one lane scores one row.  With the query quantised exactly as
// in stb_scan_q8 (q~ = q16 / S, |q^_i - q~_i| <= 0.6 / S):
//     c  <=  q^ . x~ + rho  <=  s (16 q~ . h + 7.5 sum q~) + rho + (0.6 / S) ||x~||_1
//     ||x~||_1 <= 16 ||x~||_2 <= 16 (1 + rho) <= 32.3        (rho <= 128 s <= 1.01)
//     u4 = s (16 q16 . h + 7.5 sum q16) / S + rho + 19.4 / S          >=  c - 1e-5
// (q16 . h = q16 . (h + 8) - 8 sum q16, exact in int32).  The coarse pass streams the plane and
// {s, rho}, 136 B/row, and skips every row with u4 + STB_Q4_SKIP_EPS < T, where T is a proven
// lower bound of this launch's k-th best exact cosine (below): a skipped row has c < c_k, so it
// can neither be a result nor tie with one.  Every other row is queued per warp; each 32 queued
// rows are scored from their int8 codes with the arithmetic of stb_scan_q8 and handed to the
// sink, so the lists, drop bounds and completeness proof are the q8 tier's, over the rows that
// were not skipped.
// T: a refined row also has a lower bound l8 = s (dot / S - h_l1) - e_q - 2e-5 <= c - 1e-5, which
// is max-ed into word (row mod k) of k words.  T = min of the k words is the l8 of k distinct
// rows, so at least k rows have c >= T.  A word is u64 (tag << 32 | ordered l8) and the tag
// identifies the launch: a later launch that shares the slot writes larger words, a word with
// another tag reads as "no bound", so slots are never cleared and overlapped launches need no
// ordering between them.  Warps re-read the words once per tile.
#define STB_Q4_SCAN_U 8         // 32-row tiles (4 * U): one row x 8 LDG.128 per lane in flight (4 KiB per warp)
#define STB_Q4_SPARE 64         // queued rows per warp: < 32 left over + one tile's worth ...
#define STB_Q4_QUEUE (STB_Q4_SPARE + 4)                 // ... + a spare slot for lanes with nothing to store (16-B aligned)
struct StbQ4Args {
  const uint8_t *plane;          // nibbles, 128 B per row in 32-row tiles (stb_q4_plane_offset)
  const float2 *sr;              // [n] {s, rho}
  unsigned long long *thr;       // the k threshold words of this launch
  uint32_t tag;                  // this launch's tag (never 0)
  uint32_t top_k;                // k >= 1 words
  unsigned long long *refined;   // debug counter: rows refined from the int8 codes
};

// c + sum of the four products of a's unsigned bytes with b's signed bytes
__device__ __forceinline__ int stb_dp4a_us(uint32_t a, uint32_t b, int c) {
  int d;
  asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}

// Test hook (stb_debug_q4_scan, DUMP = 1): per local row, the u4 and the T it was tested against, and for refined
// rows the l8 before stb_f2ord; pin != 0 holds T at -inf, so every row is refined.
struct StbQ4Dump {
  float *u4, *t, *l8;
  int pin;
};

// One query as the prefilter sees it: its words in shared memory (layout: stb_scan_q4) and the constants of its
// bounds.  The guest of a pair keeps a copy of the constants, its threshold words and k in shared memory.
struct StbQ4Side {
  float inv_S, h_l1, e_q;        // StbQ8Query
  float A, B, e_q4;              // u4 = s (A D + B) + rho + e_q4
  int sumq;                      // sum of the q16 components
  int unusable;
  unsigned long long *thr;       // threshold words, their tag and count
  uint32_t tag;
  int kw;
};

// Writes the warp's copy of the query words of q to pw (every lane of the warp calls it) and returns its constants.
__device__ __forceinline__ StbQ4Side stb_q4_query(const float *q, uint32_t *pw, int lane) {
  const int g = lane >> 3, j = lane & 7;
  const StbQ8Query Q = stb_q8_query(q, j);
  // query words in shared memory, read by every lane at once.  Chunk m, word k (components 32m + 4k .. +3
  // pair with its low nibbles, 32m + 16 + 4k .. +3 with its high nibbles): {low hi, low lo, high hi, high lo}
  // byte words at pw[(4m + k) * 4 + {0..3}]; the int8 codes' words (StbQ8Query) of refine lane j at
  // pw[128 + 16 j + {0..7: hi, 8..15: lo}]
  int sumq = 0;
  {
    const float4 *qv = reinterpret_cast<const float4 *>(q);
    int l1 = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      uint32_t hw, lw;
      stb_q16_words(__ldg(qv + 8 * j + i), Q.qs, Q.unusable, hw, lw, l1, sumq);
      if (g == 0) {
        *reinterpret_cast<uint2 *>(pw + (4 * j + (i & 3)) * 4 + (i < 4 ? 0 : 2)) = make_uint2(hw, lw);
        pw[128 + 16 * j + i] = Q.qhi[i];
        pw[128 + 16 * j + 8 + i] = Q.qlo[i];
      }
    }
    __syncwarp();
  }
  sumq += __shfl_xor_sync(0xffffffffu, sumq, 4);
  sumq += __shfl_xor_sync(0xffffffffu, sumq, 2);
  sumq += __shfl_xor_sync(0xffffffffu, sumq, 1);
  StbQ4Side S;
  S.inv_S = Q.inv_S; S.h_l1 = Q.h_l1; S.e_q = Q.e_q;
  S.A = 16.0f * Q.inv_S;
  S.B = 7.5f * (float)sumq * Q.inv_S;
  S.e_q4 = 19.4f * Q.inv_S;
  S.sumq = sumq;
  S.unusable = Q.unusable ? 1 : 0;
  S.thr = nullptr; S.tag = 0u; S.kw = 1;
  return S;
}

// ---- pairs: one read of each plane tile scores two back-to-back queries ----------------------------------
// A q8 top-k launch of an overlapped series is a HOST or a GUEST (stb_launch_topk_t).  A guest is two launches:
// stb_pair_join_kernel, which the host releases at its start, and its own scan kernel.  The join publishes
// the guest's query in the host's seat and then adds STB_PAIR_JUMP to the host's ticket counter: the ticket v
// the add returns is the join point.  Host draws at or above the jump are tickets >= v, and those below
// n_tickets score their tiles for both queries; after the host's own tickets run out its warps draw tickets
// [0, v) again from the seat's wrap word and score them for the guest alone.  So each tile is scored once for
// each query, and the jump tells a draw that it follows the join with no window between the two.  The host
// then runs the tail (CTA merge, tree merge, re-rank, proof, hits) once per query.  A join whose add finds
// every ticket drawn refuses (the host's warps, whose failing draws may follow the jump, read the decision
// from the seat: the join kernel writes it right after its add, and it is running); so does a query the q8
// tier cannot use, without a jump.  A refused guest's scan kernel scans by itself.  The host books the jump on
// its counter when the guest launches; a join without one adds it once the host has completed.
__device__ __forceinline__ unsigned long long stb_ld_acquire_gpu(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// A join kernel starts when its host has drawn ~30k tiles (H100, 10M and 1M rows: median join tiles 29.4k and
// 27.1k), so a pair reads (n + 30k) tiles for two queries.  Below ~60k tiles (1.9M rows) that saves too little
// to pay for running the hosts one after the other, and the series co-scans instead (1M rows: 0.070 ms per
// query paired, 0.053 co-scanning).
#define STB_PAIR_MIN_TILES 60000
#define STB_PAIR_JUMP (1ull << 31)   // > every ticket count (tiles < 2^27); a jumped ticket still fits 32 bits
// seat words: common.cuh (STB_SEAT_*)
#define STB_PAIR_SCRATCH (STB_Q4_QUEUE + 256 + 16)   // per warp: the guest's queue, words and StbQ4Side

template <int U, int RANGES, int DUMP = 0, bool PAIR = false, class Sink>
__device__ __forceinline__ bool stb_scan_q4(const ScanArgs &args, const uint8_t *q8, const float *q8_scale, const StbQ4Args &q4a,
                                            uint32_t *wq, uint32_t *pw, Sink &sink, const uint32_t *off = nullptr,
                                            const StbQ4Dump *dump = nullptr, unsigned long long *seat = nullptr,
                                            uint32_t *gscr = nullptr, Sink *sink2 = nullptr) {
  static_assert(4 * U == STB_Q4_TILE_ROWS && STB_Q8_MAX_K <= 32, "one plane tile per warp tile, one row per lane; one lane per threshold word");
  static_assert(!PAIR || (RANGES == 0 && DUMP == 0), "pairs scan whole shards");
  static_assert(sizeof(StbQ4Side) <= 16 * 4, "guest constants");
  const int lane = threadIdx.x & 31;
  const int g = lane >> 3;   // refine: row group inside the warp
  const int j = lane & 7;    // refine: int8 code bytes [16j, 16j+16) and [128+16j, ...)
  const StbQ4Side S1 = stb_q4_query(args.q, pw, lane);   // its threshold words, tag and k: q4a
  unsigned tcache = 0u;              // lane w < k: best ordered l8 of word w this warp knows (0: none)
  int qn = 0;                        // queued rows (warp-uniform)
  unsigned refined = 0u;
  // the guest (PAIR): queue, words and constants in gscr, list in *sink2
  uint32_t *wq2 = gscr, *pw2 = gscr + STB_Q4_QUEUE;
  StbQ4Side *side2 = reinterpret_cast<StbQ4Side *>(gscr + STB_Q4_QUEUE + 256);
  unsigned tcache2 = 0u;
  int qn2 = 0;

  // the first 32 queue slots of one query (0xffffffff: empty; slot 0 is never empty)
  auto refine = [&](const uint32_t *q_wq, const uint32_t *q_pw, const StbQ4Side &S, unsigned long long *thr, uint32_t tag, int kw,
                    auto &snk, unsigned tc) {
    uint32_t row[8];
    bool valid[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      row[u] = q_wq[u * 4 + g];
      valid[u] = row[u] != 0xffffffffu;
      if (!valid[u]) row[u] = q_wq[0];
    }
    int dot[8];
    float sc_row[8];
#pragma unroll
    for (int h = 0; h < 2; ++h) {          // two halves of 4 rows: the coarse pass's state stays in registers
      const uint32_t rh[4] = {row[4 * h], row[4 * h + 1], row[4 * h + 2], row[4 * h + 3]};
      int dh[4];
      float sh[4];
      stb_q8_dots<4>(q_pw + 128 + 16 * j, q_pw + 128 + 16 * j + 8, q8, q8_scale, rh, j, dh, sh);
#pragma unroll
      for (int u = 0; u < 4; ++u) { dot[4 * h + u] = dh[u]; sc_row[4 * h + u] = sh[u]; }
    }
    int d = 0;
    float sc = 0.f;
    uint32_t r = 0;
    bool v = false;
#pragma unroll
    for (int u = 0; u < 8; ++u)
      if (j == u) { d = dot[u]; sc = sc_row[u]; r = row[u]; v = valid[u]; }
    const float s = !v ? -CUDART_INF_F : (S.unusable ? CUDART_INF_F : fmaf(sc, fmaf((float)d, S.inv_S, S.h_l1), S.e_q));
    refined += (unsigned)__popc(__ballot_sync(0xffffffffu, v));
    snk.template consume<32>(s, r);
    if (S.unusable) return;
    // publish the lower bounds that beat the published value of their word (rare after the first tickets);
    // the warp learns its own contributions with the next read
    const float l8 = fmaf(sc, fmaf((float)d, S.inv_S, -S.h_l1), -S.e_q) - (float)STB_Q8_SCAN_EPS;
    if constexpr (DUMP) {
      if (v) dump->l8[r] = l8;
    }
    const unsigned o8 = stb_f2ord(l8);
    const int w = (int)(r % (uint32_t)kw);
    const unsigned known = __shfl_sync(0xffffffffu, tc, w);   // every lane takes part in the shuffle
    if (v && o8 > known) atomicMax(thr + w, ((unsigned long long)tag << 32) | o8);
  };

  // one query's side of a tile: fold in its threshold words, test the row's bound, queue it, refine 32 queued rows
  auto pass = [&](int lh, int ll, int hh, int hl, float2 sr, unsigned tw, const StbQ4Side &S, unsigned long long *thr,
                  uint32_t tag, int kw, unsigned &tc, uint32_t *q_wq, const uint32_t *q_pw, int &q_n, auto &snk, bool valid, uint32_t row) {
    if (lane < kw) tc = max(tc, tw);  // tw: the word's ordered l8 if it carries the query's tag, else 0
    float T;
    {
      const unsigned tmin = __reduce_min_sync(0xffffffffu, lane < kw ? tc : 0xffffffffu);
      T = tmin ? stb_ord2f(tmin) : -CUDART_INF_F;
    }
    const int D = (lh + (hh >> 4)) * 256 + (ll + (hl >> 4)) - 8 * S.sumq;   // q16 . h (hh, hl: multiples of 16)
    const float u4 = fmaf(sr.x, fmaf((float)D, S.A, S.B), sr.y + S.e_q4);
    if constexpr (DUMP) {
      if (dump->pin) T = -CUDART_INF_F;
      if (valid) { dump->u4[row] = u4; dump->t[row] = T; }
    }
    // an unusable query publishes no bound (refine), so T stays -inf and every valid row is queued
    const bool want = valid && !(u4 + (float)STB_Q4_SKIP_EPS < T);
    const unsigned mk = __ballot_sync(0xffffffffu, want);
    q_wq[want ? q_n + __popc(mk & ((1u << lane) - 1u)) : STB_Q4_SPARE] = row;
    q_n += __popc(mk);
    if (q_n >= 32) {                 // q_n < 64: one batch at most
      __syncwarp();
      refine(q_wq, q_pw, S, thr, tag, kw, snk, tc);
      const uint32_t rest = (32 + lane < q_n) ? q_wq[32 + lane] : 0u;
      __syncwarp();
      q_wq[(32 + lane < q_n) ? lane : STB_Q4_SPARE] = rest;
      q_n -= 32;
    }
  };

  constexpr uint64_t tile_rows = 4 * U;
  const uint64_t n_tiles = (args.n_virtual + tile_rows - 1) / tile_rows;
  const uint32_t n_rows = (uint32_t)args.n_virtual;
  StbRowMap<RANGES> rmap;
  rmap.restart();
  // M & 1: score the tile for the launch's own query, M & 2: for the guest.  M == 3 is the pair's tile body: one
  // set of plane loads feeds two sets of dp4a accumulators.
  auto tile_body = [&](uint64_t tile, bool first, auto mode) {
    constexpr int M = decltype(mode)::value;
    if (first) rmap.restart();
    const StbQ4Side &S2 = *side2;      // read where used: shared memory, not registers
    // lane w < k: threshold word w as the other warps left it; issued with the tile's loads, folded in below
    unsigned long long tw = 0ull, tw2 = 0ull;
    if constexpr ((M & 1) != 0) tw = lane < (int)q4a.top_k ? __ldcg(q4a.thr + lane) : 0ull;
    if constexpr ((M & 2) != 0) tw2 = lane < S2.kw ? __ldcg(S2.thr + lane) : 0ull;
    // lane l owns virtual row 32 tile + l (< 2^32: a shard holds at most 2^32 - 2 rows); past the end it
    // reads the last row and is not queued
    const uint32_t v = (uint32_t)tile * (uint32_t)tile_rows + (uint32_t)lane;
    const bool valid = v < n_rows;
    const uint32_t row = rmap.map(args, valid ? v : n_rows - 1);
    const uint8_t *p = q4a.plane + stb_q4_plane_offset(row, 0);
    uint4 a[8];
#pragma unroll
    for (int m = 0; m < 8; ++m) {
      const float4 t = stb_ld_stream(reinterpret_cast<const float4 *>(p + m * 512));
      a[m] = make_uint4(__float_as_uint(t.x), __float_as_uint(t.y), __float_as_uint(t.z), __float_as_uint(t.w));
    }
    const float2 sr = __ldg(q4a.sr + row);
    // the threshold words as one register each: 0 unless the word carries the query's tag
    const unsigned tv = (uint32_t)(tw >> 32) == q4a.tag ? (unsigned)tw : 0u;
    unsigned tv2 = 0u;
    if constexpr ((M & 2) != 0) tv2 = (uint32_t)(tw2 >> 32) == S2.tag ? (unsigned)tw2 : 0u;
    // low nibbles x {hi, lo} query bytes, 16 x high nibbles x {hi, lo}: exact in int32
    int lh = 0, ll = 0, hh = 0, hl = 0, lh2 = 0, ll2 = 0, hh2 = 0, hl2 = 0;
#pragma unroll
    for (int m = 0; m < 8; ++m) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t w = k == 0 ? a[m].x : (k == 1 ? a[m].y : (k == 2 ? a[m].z : a[m].w));
        const uint32_t lo = w & 0x0F0F0F0Fu, hi = w & 0xF0F0F0F0u;
        if constexpr ((M & 1) != 0) {
          const uint4 qw = *reinterpret_cast<const uint4 *>(pw + (4 * m + k) * 4);
          lh = __dp4a((int)lo, (int)qw.x, lh);
          ll = __dp4a((int)lo, (int)qw.y, ll);
          hh = stb_dp4a_us(hi, qw.z, hh);
          hl = stb_dp4a_us(hi, qw.w, hl);
        }
        if constexpr ((M & 2) != 0) {
          const uint4 qw = *reinterpret_cast<const uint4 *>(pw2 + (4 * m + k) * 4);
          lh2 = __dp4a((int)lo, (int)qw.x, lh2);
          ll2 = __dp4a((int)lo, (int)qw.y, ll2);
          hh2 = stb_dp4a_us(hi, qw.z, hh2);
          hl2 = stb_dp4a_us(hi, qw.w, hl2);
        }
      }
    }
    if constexpr ((M & 1) != 0) pass(lh, ll, hh, hl, sr, tv, S1, q4a.thr, q4a.tag, (int)q4a.top_k, tcache, wq, pw, qn, sink, valid, row);
    if constexpr ((M & 2) != 0) pass(lh2, ll2, hh2, hl2, sr, tv2, S2, S2.thr, S2.tag, S2.kw, tcache2, wq2, pw2, qn2, *sink2, valid, row);
  };

  bool joined = false;               // warp-uniform; the same in every warp once the scan is over
  bool paired = false;
  if constexpr (PAIR) paired = seat != nullptr;
  if (!paired) {
    stb_for_each_tile<RANGES, 2>(args, n_tiles, off, [&](uint64_t tile, bool first) {
      tile_body(tile, first, std::integral_constant<int, 1>());
    });
  } else if constexpr (PAIR) {
    // the host of a pair: stb_for_each_tile's ticket loop, with the join read off every draw
    auto draw = [&]() -> uint32_t {     // relative to the launch's start: < 2^32 with the jump
      uint32_t t = 0;
      if (lane == 0) t = (uint32_t)(atomicAdd(args.tickets, 1ull) - args.t_base);
      return __shfl_sync(0xffffffffu, t, 0);
    };
    auto run_ticket = [&](uint64_t t, auto mode) {
      stb_ticket_walk<0>(args, t, n_tiles, off, [&](uint64_t tile, bool) { tile_body(tile, false, mode); });
    };
    // host tickets until a draw carries the jump (or fails), then the pair's tickets
    uint32_t cur = draw();
    while (cur < STB_PAIR_JUMP && stb_ticket_first_tile(cur, args.t_bulk) < n_tiles) {
      const uint32_t nxt = draw();        // drawn before the ticket is scored (stb_for_each_tile)
      run_ticket(cur, std::integral_constant<int, 1>());
      cur = nxt;
    }
    joined = cur >= STB_PAIR_JUMP;
    if (joined) {
      // the first draw after the join: the seat holds what the join kernel wrote before its jump
      __threadfence();
      StbQ4Side S = stb_q4_query(reinterpret_cast<const float *>(__ldcg(seat + STB_SEAT_Q)), pw2, lane);
      const unsigned long long info = __ldcg(seat + STB_SEAT_INFO);
      S.thr = reinterpret_cast<unsigned long long *>(__ldcg(seat + STB_SEAT_THR));
      S.tag = (uint32_t)(info >> 32);
      S.kw = (int)(uint32_t)info;
      if (lane == 0) *side2 = S;
      __syncwarp();
      cur -= (uint32_t)STB_PAIR_JUMP;
      while (stb_ticket_first_tile(cur, args.t_bulk) < n_tiles) {
        const uint32_t nxt = draw() - (uint32_t)STB_PAIR_JUMP;
        run_ticket(cur, std::integral_constant<int, 3>());
        cur = nxt;
      }
    }
    if (joined) {
      // the join kernel writes its decision right after its jump, and it is running: wait for the word.  A
      // warp whose only draw after the jump failed cannot tell a late refusal from a join without it.
      uint32_t d = 0;                    // 0x80000000 | v: joined at ticket v
      if (lane == 0) {
        const uint32_t gtag = side2->tag;
        unsigned long long w;
        do w = stb_ld_acquire_gpu(seat + STB_SEAT_DECIDED); while ((uint32_t)(w >> 32) != gtag);
        d = (uint32_t)w;
      }
      d = __shfl_sync(0xffffffffu, d, 0);
      joined = (d & 0x80000000u) != 0;
      if (lane == 0) gscr[STB_PAIR_SCRATCH - 1] = d & 0x7fffffffu;   // v: in shared memory, the wrap's tile body needs the registers
      __syncwarp();
    }
    if (joined) {
      // the guest-only wrap: tickets [0, v), drawn from the seat's wrap word (tagged with this launch's tag)
      unsigned long long *wrap = seat + STB_SEAT_WRAP;
      const volatile uint32_t *v = gscr + STB_PAIR_SCRATCH - 1;
      for (;;) {
        unsigned long long w = 0;
        if (lane == 0) {
          unsigned long long c = __ldcg(wrap);
          while ((uint32_t)(c >> 32) != q4a.tag) {
            const unsigned long long prev = atomicCAS(wrap, c, (unsigned long long)q4a.tag << 32);
            c = prev == c ? (unsigned long long)q4a.tag << 32 : prev;
          }
          w = atomicAdd(wrap, 1ull) & 0xffffffffull;
        }
        w = __shfl_sync(0xffffffffu, w, 0);
        if (w >= *v) break;
        run_ticket(w, std::integral_constant<int, 2>());
      }
    }
  }
  if (qn > 0) {                      // the rest, with the empty slots marked
    wq[lane >= qn ? lane : STB_Q4_SPARE] = 0xffffffffu;
    __syncwarp();
    refine(wq, pw, S1, q4a.thr, q4a.tag, (int)q4a.top_k, sink, tcache);
  }
  if constexpr (PAIR) {
    if (joined && qn2 > 0) {
      const StbQ4Side &S2 = *side2;
      wq2[lane >= qn2 ? lane : STB_Q4_SPARE] = 0xffffffffu;
      __syncwarp();
      refine(wq2, pw2, S2, S2.thr, S2.tag, S2.kw, *sink2, tcache2);
    }
  }
  if (lane == 0 && refined) atomicAdd(q4a.refined, (unsigned long long)refined);
  return joined;
}

// q8 builder: one warp per row (row_encode.cuh: stb_q8_encode_row).  The same pass writes the nibble
// plane and {s, rho} of the top-k scan's prefilter (stb_scan_q4).
__global__ void __launch_bounds__(256)
stb_q8_build_kernel(const float4 *__restrict__ rows, uint64_t first_row, uint64_t n_rows, uint8_t *__restrict__ out,
                    float *__restrict__ scale, uint8_t *__restrict__ plane, float2 *__restrict__ sr, int *bad_flag,
                    uint64_t rows_first) {
  const int lane = threadIdx.x & 31;
  const uint64_t row = first_row + (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= n_rows) return;
  const float4 v0 = __ldg(rows + (row - rows_first) * STB_ROW_F4 + 2 * lane);
  const float4 v1 = __ldg(rows + (row - rows_first) * STB_ROW_F4 + 2 * lane + 1);
  stb_q8_encode_row(v0, v1, lane, row, out, scale, plane, sr, bad_flag);
}

int stb_launch_q8_build(stb_ctx *ctx, const float *rows_dev, uint64_t first_row, uint64_t n_rows, uint8_t *out,
                        float *scale, uint8_t *plane, float2 *sr, int *bad_flag_dev, uint64_t rows_first) {
  if (first_row >= n_rows) return STB_OK;
  const unsigned blocks = (unsigned)((n_rows - first_row + 7) / 8);
  stb_q8_build_kernel<<<blocks, 256, 0, ctx->stream>>>(reinterpret_cast<const float4 *>(rows_dev), first_row, n_rows, out, scale,
                                                       plane, sr, bad_flag_dev, rows_first);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// ---------------------------------------------------------------- top-K' sink ---
template <int E>
struct TopSink {
  float ls[E];
  uint32_t lr[E];
  float thr;   // min score in the list (warp-uniform); -inf while not full
  int lane;
  int fill;    // slots bulk-filled so far (warp-uniform); 32*E once the fill phase is over
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int e = 0; e < E; ++e) { ls[e] = -CUDART_INF_F; lr[e] = 0xffffffffu; }
    thr = -CUDART_INF_F;
    lane = threadIdx.x & 31;
    fill = 0;
  }
  __device__ __forceinline__ float warp_min(float m) const {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, off));
    return m;
  }
  __device__ __forceinline__ void insert(float cs, uint32_t cr) {
    float m = ls[0];
    int mi = 0;
#pragma unroll
    for (int e = 1; e < E; ++e)
      if (ls[e] < m) { m = ls[e]; mi = e; }
    unsigned owners = __ballot_sync(0xffffffffu, m == thr);
    int owner = __ffs(owners) - 1;
    if (lane == owner) {
#pragma unroll
      for (int e = 0; e < E; ++e)
        if (e == mi) { ls[e] = cs; lr[e] = cr; }
    }
    m = ls[0];
#pragma unroll
    for (int e = 1; e < E; ++e) m = fminf(m, ls[e]);
    thr = warp_min(m);
  }
  // Bulk fill: while the list has room and tiles are complete, the tile's rows are
  // gathered straight into the free slots (slot -> lane slot%32, entry slot/32) with two
  // shuffles, instead of one min-reduction per row.  ROWS = rows a full tile carries,
  // sitting in lanes g*8+u (g < 4, u < ROWS/4).
  template <int ROWS>
  __device__ __forceinline__ bool try_fill(float s, uint32_t r, unsigned vmask) {
    constexpr int KP = 32 * E;
    constexpr int UU = ROWS / 4;
    unsigned full = 0u;
#pragma unroll
    for (int g = 0; g < 4; ++g)
#pragma unroll
      for (int u = 0; u < UU; ++u) full |= 1u << (g * 8 + u);
    if (fill >= KP) return false;
    if (vmask != full || fill + ROWS > KP) {      // ragged tile: leave the fill phase for good
      fill = KP;
      return false;
    }
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int d = e * 32 + lane - fill;          // which row of the tile this slot takes
      const bool want = (d >= 0 && d < ROWS);
      const int src = want ? ((d / UU) * 8 + (d % UU)) : 0;
      const float cs = __shfl_sync(0xffffffffu, s, src);
      const uint32_t cr = __shfl_sync(0xffffffffu, r, src);
      if (want) { ls[e] = cs; lr[e] = cr; }
    }
    fill += ROWS;
    if (fill >= KP) {
      float m = ls[0];
#pragma unroll
      for (int e = 1; e < E; ++e) m = fminf(m, ls[e]);
      thr = warp_min(m);
    }
    return true;
  }
  template <int ROWS>
  __device__ __forceinline__ void consume(float s, uint32_t r) {
    if (fill < 32 * E) {
      const unsigned vmask = __ballot_sync(0xffffffffu, s > -CUDART_INF_F);
      if (try_fill<ROWS>(s, r, vmask)) return;
    }
    (*this)(s, r);
  }
  __device__ __forceinline__ void operator()(float s, uint32_t r) {
    unsigned mask = __ballot_sync(0xffffffffu, s > thr);
    while (mask) {
      int src = __ffs(mask) - 1;
      mask &= mask - 1;
      float cs = __shfl_sync(0xffffffffu, s, src);
      uint32_t cr = __shfl_sync(0xffffffffu, r, src);
      if (cs > thr) insert(cs, cr);
    }
  }
};

__device__ __forceinline__ void stb_cta_sort_keys(uint64_t *keys, int n) {
  static_assert(STB_SCAN_THREADS == 256, "register sort assumes 256 threads");
  if (n <= 256) stb_cta_sort_keys_t<1>(keys, n);
  else stb_cta_sort_keys_t<4>(keys, n);
}

// Co-scan: a launch that co-runs with its predecessor on the same corpus starts its pass where the
// predecessor is reading, so the second read of each tile is an L2 hit.  The first CTA to arrive fixes
// the offset in this launch's tagged word (tag << 32 | offset, never cleared, like the q4 threshold
// words); the others take its value.  The offset is a hint: a stale read of the predecessor's word or
// counter (launch_dependents orders no memory) gives another valid offset and only costs sharing.
// Nothing waits on the other grid.
struct StbCoscanArgs {
  unsigned long long *word;               // null: no co-scan, offset 0
  uint32_t tag;
  uint32_t pred_tag;                      // 0: no predecessor to follow (offset 0)
  const unsigned long long *pred_word;    // the predecessor's offset word ...
  const unsigned long long *pred_tickets; // ... its ticket counter, the counter's value at its start ...
  unsigned long long pred_t_base;
  uint64_t pred_t_bulk;                   // ... and its bulk ticket count (same tile count as this launch)
};

// join_front >= 0: a joined guest, whose pass starts at its join tile of the host's pass (the predecessor's).
__device__ __forceinline__ uint32_t stb_coscan_offset(const StbCoscanArgs &c, uint64_t n_tiles, int64_t join_front = -1) {
  unsigned long long cur = __ldcg(c.word);
  while ((uint32_t)(cur >> 32) != c.tag) {
    uint64_t off = 0;
    if (c.pred_tag) {
      const unsigned long long pw = __ldcg(c.pred_word);
      const uint64_t p_off = (uint32_t)(pw >> 32) == c.pred_tag ? (uint32_t)pw % n_tiles : 0;
      // the predecessor's frontier: the first tile of its next undrawn ticket (stb_for_each_tile)
      const unsigned long long drawn = __ldcg(c.pred_tickets) - c.pred_t_base;
      uint64_t front = n_tiles;
      if (join_front >= 0) front = (uint64_t)join_front;
      else if (drawn < n_tiles) front = stb_ticket_first_tile(drawn, c.pred_t_bulk);
      off = (p_off + (front < n_tiles ? front : 0)) % n_tiles;
    }
    const unsigned long long mine = ((unsigned long long)c.tag << 32) | off;
    const unsigned long long prev = atomicCAS(c.word, cur, mine);
    cur = prev == cur ? mine : prev;
  }
  return (uint32_t)cur % n_tiles;
}

// A pair (SRC == 2, RANGES == 0; see "pairs" above).  Host: its seat and the guest tail's tree-merge scratch.
// Guest: the seat's decided word and the tag it waits for, and its own ticket counter's booked advance.
struct StbPairArgs {
  unsigned long long *seat;            // host; null: no guest can join
  uint64_t *keys2;
  unsigned int *counters2;
  const unsigned long long *decided;   // guest; null: not a guest
  uint32_t tag;
  unsigned long long booked;
};

struct TopkArgs {
  ScanArgs scan;
  StbCoscanArgs co;
  StbPairArgs pair;
  uint64_t row_base;
  uint64_t *keys;            // sorted best-KP lists of every tree level
  unsigned int *counters;    // one arrival ticket per tree group, all levels
  stb_hit *out_hits;
  uint32_t *out_status;
  uint32_t top_k;
  StbXchgArgs xchg;          // world == 0: no cross-GPU exchange
  const uint8_t *shadow;    // SRC == 1: 16-bit normalised corpus shadow (UMMA tile layout)
  uint32_t early_trigger;    // overlapped launch: release the dependent launch at kernel start
  const uint8_t *q8;         // SRC == 2: int8 codes [n][256] ...
  const float *q8_scale;     //           ... and per-row scales [n]
  StbQ4Args q4;              //           ... and the prefilter's copy, threshold words, debug counter
};

// ---- peer-memory exchange (fused K1 -> all-gather -> K4) ------------------------------
// Every rank owns one exchange buffer (cudaMalloc, mapped into all peers through CUDA
// IPC or peer access):  flags[S][world] u64 | status[S][world] u32 | hits[S][world][max_k].
// The final CTA of rank r stores its k hits into slot (seq % S), lane r of EVERY peer's
// buffer over NVLink, fences, release-stores seq into the peers' flags, then
// acquire-spins on its own flags until all `world` lanes carry seq, and merges.
__device__ __forceinline__ void stb_st_release_sys(unsigned long long *p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long stb_ld_acquire_sys(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long *stb_x_flags(const StbXchgArgs &x, int peer) {
  return reinterpret_cast<unsigned long long *>(x.base[peer]);
}
__device__ __forceinline__ uint32_t *stb_x_status(const StbXchgArgs &x, int peer) {
  return reinterpret_cast<uint32_t *>(x.base[peer] + (size_t)STB_XCHG_SLOTS * x.world * 8);
}
__device__ __forceinline__ stb_hit *stb_x_hits(const StbXchgArgs &x, int peer) {
  return reinterpret_cast<stb_hit *>(x.base[peer] + (size_t)STB_XCHG_SLOTS * x.world * 16);
}

// Sort the first `c` keys of skeys (padded with INVALID to a power of two >= KP).
__device__ __forceinline__ int stb_pad_and_sort(uint64_t *skeys, int c, int min_n) {
  int n = min_n;
  while (n < c) n <<= 1;
  const int span = n <= 256 ? 256 : STB_SORT_CAP;   // the register sort writes back its whole span
  for (int i = c + threadIdx.x; i < span; i += blockDim.x) skeys[i] = STB_KEY_INVALID;
  __syncthreads();
  stb_cta_sort_keys(skeys, n);
  return n;
}

#define STB_RR_STRIDE 260   // floats per staged row (1 KiB + 16 B pad: conflict-free LDS.128)

// The join kernel of a guest (see "pairs" above): one warp beside the host's CTAs.  It decides, writes the seat's
// decided word, releases the guest's scan kernel and completes only after the host has.
struct StbPairJoinArgs {
  unsigned long long *seat;        // the host's seat
  unsigned long long *tickets;     // the host's ticket counter ...
  unsigned long long t_base;       // ... its value at the host's start and the host's ticket count
  uint64_t n_tickets;
  uint64_t v_floor;                // test hook (stb_debug_pair_floor): join no earlier than ticket v_floor
  const float *q;                  // the guest: query, outputs, k, threshold words and tag
  stb_hit *hits;
  uint32_t *status;
  uint32_t top_k;
  unsigned long long *thr;
  uint32_t tag;
};

// A warp's registers come from one of the SM's four 16K-register sub-partitions.  Two q8 scan CTAs put four
// warps of 120 registers on each (15,360), so the join's one warp must make do with the 1,024 left: 32 each.
#define STB_PAIR_JOIN_REGS 32
__global__ void __maxnreg__(STB_PAIR_JOIN_REGS) stb_pair_join_kernel(const StbPairJoinArgs a) {
  const StbQ8Query Q = stb_q8_query(a.q, threadIdx.x & 7);
  bool jumped = false;
  if (threadIdx.x == 0) {
    unsigned long long decided = (unsigned long long)a.tag << 32;   // refused
    if (!Q.unusable) {
      unsigned long long *s = a.seat;
      s[STB_SEAT_Q] = reinterpret_cast<unsigned long long>(a.q);
      s[STB_SEAT_HITS] = reinterpret_cast<unsigned long long>(a.hits);
      s[STB_SEAT_STATUS] = reinterpret_cast<unsigned long long>(a.status);
      s[STB_SEAT_THR] = reinterpret_cast<unsigned long long>(a.thr);
      s[STB_SEAT_INFO] = ((unsigned long long)a.tag << 32) | a.top_k;
      if (a.v_floor) {                               // the host is running: it draws on or runs out
        unsigned long long t;
        do t = stb_ld_acquire_gpu(a.tickets) - a.t_base; while (t < a.v_floor && t < a.n_tickets);
      }
      __threadfence();                               // the seat before the jump
      // an atomic add, not a CAS: the host's warps draw hundreds of tickets per microsecond
      const unsigned long long t = atomicAdd(a.tickets, STB_PAIR_JUMP) - a.t_base;
      jumped = true;
      if (t < a.n_tickets) decided |= 0x80000000ull | t;   // joined at ticket t
    }
    a.seat[STB_SEAT_DECIDED] = decided;
    __threadfence();
  }
  __syncwarp();
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // complete after the host: the guest's scan kernel waits on this grid, the next launch on the guest's
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (threadIdx.x == 0 && !jumped) atomicAdd(a.tickets, STB_PAIR_JUMP);   // the jump the host booked, after its last draw
}

// E: 32*E candidates per warp / CTA / inner tree list.  EF: the ROOT of the merge tree (the CTA
// itself when the grid is one CTA) keeps 32*EF >= 32*E candidates for the exact re-rank.
// EF > E lets a tier with a wide error term (q8) re-rank 128 rows while every level below the
// root moves 32-key lists -- the tail costs what the f32 tier's does.  Completeness is tracked
// explicitly: every node that drops keys publishes the best score it dropped (<= its last kept
// key), the bounds are max-reduced up the tree, and the proof compares the k-th exact distance
// with that bound instead of "the K'-th key of one uniform list".
template <int E, int U, int RANGES, int SRC = 0, int EF = E>
__device__ __forceinline__ void stb_scan_topk_body(const TopkArgs &args) {
  // SRC 0: scores from the f32 rows; SRC 1: from the 16-bit shadow (wider proof margin);
  // SRC 2: upper bounds of the exact cosine from the int8 copy (margin folded into the score)
  constexpr double kScoreEps = SRC == 1 ? STB_SHADOW_SCAN_EPS : (SRC == 2 ? STB_Q8_SCAN_EPS : STB_SCORE_EPS);
  constexpr int KP = 32 * E;          // list length below the root
  constexpr int KF = 32 * EF;         // candidates the root keeps
  constexpr int KPS = KP + 1;         // published list stride: KP keys + the node's drop bound
  constexpr bool kPair = SRC == 2 && RANGES == 0;   // q8 whole-shard scans host and guest pairs
  static_assert(EF >= E && 8 * KP <= STB_SORT_CAP && KF <= STB_SORT_CAP / 2, "list sizes");
  __shared__ uint64_t skeys[STB_SORT_CAP];
  __shared__ unsigned int s_T, s_cnt, s_ticket, s_bound, s_nin;
  __shared__ unsigned long long s_T64;
  __shared__ double sqd[STB_D];                  // query in f64 (exact conversion)
  __shared__ __align__(16) float srows[32 * STB_RR_STRIDE];
  __shared__ double s_d[KF], s_r2[KF], s_q2;
  __shared__ uint64_t s_r[KF];
  __shared__ int s_nv[2];
  __shared__ double s_cthr;
  __shared__ int s_done;
  __shared__ unsigned int s_timeout;

  // co-scan: the tile this launch's pass starts at, fixed before the dependent is released so that
  // the dependent's first CTA can read it
  __shared__ uint32_t s_off;          // (stb_for_each_tile reads it with RANGES == 0 only)
  if constexpr (RANGES == 0) {
    __shared__ int s_guest_joined;
    const uint64_t n_tiles = (args.scan.n_virtual + 4 * U - 1) / (4 * U);
    if (threadIdx.x == 0) {
      int64_t front = -1;
      s_guest_joined = 0;
      if (kPair && args.pair.decided) {
        // a guest: the join kernel wrote the decided word before it released this grid
        unsigned long long w;
        do w = stb_ld_acquire_gpu(args.pair.decided); while ((uint32_t)(w >> 32) != args.pair.tag);
        if (w & 0x80000000ull) {
          s_guest_joined = 1;
          front = (int64_t)stb_ticket_first_tile((uint32_t)w & 0x7fffffffu, args.scan.t_bulk);   // the host's plan: same grid
        }
      }
      s_off = args.co.word ? stb_coscan_offset(args.co, n_tiles, front) : 0u;
    }
    __syncthreads();
    if (s_guest_joined) {
      // the host scores this query: release the next launch; one CTA completes after the host (through the
      // join kernel) and books this launch's tickets
      asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
      if (blockIdx.x == 0) {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        if (threadIdx.x == 0) atomicAdd(args.scan.tickets, args.pair.booked);
      }
      return;
    }
  }
  // Overlapped launches (asynchronous entry points): the grid lets the NEXT query's grid in right away, so
  // the ~10 us in which a draining grid leaves HBM idle (CTA merge before exit, launch, ramp-up) are covered
  // by the other scan, and a pair's join kernel runs while its host starts.
  // Tails stay ordered: everything after the scan sits behind griddepcontrol.wait.
  if (args.early_trigger) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  TopSink<E> sink, sink2;
  sink.init();
  bool joined = false;
  if constexpr (SRC == 2) {
    // the refine queues live in the re-rank staging area, which is first used after the CTA merge
    // (per warp: STB_Q4_QUEUE queued rows + 256 query words; a host's guest: STB_PAIR_SCRATCH more)
    static_assert(STB_SCAN_WARPS * (STB_Q4_QUEUE + 256 + STB_PAIR_SCRATCH) <= 32 * STB_RR_STRIDE, "q4 scratch");
    uint32_t *scratch = reinterpret_cast<uint32_t *>(srows) + (threadIdx.x >> 5) * (STB_Q4_QUEUE + 256);
    uint32_t *gscr = reinterpret_cast<uint32_t *>(srows) + STB_SCAN_WARPS * (STB_Q4_QUEUE + 256) + (threadIdx.x >> 5) * STB_PAIR_SCRATCH;
    sink2.init();
    joined = stb_scan_q4<U, RANGES, 0, kPair>(args.scan, args.q8, args.q8_scale, args.q4, scratch, scratch + STB_Q4_QUEUE, sink, &s_off,
                                              nullptr, args.pair.seat, gscr, &sink2);
  } else if constexpr (SRC == 1) stb_scan_shadow<U, RANGES>(args.scan, args.shadow, sink, &s_off);
  else stb_scan_rows<U, RANGES>(args.scan, sink, &s_off);
  // Programmatic dependent launch: the scan above reads only the corpus and the query,
  // so the NEXT query's kernel may start streaming as soon as every CTA of this one has
  // left its scan loop; this kernel's merge / re-rank tail then overlaps with it.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  // The tail of one query: CTA merge, tree merge over tkeys / tcnt, exact re-rank, proof and output.  A pair's
  // host runs it for its own query, then for the guest's.
  auto tail = [&](TopSink<E> &snk, const float *tq, uint32_t tk, stb_hit *th, uint32_t *ts, uint64_t *tkeys, unsigned int *tcnt,
                  bool xchg) {
    __syncthreads();

    // ---- CTA merge ------------------------------------------------------------------
    // T = max over warps of the warp list minimum is a lower bound of the CTA's KP-th
    // best score (that warp alone holds KP keys >= its minimum), so only keys >= T can
    // matter: compact those (typically ~KP..2KP of the 8*KP) and sort the small set.
    // Drop bounds are ordered scores (stb_f2ord); 0 = "nothing dropped so far".
    const int lane = threadIdx.x & 31;
    const unsigned kOrdNegInf = 0x007fffffu;       // stb_f2ord(-inf): a list that never filled
    if (threadIdx.x == 0) { s_T = 0u; s_cnt = 0u; }
    __syncthreads();
    if (lane == 0) atomicMax(&s_T, stb_f2ord(snk.thr));
    __syncthreads();
    {
      const unsigned T = s_T;
#pragma unroll
      for (int e = 0; e < E; ++e) {
        const bool take = snk.lr[e] != 0xffffffffu && stb_f2ord(snk.ls[e]) >= T;
        const unsigned m = __ballot_sync(0xffffffffu, take);
        unsigned base = 0u;
        if (lane == 0 && m) base = atomicAdd(&s_cnt, (unsigned)__popc(m));   // <= 8*KP <= STB_SORT_CAP
        base = __shfl_sync(0xffffffffu, base, 0);
        if (take) skeys[base + __popc(m & ((1u << lane) - 1u))] = stb_make_key(snk.ls[e], snk.lr[e]);
      }
    }
    __syncthreads();
    unsigned bound;                                // uniform per CTA from here on
    {
      const int c = (int)s_cnt;
      stb_pad_and_sort(skeys, c, KP);
      const int keep = (gridDim.x == 1) ? KF : KP;
      // warps dropped keys below their own minimum (<= T); the compaction dropped keys < T
      bound = (s_T > kOrdNegInf) ? s_T : 0u;
      if (c > keep) bound = max(bound, stb_f2ord(stb_key_score(skeys[keep - 1])));
    }

    // Everything below writes scratch shared with the PREVIOUS launch on this stream
    // (keys, tickets, exchange slots): wait until that grid has completed and flushed.
    asm volatile("griddepcontrol.wait;" ::: "memory");

    // ---- tree merge across CTAs ------------------------------------------------------------
    // Lists of KP sorted keys (+ their drop bound) are merged F = 1024/KP at a time by the last
    // CTA to arrive in each group (atomic ticket + fences), level by level: 296 -> 10 -> 1 lists
    // at E = 1.  Each merge is one register/shuffle bitonic sort of <= 1024 keys; the groups of a
    // level run in parallel on different SMs.  Level l's lists live at key offset
    // lvl_key_off*KPS, its tickets at counters[lvl_cnt_off + group].
    {
      constexpr int F = STB_SORT_CAP / KP;
      uint32_t lists = gridDim.x, my_id = blockIdx.x, lvl_key_off = 0, lvl_cnt_off = 0;
      while (lists > 1) {
        uint64_t *lvl = tkeys + (size_t)lvl_key_off * KPS;
        for (int i = threadIdx.x; i < KP; i += blockDim.x) lvl[(size_t)my_id * KPS + i] = skeys[i];
        if (threadIdx.x == 0) lvl[(size_t)my_id * KPS + KP] = (uint64_t)bound;
        __threadfence();
        __syncthreads();
        const uint32_t group = my_id / F, first = group * F;
        const uint32_t n_in = min((uint32_t)F, lists - first);
        if (threadIdx.x == 0) s_ticket = atomicAdd(tcnt + lvl_cnt_off + group, 1u);
        __syncthreads();
        if (s_ticket != n_in - 1) return;            // not the last of my group: done
        __threadfence();
        if (threadIdx.x == 0) tcnt[lvl_cnt_off + group] = 0u;   // re-arm for the next launch
        const uint32_t groups = (lists + F - 1) / F;
        const int keep = (groups == 1) ? KF : KP;     // the root keeps the re-rank set
        {
          // Pre-filter before sorting: every list is sorted best-first, so with
          // r = ceil(keep / n_in) - 1 the worst of the lists' r-th keys is a lower bound of the
          // group's keep-th best (n_in * (r+1) >= keep keys are at least that good).  Only keys at
          // or above it can survive the merge -- typically ~100 of the 1024 -- and the sort
          // shrinks from the 1024-key to the 256-key network.  r >= KP (fewer than `keep` keys
          // in total): nothing can be filtered.
          constexpr int PER = STB_SORT_CAP / STB_SCAN_THREADS;
          uint64_t v[PER];
          const uint32_t r = (keep + n_in - 1) / n_in - 1;
          if (threadIdx.x == 0) { s_T64 = (r >= (uint32_t)KP) ? STB_KEY_INVALID : 0ull; s_cnt = 0u; s_bound = 0u; s_nin = 0u; }
          __syncthreads();
          unsigned my_valid = 0;
#pragma unroll
          for (int u = 0; u < PER; ++u) {
            const int i = threadIdx.x + u * STB_SCAN_THREADS;
            const uint32_t li = i / KP;
            v[u] = (li < n_in) ? __ldcg(lvl + (size_t)(first + li) * KPS + (i % KP)) : STB_KEY_INVALID;
            my_valid += (v[u] != STB_KEY_INVALID) ? 1u : 0u;
            if (li < n_in && (uint32_t)(i % KP) == r) atomicMax(&s_T64, v[u]);   // INVALID (all ones) disables the filter
          }
          if (threadIdx.x < n_in) atomicMax(&s_bound, (unsigned)__ldcg(lvl + (size_t)(first + threadIdx.x) * KPS + KP));
          my_valid = __reduce_add_sync(0xffffffffu, my_valid);
          if (lane == 0 && my_valid) atomicAdd(&s_nin, my_valid);
          __syncthreads();
          const uint64_t T = s_T64;
#pragma unroll
          for (int u = 0; u < PER; ++u) {
            const bool take = v[u] != STB_KEY_INVALID && v[u] <= T;
            const unsigned m = __ballot_sync(0xffffffffu, take);
            unsigned base = 0u;
            if (lane == 0 && m) base = atomicAdd(&s_cnt, (unsigned)__popc(m));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (take) skeys[base + __popc(m & ((1u << lane) - 1u))] = v[u];
          }
        }
        __syncthreads();
        stb_pad_and_sort(skeys, (int)s_cnt, KP);
        bound = s_bound;
        if ((int)s_nin > keep) bound = max(bound, stb_f2ord(stb_key_score(skeys[keep - 1])));
        lvl_key_off += lists;
        lvl_cnt_off += groups;
        lists = groups;
        my_id = group;
      }
    }

    // ---- exact re-rank of the best KF in canonical arithmetic --------------------------
    // Rows are staged through shared memory (coalesced, one DRAM latency), then one
    // thread per candidate accumulates (ab, r2) with stb_canon_dot and scores it with stb_canon_dist.
    for (int i = threadIdx.x; i < STB_D; i += blockDim.x) sqd[i] = (double)__ldg(tq + i);
    if (threadIdx.x < 2) s_nv[threadIdx.x] = 0;
    if (threadIdx.x < KF) { s_d[threadIdx.x] = CUDART_INF; s_r[threadIdx.x] = 0xffffffffffffffffull; }
    __syncthreads();
    if (threadIdx.x == 5 * 32) s_q2 = stb_canon_q2(sqd);   // an otherwise idle warp: ||q||^2 once
    // Candidates are sorted by approximate score (or upper bound) best-first and re-scored 32 at a
    // time.  After the first 32 the k-th best EXACT cosine c_k among them is known; a later
    // candidate whose score + eps is below c_k cannot enter the top-k, and neither can anything
    // after it -- with K' = 128 (q8) this usually ends the re-rank after one pass instead of four.
    if (threadIdx.x == 0) { s_cthr = -CUDART_INF; s_done = 0; }
    for (int chunk = 0; chunk < EF; ++chunk) {
      if (chunk > 0) {
        const uint64_t nk = skeys[chunk * 32];                            // uniform
        if (nk == STB_KEY_INVALID || (double)stb_key_score(nk) + kScoreEps < s_cthr) break;
      }
      {
        constexpr int PER = 32 * STB_ROW_F4 / STB_SCAN_THREADS;   // float4 per thread
        float4 v[PER];
#pragma unroll
        for (int u = 0; u < PER; ++u) {
          const int t = threadIdx.x + u * STB_SCAN_THREADS;
          const uint64_t key = skeys[chunk * 32 + (t >> 6)];
          v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (key != STB_KEY_INVALID)
            v[u] = __ldg(args.scan.rows + (size_t)stb_key_row(key) * STB_ROW_F4 + (t & 63));
        }
#pragma unroll
        for (int u = 0; u < PER; ++u) {
          const int t = threadIdx.x + u * STB_SCAN_THREADS;
          *reinterpret_cast<float4 *>(srows + (t >> 6) * STB_RR_STRIDE + (t & 63) * 4) = v[u];
        }
      }
      __syncthreads();
      // 8 candidates per warp on 4 warps (one per SM sub-partition): the f64 chains are
      // latency-bound, so spreading them quarters the issue time
      if (threadIdx.x < 128 && lane < 8) {
        const int cl = (threadIdx.x >> 5) * 8 + lane;          // candidate inside the chunk
        const int ci = chunk * 32 + cl;
        if (skeys[ci] != STB_KEY_INVALID) {
          double ab, r2;
          stb_canon_dot<false>(sqd, reinterpret_cast<const float4 *>(srows + cl * STB_RR_STRIDE), ab, r2);
          s_d[ci] = ab;          // finalised below once ||q||^2 is known
          s_r2[ci] = r2;
        }
      }
      __syncthreads();
      if (threadIdx.x == 0) s_done = chunk + 1;
      if (chunk == 0 && EF > 1 && tk <= 32) {
        if (threadIdx.x < 32) {
          const uint64_t key = skeys[lane];
          double dist = CUDART_INF;
          if (key != STB_KEY_INVALID) {
            dist = stb_canon_dist(s_d[lane], s_q2, s_r2[lane]);
            if (!(dist < STB_DEFAULT_MAX_DIST)) dist = CUDART_INF;
          }
          int rank = 0;
#pragma unroll
          for (int jj = 0; jj < 32; ++jj) {
            const double dj = __shfl_sync(0xffffffffu, dist, jj);
            rank += (dj < dist || (dj == dist && jj < lane)) ? 1 : 0;
          }
          const unsigned passing = __ballot_sync(0xffffffffu, dist < CUDART_INF);
          if ((uint32_t)__popc(passing) >= tk && rank == (int)tk - 1) s_cthr = 1.0 - dist;
        }
        __syncthreads();
      }
    }
    __syncthreads();
    if (threadIdx.x < KF) {
      const uint64_t key = skeys[threadIdx.x];
      double d = CUDART_INF;
      uint64_t grow = 0xffffffffffffffffull;
      if (key != STB_KEY_INVALID) atomicAdd(&s_nv[0], 1);     // valid candidates (re-scored or provably outside the top-k)
      if (key != STB_KEY_INVALID && (int)threadIdx.x < 32 * s_done) {
        const double dist = stb_canon_dist(s_d[threadIdx.x], s_q2, s_r2[threadIdx.x]);
        if (dist < STB_DEFAULT_MAX_DIST) {
          d = dist;
          grow = args.row_base + (uint64_t)stb_key_row(key);
          atomicAdd(&s_nv[1], 1);                   // passing
        }
      }
      s_d[threadIdx.x] = d;
      s_r[threadIdx.x] = grow;
    }
    __syncthreads();
    stb_cta_sort_hits(s_d, s_r, KF);
    const int n_valid = s_nv[0], n_pass = s_nv[1];
    const uint32_t k = tk;
    const uint32_t n_out = min((uint32_t)n_pass, k);
    bool complete;
    if (bound == 0u) complete = true;    // no node dropped a key: every scorable row is a candidate
    else {
      // every row that is not a candidate scored <= the best dropped score
      const float s_drop = stb_ord2f(bound);
      complete = (n_out == k) && ((1.0 - (double)s_drop - kScoreEps) > s_d[k - 1]);
    }
    if (!xchg || args.xchg.world <= 1) {
      stb_write_hits(th, s_d, s_r, n_out, k);
      if (threadIdx.x == 0) {
        ts[0] = n_out;
        ts[1] = complete ? 1u : 0u;
        ts[2] = (uint32_t)n_valid;
        ts[3] = (uint32_t)KF | ((uint32_t)SRC << 16);
      }
      return;
    }

    // ---- fused exchange over NVLink peer memory + global merge ---------------------------
    const StbXchgArgs &X = args.xchg;
    const int world = (int)X.world, me = (int)X.rank;
    const size_t lane_off = (size_t)X.slot * world + me;
    for (int p = 0; p < world; ++p) stb_write_hits(stb_x_hits(X, p) + lane_off * X.max_k, s_d, s_r, n_out, k);
    if (threadIdx.x < world) stb_x_status(X, threadIdx.x)[lane_off] = (complete ? 1u : 0u) | (n_out << 8);
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < world) stb_st_release_sys(stb_x_flags(X, threadIdx.x) + lane_off, X.seq);
    if (threadIdx.x == 0) s_timeout = 0u;
    __syncthreads();
    if (threadIdx.x < world) {
      const unsigned long long *f = stb_x_flags(X, me) + (size_t)X.slot * world + threadIdx.x;
      const long long t0 = clock64();
      while (stb_ld_acquire_sys(f) != X.seq) {
        if (clock64() - t0 > STB_XCHG_TIMEOUT_CYCLES) { s_timeout = 1u; break; }   // a peer is gone
      }
    }
    __syncthreads();
    // merge world x k hits by (distance,row); buffers alias the re-rank staging area
    double *md = reinterpret_cast<double *>(srows);
    uint64_t *mr = reinterpret_cast<uint64_t *>(srows) + 1024;
    const int n_in = world * (int)k;
    int n_sort = 2;
    while (n_sort < n_in) n_sort <<= 1;
    const stb_hit *lh = stb_x_hits(X, me) + (size_t)X.slot * world * X.max_k;
    for (int i = threadIdx.x; i < n_sort; i += blockDim.x) {
      double d = CUDART_INF;
      uint64_t r = 0xffffffffffffffffull;
      if (i < n_in) {
        const stb_hit *src = lh + (size_t)(i / (int)k) * X.max_k + (i % (int)k);
        d = __ldcv(&src->distance);
        r = __ldcv(&src->row);
      }
      md[i] = d; mr[i] = r;
    }
    __syncthreads();
    stb_cta_sort_hits(md, mr, (uint32_t)n_sort);
    stb_write_hits(th, md, mr, k, k);     // n_sort >= world * k: no padding
    if (threadIdx.x == 0) {
      uint32_t all_complete = s_timeout ? 0u : 1u, total = 0u;
      const uint32_t *st = stb_x_status(X, me) + (size_t)X.slot * world;
      for (int p = 0; p < world; ++p) {
        uint32_t v = __ldcv(st + p);
        all_complete &= (v & 1u);
        total += v >> 8;
      }
      ts[0] = min(total, k);
      ts[1] = all_complete;
      ts[2] = s_timeout ? STB_XCHG_STATUS_TIMEOUT : (uint32_t)n_valid;
      ts[3] = (uint32_t)KF | ((uint32_t)SRC << 16);
    }
  };
  // every warp of a pair's host learns the join by its last (failing) draw at the latest: the CTA agrees.  The
  // flag waits in shared memory while the host's tail runs.
  __shared__ int s_pair_joined;
  if constexpr (kPair) {
    if (threadIdx.x == 0) s_pair_joined = 0;
    __syncthreads();
    if (joined && (threadIdx.x & 31) == 0) s_pair_joined = 1;
  }
  tail(sink, args.scan.q, args.top_k, args.out_hits, args.out_status, args.keys, args.counters, true);
  if constexpr (kPair) {
    if (s_pair_joined) {
      const unsigned long long *s = args.pair.seat;
      tail(sink2, reinterpret_cast<const float *>(__ldcg(s + STB_SEAT_Q)), (uint32_t)__ldcg(s + STB_SEAT_INFO),
           reinterpret_cast<stb_hit *>(__ldcg(s + STB_SEAT_HITS)), reinterpret_cast<uint32_t *>(__ldcg(s + STB_SEAT_STATUS)),
           args.pair.keys2, args.pair.counters2, false);
    }
  }
}

template <int E, int U, int RANGES, int SRC = 0, int EF = E>
__global__ void __launch_bounds__(STB_SCAN_THREADS, STB_SCAN_MINB)
stb_scan_topk_kernel(const TopkArgs args) {
  stb_scan_topk_body<E, U, RANGES, SRC, EF>(args);
}

// The q8 tier: at most STB_Q8_SCAN_REGS registers, so that two CTAs leave an SM room for a pair's join kernel
// (__maxnreg__ excludes __launch_bounds__; 256 x 120 x 2 <= 65536 keeps the 2 CTAs per SM).
#define STB_Q8_SCAN_REGS 120
template <int E, int U, int RANGES, int EF>
__global__ void __maxnreg__(STB_Q8_SCAN_REGS)
stb_scan_topk_kernel_q8(const TopkArgs args) {
  stb_scan_topk_body<E, U, RANGES, 2, EF>(args);
}

uint32_t stb_scan_topk_max_k(void) { return 96; }

static int stb_pick_e(uint32_t top_k) {
  if (top_k <= 16) return 1;   // K' = 32
  if (top_k <= 40) return 2;   // K' = 64
  return 4;                    // K' = 128
}

#define STB_SHADOW_SCAN_U 4     // 4 rows x 4 LDG.128 per lane in flight = the f32 path's 2 x 8
#define STB_Q8_SCAN_U 8         // 8 rows x 2 LDG.128

// overlapped: a co-scan launch (no exchange, no ranges; stb_launch_scan_topk)
template <int E, int RANGES, int SRC = 0, int EF = E>
static int stb_launch_topk_t(stb_ctx *ctx, const TopkArgs &a_in, bool overlapped) {
  constexpr int kU = SRC == 2 ? STB_Q4_SCAN_U : (SRC == 1 ? STB_SHADOW_SCAN_U : STB_SCAN_U);
  void (*kern)(const TopkArgs);
  if constexpr (SRC == 2) kern = stb_scan_topk_kernel_q8<E, kU, RANGES, EF>;
  else kern = stb_scan_topk_kernel<E, kU, RANGES, SRC, EF>;
  // resident CTAs per SM the grid is sized for: what the occupancy calculator allows (2 with the
  // 128-register budget)
  int occ = 0;
  STB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, STB_SCAN_THREADS, 0));
  if (occ < 1) occ = 1;
  TopkArgs a = a_in;
  memset(&a.pair, 0, sizeof(a.pair));
  overlapped = overlapped && occ >= 2;
  // q8 whole-shard launches of an overlapped series come in pairs (see "pairs"): a host fills the SMs, and
  // the guest after it is scored by it.  Other overlapped launches: two consecutive grids co-reside, one CTA
  // per SM each.
  const uint64_t tiles = (a.scan.n_virtual + 4 * kU - 1) / (4 * kU);
  const bool pairable = SRC == 2 && RANGES == 0 && overlapped && a.xchg.world == 0 && tiles >= STB_PAIR_MIN_TILES;
  if (overlapped && !pairable) occ = 1;
  a.early_trigger = overlapped ? 1u : 0u;
  uint64_t want = (tiles + STB_SCAN_WARPS - 1) / STB_SCAN_WARPS;
  uint64_t grid = (uint64_t)ctx->sm_count * occ;
  // a pair's host leaves two CTA slots to the pair before it, whose last tail CTA and guest CTA outlive its
  // other CTAs: so the whole grid, and with it the next join kernel, starts while they finish
  if (pairable && grid > 2) grid -= 2;
  if (want < grid) grid = want < 1 ? 1 : want;
  // scratch: lists (KP keys + bound) for all tree levels (< 2 * grid lists), counters (< grid groups)
  size_t need_keys = (size_t)2 * grid * (32 * E + 1) + STB_SORT_CAP;
  if (need_keys > ctx->block_keys.cap || grid + 8 > ctx->counters.cap) {
    stb_set_error("scan scratch too small (grid=%llu)", (unsigned long long)grid);
    return STB_ERR_STATE;
  }
  const uint64_t warps_total = grid * STB_SCAN_WARPS;
  const StbTicketPlan plan = stb_ticket_plan(tiles, warps_total);
  a.scan.t_bulk = plan.t_bulk;
  // a pair host's guest merges its lists through the second half of the scratch
  if (pairable && (2 * need_keys > ctx->block_keys.cap || 2 * (grid + 8) > ctx->counters.cap)) {
    stb_set_error("scan scratch too small for a pair (grid=%llu)", (unsigned long long)grid);
    return STB_ERR_STATE;
  }
  // the launch's number gives its slot and tag (StbScanSeries)
  StbScanSeries &ser = ctx->series;
  if ((uint32_t)++ser.launches == 0) {
    const int rc = ser.reset(ctx->stream);
    if (rc != STB_OK) return rc;
    ++ser.launches;
  }
  const int slot = (int)(ser.launches % STB_TICKET_SLOTS), prev_slot = (int)((ser.launches - 1) % STB_TICKET_SLOTS);
  const uint32_t tag = (uint32_t)ser.launches;
  const StbSeriesLaunch &prev = ser.launch[prev_slot];
  a.scan.tickets = ser.tickets + slot;
  a.scan.t_base = ser.ticket_next[slot];
  ser.ticket_next[slot] += plan.n_tickets + warps_total;
  if constexpr (SRC == 2) {
    a.q4.thr = ser.q4_thr + (size_t)slot * STB_Q4_WORDS;
    a.q4.tag = tag;
  }
  // co-scan: follow the last launch if it was one too, on the same corpus copy and rows (hence the
  // same tiles); any other launch in between -- synchronous, sharded, ranged -- ends the series
  if (overlapped) {
    a.co.word = ser.coscan_off + slot;
    a.co.tag = tag;
    if (prev.coscan && prev.rows == a.scan.rows && prev.src == SRC && prev.n_virtual == a.scan.n_virtual && prev.tiles == tiles) {
      a.co.pred_tag = prev.tag;
      a.co.pred_word = ser.coscan_off + prev_slot;
      a.co.pred_tickets = ser.tickets + prev_slot;
      a.co.pred_t_base = prev.t_base;
      a.co.pred_t_bulk = prev.t_bulk;
    }
  }
  // pairs: a pairable launch right after a host with an open seat on the same rows becomes its guest; a
  // pairable launch that is not a guest opens its own seat
  const bool guest = pairable && prev.seat_open && prev.rows == a.scan.rows && prev.n_virtual == a.scan.n_virtual;
  ser.launch[slot] = StbSeriesLaunch{tag, a.scan.t_base, plan.t_bulk, plan.n_tickets, overlapped, guest ? prev_slot : -1,
                                     a.scan.rows, SRC, a.scan.n_virtual, tiles, pairable && !guest};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;   // PDL, see the kernel
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  if (guest) {
    unsigned long long *seat = ser.seats + (size_t)prev_slot * STB_SEAT_WORDS;
    StbPairJoinArgs j;
    j.seat = seat;
    j.tickets = ser.tickets + prev_slot;
    j.t_base = prev.t_base;
    j.n_tickets = prev.n_tickets;
    j.v_floor = ser.pair_floor;
    j.q = a.scan.q; j.hits = a.out_hits; j.status = a.out_status; j.top_k = a.top_k;
    j.thr = a.q4.thr; j.tag = tag;
    a.pair.decided = seat + STB_SEAT_DECIDED;
    a.pair.tag = tag;
    a.pair.booked = plan.n_tickets + warps_total;
    ser.ticket_next[prev_slot] += STB_PAIR_JUMP;    // the join's jump (a refusing join adds it after the host)
    cudaLaunchConfig_t jc;
    memset(&jc, 0, sizeof(jc));
    jc.gridDim = dim3(1);
    jc.blockDim = dim3(32);
    jc.stream = ctx->stream;
    jc.attrs = attr;
    jc.numAttrs = 1;
    STB_CUDA(cudaLaunchKernelEx(&jc, stb_pair_join_kernel, j));
    ctx->kernel_launches++;
  } else if (pairable) {
    a.pair.seat = ser.seats + (size_t)slot * STB_SEAT_WORDS;
    a.pair.keys2 = ctx->block_keys + need_keys;
    a.pair.counters2 = ctx->counters + grid + 8;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(STB_SCAN_THREADS);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = ctx->stream;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  STB_CUDA(cudaLaunchKernelEx(&cfg, kern, a));
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

template <int RANGES>
static int stb_launch_topk_r(stb_ctx *ctx, const TopkArgs &a, int tier, uint32_t top_k, bool ov) {
  const int e = stb_pick_e(top_k);
  // q8: 32-key lists below the root, 128 candidates re-ranked at the root (see stb_scan_q8)
  if (tier == STB_TIER_Q8) return stb_launch_topk_t<1, RANGES, 2, 4>(ctx, a, ov);
  if (tier == STB_TIER_H16) {
    switch (e) {
      case 1: return stb_launch_topk_t<1, RANGES, 1>(ctx, a, ov);
      case 2: return stb_launch_topk_t<2, RANGES, 1>(ctx, a, ov);
      default: return stb_launch_topk_t<4, RANGES, 1>(ctx, a, ov);
    }
  }
  switch (e) {
    case 1: return stb_launch_topk_t<1, RANGES, 0>(ctx, a, ov);
    case 2: return stb_launch_topk_t<2, RANGES, 0>(ctx, a, ov);
    default: return stb_launch_topk_t<4, RANGES, 0>(ctx, a, ov);
  }
}

int stb_launch_scan_topk(stb_ctx *ctx, const stb_corpus *c, int tier, const float *q_dev, uint32_t top_k,
                         const StbRowRanges &ranges, stb_hit *out_hits_dev, uint32_t *out_status_dev,
                         const StbXchgArgs *xchg, bool overlapped) {
  if (overlapped && (xchg || ranges.n)) { stb_set_error("scan_topk: an overlapped launch takes no exchange or ranges"); return STB_ERR_ARG; }
  TopkArgs a;
  a.scan = stb_scan_args(c, q_dev, ranges);
  memset(&a.co, 0, sizeof(a.co));
  a.row_base = c->row_base;
  a.keys = ctx->block_keys;
  a.counters = ctx->counters;
  a.out_hits = out_hits_dev;
  a.out_status = out_status_dev;
  a.top_k = top_k;
  if (xchg) a.xchg = *xchg; else memset(&a.xchg, 0, sizeof(a.xchg));
  a.early_trigger = 0;
  a.shadow = c->shadow.tiles;
  a.q8 = c->q8.codes;
  a.q8_scale = c->q8.scale;
  memset(&a.q4, 0, sizeof(a.q4));
  if (tier == STB_TIER_Q8 && (top_k > STB_Q8_MAX_K || !c->tier_usable(tier))) { stb_set_error("scan_topk: q8 tier unavailable"); return STB_ERR_STATE; }
  if (tier == STB_TIER_Q8) {
    a.q4.plane = c->q8.plane;   // its threshold words and tag: the launch's slot of the series (stb_launch_topk_t)
    a.q4.sr = c->q8.sr;
    a.q4.top_k = top_k > 0 ? top_k : 1;
    a.q4.refined = ctx->q4_refined;
  }
  if (tier == STB_TIER_H16 && !c->tier_usable(tier)) { stb_set_error("scan_topk: h16 tier unavailable"); return STB_ERR_STATE; }
  return ranges.n > 0 ? stb_launch_topk_r<1>(ctx, a, tier, top_k, overlapped) : stb_launch_topk_r<0>(ctx, a, tier, top_k, overlapped);
}

// ---- the series of top-k launches (StbScanSeries, common.cuh) ----------------------------------------------
int StbScanSeries::init(cudaStream_t stream) {
  int rc;
  if ((rc = tickets.alloc(STB_TICKET_SLOTS)) != STB_OK || (rc = coscan_off.alloc(STB_TICKET_SLOTS)) != STB_OK ||
      (rc = q4_thr.alloc(STB_TICKET_SLOTS * STB_Q4_WORDS)) != STB_OK || (rc = seats.alloc(STB_TICKET_SLOTS * STB_SEAT_WORDS)) != STB_OK)
    return rc;
  return reset(stream);
}

int StbScanSeries::reset(cudaStream_t stream) {
  for (StbBuf<unsigned long long> *b : {&tickets, &coscan_off, &q4_thr, &seats})
    STB_CUDA(cudaMemsetAsync(*b, 0, b->cap * sizeof(unsigned long long), stream));
  memset(ticket_next, 0, sizeof(ticket_next));
  memset(launch, 0, sizeof(launch));
  return STB_OK;
}

void StbScanSeries::forget_rows(const void *rows, bool rewritten) {
  StbSeriesLaunch &last = launch[launches % STB_TICKET_SLOTS];
  if (last.rows != rows) return;
  last.seat_open = false;                // a guest after this starts its own pair
  if (rewritten) last.rows = nullptr;    // the next co-scan starts at tile 0
}

// The slot of the launch `back` launches before the last one (back < STB_TICKET_SLOTS), -1 if there was none.
static int stb_series_recent(const StbScanSeries &s, uint32_t back) {
  if (s.launches <= back) return -1;
  const uint64_t n = s.launches - back;
  const uint32_t tag = s.launch[n % STB_TICKET_SLOTS].tag;
  return tag != 0 && tag == (uint32_t)n ? (int)(n % STB_TICKET_SLOTS) : -1;
}

// K1's tile tickets: every top-k launch must advance the device counter by exactly what the host
// booked for it (n_tickets + total_warps); a mismatch would make later launches skip or repeat
// tiles.  Synchronises; returns STB_ERR_STATE on a mismatch.
int stb_debug_ticket_check(stb_ctx *ctx, uint64_t *device_value, uint64_t *host_value) {
  int rc = stb_ctx_use(ctx);
  if (rc) return rc;
  const StbScanSeries &s = ctx->series;
  unsigned long long v[STB_TICKET_SLOTS];
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  STB_CUDA(cudaMemcpy(v, s.tickets, sizeof(v), cudaMemcpyDeviceToHost));
  unsigned long long dsum = 0, hsum = 0;
  int bad = -1;
  for (int i = 0; i < STB_TICKET_SLOTS; ++i) { dsum += v[i]; hsum += s.ticket_next[i]; if (v[i] != s.ticket_next[i] && bad < 0) bad = i; }
  if (device_value) *device_value = dsum;          // sums over the slots
  if (host_value) *host_value = hsum;
  if (bad >= 0) { stb_set_error("ticket counter %d is %llu, host expects %llu", bad, v[bad], s.ticket_next[bad]); return STB_ERR_STATE; }
  return STB_OK;
}

// The tile offsets K1's last n top-k launches started their pass at, oldest first; 0xffffffff for a launch
// that did not co-scan.  Synchronises.
int stb_debug_coscan_offsets(stb_ctx *ctx, uint32_t n, uint32_t *out) {
  int rc = stb_ctx_use(ctx);
  if (rc) return rc;
  if (n > STB_TICKET_SLOTS || (n && !out)) { stb_set_error("coscan_offsets: n must be 0..%d", STB_TICKET_SLOTS); return STB_ERR_ARG; }
  unsigned long long w[STB_TICKET_SLOTS];
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  STB_CUDA(cudaMemcpy(w, ctx->series.coscan_off, sizeof(w), cudaMemcpyDeviceToHost));
  for (uint32_t i = 0; i < n; ++i) {
    out[i] = 0xffffffffu;
    const int k = stb_series_recent(ctx->series, n - 1 - i);
    if (k >= 0 && ctx->series.launch[k].coscan && (uint32_t)(w[k] >> 32) == ctx->series.launch[k].tag) out[i] = (uint32_t)w[k];
  }
  return STB_OK;
}

// Where K1's last n top-k launches joined their host, oldest first: the join tile (the first tile of the join
// ticket), -1 for a launch that was not a guest, -2 for a guest whose join was refused.  Synchronises.
int stb_debug_pair_joins(stb_ctx *ctx, uint32_t n, int64_t *out) {
  int rc = stb_ctx_use(ctx);
  if (rc) return rc;
  if (n > STB_TICKET_SLOTS || (n && !out)) { stb_set_error("pair_joins: n must be 0..%d", STB_TICKET_SLOTS); return STB_ERR_ARG; }
  unsigned long long w[STB_TICKET_SLOTS * STB_SEAT_WORDS];
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  STB_CUDA(cudaMemcpy(w, ctx->series.seats, sizeof(w), cudaMemcpyDeviceToHost));
  for (uint32_t i = 0; i < n; ++i) {
    out[i] = -1;
    const int k = stb_series_recent(ctx->series, n - 1 - i);
    if (k < 0) continue;
    const StbSeriesLaunch &r = ctx->series.launch[k];
    if (r.host < 0) continue;
    const unsigned long long d = w[r.host * STB_SEAT_WORDS + STB_SEAT_DECIDED];
    if ((uint32_t)(d >> 32) != r.tag) continue;                         // a later pair reused the seat
    out[i] = d & 0x80000000ull ? (int64_t)stb_ticket_first_tile((uint32_t)d & 0x7fffffffu, r.t_bulk) : -2;
  }
  return STB_OK;
}

// Test hook: a join waits until its host has drawn v_floor tickets (0: joins as early as it runs).
int stb_debug_pair_floor(stb_ctx *ctx, uint64_t v_floor) {
  int rc = stb_ctx_use(ctx);
  if (rc) return rc;
  ctx->series.pair_floor = v_floor;
  return STB_OK;
}

// ------------------------------------------------------------------ collect path ---
struct CollectSink {
  float floor_;
  uint32_t *out;
  unsigned long long *count;
  uint64_t cap;
  template <int ROWS>
  __device__ __forceinline__ void consume(float s, uint32_t r) { (*this)(s, r); }
  __device__ __forceinline__ void operator()(float s, uint32_t r) {
    bool hit = (s >= floor_) && (s > -CUDART_INF_F);   // -inf marks lanes that carry no row
    unsigned mask = __ballot_sync(0xffffffffu, hit);
    if (mask == 0) return;
    int lane = threadIdx.x & 31;
    int leader = __ffs(mask) - 1;
    unsigned long long base = 0;
    if (lane == leader) base = atomicAdd(count, (unsigned long long)__popc(mask));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (hit) {
      unsigned long long idx = base + __popc(mask & ((1u << lane) - 1));
      if (idx < cap) out[idx] = r;
    }
  }
};

struct CollectArgs {
  ScanArgs scan;
  float cos_floor;
  uint32_t *out;
  unsigned long long *count;
  uint64_t cap;
  const uint8_t *q8;         // SRC == 2: scores are the q8 tier's upper bounds of the exact cosine
  const float *q8_scale;
};

template <int U, bool RANGES, int SRC = 0>
__global__ void __launch_bounds__(STB_SCAN_THREADS, STB_SCAN_MINB)
stb_scan_collect_kernel(const CollectArgs args) {
  CollectSink sink{args.cos_floor, args.out, args.count, args.cap};
  if constexpr (SRC == 2) stb_scan_q8<U, RANGES>(args.scan, args.q8, args.q8_scale, sink);
  else stb_scan_rows<U, RANGES>(args.scan, sink);
}

int stb_launch_scan_collect(stb_ctx *ctx, const stb_corpus *c, int tier, const float *q_dev, float cos_floor,
                            const StbRowRanges &ranges) {
  CollectArgs a;
  a.scan = stb_scan_args(c, q_dev, ranges);
  a.q8 = c->q8.codes; a.q8_scale = c->q8.scale;
  a.cos_floor = cos_floor;
  a.out = ctx->collect_rows;
  a.count = ctx->collect_count;
  a.cap = ctx->collect_rows.cap;
  STB_CUDA(cudaMemsetAsync(ctx->collect_count, 0, sizeof(unsigned long long), ctx->stream));
  const unsigned grid = stb_scan_grid(ctx, ranges.n_virtual, tier == STB_TIER_Q8 ? STB_Q8_SCAN_U : STB_SCAN_U);
  if (tier == STB_TIER_Q8) {
    if (!c->tier_usable(tier)) { stb_set_error("scan_collect: q8 tier unavailable"); return STB_ERR_STATE; }
    if (ranges.n > 0) stb_scan_collect_kernel<STB_Q8_SCAN_U, true, 2><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a);
    else stb_scan_collect_kernel<STB_Q8_SCAN_U, false, 2><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a);
  } else if (ranges.n > 0)
    stb_scan_collect_kernel<STB_SCAN_U, true><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a);
  else
    stb_scan_collect_kernel<STB_SCAN_U, false><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// ------------------------------------------------------------ histogram pass (large k) ---
// For top_k beyond the register lists: one scan builds a 4096-bin histogram of the
// approximate cosine (bin b covers cos in (1-(b+1)/2048, 1-b/2048]), the host picks the bin that
// contains the k-th best, and the collect pass gathers everything at or above that bin's lower edge
// (minus the score error bound).  Forced candidates (score +inf: rows that cannot be scored safely) are
// not counted: the collect pass takes them whatever the floor, so the k-th bin is the k-th best of the
// scored rows -- counting them would put the floor above a row of the exact top-k.
#define STB_HIST_BINS 4096
struct HistSink {
  unsigned int *hist;   // shared-memory histogram of this CTA
  template <int ROWS>
  __device__ __forceinline__ void consume(float s, uint32_t) {
    if (s > -CUDART_INF_F && s < CUDART_INF_F) {
      float b = floorf((1.0f - s) * (STB_HIST_BINS / 2.0f));
      int bin = b < 0.f ? 0 : (b > (float)(STB_HIST_BINS - 1) ? STB_HIST_BINS - 1 : (int)b);   // NaN cannot occur
      atomicAdd(hist + bin, 1u);
    }
  }
};

template <int U, bool RANGES, int SRC = 0>
__global__ void __launch_bounds__(STB_SCAN_THREADS, STB_SCAN_MINB)
stb_scan_hist_kernel(const ScanArgs scan, unsigned int *global_hist, const uint8_t *q8, const float *q8_scale) {
  __shared__ unsigned int s_hist[STB_HIST_BINS];
  for (int i = threadIdx.x; i < STB_HIST_BINS; i += blockDim.x) s_hist[i] = 0u;
  __syncthreads();
  HistSink sink{s_hist};
  if constexpr (SRC == 2) stb_scan_q8<U, RANGES>(scan, q8, q8_scale, sink);
  else stb_scan_rows<U, RANGES>(scan, sink);
  __syncthreads();
  for (int i = threadIdx.x; i < STB_HIST_BINS; i += blockDim.x)
    if (s_hist[i]) atomicAdd(global_hist + i, s_hist[i]);
}

int stb_launch_scan_hist(stb_ctx *ctx, const stb_corpus *c, int tier, const float *q_dev, const StbRowRanges &ranges,
                         unsigned int *hist_dev) {
  const ScanArgs a = stb_scan_args(c, q_dev, ranges);
  STB_CUDA(cudaMemsetAsync(hist_dev, 0, STB_HIST_BINS * sizeof(unsigned int), ctx->stream));
  const unsigned grid = stb_scan_grid(ctx, ranges.n_virtual, tier == STB_TIER_Q8 ? STB_Q8_SCAN_U : STB_SCAN_U);
  if (tier == STB_TIER_Q8) {
    if (!c->tier_usable(tier)) { stb_set_error("scan_hist: q8 tier unavailable"); return STB_ERR_STATE; }
    if (ranges.n > 0) stb_scan_hist_kernel<STB_Q8_SCAN_U, true, 2><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a, hist_dev, c->q8.codes, c->q8.scale);
    else stb_scan_hist_kernel<STB_Q8_SCAN_U, false, 2><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a, hist_dev, c->q8.codes, c->q8.scale);
  } else if (ranges.n > 0)
    stb_scan_hist_kernel<STB_SCAN_U, true><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a, hist_dev, nullptr, nullptr);
  else
    stb_scan_hist_kernel<STB_SCAN_U, false><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a, hist_dev, nullptr, nullptr);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// ------------------------------------------------------------------- test hooks ---
// stb_debug_scan_scores / stb_debug_q4_scan (api.cu): the production passes with a sink that records, per local
// row, the score the pass handed it and how many times.  Static warp-strided schedule, like the histogram pass.
struct DumpSink {
  float *score;
  unsigned int *seen;
  template <int ROWS>
  __device__ __forceinline__ void consume(float s, uint32_t r) {
    if (s != -CUDART_INF_F) {   // -inf marks lanes that carry no row; a NaN score is recorded
      score[r] = s;
      atomicAdd(seen + r, 1u);
    }
  }
};

template <int U, bool RANGES, int SRC>
__global__ void __launch_bounds__(STB_SCAN_THREADS, STB_SCAN_MINB)
stb_debug_scan_kernel(const ScanArgs scan, const uint8_t *shadow, const uint8_t *q8, const float *q8_scale, DumpSink sink) {
  if constexpr (SRC == 2) stb_scan_q8<U, RANGES>(scan, q8, q8_scale, sink);
  else if constexpr (SRC == 1) stb_scan_shadow<U, RANGES>(scan, shadow, sink);
  else stb_scan_rows<U, RANGES>(scan, sink);
}

int stb_launch_debug_scan(stb_ctx *ctx, const stb_corpus *c, int tier, const float *q_dev, const StbRowRanges &ranges,
                          float *score, unsigned int *seen) {
  const ScanArgs a = stb_scan_args(c, q_dev, ranges);
  const DumpSink sink{score, seen};
  const bool r = ranges.n > 0;
  if (tier == STB_TIER_Q8) {
    const unsigned grid = stb_scan_grid(ctx, ranges.n_virtual, STB_Q8_SCAN_U);
    if (r) stb_debug_scan_kernel<STB_Q8_SCAN_U, true, 2><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a, nullptr, c->q8.codes, c->q8.scale, sink);
    else stb_debug_scan_kernel<STB_Q8_SCAN_U, false, 2><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a, nullptr, c->q8.codes, c->q8.scale, sink);
  } else if (tier == STB_TIER_H16) {
    const unsigned grid = stb_scan_grid(ctx, ranges.n_virtual, STB_SHADOW_SCAN_U);
    if (r) stb_debug_scan_kernel<STB_SHADOW_SCAN_U, true, 1><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a, c->shadow.tiles, nullptr, nullptr, sink);
    else stb_debug_scan_kernel<STB_SHADOW_SCAN_U, false, 1><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a, c->shadow.tiles, nullptr, nullptr, sink);
  } else {
    const unsigned grid = stb_scan_grid(ctx, ranges.n_virtual, STB_SCAN_U);
    if (r) stb_debug_scan_kernel<STB_SCAN_U, true, 0><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a, nullptr, nullptr, nullptr, sink);
    else stb_debug_scan_kernel<STB_SCAN_U, false, 0><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a, nullptr, nullptr, nullptr, sink);
  }
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// stb_scan_q4 with DUMP = 1; its queues live in static shared memory (the top-k kernel lends them its re-rank area)
template <bool RANGES>
__global__ void __launch_bounds__(STB_SCAN_THREADS, STB_SCAN_MINB)
stb_debug_q4_kernel(const ScanArgs scan, const uint8_t *q8, const float *q8_scale, const StbQ4Args q4a, DumpSink sink,
                    const StbQ4Dump dump) {
  __shared__ __align__(16) uint32_t s_scratch[STB_SCAN_WARPS * (STB_Q4_QUEUE + 256)];
  uint32_t *scratch = s_scratch + (threadIdx.x >> 5) * (STB_Q4_QUEUE + 256);
  DumpSink s = sink;
  stb_scan_q4<STB_Q4_SCAN_U, RANGES, 1>(scan, q8, q8_scale, q4a, scratch, scratch + STB_Q4_QUEUE, s, nullptr, &dump);
}

int stb_launch_debug_q4(stb_ctx *ctx, const stb_corpus *c, const float *q_dev, uint32_t top_k, const StbRowRanges &ranges,
                        unsigned long long *words, unsigned long long *refined, int pin, float *u4, float *t, float *l8,
                        float *u8, unsigned int *seen) {
  const ScanArgs a = stb_scan_args(c, q_dev, ranges);
  StbQ4Args q4a;
  q4a.plane = c->q8.plane;
  q4a.sr = c->q8.sr;
  q4a.thr = words;
  q4a.tag = 1u;
  q4a.top_k = top_k;
  q4a.refined = refined;
  const DumpSink sink{u8, seen};
  const StbQ4Dump dump{u4, t, l8, pin};
  const unsigned grid = stb_scan_grid(ctx, ranges.n_virtual, STB_Q4_SCAN_U);
  if (ranges.n > 0) stb_debug_q4_kernel<true><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a, c->q8.codes, c->q8.scale, q4a, sink, dump);
  else stb_debug_q4_kernel<false><<<grid, STB_SCAN_THREADS, 0, ctx->stream>>>(a, c->q8.codes, c->q8.scale, q4a, sink, dump);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// Exact canonical distance of each collected row; one thread per row.
__global__ void stb_exact_kernel(const float4 *rows, uint64_t row_base, const float *q,
                                 const uint32_t *row_ids, uint64_t m, double limit,
                                 stb_hit *hits, uint64_t m_padded,
                                 unsigned long long *pass_count) {
  __shared__ double sqd[STB_D];
  __shared__ double s_q2;
  for (int i = threadIdx.x; i < STB_D; i += blockDim.x) sqd[i] = (double)__ldg(q + i);
  __syncthreads();
  if (threadIdx.x == 0) s_q2 = stb_canon_q2(sqd);
  __syncthreads();
  uint64_t idx = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= m_padded) return;
  stb_hit h;
  h.distance = CUDART_INF;
  h.row = 0xffffffffffffffffull;
  if (idx < m) {
    uint32_t row = row_ids[idx];
    double ab, r2;
    stb_canon_dot<true>(sqd, rows + (size_t)row * STB_ROW_F4, ab, r2);
    const double dist = stb_canon_dist(ab, s_q2, r2);
    if (dist < limit) {
      h.distance = dist;
      h.row = row_base + (uint64_t)row;
      atomicAdd(pass_count, 1ull);
    }
  }
  hits[idx] = h;
}

int stb_launch_exact(stb_ctx *ctx, const float *rows, uint64_t row_base,
                     const float *q_dev, const uint32_t *row_ids, uint64_t m,
                     double limit, stb_hit *hits, uint64_t m_padded,
                     unsigned long long *pass_count) {
  STB_CUDA(cudaMemsetAsync(pass_count, 0, sizeof(unsigned long long), ctx->stream));
  if (m_padded == 0) return STB_OK;
  unsigned blocks = (unsigned)((m_padded + 127) / 128);
  stb_exact_kernel<<<blocks, 128, 0, ctx->stream>>>(reinterpret_cast<const float4 *>(rows),
                                                     row_base, q_dev, row_ids, m, limit, hits,
                                                     m_padded, pass_count);
  STB_CUDA(cudaGetLastError());
  ctx->kernel_launches++;
  return STB_OK;
}

// Global bitonic sort of hits by (distance,row): one launch per (k,j) step above
// the shared-memory span, fused steps inside a 1024-element span.
__global__ void stb_bitonic_global_step(stb_hit *h, uint64_t n, uint64_t k, uint64_t j) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t ixj = i ^ j;
  if (ixj > i) {
    stb_hit a = h[i], b = h[ixj];
    bool up = ((i & k) == 0);
    bool gt = stb_hit_less(b.distance, b.row, a.distance, a.row);
    if (gt == up) { h[i] = b; h[ixj] = a; }
  }
}

// Sorts all steps with j < 1024 of stage k inside shared memory (span 1024).
__global__ void stb_bitonic_local(stb_hit *h, uint64_t n, uint64_t k_first, uint64_t k_last) {
  __shared__ double sd[1024];
  __shared__ uint64_t sr[1024];
  const uint64_t base = (uint64_t)blockIdx.x * 1024;
  for (int t = threadIdx.x; t < 1024; t += blockDim.x) {
    stb_hit x = h[base + t];
    sd[t] = x.distance; sr[t] = x.row;
  }
  __syncthreads();
  for (uint64_t k = k_first; k <= k_last; k <<= 1) {
    uint64_t jstart = (k >> 1) < 512 ? (k >> 1) : 512;
    for (uint64_t j = jstart; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < 1024; t += blockDim.x) {
        uint64_t i = base + t, ixj = i ^ j;
        if (ixj > i) {
          int u = (int)(ixj - base);
          bool up = ((i & k) == 0);
          bool gt = stb_hit_less(sd[u], sr[u], sd[t], sr[t]);
          if (gt == up) {
            double td = sd[t]; uint64_t tr = sr[t];
            sd[t] = sd[u]; sr[t] = sr[u]; sd[u] = td; sr[u] = tr;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int t = threadIdx.x; t < 1024; t += blockDim.x) {
    stb_hit x; x.distance = sd[t]; x.row = sr[t];
    h[base + t] = x;
  }
}

int stb_launch_sort_hits(stb_ctx *ctx, stb_hit *hits, uint64_t n) {
  if (n < 2) return STB_OK;
  if (n < 1024 || (n & (n - 1))) { stb_set_error("sort size must be a power of two >= 1024"); return STB_ERR_ARG; }
  unsigned lblocks = (unsigned)(n / 1024);
  // stages k = 2..1024 entirely local
  stb_bitonic_local<<<lblocks, 256, 0, ctx->stream>>>(hits, n, 2, 1024);
  ctx->kernel_launches++;
  for (uint64_t k = 2048; k <= n; k <<= 1) {
    for (uint64_t j = k >> 1; j >= 1024; j >>= 1) {
      unsigned gblocks = (unsigned)((n + 255) / 256);
      stb_bitonic_global_step<<<gblocks, 256, 0, ctx->stream>>>(hits, n, k, j);
      ctx->kernel_launches++;
    }
    stb_bitonic_local<<<lblocks, 256, 0, ctx->stream>>>(hits, n, k, k);
    ctx->kernel_launches++;
  }
  STB_CUDA(cudaGetLastError());
  return STB_OK;
}

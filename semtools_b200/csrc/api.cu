// C ABI of libsemtools_b200.so (include/semtools_b200.h).  Host-side orchestration
// only: argument checking, HBM residency, staging copies, and the exact
// fallback ladder around the scan kernel.  No CPU implementation of any kernel
// exists in this library: without an sm_90 device every entry point fails.
#include <stdarg.h>
#include <stdlib.h>

#include <algorithm>
#include <cmath>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "common.cuh"
#include "row_encode.cuh"

static thread_local char g_err[512] = "";

void stb_set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// ------------------------------------------------------------------- context ---
// Live-context registry: tables/corpora may outlive their context (garbage-collected
// host languages destroy in any order); their destructors must not touch a dead one.
static std::mutex g_ctx_mu;
static std::unordered_set<const stb_ctx *> g_ctx_live;
static bool ctx_alive(const stb_ctx *ctx) {
  std::lock_guard<std::mutex> lk(g_ctx_mu);
  return g_ctx_live.count(ctx) != 0;
}

static int ctx_use(const stb_ctx *ctx) {
  if (!ctx) { stb_set_error("null context"); return STB_ERR_ARG; }
  if (!ctx_alive(ctx)) { stb_set_error("context was destroyed"); return STB_ERR_STATE; }
  STB_CUDA(cudaSetDevice(ctx->device));
  return STB_OK;
}

int stb_ctx_use(const stb_ctx *ctx) { return ctx_use(ctx); }
bool stb_ctx_alive(const stb_ctx *ctx) { return ctx_alive(ctx); }

bool stb_ranges_ordered(const uint64_t *ranges, uint32_t n) {
  uint64_t prev_end = 0;
  for (uint32_t i = 0; i < n; ++i) {
    const uint64_t b = ranges[2 * i], e = ranges[2 * i + 1];
    if (e < b || (i > 0 && b < prev_end)) return false;
    prev_end = e;
  }
  return true;
}

extern "C" {

int stb_version(void) { return 100; }
const char *stb_last_error(void) { return g_err; }

int stb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int stb_ctx_create(int device, void *cuda_stream, stb_ctx **out) {
  if (!out) { stb_set_error("out is null"); return STB_ERR_ARG; }
  *out = nullptr;
  int n = stb_device_count();
  if (n <= 0) { stb_set_error("no CUDA device visible (this library has no CPU path)"); return STB_ERR_CUDA; }
  if (device < 0 || device >= n) { stb_set_error("device %d out of range (0..%d)", device, n - 1); return STB_ERR_ARG; }
  STB_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  STB_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    stb_set_error("device %d is sm_%d%d; libsemtools_b200 ships sm_90a code only", device, prop.major, prop.minor);
    return STB_ERR_CUDA;
  }
  stb_ctx *c = new (std::nothrow) stb_ctx();
  if (!c) { stb_set_error("out of host memory"); return STB_ERR_NOMEM; }
  c->device = device;
  c->sm_count = prop.multiProcessorCount;
  if (cuda_stream) { c->stream = (cudaStream_t)cuda_stream; c->own_stream = false; }
  else {
    cudaError_t e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) { stb_set_error("cudaStreamCreate: %s", cudaGetErrorString(e)); delete c; return STB_ERR_CUDA; }
    c->own_stream = true;
  }
  int rc = STB_OK;
  const size_t max_grid = (size_t)c->sm_count * 8;
  if ((rc = c->block_keys.alloc(2 * max_grid * 129 + STB_SORT_CAP)) != STB_OK ||
      (rc = c->counters.alloc(max_grid + 64)) != STB_OK ||
      (rc = c->q_dev.alloc(STB_D)) != STB_OK ||
      (rc = c->status_dev.alloc(8)) != STB_OK ||
      (rc = c->collect_count.alloc(2)) != STB_OK ||
      (rc = c->err_flag.alloc(1)) != STB_OK ||
      (rc = c->embed_flag.alloc(1)) != STB_OK ||
      (rc = c->hist_dev.alloc(4096)) != STB_OK ||
      (rc = c->series.init(c->stream)) != STB_OK ||
      (rc = c->q4_refined.alloc(1)) != STB_OK ||
      (rc = c->hits_dev.alloc(1024)) != STB_OK ||
      (rc = c->q_pin.alloc(STB_D)) != STB_OK ||
      (rc = c->status_pin.alloc(8)) != STB_OK ||
      (rc = c->hits_pin.alloc(1024)) != STB_OK)
    goto fail;
  if (cudaMemset(c->counters, 0, c->counters.cap * sizeof(unsigned int)) != cudaSuccess ||
      cudaMemset(c->q4_refined, 0, sizeof(unsigned long long)) != cudaSuccess ||
      cudaMemset(c->err_flag, 0, sizeof(int)) != cudaSuccess ||
      cudaMemset(c->embed_flag, 0, sizeof(int)) != cudaSuccess) {
    stb_set_error("context staging allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
    rc = STB_ERR_NOMEM;
    goto fail;
  }
  { std::lock_guard<std::mutex> lk(g_ctx_mu); g_ctx_live.insert(c); }
  *out = c;
  return STB_OK;
fail:
  stb_ctx_destroy(c);
  return rc;
}

int stb_ctx_destroy(stb_ctx *c) {
  if (!c) return STB_OK;
  { std::lock_guard<std::mutex> lk(g_ctx_mu); g_ctx_live.erase(c); }
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  const cudaStream_t own = c->own_stream ? c->stream : nullptr;
  delete c;   // the buffers go with it
  if (own) cudaStreamDestroy(own);
  cudaGetLastError();
  return STB_OK;
}

int stb_ctx_sync(stb_ctx *ctx) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  return STB_OK;
}

void *stb_ctx_stream(stb_ctx *ctx) { return ctx ? (void *)ctx->stream : nullptr; }

// Rows the q8 tier's prefilter passed on to the int8 codes, summed over the top-k launches since the
// last reset.  Synchronises.
int stb_debug_q4_refined(stb_ctx *ctx, int reset, uint64_t *refined) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  unsigned long long v = 0;
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  STB_CUDA(cudaMemcpy(&v, ctx->q4_refined, sizeof(v), cudaMemcpyDeviceToHost));
  if (reset) STB_CUDA(cudaMemset(ctx->q4_refined, 0, sizeof(v)));
  if (refined) *refined = v;
  return STB_OK;
}

int stb_ctx_counters(const stb_ctx *ctx, uint64_t *kernel_launches, uint64_t *fallback_searches) {
  if (!ctx) { stb_set_error("null context"); return STB_ERR_ARG; }
  if (kernel_launches) *kernel_launches = ctx->kernel_launches;
  if (fallback_searches) *fallback_searches = ctx->fallback_searches;
  return STB_OK;
}

// --------------------------------------------------------------------- table ---
int stb_table_load(stb_ctx *ctx, const float *E, uint64_t V, uint32_t D, const float *weights,
                   uint64_t n_weights, const uint32_t *mapping, uint64_t n_mapping, int normalize,
                   stb_table **out) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!out || !E || V == 0) { stb_set_error("table_load: null/empty table"); return STB_ERR_ARG; }
  if (D != STB_D) { stb_set_error("table_load: D=%u, only %u supported", D, STB_D); return STB_ERR_ARG; }
  if (V > 0xffffffffull) { stb_set_error("table_load: V exceeds 2^32 rows"); return STB_ERR_ARG; }
  stb_table *t = new (std::nothrow) stb_table();
  if (!t) { stb_set_error("out of host memory"); return STB_ERR_NOMEM; }
  t->ctx = ctx; t->V = V; t->normalize = normalize ? 1 : 0;
  t->n_weights = weights ? n_weights : 0;
  t->n_mapping = mapping ? n_mapping : 0;
  if ((rc = t->E.alloc(V * STB_D)) != STB_OK || (t->n_weights && (rc = t->weights.alloc(t->n_weights)) != STB_OK) ||
      (t->n_mapping && (rc = t->mapping.alloc(t->n_mapping)) != STB_OK)) {
    stb_table_destroy(t);
    return rc;
  }
  cudaError_t e = cudaMemcpyAsync(t->E, E, V * STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess && t->n_weights)
    e = cudaMemcpyAsync(t->weights, weights, t->n_weights * sizeof(float), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess && t->n_mapping)
    e = cudaMemcpyAsync(t->mapping, mapping, t->n_mapping * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (e != cudaSuccess) {
    stb_set_error("table_load: upload failed: %s", cudaGetErrorString(e));
    stb_table_destroy(t);
    return STB_ERR_CUDA;
  }
  *out = t;
  return STB_OK;
}

int stb_table_destroy(stb_table *t) {
  if (!t) return STB_OK;
  if (t->ctx && ctx_alive(t->ctx)) { cudaSetDevice(t->ctx->device); cudaStreamSynchronize(t->ctx->stream); }
  else cudaDeviceSynchronize();
  cudaGetLastError();
  delete t;
  return STB_OK;
}

// -------------------------------------------------------------------- corpus ---
// A grown corpus copy gets the first `bytes` of the old one: copied on the stream and waited for, also when the
// copy fails, so either buffer may be freed on return.
static int copy_prefix(stb_ctx *ctx, void *dst, const void *src, size_t bytes) {
  cudaError_t e = bytes ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, ctx->stream) : cudaSuccess;
  const cudaError_t se = cudaStreamSynchronize(ctx->stream);
  if (e == cudaSuccess) e = se;
  if (e != cudaSuccess) { stb_set_error("corpus grow copy: %s", cudaGetErrorString(e)); return STB_ERR_CUDA; }
  return STB_OK;
}

}  // extern "C"
// ---- the candidate copies (StbCopy, common.cuh) ----
// What sets the two copies apart beyond their buffers: growth to room for `cap` rows that keeps the first `keep`
// (nothing changes when an allocation fails), the builder of rows [r0, r1) from rows_dev, whose first row is
// row rows_first, and the message of a copy that holds rows which cannot be normalised.
static int copy_realloc(stb_ctx *ctx, StbShadowCopy &k, uint64_t cap, uint64_t keep) {
  StbShadowBufs g;
  int rc;
  if ((rc = g.tiles.alloc(StbShadowBufs::bytes(cap))) != STB_OK ||
      (rc = copy_prefix(ctx, g.tiles, k.tiles, StbShadowBufs::bytes(keep))) != STB_OK)   // keep: whole tiles
    return rc;
  static_cast<StbShadowBufs &>(k) = std::move(g);
  return STB_OK;
}
// int8 codes + scales, 260 B/row, and the top-k prefilter's nibble plane + {s, rho}, 136 B/row
static int copy_realloc(stb_ctx *ctx, StbQ8Copy &k, uint64_t cap, uint64_t keep) {
  StbQ8Bufs g;
  int rc;
  if ((rc = g.codes.alloc(cap * 256ull)) != STB_OK || (rc = g.scale.alloc(cap)) != STB_OK ||
      (rc = g.plane.alloc(stb_q4_plane_bytes(cap))) != STB_OK || (rc = g.sr.alloc(cap)) != STB_OK)
    return rc;
  if (k.allocated() && keep &&
      ((rc = copy_prefix(ctx, g.codes, k.codes, keep * 256ull)) != STB_OK ||
       (rc = copy_prefix(ctx, g.scale, k.scale, keep * sizeof(float))) != STB_OK ||
       (rc = copy_prefix(ctx, g.plane, k.plane, stb_q4_plane_bytes(keep))) != STB_OK ||   // whole tiles
       (rc = copy_prefix(ctx, g.sr, k.sr, keep * sizeof(float2))) != STB_OK))
    return rc;
  static_cast<StbQ8Bufs &>(k) = std::move(g);
  return STB_OK;
}
static int copy_build(stb_ctx *ctx, StbShadowCopy &k, const float *rows_dev, uint64_t r0, uint64_t r1, uint64_t rows_first) {
  return stb_launch_shadow_build(ctx, rows_dev, r1, 256, k.tiles, ctx->err_flag, r0, nullptr, rows_first);
}
static int copy_build(stb_ctx *ctx, StbQ8Copy &k, const float *rows_dev, uint64_t r0, uint64_t r1, uint64_t rows_first) {
  return stb_launch_q8_build(ctx, rows_dev, r0, r1, k.codes, k.scale, k.plane, k.sr, ctx->err_flag, rows_first);
}
static const char *copy_bad_rows(const StbShadowCopy &) {
  return "search_batch: corpus holds rows whose norm is not a normal fp32 number; use stb_search";
}
static const char *copy_bad_rows(const StbQ8Copy &) { return "q8 tier: corpus holds rows whose norm is not a normal fp32 number"; }

// Rows [first, n) of a host-rows corpus for a copy builder: uploaded into the context's staging buffer in chunks
// of at most STB_MUT_CHUNK_ROWS rows (a multiple of the shadow's 256-row tile), fn(stage, r0, r1, r0) per chunk.
template <class F>
static int host_rows_staged(stb_corpus *c, uint64_t first, F &&fn) {
  stb_ctx *ctx = c->ctx;
  if (first >= c->n) return STB_OK;
  const uint64_t chunk = std::min<uint64_t>(c->n - first, STB_MUT_CHUNK_ROWS);
  int rc;
  if ((rc = ctx->mut_stage.reserve(chunk * STB_D)) != STB_OK) return rc;
  for (uint64_t r0 = first; r0 < c->n; r0 += chunk) {
    const uint64_t m = std::min(chunk, c->n - r0);
    STB_CUDA(cudaMemcpyAsync(ctx->mut_stage, c->rows_host + r0 * STB_D, m * STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = fn(ctx->mut_stage, r0, r0 + m, r0)) != STB_OK) return rc;
  }
  return STB_OK;
}

// The one build-or-extend of a copy: makes it cover every row, converting only the rows behind its usable prefix
// (all of them when it has none or is bad), from HBM or, on a host-rows corpus, through the staging buffer.  A
// host-rows corpus gets here for its shadow, or to re-encode a q8 copy a mutation dropped as unusable.
// STB_ERR_STATE: the copy holds rows that cannot be normalised in fp32, and is unusable.
template <class Copy>
static int corpus_ensure(stb_ctx *ctx, stb_corpus *c, Copy &k) {
  if (!k.covers(c->n)) {
    const uint64_t first = k.prefix(c->n);
    int rc;
    if (!k.has_room(c->n) && (rc = copy_realloc(ctx, k, std::max<uint64_t>(c->n, c->capacity), first)) != STB_OK) return rc;
    STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
    const auto build = [&](const float *rows, uint64_t r0, uint64_t r1, uint64_t rows_first) {
      return copy_build(ctx, k, rows, r0, r1, rows_first);
    };
    if ((rc = c->host_rows ? host_rows_staged(c, first, build) : build(c->rows, first, c->n, 0)) != STB_OK) return rc;
    int flag = 0;
    STB_CUDA(cudaMemcpyAsync(&flag, ctx->err_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
    STB_CUDA(cudaStreamSynchronize(ctx->stream));
    k.rows = c->n;
    k.bad = flag != 0;
  }
  if (k.bad) { stb_set_error("%s", copy_bad_rows(k)); return STB_ERR_STATE; }
  return STB_OK;
}
extern "C" {

// A host-rows corpus grows both halves together: new mapped rows and a new q8 copy, then the old ones are
// copied and freed (so growing briefly holds two host buffers).  A failed allocation changes nothing.
static int host_corpus_reserve(stb_corpus *c, uint64_t ncap) {
  stb_ctx *ctx = c->ctx;
  StbBuf<float, STB_MEM_MAPPED> grown;
  cudaError_t e = cudaSuccess;
  if (grown.alloc(ncap * STB_D, &e) != STB_OK) {
    stb_set_error("corpus: cannot allocate %llu rows of page-locked host memory: %s", (unsigned long long)ncap, cudaGetErrorString(e));
    return STB_ERR_NOMEM;
  }
  int rc = copy_realloc(ctx, c->q8, ncap, c->n);
  if (rc != STB_OK) return rc;
  STB_CUDA(cudaStreamSynchronize(ctx->stream));   // kernels write the rows (update, remove)
  if (c->rows_host) memcpy(grown, c->rows_host, c->n * STB_D * sizeof(float));
  c->rows_host = std::move(grown);
  c->rows = c->rows_host.dev;
  c->capacity = ncap;
  return STB_OK;
}

static int corpus_reserve(stb_corpus *c, uint64_t need) {
  if (need <= c->capacity && c->rows) return STB_OK;
  if (need > 0xfffffffeull) { stb_set_error("corpus shard exceeds 2^32-2 rows; shard it"); return STB_ERR_ARG; }
  uint64_t ncap = std::max<uint64_t>(std::max<uint64_t>(need, 1024), c->capacity + c->capacity / 2);
  if (c->host_rows) return host_corpus_reserve(c, ncap);
  StbBuf<float> grown;
  int rc;
  if ((rc = grown.alloc(ncap * STB_D)) != STB_OK) return rc;
  if (c->rows && c->n && (rc = copy_prefix(c->ctx, grown, c->rows, c->n * STB_D * sizeof(float))) != STB_OK) return rc;
  c->dev_rows = std::move(grown);
  c->rows = c->dev_rows;
  c->capacity = ncap;
  return STB_OK;
}

int stb_corpus_create(stb_ctx *ctx, uint32_t D, uint64_t capacity_rows, uint64_t row_base, stb_corpus **out) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!out) { stb_set_error("out is null"); return STB_ERR_ARG; }
  if (D != STB_D) { stb_set_error("corpus_create: D=%u, only %u supported", D, STB_D); return STB_ERR_ARG; }
  stb_corpus *c = new (std::nothrow) stb_corpus();
  if (!c) { stb_set_error("out of host memory"); return STB_ERR_NOMEM; }
  c->ctx = ctx; c->row_base = row_base;
  rc = corpus_reserve(c, std::max<uint64_t>(capacity_rows, 1));
  if (rc) { delete c; return rc; }
  *out = c;
  return STB_OK;
}

int stb_corpus_create_host(stb_ctx *ctx, uint32_t D, uint64_t capacity_rows, uint64_t row_base, stb_corpus **out) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!out) { stb_set_error("out is null"); return STB_ERR_ARG; }
  if (D != STB_D) { stb_set_error("corpus_create_host: D=%u, only %u supported", D, STB_D); return STB_ERR_ARG; }
  if (capacity_rows > 0xfffffffeull) { stb_set_error("corpus shard exceeds 2^32-2 rows; shard it"); return STB_ERR_ARG; }
  stb_corpus *c = new (std::nothrow) stb_corpus();
  if (!c) { stb_set_error("out of host memory"); return STB_ERR_NOMEM; }
  c->ctx = ctx; c->row_base = row_base; c->host_rows = 1;
  rc = host_corpus_reserve(c, std::max<uint64_t>(capacity_rows, 1));
  if (rc) { delete c; return rc; }
  *out = c;
  return STB_OK;
}

int stb_corpus_destroy(stb_corpus *c) {
  if (!c) return STB_OK;
  if (c->ctx && ctx_alive(c->ctx)) { cudaSetDevice(c->ctx->device); cudaStreamSynchronize(c->ctx->stream); }
  else cudaDeviceSynchronize();
  cudaGetLastError();
  delete c;
  return STB_OK;
}

// The reduced-width copies (K2 shadow, K1 tiers) cover a PREFIX of the rows: an append leaves the
// prefix valid and the next query / prepare only converts the new rows (StbCopy::rows < n);
// an update or a removal re-encodes the copies at the rows it writes, so they stay built; a clear drops
// them.  Anything but an append starts a new epoch; an update or a removal also ends a co-scan series on
// the corpus (the next asynchronous top-k query starts at tile 0).
enum CorpusChange { CORPUS_APPEND, CORPUS_ROWS_REWRITTEN, CORPUS_CLEAR };
static void corpus_changed(stb_corpus *c, CorpusChange kind) {
  if (kind == CORPUS_CLEAR) { c->shadow.drop(); c->q8.drop(); }
  if (kind != CORPUS_APPEND) ++c->epoch;
  c->ctx->series.forget_rows(c->rows, kind == CORPUS_ROWS_REWRITTEN);
  c->searches_since_change = 0;
  memset(c->tier_tries, 0, sizeof(c->tier_tries));
  memset(c->tier_proven, 0, sizeof(c->tier_proven));
}

// The commit kernel's arguments (corpus_update.cu): the rows, the staging buffer, and each allocated copy with the
// rows of it the kernel keeps current; it raises flags[0] for a q8 row and flags[1] for a shadow row that cannot
// be normalised.
static StbCorpusWriteArgs corpus_write_args(stb_corpus *c, uint64_t q8_cover, uint64_t shadow_cover) {
  StbCorpusWriteArgs a;
  memset(&a, 0, sizeof(a));
  a.rows = reinterpret_cast<float4 *>(c->rows);
  a.stage = reinterpret_cast<const float4 *>(c->ctx->mut_stage.p);
  a.q8 = c->q8.codes; a.q8_scale = c->q8.scale; a.q4 = c->q8.plane; a.q4_sr = c->q8.sr;
  a.q8_rows = c->q8.allocated() ? q8_cover : 0;
  a.shadow = c->shadow.tiles;
  a.shadow_rows = c->shadow.allocated() ? shadow_cover : 0;
  a.flags = c->ctx->mut_flags;
  return a;
}

// Appending to a host-rows corpus: staged rows [0, m) become rows first .. first + m - 1.  The commit kernel of the
// in-place mutations writes them to the host rows and encodes their q8 entries from HBM in the same pass; the
// 16-bit shadow stays the prefix it was.  The caller books the rows (host_append_finish) once every chunk is in.
static int host_append_chunk(stb_corpus *c, const float *stage_dev, uint64_t first, uint64_t m) {
  StbCorpusWriteArgs a = corpus_write_args(c, first + m, 0);
  a.stage = reinterpret_cast<const float4 *>(stage_dev);
  a.first = first;
  a.m = m;
  return stb_launch_corpus_write(c->ctx, a);
}
static int host_append_begin(stb_corpus *c, uint64_t n, uint64_t stage_rows) {
  stb_ctx *ctx = c->ctx;
  int rc;
  if ((rc = corpus_reserve(c, c->n + n)) != STB_OK) return rc;
  if (stage_rows && (rc = ctx->mut_stage.reserve(stage_rows * STB_D)) != STB_OK) return rc;
  if ((rc = ctx->mut_flags.reserve(2)) != STB_OK) return rc;
  STB_CUDA(cudaMemsetAsync(ctx->mut_flags, 0, 2 * sizeof(int), ctx->stream));
  return STB_OK;
}
// synchronises; a row of the call that cannot be normalised marks the q8 copy unusable, as a build does
static int host_append_finish(stb_corpus *c, uint64_t n) {
  int flags[2] = {0, 0};
  STB_CUDA(cudaMemcpyAsync(flags, c->ctx->mut_flags, sizeof(flags), cudaMemcpyDeviceToHost, c->ctx->stream));
  STB_CUDA(cudaStreamSynchronize(c->ctx->stream));
  c->n += n;
  c->q8.rows = c->n;
  c->q8.mark_bad(flags[0]);
  corpus_changed(c, CORPUS_APPEND);
  return STB_OK;
}

static int corpus_append_impl(stb_corpus *c, const float *rows, uint64_t n, cudaMemcpyKind kind) {
  if (!c) { stb_set_error("null corpus"); return STB_ERR_ARG; }
  int rc = ctx_use(c->ctx);
  if (rc) return rc;
  if (n == 0) return STB_OK;
  if (!rows) { stb_set_error("corpus_append: rows is null"); return STB_ERR_ARG; }
  if (c->host_rows) {
    // host rows: each row goes up once (through the staging buffer unless it is in HBM already)
    const bool up = kind == cudaMemcpyHostToDevice;
    const uint64_t chunk = std::min<uint64_t>(n, STB_MUT_CHUNK_ROWS);
    if ((rc = host_append_begin(c, n, up ? chunk : 0)) != STB_OK) return rc;
    for (uint64_t i0 = 0; i0 < n; i0 += chunk) {
      const uint64_t m = std::min(chunk, n - i0);
      const float *src = rows + i0 * STB_D;
      if (up) {   // stream order keeps the copy behind the previous chunk's kernel
        STB_CUDA(cudaMemcpyAsync(c->ctx->mut_stage, src, m * STB_D * sizeof(float), cudaMemcpyHostToDevice, c->ctx->stream));
        src = c->ctx->mut_stage;
      }
      if ((rc = host_append_chunk(c, src, c->n + i0, m)) != STB_OK) return rc;
    }
    return host_append_finish(c, n);
  }
  if ((rc = corpus_reserve(c, c->n + n)) != STB_OK) return rc;
  STB_CUDA(cudaMemcpyAsync(c->rows + c->n * STB_D, rows, n * STB_D * sizeof(float), kind, c->ctx->stream));
  STB_CUDA(cudaStreamSynchronize(c->ctx->stream));
  c->n += n;
  corpus_changed(c, CORPUS_APPEND);
  return STB_OK;
}

int stb_corpus_append(stb_corpus *c, const float *rows, uint64_t n) {
  return corpus_append_impl(c, rows, n, cudaMemcpyHostToDevice);
}
int stb_corpus_append_dev(stb_corpus *c, const float *rows_dev, uint64_t n) {
  return corpus_append_impl(c, rows_dev, n, cudaMemcpyDeviceToDevice);
}
int stb_corpus_clear(stb_corpus *c) {
  if (!c) { stb_set_error("null corpus"); return STB_ERR_ARG; }
  if (!ctx_alive(c->ctx)) { stb_set_error("context was destroyed"); return STB_ERR_STATE; }
  c->n = 0;
  corpus_changed(c, CORPUS_CLEAR);
  return STB_OK;
}
int stb_corpus_rows(const stb_corpus *c, uint64_t *n) {
  if (!c || !n) { stb_set_error("null argument"); return STB_ERR_ARG; }
  *n = c->n;
  return STB_OK;
}
int stb_corpus_data_dev(const stb_corpus *c, float **rows_dev) {
  if (!c || !rows_dev) { stb_set_error("null argument"); return STB_ERR_ARG; }
  if (c->host_rows) { stb_set_error("corpus_data_dev: the rows of this corpus are in host memory; there is no device matrix"); return STB_ERR_STATE; }
  *rows_dev = c->rows;
  return STB_OK;
}
int stb_corpus_read(const stb_corpus *c, uint64_t first, uint64_t n, float *rows) {
  if (!c || (!rows && n)) { stb_set_error("null argument"); return STB_ERR_ARG; }
  int rc = ctx_use(c->ctx);
  if (rc) return rc;
  if (first > c->n || n > c->n - first) { stb_set_error("corpus_read: rows [%llu,+%llu) outside corpus of %llu",
      (unsigned long long)first, (unsigned long long)n, (unsigned long long)c->n); return STB_ERR_RANGE; }
  if (n == 0) return STB_OK;
  if (c->host_rows) {   // after the kernels that write rows
    STB_CUDA(cudaStreamSynchronize(c->ctx->stream));
    memcpy(rows, c->rows_host + first * STB_D, n * STB_D * sizeof(float));
    return STB_OK;
  }
  STB_CUDA(cudaMemcpyAsync(rows, c->rows + first * STB_D, n * STB_D * sizeof(float), cudaMemcpyDeviceToHost, c->ctx->stream));
  STB_CUDA(cudaStreamSynchronize(c->ctx->stream));
  return STB_OK;
}

// ---------------------------------------------------------------------- embed ---
int stb_embed(stb_ctx *ctx, const stb_table *table, const uint64_t *offsets, const uint32_t *ids,
              uint64_t n_lines, float *out, stb_corpus *append_to) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!table) { stb_set_error("embed: null table"); return STB_ERR_ARG; }
  if (table->ctx != ctx || (append_to && append_to->ctx != ctx)) { stb_set_error("embed: handles belong to another context"); return STB_ERR_ARG; }
  if (n_lines == 0) return STB_OK;
  if (!offsets) { stb_set_error("embed: offsets is null"); return STB_ERR_ARG; }
  if (offsets[0] != 0) { stb_set_error("embed: offsets[0] must be 0"); return STB_ERR_ARG; }
  const uint64_t total = offsets[n_lines];
  for (uint64_t i = 0; i < n_lines; ++i)
    if (offsets[i + 1] < offsets[i]) { stb_set_error("embed: offsets not monotone at line %llu", (unsigned long long)i); return STB_ERR_ARG; }
  if (total && !ids) { stb_set_error("embed: ids is null"); return STB_ERR_ARG; }
  if ((rc = ctx->embed_off_dev.reserve(n_lines + 1, 4096)) != STB_OK) return rc;
  if ((rc = ctx->embed_ids_dev.reserve(std::max<uint64_t>(total, 1), 65536)) != STB_OK) return rc;
  if (append_to && append_to->host_rows) {
    // K3 writes chunks of lines into the staging buffer; each chunk is committed to the host rows and its q8
    // entries from there.  The rows are booked only if no token was out of range.
    const uint64_t chunk = std::min<uint64_t>(n_lines, STB_MUT_CHUNK_ROWS);
    if ((rc = host_append_begin(append_to, n_lines, chunk)) != STB_OK) return rc;
    STB_CUDA(cudaMemcpyAsync(ctx->embed_off_dev, offsets, (n_lines + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->stream));
    if (total) STB_CUDA(cudaMemcpyAsync(ctx->embed_ids_dev, ids, total * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
    STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
    for (uint64_t l0 = 0; l0 < n_lines; l0 += chunk) {
      const uint64_t m = std::min(chunk, n_lines - l0);
      if ((rc = stb_launch_embed(ctx, table, ctx->embed_off_dev + l0, ctx->embed_ids_dev, m, ctx->mut_stage, ctx->err_flag)) != STB_OK) return rc;
      if (out) STB_CUDA(cudaMemcpyAsync(out + l0 * STB_D, ctx->mut_stage, m * STB_D * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
      if ((rc = host_append_chunk(append_to, ctx->mut_stage, append_to->n + l0, m)) != STB_OK) return rc;
    }
    int flag = 0;
    STB_CUDA(cudaMemcpyAsync(&flag, ctx->err_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
    STB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (flag) { stb_set_error("embed: a token id maps outside the %llu-row table", (unsigned long long)table->V); return STB_ERR_RANGE; }
    return host_append_finish(append_to, n_lines);
  }
  float *dst = nullptr;
  if (append_to) {
    if ((rc = corpus_reserve(append_to, append_to->n + n_lines)) != STB_OK) return rc;
    dst = append_to->rows + append_to->n * STB_D;
  } else {
    if ((rc = ctx->embed_out_dev.reserve(n_lines * STB_D, 4096 * STB_D)) != STB_OK) return rc;
    dst = ctx->embed_out_dev;
  }
  STB_CUDA(cudaMemcpyAsync(ctx->embed_off_dev, offsets, (n_lines + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->stream));
  if (total) STB_CUDA(cudaMemcpyAsync(ctx->embed_ids_dev, ids, total * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  // the call's own tokens are reported through its return value: the scratch flag, never the sticky
  // stb_embed_dev flag, and it is zeroed again after reading like every other synchronous user
  STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
  if ((rc = stb_launch_embed(ctx, table, ctx->embed_off_dev, ctx->embed_ids_dev, n_lines, dst, ctx->err_flag)) != STB_OK) return rc;
  int flag = 0;
  STB_CUDA(cudaMemcpyAsync(&flag, ctx->err_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
  if (out) STB_CUDA(cudaMemcpyAsync(out, dst, n_lines * STB_D * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (flag) { stb_set_error("embed: a token id maps outside the %llu-row table", (unsigned long long)table->V); return STB_ERR_RANGE; }
  if (append_to) { append_to->n += n_lines; corpus_changed(append_to, CORPUS_APPEND); }
  return STB_OK;
}

// The rows of stb_embed from text: per chunk of lines, the GPU tokenizer (tokenize.cu) leaves the chunk's CSR in
// embed_off_dev / embed_ids_dev and K3 pools it, into the corpus or the output staging; rows are booked at the end
// only if no token was out of range, as stb_embed does.
int stb_embed_text(stb_ctx *ctx, const stb_tokenizer *tok, const stb_table *table, const uint8_t *text,
                   const uint64_t *text_offsets, uint64_t n_lines, uint32_t max_length, float *out, stb_corpus *append_to) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!tok || !table) { stb_set_error("embed_text: null tokenizer or table"); return STB_ERR_ARG; }
  if (stb_tokenizer_ctx(tok) != ctx || table->ctx != ctx || (append_to && append_to->ctx != ctx)) {
    stb_set_error("embed_text: handles belong to another context"); return STB_ERR_ARG;
  }
  if (n_lines == 0) return STB_OK;
  StbTextHost h;
  if ((rc = stb_text_host(tok, text, text_offsets, n_lines, max_length, h)) != STB_OK) return rc;
  const bool host_rows = append_to && append_to->host_rows;
  const uint64_t n0 = append_to ? append_to->n : 0;
  if (host_rows) { if ((rc = host_append_begin(append_to, n_lines, std::min<uint64_t>(n_lines, STB_TEXT_CHUNK_LINES))) != STB_OK) return rc; }
  else if (append_to) { if ((rc = corpus_reserve(append_to, n0 + n_lines)) != STB_OK) return rc; }
  else if ((rc = ctx->embed_out_dev.reserve(std::min<uint64_t>(n_lines, STB_TEXT_CHUNK_LINES) * STB_D, 4096 * STB_D)) != STB_OK) return rc;
  if ((rc = stb_tok_reserve(ctx, tok, h, text_offsets, max_length)) != STB_OK) return rc;
  STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
  STB_CUDA(cudaMemsetAsync(ctx->tok_flag, 0, sizeof(int), ctx->stream));
  for (size_t c = 0; c + 1 < h.chunk_at.size(); ++c) {
    const uint64_t l0 = h.chunk_at[c], m = h.chunk_at[c + 1] - l0;
    if ((rc = stb_tok_chunk(ctx, tok, h, text, text_offsets, l0, m, max_length)) != STB_OK) return rc;
    float *dst = host_rows ? ctx->mut_stage.p : append_to ? append_to->rows + (n0 + l0) * STB_D : ctx->embed_out_dev.p;
    if ((rc = stb_launch_embed(ctx, table, ctx->embed_off_dev, ctx->embed_ids_dev, m, dst, ctx->err_flag)) != STB_OK) return rc;
    if (out) STB_CUDA(cudaMemcpyAsync(out + l0 * STB_D, dst, m * STB_D * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    if (host_rows && (rc = host_append_chunk(append_to, ctx->mut_stage, n0 + l0, m)) != STB_OK) return rc;
  }
  int flag[2] = {0, 0};
  STB_CUDA(cudaMemcpyAsync(&flag[0], ctx->err_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaMemcpyAsync(&flag[1], ctx->tok_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (flag[1]) { stb_set_error("embed_text: a GPU piece overflowed its bound (flag %d)", flag[1]); return STB_ERR_STATE; }
  if (flag[0]) { stb_set_error("embed: a token id maps outside the %llu-row table", (unsigned long long)table->V); return STB_ERR_RANGE; }
  if (host_rows) return host_append_finish(append_to, n_lines);
  if (append_to) { append_to->n += n_lines; corpus_changed(append_to, CORPUS_APPEND); }
  return STB_OK;
}

int stb_embed_dev(stb_ctx *ctx, const stb_table *table, const uint64_t *offsets_dev,
                  const uint32_t *ids_dev, uint64_t n_lines, float *out_dev) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!table || table->ctx != ctx) { stb_set_error("embed_dev: bad table"); return STB_ERR_ARG; }
  if (n_lines == 0) return STB_OK;
  if (!offsets_dev || !ids_dev || !out_dev) { stb_set_error("embed_dev: null device pointer"); return STB_ERR_ARG; }
  return stb_launch_embed(ctx, table, offsets_dev, ids_dev, n_lines, out_dev, ctx->embed_flag);
}

int stb_embed_status(stb_ctx *ctx) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  int flag = 0;
  STB_CUDA(cudaMemcpyAsync(&flag, ctx->embed_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaMemsetAsync(ctx->embed_flag, 0, sizeof(int), ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (flag) { stb_set_error("embed: a token id maps outside the table"); return STB_ERR_RANGE; }
  return STB_OK;
}

// --------------------------------------------------------------------- search ---
// STB_SCAN_TIER = f32 | h16 | q8: the narrowest candidate tier K1 may use (default q8).  Read per
// call so one process can compare tiers; results are identical whatever the value.
static int stb_env_max_tier() {
  const char *e = getenv("STB_SCAN_TIER");
  if (!e || !e[0]) return STB_TIER_Q8;
  if (e[0] == 'f') return STB_TIER_F32;
  if (e[0] == 'h') return STB_TIER_H16;
  return STB_TIER_Q8;
}
// What a K1 entry point may do to a reduced-width candidate copy that does not cover every row yet:
// build it from nothing (or rebuild one marked bad), and convert the rows appended behind a valid prefix.
struct K1CopyPolicy {
  bool build, extend;
};
static const K1CopyPolicy kBuiltOnly = {false, false};

// The one rule for K1's candidate copies: sets *ready when the scan may read tier `tier` of c now.  It
// applies the STB_SCAN_TIER cap, the q8 tier's k-limit (top_k: k of the top-k scan; 0 for the collect
// and histogram passes, which have none) and the copy's state, building or extending the copy as the
// policy allows.  Rows that cannot be normalised in fp32 make a copy unusable (the builder's
// STB_ERR_STATE), which is not an error of the search.  f32 is always ready.
static int k1_copy_ready(stb_ctx *ctx, stb_corpus *c, int tier, uint32_t top_k, K1CopyPolicy policy, bool *ready) {
  *ready = tier == STB_TIER_F32;
  if (*ready || tier > stb_env_max_tier() || (tier == STB_TIER_Q8 && top_k > STB_Q8_MAX_K)) return STB_OK;
  const auto ready_or_build = [&](auto &k) -> int {
    if (k.covers(c->n)) { *ready = k.usable(c->n); return STB_OK; }
    if (!policy.build && !(policy.extend && k.built() > 0)) return STB_OK;
    const int rc = corpus_ensure(ctx, c, k);
    *ready = rc == STB_OK;
    return rc == STB_ERR_STATE ? STB_OK : rc;
  };
  return tier == STB_TIER_Q8 ? ready_or_build(c->q8) : ready_or_build(c->shadow);
}

// The single-GPU asynchronous entry points (stb_search_topk_dev, stb_search_many without an exchange) always
// use the overlapped launch mode and co-scan (scan_topk.cu: stb_coscan_offset): back-to-back queries share
// each tile's HBM read.  The sharded forms (stb_search_topk_xchg, stb_search_many with an exchange) launch
// like the synchronous entry points (full grid, dependent released after the scan).
// All of them read the narrowest copy that is fully built and usable; `policy` may let the q8 copy be built or
// extended first, and nothing else builds one (stb_corpus_prepare does).  On a host-rows corpus they read an HBM
// copy or launch nothing: an f32 top-k scan would stream the whole matrix over the host link.
static int k1_async_tier(stb_ctx *ctx, const stb_corpus *c, uint32_t top_k, K1CopyPolicy policy, const char *what, int *tier) {
  for (*tier = STB_TIER_Q8; *tier > STB_TIER_F32; --*tier) {
    bool ready = false;
    const int rc = k1_copy_ready(ctx, const_cast<stb_corpus *>(c), *tier, top_k, *tier == STB_TIER_Q8 ? policy : kBuiltOnly, &ready);
    if (rc != STB_OK) return rc;
    if (ready) return STB_OK;
  }
  if (c->host_rows) {
    stb_set_error("%s: the rows of this corpus are in host memory and no HBM copy serves this top_k "
                  "(q8: top_k <= %d; 16-bit shadow: stb_corpus_prepare); use stb_search", what, STB_Q8_MAX_K);
    return STB_ERR_STATE;
  }
  return STB_OK;
}
// Deliberate scope limit: host-rows corpora are not sharded over an exchange.
static int host_rows_refuse(const stb_corpus *c, const char *what) {
  if (c && c->host_rows) { stb_set_error("%s: not available on a corpus whose rows are in host memory", what); return STB_ERR_STATE; }
  return STB_OK;
}

// The status words a K1 top-k scan stores beside its hits: [0] the hits (at most top_k), [1] non-zero when the
// scan proved them, [2] STB_XCHG_STATUS_TIMEOUT when a peer of a sharded scan never arrived.
struct K1Status {
  uint32_t n;
  bool proven, timeout;
};
static K1Status k1_status(const uint32_t *st, uint32_t top_k) {
  return {std::min(st[0], top_k), st[1] != 0, st[2] == STB_XCHG_STATUS_TIMEOUT};
}

// The distance limit of a search's hits, strict (distance < limit): max_distance.unwrap_or(100.0), which a top-k
// search also caps at STB_DEFAULT_MAX_DIST and threshold mode takes as given.  A NaN cap passes nothing: no
// distance compares below it.
static double k1_limit(bool threshold_all, int has_max, double max_distance) {
  if (!has_max) return STB_DEFAULT_MAX_DIST;
  return threshold_all || !(max_distance > STB_DEFAULT_MAX_DIST) ? max_distance : STB_DEFAULT_MAX_DIST;
}

// The collect floor for the rows at distance < d, from scores that may sit up to `margin` below the exact
// cosine 1 - d.  A NaN d collects nothing.
static float k1_floor(double d, double margin) { return d == d ? (float)(1.0 - d - margin) : INFINITY; }

// The distance cap of a top-k result sorted by (distance, row): how many leading hits pass the top-k limit
// (k1_limit).  Where top_k always caps (store-query mode, the top-k fast path) the capped result is this
// prefix of the uncapped one.
static uint64_t capped_hits(const stb_hit *hits, uint64_t n, int has_max, double max_distance) {
  const double limit = k1_limit(false, has_max, max_distance);
  uint64_t i = 0;
  while (i < n && hits[i].distance < limit) ++i;
  return i;
}

// ---- row ranges: global -> local, clipped to this shard and uploaded in the layout of StbRowRanges (common.cuh).
// Without ranges the passes read every row; n_virtual = 0: no row lies in them.
static int k1_upload_ranges(stb_ctx *ctx, const stb_corpus *c, const char *what, const uint64_t *row_ranges, uint32_t n_ranges,
                            StbRowRanges *out) {
  *out = {nullptr, 0, c->n};
  if (!row_ranges) return STB_OK;
  std::vector<uint64_t> vstart, rbegin;
  vstart.reserve(n_ranges + 1); rbegin.reserve(n_ranges);
  uint64_t acc = 0;
  int rc;
  if ((rc = stb_clip_ranges(what, row_ranges, n_ranges, c->row_base, c->n, [&](uint64_t b, uint64_t e) {
         vstart.push_back(acc); rbegin.push_back(b);
         acc += e - b;
       })) != STB_OK) return rc;
  out->n_virtual = acc;
  if (acc == 0) return STB_OK;
  vstart.push_back(acc);
  std::vector<uint64_t> packed(vstart);
  packed.insert(packed.end(), rbegin.begin(), rbegin.end());
  if ((rc = ctx->ranges_dev.reserve(packed.size(), 4096)) != STB_OK) return rc;
  STB_CUDA(cudaMemcpyAsync(ctx->ranges_dev, packed.data(), packed.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));   // `packed` dies at scope end
  *out = {ctx->ranges_dev, (uint32_t)rbegin.size(), acc};
  return STB_OK;
}

// A host query into ctx->q_dev, through the pinned staging buffer.
static int k1_stage_query(stb_ctx *ctx, const float *q) {
  memcpy(ctx->q_pin, q, STB_D * sizeof(float));
  STB_CUDA(cudaMemcpyAsync(ctx->q_dev, ctx->q_pin, STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  return STB_OK;
}

// Exact path for any input: collect rows whose approximate cosine >= cos_floor,
// score them canonically, keep distance < limit, sort by (distance,row).
// On return ctx->collect_hits holds the sorted hits and *n_pass their count.
static int collect_exact_sorted(stb_ctx *ctx, const stb_corpus *c, float cos_floor, double limit, const StbRowRanges &ranges,
                                uint64_t *n_pass, int tier = STB_TIER_F32) {
  int rc;
  unsigned long long count = 0;
  if ((rc = ctx->collect_rows.reserve(1, 1u << 20)) != STB_OK) return rc;
  for (int attempt = 0; attempt < 3; ++attempt) {
    if ((rc = stb_launch_scan_collect(ctx, c, tier, ctx->q_dev, cos_floor, ranges)) != STB_OK) return rc;
    STB_CUDA(cudaMemcpyAsync(&count, ctx->collect_count, sizeof(count), cudaMemcpyDeviceToHost, ctx->stream));
    STB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (count <= ctx->collect_rows.cap) break;
    if ((rc = ctx->collect_rows.reserve((size_t)count)) != STB_OK) return rc;
  }
  if (count > ctx->collect_rows.cap) { stb_set_error("collect buffer could not be sized"); return STB_ERR_STATE; }
  uint64_t m = count, m_padded = 1024;
  while (m_padded < m) m_padded <<= 1;
  if ((rc = ctx->collect_hits.reserve((size_t)m_padded)) != STB_OK) return rc;
  if ((rc = stb_launch_exact(ctx, c->rows, c->row_base, ctx->q_dev, ctx->collect_rows, m, limit,
                             ctx->collect_hits, m_padded, ctx->collect_count + 1)) != STB_OK) return rc;
  if ((rc = stb_launch_sort_hits(ctx, ctx->collect_hits, m_padded)) != STB_OK) return rc;
  unsigned long long pass = 0;
  STB_CUDA(cudaMemcpyAsync(&pass, ctx->collect_count + 1, sizeof(pass), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  *n_pass = pass;
  return STB_OK;
}

// The top-k tier ladder: q8 (260 B/row) -> h16 (512 B/row) -> f32 (1 KiB/row; not on a host-rows corpus).  Every
// tier ends in the same exact f64 re-rank and proves its own result; one that cannot is retried one tier up, so
// the answer is the oracle's whichever tier produced it.  A reduced-width tier that keeps failing its proofs on
// this corpus is dropped.  Each scan's last CTA stores the k hits + status straight into the pinned host buffers
// (UVA: cudaMallocHost memory is device-accessible), which takes the two D2H copies off the stream; kernel
// completion makes the stores visible to the host.  *proven: the last scan proved its hits.
static int k1_topk_ladder(stb_ctx *ctx, stb_corpus *c, const StbRowRanges &ranges, uint32_t top_k, K1CopyPolicy lazy,
                          bool *proven) {
  *proven = false;
  const int last = c->host_rows ? STB_TIER_H16 : STB_TIER_F32;
  for (int tier = STB_TIER_Q8; tier >= last && !*proven; --tier) {
    if (tier != STB_TIER_F32 && c->tier_tries[tier] >= 8 && 2 * c->tier_proven[tier] < c->tier_tries[tier]) continue;
    bool ready = false;
    int rc;
    if ((rc = k1_copy_ready(ctx, c, tier, top_k, lazy, &ready)) != STB_OK) return rc;
    if (!ready) continue;
    if ((rc = stb_launch_scan_topk(ctx, c, tier, ctx->q_dev, top_k, ranges, ctx->hits_pin, ctx->status_pin)) != STB_OK) return rc;
    STB_CUDA(cudaStreamSynchronize(ctx->stream));
    *proven = k1_status(ctx->status_pin, top_k).proven;
    c->tier_tries[tier]++;
    if (*proven) c->tier_proven[tier]++;
  }
  return STB_OK;
}

// The k-th-bin route (top_k beyond the register lists; on a host-rows corpus any top-k no copy proved): a histogram
// pass finds the score bin of the k-th best row, then the collect pass takes only the rows at or above that bin
// (a bin at the end: fewer than k rows, take all).  The q8 passes come first when the copy is usable.  Their
// histogram is over UPPER BOUNDS, which sit up to ~0.02-0.04 above the exact cosines, so the floor is put 0.04
// below the k-th best bound and the result is PROVEN afterwards: every row that was not collected has
// c < floor + 2e-5; if the k-th exact distance found is below 1 - floor - 2e-5 nothing outside can enter or tie.
// Otherwise (a fallback search) the f32 passes answer, with the floor 2 * STB_SCORE_EPS below the bin.
static int k1_kth_bin_collect(stb_ctx *ctx, const stb_corpus *c, const StbRowRanges &ranges, uint32_t top_k, double limit,
                              bool use_q8, uint64_t *n_pass) {
  std::vector<unsigned int> hist(4096);
  int rc;
  for (const int tier : {STB_TIER_Q8, STB_TIER_F32}) {
    const bool q8 = tier == STB_TIER_Q8;
    if (q8 && !use_q8) continue;
    if ((rc = stb_launch_scan_hist(ctx, c, tier, ctx->q_dev, ranges, ctx->hist_dev)) != STB_OK) return rc;
    STB_CUDA(cudaMemcpyAsync(hist.data(), ctx->hist_dev, 4096 * sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
    STB_CUDA(cudaStreamSynchronize(ctx->stream));
    uint64_t cum = 0;
    int b = 0;
    for (; b < 4096; ++b) { cum += hist[b]; if (cum >= top_k) break; }
    const float floor_cos = b < 4095 ? k1_floor((double)(b + 1) / 2048.0, q8 ? 0.04 : 2.0 * STB_SCORE_EPS) : -INFINITY;
    if ((rc = collect_exact_sorted(ctx, c, floor_cos, limit, ranges, n_pass, tier)) != STB_OK) return rc;
    if (!q8 || floor_cos == -INFINITY) return STB_OK;
    if (*n_pass >= top_k) {
      stb_hit kth;
      STB_CUDA(cudaMemcpyAsync(&kth, ctx->collect_hits + (top_k - 1), sizeof(kth), cudaMemcpyDeviceToHost, ctx->stream));
      STB_CUDA(cudaStreamSynchronize(ctx->stream));
      if (kth.distance < 1.0 - (double)floor_cos - 2.0 * STB_Q8_SCAN_EPS) return STB_OK;
    }
    ctx->fallback_searches++;
  }
  return STB_OK;
}

// A search's n sorted hits to the caller: the first min(n, cap) from `src` (device memory, or pinned host memory
// the kernel stored into), *out_n = n, and STB_ERR_CAPACITY when they do not all fit.
static int k1_copy_out(stb_ctx *ctx, const stb_hit *src, bool on_device, uint64_t n, stb_hit *out_hits, uint64_t cap,
                       uint64_t *out_n) {
  const uint64_t m = std::min(n, cap);
  *out_n = n;
  if (m && on_device) {
    STB_CUDA(cudaMemcpyAsync(out_hits, src, m * sizeof(stb_hit), cudaMemcpyDeviceToHost, ctx->stream));
    STB_CUDA(cudaStreamSynchronize(ctx->stream));
  } else if (m) {
    memcpy(out_hits, src, m * sizeof(stb_hit));
  }
  if (n > cap) { stb_set_error("search: %llu hits, capacity %llu", (unsigned long long)n, (unsigned long long)cap); return STB_ERR_CAPACITY; }
  return STB_OK;
}

int stb_search(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t top_k, int has_max,
               double max_distance, int mode, const uint64_t *row_ranges, uint32_t n_ranges,
               stb_hit *out_hits, uint64_t cap, uint64_t *out_n) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!corpus || !q || !out_n) { stb_set_error("search: null argument"); return STB_ERR_ARG; }
  if (corpus->ctx != ctx) { stb_set_error("search: corpus belongs to another context"); return STB_ERR_ARG; }
  if (mode != STB_MODE_SEARCH_DOCUMENTS && mode != STB_MODE_STORE_QUERY) { stb_set_error("search: bad mode %d", mode); return STB_ERR_ARG; }
  if (n_ranges && !row_ranges) { stb_set_error("search: row_ranges is null"); return STB_ERR_ARG; }
  if (cap && !out_hits) { stb_set_error("search: out_hits is null"); return STB_ERR_ARG; }
  *out_n = 0;
  const bool threshold_all = (mode == STB_MODE_SEARCH_DOCUMENTS) && has_max;   // src/search/mod.rs:115-116
  if (!threshold_all && top_k == 0) return STB_OK;                             // take(0) / store.rs:489-491
  if (mode == STB_MODE_STORE_QUERY && row_ranges && n_ranges == 0) return STB_OK;  // empty subset, store.rs:489
  if (corpus->n == 0) return STB_OK;

  StbRowRanges ranges;
  if ((rc = k1_upload_ranges(ctx, corpus, "search", row_ranges, n_ranges, &ranges)) != STB_OK) return rc;
  if (ranges.n_virtual == 0) return STB_OK;
  if ((rc = k1_stage_query(ctx, q)) != STB_OK) return rc;

  // The reduced-width candidate copies are used when they exist (stb_corpus_prepare) and built lazily
  // from the second search since the corpus last changed, on >= 32768 rows: a one-shot CLI query must
  // not pay a full extra pass to save half of one.  A copy that covers a prefix (rows were appended
  // since) is extended right away: converting the new rows costs far less than scanning everything at
  // 1 KiB/row.
  // A host-rows corpus builds nothing lazily: its q8 copy is always current, and its shadow is read when
  // stb_corpus_prepare or K2 built it.  No pass streams its f32 rows while an HBM copy can answer: a top-k
  // query no copy proves goes to the k-th-bin route below, not to the f32 top-k scan.
  stb_corpus *cm = const_cast<stb_corpus *>(corpus);
  const bool host = cm->host_rows != 0;
  const K1CopyPolicy lazy = {!host && cm->searches_since_change >= 1 && cm->n >= 32768, true};
  cm->searches_since_change++;

  const double limit = k1_limit(threshold_all, has_max, max_distance);
  if (!threshold_all && top_k <= stb_scan_topk_max_k()) {
    bool proven = false;
    if ((rc = k1_topk_ladder(ctx, cm, ranges, top_k, lazy, &proven)) != STB_OK) return rc;
    const uint32_t n_hits = k1_status(ctx->status_pin, top_k).n;
    if (proven) return k1_copy_out(ctx, ctx->hits_pin, false, capped_hits(ctx->hits_pin, n_hits, has_max, max_distance), out_hits, cap, out_n);
    if (!host) {
      // the f32 scan's candidate margin is not provable: exact collect pass down to its k-th hit
      ctx->fallback_searches++;
      const float floor_cos = n_hits == top_k ? k1_floor(ctx->hits_pin[top_k - 1].distance, 2.0 * STB_SCORE_EPS) : -INFINITY;
      uint64_t n_pass = 0;
      if ((rc = collect_exact_sorted(ctx, corpus, floor_cos, limit, ranges, &n_pass)) != STB_OK) return rc;
      return k1_copy_out(ctx, ctx->collect_hits, true, std::min<uint64_t>(n_pass, top_k), out_hits, cap, out_n);
    }
  }
  // ---- threshold mode, or the k-th-bin route: collect -> exact -> sort
  // When the int8 copy exists (or may be built: same lazy rule as the top-k tiers) the streaming
  // passes read it instead of the f32 rows: its scores are upper bounds u >= c - 2e-5 of the exact
  // cosine, so "u >= floor" collects a superset of "c >= floor" at a quarter of the bytes.
  bool use_q8 = false;
  if ((rc = k1_copy_ready(ctx, cm, STB_TIER_Q8, 0, lazy, &use_q8)) != STB_OK) return rc;
  uint64_t n_pass = 0;
  if (threshold_all)
    rc = collect_exact_sorted(ctx, corpus, k1_floor(max_distance, use_q8 ? 2.0 * STB_Q8_SCAN_EPS : STB_SCORE_EPS), limit, ranges,
                              &n_pass, use_q8 ? STB_TIER_Q8 : STB_TIER_F32);
  else
    rc = k1_kth_bin_collect(ctx, corpus, ranges, top_k, limit, use_q8, &n_pass);
  if (rc != STB_OK) return rc;
  return k1_copy_out(ctx, ctx->collect_hits, true, threshold_all ? n_pass : std::min<uint64_t>(n_pass, top_k), out_hits, cap, out_n);
}

int stb_search_topk_dev(stb_ctx *ctx, const stb_corpus *corpus, const float *q_dev, uint32_t top_k,
                        stb_hit *out_hits_dev, uint32_t *out_status_dev) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!corpus || !q_dev || !out_hits_dev || !out_status_dev) { stb_set_error("search_topk_dev: null argument"); return STB_ERR_ARG; }
  if (corpus->ctx != ctx) { stb_set_error("search_topk_dev: corpus belongs to another context"); return STB_ERR_ARG; }
  if (top_k == 0 || top_k > stb_scan_topk_max_k()) { stb_set_error("search_topk_dev: top_k must be 1..%u", stb_scan_topk_max_k()); return STB_ERR_ARG; }
  if (corpus->n == 0) { stb_set_error("search_topk_dev: empty corpus"); return STB_ERR_STATE; }
  // candidates from the narrowest copy that already exists; status[1] says whether the result is
  // proven, the caller's fallback is unchanged
  int tier;
  if ((rc = k1_async_tier(ctx, corpus, top_k, kBuiltOnly, "search_topk_dev", &tier)) != STB_OK) return rc;
  return stb_launch_scan_topk(ctx, corpus, tier, q_dev, top_k, {nullptr, 0, corpus->n}, out_hits_dev, out_status_dev, nullptr, true);
}

// ------------------------------------------------------------ peer-memory exchange ---
static size_t xchg_bytes(uint32_t world, uint32_t max_k) {
  return (size_t)STB_XCHG_SLOTS * world * 16 + (size_t)STB_XCHG_SLOTS * world * max_k * sizeof(stb_hit);
}

static size_t xchg_batch_slot_bytes(uint32_t world, uint32_t max_nq, uint32_t max_k) {
  const size_t head = ((size_t)world * 8 + (size_t)world * max_nq * 4 + 15) & ~(size_t)15;   // flags | status, 16-byte aligned
  return ((head + (size_t)world * max_nq * max_k * sizeof(stb_hit)) + 255) & ~(size_t)255;
}

static int xchg_create_impl(stb_ctx *ctx, uint32_t world, uint32_t rank, uint32_t max_k, uint32_t max_nq, stb_xchg **out) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!out) { stb_set_error("xchg_create: out is null"); return STB_ERR_ARG; }
  if (world < 1 || world > STB_XCHG_MAX_WORLD || rank >= world) { stb_set_error("xchg_create: world must be 1..%d and rank < world", STB_XCHG_MAX_WORLD); return STB_ERR_ARG; }
  if (max_k < 1 || max_k > stb_scan_topk_max_k()) { stb_set_error("xchg_create: max_k must be 1..%u", stb_scan_topk_max_k()); return STB_ERR_ARG; }
  if (max_nq > 65536 || (uint64_t)world * max_k > 2048) { stb_set_error("xchg_create: batch area too large (max_nq <= 65536, world * max_k <= 2048)"); return STB_ERR_ARG; }
  stb_xchg *x = new (std::nothrow) stb_xchg();
  if (!x) { stb_set_error("out of host memory"); return STB_ERR_NOMEM; }
  x->ctx = ctx; x->world = world; x->rank = rank; x->max_k = max_k; x->max_nq = max_nq;
  x->batch_off = (xchg_bytes(world, max_k) + 255) & ~(size_t)255;
  x->batch_slot_bytes = max_nq ? xchg_batch_slot_bytes(world, max_nq, max_k) : 0;
  x->bytes = x->batch_off + 2 * x->batch_slot_bytes;
  // plain device memory: required for cudaIpcGetMemHandle
  if ((rc = x->local.alloc(x->bytes)) != STB_OK || (rc = x->batch_ticket.alloc(1)) != STB_OK) { delete x; return rc; }
  cudaError_t e = cudaMemset(x->local, 0, x->bytes);
  if (e == cudaSuccess) e = cudaMemset(x->batch_ticket, 0, sizeof(unsigned int));
  // cudaMemset on device memory may return before it ran (legacy default stream, which a non-blocking
  // stream does not order against): the zeroed flags must be in place before any peer can store to them
  const cudaError_t se = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = se;
  if (e != cudaSuccess) { cudaGetLastError(); stb_set_error("xchg_create: %s", cudaGetErrorString(e)); delete x; return STB_ERR_NOMEM; }
  x->peers[rank] = x->local;
  x->connected = (world == 1);
  *out = x;
  return STB_OK;
}

int stb_xchg_create(stb_ctx *ctx, uint32_t world, uint32_t rank, uint32_t max_k, stb_xchg **out) {
  return xchg_create_impl(ctx, world, rank, max_k, 0, out);
}
int stb_xchg_create_batch(stb_ctx *ctx, uint32_t world, uint32_t rank, uint32_t max_k, uint32_t max_nq, stb_xchg **out) {
  if (max_nq == 0) { stb_set_error("xchg_create_batch: max_nq must be > 0"); return STB_ERR_ARG; }
  return xchg_create_impl(ctx, world, rank, max_k, max_nq, out);
}

int stb_xchg_destroy(stb_xchg *x) {
  if (!x) return STB_OK;
  if (x->ctx && ctx_alive(x->ctx)) { cudaSetDevice(x->ctx->device); cudaStreamSynchronize(x->ctx->stream); }
  else cudaDeviceSynchronize();
  for (uint32_t r = 0; r < x->world; ++r)
    if (x->ipc_opened[r] && x->peers[r]) cudaIpcCloseMemHandle(x->peers[r]);
  cudaGetLastError();
  delete x;
  return STB_OK;
}

int stb_xchg_local_handle(stb_xchg *x, uint8_t handle[STB_IPC_HANDLE_BYTES]) {
  if (!x || !handle) { stb_set_error("xchg_local_handle: null argument"); return STB_ERR_ARG; }
  int rc = ctx_use(x->ctx);
  if (rc) return rc;
  static_assert(sizeof(cudaIpcMemHandle_t) == STB_IPC_HANDLE_BYTES, "IPC handle size");
  cudaIpcMemHandle_t h;
  STB_CUDA(cudaIpcGetMemHandle(&h, x->local));
  memcpy(handle, &h, sizeof(h));
  return STB_OK;
}

int stb_xchg_connect(stb_xchg *x, const uint8_t *handles) {
  if (!x || !handles) { stb_set_error("xchg_connect: null argument"); return STB_ERR_ARG; }
  int rc = ctx_use(x->ctx);
  if (rc) return rc;
  for (uint32_t r = 0; r < x->world; ++r) {
    if (r == x->rank || x->peers[r]) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + (size_t)r * STB_IPC_HANDLE_BYTES, sizeof(h));
    void *p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      cudaGetLastError();
      stb_set_error("xchg_connect: cannot map rank %u's buffer (%s); use the NCCL path", r, cudaGetErrorString(e));
      return STB_ERR_CUDA;
    }
    x->peers[r] = (unsigned char *)p;
    x->ipc_opened[r] = true;
  }
  x->connected = true;
  return STB_OK;
}

int stb_xchg_connect_local(stb_xchg *x, stb_xchg *const *peers) {
  if (!x || !peers) { stb_set_error("xchg_connect_local: null argument"); return STB_ERR_ARG; }
  int rc = ctx_use(x->ctx);
  if (rc) return rc;
  for (uint32_t r = 0; r < x->world; ++r) {
    if (r == x->rank) continue;
    if (!peers[r] || peers[r]->world != x->world || peers[r]->rank != r || peers[r]->max_k != x->max_k || peers[r]->max_nq != x->max_nq) { stb_set_error("xchg_connect_local: peer %u mismatched", r); return STB_ERR_ARG; }
    const int pd = peers[r]->ctx->device;
    if (pd != x->ctx->device) {
      int can = 0;
      STB_CUDA(cudaDeviceCanAccessPeer(&can, x->ctx->device, pd));
      if (!can) { stb_set_error("xchg_connect_local: device %d cannot access device %d", x->ctx->device, pd); return STB_ERR_CUDA; }
      cudaError_t e = cudaDeviceEnablePeerAccess(pd, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { stb_set_error("cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(e)); return STB_ERR_CUDA; }
      cudaGetLastError();
    }
    x->peers[r] = peers[r]->local;
  }
  x->connected = true;
  return STB_OK;
}

int stb_search_topk_xchg(stb_ctx *ctx, const stb_corpus *corpus, const float *q_dev, uint32_t top_k,
                         stb_xchg *x, stb_hit *out_hits_dev, uint32_t *out_status_dev) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!corpus || !q_dev || !x || !out_hits_dev || !out_status_dev) { stb_set_error("search_topk_xchg: null argument"); return STB_ERR_ARG; }
  if (corpus->ctx != ctx || x->ctx != ctx) { stb_set_error("search_topk_xchg: handles belong to another context"); return STB_ERR_ARG; }
  if ((rc = host_rows_refuse(corpus, "search_topk_xchg")) != STB_OK) return rc;
  if (!x->connected) { stb_set_error("search_topk_xchg: exchange not connected"); return STB_ERR_STATE; }
  if (x->dead) { stb_set_error("search_topk_xchg: this exchange saw a peer time-out; destroy it on every rank"); return STB_ERR_STATE; }
  if (top_k == 0 || top_k > x->max_k) { stb_set_error("search_topk_xchg: top_k must be 1..%u", x->max_k); return STB_ERR_ARG; }
  int tier;
  if ((rc = k1_async_tier(ctx, corpus, top_k, kBuiltOnly, "search_topk_xchg", &tier)) != STB_OK) return rc;
  StbXchgArgs a;
  memset(&a, 0, sizeof(a));
  for (uint32_t r = 0; r < x->world; ++r) a.base[r] = x->peers[r];
  a.world = x->world; a.rank = x->rank; a.max_k = x->max_k;
  a.seq = ++x->seq;
  a.slot = (uint32_t)(a.seq % STB_XCHG_SLOTS);
  return stb_launch_scan_topk(ctx, corpus, tier, q_dev, top_k, {nullptr, 0, corpus->n}, out_hits_dev, out_status_dev, &a);
}

// ----------------------------------------------------------------- K2 batched search ---
int stb_corpus_prepare(stb_corpus *corpus, int what) {
  if (!corpus) { stb_set_error("null corpus"); return STB_ERR_ARG; }
  if (what & ~(STB_PREPARE_Q8 | STB_PREPARE_H16)) { stb_set_error("corpus_prepare: unknown flag"); return STB_ERR_ARG; }
  int rc = ctx_use(corpus->ctx);
  if (rc) return rc;
  if (corpus->n == 0) return STB_OK;
  // rows that cannot be normalised in fp32 make a copy unusable (STB_ERR_STATE): not an error of
  // this call -- searches simply stay on the f32 rows
  if (what & STB_PREPARE_Q8) { rc = corpus_ensure(corpus->ctx, corpus, corpus->q8); if (rc != STB_OK && rc != STB_ERR_STATE) return rc; }
  if (what & STB_PREPARE_H16) { rc = corpus_ensure(corpus->ctx, corpus, corpus->shadow); if (rc != STB_OK && rc != STB_ERR_STATE) return rc; }
  return STB_OK;
}

int stb_corpus_tier_stats(const stb_corpus *corpus, uint32_t tries[3], uint32_t proven[3], uint64_t built_rows[3]) {
  if (!corpus) { stb_set_error("null corpus"); return STB_ERR_ARG; }
  for (int t = 0; t < 3; ++t) {
    if (tries) tries[t] = corpus->tier_tries[t];
    if (proven) proven[t] = corpus->tier_proven[t];
  }
  if (built_rows) {
    built_rows[STB_TIER_F32] = corpus->n;
    built_rows[STB_TIER_H16] = corpus->shadow.built();   // < n after an append: a valid prefix
    built_rows[STB_TIER_Q8] = corpus->q8.built();
  }
  return STB_OK;
}

// ------------------------------------------------------------- in-place mutations ---
// stb_corpus_update / stb_corpus_remove (kernels: corpus_update.cu).  Validation comes first: a refused
// call writes nothing.  A copy already marked bad is dropped (its flag is recomputed by the next build);
// the others stay built and are re-encoded at every row the call writes inside their prefix.
static int corpus_mutation_check(stb_corpus *c, const char *what) {
  if (c->ivfpq_live) {
    stb_set_error("%s: %u IVF-PQ index(es) on this corpus refer to its rows; destroy them first", what, c->ivfpq_live);
    return STB_ERR_STATE;
  }
  return STB_OK;
}

static void corpus_drop_bad_copies(stb_corpus *c) {
  if (c->q8.bad) c->q8.drop();
  if (c->shadow.bad) c->shadow.drop();
}

// reads the bad-row flags the call's kernels raised (synchronises) and books the change
static int corpus_mutation_finish(stb_corpus *c) {
  stb_ctx *ctx = c->ctx;
  int flags[2] = {0, 0};
  STB_CUDA(cudaMemcpyAsync(flags, ctx->mut_flags, sizeof(flags), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  c->q8.mark_bad(flags[0]);
  c->shadow.mark_bad(flags[1]);
  corpus_changed(c, CORPUS_ROWS_REWRITTEN);
  // a host-rows corpus keeps its q8 copy current: one dropped as unusable is re-encoded from the rows now
  if (c->host_rows && c->q8.rows < c->n) {
    const int rc = corpus_ensure(ctx, c, c->q8);
    if (rc != STB_OK && rc != STB_ERR_STATE) return rc;
  }
  return STB_OK;
}

}  // extern "C"

int stb_corpus_update_impl(stb_corpus *c, const uint64_t *idx, const float *rows, uint64_t n, const char *what,
                           StbCorpusHook *hook) {
  if (!c) { stb_set_error("null corpus"); return STB_ERR_ARG; }
  int rc = ctx_use(c->ctx);
  if (rc) return rc;
  if (n == 0) return STB_OK;
  if (!idx || !rows) { stb_set_error("%s: null argument", what); return STB_ERR_ARG; }
  if ((rc = hook ? hook->check() : corpus_mutation_check(c, what)) != STB_OK) return rc;
  for (uint64_t i = 0; i < n; ++i) {
    if (idx[i] < c->row_base || idx[i] - c->row_base >= c->n || (i > 0 && idx[i] <= idx[i - 1])) {
      stb_set_error("%s: idx[%llu] = %llu is out of order or outside rows [%llu, %llu)", what, (unsigned long long)i,
                    (unsigned long long)idx[i], (unsigned long long)c->row_base, (unsigned long long)(c->row_base + c->n));
      return STB_ERR_RANGE;
    }
  }
  stb_ctx *ctx = c->ctx;
  const uint64_t chunk = std::min<uint64_t>(n, STB_MUT_CHUNK_ROWS);
  if ((rc = ctx->mut_stage.reserve(chunk * STB_D)) != STB_OK) return rc;
  if ((rc = ctx->mut_idx.reserve(chunk)) != STB_OK) return rc;
  if ((rc = ctx->mut_flags.reserve(2)) != STB_OK) return rc;
  if (hook) {
    // the hook sees its rows in the staging buffer before anything is written; an update of one chunk stays
    // staged for the write below, a larger one is uploaded again
    if ((rc = hook->begin()) != STB_OK) return rc;
    for (uint64_t i0 = 0; i0 < hook->staged_rows; i0 += chunk) {
      const uint64_t m = std::min(chunk, n - i0);
      STB_CUDA(cudaMemcpyAsync(ctx->mut_stage, rows + i0 * STB_D, m * STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
      if ((rc = hook->staged(ctx->mut_stage, i0, m)) != STB_OK) return rc;
    }
    if ((rc = hook->ready()) != STB_OK) return rc;
  }
  const bool staged = hook && hook->staged_rows && n <= chunk;
  corpus_drop_bad_copies(c);
  STB_CUDA(cudaMemsetAsync(ctx->mut_flags, 0, 2 * sizeof(int), ctx->stream));
  StbCorpusWriteArgs a = corpus_write_args(c, c->q8.rows, c->shadow.rows);
  a.idx = ctx->mut_idx;
  std::vector<uint64_t> local(chunk);
  for (uint64_t i0 = 0; i0 < n; i0 += chunk) {
    a.m = std::min(chunk, n - i0);
    for (uint64_t i = 0; i < a.m; ++i) local[i] = idx[i0 + i] - c->row_base;
    // the previous chunk's kernel reads the staging buffers: stream order keeps these copies behind it
    STB_CUDA(cudaMemcpyAsync(ctx->mut_idx, local.data(), a.m * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->stream));
    if (!staged)
      STB_CUDA(cudaMemcpyAsync(ctx->mut_stage, rows + i0 * STB_D, a.m * STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = stb_launch_corpus_write(ctx, a)) != STB_OK) return rc;
    if (i0 + chunk < n) STB_CUDA(cudaStreamSynchronize(ctx->stream));   // `local` is refilled next
  }
  return corpus_mutation_finish(c);
}

extern "C" {

int stb_corpus_update(stb_corpus *c, const uint64_t *idx, const float *rows, uint64_t n) {
  return stb_corpus_update_impl(c, idx, rows, n, "corpus_update", nullptr);
}

}  // extern "C"

int stb_corpus_remove_impl(stb_corpus *c, const uint64_t *ranges, uint32_t n_ranges, const char *what, StbCorpusHook *hook) {
  if (!c) { stb_set_error("null corpus"); return STB_ERR_ARG; }
  int rc = ctx_use(c->ctx);
  if (rc) return rc;
  if (n_ranges == 0) return STB_OK;
  if (!ranges) { stb_set_error("%s: ranges is null", what); return STB_ERR_ARG; }
  if ((rc = hook ? hook->check() : corpus_mutation_check(c, what)) != STB_OK) return rc;
  if (!stb_ranges_ordered(ranges, n_ranges)) { stb_set_error("%s: ranges must be ascending, disjoint, half-open", what); return STB_ERR_RANGE; }
  const uint64_t lo = c->row_base, hi = c->row_base + c->n;
  for (uint32_t i = 0; i < n_ranges; ++i)
    if (!(ranges[2 * i] < ranges[2 * i + 1]) || ranges[2 * i] < lo || ranges[2 * i + 1] > hi) {
      stb_set_error("%s: range %u [%llu, %llu) is empty or outside rows [%llu, %llu)", what, i, (unsigned long long)ranges[2 * i],
                    (unsigned long long)ranges[2 * i + 1], (unsigned long long)lo, (unsigned long long)hi);
      return STB_ERR_RANGE;
    }
  stb_ctx *ctx = c->ctx;
  // kept segments behind the first removed row, as {destination, source} local rows; the rows each copy covers
  // afterwards (a copy marked bad is dropped below: it covers none)
  std::vector<uint64_t> seg;
  uint64_t removed = 0;
  const uint64_t first = ranges[0] - lo;
  uint64_t dst = first;
  for (uint32_t i = 0; i < n_ranges; ++i) {
    const uint64_t b = ranges[2 * i] - lo, e = ranges[2 * i + 1] - lo;
    const uint64_t next = (i + 1 < n_ranges) ? ranges[2 * i + 2] - lo : c->n;
    removed += e - b;
    if (next > e) { seg.push_back(dst); seg.push_back(e); dst += next - e; }
  }
  const uint64_t moved = dst - first;
  const uint64_t q8_left = c->q8.covered_after_remove(ranges, n_ranges, lo);
  const uint64_t shadow_left = c->shadow.covered_after_remove(ranges, n_ranges, lo);
  if ((rc = ctx->mut_flags.reserve(2)) != STB_OK) return rc;
  if (moved) {
    const uint64_t chunk = std::min<uint64_t>(moved, STB_MUT_CHUNK_ROWS);
    if ((rc = ctx->mut_stage.reserve(chunk * STB_D)) != STB_OK) return rc;
    if ((rc = ctx->mut_idx.reserve(seg.size())) != STB_OK) return rc;
  }
  if (hook && ((rc = hook->begin()) != STB_OK || (rc = hook->ready()) != STB_OK)) return rc;
  corpus_drop_bad_copies(c);
  STB_CUDA(cudaMemsetAsync(ctx->mut_flags, 0, 2 * sizeof(int), ctx->stream));
  if (moved) {
    // Chunks in output order.  The sources of a chunk lie at or beyond its own output rows, so the gather
    // reads rows no earlier chunk has overwritten, and it completes before the commit writes.
    STB_CUDA(cudaMemcpyAsync(ctx->mut_idx, seg.data(), seg.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->stream));
    const uint32_t n_seg = (uint32_t)(seg.size() / 2);
    StbCorpusWriteArgs a = corpus_write_args(c, q8_left, shadow_left);
    for (uint64_t d0 = first; d0 < first + moved; d0 += STB_MUT_CHUNK_ROWS) {
      a.first = d0;
      a.m = std::min<uint64_t>(STB_MUT_CHUNK_ROWS, first + moved - d0);
      if ((rc = stb_launch_corpus_gather(ctx, c->rows, ctx->mut_idx, n_seg, a.first, a.m, ctx->mut_stage)) != STB_OK) return rc;
      if ((rc = stb_launch_corpus_write(ctx, a)) != STB_OK) return rc;
    }
    STB_CUDA(cudaStreamSynchronize(ctx->stream));   // `seg` dies at scope end
  }
  // the shadow's last covered tile ends in zero padding, as a build of `shadow_left` rows leaves it
  if (c->shadow.allocated() && shadow_left % 256 &&
      (rc = stb_launch_shadow_build(ctx, c->rows, shadow_left, 256, c->shadow.tiles, ctx->mut_flags + 1, shadow_left)) != STB_OK) return rc;
  c->n -= removed;
  c->q8.rows = q8_left;
  c->shadow.rows = shadow_left;
  return corpus_mutation_finish(c);
}

extern "C" {

int stb_corpus_remove(stb_corpus *c, const uint64_t *ranges, uint32_t n_ranges) {
  return stb_corpus_remove_impl(c, ranges, n_ranges, "corpus_remove", nullptr);
}

int stb_debug_corpus_copy(const stb_corpus *c, int which, uint64_t first, uint64_t n, void *out, uint64_t *covered) {
  if (!c || (n && !out)) { stb_set_error("debug_corpus_copy: null argument"); return STB_ERR_ARG; }
  int rc = ctx_use(c->ctx);
  if (rc) return rc;
  const void *src = nullptr;
  size_t unit = 0;
  uint64_t rows = c->q8.covered(), units = rows;
  switch (which) {
    case STB_COPY_Q8_CODES: src = c->q8.codes; unit = 256; break;
    case STB_COPY_Q8_SCALES: src = c->q8.scale; unit = sizeof(float); break;
    case STB_COPY_Q8_PLANE: src = c->q8.plane; unit = 128; break;
    case STB_COPY_Q8_SR: src = c->q8.sr; unit = sizeof(float2); break;
    case STB_COPY_H16_TILES:
      src = c->shadow.tiles; unit = 131072; rows = c->shadow.covered(); units = (rows + 255) / 256; break;
    default: stb_set_error("debug_corpus_copy: unknown copy %d", which); return STB_ERR_ARG;
  }
  if (covered) *covered = rows;
  if (first > units || n > units - first) {
    stb_set_error("debug_corpus_copy: [%llu, +%llu) outside the %llu the copy covers", (unsigned long long)first,
                  (unsigned long long)n, (unsigned long long)units);
    return STB_ERR_RANGE;
  }
  if (n == 0) return STB_OK;
  if (which == STB_COPY_Q8_PLANE) {   // the tiles that hold the rows, gathered back into row order
    const uint64_t t0 = first / STB_Q4_TILE_ROWS;
    const size_t off = stb_q4_plane_bytes(t0 * STB_Q4_TILE_ROWS), bytes = stb_q4_plane_bytes(first + n) - off;
    uint8_t *tiles = (uint8_t *)malloc(bytes);
    if (!tiles) { stb_set_error("debug_corpus_copy: cannot allocate %llu bytes", (unsigned long long)bytes); return STB_ERR_NOMEM; }
    cudaError_t e = cudaMemcpyAsync(tiles, (const uint8_t *)src + off, bytes, cudaMemcpyDeviceToHost, c->ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->ctx->stream);
    if (e == cudaSuccess) stb_q4_plane_gather(tiles, first, n, (uint8_t *)out);
    free(tiles);
    STB_CUDA(e);
    return STB_OK;
  }
  STB_CUDA(cudaMemcpyAsync(out, (const uint8_t *)src + first * unit, n * unit, cudaMemcpyDeviceToHost, c->ctx->stream));
  STB_CUDA(cudaStreamSynchronize(c->ctx->stream));
  return STB_OK;
}

int stb_corpus_prepare_batch(stb_corpus *corpus) {
  if (!corpus) { stb_set_error("null corpus"); return STB_ERR_ARG; }
  int rc = ctx_use(corpus->ctx);
  if (rc) return rc;
  if (corpus->n == 0) return STB_OK;
  return corpus_ensure(corpus->ctx, corpus, corpus->shadow);
}

}  // extern "C"

// ---- K2 host calls -------------------------------------------------------------------------------------------
// The record of the last K2 call, which stb_debug_batch_last returns: route, nq, two route words (routes 1-4,
// 7 and 8: n_sample, stride; 5 and 10: retried queries, K1 queries; 6 and 9: tensor groups, K1 queries), n_seg,
// seg_cap.  Routes 7-10 are the routes of a corpus whose shadow does not fit (k2_route).
enum K2Route : uint32_t { kRouteV1 = 1, kRouteV2 = 2, kRouteFiltered = 3, kRouteFilteredK1 = 4, kRouteThreshold = 5,
                          kRouteSubsets = 6, kRouteQ8 = 7, kRouteFilteredQ8 = 8, kRouteSubsetsQ8 = 9,
                          kRouteThresholdQ8 = 10 };
static void k2_record(stb_ctx *ctx, K2Route route, uint32_t nq, uint32_t a = 0, uint32_t b = 0, uint32_t n_seg = 0,
                      uint32_t seg_cap = 0) {
  const uint32_t words[6] = {route, nq, a, b, n_seg, seg_cap};
  memcpy(ctx->b_last, words, sizeof(words));
}

// The shadow as every K2 search call sees it.  batch_shadow is corpus_ensure, for a call that then reads the
// shadow.  batch_shadow_fits is for a call whose shadow plan does not fit but whose q8 plan does: it would not read
// the shadow, so none is built; it asks only whether corpus_ensure could allocate it (STB_ERR_NOMEM if not),
// with a trial allocation of the same size, released at once.  STB_ERR_NOMEM is the trigger of the q8 routes.
// While stb_debug_batch_no_shadow is on, both return STB_ERR_NOMEM without building or touching the shadow.
static int batch_no_shadow_hook(const stb_ctx *ctx) {
  if (!ctx->b_no_shadow) return STB_OK;
  stb_set_error("search_batch: the 16-bit shadow is off on this context (stb_debug_batch_no_shadow)");
  return STB_ERR_NOMEM;
}
static int batch_shadow(stb_ctx *ctx, stb_corpus *c) {
  const int rc = batch_no_shadow_hook(ctx);
  return rc != STB_OK ? rc : corpus_ensure(ctx, c, c->shadow);
}
static int batch_shadow_fits(stb_ctx *ctx, const stb_corpus *c) {
  const int rc = batch_no_shadow_hook(ctx);
  if (rc != STB_OK) return rc;
  if (c->shadow.has_room(c->n)) return STB_OK;
  StbBuf<uint8_t> trial;
  return trial.alloc(StbShadowBufs::bytes(std::max<uint64_t>(c->n, c->capacity)));
}

// The copy a K2 call reads: the 16-bit shadow, the q8 copy (where the shadow does not fit in HBM), or neither
// (K1 answers).  k2_route(on_q8, route): the number of a pipeline's route where the q8 copy stands in for the
// shadow: 2 -> 7, 3 -> 8, 6 -> 9, 5 -> 10.
enum class K2Copy { kShadow, kQ8, kNone };
static K2Route k2_route(bool on_q8, K2Route route) {
  if (!on_q8) return route;
  return route == kRouteV2 ? kRouteQ8 : route == kRouteFiltered ? kRouteFilteredQ8
       : route == kRouteSubsets ? kRouteSubsetsQ8 : route == kRouteThreshold ? kRouteThresholdQ8 : route;
}

// Which copy a K2 call reads.  reads_shadow: the call's shadow plan fits (the shadow is built, batch_shadow);
// q8_usable: its q8 plan fits.  With only the latter, the shadow is asked for with batch_shadow_fits; with neither,
// nothing is asked (kNone, STB_OK).  A shadow that does not fit (STB_ERR_NOMEM) makes the call read the q8 copy,
// built or extended here, if q8_usable and that copy can be used.  Hard errors are returned; otherwise *out says
// which copy, whether the shadow was missing (which picks the route number) and, for kNone, why: STB_ERR_STATE
// (rows K2 cannot normalise) or the shadow's STB_ERR_NOMEM, whose message is kept in shadow_err and is the last error.
struct K2Choice {
  K2Copy copy = K2Copy::kNone;
  bool shadow_missing = false;
  int status = STB_OK;
  std::string shadow_err;
};
static int k2_choose_copy(stb_ctx *ctx, stb_corpus *corpus, bool reads_shadow, bool q8_usable, K2Choice *out) {
  *out = K2Choice{};
  if (!reads_shadow && !q8_usable) return STB_OK;
  int rc = reads_shadow ? batch_shadow(ctx, corpus) : batch_shadow_fits(ctx, corpus);
  if (rc == STB_OK && reads_shadow) out->copy = K2Copy::kShadow;
  if (rc == STB_OK || rc == STB_ERR_STATE) { out->status = rc; return STB_OK; }
  if (rc != STB_ERR_NOMEM) return rc;
  out->shadow_missing = true;
  out->status = rc;
  out->shadow_err = stb_last_error();
  if (!q8_usable) return STB_OK;
  if ((rc = corpus_ensure(ctx, corpus, corpus->q8)) == STB_OK) { out->copy = K2Copy::kQ8; return STB_OK; }
  if (rc != STB_ERR_NOMEM && rc != STB_ERR_STATE) return rc;
  stb_set_error("%s", out->shadow_err.c_str());
  return STB_OK;
}

// Keys per (query, CTA) segment of the emitting pass of v2 and route 6: ~5 expected at 10M rows / 132 CTAs.
static constexpr uint32_t kSegCap = 64;

// Pipeline v2's sample size and fit rule over the n_cover tiles it may sample: the COMPLETE tiles of the
// shard (a padding row must never stand in for a real one), or, filtered, the listed tiles (tiles holding an
// eligible row; the sampling epilogue takes their maxima over eligible rows only).
//   ~4 tiles per SM, strided over the n_cover.  Expected candidates per query ~ top_k * n_cover / n_sample *
//   e^(2 EPS x / sigma^2) (x = top score, sigma = 1/16 for the benchmark's rows: factor ~1.2 with the fp16
//   shadow's EPS = 0.0012, ~3.8 with bf16's 0.0080).  Shards so large that this exceeds half of the finish
//   kernel's 4096-key capacity sample 1/64 of the tiles instead (threshold kernel: CTA-per-query variant,
//   <= 8192 tiles); beyond that v2 does not fit.
struct BatchV2Plan {
  uint32_t n_sample, stride;
  bool fits;
};
static BatchV2Plan batch_v2_plan(const stb_ctx *ctx, uint32_t n_cover, uint32_t top_k) {
  uint32_t n_sample = std::min<uint32_t>(n_cover, std::min<uint32_t>(4u * (uint32_t)ctx->sm_count, 608u));
  const uint32_t margin_factor = STB_SHADOW_F16 ? 2u : 4u;
  auto expected_emitted = [&](uint32_t ns) { return ns ? (uint64_t)top_k * margin_factor * ((n_cover + ns - 1) / ns) : 0; };
  if (expected_emitted(n_sample) > 2048) {
    const uint32_t sm = (uint32_t)ctx->sm_count;
    n_sample = std::min<uint32_t>(std::min<uint32_t>(n_cover, 8192u), (n_cover / 64 + sm - 1) / sm * sm);
  }
  const bool fits = top_k <= 64 && n_sample >= top_k && expected_emitted(n_sample) <= 2048;
  return {n_sample, fits ? n_cover / n_sample : 0u, fits};
}

// Route 7's sample size and fit rule (v2's, batch_scan.cu: "Route 7", with the q8 bounds in place of the shadow's
// EPS).  A row's bounds are u, l = a +- w with w = s h_l1 + e_q (~0.011 on the benchmark's rows: s ~ 0.21 / 127,
// h_l1 ~ ||q^||_1 / 2 ~ 6.4), and the threshold sits w below the sampled k-th cosine, so the emitted rows are those
// with a >= S - 2w instead of v2's a >= S - 2 EPS: ~e^(2 w x / sigma^2) ~ 7.2 times the top_k * n_cover / n_sample
// rows that reach the sampled k-th score (x ~ 0.35, sigma = 1/16), taken as 8.  The sample is ~4 tiles per SM,
// or as many as keep that estimate within half of the finish's 4096-key capacity (a multiple of the SM count,
// at most kQ8MaxSample: the threshold kernel's CTA-per-query variant holds that many maxima in 192 KiB of shared
// memory); any tile may be sampled, since rows past n are masked out of the maxima.  So a batch fits while
// ceil(n_tiles / 49152) <= floor(256 / top_k), top_k <= 64: every top_k up to ~50M rows, top_k <= 32 up to
// ~100M, top_k <= 16 up to ~200M (tests/test_batch_q8_plan.py).  Batches that do not fit are answered by K1.
static constexpr uint32_t kQ8MaxSample = 49152;
static BatchV2Plan batch_q8_plan(uint32_t sm, uint32_t n_cover, uint32_t top_k) {
  if (top_k == 0 || top_k > 64 || n_cover == 0 || sm == 0) return {0, 0, false};
  const uint32_t per_sample = 2048u / (8u * top_k);            // tiles one sampled tile may stand for (>= 4)
  uint32_t n_sample = std::max<uint32_t>(std::min<uint32_t>(4u * sm, 608u), (n_cover + per_sample - 1) / per_sample);
  if (n_sample > 608u) n_sample = std::min<uint32_t>((n_sample + sm - 1) / sm * sm, kQ8MaxSample);
  n_sample = std::min(n_sample, n_cover);
  const bool fits = n_sample >= top_k && (n_cover + n_sample - 1) / n_sample <= per_sample;
  return {n_sample, fits ? n_cover / n_sample : 0u, fits};
}

// The plan of the top-k passes over n_cover tiles on `copy`
static BatchV2Plan k2_plan(const stb_ctx *ctx, K2Copy copy, uint32_t n_cover, uint32_t top_k) {
  return copy == K2Copy::kQ8 ? batch_q8_plan((uint32_t)ctx->sm_count, n_cover, top_k) : batch_v2_plan(ctx, n_cover, top_k);
}

// The query tiles of q_dev[0, nq) for a GEMM on `copy`, q_pad slots in ctx->bq_tiles with every query's unusable
// flag in ctx->b_qbad: the shadow's, or the q8 copy's with the per-query constants in ctx->b_q8c
static int k2_query_tiles(stb_ctx *ctx, K2Copy copy, const float *q_dev, uint32_t nq, uint32_t q_pad) {
  if (copy == K2Copy::kQ8) return stb_launch_q8_query_tiles(ctx, q_dev, nq, q_pad, ctx->bq_tiles, ctx->b_q8c, ctx->b_qbad, nullptr);
  STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
  return stb_launch_shadow_build(ctx, q_dev, nq, 128, ctx->bq_tiles, ctx->err_flag, 0, ctx->b_qbad);
}

// GEMM pass p of the m_tiles query tiles in ctx->bq_tiles over the corpus's `copy`
static int k2_gemm(stb_ctx *ctx, const stb_corpus *corpus, K2Copy copy, uint32_t m_tiles, StbGemmPass p) {
  p.a_tiles = ctx->bq_tiles; p.m_tiles = m_tiles; p.n_rows = corpus->n;
  if (copy == K2Copy::kQ8) { p.copy = STB_GEMM_Q8; p.b_tiles = corpus->q8.codes; p.q8_scale = corpus->q8.scale; p.qc = ctx->b_q8c; }
  else p.b_tiles = corpus->shadow.tiles;
  return stb_launch_gemm(ctx, p);
}

// The top-k passes of routes 2, 3, 7 and 8 (batch_scan.cu) on `copy`: query tiles -> sampled threshold ->
// candidate-emitting GEMM -> exact finish (on the q8 copy: thresholds on the lower bounds, the upper bounds emitted,
// the finish with the q8 proof).  Unfiltered (tile_ids == NULL) the sample covers the tiles 0 .. n_cover-1 and the
// emission every tile; filtered, both cover the n_cover listed tiles tile_ids[] with the eligible-row bitmap.  p
// (k2_plan over n_cover) must fit.  Every buffer comes first: a call refused for lack of memory leaves the record
// as it was.
static int k2_topk_run(stb_ctx *ctx, const stb_corpus *corpus, K2Copy copy, const float *q_dev, uint32_t nq,
                       uint32_t top_k, uint32_t n_cover, BatchV2Plan p, const uint32_t *tile_ids, const uint32_t *bitmap,
                       stb_hit *out_hits_dev, uint32_t *out_status_dev) {
  int rc;
  const bool q8 = copy == K2Copy::kQ8;
  const uint32_t m_tiles = (nq + 127) / 128, q_pad = m_tiles * 128;
  const uint32_t n_emit = tile_ids ? n_cover : (uint32_t)((corpus->n + 255) / 256);
  const uint32_t n_seg = stb_batch_emit_grid(ctx, n_emit);
  if ((rc = ctx->b_qbad.reserve((size_t)q_pad)) != STB_OK) return rc;
  if (q8 && (rc = ctx->b_q8c.reserve((size_t)q_pad)) != STB_OK) return rc;
  if ((rc = ctx->bq_tiles.reserve((size_t)q_pad * 512)) != STB_OK) return rc;
  if ((rc = ctx->b_tilemax.reserve((size_t)p.n_sample * q_pad)) != STB_OK) return rc;
  if ((rc = ctx->b_thr.reserve((size_t)q_pad)) != STB_OK) return rc;
  if ((rc = ctx->b_cnt.reserve((size_t)q_pad * n_seg)) != STB_OK) return rc;
  if ((rc = ctx->b_keys.reserve((size_t)q_pad * n_seg * kSegCap)) != STB_OK) return rc;
  k2_record(ctx, k2_route(q8, tile_ids ? kRouteFiltered : kRouteV2), nq, p.n_sample, p.stride, n_seg, kSegCap);
  STB_CUDA(cudaMemsetAsync(ctx->b_cnt, 0, (size_t)q_pad * n_seg * sizeof(uint32_t), ctx->stream));
  if ((rc = k2_query_tiles(ctx, copy, q_dev, nq, q_pad)) != STB_OK) return rc;
  StbGemmPass pass;
  pass.select = tile_ids ? STB_GEMM_LISTED : STB_GEMM_ALL;
  pass.tile_ids = tile_ids; pass.bitmap = bitmap;
  pass.n_tiles = p.n_sample; pass.tile_stride = p.stride; pass.tilemax = ctx->b_tilemax;
  if ((rc = k2_gemm(ctx, corpus, copy, m_tiles, pass)) != STB_OK) return rc;
  // the q8 copy's threshold sits STB_Q8_SCAN_EPS lower, and an unusable query (zero, or not normalisable) emits
  // nothing and comes back unproven
  rc = q8 ? stb_launch_batch_thresh(ctx, ctx->b_tilemax, p.n_sample, nq, q_pad, top_k, ctx->b_thr, (float)STB_Q8_SCAN_EPS, ctx->b_qbad)
          : stb_launch_batch_thresh(ctx, ctx->b_tilemax, p.n_sample, nq, q_pad, top_k, ctx->b_thr);
  if (rc != STB_OK) return rc;
  pass.epi = STB_EPI_EMIT;
  pass.n_tiles = n_emit; pass.tile_stride = 1; pass.tilemax = nullptr;
  pass.thr = ctx->b_thr; pass.cand_cnt = ctx->b_cnt; pass.cand_keys = ctx->b_keys; pass.cand_cap = kSegCap;
  if ((rc = k2_gemm(ctx, corpus, copy, m_tiles, pass)) != STB_OK) return rc;
  return stb_launch_batch_finish2(ctx, ctx->b_keys, ctx->b_cnt, n_seg, kSegCap, nq, top_k, corpus->rows, corpus->n,
                                  corpus->row_base, q_dev, ctx->b_qbad, out_hits_dev, out_status_dev,
                                  q8 ? (const float *)corpus->q8.scale : nullptr, q8 ? (const float4 *)ctx->b_q8c : nullptr,
                                  q8 ? (const float *)ctx->b_thr : nullptr);
}

// The listed tiles of clipped local [begin, end) pairs: the shadow tiles a range touches (ascending, disjoint
// ranges -> ascending tiles).
static std::vector<uint32_t> listed_tiles(const std::vector<uint32_t> &loc) {
  std::vector<uint32_t> tiles;
  for (size_t r = 0; r < loc.size(); r += 2)
    for (uint32_t t = loc[r] / 256; t <= (loc[r + 1] - 1) / 256; ++t)
      if (tiles.empty() || tiles.back() < t) tiles.push_back(t);
  return tiles;
}

// How a K2 host call answers query i once its tensor passes are done (k2_complete).
struct K2Answer {
  enum Kind { kEmpty, kProven, kK1 } kind;
  const stb_hit *hits;       // kProven: the proven result, `n` hits (it may already be the output row)
  uint64_t n;
  const uint64_t *ranges;    // kK1: the query's ranges, as stb_search takes them
  uint32_t n_ranges;
};

// Completes a K2 host call: query i gets 0 hits, its proven tensor result capped at max_distance, or K1's answer
// (stb_search in `mode`, counted in fallback_searches), as answer(i) says; every row is then padded to top_k.
// *n_k1 (if given): the queries K1 answered.
template <class Answer>
static int k2_complete(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t nq, uint32_t top_k, int has_max,
                       double max_distance, int mode, Answer &&answer, stb_hit *out_hits, uint32_t *out_n,
                       uint32_t *n_k1 = nullptr) {
  uint32_t k1 = 0;
  for (uint32_t i = 0; i < nq; ++i) {
    stb_hit *oh = out_hits + (size_t)i * top_k;
    const K2Answer a = answer(i);
    uint64_t n = 0;
    if (a.kind == K2Answer::kProven) {
      if (a.hits != oh) memcpy(oh, a.hits, (size_t)top_k * sizeof(stb_hit));
      n = capped_hits(oh, a.n, has_max, max_distance);
    } else if (a.kind == K2Answer::kK1) {
      ctx->fallback_searches++;
      k1++;
      const int rc = stb_search(ctx, corpus, q + (size_t)i * STB_D, top_k, has_max, max_distance, mode, a.ranges, a.n_ranges,
                                oh, top_k, &n);
      if (rc != STB_OK) return rc;
    }
    out_n[i] = (uint32_t)n;
    stb_pad_hits(oh, n, top_k);
  }
  if (n_k1) *n_k1 = k1;
  return STB_OK;
}

// The filtered top-k passes for nq host queries over `loc` (clipped local [begin, end) pairs) and its listed tiles, on
// `copy` (route 3 on the shadow, 8 on the q8 copy); k2_plan over the listed tiles must fit.  Hits land in
// out_hits [nq][top_k], {hits, proven} in status [nq][2].
static int filtered_tensor_run(stb_ctx *ctx, stb_corpus *corpus, K2Copy copy, const float *q, uint32_t nq, uint32_t top_k,
                               const std::vector<uint32_t> &loc, const std::vector<uint32_t> &tiles, stb_hit *out_hits,
                               uint32_t *status) {
  int rc;
  const uint64_t n_words = (corpus->n + 255) / 256 * 8;
  if ((rc = ctx->bq_dev.reserve((size_t)nq * STB_D)) != STB_OK) return rc;
  if ((rc = ctx->bh_dev.reserve((size_t)nq * top_k)) != STB_OK) return rc;
  if ((rc = ctx->bs_dev.reserve((size_t)nq * 2)) != STB_OK) return rc;
  if ((rc = ctx->b_franges.reserve(loc.size(), 2048)) != STB_OK) return rc;
  if ((rc = ctx->b_ftiles.reserve(tiles.size(), 1024)) != STB_OK) return rc;
  if ((rc = ctx->b_fbits.reserve((size_t)n_words)) != STB_OK) return rc;
  STB_CUDA(cudaMemcpyAsync(ctx->bq_dev, q, (size_t)nq * STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  STB_CUDA(cudaMemcpyAsync(ctx->b_franges, loc.data(), loc.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  STB_CUDA(cudaMemcpyAsync(ctx->b_ftiles, tiles.data(), tiles.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = stb_launch_row_bitmap(ctx, ctx->b_franges, (uint32_t)(loc.size() / 2), n_words, ctx->b_fbits)) != STB_OK) return rc;
  const uint32_t n_listed = (uint32_t)tiles.size();
  if ((rc = k2_topk_run(ctx, corpus, copy, ctx->bq_dev, nq, top_k, n_listed, k2_plan(ctx, copy, n_listed, top_k), ctx->b_ftiles,
                        ctx->b_fbits, ctx->bh_dev, ctx->bs_dev)) != STB_OK) return rc;
  STB_CUDA(cudaMemcpyAsync(out_hits, ctx->bh_dev, (size_t)nq * top_k * sizeof(stb_hit), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaMemcpyAsync(status, ctx->bs_dev, (size_t)nq * 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));        // `loc` and `tiles` are read by the copies above
  return STB_OK;
}

// The store query (stb_search in STB_MODE_STORE_QUERY) for a batch, over `loc`: the caller's row_ranges clipped
// to local [begin, end) pairs (K1 answers with the former).  The eligible rows' bitmap and the listed tiles both
// come from `loc`; the filtered top-k passes run on the copy k2_choose_copy picks from the two plans over the listed
// tiles (route 3 on the shadow, 8 on the q8 copy).  K1 answers every query the tensor passes leave unproven, and
// all of them when nothing runs on the tensor cores (route 4).  The cap is applied on the host: store-query hits
// are a prefix of the uncapped top-k.
static int batch_filtered_run(stb_ctx *ctx, stb_corpus *corpus, const float *q, uint32_t nq, uint32_t top_k, int has_max,
                              double max_distance, const std::vector<uint32_t> &loc, const uint64_t *row_ranges,
                              uint32_t n_ranges, stb_hit *out_hits, uint32_t *out_n) {
  int rc;
  k2_record(ctx, kRouteFilteredK1, nq);
  if (loc.empty())
    return k2_complete(ctx, corpus, q, nq, top_k, has_max, max_distance, STB_MODE_STORE_QUERY,
                       [](uint32_t) { return K2Answer{K2Answer::kEmpty}; }, out_hits, out_n);
  const std::vector<uint32_t> tiles = listed_tiles(loc);
  const uint32_t n_listed = (uint32_t)tiles.size();
  K2Choice ch;
  if ((rc = k2_choose_copy(ctx, corpus, k2_plan(ctx, K2Copy::kShadow, n_listed, top_k).fits,
                           k2_plan(ctx, K2Copy::kQ8, n_listed, top_k).fits, &ch)) != STB_OK) return rc;
  const bool tensor_ok = ch.copy != K2Copy::kNone;
  std::vector<uint32_t> status((size_t)nq * 2, 0);
  if (tensor_ok && (rc = filtered_tensor_run(ctx, corpus, ch.copy, q, nq, top_k, loc, tiles, out_hits, status.data())) != STB_OK)
    return rc;
  return k2_complete(ctx, corpus, q, nq, top_k, has_max, max_distance, STB_MODE_STORE_QUERY, [&](uint32_t i) -> K2Answer {
    if (tensor_ok && status[2 * i + 1]) return {K2Answer::kProven, out_hits + (size_t)i * top_k, status[2 * i]};
    return {K2Answer::kK1, nullptr, 0, row_ranges, n_ranges};
  }, out_hits, out_n);
}

// stb_search_batch_dev; q8_route: the q8 copy whatever the shadow's state (stb_debug_batch_q8)
static int batch_dev_impl(stb_ctx *ctx, const stb_corpus *corpus_c, const float *q_dev, uint32_t nq, uint32_t top_k,
                          stb_hit *out_hits_dev, uint32_t *out_status_dev, bool q8_route) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  stb_corpus *corpus = const_cast<stb_corpus *>(corpus_c);
  if (!corpus || !q_dev || !out_hits_dev || !out_status_dev) { stb_set_error("search_batch_dev: null argument"); return STB_ERR_ARG; }
  if (corpus->ctx != ctx) { stb_set_error("search_batch_dev: corpus belongs to another context"); return STB_ERR_ARG; }
  if (nq == 0) return STB_OK;
  if (top_k == 0 || top_k > 1024) { stb_set_error("search_batch_dev: top_k must be 1..1024"); return STB_ERR_ARG; }
  if (corpus->n == 0) { stb_set_error("search_batch_dev: empty corpus"); return STB_ERR_STATE; }
  K2Choice ch;
  if (q8_route) {
    if ((rc = corpus_ensure(ctx, corpus, corpus->q8)) != STB_OK) return rc;
    ch.copy = K2Copy::kQ8;
  } else if ((rc = k2_choose_copy(ctx, corpus, true, true, &ch)) != STB_OK) {
    return rc;
  }
  // neither copy can be used: refused with the status and message that say why, nothing written
  if (ch.copy == K2Copy::kNone) return ch.status;
  const uint32_t m_tiles = (nq + 127) / 128, q_pad = m_tiles * 128;
  const uint32_t n_tiles = (uint32_t)((corpus->n + 255) / 256), n_sub = n_tiles * 8;
  // The top-k passes (k2_topk_run) prove every query for any top_k <= 64 unless a capacity overflows.  Their sample
  // covers the shadow's complete tiles (a padding row must never stand in for a real one), or any tile of the q8
  // copy, whose maxima leave out the rows past n.
  const uint32_t n_cover = ch.copy == K2Copy::kQ8 ? n_tiles : (uint32_t)(corpus->n / 256);
  const BatchV2Plan plan = k2_plan(ctx, ch.copy, n_cover, top_k);
  if (plan.fits) {
    rc = k2_topk_run(ctx, corpus, ch.copy, q_dev, nq, top_k, n_cover, plan, nullptr, nullptr, out_hits_dev, out_status_dev);
    // where the q8 copy stands in for the shadow, running out of memory there is the shadow's refusal
    if (ch.shadow_missing && (rc == STB_ERR_NOMEM || rc == STB_ERR_STATE)) { stb_set_error("%s", ch.shadow_err.c_str()); return STB_ERR_NOMEM; }
    return rc;
  }
  if (ch.copy == K2Copy::kQ8) {
    // the q8 plan does not fit: every query comes back unproven
    std::vector<stb_hit> pad((size_t)nq * top_k);
    stb_pad_hits(pad.data(), 0, pad.size());
    STB_CUDA(cudaMemcpyAsync(out_hits_dev, pad.data(), pad.size() * sizeof(stb_hit), cudaMemcpyHostToDevice, ctx->stream));
    STB_CUDA(cudaMemsetAsync(out_status_dev, 0, (size_t)nq * 2 * sizeof(uint32_t), ctx->stream));
    STB_CUDA(cudaStreamSynchronize(ctx->stream));       // `pad` is read by the copy
    k2_record(ctx, kRouteQ8, nq);
    return STB_OK;
  }
  // The round-1 maxima/select/finish pipeline (v1) runs on the shadow for top_k > 64 and wherever v2 does not fit.
  // One flag per query, written by the query shadow build: a query that cannot be normalised in fp32
  // has a zero (or NaN) shadow whose scores bound nothing, and both finish kernels report it unproven
  if ((rc = ctx->b_qbad.reserve((size_t)q_pad)) != STB_OK) return rc;
  k2_record(ctx, kRouteV1, nq);
  // selection slices: enough CTAs (m_tiles x n_slices) to hide the latency of the streaming
  // read; the finish kernel merges n_slices x 32 <= 4096 candidate tiles per query
  uint32_t n_slices = std::max<uint32_t>(1, std::min<uint32_t>(128, 1536 / m_tiles));
  n_slices = std::min<uint32_t>(n_slices, std::max<uint32_t>(1, n_tiles / 48));
  if ((rc = ctx->bq_tiles.reserve((size_t)q_pad * 512)) != STB_OK) return rc;
  if ((rc = ctx->b_submax.reserve((size_t)n_sub * q_pad)) != STB_OK) return rc;
  if ((rc = ctx->b_tilemax.reserve((size_t)n_tiles * q_pad)) != STB_OK) return rc;
  if ((rc = ctx->b_cand.reserve((size_t)q_pad * n_slices * 32)) != STB_OK) return rc;
  // query tiles: padding queries beyond nq are written as zeros by the shadow builder
  if ((rc = k2_query_tiles(ctx, K2Copy::kShadow, q_dev, nq, q_pad)) != STB_OK) return rc;
  StbGemmPass maxima;
  maxima.n_tiles = n_tiles; maxima.submax = ctx->b_submax; maxima.tilemax = ctx->b_tilemax;
  if ((rc = k2_gemm(ctx, corpus, K2Copy::kShadow, m_tiles, maxima)) != STB_OK) return rc;
  // two-level selection: the best tiles by tile maximum (1/8 of the data), refined to
  // sub-tiles inside the finish kernel
  if ((rc = stb_launch_batch_select(ctx, ctx->b_tilemax, n_tiles, q_pad, n_slices, ctx->b_cand)) != STB_OK) return rc;
  return stb_launch_batch_finish(ctx, ctx->b_cand, n_slices, n_sub, nq, top_k, corpus->rows, corpus->n,
                                 corpus->row_base, q_dev, ctx->b_qbad, out_hits_dev, out_status_dev, ctx->b_submax, q_pad);
}

// stb_search_batch on batch_dev_impl's route choice
static int batch_host_impl(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t nq, uint32_t top_k,
                           stb_hit *out_hits, uint32_t *out_n, bool q8_route) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!corpus || !q || !out_hits || !out_n) { stb_set_error("search_batch: null argument"); return STB_ERR_ARG; }
  if (nq == 0) return STB_OK;
  for (uint32_t i = 0; i < nq; ++i) out_n[i] = 0;
  if (top_k == 0 || corpus->n == 0) return STB_OK;
  bool tensor_ok = top_k <= 1024;
  std::vector<uint32_t> status((size_t)nq * 2, 0);
  if (tensor_ok) {
    if ((rc = ctx->bq_dev.reserve((size_t)nq * STB_D)) != STB_OK) return rc;
    if ((rc = ctx->bh_dev.reserve((size_t)nq * top_k)) != STB_OK) return rc;
    if ((rc = ctx->bs_dev.reserve((size_t)nq * 2)) != STB_OK) return rc;
    STB_CUDA(cudaMemcpyAsync(ctx->bq_dev, q, (size_t)nq * STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    rc = batch_dev_impl(ctx, corpus, ctx->bq_dev, nq, top_k, ctx->bh_dev, ctx->bs_dev, q8_route);
    if (rc == STB_ERR_STATE) { tensor_ok = false; }        // un-normalisable rows: K1 handles them
    else if (rc != STB_OK) return rc;
    else {
      // a query that could not be normalised comes back unproven (status[2q+1] = 0) like any other
      STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
      STB_CUDA(cudaMemcpyAsync(out_hits, ctx->bh_dev, (size_t)nq * top_k * sizeof(stb_hit), cudaMemcpyDeviceToHost, ctx->stream));
      STB_CUDA(cudaMemcpyAsync(status.data(), ctx->bs_dev, (size_t)nq * 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
      STB_CUDA(cudaStreamSynchronize(ctx->stream));
    }
  }
  // queries the tensor path could not prove (or could not run): exact single-query path
  return k2_complete(ctx, corpus, q, nq, top_k, 0, 0.0, STB_MODE_SEARCH_DOCUMENTS, [&](uint32_t i) -> K2Answer {
    if (tensor_ok && status[2 * i + 1]) return {K2Answer::kProven, out_hits + (size_t)i * top_k, status[2 * i]};
    return {K2Answer::kK1};
  }, out_hits, out_n);
}

extern "C" {

int stb_search_batch_dev(stb_ctx *ctx, const stb_corpus *corpus, const float *q_dev, uint32_t nq,
                         uint32_t top_k, stb_hit *out_hits_dev, uint32_t *out_status_dev) {
  return batch_dev_impl(ctx, corpus, q_dev, nq, top_k, out_hits_dev, out_status_dev, false);
}

int stb_search_batch(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t nq, uint32_t top_k,
                     stb_hit *out_hits, uint32_t *out_n) {
  return batch_host_impl(ctx, corpus, q, nq, top_k, out_hits, out_n, false);
}

int stb_debug_batch_q8(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t nq, uint32_t top_k,
                       stb_hit *out_hits, uint32_t *out_n) {
  return batch_host_impl(ctx, corpus, q, nq, top_k, out_hits, out_n, true);
}

int stb_search_batch_filtered(stb_ctx *ctx, const stb_corpus *corpus_c, const float *q, uint32_t nq, uint32_t top_k,
                              int has_max, double max_distance, const uint64_t *row_ranges, uint32_t n_ranges,
                              stb_hit *out_hits, uint32_t *out_n) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  stb_corpus *corpus = const_cast<stb_corpus *>(corpus_c);
  if (!corpus) { stb_set_error("search_batch_filtered: null corpus"); return STB_ERR_ARG; }
  if (corpus->ctx != ctx) { stb_set_error("search_batch_filtered: corpus belongs to another context"); return STB_ERR_ARG; }
  if (n_ranges && !row_ranges) { stb_set_error("search_batch_filtered: row_ranges is null"); return STB_ERR_ARG; }
  if (nq == 0) return STB_OK;
  if (!q || !out_n || (top_k && !out_hits)) { stb_set_error("search_batch_filtered: null argument"); return STB_ERR_ARG; }
  // stb_search's early outs come before it reads the ranges (store.rs:489-491: top_k 0, the empty subset)
  std::vector<uint32_t> loc;                             // clipped local [begin, end) pairs
  if (top_k && !(row_ranges && n_ranges == 0) && corpus->n) {
    if (!row_ranges) loc = {0u, (uint32_t)corpus->n};
    else if ((rc = stb_clip_ranges_u32("search_batch_filtered", row_ranges, n_ranges, corpus->row_base, corpus->n, &loc)) != STB_OK)
      return rc;                                         // refused before anything is written
  }
  return batch_filtered_run(ctx, corpus, q, nq, top_k, has_max, max_distance, loc, row_ranges, n_ranges, out_hits, out_n);
}

}  // extern "C"

// ---- one filter per query for a batch (stb_search_batch_subsets, route 6) -----------------------------------
// The work list of one pass: for every corpus tile some tensor group covers (ascending), the query tiles that
// meet it, each with the mask slot of both 64-query halves (zero_slot: the half's group does not cover the
// tile) and, sampling, the half's column of its group's sample.  A group's halves are consecutive, so walking
// groups in order yields every tile's query tiles in ascending order, and at most two halves share one.
struct SubsetsWork {
  std::vector<uint32_t> tiles, item_off, cta_tiles;
  std::vector<uint4> items;
};
static void subsets_work(const std::vector<std::vector<uint32_t>> &tiles_of, const std::vector<uint32_t> &half0,
                         const std::vector<uint32_t> &n_halves, uint32_t n_tiles, bool sample, uint32_t zero_slot,
                         uint32_t grid_cap, SubsetsWork *w) {
  const uint32_t T = (uint32_t)tiles_of.size();
  std::vector<uint32_t> off(n_tiles + 1, 0);
  for (uint32_t g = 0; g < T; ++g)
    for (uint32_t t : tiles_of[g]) off[t + 1]++;
  for (uint32_t t = 0; t < n_tiles; ++t) off[t + 1] += off[t];
  std::vector<uint32_t> grp(off[n_tiles]), col(off[n_tiles]), at(off.begin(), off.end() - 1);
  for (uint32_t g = 0; g < T; ++g)
    for (uint32_t j = 0; j < (uint32_t)tiles_of[g].size(); ++j) {
      const uint32_t p = at[tiles_of[g][j]]++;
      grp[p] = g;
      col[p] = sample ? j : 0xffffu;
    }
  w->tiles.clear(); w->items.clear();
  w->item_off.assign(1, 0);
  for (uint32_t t = 0; t < n_tiles; ++t) {
    if (off[t] == off[t + 1]) continue;
    w->tiles.push_back(t);
    const size_t first = w->items.size();
    for (uint32_t p = off[t]; p < off[t + 1]; ++p) {
      const uint32_t g = grp[p];
      for (uint32_t H = half0[g]; H < half0[g] + n_halves[g]; ++H) {
        if (w->items.size() == first || w->items.back().x != H / 2)
          w->items.push_back(make_uint4(H / 2, zero_slot, zero_slot, 0xffffffffu));
        uint4 &it = w->items.back();
        const uint32_t slot = g * n_tiles + t;
        if (H & 1) { it.z = slot; it.w = (it.w & 0xffffu) | (col[p] << 16); }
        else { it.y = slot; it.w = (it.w & 0xffff0000u) | col[p]; }
      }
    }
    w->item_off.push_back((uint32_t)w->items.size());
  }
  // CTAs take consecutive corpus tiles of equal work, a tile costing its items plus 2: reading the 128 KiB tile
  // at an SM's share of HBM bandwidth takes about as long as two items' MMAs
  const uint32_t n_union = (uint32_t)w->tiles.size();
  const uint32_t grid = std::min(n_union, grid_cap);
  const uint64_t total = (uint64_t)w->items.size() + 2ull * n_union;
  w->cta_tiles.assign(1, 0);
  uint64_t acc = 0;
  for (uint32_t u = 0; u < n_union; ++u) {
    while (w->cta_tiles.size() < grid && acc >= total * w->cta_tiles.size() / grid) w->cta_tiles.push_back(u);
    acc += w->item_off[u + 1] - w->item_off[u] + 2;
  }
  while (w->cta_tiles.size() <= grid) w->cta_tiles.push_back(n_union);
}

// Route 9: stb_search_batch_subsets where the shadow does not fit, with several groups (group[i]: query i's group
// in `lists`, or kNone for a query with no clipped range; listed[g]: group g's listed tiles).  On the q8 copy (copy
// kQ8), each group whose q8 plan fits over its listed tiles runs the filtered top-k passes on its own queries, one
// group after another; K1 answers the other groups (all of them with copy kNone) and every query the passes leave
// unproven.
static int subsets_q8_run(stb_ctx *ctx, stb_corpus *corpus, K2Copy copy, const float *q, uint32_t nq, uint32_t top_k,
                          int has_max, double max_distance, const std::vector<uint32_t> &group,
                          const std::vector<const std::vector<uint32_t> *> &lists,
                          const std::vector<std::vector<uint32_t>> &listed, const uint64_t *range_offsets,
                          const uint64_t *row_ranges, stb_hit *out_hits, uint32_t *out_n) {
  constexpr uint32_t kNone = 0xffffffffu;
  int rc;
  const uint32_t G = (uint32_t)lists.size();
  std::vector<std::vector<uint32_t>> members(G);
  for (uint32_t i = 0; i < nq; ++i)
    if (group[i] != kNone) members[group[i]].push_back(i);
  const bool any = copy == K2Copy::kQ8;
  // per caller query: the tensor result and {hits, proven}; the output is written only once every group has run,
  // so a group refused for lack of scratch leaves it untouched
  std::vector<uint32_t> status((size_t)nq * 2, 0), gstatus;
  std::vector<stb_hit> hits(any ? (size_t)nq * top_k : 0), ghits;
  std::vector<float> gq;
  uint32_t n_tensor = 0;
  for (uint32_t g = 0; any && g < G; ++g) {
    if (!k2_plan(ctx, copy, (uint32_t)listed[g].size(), top_k).fits) continue;
    const std::vector<uint32_t> &mem = members[g];
    const uint32_t m = (uint32_t)mem.size();
    gq.resize((size_t)m * STB_D);
    ghits.resize((size_t)m * top_k);
    gstatus.assign((size_t)m * 2, 0);
    for (uint32_t j = 0; j < m; ++j) memcpy(gq.data() + (size_t)j * STB_D, q + (size_t)mem[j] * STB_D, STB_D * sizeof(float));
    if ((rc = filtered_tensor_run(ctx, corpus, copy, gq.data(), m, top_k, *lists[g], listed[g], ghits.data(),
                                  gstatus.data())) != STB_OK) return rc;
    for (uint32_t j = 0; j < m; ++j) {
      memcpy(hits.data() + (size_t)mem[j] * top_k, ghits.data() + (size_t)j * top_k, (size_t)top_k * sizeof(stb_hit));
      status[2 * (size_t)mem[j]] = gstatus[2 * j];
      status[2 * (size_t)mem[j] + 1] = gstatus[2 * j + 1];
    }
    n_tensor++;
  }
  uint32_t k1;
  if ((rc = k2_complete(ctx, corpus, q, nq, top_k, has_max, max_distance, STB_MODE_STORE_QUERY, [&](uint32_t i) -> K2Answer {
         if (group[i] == kNone) return {K2Answer::kEmpty};
         if (status[2 * (size_t)i + 1]) return {K2Answer::kProven, hits.data() + (size_t)i * top_k, status[2 * (size_t)i]};
         return {K2Answer::kK1, nullptr, 0, row_ranges + 2 * range_offsets[i], (uint32_t)(range_offsets[i + 1] - range_offsets[i])};
       }, out_hits, out_n, &k1)) != STB_OK) return rc;
  k2_record(ctx, kRouteSubsetsQ8, nq, n_tensor, k1);
  return STB_OK;
}

extern "C" {

// The store query for a batch in which every query names its own subset (route 6).  Queries whose clipped
// ranges are identical form one group; one group for the whole batch is stb_search_batch_filtered's call.
// Otherwise every group whose v2 plan fits runs on the tensor cores, each occupying whole 64-query halves of
// the query slots: one sampling pass over the union of the groups' sampled tiles, the per-slot threshold, one
// emitting pass over the union of their listed tiles, finish2 over the groups' queries in compact order.  K1
// answers the other groups and every query the tensor passes leave unproven.  Where the shadow does not fit,
// route 9 (subsets_q8_run) runs instead.
int stb_search_batch_subsets(stb_ctx *ctx, const stb_corpus *corpus_c, const float *q, uint32_t nq, uint32_t top_k,
                             int has_max, double max_distance, const uint64_t *range_offsets, const uint64_t *row_ranges,
                             stb_hit *out_hits, uint32_t *out_n) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  stb_corpus *corpus = const_cast<stb_corpus *>(corpus_c);
  if (!corpus) { stb_set_error("search_batch_subsets: null corpus"); return STB_ERR_ARG; }
  if (corpus->ctx != ctx) { stb_set_error("search_batch_subsets: corpus belongs to another context"); return STB_ERR_ARG; }
  if (nq == 0) return STB_OK;
  if (!range_offsets || !q || !out_n || (top_k && !out_hits)) { stb_set_error("search_batch_subsets: null argument"); return STB_ERR_ARG; }
  if (range_offsets[0] != 0) { stb_set_error("search_batch_subsets: range_offsets[0] must be 0"); return STB_ERR_ARG; }
  for (uint32_t i = 0; i < nq; ++i)
    if (range_offsets[i + 1] < range_offsets[i] || range_offsets[i + 1] - range_offsets[i] > UINT32_MAX) {
      stb_set_error("search_batch_subsets: range_offsets decrease (or exceed 2^32 - 1 ranges) at query %u", i);
      return STB_ERR_ARG;
    }
  if (range_offsets[nq] && !row_ranges) { stb_set_error("search_batch_subsets: row_ranges is null"); return STB_ERR_ARG; }
  auto n_of = [&](uint32_t i) { return (uint32_t)(range_offsets[i + 1] - range_offsets[i]); };
  auto ranges_of = [&](uint32_t i) { return row_ranges + 2 * range_offsets[i]; };
  // clip every query's ranges as stb_search would (its refusals come before anything is written); a query with
  // no clipped range has 0 hits (store.rs:489-491, or no row of this shard), the others are grouped
  constexpr uint32_t kNone = 0xffffffffu;
  std::map<std::vector<uint32_t>, uint32_t> ids;
  std::vector<const std::vector<uint32_t> *> lists;       // group -> clipped local [begin, end) pairs
  std::vector<uint32_t> group(nq, kNone);
  if (top_k && corpus->n) {
    std::vector<uint32_t> loc;
    // a range list given again (byte for byte) has the first one's status and group: each distinct list is
    // validated and clipped once (queries: those that clipped it, by a fingerprint of count and end points)
    std::unordered_map<uint64_t, std::vector<uint32_t>> clipped;
    for (uint32_t i = 0; i < nq; ++i) {
      const uint32_t n = n_of(i);
      if (n == 0) continue;
      const uint64_t *r = ranges_of(i);
      const uint64_t fp = (uint64_t)n * 0x9e3779b97f4a7c15ull ^ r[0] ^ (r[2 * (size_t)n - 1] << 1) ^ (r[n] << 2);
      std::vector<uint32_t> &same = clipped[fp];
      auto j = std::find_if(same.begin(), same.end(), [&](uint32_t j) {
        return n_of(j) == n && memcmp(ranges_of(j), r, 2 * (size_t)n * sizeof(uint64_t)) == 0;
      });
      if (j != same.end()) { group[i] = group[*j]; continue; }
      same.push_back(i);
      loc.clear();
      if ((rc = stb_clip_ranges_u32("search_batch_subsets", ranges_of(i), n_of(i), corpus->row_base, corpus->n, &loc)) != STB_OK)
        return rc;
      if (loc.empty()) continue;
      auto it = ids.find(loc);                             // a new key is copied only once
      if (it == ids.end()) {
        it = ids.emplace(loc, (uint32_t)lists.size()).first;
        lists.push_back(&it->first);
      }
      group[i] = it->second;
    }
  }
  const uint32_t G = (uint32_t)lists.size();
  if (G == 1 && std::find(group.begin(), group.end(), kNone) == group.end())
    return batch_filtered_run(ctx, corpus, q, nq, top_k, has_max, max_distance, *lists[0], ranges_of(0), n_of(0), out_hits, out_n);
  k2_record(ctx, kRouteSubsets, nq);
  // the plan of every group; groups whose plan fits run on the tensor cores (tensor group tg = tensor[g])
  const uint32_t n_tiles = (uint32_t)((corpus->n + 255) / 256);
  std::vector<std::vector<uint32_t>> listed(G);
  std::vector<BatchV2Plan> plan(G);
  std::vector<uint32_t> tensor(G, kNone), tgroups;
  for (uint32_t g = 0; g < G; ++g) {
    listed[g] = listed_tiles(*lists[g]);
    plan[g] = batch_v2_plan(ctx, (uint32_t)listed[g].size(), top_k);
    if (plan[g].fits) tgroups.push_back(g);
  }
  if ((uint64_t)tgroups.size() * n_tiles >= UINT32_MAX) tgroups.clear();   // mask slots are 32-bit
  // the shadow is asked for whenever a group fits either plan, and built only where route 6 reads it
  bool q8_fits = false;
  for (uint32_t g = 0; g < G && !q8_fits; ++g) q8_fits = k2_plan(ctx, K2Copy::kQ8, (uint32_t)listed[g].size(), top_k).fits;
  K2Choice ch;
  rc = k2_choose_copy(ctx, corpus, !tgroups.empty(), q8_fits, &ch);
  if (ch.shadow_missing) k2_record(ctx, kRouteSubsetsQ8, nq);       // even if K1 answers every query
  if (rc != STB_OK) return rc;
  if (ch.shadow_missing)
    return subsets_q8_run(ctx, corpus, ch.copy, q, nq, top_k, has_max, max_distance, group, lists, listed, range_offsets,
                          row_ranges, out_hits, out_n);
  if (ch.copy != K2Copy::kShadow) tgroups.clear();         // e.g. un-normalisable rows: K1 answers every query
  const uint32_t T = (uint32_t)tgroups.size();
  for (uint32_t tg = 0; tg < T; ++tg) tensor[tgroups[tg]] = tg;
  // query slots: tensor group tg owns halves [half0[tg], half0[tg] + n_halves[tg]), its queries in caller order;
  // row r of the compact order is query qrow[r]
  std::vector<uint32_t> members(T, 0), half0(T), n_halves(T), row_of(nq, kNone), slot_of(nq, kNone), qrow;
  for (uint32_t i = 0; i < nq; ++i)
    if (group[i] != kNone && tensor[group[i]] != kNone) members[tensor[group[i]]]++;
  uint32_t halves = 0;
  for (uint32_t tg = 0; tg < T; ++tg) { half0[tg] = halves; n_halves[tg] = (members[tg] + 63) / 64; halves += n_halves[tg]; }
  const uint32_t m_tiles = (halves + 1) / 2, q_pad = m_tiles * 128;
  std::vector<uint32_t> slot_row(q_pad, kNone), fill(T, 0);
  for (uint32_t i = 0; i < nq; ++i) {
    if (group[i] == kNone || tensor[group[i]] == kNone) continue;
    const uint32_t tg = tensor[group[i]], j = fill[tg]++;
    slot_of[i] = half0[tg] * 64 + j;
    row_of[i] = (uint32_t)qrow.size();
    slot_row[slot_of[i]] = row_of[i];
    qrow.push_back(i);
  }
  const uint32_t nt = (uint32_t)qrow.size();
  std::vector<uint32_t> status((size_t)nt * 2, 0);
  std::vector<stb_hit> hits((size_t)nt * top_k);
  uint32_t n_seg = 0;
  if (T) {
    std::vector<std::vector<uint32_t>> sampled(T), tiles_of(T);
    uint32_t n_cols = 0;
    for (uint32_t tg = 0; tg < T; ++tg) {
      const uint32_t g = tgroups[tg];
      for (uint32_t j = 0; j < plan[g].n_sample; ++j) sampled[tg].push_back(listed[g][(size_t)j * plan[g].stride]);
      n_cols = std::max(n_cols, plan[g].n_sample);
      tiles_of[tg] = std::move(listed[g]);
    }
    const uint32_t zero_slot = T * n_tiles;
    SubsetsWork ws, we;
    subsets_work(sampled, half0, n_halves, n_tiles, true, zero_slot, (uint32_t)ctx->sm_count, &ws);
    subsets_work(tiles_of, half0, n_halves, n_tiles, false, zero_slot, (uint32_t)ctx->sm_count, &we);
    n_seg = stb_batch_emit_grid(ctx, (uint32_t)we.tiles.size());
    // one upload: items (16-byte aligned at the front), then the u32 arrays
    std::vector<uint32_t> up;
    auto put = [&](const void *p, size_t words) { const size_t o = up.size(); up.resize(o + words); memcpy(up.data() + o, p, words * 4); return o; };
    const size_t o_is = put(ws.items.data(), 4 * ws.items.size()), o_ie = put(we.items.data(), 4 * we.items.size());
    const size_t o_ts = put(ws.tiles.data(), ws.tiles.size()), o_os = put(ws.item_off.data(), ws.item_off.size());
    const size_t o_cs = put(ws.cta_tiles.data(), ws.cta_tiles.size());
    const size_t o_te = put(we.tiles.data(), we.tiles.size()), o_oe = put(we.item_off.data(), we.item_off.size());
    const size_t o_ce = put(we.cta_tiles.data(), we.cta_tiles.size()), o_sr = put(slot_row.data(), slot_row.size());
    // every tensor group's clipped ranges, back to back, for its bitmap
    std::vector<uint32_t> rr, rr_off(T + 1, 0);
    for (uint32_t tg = 0; tg < T; ++tg) {
      const std::vector<uint32_t> &loc = *lists[tgroups[tg]];
      rr.insert(rr.end(), loc.begin(), loc.end());
      rr_off[tg + 1] = (uint32_t)rr.size();
    }
    const uint64_t n_words = (uint64_t)n_tiles * 8;
    if ((rc = ctx->s_work.reserve(up.size())) != STB_OK) return rc;
    if ((rc = ctx->b_franges.reserve(rr.size(), 2048)) != STB_OK) return rc;
    if ((rc = ctx->b_fbits.reserve((size_t)(T * n_words + 8))) != STB_OK) return rc;
    if ((rc = ctx->bq_dev.reserve((size_t)nt * STB_D)) != STB_OK) return rc;
    if ((rc = ctx->s_qslots.reserve((size_t)q_pad * STB_D)) != STB_OK) return rc;
    if ((rc = ctx->s_qbad.reserve((size_t)nt)) != STB_OK) return rc;
    if ((rc = ctx->b_qbad.reserve((size_t)q_pad)) != STB_OK) return rc;
    if ((rc = ctx->bq_tiles.reserve((size_t)q_pad * 512)) != STB_OK) return rc;
    if ((rc = ctx->b_tilemax.reserve((size_t)n_cols * q_pad)) != STB_OK) return rc;
    if ((rc = ctx->b_thr.reserve((size_t)q_pad)) != STB_OK) return rc;
    if ((rc = ctx->b_cnt.reserve((size_t)nt * n_seg)) != STB_OK) return rc;
    if ((rc = ctx->b_keys.reserve((size_t)nt * n_seg * kSegCap)) != STB_OK) return rc;
    if ((rc = ctx->bh_dev.reserve((size_t)nt * top_k)) != STB_OK) return rc;
    if ((rc = ctx->bs_dev.reserve((size_t)nt * 2)) != STB_OK) return rc;
    std::vector<float> qc((size_t)nt * STB_D);
    for (uint32_t r = 0; r < nt; ++r) memcpy(qc.data() + (size_t)r * STB_D, q + (size_t)qrow[r] * STB_D, STB_D * sizeof(float));
    STB_CUDA(cudaMemcpyAsync(ctx->s_work, up.data(), up.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    STB_CUDA(cudaMemcpyAsync(ctx->b_franges, rr.data(), rr.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    STB_CUDA(cudaMemcpyAsync(ctx->bq_dev, qc.data(), qc.size() * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    STB_CUDA(cudaMemsetAsync(ctx->b_fbits + T * n_words, 0, 8 * sizeof(uint32_t), ctx->stream));   // the zero slot
    STB_CUDA(cudaMemsetAsync(ctx->b_cnt, 0, (size_t)nt * n_seg * sizeof(uint32_t), ctx->stream));
    STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
    for (uint32_t tg = 0; tg < T; ++tg)
      if ((rc = stb_launch_row_bitmap(ctx, ctx->b_franges + rr_off[tg], (rr_off[tg + 1] - rr_off[tg]) / 2, n_words,
                                      ctx->b_fbits + tg * n_words)) != STB_OK) return rc;
    const uint32_t *W = ctx->s_work;
    const uint32_t *d_slot_row = W + o_sr;
    if ((rc = stb_launch_batch_slots_gather(ctx, ctx->bq_dev, d_slot_row, q_pad, ctx->s_qslots)) != STB_OK) return rc;
    if ((rc = stb_launch_shadow_build(ctx, ctx->s_qslots, q_pad, 128, ctx->bq_tiles, ctx->err_flag, 0, ctx->b_qbad)) != STB_OK) return rc;
    if ((rc = stb_launch_batch_slots_prep(ctx, d_slot_row, ctx->b_qbad, q_pad, ctx->s_qbad, ctx->b_tilemax,
                                          (uint64_t)n_cols * q_pad)) != STB_OK) return rc;
    StbGemmPass pass;
    pass.select = STB_GEMM_WORK; pass.bitmap = ctx->b_fbits;
    pass.tile_ids = W + o_ts; pass.n_tiles = (uint32_t)ws.tiles.size(); pass.cta_tiles = W + o_cs; pass.item_off = W + o_os;
    pass.items = reinterpret_cast<const uint4 *>(W + o_is); pass.tile_stride = n_cols; pass.tilemax = ctx->b_tilemax;
    if ((rc = k2_gemm(ctx, corpus, K2Copy::kShadow, m_tiles, pass)) != STB_OK) return rc;
    if ((rc = stb_launch_batch_thresh(ctx, ctx->b_tilemax, n_cols, q_pad, q_pad, top_k, ctx->b_thr)) != STB_OK) return rc;
    pass.epi = STB_EPI_EMIT;
    pass.tile_ids = W + o_te; pass.n_tiles = (uint32_t)we.tiles.size(); pass.cta_tiles = W + o_ce; pass.item_off = W + o_oe;
    pass.items = reinterpret_cast<const uint4 *>(W + o_ie); pass.tile_stride = 1; pass.tilemax = nullptr;
    pass.slot_row = d_slot_row; pass.thr = ctx->b_thr; pass.cand_cnt = ctx->b_cnt; pass.cand_keys = ctx->b_keys;
    pass.cand_cap = kSegCap;
    if ((rc = k2_gemm(ctx, corpus, K2Copy::kShadow, m_tiles, pass)) != STB_OK) return rc;
    if ((rc = stb_launch_batch_finish2(ctx, ctx->b_keys, ctx->b_cnt, n_seg, kSegCap, nt, top_k, corpus->rows, corpus->n,
                                       corpus->row_base, ctx->bq_dev, ctx->s_qbad, ctx->bh_dev, ctx->bs_dev)) != STB_OK) return rc;
    STB_CUDA(cudaMemcpyAsync(hits.data(), ctx->bh_dev, hits.size() * sizeof(stb_hit), cudaMemcpyDeviceToHost, ctx->stream));
    STB_CUDA(cudaMemcpyAsync(status.data(), ctx->bs_dev, status.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    STB_CUDA(cudaStreamSynchronize(ctx->stream));           // the host arrays above are read by the copies
  }
  // each caller query's slot and compact row, for stb_debug_batch_last
  ctx->s_map.assign(slot_of.begin(), slot_of.begin() + nq);
  ctx->s_map.insert(ctx->s_map.end(), row_of.begin(), row_of.begin() + nq);
  uint32_t k1;
  if ((rc = k2_complete(ctx, corpus, q, nq, top_k, has_max, max_distance, STB_MODE_STORE_QUERY, [&](uint32_t i) -> K2Answer {
         const uint32_t r = row_of[i];
         if (group[i] == kNone) return {K2Answer::kEmpty};
         if (r != kNone && status[2 * (size_t)r + 1]) return {K2Answer::kProven, hits.data() + (size_t)r * top_k, status[2 * (size_t)r]};
         return {K2Answer::kK1, nullptr, 0, ranges_of(i), n_of(i)};
       }, out_hits, out_n, &k1)) != STB_OK) return rc;
  k2_record(ctx, kRouteSubsets, nq, T, k1, n_seg, T ? kSegCap : 0u);
  return STB_OK;
}

}  // extern "C"

// ---- threshold mode for a batch (stb_search_batch_threshold, route 5) ---------------------------------------
// delta: |canonical f64 distance - (1 - exact cosine)| of any pair of f32 vectors the shadow can normalise is
// below ~1e-13 (256-term f64 FMA chains, two square roots, one division; DESIGN §5); 1e-12 leaves 10x slack.
#define STB_THR_DELTA 1.0e-12
#define STB_THR_SEG_CAP 64u        // first pass: keys per (query, CTA), as pipeline v2
static_assert(STB_THR_SEG_CAP == kSegCap, "route 5's first pass uses pipeline v2's segment capacity");
#define STB_THR_CHUNK 4096u        // queries per pipeline run (keeps every candidate count within int)

// The emission threshold of the queries the tensor cores answer: ((1 - M) - eps) - delta in f64, rounded toward
// -inf to f32.  Every row with canonical d < M has exact cosine c > 1 - M - delta, so its score a >= c - EPS on
// the shadow (eps = EPS), and its upper bound u >= c - 1e-5 on the q8 copy (eps = STB_Q8_SCAN_EPS, route 10).
static float thr_emission_value(double max_distance, double eps) {
  const double x = ((1.0 - max_distance) - eps) - STB_THR_DELTA;
  float f = (float)x;
  if ((double)f > x) f = std::nextafter(f, -INFINITY);
  return f;
}

// One chunk of queries q[0, n) (global indices c0 ..) on the tensor cores, on `copy`: the shadow (route 5) or the q8
// copy (route 10: the queries' q8 tiles and unusable flags, K1's upper bounds u as the emitted scores).  On return
// slot_query[s] / pass[s] are the chunk-local query and hit count of every answered slot, k1 lists the queries K1
// must answer, and the sorted hits of slot s sit at ctx->t_buf (distance bits at [0, K), rows at [K, 2K)) from
// (*off)[s].
struct ThrChunk {
  std::vector<uint32_t> slot_query, pass, k1;
  std::vector<int> off;
  uint32_t retried = 0;
};
static int thr_chunk_run(stb_ctx *ctx, stb_corpus *corpus, const float *q, uint32_t c0, uint32_t n, double max_distance,
                         float t, K2Copy copy, ThrChunk *out) {
  int rc;
  const uint32_t m_tiles = (n + 127) / 128, q_pad = m_tiles * 128;
  const uint32_t n_tiles = (uint32_t)((corpus->n + 255) / 256);
  const uint32_t n_seg = stb_batch_emit_grid(ctx, n_tiles);
  float *thr = ctx->b_thr + c0;
  uint32_t *cnt = ctx->b_cnt + (size_t)c0 * n_seg;
  if ((rc = ctx->bq_dev.reserve((size_t)n * STB_D)) != STB_OK) return rc;
  if ((rc = ctx->b_qbad.reserve((size_t)q_pad)) != STB_OK) return rc;
  if ((rc = ctx->bq_tiles.reserve((size_t)q_pad * 512)) != STB_OK) return rc;
  if ((rc = ctx->b_keys.reserve((size_t)q_pad * n_seg * STB_THR_SEG_CAP)) != STB_OK) return rc;
  if (copy == K2Copy::kQ8 && (rc = ctx->b_q8c.reserve((size_t)q_pad)) != STB_OK) return rc;
  STB_CUDA(cudaMemcpyAsync(ctx->bq_dev, q, (size_t)n * STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  STB_CUDA(cudaMemsetAsync(cnt, 0, (size_t)q_pad * n_seg * sizeof(uint32_t), ctx->stream));
  // the unusable flags mark the queries that cannot be normalised (on the q8 copy, the zero query too): their
  // threshold is +inf, K1 answers them
  StbGemmPass emit;
  emit.epi = STB_EPI_EMIT; emit.n_tiles = n_tiles; emit.thr = thr; emit.cand_cnt = cnt; emit.cand_keys = ctx->b_keys;
  emit.cand_cap = STB_THR_SEG_CAP;
  if ((rc = k2_query_tiles(ctx, copy, ctx->bq_dev, n, q_pad)) != STB_OK) return rc;
  if ((rc = stb_launch_batch_thr_dist(ctx, ctx->bq_dev, ctx->b_qbad, n, q_pad, t, thr)) != STB_OK) return rc;
  if ((rc = k2_gemm(ctx, corpus, copy, m_tiles, emit)) != STB_OK) return rc;
  std::vector<uint32_t> hcnt((size_t)n * n_seg);
  std::vector<float> hthr(n);
  STB_CUDA(cudaMemcpyAsync(hcnt.data(), cnt, hcnt.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaMemcpyAsync(hthr.data(), thr, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));

  // Route: a query excluded by its threshold goes to K1; one whose segments all fit is answered from the first
  // pass; one with an overflowed segment is re-emitted while the re-emission's keys stay within the budget, and
  // goes to K1 beyond it.  Slots: the first-pass queries in query order, then the re-emitted ones.
  std::vector<uint32_t> direct, retry;
  std::vector<uint64_t> totals(n, 0);
  uint64_t retry_keys = 0;
  for (uint32_t i = 0; i < n; ++i) {
    if (hthr[i] == INFINITY) { out->k1.push_back(i); continue; }
    bool over = false;
    for (uint32_t s = 0; s < n_seg; ++s) {
      const uint32_t c = hcnt[(size_t)i * n_seg + s];
      totals[i] += c;
      over |= c > STB_THR_SEG_CAP;
    }
    if (!over) direct.push_back(i);
    else if (retry_keys + totals[i] <= STB_BATCH_THRESHOLD_RETRY_KEYS) { retry.push_back(i); retry_keys += totals[i]; }
    else out->k1.push_back(i);
  }
  out->retried = (uint32_t)retry.size();
  const uint32_t n_direct = (uint32_t)direct.size(), n_retry = out->retried, n_slots = n_direct + n_retry;
  out->slot_query = direct;
  out->slot_query.insert(out->slot_query.end(), retry.begin(), retry.end());
  out->pass.assign(n_slots, 0);
  out->off.assign(n_slots + 1, 0);
  if (n_slots == 0) return STB_OK;
  // key layout: slot s owns [off[s], off[s+1]); a first-pass segment lands at dst, a re-emitted one at segoff
  const uint32_t r_tiles = (n_retry + 127) / 128, r_pad = r_tiles * 128;
  std::vector<uint64_t> dst((size_t)n * n_seg, ~0ull), segoff((size_t)r_pad * n_seg + 1, 0);
  uint64_t at = 0;
  for (uint32_t s = 0; s < n_slots; ++s) {
    const uint32_t i = out->slot_query[s];
    out->off[s] = (int)at;
    for (uint32_t g = 0; g < n_seg; ++g) {
      if (s < n_direct) dst[(size_t)i * n_seg + g] = at;
      else segoff[(size_t)(s - n_direct) * n_seg + g] = at;
      at += hcnt[(size_t)i * n_seg + g];
    }
  }
  out->off[n_slots] = (int)at;
  for (size_t j = (size_t)n_retry * n_seg; j < segoff.size(); ++j) segoff[j] = at;   // padding slots: empty
  const int K = (int)at;
  if ((rc = ctx->t_buf.reserve(std::max<size_t>(4 * (size_t)K, 1))) != STB_OK) return rc;
  if ((rc = ctx->t_off.reserve((size_t)n_slots + 1)) != STB_OK) return rc;
  if ((rc = ctx->t_slot.reserve(2 * (size_t)n_slots)) != STB_OK) return rc;
  if ((rc = ctx->t_dst.reserve(dst.size())) != STB_OK) return rc;
  size_t sort_bytes = 0;
  if ((rc = stb_batch_thr_sort_bytes(ctx, K, n_slots, ctx->t_off, &sort_bytes)) != STB_OK) return rc;
  if ((rc = ctx->t_sort_tmp.reserve(sort_bytes)) != STB_OK) return rc;
  uint64_t *A = ctx->t_buf, *B = A + K, *C = B + K, *D = C + K;
  STB_CUDA(cudaMemcpyAsync(ctx->t_off, out->off.data(), out->off.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
  STB_CUDA(cudaMemcpyAsync(ctx->t_slot, out->slot_query.data(), n_slots * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  STB_CUDA(cudaMemcpyAsync(ctx->t_dst, dst.data(), dst.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = stb_launch_batch_thr_compact(ctx, ctx->b_keys, cnt, ctx->t_dst, (uint64_t)n * n_seg, STB_THR_SEG_CAP, A)) != STB_OK) return rc;
  if (n_retry) {
    // one more pass over the re-emitted queries' tiles, rebuilt from their f32 rows: the same bits, the same emitted
    // rows; into segments sized by the first pass's exact counts (the first pass's flags and q8 constants are no
    // longer read, r_pad <= q_pad)
    if ((rc = ctx->t_segoff.reserve(segoff.size())) != STB_OK) return rc;
    if ((rc = ctx->t_cur.reserve((size_t)r_pad * n_seg)) != STB_OK) return rc;
    if ((rc = ctx->t_rq.reserve((size_t)n_retry * STB_D)) != STB_OK) return rc;
    if ((rc = ctx->t_rthr.reserve((size_t)r_pad)) != STB_OK) return rc;
    STB_CUDA(cudaMemcpyAsync(ctx->t_segoff, segoff.data(), segoff.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->stream));
    STB_CUDA(cudaMemsetAsync(ctx->t_cur, 0, (size_t)r_pad * n_seg * sizeof(uint32_t), ctx->stream));
    if ((rc = stb_launch_batch_thr_gather(ctx, ctx->bq_dev, thr, ctx->t_slot + n_direct, n_retry, r_pad, ctx->t_rq,
                                          ctx->t_rthr)) != STB_OK) return rc;
    emit.epi = STB_EPI_EMIT_SIZED; emit.thr = ctx->t_rthr; emit.cand_cnt = ctx->t_cur; emit.cand_keys = A;
    emit.cand_cap = 0; emit.seg_off = ctx->t_segoff;
    if ((rc = k2_query_tiles(ctx, copy, ctx->t_rq, n_retry, r_pad)) != STB_OK) return rc;
    if ((rc = k2_gemm(ctx, corpus, copy, r_tiles, emit)) != STB_OK) return rc;
  }
  // exact finish: rows ascending -> canonical re-score, d < M -> stable sort by distance = (distance, row) order
  if ((rc = stb_batch_thr_sort_rows(ctx, ctx->t_sort_tmp, sort_bytes, K, n_slots, ctx->t_off, A, B)) != STB_OK) return rc;
  if ((rc = stb_launch_batch_thr_rescore(ctx, B, ctx->t_off, ctx->t_slot, n_slots, ctx->bq_dev, corpus->rows,
                                         corpus->row_base, max_distance, C, D, ctx->t_slot + n_slots)) != STB_OK) return rc;
  if ((rc = stb_batch_thr_sort_dist(ctx, ctx->t_sort_tmp, sort_bytes, K, n_slots, ctx->t_off, C, A, D, B)) != STB_OK) return rc;
  STB_CUDA(cudaMemcpyAsync(out->pass.data(), ctx->t_slot + n_slots, n_slots * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  return STB_OK;
}

extern "C" {

// Threshold mode of search_documents for a batch (route 5; route 10 where the shadow does not fit).  Chunks of
// STB_THR_CHUNK queries run the tensor-core pipeline (thr_chunk_run) on the copy k2_choose_copy picks; K1
// (stb_search) answers the queries it leaves (all of them when neither copy can be used), and each chunk's hits are
// laid out once all its counts are known: a chunk's output is one contiguous stretch of the concatenation.
int stb_search_batch_threshold(stb_ctx *ctx, const stb_corpus *corpus_c, const float *q, uint32_t nq, double max_distance,
                               stb_hit *out_hits, uint64_t cap, uint64_t *out_offsets) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  stb_corpus *corpus = const_cast<stb_corpus *>(corpus_c);
  if (!corpus) { stb_set_error("search_batch_threshold: null corpus"); return STB_ERR_ARG; }
  if (corpus->ctx != ctx) { stb_set_error("search_batch_threshold: corpus belongs to another context"); return STB_ERR_ARG; }
  if (nq == 0) return STB_OK;
  if (!q || !out_offsets || (cap && !out_hits)) { stb_set_error("search_batch_threshold: null argument"); return STB_ERR_ARG; }
  k2_record(ctx, kRouteThreshold, nq);
  for (uint32_t i = 0; i <= nq; ++i) out_offsets[i] = 0;
  if (corpus->n == 0 || !(max_distance > 0.0)) return STB_OK;      // NaN or <= 0: no distance is below it
  K2Choice choice;
  if ((rc = k2_choose_copy(ctx, corpus, true, true, &choice)) != STB_OK) return rc;
  const K2Route route = k2_route(choice.shadow_missing, kRouteThreshold);
  if (choice.shadow_missing) k2_record(ctx, route, nq);             // route 10, even if K1 answers all
  const bool tensor_ok = choice.copy != K2Copy::kNone;
  const uint32_t n_seg = tensor_ok ? stb_batch_emit_grid(ctx, (uint32_t)((corpus->n + 255) / 256)) : 0u;
  const size_t nq_pad = ((size_t)nq + 127) / 128 * 128;
  if (tensor_ok) {
    if ((rc = ctx->b_thr.reserve(nq_pad)) != STB_OK) return rc;
    if ((rc = ctx->b_cnt.reserve(nq_pad * n_seg)) != STB_OK) return rc;
  }
  double eps = STB_Q8_SCAN_EPS;
  if (choice.copy == K2Copy::kShadow) stb_batch_build_params(nullptr, &eps);
  const float t = thr_emission_value(max_distance, eps);
  std::unique_ptr<stb_hit[]> k1_buf;                                 // one K1 result: at most every row
  uint32_t retried = 0, k1_total = 0;
  for (uint32_t c0 = 0; c0 < nq; c0 += STB_THR_CHUNK) {
    const uint32_t n = std::min(STB_THR_CHUNK, nq - c0);
    ThrChunk ch;
    if (tensor_ok) {
      if ((rc = thr_chunk_run(ctx, corpus, q + (size_t)c0 * STB_D, c0, n, max_distance, t, choice.copy, &ch)) != STB_OK) return rc;
    } else {
      for (uint32_t i = 0; i < n; ++i) ch.k1.push_back(i);
    }
    retried += ch.retried;
    k1_total += (uint32_t)ch.k1.size();
    std::vector<uint64_t> count(n, 0);
    for (size_t s = 0; s < ch.slot_query.size(); ++s) count[ch.slot_query[s]] = ch.pass[s];
    std::vector<std::vector<stb_hit>> k1_hits(ch.k1.size());
    for (size_t j = 0; j < ch.k1.size(); ++j) {
      if (!k1_buf) k1_buf.reset(new (std::nothrow) stb_hit[corpus->n]);
      if (!k1_buf) { stb_set_error("search_batch_threshold: host allocation failed"); return STB_ERR_NOMEM; }
      ctx->fallback_searches++;
      uint64_t m = 0;
      if ((rc = stb_search(ctx, corpus, q + (size_t)(c0 + ch.k1[j]) * STB_D, 0, 1, max_distance, STB_MODE_SEARCH_DOCUMENTS,
                           nullptr, 0, k1_buf.get(), corpus->n, &m)) != STB_OK) return rc;
      k1_hits[j].assign(k1_buf.get(), k1_buf.get() + m);
      count[ch.k1[j]] = m;
    }
    for (uint32_t i = 0; i < n; ++i) out_offsets[c0 + i + 1] = out_offsets[c0 + i] + count[i];
    const uint64_t base = out_offsets[c0], total = out_offsets[c0 + n] - base;
    const uint64_t n_copy = base < cap ? std::min(total, cap - base) : 0;
    if (n_copy && !ch.slot_query.empty()) {
      // the tensor-answered queries' hits at their place in this chunk's stretch (K1's are filled in below)
      const uint32_t n_slots = (uint32_t)ch.slot_query.size();
      const int K = ch.off[n_slots];
      std::vector<uint64_t> out_at(n_slots);
      for (uint32_t s = 0; s < n_slots; ++s) out_at[s] = out_offsets[c0 + ch.slot_query[s]] - base;
      if ((rc = ctx->t_out_at.reserve((size_t)n_slots)) != STB_OK) return rc;
      if ((rc = ctx->t_hits.reserve(std::max<size_t>(total, 1))) != STB_OK) return rc;
      STB_CUDA(cudaMemcpyAsync(ctx->t_out_at, out_at.data(), n_slots * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->stream));
      if ((rc = stb_launch_batch_thr_write(ctx, ctx->t_buf, ctx->t_buf + K, ctx->t_off, ctx->t_slot + n_slots, n_slots,
                                           ctx->t_out_at, ctx->t_hits)) != STB_OK) return rc;
      STB_CUDA(cudaMemcpyAsync(out_hits + base, ctx->t_hits, n_copy * sizeof(stb_hit), cudaMemcpyDeviceToHost, ctx->stream));
      STB_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    for (size_t j = 0; j < ch.k1.size(); ++j) {
      const uint64_t o = out_offsets[c0 + ch.k1[j]];
      if (o < cap) memcpy(out_hits + o, k1_hits[j].data(), std::min<uint64_t>(k1_hits[j].size(), cap - o) * sizeof(stb_hit));
    }
  }
  k2_record(ctx, route, nq, retried, k1_total, n_seg, tensor_ok ? STB_THR_SEG_CAP : 0u);
  if (out_offsets[nq] > cap) {
    stb_set_error("search_batch_threshold: %llu hits, capacity %llu", (unsigned long long)out_offsets[nq], (unsigned long long)cap);
    return STB_ERR_CAPACITY;
  }
  return STB_OK;
}

// Sharded K2: every rank answers the nq queries on its shard (stb_search_batch_dev), then ONE exchange over
// NVLink peer memory -- each rank stores its nq x k hits + per-query proof flags into every peer's batch slot
// (push kernel), waits for all peers' sequence flags and merges per query (merge kernel).  Two launches, no
// NCCL call.  out_status_dev[2q] = hits of query q, [2q+1] = 1 iff EVERY rank proved its part, 2 = a peer
// never arrived.  Unproven queries: re-run them with stb_search_xchg / stb_search_many(x) (collective: every
// rank sees the same flags).
int stb_search_batch_xchg_dev(stb_ctx *ctx, const stb_corpus *corpus, const float *q_dev, uint32_t nq, uint32_t top_k,
                              stb_xchg *x, stb_hit *out_hits_dev, uint32_t *out_status_dev) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!corpus || !q_dev || !x || !out_hits_dev || !out_status_dev) { stb_set_error("search_batch_xchg_dev: null argument"); return STB_ERR_ARG; }
  if (corpus->ctx != ctx || x->ctx != ctx) { stb_set_error("search_batch_xchg_dev: handles belong to another context"); return STB_ERR_ARG; }
  if ((rc = host_rows_refuse(corpus, "search_batch_xchg_dev")) != STB_OK) return rc;
  if (!x->connected) { stb_set_error("search_batch_xchg_dev: exchange not connected"); return STB_ERR_STATE; }
  if (x->dead) { stb_set_error("search_batch_xchg_dev: this exchange saw a peer time-out; destroy it on every rank"); return STB_ERR_STATE; }
  if (nq == 0) return STB_OK;
  if (x->max_nq == 0 || nq > x->max_nq || top_k == 0 || top_k > x->max_k) { stb_set_error("search_batch_xchg_dev: needs stb_xchg_create_batch with max_nq >= %u, max_k >= %u", nq, top_k); return STB_ERR_ARG; }
  if ((rc = ctx->bh_dev.reserve((size_t)nq * top_k)) != STB_OK) return rc;
  if ((rc = ctx->bs_dev.reserve((size_t)nq * 2)) != STB_OK) return rc;
  if ((rc = stb_search_batch_dev(ctx, corpus, q_dev, nq, top_k, ctx->bh_dev, ctx->bs_dev)) != STB_OK) return rc;
  StbBatchXchgArgs a;
  memset(&a, 0, sizeof(a));
  a.world = x->world; a.rank = x->rank; a.max_nq = x->max_nq; a.max_k = x->max_k; a.nq = nq; a.top_k = top_k;
  a.seq = ++x->batch_seq;
  a.ticket = x->batch_ticket;
  for (uint32_t r = 0; r < x->world; ++r) a.slot[r] = x->peers[r] + x->batch_off + (size_t)(a.seq & 1) * x->batch_slot_bytes;
  return stb_launch_batch_xchg(ctx, a, ctx->bh_dev, ctx->bs_dev, out_hits_dev, out_status_dev);
}

int stb_debug_batch_last(stb_ctx *ctx, uint32_t info[6], float *thr, uint32_t *cand_cnt) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!info) { stb_set_error("debug_batch_last: null info"); return STB_ERR_ARG; }
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  memcpy(info, ctx->b_last, sizeof(ctx->b_last));
  const uint32_t route = ctx->b_last[0], nq = ctx->b_last[1], n_seg = ctx->b_last[4];
  if (route == kRouteSubsets && n_seg && nq) {
    // slot-indexed thresholds, compact-row counts -> caller order (+inf, 0: a query the tensor passes did not take)
    const uint32_t *slot = ctx->s_map.data(), *row = slot + nq;
    uint32_t n_slots = 0, n_rows = 0;
    for (uint32_t i = 0; i < nq; ++i) {
      if (slot[i] != 0xffffffffu) n_slots = std::max(n_slots, slot[i] + 1);
      if (row[i] != 0xffffffffu) n_rows = std::max(n_rows, row[i] + 1);
    }
    std::vector<float> t(n_slots);
    std::vector<uint32_t> c((size_t)n_rows * n_seg);
    STB_CUDA(cudaMemcpy(t.data(), ctx->b_thr, t.size() * sizeof(float), cudaMemcpyDeviceToHost));
    STB_CUDA(cudaMemcpy(c.data(), ctx->b_cnt, c.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    for (uint32_t i = 0; i < nq; ++i) {
      if (thr) thr[i] = slot[i] == 0xffffffffu ? INFINITY : t[slot[i]];
      for (uint32_t s = 0; cand_cnt && s < n_seg; ++s) cand_cnt[(size_t)i * n_seg + s] = row[i] == 0xffffffffu ? 0u : c[(size_t)row[i] * n_seg + s];
    }
    return STB_OK;
  }
  if ((route == kRouteV2 || route == kRouteFiltered ||
       ((route == kRouteThreshold || route == kRouteQ8 || route == kRouteFilteredQ8 || route == kRouteThresholdQ8) && n_seg)) && nq) {
    if (thr) STB_CUDA(cudaMemcpy(thr, ctx->b_thr, (size_t)nq * sizeof(float), cudaMemcpyDeviceToHost));
    if (cand_cnt) STB_CUDA(cudaMemcpy(cand_cnt, ctx->b_cnt, (size_t)nq * n_seg * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  }
  return STB_OK;
}

int stb_debug_batch_no_shadow(stb_ctx *ctx, int on) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  ctx->b_no_shadow = on ? 1 : 0;
  return STB_OK;
}

int stb_debug_batch_q8_plan(uint32_t sm_count, uint64_t n_rows, uint32_t top_k, uint32_t plan[3]) {
  if (!plan || n_rows > 0xffffffffull * 256) { stb_set_error("debug_batch_q8_plan: bad argument"); return STB_ERR_ARG; }
  const BatchV2Plan p = batch_q8_plan(sm_count, (uint32_t)((n_rows + 255) / 256), top_k);
  plan[0] = p.n_sample; plan[1] = p.stride; plan[2] = p.fits ? 1u : 0u;
  return STB_OK;
}

int stb_debug_batch_params(int *shadow_is_f16, double *eps) {
  stb_batch_build_params(shadow_is_f16, eps);
  return STB_OK;
}

// ------------------------------------------------------------------- K2 debug hook ---
// Runs shadow build + wgmma GEMM on host inputs and returns the FULL approximate score matrix (the debug pass) and
// the per-32-row maxima (the sampling pass) (tests only: validates descriptors / accumulator layout / epilogues
// against a reference matmul).
int stb_debug_batch_gemm(stb_ctx *ctx, const float *q, uint32_t nq, const float *rows, uint64_t n,
                         float *out_full, float *out_submax) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!q || !rows || !out_full || nq == 0 || n == 0) { stb_set_error("debug_batch_gemm: bad argument"); return STB_ERR_ARG; }
  const uint32_t m_tiles = (nq + 127) / 128;
  const uint32_t n_tiles = (uint32_t)((n + 255) / 256);
  const size_t q_pad = (size_t)m_tiles * 128, n_pad = (size_t)n_tiles * 256;
  StbBuf<float> dq, dr, dfull, dsub, dtile;
  StbBuf<uint8_t> da, db;
  StbBuf<int> dbad;
  if ((rc = dq.alloc((size_t)nq * STB_D)) != STB_OK || (rc = dr.alloc(n * STB_D)) != STB_OK ||
      (rc = da.alloc(q_pad * 512)) != STB_OK || (rc = db.alloc(n_pad * 512)) != STB_OK ||
      (rc = dfull.alloc(q_pad * n_pad)) != STB_OK || (rc = dsub.alloc((size_t)n_tiles * 8 * q_pad)) != STB_OK ||
      (rc = dtile.alloc((size_t)n_tiles * q_pad)) != STB_OK || (rc = dbad.alloc(1)) != STB_OK)
    return rc;
  cudaError_t e = cudaMemsetAsync(dbad, 0, 4, ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dq, q, (size_t)nq * 1024, cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dr, rows, n * 1024, cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) rc = stb_launch_shadow_build(ctx, dq, nq, 128, da, dbad);
  if (e == cudaSuccess && rc == STB_OK) rc = stb_launch_shadow_build(ctx, dr, n, 256, db, dbad);
  StbGemmPass p;
  p.epi = STB_EPI_DEBUG; p.a_tiles = da; p.b_tiles = db; p.m_tiles = m_tiles; p.n_tiles = n_tiles; p.n_rows = n;
  p.full_out = dfull;
  if (e == cudaSuccess && rc == STB_OK) rc = stb_launch_gemm(ctx, p);
  p.epi = STB_EPI_SAMPLE; p.submax = dsub; p.tilemax = dtile;
  if (e == cudaSuccess && rc == STB_OK) rc = stb_launch_gemm(ctx, p);
  if (e == cudaSuccess && rc == STB_OK) e = cudaMemcpyAsync(out_full, dfull, q_pad * n_pad * 4, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess && rc == STB_OK && out_submax) e = cudaMemcpyAsync(out_submax, dsub, (size_t)n_tiles * 8 * q_pad * 4, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess && rc == STB_OK) e = cudaStreamSynchronize(ctx->stream);
  if (e != cudaSuccess) { stb_set_error("debug_batch_gemm: %s", cudaGetErrorString(e)); cudaGetLastError(); return STB_ERR_CUDA; }
  return rc;
}

// The q8 copy's query tiles and integer GEMM over a corpus's q8 copy (built or extended first): per query its q16
// [nq][256], and per (query, row) the int32 dot and the bounds u, l [nq][n].
int stb_debug_batch_q8_gemm(stb_ctx *ctx, const stb_corpus *corpus_c, const float *q, uint32_t nq, int16_t *q16,
                            int32_t *dot, float *u, float *l) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  stb_corpus *corpus = const_cast<stb_corpus *>(corpus_c);
  if (!corpus || !q || !q16 || !dot || !u || !l || nq == 0 || corpus->n == 0) { stb_set_error("debug_batch_q8_gemm: bad argument"); return STB_ERR_ARG; }
  if (corpus->ctx != ctx) { stb_set_error("debug_batch_q8_gemm: corpus belongs to another context"); return STB_ERR_ARG; }
  if ((rc = corpus_ensure(ctx, corpus, corpus->q8)) != STB_OK) return rc;
  const uint32_t m_tiles = (nq + 127) / 128;
  const size_t q_pad = (size_t)m_tiles * 128, n = corpus->n, n_pad = (n + 255) / 256 * 256;
  StbBuf<float> dq, du, dl;
  StbBuf<uint8_t> da;
  StbBuf<float4> dc;
  StbBuf<uint32_t> dbad;
  StbBuf<int16_t> d16;
  StbBuf<int32_t> ddot;
  if ((rc = dq.alloc((size_t)nq * STB_D)) != STB_OK || (rc = da.alloc(q_pad * 512)) != STB_OK || (rc = dc.alloc(q_pad)) != STB_OK ||
      (rc = dbad.alloc(q_pad)) != STB_OK || (rc = d16.alloc((size_t)nq * STB_D)) != STB_OK ||
      (rc = ddot.alloc(q_pad * n_pad)) != STB_OK || (rc = du.alloc(q_pad * n_pad)) != STB_OK || (rc = dl.alloc(q_pad * n_pad)) != STB_OK)
    return rc;
  StbGemmPass p;
  p.copy = STB_GEMM_Q8; p.epi = STB_EPI_DEBUG; p.a_tiles = da; p.m_tiles = m_tiles; p.n_tiles = (uint32_t)(n_pad / 256);
  p.n_rows = n; p.b_tiles = corpus->q8.codes; p.q8_scale = corpus->q8.scale; p.qc = dc;
  p.dot_out = ddot; p.u_out = du; p.l_out = dl;
  STB_CUDA(cudaMemcpyAsync(dq, q, (size_t)nq * STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = stb_launch_q8_query_tiles(ctx, dq, nq, (uint32_t)q_pad, da, dc, dbad, d16)) != STB_OK ||
      (rc = stb_launch_gemm(ctx, p)) != STB_OK)
    return rc;
  STB_CUDA(cudaMemcpyAsync(q16, d16, (size_t)nq * STB_D * sizeof(int16_t), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaMemcpy2DAsync(dot, n * 4, ddot, n_pad * 4, n * 4, nq, cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaMemcpy2DAsync(u, n * 4, du, n_pad * 4, n * 4, nq, cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaMemcpy2DAsync(l, n * 4, dl, n_pad * 4, n * 4, nq, cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  return STB_OK;
}

// ------------------------------------------------------------------- K1 debug hooks ---
// The scan passes' per-row scores, for tests that check each pass's contract row by row (DESIGN.md section 5).

// Query and ranges staged like stb_search's; per-row device outputs: `floats` arrays of n f32 (NaN-filled) and one of
// n u32 (zeroed), in the one buffer f_dev.
static int k1_debug_stage(stb_ctx *ctx, const stb_corpus *c, const char *what, const float *q, const uint64_t *row_ranges,
                          uint32_t n_ranges, int floats, StbBuf<float> &f_dev, unsigned int **u_dev, StbRowRanges *ranges) {
  int rc;
  if ((rc = k1_upload_ranges(ctx, c, what, row_ranges, n_ranges, ranges)) != STB_OK) return rc;
  if ((rc = k1_stage_query(ctx, q)) != STB_OK) return rc;
  const size_t n = c->n;
  if ((rc = f_dev.alloc(n * (floats + 1))) != STB_OK) return rc;
  *u_dev = (unsigned int *)(f_dev + n * floats);
  STB_CUDA(cudaMemsetAsync(f_dev, 0xff, n * sizeof(float) * floats, ctx->stream));
  STB_CUDA(cudaMemsetAsync(*u_dev, 0, n * sizeof(unsigned int), ctx->stream));
  return STB_OK;
}

int stb_debug_scan_scores(stb_ctx *ctx, const stb_corpus *corpus, int tier, const float *q, const uint64_t *row_ranges,
                          uint32_t n_ranges, uint64_t cap, float *scores, uint32_t *seen, uint32_t *hist) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!corpus || !q || !scores || !seen || (n_ranges && !row_ranges)) { stb_set_error("debug_scan_scores: null argument"); return STB_ERR_ARG; }
  if (corpus->ctx != ctx) { stb_set_error("debug_scan_scores: corpus belongs to another context"); return STB_ERR_ARG; }
  if (tier < STB_TIER_F32 || tier > STB_TIER_Q8) { stb_set_error("debug_scan_scores: unknown tier %d", tier); return STB_ERR_ARG; }
  if (hist && tier == STB_TIER_H16) { stb_set_error("debug_scan_scores: no histogram pass reads the 16-bit shadow"); return STB_ERR_ARG; }
  if (cap < corpus->n) { stb_set_error("debug_scan_scores: outputs hold %llu rows, the corpus %llu", (unsigned long long)cap, (unsigned long long)corpus->n); return STB_ERR_ARG; }
  if (!corpus->tier_usable(tier)) { stb_set_error("debug_scan_scores: tier %d copy not built or unusable", tier); return STB_ERR_STATE; }
  if (hist) memset(hist, 0, 4096 * sizeof(uint32_t));
  if (corpus->n == 0) return STB_OK;
  StbBuf<float> d_score;
  unsigned int *d_seen = nullptr;
  StbRowRanges ranges = {nullptr, 0, 0};
  if ((rc = k1_debug_stage(ctx, corpus, "debug_scan_scores", q, row_ranges, n_ranges, 1, d_score, &d_seen, &ranges)) == STB_OK &&
      ranges.n_virtual) {
    rc = stb_launch_debug_scan(ctx, corpus, tier, ctx->q_dev, ranges, d_score, d_seen);
    if (rc == STB_OK && hist) rc = stb_launch_scan_hist(ctx, corpus, tier, ctx->q_dev, ranges, ctx->hist_dev);
  }
  cudaError_t e = cudaSuccess;
  if (rc == STB_OK) e = cudaMemcpyAsync(scores, d_score, corpus->n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream);
  if (rc == STB_OK && e == cudaSuccess) e = cudaMemcpyAsync(seen, d_seen, corpus->n * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream);
  if (rc == STB_OK && e == cudaSuccess && hist && ranges.n_virtual)
    e = cudaMemcpyAsync(hist, ctx->hist_dev, 4096 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (rc == STB_OK && e != cudaSuccess) { stb_set_error("debug_scan_scores: %s", cudaGetErrorString(e)); cudaGetLastError(); return STB_ERR_CUDA; }
  return rc;
}

int stb_debug_q4_scan(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t top_k, const uint64_t *row_ranges,
                      uint32_t n_ranges, int pin, uint64_t cap, float *u4, float *t, uint32_t *refined, float *u8, float *l8,
                      uint64_t *words) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!corpus || !q || !u4 || !t || !refined || !u8 || !l8 || !words || (n_ranges && !row_ranges)) {
    stb_set_error("debug_q4_scan: null argument");
    return STB_ERR_ARG;
  }
  if (corpus->ctx != ctx) { stb_set_error("debug_q4_scan: corpus belongs to another context"); return STB_ERR_ARG; }
  if (top_k < 1 || top_k > STB_Q8_MAX_K) { stb_set_error("debug_q4_scan: top_k must be 1..%d", STB_Q8_MAX_K); return STB_ERR_ARG; }
  if (cap < corpus->n) { stb_set_error("debug_q4_scan: outputs hold %llu rows, the corpus %llu", (unsigned long long)cap, (unsigned long long)corpus->n); return STB_ERR_ARG; }
  if (!corpus->tier_usable(STB_TIER_Q8)) { stb_set_error("debug_q4_scan: q8 copy not built or unusable"); return STB_ERR_STATE; }
  memset(words, 0, top_k * sizeof(uint64_t));
  if (corpus->n == 0) return STB_OK;
  const size_t n = corpus->n;
  StbBuf<float> d_f;
  unsigned int *d_seen = nullptr;
  StbBuf<unsigned long long> d_words;
  StbRowRanges ranges = {nullptr, 0, 0};
  rc = k1_debug_stage(ctx, corpus, "debug_q4_scan", q, row_ranges, n_ranges, 4, d_f, &d_seen, &ranges);
  cudaError_t e = cudaSuccess;
  if (rc == STB_OK && (rc = d_words.alloc(STB_Q4_WORDS + 1)) == STB_OK)   // the words, then the refined counter
    e = cudaMemsetAsync(d_words, 0, (STB_Q4_WORDS + 1) * sizeof(unsigned long long), ctx->stream);
  if (rc == STB_OK && e == cudaSuccess && ranges.n_virtual)
    rc = stb_launch_debug_q4(ctx, corpus, ctx->q_dev, top_k, ranges, d_words, d_words + STB_Q4_WORDS, pin, d_f, d_f + n,
                             d_f + 2 * n, d_f + 3 * n, d_seen);
  float *outs[4] = {u4, t, l8, u8};
  for (int i = 0; i < 4 && rc == STB_OK && e == cudaSuccess; ++i)
    e = cudaMemcpyAsync(outs[i], d_f + i * n, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream);
  if (rc == STB_OK && e == cudaSuccess) e = cudaMemcpyAsync(refined, d_seen, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream);
  if (rc == STB_OK && e == cudaSuccess) e = cudaMemcpyAsync(words, d_words, top_k * sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (rc == STB_OK && e != cudaSuccess) { stb_set_error("debug_q4_scan: %s", cudaGetErrorString(e)); cudaGetLastError(); return STB_ERR_CUDA; }
  return rc;
}

int stb_search_xchg(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t top_k, stb_xchg *x,
                    stb_hit *out_hits, uint32_t *out_n, int *out_complete) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!q || !out_hits || !out_n || !out_complete) { stb_set_error("search_xchg: null argument"); return STB_ERR_ARG; }
  if ((rc = host_rows_refuse(corpus, "search_xchg")) != STB_OK) return rc;
  if ((rc = k1_stage_query(ctx, q)) != STB_OK) return rc;
  // the merge CTA stores the hits + status straight into pinned host memory
  if ((rc = stb_search_topk_xchg(ctx, corpus, ctx->q_dev, top_k, x, ctx->hits_pin, ctx->status_pin)) != STB_OK) return rc;
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  const K1Status st = k1_status(ctx->status_pin, top_k);
  memcpy(out_hits, ctx->hits_pin, st.n * sizeof(stb_hit));
  *out_n = st.n;
  *out_complete = st.proven ? 1 : 0;
  if (st.timeout) { x->dead = true; stb_set_error("search_xchg: a peer rank never arrived (timeout)"); return STB_ERR_STATE; }
  return STB_OK;
}

// Many independent single queries with ONE synchronisation: queries are staged through pinned
// memory in one H2D copy, the nq scan kernels are enqueued back to back (PDL overlaps each tail
// with the next scan) and every kernel's final CTA stores its hits + status straight into pinned
// host memory.  Unproven queries are re-run through stb_search (x == NULL) or reported
// (x != NULL: all ranks see the same flag and fall back together).
int stb_search_many(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t nq, uint32_t top_k, stb_xchg *x,
                    stb_hit *out_hits, uint32_t *out_n, uint8_t *out_complete) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!corpus || !q || !out_hits || !out_n) { stb_set_error("search_many: null argument"); return STB_ERR_ARG; }
  if (corpus->ctx != ctx || (x && x->ctx != ctx)) { stb_set_error("search_many: handles belong to another context"); return STB_ERR_ARG; }
  if (x && (rc = host_rows_refuse(corpus, "search_many with an exchange")) != STB_OK) return rc;
  if (nq == 0) return STB_OK;
  for (uint32_t i = 0; i < nq; ++i) { out_n[i] = 0; if (out_complete) out_complete[i] = 1; }
  if (top_k == 0 || corpus->n == 0) {
    if (x && corpus->n == 0) { stb_set_error("search_many: empty shard in a sharded search"); return STB_ERR_STATE; }
    return STB_OK;
  }
  if (x && top_k > x->max_k) { stb_set_error("search_many: top_k must be 1..%u", x->max_k); return STB_ERR_ARG; }
  const bool scan = top_k <= stb_scan_topk_max_k();   // beyond the register lists: every query takes stb_search
  if (scan) {
    // many queries amortise the int8 copy: build or extend it now (same size rule as the lazy build);
    // otherwise the launches read the narrowest copy already built
    const bool eager = nq >= 2 && corpus->n >= 32768;
    int tier;
    if ((rc = k1_async_tier(ctx, corpus, top_k, {eager, eager}, "search_many", &tier)) != STB_OK) return rc;
    if ((rc = ctx->bq_dev.reserve((size_t)nq * STB_D)) != STB_OK) return rc;
    if ((rc = ctx->hits_pin.reserve((size_t)nq * top_k, 2 * ctx->hits_pin.cap)) != STB_OK) return rc;
    if ((size_t)nq * STB_D > ctx->many_q_pin.cap || (size_t)nq * 4 > ctx->many_status_pin.cap) {
      const size_t cap = std::max<size_t>((size_t)nq, 64);
      if ((rc = ctx->many_q_pin.alloc(cap * STB_D)) != STB_OK || (rc = ctx->many_status_pin.alloc(cap * 4)) != STB_OK) return rc;
    }
    memcpy(ctx->many_q_pin, q, (size_t)nq * STB_D * sizeof(float));
    STB_CUDA(cudaMemcpyAsync(ctx->bq_dev, ctx->many_q_pin, (size_t)nq * STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    for (uint32_t i = 0; i < nq; ++i) {
      stb_hit *oh = ctx->hits_pin + (size_t)i * top_k;
      uint32_t *os = ctx->many_status_pin + 4 * (size_t)i;
      if (x) rc = stb_search_topk_xchg(ctx, corpus, ctx->bq_dev + (size_t)i * STB_D, top_k, x, oh, os);
      else rc = stb_launch_scan_topk(ctx, corpus, tier, ctx->bq_dev + (size_t)i * STB_D, top_k, {nullptr, 0, corpus->n}, oh, os,
                                     nullptr, nq > 1);
      if (rc != STB_OK) { cudaStreamSynchronize(ctx->stream); return rc; }
    }
    STB_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  for (uint32_t i = 0; i < nq; ++i) {
    if (scan) {
      const K1Status st = k1_status(ctx->many_status_pin + 4 * (size_t)i, top_k);
      if (x && st.timeout) { x->dead = true; stb_set_error("search_many: a peer rank never arrived (timeout)"); return STB_ERR_STATE; }
      if (st.proven) {
        memcpy(out_hits + (size_t)i * top_k, ctx->hits_pin + (size_t)i * top_k, st.n * sizeof(stb_hit));
        out_n[i] = st.n;
        continue;
      }
      if (x) {
        if (out_complete) out_complete[i] = 0;             // every rank sees the same flag: fall back together
        continue;
      }
    }
    uint64_t n = 0;                                        // tier ladder / collect path
    rc = stb_search(ctx, corpus, q + (size_t)i * STB_D, top_k, 0, 0.0, STB_MODE_SEARCH_DOCUMENTS, nullptr, 0,
                    out_hits + (size_t)i * top_k, top_k, &n);
    if (rc != STB_OK) return rc;
    out_n[i] = (uint32_t)n;
  }
  return STB_OK;
}

// ---------------------------------------------------------------------- merge ---
int stb_hits_merge_dev(stb_ctx *ctx, const stb_hit *lists_dev, uint32_t n_lists, uint32_t per_list,
                       uint32_t top_k, stb_hit *out_dev) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!lists_dev || !out_dev || n_lists == 0 || per_list == 0 || top_k == 0) { stb_set_error("hits_merge: bad argument"); return STB_ERR_ARG; }
  return stb_launch_hits_merge(ctx, lists_dev, n_lists, per_list, top_k, out_dev);
}

int stb_hits_merge_batch_dev(stb_ctx *ctx, const stb_hit *lists_dev, uint32_t n_lists, uint32_t nq,
                             uint32_t per_list, uint32_t top_k, stb_hit *out_dev) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!lists_dev || !out_dev || n_lists == 0 || per_list == 0 || top_k == 0) { stb_set_error("hits_merge_batch: bad argument"); return STB_ERR_ARG; }
  if (nq == 0) return STB_OK;
  return stb_launch_hits_merge_batch(ctx, lists_dev, n_lists, nq, per_list, top_k, out_dev);
}

int stb_hits_merge(stb_ctx *ctx, const stb_hit *lists, uint32_t n_lists, uint32_t per_list,
                   uint32_t top_k, stb_hit *out, uint32_t *out_n) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!lists || !out || !out_n || n_lists == 0 || per_list == 0) { stb_set_error("hits_merge: bad argument"); return STB_ERR_ARG; }
  *out_n = 0;
  if (top_k == 0) return STB_OK;
  const size_t total = (size_t)n_lists * per_list;
  if ((rc = ctx->hits_dev.reserve(total + top_k)) != STB_OK) return rc;
  if ((rc = ctx->hits_pin.reserve(std::max<size_t>(total, top_k), 2 * ctx->hits_pin.cap)) != STB_OK) return rc;
  memcpy(ctx->hits_pin, lists, total * sizeof(stb_hit));
  STB_CUDA(cudaMemcpyAsync(ctx->hits_dev, ctx->hits_pin, total * sizeof(stb_hit), cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = stb_launch_hits_merge(ctx, ctx->hits_dev, n_lists, per_list, top_k, ctx->hits_dev + total)) != STB_OK) return rc;
  STB_CUDA(cudaMemcpyAsync(ctx->hits_pin, ctx->hits_dev + total, top_k * sizeof(stb_hit), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  uint32_t n = 0;
  for (uint32_t i = 0; i < top_k; ++i) {
    if (ctx->hits_pin[i].row == 0xffffffffffffffffull) break;
    out[n++] = ctx->hits_pin[i];
  }
  *out_n = n;
  return STB_OK;
}

// ------------------------------------------------------------------------ ids ---
uint64_t stb_fnv1a64(const uint8_t *bytes, uint64_t len) {
  uint64_t h = 0xcbf29ce484222325ull;
  for (uint64_t i = 0; i < len; ++i) { h ^= bytes[i]; h *= 0x100000001b3ull; }
  return h;
}

uint64_t stb_line_id(const uint8_t *path, uint64_t path_len, int32_t line_number) {
  uint64_t h = 0xcbf29ce484222325ull;
  for (uint64_t i = 0; i < path_len; ++i) { h ^= path[i]; h *= 0x100000001b3ull; }
  const uint32_t u = (uint32_t)line_number;
  for (int b = 0; b < 4; ++b) { h ^= (u >> (8 * b)) & 0xffu; h *= 0x100000001b3ull; }
  return h;
}

// LineEmbedding::id for many rows at once: rows = n_rows x (path index, line_number) int32, paths
// given as one byte blob + n_paths+1 offsets.  The FNV state after each path is computed once.
int stb_line_ids(const uint8_t *path_bytes, const uint64_t *path_offsets, uint32_t n_paths, const int32_t *rows,
                 uint64_t n_rows, uint64_t *out_ids) {
  if ((n_paths && (!path_bytes || !path_offsets)) || (n_rows && (!rows || !out_ids))) { stb_set_error("line_ids: null argument"); return STB_ERR_ARG; }
  std::vector<uint64_t> prefix(n_paths);
  for (uint32_t p = 0; p < n_paths; ++p) {
    uint64_t h = 0xcbf29ce484222325ull;
    for (uint64_t i = path_offsets[p]; i < path_offsets[p + 1]; ++i) { h ^= path_bytes[i]; h *= 0x100000001b3ull; }
    prefix[p] = h;
  }
  for (uint64_t r = 0; r < n_rows; ++r) {
    const int32_t pi = rows[2 * r];
    if (pi < 0 || (uint32_t)pi >= n_paths) { stb_set_error("line_ids: row %llu refers to path %d of %u", (unsigned long long)r, pi, n_paths); return STB_ERR_RANGE; }
    uint64_t h = prefix[pi];
    const uint32_t u = (uint32_t)rows[2 * r + 1];
    for (int b = 0; b < 4; ++b) { h ^= (u >> (8 * b)) & 0xffu; h *= 0x100000001b3ull; }
    out_ids[r] = h;
  }
  return STB_OK;
}

}  // extern "C"

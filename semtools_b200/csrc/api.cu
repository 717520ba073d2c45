// C ABI of libsemtools_b200.so (include/semtools_b200.h).  Host-side orchestration
// only: argument checking, HBM residency, staging copies, and the exact
// fallback ladder around the scan kernel.  No CPU implementation of any kernel
// exists in this library: without an sm_90 device every entry point fails.
#include <stdarg.h>
#include <stdlib.h>

#include <algorithm>
#include <mutex>
#include <new>
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

template <class T>
static int dev_reserve(T **p, size_t *cap, size_t need, size_t floor_cap = 0) {
  if (need <= *cap && *p) return STB_OK;
  size_t ncap = std::max(std::max(need, floor_cap), *cap + *cap / 2);
  T *np = nullptr;
  cudaError_t e = cudaMalloc((void **)&np, ncap * sizeof(T));
  if (e != cudaSuccess) {
    cudaGetLastError();
    stb_set_error("cudaMalloc(%zu bytes) failed: %s", ncap * sizeof(T), cudaGetErrorString(e));
    return STB_ERR_NOMEM;
  }
  if (*p) cudaFree(*p);
  *p = np;
  *cap = ncap;
  return STB_OK;
}

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
  memset(c, 0, sizeof(*c));
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
  if ((rc = dev_reserve(&c->block_keys, &c->block_keys_cap, 2 * max_grid * 129 + STB_SORT_CAP)) != STB_OK) goto fail;
  if ((rc = dev_reserve(&c->counters, &c->counters_cap, max_grid + 64)) != STB_OK) goto fail;
  {
    size_t one = 0;
    if ((rc = dev_reserve(&c->q_dev, &one, STB_D)) != STB_OK) goto fail;
    one = 0;
    if ((rc = dev_reserve(&c->status_dev, &one, 8)) != STB_OK) goto fail;
    one = 0;
    if ((rc = dev_reserve(&c->collect_count, &one, 2)) != STB_OK) goto fail;
    one = 0;
    if ((rc = dev_reserve(&c->err_flag, &one, 1)) != STB_OK) goto fail;
    one = 0;
    if ((rc = dev_reserve(&c->embed_flag, &one, 1)) != STB_OK) goto fail;
    one = 0;
    if ((rc = dev_reserve(&c->hist_dev, &one, 4096)) != STB_OK) goto fail;
    one = 0;
    if ((rc = dev_reserve(&c->tickets, &one, STB_TICKET_SLOTS)) != STB_OK) goto fail;
    one = 0;
    if ((rc = dev_reserve(&c->q4_thr, &one, STB_TICKET_SLOTS * STB_Q4_WORDS)) != STB_OK) goto fail;
    one = 0;
    if ((rc = dev_reserve(&c->q4_refined, &one, 1)) != STB_OK) goto fail;
    one = 0;
    if ((rc = dev_reserve(&c->coscan_off, &one, STB_TICKET_SLOTS)) != STB_OK) goto fail;
  }
  if ((rc = dev_reserve(&c->hits_dev, &c->hits_cap, 1024)) != STB_OK) goto fail;
  if (cudaMemset(c->counters, 0, c->counters_cap * sizeof(unsigned int)) != cudaSuccess ||
      cudaMemset(c->tickets, 0, STB_TICKET_SLOTS * sizeof(unsigned long long)) != cudaSuccess ||
      cudaMemset(c->q4_thr, 0, STB_TICKET_SLOTS * STB_Q4_WORDS * sizeof(unsigned long long)) != cudaSuccess ||
      cudaMemset(c->q4_refined, 0, sizeof(unsigned long long)) != cudaSuccess ||
      cudaMemset(c->coscan_off, 0, STB_TICKET_SLOTS * sizeof(unsigned long long)) != cudaSuccess ||
      cudaMemset(c->err_flag, 0, sizeof(int)) != cudaSuccess ||
      cudaMemset(c->embed_flag, 0, sizeof(int)) != cudaSuccess ||
      cudaMallocHost((void **)&c->q_pin, STB_D * sizeof(float)) != cudaSuccess ||
      cudaMallocHost((void **)&c->status_pin, 8 * sizeof(uint32_t)) != cudaSuccess ||
      cudaMallocHost((void **)&c->hits_pin, 1024 * sizeof(stb_hit)) != cudaSuccess) {
    stb_set_error("context staging allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
    rc = STB_ERR_NOMEM;
    goto fail;
  }
  c->hits_pin_cap = 1024;
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
  cudaFree(c->block_keys); cudaFree(c->counters); cudaFree(c->q_dev); cudaFree(c->hits_dev);
  cudaFree(c->status_dev); cudaFree(c->collect_rows); cudaFree(c->collect_count);
  cudaFree(c->collect_hits); cudaFree(c->ranges_dev); cudaFree(c->err_flag); cudaFree(c->embed_flag);
  cudaFree(c->tickets); cudaFree(c->q4_thr); cudaFree(c->q4_refined); cudaFree(c->coscan_off);
  cudaFree(c->hist_dev); cudaFree(c->bq_tiles); cudaFree(c->b_submax); cudaFree(c->b_tilemax); cudaFree(c->b_cand);
  cudaFree(c->b_thr); cudaFree(c->b_cnt); cudaFree(c->b_keys); cudaFree(c->b_qbad);
  cudaFree(c->b_franges); cudaFree(c->b_ftiles); cudaFree(c->b_fbits);
  cudaFree(c->bq_dev); cudaFree(c->bh_dev); cudaFree(c->bs_dev); cudaFree(c->embed_off_dev); cudaFree(c->embed_ids_dev); cudaFree(c->embed_out_dev);
  cudaFree(c->mut_stage); cudaFree(c->mut_idx); cudaFree(c->mut_flags);
  if (c->q_pin) cudaFreeHost(c->q_pin);
  if (c->hits_pin) cudaFreeHost(c->hits_pin);
  if (c->status_pin) cudaFreeHost(c->status_pin);
  if (c->many_q_pin) cudaFreeHost(c->many_q_pin);
  if (c->many_status_pin) cudaFreeHost(c->many_status_pin);
  if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
  cudaGetLastError();
  delete c;
  return STB_OK;
}

int stb_ctx_sync(stb_ctx *ctx) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  return STB_OK;
}

void *stb_ctx_stream(stb_ctx *ctx) { return ctx ? (void *)ctx->stream : nullptr; }

// K1's tile tickets: every top-k launch must advance the device counter by exactly what the host
// booked for it (n_tickets + total_warps); a mismatch would make later launches skip or repeat
// tiles.  Synchronises; returns STB_ERR_STATE on a mismatch.
int stb_debug_ticket_check(stb_ctx *ctx, uint64_t *device_value, uint64_t *host_value) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  unsigned long long v[STB_TICKET_SLOTS];
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  STB_CUDA(cudaMemcpy(v, ctx->tickets, sizeof(v), cudaMemcpyDeviceToHost));
  unsigned long long dsum = 0, hsum = 0;
  int bad = -1;
  for (int i = 0; i < STB_TICKET_SLOTS; ++i) { dsum += v[i]; hsum += ctx->ticket_next[i]; if (v[i] != ctx->ticket_next[i] && bad < 0) bad = i; }
  if (device_value) *device_value = dsum;          // sums over the counter ring
  if (host_value) *host_value = hsum;
  if (bad >= 0) { stb_set_error("ticket counter %d is %llu, host expects %llu", bad, v[bad], ctx->ticket_next[bad]); return STB_ERR_STATE; }
  return STB_OK;
}

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

// The tile offsets K1's last n top-k launches on the ticket ring started their pass at, oldest first;
// 0xffffffff for a launch that did not co-scan (or whose slot a later launch reused).  Synchronises.
int stb_debug_coscan_offsets(stb_ctx *ctx, uint32_t n, uint32_t *out) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (n > STB_TICKET_SLOTS || (n && !out)) { stb_set_error("coscan_offsets: n must be 0..%d", STB_TICKET_SLOTS); return STB_ERR_ARG; }
  unsigned long long w[STB_TICKET_SLOTS];
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  STB_CUDA(cudaMemcpy(w, ctx->coscan_off, sizeof(w), cudaMemcpyDeviceToHost));
  for (uint32_t i = 0; i < n; ++i) {
    out[i] = 0xffffffffu;
    if (ctx->topk_launches < n - i) continue;
    const int slot = (int)((ctx->topk_launches - (n - i)) % STB_TICKET_SLOTS);
    const uint32_t tag = ctx->coscan_tag[slot];
    if (tag && (uint32_t)(w[slot] >> 32) == tag) out[i] = (uint32_t)w[slot];
  }
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
  memset(t, 0, sizeof(*t));
  t->ctx = ctx; t->V = V; t->normalize = normalize ? 1 : 0;
  t->n_weights = weights ? n_weights : 0;
  t->n_mapping = mapping ? n_mapping : 0;
  cudaError_t e = cudaMalloc((void **)&t->E, V * STB_D * sizeof(float));
  if (e == cudaSuccess && t->n_weights) e = cudaMalloc((void **)&t->weights, t->n_weights * sizeof(float));
  if (e == cudaSuccess && t->n_mapping) e = cudaMalloc((void **)&t->mapping, t->n_mapping * sizeof(uint32_t));
  if (e != cudaSuccess) {
    cudaGetLastError();
    stb_set_error("table_load: device allocation failed: %s", cudaGetErrorString(e));
    stb_table_destroy(t);
    return STB_ERR_NOMEM;
  }
  e = cudaMemcpyAsync(t->E, E, V * STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream);
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
  cudaFree(t->E); cudaFree(t->weights); cudaFree(t->mapping);
  cudaGetLastError();
  delete t;
  return STB_OK;
}

// -------------------------------------------------------------------- corpus ---
static int corpus_reserve(stb_corpus *c, uint64_t need) {
  if (need <= c->capacity && c->rows) return STB_OK;
  if (need > 0xfffffffeull) { stb_set_error("corpus shard exceeds 2^32-2 rows; shard it"); return STB_ERR_ARG; }
  uint64_t ncap = std::max<uint64_t>(std::max<uint64_t>(need, 1024), c->capacity + c->capacity / 2);
  float *np = nullptr;
  cudaError_t e = cudaMalloc((void **)&np, ncap * STB_D * sizeof(float));
  if (e != cudaSuccess) {
    cudaGetLastError();
    stb_set_error("corpus: cudaMalloc(%llu rows) failed: %s", (unsigned long long)ncap, cudaGetErrorString(e));
    return STB_ERR_NOMEM;
  }
  if (c->rows && c->n) {
    e = cudaMemcpyAsync(np, c->rows, c->n * STB_D * sizeof(float), cudaMemcpyDeviceToDevice, c->ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->ctx->stream);
    if (e != cudaSuccess) { cudaFree(np); stb_set_error("corpus grow copy: %s", cudaGetErrorString(e)); return STB_ERR_CUDA; }
  }
  if (c->rows) cudaFree(c->rows);
  c->rows = np;
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
  memset(c, 0, sizeof(*c));
  c->ctx = ctx; c->row_base = row_base;
  rc = corpus_reserve(c, std::max<uint64_t>(capacity_rows, 1));
  if (rc) { delete c; return rc; }
  *out = c;
  return STB_OK;
}

int stb_corpus_destroy(stb_corpus *c) {
  if (!c) return STB_OK;
  if (c->ctx && ctx_alive(c->ctx)) { cudaSetDevice(c->ctx->device); cudaStreamSynchronize(c->ctx->stream); }
  else cudaDeviceSynchronize();
  cudaFree(c->shadow);
  cudaFree(c->q8);
  cudaFree(c->q8_scale);
  cudaFree(c->q4);
  cudaFree(c->q4_sr);
  cudaFree(c->rows);
  cudaGetLastError();
  delete c;
  return STB_OK;
}

// The reduced-width copies (K2 shadow, K1 tiers) cover a PREFIX of the rows: an append leaves the
// prefix valid and the next query / prepare only converts the new rows (q8_rows / shadow_rows < n);
// an update or a removal re-encodes the copies at the rows it writes, so they stay built; a clear drops
// them.  Anything but an append starts a new epoch; an update or a removal also ends a co-scan series on
// the corpus (the next asynchronous top-k query starts at tile 0).
enum CorpusChange { CORPUS_APPEND, CORPUS_ROWS_REWRITTEN, CORPUS_CLEAR };
static void corpus_changed(stb_corpus *c, CorpusChange kind) {
  if (kind == CORPUS_CLEAR) { c->shadow_rows = 0; c->q8_rows = 0; }
  if (kind != CORPUS_APPEND) ++c->epoch;
  if (kind == CORPUS_ROWS_REWRITTEN && c->ctx->coscan_prev.rows == c->rows) c->ctx->coscan_prev.rows = nullptr;
  c->searches_since_change = 0;
  memset(c->tier_tries, 0, sizeof(c->tier_tries));
  memset(c->tier_proven, 0, sizeof(c->tier_proven));
}

static int corpus_append_impl(stb_corpus *c, const float *rows, uint64_t n, cudaMemcpyKind kind) {
  if (!c) { stb_set_error("null corpus"); return STB_ERR_ARG; }
  int rc = ctx_use(c->ctx);
  if (rc) return rc;
  if (n == 0) return STB_OK;
  if (!rows) { stb_set_error("corpus_append: rows is null"); return STB_ERR_ARG; }
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
  if ((rc = dev_reserve(&ctx->embed_off_dev, &ctx->embed_off_cap, n_lines + 1, 4096)) != STB_OK) return rc;
  if ((rc = dev_reserve(&ctx->embed_ids_dev, &ctx->embed_ids_cap, std::max<uint64_t>(total, 1), 65536)) != STB_OK) return rc;
  float *dst = nullptr;
  if (append_to) {
    if ((rc = corpus_reserve(append_to, append_to->n + n_lines)) != STB_OK) return rc;
    dst = append_to->rows + append_to->n * STB_D;
  } else {
    if ((rc = dev_reserve(&ctx->embed_out_dev, &ctx->embed_out_cap, n_lines * STB_D, 4096 * STB_D)) != STB_OK) return rc;
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
static int corpus_ensure_shadow(stb_ctx *ctx, stb_corpus *c);   // defined with the K2 entry points
static int corpus_ensure_q8(stb_ctx *ctx, stb_corpus *c);

// STB_SCAN_TIER = f32 | h16 | q8: the narrowest candidate tier K1 may use (default q8).  Read per
// call so one process can compare tiers; results are identical whatever the value.
static int stb_env_max_tier() {
  const char *e = getenv("STB_SCAN_TIER");
  if (!e || !e[0]) return STB_TIER_Q8;
  if (e[0] == 'f') return STB_TIER_F32;
  if (e[0] == 'h') return STB_TIER_H16;
  return STB_TIER_Q8;
}
// The single-GPU asynchronous entry points (stb_search_topk_dev, stb_search_many without an exchange) always
// use the overlapped launch mode and co-scan (scan_topk.cu: stb_coscan_offset): back-to-back queries share
// each tile's HBM read.  The sharded forms (stb_search_topk_xchg, stb_search_many with an exchange) launch
// like the synchronous entry points (full grid, dependent released after the scan).

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
  const bool q8 = tier == STB_TIER_Q8;
  const bool have = q8 ? c->q8 != nullptr : c->shadow != nullptr;
  const uint64_t rows = q8 ? c->q8_rows : c->shadow_rows;
  const bool bad = q8 ? c->q8_bad : c->shadow_bad;
  if (have && rows == c->n) { *ready = !bad; return STB_OK; }
  if (!policy.build && !(policy.extend && have && rows > 0 && !bad)) return STB_OK;
  const int rc = q8 ? corpus_ensure_q8(ctx, c) : corpus_ensure_shadow(ctx, c);
  *ready = rc == STB_OK;
  return rc == STB_ERR_STATE ? STB_OK : rc;
}

// The narrowest copy that is fully built and usable: the asynchronous entry points never build one
// (stb_corpus_prepare does).
static int best_built_tier(stb_ctx *ctx, const stb_corpus *c, uint32_t top_k) {
  for (int tier = STB_TIER_Q8; tier > STB_TIER_F32; --tier) {
    bool ready = false;
    k1_copy_ready(ctx, const_cast<stb_corpus *>(c), tier, top_k, kBuiltOnly, &ready);   // builds nothing: cannot fail
    if (ready) return tier;
  }
  return STB_TIER_F32;
}

static int ensure_hits_pin(stb_ctx *ctx, size_t need) {
  if (need <= ctx->hits_pin_cap) return STB_OK;
  stb_hit *np = nullptr;
  size_t ncap = std::max(need, ctx->hits_pin_cap * 2);
  if (cudaMallocHost((void **)&np, ncap * sizeof(stb_hit)) != cudaSuccess) {
    cudaGetLastError();
    stb_set_error("pinned staging allocation failed");
    return STB_ERR_NOMEM;
  }
  cudaFreeHost(ctx->hits_pin);
  ctx->hits_pin = np;
  ctx->hits_pin_cap = ncap;
  return STB_OK;
}

// The distance cap of a top-k result sorted by (distance, row): how many leading hits have distance <
// max_distance (strict; a NaN cap passes none).  Where top_k always caps (store-query mode, the top-k fast
// path) the capped result is this prefix of the uncapped one.
static uint64_t capped_hits(const stb_hit *hits, uint64_t n, int has_max, double max_distance) {
  uint64_t i = 0;
  while (i < n && !(has_max && !(hits[i].distance < max_distance))) ++i;
  return i;
}

// Exact path for any input: collect rows whose approximate cosine >= cos_floor,
// score them canonically, keep distance < limit, sort by (distance,row).
// On return ctx->collect_hits holds the sorted hits and *n_pass their count.
static int collect_exact_sorted(stb_ctx *ctx, const stb_corpus *c, float cos_floor, double limit,
                                const uint64_t *ranges_dev, uint32_t n_ranges, uint64_t n_virtual,
                                uint64_t *n_pass, int tier = STB_TIER_F32) {
  int rc;
  unsigned long long count = 0;
  if ((rc = dev_reserve(&ctx->collect_rows, &ctx->collect_cap, 1, 1u << 20)) != STB_OK) return rc;
  for (int attempt = 0; attempt < 3; ++attempt) {
    if ((rc = stb_launch_scan_collect(ctx, c, tier, ctx->q_dev, cos_floor, ranges_dev, n_ranges, n_virtual)) != STB_OK) return rc;
    STB_CUDA(cudaMemcpyAsync(&count, ctx->collect_count, sizeof(count), cudaMemcpyDeviceToHost, ctx->stream));
    STB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (count <= ctx->collect_cap) break;
    if ((rc = dev_reserve(&ctx->collect_rows, &ctx->collect_cap, (size_t)count)) != STB_OK) return rc;
  }
  if (count > ctx->collect_cap) { stb_set_error("collect buffer could not be sized"); return STB_ERR_STATE; }
  uint64_t m = count, m_padded = 1024;
  while (m_padded < m) m_padded <<= 1;
  if ((rc = dev_reserve(&ctx->collect_hits, &ctx->collect_hits_cap, (size_t)m_padded)) != STB_OK) return rc;
  if ((rc = stb_launch_exact(ctx, c->rows, c->row_base, ctx->q_dev, ctx->collect_rows, m, limit,
                             ctx->collect_hits, m_padded, ctx->collect_count + 1)) != STB_OK) return rc;
  if ((rc = stb_launch_sort_hits(ctx, ctx->collect_hits, m_padded)) != STB_OK) return rc;
  unsigned long long pass = 0;
  STB_CUDA(cudaMemcpyAsync(&pass, ctx->collect_count + 1, sizeof(pass), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  *n_pass = pass;
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

  // ---- row ranges: global -> local, clipped to this shard ----------------------
  const uint64_t *ranges_dev = nullptr;
  uint32_t n_loc = 0;
  uint64_t n_virtual = corpus->n;
  if (row_ranges) {
    std::vector<uint64_t> vstart, rbegin;
    vstart.reserve(n_ranges + 1); rbegin.reserve(n_ranges);
    uint64_t acc = 0;
    if ((rc = stb_clip_ranges("search", row_ranges, n_ranges, corpus->row_base, corpus->n, [&](uint64_t b, uint64_t e) {
           vstart.push_back(acc); rbegin.push_back(b);
           acc += e - b;
         })) != STB_OK) return rc;
    if (acc == 0) return STB_OK;
    vstart.push_back(acc);
    n_loc = (uint32_t)rbegin.size();
    n_virtual = acc;
    std::vector<uint64_t> packed(vstart);
    packed.insert(packed.end(), rbegin.begin(), rbegin.end());
    if ((rc = dev_reserve(&ctx->ranges_dev, &ctx->ranges_cap, packed.size(), 4096)) != STB_OK) return rc;
    STB_CUDA(cudaMemcpyAsync(ctx->ranges_dev, packed.data(), packed.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->stream));
    STB_CUDA(cudaStreamSynchronize(ctx->stream));   // `packed` dies at scope end
    ranges_dev = ctx->ranges_dev;
  }

  memcpy(ctx->q_pin, q, STB_D * sizeof(float));
  STB_CUDA(cudaMemcpyAsync(ctx->q_dev, ctx->q_pin, STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));

  // The reduced-width candidate copies are used when they exist (stb_corpus_prepare) and built lazily
  // from the second search since the corpus last changed, on >= 32768 rows: a one-shot CLI query must
  // not pay a full extra pass to save half of one.  A copy that covers a prefix (rows were appended
  // since) is extended right away: converting the new rows costs far less than scanning everything at
  // 1 KiB/row.
  stb_corpus *cm = const_cast<stb_corpus *>(corpus);
  const K1CopyPolicy lazy = {cm->searches_since_change >= 1 && cm->n >= 32768, true};
  cm->searches_since_change++;

  uint64_t total = 0;
  const stb_hit *src_dev = nullptr;   // sorted device hits to copy out (collect path)
  if (!threshold_all && top_k <= stb_scan_topk_max_k()) {
    // ---- fast path: one kernel, k*16+16 bytes back -----------------------------
    // The kernel's last CTA stores the k hits + status straight into the pinned host buffers
    // (UVA: cudaMallocHost memory is device-accessible), which takes the two D2H copies off the
    // stream; kernel completion makes the stores visible to the host.
    auto run_fast = [&](int tier) -> int {
      int r;
      if ((r = stb_launch_scan_topk(ctx, corpus, tier, ctx->q_dev, top_k, ranges_dev, n_loc, n_virtual, ctx->hits_pin,
                                    ctx->status_pin)) != STB_OK) return r;
      STB_CUDA(cudaStreamSynchronize(ctx->stream));
      return STB_OK;
    };
    // Tier ladder: q8 (260 B/row) -> h16 (512 B/row) -> f32 (1 KiB/row).  Every tier ends in the
    // same exact f64 re-rank and proves its own result; one that cannot is retried one tier up, so
    // the answer is the oracle's whichever tier produced it.  A tier that keeps failing its proofs
    // on this corpus is dropped.
    bool proven = false;
    for (int tier = STB_TIER_Q8; tier >= STB_TIER_H16 && !proven; --tier) {
      if (cm->tier_tries[tier] >= 8 && 2 * cm->tier_proven[tier] < cm->tier_tries[tier]) continue;
      bool ready = false;
      if ((rc = k1_copy_ready(ctx, cm, tier, top_k, lazy, &ready)) != STB_OK) return rc;
      if (!ready) continue;
      if ((rc = run_fast(tier)) != STB_OK) return rc;
      proven = ctx->status_pin[1] != 0;
      cm->tier_tries[tier]++;
      if (proven) cm->tier_proven[tier]++;
    }
    if (!proven) {
      if ((rc = run_fast(STB_TIER_F32)) != STB_OK) return rc;
      cm->tier_tries[STB_TIER_F32]++;
      if (ctx->status_pin[1]) cm->tier_proven[STB_TIER_F32]++;
    }
    const uint32_t n_hits = ctx->status_pin[0];
    if (ctx->status_pin[1]) {
      const uint64_t n = capped_hits(ctx->hits_pin, n_hits, has_max, max_distance);
      if (n && cap) memcpy(out_hits, ctx->hits_pin, std::min(n, cap) * sizeof(stb_hit));
      *out_n = n;
      if (n > cap) { stb_set_error("search: %llu hits, capacity %llu", (unsigned long long)n, (unsigned long long)cap); return STB_ERR_CAPACITY; }
      return STB_OK;
    }
    // ---- candidate margin not provable: exact collect pass --------------------
    ctx->fallback_searches++;
    float floor_cos = -INFINITY;
    if (n_hits == top_k) floor_cos = (float)(1.0 - ctx->hits_pin[top_k - 1].distance - 2.0 * STB_SCORE_EPS);
    uint64_t n_pass = 0;
    if ((rc = collect_exact_sorted(ctx, corpus, floor_cos, has_max ? std::min(max_distance, STB_DEFAULT_MAX_DIST) : STB_DEFAULT_MAX_DIST,
                                   ranges_dev, n_loc, n_virtual, &n_pass)) != STB_OK) return rc;
    total = std::min<uint64_t>(n_pass, top_k);
    src_dev = ctx->collect_hits;
  } else {
    // ---- threshold mode / top_k beyond the register lists: collect -> exact -> sort --------------
    // When the int8 copy exists (or may be built: same lazy rule as the top-k tiers) the streaming
    // passes read it instead of the f32 rows: its scores are upper bounds u >= c - 2e-5 of the exact
    // cosine, so "u >= floor" collects a superset of "c >= floor" at a quarter of the bytes.
    bool use_q8 = false;
    if ((rc = k1_copy_ready(ctx, cm, STB_TIER_Q8, 0, lazy, &use_q8)) != STB_OK) return rc;
    float floor_cos = -INFINITY;
    double limit = STB_DEFAULT_MAX_DIST;
    uint64_t n_pass = 0;
    bool done = false;
    if (threshold_all) {
      limit = max_distance;
      floor_cos = (float)(1.0 - max_distance - (use_q8 ? 2.0 * STB_Q8_SCAN_EPS : STB_SCORE_EPS));
      if (!(max_distance == max_distance)) floor_cos = INFINITY;   // NaN threshold: nothing passes
      if ((rc = collect_exact_sorted(ctx, corpus, floor_cos, limit, ranges_dev, n_loc, n_virtual, &n_pass,
                                     use_q8 ? STB_TIER_Q8 : STB_TIER_F32)) != STB_OK) return rc;
      done = true;
    } else {
      if (has_max) {
        limit = std::min(max_distance, STB_DEFAULT_MAX_DIST);
        if (!(max_distance == max_distance)) limit = -1.0;
      }
      // top_k beyond the register lists: histogram pass to find the score bin of the k-th
      // best, then collect only rows at or above that bin (instead of the whole shard)
      std::vector<unsigned int> hist(4096);
      auto kth_bin = [&](int tier, int *bin) -> int {
        int r;
        if ((r = stb_launch_scan_hist(ctx, corpus, tier, ctx->q_dev, ranges_dev, n_loc, n_virtual, ctx->hist_dev)) != STB_OK) return r;
        STB_CUDA(cudaMemcpyAsync(hist.data(), ctx->hist_dev, 4096 * sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
        STB_CUDA(cudaStreamSynchronize(ctx->stream));
        uint64_t cum = 0;
        int b = 0;
        for (; b < 4096; ++b) { cum += hist[b]; if (cum >= top_k) break; }
        *bin = b;
        return STB_OK;
      };
      if (use_q8) {
        // q8: the histogram is over UPPER BOUNDS, which sit up to ~0.02-0.04 above the exact cosines, so the
        // floor is put 0.04 below the k-th best bound and the result is PROVEN afterwards: every row that
        // was not collected has c < floor + 2e-5; if the k-th exact distance found is below
        // 1 - floor - 2e-5 nothing outside can enter or tie.  Otherwise the f32 passes below answer.
        int b = 0;
        if ((rc = kth_bin(STB_TIER_Q8, &b)) != STB_OK) return rc;
        floor_cos = (b < 4095) ? (float)(1.0 - (double)(b + 1) / 2048.0 - 0.04) : -INFINITY;
        if ((rc = collect_exact_sorted(ctx, corpus, floor_cos, limit, ranges_dev, n_loc, n_virtual, &n_pass, STB_TIER_Q8)) != STB_OK) return rc;
        if (floor_cos == -INFINITY) done = true;             // everything was collected
        else if (n_pass >= top_k) {
          stb_hit kth;
          STB_CUDA(cudaMemcpyAsync(&kth, ctx->collect_hits + (top_k - 1), sizeof(kth), cudaMemcpyDeviceToHost, ctx->stream));
          STB_CUDA(cudaStreamSynchronize(ctx->stream));
          done = kth.distance < 1.0 - (double)floor_cos - 2.0 * STB_Q8_SCAN_EPS;
        }
        if (!done) ctx->fallback_searches++;
      }
      if (!done) {
        int b = 0;
        if ((rc = kth_bin(STB_TIER_F32, &b)) != STB_OK) return rc;
        floor_cos = (b < 4095) ? (float)(1.0 - (double)(b + 1) / 2048.0 - 2.0 * STB_SCORE_EPS) : -INFINITY;   // else: fewer than k rows, take all
        if ((rc = collect_exact_sorted(ctx, corpus, floor_cos, limit, ranges_dev, n_loc, n_virtual, &n_pass)) != STB_OK) return rc;
      }
    }
    total = threshold_all ? n_pass : std::min<uint64_t>(n_pass, top_k);
    src_dev = ctx->collect_hits;
  }
  *out_n = total;
  uint64_t ncopy = std::min(total, cap);
  if (ncopy) {
    STB_CUDA(cudaMemcpyAsync(out_hits, src_dev, ncopy * sizeof(stb_hit), cudaMemcpyDeviceToHost, ctx->stream));
    STB_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  if (total > cap) { stb_set_error("search: %llu hits, capacity %llu", (unsigned long long)total, (unsigned long long)cap); return STB_ERR_CAPACITY; }
  return STB_OK;
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
  return stb_launch_scan_topk(ctx, corpus, best_built_tier(ctx, corpus, top_k), q_dev, top_k, nullptr, 0, corpus->n,
                              out_hits_dev, out_status_dev, nullptr, true);
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
  memset(x, 0, sizeof(*x));
  x->ctx = ctx; x->world = world; x->rank = rank; x->max_k = max_k; x->max_nq = max_nq;
  x->batch_off = (xchg_bytes(world, max_k) + 255) & ~(size_t)255;
  x->batch_slot_bytes = max_nq ? xchg_batch_slot_bytes(world, max_nq, max_k) : 0;
  x->bytes = x->batch_off + 2 * x->batch_slot_bytes;
  // plain cudaMalloc memory: required for cudaIpcGetMemHandle
  cudaError_t e = cudaMalloc((void **)&x->local, x->bytes);
  if (e == cudaSuccess) e = cudaMemset(x->local, 0, x->bytes);
  if (e == cudaSuccess) e = cudaMalloc((void **)&x->batch_ticket, sizeof(unsigned int));
  if (e == cudaSuccess) e = cudaMemset(x->batch_ticket, 0, sizeof(unsigned int));
  // cudaMemset on device memory may return before it ran (legacy default stream, which a non-blocking
  // stream does not order against): the zeroed flags must be in place before any peer can store to them
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { cudaGetLastError(); cudaFree(x->local); stb_set_error("xchg_create: %s", cudaGetErrorString(e)); delete x; return STB_ERR_NOMEM; }
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
  cudaFree(x->batch_ticket);
  cudaFree(x->local);
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
  if (!x->connected) { stb_set_error("search_topk_xchg: exchange not connected"); return STB_ERR_STATE; }
  if (x->dead) { stb_set_error("search_topk_xchg: this exchange saw a peer time-out; destroy it on every rank"); return STB_ERR_STATE; }
  if (top_k == 0 || top_k > x->max_k) { stb_set_error("search_topk_xchg: top_k must be 1..%u", x->max_k); return STB_ERR_ARG; }
  StbXchgArgs a;
  memset(&a, 0, sizeof(a));
  for (uint32_t r = 0; r < x->world; ++r) a.base[r] = x->peers[r];
  a.world = x->world; a.rank = x->rank; a.max_k = x->max_k;
  a.seq = ++x->seq;
  a.slot = (uint32_t)(a.seq % STB_XCHG_SLOTS);
  return stb_launch_scan_topk(ctx, corpus, best_built_tier(ctx, corpus, top_k), q_dev, top_k, nullptr, 0, corpus->n,
                              out_hits_dev, out_status_dev, &a);
}

// ----------------------------------------------------------------- K2 batched search ---
static int corpus_ensure_shadow(stb_ctx *ctx, stb_corpus *c) {
  if (c->shadow && c->shadow_rows == c->n) {
    if (c->shadow_bad) { stb_set_error("search_batch: corpus holds rows whose norm is not a normal fp32 number; use stb_search"); return STB_ERR_STATE; }
    return STB_OK;
  }
  const uint64_t tiles = (c->n + 255) / 256;
  uint64_t first = (c->shadow && c->shadow_rows < c->n && !c->shadow_bad) ? (c->shadow_rows / 256) * 256 : 0;   // valid prefix, whole tiles
  if (tiles > c->shadow_cap_tiles || !c->shadow) {
    uint8_t *np = nullptr;
    const uint64_t cap_tiles = std::max<uint64_t>(tiles, (c->capacity + 255) / 256);
    cudaError_t e = cudaMalloc((void **)&np, cap_tiles * 131072ull);
    if (e != cudaSuccess) { cudaGetLastError(); stb_set_error("search_batch: cannot allocate the %llu MiB 16-bit shadow", (unsigned long long)(cap_tiles >> 3)); return STB_ERR_NOMEM; }
    if (c->shadow && first) STB_CUDA(cudaMemcpyAsync(np, c->shadow, (first / 256) * 131072ull, cudaMemcpyDeviceToDevice, ctx->stream));
    else first = 0;
    STB_CUDA(cudaStreamSynchronize(ctx->stream));
    cudaFree(c->shadow);
    c->shadow = np;
    c->shadow_cap_tiles = cap_tiles;
  }
  int rc;
  STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
  if ((rc = stb_launch_shadow_build(ctx, c->rows, c->n, 256, c->shadow, ctx->err_flag, first)) != STB_OK) return rc;
  int flag = 0;
  STB_CUDA(cudaMemcpyAsync(&flag, ctx->err_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  c->shadow_rows = c->n;
  c->shadow_bad = (first ? c->shadow_bad : 0) | flag;
  if (c->shadow_bad) { stb_set_error("search_batch: corpus holds rows whose norm is not a normal fp32 number; use stb_search"); return STB_ERR_STATE; }
  return STB_OK;
}

static int corpus_ensure_q8(stb_ctx *ctx, stb_corpus *c) {
  if (c->q8 && c->q8_rows == c->n) {
    if (c->q8_bad) { stb_set_error("q8 tier: corpus holds rows whose norm is not a normal fp32 number"); return STB_ERR_STATE; }
    return STB_OK;
  }
  uint64_t first = (c->q8 && c->q8_rows < c->n && !c->q8_bad) ? c->q8_rows : 0;      // valid prefix: convert only the new rows
  if (c->n > c->q8_cap_rows || !c->q8) {
    // int8 codes + scales (260 B/row) and the top-k prefilter's nibble plane + {s, rho} (136 B/row)
    uint8_t *np = nullptr, *pp = nullptr;
    float *ns = nullptr;
    float2 *sp = nullptr;
    const uint64_t cap = std::max<uint64_t>(c->n, c->capacity);
    cudaError_t e = cudaMalloc((void **)&np, cap * 256ull);
    if (e == cudaSuccess) e = cudaMalloc((void **)&ns, cap * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc((void **)&pp, stb_q4_plane_bytes(cap));
    if (e == cudaSuccess) e = cudaMalloc((void **)&sp, cap * sizeof(float2));
    if (e != cudaSuccess) {
      cudaGetLastError(); cudaFree(np); cudaFree(ns); cudaFree(pp);
      stb_set_error("q8 tier: cannot allocate %llu MiB", (unsigned long long)(cap * 396 >> 20));
      return STB_ERR_NOMEM;
    }
    if (c->q8 && first) {
      STB_CUDA(cudaMemcpyAsync(np, c->q8, first * 256ull, cudaMemcpyDeviceToDevice, ctx->stream));
      STB_CUDA(cudaMemcpyAsync(ns, c->q8_scale, first * sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
      STB_CUDA(cudaMemcpyAsync(pp, c->q4, stb_q4_plane_bytes(first), cudaMemcpyDeviceToDevice, ctx->stream));   // whole tiles
      STB_CUDA(cudaMemcpyAsync(sp, c->q4_sr, first * sizeof(float2), cudaMemcpyDeviceToDevice, ctx->stream));
      STB_CUDA(cudaStreamSynchronize(ctx->stream));
    } else first = 0;
    cudaFree(c->q8); cudaFree(c->q8_scale); cudaFree(c->q4); cudaFree(c->q4_sr);
    c->q8 = np; c->q8_scale = ns; c->q4 = pp; c->q4_sr = sp; c->q8_cap_rows = cap;
  }
  int rc;
  STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
  if ((rc = stb_launch_q8_build(ctx, c->rows, first, c->n, c->q8, c->q8_scale, c->q4, c->q4_sr, ctx->err_flag)) != STB_OK) return rc;
  int flag = 0;
  STB_CUDA(cudaMemcpyAsync(&flag, ctx->err_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  c->q8_rows = c->n;
  c->q8_bad = (first ? c->q8_bad : 0) | flag;
  if (c->q8_bad) { stb_set_error("q8 tier: corpus holds rows whose norm is not a normal fp32 number"); return STB_ERR_STATE; }
  return STB_OK;
}

int stb_corpus_prepare(stb_corpus *corpus, int what) {
  if (!corpus) { stb_set_error("null corpus"); return STB_ERR_ARG; }
  if (what & ~(STB_PREPARE_Q8 | STB_PREPARE_H16)) { stb_set_error("corpus_prepare: unknown flag"); return STB_ERR_ARG; }
  int rc = ctx_use(corpus->ctx);
  if (rc) return rc;
  if (corpus->n == 0) return STB_OK;
  // rows that cannot be normalised in fp32 make a copy unusable (STB_ERR_STATE): not an error of
  // this call -- searches simply stay on the f32 rows
  if (what & STB_PREPARE_Q8) { rc = corpus_ensure_q8(corpus->ctx, corpus); if (rc != STB_OK && rc != STB_ERR_STATE) return rc; }
  if (what & STB_PREPARE_H16) { rc = corpus_ensure_shadow(corpus->ctx, corpus); if (rc != STB_OK && rc != STB_ERR_STATE) return rc; }
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
    built_rows[STB_TIER_H16] = (corpus->shadow && !corpus->shadow_bad) ? corpus->shadow_rows : 0;   // < n after an append: a valid prefix
    built_rows[STB_TIER_Q8] = (corpus->q8 && !corpus->q8_bad) ? corpus->q8_rows : 0;
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
  if (c->q8_bad) { c->q8_rows = 0; c->q8_bad = 0; }
  if (c->shadow_bad) { c->shadow_rows = 0; c->shadow_bad = 0; }
}

static StbCorpusWriteArgs corpus_write_args(stb_corpus *c, uint64_t q8_rows, uint64_t shadow_rows) {
  StbCorpusWriteArgs a;
  memset(&a, 0, sizeof(a));
  a.rows = reinterpret_cast<float4 *>(c->rows);
  a.stage = reinterpret_cast<const float4 *>(c->ctx->mut_stage);
  a.q8 = c->q8; a.q8_scale = c->q8_scale; a.q4 = c->q4; a.q4_sr = c->q4_sr;
  a.q8_rows = c->q8 ? q8_rows : 0;
  a.shadow = c->shadow;
  a.shadow_rows = c->shadow ? shadow_rows : 0;
  a.flags = c->ctx->mut_flags;
  return a;
}

// reads the bad-row flags the call's kernels raised (synchronises) and books the change
static int corpus_mutation_finish(stb_corpus *c) {
  stb_ctx *ctx = c->ctx;
  int flags[2] = {0, 0};
  STB_CUDA(cudaMemcpyAsync(flags, ctx->mut_flags, sizeof(flags), cudaMemcpyDeviceToHost, ctx->stream));
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (flags[0]) c->q8_bad = 1;
  if (flags[1]) c->shadow_bad = 1;
  corpus_changed(c, CORPUS_ROWS_REWRITTEN);
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
  if ((rc = dev_reserve(&ctx->mut_stage, &ctx->mut_stage_cap, chunk * STB_D)) != STB_OK) return rc;
  if ((rc = dev_reserve(&ctx->mut_idx, &ctx->mut_idx_cap, chunk)) != STB_OK) return rc;
  if ((rc = dev_reserve(&ctx->mut_flags, &ctx->mut_flags_cap, 2)) != STB_OK) return rc;
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
  StbCorpusWriteArgs a = corpus_write_args(c, c->q8_rows, c->shadow_rows);
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
  // kept segments behind the first removed row, as {destination, source} local rows; removed rows inside the
  // prefix each copy covers (a copy marked bad is dropped below: it covers none)
  std::vector<uint64_t> seg;
  const uint64_t q8_had = c->q8_bad ? 0 : c->q8_rows, shadow_had = c->shadow_bad ? 0 : c->shadow_rows;
  uint64_t removed = 0, removed_q8 = 0, removed_shadow = 0;
  const uint64_t first = ranges[0] - lo;
  uint64_t dst = first;
  for (uint32_t i = 0; i < n_ranges; ++i) {
    const uint64_t b = ranges[2 * i] - lo, e = ranges[2 * i + 1] - lo;
    const uint64_t next = (i + 1 < n_ranges) ? ranges[2 * i + 2] - lo : c->n;
    removed += e - b;
    if (q8_had > b) removed_q8 += std::min(e, q8_had) - b;
    if (shadow_had > b) removed_shadow += std::min(e, shadow_had) - b;
    if (next > e) { seg.push_back(dst); seg.push_back(e); dst += next - e; }
  }
  const uint64_t moved = dst - first;
  const uint64_t q8_rows = q8_had - removed_q8, shadow_rows = shadow_had - removed_shadow;
  if ((rc = dev_reserve(&ctx->mut_flags, &ctx->mut_flags_cap, 2)) != STB_OK) return rc;
  if (moved) {
    const uint64_t chunk = std::min<uint64_t>(moved, STB_MUT_CHUNK_ROWS);
    if ((rc = dev_reserve(&ctx->mut_stage, &ctx->mut_stage_cap, chunk * STB_D)) != STB_OK) return rc;
    if ((rc = dev_reserve(&ctx->mut_idx, &ctx->mut_idx_cap, seg.size())) != STB_OK) return rc;
  }
  if (hook && ((rc = hook->begin()) != STB_OK || (rc = hook->ready()) != STB_OK)) return rc;
  corpus_drop_bad_copies(c);
  STB_CUDA(cudaMemsetAsync(ctx->mut_flags, 0, 2 * sizeof(int), ctx->stream));
  if (moved) {
    // Chunks in output order.  The sources of a chunk lie at or beyond its own output rows, so the gather
    // reads rows no earlier chunk has overwritten, and it completes before the commit writes.
    STB_CUDA(cudaMemcpyAsync(ctx->mut_idx, seg.data(), seg.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->stream));
    const uint32_t n_seg = (uint32_t)(seg.size() / 2);
    StbCorpusWriteArgs a = corpus_write_args(c, q8_rows, shadow_rows);
    for (uint64_t d0 = first; d0 < first + moved; d0 += STB_MUT_CHUNK_ROWS) {
      a.first = d0;
      a.m = std::min<uint64_t>(STB_MUT_CHUNK_ROWS, first + moved - d0);
      if ((rc = stb_launch_corpus_gather(ctx, c->rows, ctx->mut_idx, n_seg, a.first, a.m, ctx->mut_stage)) != STB_OK) return rc;
      if ((rc = stb_launch_corpus_write(ctx, a)) != STB_OK) return rc;
    }
    STB_CUDA(cudaStreamSynchronize(ctx->stream));   // `seg` dies at scope end
  }
  // the shadow's last covered tile ends in zero padding, as a build of `shadow_rows` rows leaves it
  if (c->shadow && shadow_rows % 256 &&
      (rc = stb_launch_shadow_build(ctx, c->rows, shadow_rows, 256, c->shadow, ctx->mut_flags + 1, shadow_rows)) != STB_OK) return rc;
  c->n -= removed;
  c->q8_rows = q8_rows;
  c->shadow_rows = shadow_rows;
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
  uint64_t rows = c->q8 ? c->q8_rows : 0, units = rows;
  switch (which) {
    case STB_COPY_Q8_CODES: src = c->q8; unit = 256; break;
    case STB_COPY_Q8_SCALES: src = c->q8_scale; unit = sizeof(float); break;
    case STB_COPY_Q8_PLANE: src = c->q4; unit = 128; break;
    case STB_COPY_Q8_SR: src = c->q4_sr; unit = sizeof(float2); break;
    case STB_COPY_H16_TILES:
      src = c->shadow; unit = 131072; rows = c->shadow ? c->shadow_rows : 0; units = (rows + 255) / 256; break;
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
  return corpus_ensure_shadow(corpus->ctx, corpus);
}

}  // extern "C"

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

// Pipeline v2 (batch_scan.cu): sampled threshold -> candidate-emitting wgmma epilogue -> exact finish.
// Unfiltered (tile_ids == NULL) it samples and emits over the shadow tiles 0 .. n_cover-1 (the sample over
// complete tiles only); filtered over the n_cover listed tiles tile_ids[] with the eligible-row bitmap.
static int batch_v2_run(stb_ctx *ctx, const stb_corpus *corpus, const float *q_dev, uint32_t nq, uint32_t top_k,
                        uint32_t n_cover, BatchV2Plan p, const uint32_t *tile_ids, const uint32_t *bitmap,
                        stb_hit *out_hits_dev, uint32_t *out_status_dev) {
  int rc;
  const uint32_t m_tiles = (nq + 127) / 128, q_pad = m_tiles * 128;
  const uint32_t n_tiles = (uint32_t)((corpus->n + 255) / 256);
  const uint32_t n_emit = tile_ids ? n_cover : n_tiles;
  constexpr uint32_t kSegCap = 64;                      // per (query, CTA): ~5 expected at 10M rows / 132 CTAs
  const uint32_t n_seg = stb_batch_emit_grid(ctx, n_emit);
  const uint32_t last[6] = {tile_ids ? 3u : 2u, nq, p.n_sample, p.stride, n_seg, kSegCap};
  memcpy(ctx->b_last, last, sizeof(last));
  if ((rc = dev_reserve(&ctx->b_qbad, &ctx->b_qbad_cap, (size_t)q_pad)) != STB_OK) return rc;
  if ((rc = dev_reserve(&ctx->bq_tiles, &ctx->bq_tiles_cap, (size_t)q_pad * 512)) != STB_OK) return rc;
  if ((rc = dev_reserve(&ctx->b_tilemax, &ctx->b_tilemax_cap, (size_t)p.n_sample * q_pad)) != STB_OK) return rc;
  if ((rc = dev_reserve(&ctx->b_thr, &ctx->b_thr_cap, (size_t)q_pad)) != STB_OK) return rc;
  if ((rc = dev_reserve(&ctx->b_cnt, &ctx->b_cnt_cap, (size_t)q_pad * n_seg)) != STB_OK) return rc;
  if ((rc = dev_reserve(&ctx->b_keys, &ctx->b_keys_cap, (size_t)q_pad * n_seg * kSegCap)) != STB_OK) return rc;
  STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
  STB_CUDA(cudaMemsetAsync(ctx->b_cnt, 0, (size_t)q_pad * n_seg * sizeof(uint32_t), ctx->stream));
  if ((rc = stb_launch_shadow_build(ctx, q_dev, nq, 128, ctx->bq_tiles, ctx->err_flag, 0, ctx->b_qbad)) != STB_OK) return rc;
  if (tile_ids)
    rc = stb_launch_batch_gemm_sample_filtered(ctx, ctx->bq_tiles, m_tiles, corpus->shadow, tile_ids, bitmap, p.n_sample,
                                               p.stride, ctx->b_tilemax);
  else
    rc = stb_launch_batch_gemm_strided(ctx, ctx->bq_tiles, m_tiles, corpus->shadow, p.n_sample, p.stride, nullptr,
                                       ctx->b_tilemax, nullptr);
  if (rc != STB_OK) return rc;
  if ((rc = stb_launch_batch_thresh(ctx, ctx->b_tilemax, p.n_sample, nq, q_pad, top_k, ctx->b_thr)) != STB_OK) return rc;
  if (tile_ids)
    rc = stb_launch_batch_gemm_emit_filtered(ctx, ctx->bq_tiles, m_tiles, corpus->shadow, tile_ids, bitmap, n_cover,
                                             corpus->n, ctx->b_thr, ctx->b_cnt, ctx->b_keys, kSegCap);
  else
    rc = stb_launch_batch_gemm_emit(ctx, ctx->bq_tiles, m_tiles, corpus->shadow, n_tiles, corpus->n, ctx->b_thr,
                                    ctx->b_cnt, ctx->b_keys, kSegCap);
  if (rc != STB_OK) return rc;
  return stb_launch_batch_finish2(ctx, ctx->b_keys, ctx->b_cnt, n_seg, kSegCap, nq, top_k, corpus->rows, corpus->n,
                                  corpus->row_base, q_dev, ctx->b_qbad, out_hits_dev, out_status_dev);
}

extern "C" {

int stb_search_batch_dev(stb_ctx *ctx, const stb_corpus *corpus_c, const float *q_dev, uint32_t nq,
                         uint32_t top_k, stb_hit *out_hits_dev, uint32_t *out_status_dev) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  stb_corpus *corpus = const_cast<stb_corpus *>(corpus_c);
  if (!corpus || !q_dev || !out_hits_dev || !out_status_dev) { stb_set_error("search_batch_dev: null argument"); return STB_ERR_ARG; }
  if (corpus->ctx != ctx) { stb_set_error("search_batch_dev: corpus belongs to another context"); return STB_ERR_ARG; }
  if (nq == 0) return STB_OK;
  if (top_k == 0 || top_k > 1024) { stb_set_error("search_batch_dev: top_k must be 1..1024"); return STB_ERR_ARG; }
  if (corpus->n == 0) { stb_set_error("search_batch_dev: empty corpus"); return STB_ERR_STATE; }
  if ((rc = corpus_ensure_shadow(ctx, corpus)) != STB_OK) return rc;
  const uint32_t m_tiles = (nq + 127) / 128, q_pad = m_tiles * 128;
  const uint32_t n_tiles = (uint32_t)((corpus->n + 255) / 256), n_sub = n_tiles * 8;
  // Pipeline v2 (default, batch_v2_run).  Proves every query for any top_k <= 64 unless a capacity
  // overflows.  The round-1 maxima/select/finish pipeline (v1) runs for top_k > 64 and wherever v2 does not fit.
  const uint32_t n_full = (uint32_t)(corpus->n / 256);
  const BatchV2Plan plan = batch_v2_plan(ctx, n_full, top_k);
  if (plan.fits) return batch_v2_run(ctx, corpus, q_dev, nq, top_k, n_full, plan, nullptr, nullptr, out_hits_dev, out_status_dev);
  // one flag per query, written by the query shadow build: a query that cannot be normalised in fp32
  // has a zero (or NaN) shadow whose scores bound nothing, and both finish kernels report it unproven
  if ((rc = dev_reserve(&ctx->b_qbad, &ctx->b_qbad_cap, (size_t)q_pad)) != STB_OK) return rc;
  const uint32_t last[6] = {1u, nq, 0u, 0u, 0u, 0u};
  memcpy(ctx->b_last, last, sizeof(last));
  // selection slices: enough CTAs (m_tiles x n_slices) to hide the latency of the streaming
  // read; the finish kernel merges n_slices x 32 <= 4096 candidate tiles per query
  uint32_t n_slices = std::max<uint32_t>(1, std::min<uint32_t>(128, 1536 / m_tiles));
  n_slices = std::min<uint32_t>(n_slices, std::max<uint32_t>(1, n_tiles / 48));
  if ((rc = dev_reserve(&ctx->bq_tiles, &ctx->bq_tiles_cap, (size_t)q_pad * 512)) != STB_OK) return rc;
  if ((rc = dev_reserve(&ctx->b_submax, &ctx->b_submax_cap, (size_t)n_sub * q_pad)) != STB_OK) return rc;
  if ((rc = dev_reserve(&ctx->b_tilemax, &ctx->b_tilemax_cap, (size_t)n_tiles * q_pad)) != STB_OK) return rc;
  if ((rc = dev_reserve(&ctx->b_cand, &ctx->b_cand_cap, (size_t)q_pad * n_slices * 32)) != STB_OK) return rc;
  // query tiles: padding queries beyond nq are written as zeros by the shadow builder
  STB_CUDA(cudaMemsetAsync(ctx->err_flag, 0, sizeof(int), ctx->stream));
  if ((rc = stb_launch_shadow_build(ctx, q_dev, nq, 128, ctx->bq_tiles, ctx->err_flag, 0, ctx->b_qbad)) != STB_OK) return rc;
  if ((rc = stb_launch_batch_gemm(ctx, ctx->bq_tiles, m_tiles, corpus->shadow, n_tiles, ctx->b_submax, ctx->b_tilemax, nullptr)) != STB_OK) return rc;
  // two-level selection: the best tiles by tile maximum (1/8 of the data), refined to
  // sub-tiles inside the finish kernel
  if ((rc = stb_launch_batch_select(ctx, ctx->b_tilemax, n_tiles, q_pad, n_slices, ctx->b_cand)) != STB_OK) return rc;
  return stb_launch_batch_finish(ctx, ctx->b_cand, n_slices, n_sub, nq, top_k, corpus->rows, corpus->n,
                                 corpus->row_base, q_dev, ctx->b_qbad, out_hits_dev, out_status_dev, ctx->b_submax, q_pad);
}

int stb_search_batch(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t nq, uint32_t top_k,
                     stb_hit *out_hits, uint32_t *out_n) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!corpus || !q || !out_hits || !out_n) { stb_set_error("search_batch: null argument"); return STB_ERR_ARG; }
  if (nq == 0) return STB_OK;
  for (uint32_t i = 0; i < nq; ++i) out_n[i] = 0;
  if (top_k == 0 || corpus->n == 0) return STB_OK;
  bool tensor_ok = top_k <= 1024;
  std::vector<uint32_t> status((size_t)nq * 2, 0);
  if (tensor_ok) {
    if ((rc = dev_reserve(&ctx->bq_dev, &ctx->bq_dev_cap, (size_t)nq * STB_D)) != STB_OK) return rc;
    if ((rc = dev_reserve(&ctx->bh_dev, &ctx->bh_dev_cap, (size_t)nq * top_k)) != STB_OK) return rc;
    if ((rc = dev_reserve(&ctx->bs_dev, &ctx->bs_dev_cap, (size_t)nq * 2)) != STB_OK) return rc;
    STB_CUDA(cudaMemcpyAsync(ctx->bq_dev, q, (size_t)nq * STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    rc = stb_search_batch_dev(ctx, corpus, ctx->bq_dev, nq, top_k, ctx->bh_dev, ctx->bs_dev);
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
  for (uint32_t i = 0; i < nq; ++i) {
    if (tensor_ok && status[2 * i + 1]) { out_n[i] = status[2 * i]; continue; }
    ctx->fallback_searches++;
    uint64_t n = 0;
    rc = stb_search(ctx, corpus, q + (size_t)i * STB_D, top_k, 0, 0.0, STB_MODE_SEARCH_DOCUMENTS, nullptr, 0,
                    out_hits + (size_t)i * top_k, top_k, &n);
    if (rc != STB_OK) return rc;
    out_n[i] = (uint32_t)n;
    for (uint64_t j = n; j < top_k; ++j) { out_hits[(size_t)i * top_k + j].distance = INFINITY; out_hits[(size_t)i * top_k + j].row = 0xffffffffffffffffull; }
  }
  return STB_OK;
}

// The store query (stb_search in STB_MODE_STORE_QUERY) for a batch.  The eligible rows' bitmap and the listed
// tiles both come from one list of clipped ranges; filtered v2 runs when its plan fits over the listed tiles,
// and K1 answers every query it leaves unproven (or all of them, route 4).  The cap is applied on the host:
// store-query hits are a prefix of the uncapped top-k.
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
  auto pad = [&](uint32_t i, uint64_t n) {               // the unused tail, as the kernels pad it
    for (uint64_t j = n; j < top_k; ++j) { out_hits[(size_t)i * top_k + j].distance = INFINITY; out_hits[(size_t)i * top_k + j].row = 0xffffffffffffffffull; }
  };
  // stb_search's early outs come before it reads the ranges (store.rs:489-491: top_k 0, the empty subset)
  std::vector<uint32_t> loc;                             // clipped local [begin, end) pairs
  if (top_k && !(row_ranges && n_ranges == 0) && corpus->n) {
    if (row_ranges) {
      loc.reserve(2 * (size_t)n_ranges);
      if ((rc = stb_clip_ranges("search_batch_filtered", row_ranges, n_ranges, corpus->row_base, corpus->n,
                                [&](uint64_t b, uint64_t e) { loc.push_back((uint32_t)b); loc.push_back((uint32_t)e); })) != STB_OK)
        return rc;                                       // refused before anything is written
    } else {
      loc = {0u, (uint32_t)corpus->n};
    }
  }
  const uint32_t none[6] = {4u, nq, 0u, 0u, 0u, 0u};
  memcpy(ctx->b_last, none, sizeof(none));
  if (loc.empty()) {
    for (uint32_t i = 0; i < nq; ++i) { out_n[i] = 0; pad(i, 0); }
    return STB_OK;
  }
  // listed tiles: the shadow tiles a clipped range touches (ascending, disjoint ranges -> ascending tiles)
  std::vector<uint32_t> tiles;
  for (size_t r = 0; r < loc.size(); r += 2)
    for (uint32_t t = loc[r] / 256; t <= (loc[r + 1] - 1) / 256; ++t)
      if (tiles.empty() || tiles.back() < t) tiles.push_back(t);
  const uint32_t n_listed = (uint32_t)tiles.size();
  const BatchV2Plan plan = batch_v2_plan(ctx, n_listed, top_k);
  bool tensor_ok = plan.fits;
  if (tensor_ok) {
    rc = corpus_ensure_shadow(ctx, corpus);
    if (rc == STB_ERR_STATE) tensor_ok = false;          // un-normalisable rows: K1 handles them
    else if (rc != STB_OK) return rc;
  }
  std::vector<uint32_t> status((size_t)nq * 2, 0);
  if (tensor_ok) {
    const uint64_t n_words = (corpus->n + 255) / 256 * 8;
    if ((rc = dev_reserve(&ctx->bq_dev, &ctx->bq_dev_cap, (size_t)nq * STB_D)) != STB_OK) return rc;
    if ((rc = dev_reserve(&ctx->bh_dev, &ctx->bh_dev_cap, (size_t)nq * top_k)) != STB_OK) return rc;
    if ((rc = dev_reserve(&ctx->bs_dev, &ctx->bs_dev_cap, (size_t)nq * 2)) != STB_OK) return rc;
    if ((rc = dev_reserve(&ctx->b_franges, &ctx->b_franges_cap, loc.size(), 2048)) != STB_OK) return rc;
    if ((rc = dev_reserve(&ctx->b_ftiles, &ctx->b_ftiles_cap, tiles.size(), 1024)) != STB_OK) return rc;
    if ((rc = dev_reserve(&ctx->b_fbits, &ctx->b_fbits_cap, (size_t)n_words)) != STB_OK) return rc;
    STB_CUDA(cudaMemcpyAsync(ctx->bq_dev, q, (size_t)nq * STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    STB_CUDA(cudaMemcpyAsync(ctx->b_franges, loc.data(), loc.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
    STB_CUDA(cudaMemcpyAsync(ctx->b_ftiles, tiles.data(), tiles.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = stb_launch_row_bitmap(ctx, ctx->b_franges, (uint32_t)(loc.size() / 2), n_words, ctx->b_fbits)) != STB_OK) return rc;
    if ((rc = batch_v2_run(ctx, corpus, ctx->bq_dev, nq, top_k, n_listed, plan, ctx->b_ftiles, ctx->b_fbits, ctx->bh_dev,
                           ctx->bs_dev)) != STB_OK) return rc;
    STB_CUDA(cudaMemcpyAsync(out_hits, ctx->bh_dev, (size_t)nq * top_k * sizeof(stb_hit), cudaMemcpyDeviceToHost, ctx->stream));
    STB_CUDA(cudaMemcpyAsync(status.data(), ctx->bs_dev, (size_t)nq * 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    STB_CUDA(cudaStreamSynchronize(ctx->stream));        // `loc` and `tiles` are read by the copies above
  }
  for (uint32_t i = 0; i < nq; ++i) {
    stb_hit *oh = out_hits + (size_t)i * top_k;
    uint64_t n = 0;
    if (tensor_ok && status[2 * i + 1]) {
      n = capped_hits(oh, status[2 * i], has_max, max_distance);
    } else {
      ctx->fallback_searches++;
      rc = stb_search(ctx, corpus, q + (size_t)i * STB_D, top_k, has_max, max_distance, STB_MODE_STORE_QUERY, row_ranges,
                      n_ranges, oh, top_k, &n);
      if (rc != STB_OK) return rc;
    }
    out_n[i] = (uint32_t)n;
    pad(i, n);
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
  if (!x->connected) { stb_set_error("search_batch_xchg_dev: exchange not connected"); return STB_ERR_STATE; }
  if (x->dead) { stb_set_error("search_batch_xchg_dev: this exchange saw a peer time-out; destroy it on every rank"); return STB_ERR_STATE; }
  if (nq == 0) return STB_OK;
  if (x->max_nq == 0 || nq > x->max_nq || top_k == 0 || top_k > x->max_k) { stb_set_error("search_batch_xchg_dev: needs stb_xchg_create_batch with max_nq >= %u, max_k >= %u", nq, top_k); return STB_ERR_ARG; }
  if ((rc = dev_reserve(&ctx->bh_dev, &ctx->bh_dev_cap, (size_t)nq * top_k)) != STB_OK) return rc;
  if ((rc = dev_reserve(&ctx->bs_dev, &ctx->bs_dev_cap, (size_t)nq * 2)) != STB_OK) return rc;
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
  const uint32_t nq = ctx->b_last[1], n_seg = ctx->b_last[4];
  if ((ctx->b_last[0] == 2u || ctx->b_last[0] == 3u) && nq) {
    if (thr) STB_CUDA(cudaMemcpy(thr, ctx->b_thr, (size_t)nq * sizeof(float), cudaMemcpyDeviceToHost));
    if (cand_cnt) STB_CUDA(cudaMemcpy(cand_cnt, ctx->b_cnt, (size_t)nq * n_seg * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  }
  return STB_OK;
}

int stb_debug_batch_params(int *shadow_is_f16, double *eps) {
  stb_batch_build_params(shadow_is_f16, eps);
  return STB_OK;
}

// ------------------------------------------------------------------- K2 debug hook ---
// Runs shadow build + wgmma GEMM on host inputs and returns the FULL approximate score
// matrix (tests only: validates descriptors / accumulator layout / epilogue against a reference matmul).
int stb_debug_batch_gemm(stb_ctx *ctx, const float *q, uint32_t nq, const float *rows, uint64_t n,
                         float *out_full, float *out_submax) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!q || !rows || !out_full || nq == 0 || n == 0) { stb_set_error("debug_batch_gemm: bad argument"); return STB_ERR_ARG; }
  const uint32_t m_tiles = (nq + 127) / 128;
  const uint32_t n_tiles = (uint32_t)((n + 255) / 256);
  const size_t q_pad = (size_t)m_tiles * 128, n_pad = (size_t)n_tiles * 256;
  float *dq = nullptr, *dr = nullptr, *dfull = nullptr, *dsub = nullptr, *dtile = nullptr;
  uint8_t *da = nullptr, *db = nullptr;
  int *dbad = nullptr;
  cudaError_t e = cudaMalloc(&dq, (size_t)nq * 1024);
  if (e == cudaSuccess) e = cudaMalloc(&dr, n * 1024);
  if (e == cudaSuccess) e = cudaMalloc(&da, q_pad * 512);
  if (e == cudaSuccess) e = cudaMalloc(&db, n_pad * 512);
  if (e == cudaSuccess) e = cudaMalloc(&dfull, q_pad * n_pad * 4);
  if (e == cudaSuccess) e = cudaMalloc(&dsub, (size_t)n_tiles * 8 * q_pad * 4);
  if (e == cudaSuccess) e = cudaMalloc(&dtile, (size_t)n_tiles * q_pad * 4);
  if (e == cudaSuccess) e = cudaMalloc(&dbad, 4);
  if (e == cudaSuccess) e = cudaMemsetAsync(dbad, 0, 4, ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dq, q, (size_t)nq * 1024, cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dr, rows, n * 1024, cudaMemcpyHostToDevice, ctx->stream);
  rc = STB_OK;
  if (e == cudaSuccess) rc = stb_launch_shadow_build(ctx, dq, nq, 128, da, dbad);
  if (e == cudaSuccess && rc == STB_OK) rc = stb_launch_shadow_build(ctx, dr, n, 256, db, dbad);
  if (e == cudaSuccess && rc == STB_OK) rc = stb_launch_batch_gemm(ctx, da, m_tiles, db, n_tiles, dsub, dtile, dfull);
  if (e == cudaSuccess && rc == STB_OK) e = cudaMemcpyAsync(out_full, dfull, q_pad * n_pad * 4, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess && rc == STB_OK && out_submax) e = cudaMemcpyAsync(out_submax, dsub, (size_t)n_tiles * 8 * q_pad * 4, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess && rc == STB_OK) e = cudaStreamSynchronize(ctx->stream);
  cudaFree(dq); cudaFree(dr); cudaFree(da); cudaFree(db); cudaFree(dfull); cudaFree(dsub); cudaFree(dtile); cudaFree(dbad);
  if (e != cudaSuccess) { stb_set_error("debug_batch_gemm: %s", cudaGetErrorString(e)); cudaGetLastError(); return STB_ERR_CUDA; }
  return rc;
}

int stb_search_xchg(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t top_k, stb_xchg *x,
                    stb_hit *out_hits, uint32_t *out_n, int *out_complete) {
  int rc = ctx_use(ctx);
  if (rc) return rc;
  if (!q || !out_hits || !out_n || !out_complete) { stb_set_error("search_xchg: null argument"); return STB_ERR_ARG; }
  memcpy(ctx->q_pin, q, STB_D * sizeof(float));
  STB_CUDA(cudaMemcpyAsync(ctx->q_dev, ctx->q_pin, STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  // the merge CTA stores the hits + status straight into pinned host memory
  if ((rc = stb_search_topk_xchg(ctx, corpus, ctx->q_dev, top_k, x, ctx->hits_pin, ctx->status_pin)) != STB_OK) return rc;
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  const uint32_t n = std::min<uint32_t>(ctx->status_pin[0], top_k);
  memcpy(out_hits, ctx->hits_pin, n * sizeof(stb_hit));
  *out_n = n;
  *out_complete = ctx->status_pin[1] ? 1 : 0;
  if (ctx->status_pin[2] == 0xfffffffeu) { x->dead = true; stb_set_error("search_xchg: a peer rank never arrived (timeout)"); return STB_ERR_STATE; }
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
  if (nq == 0) return STB_OK;
  for (uint32_t i = 0; i < nq; ++i) { out_n[i] = 0; if (out_complete) out_complete[i] = 1; }
  if (top_k == 0 || corpus->n == 0) {
    if (x && corpus->n == 0) { stb_set_error("search_many: empty shard in a sharded search"); return STB_ERR_STATE; }
    return STB_OK;
  }
  if (top_k > (x ? x->max_k : stb_scan_topk_max_k())) {
    if (x) { stb_set_error("search_many: top_k must be 1..%u", x->max_k); return STB_ERR_ARG; }
    for (uint32_t i = 0; i < nq; ++i) {                    // beyond the register lists: the general path, query by query
      uint64_t n = 0;
      rc = stb_search(ctx, corpus, q + (size_t)i * STB_D, top_k, 0, 0.0, STB_MODE_SEARCH_DOCUMENTS, nullptr, 0,
                      out_hits + (size_t)i * top_k, top_k, &n);
      if (rc != STB_OK) return rc;
      out_n[i] = (uint32_t)n;
    }
    return STB_OK;
  }
  // many queries amortise the int8 copy: build or extend it now (same size rule as the lazy build);
  // otherwise the launches read the narrowest copy already built
  const bool eager = nq >= 2 && corpus->n >= 32768;
  bool q8_ready = false;
  if ((rc = k1_copy_ready(ctx, const_cast<stb_corpus *>(corpus), STB_TIER_Q8, top_k, {eager, eager}, &q8_ready)) != STB_OK) return rc;
  if ((rc = dev_reserve(&ctx->bq_dev, &ctx->bq_dev_cap, (size_t)nq * STB_D)) != STB_OK) return rc;
  if ((rc = ensure_hits_pin(ctx, (size_t)nq * top_k)) != STB_OK) return rc;
  if ((size_t)nq * STB_D > ctx->many_q_pin_cap) {
    float *np = nullptr; uint32_t *ns = nullptr;
    const size_t cap = std::max<size_t>((size_t)nq, 64);
    if (cudaMallocHost((void **)&np, cap * STB_D * sizeof(float)) != cudaSuccess ||
        cudaMallocHost((void **)&ns, cap * 4 * sizeof(uint32_t)) != cudaSuccess) {
      cudaGetLastError(); if (np) cudaFreeHost(np);
      stb_set_error("search_many: pinned staging allocation failed"); return STB_ERR_NOMEM;
    }
    if (ctx->many_q_pin) cudaFreeHost(ctx->many_q_pin);
    if (ctx->many_status_pin) cudaFreeHost(ctx->many_status_pin);
    ctx->many_q_pin = np; ctx->many_status_pin = ns; ctx->many_q_pin_cap = cap * STB_D;
  }
  memcpy(ctx->many_q_pin, q, (size_t)nq * STB_D * sizeof(float));
  STB_CUDA(cudaMemcpyAsync(ctx->bq_dev, ctx->many_q_pin, (size_t)nq * STB_D * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  const int tier = q8_ready ? STB_TIER_Q8 : best_built_tier(ctx, corpus, top_k);
  for (uint32_t i = 0; i < nq; ++i) {
    stb_hit *oh = ctx->hits_pin + (size_t)i * top_k;
    uint32_t *os = ctx->many_status_pin + 4 * (size_t)i;
    if (x) rc = stb_search_topk_xchg(ctx, corpus, ctx->bq_dev + (size_t)i * STB_D, top_k, x, oh, os);
    else rc = stb_launch_scan_topk(ctx, corpus, tier, ctx->bq_dev + (size_t)i * STB_D, top_k, nullptr, 0, corpus->n, oh, os, nullptr,
                                   nq > 1);
    if (rc != STB_OK) { cudaStreamSynchronize(ctx->stream); return rc; }
  }
  STB_CUDA(cudaStreamSynchronize(ctx->stream));
  for (uint32_t i = 0; i < nq; ++i) {
    const uint32_t *st = ctx->many_status_pin + 4 * (size_t)i;
    if (x && st[2] == 0xfffffffeu) { x->dead = true; stb_set_error("search_many: a peer rank never arrived (timeout)"); return STB_ERR_STATE; }
    if (st[1]) {
      const uint32_t n = std::min<uint32_t>(st[0], top_k);
      memcpy(out_hits + (size_t)i * top_k, ctx->hits_pin + (size_t)i * top_k, n * sizeof(stb_hit));
      out_n[i] = n;
    } else if (x) {
      if (out_complete) out_complete[i] = 0;               // every rank sees the same flag: fall back together
    } else {
      uint64_t n = 0;                                      // tier ladder / collect path
      rc = stb_search(ctx, corpus, q + (size_t)i * STB_D, top_k, 0, 0.0, STB_MODE_SEARCH_DOCUMENTS, nullptr, 0,
                      out_hits + (size_t)i * top_k, top_k, &n);
      if (rc != STB_OK) return rc;
      out_n[i] = (uint32_t)n;
    }
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
  if ((rc = dev_reserve(&ctx->hits_dev, &ctx->hits_cap, total + top_k)) != STB_OK) return rc;
  if ((rc = ensure_hits_pin(ctx, std::max<size_t>(total, top_k))) != STB_OK) return rc;
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

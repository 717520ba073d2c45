/*
 * semtools_b200.h -- C ABI of the H100-native `search` hot path of semtools.
 *
 * The reference (run-llama/semtools v3.0.0, paths relative to the reference repository root)
 * has no FFI layer of its own: the seam is a set of Rust calls into two
 * third-party crates (model2vec-rs, simsimd) plus its own scan/sort loop.  Each
 * entry point below names the reference interface it replaces; INTEGRATION.md
 * shows the `extern "C"` block a semtools maintainer would add.
 *
 * Conventions
 *   - every function returns 0 (STB_OK) or a negative stb_status;
 *     stb_last_error() returns the message of the calling thread's last failure
 *   - nothing throws or aborts across this boundary
 *   - the caller owns every buffer it passes; the library owns everything
 *     behind the opaque handles; outputs go to caller-allocated arrays with
 *     explicit capacities
 *   - one host thread per context at a time (the reference runs the whole
 *     search path on one blocking thread, src/bin/semtools.rs:134-135)
 *   - pointers named *_dev are CUDA device pointers on the context's device,
 *     everything else is host memory
 *   - there is NO CPU fallback: without a usable sm_90 device every call fails
 *     with STB_ERR_CUDA
 *
 * Vector width is fixed at 256 f32 (LINE_EMBEDDING_SIZE,
 * src/workspace/store.rs:37); other widths fail with STB_ERR_ARG.
 *
 * Environment switches (read per call; results are identical whatever their
 * value -- they select how candidates are found, never how the returned
 * distances are computed): STB_SCAN_TIER=f32|h16|q8 (narrowest candidate copy K1
 * may read, default q8), STB_IVFPQ_BATCH_KEEP=k (INTEGRATION.md, 5b).
 */
#ifndef SEMTOOLS_B200_H
#define SEMTOOLS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define STB_DIM 256u

typedef enum stb_status {
  STB_OK = 0,
  STB_ERR_ARG = -1,      /* bad argument (null handle, wrong width, ...)          */
  STB_ERR_CUDA = -2,     /* CUDA runtime failure / no sm_90 device                */
  STB_ERR_NOMEM = -3,    /* host or device allocation failed                       */
  STB_ERR_RANGE = -4,    /* token id / row range outside the table or corpus       */
  STB_ERR_CAPACITY = -5, /* result does not fit `cap`; *out_n holds the full count */
  STB_ERR_STATE = -6     /* call not valid in the handle's current state           */
} stb_status;

typedef struct stb_ctx stb_ctx;       /* one CUDA device + stream + scratch        */
typedef struct stb_table stb_table;   /* model2vec embedding table resident in HBM */
typedef struct stb_corpus stb_corpus; /* row-major N x 256 f32 line-vector matrix  */
typedef struct stb_tokenizer stb_tokenizer; /* tokenizer.json loaded; Unigram model in HBM */

/* One search hit: (distance, global row) -- 16 bytes, the unit of the
 * cross-GPU top-k exchange.  `row` is the line's position in (document order,
 * line order), i.e. the reference's iteration order (src/search/mod.rs:84-85),
 * so ordering by (distance, row) reproduces its stable sort (:107-111). */
typedef struct stb_hit {
  double distance;
  uint64_t row;
} stb_hit;

int stb_version(void);
const char *stb_last_error(void);

/* Device count visible to the library (0 if no driver / no GPU). */
int stb_device_count(void);

/* ---- context ----------------------------------------------------------------
 * `cuda_stream` may be NULL (the library creates its own non-blocking stream) or
 * an existing cudaStream_t that every kernel/copy of this context is issued on
 * (lets a host framework time the work with its own events).  NULL never means
 * "the default stream": pass cudaStreamLegacy / cudaStreamPerThread for those.
 * Tables and corpora may be destroyed after their context (any order is safe). */
int stb_ctx_create(int device, void *cuda_stream, stb_ctx **out);
int stb_ctx_destroy(stb_ctx *ctx);
int stb_ctx_sync(stb_ctx *ctx);
/* cudaStream_t the context launches on. */
void *stb_ctx_stream(stb_ctx *ctx);

/* ---- embedding table ---------------------------------------------------------
 * Replaces the tensors held by StaticModel after
 * StaticModel::from_pretrained(MODEL_NAME, None, None, None)
 * (src/cmds/search.rs:123-128, src/search/mod.rs:16): table E[V][256] f32,
 * optional per-token weights[n_weights], optional token->row mapping[n_mapping],
 * and the `normalize` flag from config.json.  Uploaded once, read-only after. */
int stb_table_load(stb_ctx *ctx, const float *E, uint64_t V, uint32_t D,
                   const float *weights, uint64_t n_weights,
                   const uint32_t *mapping, uint64_t n_mapping, int normalize,
                   stb_table **out);
int stb_table_destroy(stb_table *table);

/* ---- corpus -------------------------------------------------------------------
 * Replaces Document.embeddings: Vec<Vec<f32>> (src/search/mod.rs:18-22) and the
 * line_embeddings shard's vectors (src/workspace/store.rs:140-160) with ONE
 * contiguous matrix in HBM.  `row_base` is the global row id of local row 0
 * (non-zero when this context holds one row-shard of a larger corpus). */
int stb_corpus_create(stb_ctx *ctx, uint32_t D, uint64_t capacity_rows,
                      uint64_t row_base, stb_corpus **out);
/* A corpus larger than HBM: its f32 rows live in page-locked, device-mapped host memory that the library
 * allocates and owns, and only the q8 copy (396 B per row) lives in HBM, so one 80 GB card holds ~190M rows
 * instead of ~50M.  It returns an ordinary stb_corpus handle; the hits of every search are bit for bit those
 * of a device corpus holding the same rows, because every route ends in the same canonical re-rank, which
 * reads the candidate rows over the host link.  Only the route differs.
 *  - The q8 copy is always current.  Creation allocates the host rows and the q8 copy for capacity_rows;
 *    STB_ERR_NOMEM if either fails, and nothing is created.  stb_corpus_append, stb_corpus_append_dev,
 *    stb_embed with append_to, stb_corpus_update and stb_corpus_remove encode the rows they add or write into
 *    the q8 copy from HBM in the same call: there is no lazy build.  Its bytes are those stb_corpus_prepare
 *    (STB_PREPARE_Q8) writes on a device corpus holding the same rows; a row that cannot be normalised marks it
 *    unusable as on a device corpus (stb_corpus_tier_stats: built_rows[q8] = 0), and searches then use the f32
 *    passes.  An update or removal on a corpus whose copy is unusable re-encodes the whole copy from the rows.
 *  - Appending.  stb_corpus_append uploads each row once, into the context's staging buffer (chunks of at most
 *    262144 rows, 256 MiB of HBM, the buffer stb_corpus_update uses); one kernel writes the chunk to the host
 *    rows and encodes its q8 entries.  stb_corpus_append_dev does the same from the caller's device rows, and
 *    stb_embed with append_to lets K3 write chunks of lines into the staging buffer.  A call that fails appends
 *    nothing.  Growing past the capacity allocates new host rows and a new q8 copy and then frees the old ones:
 *    while it runs the corpus holds two host buffers (1 KiB per row each).
 *  - stb_corpus_update / stb_corpus_remove: arguments, validation, atomicity, epochs, the tier statistics and
 *    the end of a co-scan series are the device corpus's.  The kernels write the host rows in place through the
 *    mapped pointer; neither holds a second copy of the rows.  Their cost is the host link's: an update moves
 *    each written row up once and down once (~2 KiB per row); a removal reads and writes every row behind the
 *    first removed one over the link (~2 KiB per moved row).  Measured on an H100 80GB HBM3 at 700 W with 10M
 *    rows: an update of 10000 rows 2.9 ms (device corpus 2.1 ms); a removal of 10000 rows at the middle, which
 *    moves 5M rows, 673 ms (device corpus 9.3 ms).
 *  - stb_search never streams the f32 rows while an HBM copy can answer: top_k <= 16 without a threshold takes
 *    the q8 top-k scan; a result it cannot prove, and any top_k <= 96, next takes the 16-bit top-k scan if the
 *    shadow exists (stb_corpus_prepare(STB_PREPARE_H16) or K2 built it; it is never built lazily here), and
 *    otherwise the q8 histogram -> q8 collect -> proof route that top_k > 96 and threshold mode take.  The f32
 *    passes, which stream the rows over the host link, run only when that route cannot prove its result or the
 *    q8 copy is unusable; stb_ctx_counters' fallback count counts those searches, and stb_corpus_tier_stats
 *    shows no f32 top-k scan.
 *  - stb_search_topk_dev and stb_search_many (without an exchange) read the q8 copy (top_k <= 16) or the
 *    16-bit shadow if it is built; otherwise they return STB_ERR_STATE and launch nothing.
 *  - K2 (stb_search_batch, _dev, _filtered, _threshold) works as on a device corpus: the shadow (512 B per row
 *    of HBM; STB_ERR_NOMEM when it does not fit) is built from the host rows through the staging buffer, and
 *    the re-scores and the K1 fallback read the host rows.
 *  - Refused with STB_ERR_STATE, nothing changed: stb_corpus_data_dev (there is no device matrix to hand to a
 *    zero-copy producer), stb_ivfpq_build, and the exchange forms (stb_search_topk_xchg, stb_search_xchg,
 *    stb_search_batch_xchg_dev, stb_search_many with an exchange).  These are scope limits of this release,
 *    not technical ones.
 *  - stb_corpus_read, _clear, _rows, _prepare and destroy work as on a device corpus; the corpus may outlive
 *    its context.
 * Cost of the K1 re-rank over the host link, on an H100 80GB HBM3 at 700 W with 10M rows: not visible at
 * top_k = 10 (1754 vs 1753 q/s through stb_search, within noise), so the kernels read the mapped rows as they
 * are.  The collect routes re-rank more rows: top_k = 50 500 vs 546 q/s, threshold 814 vs 838 q/s. */
int stb_corpus_create_host(stb_ctx *ctx, uint32_t D, uint64_t capacity_rows, uint64_t row_base, stb_corpus **out);
int stb_corpus_destroy(stb_corpus *corpus);
int stb_corpus_append(stb_corpus *corpus, const float *rows, uint64_t n);
int stb_corpus_append_dev(stb_corpus *corpus, const float *rows_dev, uint64_t n);
int stb_corpus_clear(stb_corpus *corpus);
int stb_corpus_rows(const stb_corpus *corpus, uint64_t *n);
/* device pointer of local row 0 (for zero-copy producers). */
int stb_corpus_data_dev(const stb_corpus *corpus, float **rows_dev);
/* copy rows [first, first+n) back to the host (tests, store write-back). */
int stb_corpus_read(const stb_corpus *corpus, uint64_t first, uint64_t n,
                    float *rows);
/* Replace and delete rows in HBM (a long-lived host that changes or drops a document's lines without
 * clearing and re-uploading the corpus; the reference's upsert by id and delete by path filter,
 * src/workspace/store.rs:298-357,402-434).
 * stb_corpus_update: idx holds n GLOBAL row ids (row_base + local), strictly ascending, each below
 *   row_base + rows; rows is n x 256 f32 (host).  Row idx[i] becomes rows[i].
 * stb_corpus_remove: ranges holds n_ranges half-open [begin, end) pairs of GLOBAL rows, ascending and
 *   disjoint as in stb_search, each non-empty and inside the corpus.  The rows after a removed range
 *   move down; their order is kept.
 * Both are synchronous on the context's stream, like stb_corpus_append:
 *  - Validation first: a refused call writes nothing, the rows and the candidate copies stay byte for
 *    byte as they were.  Unsorted, duplicate or out-of-range idx, and unsorted, overlapping, empty or
 *    out-of-range ranges: STB_ERR_RANGE.  A NULL pointer with n > 0 (n_ranges > 0): STB_ERR_ARG.
 *    n == 0 and n_ranges == 0 do nothing.
 *  - STB_ERR_STATE while an IVF-PQ index built on this corpus is alive (stb_ivfpq_build .. destroy): the
 *    index refers to rows by position and re-ranks from the rows.
 *  - The candidate copies (q8 tier, 16-bit shadow) that exist stay built: each keeps covering a prefix of
 *    the rows (all of them unless rows were appended and not yet converted), and that prefix is byte for
 *    byte what stb_corpus_prepare writes on a fresh corpus holding the same rows, the zero padding of the
 *    shadow's last tile included.  A copy marked unusable before the call (a row that cannot be normalised
 *    in fp32) is dropped, so the next prepare or lazy build decides anew; otherwise a written row that
 *    cannot be normalised marks the copy unusable, as a build does.
 *  - Both start a new epoch (stb_ivfpq_extend refuses the corpus as after stb_corpus_clear), reset the
 *    per-tier bookkeeping of stb_corpus_tier_stats, and end a co-scan series: the next asynchronous top-k
 *    query starts its pass at tile 0.  The allocation never shrinks.
 *  - Work already enqueued on the stream (e.g. stb_search_topk_dev) finishes on the old rows first.
 * Cost: update moves ~4 KiB of HBM traffic per row plus its 1 KiB upload; remove ~5 KiB per row behind the
 * first removed row.  Extra device memory: a staging buffer of at most 262144 rows (256 MiB), kept by the
 * context, never a second copy of the corpus. */
int stb_corpus_update(stb_corpus *corpus, const uint64_t *idx, const float *rows, uint64_t n);
int stb_corpus_remove(stb_corpus *corpus, const uint64_t *ranges, uint32_t n_ranges);

/* ---- K3: gather + mean-pool + L2-normalise -------------------------------------
 * Replaces model.encode_with_args(&lines, Some(2048), 16384)
 * (src/search/mod.rs:69, src/cmds/search.rs:154) and model.encode_single(q)
 * (src/search/mod.rs:138,153; src/cmds/search.rs:136) MINUS tokenisation, which
 * stays on the host: the caller passes the token ids of each line as a CSR batch
 * (offsets[n_lines+1], ids[offsets[n_lines]]), already unk-dropped and truncated
 * (2048 ids per corpus line, 512 for the query).  Output row i is bit-identical
 * to pool_ids(ids of line i) of model2vec-rs 0.1.3, subnormals included (no
 * flush-to-zero).  One exception: a component that is NaN is NaN exactly where
 * pool_ids gives NaN, but its payload is the canonical quiet NaN 0x7fffffff, not
 * the payload a CPU may propagate from a NaN in the table or the weights.
 * `out` (host, n_lines x 256) and `append_to` may each be NULL; with `append_to`
 * the rows are written straight into the corpus in HBM and never visit the host.
 * A token whose table row is out of range fails the call with STB_ERR_RANGE
 * (upstream panics) and appends nothing.  The call reports its own tokens only
 * through its return value, never through the stb_embed_dev flag below. */
int stb_embed(stb_ctx *ctx, const stb_table *table, const uint64_t *offsets,
              const uint32_t *ids, uint64_t n_lines, float *out,
              stb_corpus *append_to);

/* Asynchronous device-resident form of stb_embed: CSR and output already in HBM
 * (out_dev: n_lines x 256 f32, e.g. a slice of stb_corpus_data_dev), nothing
 * synchronises.  A token outside the table sets a sticky per-context flag instead
 * of failing (its line is pooled as if the token were row 0);
 * stb_embed_status() synchronises the stream, returns STB_ERR_RANGE if the flag was
 * set since the last call, and clears it.  Only stb_embed_dev sets the flag and
 * only stb_embed_status clears it: no other call on the context (searches, copy
 * builds, stb_embed) reads or writes it. */
int stb_embed_dev(stb_ctx *ctx, const stb_table *table, const uint64_t *offsets_dev,
                  const uint32_t *ids_dev, uint64_t n_lines, float *out_dev);
int stb_embed_status(stb_ctx *ctx);

/* ---- K3 from text: the tokenizer on the GPU ----------------------------------------
 * The same rows as stb_embed, from the lines' text instead of their token ids: the tokenisation half of
 * encode_with_args (tokenizer.encode_batch_fast(add_special_tokens = false), the unk_token drop, truncation to
 * max_length ids) moves into the library.
 *
 * stb_tokenizer_load takes the bytes of a tokenizer.json.  The library parses it with the C++ host's
 * tokenizer (host/semtools_tokenizer.hpp, HfTokenizer): a shape that tokenizer refuses fails with
 * STB_ERR_ARG and its message.  A loaded handle belongs to `ctx`; its Unigram model (byte trie, f64 scores,
 * unk id) is resident in HBM.
 *
 * Which lines are tokenised on the GPU is decided by stb_tokenizer_gpu_lines alone (pure host code): taken[i]
 * = 1 iff the tokenizer has the GPU shape -- a Unigram model with an unk_id, one Metaspace pre-tokenizer with
 * split = true whose replacement is one non-ASCII character, normaliser steps among Lowercase, Precompiled,
 * Replace(" {2,}" -> " "), Strip and Prepend (printable ASCII text) -- and line i
 *   - is printable ASCII (0x20-0x7E) only,
 *   - has only bytes that every Precompiled step leaves alone, as they are and lowercased,
 *   - contains no added token's content, neither as given nor after normalisation,
 *   - has no run of non-space bytes whose length, plus the replacement's bytes and the Prepend steps' bytes,
 *     exceeds STB_TOKENIZER_PIECE_CAP (a Metaspace piece is the replacement plus such a run).
 * Any other shape (WhitespaceSplit, Sequence pre-tokenizers, a string Replace, NFKC, ...) loads, and no line is taken.
 *
 * stb_embed_text: lines are text[text_offsets[i], text_offsets[i + 1]) (text_offsets[0] = 0), already cut
 * by model2vec's truncate_str.  Taken lines are uploaded and tokenised on the GPU (normalise, Metaspace split,
 * a Viterbi that follows the host's exactly: f64 scores, strict > on ties, unknown characters at
 * min_score - 10, consecutive unknowns fused into one unk id); declined lines are tokenised on host threads by
 * the same tokenizer.  The ids of both form one CSR in HBM, which the K3 kernel of stb_embed pools.  Rows,
 * `out`, `append_to` and STB_ERR_RANGE are exactly stb_embed's on the ids encode_with_args would produce
 * (a failed call appends nothing).  A line the host tokenizer refuses (e.g. NFKC on non-ASCII text) fails
 * the call with STB_ERR_ARG before anything is written.  Large inputs are processed in chunks of
 * context scratch that grows on demand.
 *
 * stb_debug_tokenize returns the CSR stb_embed_text would pool (ids_offsets[n_lines + 1] always; ids while
 * they fit ids_cap, else STB_ERR_CAPACITY) and, if taken is not NULL, the rule's verdict.
 *
 * stb_tokenizer_load_ex(..., STB_TOKENIZER_UTF8, ...) loads a handle whose GPU rule is UTF-8 text (flags = 0 is
 * stb_tokenizer_load).  For the same GPU shape, plus the Precompiled charsmaps, the grapheme-break properties and
 * the lowercase map resident in HBM, stb_tokenizer_gpu_lines takes a line iff it
 *   - is valid UTF-8 (shortest form, no surrogates, nothing above U+10FFFF) -- control characters, NUL, tab, the
 *     Metaspace replacement and every script are allowed,
 *   - contains no added token's content, neither as given nor (for normalized = true tokens) after normalisation.
 * The kernels normalise such a line by the tokenizer's steps in order (Precompiled grapheme cluster by cluster,
 * UAX #29), split it on spaces and on the replacement character, and run the Viterbi.  A line they cannot finish
 * exactly is given back to the host tokenizer inside the same call: its normalised text outgrows twice its bytes
 * plus the Prepend bytes, a Metaspace piece exceeds STB_TOKENIZER_PIECE_CAP, or -- under prepend_scheme "first" --
 * the normaliser removed the line's leading characters (HF decides "first" by the original offset).  For such a
 * handle stb_debug_tokenize's taken[i] = 1 means line i's ids came from the GPU (a subset of the rule's lines).
 * Every line gets exactly the ids a flags-0 handle of the same tokenizer.json gives it, so rows, errors and
 * "a failed call appends nothing" are the same; only where the work runs differs. */
#define STB_TOKENIZER_PIECE_CAP 256u
#define STB_TOKENIZER_UTF8 1u
int stb_tokenizer_load(stb_ctx *ctx, const uint8_t *json, uint64_t len, stb_tokenizer **out);
int stb_tokenizer_load_ex(stb_ctx *ctx, const uint8_t *json, uint64_t len, uint32_t flags, stb_tokenizer **out);
int stb_tokenizer_destroy(stb_tokenizer *tok);
int stb_tokenizer_gpu_lines(const stb_tokenizer *tok, const uint8_t *text, const uint64_t *text_offsets,
                            uint64_t n_lines, uint8_t *taken);
int stb_embed_text(stb_ctx *ctx, const stb_tokenizer *tok, const stb_table *table,
                   const uint8_t *text, const uint64_t *text_offsets, uint64_t n_lines,
                   uint32_t max_length, float *out, stb_corpus *append_to);
int stb_debug_tokenize(stb_ctx *ctx, const stb_tokenizer *tok, const uint8_t *text,
                       const uint64_t *text_offsets, uint64_t n_lines, uint32_t max_length,
                       uint64_t *ids_offsets, uint32_t *ids, uint64_t ids_cap, uint8_t *taken);

/* ---- K1 + K4: cosine scan, top-k / threshold, exact re-rank ---------------------
 * Replaces search_documents' scan/filter/sort/take (src/search/mod.rs:84-119,
 * one f32::cosine per line at :86) and, with `row_ranges`, the filtered query of
 * Store::search_line_embeddings (src/workspace/store.rs:481-546).
 *
 *   q            256 f32 query vector (host)
 *   top_k        config.top_k (:118)
 *   has_max /    config.max_distance (:88): a hit needs distance < max_distance
 *   max_distance (strict; 100.0 when absent).
 *   mode         STB_MODE_SEARCH_DOCUMENTS: has_max lifts the top_k cap (:115-119)
 *                STB_MODE_STORE_QUERY:      top_k always caps (store.rs:517,543)
 *   row_ranges   NULL, or n_ranges half-open [begin,end) pairs of GLOBAL rows,
 *                ascending and disjoint: only these rows are scanned
 *   out_hits     cap entries; on return the first min(*out_n, cap) are filled,
 *                ordered by (distance asc, row asc); distances are the canonical
 *                f64 cosine distance (oracle/semtools_oracle.c: orc_cosine_f32)
 *   out_n        full result count; if it exceeds cap the call returns
 *                STB_ERR_CAPACITY after filling cap entries
 * On a sharded corpus (row_base != 0 or several contexts) the result is the
 * shard-local answer; merge shards with stb_hits_merge*. */
#define STB_MODE_SEARCH_DOCUMENTS 0
#define STB_MODE_STORE_QUERY 1
int stb_search(stb_ctx *ctx, const stb_corpus *corpus, const float *q,
               uint32_t top_k, int has_max, double max_distance, int mode,
               const uint64_t *row_ranges, uint32_t n_ranges, stb_hit *out_hits,
               uint64_t cap, uint64_t *out_n);

/* Candidate tiers.  The scan is HBM-bound, so the way to go faster than the f32 roofline is
 * to read fewer bytes: stb_search can draw its candidates from a reduced-width copy of the
 * corpus -- "q8": int8 codes + one f32 scale per row, 260 B/row, top_k <= 16; "h16": the
 * 16-bit L2-normalised shadow K2 multiplies, 512 B/row -- and re-ranks them in the canonical
 * f64 arithmetic on the f32 rows exactly as before.  Each tier proves its own result (rounding
 * bound of the copy vs. the gap to the best row it dropped); an unproven query is retried on
 * the next wider tier, so the hits are identical to the f32 path's.  stb_search builds the
 * copies lazily (second query on an unchanged corpus of >= 32768 rows);
 * stb_corpus_prepare builds them now.  Costs +25 % / +50 % HBM.  No reference analogue
 * (the reference keeps Vec<Vec<f32>>, src/search/mod.rs:18-22). */
#define STB_PREPARE_Q8 1
#define STB_PREPARE_H16 2
int stb_corpus_prepare(stb_corpus *corpus, int what);
/* Per-tier bookkeeping of stb_search on this corpus since its last change, index = tier
 * (0 f32, 1 h16, 2 q8): fast-path scans tried / proven, and the rows each copy covers
 * (0 = not built or refused).  Any pointer may be NULL. */
int stb_corpus_tier_stats(const stb_corpus *corpus, uint32_t tries[3], uint32_t proven[3],
                          uint64_t built_rows[3]);

/* Asynchronous device-resident form of the top-k search (no threshold, no
 * ranges): query and results stay in HBM, nothing synchronises.  out_hits_dev
 * receives top_k entries (unused tail: distance = +inf, row = UINT64_MAX) and
 * out_status_dev[0] the hit count, out_status_dev[1] a completeness flag
 * (1 = provably the exact top-k; 0 = the candidate margin check failed and the
 * caller must fall back to stb_search, which handles it internally),
 * out_status_dev[3] = K' | tier << 16 (tier: 0 f32, 1 h16, 2 q8).  Reads the
 * narrowest copy that is already built (never builds one). */
int stb_search_topk_dev(stb_ctx *ctx, const stb_corpus *corpus,
                        const float *q_dev, uint32_t top_k, stb_hit *out_hits_dev,
                        uint32_t *out_status_dev);

/* ---- K2: batched queries on the tensor cores ------------------------------------------
 * Q independent top-k searches (the semantics of Q calls of search_documents,
 * src/search/mod.rs:77-120, without max_distance) in one pass over the corpus: an
 * L2-normalised 16-bit copy of the corpus (fp16 by default, bf16 with -DSTB_SHADOW_F16=0;
 * built lazily, 512 B/row, extended after appends; stb_corpus_prepare_batch builds it ahead
 * of time) is multiplied with the query tile on the wgmma tensor cores.  Pipeline v2 (top_k <= 64
 * when the sampled threshold fits, see DESIGN §4) emits every row whose approximate score reaches a
 * per-query threshold and re-scores those exactly; pipeline v1 (top_k > 64, or wherever v2 does not
 * fit) re-scores the 32 most promising 32-row sub-tiles per query.  Re-scores use the
 * canonical f64 distance on the f32 rows, and a result is accepted only if the 16-bit error bound
 * proves no other row can enter the top-k; unproven queries are answered by the single-query path
 * (stb_search).  Results are therefore identical to stb_search.
 * Where the shadow cannot be allocated (a corpus too large for HBM to hold it beside the rows and the q8
 * copy), both forms read the q8 copy instead (route 7, built or extended first; DESIGN §4): the queries are
 * quantised to 16 bits as K1 quantises them, their two bytes are multiplied with the int8 codes on the int8
 * tensor cores, and the threshold, emission, exact re-score and proof run on K1's upper and lower bounds.
 * It returns what the shadow's routes would: the host form's hits and counts are bit for bit stb_search's,
 * and a query the _dev form marks proven carries exactly stb_search's hits.  It runs when its sampled threshold
 * fits: top_k <= 64 up to ~50M rows, top_k <= 32 up to ~100M, top_k <= 16 up to ~200M (in general
 * ceil(ceil(n / 256) / 49152) <= floor(256 / top_k); stb_debug_batch_q8_plan).  Otherwise every query comes
 * back unproven, and the host form answers it through stb_search.
 * Zero and unnormalisable queries are never proven there.  If the q8 copy cannot be used either (it does not
 * fit, or a row cannot be normalised), the call fails with the shadow's STB_ERR_NOMEM and writes nothing.
 *   q         nq x 256 f32 (host);  out_hits nq x top_k (unused tail: +inf / UINT64_MAX)
 *   out_n     nq counts */
int stb_corpus_prepare_batch(stb_corpus *corpus);
int stb_search_batch(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t nq,
                     uint32_t top_k, stb_hit *out_hits, uint32_t *out_n);
/* Asynchronous device-resident form: out_status_dev[2*i] = hits of query i,
 * [2*i+1] = 1 iff proven exact (0: re-run query i through stb_search).  A query that cannot be
 * normalised in fp32 (a NaN or infinite component, or a non-zero fp32 squared norm outside
 * [1e-30, 1e30]) is never proven; the other queries of the batch are unaffected.  A zero query is
 * valid but every row ties with it, so it is proven only on corpora of at most top_k rows.
 * Corpus rows that cannot be normalised make the call fail with STB_ERR_STATE. */
int stb_search_batch_dev(stb_ctx *ctx, const stb_corpus *corpus, const float *q_dev,
                         uint32_t nq, uint32_t top_k, stb_hit *out_hits_dev,
                         uint32_t *out_status_dev);
/* The workspace query (Store::search_line_embeddings, src/workspace/store.rs:481-546) for a batch:
 * for every query i, out_hits[i*top_k ..] and out_n[i] equal, bit for bit, what
 *   stb_search(ctx, corpus, q_i, top_k, has_max, max_distance, STB_MODE_STORE_QUERY, row_ranges, n_ranges, ...)
 * returns (unused tail: +inf / UINT64_MAX).  row_ranges are GLOBAL rows as stb_search takes them and are
 * clipped to the shard; NULL = every row; non-NULL with n_ranges == 0 = the empty subset (every count 0).
 * Ranges stb_search refuses are refused with the same status before anything is written.  Any top_k.
 * Pipeline v2 runs on the eligible rows only (its sample over the 256-row tiles that hold an eligible row,
 * ineligible scores masked out of both epilogues) when top_k <= 64 and the plan fits; K1 (stb_search)
 * answers every query it leaves unproven, and all queries otherwise.  Pipeline v1 is never used here.
 * Where the 16-bit shadow does not fit in HBM, the same passes run on the q8 copy and the int8 tensor cores
 * (route 8, as stb_search_batch's route 7, over the listed tiles) when top_k <= 64 and the q8 plan fits, whether or
 * not v2's does.  The shadow is built only where v2's plan fits; where only the q8 plan fits, the call asks whether
 * the shadow could be allocated with a trial allocation, released at once.  K1 answers
 * the rest, and every query when the q8 copy cannot be used either.  The shadow's STB_ERR_NOMEM is never returned;
 * a failure to reserve scratch is (STB_ERR_NOMEM, before anything is written).
 * The distance cap (strict; a NaN cap passes nothing) is applied to the sorted hits on the host. */
int stb_search_batch_filtered(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t nq,
                              uint32_t top_k, int has_max, double max_distance,
                              const uint64_t *row_ranges, uint32_t n_ranges,
                              stb_hit *out_hits, uint32_t *out_n);
/* The workspace query for a batch in which every query names its own subset (an agent host's tool calls, a
 * server over one workspace): for every query i, out_hits[i*top_k ..] and out_n[i] equal, bit for bit, what
 *   stb_search(ctx, corpus, q_i, top_k, has_max, max_distance, STB_MODE_STORE_QUERY,
 *              row_ranges + 2*range_offsets[i], range_offsets[i+1] - range_offsets[i], ...)
 * returns (unused tail: +inf / UINT64_MAX).
 *   range_offsets  nq + 1 entries, range_offsets[0] = 0, non-decreasing: query i's ranges are
 *                  row_ranges[2*range_offsets[i] .. 2*range_offsets[i+1]), GLOBAL [begin, end) pairs clipped to the
 *                  shard.  A query with zero ranges has the empty subset and 0 hits; there is no NULL meaning "every
 *                  row" (pass the shard's own range for that).
 * Refused before anything is written: range_offsets[0] != 0, decreasing offsets, or row_ranges == NULL with
 * range_offsets[nq] > 0 (STB_ERR_ARG); a query's ranges that stb_search refuses (the same status).  nq == 0 is a
 * no-op; top_k == 0 sets every count to 0.  Host-rows corpora are served as stb_search_batch_filtered serves them.
 * Queries whose clipped ranges are identical form one group.  One group for the whole batch is exactly
 * stb_search_batch_filtered on it (route 3 or 4).  Otherwise (route 6) every group whose v2 plan fits over its
 * listed tiles (top_k <= 64) runs on the tensor cores, each in whole 64-query halves of the query tiles, with
 * one sampling pass and one emitting pass for all of them; K1 (stb_search, with the query's own ranges)
 * answers the other groups and every query the tensor passes leave unproven.  Extra device memory, in context
 * scratch that grows on demand: one eligible-row bitmap per tensor group (N/8 bytes each, whose 8-word slices
 * are the mask slots a work item names; 64 bytes of mask words reach shared memory per item), the two passes'
 * work lists (16 bytes per (corpus tile, query tile) item, 4 per listed tile and per CTA), the queries in slot
 * order (1 KiB per slot, 64 slots per half), and the per-group sample, laid out [query tile][largest
 * n_sample][128 queries].
 * Where the 16-bit shadow does not fit in HBM and a group fits either plan (the shadow is asked for as in
 * stb_search_batch_filtered), route 9 runs instead: each group whose q8 plan fits runs route 8's passes
 * (stb_search_batch_filtered) on its own queries, one group after another; K1 answers the rest, and every query
 * when the q8 copy cannot be used either.  The shadow's STB_ERR_NOMEM is never returned. */
int stb_search_batch_subsets(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t nq,
                             uint32_t top_k, int has_max, double max_distance,
                             const uint64_t *range_offsets, const uint64_t *row_ranges,
                             stb_hit *out_hits, uint32_t *out_n);
/* Threshold mode of search_documents (src/search/mod.rs:88-89,115-116) for a batch: for every query i,
 * out_hits[out_offsets[i] .. out_offsets[i+1]) equals, bit for bit, the hits of
 *   stb_search(ctx, corpus, q_i, 0, 1, max_distance, STB_MODE_SEARCH_DOCUMENTS, NULL, 0, ...)
 * (every row with canonical distance < max_distance, ordered by (distance, row), global rows).
 *   q            nq x 256 f32 (host)
 *   out_offsets  nq + 1 entries, out_offsets[0] = 0; the hits of all queries are concatenated in query order
 *   out_hits     cap entries (may be NULL when cap == 0).  If out_offsets[nq] > cap the first cap hits of the
 *                concatenation are filled, every offset is still written and the call returns STB_ERR_CAPACITY.
 * nq == 0 does nothing.  NULL q or out_offsets, or a corpus of another context: STB_ERR_ARG.  An empty corpus,
 * and a max_distance that is NaN or <= 0, give every count 0 without a launch; +inf passes every row.  No top_k
 * (threshold mode drops the cap) and no row ranges.
 * Route (DESIGN §4, K2 item 6): the emitting wgmma pass with a per-query threshold derived from max_distance
 * (DESIGN §5) into 64 keys per (query, CTA); queries with an overflowed segment get one more pass into exactly
 * sized segments, as long as that pass's keys stay within STB_BATCH_THRESHOLD_RETRY_KEYS (128 MiB of keys);
 * then the exact canonical re-score.  stb_search answers the rest: queries that cannot be normalised, the zero
 * query, queries beyond the budget, and every query when the corpus holds rows that cannot be normalised.
 * Where the 16-bit shadow does not fit in HBM (route 10), the same two passes run on the q8 copy and the int8
 * tensor cores, with thr = RD_f32(((1 - M) - 2e-5) - 1e-12) on K1's upper bounds; their band is wider, so more
 * queries need the second pass or pass the budget and go to stb_search.  If the q8 copy cannot be used either,
 * stb_search answers every query; the shadow's STB_ERR_NOMEM is never returned. */
#define STB_BATCH_THRESHOLD_RETRY_KEYS (1ull << 24)
/* Eligibility scratch of one stb_ivfpq_search_subsets launch (256 MiB): each distinct subset of a launch takes
 * ceil(rows / 32) + nlist words, and a launch holds as many subsets as fit (at least one). */
#define STB_IVFPQ_SUBSET_SCRATCH (1ull << 28)
int stb_search_batch_threshold(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t nq,
                               double max_distance, stb_hit *out_hits, uint64_t cap, uint64_t *out_offsets);

/* ---- fused multi-GPU search: K1 -> exchange over NVLink peer memory -> K4 -------------
 * One process (or thread) per GPU, one stb_xchg per rank.  Each rank allocates an
 * exchange buffer; the ranks trade its 64-byte CUDA IPC handle through whatever channel
 * the host has (MPI, torch.distributed, a pipe ...) and connect.  After that
 * stb_search_topk_xchg is ONE kernel per query per rank: the scan's final CTA stores its
 * k hits directly into every peer's buffer, release-stores a sequence flag, waits for
 * the peers' flags and merges by (distance,row) -- no NCCL call, no second launch.
 * All ranks must issue the same sequence of stb_search_topk_xchg calls (same top_k).
 * Within one process (several contexts), use stb_xchg_connect_local instead of IPC.
 *   out_status_dev[0] = hits, [1] = 1 iff every rank proved its shard result exact
 *   (0 -> run the per-shard stb_search + stb_hits_merge path), [2] = 0xfffffffe if a
 *   peer never arrived.  The wait is bounded (~15 s of SM cycles): ranks may enter a call seconds
 *   apart, not more.  After a timeout the ranks no longer agree on what was exchanged: stop using
 *   the exchange (destroy it on every rank); do NOT re-run queries on it, a surplus call waits a
 *   full bound for peers that will not come.  The synchronous entry points (stb_search_xchg,
 *   stb_search_many) mark the exchange dead when they see the timeout: every later call on it
 *   returns STB_ERR_STATE at once. */
typedef struct stb_xchg stb_xchg;
#define STB_IPC_HANDLE_BYTES 64
#define STB_XCHG_MAX_RANKS 8
int stb_xchg_create(stb_ctx *ctx, uint32_t world, uint32_t rank, uint32_t max_k,
                    stb_xchg **out);
int stb_xchg_destroy(stb_xchg *x);
int stb_xchg_local_handle(stb_xchg *x, uint8_t handle[STB_IPC_HANDLE_BYTES]);
/* handles: world x 64 bytes, entry r = rank r's handle (own entry ignored). */
int stb_xchg_connect(stb_xchg *x, const uint8_t *handles);
/* same-process variant: peers[r] = the stb_xchg of rank r (peers[rank] == x). */
int stb_xchg_connect_local(stb_xchg *x, stb_xchg *const *peers);
int stb_search_topk_xchg(stb_ctx *ctx, const stb_corpus *corpus, const float *q_dev,
                         uint32_t top_k, stb_xchg *x, stb_hit *out_hits_dev,
                         uint32_t *out_status_dev);
/* Sharded K2 over the same peer-memory exchange.  stb_xchg_create_batch allocates, behind the single-query
 * area, two batch slots of world x max_nq x max_k hits (+ flags and per-query proof bits); everything else
 * (handles, connect, destroy, stb_search_topk_xchg) works as with stb_xchg_create.
 * stb_search_batch_xchg_dev = stb_search_batch_dev on the local shard, then a push kernel (this rank's
 * nq x k hits into every peer's slot over NVLink, release-stored sequence flag) and a merge kernel (waits
 * for every peer's flag, merges each query's world x k hits by (distance,row)): two launches, no NCCL.
 *   out_status_dev[2q] = hits of query q, [2q+1] = 1 iff every rank proved its part, so a query that
 *   cannot be normalised is unproven on every rank (0: re-run query q
 *   through stb_search_xchg / stb_search_many on every rank; 2: a peer never arrived -- see above:
 *   treat the exchange as dead, the flags of this batch are not the same on every rank).
 * All ranks must issue the same sequence of calls. */
int stb_xchg_create_batch(stb_ctx *ctx, uint32_t world, uint32_t rank, uint32_t max_k, uint32_t max_nq,
                          stb_xchg **out);
int stb_search_batch_xchg_dev(stb_ctx *ctx, const stb_corpus *corpus, const float *q_dev, uint32_t nq,
                              uint32_t top_k, stb_xchg *x, stb_hit *out_hits_dev, uint32_t *out_status_dev);

/* ---- K5: IVF-PQ index (approximate) ------------------------------------------------------
 * NOT a replacement of any reference code: this snapshot of semtools has no IVF_PQ (the
 * store is qdrant-edge with a plain index, src/workspace/store.rs:129-130,156-157; the
 * string survives only in README.md:125).  Self-specified for BASELINE config 5 and
 * measured by recall against stb_search: coarse spherical k-means (nlist lists), 32 x 8-bit
 * product quantiser on the residual, ADC lookup-table scan of the nprobe best lists,
 * exact re-rank of the `rerank` best candidates.  Returned distances are exact canonical
 * distances; only the candidate set is approximate.  The index covers rows [0, rows) of its
 * corpus (stb_ivfpq_stats): the rows present at the build and those stb_ivfpq_extend has added
 * since; rows appended after that are not searched until the next extend.  It must be destroyed
 * before its corpus; while it is alive stb_corpus_update and stb_corpus_remove refuse the corpus
 * (stb_ivfpq_update and stb_ivfpq_remove change the corpus and the index together).
 * Forced rows: rows with a non-finite component or an fp32 squared norm outside [1e-30, 1e30]
 * (K1's forced candidates) are kept out of training and of the inverted lists; every search
 * re-ranks them exactly besides the ADC candidates.  More than 1024 such rows: the build fails
 * with STB_ERR_STATE.  With nprobe = nlist and rerank >= the codes scanned (v2: <= 1024 codes;
 * v1: <= 4096), every row is re-ranked and the hits equal stb_search's.
 * stb_ivfpq_search: nprobe is clamped to [1, min(nlist, 1024)], rerank to [top_k, 4096];
 * top_k > 4096 is STB_ERR_ARG.  *out_scanned = codes scanned (forced rows not counted).  It runs the
 * fused search (v2, stb_ivfpq_search_dev's) when rerank <= 1024 and top_k <= 1024, and the
 * multi-launch search (v1) when rerank or top_k exceeds 1024.  v2's funnel: 32-code chunks dealt over 32
 * CTAs then 16 warps, 64 best per warp, 64 best per CTA, then the `rerank` best of those 2048; it
 * returns the `rerank` best ADC scores exactly when no warp and no CTA holds more than 64 of them.
 * v1: 64 best per warp over enough warps to hold min(rerank, codes scanned) candidates. */
typedef struct stb_ivfpq stb_ivfpq;
int stb_ivfpq_build(stb_ctx *ctx, const stb_corpus *corpus, uint32_t nlist, uint32_t train_rows,
                    uint32_t iters, stb_ivfpq **out);
int stb_ivfpq_destroy(stb_ivfpq *index);
/* Index the rows appended to the index's corpus since the build or the last extend:
 * rows [indexed, corpus rows).  Centroids and codebooks are not retrained.
 * *out_added (may be NULL) = rows added, 0 when there were none.
 * Synchronous: searches enqueued before the call see the old index, later ones the new.
 * On any error the index is unchanged and still usable.
 * STB_ERR_STATE: the corpus was cleared since the index last read it,
 * or the forced rows would exceed 1024.
 * Each new row gets the list and code the build would give it; within a list the new rows follow the
 * old entries in ascending row order (a built index's lists are in ascending row order too), so two
 * extends give the lists one extend of both parts gives.  Cost: the new rows' assignment and encoding
 * plus one copy of the lists (36 B per row); extra memory while it runs: that copy and 48 B per new row. */
int stb_ivfpq_extend(stb_ivfpq *index, uint64_t *out_added);
/* Replace and delete rows of the index's corpus and keep the index current, without retraining.
 * stb_ivfpq_update / stb_ivfpq_remove apply stb_corpus_update / stb_corpus_remove to the index's corpus:
 * the arguments, their validation, the error codes, the chunking, the maintained q8 and 16-bit copies, the
 * new epoch, the reset of the tier statistics and the end of a co-scan series are exactly those calls'.
 * Instead of refusing a corpus with a live index they refuse (STB_ERR_STATE, nothing written):
 *  - another live index on the same corpus;
 *  - a corpus cleared since the index last read it (as stb_ivfpq_extend);
 *  - a call that would leave more than 1024 forced rows.
 * After success:
 *  - Centroids and codebooks are the same bits: nothing is retrained.
 *  - A removed indexed row leaves its list or the forced list; every entry behind it is renumbered (row
 *    minus the removed rows below it).  stb_ivfpq_stats' rows drops by the removed rows that were indexed.
 *  - A replaced indexed row gets the list and code the build would give its new value (a copy of another
 *    indexed row: that row's list and code, bit for bit); it may move between a list and the forced list.
 *  - Every list and the forced list stay in ascending row order.  The index is therefore a function of the
 *    quantisers and the current rows: what the build's add phase with the same quantisers makes of rows
 *    [0, indexed).  Any sequence of extend, update and remove calls that reaches the same rows reaches the
 *    same index.
 *  - Rows appended but not yet extended stay outside the index: updating them changes only the corpus,
 *    removing them shortens that tail, and the next stb_ivfpq_extend indexes exactly the rows after the
 *    indexed prefix.
 *  - The index records the corpus's new epoch: extend and the searches keep working.
 * Atomicity: on STB_ERR_ARG, STB_ERR_RANGE, STB_ERR_STATE or STB_ERR_NOMEM the corpus (rows and copies) and
 * the index are byte for byte unchanged and the index stays usable.  Every buffer the index needs is
 * allocated, and the replaced rows are encoded and the forced rows counted, before the corpus is written.
 * The new rows are encoded from the corpus's staging buffer: an update of at most 262144 rows is uploaded
 * once, a larger one twice (once to encode and count, once to write).
 * Synchronous: searches enqueued before the call see the old rows and index, later ones the new.
 * Cost, besides the corpus call's: the assignment and encoding of the replaced indexed rows and one pass
 * over the lists (read and write, 36 B per entry).  Extra device memory while it runs: one copy of the lists,
 * 48 B per replaced row, a bitmap of the indexed rows and 8 B per listed entry. */
int stb_ivfpq_update(stb_ivfpq *index, const uint64_t *idx, const float *rows, uint64_t n);
int stb_ivfpq_remove(stb_ivfpq *index, const uint64_t *ranges, uint32_t n_ranges);
int stb_ivfpq_stats(const stb_ivfpq *index, uint64_t *rows, uint32_t *nlist, uint32_t *max_list,
                    uint64_t *index_bytes);
/* Save an index to a file and load it onto its corpus in another process, without retraining or re-encoding.
 * File format, version 1, little-endian.  A 216-byte header, then the six sections back to back, in order:
 *     0  char     magic[8] = "STBIVFPQ"
 *     8  u32      version = 1, d = 256, pq_m = 32, pq_ksub = 256, pq_dsub = 8, nlist
 *    32  u64      n (rows indexed), n_listed, n_forced, rows_digest
 *    64  6 x {u64 offset, u64 bytes, u64 checksum}, one per section
 *   208  u64      header_checksum = digest(the header's bytes [0, 208))
 *   216  centroids f32[nlist][256], codebooks f32[32][256][8], list_off u32[nlist + 1], order u32[n_listed],
 *        codes u8[n_listed][32], forced u32[n_forced] -- exactly stb_debug_ivfpq_export's arrays.  Section k
 *        starts where section k - 1 ends (the first at 216) and the file ends with the last one.
 *   The checksum of a section is digest(its bytes); rows_digest = digest(the corpus rows [0, n) as stored: n x
 *   256 f32, 1 KiB per row).  Nothing else is stored: no query scratch, batch state or tuning value.
 * The digest of a byte string s of L bytes (all arithmetic mod 2^64):
 *     mix(z):  z ^= z >> 30; z *= 0xBF58476D1CE4E5B9; z ^= z >> 27; z *= 0x94D049BB133111EB; z ^= z >> 31
 *     s is zero-padded to whole 1 KiB blocks; w(b, i) = little-endian u64 at byte 1024 b + 8 i (i < 128)
 *     h(b)     = sum over i of mix(w(b, i) ^ (i + 1) * 0x9E3779B97F4A7C15)
 *     digest   = sum over b of mix(h(b) ^ (b + 1) * 0xC2B2AE3D27D4EB4F)  +  mix(L ^ 0x165667B19E3779F9)
 *   It is order-sensitive (a word's position and its block's enter its term) and parallel over blocks: the GPU
 *   computes every section checksum, after the section reached HBM, and rows_digest, a block per row.  It
 *   detects a wrong corpus or accidental damage; it is NOT cryptographic and does not authenticate a file.
 * stb_ivfpq_save: synchronous (waits for the index's enqueued work); the index is not changed.  Writes the
 *   file through a 32 MiB pinned buffer (never a second host copy of the index) to a new file beside `path`
 *   (path + ".tmp.<pid>.<k>", the next k while that name exists), fsyncs it and renames it over `path`, so a
 *   reader sees the old file or the whole new one.  On any failure `path` is untouched and the temporary file removed.  The same index gives the same
 *   bytes.  STB_ERR_ARG: a NULL argument, or a path that cannot be written.  STB_ERR_STATE: the corpus was
 *   cleared since the index last read it (as stb_ivfpq_extend).
 * stb_ivfpq_load: a new index on `corpus` equal to the saved one: stb_debug_ivfpq_export and stb_ivfpq_stats
 *   return the saved values, every search, extend, update and remove behaves as on the original, bit for bit.
 *   The corpus may have another row_base (hits carry this corpus's global rows) and rows appended after
 *   [0, n): they stay outside the index until stb_ivfpq_extend.  The file is untrusted input; in order:
 *    1. corpus of another context: STB_ERR_ARG; a host-rows corpus: STB_ERR_STATE (as stb_ivfpq_build);
 *    2. before anything is allocated, STB_ERR_ARG with a message naming the field: the file cannot be read or is
 *       shorter than the header; magic, version, shape constants; header_checksum; 1 <= nlist <= 8192;
 *       n_forced <= 1024; n_listed + n_forced == n < 2^32; each section's offset and bytes as the counts give
 *       them, and the file ends where the last section ends.  Then a corpus with fewer than n rows: STB_ERR_STATE;
 *    3. the sections are read through the pinned buffer into the index's own buffers and their checksums
 *       computed on the GPU: a mismatch is STB_ERR_ARG;
 *    4. one GPU pass over the lists, STB_ERR_ARG unless list_off[0] == 0, list_off never decreases and
 *       list_off[nlist] == n_listed; every order entry is < n and each list strictly ascending; forced is
 *       strictly ascending and < n; no row appears twice across order and forced (a bitmap of n bits) -- with
 *       the counts, every row of [0, n) appears exactly once;
 *    5. one GPU pass over the corpus rows [0, n): their digest must equal rows_digest (else STB_ERR_STATE), and
 *       forced must be exactly the rows that cannot be normalised (the build's rule; else STB_ERR_ARG).
 *   Only then is the index installed (query scratch, corpus epoch, the corpus's live-index count).  On every
 *   refusal nothing stays allocated, the corpus is not counted as indexed (stb_corpus_update still works), and
 *   the context stays usable.  Checks 2 and 4 run before any kernel reads list_off, order or forced as indices.
 *   The codes and list assignments are not re-derived (that is the build's add phase, which loading skips).
 *   Guarantees: accidental damage is caught by the checksums and a different corpus by the digest; a crafted
 *   file with consistent checksums can at worst lower recall -- every kernel stays in bounds and every returned
 *   distance is still the exact canonical distance of its row. */
int stb_ivfpq_save(const stb_ivfpq *index, const char *path);
int stb_ivfpq_load(stb_ctx *ctx, const stb_corpus *corpus, const char *path, stb_ivfpq **out);
int stb_ivfpq_search(stb_ivfpq *index, const float *q, uint32_t nprobe, uint32_t top_k,
                     uint32_t rerank, stb_hit *out_hits, uint32_t *out_n, uint64_t *out_scanned);
/* Asynchronous device-resident form (query, hits and status stay in HBM, nothing synchronises): the
 * sharded index is one of these per rank, an all-gather of the k hits and stb_hits_merge_dev.
 * out_hits_dev: top_k entries (unused tail +inf / UINT64_MAX); out_status_dev[0] = hits, [1] = codes
 * scanned.  top_k must be 1..1024; rerank is capped at 1024. */
int stb_ivfpq_search_dev(stb_ivfpq *index, const float *q_dev, uint32_t nprobe, uint32_t top_k,
                         uint32_t rerank, stb_hit *out_hits_dev, uint32_t *out_status_dev);
/* Batched search: nq queries (q / q_dev: nq x 256 f32) in one pass over the GPU.
 * out_hits: nq x top_k, entry i*top_k.. belongs to query i, unused tail (+inf, UINT64_MAX).
 * Host form: out_n[i] = hits of query i, out_scanned[i] (may be NULL) = codes scanned for it; any nq,
 * in chunks of 4096 queries with one synchronisation each; top_k == 0 sets every count to 0.
 * Device form: asynchronous on the context's stream, never synchronises; out_status_dev[2i] = hits,
 * [2i+1] = codes scanned; nq <= 4096 (more is STB_ERR_ARG).  Both: nq == 0 is a no-op; top_k must be
 * 1..1024 (else STB_ERR_ARG); nprobe is clamped to [1, min(nlist, 1024)], rerank to [top_k, 1024].
 * Scratch grows on demand (cudaFree/cudaMalloc, which synchronise, on the first call at a larger nq),
 * belongs to the index and is separate from the single-query search's.
 * Each query's answer is independent of the others in the batch and of the chunking:
 *  - coarse scores, probe list (nprobe best by coarse score desc, list id asc) and LUT are bit-identical
 *    to stb_ivfpq_search_dev's for that query, bad queries (zero, NaN / inf components, huge or tiny
 *    scales) included;
 *  - ADC score = coarse[list] + LUT[0][c0] + ... + LUT[31][c31], summed in that order in fp32;
 *  - candidates: exactly the `rerank` best scanned codes by (ADC score desc, code position asc); a code
 *    whose score is NaN or -inf is none.  Each of the 64 scan warps of a query keeps its 64 best codes;
 *    when one of them dropped a code that would have been a candidate, the query is answered by an exact
 *    slower route (a radix select over all its codes), never approximately;
 *  - hits: the candidates' rows and the forced rows re-ranked with the canonical distance, as above.
 * So with nprobe = nlist and rerank >= the codes scanned the hits equal stb_search's, and whenever v2's
 * funnel returns the `rerank` best ADC scores the hits equal stb_ivfpq_search_dev's. */
int stb_ivfpq_search_batch(stb_ivfpq *index, const float *q, uint32_t nq, uint32_t nprobe, uint32_t top_k,
                           uint32_t rerank, stb_hit *out_hits, uint32_t *out_n, uint64_t *out_scanned);
int stb_ivfpq_search_batch_dev(stb_ivfpq *index, const float *q_dev, uint32_t nq, uint32_t nprobe,
                               uint32_t top_k, uint32_t rerank, stb_hit *out_hits_dev, uint32_t *out_status_dev);
/* Filtered batched search: the query of Store::search_line_embeddings (src/workspace/store.rs:481-546)
 * on the index -- only rows of a subset, an optional distance cap, top_k always caps
 * (STB_MODE_STORE_QUERY semantics).  Shapes and argument rules are stb_ivfpq_search_batch's host form:
 * nq == 0 is a no-op; top_k == 0 sets every count to 0; top_k > 1024 is STB_ERR_ARG; nprobe is clamped
 * to [1, min(nlist, 1024)], rerank to [top_k, 1024]; any nq, in chunks of 4096 with one synchronisation
 * each; the scratch belongs to the index and grows on demand.
 *  - Filter: row_ranges holds n_ranges half-open [begin, end) pairs of GLOBAL rows, ascending and disjoint
 *    as in stb_search (otherwise STB_ERR_RANGE before any launch, nothing written), clipped to the indexed
 *    rows [row_base, row_base + rows) of stb_ivfpq_stats: rows appended but not yet extended into the index
 *    are never returned.  row_ranges == NULL: every indexed row is eligible.  Non-NULL with n_ranges == 0:
 *    the empty subset, every count 0 (store.rs:489).  n_ranges > 0 with NULL: STB_ERR_ARG.
 *  - Eligible: a listed code whose row (row_base + order[i]) lies in a range; a forced row under the same rule.
 *  - Probe list: the lists in the unfiltered order (coarse score desc, list id asc), skipping every list
 *    with no eligible code; the first min(nprobe, E) of them are probed, E = lists with an eligible code.
 *    Coarse scores and LUT are bit-identical to stb_ivfpq_search_batch's for that query.
 *  - Candidates: exactly the `rerank` best eligible probed codes by (ADC score desc, code position asc);
 *    a code whose score is NaN or -inf is none; a scan warp that overflows takes the batch's exact slow route.
 *  - Hits: the candidates' rows and the eligible forced rows, canonical distance; a hit needs
 *    distance < max_distance (strict; min(max_distance, 100) as stb_search) when has_max, else < 100;
 *    ordered by (distance, row); at most top_k.
 *  - Counts: out_n[i] = hits of query i; out_scanned[i] (may be NULL) = eligible codes in its probed lists.
 *    out_hits: nq x top_k as stb_ivfpq_search_batch's, unused entries (+inf, UINT64_MAX).
 * Cost per call, shared by its queries: a bitmap of the eligible rows (ceil(rows / 32) words) and one
 * read of order[] (4 B per listed row) that counts each list's eligible codes.
 * What follows:
 *  - nprobe = nlist and rerank >= the eligible codes: the hits equal stb_search(..., has_max, max_distance,
 *    STB_MODE_STORE_QUERY, row_ranges, n_ranges, ...) bit for bit;
 *  - a query that normalises in fp32 (finite components, fp32 squared norm in [1e-30, 1e30]), no threshold,
 *    nprobe >= top_k: min(top_k, eligible indexed rows) hits, as many as the exact scan (the canonical
 *    distance is never NaN nor above 2, so every re-ranked row is a hit, and each probed list holds an
 *    eligible code);
 *  - row_ranges == NULL, no threshold and no empty list among the nprobe best: the hits equal
 *    stb_ivfpq_search_batch's.
 * stb_debug_ivfpq_batch_last describes a filtered call too: info[1] is the clamped nprobe, probe[] the lists
 * actually probed followed by 0xffffffff. */
int stb_ivfpq_search_filtered(stb_ivfpq *index, const float *q, uint32_t nq, uint32_t nprobe, uint32_t top_k,
                              uint32_t rerank, int has_max, double max_distance,
                              const uint64_t *row_ranges, uint32_t n_ranges,
                              stb_hit *out_hits, uint32_t *out_n, uint64_t *out_scanned);
/* Filtered batched search over many subsets in one call: a batch of store queries (a server's or an agent
 * host's) that name different folders, each distinct subset passed once.
 *  - Subsets: subset_offsets has n_subsets + 1 entries, subset_offsets[0] = 0, never decreasing; subset s is
 *    row_ranges[2*subset_offsets[s] .. 2*subset_offsets[s+1]), GLOBAL [begin, end) pairs as stb_search takes
 *    them, clipped to the indexed rows as stb_ivfpq_search_filtered clips them.  A subset with no ranges, or
 *    none left after clipping, is the empty subset.
 *  - Queries: q is nq x 256 f32 (host); query i searches subset subset_of[i] (< n_subsets).
 *  - Contract: for every query i, out_hits[i*top_k ..], out_n[i] and out_scanned[i] equal, bit for bit, what
 *      stb_ivfpq_search_filtered(index, q_i, 1, nprobe, top_k, rerank, has_max, max_distance,
 *                                <ranges of subset subset_of[i]>, <their count>, ...)
 *    returns (a batched query's answer depends neither on the other queries nor on the launches).
 *  - Argument rules are stb_ivfpq_search_filtered's: nq == 0 is a no-op; top_k == 0 sets every count to 0;
 *    top_k > 1024 is STB_ERR_ARG; nprobe is clamped to [1, min(nlist, 1024)], rerank to [top_k, 1024];
 *    out_scanned may be NULL.  A query of an empty subset gets 0 hits and 0 scanned and takes no part in
 *    any launch.
 *  - Refusals, all before anything is written or launched: STB_ERR_ARG for a NULL pointer that is needed
 *    (row_ranges may be NULL when subset_offsets[n_subsets] == 0), subset_offsets[0] != 0, decreasing
 *    offsets, a subset of more than 2^32 - 1 ranges, or subset_of[i] >= n_subsets; STB_ERR_RANGE when any
 *    subset holds ranges stb_search refuses -- every subset is validated, also those no query names.
 *  - Launches: the queries in caller order, at most 4096 per launch and no more distinct subsets than
 *    STB_IVFPQ_SUBSET_SCRATCH holds (each takes an eligible-row bitmap of ceil(rows / 32) words and nlist
 *    counts; a launch holds at least one query).  Each launch: one bitmap launch and one count launch for
 *    all its subsets, the four batched kernels, one synchronisation.  The bitmap and count launches are
 *    skipped when the previous launch of the same call named exactly the same subsets, in the same order of
 *    first appearance: the scratch still holds their bitmaps and counts.  The scratch belongs to the index
 *    and grows on demand.
 * stb_debug_ivfpq_batch_last describes the call's last launch: slot j is the j-th query of that launch
 * (in caller order, queries of empty subsets skipped). */
int stb_ivfpq_search_subsets(stb_ivfpq *index, const float *q, uint32_t nq, uint32_t nprobe, uint32_t top_k,
                             uint32_t rerank, int has_max, double max_distance,
                             uint32_t n_subsets, const uint64_t *subset_offsets, const uint64_t *row_ranges,
                             const uint32_t *subset_of, stb_hit *out_hits, uint32_t *out_n, uint64_t *out_scanned);
/* Threshold mode of search_documents (src/search/mod.rs:88-89,115-119) on the index, for a batch: every row of
 * the query's probed lists (and every forced row) under max_distance, with no top_k cap.
 *  - Probe: for query i the coarse scores, probe list and LUT are bit for bit stb_ivfpq_search_batch's; nprobe is
 *    clamped to [1, min(nlist, 1024)].  stb_debug_ivfpq_batch_last describes the call's last launch, with
 *    info = {nq, nprobe, 0, 0}.
 *  - Cutoff: t = RD_f32((1 - max_distance) - slack), computed in f64 and rounded toward -inf.
 *  - Candidates: when t = -inf (max_distance or slack +inf), every code of the probed lists; otherwise every such
 *    code whose ADC score s (stb_ivfpq_search_batch's fp32 sum, in the same order) satisfies s >= t, so a NaN
 *    score is none.  Plus every forced row.
 *  - Hits: the candidate rows whose canonical distance (as on every K5 path) is < max_distance (strict), GLOBAL
 *    rows, each query's ordered by (distance, row).
 *  - Output as stb_search_batch_threshold's: out_offsets has nq + 1 entries, out_offsets[0] = 0, the hits of all
 *    queries concatenated in query order; if out_offsets[nq] > cap the first cap hits are written, every offset
 *    is still written and the call returns STB_ERR_CAPACITY.  out_hits may be NULL only when cap == 0.
 *  - Counts (either pointer may be NULL): out_scanned[i] = codes in the probed lists, as stb_ivfpq_search_batch
 *    reports them; out_reranked[i] = candidate codes plus forced rows, the rows whose f32 row was read.
 *  - Arguments: nq == 0 is a no-op; a NULL index, q or out_offsets is STB_ERR_ARG, as is a NaN or negative slack.
 *    A max_distance that is NaN or <= 0 sets every offset and count to 0 and launches nothing.
 *  - Launches: queries in chunks of at most 4096 (probe stage, one pass that counts each query's candidates per
 *    block of 16384 probed codes, one synchronisation), then launches of at most STB_IVFPQ_THRESHOLD_KEYS
 *    candidate keys (or one block, if a block alone holds more) that emit the keys and finish them as
 *    stb_search_batch_threshold does (sort by row, canonical re-score, stable sort by distance).  A query with
 *    more candidates than a launch holds is split at block boundaries and its pieces merged into (distance, row)
 *    order, so a query's answer depends neither on the other queries, nor on the chunking, nor on the budget.
 *    Scratch belongs to the index and grows on demand (the keys of a launch: 32 B each, plus the sorts').
 * What follows:
 *  - every returned hit is a threshold hit of stb_search for that query, with the same distance bits: only the
 *    recall is approximate;
 *  - with nprobe >= nlist (so nlist <= 1024) and slack = +inf every indexed row is re-scored, so the hits are
 *    the canonical threshold answer over the indexed rows, forced rows included; for a query with finite
 *    components (zero and huge ones included) they equal, bit for bit, those of
 *      stb_search(ctx, corpus, q_i, 0, 1, max_distance, STB_MODE_SEARCH_DOCUMENTS, NULL, 0, ...)
 *    and of stb_search_batch_threshold (for a query with a NaN or infinite component every canonical distance
 *    is 0, and every indexed row is a hit);
 *  - the hit set is monotone: raising nprobe (the probe list is a prefix of the coarse order) or slack never
 *    removes a hit. */
#define STB_IVFPQ_THRESHOLD_KEYS (1ull << 24)   /* candidate keys one launch holds (128 MiB) */
int stb_ivfpq_search_threshold(stb_ivfpq *index, const float *q, uint32_t nq, uint32_t nprobe,
                               double max_distance, double slack,
                               stb_hit *out_hits, uint64_t cap, uint64_t *out_offsets,
                               uint64_t *out_scanned, uint64_t *out_reranked);

/* Host-buffer form of the fused multi-GPU search (the call a sharded host makes per query):
 * pinned H2D of the query, ONE kernel (scan + NVLink exchange + merge), D2H of the merged
 * hits, stream sync.  *out_complete = 0 means some rank could not prove its shard result
 * (all ranks see the same flag): run stb_search per shard + stb_hits_merge instead. */
int stb_search_xchg(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t top_k,
                    stb_xchg *x, stb_hit *out_hits, uint32_t *out_n, int *out_complete);

/* Many independent single queries, one synchronisation (a host that has several queries in hand:
 * an agent's tool calls, a batch of CLI invocations).  q: nq x 256 f32 (host); out_hits: nq x top_k
 * (entry i*top_k.. of query i), out_n: nq counts.  Each query is its own scan (use stb_search_batch
 * when nq is in the hundreds: one pass over the corpus for all of them); the kernels are enqueued
 * back to back, so every tail overlaps the next scan, and hits are written straight to pinned host
 * memory.  x == NULL: results are exactly stb_search's (an unproven query is re-run through it).
 * x != NULL: the sharded form of stb_search_xchg -- out_complete[i] = 0 marks a query some rank could
 * not prove (every rank sees the same flags).  out_complete may be NULL when x is NULL.
 * Validation state: the x == NULL form is covered by the GPU suite; the x != NULL form is the same kernel
 * stb_search_xchg launches, enqueued nq times, but has not yet run on a multi-GPU box. */
int stb_search_many(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t nq, uint32_t top_k,
                    stb_xchg *x, stb_hit *out_hits, uint32_t *out_n, uint8_t *out_complete);

/* ---- K4: merge per-shard hit lists -----------------------------------------------
 * The final sort_by + take of src/search/mod.rs:107-119 applied across row
 * shards: `lists_dev` holds n_lists x per_list hits (e.g. the all-gathered
 * per-GPU top-k; padding entries are (+inf, UINT64_MAX)); writes the top_k best by
 * (distance, row) to out_dev.  An entry whose row is UINT64_MAX or whose distance
 * is NaN is padding and dropped wherever it sits; +inf on a real row is kept.
 * -0.0 and +0.0 tie (then ordered by row) and keep their bits.  out_dev gets
 * exactly top_k entries, the tail padded with (+inf, UINT64_MAX).
 * n_lists*per_list <= 4096.  Asynchronous on the context's stream. */
int stb_hits_merge_dev(stb_ctx *ctx, const stb_hit *lists_dev, uint32_t n_lists,
                       uint32_t per_list, uint32_t top_k, stb_hit *out_dev);
/* Batched form for sharded K2: lists_dev[n_lists][nq][per_list] (e.g. the all-gathered
 * per-rank results of stb_search_batch_dev) -> out_dev[nq][top_k]; n_lists*per_list <= 2048. */
int stb_hits_merge_batch_dev(stb_ctx *ctx, const stb_hit *lists_dev, uint32_t n_lists,
                             uint32_t nq, uint32_t per_list, uint32_t top_k, stb_hit *out_dev);
/* Host-buffer convenience wrapper (copies in, merges on the GPU, copies out): out
 * gets the *out_n <= top_k valid hits, without the padding tail. */
int stb_hits_merge(stb_ctx *ctx, const stb_hit *lists, uint32_t n_lists,
                   uint32_t per_list, uint32_t top_k, stb_hit *out,
                   uint32_t *out_n);

/* ---- ids -------------------------------------------------------------------------
 * fnv1a_hash (src/workspace/store.rs:651-661); DocMeta::id (:75-80) is
 * stb_fnv1a64(path); LineEmbedding::id (:82-89) is stb_line_id. Pure host code. */
uint64_t stb_fnv1a64(const uint8_t *bytes, uint64_t len);
uint64_t stb_line_id(const uint8_t *path, uint64_t path_len, int32_t line_number);
/* stb_line_id for n_rows (path index, line_number) int32 pairs at once (rebuilding a store's
 * id map): paths = one byte blob + n_paths+1 offsets.  STB_ERR_RANGE on a bad path index. */
int stb_line_ids(const uint8_t *path_bytes, const uint64_t *path_offsets, uint32_t n_paths,
                 const int32_t *rows, uint64_t n_rows, uint64_t *out_ids);

/* ---- introspection (bench / tests) -------------------------------------------------
 * Counters since context creation: kernels launched by this library on the
 * context, and how many searches needed the fallback pass. */
int stb_ctx_counters(const stb_ctx *ctx, uint64_t *kernel_launches,
                     uint64_t *fallback_searches);
/* Consistency check of K1's dynamic tile schedule (synchronises): the device-side ticket counter
 * must equal the value the host booked over all launches so far; STB_ERR_STATE otherwise. */
int stb_debug_ticket_check(stb_ctx *ctx, uint64_t *device_value, uint64_t *host_value);
/* Rows the q8 tier's top-k prefilter passed on to the int8 codes, summed over the
 * top-k launches since the last reset (reset != 0 zeroes the counter after reading it).
 * Synchronises the context's stream. */
int stb_debug_q4_refined(stb_ctx *ctx, int reset, uint64_t *refined);
/* The tile offsets at which K1's last n (<= 8) top-k launches on the context started their pass,
 * oldest first; 0xffffffff for a launch that did not co-scan.  A series of stb_search_topk_dev
 * calls on one corpus co-scans: each query after the first starts where its predecessor is
 * reading.  Synchronises the context's stream. */
int stb_debug_coscan_offsets(stb_ctx *ctx, uint32_t n, uint32_t *out);
/* Test hooks for K1's pairs: a q8 top-k query of an asynchronous series (stb_search_topk_dev, stb_search_many
 * without an exchange) that follows a query on the same corpus joins its running scan, which scores both
 * queries from one read of each plane tile.  stb_debug_pair_joins: for the last n (<= 8) top-k launches on
 * the context, oldest first, the tile at which each joined its host; -1 for a launch that was not such a
 * guest, -2 for a guest whose join was refused (it scanned alone).  Synchronises the context's stream.
 * stb_debug_pair_floor: later joins wait until their host has drawn v_floor tile tickets (0: no wait). */
int stb_debug_pair_joins(stb_ctx *ctx, uint32_t n, int64_t *out);
int stb_debug_pair_floor(stb_ctx *ctx, uint64_t v_floor);
/* Test hook for the candidate copies: copies entries [first, first+n) of one copy to `out` and sets
 * *covered (may be NULL) to the rows the copy covers (0: not built).  which = STB_COPY_Q8_CODES (256 B per
 * row), _Q8_SCALES (f32 per row), _Q8_PLANE (nibble plane, 128 B per row), _Q8_SR ({s, rho}, 2 x f32 per
 * row): entries are rows < covered; STB_COPY_H16_TILES: entries are whole 256-row tiles of the 16-bit shadow
 * (131072 B each), tiles < ceil(covered / 256).  Beyond that: STB_ERR_RANGE.  Synchronises the stream. */
#define STB_COPY_Q8_CODES 0
#define STB_COPY_Q8_SCALES 1
#define STB_COPY_Q8_PLANE 2
#define STB_COPY_Q8_SR 3
#define STB_COPY_H16_TILES 4
int stb_debug_corpus_copy(const stb_corpus *corpus, int which, uint64_t first, uint64_t n, void *out,
                          uint64_t *covered);
/* Test hooks for K1's per-row score contracts (DESIGN.md section 5).  Both run the production scan code on
 * query q (256 f32, host) over the corpus's rows or over row_ranges (global [begin, end) pairs, as
 * stb_search takes them; NULL with n_ranges = 0: every row), ignore STB_SCAN_TIER and synchronise the stream.
 * Outputs are per LOCAL row, cap >= the corpus's rows; a row outside the ranges keeps score NaN and count 0.
 * stb_debug_scan_scores: tier 0 / 1 / 2 picks the pass (f32 rows / 16-bit shadow / int8 codes, the order of
 *   stb_corpus_tier_stats); scores[row] is the score the pass gave the row and seen[row] how many times it was scored.
 *   hist (may be NULL; f32 and q8 only) receives the 4096-bin histogram of the large-k route's pass.
 * stb_debug_q4_scan: the q8 tier's prefiltered top-k scan for top_k (1..16) with threshold words of its own;
 *   per row its 4-bit bound u4 and the threshold T it was tested against, refined[row] = times it was scored
 *   from the int8 codes and, for such rows, that score u8 and the lower bound l8 it published; words receives
 *   the top_k final threshold words (tag 1 in the high half).  pin != 0 holds T at -inf: every row is refined.
 * STB_ERR_ARG: a null pointer or cap too small; STB_ERR_STATE: the tier's copy is not built or unusable. */
int stb_debug_scan_scores(stb_ctx *ctx, const stb_corpus *corpus, int tier, const float *q,
                          const uint64_t *row_ranges, uint32_t n_ranges, uint64_t cap, float *scores,
                          uint32_t *seen, uint32_t *hist);
int stb_debug_q4_scan(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t top_k,
                      const uint64_t *row_ranges, uint32_t n_ranges, int pin, uint64_t cap, float *u4,
                      float *t, uint32_t *refined, float *u8, float *l8, uint64_t *words);
/* Test hook for K2: shadow build + wgmma GEMM on host inputs; out_full receives the
 * approximate cosine matrix [ceil(nq/128)*128][ceil(n/256)*256] (f32), out_submax (may be
 * NULL) the per-32-row maxima [ceil(nq/128)][ceil(n/256)*8][128]. */
int stb_debug_batch_gemm(stb_ctx *ctx, const float *q, uint32_t nq, const float *rows,
                         uint64_t n, float *out_full, float *out_submax);
/* Test hook for K2's route 7: stb_search_batch run on the q8 copy whatever the state of the 16-bit shadow
 * (it builds no shadow and leaves an existing one untouched), with the same outputs and the same answer by
 * stb_search for every query the route leaves unproven. */
int stb_debug_batch_q8(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t nq, uint32_t top_k,
                       stb_hit *out_hits, uint32_t *out_n);
/* Test hook for K2's q8 routes: while on != 0, every K2 search call on ctx (stb_search_batch, its _dev form and the
 * filtered, subsets and threshold calls) behaves as if the 16-bit shadow did not fit in HBM, so it takes its q8
 * route (7, 8, 9 or 10).  It builds no shadow and leaves a built shadow's bytes as they are.  Off by default. */
int stb_debug_batch_no_shadow(stb_ctx *ctx, int on);
/* Test hook for K2's route 7: the query quantisation and the integer GEMM over the corpus's q8 copy (built or
 * extended first).  q16 receives [nq][256] the 16-bit query components, dot [nq][n] the int32 products with
 * the int8 codes, u and l [nq][n] the upper and lower bounds of the exact cosine computed from them. */
int stb_debug_batch_q8_gemm(stb_ctx *ctx, const stb_corpus *corpus, const float *q, uint32_t nq, int16_t *q16,
                            int32_t *dot, float *u, float *l);
/* Test hook for K5: synchronous copies of a built index into host buffers; a NULL pointer skips
 * that array.  centroids [nlist][256] f32, codebooks [32][256][8] f32, list_off [nlist+1],
 * order [m] (local row of each code), codes [m][32] u8, forced [n - m] (local rows outside the
 * lists, ascending), where m = list_off[nlist]. */
int stb_debug_ivfpq_export(const stb_ivfpq *index, float *centroids, float *codebooks,
                           uint32_t *list_off, uint32_t *order, uint8_t *codes, uint32_t *forced);
/* Test hook for K5: describes the most recent batched search on the index (either form; the last
 * chunk of a chunked host call), synchronising the stream.  info = {nq, nprobe, top_k, rerank} after
 * clamping; for query i, coarse receives [nlist] scores, probe [nprobe] list ids in probe order and
 * lut [32][256].  Any pointer may be NULL.  STB_ERR_STATE before any batched search, STB_ERR_ARG for
 * i >= nq. */
int stb_debug_ivfpq_batch_last(const stb_ivfpq *index, uint32_t i, uint32_t info[4], float *coarse,
                               uint32_t *probe, float *lut);
/* Test hook for K5's threshold search: candidate keys per launch for this index (0 = STB_IVFPQ_THRESHOLD_KEYS;
 * more than that is STB_ERR_ARG).  Lowering it splits queries between launches without changing any answer. */
int stb_debug_ivfpq_threshold_keys(stb_ivfpq *index, uint64_t keys);
/* Test hook for K5's stb_ivfpq_load: host milliseconds of the load that made this index, ms[0] reading the file
 * and uploading its sections, ms[1] the GPU verification (checksums, lists, rows); both 0 for a built index. */
int stb_debug_ivfpq_load_ms(const stb_ivfpq *index, double ms[2]);
/* Test hook for K2: describes the most recent stb_search_batch_dev, stb_search_batch_filtered,
 * stb_search_batch_subsets or stb_search_batch_threshold on ctx (synchronises the stream).  info = {route, nq, a,
 * b, n_seg, seg_cap}; route 1 = v1, 2 = v2, 3 = filtered v2, 4 = a filtered call that launched nothing on the
 * tensor cores (K1 answered it, or nothing could be returned), 5 = threshold mode, 6 = one filter per query
 * group, 7 = v2 on the q8 copy and the int8 tensor cores (the shadow did not fit, or stb_debug_batch_q8),
 * 8-10 = below, 0 = none yet.  Slots 2-3 (a, b):
 *   routes 1-4, 7: n_sample, stride -- v2's sampled tiles (0, stride, 2*stride, ...; after route 3 they count
 *               listed tiles, the tiles holding an eligible row, in ascending order); 0 after routes 1 and 4
 *               and after a route 7 call whose batch did not fit its plan (n_seg and seg_cap are 0 then too);
 *   route 5:    the queries re-emitted by the second tensor pass, and the queries stb_search answered;
 *   route 6:    the groups that ran on the tensor cores, and the queries stb_search answered.  After a route 6
 *               call that ran the tensor passes, thr and cand_cnt are in caller query order; a query those
 *               passes did not take has threshold +inf and zero counts.
 *   routes 8-10: routes 3, 6 and 5 on the q8 copy (the shadow did not fit, or stb_debug_batch_no_shadow), with
 *               the words of those routes; route 9 reports n_seg = seg_cap = 0.  A filtered call that launched
 *               nothing on the tensor cores records route 4 whatever the reason: neither plan fits, the shadow fits
 *               but its plan does not, its rows cannot be normalised, or the shadow does not fit and then the q8
 *               plan does not fit or the q8 copy cannot be used.  A subsets call whose shadow does not fit records
 *               route 9, with 0 groups when none ran on the tensor cores; a threshold call whose shadow does not
 *               fit records route 10, with n_seg = 0 and every query answered by stb_search when the q8 copy
 *               cannot be used.
 * n_seg and seg_cap are the emitting grid and the first pass's per-(query, CTA) key capacity, 0 after routes 1
 * and 4 and after a route 5 or 10 call that launched nothing.  After routes 2, 3 and a route 5, 7, 8 or 10 call that ran the
 * tensor pass, thr (may be NULL) receives the nq emission thresholds and cand_cnt (may be NULL) the raw
 * first-pass emission counts [nq][n_seg]; a count above seg_cap marks an overflowed segment. */
int stb_debug_batch_last(stb_ctx *ctx, uint32_t info[6], float *thr, uint32_t *cand_cnt);
/* Build parameters of K2 (host-only): element type of the shadow the tensor-core pass runs on
 * (0 = bf16, 1 = fp16) and the bound |approximate - exact cosine| <= eps its selection uses. */
int stb_debug_batch_params(int *shadow_is_f16, double *eps);
/* Route 7's plan (host-only): for a card with sm_count SMs, a corpus of n_rows rows and top_k, plan = {sampled
 * tiles, sample stride, 1 if the batch runs on the route (0: stb_search answers every query)}. */
int stb_debug_batch_q8_plan(uint32_t sm_count, uint64_t n_rows, uint32_t top_k, uint32_t plan[3]);

#ifdef __cplusplus
}
#endif
#endif /* SEMTOOLS_B200_H */

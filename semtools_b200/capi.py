"""ctypes binding of include/semtools_b200.h -- one Python callable per C entry
point, same names, same argument meaning.  Raises StbError on any negative
status; never substitutes a CPU computation."""
from __future__ import annotations

import contextlib
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("STB_LIB_PATH") or os.path.join(_HERE, "lib", "libsemtools_b200.so")

STB_DIM = 256
STB_OK, STB_ERR_ARG, STB_ERR_CUDA, STB_ERR_NOMEM = 0, -1, -2, -3
STB_ERR_RANGE, STB_ERR_CAPACITY, STB_ERR_STATE = -4, -5, -6
STB_MODE_SEARCH_DOCUMENTS, STB_MODE_STORE_QUERY = 0, 1
STB_COPY_Q8_CODES, STB_COPY_Q8_SCALES, STB_COPY_Q8_PLANE, STB_COPY_Q8_SR, STB_COPY_H16_TILES = 0, 1, 2, 3, 4

# every symbol include/semtools_b200.h declares (tests check the .so exports all)
SYMBOLS = [
    "stb_version", "stb_last_error", "stb_device_count", "stb_ctx_create", "stb_ctx_destroy",
    "stb_ctx_sync", "stb_ctx_stream", "stb_table_load", "stb_table_destroy", "stb_corpus_create", "stb_corpus_create_host",
    "stb_corpus_destroy", "stb_corpus_append", "stb_corpus_append_dev", "stb_corpus_clear",
    "stb_corpus_rows", "stb_corpus_data_dev", "stb_corpus_read", "stb_corpus_update", "stb_corpus_remove", "stb_embed", "stb_embed_dev",
    "stb_embed_status", "stb_search",
    "stb_search_topk_dev", "stb_corpus_prepare", "stb_corpus_tier_stats", "stb_corpus_prepare_batch", "stb_search_batch", "stb_search_batch_dev",
    "stb_search_batch_filtered", "stb_search_batch_subsets", "stb_search_batch_threshold",
    "stb_xchg_create", "stb_xchg_destroy", "stb_xchg_local_handle",
    "stb_xchg_connect", "stb_xchg_connect_local", "stb_search_topk_xchg", "stb_search_xchg", "stb_search_many", "stb_xchg_create_batch", "stb_search_batch_xchg_dev", "stb_ivfpq_build",
    "stb_ivfpq_destroy", "stb_ivfpq_extend", "stb_ivfpq_stats", "stb_ivfpq_search", "stb_ivfpq_search_dev", "stb_hits_merge_dev", "stb_hits_merge_batch_dev", "stb_hits_merge", "stb_fnv1a64", "stb_line_id", "stb_line_ids",
    "stb_ctx_counters", "stb_debug_ticket_check", "stb_debug_q4_refined", "stb_debug_coscan_offsets", "stb_debug_pair_joins", "stb_debug_pair_floor", "stb_debug_batch_gemm", "stb_debug_batch_params",
    "stb_debug_batch_last", "stb_debug_batch_q8", "stb_debug_batch_no_shadow", "stb_debug_batch_q8_gemm", "stb_debug_batch_q8_plan", "stb_debug_corpus_copy", "stb_debug_scan_scores", "stb_debug_q4_scan",
    "stb_debug_ivfpq_export",
    "stb_ivfpq_search_batch", "stb_ivfpq_search_batch_dev", "stb_debug_ivfpq_batch_last",
    "stb_ivfpq_search_filtered", "stb_ivfpq_search_subsets", "stb_ivfpq_update", "stb_ivfpq_remove",
    "stb_ivfpq_search_threshold", "stb_debug_ivfpq_threshold_keys", "stb_ivfpq_save", "stb_ivfpq_load", "stb_debug_ivfpq_load_ms",
    "stb_tokenizer_load", "stb_tokenizer_load_ex", "stb_tokenizer_destroy", "stb_tokenizer_gpu_lines", "stb_embed_text", "stb_debug_tokenize",
]
STB_TOKENIZER_PIECE_CAP = 256
STB_TOKENIZER_UTF8 = 1


class StbHit(C.Structure):
    _fields_ = [("distance", C.c_double), ("row", C.c_uint64)]


HIT_DTYPE = np.dtype([("distance", np.float64), ("row", np.uint64)])


class StbError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"stb status {status}: {message}")
        self.status = status


_lib = None
vp = C.c_void_p
u64, u32, i32, f64 = C.c_uint64, C.c_uint32, C.c_int, C.c_double


def lib() -> C.CDLL:
    """Load libsemtools_b200.so; fails loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(scripts/build_lib.sh).  semtools_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    L.stb_version.restype = i32
    L.stb_last_error.restype = C.c_char_p
    L.stb_device_count.restype = i32
    L.stb_ctx_create.argtypes = [i32, vp, C.POINTER(vp)]
    L.stb_ctx_destroy.argtypes = [vp]
    L.stb_ctx_sync.argtypes = [vp]
    L.stb_ctx_stream.argtypes = [vp]
    L.stb_ctx_stream.restype = vp
    L.stb_table_load.argtypes = [vp, vp, u64, u32, vp, u64, vp, u64, i32, C.POINTER(vp)]
    L.stb_table_destroy.argtypes = [vp]
    L.stb_corpus_create.argtypes = [vp, u32, u64, u64, C.POINTER(vp)]
    L.stb_corpus_create_host.argtypes = [vp, u32, u64, u64, C.POINTER(vp)]
    L.stb_corpus_destroy.argtypes = [vp]
    L.stb_corpus_append.argtypes = [vp, vp, u64]
    L.stb_corpus_append_dev.argtypes = [vp, vp, u64]
    L.stb_corpus_clear.argtypes = [vp]
    L.stb_corpus_rows.argtypes = [vp, C.POINTER(u64)]
    L.stb_corpus_data_dev.argtypes = [vp, C.POINTER(vp)]
    L.stb_corpus_read.argtypes = [vp, u64, u64, vp]
    L.stb_corpus_update.argtypes = [vp, vp, vp, u64]
    L.stb_corpus_remove.argtypes = [vp, vp, u32]
    L.stb_debug_corpus_copy.argtypes = [vp, i32, u64, u64, vp, C.POINTER(u64)]
    L.stb_debug_scan_scores.argtypes = [vp, vp, i32, vp, vp, u32, u64, vp, vp, vp]
    L.stb_debug_q4_scan.argtypes = [vp, vp, vp, u32, vp, u32, i32, u64, vp, vp, vp, vp, vp, vp]
    L.stb_embed.argtypes = [vp, vp, vp, vp, u64, vp, vp]
    L.stb_embed_dev.argtypes = [vp, vp, vp, vp, u64, vp]
    L.stb_embed_status.argtypes = [vp]
    L.stb_search.argtypes = [vp, vp, vp, u32, i32, f64, i32, vp, u32, vp, u64, C.POINTER(u64)]
    L.stb_search_topk_dev.argtypes = [vp, vp, vp, u32, vp, vp]
    L.stb_corpus_prepare_batch.argtypes = [vp]
    L.stb_corpus_prepare.argtypes = [vp, i32]
    L.stb_corpus_tier_stats.argtypes = [vp, vp, vp, vp]
    L.stb_search_batch.argtypes = [vp, vp, vp, u32, u32, vp, vp]
    L.stb_search_batch_dev.argtypes = [vp, vp, vp, u32, u32, vp, vp]
    L.stb_search_batch_filtered.argtypes = [vp, vp, vp, u32, u32, i32, f64, vp, u32, vp, vp]
    L.stb_search_batch_subsets.argtypes = [vp, vp, vp, u32, u32, i32, f64, vp, vp, vp, vp]
    L.stb_search_batch_threshold.argtypes = [vp, vp, vp, u32, f64, vp, u64, vp]
    L.stb_xchg_create.argtypes = [vp, u32, u32, u32, C.POINTER(vp)]
    L.stb_xchg_destroy.argtypes = [vp]
    L.stb_xchg_local_handle.argtypes = [vp, vp]
    L.stb_xchg_connect.argtypes = [vp, vp]
    L.stb_xchg_connect_local.argtypes = [vp, C.POINTER(vp)]
    L.stb_search_topk_xchg.argtypes = [vp, vp, vp, u32, vp, vp, vp]
    L.stb_search_xchg.argtypes = [vp, vp, vp, u32, vp, vp, C.POINTER(u32), C.POINTER(i32)]
    L.stb_search_many.argtypes = [vp, vp, vp, u32, u32, vp, vp, vp, vp]
    L.stb_xchg_create_batch.argtypes = [vp, u32, u32, u32, u32, C.POINTER(vp)]
    L.stb_search_batch_xchg_dev.argtypes = [vp, vp, vp, u32, u32, vp, vp, vp]
    L.stb_ivfpq_build.argtypes = [vp, vp, u32, u32, u32, C.POINTER(vp)]
    L.stb_ivfpq_destroy.argtypes = [vp]
    L.stb_ivfpq_extend.argtypes = [vp, C.POINTER(u64)]
    L.stb_ivfpq_update.argtypes = [vp, vp, vp, u64]
    L.stb_ivfpq_remove.argtypes = [vp, vp, u32]
    L.stb_ivfpq_stats.argtypes = [vp, C.POINTER(u64), C.POINTER(u32), C.POINTER(u32), C.POINTER(u64)]
    L.stb_ivfpq_search.argtypes = [vp, vp, u32, u32, u32, vp, C.POINTER(u32), C.POINTER(u64)]
    L.stb_ivfpq_search_dev.argtypes = [vp, vp, u32, u32, u32, vp, vp]
    L.stb_hits_merge_dev.argtypes = [vp, vp, u32, u32, u32, vp]
    L.stb_hits_merge_batch_dev.argtypes = [vp, vp, u32, u32, u32, u32, vp]
    L.stb_hits_merge.argtypes = [vp, vp, u32, u32, u32, vp, C.POINTER(u32)]
    L.stb_fnv1a64.argtypes = [C.c_char_p, u64]
    L.stb_fnv1a64.restype = u64
    L.stb_line_id.argtypes = [C.c_char_p, u64, C.c_int32]
    L.stb_line_ids.argtypes = [vp, vp, u32, vp, u64, vp]
    L.stb_line_id.restype = u64
    L.stb_ctx_counters.argtypes = [vp, C.POINTER(u64), C.POINTER(u64)]
    L.stb_debug_ticket_check.argtypes = [vp, C.POINTER(u64), C.POINTER(u64)]
    L.stb_debug_q4_refined.argtypes = [vp, i32, C.POINTER(u64)]
    L.stb_debug_coscan_offsets.argtypes = [vp, u32, vp]
    L.stb_debug_pair_joins.argtypes = [vp, u32, vp]
    L.stb_debug_pair_floor.argtypes = [vp, u64]
    L.stb_debug_batch_gemm.argtypes = [vp, vp, u32, vp, u64, vp, vp]
    L.stb_debug_batch_params.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_double)]
    L.stb_debug_batch_last.argtypes = [vp, vp, vp, vp]
    L.stb_debug_batch_q8.argtypes = [vp, vp, vp, u32, u32, vp, vp]
    L.stb_debug_batch_no_shadow.argtypes = [vp, i32]
    L.stb_debug_batch_q8_gemm.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp]
    L.stb_debug_batch_q8_plan.argtypes = [u32, u64, u32, vp]
    L.stb_debug_ivfpq_export.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    L.stb_ivfpq_search_batch.argtypes = [vp, vp, u32, u32, u32, u32, vp, vp, vp]
    L.stb_ivfpq_search_batch_dev.argtypes = [vp, vp, u32, u32, u32, u32, vp, vp]
    L.stb_debug_ivfpq_batch_last.argtypes = [vp, u32, vp, vp, vp, vp]
    L.stb_ivfpq_search_filtered.argtypes = [vp, vp, u32, u32, u32, u32, i32, f64, vp, u32, vp, vp, vp]
    L.stb_ivfpq_search_subsets.argtypes = [vp, vp, u32, u32, u32, u32, i32, f64, u32, vp, vp, vp, vp, vp, vp]
    L.stb_ivfpq_search_threshold.argtypes = [vp, vp, u32, u32, f64, f64, vp, u64, vp, vp, vp]
    L.stb_debug_ivfpq_threshold_keys.argtypes = [vp, u64]
    L.stb_ivfpq_save.argtypes = [vp, C.c_char_p]
    L.stb_ivfpq_load.argtypes = [vp, vp, C.c_char_p, C.POINTER(vp)]
    L.stb_debug_ivfpq_load_ms.argtypes = [vp, vp]
    L.stb_tokenizer_load.argtypes = [vp, vp, u64, C.POINTER(vp)]
    L.stb_tokenizer_load_ex.argtypes = [vp, vp, u64, u32, C.POINTER(vp)]
    L.stb_tokenizer_destroy.argtypes = [vp]
    L.stb_tokenizer_gpu_lines.argtypes = [vp, vp, vp, u64, vp]
    L.stb_embed_text.argtypes = [vp, vp, vp, vp, vp, u64, u32, vp, vp]
    L.stb_debug_tokenize.argtypes = [vp, vp, vp, vp, u64, u32, vp, vp, u64, vp]
    for name in SYMBOLS:
        fn = getattr(L, name)
        if fn.restype is C.c_int and name not in ("stb_version", "stb_device_count"):
            fn.restype = i32
    _lib = L
    return L


def _check(rc: int, allow_capacity: bool = False) -> int:
    if rc < 0 and not (allow_capacity and rc == STB_ERR_CAPACITY):
        raise StbError(rc, lib().stb_last_error().decode("utf-8", "replace"))
    return rc


def _np_ptr(a):
    return None if a is None else a.ctypes.data_as(vp)


def device_count() -> int:
    return int(lib().stb_device_count())


def batch_params():
    """(shadow_is_f16, eps) of this build's K2 path (stb_debug_batch_params; host-only)."""
    f16, eps = C.c_int(0), C.c_double(0.0)
    _check(lib().stb_debug_batch_params(C.byref(f16), C.byref(eps)))
    return bool(f16.value), float(eps.value)


def batch_q8_plan(sm_count: int, n_rows: int, top_k: int):
    """(n_sample, stride, fits) of K2 route 7's plan for a card with sm_count SMs (stb_debug_batch_q8_plan;
    host-only)."""
    out = np.zeros(3, dtype=np.uint32)
    _check(lib().stb_debug_batch_q8_plan(sm_count, n_rows, top_k, _np_ptr(out)))
    return int(out[0]), int(out[1]), bool(out[2])


def fnv1a64(data: bytes) -> int:
    """fnv1a_hash / DocMeta::id (reference src/workspace/store.rs:651-661, :75-80)."""
    return int(lib().stb_fnv1a64(data, len(data)))


def line_id(path: str, line_number: int) -> int:
    """LineEmbedding::id (reference src/workspace/store.rs:82-89)."""
    b = path.encode("utf-8")
    return int(lib().stb_line_id(b, len(b), line_number))


def line_ids(paths, rows) -> np.ndarray:
    """stb_line_ids: LineEmbedding ids of all rows ((path index, line_number) int32 pairs) in one
    native call (a store with millions of rows used to make one ctypes call per row)."""
    rows = np.ascontiguousarray(rows, dtype=np.int32).reshape(-1, 2)
    enc = [p.encode("utf-8") for p in paths]
    offs = np.zeros(len(enc) + 1, dtype=np.uint64)
    if enc:
        offs[1:] = np.cumsum([len(b) for b in enc])
    blob = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8)
    out = np.zeros(len(rows), dtype=np.uint64)
    _check(lib().stb_line_ids(_np_ptr(blob), _np_ptr(offs), len(enc), _np_ptr(rows), len(rows), _np_ptr(out)))
    return out


class Context:
    """stb_ctx: one CUDA device + stream.  `stream` is an optional raw cudaStream_t."""

    def __init__(self, device: int = 0, stream: int | None = None):
        self._h = vp()
        _check(lib().stb_ctx_create(device, vp(stream) if stream else None, C.byref(self._h)))
        self.device = device

    def close(self):
        if getattr(self, "_h", None) is not None and self._h and _lib is not None:
            _lib.stb_ctx_destroy(self._h)
            self._h = None

    __del__ = close

    def sync(self):
        _check(lib().stb_ctx_sync(self._h))

    @property
    def stream(self) -> int:
        return int(lib().stb_ctx_stream(self._h) or 0)

    def counters(self):
        a, b = u64(0), u64(0)
        _check(lib().stb_ctx_counters(self._h, C.byref(a), C.byref(b)))
        return {"kernel_launches": int(a.value), "fallback_searches": int(b.value)}

    def ticket_check(self):
        """stb_debug_ticket_check: (device counter, host-booked value); raises StbError on a mismatch."""
        a, b = u64(0), u64(0)
        _check(lib().stb_debug_ticket_check(self._h, C.byref(a), C.byref(b)))
        return int(a.value), int(b.value)

    def coscan_offsets(self, n: int = 8):
        """stb_debug_coscan_offsets: tile offsets of the last n top-k launches, oldest first (None: no co-scan)."""
        out = np.zeros(max(n, 1), dtype=np.uint32)
        _check(lib().stb_debug_coscan_offsets(self._h, n, _np_ptr(out)))
        return [None if v == 0xFFFFFFFF else int(v) for v in out[:n]]

    def pair_joins(self, n: int = 8):
        """stb_debug_pair_joins: join tile of each of the last n top-k launches, oldest first (None: not a
        guest, "refused": a guest that scanned alone)."""
        out = np.zeros(max(n, 1), dtype=np.int64)
        _check(lib().stb_debug_pair_joins(self._h, n, _np_ptr(out)))
        return [None if v == -1 else ("refused" if v == -2 else int(v)) for v in out[:n]]

    def pair_floor(self, v_floor: int = 0):
        """stb_debug_pair_floor: later joins wait until their host has drawn v_floor tile tickets."""
        _check(lib().stb_debug_pair_floor(self._h, int(v_floor)))

    def batch_last(self):
        """stb_debug_batch_last: the most recent K2 device call on this context.  Returns a dict with
        route (1 = v1, 2 = v2, 3 = filtered v2, 4 = filtered without the tensor cores, 5 = threshold mode, 6 = one
        filter per query group, 7 = v2 on the q8 copy, 8 = filtered v2 on the q8 copy, 9 = one filter per query group
        on the q8 copy, 10 = threshold mode on the q8 copy), nq, n_sample, stride (routes 1-4, 7, 8) or retried, k1
        (routes 5, 10: queries re-emitted by the second tensor pass / answered by stb_search) or groups, k1 (routes 6,
        9: groups on the tensor cores / queries answered by stb_search), n_seg, seg_cap and, after v2 (filtered or
        not) and a route 5, 6, 7, 8 or 10 call that ran the tensor passes, thr [nq] (f32) and cand_cnt [nq][n_seg]
        (raw counts; > seg_cap marks an overflowed segment; route 6: caller order, +inf and zeros for a query the
        tensor passes did not take)."""
        info = np.zeros(6, dtype=np.uint32)
        _check(lib().stb_debug_batch_last(self._h, _np_ptr(info), None, None))
        names = {5: ("retried", "k1"), 6: ("groups", "k1"), 9: ("groups", "k1"), 10: ("retried", "k1")}.get(
            int(info[0]), ("n_sample", "stride"))
        out = dict(zip(("route", "nq") + names + ("n_seg", "seg_cap"), (int(v) for v in info)))
        if out["route"] in (2, 3) or (out["route"] in (5, 6, 7, 8, 10) and out["n_seg"]):
            thr = np.zeros(max(out["nq"], 1), dtype=np.float32)
            cnt = np.zeros((max(out["nq"], 1), max(out["n_seg"], 1)), dtype=np.uint32)
            _check(lib().stb_debug_batch_last(self._h, _np_ptr(info), _np_ptr(thr), _np_ptr(cnt)))
            out["thr"], out["cand_cnt"] = thr[: out["nq"]], cnt[: out["nq"]]
        return out

    @contextlib.contextmanager
    def batch_no_shadow(self):
        """stb_debug_batch_no_shadow: within the block, every K2 search on this context behaves as if the 16-bit
        shadow did not fit in HBM and takes its q8 route (7-10); no shadow is built or changed."""
        _check(lib().stb_debug_batch_no_shadow(self._h, 1))
        try:
            yield self
        finally:
            _check(lib().stb_debug_batch_no_shadow(self._h, 0))

    # -- K4 ------------------------------------------------------------------
    def hits_merge(self, lists: np.ndarray, top_k: int) -> np.ndarray:
        """lists: (n_lists, per_list) array of HIT_DTYPE; returns the merged top_k."""
        lists = np.ascontiguousarray(lists, dtype=HIT_DTYPE)
        n_lists, per_list = lists.shape
        out = np.zeros(max(top_k, 1), dtype=HIT_DTYPE)
        n = u32(0)
        _check(lib().stb_hits_merge(self._h, _np_ptr(lists), n_lists, per_list, top_k, _np_ptr(out),
                                    C.byref(n)))
        return out[: n.value]

    def hits_merge_batch_dev(self, lists_dev: int, n_lists: int, nq: int, per_list: int, top_k: int, out_dev: int):
        """lists_dev [n_lists][nq][per_list] -> out_dev [nq][top_k] (sharded K2)."""
        _check(lib().stb_hits_merge_batch_dev(self._h, vp(lists_dev), n_lists, nq, per_list, top_k, vp(out_dev)))

    def hits_merge_dev(self, lists_dev: int, n_lists: int, per_list: int, top_k: int, out_dev: int):
        _check(lib().stb_hits_merge_dev(self._h, vp(lists_dev), n_lists, per_list, top_k, vp(out_dev)))


class Table:
    """stb_table: the StaticModel tensors resident in HBM."""

    def __init__(self, ctx: Context, E, weights=None, mapping=None, normalize=True):
        E = np.ascontiguousarray(E, dtype=np.float32)
        w = None if weights is None else np.ascontiguousarray(weights, dtype=np.float32)
        m = None if mapping is None else np.ascontiguousarray(mapping, dtype=np.uint32)
        self.ctx = ctx
        self._h = vp()
        _check(lib().stb_table_load(ctx._h, _np_ptr(E), E.shape[0], E.shape[1], _np_ptr(w),
                                    0 if w is None else w.size, _np_ptr(m), 0 if m is None else m.size,
                                    int(normalize), C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h and _lib is not None:
            _lib.stb_table_destroy(self._h)
            self._h = None

    __del__ = close


class Tokenizer:
    """stb_tokenizer: a tokenizer.json loaded into the library (Unigram model resident in HBM).  utf8=True loads
    it with STB_TOKENIZER_UTF8: the GPU takes valid UTF-8 lines, not only printable ASCII ones (same ids)."""

    def __init__(self, ctx: Context, json_bytes: bytes, utf8: bool = False):
        self.ctx = ctx
        self._h = vp()
        buf = np.frombuffer(json_bytes, dtype=np.uint8)
        flags = STB_TOKENIZER_UTF8 if utf8 else 0
        _check(lib().stb_tokenizer_load_ex(ctx._h, _np_ptr(buf), buf.size, flags, C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h and _lib is not None:
            _lib.stb_tokenizer_destroy(self._h)
            self._h = None

    __del__ = close

    def gpu_lines(self, lines) -> np.ndarray:
        """stb_tokenizer_gpu_lines: 1 for each line the GPU tokenises (host-only)."""
        text, offsets = pack_lines(lines)
        taken = np.zeros(len(lines), dtype=np.uint8)
        _check(lib().stb_tokenizer_gpu_lines(self._h, _np_ptr(text), _np_ptr(offsets), len(lines), _np_ptr(taken)))
        return taken.astype(bool)

    def debug_tokenize(self, lines, max_length: int):
        """stb_debug_tokenize -> (offsets u64[n+1], ids u32, taken bool[n]): the CSR stb_embed_text pools."""
        text, offsets = pack_lines(lines)
        n = len(lines)
        out_off = np.zeros(n + 1, dtype=np.uint64)
        taken = np.zeros(max(n, 1), dtype=np.uint8)
        cap = int(offsets[-1]) + 2 * n + 1                    # a line of k bytes has at most k + 1 ids
        ids = np.zeros(cap, dtype=np.uint32)
        rc = _check(lib().stb_debug_tokenize(self.ctx._h, self._h, _np_ptr(text), _np_ptr(offsets), n, max_length,
                                             _np_ptr(out_off), _np_ptr(ids), cap, _np_ptr(taken)), allow_capacity=True)
        if rc == STB_ERR_CAPACITY:
            cap = int(out_off[-1])
            ids = np.zeros(max(cap, 1), dtype=np.uint32)
            _check(lib().stb_debug_tokenize(self.ctx._h, self._h, _np_ptr(text), _np_ptr(offsets), n, max_length,
                                            _np_ptr(out_off), _np_ptr(ids), cap, _np_ptr(taken)))
        return out_off, ids[: int(out_off[-1])].copy(), taken[:n].astype(bool)


def pack_lines(lines):
    """Lines (str or bytes) -> (UTF-8 text u8, offsets u64[n+1])."""
    enc = [l.encode("utf-8") if isinstance(l, str) else bytes(l) for l in lines]
    offsets = np.zeros(len(enc) + 1, dtype=np.uint64)
    if enc:
        offsets[1:] = np.cumsum([len(b) for b in enc])
    text = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8)
    return text, offsets


class Corpus:
    """stb_corpus: contiguous N x 256 f32 line-vector matrix in HBM."""
    host_rows = False

    def __init__(self, ctx: Context, capacity_rows: int = 1024, row_base: int = 0):
        self.ctx = ctx
        self.row_base = row_base
        self._h = vp()
        _check(lib().stb_corpus_create(ctx._h, STB_DIM, capacity_rows, row_base, C.byref(self._h)))

    @classmethod
    def in_host_memory(cls, ctx: Context, capacity_rows: int = 1024, row_base: int = 0) -> "Corpus":
        """stb_corpus_create_host: the f32 rows in page-locked host memory, only the q8 copy in HBM (a corpus
        larger than the card's memory; the same hits as a device corpus, see the header for the routes)."""
        self = cls.__new__(cls)
        self.ctx, self.row_base, self.host_rows = ctx, row_base, True
        self._h = vp()
        _check(lib().stb_corpus_create_host(ctx._h, STB_DIM, capacity_rows, row_base, C.byref(self._h)))
        return self

    def close(self):
        if getattr(self, "_h", None) is not None and self._h and _lib is not None:
            _lib.stb_corpus_destroy(self._h)
            self._h = None

    __del__ = close

    def append(self, rows: np.ndarray):
        rows = np.ascontiguousarray(rows, dtype=np.float32)
        if rows.size == 0:
            return
        if rows.ndim != 2 or rows.shape[1] != STB_DIM:
            raise StbError(STB_ERR_ARG, f"rows must be (n,{STB_DIM}) f32")
        _check(lib().stb_corpus_append(self._h, _np_ptr(rows), rows.shape[0]))

    def append_dev(self, rows_dev: int, n: int):
        _check(lib().stb_corpus_append_dev(self._h, vp(rows_dev), n))

    def clear(self):
        _check(lib().stb_corpus_clear(self._h))

    def __len__(self) -> int:
        n = u64(0)
        _check(lib().stb_corpus_rows(self._h, C.byref(n)))
        return int(n.value)

    @property
    def data_dev(self) -> int:
        p = vp()
        _check(lib().stb_corpus_data_dev(self._h, C.byref(p)))
        return int(p.value or 0)

    def read(self, first: int = 0, n: int | None = None) -> np.ndarray:
        n = len(self) - first if n is None else n
        out = np.empty((n, STB_DIM), dtype=np.float32)
        _check(lib().stb_corpus_read(self._h, first, n, _np_ptr(out)))
        return out

    def update(self, idx, rows):
        """stb_corpus_update: rows[i] replaces global row idx[i] (idx strictly ascending); the candidate
        copies that exist are re-encoded at those rows and stay built."""
        idx = np.ascontiguousarray(idx, dtype=np.uint64).reshape(-1)
        rows = np.ascontiguousarray(rows, dtype=np.float32).reshape(-1, STB_DIM)
        if rows.shape[0] != idx.size:
            raise StbError(STB_ERR_ARG, f"{idx.size} row ids for {rows.shape[0]} rows")
        if idx.size:
            _check(lib().stb_corpus_update(self._h, _np_ptr(idx), _np_ptr(rows), idx.size))

    def remove(self, ranges):
        """stb_corpus_remove: delete the global rows of (n, 2) half-open [begin, end) ranges (ascending,
        disjoint, non-empty); later rows move down in order, the candidate copies follow them."""
        rr = np.ascontiguousarray(ranges, dtype=np.uint64).reshape(-1, 2)
        if rr.shape[0]:
            _check(lib().stb_corpus_remove(self._h, _np_ptr(rr), rr.shape[0]))

    def debug_copy(self, which: int, first: int = 0, n: int | None = None):
        """stb_debug_corpus_copy: (entries [first, first+n) of one candidate copy, rows the copy covers).
        which: STB_COPY_Q8_CODES / _Q8_SCALES / _Q8_PLANE / _Q8_SR (entries are rows) or STB_COPY_H16_TILES
        (entries are 256-row tiles of 131072 bytes); n=None: every covered entry from `first` on."""
        covered = u64(0)
        _check(lib().stb_debug_corpus_copy(self._h, which, 0, 0, None, C.byref(covered)))
        cov = int(covered.value)
        units = (cov + 255) // 256 if which == STB_COPY_H16_TILES else cov
        n = units - first if n is None else n
        shape, dtype = {STB_COPY_Q8_CODES: ((n, 256), np.int8), STB_COPY_Q8_SCALES: ((n,), np.float32),
                        STB_COPY_Q8_PLANE: ((n, 128), np.uint8), STB_COPY_Q8_SR: ((n, 2), np.float32),
                        STB_COPY_H16_TILES: ((n, 131072), np.uint8)}[which]
        out = np.zeros(shape, dtype=dtype)
        _check(lib().stb_debug_corpus_copy(self._h, which, first, n, _np_ptr(out) if n else None, C.byref(covered)))
        return out, cov

    @staticmethod
    def _debug_args(q, row_ranges):
        q = np.ascontiguousarray(q, dtype=np.float32)
        if q.size != STB_DIM:
            raise StbError(STB_ERR_ARG, f"query must have {STB_DIM} floats")
        if row_ranges is None:
            return q, None, 0
        rr = np.ascontiguousarray(row_ranges, dtype=np.uint64).reshape(-1, 2)
        return q, (rr if rr.shape[0] else np.zeros((1, 2), dtype=np.uint64)), rr.shape[0]

    def debug_scan_scores(self, q, tier: str = "f32", row_ranges=None, hist: bool = False):
        """stb_debug_scan_scores: (score [n] f32, times scored [n] u32, 4096-bin histogram or None) of one K1
        pass, tier "f32" | "h16" | "q8", per local row; rows outside row_ranges keep NaN and 0."""
        q, rr, n_rr = self._debug_args(q, row_ranges)
        n = len(self)
        scores, seen = np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.uint32)
        h = np.zeros(4096, np.uint32) if hist else None
        _check(lib().stb_debug_scan_scores(self.ctx._h, self._h, ("f32", "h16", "q8").index(tier), _np_ptr(q), _np_ptr(rr), n_rr,
                                           n, _np_ptr(scores), _np_ptr(seen), _np_ptr(h)))
        return scores[:n], seen[:n], h

    def debug_q4_scan(self, q, top_k: int, row_ranges=None, pin: bool = True):
        """stb_debug_q4_scan: the q8 tier's prefiltered top-k scan, per local row.  Returns a dict of numpy
        arrays: u4, t (the threshold the row was tested against), refined (times scored from the int8 codes), u8,
        l8 (refined rows; NaN elsewhere), and words [top_k] u64 (the final threshold words)."""
        q, rr, n_rr = self._debug_args(q, row_ranges)
        n = len(self)
        out = {k: np.zeros(max(n, 1), np.float32) for k in ("u4", "t", "u8", "l8")}
        out["refined"] = np.zeros(max(n, 1), np.uint32)
        words = np.zeros(max(top_k, 1), np.uint64)
        _check(lib().stb_debug_q4_scan(self.ctx._h, self._h, _np_ptr(q), top_k, _np_ptr(rr), n_rr, int(pin), n,
                                       _np_ptr(out["u4"]), _np_ptr(out["t"]), _np_ptr(out["refined"]), _np_ptr(out["u8"]),
                                       _np_ptr(out["l8"]), _np_ptr(words)))
        out = {k: v[:n] for k, v in out.items()}
        out["words"] = words[:top_k]
        return out

    # -- K1 + K4 -------------------------------------------------------------
    def search(self, q, top_k: int = 3, max_distance: float | None = None,
               mode: int = STB_MODE_SEARCH_DOCUMENTS, row_ranges=None, cap: int | None = None):
        """stb_search.  Returns a HIT_DTYPE array ordered by (distance,row)."""
        q = np.ascontiguousarray(q, dtype=np.float32)
        if q.size != STB_DIM:
            raise StbError(STB_ERR_ARG, f"query must have {STB_DIM} floats")
        rr, n_rr = None, 0
        if row_ranges is not None:
            rr = np.ascontiguousarray(row_ranges, dtype=np.uint64).reshape(-1, 2)
            n_rr = rr.shape[0]
            if n_rr == 0:
                rr = np.zeros((1, 2), dtype=np.uint64)   # non-null pointer, zero ranges
        if cap is None:
            cap = max(top_k, 1) if (max_distance is None or mode == STB_MODE_STORE_QUERY) else max(top_k, 4096)
        while True:
            out = np.zeros(max(cap, 1), dtype=HIT_DTYPE)
            n = u64(0)
            rc = _check(lib().stb_search(self.ctx._h, self._h, _np_ptr(q), top_k,
                                         int(max_distance is not None), float(max_distance or 0.0), mode,
                                         _np_ptr(rr), n_rr, _np_ptr(out), cap, C.byref(n)), allow_capacity=True)
            if rc == STB_ERR_CAPACITY:
                cap = int(n.value)
                continue
            return out[: int(n.value)]

    def search_many(self, queries, top_k: int = 10, xchg=None):
        """stb_search_many: nq independent single queries, one synchronisation.  Returns a list of
        HIT_DTYPE arrays (x is None) or (list, complete flags) for the sharded form."""
        queries = np.ascontiguousarray(queries, dtype=np.float32)
        if queries.ndim != 2 or queries.shape[1] != STB_DIM:
            raise StbError(STB_ERR_ARG, f"queries must be (nq,{STB_DIM}) f32")
        nq = queries.shape[0]
        out = np.zeros((nq, max(top_k, 1)), dtype=HIT_DTYPE)
        cnt = np.zeros(max(nq, 1), dtype=np.uint32)
        ok = np.ones(max(nq, 1), dtype=np.uint8)
        _check(lib().stb_search_many(self.ctx._h, self._h, _np_ptr(queries), nq, top_k, xchg._h if xchg is not None else None,
                                     _np_ptr(out), _np_ptr(cnt), _np_ptr(ok)))
        res = [out[i, : cnt[i]] for i in range(nq)]
        return res if xchg is None else (res, ok[:nq].astype(bool))

    # -- K2 -----------------------------------------------------------------
    def prepare(self, what: int = 3):
        """stb_corpus_prepare: build the reduced-width candidate copies now
        (STB_PREPARE_Q8 = 1, STB_PREPARE_H16 = 2)."""
        _check(lib().stb_corpus_prepare(self._h, what))

    def tier_stats(self):
        """stb_corpus_tier_stats -> {"f32"|"h16"|"q8": {"tries", "proven", "built_rows"}}."""
        tries, proven = np.zeros(3, np.uint32), np.zeros(3, np.uint32)
        built = np.zeros(3, np.uint64)
        _check(lib().stb_corpus_tier_stats(self._h, _np_ptr(tries), _np_ptr(proven), _np_ptr(built)))
        return {name: {"tries": int(tries[i]), "proven": int(proven[i]), "built_rows": int(built[i])}
                for i, name in enumerate(("f32", "h16", "q8"))}

    def prepare_batch(self):
        """stb_corpus_prepare_batch: build the 16-bit tensor-core shadow now."""
        _check(lib().stb_corpus_prepare_batch(self._h))

    def search_batch(self, queries, top_k: int = 10):
        """stb_search_batch.  Returns a list of HIT_DTYPE arrays, one per query."""
        queries = np.ascontiguousarray(queries, dtype=np.float32)
        if queries.ndim != 2 or queries.shape[1] != STB_DIM:
            raise StbError(STB_ERR_ARG, f"queries must be (nq,{STB_DIM}) f32")
        nq = queries.shape[0]
        out = np.zeros((nq, max(top_k, 1)), dtype=HIT_DTYPE)
        cnt = np.zeros(max(nq, 1), dtype=np.uint32)
        _check(lib().stb_search_batch(self.ctx._h, self._h, _np_ptr(queries), nq, top_k, _np_ptr(out), _np_ptr(cnt)))
        return [out[i, : cnt[i]] for i in range(nq)]

    def debug_batch_q8(self, queries, top_k: int = 10):
        """stb_debug_batch_q8: search_batch on route 7 (the q8 copy on the int8 tensor cores) whatever the state of
        the 16-bit shadow.  Returns a list of HIT_DTYPE arrays, one per query."""
        queries = np.ascontiguousarray(queries, dtype=np.float32)
        if queries.ndim != 2 or queries.shape[1] != STB_DIM:
            raise StbError(STB_ERR_ARG, f"queries must be (nq,{STB_DIM}) f32")
        nq = queries.shape[0]
        out = np.zeros((nq, max(top_k, 1)), dtype=HIT_DTYPE)
        cnt = np.zeros(max(nq, 1), dtype=np.uint32)
        _check(lib().stb_debug_batch_q8(self.ctx._h, self._h, _np_ptr(queries), nq, top_k, _np_ptr(out), _np_ptr(cnt)))
        return [out[i, : cnt[i]] for i in range(nq)]

    def debug_batch_q8_gemm(self, queries):
        """stb_debug_batch_q8_gemm: route 7's query quantisation and integer GEMM.  Returns (q16 [nq, 256] int16,
        dot [nq, n] int32, u [nq, n] f32, l [nq, n] f32)."""
        queries = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, STB_DIM)
        nq, n = queries.shape[0], len(self)
        q16 = np.zeros((nq, STB_DIM), dtype=np.int16)
        dot = np.zeros((nq, n), dtype=np.int32)
        u = np.zeros((nq, n), dtype=np.float32)
        l = np.zeros((nq, n), dtype=np.float32)
        _check(lib().stb_debug_batch_q8_gemm(self.ctx._h, self._h, _np_ptr(queries), nq, _np_ptr(q16), _np_ptr(dot),
                                             _np_ptr(u), _np_ptr(l)))
        return q16, dot, u, l

    def search_batch_filtered(self, queries, row_ranges=None, top_k: int = 10, max_distance: float | None = None):
        """stb_search_batch_filtered: for each query, what search(q, top_k, max_distance, STB_MODE_STORE_QUERY,
        row_ranges) returns (row_ranges: (n, 2) global [begin, end) pairs; None = every row, empty = no row).
        Returns a list of HIT_DTYPE arrays, one per query."""
        queries = np.ascontiguousarray(queries, dtype=np.float32)
        if queries.ndim != 2 or queries.shape[1] != STB_DIM:
            raise StbError(STB_ERR_ARG, f"queries must be (nq,{STB_DIM}) f32")
        nq = queries.shape[0]
        rr, n_rr = None, 0
        if row_ranges is not None:
            rr = np.ascontiguousarray(row_ranges, dtype=np.uint64).reshape(-1, 2)
            n_rr = rr.shape[0]
            if n_rr == 0:
                rr = np.zeros((1, 2), dtype=np.uint64)   # non-null pointer, zero ranges
        out = np.zeros((nq, max(top_k, 1)), dtype=HIT_DTYPE)
        cnt = np.zeros(max(nq, 1), dtype=np.uint32)
        _check(lib().stb_search_batch_filtered(self.ctx._h, self._h, _np_ptr(queries), nq, top_k,
                                               int(max_distance is not None), float(max_distance or 0.0),
                                               _np_ptr(rr), n_rr, _np_ptr(out), _np_ptr(cnt)))
        return [out[i, : cnt[i]] for i in range(nq)]

    def search_batch_subsets(self, queries, ranges_per_query, top_k: int = 10, max_distance: float | None = None):
        """stb_search_batch_subsets: for each query i, what search(queries[i], top_k, max_distance,
        STB_MODE_STORE_QUERY, ranges_per_query[i]) returns (each an (n, 2) array of global [begin, end) pairs;
        n = 0 is the empty subset).  Returns a list of HIT_DTYPE arrays, one per query."""
        queries = np.ascontiguousarray(queries, dtype=np.float32)
        if queries.ndim != 2 or queries.shape[1] != STB_DIM:
            raise StbError(STB_ERR_ARG, f"queries must be (nq,{STB_DIM}) f32")
        nq = queries.shape[0]
        if len(ranges_per_query) != nq:
            raise StbError(STB_ERR_ARG, f"{len(ranges_per_query)} range lists for {nq} queries")
        parts = [np.asarray(r, dtype=np.uint64).reshape(-1, 2) for r in ranges_per_query]
        offsets = np.zeros(nq + 1, dtype=np.uint64)
        offsets[1:] = np.cumsum([len(p) for p in parts]) if nq else []
        rr = np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros((0, 2), np.uint64), dtype=np.uint64)
        if len(rr) == 0:
            rr = np.zeros((1, 2), dtype=np.uint64)
        out = np.zeros((nq, max(top_k, 1)), dtype=HIT_DTYPE)
        cnt = np.zeros(max(nq, 1), dtype=np.uint32)
        _check(lib().stb_search_batch_subsets(self.ctx._h, self._h, _np_ptr(queries), nq, top_k,
                                              int(max_distance is not None), float(max_distance or 0.0),
                                              _np_ptr(offsets), _np_ptr(rr), _np_ptr(out), _np_ptr(cnt)))
        return [out[i, : cnt[i]] for i in range(nq)]

    def search_batch_threshold(self, queries, max_distance: float, cap: int | None = None):
        """stb_search_batch_threshold: for each query, what search(q, 0, max_distance) returns in threshold mode
        (every row with distance < max_distance).  Starts from a modest capacity and retries once with the
        reported total.  Returns a list of HIT_DTYPE arrays, one per query."""
        queries = np.ascontiguousarray(queries, dtype=np.float32)
        if queries.ndim != 2 or queries.shape[1] != STB_DIM:
            raise StbError(STB_ERR_ARG, f"queries must be (nq,{STB_DIM}) f32")
        nq = queries.shape[0]
        if cap is None:
            cap = max(nq, 1) * 64
        offsets = np.zeros(nq + 1, dtype=np.uint64)
        while True:
            out = np.zeros(max(cap, 1), dtype=HIT_DTYPE)
            rc = _check(lib().stb_search_batch_threshold(self.ctx._h, self._h, _np_ptr(queries), nq, float(max_distance),
                                                         _np_ptr(out), cap, _np_ptr(offsets)), allow_capacity=True)
            if rc == STB_ERR_CAPACITY:
                cap = int(offsets[nq])
                continue
            return [out[int(offsets[i]): int(offsets[i + 1])] for i in range(nq)]

    def search_batch_dev(self, q_dev: int, nq: int, top_k: int, out_hits_dev: int, out_status_dev: int):
        """stb_search_batch_dev: asynchronous, everything stays in HBM."""
        _check(lib().stb_search_batch_dev(self.ctx._h, self._h, vp(q_dev), nq, top_k, vp(out_hits_dev),
                                          vp(out_status_dev)))

    def search_topk_dev(self, q_dev: int, top_k: int, out_hits_dev: int, out_status_dev: int):
        """stb_search_topk_dev: asynchronous, everything stays in HBM."""
        _check(lib().stb_search_topk_dev(self.ctx._h, self._h, vp(q_dev), top_k, vp(out_hits_dev),
                                         vp(out_status_dev)))


class IvfPq:
    """stb_ivfpq: approximate IVF-PQ index over a corpus (K5; self-specified, see header)."""

    def __init__(self, corpus: "Corpus", nlist: int = 4096, train_rows: int = 262144, iters: int = 8):
        self.corpus = corpus
        self._h = vp()
        _check(lib().stb_ivfpq_build(corpus.ctx._h, corpus._h, nlist, train_rows, iters, C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h and _lib is not None:
            _lib.stb_ivfpq_destroy(self._h)
            self._h = None

    __del__ = close

    def save(self, path):
        """stb_ivfpq_save: write the index to `path` (atomically replaced); the corpus rows are not stored."""
        _check(lib().stb_ivfpq_save(self._h, os.fsencode(path)))

    @classmethod
    def load(cls, corpus: "Corpus", path) -> "IvfPq":
        """stb_ivfpq_load: the index saved at `path`, on a corpus whose first rows are the ones it was saved with."""
        self = cls.__new__(cls)
        self.corpus = corpus
        self._h = vp()
        _check(lib().stb_ivfpq_load(corpus.ctx._h, corpus._h, os.fsencode(path), C.byref(self._h)))
        return self

    def load_ms(self):
        """stb_debug_ivfpq_load_ms: (read + upload, verification) milliseconds of the load that made this index."""
        ms = np.zeros(2, dtype=np.float64)
        _check(lib().stb_debug_ivfpq_load_ms(self._h, _np_ptr(ms)))
        return float(ms[0]), float(ms[1])

    def extend(self) -> int:
        """stb_ivfpq_extend: index the rows appended to the corpus since the build or the last extend
        (same quantisers); returns how many were added."""
        added = u64(0)
        _check(lib().stb_ivfpq_extend(self._h, C.byref(added)))
        return int(added.value)

    def update(self, idx, rows):
        """stb_ivfpq_update: Corpus.update on the index's corpus, and the replaced indexed rows get the list
        and code of their new value (same quantisers)."""
        idx = np.ascontiguousarray(idx, dtype=np.uint64).reshape(-1)
        rows = np.ascontiguousarray(rows, dtype=np.float32).reshape(-1, STB_DIM)
        if rows.shape[0] != idx.size:
            raise StbError(STB_ERR_ARG, f"{idx.size} row ids for {rows.shape[0]} rows")
        if idx.size:
            _check(lib().stb_ivfpq_update(self._h, _np_ptr(idx), _np_ptr(rows), idx.size))

    def remove(self, ranges):
        """stb_ivfpq_remove: Corpus.remove on the index's corpus; the removed rows leave the index and the
        entries behind them are renumbered."""
        rr = np.ascontiguousarray(ranges, dtype=np.uint64).reshape(-1, 2)
        if rr.shape[0]:
            _check(lib().stb_ivfpq_remove(self._h, _np_ptr(rr), rr.shape[0]))

    def stats(self):
        rows, nbytes, nlist, mx = u64(0), u64(0), u32(0), u32(0)
        _check(lib().stb_ivfpq_stats(self._h, C.byref(rows), C.byref(nlist), C.byref(mx), C.byref(nbytes)))
        return {"rows": int(rows.value), "nlist": int(nlist.value), "max_list": int(mx.value),
                "index_bytes": int(nbytes.value)}

    def search(self, q, nprobe: int = 64, top_k: int = 10, rerank: int = 256):
        q = np.ascontiguousarray(q, dtype=np.float32)
        out = np.zeros(max(top_k, 1), dtype=HIT_DTYPE)
        n, scanned = u32(0), u64(0)
        _check(lib().stb_ivfpq_search(self._h, _np_ptr(q), nprobe, top_k, rerank, _np_ptr(out), C.byref(n),
                                      C.byref(scanned)))
        return out[: n.value], int(scanned.value)

    def export(self):
        """stb_debug_ivfpq_export: the built index as numpy arrays (centroids, codebooks, list_off,
        order, codes, forced); m = list_off[-1] rows are in the lists, the others in `forced`."""
        nlist, n = self.stats()["nlist"], self.stats()["rows"]
        list_off = np.zeros(nlist + 1, dtype=np.uint32)
        _check(lib().stb_debug_ivfpq_export(self._h, None, None, _np_ptr(list_off), None, None, None))
        m = int(list_off[-1])
        centroids = np.zeros((nlist, STB_DIM), dtype=np.float32)
        codebooks = np.zeros((32, 256, 8), dtype=np.float32)
        order = np.zeros(max(m, 1), dtype=np.uint32)
        codes = np.zeros((max(m, 1), 32), dtype=np.uint8)
        forced = np.zeros(max(n - m, 1), dtype=np.uint32)
        _check(lib().stb_debug_ivfpq_export(self._h, _np_ptr(centroids), _np_ptr(codebooks), _np_ptr(list_off),
                                            _np_ptr(order), _np_ptr(codes), _np_ptr(forced)))
        return {"centroids": centroids, "codebooks": codebooks, "list_off": list_off, "order": order[:m],
                "codes": codes[:m], "forced": forced[: n - m]}

    def search_dev(self, q_dev: int, nprobe: int, top_k: int, rerank: int, out_hits_dev: int, out_status_dev: int):
        """stb_ivfpq_search_dev: asynchronous, everything stays in HBM."""
        _check(lib().stb_ivfpq_search_dev(self._h, vp(q_dev), nprobe, top_k, rerank, vp(out_hits_dev), vp(out_status_dev)))

    def search_batch(self, queries, nprobe: int = 64, top_k: int = 10, rerank: int = 256):
        """stb_ivfpq_search_batch: (hits [nq, top_k] of HIT_DTYPE, padded with (+inf, UINT64_MAX);
        n [nq] hit counts; scanned [nq] codes scanned)."""
        queries = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, STB_DIM)
        nq = queries.shape[0]
        out = np.zeros((nq, top_k), dtype=HIT_DTYPE)
        n = np.zeros(nq, dtype=np.uint32)
        scanned = np.zeros(nq, dtype=np.uint64)
        _check(lib().stb_ivfpq_search_batch(self._h, _np_ptr(queries), nq, nprobe, top_k, rerank,
                                            _np_ptr(out) if out.size else None, _np_ptr(n), _np_ptr(scanned)))
        return out, n, scanned

    def search_filtered(self, queries, row_ranges=None, max_distance: float | None = None, nprobe: int = 64,
                        top_k: int = 10, rerank: int = 256):
        """stb_ivfpq_search_filtered: search_batch restricted to the rows of row_ranges ((n, 2) global
        [begin, end) pairs as Corpus.search takes them; None = every indexed row, empty = no row), with an
        optional distance cap.  Returns (hits [nq, top_k] padded with (+inf, UINT64_MAX), n [nq] hit counts,
        scanned [nq] eligible codes scanned)."""
        queries = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, STB_DIM)
        nq = queries.shape[0]
        rr, n_rr = None, 0
        if row_ranges is not None:
            rr = np.ascontiguousarray(row_ranges, dtype=np.uint64).reshape(-1, 2)
            n_rr = rr.shape[0]
            if n_rr == 0:
                rr = np.zeros((1, 2), dtype=np.uint64)   # non-null pointer, zero ranges
        out = np.zeros((nq, top_k), dtype=HIT_DTYPE)
        n = np.zeros(nq, dtype=np.uint32)
        scanned = np.zeros(nq, dtype=np.uint64)
        _check(lib().stb_ivfpq_search_filtered(self._h, _np_ptr(queries), nq, nprobe, top_k, rerank,
                                               int(max_distance is not None), float(max_distance or 0.0),
                                               _np_ptr(rr), n_rr, _np_ptr(out) if out.size else None, _np_ptr(n),
                                               _np_ptr(scanned)))
        return out, n, scanned

    def search_subsets(self, queries, subsets, subset_of, max_distance: float | None = None, nprobe: int = 64,
                       top_k: int = 10, rerank: int = 256):
        """stb_ivfpq_search_subsets: search_filtered for a batch whose queries name different subsets.  subsets
        is a list of (n, 2) global [begin, end) range arrays, each distinct subset given once (an empty array is
        the empty subset); query i searches subsets[subset_of[i]].  Returns what search_filtered returns: (hits
        [nq, top_k] padded with (+inf, UINT64_MAX), n [nq] hit counts, scanned [nq] eligible codes scanned)."""
        queries = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, STB_DIM)
        nq = queries.shape[0]
        subset_of = np.ascontiguousarray(subset_of, dtype=np.uint32).reshape(-1)
        if len(subset_of) != nq:
            raise ValueError(f"subset_of has {len(subset_of)} entries for {nq} queries")
        parts = [np.asarray(r, dtype=np.uint64).reshape(-1, 2) for r in subsets]
        offsets = np.zeros(len(parts) + 1, dtype=np.uint64)
        offsets[1:] = np.cumsum([len(r) for r in parts], dtype=np.uint64)
        rr = np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros((0, 2), np.uint64), dtype=np.uint64)
        out = np.zeros((nq, top_k), dtype=HIT_DTYPE)
        n = np.zeros(nq, dtype=np.uint32)
        scanned = np.zeros(nq, dtype=np.uint64)
        _check(lib().stb_ivfpq_search_subsets(self._h, _np_ptr(queries), nq, nprobe, top_k, rerank,
                                              int(max_distance is not None), float(max_distance or 0.0), len(parts),
                                              _np_ptr(offsets), _np_ptr(rr) if rr.size else None, _np_ptr(subset_of),
                                              _np_ptr(out) if out.size else None, _np_ptr(n), _np_ptr(scanned)))
        return out, n, scanned

    def search_threshold(self, queries, nprobe: int = 64, max_distance: float = 0.5, slack: float = 0.0,
                         cap: int | None = None):
        """stb_ivfpq_search_threshold: for each query, every row of its probed lists (and every forced row) with
        distance < max_distance whose ADC score reaches RD_f32((1 - max_distance) - slack).  Starts from a modest
        capacity and retries once with the reported total.  Returns (list of HIT_DTYPE arrays, one per query,
        scanned [nq] codes in the probed lists, reranked [nq] rows re-scored)."""
        queries = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, STB_DIM)
        nq = queries.shape[0]
        if cap is None:
            cap = max(nq, 1) * 64
        offsets = np.zeros(nq + 1, dtype=np.uint64)
        scanned = np.zeros(nq, dtype=np.uint64)
        reranked = np.zeros(nq, dtype=np.uint64)
        while True:
            out = np.zeros(max(cap, 1), dtype=HIT_DTYPE)
            rc = _check(lib().stb_ivfpq_search_threshold(self._h, _np_ptr(queries), nq, nprobe, float(max_distance),
                                                         float(slack), _np_ptr(out), cap, _np_ptr(offsets),
                                                         _np_ptr(scanned), _np_ptr(reranked)), allow_capacity=True)
            if rc == STB_ERR_CAPACITY:
                cap = int(offsets[nq])
                continue
            return [out[int(offsets[i]): int(offsets[i + 1])] for i in range(nq)], scanned, reranked

    def set_threshold_keys(self, keys: int):
        """stb_debug_ivfpq_threshold_keys: candidate keys per launch of search_threshold (0 = the default)."""
        _check(lib().stb_debug_ivfpq_threshold_keys(self._h, keys))

    def search_batch_dev(self, q_dev: int, nq: int, nprobe: int, top_k: int, rerank: int, out_hits_dev: int,
                         out_status_dev: int):
        """stb_ivfpq_search_batch_dev: asynchronous; hits [nq][top_k], status [nq][2] = (hits, codes scanned)."""
        _check(lib().stb_ivfpq_search_batch_dev(self._h, vp(q_dev), nq, nprobe, top_k, rerank, vp(out_hits_dev),
                                                vp(out_status_dev)))

    def batch_last(self, i: int):
        """stb_debug_ivfpq_batch_last: the last batched search's clamped {nq, nprobe, top_k, rerank} and
        query i's coarse scores [nlist], probe list [nprobe] and LUT [32][256]."""
        info = np.zeros(4, dtype=np.uint32)
        _check(lib().stb_debug_ivfpq_batch_last(self._h, i, _np_ptr(info), None, None, None))
        coarse = np.zeros(self.stats()["nlist"], dtype=np.float32)
        probe = np.zeros(max(int(info[1]), 1), dtype=np.uint32)
        lut = np.zeros((32, 256), dtype=np.float32)
        _check(lib().stb_debug_ivfpq_batch_last(self._h, i, None, _np_ptr(coarse), _np_ptr(probe), _np_ptr(lut)))
        return {"nq": int(info[0]), "nprobe": int(info[1]), "top_k": int(info[2]), "rerank": int(info[3]),
                "coarse": coarse, "probe": probe[: int(info[1])], "lut": lut}


class Exchange:
    """stb_xchg: peer-memory exchange buffers for the fused multi-GPU search."""
    HANDLE_BYTES = 64

    def __init__(self, ctx: Context, world: int, rank: int, max_k: int, max_nq: int = 0):
        """max_nq > 0 also allocates the batch area for the sharded K2 exchange (stb_xchg_create_batch)."""
        self.ctx, self.world, self.rank, self.max_k, self.max_nq = ctx, world, rank, max_k, max_nq
        self._h = vp()
        if max_nq:
            _check(lib().stb_xchg_create_batch(ctx._h, world, rank, max_k, max_nq, C.byref(self._h)))
        else:
            _check(lib().stb_xchg_create(ctx._h, world, rank, max_k, C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h and _lib is not None:
            _lib.stb_xchg_destroy(self._h)
            self._h = None

    __del__ = close

    def local_handle(self) -> bytes:
        buf = (C.c_uint8 * self.HANDLE_BYTES)()
        _check(lib().stb_xchg_local_handle(self._h, buf))
        return bytes(buf)

    def connect(self, handles: list):
        """handles[r] = rank r's 64-byte IPC handle (other processes)."""
        blob = b"".join(handles)
        assert len(blob) == self.world * self.HANDLE_BYTES
        buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
        _check(lib().stb_xchg_connect(self._h, buf))

    def connect_local(self, peers: list):
        """peers[r] = the Exchange of rank r living in this process."""
        arr = (vp * self.world)(*[p._h for p in peers])
        _check(lib().stb_xchg_connect_local(self._h, arr))

    def search(self, corpus: "Corpus", q, top_k: int):
        """stb_search_xchg: host query in, merged global hits out; returns (hits, complete)."""
        q = np.ascontiguousarray(q, dtype=np.float32)
        out = np.zeros(max(top_k, 1), dtype=HIT_DTYPE)
        n, ok = u32(0), i32(0)
        _check(lib().stb_search_xchg(self.ctx._h, corpus._h, _np_ptr(q), top_k, self._h, _np_ptr(out), C.byref(n),
                                     C.byref(ok)))
        return out[: n.value], bool(ok.value)

    def search_batch_dev(self, corpus: "Corpus", q_dev: int, nq: int, top_k: int, out_hits_dev: int, out_status_dev: int):
        """stb_search_batch_xchg_dev: K2 on the local shard + fused NVLink exchange + per-query merge."""
        _check(lib().stb_search_batch_xchg_dev(self.ctx._h, corpus._h, vp(q_dev), nq, top_k, self._h, vp(out_hits_dev),
                                               vp(out_status_dev)))

    def search_topk(self, corpus: "Corpus", q_dev: int, top_k: int, out_hits_dev: int, out_status_dev: int):
        """stb_search_topk_xchg: one kernel = scan + NVLink exchange + global merge."""
        _check(lib().stb_search_topk_xchg(self.ctx._h, corpus._h, vp(q_dev), top_k, self._h, vp(out_hits_dev),
                                          vp(out_status_dev)))


def embed_dev(ctx: Context, table: Table, offsets_dev: int, ids_dev: int, n_lines: int, out_dev: int):
    """stb_embed_dev: asynchronous, CSR and output already in HBM."""
    _check(lib().stb_embed_dev(ctx._h, table._h, vp(offsets_dev), vp(ids_dev), n_lines, vp(out_dev)))


def embed_status(ctx: Context):
    """stb_embed_status: sync + raise StbError(STB_ERR_RANGE) if a token was out of range."""
    _check(lib().stb_embed_status(ctx._h))


def embed(ctx: Context, table: Table, offsets, ids, out: bool = True, append_to: Corpus | None = None):
    """stb_embed (K3).  offsets: (n_lines+1,) u64 CSR; ids: u32 token ids."""
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    ids = np.ascontiguousarray(ids, dtype=np.uint32)
    n_lines = offsets.size - 1
    res = np.empty((n_lines, STB_DIM), dtype=np.float32) if out else None
    if ids.size == 0:
        ids = np.zeros(1, dtype=np.uint32)
    _check(lib().stb_embed(ctx._h, table._h, _np_ptr(offsets), _np_ptr(ids), n_lines, _np_ptr(res),
                           append_to._h if append_to is not None else None))
    return res


def embed_text(ctx: Context, tok: Tokenizer, table: Table, lines, max_length: int, out: bool = True,
               append_to: Corpus | None = None):
    """stb_embed_text: the rows of stb_embed from the lines' text (str or UTF-8 bytes), tokenised in the library."""
    text, offsets = pack_lines(lines)
    n_lines = len(lines)
    res = np.empty((n_lines, STB_DIM), dtype=np.float32) if out else None
    _check(lib().stb_embed_text(ctx._h, tok._h, table._h, _np_ptr(text), _np_ptr(offsets), n_lines, max_length,
                                _np_ptr(res), append_to._h if append_to is not None else None))
    return res

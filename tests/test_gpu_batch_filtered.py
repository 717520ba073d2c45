"""GPU: stb_search_batch_filtered, the workspace query (stb_search in store-query mode) for a batch.

Every query of a call must equal, bit for bit, what stb_search returns for it alone (hits, order, count, the
padded tail), and the oracle's orc_store_search where the corpus is small.  Filtered v2 (route 3) is checked
against its own approximate scores, as tests/test_gpu_batch_contract.py checks v2: stb_debug_batch_gemm gives
the score matrix the epilogues see, and from its eligible entries the tests predict the sample, every
threshold, every emission count and which queries need the single-query path.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest

import oracle
from conftest import unit_rows
from semtools_b200 import capi

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_BATCH = open(os.path.join(ROOT, "semtools_b200", "csrc", "batch_scan.cu")).read()
_API = open(os.path.join(ROOT, "semtools_b200", "csrc", "api.cu")).read()
SEG_CAP = int(re.search(r"constexpr\s+uint32_t\s+kSegCap\s*=\s*(\d+)", _API).group(1))
F2_KEYS = int(re.search(r"#define\s+STB_F2_KEYS\s+(\d+)", _BATCH).group(1))
F2_RESCORE = int(re.search(r"#define\s+STB_F2_RESCORE\s+(\d+)", _BATCH).group(1))
TILE = 256
NO_ROW = 0xFFFFFFFFFFFFFFFF
KS = (1, 10, 64, 65, 200)
CAPS = (None, 0.0, 0.3, 100.0, 1e9, -1.0, float("nan"), float("inf"))


@pytest.fixture(scope="module")
def sm_count():
    torch = pytest.importorskip("torch")
    return torch.cuda.get_device_properties(0).multi_processor_count


def new_corpus(ctx, rows, row_base=0):
    c = capi.Corpus(ctx, max(len(rows), 1), row_base=row_base)
    c.append(rows)
    return c


def k1(c, q, k, cap, ranges):
    return c.search(q, top_k=k, max_distance=cap, mode=capi.STB_MODE_STORE_QUERY, row_ranges=ranges)


def same(a, b, where=""):
    assert a["row"].tolist() == b["row"].tolist(), where
    assert np.array_equal(a["distance"].view(np.uint64), b["distance"].view(np.uint64)), where


def raw_call(ctx, c, queries, k, cap, rr, n_rr, out=None, cnt=None):
    """The C entry point on preset output buffers: (status, hits [nq][k], counts [nq])."""
    queries = np.ascontiguousarray(queries, dtype=np.float32)
    nq = len(queries)
    out = np.zeros((nq, max(k, 1)), dtype=capi.HIT_DTYPE) if out is None else out
    cnt = np.zeros(max(nq, 1), dtype=np.uint32) if cnt is None else cnt
    vp = C.c_void_p
    rc = capi.lib().stb_search_batch_filtered(ctx._h, c._h, queries.ctypes.data_as(vp), nq, k, int(cap is not None),
                                              float(cap or 0.0), None if rr is None else rr.ctypes.data_as(vp), n_rr,
                                              out.ctypes.data_as(vp), cnt.ctypes.data_as(vp))
    return rc, out, cnt


def check_batch(ctx, c, queries, k, cap, ranges, where=""):
    """The batch against per-query stb_search, the padded tail included; returns the hit lists."""
    rr = None if ranges is None else np.ascontiguousarray(ranges, dtype=np.uint64).reshape(-1, 2)
    n_rr = 0 if rr is None else len(rr)
    if rr is not None and n_rr == 0:
        rr = np.zeros((1, 2), np.uint64)
    rc, out, cnt = raw_call(ctx, c, queries, k, cap, rr, n_rr)
    assert rc == 0, capi.lib().stb_last_error()
    res = []
    for i, q in enumerate(queries):
        exp = k1(c, q, k, cap, ranges)
        got = out[i, : cnt[i]]
        same(got, exp, f"{where} k={k} cap={cap} query {i}")
        if k:
            assert np.all(out[i, cnt[i]:]["distance"] == np.inf) and np.all(out[i, cnt[i]:]["row"] == NO_ROW), where
        res.append(got)
    return res


# ------------------------------------------------------------------ the route rule, restated ---
def listed_tiles(ranges, n, row_base=0):
    """api.cu stb_search_batch_filtered: the tiles a clipped range touches, ascending."""
    if ranges is None:
        ranges = [[row_base, row_base + n]]
    out = []
    for b, e in np.asarray(ranges, dtype=np.uint64).reshape(-1, 2).tolist():
        b, e = max(b, row_base) - row_base, min(e, row_base + n) - row_base
        if b < e:
            for t in range(b // TILE, (e - 1) // TILE + 1):
                if not out or out[-1] < t:
                    out.append(t)
    return np.array(out, dtype=np.int64)


def local_ranges(ranges, n, row_base=0):
    """The ranges clipped to the shard, in local rows (the oracle takes rows inside its matrix only)."""
    if ranges is None:
        return np.array([[0, n]], np.uint64)
    r = np.clip(np.asarray(ranges, dtype=np.int64).reshape(-1, 2) - row_base, 0, n)
    return r[r[:, 0] < r[:, 1]].astype(np.uint64)


def eligible_mask(ranges, n, row_base=0):
    m = np.zeros(n, bool)
    if ranges is None:
        m[:] = True
        return m
    for b, e in np.asarray(ranges, dtype=np.uint64).reshape(-1, 2).tolist():
        b, e = max(b, row_base) - row_base, min(e, row_base + n) - row_base
        if b < e:
            m[b:e] = True
    return m


def route_rule(n_listed, k, sm):
    """batch_v2_plan over the listed tiles: route 3 and its sample, else route 4 (K1 answers)."""
    f16, _ = capi.batch_params()
    n_sample = min(n_listed, min(4 * sm, 608))
    margin_factor = 2 if f16 else 4

    def expected_emitted(ns):
        return k * margin_factor * (-(-n_listed // ns)) if ns else 0
    if expected_emitted(n_sample) > 2048:
        n_sample = min(min(n_listed, 8192), (n_listed // 64 + sm - 1) // sm * sm)
    if k <= 64 and n_sample >= k and expected_emitted(n_sample) <= 2048:
        return {"route": 3, "n_sample": n_sample, "stride": n_listed // n_sample, "n_seg": min(n_listed, sm),
                "seg_cap": SEG_CAP}
    return {"route": 4, "n_sample": 0, "stride": 0, "n_seg": 0, "seg_cap": 0}


def debug_scores(ctx, queries, rows):
    queries = np.ascontiguousarray(queries, dtype=np.float32)
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    nq, n = len(queries), len(rows)
    full = np.zeros((-(-nq // 128) * 128, -(-n // TILE) * TILE), dtype=np.float32)
    vp = C.c_void_p
    capi._check(capi.lib().stb_debug_batch_gemm(ctx._h, queries.ctypes.data_as(vp), nq, rows.ctypes.data_as(vp), n,
                                                full.ctypes.data_as(vp), None))
    return full[:nq, :n]


def predict(A, elig, listed, k, info):
    """Filtered v2 from the approximate scores A [nq][n]: thresholds, emission counts [nq][n_seg], proof flags."""
    _, eps = capi.batch_params()
    nq, n = A.shape
    ns, stride, n_seg = info["n_sample"], info["stride"], info["n_seg"]
    two_eps = np.float32(2.0) * np.float32(eps)
    Am = np.where(elig[None, :], A, -np.inf).astype(np.float32)           # the sampling epilogue's mask
    pad = np.full((nq, -(-n // TILE) * TILE - n), -np.inf, np.float32)    # padding rows are never eligible
    tiles = np.concatenate([Am, pad], axis=1).reshape(nq, -1, TILE)
    s_k = np.sort(tiles[:, listed[np.arange(ns) * stride]].max(axis=2), axis=1)[:, ns - k]
    thr = (s_k.astype(np.float32) - two_eps).astype(np.float32)
    seg_of_tile = np.full(-(-n // TILE), -1)
    seg_of_tile[listed] = np.arange(len(listed)) % n_seg
    seg_of = seg_of_tile[np.arange(n) // TILE]
    cnt = np.zeros((nq, n_seg), dtype=np.int64)
    proven = np.zeros(nq, dtype=bool)
    for q in range(nq):
        emit = elig & (A[q] >= thr[q])
        cnt[q] = np.bincount(seg_of[emit], minlength=n_seg)
        sc = A[q][emit]
        m2 = len(sc)
        if len(sc) >= k:
            m2 = int(np.count_nonzero(sc >= np.float32(np.sort(sc)[len(sc) - k]) - two_eps))
        proven[q] = not ((cnt[q] > SEG_CAP).any() or len(sc) > F2_KEYS) and m2 <= F2_RESCORE
    return thr, cnt, proven


def check_route(ctx, sm, c, rows, queries, k, ranges, row_base=0, require_all_proven=False):
    """Route, sample and, for route 3, thresholds, counts and the K1 fallbacks against the restatement."""
    n = len(rows)
    listed = listed_tiles(ranges, n, row_base)
    exp = route_rule(len(listed), k, sm)
    before = ctx.counters()["fallback_searches"]
    c.search_batch_filtered(queries, ranges, top_k=k)
    fell = ctx.counters()["fallback_searches"] - before
    info = ctx.batch_last()
    assert {key: info[key] for key in exp} == exp and info["nq"] == len(queries), (info, exp)
    if exp["route"] == 4:
        assert fell >= len(queries)
        return info
    elig = eligible_mask(ranges, n, row_base)
    A = debug_scores(ctx, queries, rows)
    thr, cnt, proven = predict(A, elig, listed, k, info)
    assert np.array_equal(info["thr"].view(np.uint32), thr.view(np.uint32)), np.flatnonzero(info["thr"] != thr)[:8]
    assert np.array_equal(info["cand_cnt"].astype(np.int64), cnt), np.argwhere(info["cand_cnt"] != cnt)[:8]
    unproven = int((~proven).sum())
    assert unproven <= fell <= 2 * unproven, (unproven, fell)
    if require_all_proven:
        assert fell == 0
    return info


# ------------------------------------------------------------------ corpora and filters ---
def corpus_of(kind, rng, n):
    if kind == "duplicated":
        base = unit_rows(rng, max(n // 8, 1))
        return np.ascontiguousarray(base[rng.integers(0, len(base), n)])
    return unit_rows(rng, n)


def doc_ranges(rng, n, frac, row_base=0, mean_len=30):
    """A random subset of `documents` (consecutive lines, lognormal lengths) merged into ranges."""
    lens = np.clip(np.round(rng.lognormal(np.log(mean_len), 0.8, n)), 1, 200).astype(np.int64)
    starts = np.concatenate([[0], np.cumsum(lens)])
    starts = starts[starts < n]
    ends = np.append(starts[1:], n)
    keep = rng.random(len(starts)) < frac
    m = np.zeros(n, bool)
    for b, e in zip(starts[keep], ends[keep]):
        m[b:e] = True
    edges = np.flatnonzero(np.diff(np.concatenate([[0], m.astype(np.int8), [0]])))
    return (edges.reshape(-1, 2) + row_base).astype(np.uint64)


def filter_of(name, rng, n, row_base=0):
    if name == "none":
        return None
    if name == "all":
        return np.array([[row_base, row_base + n]], np.uint64)
    if name == "docs":
        return doc_ranges(rng, n, 0.3, row_base)
    if name == "one_tile":
        return np.array([[row_base + 5 * TILE + 17, row_base + 5 * TILE + 90]], np.uint64)
    if name == "straddle":
        edges = [t * TILE for t in range(1, n // TILE, 3)]
        return np.array([[row_base + e - 7, row_base + e + 9] for e in edges], np.uint64)
    if name == "past_end":
        return np.array([[row_base + n // 3, row_base + n // 3 + 500], [row_base + n - 300, row_base + n + 10_000],
                         [row_base + n + 20_000, row_base + n + 30_000]], np.uint64)
    raise ValueError(name)


PARITY = [("random", 40_000, "none"), ("random", 40_000, "all"), ("duplicated", 40_000, "docs"),
          ("random", 40_000 + 77, "one_tile"), ("random", 30 * TILE + 131, "straddle"),
          ("duplicated", 40_000 + 77, "past_end"), ("random", 40_000 + 77, "docs")]


@pytest.mark.parametrize("kind,n,flt", PARITY)
def test_parity_with_single_query_search(ctx, sm_count, kind, n, flt):
    rng = np.random.default_rng(n + len(flt) * 7 + len(kind))
    rows = corpus_of(kind, rng, n)
    ranges = filter_of(flt, rng, n)
    queries = unit_rows(rng, 9)
    elig = np.flatnonzero(eligible_mask(ranges, n))
    queries[0] = rows[elig[-1]]                                   # an eligible row in the last listed tile
    queries[1] = rows[elig[len(elig) // 2]] * np.float32(3.0)
    queries[2] = rows[0]                                          # row 0: eligible only for some filters
    c = new_corpus(ctx, rows)
    for k in KS:
        for cap in (CAPS if k == 10 else (None, 0.3, float("nan"))):
            res = check_batch(ctx, c, queries, k, cap, ranges, where=f"{kind}/{flt}")
        check_route(ctx, sm_count, c, rows, queries, k, ranges, require_all_proven=(kind == "random" and k <= 64
                                                                                    and flt not in ("one_tile",)))
        if k in (10, 65):
            for i in (0, 1, 5):
                r, d32 = oracle.store_search(rows, local_ranges(ranges, n), queries[i], k)
                got = c.search_batch_filtered(queries[i:i + 1], ranges, top_k=k)[0]
                assert got["row"].tolist() == [int(x) for x in r], (flt, k, i)
                assert np.array_equal(got["distance"].astype(np.float32), d32), (flt, k, i)
    assert len(res) == len(queries)


def test_shard_with_row_base(ctx, sm_count):
    rng = np.random.default_rng(17)
    row_base = 5_000_000_000
    n = 60 * TILE + 33
    rows = unit_rows(rng, n)
    docs = doc_ranges(rng, n, 0.4, row_base)
    ranges = np.concatenate([np.array([[row_base - 5000, row_base - 4000], [row_base - 1000, row_base + 300]], np.uint64),
                             docs[docs[:, 0] >= row_base + 300],                      # clipped at both ends of the shard
                             np.array([[row_base + n + 5, row_base + n + 9]], np.uint64)])
    queries = unit_rows(rng, 6)
    queries[0] = rows[100]
    c = new_corpus(ctx, rows, row_base=row_base)
    for k in (1, 10, 64, 65):
        for cap in (None, 0.2, float("inf")):
            check_batch(ctx, c, queries, k, cap, ranges, where="row_base")
        check_route(ctx, sm_count, c, rows, queries, k, ranges, row_base=row_base, require_all_proven=k <= 64)
    r, d32 = oracle.store_search(rows, local_ranges(ranges, n, row_base), queries[0], 10)
    got = c.search_batch_filtered(queries[:1], ranges, top_k=10)[0]
    assert got["row"].tolist() == [int(x) + row_base for x in r]
    assert np.array_equal(got["distance"].astype(np.float32), d32)


# ------------------------------------------------------------------ the mask ---
def at_cos(q, cos, rng, m=1):
    u = rng.standard_normal((m, 256))
    qq = q.astype(np.float64)
    u -= np.outer(u @ qq, qq)
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    x = cos * qq[None, :] + np.sqrt(1.0 - cos * cos) * u
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


@pytest.mark.parametrize("k", [1, 10, 64])
def test_adversarial_filter_is_proven_on_the_eligible_rows(ctx, sm_count, k):
    """The first half of every tile is eligible, the second half holds, for every query, an exact copy and rows
    at cosine 0.99: better than any eligible row.  Without the mask in the sampling epilogue the threshold
    would sit near 0.99 and the eligible top-k would be proven empty; without it in the emitting epilogue the
    copies would be returned.  Every query must be proven on route 3 and equal stb_search."""
    rng = np.random.default_rng(900 + k)
    n_tiles = 2 * sm_count + 40
    n = n_tiles * TILE
    rows = unit_rows(rng, n)
    queries = unit_rows(rng, 12)
    for t in range(n_tiles):
        for j, q in enumerate(queries):
            rows[t * TILE + 128 + 2 * j] = q if t % 7 == 0 else at_cos(q, 0.99, rng)[0]
            rows[t * TILE + 129 + 2 * j] = at_cos(q, 0.995, rng)[0]
    ranges = np.array([[t * TILE, t * TILE + 128] for t in range(n_tiles)], np.uint64)
    c = new_corpus(ctx, rows)
    before = ctx.counters()["fallback_searches"]
    got = c.search_batch_filtered(queries, ranges, top_k=k)
    assert ctx.counters()["fallback_searches"] == before, "filtered v2 left a query unproven"
    info = ctx.batch_last()
    assert info["route"] == 3, info
    for i, q in enumerate(queries):
        exp = k1(c, q, k, None, ranges)
        same(got[i], exp, f"query {i}")
        assert np.all(got[i]["row"] % TILE < 128) and len(got[i]) == k
        r, d32 = oracle.store_search(rows, ranges, q, k)
        assert got[i]["row"].tolist() == [int(x) for x in r]
    check_route(ctx, sm_count, c, rows, queries, k, ranges, require_all_proven=True)


# ------------------------------------------------------------------ routes x shapes ---
@pytest.mark.parametrize("n,frac,k,nq", [(70_000, 1.0, 10, 130), (140_000 + 5, 0.25, 10, 130), (140_000, 0.05, 16, 130),
                                         (200_000, 0.01, 10, 130), (64 * TILE + 200, 0.5, 64, 130),
                                         (300 * TILE + 7, 0.1, 1, 130), (400_000, 0.5, 10, 100)])
def test_route_contract_on_document_filters(ctx, sm_count, n, frac, k, nq):
    rng = np.random.default_rng(int(n * frac) + k)
    rows = unit_rows(rng, n)
    ranges = doc_ranges(rng, n, frac)
    queries = unit_rows(rng, nq)
    elig = np.flatnonzero(eligible_mask(ranges, n))
    queries[7] = rows[elig[0]]
    queries[nq - 1] = rows[elig[-1]]
    c = new_corpus(ctx, rows)
    route = route_rule(len(listed_tiles(ranges, n)), k, sm_count)["route"]
    # k = 64 over about 64 listed tiles samples them all and may overflow a capacity: the restatement says
    # which queries, and the fallback count must match it
    check_route(ctx, sm_count, c, rows, queries, k, ranges, require_all_proven=route == 3 and k <= 16)
    ids = sorted({0, 7, nq - 1} | {i for i in (127, 128) if i < nq} | set(rng.choice(nq, 10, replace=False).tolist()))
    check_batch(ctx, c, queries[ids], k, None, ranges, where=f"docs {frac}")


def test_route_boundary_listed_tiles_equal_k(ctx, sm_count):
    """n_listed == k samples every listed tile (route 3, stride 1); n_listed == k - 1 leaves it to K1."""
    rng = np.random.default_rng(77)
    n = 200 * TILE
    rows = unit_rows(rng, n)
    c = new_corpus(ctx, rows)
    queries = unit_rows(rng, 5)
    for k, n_listed, route in [(16, 16, 3), (17, 16, 4), (64, 64, 3), (64, 63, 4)]:
        tiles = np.sort(rng.choice(200, n_listed, replace=False))
        ranges = np.array([[t * TILE + 3, t * TILE + 40] for t in tiles], np.uint64)
        info = check_route(ctx, sm_count, c, rows, queries, k, ranges, require_all_proven=route == 3)
        assert info["route"] == route and (route == 4 or (info["n_sample"] == n_listed and info["stride"] == 1))
        check_batch(ctx, c, queries, k, None, ranges, where=f"{n_listed} listed")


# ------------------------------------------------------------------ arguments and edges ---
def test_argument_rules(ctx):
    rng = np.random.default_rng(5)
    rows = unit_rows(rng, 5000)
    c = new_corpus(ctx, rows)
    q = unit_rows(rng, 3)
    good = np.array([[10, 2000]], np.uint64)
    rc, _, _ = raw_call(ctx, c, q[:0], 10, None, good, 1)                                 # nq = 0
    assert rc == 0
    rc, _, cnt = raw_call(ctx, c, q, 0, None, good, 1, cnt=np.full(3, 9, np.uint32))      # top_k = 0
    assert rc == 0 and cnt.tolist() == [0, 0, 0]
    assert capi.lib().stb_search_batch_filtered(ctx._h, c._h, q.ctypes.data_as(C.c_void_p), 3, 10, 0, 0.0, None, 2,
                                                None, None) == capi.STB_ERR_ARG           # NULL with n_ranges > 0
    assert ctx.batch_last()["route"] == 4
    empty = c.search_batch_filtered(q, np.zeros((0, 2), np.uint64), top_k=10)          # the empty subset
    assert [len(h) for h in empty] == [0, 0, 0]
    rc, out, cnt = raw_call(ctx, c, q, 10, None, np.zeros((1, 2), np.uint64), 0)
    assert rc == 0 and cnt.tolist() == [0, 0, 0] and np.all(out["row"] == NO_ROW) and np.all(out["distance"] == np.inf)
    for bad in ([[100, 50]], [[0, 100], [50, 200]], [[300, 400], [0, 10]]):            # refused ranges
        bad = np.array(bad, np.uint64)
        exp = capi.lib().stb_search(ctx._h, c._h, q[0].ctypes.data_as(C.c_void_p), 10, 0, 0.0, capi.STB_MODE_STORE_QUERY,
                                    bad.ctypes.data_as(C.c_void_p), len(bad), None, 0, C.byref(C.c_uint64(0)))
        out0 = np.zeros((3, 10), dtype=capi.HIT_DTYPE)
        out0["distance"] = 0.125
        out0["row"] = 42
        cnt0 = np.full(3, 7, np.uint32)
        rc, out, cnt = raw_call(ctx, c, q, 10, None, bad, len(bad), out=out0.copy(), cnt=cnt0.copy())
        assert rc == exp == capi.STB_ERR_RANGE
        assert np.array_equal(out, out0) and np.array_equal(cnt, cnt0)
    for k in (1, 10, 1500):                                                              # any top_k
        check_batch(ctx, c, q, k, None, good, where="any k")
    check_batch(ctx, c, q, 10, 0.9, None, where="NULL ranges")


def test_bad_queries_equal_single_query_search(ctx, sm_count):
    rng = np.random.default_rng(31)
    n = 70_000
    rows = unit_rows(rng, n)
    ranges = doc_ranges(rng, n, 0.5)
    queries = list(unit_rows(rng, 10))
    nan = unit_rows(rng, 1)[0]; nan[7] = np.nan
    inf = unit_rows(rng, 1)[0]; inf[3] = np.inf
    queries += [np.zeros(256, np.float32), nan, inf, rows[11] * np.float32(1e-25), rows[12] * np.float32(1e20),
                rows[13] * np.float32(1e-20)]
    queries = np.ascontiguousarray(np.stack(queries), dtype=np.float32)
    c = new_corpus(ctx, rows)
    for k in (10, 64):
        check_batch(ctx, c, queries, k, None, ranges, where="bad queries")
        check_batch(ctx, c, queries, k, 0.8, ranges, where="bad queries, cap")
    assert ctx.batch_last()["route"] == 3


def test_unnormalisable_corpus_row_goes_to_k1(ctx):
    rng = np.random.default_rng(32)
    n = 50_000
    rows = unit_rows(rng, n)
    rows[1234] *= np.float32(1e25)                                 # squared norm overflows fp32
    ranges = doc_ranges(rng, n, 0.5)
    queries = unit_rows(rng, 6)
    queries[0] = rows[1234] / np.float32(1e25)
    c = new_corpus(ctx, rows)
    check_batch(ctx, c, queries, 10, None, ranges, where="bad row")
    check_batch(ctx, c, queries, 10, None, None, where="bad row, no filter")
    assert ctx.batch_last()["route"] == 4


# ------------------------------------------------------------------ corpus changes ---
def test_after_append_update_and_remove(ctx, sm_count):
    rng = np.random.default_rng(41)
    rows = unit_rows(rng, 80 * TILE + 300)
    queries = unit_rows(rng, 8)
    queries[0] = rows[80 * TILE + 299]
    c = capi.Corpus(ctx, len(rows))
    c.append(rows[: 50 * TILE + 130])
    ranges = doc_ranges(rng, len(rows), 0.4)
    check_batch(ctx, c, queries, 10, None, ranges, where="prefix")
    c.append(rows[50 * TILE + 130:])                               # the shadow is extended behind a ragged tile
    check_batch(ctx, c, queries, 10, None, ranges, where="append")
    check_route(ctx, sm_count, c, rows, queries, 10, ranges, require_all_proven=True)
    idx = np.sort(rng.choice(len(rows), 300, replace=False)).astype(np.uint64)
    new = unit_rows(rng, 300)
    new[0] = queries[1]
    c.update(idx, new)
    rows[idx.astype(np.int64)] = new
    check_batch(ctx, c, queries, 10, 0.9, ranges, where="update")
    check_route(ctx, sm_count, c, rows, queries, 10, ranges, require_all_proven=True)
    c.remove(np.array([[100, 4000], [20_000, 20_001]], np.uint64))
    rows = np.delete(rows, np.r_[100:4000, 20_000], axis=0)
    assert len(c) == len(rows)
    check_batch(ctx, c, queries, 10, None, ranges, where="remove")
    check_route(ctx, sm_count, c, rows, queries, 10, ranges, require_all_proven=True)


# ------------------------------------------------------------------ the workspace store ---
def test_store_batch_equals_single_queries(ctx, monkeypatch, tmp_path):
    from semtools_b200.workspace import LineEmbedding, Store
    monkeypatch.setenv("HOME", str(tmp_path))
    rng = np.random.default_rng(51)
    ws_dir = tmp_path / ".semtools" / "workspaces" / "batch"
    ws_dir.mkdir(parents=True)
    s = Store.open(str(ws_dir), ctx)
    paths = [f"/docs/f{i}.txt" for i in range(60)]
    lines = []
    for p in paths:
        for ln in range(int(rng.integers(5, 400))):
            lines.append(LineEmbedding(p, ln, unit_rows(rng, 1)[0]))
    s.upsert_line_embeddings(lines)
    queries = unit_rows(rng, 20)
    queries[0] = lines[len(lines) // 2].embedding
    for subset, k, cap in [(paths[::3], 10, None), (paths[5:9], 3, 0.9), (paths, 64, None), ([], 10, None),
                           (["/nope.txt"], 10, None), (paths[:2], 0, None), (paths[10:40], 200, 0.95)]:
        got = s.search_line_embeddings_batch(queries, subset, k, cap)
        assert len(got) == len(queries)
        for i, q in enumerate(queries):
            assert got[i] == s.search_line_embeddings(q, subset, k, cap), (subset[:2], k, cap, i)

"""GPU: stb_search_batch_threshold, threshold mode of search_documents for a whole batch (route 5).

Every query of a call must equal, bit for bit (rows, order, f64 distances), what stb_search returns for it alone
in threshold mode, and the oracle's where the corpus is small.  The emission pass is checked against its own
approximate scores: stb_debug_batch_gemm gives the score matrix the epilogue sees, and from it the tests predict
every per-(query, CTA) count from the documented threshold.  Every route is reached through the data.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest

import oracle
from conftest import unit_rows
from semtools_b200 import capi
from semtools_b200.search import SearchConfig, Searcher

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_API = open(os.path.join(ROOT, "semtools_b200", "csrc", "api.cu")).read()
_HDR = open(os.path.join(ROOT, "include", "semtools_b200.h")).read()
DELTA = float(re.search(r"#define\s+STB_THR_DELTA\s+(\S+)", _API).group(1))
SEG_CAP = int(re.search(r"#define\s+STB_THR_SEG_CAP\s+(\d+)u", _API).group(1))
BUDGET = eval(re.search(r"#define\s+STB_BATCH_THRESHOLD_RETRY_KEYS\s+\((\S+ << \d+)\)", _HDR).group(1).replace("ull", ""))
TILE = 256
NQS = (1, 127, 128, 129, 300)


@pytest.fixture(scope="module")
def sm_count():
    torch = pytest.importorskip("torch")
    return torch.cuda.get_device_properties(0).multi_processor_count


def new_corpus(ctx, rows, row_base=0):
    c = capi.Corpus(ctx, max(len(rows), 1), row_base=row_base)
    c.append(rows)
    return c


def raw_call(ctx, c, queries, m, cap, hits=True, offsets=True):
    """The C entry point: (status, hits [cap], offsets [nq + 1])."""
    queries = np.ascontiguousarray(queries, dtype=np.float32)
    nq = len(queries)
    out = np.zeros(max(cap, 1), dtype=capi.HIT_DTYPE)
    off = np.full(nq + 1, 12345, dtype=np.uint64)
    vp = C.c_void_p
    rc = capi.lib().stb_search_batch_threshold(ctx._h, c._h, queries.ctypes.data_as(vp) if nq else None, nq, float(m),
                                               out.ctypes.data_as(vp) if hits else None, cap,
                                               off.ctypes.data_as(vp) if offsets else None)
    return rc, out, off


def k1(c, q, m):
    return c.search(q, top_k=0, max_distance=m)


def same(a, b, where=""):
    assert len(a) == len(b), f"{where}: {len(a)} hits, expected {len(b)}"
    assert a["row"].tolist() == b["row"].tolist(), where
    assert np.array_equal(a["distance"].view(np.uint64), b["distance"].view(np.uint64)), where


def expected_thr(m, eps):
    """The documented emission threshold: ((1 - M) - EPS) - delta in f64, rounded toward -inf to f32."""
    x = ((np.float64(1.0) - np.float64(m)) - np.float64(eps)) - np.float64(DELTA)
    f = np.float32(x)
    if np.float64(f) > x:
        f = np.nextafter(f, np.float32(-np.inf))
    return f


def check_batch(ctx, c, queries, m, refs=None, where=""):
    """The batch against per-query stb_search (refs: precomputed per-query results); returns stb_debug_batch_last."""
    got = c.search_batch_threshold(queries, m)
    info = ctx.batch_last()
    assert info["route"] == 5 and info["nq"] == len(queries)
    for i, q in enumerate(queries):
        same(got[i], refs[i] if refs is not None else k1(c, q, m), f"{where} M={m!r} query {i}")
    return info


# ------------------------------------------------------------------------------------------------ corpora ---
def bench_like(rng, n):
    """Unit rows with 0.1 % duplicated rows and 0.01 % zero rows."""
    rows = unit_rows(rng, n)
    nd = max(1, n // 1000)
    rows[rng.choice(n, nd, replace=False)] = rows[rng.choice(n, nd, replace=False)]
    rows[rng.choice(n, max(1, n // 10000), replace=False)] = 0.0
    return rows


def clustered(rng, n, k=40, spread=0.08):
    centres = unit_rows(rng, k)
    x = centres[rng.integers(0, k, n)] + spread * rng.standard_normal((n, 256)).astype(np.float32) / 16
    return np.ascontiguousarray(x / np.linalg.norm(x, axis=1, keepdims=True), dtype=np.float32)


def queries_for(rng, rows, nq):
    """Half perturbed corpus rows, half exact corpus rows (their duplicates tie), one fresh random row."""
    idx = rng.integers(0, len(rows), nq)
    q = rows[idx].copy()
    h = nq // 2
    q[:h] += 0.02 * rng.standard_normal((h, 256)).astype(np.float32) / 16
    q[-1] = unit_rows(rng, 1)[0]
    q[np.linalg.norm(q, axis=1) == 0] = unit_rows(rng, 1)[0]          # zero queries have their own test
    return np.ascontiguousarray(q, dtype=np.float32)


def thresholds(rows, queries):
    """tiny (duplicates only), ~10 and ~1000 hits per query, 1.0, nextafter(1.0, 2), 2.0, +inf."""
    q = queries[: min(16, len(queries))].astype(np.float64)
    r = rows.astype(np.float64)
    rn = np.linalg.norm(r, axis=1)
    d = 1.0 - (q @ r.T) / np.maximum(np.linalg.norm(q, axis=1)[:, None] * rn[None, :], 1e-300)
    d = np.sort(d, axis=1)
    return [1e-12, float(np.median(d[:, 10])), float(np.median(d[:, min(1000, d.shape[1] - 1)])), 1.0,
            float(np.nextafter(1.0, 2.0)), 2.0, float("inf")]


CORPORA = {"bench": lambda rng: bench_like(rng, 20000 + 77), "clustered": lambda rng: clustered(rng, 12000),
           "ragged": lambda rng: bench_like(rng, 3 * TILE + 37)}


@pytest.mark.parametrize("kind", sorted(CORPORA))
def test_parity_with_k1_and_oracle(ctx, kind):
    rng = np.random.default_rng({"bench": 11, "clustered": 12, "ragged": 13}[kind])
    rows = CORPORA[kind](rng)
    c = new_corpus(ctx, rows)
    queries = queries_for(rng, rows, max(NQS))
    small = len(rows) < 1000
    for m in thresholds(rows, queries):
        refs = [k1(c, q, m) for q in queries]
        if small:
            for i in range(0, len(queries), 37):
                r, d = oracle.search_rows(rows, queries[i], 0, m)
                assert refs[i]["row"].tolist() == [int(x) for x in r], (kind, m, i)
                assert np.array_equal(refs[i]["distance"].view(np.uint64), np.asarray(d, np.float64).view(np.uint64))
        for nq in NQS:
            info = check_batch(ctx, c, queries[:nq], m, refs[:nq], f"{kind} nq={nq}")
            assert info["n_seg"] > 0 and info["k1"] == 0, info


# ------------------------------------------------------------------------------------------------ boundary ---
def at_cos(q, cos, rng):
    """A row at cosine ~cos to the unit query q."""
    u = rng.standard_normal(256)
    u -= (u @ q) * q
    u /= np.linalg.norm(u)
    return (cos * q + np.sqrt(max(0.0, 1 - cos * cos)) * u).astype(np.float32)


def test_boundary_is_strict_and_loses_nothing(ctx):
    rng = np.random.default_rng(21)
    f16, eps = capi.batch_params()
    q = unit_rows(rng, 1)[0].astype(np.float64)
    cosines = [0.999, 0.95, 0.7, 0.3, 0.05, 0.0, -0.2]
    # rows whose canonical distance sits on an f32 rounding edge of thr: 1 - M - EPS - delta = an f32 value
    for t in (np.float32(0.5), np.float32(0.25), np.float32(-0.125)):
        for nb in (np.nextafter(t, np.float32(-1)), t, np.nextafter(t, np.float32(1))):
            cosines.append(float(nb) + eps + DELTA)
    planted = np.stack([at_cos(q, cs, rng) for cs in cosines])
    rows = np.concatenate([unit_rows(rng, 3000), planted])
    rows = rows[rng.permutation(len(rows))]
    c = new_corpus(ctx, rows)
    qf = q.astype(np.float32)
    queries = np.stack([qf] * 3 + [unit_rows(rng, 1)[0]])
    for p in planted:
        ri = int(np.flatnonzero((rows == p).all(axis=1))[0])
        m = float(oracle.search_rows(rows[ri: ri + 1], qf, 0, 1e9)[1][0])      # canonical distance of the planted row
        for mm, present in ((m, False), (float(np.nextafter(m, np.inf)), True)):
            if mm <= 0:
                continue
            got = c.search_batch_threshold(queries, mm)
            info = ctx.batch_last()
            assert (ri in got[0]["row"].tolist()) == present, (m, mm, present)
            assert info["k1"] == 0
            assert np.float32(info["thr"][0]).tobytes() == expected_thr(mm, eps).tobytes()
            for i in range(len(queries)):
                same(got[i], k1(c, queries[i], mm), f"M={mm!r} query {i}")


# ------------------------------------------------------------------------------------- emission contract ---
def debug_scores(ctx, queries, rows):
    queries = np.ascontiguousarray(queries, dtype=np.float32)
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    nq, n = len(queries), len(rows)
    full = np.zeros((-(-nq // 128) * 128, -(-n // TILE) * TILE), dtype=np.float32)
    vp = C.c_void_p
    capi._check(capi.lib().stb_debug_batch_gemm(ctx._h, queries.ctypes.data_as(vp), nq, rows.ctypes.data_as(vp), n,
                                                full.ctypes.data_as(vp), None))
    return full[:nq, :n]


@pytest.mark.parametrize("n", [5 * TILE + 17, 600 * TILE + 3])
def test_emission_contract(ctx, sm_count, n):
    rng = np.random.default_rng(31 + n)
    f16, eps = capi.batch_params()
    rows = bench_like(rng, n)
    c = new_corpus(ctx, rows)
    queries = queries_for(rng, rows, 130)
    queries[5] = 0.0                                                   # zero query
    queries[6, 3] = np.nan                                             # cannot be normalised
    A = debug_scores(ctx, queries, rows)
    n_seg = min(-(-n // TILE), sm_count)
    seg_of = (np.arange(n) // TILE) % n_seg
    # 1.5 emits nearly every row: on the large corpus the re-emission would pass its budget
    for m in (0.3, 0.8, 1.0, 1.5) if n < 10000 else (0.3, 0.8, 1.0):
        c.search_batch_threshold(queries, m)
        info = ctx.batch_last()
        assert info["n_seg"] == n_seg and info["seg_cap"] == SEG_CAP
        t = expected_thr(m, eps)
        thr = info["thr"]
        for i in range(len(queries)):
            exp = np.float32(np.inf) if i in (5, 6) else t
            assert thr[i].tobytes() == exp.tobytes(), (m, i, thr[i], exp)
            want = np.zeros(n_seg, np.int64) if i in (5, 6) else np.bincount(seg_of[A[i] >= t], minlength=n_seg)
            assert np.array_equal(info["cand_cnt"][i].astype(np.int64), want), (m, i)
        assert info["k1"] == 2


# ------------------------------------------------------------------------------------------------ routes ---
def test_route_one_pass(ctx):
    rng = np.random.default_rng(41)
    rows = bench_like(rng, 40000)
    c = new_corpus(ctx, rows)
    queries = queries_for(rng, rows, 64)
    before = ctx.counters()["fallback_searches"]
    info = check_batch(ctx, c, queries, 0.75)
    assert (info["retried"], info["k1"]) == (0, 0)
    assert int(info["cand_cnt"].max()) <= SEG_CAP
    assert ctx.counters()["fallback_searches"] == before


def test_route_retry(ctx, sm_count):
    rng = np.random.default_rng(42)
    n_tiles = 2 * sm_count + 5
    rows = unit_rows(rng, n_tiles * TILE)
    queries = unit_rows(rng, 4)
    t0 = 7
    near = queries[0] + 1e-3 * rng.standard_normal((SEG_CAP + 30, 256)).astype(np.float32) / 16
    rows[t0 * TILE: t0 * TILE + len(near)] = near / np.linalg.norm(near, axis=1, keepdims=True)
    rows[(t0 + sm_count) * TILE + 3] = queries[0]                     # same CTA, another tile
    c = new_corpus(ctx, rows)
    before = ctx.counters()["fallback_searches"]
    info = check_batch(ctx, c, queries, 0.01)
    assert info["retried"] == 1 and info["k1"] == 0, info
    assert info["cand_cnt"][0][t0 % sm_count] == SEG_CAP + 31
    assert ctx.counters()["fallback_searches"] == before
    got = c.search_batch_threshold(queries, 0.01)
    assert len(got[0]) == SEG_CAP + 31


def test_route_k1_bad_and_zero_queries(ctx):
    rng = np.random.default_rng(43)
    rows = bench_like(rng, 5000)
    rows[[17, 4000, 4999]] = 0.0
    zeros = np.flatnonzero(~rows.any(axis=1)).tolist()
    c = new_corpus(ctx, rows)
    queries = queries_for(rng, rows, 8)
    queries[1, 0] = np.nan
    queries[2, 9] = np.inf
    queries[3] = 1e20                                                  # squared norm beyond fp32
    queries[4] = 0.0
    for m in (0.5, 1.0, float(np.nextafter(1.0, 2.0)), 3.0):
        before = ctx.counters()["fallback_searches"]
        got = c.search_batch_threshold(queries, m)
        info = ctx.batch_last()
        assert info["k1"] == 4 and info["n_seg"] > 0, info
        assert ctx.counters()["fallback_searches"] >= before + 4
        for i in range(len(queries)):
            same(got[i], k1(c, queries[i], m), f"M={m} query {i}")
        if m <= 1.0:                                                   # the zero query finds the zero rows at 0
            assert sorted(got[4]["row"].tolist()) == zeros and not got[4]["distance"].any()


def test_route_k1_rows_that_cannot_be_normalised(ctx):
    rng = np.random.default_rng(44)
    rows = unit_rows(rng, 3000)
    rows[1234] = 1e20
    c = new_corpus(ctx, rows)
    queries = queries_for(rng, unit_rows(rng, 3000), 5)
    info = check_batch(ctx, c, queries, 0.8)
    assert (info["k1"], info["n_seg"], info["seg_cap"]) == (5, 0, 0), info


def test_route_k1_beyond_the_budget(ctx):
    rng = np.random.default_rng(45)
    n, nq = 60000, 300
    assert nq * n > BUDGET
    rows = unit_rows(rng, n)
    c = new_corpus(ctx, rows)
    queries = unit_rows(rng, nq)
    got = c.search_batch_threshold(queries, float("inf"))
    info = ctx.batch_last()
    assert info["retried"] == BUDGET // n and info["k1"] == nq - BUDGET // n, info
    for i in [0, 1, info["retried"] - 1, info["retried"], nq - 1]:
        same(got[i], k1(c, queries[i], float("inf")), f"query {i}")
    assert all(len(g) == n for g in got)


# ---------------------------------------------------------------------------------------- argument rules ---
def test_argument_rules(ctx):
    rng = np.random.default_rng(51)
    rows = bench_like(rng, 2000)
    c = new_corpus(ctx, rows)
    queries = queries_for(rng, rows, 9)
    vp = C.c_void_p
    L = capi.lib()
    assert raw_call(ctx, c, queries[:0], 0.5, 10)[0] == 0
    off = np.zeros(10, np.uint64)
    out = np.zeros(10, capi.HIT_DTYPE)
    assert L.stb_search_batch_threshold(ctx._h, c._h, None, 9, 0.5, out.ctypes.data_as(vp), 10, off.ctypes.data_as(vp)) == capi.STB_ERR_ARG
    assert raw_call(ctx, c, queries, 0.5, 10, offsets=False)[0] == capi.STB_ERR_ARG
    assert raw_call(ctx, c, queries, 0.5, 10, hits=False)[0] == capi.STB_ERR_ARG
    other = capi.Context(0)
    try:
        oc = new_corpus(other, rows)
        assert raw_call(ctx, oc, queries, 0.5, 10)[0] == capi.STB_ERR_ARG
        oc.close()
    finally:
        other.close()
    empty = capi.Corpus(ctx, 16)
    rc, _, off = raw_call(ctx, empty, queries, 0.5, 10)
    assert rc == 0 and not off.any()
    for m in (float("nan"), 0.0, -0.0, -1.0, float("-inf")):
        rc, _, off = raw_call(ctx, c, queries, m, 10)
        assert rc == 0 and not off.any(), m
        info = ctx.batch_last()
        assert info["route"] == 5 and info["n_seg"] == 0
    refs = [k1(c, q, 0.8) for q in queries]
    total = sum(len(r) for r in refs)
    exp_off = np.concatenate([[0], np.cumsum([len(r) for r in refs])]).astype(np.uint64)
    concat = np.concatenate(refs)
    for cap in (total, total - 1, total // 2, 1):
        rc, out, off = raw_call(ctx, c, queries, 0.8, cap)
        assert rc == (0 if cap >= total else capi.STB_ERR_CAPACITY)
        assert np.array_equal(off, exp_off)
        same(out[:min(cap, total)], concat[:cap])
    rc, _, off = raw_call(ctx, c, queries, 0.8, 0, hits=False)
    assert rc == capi.STB_ERR_CAPACITY and np.array_equal(off, exp_off)


# ------------------------------------------------------------------------------------ shard and mutation ---
def test_row_base_and_mutations(ctx):
    rng = np.random.default_rng(61)
    rows = bench_like(rng, 9000)
    c = new_corpus(ctx, rows, row_base=100000)
    queries = queries_for(rng, rows, 40)
    got = c.search_batch_threshold(queries, 0.8)
    assert min(int(g["row"].min()) for g in got if len(g)) >= 100000
    check_batch(ctx, c, queries, 0.8, where="row_base")
    c.append(bench_like(rng, 700))
    check_batch(ctx, c, queries, 0.8, where="append")
    idx = (np.sort(rng.choice(len(c), 50, replace=False)) + 100000).astype(np.uint64)
    c.update(idx, queries[rng.integers(0, len(queries), 50)])
    check_batch(ctx, c, queries, 0.8, where="update")
    c.remove(np.array([[100000 + 10, 100000 + 900], [100000 + 5000, 100000 + 5003]], dtype=np.uint64))
    check_batch(ctx, c, queries, 0.8, where="remove")


# ---------------------------------------------------------------------------------------------- Python ---
def test_searcher_batch_equals_per_query(ctx):
    rng = np.random.default_rng(71)
    s = Searcher(ctx, capi.Corpus(ctx, 4096))
    docs = []
    for d in range(6):
        n = int(rng.integers(1, 400))
        emb = unit_rows(rng, n)
        lines = [f"doc{d} line {i}" for i in range(n)]
        s.add_document_embeddings(f"doc{d}.txt", lines, emb)
        docs.append(emb)
    allrows = np.concatenate(docs)
    queries = np.concatenate([allrows[[0, len(docs[0]) - 1, len(allrows) - 1]], queries_for(rng, allrows, 20)])
    for cfg in (SearchConfig(n_lines=3, top_k=5), SearchConfig(n_lines=3, top_k=3, max_distance=0.85),
                SearchConfig(n_lines=1, top_k=1, max_distance=1e-9), SearchConfig(n_lines=2, max_distance=2.0)):
        batch = s.search_documents_batch(queries, cfg)
        assert len(batch) == len(queries)
        for i, q in enumerate(queries):
            assert batch[i] == s.search_documents(q, cfg), (cfg, i)
    edge = s.search_documents_batch(queries[:3], SearchConfig(n_lines=3, max_distance=1e-9))
    assert edge[0][0].start == 0 and edge[2][0].end == len(docs[-1])

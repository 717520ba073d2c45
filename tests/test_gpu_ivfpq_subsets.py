"""GPU: K5 IVF-PQ search over many subsets in one call (stb_ivfpq_search_subsets, csrc/ivfpq.cu).

Its contract is per query: hits, count and codes scanned equal, bit for bit, stb_ivfpq_search_filtered called
with that one query and its subset's ranges.  Each test here compares against those per-query calls, and, where
the search is exhaustive, against the exact store query of the corpus.
"""

import os
import re
import sys

import numpy as np
import pytest

from semtools_b200 import capi

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_ivfpq_batch import (MAX_NQ, RERANK_CAP, U64MAX, build, clustered, edge_corpus,  # noqa: E402
                                  edge_queries, make_centers)
from test_gpu_ivfpq_filter import assert_store_query, doc_filter, ranges_of  # noqa: E402

pytestmark = pytest.mark.gpu

_HDR = open(os.path.join(os.path.dirname(__file__), "..", "include", "semtools_b200.h")).read()
SUBSET_SCRATCH = eval(re.search(r"#define\s+STB_IVFPQ_SUBSET_SCRATCH\s+\((\S+ << \d+)\)", _HDR).group(1).replace("ull", ""))


# ------------------------------------------------------------------------------------------ helpers ---
def per_query(idx, Q, subsets, subset_of, **kw):
    """What the contract names: one stb_ivfpq_search_filtered call per query, with its subset's ranges."""
    out = []
    for i, q in enumerate(Q):
        out.append(idx.search_filtered(q[None], subsets[subset_of[i]], **kw))
    return out


def assert_equals_per_query(got, want):
    hits, n, sc = got
    for i, (wh, wn, ws) in enumerate(want):
        assert hits[i].tobytes() == wh[0].tobytes(), i
        assert int(n[i]) == int(wn[0]) and int(sc[i]) == int(ws[0]), i


def uneven_subset_of(rng, nq, named):
    """Queries dealt unevenly to the subsets listed in `named` (weights 1, 2, 4, ...)."""
    w = 2.0 ** np.arange(len(named))
    return np.asarray(named, np.uint32)[rng.choice(len(named), nq, p=w / w.sum())]


def launches_of(subset_of, empty, set_cap):
    """The call's cut: queries in caller order, empty-subset queries skipped, at most MAX_NQ queries and set_cap
    distinct subsets per launch.  Returns the list of launches, each a list of query indices."""
    out, cur, sets = [], [], set()
    for i, s in enumerate(subset_of.tolist()):
        if empty[s]:
            continue
        if len(cur) == MAX_NQ or (s not in sets and len(sets) == set_cap):
            out.append(cur); cur, sets = [], set()
        cur.append(i); sets.add(s)
    if cur:
        out.append(cur)
    return out


def raw_call(idx, Q, offsets, ranges, subset_of, top_k=10, n_subsets=None, scanned=True):
    """The C call on sentinel-filled outputs: (status, hits, n, scanned)."""
    nq = len(Q)
    out = np.full((nq, max(top_k, 1)), 7, dtype=capi.HIT_DTYPE)
    n = np.full(nq, 77, np.uint32)
    sc = np.full(nq, 777, np.uint64)
    ptr = lambda a: None if a is None else capi._np_ptr(a)  # noqa: E731
    ns = len(offsets) - 1 if n_subsets is None else n_subsets
    rc = capi.lib().stb_ivfpq_search_subsets(idx._h, ptr(Q), nq, 8, top_k, 64, 0, 0.0, ns, ptr(offsets), ptr(ranges),
                                             ptr(subset_of), capi._np_ptr(out), capi._np_ptr(n),
                                             capi._np_ptr(sc) if scanned else None)
    return rc, out, n, sc


# ------------------------------------------------------------------------- equality, partial probe ---
@pytest.fixture(scope="module")
def sub_index(ctx):
    rng = np.random.default_rng(7070)
    n, nlist = 60_000, 128
    centers = make_centers(rng, 64)
    rows = clustered(rng, centers, n)
    Q = np.concatenate([clustered(rng, centers, 40), rng.standard_normal((2, 256)).astype(np.float32)])
    rows[321] = Q[0] * np.float32(1e-25)                      # forced rows
    rows[9876, 9] = np.nan
    base = 21 << 32
    c, idx = build(ctx, rows, nlist, row_base=base, iters=6)
    subsets = [doc_filter(rng, n, 0.25, base)[1], doc_filter(rng, n, 0.05, base)[1],
               np.array([[base + 4000, base + 4050]], np.uint64),     # named by no query
               doc_filter(rng, n, 0.01, base)[1], np.array([[base + 10_000, base + 25_000]], np.uint64),
               np.array([[base, base + n]], np.uint64), np.zeros((0, 2), np.uint64),
               doc_filter(rng, n, 0.05, base)[1]]                     # named by no query
    yield rows, Q, c, idx, base, nlist, subsets
    idx.close(); c.close()


@pytest.mark.parametrize("capped", [False, True])
@pytest.mark.parametrize("rerank", [10, 256, 1024])
@pytest.mark.parametrize("nprobe", [8, 64, "nlist"])
def test_equals_the_filtered_call_per_query(sub_index, nprobe, rerank, capped):
    rows, Q, c, idx, base, nlist, subsets = sub_index
    nprobe = nlist if nprobe == "nlist" else nprobe
    rng = np.random.default_rng(nprobe * 7 + rerank + capped)
    subset_of = uneven_subset_of(rng, len(Q), [0, 1, 3, 4, 5, 6])
    kw = dict(max_distance=0.45 if capped else None, nprobe=nprobe, top_k=10, rerank=rerank)
    got = idx.search_subsets(Q, subsets, subset_of, **kw)
    assert_equals_per_query(got, per_query(idx, Q, subsets, subset_of, **kw))
    assert np.all(got[1][subset_of == 6] == 0) and (capped or np.all(got[1][subset_of != 6] > 0))


def test_the_overflow_route_equals_the_filtered_call(sub_index, monkeypatch):
    """STB_IVFPQ_BATCH_KEEP=1: every scan warp keeps one code, so queries take the exact slow route."""
    rows, Q, c, idx, base, nlist, subsets = sub_index
    subset_of = uneven_subset_of(np.random.default_rng(5), len(Q), [0, 1, 3, 4, 5])
    monkeypatch.setenv("STB_IVFPQ_BATCH_KEEP", "1")
    for rerank in (64, 1024):
        kw = dict(nprobe=16, top_k=10, rerank=rerank)
        got = idx.search_subsets(Q, subsets, subset_of, **kw)
        assert_equals_per_query(got, per_query(idx, Q, subsets, subset_of, **kw))
    monkeypatch.delenv("STB_IVFPQ_BATCH_KEEP")
    assert_equals_per_query(got, per_query(idx, Q, subsets, subset_of, **kw))   # and the default route agrees


# ------------------------------------------------------------------------------ exhaustive = exact ---
def test_exhaustive_equals_the_store_query(ctx):
    rng = np.random.default_rng(8181)
    n, base, extra = 3000, 5 << 32, 300
    rows, p = edge_corpus(rng, n)
    rows[p[14]] = rows[p[15]] * np.float32(1e-20)               # forced: zero rows, NaN / inf, 1e-25 and 1e-20 scales
    appended = clustered(rng, make_centers(rng, 4), extra)
    c, idx = build(ctx, rows, 8, row_base=base, extra=extra)
    c.append(appended)                                           # appended, not extended: never returned
    try:
        Q = np.stack(edge_queries(rng, rows, p) + [appended[0], appended[1]])
        m = np.zeros(n, bool)
        m[np.sort(rng.choice(n - 4, 250, replace=False))] = True
        forced = np.zeros(n, bool); forced[p] = True; forced[rng.choice(n, 150, replace=False)] = True
        subsets = [np.array([[base + n // 3, base + n // 3 + 700]], np.uint64), ranges_of(m, base), ranges_of(forced, base),
                   np.array([[base + n - 400, base + n + extra]], np.uint64),          # 400 indexed + every appended row
                   np.array([[base + n, base + n + extra]], np.uint64),               # appended rows only: empty
                   np.zeros((0, 2), np.uint64)]
        subset_of = uneven_subset_of(rng, len(Q), list(range(len(subsets))))
        subset_of[:len(subsets)] = np.arange(len(subsets))
        for top_k in (10, 1024):
            hits, cnt, sc = idx.search_subsets(Q, subsets, subset_of, nprobe=8, top_k=top_k, rerank=RERANK_CAP)
            assert np.all(hits["row"][hits["row"] != U64MAX] < base + n)
            for i, q in enumerate(Q):
                rr = subsets[subset_of[i]]
                indexed = np.clip(rr.astype(np.int64), base, base + n).astype(np.uint64)
                indexed = indexed[indexed[:, 0] < indexed[:, 1]]
                if len(indexed) == 0:
                    assert cnt[i] == 0 and sc[i] == 0 and np.all(hits[i]["row"] == U64MAX)
                    continue
                assert_store_query(hits[i], cnt[i], c, rows, q, top_k, indexed, base)
            assert_equals_per_query((hits, cnt, sc), per_query(idx, Q, subsets, subset_of, nprobe=8, top_k=top_k,
                                                                rerank=RERANK_CAP))
    finally:
        idx.close(); c.close()


# ---------------------------------------------------------------------------------------- chunking ---
def test_more_than_one_launch_of_queries(ctx):
    rng = np.random.default_rng(919)
    centers = make_centers(rng, 16)
    rows = clustered(rng, centers, 5000)
    base = 1 << 40
    c, idx = build(ctx, rows, 16, row_base=base)
    try:
        subsets = [doc_filter(rng, len(rows), f, base)[1] for f in (0.3, 0.1, 0.02)] + [np.zeros((0, 2), np.uint64)]
        Q = clustered(rng, centers, MAX_NQ + 900)
        subset_of = uneven_subset_of(rng, len(Q), [3, 0, 1, 2])
        kw = dict(nprobe=4, top_k=8, rerank=64)
        got = idx.search_subsets(Q, subsets, subset_of, **kw)
        launches = launches_of(subset_of, [False, False, False, True], 1 << 30)
        assert len(launches) == 2
        _check_last_launch(idx, Q, subsets, subset_of, launches[-1], kw)
        assert_equals_per_query(got, per_query(idx, Q, subsets, subset_of, **kw))
    finally:
        idx.close(); c.close()


@pytest.mark.parametrize("shape, launches", [
    ("batch", 2 * 4),                        # two launches of the four batched kernels
    ("filtered", 2 + 2 * 4),                 # one eligibility pass (bitmap, counts) per call
    ("filtered_every_row", 1 + 4),           # no bitmap: the counts are the list lengths
    ("subsets_different", 2 * (2 + 4)),      # each launch names another subset: a pass per launch
    ("subsets_same", 2 + 2 * 4),             # the second launch names the first one's subset: its pass is reused
])
def test_kernel_launches_per_call(ctx, sub_index, shape, launches):
    """The host forms share one loop: their launch counts, and the hits of a launch whose pass was skipped."""
    rows, Q, c, idx, base, nlist, subsets = sub_index
    QQ = np.ascontiguousarray(np.resize(Q, (MAX_NQ + 1, 256)))
    kw = dict(nprobe=8, top_k=10, rerank=64)
    before = ctx.counters()["kernel_launches"]
    if shape == "batch":
        idx.search_batch(QQ, **kw)
    elif shape == "filtered":
        idx.search_filtered(QQ, subsets[0], **kw)
    elif shape == "filtered_every_row":
        idx.search_filtered(Q, None, **kw)
    else:
        subset_of = np.zeros(len(QQ), np.uint32)
        if shape == "subsets_different":
            subset_of[MAX_NQ:] = 1
        got = idx.search_subsets(QQ, subsets, subset_of, **kw)
    assert ctx.counters()["kernel_launches"] - before == launches
    if shape.startswith("subsets"):
        for sl in (slice(0, MAX_NQ), slice(MAX_NQ, None)):
            want = idx.search_filtered(QQ[sl], subsets[subset_of[sl][0]], **kw)
            assert all(g[sl].tobytes() == w.tobytes() for g, w in zip(got, want)), sl


def _check_last_launch(idx, Q, subsets, subset_of, last, kw):
    """batch_last describes the call's last launch: slot j = its j-th query, as the single filtered call has it."""
    info = [idx.batch_last(j) for j in (0, len(last) - 1)]
    assert info[0]["nq"] == len(last)
    with pytest.raises(capi.StbError):
        idx.batch_last(len(last))
    for j, inf in zip((0, len(last) - 1), info):
        i = last[j]
        idx.search_filtered(Q[i:i + 1], subsets[subset_of[i]], **kw)
        one = idx.batch_last(0)
        assert np.array_equal(inf["probe"], one["probe"]) and np.array_equal(inf["coarse"], one["coarse"])


def test_the_scratch_cap_splits_the_subsets(ctx):
    """An index wide enough that STB_IVFPQ_SUBSET_SCRATCH holds fewer distinct subsets than the batch names."""
    rng = np.random.default_rng(2024)
    n, nlist, base = 1 << 20, 64, 9 << 32
    centers = make_centers(rng, 32)
    rows = np.empty((n, 256), np.float32)
    for s in range(0, n, 1 << 16):
        x = centers[rng.integers(0, len(centers), 1 << 16)] + rng.standard_normal(size=(1 << 16, 256), dtype=np.float32) * np.float32(0.04)
        rows[s:s + (1 << 16)] = x / np.linalg.norm(x, axis=1, keepdims=True)
    c = capi.Corpus(ctx, n, row_base=base)
    c.append(rows)
    idx = capi.IvfPq(c, nlist=nlist, train_rows=65536, iters=4)
    try:
        set_cap = SUBSET_SCRATCH // (((n + 31) // 32 + nlist) * 4)
        n_sets = set_cap + 60
        subsets = [np.array([[base + s * 480, base + s * 480 + 300 + s % 50]], np.uint64) for s in range(n_sets)]
        subsets[7] = np.array([[base + 3000, base + 53_000]], np.uint64)
        Q = np.ascontiguousarray(rows[rng.integers(0, n, n_sets + 200)] + np.float32(0.01))
        subset_of = np.arange(len(Q), dtype=np.uint32) % n_sets
        kw = dict(nprobe=8, top_k=10, rerank=128)
        got = idx.search_subsets(Q, subsets, subset_of, **kw)
        launches = launches_of(subset_of, [False] * n_sets, set_cap)
        assert len(launches) == 2 and len(launches[1]) == 60 + 200
        _check_last_launch(idx, Q, subsets, subset_of, launches[-1], kw)
        assert_equals_per_query(got, per_query(idx, Q, subsets, subset_of, **kw))
        assert np.all(got[1] > 0)
    finally:
        idx.close(); c.close()


# ----------------------------------------------------------------------------- refusals and edges ---
def test_refusals_write_and_launch_nothing(ctx, sub_index):
    rows, Q, c, idx, base, nlist, subsets = sub_index
    Q3 = np.ascontiguousarray(Q[:3])
    good = np.array([[base, base + 100], [base + 200, base + 300], [base + 500, base + 900]], np.uint64)
    off = np.array([0, 2, 3], np.uint64)
    so = np.array([0, 1, 0], np.uint32)
    rc, out, n, sc = raw_call(idx, Q3, off, good, so)
    assert rc == capi.STB_OK and np.all(n > 0)
    cases = [  # (expected status, offsets, ranges, subset_of, q, n_subsets)
        (capi.STB_ERR_ARG, off, good, so, None, None),                                   # NULL q
        (capi.STB_ERR_ARG, None, good, so, Q3, 2),                                       # NULL offsets
        (capi.STB_ERR_ARG, off, None, so, Q3, None),                                     # NULL ranges, 3 ranges named
        (capi.STB_ERR_ARG, off, good, None, Q3, None),                                   # NULL subset_of
        (capi.STB_ERR_ARG, np.array([1, 2, 3], np.uint64), good, so, Q3, None),          # offsets[0] != 0
        (capi.STB_ERR_ARG, np.array([0, 2, 1], np.uint64), good, so, Q3, None),          # decreasing
        (capi.STB_ERR_ARG, off, good, np.array([0, 2, 0], np.uint32), Q3, None),         # subset_of >= n_subsets
        (capi.STB_ERR_RANGE, np.array([0, 2, 3, 4], np.uint64),                          # unnamed subset 2 malformed
         np.concatenate([good, [[base + 50, base + 10]]]).astype(np.uint64), so, Q3, None),
        (capi.STB_ERR_RANGE, np.array([0, 2, 3], np.uint64),                             # overlapping ranges
         np.array([[base, base + 100], [base + 50, base + 300], [base + 500, base + 900]], np.uint64), so, Q3, None),
    ]
    for k, (status, o, r, s, q, ns) in enumerate(cases):
        before = ctx.counters()["kernel_launches"]
        nq_q = Q3 if q is None else q
        out = np.full((3, 10), 7, dtype=capi.HIT_DTYPE)
        n = np.full(3, 77, np.uint32)
        sc = np.full(3, 777, np.uint64)
        ptr = lambda a: None if a is None else capi._np_ptr(a)  # noqa: E731
        rc = capi.lib().stb_ivfpq_search_subsets(idx._h, ptr(q), len(nq_q), 8, 10, 64, 0, 0.0,
                                                 len(o) - 1 if ns is None else ns, ptr(o), ptr(r), ptr(s),
                                                 capi._np_ptr(out), capi._np_ptr(n), capi._np_ptr(sc))
        assert rc == status, k
        assert np.all(out["row"] == 7) and np.all(n == 77) and np.all(sc == 777), k
        assert ctx.counters()["kernel_launches"] == before, k
    with pytest.raises(capi.StbError) as e:
        idx.search_subsets(Q3, [good], [0, 0, 0], top_k=1025)
    assert e.value.status == capi.STB_ERR_ARG


def test_edges_launch_nothing(ctx, sub_index):
    rows, Q, c, idx, base, nlist, subsets = sub_index
    n_rows = len(rows)
    before = ctx.counters()["kernel_launches"]
    got, n, sc = idx.search_subsets(np.zeros((0, 256), np.float32), subsets, [])       # nq = 0
    assert len(n) == 0
    got, n, sc = idx.search_subsets(Q, subsets, np.zeros(len(Q), np.uint32), top_k=0)  # top_k = 0
    assert got.shape == (len(Q), 0) and np.all(n == 0) and np.all(sc == 0)
    empties = [np.zeros((0, 2), np.uint64), np.array([[base + n_rows, base + n_rows + 100]], np.uint64),
               np.array([[0, base]], np.uint64), np.array([[base + 5, base + 5]], np.uint64)]
    so = np.arange(len(Q), dtype=np.uint32) % len(empties)
    got, n, sc = idx.search_subsets(Q, empties, so)                                      # every subset empty
    assert np.all(n == 0) and np.all(sc == 0) and np.all(got["row"] == U64MAX) and np.all(np.isinf(got["distance"]))
    assert ctx.counters()["kernel_launches"] == before
    # out_scanned may be NULL; empty-subset queries are padded amid answered ones
    off = np.array([0, 1, 1], np.uint64)
    rr = np.array([[base, base + 30_000]], np.uint64)
    so = np.array([1, 0, 1], np.uint32)
    rc, out, n, sc = raw_call(idx, np.ascontiguousarray(Q[:3]), off, rr, so, scanned=False)
    assert rc == capi.STB_OK and np.all(sc == 777)
    want = idx.search_filtered(Q[1:2], rr, nprobe=8, top_k=10, rerank=64)
    assert out[1].tobytes() == want[0][0].tobytes() and n[1] == want[1][0]
    assert n[0] == 0 and n[2] == 0 and np.all(out["row"][[0, 2]] == U64MAX)

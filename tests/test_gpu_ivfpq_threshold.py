"""GPU: K5 IVF-PQ threshold search (stb_ivfpq_search_threshold, csrc/ivfpq.cu) against a prediction.

The probe stage is the batched search's, so stb_debug_ivfpq_batch_last gives each query's coarse scores, probe
list and LUT, from which numpy reproduces every ADC score bit for bit (test_gpu_ivfpq_batch.adc_keys).  The
prediction takes the probed codes whose score reaches the cutoff t = RD_f32((1 - M) - slack) (all of them when
t = -inf), adds the forced rows, and keeps the rows whose oracle distance is below M, in (distance, row) order.
"""

import os
import re
import sys

import numpy as np
import pytest

import oracle
from semtools_b200 import capi

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_ivfpq_batch import (INVALID, adc_keys, bad_queries, build, clustered, edge_corpus,  # noqa: E402
                                  edge_queries, make_centers)

pytestmark = pytest.mark.gpu

_SRC = open(os.path.join(os.path.dirname(__file__), "..", "semtools_b200", "csrc", "ivfpq.cu")).read()
BLOCK = int(re.search(r"#define IVFT_BLOCK (\d+)", _SRC).group(1))
_HDR = open(os.path.join(os.path.dirname(__file__), "..", "include", "semtools_b200.h")).read()
KEYS = eval(re.search(r"#define\s+STB_IVFPQ_THRESHOLD_KEYS\s+\((\S+ << \d+)\)", _HDR).group(1).replace("ull", ""))
INF = float("inf")


# ------------------------------------------------------------------------------------------ helpers ---
def key_scores(keys):
    """The fp32 ADC score a stb_make_key key holds (NaN for INVALID)."""
    ordv = ~(keys >> np.uint64(32)).astype(np.uint32)
    b = np.where(ordv & np.uint32(0x80000000), ordv & np.uint32(0x7FFFFFFF), ~ordv).astype(np.uint32)
    return b.view(np.float32)


def cutoff(m, slack):
    """RD_f32((1 - m) - slack), the difference taken in f64."""
    x = (1.0 - m) - slack
    f = np.float32(x)
    if float(f) > x:
        f = np.nextafter(f, np.float32(-np.inf))
    return f


def predict(E, info, rows, q, m, slack, base):
    """(hits, codes scanned, rows re-scored) the threshold search must return for this query."""
    pos, keys = adc_keys(E, info)
    t = cutoff(m, slack)
    if t == -np.inf:
        cand = pos
    else:
        with np.errstate(invalid="ignore"):
            cand = pos[(keys != INVALID) & (key_scores(keys) >= t)]
    mem = np.sort(np.concatenate([E["order"][cand].astype(np.int64), E["forced"].astype(np.int64)]))
    want = np.zeros(0, capi.HIT_DTYPE)
    if len(mem):
        rr, dd = oracle.search_rows(rows[mem], q, top_k=0, max_distance=m)
        want = np.zeros(len(rr), capi.HIT_DTYPE)
        want["row"] = mem[np.asarray(rr, np.int64)].astype(np.uint64) + np.uint64(base)
        want["distance"] = dd
    return want, len(pos), len(mem)


def check_prediction(idx, E, rows, Q, m, slack, base, nprobe, got):
    hits, scanned, reranked = got
    for i, q in enumerate(Q):
        info = idx.batch_last(i)
        assert (info["nq"], info["nprobe"], info["top_k"], info["rerank"]) == (len(Q), nprobe, 0, 0)
        want, n_scan, n_re = predict(E, info, rows, q, m, slack, base)
        assert int(scanned[i]) == n_scan and int(reranked[i]) == n_re, (i, m, slack)
        assert hits[i].tobytes() == want.tobytes(), (i, m, slack)


def same(a, b, what=""):
    assert len(a) == len(b), (what, len(a), len(b))
    assert a.tobytes() == b.tobytes(), what


def raw(idx, Q, nq, m, slack, cap, out=True, offsets=True, counts=True, nprobe=8):
    """The C call on sentinel-filled outputs: (status, hits, offsets, scanned, reranked)."""
    hits = np.full(max(cap, 1), 7, dtype=capi.HIT_DTYPE)
    off = np.full(nq + 1, 77, np.uint64)
    sc = np.full(max(nq, 1), 777, np.uint64)
    rk = np.full(max(nq, 1), 777, np.uint64)
    p = capi._np_ptr
    rc = capi.lib().stb_ivfpq_search_threshold(idx._h if idx is not None else None, p(Q) if Q is not None else None, nq,
                                               nprobe, m, slack, p(hits) if out else None, cap,
                                               p(off) if offsets else None, p(sc) if counts else None,
                                               p(rk) if counts else None)
    return rc, hits, off, sc, rk


# ---------------------------------------------------------------------- clustered index (partial probe) ---
@pytest.fixture(scope="module")
def clustered_index(ctx):
    rng = np.random.default_rng(9191)
    n, nlist = 60_000, 64
    centers = make_centers(rng, 64)
    rows = clustered(rng, centers, n)
    Q = np.concatenate([clustered(rng, centers, 20), rng.standard_normal((2, 256)).astype(np.float32),
                        np.stack(bad_queries(rng))])
    rows[321] = Q[0] * np.float32(1e-25)                    # forced rows
    rows[7654, 9] = np.nan
    base = 11 << 32
    c, idx = build(ctx, rows, nlist, row_base=base, iters=6)
    E = idx.export()
    assert len(E["forced"]) == 2
    yield rows, Q, c, idx, E, base, centers
    idx.close(); c.close()


@pytest.mark.parametrize("m,slack", [(0.2, 0.0), (0.27, 0.0), (0.27, 0.02), (0.35, 0.1), (0.3, INF), (INF, 0.0)])
def test_predicted_bits_at_partial_probe(clustered_index, m, slack):
    rows, Q, c, idx, E, base, _ = clustered_index
    got = idx.search_threshold(Q, nprobe=8, max_distance=m, slack=slack)
    check_prediction(idx, E, rows, Q, m, slack, base, 8, got)
    if slack == 0.0 and m < 1:
        assert sum(len(h) for h in got[0]) > 0


def test_every_hit_is_an_exact_hit_and_the_set_is_monotone(clustered_index):
    rows, Q, c, idx, E, base, _ = clustered_index
    m = 0.3
    exact = c.search_batch_threshold(Q, m)
    prev = None
    for nprobe in (1, 2, 4, 8, 16, 64):
        hits, scanned, _ = idx.search_threshold(Q, nprobe=nprobe, max_distance=m, slack=0.02)
        sets = [set(zip(h["row"].tolist(), h["distance"].view(np.uint64).tolist())) for h in hits]
        for i in range(len(Q)):
            assert sets[i] <= set(zip(exact[i]["row"].tolist(), exact[i]["distance"].view(np.uint64).tolist())), i
            if prev is not None:
                assert prev[i] <= sets[i], (nprobe, i)
        prev = sets
    prev = None
    for slack in (0.0, 0.005, 0.02, 0.1, 0.5, INF):
        hits, _, reranked = idx.search_threshold(Q, nprobe=4, max_distance=m, slack=slack)
        sets = [set(h["row"].tolist()) for h in hits]
        if prev is not None:
            assert all(p <= s for p, s in zip(prev[0], sets)), slack
            assert np.all(prev[1] <= reranked), slack
        prev = (sets, reranked)


# ------------------------------------------------------------------------- exhaustive search is exact ---
@pytest.mark.parametrize("n", [700, 1031])
def test_exhaustive_probe_with_infinite_slack_is_exact(ctx, n):
    rng = np.random.default_rng(800 + n)
    rows, p = edge_corpus(rng, n)
    base = 3 << 32
    c, idx = build(ctx, rows, nlist=3, row_base=base)
    Q = np.stack(edge_queries(rng, rows, p) + bad_queries(rng) + [rng.standard_normal(256).astype(np.float32)
                                                                  for _ in range(3)] + [rows[p[13]], rows[p[3]]])
    try:
        assert len(idx.export()["forced"]) > 0
        for m in (0.05, 0.5, 1.0, 1.7, INF):
            got, scanned, reranked = idx.search_threshold(Q, nprobe=3, max_distance=m, slack=INF)
            assert np.all(reranked == n) and np.all(scanned + len(idx.export()["forced"]) == n)
            k2 = c.search_batch_threshold(Q, m)
            for i, q in enumerate(Q):
                rr, dd = oracle.search_rows(rows, q, top_k=0, max_distance=m)
                want = np.zeros(len(rr), capi.HIT_DTYPE)
                want["row"] = np.asarray(rr, np.uint64) + np.uint64(base)
                want["distance"] = dd
                same(got[i], want, f"M={m} query {i} vs the oracle")
                if not np.all(np.isfinite(q)):
                    continue                   # every row's canonical distance is 0; stb_search is not pinned there
                same(got[i], c.search(q, top_k=0, max_distance=m), f"M={m} query {i} vs stb_search")
                same(got[i], k2[i], f"M={m} query {i} vs stb_search_batch_threshold")
    finally:
        idx.close(); c.close()


# ---------------------------------------------------------------------------------------- split path ---
def test_split_queries_answer_as_with_the_default_budget(clustered_index):
    rows, Q, c, idx, E, base, centers = clustered_index
    m, slack, nprobe = 0.3, 0.1, 32
    want, w_sc, w_rk = idx.search_threshold(Q, nprobe=nprobe, max_distance=m, slack=slack)
    assert int(w_sc.max()) > BLOCK                          # queries span more than one block
    big = int(np.argmax(w_rk))
    budget = int(w_rk[big]) // 3
    assert budget > 0
    idx.set_threshold_keys(budget)
    try:
        one, o_sc, o_rk = idx.search_threshold(Q[big:big + 1], nprobe=nprobe, max_distance=m, slack=slack)
        same(one[0], want[big], "one query over several launches")
        assert int(o_sc[0]) == int(w_sc[big]) and int(o_rk[0]) == int(w_rk[big])
        got = idx.search_threshold(Q, nprobe=nprobe, max_distance=m, slack=slack)
        check_prediction(idx, E, rows, Q, m, slack, base, nprobe, got)
        for i in range(len(Q)):
            same(got[0][i], want[i], f"query {i}")
    finally:
        idx.set_threshold_keys(0)

    rng = np.random.default_rng(5)
    B = np.concatenate([clustered(rng, centers, 5000 - len(Q)), Q])
    ref, r_sc, r_rk = idx.search_threshold(B, nprobe=nprobe, max_distance=m, slack=slack)
    perm = rng.permutation(len(B))
    idx.set_threshold_keys(int(np.median(r_rk)) + 1)
    try:
        got, g_sc, g_rk = idx.search_threshold(B[perm], nprobe=nprobe, max_distance=m, slack=slack)
    finally:
        idx.set_threshold_keys(0)
    assert np.array_equal(g_sc, r_sc[perm]) and np.array_equal(g_rk, r_rk[perm])
    for i, j in enumerate(perm):
        same(got[i], ref[j], f"permuted slot {i} (query {j})")
    info = idx.batch_last(0)
    assert (info["nq"], info["nprobe"]) == (len(B) - 4096, nprobe)     # the last chunk's launch


def test_budget_hook_limits(clustered_index):
    idx = clustered_index[3]
    with pytest.raises(capi.StbError) as e:
        idx.set_threshold_keys(KEYS + 1)
    assert e.value.status == capi.STB_ERR_ARG
    idx.set_threshold_keys(KEYS)
    idx.set_threshold_keys(0)


# ------------------------------------------------------------------------------------------ capacity ---
def test_capacity_writes_the_first_hits_and_every_offset(clustered_index):
    rows, Q, c, idx, E, base, _ = clustered_index
    Qc = np.ascontiguousarray(Q)
    full, sc, rk = idx.search_threshold(Qc, nprobe=8, max_distance=0.3, slack=0.05)
    cat = np.concatenate(full)
    offs = np.concatenate([[0], np.cumsum([len(h) for h in full])]).astype(np.uint64)
    assert len(cat) > 10
    for cap in (0, 1, len(cat) // 2, len(cat) - 1):
        rc, hits, off, gsc, grk = raw(idx, Qc, len(Qc), 0.3, 0.05, cap, out=cap > 0)
        assert rc == capi.STB_ERR_CAPACITY, cap
        assert np.array_equal(off, offs) and np.array_equal(gsc[: len(Qc)], sc) and np.array_equal(grk[: len(Qc)], rk)
        assert hits[:cap].tobytes() == cat[:cap].tobytes(), cap
        assert np.all(hits["row"][cap:] == 7)                          # nothing past cap
    rc, hits, off, _, _ = raw(idx, Qc, len(Qc), 0.3, 0.05, len(cat))
    assert rc == 0 and hits.tobytes() == cat.tobytes() and np.array_equal(off, offs)


# ------------------------------------------------------------------------------------ argument rules ---
def test_argument_rules(ctx, clustered_index):
    rows, Q, c, idx, E, base, _ = clustered_index
    Qc = np.ascontiguousarray(Q[:4])
    rc, _, off, sc, _ = raw(idx, Qc, 0, 0.5, 0.0, 10)                  # nq == 0: no-op, nothing written
    assert rc == 0 and np.all(off == 77) and np.all(sc == 777)
    assert raw(None, Qc, 0, 0.5, 0.0, 10)[0] == capi.STB_ERR_ARG       # null index
    for m in (float("nan"), 0.0, -0.0, -1.0, -INF):
        before = ctx.counters()["kernel_launches"]
        rc, hits, off, sc, rk = raw(idx, Qc, 4, m, 0.0, 10)
        assert rc == 0 and np.all(off == 0) and np.all(sc[:4] == 0) and np.all(rk[:4] == 0), m
        assert np.all(hits["row"] == 7)
        assert ctx.counters()["kernel_launches"] == before, m
        assert raw(idx, Qc, 4, m, 0.0, 10, counts=False)[0] == 0
    for slack in (float("nan"), -1e-300, -1.0, -INF):
        assert raw(idx, Qc, 4, 0.5, slack, 10)[0] == capi.STB_ERR_ARG, slack
    assert raw(idx, None, 4, 0.5, 0.0, 10)[0] == capi.STB_ERR_ARG      # null q
    assert raw(idx, Qc, 4, 0.5, 0.0, 10, offsets=False)[0] == capi.STB_ERR_ARG
    assert raw(idx, Qc, 4, 0.5, 0.0, 10, out=False)[0] == capi.STB_ERR_ARG   # null out_hits with cap > 0
    rc, _, off, _, _ = raw(idx, Qc, 4, 0.5, 0.0, 0, out=False)         # cap 0: only the offsets
    assert rc in (0, capi.STB_ERR_CAPACITY) and off[0] == 0
    rc, _, _, sc, rk = raw(idx, Qc, 4, 0.3, 0.0, 1 << 16, counts=False)
    assert rc == 0 and np.all(sc == 777) and np.all(rk == 777)
    for nprobe, want in [(0, 1), (5000, 64)]:                          # nprobe clamped to [1, min(nlist, 1024)]
        idx.search_threshold(Qc, nprobe=nprobe, max_distance=0.3)
        assert idx.batch_last(0)["nprobe"] == want


# ------------------------------------------------------------------------------- after index changes ---
def test_prediction_after_extend_update_and_remove(ctx):
    rng = np.random.default_rng(2718)
    centers = make_centers(rng, 32)
    rows = clustered(rng, centers, 24_000)
    extra = clustered(rng, centers, 3000)
    c, idx = build(ctx, rows, nlist=32, row_base=1 << 32, extra=len(extra))
    Q = np.concatenate([clustered(rng, centers, 12), np.stack(bad_queries(rng))])
    try:
        c.append(extra)
        assert idx.extend() == len(extra)
        cur = np.concatenate([rows, extra])
        upd = np.array([5, 100, 20_000, 25_000], np.uint64)
        new = clustered(rng, centers, len(upd))
        new[1] = 0.0                                                   # becomes a forced row
        idx.update(upd + np.uint64(1 << 32), new)
        cur[upd.astype(np.int64)] = new
        idx.remove(np.array([[(1 << 32) + 1000, (1 << 32) + 1500]], np.uint64))
        cur = np.delete(cur, np.arange(1000, 1500), axis=0)
        E = idx.export()
        assert len(E["forced"]) == 1
        for m, slack in [(0.27, 0.0), (0.3, 0.05), (0.3, INF)]:
            got = idx.search_threshold(Q, nprobe=6, max_distance=m, slack=slack)
            check_prediction(idx, E, cur, Q, m, slack, 1 << 32, 6, got)
    finally:
        idx.close(); c.close()

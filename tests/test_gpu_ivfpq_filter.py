"""GPU: K5 IVF-PQ filtered search (stb_ivfpq_search_filtered, csrc/ivfpq.cu) against the exact filtered scan
and against a prediction from the index itself.

The filtered search is the batched search with an eligibility rule, so its answers are predictable the same
way (helpers from test_gpu_ivfpq_batch.py): the hook's coarse scores fix the probe list (lists with an
eligible code, in the unfiltered order), the hook's LUT fixes every ADC score, and the `rerank` best
eligible keys plus the eligible forced rows, re-ranked with the oracle, are the hits bit for bit.
"""

import ctypes as C
import os
import sys

import numpy as np
import pytest

import oracle
from semtools_b200 import capi

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_ivfpq_batch import (INVALID, RERANK_CAP, U64MAX, WARP_KEEP, adc_keys, assert_hits, build,  # noqa: E402
                                  clustered, edge_corpus, edge_queries, make_centers, np_keys, scan_routes,
                                  winners)

pytestmark = pytest.mark.gpu

NO_LIST = 0xFFFFFFFF
MAX_DIST = 100.0


# ------------------------------------------------------------------------------------------ helpers ---
def ranges_of(mask, base):
    """Global [begin, end) ranges of the True runs of a local row mask (as Store._ranges_for builds them)."""
    edges = np.flatnonzero(np.diff(np.concatenate([[0], mask.astype(np.int8), [0]])))
    return (edges.reshape(-1, 2).astype(np.uint64) + np.uint64(base))


def mask_of(ranges, base, n):
    m = np.zeros(n, bool)
    for b, e in np.asarray(ranges, np.uint64).reshape(-1, 2).tolist():
        b, e = max(b, base), min(e, base + n)
        if b < e:
            m[b - base:e - base] = True
    return m


def elig_per_list(E, mask):
    off = E["list_off"].astype(np.int64)
    nlist = len(off) - 1
    lst = np.repeat(np.arange(nlist), np.diff(off))
    return np.bincount(lst, weights=mask[E["order"]].astype(np.float64), minlength=nlist).astype(np.int64)


def probe_of(coarse, elig, nprobe):
    """The filtered probe list: lists with an eligible code in (coarse desc, list id asc) order, the first
    nprobe of them, padded with NO_LIST."""
    order = np.argsort(np_keys(coarse, np.arange(len(coarse))), kind="stable")
    sel = order[elig[order] > 0][:nprobe]
    return np.concatenate([sel, np.full(nprobe - len(sel), NO_LIST)]).astype(np.int64)


def filtered_keys(E, info, mask):
    """(code positions of the probed lists in probe order, keys with INVALID for ineligible codes)."""
    probe = info["probe"][info["probe"] != NO_LIST]
    pos, keys = adc_keys(E, {**info, "probe": probe})
    return pos, np.where(mask[E["order"][pos]], keys, INVALID)


def predict_filtered(E, info, rows, q, top_k, base, mask, limit=MAX_DIST):
    """(global rows, distances, eligible codes scanned) the filtered search must return."""
    pos, keys = filtered_keys(E, info, mask)
    w = winners(keys, info["rerank"])
    cand = E["order"][(w & np.uint64(0xFFFFFFFF)).astype(np.int64)].astype(np.int64)
    forced = E["forced"].astype(np.int64)
    mem = np.concatenate([cand, forced[mask[forced]]])
    n_scan = int(mask[E["order"][pos]].sum())
    if len(mem) == 0:
        return [], np.zeros(0), n_scan
    d = oracle.distances(rows[mem], q)
    ok = d < limit
    mem, d = mem[ok], d[ok]
    o = np.lexsort((mem, d))[:top_k]
    return [int(mem[i]) + base for i in o], d[o].astype(np.float64), n_scan


def check_predicted(idx, E, rows, Q, got, n, scanned, top_k, base, mask, nprobe, limit=MAX_DIST):
    elig = elig_per_list(E, mask)
    for i, q in enumerate(Q):
        info = idx.batch_last(i)
        assert info["probe"].tolist() == probe_of(info["coarse"], elig, nprobe).tolist(), i
        want_rows, want_d, n_scan = predict_filtered(E, info, rows, q, top_k, base, mask, limit)
        assert int(scanned[i]) == n_scan, i
        assert_hits(got[i], n[i], want_rows, want_d)


def assert_store_query(got, n, c, rows, q, top_k, ranges, base, max_distance=None):
    """Bit for bit against stb_search in store-query mode; rows and f32 distances against the oracle."""
    want = c.search(q, top_k, max_distance, capi.STB_MODE_STORE_QUERY, row_ranges=ranges)
    assert int(n) == len(want)
    assert got["row"][:n].tolist() == want["row"].tolist()
    assert np.array_equal(got["distance"][:n].view(np.uint64), want["distance"].view(np.uint64))
    assert np.all(got["row"][n:] == U64MAX)
    if max_distance is not None and float(np.float32(max_distance)) != max_distance:
        return                                                 # the oracle takes the cap as f32
    loc = np.asarray(ranges, np.uint64).reshape(-1, 2).astype(np.int64) - base
    loc = np.clip(loc, 0, len(rows))
    orow, od = oracle.store_search(rows, loc[loc[:, 0] < loc[:, 1]], q, top_k, max_distance)
    assert got["row"][:n].tolist() == [int(r) + base for r in orow]
    assert np.array_equal(got["distance"][:n].astype(np.float32).view(np.uint32), od.view(np.uint32))


def doc_filter(rng, n, frac, base, max_len=40):
    """Random "documents" (runs of 1..max_len rows) each kept with probability frac."""
    lens = rng.integers(1, max_len + 1, n)
    starts = np.concatenate([[0], np.cumsum(lens)])
    starts = starts[starts < n]
    keep = rng.random(len(starts)) < frac
    mask = np.zeros(n, bool)
    for s, k in zip(np.append(starts, n)[:-1], keep):
        if k:
            e = starts[starts > s][0] if np.any(starts > s) else n
            mask[s:e] = True
    return mask, ranges_of(mask, base)


# ------------------------------------------------------------------------- exhaustive = exact scan ---
def exhaustive_filters(rng, n, base, E, special):
    """One range, hundreds of small ranges, ranges cutting through lists, ranges covering forced rows;
    each selects at most RERANK_CAP eligible codes."""
    out = {"one_range": np.array([[base + n // 3, base + n // 3 + 700]], np.uint64)}
    m = np.zeros(n, bool)
    starts = np.sort(rng.choice(n - 4, 300, replace=False))
    for s in starts:
        m[s:s + rng.integers(1, 4)] = True
    out["hundreds_small"] = ranges_of(m, base)
    off = E["list_off"].astype(np.int64)
    big = int(np.argmax(np.diff(off)))
    m = np.zeros(n, bool)
    lr = E["order"][off[big]:off[big + 1]].astype(np.int64)
    m[lr[::2]] = True                                        # every other row of the largest list
    out["cut_through_a_list"] = ranges_of(m, base)
    m = np.zeros(n, bool)
    m[special] = True
    m[rng.choice(n, 200, replace=False)] = True
    out["forced_rows"] = ranges_of(m, base)
    return out


@pytest.mark.parametrize("data", ["clustered", "edge"])
def test_exhaustive_filtered_equals_the_exact_scan(ctx, data):
    rng = np.random.default_rng(900 + len(data))
    n, base = 3000, 11 << 32
    if data == "edge":
        rows, p = edge_corpus(rng, n)
        Q = np.stack(edge_queries(rng, rows, p))
        special = p
    else:
        centers = make_centers(rng, 16)
        rows = clustered(rng, centers, n)
        rows[17] = 0.0; rows[2500, 3] = np.nan                  # forced rows
        Q = np.concatenate([clustered(rng, centers, 4), rng.standard_normal((1, 256)).astype(np.float32)])
        special = np.array([17, 2500, 18, 2499])
    nlist = 8
    c, idx = build(ctx, rows, nlist, row_base=base)
    E = idx.export()
    try:
        for name, rr in exhaustive_filters(rng, n, base, E, special).items():
            mask = mask_of(rr, base, n)
            assert mask[E["order"]].sum() <= RERANK_CAP, name
            for top_k in (10, 1024):
                got, cnt, sc = idx.search_filtered(Q, rr, nprobe=nlist, top_k=top_k, rerank=RERANK_CAP)
                for i, q in enumerate(Q):
                    assert int(sc[i]) == int(mask[E["order"]].sum())
                    assert_store_query(got[i], cnt[i], c, rows, q, top_k, rr, base)
                    # caps: one above the k-th hit's distance, and exactly at it (the hit is excluded)
                    if cnt[i] >= 4:
                        for cap in (float(got[i]["distance"][3]), float(np.nextafter(got[i]["distance"][3], 9.0)), 0.5):
                            g2, c2, _ = idx.search_filtered(q[None], rr, max_distance=cap, nprobe=nlist, top_k=top_k,
                                                            rerank=RERANK_CAP)
                            assert np.all(g2[0]["distance"][:c2[0]] < cap)
                            assert_store_query(g2[0], c2[0], c, rows, q, top_k, rr, base, max_distance=cap)
    finally:
        idx.close(); c.close()


# ---------------------------------------------------------------------------- partial probe, predicted ---
@pytest.fixture(scope="module")
def filt_index(ctx):
    rng = np.random.default_rng(6060)
    n, nlist = 60_000, 64
    centers = make_centers(rng, 64)
    rows = clustered(rng, centers, n)
    Q = np.concatenate([clustered(rng, centers, 16), rng.standard_normal((2, 256)).astype(np.float32)])
    rows[321] = Q[0] * np.float32(1e-25)                      # forced rows
    rows[9876, 9] = np.nan
    base = 13 << 32
    c, idx = build(ctx, rows, nlist, row_base=base, iters=6)
    E = idx.export()
    yield rows, Q, c, idx, E, base, rng
    idx.close(); c.close()


def partial_filters(rows, E, base, rng):
    n = len(rows)
    out = {}
    for frac in (0.25, 0.05):
        out[f"docs_{frac}"] = doc_filter(rng, n, frac, base)[1]
    off = E["list_off"].astype(np.int64)
    m = np.zeros(n, bool)                                    # only 3 lists hold eligible codes: E < nprobe
    for l in (5, 17, 40):
        m[E["order"][off[l]:off[l + 1]]] = True
    m[321] = True
    out["three_lists"] = ranges_of(m, base)
    out["block"] = np.array([[base + 10_000, base + 25_000]], np.uint64)
    return out


@pytest.mark.parametrize("rerank", [10, 256, 1024])
def test_predicted_bits_at_partial_probe(filt_index, rerank):
    rows, Q, c, idx, E, base, rng = filt_index
    nprobe, top_k = 8, 10
    for name, rr in partial_filters(rows, E, base, np.random.default_rng(rerank)).items():
        mask = mask_of(rr, base, len(rows))
        got, n, sc = idx.search_filtered(Q, rr, nprobe=nprobe, top_k=top_k, rerank=rerank)
        info = idx.batch_last(0)
        assert (info["nq"], info["nprobe"], info["top_k"], info["rerank"]) == (len(Q), nprobe, top_k, rerank)
        check_predicted(idx, E, rows, Q, got, n, sc, top_k, base, mask, nprobe)
        if name == "three_lists":
            assert all(idx.batch_last(i)["probe"].tolist()[3:] == [NO_LIST] * 5 for i in range(len(Q)))
        # with a cap between hits: the same candidates, fewer hits
        cap = float(np.median(got["distance"][:, 0]))
        g2, n2, s2 = idx.search_filtered(Q, rr, max_distance=cap, nprobe=nprobe, top_k=top_k, rerank=rerank)
        check_predicted(idx, E, rows, Q, g2, n2, s2, top_k, base, mask, nprobe, limit=cap)
        assert np.array_equal(s2, sc) and np.all(n2 <= n) and np.any(n2 < n)


# ------------------------------------------------------------------------ selective filter, far away ---
def test_selective_filter_far_from_the_query(filt_index):
    """The eligible rows live only in lists none of the nprobe best lists of any query: post-filtering the
    unfiltered search finds (almost) nothing, the filtered search returns min(top_k, eligible rows)."""
    rows, Q, c, idx, E, base, rng = filt_index
    nprobe, top_k = 8, 10
    Qn = Q[:16]
    idx.search_batch(Qn, nprobe=nprobe, top_k=top_k, rerank=256)
    probed = set()
    for i in range(len(Qn)):
        probed |= set(idx.batch_last(i)["probe"].tolist())
    off = E["list_off"].astype(np.int64)
    far = [l for l in range(len(off) - 1) if l not in probed and off[l + 1] > off[l]]
    assert len(far) >= 4
    m = np.zeros(len(rows), bool)
    for l in far[:2]:
        lr = E["order"][off[l]:off[l + 1]]
        m[lr[: max(3, len(lr) // 200)]] = True                # a handful of rows of two far lists
    rr = ranges_of(m, base)
    n_elig = int(m.sum())
    ub, un, _ = idx.search_batch(Qn, nprobe=nprobe, top_k=top_k, rerank=256)
    got, n, sc = idx.search_filtered(Qn, rr, nprobe=nprobe, top_k=top_k, rerank=256)
    for i, q in enumerate(Qn):
        assert int(n[i]) == min(top_k, n_elig)
        exact = c.search(q, top_k, None, capi.STB_MODE_STORE_QUERY, row_ranges=rr)
        assert int(n[i]) == len(exact)
        post = [r for r in ub[i]["row"][: un[i]].tolist() if m[r - base]]
        assert len(post) < int(n[i])
    check_predicted(idx, E, rows, Qn, got, n, sc, top_k, base, m, nprobe)


# --------------------------------------------------------------------------------------- slow route ---
@pytest.mark.parametrize("rerank", [64, 1024])
def test_warp_capacity_at_its_limit_and_one_past(filt_index, monkeypatch, rerank):
    rows, Q, c, idx, E, base, rng = filt_index
    mask, rr = doc_filter(np.random.default_rng(rerank + 1), len(rows), 0.3, base)
    got, n, sc = idx.search_filtered(Q, rr, nprobe=8, top_k=10, rerank=rerank)
    keys_of = [filtered_keys(E, idx.batch_last(i), mask)[1] for i in range(len(Q))]
    most = max(scan_routes(k, rerank, WARP_KEEP)[1] for k in keys_of)
    assert 1 < most <= WARP_KEEP
    for keep, any_slow in [(most, False), (most - 1, True), (1, True)]:
        routes = [scan_routes(k, rerank, keep)[0] for k in keys_of]
        assert (not all(routes)) == any_slow, keep
        monkeypatch.setenv("STB_IVFPQ_BATCH_KEEP", str(keep))
        try:
            got, n, sc = idx.search_filtered(Q, rr, nprobe=8, top_k=10, rerank=rerank)
        finally:
            monkeypatch.delenv("STB_IVFPQ_BATCH_KEEP")
        check_predicted(idx, E, rows, Q, got, n, sc, 10, base, mask, 8)


# ----------------------------------------------------------------------------- unfiltered equivalence ---
@pytest.mark.parametrize("nprobe,rerank", [(8, 256), (32, 1024)])
def test_no_filter_equals_the_batch(filt_index, nprobe, rerank):
    rows, Q, c, idx, E, base, rng = filt_index
    sizes = np.diff(E["list_off"].astype(np.int64))
    want, wn, ws = idx.search_batch(Q, nprobe=nprobe, top_k=10, rerank=rerank)
    for i in range(len(Q)):
        assert np.all(sizes[idx.batch_last(i)["probe"]] > 0)
    got, n, sc = idx.search_filtered(Q, None, nprobe=nprobe, top_k=10, rerank=rerank)
    assert np.array_equal(got, want) and np.array_equal(n, wn) and np.array_equal(sc, ws)


# ----------------------------------------------------------------------------------------- boundaries ---
def raw_call(idx, Q, ranges_ptr, n_ranges, top_k=10):
    nq = len(Q)
    out = np.full((nq, max(top_k, 1)), 7, dtype=capi.HIT_DTYPE)
    n = np.full(nq, 77, np.uint32)
    sc = np.full(nq, 777, np.uint64)
    rc = capi.lib().stb_ivfpq_search_filtered(idx._h, capi._np_ptr(Q), nq, 8, top_k, 64, 0, 0.0, ranges_ptr, n_ranges,
                                              capi._np_ptr(out), capi._np_ptr(n), capi._np_ptr(sc))
    return rc, out, n, sc


def test_boundaries(ctx, filt_index):
    rows, Q, c, idx, E, base, rng = filt_index
    n_rows = len(rows)
    # empty subset, ranges outside the index
    for rr in (np.zeros((0, 2), np.uint64), np.array([[base + n_rows, base + n_rows + 100]], np.uint64),
               np.array([[0, base]], np.uint64), np.array([[base + 5, base + 5]], np.uint64)):
        got, n, sc = idx.search_filtered(Q, rr, nprobe=8, top_k=10)
        assert np.all(n == 0) and np.all(sc == 0) and np.all(got["row"] == U64MAX)
    # malformed ranges: STB_ERR_RANGE, nothing written; n_ranges > 0 with NULL: STB_ERR_ARG
    for bad in ([[base + 10, base + 5]], [[base, base + 10], [base + 5, base + 20]]):
        arr = np.ascontiguousarray(bad, dtype=np.uint64)
        rc, out, n, sc = raw_call(idx, Q[:3], capi._np_ptr(arr), len(arr))
        assert rc == capi.STB_ERR_RANGE
        assert np.all(out["row"] == 7) and np.all(n == 77) and np.all(sc == 777)
        with pytest.raises(capi.StbError) as e:
            idx.search_filtered(Q, arr)
        assert e.value.status == capi.STB_ERR_RANGE
    rc, out, n, sc = raw_call(idx, Q[:3], None, 2)
    assert rc == capi.STB_ERR_ARG and np.all(n == 77)
    # top_k 0 and 1025
    rr = np.array([[base, base + 1000]], np.uint64)
    got, n, sc = idx.search_filtered(Q, rr, top_k=0)
    assert np.all(n == 0) and np.all(sc == 0)
    with pytest.raises(capi.StbError) as e:
        idx.search_filtered(Q, rr, top_k=1025)
    assert e.value.status == capi.STB_ERR_ARG
    got, n, sc = idx.search_filtered(np.zeros((0, 256), np.float32), rr)        # nq = 0: no-op
    assert len(n) == 0
    # a filtered call between two unfiltered ones changes neither
    a = idx.search_batch(Q, nprobe=8, top_k=10, rerank=256)
    fa = idx.search_filtered(Q, rr, nprobe=8, top_k=10, rerank=256)
    b = idx.search_batch(Q, nprobe=8, top_k=10, rerank=256)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert idx.batch_last(0)["probe"].tolist() != []
    fb = idx.search_filtered(Q, rr, nprobe=8, top_k=10, rerank=256)
    assert all(np.array_equal(x, y) for x, y in zip(fa, fb))


def test_appended_rows_and_extend(ctx):
    rng = np.random.default_rng(4711)
    centers = make_centers(rng, 16)
    rows = clustered(rng, centers, 6000)
    extra = clustered(rng, centers, 500)
    base = 3 << 32
    c, idx = build(ctx, rows, 16, row_base=base, extra=len(extra))
    c.append(extra)
    allrows = np.concatenate([rows, extra])
    try:
        Q = extra[:6]                                           # each query's best row is appended
        rr = np.array([[base + 5500, base + 6500]], np.uint64)    # 500 indexed rows, then the 500 appended
        got, n, sc = idx.search_filtered(Q, rr, nprobe=16, top_k=10, rerank=1024)
        assert np.all(got["row"][got["row"] != U64MAX] < base + 6000) and np.all(n == 10)
        E = idx.export()
        check_predicted(idx, E, rows, Q, got, n, sc, 10, base, mask_of(rr, base, 6000), 16)
        assert np.all(sc == 500)
        assert idx.extend() == len(extra)
        E = idx.export()
        got, n, sc = idx.search_filtered(Q, rr, nprobe=16, top_k=10, rerank=1024)
        check_predicted(idx, E, allrows, Q, got, n, sc, 10, base, mask_of(rr, base, 6500), 16)
        assert [int(got[i]["row"][0]) for i in range(len(Q))] == [base + 6000 + i for i in range(len(Q))]
        for i, q in enumerate(Q):                                # every eligible code re-ranked: the exact scan
            assert_store_query(got[i], n[i], c, allrows, q, 10, rr, base)
    finally:
        idx.close(); c.close()


def test_chunked_call_equals_per_query_calls(ctx):
    rng = np.random.default_rng(515)
    centers = make_centers(rng, 16)
    rows = clustered(rng, centers, 5000)
    c, idx = build(ctx, rows, 16, row_base=1 << 40)
    try:
        mask, rr = doc_filter(rng, len(rows), 0.2, 1 << 40)
        Q = clustered(rng, centers, 4097)
        got, n, sc = idx.search_filtered(Q, rr, nprobe=4, top_k=8, rerank=64)
        for i in range(len(Q)):
            g1, n1, s1 = idx.search_filtered(Q[i:i + 1], rr, nprobe=4, top_k=8, rerank=64)
            assert np.array_equal(g1[0], got[i]) and n1[0] == n[i] and s1[0] == sc[i], i
        E = idx.export()
        check_predicted(idx, E, rows, Q[-1:], got[-1:], n[-1:], sc[-1:], 8, 1 << 40, mask, 4)
    finally:
        idx.close(); c.close()

"""GPU: K5 IVF-PQ index extended after the build (stb_ivfpq_extend, csrc/ivfpq.cu).

An extended index is held to the contracts of a built one.  Its layout is read back with
stb_debug_ivfpq_export and compared with the export before the extend: the quantisers are the same bits,
each list keeps its old entries as a prefix and gains the appended rows assigned to it in ascending row
order, and the forced side list grows by the appended forced rows.  An appended copy of an indexed row gets
that row's list and code bit for bit; fresh rows are checked against the f64 bounds of
test_gpu_ivfpq_contract.py::test_index_invariants.  Searches over an extended index are checked as the
other K5 files check a built one: exhaustive searches against the oracle, partial probes against the
batched search's prediction (helpers from test_gpu_ivfpq_batch.py).
"""

import os
import sys

import numpy as np
import pytest

import oracle
from semtools_b200 import capi

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_ivfpq_batch import (F64_SLOP, FUSED_CAP, INV_REL, RERANK_CAP, U, WARP_KEEP, adc_keys,  # noqa: E402
                                  assert_hits, bad_queries, check_batch, clustered, edge_corpus, edge_queries,
                                  forced_ref, gamma, make_centers, predict, scan_routes, search_on_route,
                                  v2_precondition)

pytestmark = pytest.mark.gpu

WORKSPACE_BATCH = 16384          # rows a workspace upsert appends at a time


def build(ctx, rows, nlist, capacity, row_base=0, iters=4):
    c = capi.Corpus(ctx, capacity, row_base=row_base)
    c.append(rows)
    return c, capi.IvfPq(c, nlist=nlist, train_rows=len(rows), iters=iters)


def lists_of(E):
    off = E["list_off"].astype(np.int64)
    return [(E["order"][off[l]:off[l + 1]], E["codes"][off[l]:off[l + 1]]) for l in range(len(off) - 1)]


def list_and_code(E, n):
    """(list of each row or -1 for a forced row, code of each row) over rows 0..n-1."""
    off = E["list_off"].astype(np.int64)
    lst = np.full(n, -1, np.int64)
    lst[E["order"]] = np.repeat(np.arange(len(off) - 1), np.diff(off))
    code = np.zeros((n, 32), np.uint8)
    code[E["order"]] = E["codes"]
    return lst, code


def same_export(a, b):
    return all(np.array_equal(a[k], b[k]) for k in ("centroids", "codebooks", "list_off", "order", "codes", "forced"))


def check_extension(E0, E1, rows, n0, n1):
    """E1 = E0 extended by rows [n0, n1)."""
    assert np.array_equal(E1["centroids"].view(np.uint32), E0["centroids"].view(np.uint32))
    assert np.array_equal(E1["codebooks"].view(np.uint32), E0["codebooks"].view(np.uint32))
    new_forced = np.flatnonzero(forced_ref(rows[n0:n1])) + n0
    assert np.array_equal(E1["forced"], np.concatenate([E0["forced"], new_forced]).astype(np.uint32))
    added = []
    for (o0, c0), (o1, c1) in zip(lists_of(E0), lists_of(E1)):
        assert np.array_equal(o1[:len(o0)], o0) and np.array_equal(c1[:len(o0)], c0)
        suffix = o1[len(o0):].astype(np.int64)
        assert np.all(suffix >= n0) and np.all(suffix < n1) and np.all(np.diff(suffix) > 0)
        assert np.all(np.diff(o1.astype(np.int64)) > 0)           # a built list is ascending too
        added.append(suffix)
    added = np.concatenate(added)
    assert np.array_equal(np.sort(np.concatenate([added, new_forced])), np.arange(n0, n1))
    assert np.array_equal(np.sort(np.concatenate([E1["order"], E1["forced"]])), np.arange(n1))


def check_assignment_and_codes(E, rows, sel):
    """The f64 bounds of test_gpu_ivfpq_contract.py::test_index_invariants for the listed rows `sel`: the
    assigned centroid is within the fp32 dot's error of the best, and each sub-space code is within the
    residual's and the distance's error of the nearest codebook entry."""
    lst, code = list_and_code(E, len(rows))
    sel = sel[lst[sel] >= 0]
    C = E["centroids"].astype(np.float64)
    X = rows[sel].astype(np.float64)
    L = lst[sel]
    g = gamma(256) + F64_SLOP
    for a in range(0, len(sel), 512):
        xb = X[a:a + 512]
        G, A = xb @ C.T, np.abs(xb) @ np.abs(C).T
        mine = np.arange(len(xb)), L[a:a + 512]
        assert np.all(G[mine] + g * A[mine] >= np.max(G - g * A, axis=1))
    cb = E["codebooks"].astype(np.float64)
    xh = X / np.linalg.norm(X, axis=1, keepdims=True)
    res = xh - C[L]
    k1 = ((1 + INV_REL) * (1 + U) - 1) * (1 + U)
    eps = np.abs(xh) * k1 + (np.abs(xh) + np.abs(C[L])) * U
    g10 = gamma(10) + F64_SLOP
    codes = code[sel]
    for s in range(32):
        for a in range(0, len(sel), 1024):
            R = res[a:a + 1024, None, 8 * s:8 * s + 8]
            ep = eps[a:a + 1024, None, 8 * s:8 * s + 8]
            diff = np.abs(R - cb[s][None])
            D = np.sum(diff ** 2, axis=2)
            beta = np.sum(ep * (2 * diff + ep), axis=2) + g10 * np.sum((diff + ep) ** 2, axis=2)
            ch = codes[a:a + 1024, s].astype(np.int64)
            i = np.arange(len(ch))
            assert np.all(D[i, ch] - beta[i, ch] <= np.min(D + beta, axis=1)), (s, a)


# ------------------------------------------------------------------------------------------- layout ---
def test_layout_over_a_series_of_extends(ctx):
    rng = np.random.default_rng(601)
    centers = make_centers(rng, 64)
    n0 = 20_000
    parts = [clustered(rng, centers, n0), clustered(rng, centers, 1)] + \
        [clustered(rng, centers, WORKSPACE_BATCH) for _ in range(3)]
    parts[0][17, 3] = np.nan
    parts[2][5] = 0.0                                           # forced rows in the appended batches
    parts[3][WORKSPACE_BATCH - 1] *= np.float32(1e22)
    rows = np.concatenate(parts)
    c, idx = build(ctx, parts[0], nlist=64, capacity=len(rows))
    try:
        E = idx.export()
        for (o, _) in lists_of(E):                              # the build's lists are ascending
            assert np.all(np.diff(o.astype(np.int64)) > 0)
        assert idx.extend() == 0                                # nothing appended: nothing changes
        assert same_export(idx.export(), E) and idx.stats()["rows"] == n0
        n = n0
        for part in parts[1:]:
            c.append(part)
            assert idx.extend() == len(part)
            E1 = idx.export()
            check_extension(E, E1, rows, n, n + len(part))
            n += len(part)
            assert idx.stats()["rows"] == n and idx.stats()["index_bytes"] > 0
            assert idx.extend() == 0 and same_export(idx.export(), E1)
            E = E1
    finally:
        idx.close(); c.close()


def test_appended_copies_get_their_originals_bits_and_fresh_rows_the_build_s_rule(ctx):
    rng = np.random.default_rng(602)
    centers = make_centers(rng, 32)
    n0, m, fresh = 8000, 5000, 3000
    base = clustered(rng, centers, n0)
    base[7, 5] = np.nan; base[4000] = 0.0
    extra = clustered(rng, centers, fresh)
    extra[11] *= np.float32(1e-25)
    rows = np.concatenate([base, base[:m], extra])
    c, idx = build(ctx, base, nlist=64, capacity=len(rows))
    try:
        E0 = idx.export()
        c.append(base[:m])
        assert idx.extend() == m
        c.append(extra)
        assert idx.extend() == fresh
        E = idx.export()
        check_extension(E0, E, rows, n0, len(rows))
        lst, code = list_and_code(E, len(rows))
        assert np.array_equal(lst[n0:n0 + m], lst[:m])          # copies: the original's list (-1: forced) ...
        assert np.array_equal(code[n0:n0 + m][lst[:m] >= 0], code[:m][lst[:m] >= 0])   # ... and code
        assert lst[n0 + 7] == -1 and lst[n0 + m + 11] == -1
        check_assignment_and_codes(E, rows, np.arange(n0 + m, len(rows)))
    finally:
        idx.close(); c.close()


# ------------------------------------------------------------------------- exhaustive search is exact ---
@pytest.mark.parametrize("n,n0", [(1000, 400), (3000, 1200)])
def test_exhaustive_search_over_an_extended_index_is_exact(ctx, n, n0):
    """Edge rows (NaN / +-inf, zero, 1e-25, 1e22, duplicates) on both sides of the build, two extends,
    nlist 3, row_base >= 2^32: with every list probed and every code re-ranked, each search path returns
    the oracle's answer over all n rows."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(603 + n)
    rows, p = edge_corpus(rng, n)
    assert np.any(p < n0) and np.any(p >= n0)
    assert forced_ref(rows[:n0]).any() and forced_ref(rows[n0:]).any()
    base = 3 << 32
    c, idx = build(ctx, rows[:n0], nlist=3, capacity=n, row_base=base)
    try:
        half = (n0 + n) // 2
        for a, b in [(n0, half), (half, n)]:
            c.append(rows[a:b])
            assert idx.extend() == b - a
        n_listed = n - int(forced_ref(rows).sum())
        assert idx.stats()["rows"] == n
        Q = np.stack(edge_queries(rng, rows, p) + [rows[p[13]], rows[p[3]]])
        ks = sorted({1, 10, 1024, n})

        def oracle_hits(q, k):
            want_rows, want_d = oracle.search_rows(rows, q, k)
            return [int(r) + base for r in want_rows], np.asarray(want_d, np.float64)

        def single(k, rerank_min=0):
            for q in Q:
                got, n_scan = search_on_route(ctx, idx, q, 3, k, max(n, k, rerank_min))
                assert n_scan == n_listed
                want_rows, want_d = oracle_hits(q, k)
                assert got["row"].tolist() == want_rows
                assert np.array_equal(got["distance"].view(np.uint64), want_d.view(np.uint64))

        if n_listed > 1024:
            for k in ks:                                        # v1 by itself (rerank > 1024)
                single(k)
            return
        for k in ks:
            single(k)                                           # fused v2
        for k in ks:
            single(k, FUSED_CAP + 1)                            # v1
        dev = torch.device("cuda:0")
        q_dev = torch.from_numpy(np.ascontiguousarray(Q)).to(dev)
        for k in (1, 10, 1024):
            got, cnt, scanned = idx.search_batch(Q, nprobe=3, top_k=k, rerank=RERANK_CAP)
            hits = torch.zeros((len(Q), k, 2), dtype=torch.float64, device=dev)
            st = torch.zeros((len(Q), 2), dtype=torch.int32, device=dev)
            torch.cuda.synchronize()
            idx.search_batch_dev(q_dev.data_ptr(), len(Q), 3, k, RERANK_CAP, hits.data_ptr(), st.data_ptr())
            c.ctx.sync()
            raw = np.ascontiguousarray(hits.cpu().numpy()).view(capi.HIT_DTYPE).reshape(len(Q), k)
            sth = st.cpu().numpy()
            for i, q in enumerate(Q):
                want_rows, want_d = oracle_hits(q, k)
                assert int(scanned[i]) == n_listed and int(sth[i, 1]) == n_listed
                assert_hits(got[i], cnt[i], want_rows, want_d)
                assert_hits(raw[i], sth[i, 0], want_rows, want_d)
    finally:
        idx.close(); c.close()


# ---------------------------------------------------------------------- clustered index (partial probe) ---
@pytest.fixture(scope="module")
def extended_index(ctx):
    rng = np.random.default_rng(604)
    n0, n, nlist = 40_000, 60_000, 64
    centers = make_centers(rng, 64)
    rows = clustered(rng, centers, n)
    Q = np.concatenate([clustered(rng, centers, 24), rng.standard_normal((2, 256)).astype(np.float32)])
    rows[123] = Q[0] * np.float32(1e-25)                    # forced, in the build
    rows[45_678, 9] = np.nan                                 # forced, appended
    rows[50_000] = Q[1]                                      # appended exact matches of two queries
    rows[59_999] = Q[2]
    base = 7 << 32
    c, idx = build(ctx, rows[:n0], nlist, capacity=n, row_base=base, iters=6)
    for a, b in [(n0, 50_000), (50_000, n)]:
        c.append(rows[a:b])
        idx.extend()
    E = idx.export()
    yield rows, Q, c, idx, E, base
    idx.close(); c.close()


@pytest.mark.parametrize("rerank", [64, 1024])
def test_predicted_bits_at_partial_probe_after_extend(extended_index, rerank):
    rows, Q, c, idx, E, base = extended_index
    assert len(E["order"]) + len(E["forced"]) == len(rows) and E["forced"].tolist() == [123, 45_678]
    got, n, scanned = idx.search_batch(Q, nprobe=8, top_k=10, rerank=rerank)
    check_batch(idx, E, rows, Q, got, n, scanned, 10, base)
    # the appended copies of queries 1 and 2 come back (behind the appended NaN row: distance 0, lower row)
    assert got[1]["row"][:2].tolist() == [base + 45_678, base + 50_000]
    assert got[2]["row"][:2].tolist() == [base + 45_678, base + 59_999]


def test_single_v2_agrees_with_the_batch_where_exact_after_extend(extended_index):
    rows, Q, c, idx, E, base = extended_index
    Qb = np.concatenate([Q, np.stack(bad_queries(np.random.default_rng(5)))])
    got, n, scanned = idx.search_batch(Qb, nprobe=8, top_k=10, rerank=512)
    agreed = 0
    for i, q in enumerate(Qb):
        info = idx.batch_last(i)
        _, keys = adc_keys(E, info)
        want_rows, want_d, _ = predict(E, info, rows, q, 10, base)
        assert_hits(got[i], n[i], want_rows, want_d)
        if v2_precondition(keys, 512):
            one, s1 = idx.search(q, nprobe=8, top_k=10, rerank=512)
            assert s1 == int(scanned[i]) and np.array_equal(got[i][: n[i]], one), i
            agreed += 1
    assert agreed >= len(Q) // 2


def test_skewed_append_takes_the_exact_slow_route(ctx, monkeypatch):
    """Tens of thousands of rows appended around one centre: one list grows far past 2048 codes and past
    what the scan warps keep, and the batch still answers as predicted."""
    rng = np.random.default_rng(605)
    centers = make_centers(rng, 64)
    n0, m = 30_000, 40_000
    rows = np.concatenate([clustered(rng, centers, n0), clustered(rng, centers[:1], m)])
    c, idx = build(ctx, rows[:n0], nlist=64, capacity=len(rows), row_base=1 << 32)
    try:
        sizes0 = np.diff(idx.export()["list_off"].astype(np.int64))
        c.append(rows[n0:])
        assert idx.extend() == m
        E = idx.export()
        sizes = np.diff(E["list_off"].astype(np.int64))
        big = int(np.argmax(sizes - sizes0))
        assert sizes[big] - sizes0[big] > m // 4 and sizes[big] > 4 * 2048
        Q = np.concatenate([clustered(rng, centers[:1], 12), clustered(rng, centers, 4)])
        rerank = 1024
        got, n, scanned = idx.search_batch(Q, nprobe=4, top_k=10, rerank=rerank)
        check_batch(idx, E, rows, Q, got, n, scanned, 10, base=1 << 32)
        keys_of = [adc_keys(E, idx.batch_last(i))[1] for i in range(len(Q))]
        assert max(len(k) for k in keys_of) >= sizes[big]    # the grown list was probed
        most = max(scan_routes(k, rerank, WARP_KEEP)[1] for k in keys_of)
        keep = max(1, most // 2)                              # some warp holds more winners than it keeps
        assert not all(scan_routes(k, rerank, keep)[0] for k in keys_of)
        monkeypatch.setenv("STB_IVFPQ_BATCH_KEEP", str(keep))
        try:
            got, n, scanned = idx.search_batch(Q, nprobe=4, top_k=10, rerank=rerank)
        finally:
            monkeypatch.delenv("STB_IVFPQ_BATCH_KEEP")
        check_batch(idx, E, rows, Q, got, n, scanned, 10, base=1 << 32)
    finally:
        idx.close(); c.close()


# ------------------------------------------------------------------------------------------- errors ---
def _answers(idx, Q):
    single = [idx.search(q, nprobe=4, top_k=10, rerank=256) for q in Q]
    return single, idx.search_batch(Q, nprobe=4, top_k=10, rerank=256)


def _same_answers(a, b):
    (s0, (g0, n0, sc0)), (s1, (g1, n1, sc1)) = a, b
    assert all(x[1] == y[1] and np.array_equal(x[0], y[0]) for x, y in zip(s0, s1))
    assert np.array_equal(g0, g1) and np.array_equal(n0, n1) and np.array_equal(sc0, sc1)


def test_errors_leave_the_index_usable(ctx):
    rng = np.random.default_rng(606)
    centers = make_centers(rng, 8)
    rows = clustered(rng, centers, 3000)
    rows[:1000] = 0.0                                        # 1000 forced rows
    more = clustered(rng, centers, 200)
    more[::8] = 0.0                                          # 25 more: 1025 > 1024
    c, idx = build(ctx, rows, nlist=8, capacity=len(rows) + len(more), row_base=2 << 32)
    try:
        Q = np.concatenate([rows[1000:1004], rng.standard_normal((2, 256)).astype(np.float32)])
        E, ans = idx.export(), _answers(idx, Q)
        c.append(more)
        for _ in range(2):                                   # refused each time, nothing changes
            with pytest.raises(capi.StbError) as e:
                idx.extend()
            assert e.value.status == capi.STB_ERR_STATE
            assert same_export(idx.export(), E) and idx.stats()["rows"] == len(rows)
            _same_answers(_answers(idx, Q), ans)
        c.clear()                                            # fewer rows than the index holds
        with pytest.raises(capi.StbError) as e:
            idx.extend()
        assert e.value.status == capi.STB_ERR_STATE
        c.append(rows); c.append(clustered(rng, centers, 10))   # refilled and longer: a new epoch all the same
        with pytest.raises(capi.StbError) as e:
            idx.extend()
        assert e.value.status == capi.STB_ERR_STATE
        assert same_export(idx.export(), E) and idx.stats()["rows"] == len(rows)
        _same_answers(_answers(idx, Q), ans)
        assert capi.lib().stb_ivfpq_extend(None, None) == capi.STB_ERR_ARG
    finally:
        idx.close(); c.close()


# ------------------------------------------------------------------------------------ stream ordering ---
def test_device_searches_around_an_extend_see_the_old_then_the_new_index(ctx):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(607)
    centers = make_centers(rng, 64)
    rows = clustered(rng, centers, 30_000)
    Q = clustered(rng, centers, 4096)
    extra = np.ascontiguousarray(Q[:64])                     # appended exact matches of the first queries
    c, idx = build(ctx, rows, nlist=64, capacity=len(rows) + len(extra), row_base=3 << 32)
    try:
        c.append(extra)
        before = idx.search_batch(Q, nprobe=8, top_k=10, rerank=256)
        dev = torch.device("cuda:0")
        q_dev = torch.from_numpy(Q).to(dev)
        outs = [(torch.zeros((len(Q), 10, 2), dtype=torch.float64, device=dev),
                 torch.zeros((len(Q), 2), dtype=torch.int32, device=dev)) for _ in range(2)]
        torch.cuda.synchronize()
        idx.search_batch_dev(q_dev.data_ptr(), len(Q), 8, 10, 256, outs[0][0].data_ptr(), outs[0][1].data_ptr())
        assert idx.extend() == len(extra)
        idx.search_batch_dev(q_dev.data_ptr(), len(Q), 8, 10, 256, outs[1][0].data_ptr(), outs[1][1].data_ptr())
        c.ctx.sync()
        after = idx.search_batch(Q, nprobe=8, top_k=10, rerank=256)
        assert not np.array_equal(before[0], after[0])
        assert np.all(after[0][:64]["row"][:, 0] == (3 << 32) + len(rows) + np.arange(64))
        for (h, st), (want, wn, ws) in zip(outs, (before, after)):
            raw = np.ascontiguousarray(h.cpu().numpy()).view(capi.HIT_DTYPE).reshape(len(Q), 10)
            sth = st.cpu().numpy()
            assert np.array_equal(raw, want) and np.array_equal(sth[:, 0], wn) and np.array_equal(sth[:, 1], ws)
    finally:
        idx.close(); c.close()

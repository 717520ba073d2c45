"""GPU: K5 IVF-PQ index kept current through corpus updates and removals (stb_ivfpq_update /
stb_ivfpq_remove, csrc/ivfpq.cu on top of the corpus calls in csrc/api.cu).

Each test keeps a numpy model next to the corpus: the rows, the number of indexed rows, and the (list, code)
of every indexed row (list -1: a forced row).  A removed row leaves the model, an update with a copy of
another indexed row takes that row's (list, code), and an update with a fresh value takes what the export
says once the f64 bounds of test_gpu_ivfpq_extend.py::check_assignment_and_codes accept it.  The expected
export is derived from the model alone -- each list is its rows in ascending order, the forced list likewise --
and must equal the index's byte for byte.  The corpus side is held to test_gpu_corpus_update.py's `check`,
searches to the oracle (exhaustive) or to the batched search's prediction (partial probe).
"""

import os
import sys

import numpy as np
import pytest

import oracle
from semtools_b200 import capi

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_corpus_update import CHUNK, bits, check, scattered_ranges, snapshot  # noqa: E402
from test_gpu_ivfpq_batch import (FUSED_CAP, RERANK_CAP, assert_hits, check_batch, clustered, edge_corpus,  # noqa: E402
                                  edge_queries, forced_ref, make_centers, search_on_route)
from test_gpu_ivfpq_extend import check_assignment_and_codes, list_and_code, same_export  # noqa: E402
from test_gpu_ivfpq_filter import assert_store_query  # noqa: E402

pytestmark = pytest.mark.gpu

FORCED_CAP = 1024


# ------------------------------------------------------------------------------------------- model ---
class Model:
    """Rows of the corpus, indexed rows [0, n), and (list, code) of each indexed row."""

    def __init__(self, rows, E, n):
        self.rows = np.array(rows, dtype=np.float32)
        self.n = n
        self.lst, self.code = list_and_code(E, n)
        self.C, self.cb = E["centroids"].copy(), E["codebooks"].copy()

    def remove(self, ranges, base=0):
        keep = np.ones(len(self.rows), bool)
        for b, e in np.asarray(ranges, np.int64).reshape(-1, 2):
            keep[b - base:e - base] = False
        self.rows = np.ascontiguousarray(self.rows[keep])
        k = keep[:self.n]
        self.lst, self.code, self.n = self.lst[k], self.code[k], int(k.sum())

    def update(self, loc, vals, E=None):
        """rows[loc] = vals, fresh values: the indexed ones take E's (list, code) once the f64 bounds accept them"""
        loc = np.asarray(loc, np.int64)
        self.rows[loc] = vals
        fresh = loc[loc < self.n]
        if len(fresh):
            lst, code = list_and_code(E, self.n)
            self.lst[fresh], self.code[fresh] = lst[fresh], code[fresh]
            assert np.array_equal(self.lst[fresh] < 0, forced_ref(self.rows[fresh]))
            check_assignment_and_codes(E, self.rows[:self.n], fresh)

    def copy_rows(self, dst, src):
        """rows[dst] = rows[src] (src indexed and not in dst): the copies' expected (list, code)."""
        dst, src = np.asarray(dst, np.int64), np.asarray(src, np.int64)
        self.rows[dst] = self.rows[src]
        d = dst < self.n
        self.lst[dst[d]], self.code[dst[d]] = self.lst[src[d]], self.code[src[d]]

    def extended(self, E, n):
        """after an extend to n rows: the new rows take E's (list, code) once the bounds accept them"""
        n0, self.n = self.n, n
        lst, code = list_and_code(E, n)
        self.lst, self.code = np.concatenate([self.lst, lst[n0:]]), np.concatenate([self.code, code[n0:]])
        assert np.array_equal(self.lst[n0:] < 0, forced_ref(self.rows[n0:n]))
        check_assignment_and_codes(E, self.rows[:n], np.arange(n0, n))

    def export(self):
        listed = np.flatnonzero(self.lst >= 0)
        o = listed[np.lexsort((listed, self.lst[listed]))]
        off = np.concatenate([[0], np.cumsum(np.bincount(self.lst[listed], minlength=len(self.C)))])
        return {"centroids": self.C, "codebooks": self.cb, "list_off": off.astype(np.uint32),
                "order": o.astype(np.uint32), "codes": self.code[o], "forced": np.flatnonzero(self.lst < 0).astype(np.uint32)}


def check_index(idx, c, m):
    """the index's export is the model's, byte for byte, and the corpus holds the model's rows"""
    E = idx.export()
    want = m.export()
    for k in ("centroids", "codebooks"):
        assert np.array_equal(E[k].view(np.uint32), want[k].view(np.uint32)), k
    for k in ("list_off", "order", "codes", "forced"):
        assert np.array_equal(E[k], want[k]), k
    assert idx.stats()["rows"] == m.n
    assert np.array_equal(np.sort(np.concatenate([E["order"], E["forced"]])), np.arange(m.n))
    assert np.array_equal(bits(c.read()), bits(m.rows))
    return E


def build(ctx, rows, nlist, tail=None, row_base=0, iters=4, prepare=True):
    """corpus of rows (+ an unindexed tail), copies prepared over all of them, index over rows"""
    c = capi.Corpus(ctx, len(rows) + (0 if tail is None else len(tail)), row_base=row_base)
    c.append(rows)
    idx = capi.IvfPq(c, nlist=nlist, train_rows=len(rows), iters=iters)
    if tail is not None:
        c.append(tail)
    if prepare:
        c.prepare(3)
    E = idx.export()
    m = Model(rows if tail is None else np.concatenate([rows, tail]), E, len(rows))
    return c, idx, m


# ------------------------------------------------------------------------------------------ layout ---
def test_removal_layout(ctx):
    rng = np.random.default_rng(701)
    centers = make_centers(rng, 64)
    rows, tail = clustered(rng, centers, 20_000), clustered(rng, centers, 3000)
    rows[17, 3] = np.nan; rows[5000] = 0.0; rows[19_000] *= np.float32(1e22)
    c, idx, m = build(ctx, rows, 64, tail)
    try:
        steps = [np.array([[0, 100]]),                                       # the front (forced row 17)
                 scattered_ranges(rng, m.n - 200, 50) + 10,                   # the middle
                 None]                                                        # across the indexed end
        for r in steps:
            if r is None:
                r = np.array([[m.n - 50, m.n + 200]])
            r = np.asarray(r, np.uint64)
            idx.remove(r)
            m.remove(r)
            check_index(idx, c, m)
            check(ctx, c, m.rows, maintained=False)          # forced rows: the copies are unusable
        assert idx.extend() == len(m.rows) - m.n                              # exactly the unindexed tail
        m.extended(idx.export(), len(m.rows))
        check_index(idx, c, m)
        k = 12_345                                                            # everything but one row
        r = np.array([[0, k], [k + 1, len(m.rows)]], np.uint64)
        idx.remove(r)
        m.remove(r)
        E = check_index(idx, c, m)
        assert m.n == 1 and len(E["order"]) + len(E["forced"]) == 1
        got, _ = idx.search(m.rows[0], nprobe=64, top_k=3, rerank=64)
        assert got["row"].tolist() == [0]
    finally:
        idx.close(); c.close()


def test_update_layout(ctx):
    rng = np.random.default_rng(702)
    centers = make_centers(rng, 32)
    rows, tail = clustered(rng, centers, 12_000), clustered(rng, centers, 500)
    rows[40] = 0.0; rows[41, 9] = np.inf; rows[7000] *= np.float32(1e-25)       # forced
    c, idx, m = build(ctx, rows, 32, tail, row_base=5 << 32)
    base = 5 << 32
    try:
        # copies of other indexed rows: listed -> listed, listed -> forced (copy of 40), forced -> listed
        src = np.array([40, 100, 101, 2000, 9000, 11_999])
        dst = np.array([3, 41, 500, 501, 7000, 8000])
        idx.update(dst + base, m.rows[src])
        m.copy_rows(dst, src)
        check_index(idx, c, m)
        # fresh values, and rows of the unindexed tail (the corpus only)
        loc = np.sort(np.concatenate([rng.choice(np.arange(50, 12_000), 700, replace=False), [40, 41], 12_000 + np.arange(0, 500, 7)]))
        vals = clustered(rng, centers, len(loc))
        vals[np.searchsorted(loc, 60 if 60 in loc else loc[10])] = 0.0       # listed -> forced
        idx.update(loc + base, vals)
        m.update(loc, vals, idx.export())
        E = check_index(idx, c, m)
        assert 40 not in E["forced"] and 41 not in E["forced"]               # forced -> listed
        check(ctx, c, m.rows, maintained=False)
        assert idx.extend() == 500
        m.extended(idx.export(), len(m.rows))
        check_index(idx, c, m)
    finally:
        idx.close(); c.close()


def test_update_of_several_chunks_and_its_refusal(ctx):
    """An update larger than one staging chunk is uploaded twice; refused for its forced rows, it writes
    nothing -- even when they lie in its second chunk."""
    rng = np.random.default_rng(703)
    centers = make_centers(rng, 64)
    n = CHUNK + 40_000
    rows = clustered(rng, centers, n)
    c, idx, m = build(ctx, rows, 64, prepare=False)
    try:
        loc = np.arange(1000, n, 1, dtype=np.int64)[: CHUNK + 20_000]
        src = (loc + 7) % 1000                                               # copies of rows 0..999
        vals = m.rows[src].copy()
        before, E0 = snapshot(c), idx.export()
        bad = vals.copy()
        bad[CHUNK + 100: CHUNK + 100 + FORCED_CAP + 1] = 0.0                 # 1025 forced rows, second chunk
        with pytest.raises(capi.StbError) as e:
            idx.update(loc, bad)
        assert e.value.status == capi.STB_ERR_STATE
        assert all(np.array_equal(a, b) for a, b in zip(before, snapshot(c))) and same_export(idx.export(), E0)
        idx.update(loc, vals)
        m.copy_rows(loc, src)
        check_index(idx, c, m)
    finally:
        idx.close(); c.close()


def test_same_rows_give_the_same_index(ctx):
    """Two sequences of calls reaching the same rows give byte-identical exports: one call each of update,
    remove and extend; then, from there, other values written and written back, and the last rows removed
    from the back in two calls, appended again and extended in two steps."""
    rng = np.random.default_rng(704)
    centers = make_centers(rng, 32)
    rows, tail = clustered(rng, centers, 15_000), clustered(rng, centers, 2000)
    rows[3] = 0.0; tail[5, 1] = np.nan
    c, idx, m = build(ctx, rows, 32, tail, prepare=False)
    try:
        gone = np.array([[100, 400], [5000, 5003], [14_990, 15_500]], np.uint64)    # the last crosses into the tail
        up = np.sort(rng.choice(np.arange(400, 5000), 3000, replace=False))
        vals = clustered(rng, centers, len(up))
        vals[::500] = 0.0
        idx.update(up, vals)
        idx.remove(gone)
        idx.extend()
        E1, R1 = idx.export(), c.read()
        n = len(R1)
        assert idx.stats()["rows"] == n and len(E1["forced"]) >= 6
        # other values (forced ones among them) over listed and forced rows, written in two calls
        loc = np.sort(np.concatenate([E1["forced"][:4].astype(np.int64), rng.choice(n - 3000, 2000, replace=False)]))
        loc = np.unique(loc)
        other = clustered(rng, make_centers(rng, 8), len(loc))
        other[::300] = 0.0
        h = len(loc) // 2
        idx.update(loc[h:], other[h:])
        idx.update(loc[:h], other[:h])
        assert not np.array_equal(idx.export()["order"], E1["order"])
        # the last 3000 rows removed from the back, appended again and extended in two steps
        idx.remove(np.array([[n - 1000, n]], np.uint64))
        idx.remove(np.array([[n - 3000, n - 1000]], np.uint64))
        assert idx.stats()["rows"] == n - 3000
        c.append(R1[n - 3000:n - 1500]); idx.extend()
        c.append(R1[n - 1500:]); idx.extend()
        idx.update(loc, R1[loc])                                                     # the old values back
        E2, R2 = idx.export(), c.read()
        assert np.array_equal(bits(R1), bits(R2))
        for k in ("centroids", "codebooks", "list_off", "order", "codes", "forced"):
            assert np.array_equal(bits(E1[k]), bits(E2[k])), k
    finally:
        idx.close(); c.close()


# ------------------------------------------------------------------------------------------- search ---
@pytest.mark.parametrize("n,n0", [(1200, 700)])
def test_exhaustive_search_after_a_mixed_sequence_is_exact(ctx, n, n0):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(705)
    rows, p = edge_corpus(rng, n)
    base = 3 << 32
    c, idx, m = build(ctx, rows[:n0], 3, rows[n0:], row_base=base)
    try:
        # edge values written over indexed and unindexed rows, removals on both sides of the indexed end
        loc = np.array(sorted({int(x) for x in rng.choice(n, 40, replace=False)} - {int(x) for x in p[:14]}))
        vals = clustered(rng, make_centers(rng, 8), len(loc), spread=2.0)
        vals[0] = rows[p[0]]; vals[1] = 0.0; vals[2, 5] = np.nan; vals[3, 6] = -np.inf
        vals[4] = rows[p[10]] * np.float32(1e-25); vals[5] = rows[p[12]] * np.float32(1e22); vals[6] = rows[p[0]]
        idx.update(loc + base, vals)
        m.update(loc, vals, idx.export())
        gone = np.array([[20, 90], [600, 760], [1100, 1130]], np.uint64)
        idx.remove(gone + np.uint64(base))
        m.remove(gone)
        idx.extend()
        m.extended(idx.export(), len(m.rows))
        E = check_index(idx, c, m)
        R = m.rows
        n_listed = len(E["order"])
        assert n_listed <= RERANK_CAP and len(E["forced"]) >= 6
        Q = np.stack(edge_queries(rng, R, rng.permutation(len(R))[:16]) + [vals[0], vals[5]])

        def want(q, k):
            r, d = oracle.search_rows(R, q, k)
            return [int(x) + base for x in r], np.asarray(d, np.float64)

        for k in (1, 10, 1024):
            for rerank_min in (0, FUSED_CAP + 1):                  # fused v2, then v1
                for q in Q:
                    got, n_scan = search_on_route(ctx, idx, q, 3, k, max(n_listed, k, rerank_min))
                    wr, wd = want(q, k)
                    assert n_scan == n_listed and got["row"].tolist() == wr
                    assert np.array_equal(got["distance"].view(np.uint64), wd.view(np.uint64))
            dev = torch.device("cuda:0")
            q_dev = torch.from_numpy(np.ascontiguousarray(Q)).to(dev)
            hits = torch.zeros((len(Q), k, 2), dtype=torch.float64, device=dev)
            st = torch.zeros((len(Q), 2), dtype=torch.int32, device=dev)
            hits1 = torch.zeros((k, 2), dtype=torch.float64, device=dev)
            st1 = torch.zeros(2, dtype=torch.int32, device=dev)
            torch.cuda.synchronize()
            idx.search_batch_dev(q_dev.data_ptr(), len(Q), 3, k, RERANK_CAP, hits.data_ptr(), st.data_ptr())
            c.ctx.sync()
            raw = np.ascontiguousarray(hits.cpu().numpy()).view(capi.HIT_DTYPE).reshape(len(Q), k)
            sth = st.cpu().numpy()
            got, cnt, scanned = idx.search_batch(Q, nprobe=3, top_k=k, rerank=RERANK_CAP)
            for i, q in enumerate(Q):
                wr, wd = want(q, k)
                assert int(scanned[i]) == n_listed and int(sth[i, 1]) == n_listed
                assert_hits(got[i], cnt[i], wr, wd)
                assert_hits(raw[i], sth[i, 0], wr, wd)
                idx.search_dev(q_dev[i].data_ptr(), 3, k, RERANK_CAP, hits1.data_ptr(), st1.data_ptr())
                c.ctx.sync()
                one = np.ascontiguousarray(hits1.cpu().numpy()).view(capi.HIT_DTYPE).reshape(k)
                assert_hits(one, int(st1.cpu().numpy()[0]), wr, wd)
        ranges = np.array([[base + 5, base + 300], [base + 400, base + 401], [base + 700, base + len(R) + 50]], np.uint64)
        for dist in (None, 0.9):
            got, cnt, _ = idx.search_filtered(Q, ranges, max_distance=dist, nprobe=3, top_k=10, rerank=RERANK_CAP)
            for i, q in enumerate(Q):
                assert_store_query(got[i], cnt[i], c, R, q, 10, ranges, base, dist)
    finally:
        idx.close(); c.close()


def test_predicted_hits_at_partial_probe_after_a_mixed_sequence(ctx):
    rng = np.random.default_rng(706)
    centers = make_centers(rng, 64)
    rows = clustered(rng, centers, 50_000)
    base = 9 << 32
    c, idx, m = build(ctx, rows[:40_000], 64, rows[40_000:], row_base=base, prepare=False)
    try:
        Q = np.concatenate([clustered(rng, centers, 24), rng.standard_normal((2, 256)).astype(np.float32)])
        loc = np.sort(rng.choice(45_000, 8000, replace=False))
        vals = clustered(rng, np.roll(centers, 1, axis=1), len(loc))          # rows from shifted centres
        vals[:3] = Q[:3]                                                      # exact matches of three queries
        idx.update(loc + base, vals)
        m.update(loc, vals, idx.export())
        gone = scattered_ranges(rng, 50_000, 200)
        idx.remove(gone + np.uint64(base))
        m.remove(gone)
        idx.extend()
        m.extended(idx.export(), len(m.rows))
        E = check_index(idx, c, m)
        for rerank in (64, 1024):
            got, n, scanned = idx.search_batch(Q, nprobe=8, top_k=10, rerank=rerank)
            check_batch(idx, E, m.rows, Q, got, n, scanned, 10, base)
    finally:
        idx.close(); c.close()


# ------------------------------------------------------------------------------------- corpus side ---
def test_corpus_side_tier_statistics_and_co_scan(ctx):
    from test_gpu_corpus_update import DevSeries
    rng = np.random.default_rng(707)
    centers = make_centers(rng, 32)
    rows = clustered(rng, centers, 60_001)
    c, idx, m = build(ctx, rows, 32)
    try:
        qs = clustered(rng, centers, 8)
        s = DevSeries(len(qs))
        s.launch_all(c, qs)
        for call, model_call in ((lambda: idx.update(np.arange(0, 60_000, 3), m.rows[1:60_001:3][:20_000]), None),
                                 (lambda: idx.remove(np.array([[10, 2000]], np.uint64)), None)):
            c.search(qs[0], top_k=5)
            assert sum(v["tries"] for v in c.tier_stats().values()) >= 1
            call()
            assert all(v["tries"] == 0 and v["proven"] == 0 for v in c.tier_stats().values())
            s.launch_all(c, qs)
            ctx.sync()
            assert ctx.coscan_offsets(len(qs))[0] == 0                        # the call ended the co-scan series
        m.copy_rows(np.arange(0, 60_000, 3), np.arange(1, 60_001, 3)[:20_000])
        m.remove(np.array([[10, 2000]]))
        check_index(idx, c, m)
        check(ctx, c, m.rows)
        for i, q in enumerate(qs):
            s.check(ctx, i, m.rows, q)
    finally:
        idx.close(); c.close()


# ------------------------------------------------------------------------------------------ refusals ---
def test_refusals_change_nothing(ctx):
    rng = np.random.default_rng(708)
    centers = make_centers(rng, 16)
    base = 1000
    rows = clustered(rng, centers, 20_000)
    rows[:FORCED_CAP - 2] = 0.0                                               # 1022 forced rows
    c, idx, m = build(ctx, rows, 16, clustered(rng, centers, 100), row_base=base)
    try:
        L = capi.lib()
        before, E0 = snapshot(c), idx.export()
        three = clustered(rng, centers, 3)

        def upd(ids, vals=three):
            ids = np.asarray(ids, np.uint64)
            return L.stb_ivfpq_update(idx._h, ids.ctypes.data, vals.ctypes.data, len(ids))

        def rem(r):
            r = np.asarray(r, np.uint64).reshape(-1, 2)
            return L.stb_ivfpq_remove(idx._h, r.ctypes.data, r.shape[0])

        R, A, S = capi.STB_ERR_RANGE, capi.STB_ERR_ARG, capi.STB_ERR_STATE
        zeros3 = np.zeros((3, 256), np.float32)
        one = np.array([base], np.uint64)
        cases = [
            (upd([base + 5, base + 4, base + 6]), R), (upd([base + 5, base + 5, base + 6]), R),
            (upd([base + 1, base + 2, base + 20_100]), R), (upd([base - 1, base + 2, base + 3]), R),
            (L.stb_ivfpq_update(idx._h, None, three.ctypes.data, 3), A),
            (L.stb_ivfpq_update(idx._h, one.ctypes.data, None, 1), A),
            (L.stb_ivfpq_update(None, one.ctypes.data, three.ctypes.data, 1), A),
            (rem([[base + 10, base + 20], [base + 5, base + 8]]), R), (rem([[base + 10, base + 20], [base + 19, base + 30]]), R),
            (rem([[base + 10, base + 10]]), R), (rem([[base + 10, base + 20], [base + 20_090, base + 20_101]]), R),
            (rem([[base - 2, base + 1]]), R), (L.stb_ivfpq_remove(idx._h, None, 2), A), (L.stb_ivfpq_remove(None, None, 1), A),
            (upd([base + 5000, base + 5001, base + 5002], zeros3), S),        # 1025 forced rows
        ]
        assert [rc for rc, _ in cases] == [w for _, w in cases]
        assert L.stb_ivfpq_update(idx._h, None, None, 0) == 0 and L.stb_ivfpq_remove(idx._h, None, 0) == 0
        idx2 = capi.IvfPq(c, nlist=16, train_rows=4096, iters=2)              # a second live index
        for call in (lambda: idx.update(np.array([base + 3000]), three[:1]), lambda: idx.remove(np.array([[base + 1, base + 2]])),
                     lambda: idx2.remove(np.array([[base + 1, base + 2]]))):
            with pytest.raises(capi.StbError) as e:
                call()
            assert e.value.status == S
        idx2.close()
        assert all(np.array_equal(a, b) for a, b in zip(before, snapshot(c))) and same_export(idx.export(), E0)
        # still usable: searches, an update that frees forced rows, then two more forced ones, and extend
        got, _ = idx.search(m.rows[5000], nprobe=16, top_k=1, rerank=64)
        assert got["row"].tolist() == [base + 5000]
        loc = np.array([0, 1, 5000, 5001])
        vals = np.concatenate([clustered(rng, centers, 2), zeros3[:2]])
        idx.update(loc + base, vals)
        m.update(loc, vals, idx.export())
        assert idx.extend() == 100
        m.extended(idx.export(), len(m.rows))
        check_index(idx, c, m)
        # a cleared corpus: refused, nothing written
        c.clear()
        c.append(m.rows)
        with pytest.raises(capi.StbError) as e:
            idx.remove(np.array([[base, base + 1]], np.uint64))
        assert e.value.status == S
        with pytest.raises(capi.StbError) as e:
            idx.update(np.array([base]), three[:1])
        assert e.value.status == S
        assert np.array_equal(bits(c.read()), bits(m.rows))
    finally:
        idx.close(); c.close()


# ---------------------------------------------------------------------------------- stream ordering ---
def test_device_searches_around_update_and_remove_see_old_then_new(ctx):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(709)
    centers = make_centers(rng, 64)
    rows = clustered(rng, centers, 30_000)
    Q = clustered(rng, centers, 2048)
    base = 3 << 32
    c, idx, m = build(ctx, rows, 64, row_base=base, prepare=False)
    try:
        dev = torch.device("cuda:0")
        q_dev = torch.from_numpy(Q).to(dev)
        loc = np.arange(64) * 400                                            # exact matches of the first queries
        for step in ("update", "remove"):
            before = idx.search_batch(Q, nprobe=8, top_k=10, rerank=256)
            b1 = idx.search(Q[0], nprobe=8, top_k=10, rerank=256)[0]
            outs = [(torch.zeros((len(Q), 10, 2), dtype=torch.float64, device=dev),
                     torch.zeros((len(Q), 2), dtype=torch.int32, device=dev)) for _ in range(2)]
            one = [(torch.zeros((10, 2), dtype=torch.float64, device=dev), torch.zeros(2, dtype=torch.int32, device=dev))
                   for _ in range(2)]
            torch.cuda.synchronize()
            idx.search_batch_dev(q_dev.data_ptr(), len(Q), 8, 10, 256, outs[0][0].data_ptr(), outs[0][1].data_ptr())
            idx.search_dev(q_dev[0].data_ptr(), 8, 10, 256, one[0][0].data_ptr(), one[0][1].data_ptr())
            if step == "update":
                idx.update(loc + base, Q[:64])
            else:
                idx.remove(np.array([[base, base + 3]], np.uint64))
            idx.search_batch_dev(q_dev.data_ptr(), len(Q), 8, 10, 256, outs[1][0].data_ptr(), outs[1][1].data_ptr())
            idx.search_dev(q_dev[0].data_ptr(), 8, 10, 256, one[1][0].data_ptr(), one[1][1].data_ptr())
            c.ctx.sync()
            after = idx.search_batch(Q, nprobe=8, top_k=10, rerank=256)
            a1 = idx.search(Q[0], nprobe=8, top_k=10, rerank=256)[0]
            assert not np.array_equal(before[0], after[0])
            for (h, st), (want, wn, ws) in zip(outs, (before, after)):
                raw = np.ascontiguousarray(h.cpu().numpy()).view(capi.HIT_DTYPE).reshape(len(Q), 10)
                sth = st.cpu().numpy()
                assert np.array_equal(raw, want) and np.array_equal(sth[:, 0], wn) and np.array_equal(sth[:, 1], ws)
            for (h, st), want in zip(one, (b1, a1)):
                raw = np.ascontiguousarray(h.cpu().numpy()).view(capi.HIT_DTYPE).reshape(10)
                assert np.array_equal(raw[: int(st.cpu().numpy()[0])], want)
        # after both: the first queries find their copies, moved down by the three removed rows
        assert np.all(after[0][1:64]["row"][:, 0] == base + loc[1:] - 3)
    finally:
        idx.close(); c.close()

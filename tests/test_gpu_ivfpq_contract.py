"""GPU: K5 IVF-PQ (csrc/ivfpq.cu) against an f64 reference of its own index.

K5 is self-specified (the reference has no IVF-PQ), so its reference lives here in numpy rather than
under oracle/.  Every check reads the index back with stb_debug_ivfpq_export and compares against that
same build: the build uses float atomics and an atomic scatter, so two builds differ.

The GPU computes in fp32; each check carries a bound derived from the kernel's arithmetic:
  U = 2^-24 (fp32 unit roundoff), gamma(n) = nU / (1 - nU) (a sum of n rounded terms in any order),
  rsqrtf is within 2 ulp, i.e. a relative 2^-22 (CUDA C Programming Guide, single-precision functions).
"""

import os
import sys

import numpy as np
import pytest

import oracle
from semtools_b200 import capi

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_ivfpq_batch import FUSED_CAP, search_on_route  # noqa: E402

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
RSQRT_REL = 2.0 ** -22
F64_SLOP = 2.0 ** -40          # relative: the f64 reference sums at most a few thousand terms


def gamma(n):
    return n * U / (1 - n * U)


# inv = rsqrtf(fl(sum of 256 squares)) against 1/||x||: the sum is within gamma(256) relatively, the
# square root halves that ((1 - g)^-1/2 - 1 bounds both sides), rsqrtf adds its own 2 ulp.
_G = gamma(256)
INV_REL = ((1 - _G) ** -0.5 - 1) + RSQRT_REL + ((1 - _G) ** -0.5 - 1) * RSQRT_REL


def make_centers(rng, n_centers):
    c = rng.standard_normal((n_centers, 256))
    return (c / np.linalg.norm(c, axis=1, keepdims=True)).astype(np.float32)


def clustered(rng, centers, n, spread=0.6):
    x = centers[rng.integers(0, len(centers), n)] + spread * rng.standard_normal((n, 256)).astype(np.float32) / 16.0
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    return np.ascontiguousarray(x, dtype=np.float32)


def forced_ref(rows):
    """K1's forced candidates: a non-finite component or ||x||^2 outside [1e-30, 1e30] (the test data
    keeps every finite row far from both ends, so f64 and the kernel's fp32 sum agree)."""
    with np.errstate(over="ignore", invalid="ignore"):
        ss = np.sum(rows.astype(np.float64) ** 2, axis=1)
    return ~((ss >= 1e-30) & (ss <= 1e30))


def edge_corpus(rng, n):
    """Random unit rows plus duplicates and ties, zero rows, NaN / +-inf components and rows scaled by
    1e-25 and 1e22, at positions spread over the whole corpus.  Returns (rows, special positions)."""
    x = clustered(rng, make_centers(rng, 8), n, spread=2.0)
    p = rng.permutation(n)[:16]
    x[p[1]] = x[p[0]]; x[p[2]] = x[p[0]]                    # three copies: equal distances, row order decides
    x[p[3]] = -x[p[0]]                                      # distance 2 (clamped) to a copy-query
    x[p[4]] = 0.0; x[p[5]] = 0.0                            # zero rows
    x[p[6], 3] = np.nan                                     # NaN distance -> 0 (simsimd rule)
    x[p[7], 100] = np.inf; x[p[8], 7] = -np.inf
    x[p[9]] = x[p[10]] * np.float32(1e-25)                  # fp32 ||x||^2 underflows
    x[p[11]] = x[p[12]] * np.float32(1e22)                  # fp32 ||x||^2 overflows
    x[p[13]] = x[p[0]] * np.float32(2.0)                    # same direction, different norm
    return np.ascontiguousarray(x), p


def edge_queries(rng, rows, p):
    q = rng.standard_normal(256).astype(np.float32)
    return {
        "random": q,
        "zero": np.zeros(256, np.float32),
        "scaled": (q * np.float32(1e-20)).astype(np.float32),
        "copy": rows[p[0]].copy(),
        "copy_of_tiny": rows[p[10]].copy(),
    }


def assert_exact(got, rows, q, top_k, base=0):
    want_rows, want_d = oracle.search_rows(rows, q, top_k)
    assert got["row"].tolist() == [int(r) + base for r in want_rows]
    assert np.array_equal(got["distance"].view(np.uint64), np.asarray(want_d, np.float64).view(np.uint64))


def build(ctx, rows, nlist, row_base=0, iters=4, extra=0):
    c = capi.Corpus(ctx, len(rows) + extra, row_base=row_base)
    c.append(rows)
    return c, capi.IvfPq(c, nlist=nlist, train_rows=len(rows), iters=iters)


# ----------------------------------------------------------------------------- index invariants ---
@pytest.mark.parametrize("nlist,n", [(1, 256), (3, 257), (257, 4099), (8192, 8192)])
def test_index_invariants(ctx, nlist, n):
    rng = np.random.default_rng(100 + nlist)
    rows = clustered(rng, make_centers(rng, max(nlist // 2, 2)), n)
    rows[7, 5] = np.nan; rows[n - 1] = 0.0; rows[n // 2] *= np.float32(1e22)
    c, idx = build(ctx, rows, nlist)
    E = idx.export()
    off, order, codes, forced = E["list_off"].astype(np.int64), E["order"], E["codes"], E["forced"]
    m = int(off[-1])
    # order (+ the forced side list) is a permutation of 0..n-1, list_off is consistent with it
    assert off[0] == 0 and np.all(np.diff(off) >= 0) and len(order) == m == n - len(forced)
    assert np.array_equal(np.sort(np.concatenate([order, forced])), np.arange(n))
    assert np.array_equal(forced, np.flatnonzero(forced_ref(rows)))
    assert len(forced) == 3
    # centroids: finite, unit norm (fl(v * rsqrtf(fl(||v||^2))): INV_REL and one rounding) or zero
    C = E["centroids"].astype(np.float64)
    assert np.all(np.isfinite(C)) and np.all(np.isfinite(E["codebooks"]))
    cn = np.linalg.norm(C, axis=1)
    tol = (1 + INV_REL) * (1 + U) - 1 + F64_SLOP
    assert np.all((cn == 0) | (np.abs(cn - 1) <= tol)), np.max(np.abs(cn - 1))
    lst = np.repeat(np.arange(nlist), np.diff(off))          # list of code i
    X = rows[order].astype(np.float64)
    # assignment: fp32 FMA chain of 256 terms -> |fl(x.c) - x.c| <= gamma(256) sum |x_t c_t|
    g = gamma(256) + F64_SLOP
    for a in range(0, m, 512):
        xb = X[a:a + 512]
        G, A = xb @ C.T, np.abs(xb) @ np.abs(C).T
        mine = np.arange(len(xb)), lst[a:a + 512]
        best_lo = np.max(G - g * A, axis=1)
        assert np.all(G[mine] + g * A[mine] >= best_lo)
    # codes: per sub-space argmin of ||r_s - e||^2, r = x * inv - c(list) in fp32.  Per component
    # |r~ - r| <= eps = |x^| K1 + (|x^| + |c|) U (product and difference roundings, INV_REL); the
    # fp32 distance of 8 terms adds gamma(10) relatively (difference rounding squared + FMA chain).
    cb = E["codebooks"].astype(np.float64)
    xh = X / np.linalg.norm(X, axis=1, keepdims=True)
    res = xh - C[lst]
    k1 = ((1 + INV_REL) * (1 + U) - 1) * (1 + U)
    eps = np.abs(xh) * k1 + (np.abs(xh) + np.abs(C[lst])) * U
    g10 = gamma(10) + F64_SLOP
    for s in range(32):
        for a in range(0, m, 1024):
            R = res[a:a + 1024, None, 8 * s:8 * s + 8]
            ep = eps[a:a + 1024, None, 8 * s:8 * s + 8]
            diff = np.abs(R - cb[s][None])
            D = np.sum(diff ** 2, axis=2)
            beta = np.sum(ep * (2 * diff + ep), axis=2) + g10 * np.sum((diff + ep) ** 2, axis=2)
            ch = codes[a:a + 1024, s].astype(np.int64)
            i = np.arange(len(ch))
            assert np.all(D[i, ch] - beta[i, ch] <= np.min(D + beta, axis=1)), (s, a)
    idx.close(); c.close()


# ---------------------------------------------------------------------- exhaustive search is exact ---
# nprobe = nlist and rerank >= n: every row is re-ranked, so the answer is the oracle's, bit for bit.
# v2 (fused) re-ranks every code when the probed lists hold <= 1024; v1 (multi-launch) runs for rerank > 1024,
# which the v1 cases ask for at every n.
@pytest.mark.parametrize("version,n", [("v2", 256), ("v2", 300), ("v2", 1000), ("v2", 1024),
                                       ("v1", 256), ("v1", 1000), ("v1", 1025), ("v1", 2000), ("v1", 4096)])
def test_exhaustive_search_is_exact(ctx, version, n):
    rng = np.random.default_rng(n + (7 if version == "v1" else 0))
    rows, p = edge_corpus(rng, n)
    base = 3 << 32
    c, idx = build(ctx, rows, nlist=3, row_base=base)
    n_forced = int(forced_ref(rows).sum())
    rerank_min = FUSED_CAP + 1 if version == "v1" else 0
    try:
        for name, q in edge_queries(rng, rows, p).items():
            for k in sorted({1, 10, 1024, n}):
                got, n_scan = search_on_route(ctx, idx, q, 3, k, max(n, k, rerank_min))
                assert n_scan == n - n_forced
                assert len(got) == min(k, n), (name, k)
                assert_exact(got, rows, q, k, base)
    finally:
        idx.close(); c.close()


# ----------------------------------------------------------------------- partial probe follows spec ---
def adc_reference(E, q):
    """f64 coarse scores, LUT and the bound on the GPU's error of each (see the module docstring):
    coarse~ = fl(fl(c.q) * rsqrtf(fl(q.q))): |err| <= A/|q| Kc, A = sum |c_t q_t|
    LUT~    = FMA chain of 8 fl(q_t * inv) e_t:  |err| <= B Kl, B = sum |q^_t e_t|."""
    qd = q.astype(np.float64)
    qn = np.linalg.norm(qd)
    qh = qd / qn
    C = E["centroids"].astype(np.float64)
    coarse = C @ qh
    kc = gamma(256) * (1 + INV_REL) * (1 + U) + (1 + INV_REL) * (1 + U) - 1 + F64_SLOP
    d_coarse = (np.abs(C) @ np.abs(qh)) * kc
    cb = E["codebooks"].astype(np.float64)                            # [32][256][8]
    qs = qh.reshape(32, 1, 8)
    lut = np.sum(cb * qs, axis=2)
    kl = (1 + INV_REL) * (1 + U) * (1 + gamma(8)) - 1 + F64_SLOP
    d_lut = np.sum(np.abs(cb) * np.abs(qs), axis=2) * kl
    return coarse, d_coarse, lut, d_lut


def probe_sets(lo, hi, nprobe):
    """Lists that are in the GPU's top-nprobe whatever its rounding (sure) and that may be (possible)."""
    above_sure = np.sum(hi[None, :] >= lo[:, None], axis=1) - 1      # others that may outrank j
    above_poss = np.sum(lo[None, :] > hi[:, None], axis=1)            # others that surely outrank j
    return np.flatnonzero(above_sure < nprobe), np.flatnonzero(above_poss < nprobe)


def deal_v2(total):
    """(CTA, warp) of code position v in ivf_adc_finish_kernel: 32-code chunk g -> CTA g % 32,
    warp (g / 32) % 16."""
    g = np.arange(total) // 32
    return g % 32, (g // 32) % 16


@pytest.mark.parametrize("rerank", [64, 512, 1024])
def test_partial_probe_follows_the_spec(ctx, rerank):
    rng = np.random.default_rng(rerank)
    n, nlist, nprobe = 60_000, 64, 8
    centers = make_centers(rng, 64)
    rows = clustered(rng, centers, n)
    queries = clustered(rng, centers, 12)
    rows[123] = queries[0] * np.float32(1e-25)            # forced: must come back as query 0's best hit
    rows[4567, 9] = np.nan                                  # forced: distance 0 by the simsimd rule
    c, idx = build(ctx, rows, nlist, iters=6)
    E = idx.export()
    off = E["list_off"].astype(np.int64)
    sizes = np.diff(off)
    list_of_row = np.full(n, -1)
    list_of_row[E["order"]] = np.repeat(np.arange(nlist), sizes)
    forced = set(E["forced"].tolist())
    assert forced == {123, 4567}
    r = min(rerank, 1024)
    checked = 0
    for qi, top_k in [(qi, k) for qi in range(len(queries)) for k in (10, r)]:
        q = queries[qi]
        got, n_scan = idx.search(q, nprobe=nprobe, top_k=top_k, rerank=rerank)
        hit_rows = got["row"].astype(np.int64)
        # every hit has the canonical distance and comes from a list that may be probed, or is forced
        assert np.array_equal(got["distance"].view(np.uint64), oracle.distances(rows[hit_rows], q).view(np.uint64))
        coarse, d_coarse, lut, d_lut = adc_reference(E, q)
        sure_l, poss_l = probe_sets(coarse - d_coarse, coarse + d_coarse, nprobe)
        assert all(int(h) in forced or list_of_row[h] in set(poss_l.tolist()) for h in hit_rows)
        assert sizes[sure_l].sum() <= n_scan <= sizes[poss_l].sum()
        if qi == 0:                                          # the NaN row (0) and the tiny copy (~0) lead
            assert set(hit_rows[:2].tolist()) == {123, 4567}
        if len(sure_l) != len(poss_l):
            continue                                         # probe set decided by rounding: bounds only
        assert n_scan == sizes[sure_l].sum()
        # GPU probe order (coarse desc, then list id): must be decided too, since it fixes the deal
        po = sure_l[np.lexsort((sure_l, -coarse[sure_l]))]
        if np.any(coarse[po][:-1] - d_coarse[po][:-1] <= coarse[po][1:] + d_coarse[po][1:]):
            continue
        checked += 1
        pos = np.concatenate([np.arange(off[l], off[l + 1]) for l in po])     # code position of v
        lv = np.repeat(po, sizes[po])
        cd = E["codes"][pos].astype(np.int64)
        A = coarse[lv] + np.sum(lut[np.arange(32)[None, :], cd], axis=1)
        dl = np.sum(d_lut[np.arange(32)[None, :], cd], axis=1)
        mag = np.abs(coarse[lv]) + d_coarse[lv] + np.sum(np.abs(lut[np.arange(32)[None, :], cd]), axis=1) + dl
        dA = d_coarse[lv] + dl + gamma(32) * mag            # 33 fp32 terms summed in order
        total = len(pos)
        lo, hi = A - dA, A + dA
        if total > r:
            H_r = np.sort(hi)[::-1][r - 1]
            L_r = np.sort(lo)[::-1][r - 1]
            sure = lo > H_r
            possible = hi >= L_r
        else:
            sure = possible = np.ones(total, bool)
        # the funnel's precondition: no warp and no CTA of the deal holds more than 64 possible winners
        cta, warp = deal_v2(total)
        assert np.bincount(cta[possible], minlength=32).max() <= 64
        assert np.bincount(cta[possible] * 16 + warp[possible], minlength=512).max() <= 64
        assert sure.sum() >= min(r, total) / 2                # the bound is not uselessly loose
        # no sure winner (nor forced row) beats the last hit without being returned
        cand = np.concatenate([E["order"][pos[sure]].astype(np.int64), np.asarray(sorted(forced), np.int64)])
        d = oracle.distances(rows[cand], q)
        last = (got["distance"][-1], int(hit_rows[-1]))
        returned = set(hit_rows.tolist())
        for row, dist in zip(cand.tolist(), d.tolist()):
            if len(got) < top_k or (dist, row) < last:
                assert row in returned, (qi, row, dist, last)
    assert checked >= len(queries), checked                # at least half of the 2 x 12 searches
    idx.close(); c.close()


# ---------------------------------------------------------------------------- edges and contract ---
@pytest.fixture(scope="module")
def edge_index(ctx):
    rng = np.random.default_rng(77)
    n = 4096
    rows, p = edge_corpus(rng, n)
    extra = np.ascontiguousarray(np.repeat(rows[p[0]][None], 8, axis=0))     # appended after the build
    c, idx = build(ctx, rows, nlist=2048, row_base=5 << 32, extra=len(extra))
    c.append(extra)
    yield rows, p, c, idx, rng
    idx.close(); c.close()


def test_nprobe_is_clamped(edge_index):
    rows, p, c, idx, rng = edge_index
    q = rows[p[0]]
    one, s1 = idx.search(q, nprobe=1, top_k=10, rerank=256)
    assert idx.search(q, nprobe=0, top_k=10, rerank=256)[1] == s1
    assert np.array_equal(idx.search(q, nprobe=0, top_k=10, rerank=256)[0], one)
    cap, s1024 = idx.search(q, nprobe=1024, top_k=10, rerank=256)
    for nprobe in (1025, 2048, 5000):                      # > 1024 and >= nlist (2048)
        got, s = idx.search(q, nprobe=nprobe, top_k=10, rerank=256)
        assert s == s1024 and np.array_equal(got, cap)
    assert s1 <= s1024 < len(rows)


def test_rerank_below_top_k_is_raised_to_top_k(edge_index):
    rows, p, c, idx, rng = edge_index
    q = rng.standard_normal(256).astype(np.float32)
    for k in (10, 300):
        a = idx.search(q, nprobe=64, top_k=k, rerank=1)
        b = idx.search(q, nprobe=64, top_k=k, rerank=k)
        assert a[1] == b[1] and np.array_equal(a[0], b[0])


def test_top_k_above_the_codes_scanned(edge_index):
    """nprobe = 1 and rerank >= the list: every code of the list and every forced row is re-ranked."""
    rows, p, c, idx, rng = edge_index
    E = idx.export()
    off = E["list_off"].astype(np.int64)
    forced = E["forced"].astype(np.int64)
    list_of_row = np.full(len(rows), -1)
    list_of_row[E["order"]] = np.repeat(np.arange(len(off) - 1), np.diff(off))
    for q in (rows[p[0]], rng.standard_normal(256).astype(np.float32)):
        got, n_scan = idx.search(q, nprobe=1, top_k=1000, rerank=1000)
        assert len(got) == n_scan + len(forced) < 1000
        local = got["row"].astype(np.int64) - (5 << 32)
        lists = set(list_of_row[local].tolist()) - {-1}
        assert len(lists) <= 1                              # one probed list, the rest are forced rows
        l = lists.pop() if lists else None
        mem = forced if l is None else np.concatenate([E["order"][off[l]:off[l + 1]].astype(np.int64), forced])
        assert n_scan == len(mem) - len(forced)
        mem = np.sort(mem)
        rr, dd = oracle.search_rows(rows[mem], q, len(mem))
        assert local.tolist() == [int(mem[i]) for i in rr]
        assert np.array_equal(got["distance"].view(np.uint64), np.asarray(dd, np.float64).view(np.uint64))


@pytest.mark.parametrize("top_k", [1025, 4096, 5000])
def test_host_top_k_above_1024(ctx, edge_index, top_k):
    """The multi-launch search takes top_k up to 4096 (exhaustive here: every list, rerank 4096);
    above that the call is refused."""
    rows, p, _, _, rng = edge_index
    c, idx = build(ctx, rows, nlist=16, row_base=5 << 32, extra=8)
    c.append(np.repeat(rows[p[0]][None], 8, axis=0))      # appended after the build: never returned
    q = rows[p[0]]
    try:
        if top_k > 4096:
            with pytest.raises(capi.StbError) as e:
                idx.search(q, nprobe=16, top_k=top_k, rerank=top_k)
            assert e.value.status == capi.STB_ERR_ARG
            return
        got, n_scan = idx.search(q, nprobe=16, top_k=top_k, rerank=4096)
        assert n_scan == len(rows) - int(forced_ref(rows).sum())
        assert_exact(got, rows, q, top_k, base=5 << 32)   # row_base >= 2^32
    finally:
        idx.close(); c.close()


def test_search_dev_matches_search_at_the_new_shapes(ctx, edge_index):
    torch = pytest.importorskip("torch")
    rows, p, c, idx, rng = edge_index
    qs = np.stack(list(edge_queries(rng, rows, p).values()))
    shapes = [(2048, 1024, 1024), (64, 10, 1024), (1, 1000, 1000), (7, 1, 0)]
    dev = torch.device("cuda:0")
    q_dev = torch.from_numpy(qs).to(dev)
    hits = torch.zeros((len(shapes), len(qs), 1024, 2), dtype=torch.float64, device=dev)
    st = torch.zeros((len(shapes), len(qs), 2), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    for si, (nprobe, k, rr) in enumerate(shapes):
        for i in range(len(qs)):
            idx.search_dev(q_dev[i].data_ptr(), nprobe, k, rr, hits[si, i].data_ptr(), st[si, i].data_ptr())
    ctx.sync()
    raw, sth = hits.cpu().numpy(), st.cpu().numpy()
    for si, (nprobe, k, rr) in enumerate(shapes):
        for i, q in enumerate(qs):
            want, n_scan = idx.search(q, nprobe=nprobe, top_k=k, rerank=rr)
            got = np.ascontiguousarray(raw[si, i, :k]).view(capi.HIT_DTYPE).reshape(-1)
            assert sth[si, i, 0] == len(want) and sth[si, i, 1] == n_scan
            assert np.array_equal(got[: len(want)], want)
            assert np.all(np.isinf(got["distance"][len(want):]))


def test_sharded_exhaustive_search_merges_to_the_oracle(ctx):
    rng = np.random.default_rng(91)
    n, k = 1600, 50
    rows, p = edge_corpus(rng, n)
    half = 700
    shards = [build(ctx, rows[:half], nlist=4, row_base=1 << 33), build(ctx, rows[half:], nlist=5, row_base=(1 << 33) + half)]
    try:
        for q in edge_queries(rng, rows, p).values():
            lists = np.zeros((2, k), dtype=capi.HIT_DTYPE)
            lists["distance"] = np.inf
            lists["row"] = np.iinfo(np.uint64).max
            for s, (c, idx) in enumerate(shards):
                got, _ = idx.search(q, nprobe=5, top_k=k, rerank=1024)
                lists[s, : len(got)] = got
            assert_exact(ctx.hits_merge(lists, k), rows, q, k, base=1 << 33)
    finally:
        for c, idx in shards:
            idx.close(); c.close()


def test_too_many_forced_rows_fail_the_build(ctx):
    rows = clustered(np.random.default_rng(3), make_centers(np.random.default_rng(4), 4), 2000)
    rows[:1025] = 0.0
    c = capi.Corpus(ctx, len(rows))
    c.append(rows)
    with pytest.raises(capi.StbError) as e:
        capi.IvfPq(c, nlist=4, train_rows=2000, iters=2)
    assert e.value.status == capi.STB_ERR_STATE
    rows[1024] = rows[1025]                                  # 1024 forced rows: the cap itself builds
    c2, idx = build(ctx, rows, nlist=4, iters=2)
    got, n_scan = idx.search(rows[1500], nprobe=4, top_k=10, rerank=1024)
    assert n_scan == 2000 - 1024
    assert_exact(got, rows, rows[1500], 10)
    idx.close(); c2.close(); c.close()

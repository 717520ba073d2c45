"""GPU: K5 IVF-PQ batched search (stb_ivfpq_search_batch / _dev, csrc/ivfpq.cu) against a prediction.

The batch's contract makes every answer predictable from its own index: with the coarse scores and the
LUT that stb_debug_ivfpq_batch_last returns, each ADC score is a plain fp32 sum in a fixed order, which
numpy reproduces bit for bit.  The prediction takes the `rerank` best keys (ADC score desc, code position
asc, as stb_make_key orders them), adds the forced rows and re-ranks them with the oracle.  The batch's
hits must equal that prediction bit for bit, whatever route the selection took.

The capacities of the selection are read from the source.  Each scan warp keeps IVFB_WARP_KEEP keys;
STB_IVFPQ_BATCH_KEEP lowers that at run time, which lets real data sit exactly at the capacity and one
past it.
"""

import os
import re

import numpy as np
import pytest

import oracle
from semtools_b200 import capi

pytestmark = pytest.mark.gpu

_SRC = os.path.join(os.path.dirname(__file__), "..", "semtools_b200", "csrc", "ivfpq.cu")


def _define(name):
    m = re.search(rf"#define {name} (\d+)", open(_SRC).read())
    assert m, name
    return int(m.group(1))


SCAN_CTAS = _define("IVFB_SCAN_CTAS")
SCAN_WARPS_PER_CTA = _define("IVFB_SCAN_THREADS") // 32
WARP_KEEP = _define("IVFB_WARP_KEEP")
MAX_NQ = _define("IVFB_MAX_NQ")
RERANK_CAP = _define("IVFB_RERANK_CAP")
FUSED_CAP = _define("ADC2_RERANK_CAP")      # stb_ivfpq_search: the fused search up to this rerank and top_k
INVALID = np.uint64(0xFFFFFFFFFFFFFFFF)
U64MAX = np.iinfo(np.uint64).max

U = 2.0 ** -24
RSQRT_REL = 2.0 ** -22
F64_SLOP = 2.0 ** -40


def gamma(n):
    return n * U / (1 - n * U)


_G = gamma(256)
INV_REL = ((1 - _G) ** -0.5 - 1) + RSQRT_REL + ((1 - _G) ** -0.5 - 1) * RSQRT_REL


# ----------------------------------------------------------------------------------- data helpers ---
def make_centers(rng, n_centers):
    c = rng.standard_normal((n_centers, 256))
    return (c / np.linalg.norm(c, axis=1, keepdims=True)).astype(np.float32)


def clustered(rng, centers, n, spread=0.6):
    x = centers[rng.integers(0, len(centers), n)] + spread * rng.standard_normal((n, 256)).astype(np.float32) / 16.0
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    return np.ascontiguousarray(x, dtype=np.float32)


def forced_ref(rows):
    with np.errstate(over="ignore", invalid="ignore"):
        ss = np.sum(rows.astype(np.float64) ** 2, axis=1)
    return ~((ss >= 1e-30) & (ss <= 1e30))


def edge_corpus(rng, n):
    """Unit rows plus duplicates, zero rows, NaN / +-inf components and rows scaled by 1e-25 and 1e22."""
    x = clustered(rng, make_centers(rng, 8), n, spread=2.0)
    p = rng.permutation(n)[:16]
    x[p[1]] = x[p[0]]; x[p[2]] = x[p[0]]
    x[p[3]] = -x[p[0]]
    x[p[4]] = 0.0; x[p[5]] = 0.0
    x[p[6], 3] = np.nan
    x[p[7], 100] = np.inf; x[p[8], 7] = -np.inf
    x[p[9]] = x[p[10]] * np.float32(1e-25)
    x[p[11]] = x[p[12]] * np.float32(1e22)
    x[p[13]] = x[p[0]] * np.float32(2.0)
    return np.ascontiguousarray(x), p


def edge_queries(rng, rows, p):
    q = rng.standard_normal(256).astype(np.float32)
    return [q, np.zeros(256, np.float32), (q * np.float32(1e-20)).astype(np.float32), rows[p[0]].copy(),
            rows[p[10]].copy()]


def bad_queries(rng):
    q = rng.standard_normal(256).astype(np.float32)
    nan = q.copy(); nan[5] = np.nan
    pinf = q.copy(); pinf[9] = np.inf
    ninf = q.copy(); ninf[200] = -np.inf
    return [np.zeros(256, np.float32), nan, pinf, ninf, (q * np.float32(1e-20)).astype(np.float32),
            (q * np.float32(1e20)).astype(np.float32)]


def search_on_route(ctx, idx, q, nprobe, top_k, rerank):
    """idx.search, checking from the context's launch count the route that rerank (in [top_k, 4096]) and top_k
    select: the fused search (2 launches) when both are <= FUSED_CAP, else the multi-launch search (more, as
    soon as a probed list holds a code)."""
    before = ctx.counters()["kernel_launches"]
    got, n_scan = idx.search(q, nprobe=nprobe, top_k=top_k, rerank=rerank)
    launches = ctx.counters()["kernel_launches"] - before
    if rerank <= FUSED_CAP and top_k <= FUSED_CAP:
        assert launches == 2, (rerank, top_k, launches)
    else:
        assert n_scan > 0 and launches > 2, (rerank, top_k, n_scan, launches)
    return got, n_scan


def build(ctx, rows, nlist, row_base=0, iters=4, extra=0):
    c = capi.Corpus(ctx, len(rows) + extra, row_base=row_base)
    c.append(rows)
    return c, capi.IvfPq(c, nlist=nlist, train_rows=len(rows), iters=iters)


# ------------------------------------------------------------------------------------- prediction ---
def np_keys(s, ids):
    """stb_make_key: (~f2ord(score)) << 32 | id, ascending = (score desc, id asc)."""
    b = np.ascontiguousarray(s, dtype=np.float32).view(np.uint32).astype(np.uint64)
    ordv = np.where(b & 0x80000000, (~b) & 0xFFFFFFFF, b | 0x80000000)
    return (((~ordv) & 0xFFFFFFFF) << np.uint64(32)) | np.asarray(ids).astype(np.uint64)


def adc_keys(E, info):
    """(code positions in probe order, their keys; INVALID for a NaN or -inf score)."""
    off = E["list_off"].astype(np.int64)
    probe = info["probe"].astype(np.int64)
    sizes = off[probe + 1] - off[probe]
    pos = np.concatenate([np.arange(off[l], off[l + 1]) for l in probe]) if len(probe) else np.zeros(0, np.int64)
    s = info["coarse"][np.repeat(probe, sizes)].astype(np.float32)
    cd = E["codes"][pos].astype(np.int64)
    for t in range(32):
        s = s + info["lut"][t][cd[:, t]]                    # fp32 + fp32, in sub-space order
    assert s.dtype == np.float32
    keys = np.where(s > -np.inf, np_keys(s, pos), INVALID)
    return pos, keys


def winners(keys, r):
    k = np.sort(keys[keys != INVALID])
    return k[:r]


def predict(E, info, rows, q, top_k, base):
    """(rows with base, distances, codes scanned) the batch must return for this query."""
    pos, keys = adc_keys(E, info)
    w = winners(keys, info["rerank"])
    cand = E["order"][(w & np.uint64(0xFFFFFFFF)).astype(np.int64)].astype(np.int64)
    mem = np.sort(np.concatenate([cand, E["forced"].astype(np.int64)]))
    if len(mem) == 0:
        return [], np.zeros(0), len(pos)
    rr, dd = oracle.search_rows(rows[mem], q, min(top_k, len(mem)))
    return [int(mem[i]) + base for i in rr], np.asarray(dd, np.float64), len(pos)


def assert_hits(got_row, n, want_rows, want_d):
    assert int(n) == len(want_rows)
    assert got_row["row"][:n].tolist() == want_rows
    assert np.array_equal(got_row["distance"][:n].view(np.uint64), want_d.view(np.uint64))
    assert np.all(np.isinf(got_row["distance"][n:])) and np.all(got_row["row"][n:] == U64MAX)


def scan_routes(keys, r, keep):
    """Per (warp of the deal, kept keys) -> is the fast route exact-by-itself (no dropped key beats the
    r-th best kept key)?  Returns (fast, max winners any warp holds)."""
    v = np.arange(len(keys))
    g = v // 32
    warp = (g % SCAN_CTAS) * SCAN_WARPS_PER_CTA + (g // SCAN_CTAS) % SCAN_WARPS_PER_CTA
    kept, drops = [], []
    for w in range(SCAN_CTAS * SCAN_WARPS_PER_CTA):
        kw = np.sort(keys[(warp == w) & (keys != INVALID)])
        kept.append(kw[:keep])
        if len(kw) > keep:
            drops.append(kw[keep])
    allk = np.sort(np.concatenate(kept)) if kept else np.zeros(0, np.uint64)
    T = allk[r - 1] if len(allk) >= r else INVALID
    fast = all(d > T for d in drops)
    win = set(winners(keys, r).tolist())
    most = max(int(np.sum(np.isin(keys[warp == w], list(win)))) for w in range(SCAN_CTAS * SCAN_WARPS_PER_CTA)) if win else 0
    return fast, most


def adc_reference(E, q):
    """f64 coarse scores and LUT with the bound on the GPU's error of each (restated from
    test_gpu_ivfpq_contract.py: coarse |err| <= A/|q| Kc, LUT |err| <= B Kl)."""
    qd = q.astype(np.float64)
    qh = qd / np.linalg.norm(qd)
    C = E["centroids"].astype(np.float64)
    coarse = C @ qh
    kc = gamma(256) * (1 + INV_REL) * (1 + U) + (1 + INV_REL) * (1 + U) - 1 + F64_SLOP
    d_coarse = (np.abs(C) @ np.abs(qh)) * kc
    cb = E["codebooks"].astype(np.float64)
    qs = qh.reshape(32, 1, 8)
    lut = np.sum(cb * qs, axis=2)
    kl = (1 + INV_REL) * (1 + U) * (1 + gamma(8)) - 1 + F64_SLOP
    d_lut = np.sum(np.abs(cb) * np.abs(qs), axis=2) * kl
    return coarse, d_coarse, lut, d_lut


def check_batch(idx, E, rows, Q, got, n, scanned, top_k, base=0):
    for i, q in enumerate(Q):
        info = idx.batch_last(i)
        want_rows, want_d, n_scan = predict(E, info, rows, q, top_k, base)
        assert int(scanned[i]) == n_scan, i
        assert_hits(got[i], n[i], want_rows, want_d)


# ------------------------------------------------------------------------- exhaustive search is exact ---
@pytest.mark.parametrize("n", [256, 700, 1031])
def test_exhaustive_batch_is_exact(ctx, n):
    rng = np.random.default_rng(500 + n)
    rows, p = edge_corpus(rng, n)
    base = 3 << 32
    c, idx = build(ctx, rows, nlist=3, row_base=base)
    n_forced = int(forced_ref(rows).sum())
    assert n - n_forced <= RERANK_CAP
    Q = np.stack(edge_queries(rng, rows, p) + [rng.standard_normal(256).astype(np.float32) for _ in range(3)]
                 + [rows[p[13]], rows[p[3]]])
    try:
        for k in (1, 10, 1024):
            got, cnt, scanned = idx.search_batch(Q, nprobe=3, top_k=k, rerank=RERANK_CAP)
            for i, q in enumerate(Q):
                want_rows, want_d = oracle.search_rows(rows, q, k)
                assert int(scanned[i]) == n - n_forced
                assert_hits(got[i], cnt[i], [int(r) + base for r in want_rows], np.asarray(want_d, np.float64))
    finally:
        idx.close(); c.close()


# ---------------------------------------------------------------------- clustered index (partial probe) ---
@pytest.fixture(scope="module")
def clustered_index(ctx):
    rng = np.random.default_rng(4242)
    n, nlist = 60_000, 64
    centers = make_centers(rng, 64)
    rows = clustered(rng, centers, n)
    Q = np.concatenate([clustered(rng, centers, 24), rng.standard_normal((2, 256)).astype(np.float32)])
    rows[123] = Q[0] * np.float32(1e-25)                    # forced rows
    rows[4567, 9] = np.nan
    base = 7 << 32
    c, idx = build(ctx, rows, nlist, row_base=base, iters=6)
    E = idx.export()
    yield rows, Q, c, idx, E, base
    idx.close(); c.close()


@pytest.mark.parametrize("rerank", [10, 64, 512, 1024])
def test_predicted_bits_at_partial_probe(clustered_index, rerank):
    rows, Q, c, idx, E, base = clustered_index
    nprobe, top_k = 8, 10
    got, n, scanned = idx.search_batch(Q, nprobe=nprobe, top_k=top_k, rerank=rerank)
    nlist = len(E["list_off"]) - 1
    for i, q in enumerate(Q):
        info = idx.batch_last(i)
        assert (info["nq"], info["nprobe"], info["top_k"], info["rerank"]) == (len(Q), nprobe, top_k, rerank)
        # the probe list: the nprobe best of the hook's coarse scores by (score desc, list id asc)
        order = np.argsort(np_keys(info["coarse"], np.arange(nlist)), kind="stable")
        assert info["probe"].tolist() == order[:nprobe].tolist()
        coarse, d_coarse, lut, d_lut = adc_reference(E, q)
        assert np.all(np.abs(info["coarse"] - coarse) <= d_coarse)
        assert np.all(np.abs(info["lut"] - lut) <= d_lut)
        want_rows, want_d, n_scan = predict(E, info, rows, q, top_k, base)
        assert int(scanned[i]) == n_scan
        assert_hits(got[i], n[i], want_rows, want_d)


def v2_precondition(keys, r):
    """v2's funnel (ivf_adc_finish_kernel) returns the r best ADC keys when no warp and no CTA of its deal
    (32-code chunk g -> CTA g % 32, warp (g / 32) % 16) holds more than 64 of them, and the r-th and
    (r+1)-th scores differ (it compares scores only)."""
    valid = keys != INVALID
    srt = np.sort(keys[valid])
    if len(srt) > r and (srt[r - 1] >> np.uint64(32)) == (srt[r] >> np.uint64(32)):
        return False
    win = np.isin(keys, srt[:r])
    g = np.arange(len(keys)) // 32
    cta, warp = g % 32, (g // 32) % 16
    return (np.bincount(cta[win], minlength=32).max(initial=0) <= 64
            and np.bincount(cta[win] * 16 + warp[win], minlength=512).max(initial=0) <= 64)


@pytest.mark.parametrize("rerank", [64, 512, 1024])
def test_agrees_with_the_single_path_where_v2_is_exact(clustered_index, rerank):
    rows, Q, c, idx, E, base = clustered_index
    Qb = np.concatenate([Q, np.stack(bad_queries(np.random.default_rng(rerank)))])
    got, n, scanned = idx.search_batch(Qb, nprobe=8, top_k=10, rerank=rerank)
    agreed = 0
    for i, q in enumerate(Qb):
        info = idx.batch_last(i)
        _, keys = adc_keys(E, info)
        want_rows, want_d, n_scan = predict(E, info, rows, q, 10, base)
        assert_hits(got[i], n[i], want_rows, want_d)
        if v2_precondition(keys, rerank):
            one, s1 = idx.search(q, nprobe=8, top_k=10, rerank=rerank)
            assert s1 == int(scanned[i])
            assert np.array_equal(got[i][: n[i]], one), i
            agreed += 1
    assert agreed >= len(Q)


def test_bad_queries_probe_and_answer_as_the_single_path(clustered_index):
    rows, Q, c, idx, E, base = clustered_index
    B = np.stack(bad_queries(np.random.default_rng(9)))
    got, n, scanned = idx.search_batch(B, nprobe=8, top_k=10, rerank=256)
    for i, q in enumerate(B):
        info = idx.batch_last(i)
        one, s1 = idx.search(q, nprobe=8, top_k=10, rerank=256)
        assert s1 == int(scanned[i]) and np.array_equal(got[i][: n[i]], one), i
        want_rows, want_d, _ = predict(E, info, rows, q, 10, base)
        assert_hits(got[i], n[i], want_rows, want_d)
    zero = idx.batch_last(0)                                   # every coarse score is 0: lists 0..7 in id order
    assert np.all(zero["coarse"] == 0) and zero["probe"].tolist() == list(range(8))


# ------------------------------------------------------------------------------- ties and capacities ---
def test_rerank_cut_inside_a_block_of_identical_codes(ctx):
    rng = np.random.default_rng(31)
    centers = make_centers(rng, 16)
    rows = clustered(rng, centers, 24_000)
    dup = rng.permutation(len(rows))[:3000]
    rows[dup] = rows[dup[0]]                                  # 3000 identical rows, spread over the corpus
    c, idx = build(ctx, rows, nlist=16, row_base=1 << 32)
    E = idx.export()
    try:
        q = rows[dup[0]] + np.float32(0.01) * rng.standard_normal(256).astype(np.float32)
        Q = np.stack([q, rows[dup[0]]])
        for rerank, k in [(512, 10), (512, 512), (1024, 1024)]:
            got, n, scanned = idx.search_batch(Q, nprobe=4, top_k=k, rerank=rerank)
            for i in range(len(Q)):
                info = idx.batch_last(i)
                pos, keys = adc_keys(E, info)
                w = winners(keys, rerank)
                # the cut falls inside the block: equal scores, the lower code positions win
                in_block = np.isin(E["order"][(w & np.uint64(0xFFFFFFFF)).astype(np.int64)], dup)
                assert in_block.sum() == rerank
            check_batch(idx, E, rows, Q, got, n, scanned, k, base=1 << 32)
    finally:
        idx.close(); c.close()


@pytest.mark.parametrize("rerank", [64, 1024])
def test_warp_capacity_at_its_limit_and_one_past(clustered_index, monkeypatch, rerank):
    """Each scan warp keeps `keep` keys.  At keep = the most winners any warp holds, the kept keys hold
    every winner (fast route); one below, some query's winners overflow a warp and that query takes the
    exact slow route.  Both must match the prediction, as must keep = 1 (every query slow)."""
    rows, Q, c, idx, E, base = clustered_index
    got, n, scanned = idx.search_batch(Q, nprobe=8, top_k=10, rerank=rerank)
    keys_of = [adc_keys(E, idx.batch_last(i))[1] for i in range(len(Q))]
    most = max(scan_routes(k, rerank, WARP_KEEP)[1] for k in keys_of)
    assert 1 < most <= WARP_KEEP
    for keep, any_slow in [(most, False), (most - 1, True), (1, True)]:
        routes = [scan_routes(k, rerank, keep)[0] for k in keys_of]
        assert (not all(routes)) == any_slow, keep
        monkeypatch.setenv("STB_IVFPQ_BATCH_KEEP", str(keep))
        try:
            got, n, scanned = idx.search_batch(Q, nprobe=8, top_k=10, rerank=rerank)
        finally:
            monkeypatch.delenv("STB_IVFPQ_BATCH_KEEP")
        check_batch(idx, E, rows, Q, got, n, scanned, 10, base)


# ------------------------------------------------------------------------------------- independence ---
def test_a_query_answers_the_same_alone_in_4096_and_permuted(clustered_index):
    rows, Q, c, idx, E, base = clustered_index
    rng = np.random.default_rng(77)
    big = np.concatenate([Q, clustered(rng, make_centers(rng, 64), 4096 - len(Q) - 6), np.stack(bad_queries(rng))])
    assert len(big) == 4096
    got, n, sc = idx.search_batch(big, nprobe=8, top_k=10, rerank=512)
    perm = rng.permutation(len(big))
    gp, np_, sp = idx.search_batch(big[perm], nprobe=8, top_k=10, rerank=512)
    assert np.array_equal(gp, got[perm]) and np.array_equal(np_, n[perm]) and np.array_equal(sp, sc[perm])
    for i in list(range(len(Q))) + [4000, 4090, 4095]:
        g1, n1, s1 = idx.search_batch(big[i:i + 1], nprobe=8, top_k=10, rerank=512)
        assert np.array_equal(g1[0], got[i]) and n1[0] == n[i] and s1[0] == sc[i]
    # bad queries do not change their neighbours' answers
    mixed = np.insert(Q, [1, 5, 9, 13, 17, 21], np.stack(bad_queries(rng)), axis=0)
    keep = np.ones(len(mixed), bool); keep[[1, 6, 11, 16, 21, 26]] = False
    gm, nm, sm = idx.search_batch(mixed, nprobe=8, top_k=10, rerank=512)
    assert np.array_equal(gm[keep], got[: len(Q)]) and np.array_equal(nm[keep], n[: len(Q)])


def test_host_chunks_equal_the_device_form(clustered_index):
    torch = pytest.importorskip("torch")
    rows, Q, c, idx, E, base = clustered_index
    rng = np.random.default_rng(5)
    nq = MAX_NQ + 37                                            # two chunks
    big = clustered(rng, make_centers(rng, 64), nq)
    got, n, sc = idx.search_batch(big, nprobe=8, top_k=16, rerank=128)
    dev = torch.device("cuda:0")
    q_dev = torch.from_numpy(big).to(dev)
    hits = torch.zeros((nq, 16, 2), dtype=torch.float64, device=dev)
    st = torch.zeros((nq, 2), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    with pytest.raises(capi.StbError) as e:
        idx.search_batch_dev(q_dev.data_ptr(), nq, 8, 16, 128, hits.data_ptr(), st.data_ptr())
    assert e.value.status == capi.STB_ERR_ARG
    for a, b in [(0, MAX_NQ), (MAX_NQ, nq)]:
        idx.search_batch_dev(q_dev[a].data_ptr(), b - a, 8, 16, 128, hits[a].data_ptr(), st[a].data_ptr())
    c.ctx.sync()
    raw = np.ascontiguousarray(hits.cpu().numpy()).view(capi.HIT_DTYPE).reshape(nq, 16)
    sth = st.cpu().numpy()
    assert np.array_equal(raw, got) and np.array_equal(sth[:, 0], n) and np.array_equal(sth[:, 1], sc)


# ------------------------------------------------------------------------------------------- edges ---
@pytest.fixture(scope="module")
def edge_index(ctx):
    rng = np.random.default_rng(78)
    n = 4096
    rows, p = edge_corpus(rng, n)
    extra = np.ascontiguousarray(np.repeat(rows[p[0]][None], 8, axis=0))     # appended after the build
    c, idx = build(ctx, rows, nlist=2048, row_base=5 << 32, extra=len(extra))
    c.append(extra)
    yield rows, p, c, idx, idx.export(), rng
    idx.close(); c.close()


def test_hook_before_any_batch_and_argument_errors(ctx, edge_index):
    rows, p, c0, _, _, rng = edge_index
    c, idx = build(ctx, rows[:600], nlist=4)
    try:
        with pytest.raises(capi.StbError) as e:
            idx.batch_last(0)
        assert e.value.status == capi.STB_ERR_STATE
        got, n, sc = idx.search_batch(np.zeros((0, 256), np.float32))     # nq = 0: no-op
        assert got.shape == (0, 10) and len(n) == 0
        idx.search_batch_dev(0, 0, 8, 10, 64, 0, 0)
        with pytest.raises(capi.StbError) as e:
            idx.batch_last(0)
        assert e.value.status == capi.STB_ERR_STATE
        Q = np.stack(edge_queries(rng, rows, p))
        got, n, sc = idx.search_batch(Q, nprobe=4, top_k=0)                 # top_k 0: every count 0
        assert np.all(n == 0) and np.all(sc == 0)
        for k in (1025, 5000):
            with pytest.raises(capi.StbError) as e:
                idx.search_batch(Q, top_k=k)
            assert e.value.status == capi.STB_ERR_ARG
        idx.search_batch(Q[:1], nprobe=4, top_k=3, rerank=3)               # nq = 1
        with pytest.raises(capi.StbError) as e:
            idx.batch_last(1)
        assert e.value.status == capi.STB_ERR_ARG
        assert idx.batch_last(0)["nq"] == 1
    finally:
        idx.close(); c.close()


def test_nprobe_and_rerank_are_clamped(edge_index):
    rows, p, c, idx, E, rng = edge_index
    Q = np.stack(edge_queries(rng, rows, p))
    ref = {}
    for nprobe, rerank, want_np, want_rr in [(0, 5, 1, 10), (1, 10, 1, 10), (1024, 2000, 1024, 1024),
                                              (1025, 1024, 1024, 1024), (5000, 1 << 30, 1024, 1024)]:
        got, n, sc = idx.search_batch(Q, nprobe=nprobe, top_k=10, rerank=rerank)
        info = idx.batch_last(0)
        assert (info["nprobe"], info["rerank"]) == (want_np, want_rr)
        key = (want_np, want_rr)
        if key in ref:
            assert np.array_equal(ref[key][0], got) and np.array_equal(ref[key][1], sc)
        ref[key] = (got, sc)
        check_batch(idx, E, rows, Q, got, n, sc, 10, base=5 << 32)


def test_padding_empty_lists_and_appended_rows(ctx):
    """8 distinct rows, 40 copies each, 64 lists: most lists are empty (equal centroids assign to the lowest
    list id).  top_k above the codes scanned pads with (+inf, UINT64_MAX); rows appended after the build
    are never returned."""
    rng = np.random.default_rng(19)
    distinct = clustered(rng, make_centers(rng, 8), 8, spread=2.0)
    rows = np.ascontiguousarray(np.repeat(distinct, 40, axis=0))
    c, idx = build(ctx, rows, nlist=64, row_base=9 << 32, extra=16)
    c.append(np.ascontiguousarray(np.repeat(distinct[:2], 8, axis=0)))
    try:
        E = idx.export()
        sizes = np.diff(E["list_off"].astype(np.int64))
        assert np.sum(sizes == 0) > 0
        Q = np.concatenate([distinct, rng.standard_normal((8, 256)).astype(np.float32)])
        saw_empty = False
        for nprobe in (1, 3, 16):
            got, n, sc = idx.search_batch(Q, nprobe=nprobe, top_k=1000, rerank=1000)
            assert np.all(n < 1000) and np.all(n == sc)
            assert np.all(got["row"][got["row"] != U64MAX] < (9 << 32) + len(rows))
            check_batch(idx, E, rows, Q, got, n, sc, 1000, base=9 << 32)
            for i in range(len(Q)):
                pl = idx.batch_last(i)["probe"]
                assert sc[i] == sizes[pl].sum()
                saw_empty |= bool(np.any(sizes[pl] == 0))
        assert saw_empty
    finally:
        idx.close(); c.close()


def test_back_to_back_device_calls_with_a_single_query_between(edge_index):
    torch = pytest.importorskip("torch")
    rows, p, c, idx, E, rng = edge_index
    Q = np.stack(edge_queries(rng, rows, p) + [rng.standard_normal(256).astype(np.float32) for _ in range(40)])
    dev = torch.device("cuda:0")
    q_dev = torch.from_numpy(Q).to(dev)
    shapes = [(len(Q), 64, 10, 256), (17, 1024, 100, 1024)]
    outs = [(torch.zeros((nq, k, 2), dtype=torch.float64, device=dev), torch.zeros((nq, 2), dtype=torch.int32, device=dev))
            for nq, _, k, _ in shapes]
    h1 = torch.zeros((1024, 2), dtype=torch.float64, device=dev)
    s1 = torch.zeros(2, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    (nq0, np0, k0, r0), (nq1, np1, k1, r1) = shapes
    idx.search_batch_dev(q_dev.data_ptr(), nq0, np0, k0, r0, outs[0][0].data_ptr(), outs[0][1].data_ptr())
    idx.search_dev(q_dev[3].data_ptr(), 64, 1024, 1024, h1.data_ptr(), s1.data_ptr())
    idx.search_batch_dev(q_dev[5].data_ptr(), nq1, np1, k1, r1, outs[1][0].data_ptr(), outs[1][1].data_ptr())
    c.ctx.sync()
    for (nq, nprobe, k, rr), (h, st), q0 in zip(shapes, outs, (0, 5)):
        want, wn, ws = idx.search_batch(Q[q0:q0 + nq], nprobe=nprobe, top_k=k, rerank=rr)
        raw = np.ascontiguousarray(h.cpu().numpy()).view(capi.HIT_DTYPE).reshape(nq, k)
        sth = st.cpu().numpy()
        assert np.array_equal(raw, want) and np.array_equal(sth[:, 0], wn) and np.array_equal(sth[:, 1], ws)
    one, ns = idx.search(Q[3], nprobe=64, top_k=1024, rerank=1024)
    raw1 = np.ascontiguousarray(h1.cpu().numpy()).view(capi.HIT_DTYPE).reshape(-1)
    assert int(s1[0]) == len(one) and int(s1[1]) == ns and np.array_equal(raw1[: len(one)], one)

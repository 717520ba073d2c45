"""GPU: K2 (csrc/batch_scan.cu) stage by stage, through the device entry point.

stb_search_batch re-runs every unproven query through K1, so a K2 that proves too little looks the same
there as a correct one.  These tests call stb_search_batch_dev instead and read the last call back with
stb_debug_batch_last (route, sampled tiles, per-query thresholds, per-(query, CTA) emission counts).

Pipeline v2 is checked against its own approximate scores: stb_debug_batch_gemm runs the same shadow
build and the same wgmma accumulation on host inputs, so its score a[q][r] is bit-identical to the one the
search's epilogues see.  From that matrix the tests predict, exactly, the threshold of every query, the
count of every emission segment and which queries the finish kernel proves.  Proven hits must equal
oracle.search_rows bit for bit.

The host routing rule (api.cu, stb_search_batch_dev) and the capacities are restated or read from the
sources below, so a change to either shows up here.
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
CSRC = os.path.join(ROOT, "semtools_b200", "csrc")


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _define(text, name):
    return int(re.search(rf"#define\s+{name}\s+(\d+)", text).group(1))


_BATCH = _src("batch_scan.cu")
SEG_CAP = int(re.search(r"constexpr\s+uint32_t\s+kSegCap\s*=\s*(\d+)", _src("api.cu")).group(1))
F2_KEYS = _define(_BATCH, "STB_F2_KEYS")
F2_RESCORE = _define(_BATCH, "STB_F2_RESCORE")
KSEL = _define(_BATCH, "STB_BATCH_KSEL")
MAX_SAMPLE = _define(_BATCH, "STB_V2_MAX_SAMPLE")
MAX_K = _define(_BATCH, "STB_V2_MAX_K")
TILE = 256
NO_ROW = np.uint64(0xFFFFFFFFFFFFFFFF)


def test_constants_are_the_documented_ones():
    assert (SEG_CAP, F2_KEYS, F2_RESCORE, KSEL, MAX_SAMPLE, MAX_K) == (64, 4096, 1024, 32, 608, 64)


@pytest.fixture(scope="module")
def sm_count():
    torch = pytest.importorskip("torch")
    return torch.cuda.get_device_properties(0).multi_processor_count


def route_rule(n, k, sm):
    """api.cu stb_search_batch_dev: which pipeline runs, and v2's sampling and emission grid."""
    f16, _ = capi.batch_params()
    n_full = n // TILE
    n_sample = min(n_full, min(4 * sm, MAX_SAMPLE))
    margin_factor = 2 if f16 else 4

    def expected_emitted(ns):
        return k * margin_factor * (-(-n_full // ns)) if ns else 0
    if expected_emitted(n_sample) > 2048:
        n_sample = min(min(n_full, 8192), (n_full // 64 + sm - 1) // sm * sm)
    v2_fits = n_sample >= k and expected_emitted(n_sample) <= 2048
    if k <= MAX_K and v2_fits:
        n_tiles = -(-n // TILE)
        return {"route": 2, "n_sample": n_sample, "stride": n_full // n_sample, "n_seg": min(n_tiles, sm),
                "seg_cap": SEG_CAP}
    return {"route": 1, "n_sample": 0, "stride": 0, "n_seg": 0, "seg_cap": 0}


def unnormalisable(queries):
    """Queries the shadow build cannot normalise in fp32 (test data keeps clear of the fp32 edges)."""
    q = queries.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        ss = np.sum(q * q, axis=1)
    finite = np.isfinite(q).all(axis=1)
    return ~finite | ((ss > 0) & ((ss < 1e-30) | (ss > 1e30)))


def debug_scores(ctx, queries, rows):
    """a[q][r]: the approximate score matrix of K2's shadow and wgmma GEMM (stb_debug_batch_gemm)."""
    queries = np.ascontiguousarray(queries, dtype=np.float32)
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    nq, n = len(queries), len(rows)
    full = np.zeros((-(-nq // 128) * 128, -(-n // TILE) * TILE), dtype=np.float32)
    vp = C.c_void_p
    capi._check(capi.lib().stb_debug_batch_gemm(ctx._h, queries.ctypes.data_as(vp), nq, rows.ctypes.data_as(vp), n,
                                                full.ctypes.data_as(vp), None))
    return full[:nq, :n]


def run_dev(ctx, corpus, queries, k):
    """stb_search_batch_dev -> (hits [nq][k] HIT_DTYPE, status [nq][2] u32, stb_debug_batch_last)."""
    torch = pytest.importorskip("torch")
    nq = len(queries)
    dev = torch.device("cuda:0")
    q_dev = torch.from_numpy(np.ascontiguousarray(queries, dtype=np.float32)).to(dev)
    hits = torch.zeros((nq, k, 2), dtype=torch.float64, device=dev)
    status = torch.full((nq, 2), 7, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    corpus.search_batch_dev(q_dev.data_ptr(), nq, k, hits.data_ptr(), status.data_ptr())
    ctx.sync()
    got = np.ascontiguousarray(hits.cpu().numpy()).view(capi.HIT_DTYPE).reshape(nq, k)
    st = status.cpu().numpy().view(np.uint32)
    return got, st, ctx.batch_last()


def check_query(hits_q, status_q, rows, q, k, row_base=0, where=""):
    """A proven query: the oracle's hits bit for bit, the count in status, the padded tail."""
    r, d = oracle.search_rows(rows, q, top_k=k)
    n_out = int(status_q[0])
    assert n_out == len(r), where
    assert hits_q["row"][:n_out].tolist() == [int(x) + row_base for x in r], where
    assert np.array_equal(hits_q["distance"][:n_out], d), where
    assert np.all(hits_q["distance"][n_out:] == np.inf) and np.all(hits_q["row"][n_out:] == NO_ROW), where


def sample_ids(nq, rng, extra=24):
    """Query tile edges plus a random sample: enough to catch a per-tile or per-query defect."""
    ids = {0, nq - 1} | {i for i in (1, 126, 127, 128, 129, 255, 256, 257) if i < nq}
    ids |= set(rng.choice(nq, min(nq, extra), replace=False).tolist())
    return sorted(ids)


def predict_v2(A, k, info, bad):
    """From the approximate scores A [nq][n]: thr [nq], counts [nq][n_seg] and the proof flag the kernels
    must produce (threshold kernel, emitting epilogue and finish2 of batch_scan.cu)."""
    _, eps = capi.batch_params()
    nq, n = A.shape
    n_full = n // TILE
    ns, stride, n_seg = info["n_sample"], info["stride"], info["n_seg"]
    two_eps = np.float32(2.0) * np.float32(eps)
    tiles = A[:, : n_full * TILE].reshape(nq, n_full, TILE)[:, np.arange(ns) * stride]
    s_k = np.sort(tiles.max(axis=2), axis=1)[:, ns - k]
    thr = (s_k.astype(np.float32) - two_eps).astype(np.float32)
    seg_of = (np.arange(n) // TILE) % n_seg
    cnt = np.zeros((nq, n_seg), dtype=np.int64)
    proven = np.zeros(nq, dtype=bool)
    m2s = np.zeros(nq, dtype=np.int64)
    for q in range(nq):
        emit = A[q] >= thr[q]
        cnt[q] = np.bincount(seg_of[emit], minlength=n_seg)
        total = int(cnt[q].sum())
        sc = A[q][emit]
        m2 = total                                                # narrowed keys (the finish sees them only
        if total >= k:                                            # when no capacity before it overflowed)
            cut = np.float32(np.sort(sc)[total - k]) - two_eps
            m2 = int(np.count_nonzero(sc >= cut))
        m2s[q] = m2
        over = (cnt[q] > SEG_CAP).any() or total > F2_KEYS
        proven[q] = not over and m2 <= F2_RESCORE and not bad[q]
    return thr, cnt, proven, m2s


def check_v2_call(ctx, rows, queries, k, got, st, info, row_base=0, rng=None, require_all_proven=False):
    """Threshold bits, emission counts and proof flags against the prediction; proven hits against the oracle."""
    bad = unnormalisable(queries)
    A = debug_scores(ctx, queries, rows)
    thr, cnt, proven, _ = predict_v2(A, k, info, bad)
    # a NaN or infinite component survives the zero scale of an unnormalisable query (NaN * 0), so its
    # scores are NaN and its threshold and counts follow NaN rules the model does not restate
    live = np.isfinite(A).all(axis=1)
    assert live[~bad].all()
    assert np.array_equal(info["thr"][live].view(np.uint32), thr[live].view(np.uint32)), \
        np.flatnonzero(info["thr"].view(np.uint32) != thr.view(np.uint32))[:8]
    assert np.array_equal(info["cand_cnt"][live].astype(np.int64), cnt[live]), \
        np.argwhere(info["cand_cnt"].astype(np.int64) != cnt)[:8]
    assert np.array_equal(st[:, 1].astype(bool), proven), np.flatnonzero(st[:, 1].astype(bool) != proven)[:8]
    if require_all_proven:
        assert proven[~bad].all()
    rng = rng or np.random.default_rng(len(queries) + k)
    for i in sample_ids(len(queries), rng):
        if st[i, 1]:
            check_query(got[i], st[i], rows, queries[i], k, row_base, where=f"query {i}")
    return A, cnt, proven


def new_corpus(ctx, rows, row_base=0):
    c = capi.Corpus(ctx, max(len(rows), 1), row_base=row_base)
    c.append(rows)
    return c


# ------------------------------------------------------------------ a. v2 stage contracts ---
def corpus_of(kind, rng, n):
    if kind == "random":
        return unit_rows(rng, n)
    if kind == "duplicated":
        base = unit_rows(rng, n // 4)
        rows = base[rng.integers(0, len(base), n)]
        return np.ascontiguousarray(rows)
    centers = unit_rows(rng, 16)
    x = centers[rng.integers(0, 16, n)] + 0.05 * rng.standard_normal((n, 256)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    return np.ascontiguousarray(x, dtype=np.float32)


@pytest.mark.parametrize("kind,n,nq,k", [("random", 70_000, 130, 10), ("duplicated", 120_000, 64, 5),
                                         ("clustered", 280_000, 40, 16), ("random", 140_001, 257, 1),
                                         ("clustered", 51_200, 20, 64)])
def test_v2_stage_contracts(ctx, sm_count, kind, n, nq, k):
    rng = np.random.default_rng(n + nq + k)
    rows = corpus_of(kind, rng, n)
    queries = unit_rows(rng, nq)
    queries[0] = rows[n // 3]
    queries[nq - 1] = rows[n - 1]
    c = new_corpus(ctx, rows)
    got, st, info = run_dev(ctx, c, queries, k)
    exp = route_rule(n, k, sm_count)
    assert exp["route"] == 2 and {key: info[key] for key in exp} == exp, (info, exp)
    check_v2_call(ctx, rows, queries, k, got, st, info, require_all_proven=(kind == "random"))


# ------------------------------------------------------------------ b. capacity edges ---
def at_cos(q, cos, rng, m=1):
    """m distinct unit rows at exact-ish cosine `cos` to the unit query q."""
    u = rng.standard_normal((m, 256))
    qq = q.astype(np.float64)
    u -= np.outer(u @ qq, qq)
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    x = cos * qq[None, :] + np.sqrt(1.0 - cos * cos) * u
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def background(rng, q, n):
    """Random unit rows with every cosine to q below 0.4 (far below the constructed ones)."""
    rows = unit_rows(rng, n)
    hi = rows @ q > 0.4
    rows[hi] *= -1.0
    return rows


def capacity_case(ctx, sm, rows, q, k, where):
    """One query: route v2, the hook's counts equal the prediction; returns (counts, proven, m2)."""
    got, st, info = run_dev(ctx, new_corpus(ctx, rows), q[None, :], k)
    assert info["route"] == 2 and info["n_seg"] == min(-(-len(rows) // TILE), sm), info
    A = debug_scores(ctx, q[None, :], rows)
    thr, cnt, proven, m2 = predict_v2(A, k, info, np.zeros(1, bool))
    assert np.array_equal(info["thr"].view(np.uint32), thr.view(np.uint32)), where
    assert np.array_equal(info["cand_cnt"].astype(np.int64), cnt), where
    assert bool(st[0, 1]) == bool(proven[0]), (where, st[0], cnt[0].max(), cnt[0].sum(), m2[0])
    if st[0, 1]:
        check_query(got[0], st[0], rows, q, k, where=where)
    host = new_corpus(ctx, rows).search_batch(q[None, :], top_k=k)[0]
    r, d = oracle.search_rows(rows, q, top_k=k)
    assert host["row"].tolist() == [int(x) for x in r] and np.array_equal(host["distance"], d), where
    return cnt[0], bool(st[0, 1]), int(m2[0])


def anchored_corpus(rng, q, n_tiles, n_seg, special_tiles):
    """Background rows, plus one anchor row at cos 0.5 in every tile outside the special tiles' segments:
    with k <= 8 the threshold sits just below 0.5, so the special segment holds exactly what is put there."""
    rows = background(rng, q, n_tiles * TILE)
    special_segs = {t % n_seg for t in special_tiles}
    anchor = at_cos(q, 0.5, rng)[0]
    for t in range(n_tiles):
        if t % n_seg not in special_segs:
            rows[t * TILE + 7] = anchor
    return rows


@pytest.mark.parametrize("n_keys", [64, 65])
def test_segment_capacity(ctx, sm_count, n_keys):
    rng = np.random.default_rng(640 + n_keys)
    q = unit_rows(rng, 1)[0]
    n_tiles = 2 * sm_count + 10
    t0 = 5
    rows = anchored_corpus(rng, q, n_tiles, sm_count, [t0])
    near = at_cos(q, 0.9, rng, n_keys)
    near[-8:] = at_cos(q, 0.95, rng, 8)                        # the top-8 at the end of the segment
    rows[t0 * TILE: t0 * TILE + n_keys] = near
    cnt, proven, _ = capacity_case(ctx, sm_count, rows, q, 8, f"{n_keys} keys in one segment")
    assert cnt[t0 % sm_count] == n_keys
    assert proven == (n_keys <= SEG_CAP)


@pytest.mark.parametrize("first,second", [(40, 24), (40, 40)])
def test_segment_cursor_across_tiles_of_one_cta(ctx, sm_count, first, second):
    rng = np.random.default_rng(first * 100 + second)
    q = unit_rows(rng, 1)[0]
    n_tiles = 2 * sm_count + 10
    t0, t1 = 3, 3 + sm_count                                   # same CTA, consecutive iterations
    rows = anchored_corpus(rng, q, n_tiles, sm_count, [t0, t1])
    near = at_cos(q, 0.9, rng, first + second)
    near[first - 4: first] = at_cos(q, 0.95, rng, 4)           # the best rows at the end of each tile's run
    near[-4:] = at_cos(q, 0.96, rng, 4)
    rows[t0 * TILE + 200: t0 * TILE + 200 + first] = near[:first]
    rows[t1 * TILE: t1 * TILE + second] = near[first:]
    cnt, proven, _ = capacity_case(ctx, sm_count, rows, q, 8, f"{first}+{second} keys in one CTA")
    assert cnt[t0 % sm_count] == first + second
    assert proven == (first + second <= SEG_CAP)


@pytest.mark.parametrize("total", [4096, 4097])
def test_total_key_capacity(ctx, sm_count, total):
    """k = 1: one row at cos 0.9 in sampled tile 0 sets the threshold, an exact copy of q in an unsampled tile
    is the answer (the only narrowed key), and total - 2 rows at cos 0.8995 fill the segments <= 40 each."""
    rng = np.random.default_rng(total)
    q = unit_rows(rng, 1)[0]
    n_full = 2 * MAX_SAMPLE + 64                              # stride 2 whatever the SM count
    info = route_rule(n_full * TILE, 1, sm_count)
    assert info["route"] == 2 and info["stride"] >= 2, info
    n_seg = info["n_seg"]
    rows = background(rng, q, n_full * TILE)
    rows[3] = at_cos(q, 0.9, rng)[0]
    copy_tile = 1                                              # tile 1 is not sampled (stride >= 2)
    rows[copy_tile * TILE + 9] = q
    m = total - 2
    assert m <= 40 * n_seg
    fill = at_cos(q, 0.8995, rng)[0]                           # one vector: every copy has the same score
    per_seg = -(-m // n_seg)
    pos = []
    for s in range(n_seg):
        for j in range(per_seg):
            if len(pos) == m:
                break
            t = s + n_seg * (2 + j // 64)                      # tiles of segment s; never tile 0 or 1
            pos.append(t * TILE + 100 + j % 64)
    rows[np.array(pos)] = fill
    cnt, proven, m2 = capacity_case(ctx, sm_count, rows, q, 1, f"{total} keys")
    assert cnt.sum() == total and cnt.max() <= 40 and m2 == 1
    assert proven == (total <= F2_KEYS)


@pytest.mark.parametrize("narrowed", [1024, 1025])
def test_rescore_capacity(ctx, sm_count, narrowed):
    """k = 1: an exact copy of q and narrowed - 1 copies of a row at cos 0.9995, all within 2 EPS of the top."""
    rng = np.random.default_rng(narrowed)
    q = unit_rows(rng, 1)[0]
    n_tiles = 200
    rows = background(rng, q, n_tiles * TILE)
    rows[5 * TILE + 17] = q
    pos = rng.choice(np.setdiff1d(np.arange(len(rows)), [5 * TILE + 17]), narrowed - 1, replace=False)
    rows[pos] = at_cos(q, 0.9995, rng)[0]
    cnt, proven, m2 = capacity_case(ctx, sm_count, rows, q, 1, f"{narrowed} narrowed")
    assert m2 == narrowed and cnt.max() <= SEG_CAP
    assert proven == (narrowed <= F2_RESCORE)


def test_narrowing_band_uses_two_eps(ctx, sm_count):
    """About 1100 rows whose scores sit between A_k - 2 EPS and A_k - EPS: the 2 EPS cut narrows them all
    (over the re-score cap: unproven); a 1 EPS cut would keep none and prove the query."""
    _, eps = capi.batch_params()
    rng = np.random.default_rng(1100)
    q = unit_rows(rng, 1)[0]
    rows = background(rng, q, 200 * TILE)
    rows[9 * TILE + 3] = q
    pos = rng.choice(np.arange(10 * TILE, len(rows)), 1100, replace=False)
    rows[pos] = at_cos(q, 1.0 - 1.5 * eps, rng, 1100)
    A = debug_scores(ctx, q[None, :], rows)[0]
    a_k = A[9 * TILE + 3]
    band = A[pos]
    assert np.all(band >= a_k - np.float32(2 * eps)) and np.all(band < a_k - np.float32(eps)), (band.min(), band.max(), a_k)
    cnt, proven, m2 = capacity_case(ctx, sm_count, rows, q, 1, "band")
    assert m2 == 1101 and not proven


# ------------------------------------------------------------------ c. routes x shapes ---
V2_SHAPES = [(1, 70_000, 10), (127, 20_001, 1), (128, 64 * TILE, 64), (129, 2 * TILE + 255, 2),
             (257, 140 * TILE + 1, 63), (2049, 40 * TILE + 255, 2), (5, 3 * TILE, 3), (129, 300 * TILE + 128, 64)]
V1_SHAPES = [(9, 63 * TILE + 200, 64), (128, 30_000, 65), (257, 20_000, 97), (3, 5000, 1024), (2049, 20 * TILE + 1, 65),
             (1, 255, 1), (5, 1000, 10), (129, 50_000, 80), (1, 16 * TILE + 255, 17), (130, 140 * TILE + 255, 96)]


@pytest.mark.parametrize("nq,n,k", V2_SHAPES)
def test_v2_route_and_shapes(ctx, sm_count, nq, n, k):
    rng = np.random.default_rng(nq * 3 + n + k)
    rows = unit_rows(rng, n)
    queries = unit_rows(rng, nq)
    queries[nq // 2] = rows[n - 1]                             # a hit in the ragged last tile
    c = new_corpus(ctx, rows)
    got, st, info = run_dev(ctx, c, queries, k)
    exp = route_rule(n, k, sm_count)
    assert exp["route"] == 2 and {key: info[key] for key in exp} == exp, (info, exp)
    check_v2_call(ctx, rows, queries, k, got, st, info, rng=rng, require_all_proven=True)


@pytest.mark.parametrize("nq,n,k", V1_SHAPES)
def test_v1_route_and_shapes(ctx, sm_count, nq, n, k):
    rng = np.random.default_rng(nq * 5 + n + k)
    rows = unit_rows(rng, n)
    queries = unit_rows(rng, nq)
    queries[0] = rows[n - 1]
    c = new_corpus(ctx, rows)
    got, st, info = run_dev(ctx, c, queries, k)
    assert route_rule(n, k, sm_count)["route"] == 1
    assert info["route"] == 1 and info["nq"] == nq, info
    assert np.all(st[:, 0] <= min(k, n))
    for i in sample_ids(nq, rng):
        if st[i, 1]:
            check_query(got[i], st[i], rows, queries[i], k, where=f"query {i}")
    if k <= 16 and n >= 20_000:
        assert st[:, 1].mean() >= 0.8                          # v1 proves small k on random rows
    ids = sample_ids(nq, rng, extra=8)
    host = c.search_batch(queries[ids], top_k=k)
    for j, i in enumerate(ids):
        r, d = oracle.search_rows(rows, queries[i], top_k=k)
        assert host[j]["row"].tolist() == [int(x) for x in r] and np.array_equal(host[j]["distance"], d), i


def test_route_boundary_n_full_equals_k(ctx, sm_count):
    """n_full == k samples every tile (v2); n_full == k - 1 falls to v1."""
    rng = np.random.default_rng(7)
    for k, n_full, route in [(16, 16, 2), (17, 16, 1), (64, 64, 2), (65, 64, 1), (64, 63, 1)]:
        n = n_full * TILE + 100
        rows = unit_rows(rng, n)
        queries = unit_rows(rng, 3)
        got, st, info = run_dev(ctx, new_corpus(ctx, rows), queries, k)
        assert info["route"] == route == route_rule(n, k, sm_count)["route"], (k, n_full, info)
        if route == 2:
            assert info["n_sample"] == n_full and info["stride"] == 1
            check_v2_call(ctx, rows, queries, k, got, st, info, require_all_proven=True)


def test_argument_handling(ctx):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(3)
    rows = unit_rows(rng, 3000)
    c = new_corpus(ctx, rows)
    dev = torch.device("cuda:0")
    q = torch.from_numpy(unit_rows(rng, 2)).to(dev)
    hits = torch.zeros((2, 1100, 2), dtype=torch.float64, device=dev)
    status = torch.zeros((2, 2), dtype=torch.int32, device=dev)
    for k in (0, 1025):
        with pytest.raises(capi.StbError) as e:
            c.search_batch_dev(q.data_ptr(), 2, k, hits.data_ptr(), status.data_ptr())
        assert e.value.status == capi.STB_ERR_ARG
    empty = capi.Corpus(ctx, 16)
    with pytest.raises(capi.StbError) as e:
        empty.search_batch_dev(q.data_ptr(), 2, 10, hits.data_ptr(), status.data_ptr())
    assert e.value.status == capi.STB_ERR_STATE
    queries = unit_rows(rng, 2)
    queries[1] = rows[2999]
    res = c.search_batch(queries, top_k=1500)                  # above the tensor path's 1024: K1
    for i in range(2):
        r, d = oracle.search_rows(rows, queries[i], top_k=1500)
        assert res[i]["row"].tolist() == [int(x) for x in r] and np.array_equal(res[i]["distance"], d)


# ------------------------------------------------------------------ d. bad and degenerate queries ---
def with_bad_queries(rng, rows, n_good):
    """Good random queries with, interleaved, a zero query, NaN / +inf / -inf components and copies of rows
    scaled by 1e-20, 1e20 and 1e-25 (the last three cannot be normalised in fp32).  Returns (queries, kinds)."""
    queries = list(unit_rows(rng, n_good))
    kinds = ["good"] * n_good
    nan = unit_rows(rng, 1)[0]; nan[7] = np.nan
    pinf = unit_rows(rng, 1)[0]; pinf[3] = np.inf
    minf = unit_rows(rng, 1)[0]; minf[200] = -np.inf
    specials = [("zero", np.zeros(256, np.float32)), ("nan", nan), ("+inf", pinf), ("-inf", minf),
                ("x1e-20", rows[11] * np.float32(1e-20)), ("x1e20", rows[12] * np.float32(1e20)),
                ("x1e-25", rows[13] * np.float32(1e-25))]
    for j, (kind, v) in enumerate(specials):
        at = (j * 37 + 5) % (len(queries) + 1)
        queries.insert(at, v.astype(np.float32))
        kinds.insert(at, kind)
    return np.ascontiguousarray(np.stack(queries), dtype=np.float32), kinds


@pytest.mark.parametrize("n,k", [(70_000, 10), (2_000, 10), (70_000, 97)])
def test_bad_queries_are_never_proven_wrong(ctx, sm_count, n, k):
    """Pipeline v2, then v1 twice: on a corpus of fewer than k complete tiles, and for k > 64."""
    route = "v2" if route_rule(n, k, sm_count)["route"] == 2 else "v1"
    assert route == ("v1" if n // TILE < k or k > MAX_K else "v2")
    rng = np.random.default_rng(n + k)
    rows = unit_rows(rng, n)
    queries, kinds = with_bad_queries(rng, rows, 40)
    bad = unnormalisable(queries)
    assert [kinds[i] for i in np.flatnonzero(bad)] == [x for x in kinds if x in ("nan", "+inf", "-inf", "x1e-20", "x1e20", "x1e-25")]
    c = new_corpus(ctx, rows)
    got, st, info = run_dev(ctx, c, queries, k)
    assert info["route"] == (2 if route == "v2" else 1)
    for i, kind in enumerate(kinds):
        if kind != "good" and st[i, 1]:
            check_query(got[i], st[i], rows, queries[i], k, where=f"{kind} query {i} proven")
    assert not st[bad, 1].any(), [kinds[i] for i in np.flatnonzero(bad & (st[:, 1] == 1))]
    good = np.array([x == "good" for x in kinds])
    if k <= 16:
        assert st[good, 1].all() if route == "v2" else st[good, 1].mean() >= 0.8
    if route == "v2":
        check_v2_call(ctx, rows, queries, k, got, st, info, rng=rng)
    before = ctx.counters()["fallback_searches"]
    host = c.search_batch(queries, top_k=k)
    unproven = int((st[:, 1] == 0).sum())
    assert unproven <= ctx.counters()["fallback_searches"] - before <= 2 * unproven
    for i in range(len(queries)):
        r, d = oracle.search_rows(rows, queries[i], top_k=k)
        assert host[i]["row"].tolist() == [int(x) for x in r], (kinds[i], i)
        assert np.array_equal(host[i]["distance"], d), (kinds[i], i)


def test_bad_queries_in_the_sharded_exchange():
    torch = pytest.importorskip("torch")
    from semtools_b200.sharded import shard_bounds
    world, k = 2, 10
    rng = np.random.default_rng(202)
    n = 40_000
    rows = unit_rows(rng, n)
    queries, kinds = with_bad_queries(rng, rows, 9)
    nq = len(queries)
    bad = unnormalisable(queries)
    dev = torch.device("cuda:0")
    ctxs = [capi.Context(0) for _ in range(world)]
    corpora, xs = [], []
    for r in range(world):
        lo, hi = shard_bounds(n, world, r)
        corpora.append(new_corpus(ctxs[r], rows[lo:hi], row_base=lo))
        xs.append(capi.Exchange(ctxs[r], world, r, k, max_nq=32))
    for x in xs:
        x.connect_local(xs)
    q_dev = torch.from_numpy(queries).to(dev)
    out = torch.zeros((world, nq, k, 2), dtype=torch.float64, device=dev)
    status = torch.zeros((world, nq, 2), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    for r in range(world):
        xs[r].search_batch_dev(corpora[r], q_dev.data_ptr(), nq, k, out[r].data_ptr(), status[r].data_ptr())
    for cx in ctxs:
        cx.sync()
    raw, st = out.cpu().numpy(), status.cpu().numpy()
    assert (st[:, :, 1] <= 1).all(), "a rank timed out waiting for a peer"
    for r in range(world):
        assert np.array_equal(st[r], st[0])
        assert not st[r, bad, 1].any(), [kinds[i] for i in np.flatnonzero(bad & (st[r, :, 1] == 1))]
        hits = np.ascontiguousarray(raw[r]).view(capi.HIT_DTYPE).reshape(nq, k)
        for i in range(nq):
            if st[r, i, 1]:
                rr, dd = oracle.search_rows(rows, queries[i], top_k=k)
                assert hits[i]["row"].tolist() == [int(v) for v in rr] and np.array_equal(hits[i]["distance"], dd), (r, i)
    good = np.array([x == "good" for x in kinds])
    assert st[0, good, 1].all()
    for x in xs:
        x.close()
    for c in corpora:
        c.close()
    for cx in ctxs:
        cx.close()


def test_bad_queries_through_k1_topk_dev(ctx):
    """stb_search_topk_dev is where sharded K2 sends its unproven queries: the same queries, one by one."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(303)
    rows = unit_rows(rng, 50_000)
    queries, kinds = with_bad_queries(rng, rows, 3)
    c = new_corpus(ctx, rows)
    k = 10
    dev = torch.device("cuda:0")
    q_dev = torch.from_numpy(queries).to(dev)
    hits = torch.zeros((len(queries), k, 2), dtype=torch.float64, device=dev)
    status = torch.zeros((len(queries), 4), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    for i in range(len(queries)):
        c.search_topk_dev(q_dev[i].data_ptr(), k, hits[i].data_ptr(), status[i].data_ptr())
    ctx.sync()
    got = np.ascontiguousarray(hits.cpu().numpy()).view(capi.HIT_DTYPE).reshape(len(queries), k)
    st = status.cpu().numpy().view(np.uint32)
    for i, kind in enumerate(kinds):
        if st[i, 1] == 1:
            check_query(got[i], st[i], rows, queries[i], k, where=f"K1 {kind} query {i}")
        else:
            res = c.search(queries[i], top_k=k)
            r, d = oracle.search_rows(rows, queries[i], top_k=k)
            assert res["row"].tolist() == [int(x) for x in r] and np.array_equal(res["distance"], d), (kind, i)


# ------------------------------------------------------------------ e. data edges ---
@pytest.mark.parametrize("k", [8, 72])
def test_data_edges(ctx, sm_count, k):
    """k = 8 runs pipeline v2, k = 72 (> 64) pipeline v1."""
    route = "v2" if k <= MAX_K else "v1"
    rng = np.random.default_rng(55)
    n_tiles = sm_count + 20
    n = n_tiles * TILE - 37                                   # ragged last tile
    rows = unit_rows(rng, n)
    queries = unit_rows(rng, 24)
    cta_edge = sm_count * TILE                                # first row of the first tile a CTA reaches second
    rows[255] = rows[256] = queries[0]                        # exact tie across a tile boundary
    rows[cta_edge - 1] = rows[cta_edge] = rows[40] = (queries[1] + 0.01 * unit_rows(rng, 1)[0])   # ties across CTAs
    rows[[3, 1000, n - 1]] = 0.0                              # zero rows
    rows[500] = queries[2] * np.float32(1e-14)                # tiny but valid
    rows[600] = queries[3] * np.float32(1e14)                 # huge but valid
    rows[700] = -queries[4]                                   # anti-parallel: distance 2 clamps
    rows[[10, 2000, 9000, n - 2]] = queries[5]                # several exact copies: distance-0 ties by row
    queries[6] = -rows[800]                                   # its worst row
    queries[7] = rows[n - 2] * np.float32(3.0)
    row_base = 5_000_000_000
    c = new_corpus(ctx, rows, row_base=row_base)
    got, st, info = run_dev(ctx, c, queries, k)
    assert info["route"] == route_rule(n, k, sm_count)["route"] == (2 if route == "v2" else 1)
    if route == "v2":
        check_v2_call(ctx, rows, queries, k, got, st, info, row_base=row_base, require_all_proven=False)
    for i in range(len(queries)):
        if st[i, 1]:
            check_query(got[i], st[i], rows, queries[i], k, row_base=row_base, where=f"query {i}")
    if st[0, 1]:
        assert got[0]["row"][:2].tolist() == [row_base + 255, row_base + 256]
    if st[5, 1]:
        assert got[5]["row"][:4].tolist() == [row_base + r for r in (10, 2000, 9000, n - 2)]
    host = c.search_batch(queries, top_k=k)
    for i in range(len(queries)):
        r, d = oracle.search_rows(rows, queries[i], top_k=k)
        assert host[i]["row"].tolist() == [int(x) + row_base for x in r] and np.array_equal(host[i]["distance"], d), i


def test_append_extends_a_ragged_shadow(ctx, sm_count):
    rng = np.random.default_rng(66)
    rows = unit_rows(rng, 60 * TILE + 300)
    queries = unit_rows(rng, 20)
    queries[0] = rows[60 * TILE + 299]                        # lands in the tile the append completes
    queries[1] = rows[50 * TILE + 100]
    c = capi.Corpus(ctx, len(rows))
    c.append(rows[: 50 * TILE + 130])
    for m in (50 * TILE + 130, 55 * TILE + 1, len(rows)):
        if m > len(c):
            c.append(rows[len(c): m])
        got, st, info = run_dev(ctx, c, queries, 5)
        assert info["route"] == route_rule(m, 5, sm_count)["route"] == 2
        check_v2_call(ctx, rows[:m], queries, 5, got, st, info, require_all_proven=True)


# ------------------------------------------------------------------ f. the error bound on the GPU ---
def test_gemm_error_bound_on_adversarial_rows(ctx):
    """|a - c| <= EPS (batch_params) for 128 queries over rows built to round badly in fp16 / bf16."""
    f16, eps = capi.batch_params()
    rng = np.random.default_rng(99)
    mant = 10 if f16 else 7
    rows = []
    for e in (-4, -5, -6):                                    # components just below a rounding midpoint
        v = 2.0 ** e * (1 + 0.498 * 2.0 ** -mant)
        m = min(250, int(1.0 / (v * v)) - 1)
        w = np.sqrt(max(1.0 - m * v * v, 0.0) / (256 - m))
        x = np.array([v] * m + [w] * (256 - m))
        for _ in range(40):
            rows.append(rng.permutation(x) * rng.choice([-1.0, 1.0], 256))
    spiky = rng.standard_normal((200, 256)) * 1e-6             # fp16-subnormal components beside one large one
    spiky[np.arange(200), rng.integers(0, 256, 200)] = 1.0
    rows += list(spiky)
    mid = rng.standard_normal((200, 256))
    mid = np.round(mid * 2 ** 12) / 2 ** 12 + 2.0 ** -13        # halfway between 12-bit grid points
    rows += list(mid)
    rows += list(unit_rows(rng, 400) * rng.choice([1e-12, 1e-3, 1.0, 1e3, 1e12], (400, 1)))
    rows += [np.zeros(256)] * 5
    rows = np.ascontiguousarray(np.stack(rows), dtype=np.float32)
    queries = np.ascontiguousarray(rows[rng.choice(len(rows) - 5, 128, replace=False)], dtype=np.float32)
    queries[:8] = unit_rows(rng, 8)
    A = debug_scores(ctx, queries, rows)
    worst = 0.0
    for i, q in enumerate(queries):
        d = oracle.distances(rows, q)
        live = d != 1.0                                       # the ab == 0 -> distance 1 rule is not a score
        err = np.abs(A[i][live].astype(np.float64) - (1.0 - d[live]))
        worst = max(worst, float(err.max()))
    assert worst <= eps, f"worst |a - c| = {worst:.6f}, margin {eps - worst:.6f} of EPS {eps}"


# ------------------------------------------------------------------ g. shards of millions of rows ---
def random_device_corpus(ctx, n, seed):
    """n random unit rows generated on the device (too many to scan on the host): (rows, corpus)."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(seed)
    R = torch.empty((n, 256), dtype=torch.float32, device=dev)
    for lo in range(0, n, 1 << 20):
        hi = min(n, lo + (1 << 20))
        x = torch.randn((hi - lo, 256), generator=g, device=dev)
        R[lo:hi] = x / x.norm(dim=1, keepdim=True)
    c = capi.Corpus(ctx, n)
    torch.cuda.synchronize()
    c.append_dev(R.data_ptr(), n)
    return R, c


def exact_topk(R, q, k):
    """oracle.search_rows over device rows R: an f32 shortlist (error ~1e-6 on unit rows), ranked by
    oracle.distances -> (rows, distances)."""
    torch = pytest.importorskip("torch")
    cos = R @ torch.from_numpy(q).to(R.device)
    kth = torch.topk(cos, k).values[-1]
    short = torch.nonzero(cos >= kth - 1e-4).flatten().cpu().numpy()
    d = oracle.distances(R[torch.from_numpy(short).to(R.device)].cpu().numpy(), q)
    order = np.lexsort((short, d))[:k]
    return short[order], d[order]


def test_big_sample_threshold_kernel(ctx, sm_count):
    """n_sample > 608 takes stb_batch_thresh_big_kernel: about 8.7M rows on 132 SMs, k = 16."""
    torch = pytest.importorskip("torch")
    k = 16
    n_full = next(f for f in range(33_000, 200_000) if route_rule(f * TILE, k, sm_count)["route"] == 2
                  and route_rule(f * TILE, k, sm_count)["n_sample"] > MAX_SAMPLE)
    n = n_full * TILE + 100
    exp = route_rule(n, k, sm_count)
    assert exp["n_sample"] > MAX_SAMPLE
    R, c = random_device_corpus(ctx, n, 8)
    rng = np.random.default_rng(8)
    queries = unit_rows(rng, 8)
    queries[0] = c.read(n - 5, 1)[0]
    queries[1] = c.read(1234567, 1)[0]
    got, st, info = run_dev(ctx, c, queries, k)
    assert {key: info[key] for key in exp} == exp, (info, exp)
    # threshold: the sampled tiles' maxima, from the debug GEMM of exactly those tiles
    sampled = np.concatenate([c.read(t * exp["stride"] * TILE, TILE) for t in range(exp["n_sample"])])
    A = debug_scores(ctx, queries, sampled)
    _, eps = capi.batch_params()
    s_k = np.sort(A.reshape(len(queries), exp["n_sample"], TILE).max(axis=2), axis=1)[:, -k]
    thr = (s_k.astype(np.float32) - np.float32(2.0) * np.float32(eps)).astype(np.float32)
    assert np.array_equal(info["thr"].view(np.uint32), thr.view(np.uint32))
    assert st[:, 1].all()
    for i in range(len(queries)):
        r, d = exact_topk(R, queries[i], k)
        assert got[i]["row"].tolist() == r.tolist(), i
        assert np.array_equal(got[i]["distance"], d), i
    c.close()
    del R
    torch.cuda.empty_cache()


def test_v1_route_when_the_second_sample_overflows(ctx, sm_count):
    """17 <= k <= 64 on a shard so large that even the 1/64 sample expects more than 2048 keys per query
    runs v1: k = 64 from about 2.2M rows on 132 SMs."""
    torch = pytest.importorskip("torch")
    k = 64
    n_full = next(f for f in range(k, 200_000) if route_rule(f * TILE, k, sm_count)["route"] == 1)
    n = n_full * TILE + 100
    assert route_rule(n, k, sm_count)["route"] == 1
    R, c = random_device_corpus(ctx, n, 9)
    rng = np.random.default_rng(9)
    queries = unit_rows(rng, 6)
    queries[0] = c.read(n - 5, 1)[0]
    got, st, info = run_dev(ctx, c, queries, k)
    assert info["route"] == 1 and info["nq"] == len(queries), info
    assert np.all(st[:, 0] <= k)
    exact = [exact_topk(R, q, k) for q in queries]
    for i, (r, d) in enumerate(exact):
        if st[i, 1]:
            assert got[i]["row"].tolist() == r.tolist() and np.array_equal(got[i]["distance"], d), i
    host = c.search_batch(queries, top_k=k)
    assert ctx.batch_last()["route"] == 1
    for i, (r, d) in enumerate(exact):
        assert host[i]["row"].tolist() == r.tolist() and np.array_equal(host[i]["distance"], d), i
    c.close()
    del R
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ h. scratch reuse ---
def test_scratch_reuse_across_shapes(ctx, sm_count):
    """Alternate corpora of different tile counts and (nq, k) pairs on one context: stale counts, keys or
    thresholds from the previous call would show."""
    rng = np.random.default_rng(1234)
    big = unit_rows(rng, (sm_count + 60) * TILE + 11)
    small = unit_rows(rng, 20 * TILE + 200)
    cb, cs = new_corpus(ctx, big), new_corpus(ctx, small)
    qa = unit_rows(rng, 300)
    qb = unit_rows(rng, 5)
    qb[0] = small[20 * TILE + 199]
    for rows, c, qs, k in [(big, cb, qa, 64), (small, cs, qb, 1), (big, cb, qa[:130], 3), (small, cs, qb, 64),
                           (big, cb, qa, 64)]:
        got, st, info = run_dev(ctx, c, qs, k)
        assert info["route"] == route_rule(len(rows), k, sm_count)["route"]
        if info["route"] == 2:
            check_v2_call(ctx, rows, qs, k, got, st, info, rng=rng, require_all_proven=True)
        else:
            for i in range(len(qs)):
                if st[i, 1]:
                    check_query(got[i], st[i], rows, qs[i], k)

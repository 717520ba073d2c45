"""K2 routes 8, 9 and 10: the filtered, per-query-subset and threshold batch calls on the q8 copy and the int8 tensor
cores, the routes they take where the 16-bit shadow does not fit in HBM.  Context.batch_no_shadow (the
stb_debug_batch_no_shadow hook) makes every K2 call on the context act as if the shadow did not fit, so the public
calls' own code path is exercised without filling the card.

Every case runs on a 300k-row device corpus and its host-rows twin, with adversarial rows (duplicates, zero rows,
rows scaled by 1e-12 and 1e12, negated rows, near-copies of the queries, rows planted at chosen cosines) and a zero
and a NaN query:
- filtered (route 8): hits and counts bit for bit stb_search's in store-query mode with the same ranges, for top_k
  1-100, with and without a cap, over document subsets of 25, 5 and 1 %, ranges that cut tiles, None and the empty
  subset; the masked sample on the ineligible half of every tile; >= 99 % proven on random rows;
- subsets (route 9): several groups, an empty and a whole-shard one, each query equal to stb_search with its own
  ranges; one group is route 8 and equals the filtered call;
- threshold (route 10): equal to stb_search in threshold mode at ~1, 100 and 5000 hits per query, on both sides of a
  planted boundary, through the retry pass and past its budget; thresholds bit for bit the documented value;
- an unusable q8 copy gives K1's answers; with the hook off the calls keep routes 3, 6 and 5, and the hook leaves a
  built shadow's bytes unchanged."""
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
_API = open(os.path.join(ROOT, "semtools_b200", "csrc", "api.cu")).read()
_HDR = open(os.path.join(ROOT, "include", "semtools_b200.h")).read()
_COMMON = open(os.path.join(ROOT, "semtools_b200", "csrc", "common.cuh")).read()
DELTA = float(re.search(r"#define\s+STB_THR_DELTA\s+(\S+)", _API).group(1))
SEG_CAP = int(re.search(r"#define\s+STB_THR_SEG_CAP\s+(\d+)u", _API).group(1))
_BUDGET = re.search(r"#define\s+STB_BATCH_THRESHOLD_RETRY_KEYS\s+\((\d+)ull << (\d+)\)", _HDR)
BUDGET = int(_BUDGET.group(1)) << int(_BUDGET.group(2))
Q8_EPS = float(re.search(r"#define\s+STB_Q8_SCAN_EPS\s+(\S+)", _COMMON).group(1))
N = 300_000
TILE = 256
TOPKS = (1, 10, 16, 64, 65, 100)
NO_ROW = np.uint64(0xFFFFFFFFFFFFFFFF)
PLANT = 1000                                               # rows planted at chosen cosines to query 0
COSINES = (0.9, 0.7, 0.5, 0.3, 0.1)


@pytest.fixture(scope="module")
def sm_count():
    torch = pytest.importorskip("torch")
    return torch.cuda.get_device_properties(0).multi_processor_count


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def same(a, b, where=""):
    assert len(a) == len(b), f"{where}: {len(a)} hits, expected {len(b)}"
    assert np.array_equal(bits(a), bits(b)), where


def at_cos(q, cos, rng):
    u = rng.standard_normal(256)
    qq = q.astype(np.float64) / np.linalg.norm(q)
    u -= (u @ qq) * qq
    u /= np.linalg.norm(u)
    return (cos * qq + np.sqrt(1.0 - cos * cos) * u).astype(np.float32)


def adversarial_rows(rng, n, q0):
    rows = unit_rows(rng, n)
    rows[100:110] = rows[5]                                 # exact duplicates: ties at every distance
    rows[200:204] = 0.0                                     # zero rows
    rows[300:310] *= np.float32(1e-12)
    rows[400:410] *= np.float32(1e12)
    rows[500:510] = -rows[500:510]
    for j, cs in enumerate(COSINES):
        rows[PLANT + j] = at_cos(q0, cs, rng)
    return np.ascontiguousarray(rows)


def queries_for(rng, rows, nq):
    q = unit_rows(rng, nq)
    near = rows[[5, 1234, 400, 300]] + np.float32(1e-3) * unit_rows(rng, 4)
    special = np.zeros((2, 256), np.float32)
    special[1, 7] = np.nan                                  # a zero query and a NaN query
    return np.ascontiguousarray(np.concatenate([q, near, -rows[[501]], special]).astype(np.float32))


@pytest.fixture(scope="module")
def data():
    rng = np.random.default_rng(20261018)
    q0 = unit_rows(rng, 1)[0]
    rows = adversarial_rows(rng, N, q0)
    queries = queries_for(rng, rows, 60)
    queries[0] = q0
    return rows, queries


@pytest.fixture(scope="module")
def pair(ctx, data):
    rows, _ = data
    dev = capi.Corpus(ctx, N)
    dev.append(rows)
    host = capi.Corpus.in_host_memory(ctx, 1024)
    for part in np.array_split(rows, 3):
        host.append(part)
    yield dev, host
    dev.close()
    host.close()


def doc_ranges(rng, n, frac, mean_len=30):
    """A random subset of documents (consecutive lines, lognormal lengths) merged into ranges."""
    lens = np.clip(np.round(rng.lognormal(np.log(mean_len), 0.8, n)), 1, 200).astype(np.int64)
    starts = np.concatenate([[0], np.cumsum(lens)])
    starts = starts[starts < n]
    ends = np.append(starts[1:], n)
    keep = rng.random(len(starts)) < frac
    m = np.zeros(n, bool)
    for b, e in zip(starts[keep], ends[keep]):
        m[b:e] = True
    edges = np.flatnonzero(np.diff(np.concatenate([[0], m.astype(np.int8), [0]])))
    return edges.reshape(-1, 2).astype(np.uint64)


def filters(rng, n):
    cut = np.array([[t * TILE - 7, t * TILE + 9] for t in range(1, n // TILE, 5)], np.uint64)   # every range cuts tiles
    return {"docs25": doc_ranges(rng, n, 0.25), "docs5": doc_ranges(rng, n, 0.05), "docs1": doc_ranges(rng, n, 0.01),
            "cut": cut, "none": None, "empty": np.zeros((0, 2), np.uint64)}


def n_listed(ranges, n):
    if ranges is None:
        return -(-n // TILE)
    tiles = set()
    for b, e in np.asarray(ranges, np.int64).reshape(-1, 2).tolist():
        b, e = max(b, 0), min(e, n)
        if b < e:
            tiles.update(range(b // TILE, (e - 1) // TILE + 1))
    return len(tiles)


def local_ranges(ranges, n):
    if ranges is None:
        return np.array([[0, n]], np.uint64)
    r = np.clip(np.asarray(ranges, dtype=np.int64).reshape(-1, 2), 0, n)
    return r[r[:, 0] < r[:, 1]].astype(np.uint64)


def store_k1(c, q, k, cap, ranges):
    return c.search(q, top_k=k, max_distance=cap, mode=capi.STB_MODE_STORE_QUERY, row_ranges=ranges)


def expected_thr(m):
    """RD_f32(((1 - M) - STB_Q8_SCAN_EPS) - delta), the route 10 threshold on the upper bounds u."""
    x = ((np.float64(1.0) - np.float64(m)) - np.float64(Q8_EPS)) - np.float64(DELTA)
    f = np.float32(x)
    if np.float64(f) > x:
        f = np.nextafter(f, np.float32(-np.inf))
    return f


# ------------------------------------------------------------------------------------------ filtered ---
def test_filtered_parity(ctx, sm_count, data, pair):
    rows, queries = data
    rng = np.random.default_rng(5)
    flts = filters(rng, N)
    for c in pair:
        with ctx.batch_no_shadow():
            for name, ranges in flts.items():
                for k in TOPKS:
                    for cap in ((None, 0.7) if k in (10, 65) else (None,)):
                        fb = ctx.counters()["fallback_searches"]
                        got = c.search_batch_filtered(queries, ranges, top_k=k, max_distance=cap)
                        fell = ctx.counters()["fallback_searches"] - fb
                        info = ctx.batch_last()
                        if name == "empty":
                            assert info["route"] == 4 and fell == 0
                        else:
                            # route 8 where the q8 plan fits; else nothing runs on the tensor cores (route 4)
                            ns, stride, fits = capi.batch_q8_plan(sm_count, n_listed(ranges, N) * TILE, k)
                            assert info["route"] == (8 if fits else 4) and info["nq"] == len(queries), (name, k, info)
                            assert (info["n_sample"], info["stride"]) == ((ns, stride) if fits else (0, 0)), (name, k, info)
                            if fits:
                                assert info["n_seg"] == min(n_listed(ranges, N), sm_count) and info["seg_cap"] == 64
                                if k <= 16:                         # the zero and NaN queries, and few others
                                    assert fell <= 4 + len(queries) // 50, (name, k, fell)
                                assert np.all(info["thr"][-2:] == np.inf)       # the zero and NaN queries emit nothing
                            else:
                                assert fell >= len(queries)
                        for i, q in enumerate(queries):
                            same(got[i], store_k1(c, q, k, cap, ranges), f"{name} k={k} cap={cap} query {i}")
            for name in ("docs5", "cut"):
                for i in (0, 61, 62):
                    r, d32 = oracle.store_search(rows, local_ranges(flts[name], N), queries[i], 10)
                    got = c.search_batch_filtered(queries[i:i + 1], flts[name], top_k=10)[0]
                    assert got["row"].tolist() == [int(x) for x in r], (name, i)
                    assert np.array_equal(got["distance"].astype(np.float32), d32), (name, i)


def test_filtered_random_rows_are_proven(ctx):
    rng = np.random.default_rng(8)
    c = capi.Corpus(ctx, N)
    c.append(unit_rows(rng, N))
    queries = unit_rows(rng, 512)
    ranges = doc_ranges(rng, N, 0.25)
    with ctx.batch_no_shadow():
        for k in (1, 10, 16, 64):
            fb = ctx.counters()["fallback_searches"]
            got = c.search_batch_filtered(queries, ranges, top_k=k)
            fell = ctx.counters()["fallback_searches"] - fb
            info = ctx.batch_last()
            assert info["route"] == 8 and fell <= len(queries) // 100, (k, fell, info)
            for i in range(0, len(queries), 7):
                same(got[i], store_k1(c, queries[i], k, None, ranges), f"k={k} query {i}")
    c.close()


@pytest.mark.parametrize("k", [1, 10, 64])
def test_filtered_masked_sample(ctx, sm_count, k):
    """The first half of every tile is eligible; the second holds exact copies of the queries and rows at cosine
    0.99 and 0.995.  Unmasked, the sample would put the threshold near those rows and the eligible top-k would go
    unemitted; every query must be proven on route 8 and equal stb_search."""
    rng = np.random.default_rng(900 + k)
    n_tiles = 2 * sm_count + 40
    rows = unit_rows(rng, n_tiles * TILE)
    queries = unit_rows(rng, 12)
    for t in range(n_tiles):
        for j, q in enumerate(queries):
            rows[t * TILE + 128 + 2 * j] = q if t % 7 == 0 else at_cos(q, 0.99, rng)
            rows[t * TILE + 129 + 2 * j] = at_cos(q, 0.995, rng)
    ranges = np.array([[t * TILE, t * TILE + 128] for t in range(n_tiles)], np.uint64)
    for c in (capi.Corpus(ctx, len(rows)), capi.Corpus.in_host_memory(ctx, 1024)):
        c.append(rows)
        with ctx.batch_no_shadow():
            before = ctx.counters()["fallback_searches"]
            got = c.search_batch_filtered(queries, ranges, top_k=k)
            assert ctx.counters()["fallback_searches"] == before, "route 8 left a query unproven"
            assert ctx.batch_last()["route"] == 8
        for i, q in enumerate(queries):
            same(got[i], store_k1(c, q, k, None, ranges), f"query {i}")
            assert np.all(got[i]["row"] % TILE < 128) and len(got[i]) == k
        c.close()


# ------------------------------------------------------------------------------------------- subsets ---
def test_subsets_groups(ctx, sm_count, data, pair):
    rows, queries = data
    rng = np.random.default_rng(9)
    lists = [doc_ranges(rng, N, 0.25), doc_ranges(rng, N, 0.05), np.zeros((0, 2), np.uint64),
             np.array([[0, N]], np.uint64), doc_ranges(rng, N, 0.01),
             np.array([[N + 10, N + 20]], np.uint64)]                  # outside the shard: no clipped range
    per_query = [lists[i % len(lists)] for i in range(len(queries))]
    for c in pair:
        with ctx.batch_no_shadow():
            for k in (10, 64, 65):
                fb = ctx.counters()["fallback_searches"]
                got = c.search_batch_subsets(queries, per_query, top_k=k, max_distance=0.9 if k == 10 else None)
                info = ctx.batch_last()
                groups = sum(capi.batch_q8_plan(sm_count, n_listed(r, N) * TILE, k)[2] for r in (lists[0], lists[1],
                                                                                                    lists[3], lists[4]))
                # route 9 where a group fits the q8 plan; else no group runs on the tensor cores (route 6, 0 groups)
                assert info["route"] == (9 if groups else 6) and info["groups"] == groups, (k, info)
                assert (info["n_seg"], info["seg_cap"]) == (0, 0), (k, info)
                assert info["k1"] <= ctx.counters()["fallback_searches"] - fb
                for i, q in enumerate(queries):
                    same(got[i], store_k1(c, q, k, 0.9 if k == 10 else None, per_query[i]), f"k={k} query {i}")
            # one group for the whole batch is the filtered call (route 8)
            one = c.search_batch_subsets(queries, [lists[1]] * len(queries), top_k=10)
            assert ctx.batch_last()["route"] == 8
            for a, b in zip(one, c.search_batch_filtered(queries, lists[1], top_k=10)):
                same(a, b)


# ---------------------------------------------------------------- the q8 plan fits where v2's does not ---
def v2_plan_fits(n_listed_tiles, k, sm):
    """api.cu batch_v2_plan's fit rule, restated (tests/test_gpu_batch_filtered.py: route_rule)."""
    f16, _ = capi.batch_params()
    margin = 2 if f16 else 4
    ns = min(n_listed_tiles, min(4 * sm, 608))

    def emitted(x):
        return k * margin * (-(-n_listed_tiles // x)) if x else 0
    if emitted(ns) > 2048:
        ns = min(min(n_listed_tiles, 8192), (n_listed_tiles // 64 + sm - 1) // sm * sm)
    return k <= 64 and ns >= k and emitted(ns) <= 2048


def test_q8_plan_beyond_the_shadow_plan(ctx, sm_count):
    """3M rows at top_k = 64: batch_v2_plan does not fit, batch_q8_plan does.  With the shadow unavailable the
    filtered and subsets calls take routes 8 and 9; where the shadow fits they keep routes 4 and 6 (K1 answers every
    query, as before) and build no shadow, since they would not read it (K1, answering on a device corpus, may build
    one lazily as it always has; on the host-rows twin it builds none, so there the check is exact)."""
    n, k = 3_000_000, 64
    rng = np.random.default_rng(64)
    ranges = doc_ranges(rng, n, 0.25)
    per = [ranges if i % 2 else None for i in range(16)]
    per = [np.array([[0, n]], np.uint64) if r is None else r for r in per]
    for r in (None, ranges):
        nl = n_listed(r, n)
        assert not v2_plan_fits(nl, k, sm_count) and capi.batch_q8_plan(sm_count, nl * TILE, k)[2], nl
    rows = unit_rows(rng, n)
    queries = np.concatenate([unit_rows(rng, 14), rows[[17, n - 3]]])
    dev = capi.Corpus(ctx, n)
    for c in (dev, capi.Corpus.in_host_memory(ctx, 1 << 20)):
        for part in np.array_split(rows, 4):
            c.append(part)
        refs = [store_k1(c, q, k, None, ranges) for q in queries]
        refs_per = [store_k1(c, q, k, None, per[i]) for i, q in enumerate(queries)]
        with ctx.batch_no_shadow():
            got = c.search_batch_filtered(queries, ranges, top_k=k)
            info = ctx.batch_last()
            assert info["route"] == 8 and info["n_sample"] > 0, info
            for i in range(len(queries)):
                same(got[i], refs[i], f"route 8 query {i}")
            got = c.search_batch_subsets(queries, per, top_k=k)
            info = ctx.batch_last()
            assert (info["route"], info["groups"]) == (9, 2), info
            for i in range(len(queries)):
                same(got[i], refs_per[i], f"route 9 query {i}")
        # the shadow fits on this card: the calls keep their routes and leave no shadow behind
        got = c.search_batch_filtered(queries, ranges, top_k=k)
        assert ctx.batch_last()["route"] == 4
        got2 = c.search_batch_subsets(queries, per, top_k=k)
        info = ctx.batch_last()
        assert (info["route"], info["groups"]) == (6, 0), info
        if c is not dev:                # K1 builds no copy lazily on a host-rows corpus: any shadow would be K2's
            assert c.tier_stats()["h16"]["built_rows"] == 0
        for i in range(len(queries)):
            same(got[i], refs[i], f"route 4 query {i}")
            same(got2[i], refs_per[i], f"route 6 query {i}")
        c.close()


# ----------------------------------------------------------------------------------------- threshold ---
def hit_thresholds(rows, queries):
    q = queries[:16].astype(np.float64)
    r = rows.astype(np.float64)
    d = 1.0 - (q @ r.T) / np.maximum(np.linalg.norm(q, axis=1)[:, None] * np.linalg.norm(r, axis=1)[None, :], 1e-300)
    d = np.sort(d, axis=1)
    return [float(np.median(d[:, j])) for j in (1, 100, 5000)]


def check_threshold(ctx, c, queries, m, usable):
    got = c.search_batch_threshold(queries, m)
    info = ctx.batch_last()
    assert info["route"] == 10 and info["nq"] == len(queries) and info["n_seg"] > 0 and info["seg_cap"] == SEG_CAP, info
    t = expected_thr(m)
    for i in range(len(queries)):
        exp = t if usable[i] else np.float32(np.inf)
        assert info["thr"][i].tobytes() == exp.tobytes(), (m, i, info["thr"][i], exp)
    for i, q in enumerate(queries):
        same(got[i], c.search(q, top_k=0, max_distance=m), f"M={m!r} query {i}")
    return info


def test_threshold_parity(ctx, data, pair):
    rows, queries = data
    usable = np.all(np.isfinite(queries), axis=1) & np.any(queries != 0, axis=1)
    for c in pair:
        with ctx.batch_no_shadow():
            for m in hit_thresholds(rows, queries):
                info = check_threshold(ctx, c, queries, m, usable)
                assert info["k1"] >= 2                              # the zero and NaN queries
            # rows planted at canonical distances just below M (kept) and at M (dropped)
            for j in range(len(COSINES)):
                m = float(oracle.search_rows(rows[PLANT + j: PLANT + j + 1], queries[0], 0, 1e9)[1][0])
                for mm, present in ((m, False), (float(np.nextafter(m, np.inf)), True)):
                    got = c.search_batch_threshold(queries[:3], mm)
                    assert ctx.batch_last()["route"] == 10
                    assert ((PLANT + j) in got[0]["row"].tolist()) == present, (m, mm)
                    same(got[0], c.search(queries[0], top_k=0, max_distance=mm))
            # a short cap: STB_ERR_CAPACITY, every offset written, the first cap hits of the concatenation
            m = hit_thresholds(rows, queries)[1]
            full = c.search_batch_threshold(queries, m)
            total = sum(len(g) for g in full)
            out = np.zeros(total - 5, dtype=capi.HIT_DTYPE)
            off = np.zeros(len(queries) + 1, dtype=np.uint64)
            vp = C.c_void_p
            rc = capi.lib().stb_search_batch_threshold(ctx._h, c._h, queries.ctypes.data_as(vp), len(queries), m,
                                                       out.ctypes.data_as(vp), total - 5, off.ctypes.data_as(vp))
            assert rc == capi.STB_ERR_CAPACITY and int(off[-1]) == total
            assert np.array_equal(bits(out), bits(np.concatenate(full)[: total - 5]))


def test_threshold_past_the_retry_budget(ctx, data, pair):
    rows, queries = data
    for c in pair:
        with ctx.batch_no_shadow():
            # M = +inf emits every row: the retry pass takes what fits its key budget, K1 the rest
            nq = BUDGET // N + 5
            clean = unit_rows(np.random.default_rng(4), nq)
            got = c.search_batch_threshold(clean, float("inf"), cap=nq * N)
            info = ctx.batch_last()
            assert info["route"] == 10 and info["retried"] == BUDGET // N and info["k1"] == 5, info
            for i in (0, BUDGET // N - 1, BUDGET // N, nq - 1):
                same(got[i], c.search(clean[i], top_k=0, max_distance=float("inf")), f"inf query {i}")
            assert all(len(g) == N for g in got)


def test_threshold_overflowing_segments_use_the_retry_pass(ctx, sm_count):
    rng = np.random.default_rng(42)
    n_tiles = 2 * sm_count + 5
    rows = unit_rows(rng, n_tiles * TILE)
    queries = unit_rows(rng, 4)
    t0 = 7
    near = queries[0] + 1e-3 * rng.standard_normal((SEG_CAP + 30, 256)).astype(np.float32) / 16
    rows[t0 * TILE: t0 * TILE + len(near)] = near / np.linalg.norm(near, axis=1, keepdims=True)
    rows[(t0 + sm_count) * TILE + 3] = queries[0]                     # same CTA, another tile
    for c in (capi.Corpus(ctx, len(rows)), capi.Corpus.in_host_memory(ctx, 1024)):
        c.append(rows)
        with ctx.batch_no_shadow():
            before = ctx.counters()["fallback_searches"]
            got = c.search_batch_threshold(queries, 0.01)
            info = ctx.batch_last()
        assert info["route"] == 10 and info["retried"] == 1 and info["k1"] == 0, info
        assert info["cand_cnt"][0][t0 % sm_count] > SEG_CAP
        assert ctx.counters()["fallback_searches"] == before
        assert len(got[0]) == SEG_CAP + 31
        for i in range(len(queries)):
            same(got[i], c.search(queries[i], top_k=0, max_distance=0.01), f"query {i}")
        c.close()


# ------------------------------------------------------------------------------------- routes and hook ---
def test_unusable_q8_copy_gives_k1_answers(ctx, data):
    rows, queries = data
    bad = rows[:120_000].copy()
    bad[321] = unit_rows(np.random.default_rng(3), 1)[0] * np.float32(1e-20)
    ranges = doc_ranges(np.random.default_rng(6), len(bad), 0.25)
    for c in (capi.Corpus(ctx, len(bad)), capi.Corpus.in_host_memory(ctx, 1024)):
        c.append(bad)
        with ctx.batch_no_shadow():
            got = c.search_batch_filtered(queries[:20], ranges, top_k=10)
            assert ctx.batch_last()["route"] == 4
            for i in range(20):
                same(got[i], store_k1(c, queries[i], 10, None, ranges))
            per = [ranges, np.array([[0, 5000]], np.uint64)] * 10
            got = c.search_batch_subsets(queries[:20], per, top_k=10)
            info = ctx.batch_last()
            assert (info["route"], info["groups"]) == (9, 0), info
            for i in range(20):
                same(got[i], store_k1(c, queries[i], 10, None, per[i]))
            got = c.search_batch_threshold(queries[:20], 0.8)
            info = ctx.batch_last()
            assert (info["route"], info["k1"], info["n_seg"]) == (10, 20, 0), info
            for i in range(20):
                same(got[i], c.search(queries[i], top_k=0, max_distance=0.8))
        c.close()


def test_routes_off_the_hook_and_shadow_untouched(ctx, data):
    rows, queries = data
    sub = np.ascontiguousarray(rows[:40_000])
    ranges = doc_ranges(np.random.default_rng(7), len(sub), 0.25)
    per = [ranges, np.array([[0, 20_000]], np.uint64)] * (len(queries) // 2) + [ranges] * (len(queries) % 2)
    c = capi.Corpus(ctx, len(sub))
    c.append(sub)
    c.prepare_batch()
    shadow = bits(c.debug_copy(capi.STB_COPY_H16_TILES)[0]).copy()
    off = (c.search_batch_filtered(queries, ranges, top_k=10), c.search_batch_subsets(queries, per, top_k=10),
           c.search_batch_threshold(queries, 0.8))
    routes = []
    for call in (lambda: c.search_batch_filtered(queries, ranges, top_k=10), lambda: c.search_batch_subsets(queries, per, top_k=10),
                 lambda: c.search_batch_threshold(queries, 0.8), lambda: c.search_batch(queries, 10)):
        call()
        routes.append(ctx.batch_last()["route"])
    assert routes == [3, 6, 5, 2], routes
    with ctx.batch_no_shadow():
        on = (c.search_batch_filtered(queries, ranges, top_k=10), c.search_batch_subsets(queries, per, top_k=10),
              c.search_batch_threshold(queries, 0.8))
        routes = []
        for call in (lambda: c.search_batch_filtered(queries, ranges, top_k=10),
                     lambda: c.search_batch_subsets(queries, per, top_k=10),
                     lambda: c.search_batch_threshold(queries, 0.8), lambda: c.search_batch(queries, 10)):
            call()
            routes.append(ctx.batch_last()["route"])
        assert routes == [8, 9, 10, 7], routes
    assert np.array_equal(bits(c.debug_copy(capi.STB_COPY_H16_TILES)[0]), shadow)
    for a_list, b_list in zip(off, on):
        for a, b in zip(a_list, b_list):
            same(a, b)
    c.search_batch_filtered(queries, ranges, top_k=10)
    assert ctx.batch_last()["route"] == 3                     # the hook is off again
    c.close()

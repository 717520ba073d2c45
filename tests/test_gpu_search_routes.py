"""K1's host routes, call shape by call shape: what one stb_search (or stb_search_many) call costs in kernel
launches, fallback searches and per-tier bookkeeping (tries, proven, rows built), on a device corpus and on a
host-rows corpus, and its hits against the oracle.  Each shape runs on a fresh corpus, so the tier counts start
from zero; the counts are the routes' fingerprint: a call that takes another route changes them."""
import numpy as np
import pytest

import oracle
from conftest import unit_rows
from semtools_b200 import capi

pytestmark = pytest.mark.gpu
N = 40_000                       # above the 32768 rows from which a copy is built lazily
TOL = 1e-5
STORE = capi.STB_MODE_STORE_QUERY
RANGES = [[100, 5000], [20_000, 30_000]]
NAN = float("nan")


def random_data():
    rng = np.random.default_rng(20261018)
    return unit_rows(rng, N), unit_rows(rng, 8)


def skewed_data():
    """Rows with one dominant component under a sign query: every row's q8 bound sits ~0.06 above its cosine,
    beyond the k-th-bin route's 0.04 margin, so the q8 collect cannot prove its result and the f32 passes answer."""
    rng = np.random.default_rng(13)
    q = np.sign(unit_rows(rng, 1)[0]).astype(np.float32)
    rows = unit_rows(rng, 20_000)
    rows[:, 0] = np.float32(3.0) * q[0]
    return np.ascontiguousarray(rows), q[None, :]


def topk(k, **kw):
    def run(c, rows, qs):
        got = c.search(qs[0], top_k=k, **kw)
        return [(got, oracle.search_rows(rows, qs[0], top_k=k, max_distance=kw.get("max_distance")))]
    return run


def store(k, ranges, max_distance=None):
    def run(c, rows, qs):
        got = c.search(qs[0], top_k=k, max_distance=max_distance, mode=STORE, row_ranges=ranges)
        return [(got, oracle.store_search(rows, ranges, qs[0], k, max_distance))]
    return run


def zero_query(c, rows, qs):
    z = np.zeros(256, np.float32)
    return [(c.search(z, top_k=10), oracle.search_rows(rows, z, top_k=10))]


def clipped_to_nothing(c, rows, qs):
    got = c.search(qs[0], top_k=10, mode=STORE, row_ranges=[[N + 10, N + 20]])
    return [(got, (np.zeros(0, np.uint64), np.zeros(0)))]


def twice(c, rows, qs):
    return topk(10)(c, rows, qs) + topk(10)(c, rows, qs)


def many(k, nq):
    def run(c, rows, qs):
        got = c.search_many(qs[:nq], top_k=k)
        return [(g, oracle.search_rows(rows, q, top_k=k)) for g, q in zip(got, qs[:nq])]
    return run


# shape: (data, stb_corpus_prepare bits before the call, STB_SCAN_TIER, the call)
SHAPES = {
    "q8_top10": (random_data, 1, None, topk(10)),
    "zero_query": (random_data, 1, None, zero_query),                 # every row ties: nothing proves it
    "h16_top50": (random_data, 3, None, topk(50)),
    "kth_bin_q8_top200": (random_data, 1, None, topk(200)),
    "kth_bin_f32_retry_top200": (skewed_data, 1, None, topk(200)),
    "threshold_q8": (random_data, 1, None, topk(0, max_distance=0.85)),
    "threshold_f32": (random_data, 1, "f32", topk(0, max_distance=0.85)),
    "nan_cap_threshold": (random_data, 1, None, topk(0, max_distance=NAN)),
    "nan_cap_top10": (random_data, 1, None, store(10, [[0, N]], NAN)),
    "nan_cap_top200": (random_data, 1, None, store(200, [[0, N]], NAN)),
    "ranges_top10": (random_data, 1, None, store(10, RANGES)),
    "ranges_top200": (random_data, 1, None, store(200, RANGES, 0.97)),
    "ranges_clipped_to_nothing": (random_data, 1, None, clipped_to_nothing),
    "lazy_build_second_search": (random_data, 0, None, twice),
    "many_top10": (random_data, 0, None, many(10, 8)),
    "many_top200": (random_data, 0, None, many(200, 3)),
}
TIERS = ("f32", "h16", "q8")


def measure(ctx, kind, shape, monkeypatch):
    """Runs one shape on a fresh corpus: ((launches, fallbacks, tries, proven, rows built), [(got, want)])."""
    data, prepare, tier, call = SHAPES[shape]
    rows, qs = data()
    c = capi.Corpus.in_host_memory(ctx, len(rows)) if kind == "host" else capi.Corpus(ctx, len(rows))
    try:
        c.append(rows)
        if prepare:
            c.prepare(prepare)
        if tier:
            monkeypatch.setenv("STB_SCAN_TIER", tier)
        c0, t0 = ctx.counters(), c.tier_stats()
        pairs = call(c, rows, qs)
        c1, t1 = ctx.counters(), c.tier_stats()
    finally:
        c.close()
    delta = tuple(tuple(t1[t][f] - t0[t][f] for t in TIERS) for f in ("tries", "proven", "built_rows"))
    return (c1["kernel_launches"] - c0["kernel_launches"], c1["fallback_searches"] - c0["fallback_searches"]) + delta, pairs


def hits_match(got, want):
    rows, d = want
    return (got["row"].tolist() == [int(r) for r in rows]
            and bool(np.all(np.abs(got["distance"] - np.asarray(d, np.float64)) <= TOL)))


# (kernel launches, fallback searches, (tries), (proven), (rows built)); tiers in the order f32, h16, q8
EXPECTED = {
    ("device", "q8_top10"): (1, 0, (0, 0, 1), (0, 0, 1), (0, 0, 0)),
    ("device", "zero_query"): (32, 1, (1, 0, 1), (0, 0, 0), (0, 0, 0)),
    ("device", "h16_top50"): (1, 0, (0, 1, 0), (0, 1, 0), (0, 0, 0)),
    ("device", "kth_bin_q8_top200"): (4, 0, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("device", "kth_bin_f32_retry_top200"): (17, 1, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("device", "threshold_q8"): (3, 0, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("device", "threshold_f32"): (3, 0, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("device", "nan_cap_threshold"): (3, 0, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("device", "nan_cap_top10"): (1, 0, (0, 0, 1), (0, 0, 1), (0, 0, 0)),
    ("device", "nan_cap_top200"): (8, 1, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("device", "ranges_top10"): (1, 0, (0, 0, 1), (0, 0, 1), (0, 0, 0)),
    ("device", "ranges_top200"): (4, 0, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("device", "ranges_clipped_to_nothing"): (0, 0, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("device", "lazy_build_second_search"): (3, 0, (1, 0, 1), (1, 0, 1), (0, 0, 40000)),
    ("device", "many_top10"): (9, 0, (0, 0, 0), (0, 0, 0), (0, 0, 40000)),
    ("device", "many_top200"): (15, 0, (0, 0, 0), (0, 0, 0), (0, 0, 40000)),
    ("host", "q8_top10"): (1, 0, (0, 0, 1), (0, 0, 1), (0, 0, 0)),
    ("host", "zero_query"): (32, 0, (0, 0, 1), (0, 0, 0), (0, 0, 0)),
    ("host", "h16_top50"): (1, 0, (0, 1, 0), (0, 1, 0), (0, 0, 0)),
    ("host", "kth_bin_q8_top200"): (4, 0, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("host", "kth_bin_f32_retry_top200"): (17, 1, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("host", "threshold_q8"): (3, 0, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("host", "threshold_f32"): (3, 0, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("host", "nan_cap_threshold"): (3, 0, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("host", "nan_cap_top10"): (1, 0, (0, 0, 1), (0, 0, 1), (0, 0, 0)),
    ("host", "nan_cap_top200"): (8, 1, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("host", "ranges_top10"): (1, 0, (0, 0, 1), (0, 0, 1), (0, 0, 0)),
    ("host", "ranges_top200"): (4, 0, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("host", "ranges_clipped_to_nothing"): (0, 0, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("host", "lazy_build_second_search"): (2, 0, (0, 0, 2), (0, 0, 2), (0, 0, 0)),
    ("host", "many_top10"): (8, 0, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    ("host", "many_top200"): (14, 0, (0, 0, 0), (0, 0, 0), (0, 0, 0)),
}


@pytest.mark.parametrize("kind", ["device", "host"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_route_costs_and_hits(ctx, kind, shape, monkeypatch):
    counts, pairs = measure(ctx, kind, shape, monkeypatch)
    assert all(hits_match(g, w) for g, w in pairs)
    assert counts == EXPECTED[(kind, shape)]

"""The q8 tier's top-k scan with its 4-bit prefilter (csrc/scan_topk.cu: stb_scan_q4) against the CPU
oracle: hits, order and distances must be the oracle's bit for bit, proven by the q8 tier itself where
the data allows it, and still right (through the wider tiers / the collect path) where it does not."""
import ctypes

import numpy as np
import pytest

import oracle
from conftest import unit_rows
from semtools_b200 import capi

pytestmark = pytest.mark.gpu


def check(hits, rows_exp, d_exp):
    assert hits["row"].tolist() == [int(r) for r in rows_exp]
    assert np.array_equal(hits["distance"], np.asarray(d_exp, dtype=np.float64))


def refined(ctx, reset=True):
    v = ctypes.c_uint64(0)
    capi._check(capi.lib().stb_debug_q4_refined(ctx._h, 1 if reset else 0, ctypes.byref(v)))
    return int(v.value)


def q8_corpus(ctx, rows):
    c = capi.Corpus(ctx, len(rows))
    c.append(rows)
    c.prepare(1)                                     # STB_PREPARE_Q8: codes + nibble plane
    return c


@pytest.fixture
def q8_only(monkeypatch):
    monkeypatch.setenv("STB_SCAN_TIER", "q8")


@pytest.mark.parametrize("n", [1, 33, 5_000, 200_000])
def test_random_rows_are_proven_by_the_q8_tier(ctx, q8_only, n):
    """n = 5000 lies below the rows the prefilter needs before T exists: every row is refined."""
    rng = np.random.default_rng(40 + n)
    rows = unit_rows(rng, n)
    c = q8_corpus(ctx, rows)
    for i, k in enumerate((1, 10, 16)):
        q = unit_rows(rng, 1)[0]
        r, d = oracle.search_rows(rows, q, top_k=k)
        check(c.search(q, top_k=k), r, d)
        if n >= 5_000:
            assert c.tier_stats()["q8"]["proven"] == i + 1


def test_heavy_duplication_still_matches(ctx, q8_only):
    rng = np.random.default_rng(41)
    rows = unit_rows(rng, 60_000)
    q = unit_rows(rng, 1)[0]
    where = rng.choice(60_000, 500, replace=False)
    rows[where] = (q + 0.01 * unit_rows(rng, 1)[0]).astype(np.float32)
    c = q8_corpus(ctx, rows)
    r, d = oracle.search_rows(rows, q, top_k=10)
    check(c.search(q, top_k=10), r, d)
    assert sorted(where)[:10] == [int(x) for x in r]


def test_ties_resolve_by_row(ctx, q8_only):
    rng = np.random.default_rng(42)
    rows = unit_rows(rng, 100_000)
    q = unit_rows(rng, 1)[0]
    best = int(np.argmax(rows @ q))
    for dst in (5, 70_000, 99_999):                  # exact copies of the best row, before and after it
        rows[dst] = rows[best]
    rows[rng.integers(0, 100_000, 4)] = 0.0
    c = q8_corpus(ctx, rows)
    for k in (1, 4, 10, 16):
        r, d = oracle.search_rows(rows, q, top_k=k)
        check(c.search(q, top_k=k), r, d)


def test_row_ranges(ctx, q8_only):
    rng = np.random.default_rng(43)
    n = 300_000
    rows = unit_rows(rng, n)
    q = unit_rows(rng, 1)[0]
    c = q8_corpus(ctx, rows)
    for ranges in ([[1000, n - 1000]], [[0, 10], [500, 150_000], [200_000, 200_001], [250_000, n]]):
        for k in (1, 10):
            r, d32 = oracle.store_search(rows, ranges, q, k)
            hits = c.search(q, top_k=k, mode=capi.STB_MODE_STORE_QUERY, row_ranges=ranges)
            assert hits["row"].tolist() == [int(x) for x in r]
            assert np.array_equal(hits["distance"].astype(np.float32), d32)


def test_corpus_extended_by_appends(ctx, q8_only):
    """The plane is extended with the codes: rows appended after the copy was built are scanned too."""
    rng = np.random.default_rng(44)
    rows = unit_rows(rng, 150_000)
    q = unit_rows(rng, 1)[0]
    c = q8_corpus(ctx, rows[:100_000])
    r, d = oracle.search_rows(rows[:100_000], q, top_k=10)
    check(c.search(q, top_k=10), r, d)
    rows[120_000] = q                                # the new best row lives in the appended part
    c.append(rows[100_000:])
    c.prepare(1)
    assert c.tier_stats()["q8"]["built_rows"] == 150_000
    r, d = oracle.search_rows(rows, q, top_k=10)
    assert int(r[0]) == 120_000
    check(c.search(q, top_k=10), r, d)
    assert c.tier_stats()["q8"]["proven"] == 1                 # tier statistics restart with the append


def test_prefilter_refines_a_small_share_of_1m_random_rows(ctx, q8_only):
    """Until the k threshold words exist every warp refines what it scans; on an H100 that warm-up is ~15 %
    of a 1M-row corpus (2.9 % of 10M rows), so the bound here leaves room for the warm-up only."""
    rng = np.random.default_rng(45)
    n = 1_000_000
    rows = unit_rows(rng, n)
    c = q8_corpus(ctx, rows)
    q = unit_rows(rng, 1)[0]
    refined(ctx)
    hits = c.search(q, top_k=10)
    m = refined(ctx)
    r, d = oracle.search_rows(rows, q, top_k=10)
    check(hits, r, d)
    assert c.tier_stats()["q8"]["proven"] == 1
    assert 0 < m < 0.25 * n, m


@pytest.mark.parametrize("kind", ["constant", "nibble_tops"])
def test_exact_match_behind_near_copies_of_the_query(ctx, q8_only, kind):
    """k+6 near-copies of the query early in a 1M-row corpus fill every threshold word with bounds close to 1
    before the exact match (cosine 1) is scanned near the end.  Its 4-bit bound must still clear T: the
    query is a row whose codes all sit at the top of their nibbles, where a wrong nibble centre under-bounds."""
    rng = np.random.default_rng(46)
    n = 1_000_000
    rows = unit_rows(rng, n)
    if kind == "constant":
        q = np.ones(256, dtype=np.float32)
    else:
        codes = np.clip(16 * rng.integers(-8, 7, 256) + 15, -127, 127)
        codes[0] = 127
        q = (codes / 127.0).astype(np.float32)
    rows[:16] = (q[None, :] + 1e-3 * unit_rows(rng, 16)).astype(np.float32)
    rows[n - 1000] = q
    c = q8_corpus(ctx, rows)
    for k in (1, 10, 16):
        r, d = oracle.search_rows(rows, q, top_k=k)
        assert int(r[0]) == n - 1000
        check(c.search(q, top_k=k), r, d)

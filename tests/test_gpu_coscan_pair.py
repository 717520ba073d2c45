"""K1 pairs (scan_topk.cu: "pairs"): in an asynchronous q8 top-k series, each query after a host joins the
host's running scan, which scores both from one read of each plane tile.  Who scores a tile must not change a
result: every query's hits and status must be the bytes a scan of the query alone gives, whether it joined,
was refused, or hosted.  stb_debug_pair_joins shows which launches joined and at which tile."""
import numpy as np
import pytest

from conftest import unit_rows
from semtools_b200 import capi

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = torch.device("cuda:0")
PAIR_MIN_ROWS = 60000 * 32          # STB_PAIR_MIN_TILES plane tiles of 32 rows: smaller series co-scan instead


def need_pairs(n):
    if n < PAIR_MIN_ROWS:
        pytest.skip("below the pair size: the series co-scans")


@pytest.fixture(scope="module", params=[1_000_000, 2_000_017], ids=["1M", "2M+17"])
def corpus(request, ctx):
    rng = np.random.default_rng(request.param % 1000)
    rows = unit_rows(rng, request.param)
    c = capi.Corpus(ctx, request.param)
    c.append(rows)
    c.prepare(1)
    del rows
    yield c, request.param
    c.close()


def solo(c, q, k):
    """The same query alone: a synchronous search, which reads its q8 scan's hits, or the exact fallback."""
    return c.search(q, top_k=k)


def run_series(ctx, c, qs, k, sync_after=None, append=None):
    """stb_search_topk_dev for every query back to back into its own slot; returns (hits, status, joins)."""
    q_dev = torch.from_numpy(np.ascontiguousarray(qs, dtype=np.float32)).to(DEV)
    hits = torch.zeros((len(qs), k, 2), dtype=torch.float64, device=DEV)
    st = torch.zeros((len(qs), 4), dtype=torch.int32, device=DEV)
    torch.cuda.synchronize()
    for i in range(len(qs)):
        if sync_after is not None and i == sync_after + 1:
            ctx.sync()
        if append is not None and i == append[0] + 1:
            c.append(append[1])
            c.prepare(1)                                               # the q8 copy covers the new rows
        c.search_topk_dev(q_dev[i].data_ptr(), k, hits[i].data_ptr(), st[i].data_ptr())
    joins = ctx.pair_joins(min(len(qs), 8))
    d, h = ctx.ticket_check()
    assert d == h
    raw = np.ascontiguousarray(hits.cpu().numpy())
    return raw, st.cpu().numpy(), joins


def assert_solo(c, raw, st, qs, k, proven=True):
    for i, q in enumerate(qs):
        ref = solo(c, q, k)
        if proven:
            assert st[i, 1] == 1, (i, st[i])
        if st[i, 1] == 1:
            got = raw[i].view(capi.HIT_DTYPE).reshape(-1)[: st[i, 0]]
            assert got.tobytes() == ref.tobytes(), (i, got, ref)
            assert st[i, 3] >> 16 == 2                                    # the q8 tier answered


@pytest.mark.parametrize("k", [1, 10, 16])
def test_device_series_pairs_and_matches_solo_scans(ctx, corpus, k):
    corpus, n = corpus
    rng = np.random.default_rng(k)
    qs = unit_rows(rng, 12)
    raw, st, joins = run_series(ctx, corpus, qs, k)
    assert_solo(corpus, raw, st, qs, k)
    if n < PAIR_MIN_ROWS:
        assert joins == [None] * 8, joins                             # co-scans, no pairs
        return
    # last 8 launches: host, guest, host, guest, ...; guests join while their host runs
    guests = joins[1::2]
    assert all(j is None for j in joins[0::2]), joins
    assert all(isinstance(j, int) for j in guests), joins
    n_tiles = -(-n // 32)
    assert all(0 <= j < n_tiles for j in guests), joins


@pytest.mark.parametrize("nq", [16, 7])
def test_search_many_pairs_and_matches_solo_scans(ctx, corpus, nq):
    corpus, n = corpus
    rng = np.random.default_rng(100 + nq)
    qs = unit_rows(rng, nq)
    many = corpus.search_many(qs, top_k=10)
    joins = ctx.pair_joins(8)
    assert any(isinstance(j, int) for j in joins) == (n >= PAIR_MIN_ROWS), joins
    for i, q in enumerate(qs):
        assert many[i].tobytes() == solo(corpus, q, 10).tobytes(), i
    d, h = ctx.ticket_check()
    assert d == h


def test_a_synchronised_guest_is_refused_and_scans_alone(ctx, corpus):
    corpus, n = corpus
    need_pairs(n)
    rng = np.random.default_rng(5)
    qs = unit_rows(rng, 4)
    raw, st, joins = run_series(ctx, corpus, qs, 10, sync_after=0)   # the host completes before the guest
    assert joins[-4:][1] == "refused" and isinstance(joins[-4:][3], int), joins
    assert_solo(corpus, raw, st, qs, 10)


def test_a_late_join_scores_the_wrap_for_the_guest(ctx, corpus):
    corpus, n = corpus
    need_pairs(n)
    rng = np.random.default_rng(6)
    qs = unit_rows(rng, 4)
    n_tiles = -(-n // 32)
    floor = n_tiles // 8                                               # bulk tickets: 4 tiles each
    ctx.pair_floor(floor)
    try:
        raw, st, joins = run_series(ctx, corpus, qs, 10)
    finally:
        ctx.pair_floor(0)
    for j in joins[-4:][1::2]:
        assert j == "refused" or j >= 4 * floor, joins
    assert any(isinstance(j, int) for j in joins[-4:][1::2]), joins
    assert_solo(corpus, raw, st, qs, 10)


def test_zero_and_unusable_queries_as_guest_and_as_host(ctx, corpus):
    corpus, n = corpus
    need_pairs(n)
    rng = np.random.default_rng(8)
    qs = unit_rows(rng, 6)
    qs[1] = 0.0                                                        # a guest the q8 tier cannot use
    qs[2] = 0.0                                                        # a host that cannot use it
    qs[5, 7] = np.inf                                                  # an unusable guest
    raw, st, joins = run_series(ctx, corpus, qs, 10)
    j = joins[-6:]
    assert j[1] == "refused" and j[5] == "refused", j
    assert isinstance(j[3], int), j                                    # a usable guest of an unusable host joins
    for i in (1, 2, 5):
        assert st[i, 1] == 0                                           # unproven, as alone: the caller falls back
    ok = [0, 3, 4]
    assert_solo(corpus, raw[ok], st[ok], qs[ok], 10)


def test_an_append_between_host_and_guest_closes_the_seat(ctx):
    rng = np.random.default_rng(9)
    n0 = PAIR_MIN_ROWS + 1000
    rows = unit_rows(rng, n0 + 40_000)
    c = capi.Corpus(ctx, n0 + 40_000)
    c.append(rows[:n0])
    c.prepare(1)
    qs = unit_rows(rng, 4)
    raw, st, joins = run_series(ctx, c, qs, 10, append=(0, rows[n0:]))
    j = joins[-4:]
    assert j[1] is None and isinstance(j[2], int), j                   # launch 1 hosts a new pair on more rows
    assert st[0, 1] == 1 and all(st[1:, 1] == 1)
    c1 = capi.Corpus(ctx, n0)
    c1.append(rows[:n0])
    got0 = raw[0].view(capi.HIT_DTYPE).reshape(-1)[: st[0, 0]]
    assert got0.tobytes() == c1.search(qs[0], top_k=10).tobytes()
    for i in (1, 2, 3):
        got = raw[i].view(capi.HIT_DTYPE).reshape(-1)[: st[i, 0]]
        assert got.tobytes() == c.search(qs[i], top_k=10).tobytes(), i
    c.close(); c1.close()

"""K1 co-scan series against an exact scan of the whole corpus.

The benchmarked query stream is a back-to-back series of stb_search_topk_dev launches in which every
launch starts its pass at the tile its predecessor is reading and wraps around the end of the corpus
(scan_topk.cu: stb_coscan_offset, stb_for_each_tile).  Its claim is that hits, order and f64 distances
are bit-identical to the oracle's for every query of such a series.  These tests hold it to that claim
at the benchmark's own corpus (1M and 10M rows), on planted adversarial rows, on rows that cannot be
normalised, and at the tile counts where the ticket arithmetic changes regime.

`exact_topk` is the reference: the oracle's canonical f64 distances over chunks of the corpus, every
row that ties the chunk's k-th distance kept, merged by (distance, row).  It scales to 10M rows with
one chunk plus the candidates in host memory, and is itself checked against oracle.search_rows on the
CPU."""
from types import SimpleNamespace

import numpy as np
import pytest

import bench
import oracle
from conftest import unit_rows
from semtools_b200 import capi

TIER_SRC = {"f32": 0, "h16": 1, "q8": 2}          # status[3] >> 16
TILE_ROWS = {"f32": 8, "h16": 16, "q8": 32}       # 4 * U rows per tile (scan_topk.cu: stb_launch_topk_t)
PREPARE = {"f32": 0, "h16": 2, "q8": 1}           # STB_PREPARE_* flag that builds the tier's copy
WIDE_K = (17, 40, 64, 96)                         # the three list classes of stb_pick_e beyond k = 16


# ------------------------------------------------------------------ reference ---
def exact_topk(read_chunk, n, queries, k, chunk=bench.CHUNK):
    """Exact top-k of every query over rows [0, n): a list of (rows u64, distances f64) ordered by
    (distance, row), as oracle.search_rows returns them.  read_chunk(first, count) gives the f32 rows."""
    queries = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, capi.STB_DIM)
    kept = [([], []) for _ in range(len(queries))]
    for lo in range(0, n, chunk):
        x = np.ascontiguousarray(read_chunk(lo, min(chunk, n - lo)), dtype=np.float32)
        for (rows, dists), q in zip(kept, queries):
            d = oracle.distances(x, q)
            sel = np.flatnonzero(d <= np.partition(d, k - 1)[k - 1]) if d.size > k else np.arange(d.size)
            sel = sel[np.lexsort((sel, d[sel]))[:k]]           # ties at the k-th distance: lowest rows first
            rows.append(sel.astype(np.uint64) + np.uint64(lo))
            dists.append(d[sel])
        del x                                                   # one chunk in host memory at a time
    out = []
    for rows, dists in kept:
        r, d = np.concatenate(rows), np.concatenate(dists)
        o = np.lexsort((r, d))[:k]
        out.append((r[o], d[o]))
    return out


def assert_exact(hits, ref, k):
    """hits (HIT_DTYPE) are the first k entries of the reference, rows and f64 distance bits."""
    r, d = ref[0][:k], ref[1][:k]
    assert hits["row"].tolist() == r.tolist()
    assert np.array_equal(hits["distance"].view(np.uint64), np.ascontiguousarray(d).view(np.uint64))


def special_rows(rng, n=97):
    """Unit rows with a tied group, duplicates at both ends, zero, NaN, +-inf and extreme rows."""
    rows = unit_rows(rng, n)
    rows[20:34] = rows[50]                       # 15 copies of one row (with row 50 itself)
    rows[0] = rows[n - 1] = rows[n // 2]         # duplicates in the first and the last chunk
    rows[3] = rows[n - 3] = 0.0
    rows[5, 9] = np.nan
    rows[40, 0] = np.inf
    rows[n - 2, 255] = -np.inf
    rows[60] *= np.float32(1e30)
    rows[61] *= np.float32(1e-30)
    return rows


@pytest.mark.parametrize("chunk", [1, 4, 7, 13, 32, 1000])
@pytest.mark.parametrize("k", [1, 5, 15, 16, 40, 97])
def test_exact_topk_equals_the_oracle_scan(chunk, k):
    rng = np.random.default_rng(7 * chunk + k)
    rows = special_rows(rng)
    n = len(rows)
    qs = np.concatenate([unit_rows(rng, 2), rows[[50, n // 2]], np.zeros((1, 256), np.float32),
                         1e-3 * unit_rows(rng, 1)])
    got = exact_topk(lambda lo, m: rows[lo:lo + m], n, qs, k, chunk=chunk)
    for q, (r, d) in zip(qs, got):
        r_exp, d_exp = oracle.search_rows(rows, q, top_k=k)
        assert r.tolist() == r_exp.tolist()
        assert np.array_equal(d.view(np.uint64), d_exp.view(np.uint64))


def test_exact_topk_keeps_a_tied_group_split_across_chunks():
    """The best row has 15 copies spread over rows 20..50; with chunks of 7 rows every chunk boundary
    cuts the group and each chunk's k-th distance is the tied one."""
    rng = np.random.default_rng(3)
    rows = special_rows(rng)
    q = rows[50].copy()
    for k in (3, 8, 15, 16):
        (r, d), = exact_topk(lambda lo, m: rows[lo:lo + m], len(rows), q[None], k, chunk=7)
        r_exp, d_exp = oracle.search_rows(rows, q, top_k=k)
        assert r.tolist() == r_exp.tolist() and np.array_equal(d, d_exp)
    # the copies and the NaN / inf rows all sit at distance 0: row order decides, across the chunks
    assert r.tolist() == [5] + list(range(20, 34)) + [40] and not d.any()


def test_exact_topk_of_a_zero_query_is_every_zero_row_then_row_order():
    rng = np.random.default_rng(4)
    rows = special_rows(rng)
    (r, d), = exact_topk(lambda lo, m: rows[lo:lo + m], len(rows), np.zeros((1, 256), np.float32), 12, chunk=10)
    r_exp, d_exp = oracle.search_rows(rows, np.zeros(256, np.float32), top_k=12)
    assert r.tolist() == r_exp.tolist() and np.array_equal(d, d_exp)
    n = len(rows)
    assert r[:5].tolist() == [3, 5, 40, n - 3, n - 2] and not d[:5].any()   # zero, NaN and inf rows tie at 0


# ------------------------------------------------------------------ device series ---
def set_tier(monkeypatch, tier):
    monkeypatch.setenv("STB_SCAN_TIER", tier)


def sm_count():
    torch = pytest.importorskip("torch")
    return torch.cuda.get_device_properties(0).multi_processor_count


def run_series(ctx, corpus, qs, order, ks):
    """Launch stb_search_topk_dev for qs[order[i]] with top-k ks[i], back to back and each into its own
    slot, as bench.timed_queries does; one synchronisation at the end.  Returns (hits per launch,
    status [launches, 4], co-scan offsets of the last 8 launches)."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda:0")
    q_dev = torch.from_numpy(np.ascontiguousarray(qs, dtype=np.float32)).to(dev)
    hits = torch.zeros((len(order), max(ks), 2), dtype=torch.float64, device=dev)
    status = torch.zeros((len(order), 4), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    for i, (j, k) in enumerate(zip(order, ks)):
        corpus.search_topk_dev(q_dev[j].data_ptr(), k, hits[i].data_ptr(), status[i].data_ptr())
    offs = ctx.coscan_offsets(8)                               # synchronises the library's stream
    d, h = ctx.ticket_check()
    assert d == h
    raw = np.ascontiguousarray(hits.cpu().numpy())
    st = status.cpu().numpy().astype(np.int64)
    out = [raw[i].view(capi.HIT_DTYPE).reshape(-1)[: st[i, 0]] for i in range(len(order))]
    return out, st, offs


@pytest.fixture(scope="module", params=[1_000_000, 10_000_000], ids=["1M", "10M"])
def headline(request, ctx):
    """The benchmark's corpus (bench.fill_shard, one rank), both reduced copies, its 64 queries and their
    exact top-96."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda:0")
    n = request.param
    c, lo, hi = bench.fill_shard(torch, dev, capi, ctx, n, 1, 0)
    assert (lo, hi) == (0, n)
    torch.cuda.empty_cache()
    c.prepare(3)
    qs = bench.gen_queries(64)
    ref = exact_topk(c.read, n, qs, max(WIDE_K))
    yield SimpleNamespace(corpus=c, n=n, qs=qs, ref=ref)
    c.close()
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("tier", ["q8", "h16", "f32"])
def test_headline_device_series_is_exact(ctx, headline, monkeypatch, tier):
    """3 x 64 back-to-back queries, k = 10: every launch proven, on the requested tier, and exact."""
    set_tier(monkeypatch, tier)
    H = headline
    order = list(range(64)) * 3
    hits, st, offs = run_series(ctx, H.corpus, H.qs, order, [10] * len(order))
    assert (st[:, 0] == 10).all() and (st[:, 1] == 1).all(), st[(st[:, 0] != 10) | (st[:, 1] != 1)]
    assert (st[:, 3] >> 16 == TIER_SRC[tier]).all()
    for i, j in enumerate(order):
        assert_exact(hits[i], H.ref[j], 10)
    n_tiles = -(-H.n // TILE_ROWS[tier])
    assert all(o is not None and 0 <= o < n_tiles for o in offs), offs
    assert any(o > 0 for o in offs), offs                     # followers start where their predecessor reads


@pytest.mark.gpu
@pytest.mark.parametrize("tier", ["q8", "h16", "f32"])
def test_headline_search_and_search_many_are_exact(ctx, headline, monkeypatch, tier):
    """The synchronous entry point (bench's e2e) and stb_search_many in groups of 16 (bench's many16)."""
    set_tier(monkeypatch, tier)
    H = headline
    for j, q in enumerate(H.qs):
        assert_exact(H.corpus.search(q, top_k=10), H.ref[j], 10)
    for g in range(0, 64, 16):
        for j, h in enumerate(H.corpus.search_many(H.qs[g:g + 16], top_k=10)):
            assert_exact(h, H.ref[g + j], 10)
    d, h = ctx.ticket_check()
    assert d == h


@pytest.mark.gpu
@pytest.mark.parametrize("tier", ["h16", "f32"])
def test_headline_series_of_wider_k_is_exact(ctx, headline, monkeypatch, tier):
    """k cycles through 17, 40, 64, 96 within one series, so consecutive launches co-scan with
    different list widths."""
    set_tier(monkeypatch, tier)
    H = headline
    order = list(range(64))
    ks = [WIDE_K[i % len(WIDE_K)] for i in order]
    hits, st, offs = run_series(ctx, H.corpus, H.qs, order, ks)
    assert (st[:, 0] == ks).all() and (st[:, 1] == 1).all(), st
    assert (st[:, 3] >> 16 == TIER_SRC[tier]).all()
    for i, (j, k) in enumerate(zip(order, ks)):
        assert_exact(hits[i], H.ref[j], k)
    assert any(o is not None and o > 0 for o in offs), offs


# ------------------------------------------------------------------ adversarial rows ---
ADV_N = 1_500_001          # n % 32 == 1: the last tile of every tier holds one row


def nibble_top_query(rng):
    """A query whose int8 codes all sit at the top of their nibbles (test_gpu_q4)."""
    codes = np.clip(16 * rng.integers(-8, 7, 256) + 15, -127, 127)
    codes[0] = 127
    return (codes / 127.0).astype(np.float32)


@pytest.fixture(scope="module")
def adversarial(ctx):
    """The benchmark's row distribution (0.1 % duplicates, 0.01 % zero rows) with planted rows:
    - three exact copies of query `a`'s best row: at row 0, in the middle and at row n-1;
    - k+6 near-copies of query `b` near the start and its exact match near the end (test_gpu_q4);
    - a duplicated pair whose row is query `dup`."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda:0")
    n = ADV_N
    rows = bench.gen_chunk_torch(torch, dev, 9001, n).cpu().numpy()
    rng = np.random.default_rng(9001)
    qa = unit_rows(rng, 1)[0]
    best = int(np.argmin(oracle.distances(rows, qa)))
    for dst in (0, n // 2, n - 1):
        rows[dst] = rows[best]
    qb = nibble_top_query(rng)
    rows[1000:1016] = (qb[None, :] + 1e-3 * unit_rows(rng, 16)).astype(np.float32)
    rows[n - 1000] = qb
    rows[700_000] = rows[300_000]
    qs = np.stack([qa, unit_rows(rng, 1)[0], qb, rows[300_000], np.zeros(256, np.float32),
                   (qa * np.float32(1e-3)).astype(np.float32), unit_rows(rng, 1)[0]])
    names = ["planted", "random", "near_copies", "dup_row", "zero", "scaled", "random"]
    c = capi.Corpus(ctx, n)
    c.append(rows)
    c.prepare(3)
    ref = exact_topk(lambda lo, m: rows[lo:lo + m], n, qs, 10)
    ties = sorted({0, best, n // 2, n - 1})
    assert ref[0][0][:len(ties)].tolist() == ties                              # the planted ties lead
    assert int(ref[2][0][0]) == n - 1000                                        # the exact match wins
    del rows                                                                    # the corpus lives in HBM from here
    yield SimpleNamespace(corpus=c, n=n, qs=qs, names=names, ref=ref)
    c.close()
    torch.cuda.empty_cache()


def check_series_contract(st, hits, order, ref, k, must_prove):
    """status[1] == 1 means exact; the queries in `must_prove` are proven wherever they fall in the
    series, including after an unproven one."""
    for i, j in enumerate(order):
        if st[i, 1] == 1:
            assert st[i, 0] == k, (i, st[i])
            assert_exact(hits[i], ref[j], k)
        else:
            assert j not in must_prove, (i, j, st[i])


@pytest.mark.gpu
@pytest.mark.parametrize("tier", ["q8", "h16", "f32"])
def test_adversarial_series_is_exact_where_proven(ctx, adversarial, monkeypatch, tier):
    set_tier(monkeypatch, tier)
    A = adversarial
    # query 0 (planted ties) is launched every 4th time, so it starts at several offsets
    cycle = [0, 1, 2, 3, 0, 4, 5, 6]
    order = cycle * 3
    hits, st, offs = run_series(ctx, A.corpus, A.qs, order, [10] * len(order))
    assert (st[:, 3] >> 16 == TIER_SRC[tier]).all()
    random = {j for j, nm in enumerate(A.names) if nm == "random"}
    check_series_contract(st, hits, order, A.ref, 10, must_prove=random)
    planted_offs = {offs[i] for i in range(8) if cycle[i] == 0}
    assert None not in planted_offs and len(planted_offs) == 2, offs
    # the many-query entry point answers every query exactly, an unproven one through stb_search
    for j, h in enumerate(A.corpus.search_many(A.qs, top_k=10)):
        assert_exact(h, A.ref[j], 10)
    d, h = ctx.ticket_check()
    assert d == h


@pytest.fixture(scope="module")
def unnormalisable(ctx):
    """Unit rows with NaN, +-inf and extreme-magnitude rows at row 0, in the middle and at row n-1:
    the q8 and h16 copies refuse them, the f32 tier scans them (their canonical distance is 0 or the
    one of the scaled row)."""
    torch = pytest.importorskip("torch")
    n = 600_001
    rows = bench.gen_chunk_torch(torch, torch.device("cuda:0"), 9002, n).cpu().numpy()
    qs = unit_rows(np.random.default_rng(9002), 4)
    m = n // 2
    rows[0, 17] = np.nan
    rows[1] = qs[0] * np.float32(1e30)            # |row|^2 overflows fp32
    rows[m, 0] = np.inf
    rows[m + 1] = qs[1] * np.float32(1e-30)       # |row|^2 underflows fp32
    rows[m + 2, 200] = -np.inf
    rows[n - 2] = qs[0] * np.float32(3e38)
    rows[n - 1, 255] = np.nan
    qs = np.concatenate([qs, np.zeros((1, 256), np.float32), (qs[2] * np.float32(1e-3))[None]])
    c = capi.Corpus(ctx, n)
    c.append(rows)
    c.prepare(3)
    ref = exact_topk(lambda lo, mm: rows[lo:lo + mm], n, qs, 10)
    assert {0, m, m + 2, n - 1} <= set(ref[2][0].tolist())            # NaN and inf rows: distance 0
    assert {1, n - 2} <= set(ref[0][0].tolist()) and m + 1 in ref[1][0].tolist()   # scaled copies of the query
    del rows
    yield SimpleNamespace(corpus=c, n=n, qs=qs, ref=ref)
    c.close()


@pytest.mark.gpu
def test_unnormalisable_rows_series_runs_on_f32_and_is_exact(ctx, unnormalisable, monkeypatch):
    monkeypatch.delenv("STB_SCAN_TIER", raising=False)
    U = unnormalisable
    order = list(range(len(U.qs))) * 3
    hits, st, offs = run_series(ctx, U.corpus, U.qs, order, [10] * len(order))
    assert (st[:, 3] >> 16 == TIER_SRC["f32"]).all(), st
    check_series_contract(st, hits, order, U.ref, 10, must_prove=set())
    assert any(o is not None and o > 0 for o in offs), offs
    for j, h in enumerate(U.corpus.search_many(U.qs, top_k=10)):
        assert_exact(h, U.ref[j], 10)
    for j, q in enumerate(U.qs):
        assert_exact(U.corpus.search(q, top_k=10), U.ref[j], 10)


# ------------------------------------------------------------------ ticket regimes ---
def regime_tile_counts(sms):
    """Tile counts around the overlapped grid's warp count W = 8 * SMs (one CTA of 8 warps per SM):
    below and above W, around 2W where the single-tile tickets end, and at 2W + 4 / 2W + 5 where the
    first bulk ticket appears (t_bulk = (tiles - min(tiles, 2W)) / 4)."""
    w = 8 * sms
    return [w - 1, w, w + 1, 2 * w - 1, 2 * w, 2 * w + 1, 2 * w + 4, 2 * w + 5]


@pytest.mark.gpu
@pytest.mark.parametrize("last", ["full", "one_row"])
@pytest.mark.parametrize("tier", ["q8", "h16", "f32"])
def test_ticket_regime_sizes_are_exact(ctx, monkeypatch, tier, last):
    """Rotating series on corpora whose tile counts straddle the ticket-regime boundaries.  Exact copies
    of query 0 at row 0, in the middle and at row n-1 tie: the wrap scans row n-1 before row 0, and the
    result must still order them by row."""
    set_tier(monkeypatch, tier)
    T = TILE_ROWS[tier]
    rng = np.random.default_rng(9003 + T + (last == "full"))
    for tiles in regime_tile_counts(sm_count()):
        n = (tiles - 1) * T + (T if last == "full" else 1)
        rows = unit_rows(rng, n)
        qs = np.concatenate([unit_rows(rng, 5), np.zeros((1, 256), np.float32)])
        for dst in (0, n // 2, n - 1):
            rows[dst] = qs[0]
        rows[n - 2] = 0.0
        c = capi.Corpus(ctx, n)
        c.append(rows)
        if PREPARE[tier]:
            c.prepare(PREPARE[tier])
        order = list(range(len(qs))) * 3
        hits, st, offs = run_series(ctx, c, qs, order, [10] * len(order))
        assert (st[:, 3] >> 16 == TIER_SRC[tier]).all(), (tiles, st)
        ref = [oracle.search_rows(rows, q, top_k=10) for q in qs]
        check_series_contract(st, hits, order, ref, 10, must_prove={0, 1, 2, 3, 4})
        assert all(o is not None and 0 <= o < tiles for o in offs), (tiles, offs)
        assert ref[0][0][:3].tolist() == [0, n // 2, n - 1]
        c.close()

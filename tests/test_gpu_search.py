"""GPU parity tests proper: K1 (+K4) through the C ABI vs the CPU oracle.

Bar (BASELINE.md section 5): top-k row indices and order bit-identical to the
oracle; distances within 1e-5 (they are in fact bit-identical: the GPU re-ranks
in the oracle's canonical arithmetic, so == is asserted and 1e-5 is the stated
tolerance)."""
import json
import os

import numpy as np
import pytest

import oracle
from conftest import unit_rows
from semtools_b200 import capi, SearchConfig, Searcher

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-5


def check(hits, rows_exp, d_exp):
    assert hits["row"].tolist() == [int(r) for r in rows_exp]
    assert np.all(np.abs(hits["distance"] - np.asarray(d_exp)) <= TOL)
    assert np.array_equal(hits["distance"], np.asarray(d_exp, dtype=np.float64))


def make_corpus(ctx, rows, row_base=0):
    c = capi.Corpus(ctx, max(len(rows), 1), row_base)
    c.append(rows)
    return c


@pytest.mark.parametrize("n", [1, 2, 7, 8, 9, 31, 32, 33, 255, 1000, 4099, 50_000])
@pytest.mark.parametrize("k", [1, 3, 10])
def test_topk_matches_oracle(ctx, n, k):
    rng = np.random.default_rng(n * 31 + k)
    rows = unit_rows(rng, n)
    q = unit_rows(rng, 1)[0]
    c = make_corpus(ctx, rows)
    r, d = oracle.search_rows(rows, q, top_k=k)
    before = ctx.counters()["fallback_searches"]
    check(c.search(q, top_k=k), r, d)
    assert ctx.counters()["fallback_searches"] == before      # random data: fast path proves it


@pytest.mark.parametrize("k", [16, 17, 40, 41, 64, 96])
def test_topk_candidate_width_classes(ctx, k):
    rng = np.random.default_rng(k)
    rows = unit_rows(rng, 20_000)
    q = unit_rows(rng, 1)[0]
    c = make_corpus(ctx, rows)
    r, d = oracle.search_rows(rows, q, top_k=k)
    check(c.search(q, top_k=k), r, d)


@pytest.mark.parametrize("k", [97, 500, 3000])
def test_topk_large_k_exact_path(ctx, k):
    rng = np.random.default_rng(k)
    rows = unit_rows(rng, 2500)
    q = unit_rows(rng, 1)[0]
    c = make_corpus(ctx, rows)
    r, d = oracle.search_rows(rows, q, top_k=k)
    check(c.search(q, top_k=k), r, d)


def test_config1_1k_lines_top3(ctx):
    """BASELINE configs[0]: 1k lines, top-k=3."""
    rng = np.random.default_rng(0x5E117001)
    rows = unit_rows(rng, 1000)
    q = unit_rows(rng, 1)[0]
    c = make_corpus(ctx, rows)
    r, d = oracle.search_rows(rows, q, top_k=3)
    check(c.search(q, top_k=3), r, d)


def test_golden_cases_through_searcher(ctx):
    z = np.load(os.path.join(G, "search_small.npz"))
    cases = json.load(open(os.path.join(G, "search_small.json")))
    offs = z["doc_offsets"].astype(int)
    s = Searcher(ctx, capi.Corpus(ctx, 1024))
    for d in range(len(offs) - 1):
        lines = [f"doc{d} line{i}" for i in range(offs[d + 1] - offs[d])]
        doc = s.add_document_embeddings(f"doc{d}.txt", lines, z["rows"][offs[d]:offs[d + 1]])
        assert (doc is None) == (len(lines) == 0)       # empty content -> None (mod.rs:57-59)
    names = [f"doc{d}.txt" for d in range(len(offs) - 1)]
    for name, case in cases.items():
        kw = case["kw"]
        res = s.search_documents(z["q"], SearchConfig(kw["n_lines"], kw["top_k"], kw.get("max_distance")))
        assert len(res) == len(case["res"]), name
        for got, (dist, row, doc, idx, start, end) in zip(res, case["res"]):
            assert (got.filename, got.match_line, got.start, got.end) == (names[doc], idx, start, end), name
            assert got.distance == dist, name
            assert got.lines == [f"doc{doc} line{i}" for i in range(start, end)]


def test_duplicates_zero_rows_and_ties(ctx):
    """0.1 % duplicates + zero rows (SURVEY 8d): ties resolve by row order."""
    rng = np.random.default_rng(77)
    rows = unit_rows(rng, 30_000)
    dup_src = rng.integers(0, 30_000, 30)
    dup_dst = rng.integers(0, 30_000, 30)
    rows[dup_dst] = rows[dup_src]
    rows[rng.integers(0, 30_000, 5)] = 0.0
    q = rows[dup_src[0]].copy()
    c = make_corpus(ctx, rows)
    for k in (1, 5, 10, 32):
        r, d = oracle.search_rows(rows, q, top_k=k)
        check(c.search(q, top_k=k), r, d)


def test_heavy_duplication_forces_exact_fallback(ctx):
    """500 exact copies of the best line: the K' candidate list cannot prove
    completeness, the exact collect pass must kick in and still match."""
    rng = np.random.default_rng(5)
    rows = unit_rows(rng, 40_000)
    q = unit_rows(rng, 1)[0]
    where = rng.choice(40_000, 500, replace=False)
    rows[where] = (q + 0.01 * unit_rows(rng, 1)[0]).astype(np.float32)
    c = make_corpus(ctx, rows)
    before = ctx.counters()["fallback_searches"]
    r, d = oracle.search_rows(rows, q, top_k=10)
    check(c.search(q, top_k=10), r, d)
    assert sorted(where)[:10] == [int(x) for x in r]
    assert ctx.counters()["fallback_searches"] == before + 1


def test_zero_query_and_all_zero_corpus(ctx):
    rng = np.random.default_rng(6)
    rows = unit_rows(rng, 300)
    rows[[4, 100, 299]] = 0.0
    zq = np.zeros(256, dtype=np.float32)
    c = make_corpus(ctx, rows)
    r, d = oracle.search_rows(rows, zq, top_k=5)        # zero rows -> 0.0, others 1.0
    check(c.search(zq, top_k=5), r, d)
    assert d[:3].tolist() == [0.0, 0.0, 0.0]
    z = np.zeros((40, 256), dtype=np.float32)
    c2 = make_corpus(ctx, z)
    r, d = oracle.search_rows(z, rows[0], top_k=3)
    check(c2.search(rows[0], top_k=3), r, d)
    assert d.tolist() == [1.0, 1.0, 1.0]


def test_unnormalised_and_scaled_rows(ctx):
    rng = np.random.default_rng(8)
    rows = (unit_rows(rng, 5000) * rng.uniform(1e-3, 1e3, (5000, 1))).astype(np.float32)
    q = (unit_rows(rng, 1)[0] * 37.5).astype(np.float32)
    c = make_corpus(ctx, rows)
    r, d = oracle.search_rows(rows, q, top_k=10)
    check(c.search(q, top_k=10), r, d)


def test_extreme_magnitude_rows_are_forced_candidates(ctx):
    rng = np.random.default_rng(12)
    rows = unit_rows(rng, 3000)
    rows[7] *= np.float32(1e-25)       # fp32 squared norm underflows
    rows[9] *= np.float32(1e22)        # fp32 squared norm overflows
    q = rows[7] * np.float32(1e25)
    c = make_corpus(ctx, rows)
    r, d = oracle.search_rows(rows, q, top_k=4)
    check(c.search(q, top_k=4), r, d)
    assert int(r[0]) == 7


@pytest.mark.parametrize("thr", [0.0, 0.5, 0.8, 0.93, 1.0, 1.0000001, 2.5])
def test_threshold_mode_returns_all_under_threshold(ctx, thr):
    """src/search/mod.rs:88-89 strict <, :115-116 threshold lifts top_k."""
    rng = np.random.default_rng(int(thr * 1000))
    rows = unit_rows(rng, 6000)
    rows[[5, 77]] = 0.0
    q = unit_rows(rng, 1)[0]
    rows[123] = q
    c = make_corpus(ctx, rows)
    r, d = oracle.search_rows(rows, q, top_k=3, max_distance=thr)
    hits = c.search(q, top_k=3, max_distance=thr)
    check(hits, r, d)
    assert np.all(hits["distance"] < thr)


def test_threshold_capacity_protocol(ctx):
    rng = np.random.default_rng(2)
    rows = unit_rows(rng, 3000)
    q = unit_rows(rng, 1)[0]
    c = make_corpus(ctx, rows)
    import ctypes as C
    out = np.zeros(4, dtype=capi.HIT_DTYPE)
    n = C.c_uint64(0)
    rc = capi.lib().stb_search(ctx._h, c._h, q.ctypes.data_as(C.c_void_p), 3, 1, 5.0, 0, None, 0,
                               out.ctypes.data_as(C.c_void_p), 4, C.byref(n))
    assert rc == capi.STB_ERR_CAPACITY and n.value == 3000
    r, d = oracle.search_rows(rows, q, top_k=3, max_distance=5.0)
    assert out["row"].tolist() == [int(x) for x in r[:4]]


def test_store_query_mode_and_row_ranges(ctx):
    """Store::search_line_embeddings semantics (store.rs:481-546): path filter ==
    row ranges; threshold does NOT lift top_k; distance reported as f32."""
    rng = np.random.default_rng(14)
    rows = unit_rows(rng, 9000)
    q = unit_rows(rng, 1)[0]
    c = make_corpus(ctx, rows)
    ranges = [[0, 10], [10, 11], [500, 1500], [4000, 4001], [8990, 9000]]
    for k, thr in [(1, None), (5, None), (20, 0.9), (7, 0.0), (64, None)]:
        r, d32 = oracle.store_search(rows, ranges, q, k, thr)
        hits = c.search(q, top_k=k, max_distance=thr, mode=capi.STB_MODE_STORE_QUERY, row_ranges=ranges)
        assert hits["row"].tolist() == [int(x) for x in r]
        assert np.array_equal(hits["distance"].astype(np.float32), d32)
    assert len(c.search(q, top_k=3, mode=capi.STB_MODE_STORE_QUERY, row_ranges=[])) == 0


def test_many_small_ranges(ctx):
    rng = np.random.default_rng(15)
    rows = unit_rows(rng, 20_000)
    q = unit_rows(rng, 1)[0]
    c = make_corpus(ctx, rows)
    starts = np.sort(rng.choice(np.arange(0, 20_000, 10), 700, replace=False))
    ranges = [[int(s), int(s + rng.integers(1, 10))] for s in starts]
    r, d32 = oracle.store_search(rows, ranges, q, 10)
    hits = c.search(q, top_k=10, mode=capi.STB_MODE_STORE_QUERY, row_ranges=ranges)
    assert hits["row"].tolist() == [int(x) for x in r]


def test_reference_store_fixture(ctx):
    """src/workspace/store.rs:753-757,814-850."""
    s = Searcher(ctx, capi.Corpus(ctx, 16))
    for i, v in enumerate((0.1, 0.5, 0.75)):
        s.add_document_embeddings(f"/test/doc{i + 1}.txt", ["line"], np.full((1, 256), v, dtype=np.float32))
    q = np.full(256, 0.1, dtype=np.float32)
    res = s.search_line_embeddings(q, ["/test/doc1.txt"], 1, 0.1)
    assert len(res) == 1 and res[0].line_number == 0 and res[0].path == "/test/doc1.txt"
    assert res[0].distance < 0.1
    assert s.search_line_embeddings(q, [], 1, 0.1) == []
    assert s.search_line_embeddings(q, ["/test/doc1.txt"], 0, 0.1) == []


def test_sharded_row_base_and_merge(ctx):
    """Row-sharding contract (SURVEY 8e): shard-local searches with row_base, then
    K4 merge == unsharded oracle."""
    rng = np.random.default_rng(16)
    rows = unit_rows(rng, 12_000)
    rows[11_000] = rows[100]                    # cross-shard exact tie
    q = rows[100].copy()
    bounds = [0, 3000, 3001, 9000, 12_000]
    lists = []
    k = 10
    for a, b in zip(bounds[:-1], bounds[1:]):
        c = make_corpus(ctx, rows[a:b], row_base=a)
        h = c.search(q, top_k=k)
        pad = np.zeros(k, dtype=capi.HIT_DTYPE)
        pad["distance"] = np.inf
        pad["row"] = np.uint64(0xFFFFFFFFFFFFFFFF)
        pad[: len(h)] = h
        lists.append(pad)
    merged = ctx.hits_merge(np.stack(lists), k)
    r, d = oracle.search_rows(rows, q, top_k=k)
    check(merged, r, d)
    assert merged["row"][:2].tolist() == [100, 11_000]


def test_device_resident_async_entry_point(ctx):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(17)
    rows = unit_rows(rng, 70_000)
    qs = unit_rows(rng, 4)
    c = make_corpus(ctx, rows)
    dev = torch.device("cuda:0")
    q_dev = torch.from_numpy(qs).to(dev)
    hits = torch.zeros((4, 10, 2), dtype=torch.float64, device=dev)
    status = torch.zeros((4, 4), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    for i in range(4):
        c.search_topk_dev(q_dev[i].data_ptr(), 10, hits[i].data_ptr(), status[i].data_ptr())
    ctx.sync()
    raw = hits.cpu().numpy()
    st = status.cpu().numpy()
    for i in range(4):
        r, d = oracle.search_rows(rows, qs[i], top_k=10)
        got = np.ascontiguousarray(raw[i]).view(capi.HIT_DTYPE).reshape(-1)
        assert st[i, 0] == 10 and st[i, 1] == 1
        check(got, r, d)


def test_error_paths(ctx):
    c = capi.Corpus(ctx, 8)
    q = np.zeros(256, dtype=np.float32)
    assert len(c.search(q, top_k=3)) == 0                       # empty corpus -> empty
    c.append(np.ones((2, 256), dtype=np.float32))
    assert len(c.search(q, top_k=0)) == 0                       # take(0)
    with pytest.raises(capi.StbError):
        c.search(np.zeros(100, dtype=np.float32))               # length mismatch
    with pytest.raises(capi.StbError):
        c.search(q, top_k=1, row_ranges=[[5, 2]])               # malformed range
    with pytest.raises(capi.StbError):
        c.read(1, 5)


def cs_batch(corpus, queries):
    return corpus.search_batch(queries, top_k=10)


def test_nan_and_inf_rows_follow_the_simsimd_rules(ctx):
    """simsimd's `result > 0 ? result : 0` turns a NaN distance into 0.0 (restated in the
    oracle), so NaN/inf rows rank FIRST; the scan must force them into the candidate set."""
    rng = np.random.default_rng(31)
    rows = unit_rows(rng, 4000)
    rows[100, 7] = np.nan
    rows[2000, 0] = np.inf
    rows[3999, 255] = -np.inf
    q = unit_rows(rng, 1)[0]
    c = make_corpus(ctx, rows)
    for k in (2, 5):
        r, d = oracle.search_rows(rows, q, top_k=k)
        check(c.search(q, top_k=k), r, d)
    assert [int(x) for x in r[:3]] == [100, 2000, 3999]


@pytest.mark.parametrize("n", [1_000_000, 10_000_000])
def test_full_size_properties(ctx, n):
    """BASELINE configs[1] (1M) and the metric's corpus size (10M): rows generated on the
    GPU; parity through size-independent properties + an oracle check on a downloaded slice."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev); g.manual_seed(0x5E117002)
    x = torch.randn((n, 256), generator=g, device=dev, dtype=torch.float32)
    x = x / x.norm(dim=1, keepdim=True)
    q = torch.randn(256, generator=g, device=dev, dtype=torch.float32)
    q = (q / q.norm()).cpu().numpy()
    planted = [3, n // 2 - 1, n - 1]
    for j, p in enumerate(planted):                               # plant near-copies of q
        x[p] = torch.from_numpy(q).to(dev) + 0.02 * (j + 1) * x[p]
    x[12345] = x[planted[0]]                                     # exact duplicate -> tie by row
    torch.cuda.synchronize()
    c = capi.Corpus(ctx, n)
    c.append_dev(x.data_ptr(), n)
    hits = c.search(q, top_k=10)
    assert hits["row"][:4].tolist() == [3, 12345, n // 2 - 1, n - 1]
    assert np.all(np.diff(hits["distance"]) >= 0)
    # every reported distance is the canonical one
    rows_h = x[torch.from_numpy(hits["row"].astype(np.int64)).to(dev)].cpu().numpy()
    for h, row in zip(hits, rows_h):
        assert h["distance"] == oracle.cosine(q, row)
    # idempotence and shard-merge consistency: top-k of the whole == merge of halves
    again = c.search(q, top_k=10)
    assert np.array_equal(again, hits)
    lists = []
    for a, b in [(0, n // 2), (n // 2, n)]:
        cs = capi.Corpus(ctx, b - a, row_base=a)
        cs.append_dev(x[a:b].data_ptr(), b - a)
        lists.append(cs.search(q, top_k=10))
        cs.close()
    assert np.array_equal(ctx.hits_merge(np.stack(lists), 10), hits)
    # the batched tensor-core path (K2) must return the same hits as the single-query path
    qs = np.stack([q, q * np.float32(2.0)])      # x2 is exact in binary fp: identical canonical distances
    for got_b in cs_batch(c, qs):
        assert np.array_equal(got_b, hits)
    # oracle on a 200k-row window containing a planted row
    lo, hi = n // 2 - 100_000, n // 2 + 100_000
    win = x[lo:hi].cpu().numpy()
    r, d = oracle.search_rows(win, q, top_k=5)
    cw = capi.Corpus(ctx, hi - lo, row_base=lo)
    cw.append_dev(x[lo:hi].data_ptr(), hi - lo)
    got = cw.search(q, top_k=5)
    check(got, r + lo, d)


@pytest.mark.parametrize("world,k", [(2, 10), (3, 1), (4, 40), (8, 10)])
def test_fused_peer_memory_exchange_single_gpu(world, k):
    """The fused K1 -> exchange -> K4 kernel (stb_search_topk_xchg): `world` contexts
    on cuda:0 stand in for `world` GPUs (same-process peer buffers); every rank must
    end up with the global top-k of the unsharded oracle."""
    torch = pytest.importorskip("torch")
    from semtools_b200.sharded import shard_bounds
    rng = np.random.default_rng(world * 100 + k)
    n = 60_000 + world
    rows = unit_rows(rng, n)
    rows[n - 1] = rows[7]                         # cross-shard exact tie
    qs = np.stack([rows[7], unit_rows(rng, 1)[0], (unit_rows(rng, 1)[0] * 3.5).astype(np.float32)])
    dev = torch.device("cuda:0")
    ctxs = [capi.Context(0) for _ in range(world)]
    corpora, xs = [], []
    for r in range(world):
        lo, hi = shard_bounds(n, world, r)
        c = capi.Corpus(ctxs[r], max(hi - lo, 1), row_base=lo)
        c.append(rows[lo:hi])
        corpora.append(c)
        xs.append(capi.Exchange(ctxs[r], world, r, max(k, 16)))
    for x in xs:
        x.connect_local(xs)
    q_dev = torch.from_numpy(qs).to(dev)
    hits = torch.zeros((world, len(qs), k, 2), dtype=torch.float64, device=dev)
    status = torch.zeros((world, len(qs), 4), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    for rep in range(3):                          # several rounds: slot reuse / sequence numbers
        for qi in range(len(qs)):
            for r in range(world):
                xs[r].search_topk(corpora[r], q_dev[qi].data_ptr(), k, hits[r, qi].data_ptr(),
                                  status[r, qi].data_ptr())
        for c in ctxs:
            c.sync()
        raw, st = hits.cpu().numpy(), status.cpu().numpy()
        for qi in range(len(qs)):
            r_exp, d_exp = oracle.search_rows(rows, qs[qi], top_k=k)
            for r in range(world):
                got = np.ascontiguousarray(raw[r, qi]).view(capi.HIT_DTYPE).reshape(-1)
                assert st[r, qi, 1] == 1 and st[r, qi, 0] == k, (world, r, qi, st[r, qi])
                check(got, r_exp, d_exp)
    # host-buffer form (stb_search_xchg): rank threads would call it concurrently; here rank 0's
    # call is issued last so its spin finds the peers' flags already set
    import threading
    res = [None] * world
    def run(r):
        res[r] = xs[r].search(corpora[r], qs[1], k)
    ths = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in ths:
        t.start()
    for t in ths:
        t.join(timeout=60)
    r_exp, d_exp = oracle.search_rows(rows, qs[1], top_k=k)
    for r in range(world):
        hits_r, ok = res[r]
        assert ok
        check(hits_r, r_exp, d_exp)
    # a zero query ties every row at distance 1.0: no rank can prove its top-k, and the
    # fused kernel must say so on every rank (status[1] == 0) instead of guessing
    zq = torch.zeros(256, dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    for r in range(world):
        xs[r].search_topk(corpora[r], zq.data_ptr(), k, hits[r, 0].data_ptr(), status[r, 0].data_ptr())
    for c in ctxs:
        c.sync()
    assert (status.cpu().numpy()[:, 0, 1] == 0).all()
    for x in xs:
        x.close()
    for c in corpora:
        c.close()
    for c in ctxs:
        c.close()


@pytest.mark.parametrize("n,k", [(200_000, 1000), (50_000, 97), (30_000, 30_000)])
def test_large_k_histogram_path(ctx, n, k):
    """top_k beyond the register lists: histogram pass + collect pass, still bit-identical;
    duplicates, zero rows and forced candidates included."""
    rng = np.random.default_rng(n + k)
    rows = unit_rows(rng, n)
    rows[rng.integers(0, n, 50)] = rows[rng.integers(0, n, 50)]
    rows[[1, n // 3]] = 0.0
    rows[7] *= np.float32(1e-25)
    q = unit_rows(rng, 1)[0]
    c = make_corpus(ctx, rows)
    r, d = oracle.search_rows(rows, q, top_k=k)
    check(c.search(q, top_k=k), r, d)
    ranges = [[10, n // 2], [n // 2 + 5, n - 3]]
    r2, d2 = oracle.store_search(rows, ranges, q, k)
    got = c.search(q, top_k=k, mode=capi.STB_MODE_STORE_QUERY, row_ranges=ranges)
    assert got["row"].tolist() == [int(x) for x in r2]


def test_hits_stored_straight_into_pinned_host_memory_match_the_oracle(ctx):
    """stb_search's scan kernel stores hits + status straight into pinned host memory (no D2H copy);
    what the host reads there is the oracle's answer, ties and the widest register list included."""
    rng = np.random.default_rng(321)
    rows = unit_rows(rng, 50_000)
    rows[777] = rows[5]
    c = capi.Corpus(ctx, 50_000)
    c.append(rows)
    for k in (1, 10, 96):
        for qi in (5, 100, 49_999):
            got = c.search(rows[qi], top_k=k)
            r, d = oracle.search_rows(rows, rows[qi], top_k=k)
            assert got["row"].tolist() == [int(x) for x in r] and np.array_equal(got["distance"], d)


def _ranges_for(rng, n, n_ranges):
    step = max(n // n_ranges, 2)
    starts = np.sort(rng.choice(np.arange(0, n - step, step), min(n_ranges, (n - step) // step), replace=False))
    ranges = [[int(s), int(s + rng.integers(1, step + 1))] for s in starts]
    if n_ranges == 1:
        ranges = [[1000, n - 1000]]
    return ranges


@pytest.mark.parametrize("tier", ["f32", "h16", "q8"])
@pytest.mark.parametrize("n,n_ranges", [(9_000, 5), (20_000, 700), (300_000, 20_000), (70_000, 1)])
def test_row_range_walk_matches_the_oracle_on_every_tier(ctx, monkeypatch, n, n_ranges, tier):
    """Workspace path filter (store.rs:495-523) = row ranges: warps walk blocks of the selected
    rows and step their range index; candidates from the f32 rows, the 16-bit shadow or the int8
    copy -- the answer must be the store query's."""
    rng = np.random.default_rng(n + n_ranges)
    rows = unit_rows(rng, n)
    rows[n // 3] = rows[n // 3 + 1]                                     # a tie inside / across ranges
    q = unit_rows(rng, 1)[0]
    c = make_corpus(ctx, rows)
    c.prepare()
    ranges = _ranges_for(rng, n, n_ranges)
    monkeypatch.setenv("STB_SCAN_TIER", tier)
    for k, thr in [(1, None), (10, None), (64, None), (10, 0.95)]:
        r, d32 = oracle.store_search(rows, ranges, q, k, thr)
        hits = c.search(q, top_k=k, max_distance=thr, mode=capi.STB_MODE_STORE_QUERY, row_ranges=ranges)
        assert hits["row"].tolist() == [int(x) for x in r]
        assert np.array_equal(hits["distance"].astype(np.float32), d32)
    st = c.tier_stats()
    if tier != "f32":
        assert st[tier]["tries"] >= 2, st                              # the reduced-width copy really was scanned


@pytest.mark.parametrize("tier", ["h16", "q8"])
@pytest.mark.parametrize("n", [1, 7, 255, 256, 257, 5_000, 70_001, 300_000])
def test_reduced_width_tiers_match_the_oracle(ctx, monkeypatch, n, tier):
    """K1 candidates from the 16-bit normalised shadow (half the bytes) or the int8 copy (a
    quarter); the re-rank is the same exact f64 pass on the f32 rows, so hits, order and distances
    are the oracle's.  Unprovable queries (zero query, mass ties, k too close to K') are retried on
    the next wider tier / the collect path."""
    rng = np.random.default_rng(1000 + n)
    rows = (unit_rows(rng, n) * rng.uniform(0.2, 5.0, (n, 1))).astype(np.float32)
    if n > 300:
        rows[n // 2] = rows[3]                         # exact duplicate: tie broken by row
        rows[17] = 0.0                                 # zero row
    c = make_corpus(ctx, rows)
    c.prepare()
    queries = [rows[3 % n], unit_rows(rng, 1)[0], unit_rows(rng, 1)[0] * np.float32(1e-3)]
    if n > 300:
        queries.append(np.zeros(256, np.float32))      # zero query: everything ties -> fallback
    monkeypatch.setenv("STB_SCAN_TIER", tier)
    for q in queries:
        for k in (1, 10, 16, 96):
            r, d = oracle.search_rows(rows, q, top_k=k)
            hits = c.search(q, top_k=k)
            assert hits["row"].tolist() == [int(x) for x in r]
            assert np.array_equal(hits["distance"], d)
    st = c.tier_stats()
    assert st[tier]["built_rows"] == n and st[tier]["tries"] > 0, st
    if n >= 5_000:
        assert 3 * st[tier]["proven"] >= st[tier]["tries"], st         # random data: the tier proves most queries itself
    # a corpus with a row that cannot be normalised in fp32: the copies are refused, f32 path answers
    if n >= 5_000:
        rows2 = rows.copy(); rows2[11] *= np.float32(1e-25)
        c2 = make_corpus(ctx, rows2)
        c2.prepare()
        r, d = oracle.search_rows(rows2, queries[1], top_k=5)
        hits = c2.search(queries[1], top_k=5)
        assert hits["row"].tolist() == [int(x) for x in r] and np.array_equal(hits["distance"], d)
        assert c2.tier_stats()[tier]["built_rows"] == 0


def test_q8_upper_bound_really_bounds_the_exact_cosine(ctx, monkeypatch):
    """Adversarial rows for the int8 tier: components just below a rounding boundary, one
    dominant component (large per-row scale), tiny components; queries with one dominant
    component.  Whatever the tier can or cannot prove, the hits must be the oracle's."""
    rng = np.random.default_rng(4242)
    n = 40_000
    rows = unit_rows(rng, n)
    rows[:2000, 0] += np.float32(3.0)                                   # dominant component -> scale ~ 1/127
    rows[2000:4000] = np.round(rows[2000:4000] * 254.0 + 0.49) / np.float32(254.0)   # near half-step boundaries
    rows[4000:4100] *= np.float32(1e-4)
    qs = [unit_rows(rng, 1)[0] for _ in range(3)]
    spike = unit_rows(rng, 1)[0]; spike[5] = 4.0
    qs.append(spike.astype(np.float32))
    qs.append(rows[100].copy())
    c = make_corpus(ctx, rows)
    c.prepare()
    monkeypatch.setenv("STB_SCAN_TIER", "q8")
    for q in qs:
        for k in (1, 5, 16):
            r, d = oracle.search_rows(rows, q, top_k=k)
            hits = c.search(q, top_k=k)
            assert hits["row"].tolist() == [int(x) for x in r]
            assert np.array_equal(hits["distance"], d)


def test_lazy_tier_build_waits_for_the_second_query(ctx, monkeypatch):
    monkeypatch.delenv("STB_SCAN_TIER", raising=False)
    rng = np.random.default_rng(99)
    rows = unit_rows(rng, 40_000)
    q = unit_rows(rng, 1)[0]
    c = make_corpus(ctx, rows)
    r, d = oracle.search_rows(rows, q, top_k=10)
    check(c.search(q, top_k=10), r, d)
    assert c.tier_stats()["q8"]["built_rows"] == 0                      # one-shot query: f32 rows only
    check(c.search(q, top_k=10), r, d)
    st = c.tier_stats()
    assert st["q8"]["built_rows"] == 40_000 and st["q8"]["proven"] == 1, st
    c.append(rows[:10])                                                 # an append leaves a valid PREFIX ...
    assert c.tier_stats()["q8"]["built_rows"] == 40_000
    rows2 = np.concatenate([rows, rows[:10]])
    r2, d2 = oracle.search_rows(rows2, rows[3], top_k=10)               # rows[3] now has an exact duplicate at row 40003
    check(c.search(rows[3], top_k=10), r2, d2)                          # ... which the next query extends (only the new rows are converted)
    st = c.tier_stats()
    assert st["q8"]["built_rows"] == 40_010 and st["q8"]["tries"] == 1, st
    c.clear()                                                           # anything else drops the copies
    assert c.tier_stats()["q8"]["built_rows"] == 0
    small = make_corpus(ctx, rows[:5000])
    small.search(q, top_k=3); small.search(q, top_k=3)
    assert small.tier_stats()["q8"]["built_rows"] == 0                  # below 32768 rows: never lazily


def test_threshold_and_large_k_build_only_the_int8_copy_lazily(ctx, monkeypatch):
    """Threshold mode and top_k beyond the register lists follow the lazy rule of the top-k tiers for
    the int8 copy alone: built on the second search since a change, extended on the first search after
    an append; the 16-bit shadow is never built and no tier counts a try."""
    monkeypatch.delenv("STB_SCAN_TIER", raising=False)
    rng = np.random.default_rng(77)
    rows = unit_rows(rng, 40_000)
    q = unit_rows(rng, 1)[0]
    c = make_corpus(ctx, rows)
    r, d = oracle.search_rows(rows, q, top_k=3, max_distance=0.9)
    check(c.search(q, top_k=3, max_distance=0.9), r, d)
    assert c.tier_stats()["q8"]["built_rows"] == 0                      # first search: f32 rows only
    check(c.search(q, top_k=3, max_distance=0.9), r, d)
    st = c.tier_stats()
    assert st["q8"]["built_rows"] == 40_000 and st["h16"]["built_rows"] == 0, st
    c.append(rows[:10])
    rows2 = np.concatenate([rows, rows[:10]])
    r, d = oracle.search_rows(rows2, q, top_k=200)
    check(c.search(q, top_k=200), r, d)
    st = c.tier_stats()
    assert st["q8"]["built_rows"] == 40_010 and st["h16"]["built_rows"] == 0, st
    assert all(v["tries"] == 0 for v in st.values()), st


def test_search_many_builds_the_int8_copy_only_for_several_queries(ctx, monkeypatch):
    """stb_search_many builds or extends the int8 copy when it holds >= 2 queries (>= 32768 rows); one
    query reads the copies already built, whatever its history, and counts no tier."""
    monkeypatch.delenv("STB_SCAN_TIER", raising=False)
    rng = np.random.default_rng(616)
    rows = unit_rows(rng, 40_000)
    qs = unit_rows(rng, 2)
    c = make_corpus(ctx, rows)
    for _ in range(3):
        got = c.search_many(qs[:1], top_k=10)
        r, d = oracle.search_rows(rows, qs[0], top_k=10)
        check(got[0], r, d)
    st = c.tier_stats()
    assert st["q8"]["built_rows"] == 0 and st["h16"]["built_rows"] == 0, st
    assert all(v["tries"] == 0 for v in st.values()), st
    c.search_many(qs, top_k=10)
    assert c.tier_stats()["q8"]["built_rows"] == 40_000
    c.append(rows[:10])
    rows2 = np.concatenate([rows, rows[:10]])
    got = c.search_many(qs[:1], top_k=10)
    r, d = oracle.search_rows(rows2, qs[0], top_k=10)
    check(got[0], r, d)
    assert c.tier_stats()["q8"]["built_rows"] == 40_000                 # one query: the prefix is not extended
    got = c.search_many(qs, top_k=10)
    for i in range(2):
        r, d = oracle.search_rows(rows2, qs[i], top_k=10)
        check(got[i], r, d)
    assert c.tier_stats()["q8"]["built_rows"] == 40_010


def test_device_entry_point_reads_only_fully_built_copies(ctx, monkeypatch):
    """stb_search_topk_dev never builds or extends a copy: it reads the narrowest one that covers every
    row and that STB_SCAN_TIER allows, which status[3] >> 16 reports (0 f32, 1 h16, 2 q8)."""
    torch = pytest.importorskip("torch")
    monkeypatch.delenv("STB_SCAN_TIER", raising=False)
    rng = np.random.default_rng(4040)
    rows = unit_rows(rng, 40_000)
    q = unit_rows(rng, 1)[0]
    c = make_corpus(ctx, rows)
    dev = torch.device("cuda:0")
    q_dev = torch.from_numpy(q).to(dev)
    hits = torch.zeros((10, 2), dtype=torch.float64, device=dev)
    status = torch.zeros(4, dtype=torch.int32, device=dev)

    def tier_read(rows_now):
        torch.cuda.synchronize()
        c.search_topk_dev(q_dev.data_ptr(), 10, hits.data_ptr(), status.data_ptr())
        ctx.sync()
        st = status.cpu().numpy()
        assert st[1] == 1, st
        r, d = oracle.search_rows(rows_now, q, top_k=10)
        check(np.ascontiguousarray(hits.cpu().numpy()).view(capi.HIT_DTYPE).reshape(-1)[: st[0]], r, d)
        return int(st[3]) >> 16

    assert [tier_read(rows) for _ in range(3)] == [0, 0, 0]            # nothing built: never builds one
    assert c.tier_stats()["q8"]["built_rows"] == 0
    c.prepare()
    assert tier_read(rows) == 2
    c.append(rows[:10])
    rows2 = np.concatenate([rows, rows[:10]])
    assert tier_read(rows2) == 0                                         # a prefix is not extended ...
    st = c.tier_stats()
    assert st["q8"]["built_rows"] == 40_000 and st["h16"]["built_rows"] == 40_000, st
    c.prepare()                                                          # ... until something else does
    assert tier_read(rows2) == 2
    monkeypatch.setenv("STB_SCAN_TIER", "h16")
    assert tier_read(rows2) == 1
    assert all(v["tries"] == 0 for v in c.tier_stats().values())


@pytest.mark.parametrize("tier", ["f32", "h16", "q8"])
def test_ticket_schedule_stays_consistent_and_order_independent(ctx, monkeypatch, tier):
    """The dynamic tile tickets must (a) leave the device counter exactly where the host booked it
    after launches of many shapes, including back-to-back PDL launches, and (b) give the oracle's
    hits whichever warp draws which tile (the co-scan starts each pass at a different tile)."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(2024)
    monkeypatch.setenv("STB_SCAN_TIER", tier)
    dev = torch.device("cuda:0")
    for n in (1, 33, 2_000, 9_473, 150_000, 700_001):
        rows = unit_rows(rng, n)
        c = make_corpus(ctx, rows)
        c.prepare()
        qs = unit_rows(rng, 6)
        q_dev = torch.from_numpy(qs).to(dev)
        hits = torch.zeros((6, 10, 2), dtype=torch.float64, device=dev)
        status = torch.zeros((6, 4), dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        for rep in range(3):
            for i in range(6):                                   # back to back: PDL overlaps tails and scans
                c.search_topk_dev(q_dev[i].data_ptr(), 10, hits[i].data_ptr(), status[i].data_ptr())
        ctx.sync()
        d, h = ctx.ticket_check()
        assert d == h
        raw, st = hits.cpu().numpy(), status.cpu().numpy()
        for i in range(6):
            r, dd = oracle.search_rows(rows, qs[i], top_k=10)
            got = np.ascontiguousarray(raw[i]).view(capi.HIT_DTYPE).reshape(-1)[: st[i, 0]]
            assert st[i, 1] == 1, (n, i, st[i])
            check(got, r, dd)


def test_search_many_equals_search_one_by_one(ctx, monkeypatch):
    """stb_search_many: nq queries enqueued back to back, one synchronisation, hits stored straight
    into pinned host memory; unproven queries (zero query) go through stb_search.  Same hits as
    the oracle for every query, for k inside and beyond the register lists."""
    monkeypatch.delenv("STB_SCAN_TIER", raising=False)
    rng = np.random.default_rng(515)
    rows = unit_rows(rng, 80_000)
    rows[70_000] = rows[9]
    c = make_corpus(ctx, rows)
    qs = unit_rows(rng, 37)
    qs[3] = 0.0                                                     # everything ties: fallback
    qs[5] = rows[9]                                                 # exact duplicate pair -> tie by row
    for k in (1, 10, 96, 200):
        got = c.search_many(qs, top_k=k)
        assert len(got) == len(qs)
        for i, q in enumerate(qs):
            r, d = oracle.search_rows(rows, q, top_k=k)
            check(got[i], r, d)
    assert c.tier_stats()["q8"]["built_rows"] == 80_000             # many queries amortise the int8 copy: built eagerly
    assert len(c.search_many(np.zeros((0, 256), np.float32), top_k=3)) == 0
    d, h = ctx.ticket_check()
    assert d == h


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_threshold_mode_counts_then_padded_payload(world):
    """SURVEY 8e / VERDICT r1 #9: search_documents with max_distance returns ALL lines under the
    threshold (mod.rs:115-116); across shards the ranks exchange counts, then a payload padded to the
    largest count, and merge by (distance,row).  `world` contexts on cuda:0 in threads stand in for
    ranks; the all-gather is a barrier-synchronised list (the NCCL one is exercised by bench.py)."""
    import threading
    from semtools_b200.sharded import ShardedCorpus, shard_bounds
    rng = np.random.default_rng(world)
    n = 50_000 + world
    rows = unit_rows(rng, n)
    rows[n - 1] = rows[11]
    q = rows[11].copy()
    barrier, slots = threading.Barrier(world), [None] * world
    results, errors = [None] * world, []

    def run(rank):
        try:
            c_ctx = capi.Context(0)
            lo, hi = shard_bounds(n, world, rank)
            c = capi.Corpus(c_ctx, hi - lo, row_base=lo)
            c.append(rows[lo:hi])

            def all_gather(local):
                slots[rank] = local.copy()
                barrier.wait(timeout=60)
                out = np.stack(slots)
                barrier.wait(timeout=60)
                return out

            sc = ShardedCorpus(rank, world, lambda qv, k, md, mode: c.search(qv, k, md, mode),
                               lambda lists, k: c_ctx.hits_merge(lists, k) if lists.size <= 4096 else
                               np.sort(lists.reshape(-1)[lists.reshape(-1)["row"] != np.uint64(0xFFFFFFFFFFFFFFFF)], order=["distance", "row"])[:k],
                               all_gather)
            out = {}
            for thr in (0.0, 0.78, 0.9, 1.0000001):
                out[thr] = sc.search(q, 3, max_distance=thr, mode=capi.STB_MODE_SEARCH_DOCUMENTS)
            out["topk"] = sc.search(q, 5, mode=capi.STB_MODE_SEARCH_DOCUMENTS)
            results[rank] = out
            c.close(); c_ctx.close()
        except Exception as e:                                  # noqa: BLE001
            errors.append((rank, repr(e)))
            barrier.abort()

    ths = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in ths:
        t.start()
    for t in ths:
        t.join(timeout=180)
    assert not errors, errors
    for thr in (0.0, 0.78, 0.9, 1.0000001):
        r, d = oracle.search_rows(rows, q, top_k=3, max_distance=thr)
        for rank in range(world):
            got = results[rank][thr]
            assert got["row"].tolist() == [int(x) for x in r], (thr, rank, len(got), len(r))
            assert np.array_equal(got["distance"], d)
    r, d = oracle.search_rows(rows, q, top_k=5)
    for rank in range(world):
        check(results[rank]["topk"], r, d)
    assert len(results[0][0.78]) > 3 and len(results[0][1.0000001]) > 20_000       # really lifted the cap, really > 4096 hits (about half the rows have cosine > 0)


@pytest.mark.parametrize("tier", ["q8", "f32"])
def test_threshold_mode_and_large_k_read_the_narrowest_copy(ctx, monkeypatch, tier):
    """Threshold mode (mod.rs:115-116) and top_k beyond the register lists run collect -> exact -> sort.
    With the int8 copy built the streaming passes read it (upper bounds of the cosine: a superset is
    collected; the large-k floor is proven afterwards) -- a quarter of the bytes, the same hits."""
    monkeypatch.setenv("STB_SCAN_TIER", tier)
    rng = np.random.default_rng(808)
    n = 120_000
    rows = unit_rows(rng, n)
    rows[rng.integers(0, n, 40)] = rows[rng.integers(0, n, 40)]
    rows[[7, n // 2]] = 0.0
    q = unit_rows(rng, 1)[0]
    rows[4321] = q
    c = make_corpus(ctx, rows)
    c.prepare()
    before = ctx.counters()["fallback_searches"]
    for thr in (0.0, 0.5, 0.8, 0.93, 1.0, 1.0000001):
        r, d = oracle.search_rows(rows, q, top_k=3, max_distance=thr)
        check(c.search(q, top_k=3, max_distance=thr), r, d)
    for k in (97, 1000, 5000):
        r, d = oracle.search_rows(rows, q, top_k=k)
        check(c.search(q, top_k=k), r, d)
    ranges = [[10, n // 2], [n // 2 + 5, n - 3]]
    r2, d2 = oracle.store_search(rows, ranges, q, 300)
    got = c.search(q, top_k=300, mode=capi.STB_MODE_STORE_QUERY, row_ranges=ranges)
    assert got["row"].tolist() == [int(x) for x in r2]
    zq = np.zeros(256, np.float32)                                   # zero query: every bound is +inf -> everything collected
    r, d = oracle.search_rows(rows, zq, top_k=3, max_distance=0.5)
    check(c.search(zq, top_k=3, max_distance=0.5), r, d)
    assert ctx.counters()["fallback_searches"] == before             # random data: the q8 floor proves itself

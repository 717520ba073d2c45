"""GPU: K2 (wgmma batched scan).  Stage 1: the tensor-core GEMM itself against a
reference matmul of the rounded 16-bit operands; stage 2 (stb_search_batch): parity with the oracle
per query.  tests/test_gpu_batch_contract.py checks each stage through the device entry point."""
import ctypes as C

import numpy as np
import pytest

import oracle
from conftest import unit_rows
from semtools_b200 import capi

pytestmark = pytest.mark.gpu


def expected_route(n, k):
    """Pipeline v2 (sampled threshold -> emitting epilogue -> exact finish) for k <= 64 on a corpus of at
    least k complete tiles; v1 (maxima/select/finish) otherwise.  These shapes stay far below the shard size
    at which v2's sample overflows (test_gpu_batch_contract.route_rule)."""
    return 2 if k <= 64 and n // 256 >= k else 1


def bf16_round(x):
    """Rounds to the element type of this build's shadow (fp16 by default, bf16 with -DSTB_SHADOW_F16=0)."""
    torch = pytest.importorskip("torch")
    dt = torch.float16 if capi.batch_params()[0] else torch.bfloat16
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(dt).to(torch.float32).numpy()


@pytest.mark.parametrize("nq,n", [(128, 256), (200, 1000), (1, 5), (384, 40_000)])
def test_tcgen05_gemm_matches_bf16_reference(ctx, nq, n):
    rng = np.random.default_rng(nq * 7 + n)
    rows = (unit_rows(rng, n) * rng.uniform(0.5, 2.0, (n, 1))).astype(np.float32)
    rows[n // 2] = 0.0
    q = unit_rows(rng, nq)
    mt, nt = (nq + 127) // 128, (n + 255) // 256
    full = np.zeros((mt * 128, nt * 256), dtype=np.float32)
    sub = np.zeros((mt, nt * 8, 128), dtype=np.float32)
    vp = C.c_void_p
    capi._check(capi.lib().stb_debug_batch_gemm(ctx._h, q.ctypes.data_as(vp), nq, rows.ctypes.data_as(vp), n,
                                                full.ctypes.data_as(vp), sub.ctypes.data_as(vp)))
    norm = np.linalg.norm(rows, axis=1, keepdims=True)
    rn = bf16_round(np.divide(rows, norm, out=np.zeros_like(rows), where=norm > 0))
    qn = bf16_round(q / np.linalg.norm(q, axis=1, keepdims=True))
    ref = qn @ rn.T
    got = full[:nq, :n]
    assert np.max(np.abs(got - ref)) < 2e-3, np.max(np.abs(got - ref))
    # exact cosine is within the rigorous bf16 bound used by the completeness proof
    exact = 1.0 - np.stack([oracle.distances(rows, q[i]) for i in range(min(nq, 4))])
    exact[:, n // 2] = 0.0
    assert np.max(np.abs(got[: exact.shape[0]] - exact)) < capi.batch_params()[1]
    # padding rows / queries are zeros; sub-tile maxima agree with the full matrix
    assert np.all(full[:, n:] == 0.0)
    exp_sub = full.reshape(mt, 128, nt * 8, 32).max(axis=3).transpose(0, 2, 1)
    assert np.array_equal(sub, exp_sub)


def check_batch(res, rows, queries, k):
    for i, q in enumerate(queries):
        r, d = oracle.search_rows(rows, q, top_k=k)
        assert res[i]["row"].tolist() == [int(x) for x in r], i
        assert np.array_equal(res[i]["distance"], d), i


@pytest.mark.parametrize("nq,n,k", [(1, 40, 3), (5, 1000, 10), (130, 70_000, 10), (300, 20_000, 1), (64, 50_000, 40),
                                    (130, 70_000, 80), (64, 50_000, 96), (20, 20_000, 200), (300, 2_000, 16),
                                    (40, 9_000, 64)])
def test_search_batch_matches_oracle(ctx, nq, n, k):
    rng = np.random.default_rng(nq + n + k)
    rows = unit_rows(rng, n)
    queries = unit_rows(rng, nq)
    c = capi.Corpus(ctx, n)
    c.append(rows)
    before = ctx.counters()["fallback_searches"]
    res = c.search_batch(queries, top_k=k)
    assert ctx.batch_last()["route"] == expected_route(n, k)
    check_batch(res, rows, queries, k)
    if n >= 20_000 and k <= 16:
        # 32 sub-tiles are re-scored per query, enough to PROVE top-k for k <= ~16 for nearly every
        # query (the margin is the worst-case bf16 bound 2u+u^2, u = 2^-8; a query whose 32nd
        # sub-tile maximum lies within it of the k-th hit is answered through the single-query
        # path, as is every larger k) -- so fallbacks stay rare, not absent
        assert ctx.counters()["fallback_searches"] - before <= max(2, nq // 8)


@pytest.mark.parametrize("route", ["v2", "v1"])
def test_search_batch_ties_zero_rows_and_unprovable_queries(ctx, route):
    k = 10 if route == "v2" else 80                            # v1: k > 64
    rng = np.random.default_rng(42)
    rows = unit_rows(rng, 30_000)
    rows[rng.integers(0, 30_000, 20)] = rows[rng.integers(0, 30_000, 20)]      # duplicates
    rows[[3, 999, 29_999]] = 0.0
    queries = unit_rows(rng, 40)
    queries[0] = rows[17]                      # exact hit (distance 0)
    queries[1] = 0.0                           # zero query: everything ties at 1.0 -> fallback
    where = rng.choice(30_000, 600, replace=False)
    rows[where] = (queries[2] + 0.005 * unit_rows(rng, 1)[0]).astype(np.float32)   # 600 near-identical best rows
    c = capi.Corpus(ctx, 30_000)
    c.append(rows)
    before = ctx.counters()["fallback_searches"]
    res = c.search_batch(queries, top_k=k)
    assert ctx.batch_last()["route"] == expected_route(30_000, k)
    check_batch(res, rows, queries, k)
    assert ctx.counters()["fallback_searches"] >= before + 2     # queries 1 and 2 cannot be proven


def test_search_batch_refuses_unnormalisable_rows_but_still_answers(ctx):
    rng = np.random.default_rng(43)
    rows = unit_rows(rng, 5000)
    rows[11] *= np.float32(1e-25)
    queries = unit_rows(rng, 3)
    queries[0] = rows[11] * np.float32(1e25)
    c = capi.Corpus(ctx, 5000)
    c.append(rows)
    res = c.search_batch(queries, top_k=5)     # tensor path refused (STATE) -> K1 for every query
    check_batch(res, rows, queries, 5)
    assert int(res[0]["row"][0]) == 11


def test_search_batch_sharded_row_base_and_rebuild_after_append(ctx):
    rng = np.random.default_rng(44)
    rows = unit_rows(rng, 24_000)
    queries = unit_rows(rng, 10)
    c = capi.Corpus(ctx, 16_000, row_base=1_000_000)
    c.append(rows[:12_000])
    c.prepare_batch()
    res = c.search_batch(queries, top_k=5)
    for i, q in enumerate(queries):
        r, d = oracle.search_rows(rows[:12_000], q, top_k=5)
        assert res[i]["row"].tolist() == [int(x) + 1_000_000 for x in r]
    c.append(rows[12_000:])                    # shadow must be rebuilt
    res = c.search_batch(queries, top_k=5)
    for i, q in enumerate(queries):
        r, d = oracle.search_rows(rows, q, top_k=5)
        assert res[i]["row"].tolist() == [int(x) + 1_000_000 for x in r]
        assert np.array_equal(res[i]["distance"], d)


@pytest.mark.parametrize("route", ["v2", "v1"])
def test_sharded_batch_search_merges_to_the_unsharded_answer(ctx, route):
    """Sharded K2: per-shard stb_search_batch_dev + stb_hits_merge_batch_dev (what ranks do
    after all-gathering their nq x k hits) == oracle over the whole corpus."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(77)
    n = 60_000 if route == "v2" else 6_000                     # v1: shards of fewer than k complete tiles
    nq, k = 70, 10
    rows = unit_rows(rng, n)
    rows[n - 1] = rows[5]                       # cross-shard exact tie
    queries = unit_rows(rng, nq)
    queries[0] = rows[5]
    bounds = [0, n // 3, n * 3 // 4, n]
    dev = torch.device("cuda:0")
    q_dev = torch.from_numpy(queries).to(dev)
    world = len(bounds) - 1
    lists = torch.zeros((world, nq, k, 2), dtype=torch.float64, device=dev)
    status = torch.zeros((world, nq, 2), dtype=torch.int32, device=dev)
    out = torch.zeros((nq, k, 2), dtype=torch.float64, device=dev)
    torch.cuda.synchronize()
    shards = []
    for r in range(world):
        c = capi.Corpus(ctx, bounds[r + 1] - bounds[r], row_base=bounds[r])
        c.append(rows[bounds[r]:bounds[r + 1]])
        shards.append(c)
        c.search_batch_dev(q_dev.data_ptr(), nq, k, lists[r].data_ptr(), status[r].data_ptr())
        assert ctx.batch_last()["route"] == expected_route(bounds[r + 1] - bounds[r], k)
    ctx.hits_merge_batch_dev(lists.data_ptr(), world, nq, k, k, out.data_ptr())
    ctx.sync()
    proven = (status[:, :, 1] == 1).all(dim=0).cpu().numpy()      # per query: every shard proved its part
    assert proven.mean() >= 0.8                                    # the rest would go to the single-query path
    got = np.ascontiguousarray(out.cpu().numpy()).view(capi.HIT_DTYPE).reshape(nq, k)
    for i in range(nq):
        if not proven[i]:
            continue
        r, d = oracle.search_rows(rows, queries[i], top_k=k)
        assert got[i]["row"].tolist() == [int(x) for x in r], i
        assert np.array_equal(got[i]["distance"], d), i
    if proven[0]:
        assert got[0]["row"][:2].tolist() == [5, n - 1]


@pytest.mark.parametrize("nq,n,k", [(1, 40, 3), (5, 1000, 10), (130, 70_000, 10), (300, 20_001, 1), (64, 50_000, 40),
                                    (3, 255, 5), (9, 256, 64), (20, 200_000, 10)])
def test_v2_search_batch_matches_oracle_without_fallback(ctx, nq, n, k):
    rng = np.random.default_rng(nq + n + k)
    rows = unit_rows(rng, n)
    queries = unit_rows(rng, nq)
    c = capi.Corpus(ctx, n)
    c.append(rows)
    before = ctx.counters()["fallback_searches"]
    res = c.search_batch(queries, top_k=k)
    check_batch(res, rows, queries, k)
    assert ctx.counters()["fallback_searches"] == before        # v2 proves every k <= 64 unless a capacity overflows
    # v2 samples complete tiles: a corpus of fewer than k of them, (1,40,3), (5,1000,10), (3,255,5) and
    # (9,256,64), is answered by v1, which proves these small shapes too
    assert ctx.batch_last()["route"] == expected_route(n, k)


def test_v2_ties_zero_rows_dense_neighbourhoods(ctx):
    rng = np.random.default_rng(42)
    rows = unit_rows(rng, 30_000)
    rows[rng.integers(0, 30_000, 20)] = rows[rng.integers(0, 30_000, 20)]
    rows[[3, 999, 29_999]] = 0.0
    queries = unit_rows(rng, 40)
    queries[0] = rows[17]
    queries[1] = 0.0                           # zero query: every row ties -> overflow -> K1 fallback
    where = rng.choice(30_000, 600, replace=False)
    rows[where] = (queries[2] + 0.005 * unit_rows(rng, 1)[0]).astype(np.float32)   # 600 identical best rows: 600 <= 1024 re-scores, ~5 per (query, CTA) segment
    where2 = rng.choice(30_000, 3000, replace=False)
    rows[where2] = (queries[3] + 0.004 * unit_rows(rng, 1)[0]).astype(np.float32)  # 3000 > re-score cap -> fallback
    c = capi.Corpus(ctx, 30_000, row_base=5_000_000_000)
    c.append(rows)
    before = ctx.counters()["fallback_searches"]
    res = c.search_batch(queries, top_k=10)
    for i, q in enumerate(queries):
        r, d = oracle.search_rows(rows, q, top_k=10)
        assert res[i]["row"].tolist() == [int(x) + 5_000_000_000 for x in r], i
        assert np.array_equal(res[i]["distance"], d), i
    # queries 1 and 3 overflow a capacity and go to K1 (whose own tie fallback counts again)
    assert ctx.counters()["fallback_searches"] - before >= 2
    # the 600 tied best rows of query 2 fit the in-kernel exact re-score: no fallback
    before = ctx.counters()["fallback_searches"]
    one = c.search_batch(queries[2:3], top_k=10)
    assert np.array_equal(one[0], res[2])
    assert ctx.counters()["fallback_searches"] == before


@pytest.mark.parametrize("world,nq,k", [(3, 24, 10), (2, 9, 1)])
def test_sharded_batch_search_with_fused_peer_memory_exchange(world, nq, k):
    """stb_search_batch_xchg_dev: K2 per shard, then push + merge kernels over peer memory (no NCCL).
    `world` contexts on cuda:0 stand in for the ranks (same-process peer buffers); every rank must end
    up with the unsharded oracle answer for every query, twice in a row (slot parity / sequence reuse).
    (nq stays small here: on ONE GPU a rank's spinning merge CTAs share the SMs with its peers' GEMMs.)"""
    torch = pytest.importorskip("torch")
    from semtools_b200.sharded import shard_bounds
    rng = np.random.default_rng(world * 10 + nq)
    n = 45_000 + world
    rows = unit_rows(rng, n)
    rows[n - 1] = rows[5]                       # cross-shard exact tie
    queries = unit_rows(rng, nq)
    queries[0] = rows[5]
    dev = torch.device("cuda:0")
    ctxs = [capi.Context(0) for _ in range(world)]
    corpora, xs = [], []
    for r in range(world):
        lo, hi = shard_bounds(n, world, r)
        c = capi.Corpus(ctxs[r], hi - lo, row_base=lo)
        c.append(rows[lo:hi])
        c.prepare()
        corpora.append(c)
        xs.append(capi.Exchange(ctxs[r], world, r, max(k, 10), max_nq=32))
    for x in xs:
        x.connect_local(xs)
    q_dev = torch.from_numpy(queries).to(dev)
    out = torch.zeros((world, nq, k, 2), dtype=torch.float64, device=dev)
    status = torch.zeros((world, nq, 2), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    for rep in range(3):
        out.zero_(); status.zero_(); torch.cuda.synchronize()
        for r in range(world):
            xs[r].search_batch_dev(corpora[r], q_dev.data_ptr(), nq, k, out[r].data_ptr(), status[r].data_ptr())
        for c in ctxs:
            c.sync()
        raw, st = out.cpu().numpy(), status.cpu().numpy()
        assert (st[:, :, 1] <= 1).all(), "a rank timed out waiting for a peer"
        for r in range(world):
            assert np.array_equal(st[r], st[0])                      # every rank sees the same proof flags
            got = np.ascontiguousarray(raw[r]).view(capi.HIT_DTYPE).reshape(nq, k)
            for i in range(nq):
                if st[r, i, 1] != 1:
                    continue
                rr, dd = oracle.search_rows(rows, queries[i], top_k=k)
                assert got[i]["row"].tolist() == [int(v) for v in rr], (rep, r, i)
                assert np.array_equal(got[i]["distance"], dd)
        assert st[0, :, 1].mean() >= 0.8
        if st[0, 0, 1] == 1 and k >= 2:
            first = np.ascontiguousarray(raw[0]).view(capi.HIT_DTYPE).reshape(nq, k)[0]
            assert first["row"][:2].tolist() == [5, n - 1]
    for x in xs:
        x.close()
    for c in corpora:
        c.close()
    for c in ctxs:
        c.close()

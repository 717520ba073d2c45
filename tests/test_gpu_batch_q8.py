"""K2 route 7: batched search on the q8 copy and the int8 tensor cores, the route stb_search_batch takes where the
16-bit shadow does not fit in HBM.  stb_debug_batch_q8 runs the host form on that route whatever the shadow's state,
so these tests reach it without filling the card.

- Parity: on a 300k-row device corpus and its host-rows twin, with adversarial rows (duplicates and ties, zero rows,
  rows scaled by 1e-12 and 1e12, negated rows, near-copies of the queries) and a zero and a NaN query, the route's
  hits and counts are bit for bit stb_search's for every top_k, and a subset matches the oracle.
- The route record is 7, and on random unit rows at top_k <= 64 at least 99 % of the queries are proven on the
  tensor cores (stb_search answers at most 1 %), on a 300k-row corpus and on a 13M-row one whose sample (~12.8k
  tiles) needs the threshold kernel's large shared-memory form; on the adversarial corpora only the zero and NaN
  queries and at most 2 % of the others go to stb_search.
- The integer GEMM: every (query, row) dot equals the int64 product of the returned q16 with the int8 codes, u and
  l are K1's q8 bounds bit for bit and bracket the f64 exact cosine.
- A corpus whose q8 copy is unusable never takes the route; the hook leaves a built shadow's bytes unchanged."""
import numpy as np
import pytest

import oracle
from conftest import unit_rows
from semtools_b200 import capi

pytestmark = pytest.mark.gpu

N = 300_000
TOPKS = (1, 10, 16, 64, 65, 100)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def same_hits(a, b):
    assert len(a) == len(b)
    assert np.array_equal(bits(a), bits(b))


def adversarial_rows(rng, n):
    rows = unit_rows(rng, n)
    rows[100:110] = rows[5]                                 # exact duplicates: ties at every distance
    rows[200:204] = 0.0                                     # zero rows
    rows[300:310] *= np.float32(1e-12)
    rows[400:410] *= np.float32(1e12)
    rows[500:510] = -rows[500:510]
    return np.ascontiguousarray(rows)


def queries_for(rng, rows, nq):
    q = unit_rows(rng, nq)
    near = rows[[5, 1234, 400, 300]] + np.float32(1e-3) * unit_rows(rng, 4)
    special = np.zeros((2, 256), np.float32)
    special[1, 7] = np.nan                                  # a zero query and a NaN query
    return np.ascontiguousarray(np.concatenate([q, near, -rows[[501]], special]).astype(np.float32))


@pytest.fixture(scope="module")
def data():
    rng = np.random.default_rng(20261017)
    rows = adversarial_rows(rng, N)
    return rows, queries_for(rng, rows, 140)


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


def test_parity_with_stb_search(ctx, data, pair):
    rows, queries = data
    for c in pair:
        for k in TOPKS:
            fb = ctx.counters()["fallback_searches"]
            got = c.debug_batch_q8(queries, k)
            fell_back = ctx.counters()["fallback_searches"] - fb
            info = ctx.batch_last()
            assert info["route"] == 7 and info["nq"] == len(queries)
            if k <= 64:
                assert info["n_sample"] > 0 and info["n_seg"] > 0
                assert fell_back <= 2 + len(queries) // 50, (k, fell_back)   # the zero and NaN queries, and few others
            else:
                # top_k > 64: stb_search answers all (the counter also counts stb_search's own internal retries)
                assert fell_back >= len(queries)
            for q, g in zip(queries, got):
                same_hits(g, c.search(q, k))
    host = pair[1]
    for i in (0, 140, 141):
        r, d = oracle.search_rows(rows, queries[i], top_k=10)
        h = host.debug_batch_q8(queries[[i]], 10)[0]
        assert np.array_equal(h["row"], np.asarray(r, dtype=np.uint64)) and np.array_equal(h["distance"], d)


def check_proven(ctx, c, queries, topks):
    for k in topks:
        before = ctx.counters()["fallback_searches"]
        got = c.debug_batch_q8(queries, k)
        info = ctx.batch_last()
        fell_back = ctx.counters()["fallback_searches"] - before
        assert info["route"] == 7 and info["stride"] >= 1, info
        assert fell_back <= len(queries) // 100, (k, fell_back, info)
        assert np.all(info["cand_cnt"] <= info["seg_cap"])
        for q, g in zip(queries, got):
            same_hits(g, c.search(q, k))


def test_random_rows_are_proven_on_the_tensor_cores(ctx):
    rng = np.random.default_rng(7)
    c = capi.Corpus(ctx, N)
    c.append(unit_rows(rng, N))
    check_proven(ctx, c, unit_rows(rng, 512), (1, 10, 16, 64))
    c.close()


def test_a_sample_past_48k_of_shared_memory(ctx):
    """13M rows at top_k = 64: the plan samples ~12.8k tiles, whose maxima take more than the 48 KiB of shared memory
    a kernel gets by default"""
    import torch
    n = 13_000_000
    n_sample, stride, fits = capi.batch_q8_plan(torch.cuda.get_device_properties(0).multi_processor_count, n, 64)
    assert fits and n_sample * 4 > 48 * 1024
    c = capi.Corpus(ctx, n)
    g = torch.Generator(device="cuda").manual_seed(11)
    for r0 in range(0, n, 1 << 20):
        m = min(1 << 20, n - r0)
        x = torch.randn((m, 256), generator=g, device="cuda", dtype=torch.float32)
        x /= x.norm(dim=1, keepdim=True)
        torch.cuda.synchronize()
        c.append_dev(x.data_ptr(), m)
        ctx.sync()
        del x
    torch.cuda.empty_cache()
    check_proven(ctx, c, unit_rows(np.random.default_rng(12), 256), (16, 64))
    assert ctx.batch_last()["n_sample"] == n_sample      # the top_k = 64 batch ran on the large sample
    c.close()


def test_integer_gemm_and_bounds(ctx, data):
    rows, queries = data
    sub = np.ascontiguousarray(rows[:5000])
    c = capi.Corpus(ctx, len(sub))
    c.append(sub)
    q16, dot, u, l = c.debug_batch_q8_gemm(queries)
    codes = c.debug_copy(capi.STB_COPY_Q8_CODES)[0].view(np.int8).reshape(len(sub), 256)
    assert np.array_equal(dot.astype(np.int64), q16.astype(np.int64) @ codes.astype(np.int64).T)
    assert np.all(np.abs(q16.astype(np.int32)) <= 32639)
    usable = [i for i in range(len(queries)) if np.all(np.isfinite(queries[i])) and np.any(queries[i] != 0)]
    assert not np.any(q16[-2:])                             # zero and NaN queries quantise to zero
    qn = queries[usable].astype(np.float64)
    qn /= np.linalg.norm(qn, axis=1, keepdims=True)
    rn = sub.astype(np.float64)
    norms = np.linalg.norm(rn, axis=1, keepdims=True)
    rn = np.divide(rn, norms, out=np.zeros_like(rn), where=norms > 0)
    cos = qn @ rn.T
    assert np.all(cos <= u[usable].astype(np.float64) + 1e-5)
    assert np.all(l[usable].astype(np.float64) <= cos + 1e-5)
    for i in usable[:4] + usable[-3:]:                      # K1's q8 bounds, bit for bit
        k1_u = c.debug_scan_scores(queries[i], "q8")[0]
        assert np.array_equal(bits(k1_u), bits(u[i]))
        k1_l = c.debug_q4_scan(queries[i], 4)["l8"]
        assert np.array_equal(bits(k1_l), bits(l[i]))
    c.close()


def test_unusable_q8_copy_never_takes_the_route(ctx, data):
    rows, queries = data
    bad = rows[:120_000].copy()
    bad[321] = unit_rows(np.random.default_rng(3), 1)[0] * np.float32(1e-20)
    small = capi.Corpus(ctx, 4096)
    small.append(rows[:4096])
    small.search_batch(queries[:8], 10)
    before = ctx.batch_last()
    for c in (capi.Corpus(ctx, len(bad)), capi.Corpus.in_host_memory(ctx, 1024)):
        c.append(bad)
        fb = ctx.counters()["fallback_searches"]
        got = c.debug_batch_q8(queries[:20], 10)
        assert ctx.counters()["fallback_searches"] - fb == 20      # stb_search answered every query
        after = ctx.batch_last()
        assert (after["route"], after["nq"]) == (before["route"], before["nq"]) != (7, 20)
        assert c.tier_stats()["q8"]["built_rows"] == 0
        for q, g in zip(queries[:20], got):
            same_hits(g, c.search(q, 10))
        c.close()
    small.close()


def test_hook_leaves_a_built_shadow_unchanged(ctx, data):
    rows, queries = data
    c = capi.Corpus(ctx, 20_000)
    c.append(rows[:20_000])
    c.prepare_batch()
    shadow = bits(c.debug_copy(capi.STB_COPY_H16_TILES)[0]).copy()
    got = c.debug_batch_q8(queries, 10)
    assert ctx.batch_last()["route"] == 7
    assert np.array_equal(bits(c.debug_copy(capi.STB_COPY_H16_TILES)[0]), shadow)
    for a, b in zip(got, c.search_batch(queries, 10)):
        same_hits(a, b)
    c.close()

"""GPU: stb_search_batch_subsets, the workspace query for a batch in which every query names its own subset.

Every query of a call must equal, bit for bit, what stb_search in store-query mode returns for it alone with its
own ranges (hits, order, count, the padded tail), and the oracle's store search on a small corpus.  Route 6 is
checked against its own approximate scores, as tests/test_gpu_batch_filtered.py checks route 3: from
stb_debug_batch_gemm's score matrix restricted to each query's eligible rows the tests predict every threshold,
every query's total emission count and which groups run on the tensor cores.
"""
import ctypes as C

import numpy as np
import pytest

import oracle
from conftest import unit_rows
from semtools_b200 import capi
from test_gpu_batch_filtered import (F2_KEYS, F2_RESCORE, SEG_CAP, TILE, debug_scores, doc_ranges, eligible_mask,
                                     listed_tiles, local_ranges, route_rule)

pytestmark = pytest.mark.gpu

NO_ROW = 0xFFFFFFFFFFFFFFFF


@pytest.fixture(scope="module")
def sm_count():
    torch = pytest.importorskip("torch")
    return torch.cuda.get_device_properties(0).multi_processor_count


def new_corpus(ctx, rows, row_base=0):
    c = capi.Corpus(ctx, max(len(rows), 1), row_base=row_base)
    c.append(rows)
    return c


def k1(c, q, k, cap, ranges):
    return c.search(q, top_k=k, max_distance=cap, mode=capi.STB_MODE_STORE_QUERY,
                    row_ranges=np.asarray(ranges, np.uint64).reshape(-1, 2))


def same(a, b, where=""):
    assert a["row"].tolist() == b["row"].tolist(), where
    assert np.array_equal(a["distance"].view(np.uint64), b["distance"].view(np.uint64)), where


def packed(ranges_per_query):
    parts = [np.asarray(r, np.uint64).reshape(-1, 2) for r in ranges_per_query]
    offs = np.zeros(len(parts) + 1, np.uint64)
    offs[1:] = np.cumsum([len(p) for p in parts])
    rr = np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros((0, 2), np.uint64), np.uint64)
    return offs, (rr if len(rr) else np.zeros((1, 2), np.uint64))


def raw_call(ctx, c, queries, k, cap, offs, rr, out=None, cnt=None):
    """The C entry point on preset output buffers (None: a NULL pointer): (status, hits [nq][k], counts [nq])."""
    queries = np.ascontiguousarray(queries, dtype=np.float32)
    nq = len(queries)
    out = np.zeros((nq, max(k, 1)), dtype=capi.HIT_DTYPE) if out is None else out
    cnt = np.zeros(max(nq, 1), dtype=np.uint32) if cnt is None else cnt
    vp = C.c_void_p
    ptr = (lambda a: None if a is None else a.ctypes.data_as(vp))
    rc = capi.lib().stb_search_batch_subsets(ctx._h, c._h, ptr(queries), nq, k, int(cap is not None), float(cap or 0.0),
                                             ptr(offs), ptr(rr), ptr(out), ptr(cnt))
    return rc, out, cnt


def check_batch(ctx, c, queries, k, cap, subsets, where=""):
    """The batch against per-query stb_search with each query's own ranges, the padded tail included."""
    offs, rr = packed(subsets)
    rc, out, cnt = raw_call(ctx, c, queries, k, cap, offs, rr)
    assert rc == 0, capi.lib().stb_last_error()
    for i, q in enumerate(queries):
        got = out[i, : cnt[i]]
        if len(np.asarray(subsets[i]).reshape(-1, 2)) == 0:
            assert cnt[i] == 0, where                             # the empty subset
        else:
            same(got, k1(c, q, k, cap, subsets[i]), f"{where} k={k} cap={cap} query {i}")
        if k:
            assert np.all(out[i, cnt[i]:]["distance"] == np.inf) and np.all(out[i, cnt[i]:]["row"] == NO_ROW), where
    return [out[i, : cnt[i]] for i in range(len(queries))]


# ------------------------------------------------------------------ batches of subsets ---
def deal(rng, sizes, subsets):
    """Queries dealt to subsets unevenly and interleaved: query i uses subsets[owner[i]]."""
    owner = np.repeat(np.arange(len(sizes)), sizes)
    rng.shuffle(owner)
    return owner, [subsets[g] for g in owner]


def special_subsets(rng, n, row_base=0):
    """Overlapping and disjoint document subsets, the whole shard, a split of one subset that clips to the same
    list, a subset outside the shard, a ragged last tile, and the empty subset."""
    a = doc_ranges(rng, n, 0.3, row_base)
    b = doc_ranges(rng, n, 0.05, row_base)
    whole = np.array([[row_base, row_base + n]], np.uint64)
    a_split = np.concatenate([a, [[row_base + n + 10, row_base + n + 20]]]).astype(np.uint64)   # clips to `a`
    outside = np.array([[row_base + n + 5, row_base + n + 500]], np.uint64)
    tail = np.array([[row_base + n - 100, row_base + n + 7]], np.uint64)                        # the ragged last tile
    first = np.array([[row_base, row_base + 40 * TILE]], np.uint64)
    over = np.array([[row_base + 30 * TILE, row_base + 90 * TILE]], np.uint64)                 # overlaps `first`
    return [a, b, whole, a_split, outside, tail, first, over, np.zeros((0, 2), np.uint64)]


@pytest.mark.parametrize("n,G", [(70_000, 1), (70_000, 2), (70_000, 7), (70_000, 64), (300_000, 7), (300_000, 64)])
def test_parity_with_single_query_search(ctx, sm_count, n, G):
    rng = np.random.default_rng(n + G)
    rows = unit_rows(rng, n)
    c = new_corpus(ctx, rows)
    if G == 1:
        subsets, sizes = [doc_ranges(rng, n, 0.25)], [300]
    else:
        subsets = special_subsets(rng, n)
        subsets += [doc_ranges(rng, n, float(f)) for f in rng.choice([0.01, 0.05, 0.25], max(G - len(subsets), 0))]
        subsets = subsets[:G]
        sizes = rng.integers(1, 20, G)
        sizes[0] = 300                                            # a group over three query tiles' halves
        sizes[min(1, G - 1)] = 65
    owner, per_query = deal(rng, sizes, subsets)
    queries = unit_rows(rng, len(owner))
    for i in range(0, len(owner), 5):                             # eligible copies: a sure hit per group
        elig = np.flatnonzero(eligible_mask(per_query[i], n))
        if len(elig):
            queries[i] = rows[elig[len(elig) // 2]]
    for k, cap in [(10, None), (10, 0.9), (1, None), (64, None)]:
        res = check_batch(ctx, c, queries, k, cap, per_query, where=f"n={n} G={G}")
        assert ctx.batch_last()["route"] == (3 if G == 1 else 6), ctx.batch_last()
    for i in rng.choice(len(owner), 6, replace=False):            # the oracle on the clipped ranges
        loc = local_ranges(per_query[i], n)
        got = c.search_batch_subsets(queries[i:i + 1], [per_query[i]], top_k=10)[0]
        if len(loc) == 0:
            assert len(got) == 0
            continue
        r, d32 = oracle.store_search(rows, loc, queries[i], 10)
        assert got["row"].tolist() == [int(x) for x in r]
        assert np.array_equal(got["distance"].astype(np.float32), d32)
    assert len(res) == len(queries)


@pytest.mark.parametrize("k", [0, 1, 10, 64, 65])
def test_top_k_and_caps(ctx, k):
    rng = np.random.default_rng(100 + k)
    n = 70_000 + 77                                               # a ragged last tile
    rows = unit_rows(rng, n)
    c = new_corpus(ctx, rows)
    subsets = special_subsets(rng, n)
    owner, per_query = deal(rng, [3, 70, 1, 5, 2, 9, 4, 6, 2], subsets)
    queries = unit_rows(rng, len(owner))
    queries[0] = rows[n - 1]
    for cap in (None, 0.0, 0.5, 1e9, float("nan"), float("inf")):
        check_batch(ctx, c, queries, k, cap, per_query, where=f"k={k}")
    info = ctx.batch_last()
    assert info["route"] == 6
    if k == 0:
        assert info["groups"] == 0 and info["k1"] == 0
    if k == 65:                                                   # all K1: v2 stops at 64
        assert info["groups"] == 0 and info["k1"] == sum(len(local_ranges(r, n)) > 0 for r in per_query)


def test_shard_with_row_base_and_the_whole_shard(ctx):
    rng = np.random.default_rng(17)
    row_base = 5_000_000_000
    n = 120 * TILE + 33
    rows = unit_rows(rng, n)
    c = new_corpus(ctx, rows, row_base=row_base)
    subsets = special_subsets(rng, n, row_base)
    subsets.append(np.array([[row_base - 5000, row_base + 700], [row_base + n - 50, row_base + n + 9]], np.uint64))
    owner, per_query = deal(rng, [4, 2, 9, 1, 3, 2, 5, 1, 2, 6], subsets)
    queries = unit_rows(rng, len(owner))
    queries[1] = rows[100]
    for k in (1, 10, 64):
        check_batch(ctx, c, queries, k, None, per_query, where="row_base")
        assert ctx.batch_last()["route"] == 6


# ------------------------------------------------------------------ the route rule, restated ---
def predict(ctx, sm, rows, queries, per_query, k):
    """Route 6 from the approximate scores: per query its threshold and total emission count, the tensor
    groups and the queries K1 answers (those of groups whose plan does not fit, and unproven ones)."""
    _, eps = capi.batch_params()
    two_eps = np.float32(2.0) * np.float32(eps)
    n = len(rows)
    A = debug_scores(ctx, queries, rows)
    keys = [local_ranges(r, n).tobytes() for r in per_query]
    groups = {}
    for i, key in enumerate(keys):
        if len(np.frombuffer(key, np.uint64)):
            groups.setdefault(key, []).append(i)
    thr = np.full(len(queries), np.inf, np.float32)
    total = np.zeros(len(queries), np.int64)
    k1_queries, tensor_groups = set(), 0
    for members in groups.values():
        rr = per_query[members[0]]
        listed = listed_tiles(rr, n)
        plan = route_rule(len(listed), k, sm)
        if plan["route"] != 3:
            k1_queries |= set(members)
            continue
        tensor_groups += 1
        elig = eligible_mask(rr, n)
        ns, stride = plan["n_sample"], plan["stride"]
        pad = np.full(-(-n // TILE) * TILE - n, -np.inf, np.float32)
        for i in members:
            a = np.concatenate([np.where(elig, A[i], -np.inf).astype(np.float32), pad]).reshape(-1, TILE)
            s_k = np.sort(a[listed[np.arange(ns) * stride]].max(axis=1))[ns - k]
            thr[i] = np.float32(s_k) - two_eps
            sc = A[i][elig & (A[i] >= thr[i])]
            total[i] = len(sc)
            m2 = len(sc)
            if len(sc) >= k:
                m2 = int(np.count_nonzero(sc >= np.float32(np.sort(sc)[len(sc) - k]) - two_eps))
            if len(sc) > F2_KEYS or m2 > F2_RESCORE:
                k1_queries.add(i)
    return thr, total, tensor_groups, k1_queries


@pytest.mark.parametrize("n,k", [(70_000, 10), (140_000 + 5, 16), (300 * TILE + 7, 1), (64 * TILE + 200, 64)])
def test_route_contract(ctx, sm_count, n, k):
    rng = np.random.default_rng(n + k)
    rows = unit_rows(rng, n)
    c = new_corpus(ctx, rows)
    subsets = [doc_ranges(rng, n, f) for f in (0.5, 0.25, 0.05, 0.01)]
    subsets.append(np.array([[3 * TILE + 5, 3 * TILE + 60]], np.uint64))        # one listed tile: K1 for k > 1
    subsets.append(np.array([[0, n]], np.uint64))
    owner, per_query = deal(rng, [130, 7, 64, 1, 3, 40], subsets)
    queries = unit_rows(rng, len(owner))
    queries[0] = rows[n - 1]
    thr, total, tg, k1_q = predict(ctx, sm_count, rows, queries, per_query, k)
    before = ctx.counters()["fallback_searches"]
    c.search_batch_subsets(queries, per_query, top_k=k)
    fell = ctx.counters()["fallback_searches"] - before
    info = ctx.batch_last()
    assert info["route"] == 6 and info["nq"] == len(queries) and info["groups"] == tg, info
    assert info["n_seg"] == min(len(set().union(*[set(listed_tiles(r, n).tolist()) for r in subsets
                                                  if route_rule(len(listed_tiles(r, n)), k, sm_count)["route"] == 3])),
                                sm_count) and info["seg_cap"] == SEG_CAP
    assert np.array_equal(info["thr"].view(np.uint32), thr.view(np.uint32)), np.flatnonzero(info["thr"] != thr)[:8]
    assert np.array_equal(info["cand_cnt"].astype(np.int64).sum(axis=1), total), \
        np.flatnonzero(info["cand_cnt"].sum(axis=1) != total)[:8]
    overflow = {i for i in range(len(queries)) if (info["cand_cnt"][i] > SEG_CAP).any()}
    # stb_search may count one more fallback of its own per query
    assert len(k1_q) <= info["k1"] <= len(k1_q | overflow) and info["k1"] <= fell <= 2 * info["k1"], \
        (info, len(k1_q), len(overflow), fell)
    if k <= 16:
        assert info["k1"] == len(k1_q)
    check_batch(ctx, c, queries, k, None, per_query, where="contract")


def test_one_group_is_the_filtered_call(ctx, sm_count):
    """Every query with the same clipped list (given with different splits): route 3, and stb_debug_batch_last
    gives what stb_search_batch_filtered gives on the same inputs."""
    rng = np.random.default_rng(9)
    n = 90_000
    rows = unit_rows(rng, n)
    c = new_corpus(ctx, rows)
    docs = doc_ranges(rng, n, 0.2)
    per_query = [docs if i % 2 else np.concatenate([docs, [[n + 1, n + 3]]]).astype(np.uint64) for i in range(150)]
    queries = unit_rows(rng, 150)
    got = c.search_batch_subsets(queries, per_query, top_k=10)
    a = ctx.batch_last()
    exp = c.search_batch_filtered(queries, docs, top_k=10)
    b = ctx.batch_last()
    assert a["route"] == 3
    for key in ("route", "nq", "n_sample", "stride", "n_seg", "seg_cap"):
        assert a[key] == b[key], key
    assert np.array_equal(a["thr"].view(np.uint32), b["thr"].view(np.uint32))
    assert np.array_equal(a["cand_cnt"], b["cand_cnt"])
    for x, y in zip(got, exp):
        same(x, y)


# ------------------------------------------------------------------ refusals ---
def test_refusals_write_nothing_and_launch_nothing(ctx):
    rng = np.random.default_rng(5)
    rows = unit_rows(rng, 5000)
    c = new_corpus(ctx, rows)
    q = unit_rows(rng, 3)
    good = [np.array([[10, 2000]], np.uint64), np.array([[0, 40]], np.uint64), np.array([[300, 4000]], np.uint64)]
    offs, rr = packed(good)

    def refused(offs, rr, status):
        out0 = np.zeros((3, 10), dtype=capi.HIT_DTYPE)
        out0["distance"] = 0.125
        out0["row"] = 42
        cnt0 = np.full(3, 7, np.uint32)
        before = ctx.counters()["kernel_launches"]
        rc, out, cnt = raw_call(ctx, c, q, 10, None, offs, rr, out=out0.copy(), cnt=cnt0.copy())
        assert rc == status, capi.lib().stb_last_error()
        assert ctx.counters()["kernel_launches"] == before
        assert np.array_equal(out, out0) and np.array_equal(cnt, cnt0)

    refused(np.array([1, 1, 2, 3], np.uint64), rr, capi.STB_ERR_ARG)               # offsets[0] != 0
    refused(np.array([0, 2, 1, 3], np.uint64), rr, capi.STB_ERR_ARG)               # decreasing
    vp = C.c_void_p
    assert capi.lib().stb_search_batch_subsets(ctx._h, c._h, q.ctypes.data_as(vp), 3, 10, 0, 0.0, offs.ctypes.data_as(vp),
                                               None, None, None) == capi.STB_ERR_ARG
    cnt0 = np.full(3, 7, np.uint32)
    out0 = np.zeros((3, 10), dtype=capi.HIT_DTYPE)
    rc = capi.lib().stb_search_batch_subsets(ctx._h, c._h, q.ctypes.data_as(vp), 3, 10, 0, 0.0, offs.ctypes.data_as(vp),
                                             None, out0.ctypes.data_as(vp), cnt0.ctypes.data_as(vp))
    assert rc == capi.STB_ERR_ARG and cnt0.tolist() == [7, 7, 7]                   # row_ranges NULL, ranges > 0
    rc = capi.lib().stb_search_batch_subsets(ctx._h, c._h, q.ctypes.data_as(vp), 3, 10, 0, 0.0, None,
                                             rr.ctypes.data_as(vp), out0.ctypes.data_as(vp), cnt0.ctypes.data_as(vp))
    assert rc == capi.STB_ERR_ARG and cnt0.tolist() == [7, 7, 7]                   # range_offsets NULL
    assert capi.lib().stb_search_batch_subsets(ctx._h, c._h, q.ctypes.data_as(vp), 3, 10, 0, 0.0, offs.ctypes.data_as(vp),
                                               rr.ctypes.data_as(vp), out0.ctypes.data_as(vp), None) == capi.STB_ERR_ARG
    for bad in ([[100, 50]], [[0, 100], [50, 200]], [[300, 400], [0, 10]]):        # one query's ranges refused
        bad = np.array(bad, np.uint64)
        exp = capi.lib().stb_search(ctx._h, c._h, q[0].ctypes.data_as(vp), 10, 0, 0.0, capi.STB_MODE_STORE_QUERY,
                                    bad.ctypes.data_as(vp), len(bad), None, 0, C.byref(C.c_uint64(0)))
        assert exp == capi.STB_ERR_RANGE
        o, r = packed([good[0], bad, good[2]])
        refused(o, r, exp)
    # nq = 0 is a no-op, top_k = 0 sets every count to 0, zero ranges everywhere: no hits and a NULL row_ranges
    rc, _, _ = raw_call(ctx, c, q[:0], 10, None, np.zeros(1, np.uint64), None)
    assert rc == 0
    rc, _, cnt = raw_call(ctx, c, q, 0, None, offs, rr, cnt=np.full(3, 9, np.uint32))
    assert rc == 0 and cnt.tolist() == [0, 0, 0]
    rc, out, cnt = raw_call(ctx, c, q, 10, None, np.zeros(4, np.uint64), None, cnt=np.full(3, 9, np.uint32))
    assert rc == 0 and cnt.tolist() == [0, 0, 0] and np.all(out["row"] == NO_ROW) and np.all(out["distance"] == np.inf)


# ------------------------------------------------------------------ inputs K1 must answer ---
def test_bad_queries_and_the_zero_query(ctx):
    rng = np.random.default_rng(31)
    n = 70_000
    rows = unit_rows(rng, n)
    c = new_corpus(ctx, rows)
    queries = list(unit_rows(rng, 10))
    nan = unit_rows(rng, 1)[0]; nan[7] = np.nan
    inf = unit_rows(rng, 1)[0]; inf[3] = np.inf
    queries += [np.zeros(256, np.float32), nan, inf, rows[11] * np.float32(1e-25), rows[12] * np.float32(1e20),
                rows[13] * np.float32(1e-20)]
    queries = np.ascontiguousarray(np.stack(queries), dtype=np.float32)
    subsets = [doc_ranges(rng, n, 0.5), doc_ranges(rng, n, 0.1), np.array([[0, n]], np.uint64)]
    per_query = [subsets[i % 3] for i in range(len(queries))]
    for k in (10, 64):
        check_batch(ctx, c, queries, k, None, per_query, where="bad queries")
        check_batch(ctx, c, queries, k, 0.8, per_query, where="bad queries, cap")
    assert ctx.batch_last()["route"] == 6


def test_unnormalisable_corpus_row_sends_every_query_to_k1(ctx):
    rng = np.random.default_rng(32)
    n = 50_000
    rows = unit_rows(rng, n)
    rows[1234] *= np.float32(1e25)                                 # squared norm overflows fp32
    c = new_corpus(ctx, rows)
    per_query = [doc_ranges(rng, n, 0.5), np.array([[0, 3000]], np.uint64), doc_ranges(rng, n, 0.2)] * 2
    queries = unit_rows(rng, 6)
    queries[0] = rows[1234] / np.float32(1e25)
    check_batch(ctx, c, queries, 10, None, per_query, where="bad row")
    info = ctx.batch_last()
    assert info["route"] == 6 and info["groups"] == 0 and info["k1"] == 6


# ------------------------------------------------------------------ corpus changes and host rows ---
def test_after_append_update_and_remove(ctx):
    rng = np.random.default_rng(41)
    rows = unit_rows(rng, 80 * TILE + 300)
    queries = unit_rows(rng, 12)
    queries[0] = rows[80 * TILE + 299]
    c = capi.Corpus(ctx, len(rows))
    c.append(rows[: 50 * TILE + 130])
    subsets = [doc_ranges(rng, len(rows), f) for f in (0.4, 0.25, 0.7)]
    per_query = [subsets[i % 3] for i in range(12)]
    check_batch(ctx, c, queries, 10, None, per_query, where="prefix")
    c.append(rows[50 * TILE + 130:])
    check_batch(ctx, c, queries, 10, None, per_query, where="append")
    idx = np.sort(rng.choice(len(rows), 300, replace=False)).astype(np.uint64)
    new = unit_rows(rng, 300)
    new[0] = queries[1]
    c.update(idx, new)
    check_batch(ctx, c, queries, 10, 0.9, per_query, where="update")
    c.remove(np.array([[100, 4000], [20_000, 20_001]], np.uint64))
    check_batch(ctx, c, queries, 10, None, per_query, where="remove")
    assert ctx.batch_last()["route"] == 6 and ctx.batch_last()["groups"] == 3


def test_host_rows_corpus_equals_its_device_twin(ctx):
    rng = np.random.default_rng(43)
    n = 100_000
    rows = unit_rows(rng, n)
    dev = new_corpus(ctx, rows)
    host = capi.Corpus.in_host_memory(ctx, n)
    for part in np.array_split(rows, 3):
        host.append(part)
    subsets = special_subsets(rng, n)
    owner, per_query = deal(rng, [5, 3, 70, 2, 1, 4, 6, 2, 3], subsets)
    queries = unit_rows(rng, len(owner))
    for k, cap in [(10, None), (64, 0.95), (65, None)]:
        a = dev.search_batch_subsets(queries, per_query, k, cap)
        b = host.search_batch_subsets(queries, per_query, k, cap)
        assert ctx.batch_last()["route"] == 6
        for i, (x, y) in enumerate(zip(a, b)):
            same(x, y, f"query {i}")
    check_batch(ctx, host, queries, 10, None, per_query, where="host rows")
    host.close()


# ------------------------------------------------------------------ the workspace store ---
def test_store_many_equals_single_queries(ctx, monkeypatch, tmp_path):
    from semtools_b200.workspace import LineEmbedding, Store
    monkeypatch.setenv("HOME", str(tmp_path))
    rng = np.random.default_rng(51)
    paths = [f"/docs/f{i}.txt" for i in range(60)]
    lines = []
    for p in paths:
        for ln in range(int(rng.integers(5, 400))):
            lines.append(LineEmbedding(p, ln, unit_rows(rng, 1)[0]))
    sd, sh = Store.open(str(tmp_path / "d"), ctx), Store.open(str(tmp_path / "h"), ctx)
    for s in (sd, sh):
        s.upsert_line_embeddings(lines)
    real_init = capi.Corpus.__init__

    def nomem(self, *a, **k):
        raise capi.StbError(capi.STB_ERR_NOMEM, "device mirror does not fit")

    monkeypatch.setattr(capi.Corpus, "__init__", nomem)
    sh._gpu_corpus()                                               # the host mirror
    monkeypatch.setattr(capi.Corpus, "__init__", real_init)
    assert sh._corpus.host_rows and not sd._gpu_corpus().host_rows
    queries = unit_rows(rng, 24)
    queries[0] = lines[len(lines) // 2].embedding
    subsets = [paths[::3], paths[5:9], paths, [], ["/nope.txt"], paths[10:40], paths[:1]]
    per_query = [subsets[i % len(subsets)] for i in range(len(queries))]
    for s in (sd, sh):
        for k, cap in [(10, None), (3, 0.9), (64, None), (0, None), (200, 0.95)]:
            got = s.search_line_embeddings_many(queries, per_query, k, cap)
            assert len(got) == len(queries)
            for i, q in enumerate(queries):
                assert got[i] == s.search_line_embeddings(q, per_query[i], k, cap), (per_query[i][:2], k, cap, i)

"""In-place corpus mutations (stb_corpus_update / stb_corpus_remove): a numpy model of the rows is kept next
to each corpus.  After every step the rows must equal the model bit for bit, every candidate copy must be
byte-equal over the prefix it covers to a fresh corpus built from the model and prepared, and a copy that
covered every row before the step must still cover every row (it was maintained, not dropped).  Searches
after a mixed sequence of changes must return exactly the oracle's hits on the model."""
import numpy as np
import pytest

import oracle
from conftest import unit_rows
from semtools_b200 import capi

pytestmark = pytest.mark.gpu

CHUNK = 262144          # staging rows per chunk (STB_MUT_CHUNK_ROWS)
COPIES = (capi.STB_COPY_Q8_CODES, capi.STB_COPY_Q8_SCALES, capi.STB_COPY_Q8_PLANE, capi.STB_COPY_Q8_SR)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def make(ctx, rows, row_base=0, prepare=True):
    c = capi.Corpus(ctx, max(len(rows), 1), row_base=row_base)
    c.append(rows)
    if prepare:
        c.prepare(3)                                                  # q8 codes and 16-bit shadow
    return c


def snapshot(c):
    """rows and every copy as bytes (for the atomicity checks)"""
    return [bits(c.read())] + [bits(c.debug_copy(w)[0]) for w in COPIES + (capi.STB_COPY_H16_TILES,)]


def check(ctx, c, model, maintained=True):
    """rows == model bit for bit; each copy equals a fresh build of the rows it covers; maintained: both
    copies cover every row (tier_stats, no prepare in between)."""
    assert len(c) == len(model)
    assert np.array_equal(bits(c.read()), bits(model))
    st = c.tier_stats()
    if maintained:
        assert st["q8"]["built_rows"] == len(model) and st["h16"]["built_rows"] == len(model), st
    cov_q8 = c.debug_copy(capi.STB_COPY_Q8_SCALES, 0, 0)[1]
    cov_h16 = c.debug_copy(capi.STB_COPY_H16_TILES, 0, 0)[1]
    fresh = {}
    for cov in {cov_q8, cov_h16} - {0}:
        fresh[cov] = make(ctx, model[:cov])
    if cov_q8:
        for w in COPIES:
            got, n = c.debug_copy(w, 0, cov_q8)
            assert n == cov_q8
            assert np.array_equal(bits(got), bits(fresh[cov_q8].debug_copy(w, 0, cov_q8)[0])), w
    if cov_h16:
        tiles = (cov_h16 + 255) // 256
        got = c.debug_copy(capi.STB_COPY_H16_TILES, 0, tiles)[0]
        assert np.array_equal(got, fresh[cov_h16].debug_copy(capi.STB_COPY_H16_TILES, 0, tiles)[0])
    for f in fresh.values():
        f.close()
    return cov_q8, cov_h16


def removed_model(model, ranges, base=0):
    keep = np.ones(len(model), dtype=bool)
    for b, e in np.asarray(ranges, dtype=np.int64).reshape(-1, 2):
        keep[b - base:e - base] = False
    return np.ascontiguousarray(model[keep])


def scattered_ranges(rng, n, count, max_len=40):
    starts = np.sort(rng.choice(n - max_len, count, replace=False))
    ranges, prev = [], 0
    for s in starts:
        s = max(int(s), prev)
        e = min(s + int(rng.integers(1, max_len)), n)
        if s < e:
            ranges.append((s, e))
            prev = e + 1
    return np.asarray(ranges, dtype=np.uint64)


def test_update_rows_keeps_the_copies_current(ctx):
    rng = np.random.default_rng(1)
    n = 40037
    model = unit_rows(rng, n)
    c = make(ctx, model)
    check(ctx, c, model)
    # row 0, the last row, a row in the partial last tile
    idx = np.array([0, n - 40, n - 1], dtype=np.uint64)
    new = unit_rows(rng, 3) * np.float32(3.5)
    c.update(idx, new)
    model[idx.astype(np.int64)] = new
    check(ctx, c, model)
    # 16384 random rows, then every row of one tile
    idx = np.sort(rng.choice(n, 16384, replace=False)).astype(np.uint64)
    new = unit_rows(rng, len(idx))
    c.update(idx, new)
    model[idx.astype(np.int64)] = new
    check(ctx, c, model)
    idx = np.arange(256 * 37, 256 * 38, dtype=np.uint64)
    new = unit_rows(rng, 256)
    c.update(idx, new)
    model[idx.astype(np.int64)] = new
    check(ctx, c, model)
    # rows of an appended tail the copies do not cover yet, and rows of the covered prefix
    tail = unit_rows(rng, 1000)
    c.append(tail)
    model = np.concatenate([model, tail])
    idx = np.array([5, n - 1, n, n + 17, n + 999], dtype=np.uint64)
    new = unit_rows(rng, len(idx))
    c.update(idx, new)
    model[idx.astype(np.int64)] = new
    assert check(ctx, c, model, maintained=False) == (n, n)
    c.prepare(3)
    check(ctx, c, model)


def test_update_batch_larger_than_one_chunk(ctx):
    rng = np.random.default_rng(2)
    n = CHUNK + 40001
    model = unit_rows(rng, n)
    c = make(ctx, model)
    idx = np.sort(rng.choice(n, CHUNK + 20000, replace=False)).astype(np.uint64)
    new = unit_rows(rng, len(idx))
    c.update(idx, new)
    model[idx.astype(np.int64)] = new
    check(ctx, c, model)


def test_remove_rows_keeps_the_copies_current(ctx):
    rng = np.random.default_rng(3)
    n = 45101
    model = unit_rows(rng, n)
    c = make(ctx, model)
    for pick in (lambda m: [[0, 1]], lambda m: [[m - 1, m]], lambda m: [[20000, 20057]]):   # first, last, one "document"
        ranges = pick(len(model))
        c.remove(np.asarray(ranges, dtype=np.uint64))
        model = removed_model(model, ranges)
        check(ctx, c, model)
    ranges = scattered_ranges(rng, len(model), 500)
    assert len(ranges) >= 450
    c.remove(ranges)
    model = removed_model(model, ranges)
    check(ctx, c, model)
    # nothing to remove: nothing changes, the tier bookkeeping included
    c.search(model[3], top_k=5)
    before, tries = snapshot(c), c.tier_stats()
    c.remove(np.zeros((0, 2), dtype=np.uint64))
    assert all(np.array_equal(a, b) for a, b in zip(before, snapshot(c))) and c.tier_stats() == tries
    # an appended tail the copies do not cover: a removal across the covered prefix's end shrinks the prefix
    cov = len(model)
    tail = unit_rows(rng, 700)
    c.append(tail)
    model = np.concatenate([model, tail])
    ranges = [[100, 300], [cov - 50, cov + 20], [cov + 600, cov + 650]]
    c.remove(np.asarray(ranges, dtype=np.uint64))
    model = removed_model(model, ranges)
    assert check(ctx, c, model, maintained=False) == (cov - 250, cov - 250)
    c.prepare(3)
    check(ctx, c, model)
    # everything, then rows again
    c.remove(np.array([[0, len(model)]], dtype=np.uint64))
    assert len(c) == 0 and c.tier_stats()["q8"]["built_rows"] == 0
    model = unit_rows(rng, 33001)
    c.append(model)
    c.prepare(3)
    check(ctx, c, model)


def test_remove_moves_a_tail_of_several_chunks(ctx):
    rng = np.random.default_rng(4)
    n = 4 * CHUNK + 12345
    model = unit_rows(rng, n)
    c = make(ctx, model)
    ranges = [[1000, 2000], [2500, 2501], [CHUNK + 7, CHUNK + 300], [3 * CHUNK, 3 * CHUNK + 5000], [n - 3, n]]
    c.remove(np.asarray(ranges, dtype=np.uint64))
    model = removed_model(model, ranges)
    assert len(model) - 1000 >= 3 * CHUNK
    check(ctx, c, model)


class DevSeries:
    """stb_search_topk_dev launches into device buffers, read back after one synchronisation."""

    def __init__(self, n_slots, k=10):
        self.torch = pytest.importorskip("torch")
        self.dev = self.torch.device("cuda:0")
        self.k = k
        self.hits = self.torch.zeros((n_slots, k, 2), dtype=self.torch.float64, device=self.dev)
        self.status = self.torch.zeros((n_slots, 4), dtype=self.torch.int32, device=self.dev)
        self.q = self.torch.zeros((n_slots, 256), dtype=self.torch.float32, device=self.dev)

    def launch_all(self, corpus, qs):
        self.q[: len(qs)].copy_(self.torch.from_numpy(qs))
        self.torch.cuda.synchronize()
        for i in range(len(qs)):
            corpus.search_topk_dev(self.q[i].data_ptr(), self.k, self.hits[i].data_ptr(), self.status[i].data_ptr())

    def check(self, ctx, slot, rows, q):
        ctx.sync()
        raw, st = self.hits[slot].cpu().numpy(), self.status[slot].cpu().numpy()
        assert st[1] == 1, st
        r, d = oracle.search_rows(rows, q, top_k=self.k)
        expect_hits(np.ascontiguousarray(raw).view(capi.HIT_DTYPE).reshape(-1)[: st[0]], r, d)


def expect_hits(hits, rows_exp, d_exp):
    assert hits["row"].tolist() == [int(r) for r in rows_exp]
    assert np.array_equal(hits["distance"], np.asarray(d_exp, dtype=np.float64))


def test_searches_after_a_mixed_sequence_are_exact(ctx, monkeypatch):
    rng = np.random.default_rng(5)
    model = unit_rows(rng, 50013)
    c = make(ctx, model)
    tail = unit_rows(rng, 3000)                                       # append
    c.append(tail)
    model = np.concatenate([model, tail])
    c.prepare(3)
    idx = np.sort(rng.choice(len(model), 5000, replace=False)).astype(np.uint64)   # update
    new = unit_rows(rng, len(idx))
    c.update(idx, new)
    model[idx.astype(np.int64)] = new
    ranges = scattered_ranges(rng, len(model), 120)                   # remove
    c.remove(ranges)
    model = removed_model(model, ranges)
    # update: near-copies of the queries, so the top hits are rows the sequence wrote
    qs = unit_rows(rng, 16)
    idx = np.sort(rng.choice(len(model), 16, replace=False)).astype(np.uint64)
    new = (qs + np.float32(0.05) * unit_rows(rng, 16)).astype(np.float32)
    c.update(idx, new)
    model[idx.astype(np.int64)] = new
    check(ctx, c, model)
    for k in (1, 10, 16, 40):
        for q in qs[:4]:
            r, d = oracle.search_rows(model, q, top_k=k)
            expect_hits(c.search(q, top_k=k), r, d)
    st = c.tier_stats()
    assert st["q8"]["proven"] >= 1 and st["h16"]["tries"] >= 1, st
    monkeypatch.setenv("STB_SCAN_TIER", "f32")
    for q in qs[:2]:
        r, d = oracle.search_rows(model, q, top_k=10)
        expect_hits(c.search(q, top_k=10), r, d)
    monkeypatch.delenv("STB_SCAN_TIER")
    for q in qs[:3]:                                                  # threshold mode
        r, d = oracle.search_rows(model, q, top_k=10, max_distance=0.9)
        expect_hits(c.search(q, top_k=10, max_distance=0.9), r, d)
    sub = np.array([[10, 4000], [9000, 9100], [30000, len(model)]], dtype=np.uint64)   # store query
    for q in qs[:3]:
        r, d32 = oracle.store_search(model, sub, q, 10, 0.98)
        hits = c.search(q, 10, 0.98, capi.STB_MODE_STORE_QUERY, row_ranges=sub)
        assert hits["row"].tolist() == [int(x) for x in r]
        assert np.array_equal(hits["distance"].astype(np.float32), d32)
    for q, hits in zip(qs, c.search_many(qs, top_k=10)):             # search_many, then a co-scan series
        r, d = oracle.search_rows(model, q, top_k=10)
        expect_hits(hits, r, d)
    s = DevSeries(len(qs))
    s.launch_all(c, qs)
    for i, q in enumerate(qs):
        s.check(ctx, i, model, q)
    for q, hits in zip(qs, c.search_batch(qs, top_k=10)):            # K2
        r, d = oracle.search_rows(model, q, top_k=10)
        expect_hits(hits, r, d)


@pytest.mark.parametrize("kind", ["nan", "inf", "tiny", "zero"])
def test_bad_rows(ctx, kind):
    rng = np.random.default_rng(6)
    model = unit_rows(rng, 36001)
    c = make(ctx, model)
    row = 20011
    bad = model[row].copy()
    if kind == "nan":
        bad[7] = np.nan
    elif kind == "inf":
        bad[7] = np.inf
    elif kind == "tiny":
        bad *= np.float32(1e-25)                                      # the fp32 squared norm underflows
    else:
        bad[:] = 0
    c.update(np.array([row], dtype=np.uint64), bad[None])
    model[row] = bad
    assert np.array_equal(bits(c.read()), bits(model))
    st = c.tier_stats()
    marked = kind != "zero"
    assert (st["q8"]["built_rows"], st["h16"]["built_rows"]) == ((0, 0) if marked else (len(model), len(model))), st
    if not marked:
        check(ctx, c, model)
    qs = np.concatenate([unit_rows(rng, 3), model[row + 1][None]])
    for q in qs:
        for k in (10, 40):
            r, d = oracle.search_rows(model, q, top_k=k)
            hits = c.search(q, top_k=k)
            assert hits["row"].tolist() == [int(x) for x in r]
            assert np.array_equal(hits["distance"], d, equal_nan=True)
    # a good row in its place; the marked copies were dropped by the update, prepare builds them anew
    good = unit_rows(rng, 1)
    c.update(np.array([row], dtype=np.uint64), good)
    model[row] = good[0]
    if marked:
        assert c.tier_stats()["q8"]["built_rows"] == 0
        c.prepare(3)
    check(ctx, c, model)
    tries = c.tier_stats()["q8"]["proven"]
    r, d = oracle.search_rows(model, qs[-1], top_k=10)
    expect_hits(c.search(qs[-1], top_k=10), r, d)
    assert c.tier_stats()["q8"]["proven"] == tries + 1


def test_removal_drops_copies_marked_bad(ctx):
    """A removal drops a copy already marked bad, so the next prepare decides anew: still bad while the bad
    row is there, built once it is gone."""
    rng = np.random.default_rng(7)
    model = unit_rows(rng, 34003)
    c = make(ctx, model)
    c.update(np.array([100], dtype=np.uint64), np.full((1, 256), np.nan, dtype=np.float32))
    model[100] = np.nan
    for ranges, built in (([[200, 300]], 0), ([[100, 101]], len(model) - 101)):
        c.remove(np.asarray(ranges, dtype=np.uint64))
        model = removed_model(model, ranges)
        assert np.array_equal(bits(c.read()), bits(model))
        st = c.tier_stats()
        assert st["q8"]["built_rows"] == 0 and st["h16"]["built_rows"] == 0
        c.prepare(3)
        st = c.tier_stats()
        assert st["q8"]["built_rows"] == built and st["h16"]["built_rows"] == built, st
    check(ctx, c, model)


def test_global_row_ids(ctx):
    rng = np.random.default_rng(8)
    base = 2 ** 32
    model = unit_rows(rng, 33301)
    c = make(ctx, model, row_base=base)
    idx = np.array([0, 1, 33300], dtype=np.uint64)
    with pytest.raises(capi.StbError) as e:
        c.update(idx, unit_rows(rng, 3))                              # local ids are not this shard's rows
    assert e.value.status == capi.STB_ERR_RANGE
    new = unit_rows(rng, 3)
    c.update(idx + np.uint64(base), new)
    model[idx.astype(np.int64)] = new
    check(ctx, c, model)
    ranges = np.array([[base + 5, base + 9], [base + 33000, base + 33301]], dtype=np.uint64)
    c.remove(ranges)
    model = removed_model(model, ranges, base)
    check(ctx, c, model)
    hits = c.search(model[40], top_k=3)
    r, d = oracle.search_rows(model, model[40], top_k=3)
    assert hits["row"].tolist() == [int(x) + base for x in r] and np.array_equal(hits["distance"], d)


def test_rejected_arguments_change_nothing(ctx):
    rng = np.random.default_rng(9)
    base = 1000
    model = unit_rows(rng, 33000)
    c = make(ctx, model, row_base=base)
    before = snapshot(c)
    L = capi.lib()
    rows3 = unit_rows(rng, 3)

    def upd(idx, rows=rows3):
        idx = np.asarray(idx, dtype=np.uint64)
        return L.stb_corpus_update(c._h, idx.ctypes.data, rows.ctypes.data, len(idx))

    def rem(ranges):
        r = np.asarray(ranges, dtype=np.uint64).reshape(-1, 2)
        return L.stb_corpus_remove(c._h, r.ctypes.data, r.shape[0])

    R, A = capi.STB_ERR_RANGE, capi.STB_ERR_ARG
    one = np.array([base], dtype=np.uint64)
    cases = [
        (upd([base + 5, base + 4, base + 6]), R),                    # unsorted
        (upd([base + 5, base + 5, base + 6]), R),                    # duplicate
        (upd([base + 1, base + 2, base + 33000]), R),                # past the end
        (upd([base - 1, base + 2, base + 3]), R),                    # below row_base
        (L.stb_corpus_update(c._h, None, rows3.ctypes.data, 3), A),
        (L.stb_corpus_update(c._h, one.ctypes.data, None, 1), A),
        (rem([[base + 10, base + 20], [base + 5, base + 8]]), R),    # unsorted
        (rem([[base + 10, base + 20], [base + 19, base + 30]]), R),  # overlapping
        (rem([[base + 10, base + 10]]), R),                          # empty
        (rem([[base + 10, base + 20], [base + 32990, base + 33001]]), R),   # past the end
        (rem([[base - 2, base + 1]]), R),                            # below row_base
        (L.stb_corpus_remove(c._h, None, 2), A),
    ]
    assert [rc for rc, _ in cases] == [want for _, want in cases]
    assert all(np.array_equal(a, b) for a, b in zip(before, snapshot(c)))
    assert L.stb_corpus_update(c._h, None, None, 0) == 0 and L.stb_corpus_remove(c._h, None, 0) == 0
    check(ctx, c, model)


def test_live_ivfpq_index_blocks_mutations(ctx):
    rng = np.random.default_rng(10)
    model = unit_rows(rng, 40000)
    c = make(ctx, model)
    index = capi.IvfPq(c, nlist=64, train_rows=8192, iters=4)
    before = snapshot(c)
    for call in (lambda: c.update(np.array([3], dtype=np.uint64), unit_rows(rng, 1)),
                 lambda: c.remove(np.array([[3, 4]], dtype=np.uint64))):
        with pytest.raises(capi.StbError) as e:
            call()
        assert e.value.status == capi.STB_ERR_STATE
    assert all(np.array_equal(a, b) for a, b in zip(before, snapshot(c)))
    index.close()
    new = unit_rows(rng, 1)
    c.update(np.array([3], dtype=np.uint64), new)
    model[3] = new[0]
    c.remove(np.array([[4, 6]], dtype=np.uint64))
    model = removed_model(model, [[4, 6]])
    check(ctx, c, model)
    index = capi.IvfPq(c, nlist=64, train_rows=8192, iters=4)
    with pytest.raises(capi.StbError):
        c.update(np.array([3], dtype=np.uint64), new)
    tail = unit_rows(rng, 500)
    c.append(tail)
    assert index.extend() == 500
    index.close()


def test_update_is_stream_ordered_after_queued_queries(ctx):
    rng = np.random.default_rng(11)
    model = unit_rows(rng, 60001)
    c = make(ctx, model)
    qs = unit_rows(rng, 8)
    old = model.copy()
    s = DevSeries(len(qs))
    s.launch_all(c, qs)                                               # enqueued, not waited for
    # replace the rows the queries would find first, and many more
    win = sorted({int(oracle.search_rows(old, q, top_k=1)[0][0]) for q in qs})
    idx = np.union1d(np.array(win), rng.choice(len(model), 20000, replace=False)).astype(np.uint64)
    new = unit_rows(rng, len(idx))
    c.update(idx, new)
    model[idx.astype(np.int64)] = new
    for i, q in enumerate(qs):
        s.check(ctx, i, old, q)                                       # the queued queries saw the old rows
    s.launch_all(c, qs)
    ctx.sync()
    assert ctx.coscan_offsets(len(qs))[0] == 0                        # the update ended the co-scan series
    for i, q in enumerate(qs):
        s.check(ctx, i, model, q)
    check(ctx, c, model)


def test_store_keeps_its_gpu_mirror(ctx, tmp_path):
    from semtools_b200.workspace import LineEmbedding, Store
    rng = np.random.default_rng(12)
    docs = {f"/d/{i}.txt": unit_rows(rng, int(n)) for i, n in enumerate(rng.integers(2000, 6000, 12))}
    store = Store.open(str(tmp_path), ctx)
    store.upsert_line_embeddings([LineEmbedding(p, j, e[j]) for p, e in docs.items() for j in range(len(e))])
    paths = list(docs)
    q = unit_rows(rng, 1)[0]
    store.search_line_embeddings(q, paths, 10)
    mirror = store._corpus
    mirror.prepare(3)
    # patch a document (same line ids), with a repeated line in the batch: the last value wins
    p = paths[3]
    patch = unit_rows(rng, 300)
    store.upsert_line_embeddings([LineEmbedding(p, j, patch[j]) for j in range(300)] +
                                 [LineEmbedding(p, 7, patch[0])])
    assert store._corpus is mirror
    assert np.array_equal(bits(mirror.read()), bits(np.asarray(store._emb)))
    store.delete_documents([paths[5]])                                # prune one document
    assert store._corpus is mirror
    assert np.array_equal(bits(mirror.read()), bits(np.asarray(store._emb)))
    st = mirror.tier_stats()
    assert st["q8"]["built_rows"] == len(mirror) == len(store._emb)
    live = [x for x in paths if x != paths[5]]
    for qq in (q, patch[7], docs[paths[9]][11]):
        got = store.search_line_embeddings(qq, live, 10)
        fresh = Store.open(str(tmp_path), ctx).search_line_embeddings(qq, live, 10)
        assert got == fresh
    assert store._corpus is mirror

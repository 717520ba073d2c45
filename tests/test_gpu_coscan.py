"""K1 co-scan: back-to-back asynchronous top-k queries on one corpus start their pass where the
previous query is reading (scan_topk.cu: stb_coscan_offset), so the two scans share each tile's
read.  The offset only decides which warp scores which row: every result must stay exactly the
oracle's, the ticket bookkeeping must hold, and a series must restart at tile 0 whenever anything
but a co-scan of the same corpus ran in between."""
import numpy as np
import pytest

import oracle
from conftest import unit_rows
from semtools_b200 import capi

pytestmark = pytest.mark.gpu
TILE_ROWS = {"f32": 8, "h16": 16, "q8": 32}


def check(hits, rows_exp, d_exp):
    assert hits["row"].tolist() == [int(r) for r in rows_exp]
    assert np.array_equal(hits["distance"], np.asarray(d_exp, dtype=np.float64))


def make_corpus(ctx, rows):
    c = capi.Corpus(ctx, max(len(rows), 1))
    c.append(rows)
    return c


class DevSeries:
    """stb_search_topk_dev launches into device buffers, read back after one synchronisation."""

    def __init__(self, n_slots, k=10):
        self.torch = pytest.importorskip("torch")
        self.dev = self.torch.device("cuda:0")
        self.k = k
        self.hits = self.torch.zeros((n_slots, k, 2), dtype=self.torch.float64, device=self.dev)
        self.status = self.torch.zeros((n_slots, 4), dtype=self.torch.int32, device=self.dev)
        self.q = self.torch.zeros((n_slots, 256), dtype=self.torch.float32, device=self.dev)

    def launch(self, corpus, slot, q):
        self.q[slot].copy_(self.torch.from_numpy(q))
        self.torch.cuda.synchronize()
        corpus.search_topk_dev(self.q[slot].data_ptr(), self.k, self.hits[slot].data_ptr(), self.status[slot].data_ptr())

    def launch_all(self, corpus, qs, reps=1):
        self.q[: len(qs)].copy_(self.torch.from_numpy(qs))
        self.torch.cuda.synchronize()
        for _ in range(reps):
            for i in range(len(qs)):
                corpus.search_topk_dev(self.q[i].data_ptr(), self.k, self.hits[i].data_ptr(), self.status[i].data_ptr())

    def check(self, ctx, slot, rows, q):
        ctx.sync()
        raw, st = self.hits[slot].cpu().numpy(), self.status[slot].cpu().numpy()
        assert st[1] == 1, st
        r, d = oracle.search_rows(rows, q, top_k=self.k)
        check(np.ascontiguousarray(raw).view(capi.HIT_DTYPE).reshape(-1)[: st[0]], r, d)


@pytest.mark.parametrize("tier", ["f32", "h16", "q8"])
def test_coscan_series_is_exact_and_rotates(ctx, monkeypatch, tier):
    rng = np.random.default_rng(4242)
    monkeypatch.setenv("STB_SCAN_TIER", tier)
    for n in (1, 33, 9_473, 150_000, 700_001):
        rows = unit_rows(rng, n)
        c = make_corpus(ctx, rows)
        c.prepare()
        qs = unit_rows(rng, 6)
        s = DevSeries(6)
        s.launch_all(c, qs, reps=3)                          # one series of 18 back-to-back queries
        offs = ctx.coscan_offsets(8)                         # its last 8 launches: all followers
        d, h = ctx.ticket_check()
        assert d == h
        for i in range(6):
            s.check(ctx, i, rows, qs[i])
        n_tiles = -(-n // TILE_ROWS[tier])
        assert all(o is not None and 0 <= o < n_tiles for o in offs), (n, offs)
        if n == 700_001:                                     # a follower starts where its predecessor reads
            assert any(o > 0 for o in offs), (n, offs)


def test_coscan_restarts_after_an_append(ctx, monkeypatch):
    monkeypatch.delenv("STB_SCAN_TIER", raising=False)
    rng = np.random.default_rng(77)
    rows = unit_rows(rng, 400_000)
    c = capi.Corpus(ctx, 500_000)
    c.append(rows[:300_000])
    c.prepare()
    qs = unit_rows(rng, 8)
    s = DevSeries(8)
    for i in range(4):
        s.launch(c, i, qs[i])
    c.append(rows[300_000:])
    for i in range(4, 8):
        s.launch(c, i, qs[i])
    offs = ctx.coscan_offsets(4)
    assert offs[0] == 0, offs                                # more rows: a new series
    for i in range(8):
        s.check(ctx, i, rows[:300_000] if i < 4 else rows, qs[i])
    d, h = ctx.ticket_check()
    assert d == h


def test_coscan_alternating_corpora_never_follow_each_other(ctx, monkeypatch):
    monkeypatch.delenv("STB_SCAN_TIER", raising=False)
    rng = np.random.default_rng(78)
    rows_a, rows_b = unit_rows(rng, 200_000), unit_rows(rng, 200_000)
    a, b = make_corpus(ctx, rows_a), make_corpus(ctx, rows_b)
    a.prepare(); b.prepare()
    qs = unit_rows(rng, 8)
    s = DevSeries(8)
    s.q.copy_(s.torch.from_numpy(qs))
    s.torch.cuda.synchronize()
    for i in range(8):
        (a if i % 2 == 0 else b).search_topk_dev(s.q[i].data_ptr(), s.k, s.hits[i].data_ptr(), s.status[i].data_ptr())
    assert ctx.coscan_offsets(8) == [0] * 8                  # same shape, other corpus: no predecessor
    for i in range(8):
        s.check(ctx, i, rows_a if i % 2 == 0 else rows_b, qs[i])


def test_coscan_series_interleaved_with_synchronous_search(ctx, monkeypatch):
    monkeypatch.delenv("STB_SCAN_TIER", raising=False)
    rng = np.random.default_rng(79)
    rows = unit_rows(rng, 300_000)
    c = make_corpus(ctx, rows)
    c.prepare()
    qs = unit_rows(rng, 7)
    s = DevSeries(7)
    s.q.copy_(s.torch.from_numpy(qs))
    s.torch.cuda.synchronize()
    sync_hits = {}
    for i in range(7):
        if i == 3:
            sync_hits[i] = c.search(qs[i], top_k=10)         # a synchronous full-grid launch ends the series
        else:
            c.search_topk_dev(s.q[i].data_ptr(), s.k, s.hits[i].data_ptr(), s.status[i].data_ptr())
    offs = ctx.coscan_offsets(4)
    assert offs[0] is None and offs[1] == 0, offs
    for i in range(7):
        if i == 3:
            r, d = oracle.search_rows(rows, qs[i], top_k=10)
            check(sync_hits[i], r, d)
        else:
            s.check(ctx, i, rows, qs[i])
    d, h = ctx.ticket_check()
    assert d == h


def test_coscan_search_many_equals_search_one_by_one(ctx, monkeypatch):
    monkeypatch.delenv("STB_SCAN_TIER", raising=False)
    rng = np.random.default_rng(80)
    rows = unit_rows(rng, 700_001)
    c = make_corpus(ctx, rows)
    c.prepare()
    qs = unit_rows(rng, 12)
    many = c.search_many(qs, top_k=10)
    offs = ctx.coscan_offsets(8)
    assert all(o is not None for o in offs) and any(o > 0 for o in offs), offs
    for i, q in enumerate(qs):
        one = c.search(q, top_k=10)
        assert np.array_equal(many[i], one)
        r, d = oracle.search_rows(rows, q, top_k=10)
        check(one, r, d)
    d, h = ctx.ticket_check()
    assert d == h

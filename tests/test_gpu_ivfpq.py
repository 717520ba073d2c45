"""GPU: K5 IVF-PQ (self-specified, parity-unpinned: the reference has no IVF_PQ).
Measured property: recall@10 against the exact scan on clustered synthetic data; every
returned (distance,row) pair must be an exact canonical distance of a real row."""
import numpy as np
import pytest

import oracle
from semtools_b200 import capi

pytestmark = pytest.mark.gpu


def make_centers(rng, n_centers=4000):
    centers = rng.standard_normal((n_centers, 256)).astype(np.float32)
    return centers / np.linalg.norm(centers, axis=1, keepdims=True)


def clustered(rng, centers, n, spread=0.6):
    x = centers[rng.integers(0, len(centers), n)] + spread * rng.standard_normal((n, 256)).astype(np.float32) / 16.0
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    return np.ascontiguousarray(x, dtype=np.float32)


def test_ivfpq_recall_and_exact_distances(ctx):
    rng = np.random.default_rng(5)
    n = 200_000
    centers = make_centers(rng)
    rows = clustered(rng, centers, n)
    c = capi.Corpus(ctx, n)
    c.append(rows)
    idx = capi.IvfPq(c, nlist=256, train_rows=65536, iters=6)
    st = idx.stats()
    assert st["rows"] == n and st["nlist"] == 256 and st["max_list"] < n // 8
    queries = clustered(rng, centers, 30)          # queries come from the corpus' own clusters
    recalls, scanned = [], []
    for q in queries:
        got, n_scan = idx.search(q, nprobe=32, top_k=10, rerank=512)
        exact = c.search(q, top_k=10)
        assert len(got) == 10
        recalls.append(len(set(got["row"].tolist()) & set(exact["row"].tolist())) / 10.0)
        scanned.append(n_scan)
        assert np.all(np.diff(got["distance"]) >= 0)
        for h in got[:3]:                                  # returned distances are exact
            assert h["distance"] == oracle.cosine(q, rows[int(h["row"])])
    assert np.mean(recalls) >= 0.9, np.mean(recalls)
    assert np.mean(scanned) < 0.3 * n                      # probed 32 of 256 lists
    # probing every list and re-ranking generously must reproduce the exact answer
    got, n_scan = idx.search(queries[0], nprobe=256, top_k=10, rerank=4096)
    assert n_scan == n
    assert got["row"].tolist() == c.search(queries[0], top_k=10)["row"].tolist()
    idx.close()


def test_v2_fused_search_matches_v1_candidates_and_exact_distances(ctx):
    """The fused search (rerank <= 1024) against the batched search, which has the same coarse scores,
    probe lists and LUT and selects its candidates exactly (stb_ivfpq_search_batch)."""
    rng = np.random.default_rng(6)
    n = 200_000
    centers = make_centers(rng)
    rows = clustered(rng, centers, n)
    c = capi.Corpus(ctx, n, row_base=7_000_000)
    c.append(rows)
    idx = capi.IvfPq(c, nlist=256, train_rows=65536, iters=6)
    queries = clustered(rng, centers, 30)
    batch, batch_n, batch_scanned = idx.search_batch(queries, nprobe=32, top_k=10, rerank=512)
    try:
        recalls = []
        for i, q in enumerate(queries):
            got, n_scan = idx.search(q, nprobe=32, top_k=10, rerank=512)
            assert n_scan == batch_scanned[i]                      # same probe lists
            assert len(got) == 10 and np.all(np.diff(got["distance"]) >= 0)
            for h in got[:3]:
                assert h["distance"] == oracle.cosine(q, rows[int(h["row"]) - 7_000_000])
            exact = c.search(q, top_k=10)
            recalls.append(len(set(got["row"].tolist()) & set(exact["row"].tolist())) / 10.0)
            # the per-warp top-64 / per-CTA top-64 reductions are lossless for the best 512 here,
            # so both searches re-rank the same candidates -> identical hits
            assert np.array_equal(got, batch[i][: batch_n[i]]), i
        assert np.mean(recalls) >= 0.9
        # probing every list: exact answer (rerank capped at 1024 in v2)
        got, n_scan = idx.search(queries[0], nprobe=256, top_k=10, rerank=1024)
        assert n_scan == n
        assert got["row"].tolist() == c.search(queries[0], top_k=10)["row"].tolist()
        # top_k larger than the number of codes probed, and a zero query
        got, _ = idx.search(queries[1], nprobe=1, top_k=1000, rerank=1000)
        assert 0 < len(got) <= 1000 and np.all(np.diff(got["distance"]) >= 0)
        got, _ = idx.search(np.zeros(256, np.float32), nprobe=4, top_k=5, rerank=64)
        assert len(got) == 5 and np.all(got["distance"] == 1.0)
    finally:
        idx.close()


def test_device_resident_search_equals_the_host_call(ctx):
    """stb_ivfpq_search_dev (asynchronous, query / hits / status in HBM; what the sharded index runs per
    rank) returns exactly the hits of stb_ivfpq_search, padded with (+inf, UINT64_MAX)."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(8)
    n = 120_000
    centers = make_centers(rng)
    rows = clustered(rng, centers, n)
    c = capi.Corpus(ctx, n, row_base=1_000_000)
    c.append(rows)
    idx = capi.IvfPq(c, nlist=128, train_rows=65536, iters=6)
    queries = clustered(rng, centers, 12)
    dev = torch.device("cuda:0")
    q_dev = torch.from_numpy(queries).to(dev)
    hits = torch.zeros((12, 20, 2), dtype=torch.float64, device=dev)
    st = torch.zeros((12, 2), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    for i in range(12):
        idx.search_dev(q_dev[i].data_ptr(), 16, 20, 256, hits[i].data_ptr(), st[i].data_ptr())
    ctx.sync()
    raw, sth = hits.cpu().numpy(), st.cpu().numpy()
    for i in range(12):
        want, n_scan = idx.search(queries[i], nprobe=16, top_k=20, rerank=256)
        got = np.ascontiguousarray(raw[i]).view(capi.HIT_DTYPE).reshape(-1)
        assert sth[i, 0] == len(want) and sth[i, 1] == n_scan
        assert np.array_equal(got[: len(want)], want)
        assert np.all(np.isinf(got["distance"][len(want):]))
    idx.close()

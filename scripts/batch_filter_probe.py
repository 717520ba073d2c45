"""K2 filtered batch probe: stb_search_batch_filtered against the K1 store query one query at a time (stb_search
in store-query mode, the same filter) and against unfiltered stb_search_batch.

python scripts/batch_filter_probe.py [rows] [nq] [k1_queries] [ivfpq_rows]
Defaults: 10M random unit rows, nq = 1024, top_k = 10, 256 queries for the K1 loop, K5 at 4M rows (0: skip).
The rows are grouped into "documents" of 1..200 lines (lognormal, median ~20, as scripts/ivfpq_filter_probe.py);
a filter is a random subset of documents holding ~100 / 25 / 5 / 1 / 0.1 % of the rows, one contiguous block of
1 % of the rows, or no filter (row_ranges = NULL).  Per filter: eligible rows, ranges, the share of 256-row
tiles holding an eligible row (listed tiles), the route (stb_debug_batch_last: 3 = filtered v2, 4 = K1 only),
queries the tensor path left to K1, ms per batch and q/s of the host call (median of 3 after a warm-up, host
to host: query upload, ranges, bitmap, both GEMM passes, finish, K1 fallbacks), q/s of the K1 loop, and whether
the first 64 queries equal K1.  For context, K5's stb_ivfpq_search_filtered q/s and recall@10 on a clustered
corpus of its own.  Prints one JSON line per measurement, the card name and power limit first."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from semtools_b200 import capi  # noqa: E402

rows = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
NQ = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
K1_Q = int(sys.argv[3]) if len(sys.argv) > 3 else 256
IVF_ROWS = int(sys.argv[4]) if len(sys.argv) > 4 else 4_000_000
top_k = 10


def emit(**kw):
    print(json.dumps(kw), flush=True)


hw = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                    capture_output=True, text=True).stdout.strip()
emit(hardware=hw)

dev = torch.device("cuda:0")
ctx = capi.Context(0)
g = torch.Generator(device=dev); g.manual_seed(1)
c = capi.Corpus(ctx, rows)
for i in range(0, rows, 1_000_000):
    n = min(1_000_000, rows - i)
    x = torch.randn((n, 256), generator=g, device=dev); x /= x.norm(dim=1, keepdim=True)
    torch.cuda.synchronize(); c.append_dev(x.data_ptr(), n)
    del x
q = torch.randn((NQ, 256), generator=g, device=dev)
Q = (q / q.norm(dim=1, keepdim=True)).contiguous().cpu().numpy()
c.prepare_batch()
c.prepare()

rng = np.random.default_rng(5)


def documents(n):
    lens = np.clip(np.round(rng.lognormal(3.0, 1.0, n)), 1, 200).astype(np.int64)
    start = np.concatenate([[0], np.cumsum(lens)])
    start = start[start < n]
    return start, np.append(start[1:], n)


def doc_subset(n, doc_start, doc_end, frac):
    keep = rng.random(len(doc_start)) < frac
    if frac >= 1.0:
        keep[:] = True
    mask = np.zeros(n + 1, np.int8)
    np.add.at(mask, doc_start[keep], 1); np.add.at(mask, doc_end[keep], -1)
    m = np.cumsum(mask)[:n] > 0
    edges = np.flatnonzero(np.diff(np.concatenate([[0], m.astype(np.int8), [0]])))
    return m, edges.reshape(-1, 2).astype(np.uint64)


def filters_for(n):
    doc_start, doc_end = documents(n)
    out = {}
    for frac in (1.0, 0.25, 0.05, 0.01, 0.001):
        out[f"docs_{frac * 100:g}%"] = doc_subset(n, doc_start, doc_end, frac)
    blk = np.zeros(n, bool); blk[n // 2: n // 2 + n // 100] = True
    out["block_1%"] = (blk, np.array([[n // 2, n // 2 + n // 100]], np.uint64))
    out["none"] = (np.ones(n, bool), None)
    return len(doc_start), out


n_docs, filters = filters_for(rows)
emit(shape=dict(rows=rows, nq=NQ, top_k=top_k, k1_queries=K1_Q), documents=n_docs)


def timed(fn, reps=3):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); t.append(time.perf_counter() - t0)
    return float(np.median(t)) * 1e3


ms = timed(lambda: c.search_batch(Q, top_k=top_k))
emit(reference="stb_search_batch unfiltered", route=ctx.batch_last()["route"], ms_per_batch=round(ms, 3),
     qps=round(NQ / ms * 1e3, 1))

for name, (mask, ranges) in filters.items():
    listed = np.add.reduceat(mask.astype(np.int32), np.arange(0, rows, 256)) > 0
    tiles, n_tiles = int(listed.sum()), len(listed)
    before = ctx.counters()["fallback_searches"]
    got = c.search_batch_filtered(Q, ranges, top_k=top_k)
    to_k1 = ctx.counters()["fallback_searches"] - before
    info = ctx.batch_last()
    ms = timed(lambda: c.search_batch_filtered(Q, ranges, top_k=top_k))
    k1 = [c.search(Q[i], top_k, None, capi.STB_MODE_STORE_QUERY, row_ranges=ranges) for i in range(min(64, NQ))]
    agree = all(np.array_equal(got[i], k1[i]) for i in range(len(k1)))
    t0 = time.perf_counter()
    for i in range(K1_Q):
        c.search(Q[i % NQ], top_k, None, capi.STB_MODE_STORE_QUERY, row_ranges=ranges)
    k1_ms = (time.perf_counter() - t0) * 1e3 / K1_Q
    emit(filter=name, eligible_rows=int(mask.sum()), ranges=0 if ranges is None else len(ranges),
         listed_tile_share=round(float(tiles) / n_tiles, 4), route=info["route"], n_sample=info["n_sample"],
         stride=info["stride"], queries_to_k1=int(to_k1), ms_per_batch=round(ms, 3), qps=round(NQ / ms * 1e3, 1),
         k1_ms_per_query=round(k1_ms, 4), k1_qps=round(1e3 / k1_ms, 1), agree_with_k1=agree)

c.close()
del c
torch.cuda.empty_cache()

# K5 for context: its own clustered corpus (scripts/ivfpq_filter_probe.py's shape), recall against K2 filtered
if IVF_ROWS:
    n_centers, spread = max(IVF_ROWS // 100, 1000), 0.6
    centers = torch.randn((n_centers, 256), generator=g, device=dev); centers /= centers.norm(dim=1, keepdim=True)
    c = capi.Corpus(ctx, IVF_ROWS)
    for i in range(0, IVF_ROWS, 1_000_000):
        n = min(1_000_000, IVF_ROWS - i)
        idx = torch.randint(0, n_centers, (n,), generator=g, device=dev)
        x = centers[idx] + spread / 16.0 * torch.randn((n, 256), generator=g, device=dev)
        x /= x.norm(dim=1, keepdim=True)
        torch.cuda.synchronize(); c.append_dev(x.data_ptr(), n)
        del x
    idx = torch.randint(0, n_centers, (NQ,), generator=g, device=dev)
    qc = centers[idx] + spread / 16.0 * torch.randn((NQ, 256), generator=g, device=dev)
    QC = (qc / qc.norm(dim=1, keepdim=True)).contiguous().cpu().numpy()
    index = capi.IvfPq(c, nlist=4096, train_rows=262144, iters=8)
    _, ivf_filters = filters_for(IVF_ROWS)
    for name, (mask, ranges) in ivf_filters.items():
        exact = c.search_batch_filtered(QC, ranges, top_k=top_k)
        ms_exact = timed(lambda: c.search_batch_filtered(QC, ranges, top_k=top_k))
        got, n, _ = index.search_filtered(QC, ranges, nprobe=64, top_k=top_k, rerank=256)
        ms = timed(lambda: index.search_filtered(QC, ranges, nprobe=64, top_k=top_k, rerank=256))
        rec = float(np.mean([len(set(got[i]["row"][: n[i]].tolist()) & set(exact[i]["row"].tolist())) / max(len(exact[i]), 1)
                             for i in range(NQ)]))
        emit(k5_filter=name, rows=IVF_ROWS, k5_qps=round(NQ / ms * 1e3, 1), k5_recall_at_10=round(rec, 4),
             k2_filtered_qps=round(NQ / ms_exact * 1e3, 1), k2_route=ctx.batch_last()["route"])
    index.close()
    c.close()

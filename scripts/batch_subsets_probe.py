"""K2 per-query subsets probe: stb_search_batch_subsets against one stb_search_batch_filtered call per distinct
subset and against the K1 store query one query at a time (stb_search in store-query mode, each query's own
ranges).

python scripts/batch_subsets_probe.py [rows] [nq] [k1_queries]
Defaults: 10M random unit rows, nq = 1024, top_k = 10, 64 queries for the K1 loop.  The rows are grouped into
"documents" of 1..200 lines (lognormal, median ~20, as scripts/batch_filter_probe.py).  For G in {1, 4, 16, 64,
256} distinct random document subsets holding ~25 / 5 / 1 % of the rows each, and subsets of 50 random
documents (the files an agent's tool call names: ~50 ranges, ~1k rows), the queries are dealt to the
subsets unevenly (weights 1 / (1 + j), shuffled; every subset gets at least one query).  Per point: the route
and stb_debug_batch_last's counts (groups on the tensor cores, queries K1 answered), ms per batch and q/s of the
new call (median of 3 after a warm-up, host to host), the same for the per-subset loop of
stb_search_batch_filtered (queries gathered per subset, results scattered back), the K1 loop's q/s on the first
k1_queries queries, and whether the first 64 queries equal K1.  Prints one JSON line per measurement, the card
name and power limit first."""
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
K1_Q = int(sys.argv[3]) if len(sys.argv) > 3 else 64
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
lens = np.clip(np.round(rng.lognormal(3.0, 1.0, rows)), 1, 200).astype(np.int64)
doc_start = np.concatenate([[0], np.cumsum(lens)])
doc_start = doc_start[doc_start < rows]
doc_end = np.append(doc_start[1:], rows)


def doc_subset(frac=None, n_docs=None):
    if n_docs is None:
        keep = rng.random(len(doc_start)) < frac
    else:
        keep = np.zeros(len(doc_start), bool); keep[rng.choice(len(doc_start), n_docs, replace=False)] = True
    mask = np.zeros(rows + 1, np.int8)
    np.add.at(mask, doc_start[keep], 1); np.add.at(mask, doc_end[keep], -1)
    m = np.cumsum(mask)[:rows] > 0
    edges = np.flatnonzero(np.diff(np.concatenate([[0], m.astype(np.int8), [0]])))
    return edges.reshape(-1, 2).astype(np.uint64)


def timed(fn, reps=3):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); t.append(time.perf_counter() - t0)
    return float(np.median(t)) * 1e3


emit(shape=dict(rows=rows, nq=NQ, top_k=top_k, k1_queries=K1_Q), documents=len(doc_start))

for frac, n_docs in ((0.25, None), (0.05, None), (0.01, None), (None, 50)):
    for G in (1, 4, 16, 64, 256):
        subsets = [doc_subset(frac, n_docs) for _ in range(G)]
        w = 1.0 / (1.0 + np.arange(G)); rng.shuffle(w)
        owner = np.concatenate([np.arange(G), rng.choice(G, NQ - G, p=w / w.sum())]) if NQ >= G else np.arange(NQ) % G
        rng.shuffle(owner)
        per_query = [subsets[j] for j in owner]
        members = [np.flatnonzero(owner == j) for j in range(G)]

        def per_subset_loop():
            out = [None] * NQ
            for j, idx in enumerate(members):
                if len(idx):
                    for i, h in zip(idx, c.search_batch_filtered(Q[idx], subsets[j], top_k=top_k)):
                        out[i] = h
            return out

        before = ctx.counters()["fallback_searches"]
        got = c.search_batch_subsets(Q, per_query, top_k=top_k)
        to_k1 = ctx.counters()["fallback_searches"] - before
        info = ctx.batch_last()
        ms = timed(lambda: c.search_batch_subsets(Q, per_query, top_k=top_k))
        loop = per_subset_loop()
        ms_loop = timed(per_subset_loop)
        k1 = [c.search(Q[i], top_k, None, capi.STB_MODE_STORE_QUERY, row_ranges=per_query[i]) for i in range(min(64, NQ))]
        agree = all(np.array_equal(got[i], k1[i]) and np.array_equal(loop[i], k1[i]) for i in range(len(k1)))
        t0 = time.perf_counter()
        for i in range(K1_Q):
            c.search(Q[i % NQ], top_k, None, capi.STB_MODE_STORE_QUERY, row_ranges=per_query[i % NQ])
        k1_ms = (time.perf_counter() - t0) * 1e3 / K1_Q
        emit(subset_share=frac, subset_docs=n_docs, ranges_per_query=round(float(np.mean([len(r) for r in per_query])), 1), subsets=G, group_sizes=dict(min=int(min(map(len, members))), max=int(max(map(len, members)))),
             route=info["route"], tensor_groups=info.get("groups"), k1_queries=info.get("k1"), fallback_searches=int(to_k1),
             ms_per_batch=round(ms, 3), qps=round(NQ / ms * 1e3, 1),
             loop_ms_per_batch=round(ms_loop, 3), loop_qps=round(NQ / ms_loop * 1e3, 1),
             k1_ms_per_query=round(k1_ms, 4), k1_qps=round(1e3 / k1_ms, 1), agree_with_k1=agree)

c.close()

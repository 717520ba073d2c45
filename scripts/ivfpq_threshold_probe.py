"""K5 threshold search probe: recall, rows re-scored and q/s of stb_ivfpq_search_threshold against the exact
threshold search of the same rows (K2's stb_search_batch_threshold, and K1 one query at a time).

python scripts/ivfpq_threshold_probe.py [rows] [nlist] [nq]
Defaults: the bench's IVF-PQ shape (4M clustered rows, rows / 100 centres, spread 0.6; nlist 4096) and 1024
queries drawn like the rows.  max_distance is chosen per query set so that the exact answer has about 10, 100 and
5000 hits per query (the median query's 10th, 100th and 5000th distance on a sample).  For each, nprobe in
{32, 64, 128} x slack in {0, 0.02, 0.05, 0.1, 0.2, 0.3}.  Prints one JSON line per measurement."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from semtools_b200 import capi  # noqa: E402

rows = int(sys.argv[1]) if len(sys.argv) > 1 else 4_000_000
nlist = int(sys.argv[2]) if len(sys.argv) > 2 else 4096
nq = int(sys.argv[3]) if len(sys.argv) > 3 else 1024
n_centers, spread = max(rows // 100, 1000), 0.6
TARGETS = (10, 100, 5000)
NPROBES = (32, 64, 128)
SLACKS = (0.0, 0.02, 0.05, 0.1, 0.2, 0.3)


def emit(**kw):
    print(json.dumps(kw), flush=True)


hw = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                    capture_output=True, text=True).stdout.strip()
emit(hardware=hw)

dev = torch.device("cuda:0")
ctx = capi.Context(0)
g = torch.Generator(device=dev); g.manual_seed(11)
centers = torch.randn((n_centers, 256), generator=g, device=dev); centers /= centers.norm(dim=1, keepdim=True)
c = capi.Corpus(ctx, rows)
X = torch.empty((rows, 256), dtype=torch.float32, device=dev)      # kept to choose max_distance
for i in range(0, rows, 1_000_000):
    n = min(1_000_000, rows - i)
    idx = torch.randint(0, n_centers, (n,), generator=g, device=dev)
    x = centers[idx] + spread / 16.0 * torch.randn((n, 256), generator=g, device=dev)
    X[i:i + n] = x / x.norm(dim=1, keepdim=True)
    torch.cuda.synchronize(); c.append_dev(X[i].data_ptr(), n)
idx = torch.randint(0, n_centers, (nq,), generator=g, device=dev)
q = centers[idx] + spread / 16.0 * torch.randn((nq, 256), generator=g, device=dev)
q = (q / q.norm(dim=1, keepdim=True)).contiguous()
qh = q.cpu().numpy()
# max_distance per target: the median sample query's target-th smallest distance (f32 GEMM; the exact counts follow)
d = 1.0 - q[:64] @ X.T
kth = torch.topk(d, max(TARGETS), dim=1, largest=False).values
M = {k: float(kth[:, k - 1].median()) for k in TARGETS}
del d, kth, X
torch.cuda.empty_cache()
t0 = time.perf_counter()
index = capi.IvfPq(c, nlist=nlist, train_rows=262144, iters=8)
ctx.sync()
emit(shape=dict(rows=rows, nlist=nlist, nq=nq), build_s=time.perf_counter() - t0, stats=index.stats())
c.prepare_batch()


def timed(fn, reps):
    """ms per call: host clock around reps synchronous calls, after one warm-up call."""
    out = fn()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t0) * 1e3 / reps, out


for target in TARGETS:
    m = M[target]
    ms, exact = timed(lambda: c.search_batch_threshold(qh, m), 3)
    n_exact = np.array([len(h) for h in exact])
    emit(target=target, max_distance=m, config="stb_search_batch_threshold (K2, exact)", nq=nq, ms=ms,
         qps=nq / ms * 1e3, hits_per_query=float(n_exact.mean()), hits_per_query_median=float(np.median(n_exact)))
    k1n = 16
    ms, _ = timed(lambda: [c.search(qh[i], top_k=0, max_distance=m) for i in range(k1n)], 2)
    emit(target=target, max_distance=m, config="stb_search (K1, exact) one query at a time", nq=k1n, ms=ms,
         qps=k1n / ms * 1e3)
    ex = [set(h["row"].tolist()) for h in exact]
    for nprobe in NPROBES:
        for slack in SLACKS:
            ms, (got, scanned, reranked) = timed(
                lambda: index.search_threshold(qh, nprobe=nprobe, max_distance=m, slack=slack), 3)
            found = sum(len(set(h["row"].tolist()) & e) for h, e in zip(got, ex))
            per_q = [len(set(h["row"].tolist()) & e) / len(e) for h, e in zip(got, ex) if len(e)]
            emit(target=target, max_distance=m, config="stb_ivfpq_search_threshold", nprobe=nprobe, slack=slack,
                 nq=nq, ms=ms, qps=nq / ms * 1e3, recall=found / max(int(n_exact.sum()), 1),
                 recall_mean_per_query=float(np.mean(per_q)) if per_q else None,
                 reranked_per_query=float(np.mean(reranked)), scanned_per_query=float(np.mean(scanned)))
emit(hardware_after=subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                   capture_output=True, text=True).stdout.strip())
index.close(); c.close()

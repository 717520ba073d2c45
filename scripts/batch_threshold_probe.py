"""K2 threshold batch probe: stb_search_batch_threshold against the same queries through stb_search in threshold
mode, one query at a time (K1).

python scripts/batch_threshold_probe.py [rows] [nq]
Defaults: 10M rows of the benchmark's synthetic distribution (unit rows, 0.1 % duplicated, 0.01 % zero), with
planted near-duplicate clusters (1..8 near-copies, noise ~1e-3 per unit row, of every query's anchor row),
nq = 1024 queries (each a slightly perturbed anchor).  Thresholds are chosen from the exact distances of 32 of
the queries to all rows so that a query has about 1, 100 and 5000 hits.  Per threshold: hits per query (mean,
median, max), the route fields of stb_debug_batch_last (queries re-emitted by the second tensor pass, queries
answered by K1), ms per batch and q/s of the host call with the capacity set to the total (median of 3 after a
warm-up, host to host), ms per query and q/s of the K1 loop over the same queries, and whether every query's
hits equal K1's bit for bit.
Prints one JSON line per measurement, the card name and power limit first."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from semtools_b200 import capi  # noqa: E402

ROWS = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
NQ = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
TARGETS = (1, 100, 5000)


def emit(**kw):
    print(json.dumps(kw), flush=True)


hw = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                    capture_output=True, text=True).stdout.strip()
emit(hardware=hw)

dev = torch.device("cuda:0")
ctx = capi.Context(0)
g = torch.Generator(device=dev); g.manual_seed(7)
chunk = 1_000_000
anchors = torch.randint(0, ROWS, (NQ,), generator=g, device=dev)
X = torch.empty((ROWS, 256), device=dev)
for i in range(0, ROWS, chunk):                        # the benchmark's distribution, chunk by chunk
    n = min(chunk, ROWS - i)
    x = torch.randn((n, 256), generator=g, device=dev); x /= x.norm(dim=1, keepdim=True)
    n_dup, n_zero = max(n // 1000, 1), max(n // 10000, 1)
    idx = torch.randint(0, n, (2 * n_dup + n_zero,), generator=g, device=dev)
    x[idx[:n_dup]] = x[idx[n_dup:2 * n_dup]]
    x[idx[2 * n_dup:]] = 0.0
    X[i:i + n] = x
    del x
# near-duplicate clusters: 1..8 noisy copies of every anchor at random rows
sizes = torch.randint(1, 9, (NQ,), generator=g, device=dev)
src = torch.repeat_interleave(anchors, sizes)
dst = torch.randint(0, ROWS, (src.numel(),), generator=g, device=dev)
y = X[src] + 1e-3 / 16 * torch.randn((src.numel(), 256), generator=g, device=dev)
X[dst] = y / y.norm(dim=1, keepdim=True)
q = X[anchors] + 1e-3 / 16 * torch.randn((NQ, 256), generator=g, device=dev)
q[X[anchors].norm(dim=1) == 0] = torch.randn((1, 256), generator=g, device=dev)
Q = (q / q.norm(dim=1, keepdim=True)).contiguous()
# thresholds: the median over 32 queries of the distance of the target-th nearest row (f64, exact enough to aim)
samp = Q[:32].double()
D = torch.empty((samp.shape[0], ROWS), dtype=torch.float64, device=dev)
for i in range(0, ROWS, chunk):
    xb = X[i:i + chunk].double()
    D[:, i:i + chunk] = 1.0 - (samp @ xb.T) / (xb.norm(dim=1).clamp_min(1e-300)[None, :] * samp.norm(dim=1)[:, None])
    del xb
s = torch.topk(D, max(TARGETS) + 1, dim=1, largest=False).values.cpu().numpy()
del D
M = {t: float(np.median(s[:, t])) for t in TARGETS}
c = capi.Corpus(ctx, ROWS)
torch.cuda.synchronize()
c.append_dev(X.data_ptr(), ROWS)
del X, y
torch.cuda.empty_cache()
Qh = Q.cpu().numpy()
c.prepare_batch()
c.prepare()
emit(shape=dict(rows=ROWS, nq=NQ, planted_copies=int(sizes.sum())), thresholds={str(t): M[t] for t in TARGETS})


def timed(fn, reps=3):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); t.append(time.perf_counter() - t0)
    return float(np.median(t)) * 1e3


for t in TARGETS:
    m = M[t]
    got = c.search_batch_threshold(Qh, m)
    info = ctx.batch_last()
    total = sum(len(h) for h in got)
    ms = timed(lambda: c.search_batch_threshold(Qh, m, cap=total))        # one pass: the capacity fits
    t0 = time.perf_counter()
    ref = [c.search(Qh[i], top_k=0, max_distance=m) for i in range(NQ)]
    k1_ms = (time.perf_counter() - t0) * 1e3 / NQ
    agree = all(len(a) == len(b) and np.array_equal(a["row"], b["row"]) and
                np.array_equal(a["distance"].view(np.uint64), b["distance"].view(np.uint64)) for a, b in zip(got, ref))
    n_hits = np.array([len(h) for h in got])
    emit(target_hits=t, max_distance=m, hits_mean=round(float(n_hits.mean()), 1), hits_median=float(np.median(n_hits)),
         hits_max=int(n_hits.max()), retried=info["retried"], k1_queries=info["k1"], ms_per_batch=round(ms, 3),
         qps=round(NQ / ms * 1e3, 1), k1_ms_per_query=round(k1_ms, 4), k1_qps=round(1e3 / k1_ms, 1),
         identical_to_k1=agree)
c.close()
ctx.close()

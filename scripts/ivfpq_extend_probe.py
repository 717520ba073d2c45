"""K5 extend probe: what stb_ivfpq_extend costs against a rebuild, and what it does to recall and q/s.

python scripts/ivfpq_extend_probe.py [rows] [base_rows] [nlist] [nprobe] [rerank] [step]
Defaults: the data of scripts/ivfpq_batch_probe.py (4M clustered rows, rows/100 centres, spread 0.6), nlist 4096,
nprobe 64, rerank 512, top_k 10, 1024 queries; the extended indexes are built on the first 3M rows and extended
by the last 1M, in one call and in calls of `step` = 16384 rows (the workspace batch).  Every build and extend is
timed with a host clock around the call and a synchronise.  Prints one JSON line per measurement."""
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
base_rows = int(sys.argv[2]) if len(sys.argv) > 2 else rows * 3 // 4
nlist = int(sys.argv[3]) if len(sys.argv) > 3 else 4096
nprobe = int(sys.argv[4]) if len(sys.argv) > 4 else 64
rerank = int(sys.argv[5]) if len(sys.argv) > 5 else 512
step = int(sys.argv[6]) if len(sys.argv) > 6 else 16384
top_k, n_centers, spread, nq = 10, max(rows // 100, 1000), 0.6, 1024


def emit(**kw):
    print(json.dumps(kw), flush=True)


hw = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                    capture_output=True, text=True).stdout.strip()
emit(hardware=hw)

dev = torch.device("cuda:0")
ctx = capi.Context(0)
g = torch.Generator(device=dev); g.manual_seed(11)
centers = torch.randn((n_centers, 256), generator=g, device=dev); centers /= centers.norm(dim=1, keepdim=True)
X = torch.empty((rows, 256), dtype=torch.float32, device=dev)
for i in range(0, rows, 1_000_000):
    n = min(1_000_000, rows - i)
    idx = torch.randint(0, n_centers, (n,), generator=g, device=dev)
    x = centers[idx] + spread / 16.0 * torch.randn((n, 256), generator=g, device=dev)
    X[i:i + n] = x / x.norm(dim=1, keepdim=True)
    del x
idx = torch.randint(0, n_centers, (nq,), generator=g, device=dev)
q = centers[idx] + spread / 16.0 * torch.randn((nq, 256), generator=g, device=dev)
q = (q / q.norm(dim=1, keepdim=True)).contiguous()
qh = q.cpu().numpy()
torch.cuda.synchronize()


def corpus(n):
    c = capi.Corpus(ctx, rows)
    c.append_dev(X.data_ptr(), n)
    return c


def timed(fn):
    ctx.sync()
    t0 = time.perf_counter()
    out = fn()
    ctx.sync()
    return out, time.perf_counter() - t0


def build(c):
    return timed(lambda: capi.IvfPq(c, nlist=nlist, train_rows=262144, iters=8))


emit(shape=dict(rows=rows, base_rows=base_rows, nlist=nlist, nprobe=nprobe, top_k=top_k, rerank=rerank, nq=nq, step=step))
c_full = corpus(rows)
full, t_full = build(c_full)
emit(config="build", rows=rows, s=t_full, stats=full.stats())

c_one = corpus(base_rows)
one, t_base = build(c_one)
c_one.append_dev(X[base_rows:].data_ptr(), rows - base_rows)
added, t_ext = timed(one.extend)
emit(config="build + extend in one call", build_rows=base_rows, build_s=t_base, extend_rows=added, extend_s=t_ext,
     total_s=t_base + t_ext, stats=one.stats())

c_step = corpus(base_rows)
stepped, t_base2 = build(c_step)
t_steps, calls = [], 0
for a in range(base_rows, rows, step):
    b = min(a + step, rows)
    c_step.append_dev(X[a:b].data_ptr(), b - a)
    added, t = timed(stepped.extend)
    assert added == b - a
    t_steps.append(t)
emit(config=f"build + extend in {step}-row calls", build_rows=base_rows, build_s=t_base2, calls=len(t_steps),
     extend_s=sum(t_steps), extend_ms_per_call=dict(mean=1e3 * float(np.mean(t_steps)), min=1e3 * min(t_steps),
                                                     max=1e3 * max(t_steps)),
     total_s=t_base2 + sum(t_steps), stats=stepped.stats())
del X
torch.cuda.empty_cache()

# recall@10 against the exact search over the same 4M rows, and batched q/s (device form, 1024 queries)
exact = c_full.search_batch(qh, top_k=top_k)
lib_stream = torch.cuda.ExternalStream(ctx.stream) if ctx.stream else torch.cuda.default_stream()
hits = torch.empty((nq, top_k, 2), dtype=torch.float64, device=dev)
status = torch.empty((nq, 2), dtype=torch.int32, device=dev)
for name, index in [("build", full), ("build + extend in one call", one), (f"build + extend in {step}-row calls", stepped)]:
    got, cnt, scanned = index.search_batch(qh, nprobe=nprobe, top_k=top_k, rerank=rerank)
    rec = [len(set(got[i, : cnt[i]]["row"].tolist()) & set(exact[i]["row"].tolist())) / top_k for i in range(nq)]
    index.search_batch_dev(q.data_ptr(), nq, nprobe, top_k, rerank, hits.data_ptr(), status.data_ptr()); ctx.sync()
    reps = 20
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(lib_stream)
    for _ in range(reps):
        index.search_batch_dev(q.data_ptr(), nq, nprobe, top_k, rerank, hits.data_ptr(), status.data_ptr())
    b.record(lib_stream); ctx.sync(); b.synchronize()
    ms = a.elapsed_time(b) / reps
    emit(index=name, recall_at_10=float(np.mean(rec)), codes_scanned_per_query=float(np.mean(scanned)),
         max_list=index.stats()["max_list"], batch_ms=ms, batch_qps=nq / ms * 1e3)
for index in (full, one, stepped):
    index.close()
for c in (c_full, c_one, c_step):
    c.close()

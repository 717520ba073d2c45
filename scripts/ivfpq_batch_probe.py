"""K5 batched search probe: q/s of stb_ivfpq_search_batch(_dev) against back-to-back single queries and the
exact K2 batch, recall@10, and a per-stage breakdown (torch.profiler, separate run).

python scripts/ivfpq_batch_probe.py [rows] [nlist] [nprobe] [rerank] [rounds] [out_dir]
Defaults: the bench's IVF-PQ shape (4M clustered rows, 40k centres, spread 0.6; nlist 4096, nprobe 64,
top_k 10, rerank 512).  Prints one JSON line per measurement."""
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
nprobe = int(sys.argv[3]) if len(sys.argv) > 3 else 64
rerank = int(sys.argv[4]) if len(sys.argv) > 4 else 512
rounds = int(sys.argv[5]) if len(sys.argv) > 5 else 2
out_dir = sys.argv[6] if len(sys.argv) > 6 else None
top_k, n_centers, spread = 10, max(rows // 100, 1000), 0.6
NQS = (1, 16, 128, 1024, 4096)


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
for i in range(0, rows, 1_000_000):
    n = min(1_000_000, rows - i)
    idx = torch.randint(0, n_centers, (n,), generator=g, device=dev)
    x = centers[idx] + spread / 16.0 * torch.randn((n, 256), generator=g, device=dev)
    x /= x.norm(dim=1, keepdim=True)
    torch.cuda.synchronize(); c.append_dev(x.data_ptr(), n)
    del x
idx = torch.randint(0, n_centers, (max(NQS),), generator=g, device=dev)
q = centers[idx] + spread / 16.0 * torch.randn((max(NQS), 256), generator=g, device=dev)
q = (q / q.norm(dim=1, keepdim=True)).contiguous()
qh = q.cpu().numpy()
t0 = time.perf_counter()
index = capi.IvfPq(c, nlist=nlist, train_rows=262144, iters=8)
ctx.sync()
emit(shape=dict(rows=rows, nlist=nlist, nprobe=nprobe, top_k=top_k, rerank=rerank), build_s=time.perf_counter() - t0,
     stats=index.stats())

hits = torch.empty((max(NQS), top_k, 2), dtype=torch.float64, device=dev)
status = torch.empty((max(NQS), 2), dtype=torch.int32, device=dev)
Q1024 = qh[:1024]


def batch_dev(nq):
    index.search_batch_dev(q.data_ptr(), nq, nprobe, top_k, rerank, hits.data_ptr(), status.data_ptr())


def singles_dev(nq):
    for i in range(nq):
        index.search_dev(q[i].data_ptr(), nprobe, top_k, rerank, hits[i].data_ptr(), status[i].data_ptr())


# the library enqueues on the context's stream: the events are recorded there
lib_stream = torch.cuda.ExternalStream(ctx.stream) if ctx.stream else torch.cuda.default_stream()


def timed_dev(fn, nq, reps):
    """ms per call from device events over reps calls (one warm-up call first)."""
    fn(nq); ctx.sync()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(lib_stream)
    for _ in range(reps):
        fn(nq)
    b.record(lib_stream); ctx.sync(); b.synchronize()
    return a.elapsed_time(b) / reps


def timed_host(fn, reps):
    fn(); ctx.sync()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    ctx.sync()
    return (time.perf_counter() - t0) * 1e3 / reps


c.prepare_batch()
for r in range(rounds):
    for nq in NQS:
        ms = timed_dev(batch_dev, nq, max(5, 8192 // nq))
        emit(round=r, config="search_batch_dev", nq=nq, ms=ms, qps=nq / ms * 1e3)
    ms = timed_host(lambda: index.search_batch(Q1024, nprobe=nprobe, top_k=top_k, rerank=rerank), 5)
    emit(round=r, config="search_batch (host)", nq=1024, ms=ms, qps=1024 / ms * 1e3)
    ms = timed_dev(singles_dev, 1024, 2)
    emit(round=r, config="search_dev x1024 back to back", nq=1024, ms=ms, qps=1024 / ms * 1e3)
    ms = timed_host(lambda: c.search_batch(Q1024, top_k=top_k), 5)
    emit(round=r, config="Corpus.search_batch (K2, exact)", nq=1024, ms=ms, qps=1024 / ms * 1e3)

# recall@10 against the exact search (first 256 queries), batch and single path
nr = 256
exact = c.search_batch(qh[:nr], top_k=top_k)
got, cnt, scanned = index.search_batch(qh[:nr], nprobe=nprobe, top_k=top_k, rerank=rerank)
rec_b = [len(set(got[i, : cnt[i]]["row"].tolist()) & set(exact[i]["row"].tolist())) / top_k for i in range(nr)]
rec_s, same = [], 0
for i in range(nr):
    one, _ = index.search(qh[i], nprobe=nprobe, top_k=top_k, rerank=rerank)
    rec_s.append(len(set(one["row"].tolist()) & set(exact[i]["row"].tolist())) / top_k)
    same += int(np.array_equal(one, got[i, : cnt[i]]))
code_bytes = float(np.mean(scanned)) * 32
emit(recall_batch=float(np.mean(rec_b)), recall_single=float(np.mean(rec_s)), batch_equals_single=f"{same}/{nr}",
     codes_scanned_per_query=float(np.mean(scanned)), code_bytes_per_query=code_bytes,
     code_bytes_per_1024_batch=code_bytes * 1024)

# per-stage breakdown (separate profiled run)
from torch.profiler import ProfilerActivity, profile  # noqa: E402
batch_dev(1024); ctx.sync()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(5):
        batch_dev(1024)
    ctx.sync()
stages = {}
for e in prof.key_averages():
    if "ivfb_" in e.key:
        stages[e.key.split("(")[0]] = round(e.device_time_total / 5 / 1e3, 4)
emit(stage_ms_per_1024_batch=stages)
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
    prof.export_chrome_trace(os.path.join(out_dir, "ivfpq_batch_trace.json"))
index.close(); c.close()

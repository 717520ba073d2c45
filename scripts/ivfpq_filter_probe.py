"""K5 filtered search probe: stb_ivfpq_search_filtered against the exact filtered scan (stb_search in
store-query mode, K1's range walk) and against "unfiltered K5, then drop the ineligible hits".

python scripts/ivfpq_filter_probe.py [rows] [nq] [out_dir]
Defaults: the bench's IVF-PQ shape (4M clustered rows, 40k centres, spread 0.6; nlist 4096, nprobe 64,
top_k 10), rerank 256 and 512, 1024 queries.  The rows are grouped into "documents" of 1..200 lines
(lognormal, median ~20); a filter is a random subset of documents holding ~100 / 25 / 5 / 1 / 0.1 % of the
rows (thousands of ranges), or one contiguous block of 1 % of the rows (a single range).  Per filter:
  recall@10 of the filtered search and of the post-filtered unfiltered search, both against the exact
  filtered scan; ms per query at nq = 1 (synchronised host calls, median of 200 after warm-up); q/s at
  nq = 1024; eligible codes scanned; ms of the exact filtered scan (median of 200 host calls); and, in a
  profiled run of its own, the device time of the eligibility pass (ivff_* kernels) per call.
Prints one JSON line per measurement."""
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
NQ = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
out_dir = sys.argv[3] if len(sys.argv) > 3 else None
nlist, nprobe, top_k, n_centers, spread = 4096, 64, 10, max(rows // 100, 1000), 0.6
RERANKS = (256, 512)
REPS = 200


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
idx = torch.randint(0, n_centers, (NQ,), generator=g, device=dev)
q = centers[idx] + spread / 16.0 * torch.randn((NQ, 256), generator=g, device=dev)
Q = (q / q.norm(dim=1, keepdim=True)).contiguous().cpu().numpy()
t0 = time.perf_counter()
index = capi.IvfPq(c, nlist=nlist, train_rows=262144, iters=8)
ctx.sync()
emit(shape=dict(rows=rows, nlist=nlist, nprobe=nprobe, top_k=top_k, reranks=RERANKS, nq=NQ),
     build_s=round(time.perf_counter() - t0, 2), stats=index.stats())

# documents and filters
rng = np.random.default_rng(5)
lens = np.clip(np.round(rng.lognormal(3.0, 1.0, rows)), 1, 200).astype(np.int64)
doc_start = np.concatenate([[0], np.cumsum(lens)])
doc_start = doc_start[doc_start < rows]
doc_end = np.append(doc_start[1:], rows)
n_docs = len(doc_start)


def doc_subset(frac):
    keep = rng.random(n_docs) < frac
    if frac >= 1.0:
        keep[:] = True
    b, e = doc_start[keep], doc_end[keep]
    # merge adjacent documents into one range, as Store._ranges_for does for consecutive rows
    mask = np.zeros(rows + 1, np.int8)
    np.add.at(mask, b, 1); np.add.at(mask, e, -1)
    m = np.cumsum(mask)[:rows] > 0
    edges = np.flatnonzero(np.diff(np.concatenate([[0], m.astype(np.int8), [0]])))
    return m, edges.reshape(-1, 2).astype(np.uint64)


filters = {}
for frac in (1.0, 0.25, 0.05, 0.01, 0.001):
    filters[f"docs_{frac * 100:g}%"] = doc_subset(frac)
blk = np.zeros(rows, bool); blk[rows // 2: rows // 2 + rows // 100] = True
filters["block_1%"] = (blk, np.array([[rows // 2, rows // 2 + rows // 100]], np.uint64))
emit(documents=n_docs, filters={k: dict(rows=int(m.sum()), ranges=len(r)) for k, (m, r) in filters.items()})


def recall(got_rows, exact_rows):
    if len(exact_rows) == 0:
        return 1.0
    return len(set(got_rows) & set(exact_rows)) / len(exact_rows)


def median_ms(fn, reps):
    for _ in range(5):
        fn()
    t = []
    for i in range(reps):
        t0 = time.perf_counter(); fn(i); t.append(time.perf_counter() - t0)
    return float(np.median(t)) * 1e3


unf = {rr: index.search_batch(Q, nprobe=nprobe, top_k=top_k, rerank=rr) for rr in RERANKS}
for name, (mask, ranges) in filters.items():
    exact = [c.search(Q[i], top_k, None, capi.STB_MODE_STORE_QUERY, row_ranges=ranges)["row"].tolist() for i in range(NQ)]
    exact_ms = median_ms(lambda i=0: c.search(Q[i % NQ], top_k, None, capi.STB_MODE_STORE_QUERY, row_ranges=ranges), REPS)
    for rr in RERANKS:
        got, n, sc = index.search_filtered(Q, ranges, nprobe=nprobe, top_k=top_k, rerank=rr)
        rec = float(np.mean([recall(got[i]["row"][: n[i]].tolist(), exact[i]) for i in range(NQ)]))
        ug, un, _ = unf[rr]
        post = [[r for r in ug[i]["row"][: un[i]].tolist() if mask[r]] for i in range(NQ)]
        rec_post = float(np.mean([recall(post[i], exact[i]) for i in range(NQ)]))
        full = float(np.mean([len(exact[i]) == n[i] for i in range(NQ)]))
        ms1 = median_ms(lambda i=0: index.search_filtered(Q[i % NQ][None], ranges, nprobe=nprobe, top_k=top_k, rerank=rr),
                        REPS)
        index.search_filtered(Q, ranges, nprobe=nprobe, top_k=top_k, rerank=rr)
        t0 = time.perf_counter()
        for _ in range(3):
            index.search_filtered(Q, ranges, nprobe=nprobe, top_k=top_k, rerank=rr)
        ms_b = (time.perf_counter() - t0) * 1e3 / 3
        emit(filter=name, rerank=rr, eligible_rows=int(mask.sum()), ranges=len(ranges), recall_at_10=round(rec, 4),
             recall_post_filter=round(rec_post, 4), full_count_share=round(full, 4),
             eligible_codes_scanned=float(np.mean(sc)), ms_nq1=round(ms1, 4), qps_nq1024=round(NQ / ms_b * 1e3, 1),
             exact_filtered_ms=round(exact_ms, 4))

# eligibility pass: device time of the ivff_* kernels per call (profiled run of its own)
from torch.profiler import ProfilerActivity, profile  # noqa: E402
for name, (mask, ranges) in filters.items():
    index.search_filtered(Q[:1], ranges, nprobe=nprobe, top_k=top_k, rerank=256)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(20):
            index.search_filtered(Q[i:i + 1], ranges, nprobe=nprobe, top_k=top_k, rerank=256)
        ctx.sync()
    st = {}
    for e in prof.key_averages():
        if "ivff_" in e.key or "ivfb_" in e.key:
            st[e.key.split("(")[0]] = round(e.device_time_total / 20 / 1e3, 4)
    emit(filter=name, eligibility_pass_ms=round(sum(v for k, v in st.items() if "ivff_" in k), 4), stage_ms_nq1=st)
    if out_dir and name == "docs_5%":
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, "ivfpq_filter_trace.json"))
index.close(); c.close()

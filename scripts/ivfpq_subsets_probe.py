"""K5 subsets search probe: stb_ivfpq_search_subsets (one call, each distinct subset passed once) against the
loop of one stb_ivfpq_search_filtered call per subset, and against the exact store query (stb_search in
store-query mode).

python scripts/ivfpq_subsets_probe.py [rows] [nq] [out_dir]
Defaults: the shape of scripts/ivfpq_filter_probe.py (4M clustered rows, 40k centres, spread 0.6, documents of
1..200 lines; nlist 4096, nprobe 64, top_k 10, rerank 256) and 1024 queries, dealt at random to G = 1, 4, 16,
64, 256 subsets, each a random set of documents holding ~25 % or ~5 % of the rows.  Per point:
  q/s of the call and of the per-subset loop (host calls, median of 3 after a warm-up; every query of the two
  forms compared bit for bit); recall@10 against the exact store query; and, in a profiled run of its own,
  the device time of each form (kernels and copies), the eligibility pass's share of it (ivff_* kernels), and
  the host-side share of the call: 1 - device time / median call time.
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
nlist, nprobe, top_k, rerank, n_centers, spread = 4096, 64, 10, 256, max(rows // 100, 1000), 0.6
GROUPS = (1, 4, 16, 64, 256)
FRACS = (0.25, 0.05)


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
index = capi.IvfPq(c, nlist=nlist, train_rows=262144, iters=8)
ctx.sync()
emit(shape=dict(rows=rows, nlist=nlist, nprobe=nprobe, top_k=top_k, rerank=rerank, nq=NQ), stats=index.stats())

rng = np.random.default_rng(5)
lens = np.clip(np.round(rng.lognormal(3.0, 1.0, rows)), 1, 200).astype(np.int64)
doc_start = np.concatenate([[0], np.cumsum(lens)])
doc_start = doc_start[doc_start < rows]
doc_end = np.append(doc_start[1:], rows)
n_docs = len(doc_start)


def doc_subset(frac):
    """Global ranges of a random set of documents, adjacent documents merged (as Store._ranges_for)."""
    keep = rng.random(n_docs) < frac
    m = np.zeros(rows + 1, np.int32)
    m[doc_start[keep]] += 1
    m[doc_end[keep]] -= 1
    on = np.cumsum(m)[:rows] > 0
    edges = np.flatnonzero(np.diff(np.concatenate([[0], on.astype(np.int8), [0]])))
    return edges.reshape(-1, 2).astype(np.uint64)


def call(subsets, subset_of):
    return index.search_subsets(Q, subsets, subset_of, nprobe=nprobe, top_k=top_k, rerank=rerank)


def loop(subsets, subset_of):
    hits = np.zeros((NQ, top_k), dtype=capi.HIT_DTYPE)
    n = np.zeros(NQ, np.uint32)
    sc = np.zeros(NQ, np.uint64)
    for s in np.unique(subset_of):
        sel = np.flatnonzero(subset_of == s)
        hits[sel], n[sel], sc[sel] = index.search_filtered(Q[sel], subsets[s], nprobe=nprobe, top_k=top_k, rerank=rerank)
    return hits, n, sc


def median_s(fn):
    fn()
    t = []
    for _ in range(3):
        t0 = time.perf_counter(); fn(); t.append(time.perf_counter() - t0)
    return float(np.median(t))


def device_ms(fn):
    """Device time of one run of fn (every kernel, copy and memset), and the ivff_* kernels' part of it."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        ctx.sync()
    tot = elig = 0.0
    for e in prof.key_averages():
        tot += e.device_time_total
        if "ivff_" in e.key:
            elig += e.device_time_total
    return tot / 1e3, elig / 1e3


def recall(got_rows, exact_rows):
    if len(exact_rows) == 0:
        return 1.0
    return len(set(got_rows) & set(exact_rows)) / len(exact_rows)


for frac in FRACS:
    for G in GROUPS:
        subsets = [doc_subset(frac) for _ in range(G)]
        subset_of = rng.integers(0, G, NQ).astype(np.uint32)
        a, b = call(subsets, subset_of), loop(subsets, subset_of)
        same = all(a[0][i].tobytes() == b[0][i].tobytes() and a[1][i] == b[1][i] and a[2][i] == b[2][i] for i in range(NQ))
        exact = [c.search(Q[i], top_k, None, capi.STB_MODE_STORE_QUERY, row_ranges=subsets[subset_of[i]])["row"].tolist()
                 for i in range(NQ)]
        rec = float(np.mean([recall(a[0][i]["row"][: a[1][i]].tolist(), exact[i]) for i in range(NQ)]))
        t_call, t_loop = median_s(lambda: call(subsets, subset_of)), median_s(lambda: loop(subsets, subset_of))
        d_call, e_call = device_ms(lambda: call(subsets, subset_of))
        d_loop, e_loop = device_ms(lambda: loop(subsets, subset_of))
        emit(frac=frac, G=G, ranges_per_subset=int(np.mean([len(s) for s in subsets])), bit_equal=bool(same),
             recall_at_10=round(rec, 4), qps_call=round(NQ / t_call, 1), qps_loop=round(NQ / t_loop, 1),
             ms_call=round(t_call * 1e3, 3), ms_loop=round(t_loop * 1e3, 3),
             device_ms_call=round(d_call, 3), device_ms_loop=round(d_loop, 3),
             eligibility_ms_call=round(e_call, 3), eligibility_ms_loop=round(e_loop, 3),
             host_share_call=round(max(0.0, 1.0 - d_call / (t_call * 1e3)), 3))
        if not same:
            sys.exit("the call and the per-subset loop differ")
index.close(); c.close()

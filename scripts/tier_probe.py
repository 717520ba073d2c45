"""K1 candidate tiers on one GPU: pipelined device-timed us/query (stb_search_topk_dev, PDL) and
synchronous end-to-end ms/query (stb_search, host query in / host hits out) per tier, plus the
row-range (workspace path filter) mode.  Every result is compared bit for bit with the f32 tier.
    python scripts/tier_probe.py [rows] [iters] [k]"""
import json, os, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from semtools_b200 import capi
rows = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 64
k = int(sys.argv[3]) if len(sys.argv) > 3 else 10
dev = torch.device("cuda:0")
s = torch.cuda.Stream(dev); torch.cuda.set_stream(s)
ctx = capi.Context(0, s.cuda_stream)
g = torch.Generator(device=dev); g.manual_seed(1)
c = capi.Corpus(ctx, rows)
for i in range(0, rows, 1_000_000):
    n = min(1_000_000, rows - i)
    x = torch.randn((n, 256), generator=g, device=dev); x /= x.norm(dim=1, keepdim=True)
    torch.cuda.synchronize(); c.append_dev(x.data_ptr(), n)
del x
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(s); c.prepare(1); e1.record(s); torch.cuda.synchronize(); q8_ms = e0.elapsed_time(e1)
e0.record(s); c.prepare(2); e1.record(s); torch.cuda.synchronize(); h16_ms = e0.elapsed_time(e1)
nq = 32
q = torch.randn((nq, 256), generator=g, device=dev); q /= q.norm(dim=1, keepdim=True)
qh = q.cpu().numpy()
out = {"rows": rows, "k": k, "build_ms": {"q8": q8_ms, "h16": h16_ms}}
ref = None
BYTES = {"f32": 1024, "h16": 512, "q8": 260}
for tier in ("f32", "h16", "q8"):
    os.environ["STB_SCAN_TIER"] = tier
    hits = torch.zeros((nq, k, 2), dtype=torch.float64, device=dev); st = torch.zeros((nq, 4), dtype=torch.int32, device=dev)
    for i in range(nq):
        c.search_topk_dev(q[i].data_ptr(), k, hits[i].data_ptr(), st[i].data_ptr())
    torch.cuda.synchronize()
    e0.record(s)
    for i in range(iters):
        c.search_topk_dev(q[i % nq].data_ptr(), k, hits[i % nq].data_ptr(), st[i % nq].data_ptr())
    e1.record(s); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / iters * 1e3
    sth = st.cpu().numpy()
    if ref is None:
        ref = hits.clone()
    proven = sth[:, 1] == 1
    same = bool(torch.equal(hits.view(torch.int64)[torch.from_numpy(proven).to(dev)], ref.view(torch.int64)[torch.from_numpy(proven).to(dev)]))
    for i in range(3):
        c.search(qh[i], top_k=k)
    t0 = time.perf_counter()
    for i in range(iters):
        c.search(qh[i % nq], top_k=k)
    e2e_ms = (time.perf_counter() - t0) / iters * 1e3
    out[tier] = {"us_per_query_pipelined": us, "GBps_read": rows * BYTES[tier] / us / 1e3, "proven": int(proven.sum()), "of": nq,
                 "tier_seen": int(sth[0, 3] >> 16), "kprime": int(sth[0, 3] & 0xffff), "proven_hits_equal_f32": same, "e2e_ms": e2e_ms}
# row ranges: 20k scattered ranges (~25% of the rows) and one full range, per tier, end to end
rng = np.random.default_rng(0)
if rows >= 1_000_000:
    starts = np.sort(rng.choice(np.arange(0, rows - 200, 200), min(20_000, rows // 400), replace=False))
    ranges = np.stack([starts, starts + rng.integers(50, 200, len(starts))], axis=1).astype(np.uint64)
    sel = int((ranges[:, 1] - ranges[:, 0]).sum())
    out["ranges"] = {"n_ranges": len(ranges), "rows_selected": sel}
    want = None
    for tier in ("f32", "h16", "q8"):
        os.environ["STB_SCAN_TIER"] = tier
        res = {}
        for name, rr in (("many", ranges), ("one", np.array([[0, rows]], dtype=np.uint64))):
            for i in range(2):
                got = c.search(qh[i], top_k=k, mode=capi.STB_MODE_STORE_QUERY, row_ranges=rr)
            t0 = time.perf_counter()
            for i in range(16):
                got = c.search(qh[i % nq], top_k=k, mode=capi.STB_MODE_STORE_QUERY, row_ranges=rr)
            ms = (time.perf_counter() - t0) / 16 * 1e3
            n_sel = sel if name == "many" else rows
            res[name + "_ms"] = ms
            res[name + "_GBps_of_selected_f32_rows"] = n_sel * 1024 / ms / 1e6
            if name == "many":
                if want is None:
                    want = got
                res["same_as_f32"] = bool(np.array_equal(got, want))
        out["ranges"][tier] = res
out["tier_stats"] = c.tier_stats()
print(json.dumps(out))

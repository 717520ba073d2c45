"""Host-rows corpora (stb_corpus_create_host) on one GPU: what keeping the f32 rows in host memory costs, and
how far past the HBM limit it goes.

1. Same rows, both placements: --rows (default 10M) seeded unit rows on a device corpus (q8 copy prepared) and on a
   host-rows corpus, in one run; the same query series alternates between the two.  Reports q/s for top_k = 10 (the
   q8 top-k scan), top_k = 50 (the q8 histogram / collect route) and a threshold query, the extra latency per query
   of the host corpus (the K1 re-rank reading its candidate rows over the host link), append throughput, and checks
   that every hit is identical.
2. Past the HBM limit: --big rows (default 64M; 100M when the host has the memory) that the device cannot hold with
   their q8 copy, appended in chunks of 1M rows (never one full matrix in numpy).  Reports append time, first-query
   time and steady q/s at top_k = 10, and checks a few timed queries against an exact f64 scan of
   stb_corpus_read chunks.  The pinned rows may take at most half of MemAvailable (the host is shared); a size that
   does not fit is reported as "not measured".

Prints one JSON object; the card's name and power limit are read in the same run.
Usage: python scripts/host_rows_probe.py [--rows 10000000] [--big 0|64000000|100000000] [--queries 200]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from semtools_b200 import capi  # noqa: E402

CHUNK = 1 << 20


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,memory.total", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, mem = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "memory": mem}
    except Exception as e:  # noqa: BLE001 - reported, not hidden
        return {"error": repr(e)}


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def unit_chunk(seed, n):
    """n seeded unit rows (f32), generated on the GPU and returned in host memory"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((n, 256), generator=g, device="cuda", dtype=torch.float32)
    x /= x.norm(dim=1, keepdim=True)
    return x.cpu().numpy()


def chunks(total, seed):
    for i, r0 in enumerate(range(0, total, CHUNK)):
        yield unit_chunk(seed * 100003 + i, min(CHUNK, total - r0))


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return out, time.perf_counter() - t


def same(a, b):
    return len(a) == len(b) and np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def placements(ctx, n, nq, reps):
    dev = capi.Corpus(ctx, n)
    host = capi.Corpus.in_host_memory(ctx, n)
    t_dev = t_host = 0.0
    for part in chunks(n, 1):
        t_dev += timed(lambda: dev.append(part))[1]
        t_host += timed(lambda: host.append(part))[1]
    dev.prepare(1)                                       # STB_PREPARE_Q8
    rng = np.random.default_rng(2)
    qs = rng.standard_normal((nq, 256)).astype(np.float32)
    qs /= np.linalg.norm(qs, axis=1, keepdims=True)
    kinds = {"top_k=10": dict(top_k=10), "top_k=50": dict(top_k=50), "threshold<0.72": dict(top_k=0, max_distance=0.72)}
    res = {k: {"device": [], "host": []} for k in kinds}
    identical = True
    for kind, kw in kinds.items():
        for c in (dev, host):                                  # warm-up of every shape
            c.search(qs[0], **kw)
        for _ in range(reps):
            hits = {}
            for name, c in (("device", dev), ("host", host)):
                t = time.perf_counter()
                hits[name] = [c.search(q, **kw) for q in qs]
                res[kind][name].append(nq / (time.perf_counter() - t))
            identical &= all(same(a, b) for a, b in zip(hits["device"], hits["host"]))
    fb = ctx.counters()["fallback_searches"]
    out = {"rows": n, "queries_per_series": nq, "series": reps, "identical": bool(identical),
           "append_rows_per_s": {"device": n / t_dev, "host": n / t_host},
           "host_tier_stats": host.tier_stats(), "fallback_searches": fb}
    for kind in kinds:
        d, h = float(np.median(res[kind]["device"])), float(np.median(res[kind]["host"]))
        out[kind] = {"device_qps": d, "host_qps": h, "host_extra_us_per_query": (1.0 / h - 1.0 / d) * 1e6}
    # update / remove cost on the host corpus (10k rows)
    idx = np.sort(rng.choice(n, 10000, replace=False)).astype(np.uint64)
    new = unit_chunk(7, 10000)
    out["update_10k_rows_s"] = {"device": timed(lambda: dev.update(idx, new))[1], "host": timed(lambda: host.update(idx, new))[1]}
    rr = np.array([[n // 2, n // 2 + 10000]], dtype=np.uint64)
    out["remove_10k_rows_at_half_s"] = {"device": timed(lambda: dev.remove(rr))[1], "host": timed(lambda: host.remove(rr))[1]}
    dev.close()
    host.close()
    return out


def exact_top(host, qs, k):
    """exact f64 top-k of every query from stb_corpus_read chunks: (row, distance) lists"""
    n = len(host)
    qd = qs.astype(np.float64)
    qn = np.sqrt((qd * qd).sum(1))
    best = [[] for _ in qs]
    for r0 in range(0, n, CHUNK):
        rows = host.read(r0, min(CHUNK, n - r0)).astype(np.float64)
        rn = np.sqrt((rows * rows).sum(1))
        d = 1.0 - (rows @ qd.T) / (rn[:, None] * qn[None, :])
        for j in range(len(qs)):
            top = np.argpartition(d[:, j], k)[:k]
            best[j] += [(float(d[t, j]), r0 + int(t)) for t in top]
    return [sorted(b)[:k] for b in best]


def past_the_limit(ctx, big, nq):
    need = big * 1024
    avail = mem_available()
    if need > avail // 2:
        return {"rows": big, "status": "not measured",
                "reason": f"pinned rows need {need / 2**30:.1f} GiB, more than half of MemAvailable ({avail / 2**30:.1f} GiB)"}
    host, t = timed(lambda: capi.Corpus.in_host_memory(ctx, big))
    t_append = t
    for part in chunks(big, 3):
        t_append += timed(lambda: host.append(part))[1]
    rng = np.random.default_rng(4)
    qs = rng.standard_normal((nq, 256)).astype(np.float32)
    qs /= np.linalg.norm(qs, axis=1, keepdims=True)
    first, t_first = timed(lambda: host.search(qs[0], 10))
    t = time.perf_counter()
    hits = [host.search(q, 10) for q in qs]
    qps = nq / (time.perf_counter() - t)
    check = exact_top(host, qs[:3], 10)
    ok = all(np.array_equal(h["row"], [r for _, r in e]) and np.allclose(h["distance"], [d for d, _ in e], rtol=0, atol=1e-12)
             for h, e in zip(hits[:3], check))
    out = {"rows": big, "append_s": t_append, "append_rows_per_s": big / t_append, "first_query_s": t_first,
           "top_k=10_qps": qps, "checked_queries": 3, "exact_match": bool(ok), "tier_stats": host.tier_stats(),
           "mem_available_gib": avail / 2**30}
    host.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--big", type=int, default=-1, help="-1: 100M if the host holds it, else 64M; 0: skip")
    ap.add_argument("--queries", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    ctx = capi.Context(0)
    out = {"card": card(), "placements": placements(ctx, a.rows, a.queries, a.reps)}
    big = a.big
    if big < 0:
        big = 100_000_000 if 100_000_000 * 1024 <= mem_available() // 2 else 64_000_000
    if big:
        out["past_hbm"] = past_the_limit(ctx, big, 50)
    out["card_after"] = card()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

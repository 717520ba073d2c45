#!/usr/bin/env python3
"""Cost of changing rows of a resident corpus in place (stb_corpus_update / stb_corpus_remove) against the
path a host without them takes (clear, append every row from host memory, prepare the candidate copies),
and the first top-k query after each.  10M rows, both copies built.  Times are device events on the
context's stream after a warm-up of every call shape.  Prints one JSON line (also written to --out).

    python scripts/corpus_update_probe.py [--rows 10000000] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from semtools_b200 import capi  # noqa: E402

CHUNK = 1 << 20


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    n = args.rows
    ctx = capi.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    g = torch.Generator(device="cuda").manual_seed(0)
    rng = np.random.default_rng(0)
    host = rng.standard_normal((min(n, CHUNK), 256)).astype(np.float32)   # host rows of the re-upload path
    host /= np.linalg.norm(host, axis=1, keepdims=True)
    qs = host[rng.choice(len(host), 16, replace=False)] + np.float32(0.1) * host[:16]

    def timed(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        return a.elapsed_time(b)

    def fill(c):
        c.clear()
        for i in range(0, n, CHUNK):
            m = min(CHUNK, n - i)
            x = torch.randn((m, 256), generator=g, device="cuda")
            x /= x.norm(dim=1, keepdim=True)
            torch.cuda.synchronize()
            c.append_dev(x.data_ptr(), m)
        c.prepare(3)

    def reupload(c):
        c.clear()
        for i in range(0, n, CHUNK):
            c.append(host[: min(CHUNK, n - i)])

    q_i = [0]

    def query(c):
        q_i[0] += 1
        return timed(lambda: c.search(qs[q_i[0] % len(qs)], top_k=10))

    c = capi.Corpus(ctx, n)
    fill(c)
    res = {"card": card(), "rows": n, "update": {}, "remove": {}, "today": {}}
    # warm-up of every call shape
    c.update(np.array([0], dtype=np.uint64), host[:1])
    c.remove(np.array([[n - 1, n]], dtype=np.uint64))
    c.append(host[:1])
    query(c)
    for m in (1, 1024, 16384, 262144):
        idx = np.sort(rng.choice(len(c), m, replace=False)).astype(np.uint64)
        rows = np.ascontiguousarray(host[:m])
        ms = timed(lambda: c.update(idx, rows))
        st = c.tier_stats()
        res["update"][str(m)] = {"ms": ms, "first_query_ms": query(c), "q8_rows": st["q8"]["built_rows"], "rows": len(c)}
        print("update", m, res["update"][str(m)], flush=True)
    cases = {
        "1000 rows near the start": np.array([[1000, 2000]], dtype=np.uint64),
        "10% scattered": None,
        "1000 rows near the end": "end",
    }
    for name, ranges in cases.items():
        cur = len(c)
        if isinstance(ranges, str):
            ranges = np.array([[cur - 5000, cur - 4000]], dtype=np.uint64)
        if ranges is None:
            starts = np.arange(0, cur - 100, 1000, dtype=np.uint64) + np.uint64(37)
            ranges = np.stack([starts, starts + np.uint64(100)], axis=1)
            ranges[-1, 1] = min(int(ranges[-1, 1]), cur)
        ms = timed(lambda: c.remove(ranges))
        removed = int((ranges[:, 1] - ranges[:, 0]).sum())
        moved = cur - int(ranges[0, 0]) - removed
        st = c.tier_stats()
        res["remove"][name] = {"ms": ms, "removed": removed, "moved_rows": moved, "first_query_ms": query(c),
                               "q8_rows": st["q8"]["built_rows"], "rows": len(c)}
        print("remove", name, res["remove"][name], flush=True)
    # today: clear + append every row from host memory, the first query (f32 tier), prepare, the next query
    t = res["today"]
    t["clear_append_ms"] = timed(lambda: reupload(c))
    t["first_query_ms"] = query(c)
    t["prepare_ms"] = timed(lambda: c.prepare(3))
    t["query_after_prepare_ms"] = query(c)
    print("today", t, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

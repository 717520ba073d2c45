"""K2 route 7 at the size it exists for: a device corpus whose 16-bit shadow does not fit in HBM.

Builds a seeded device corpus of --rows (default 45M) unit rows generated on the GPU (46 GB of f32 rows and 18 GB
of q8 copy and nibble plane: the 23 GB shadow does not fit beside them on an 80 GB card), shows that
stb_corpus_prepare_batch is refused with STB_ERR_NOMEM, then runs stb_search_batch on --queries (default 1024)
queries at top_k = 10, which takes route 7.  Every query is checked bit for bit against stb_search.  Reports the
batch's q/s against stb_search_many over the same queries, the share of queries proven on the tensor cores, and the
rows emitted per query (the finish's re-score count is not exposed; it is at most the emitted count).

A host-rows corpus past 88M rows (where its shadow stops fitting) needs ~100 GB of page-locked host memory; the
probe reports it as "not measured" when MemAvailable is below that.

Prints one JSON object; the card's name and power limit are read in the same run.
Usage: python scripts/batch_q8_probe.py [--rows 45000000] [--queries 1024] [--reps 3]
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


def mem_available_gib():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) / 2**20
    return 0.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=45_000_000)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch

    out = {"card": card(), "rows": args.rows, "queries": args.queries, "top_k": 10}
    ctx = capi.Context(0)
    corpus = capi.Corpus(ctx, args.rows)
    g = torch.Generator(device="cuda").manual_seed(20261017)
    t0 = time.perf_counter()
    for r0 in range(0, args.rows, CHUNK):
        m = min(CHUNK, args.rows - r0)
        x = torch.randn((m, 256), generator=g, device="cuda", dtype=torch.float32)
        x /= x.norm(dim=1, keepdim=True)
        torch.cuda.synchronize()
        corpus.append_dev(x.data_ptr(), m)
        ctx.sync()
        del x
    queries = torch.randn((args.queries, 256), generator=g, device="cuda", dtype=torch.float32)
    queries /= queries.norm(dim=1, keepdim=True)
    queries = queries.cpu().numpy()
    torch.cuda.empty_cache()
    out["append_s"] = round(time.perf_counter() - t0, 2)
    t0 = time.perf_counter()
    corpus.prepare(1)                                        # the q8 copy
    out["q8_build_s"] = round(time.perf_counter() - t0, 2)
    out["free_gib_after_q8"] = round(torch.cuda.mem_get_info()[0] / 2**30, 2)
    try:
        corpus.prepare_batch()
        out["prepare_batch"] = "built (the shadow fits: this size does not exercise route 7)"
    except capi.StbError as e:
        out["prepare_batch"] = {"status": e.status, "nomem": e.status == capi.STB_ERR_NOMEM}

    k = 10
    fb0 = ctx.counters()["fallback_searches"]
    got = corpus.search_batch(queries, k)                    # first call: route 7, q8 copy already built
    info = ctx.batch_last()
    out["route"] = info["route"]
    out["n_sample"], out["stride"], out["n_seg"] = info["n_sample"], info["stride"], info["n_seg"]
    out["proven"] = args.queries - (ctx.counters()["fallback_searches"] - fb0)
    if "cand_cnt" in info:
        emitted = np.minimum(info["cand_cnt"], info["seg_cap"]).sum(axis=1)
        out["emitted_per_query"] = {"mean": float(emitted.mean()), "max": int(emitted.max())}
        out["overflowed_queries"] = int((info["cand_cnt"] > info["seg_cap"]).any(axis=1).sum())
    times = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        again = corpus.search_batch(queries, k)
        times.append(time.perf_counter() - t0)
    out["batch_s"] = [round(t, 4) for t in times]
    out["batch_qps"] = round(args.queries / float(np.median(times)), 1)
    times = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        many = corpus.search_many(queries, k)
        times.append(time.perf_counter() - t0)
    out["search_many_s"] = [round(t, 4) for t in times]
    out["search_many_qps"] = round(args.queries / float(np.median(times)), 1)
    mismatch = 0
    for i in range(args.queries):
        ref = corpus.search(queries[i], k)
        for a in (got[i], again[i], many[i]):
            if len(a) != len(ref) or not np.array_equal(np.ascontiguousarray(a).view(np.uint8), ref.view(np.uint8)):
                mismatch += 1
    out["mismatched_results"] = mismatch
    avail = mem_available_gib()
    out["host_rows_past_88M"] = "not measured" if avail < 100 else "not run by this probe"
    out["host_mem_available_gib"] = round(avail, 1)
    corpus.close()
    ctx.close()
    print(json.dumps(out))
    if mismatch:
        sys.exit(1)


if __name__ == "__main__":
    main()

"""K2 routes 8, 9 and 10 at the size they exist for: a device corpus whose 16-bit shadow does not fit in HBM.

Builds a seeded device corpus of --rows (default 45M) unit rows generated on the GPU, shows that
stb_corpus_prepare_batch is refused with STB_ERR_NOMEM, then times on --queries (default 1024) queries at top_k = 10:
- stb_search_batch_filtered (route 8) over document subsets of 25, 5 and 1 % of the rows, and at top_k = 64 over
  the 25 % subset, where the shadow's v2 plan does not fit but the q8 plan does;
- stb_search_batch_subsets (route 9) with 16 and 64 groups, each a 5 % document subset of its own, and 16 groups at
  top_k = 64;
- stb_search_batch_threshold (route 10) at distances giving about 1, 100 and 5000 hits per query (read off the
  N(0, 1/256) distribution of a random unit row's cosine).
Each against K1 one query at a time (stb_search with the same arguments), which is also the reference: every query
is checked bit for bit.  At top_k = 64 the reference runs with STB_SCAN_TIER=f32: K1's default ladder would ask for
the 16-bit shadow there (its q8 tier serves top_k <= 16), which does not fit; the probe reports what that returns.  Documents are runs of consecutive rows with lognormal lengths (mean ~30), as a workspace
stores lines.

Prints one JSON object; the card's name and power limit are read in the same run.
Usage: python scripts/batch_q8_modes_probe.py [--rows 45000000] [--queries 1024] [--reps 2]
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


def doc_ranges(rng, n, frac, mean_len=30):
    """A random subset of documents (lognormal lengths, consecutive rows) as sorted [begin, end) ranges."""
    lens = np.clip(np.round(rng.lognormal(np.log(mean_len), 0.8, n // 10)), 1, 200).astype(np.int64)
    starts = np.concatenate([[0], np.cumsum(lens)])
    starts = starts[starts < n]
    ends = np.append(starts[1:], n)
    keep = rng.random(len(starts)) < frac
    return np.stack([starts[keep], ends[keep]], axis=1).astype(np.uint64)


def same(a, b):
    return len(a) == len(b) and np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def timed(fn, reps):
    res, times = None, []
    for _ in range(reps):
        t0 = time.perf_counter()
        res = fn()
        times.append(time.perf_counter() - t0)
    return res, float(np.median(times))


def run_mode(ctx, nq, batch, k1_one, reps, k1_tier=None):
    """(batch result, its q/s, K1's q/s, mismatches, route record, queries K1 answered inside the batch call).
    k1_tier: STB_SCAN_TIER for the reference calls (results are identical whatever the tier)."""
    fb0 = ctx.counters()["fallback_searches"]
    try:
        got, t_batch = timed(batch, reps)
    except capi.StbError as e:                              # reported, not hidden
        return {"batch_error": {"status": e.status, "error": str(e)[:200]}, "route": ctx.batch_last()["route"]}
    info = ctx.batch_last()
    fell = (ctx.counters()["fallback_searches"] - fb0) // reps
    if k1_tier:
        os.environ["STB_SCAN_TIER"] = k1_tier
    t0 = time.perf_counter()
    try:
        refs = [k1_one(i) for i in range(nq)]
    finally:
        os.environ.pop("STB_SCAN_TIER", None)
    t_k1 = time.perf_counter() - t0
    bad = sum(not same(got[i], refs[i]) for i in range(nq))
    rec = {key: v for key, v in info.items() if key not in ("thr", "cand_cnt")}
    return {"batch_qps": round(nq / t_batch, 1), "k1_qps": round(nq / t_k1, 1), "mismatched": bad, "route": rec,
            "fallback_searches_per_call": int(fell), "k1_tier": k1_tier or "default"}


def k1_default_tier(fn):
    """K1 at its default tier ladder: "ok", or the error it returns (top_k > 16 asks for the 16-bit shadow)."""
    try:
        fn()
        return "ok"
    except capi.StbError as e:
        return {"status": e.status, "error": str(e)[:200]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=45_000_000)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    import torch
    from scipy.stats import norm

    n, nq, k = args.rows, args.queries, 10
    out = {"card": card(), "rows": n, "queries": nq, "top_k": k}
    ctx = capi.Context(0)
    corpus = capi.Corpus(ctx, n)
    g = torch.Generator(device="cuda").manual_seed(20261018)
    for r0 in range(0, n, CHUNK):
        m = min(CHUNK, n - r0)
        x = torch.randn((m, 256), generator=g, device="cuda", dtype=torch.float32)
        x /= x.norm(dim=1, keepdim=True)
        torch.cuda.synchronize()
        corpus.append_dev(x.data_ptr(), m)
        ctx.sync()
        del x
    queries = torch.randn((nq, 256), generator=g, device="cuda", dtype=torch.float32)
    queries /= queries.norm(dim=1, keepdim=True)
    queries = np.ascontiguousarray(queries.cpu().numpy())
    torch.cuda.empty_cache()
    corpus.prepare(1)                                        # the q8 copy
    try:
        corpus.prepare_batch()
        out["prepare_batch"] = "built (the shadow fits: this size does not exercise routes 8-10)"
    except capi.StbError as e:
        out["prepare_batch"] = {"status": e.status, "nomem": e.status == capi.STB_ERR_NOMEM}

    rng = np.random.default_rng(7)
    store = capi.STB_MODE_STORE_QUERY
    for frac in (0.25, 0.05, 0.01):
        rr = doc_ranges(rng, n, frac)
        out[f"filtered_{int(frac * 100)}pct"] = run_mode(
            ctx, nq, lambda: corpus.search_batch_filtered(queries, rr, top_k=k),
            lambda i: corpus.search(queries[i], top_k=k, mode=store, row_ranges=rr), args.reps)
        if frac == 0.25:
            # top_k = 64: the shadow's v2 plan does not fit here, the q8 plan does
            out["filtered_25pct_k64"] = run_mode(
                ctx, nq, lambda: corpus.search_batch_filtered(queries, rr, top_k=64),
                lambda i: corpus.search(queries[i], top_k=64, mode=store, row_ranges=rr), args.reps, "f32")
            out["filtered_25pct_k64"]["k1_default_tier"] = k1_default_tier(
                lambda: corpus.search(queries[0], top_k=64, mode=store, row_ranges=rr))
    for groups in (16, 64):
        lists = [doc_ranges(rng, n, 0.05) for _ in range(groups)]
        per = [lists[i % groups] for i in range(nq)]
        out[f"subsets_{groups}_groups"] = run_mode(
            ctx, nq, lambda: corpus.search_batch_subsets(queries, per, top_k=k),
            lambda i: corpus.search(queries[i], top_k=k, mode=store, row_ranges=per[i]), args.reps)
        if groups == 16:
            out["subsets_16_groups_k64"] = run_mode(
                ctx, nq, lambda: corpus.search_batch_subsets(queries, per, top_k=64),
                lambda i: corpus.search(queries[i], top_k=64, mode=store, row_ranges=per[i]), args.reps, "f32")
    for hits in (1, 100, 5000):
        m = 1.0 - norm.isf(hits / n) / 16.0                 # cosine of a random unit row ~ N(0, 1/256)
        res = run_mode(ctx, nq, lambda: corpus.search_batch_threshold(queries, m, cap=nq * hits * 4),
                       lambda i: corpus.search(queries[i], top_k=0, max_distance=m), args.reps)
        res["max_distance"] = m
        out[f"threshold_{hits}_hits"] = res
    corpus.close()
    ctx.close()
    print(json.dumps(out))
    if any(isinstance(v, dict) and (v.get("mismatched") or v.get("batch_error")) for v in out.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()

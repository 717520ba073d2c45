"""K1 pairs (scan_topk.cu: "pairs") on bench.py's corpus and queries (imported from it): --queries pipelined q8
stb_search_topk_dev calls at --rows and --rows2 rows.  Per corpus it reports
  ms_per_query           CUDA events around the pipelined series (after --warmup untimed queries)
  joined_share           guests that joined their host, and the median join tile (stb_debug_pair_joins, read
                         in a second series synchronised every 8 launches, so its first pair of each 8 is typical)
  plane_tiles_per_query  plane tiles read per query, counted from the tickets: a host reads every tile for two
                         queries, a joined guest adds the tiles before its join tile (the guest-only wrap), a
                         refused one every tile; with the refined rows (stb_debug_q4_refined) it gives the bytes
                         per query: 136 B per plane row + 260 B per refined row
  kernels                mean time per launch of each kernel, from a separate torch.profiler run
and the card's name and power limit, read in the same process.  Needs a GPU.

    python scripts/pair_probe.py [--rows 10000000] [--rows2 1000000] [--queries 200] [--out FILE]
"""
import argparse
import collections
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TILE_ROWS = 32
PLANE_ROW_BYTES, CODE_ROW_BYTES = 136, 260


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--rows2", type=int, default=1_000_000)
    ap.add_argument("--topk", type=int, default=10)
    ap.add_argument("--queries", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    import bench
    from semtools_b200 import capi

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    ctx = capi.Context(0, stream.cuda_stream)
    cnt = ctypes.c_uint64(0)

    def refined(reset):
        capi._check(capi.lib().stb_debug_q4_refined(ctx._h, reset, ctypes.byref(cnt)))
        return int(cnt.value)

    n_q, warm, k = a.queries, a.warmup, a.topk
    qs = torch.from_numpy(bench.gen_queries(64)).to(dev)
    hits = torch.zeros((n_q + warm, k, 2), dtype=torch.float64, device=dev)
    st = torch.zeros((n_q + warm, 4), dtype=torch.int32, device=dev)
    results = {"card": card, "queries": n_q}
    for rows in (a.rows, a.rows2):
        if rows <= 0:
            continue
        corpus, _, _ = bench.fill_shard(torch, dev, capi, ctx, rows, 1, 0)
        corpus.prepare(1)
        n_tiles = -(-rows // TILE_ROWS)

        def launch(i):
            corpus.search_topk_dev(qs[i % 64].data_ptr(), k, hits[i].data_ptr(), st[i].data_ptr())

        for i in range(warm):
            launch(i)
        torch.cuda.synchronize(dev)
        refined(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for i in range(warm, warm + n_q):
            launch(i)
        e1.record(stream)
        torch.cuda.synchronize(dev)
        ref_rows = refined(1) / n_q
        s = st[warm:].cpu().numpy()
        rec = {"rows": rows, "tier": bench.TIER_NAMES[int(s[0, 3]) >> 16], "ms_per_query": round(e0.elapsed_time(e1) / n_q, 4),
               "all_proven": bool((s[:, 1] == 1).all()), "refined_rows_per_query": round(ref_rows)}

        # joins: the same series in groups of 8 launches, each group read back
        joins = []
        ctx.sync()
        for g in range(0, n_q, 8):
            m = min(8, n_q - g)
            for i in range(g, g + m):
                launch(warm + i)
            joins += ctx.pair_joins(m)
        guests = joins[1::2]
        joined = [j for j in guests if isinstance(j, int)]
        tiles = (len(joins) - len(guests)) * n_tiles + sum(joined) + (len(guests) - len(joined)) * n_tiles
        rec.update({"guests": len(guests), "joined_share": round(len(joined) / max(len(guests), 1), 3),
                    "median_join_tile": statistics.median(joined) if joined else None,
                    "plane_tiles_per_query": round(tiles / len(joins), 1), "n_tiles": n_tiles})
        rec["gb_per_query"] = round((rec["plane_tiles_per_query"] * TILE_ROWS * PLANE_ROW_BYTES + ref_rows * CODE_ROW_BYTES) / 1e9, 4)

        # kernel times: a separate profiled series
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(warm, warm + min(n_q, 64)):
                launch(i)
            torch.cuda.synchronize(dev)
        per = collections.defaultdict(list)
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA and "stb_" in ev.name:
                per[ev.name.split("(")[0].split("<")[0]].append(ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total)
        rec["kernels_us"] = {n: {"launches": len(v), "mean_us": round(sum(v) / len(v), 1)} for n, v in per.items()}
        print(json.dumps(rec), flush=True)
        results[str(rows)] = rec
        del corpus
        torch.cuda.synchronize(dev)
    print(json.dumps(results), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(results) + "\n")


if __name__ == "__main__":
    main()

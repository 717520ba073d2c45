"""K1 co-scan against the launch modes it replaces, on bench.py's corpus and queries (imported from it).

Each mode runs in a subprocess of its own, because the library path is fixed when it is first loaded:
  full     the parent commit (--parent-root: a checkout with its library built, loaded through
           STB_LIB_PATH with that checkout's bindings): full grid, one query per pass
  coscan   this build: overlapped grids, each query starting where its predecessor reads
  NAME     --extra NAME=PATH: another build of this tree (e.g. another ticket size), co-scan
The modes alternate over --rounds rounds.  Each subprocess builds the headline corpus (--rows) and
the config-2 corpus (--rows2) and times --queries pipelined stb_search_topk_dev calls with CUDA events
per tier (q8, h16, f32), after --warmup untimed ones.  Prints one JSON line per measurement and a
summary line with the card, its power limit and maximum SM clock (also written to --out).  Needs a GPU.

    python scripts/coscan_probe.py --parent-root DIR [--extra NAME=PATH ...] [--rounds 3] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def worker(a):
    import torch
    import bench
    from semtools_b200 import capi

    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    ctx = capi.Context(0, stream.cuda_stream)
    cnt = ctypes.c_uint64(0)

    def refined(reset):
        capi._check(capi.lib().stb_debug_q4_refined(ctx._h, reset, ctypes.byref(cnt)))
        return int(cnt.value)

    n_q, warm = a.queries, a.warmup
    qs = torch.from_numpy(bench.gen_queries(64)).to(dev)
    hits = torch.zeros((n_q + warm, a.topk, 2), dtype=torch.float64, device=dev)
    st = torch.zeros((n_q + warm, 4), dtype=torch.int32, device=dev)
    for rows in (a.rows, a.rows2):
        if rows <= 0:
            continue
        corpus, _, _ = bench.fill_shard(torch, dev, capi, ctx, rows, 1, 0)
        corpus.prepare(1)
        for tier in a.tiers.split(","):
            os.environ["STB_SCAN_TIER"] = tier
            for i in range(warm):
                corpus.search_topk_dev(qs[i % 64].data_ptr(), a.topk, hits[i].data_ptr(), st[i].data_ptr())
            torch.cuda.synchronize(dev)
            refined(1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for i in range(warm, warm + n_q):
                corpus.search_topk_dev(qs[i % 64].data_ptr(), a.topk, hits[i].data_ptr(), st[i].data_ptr())
            e1.record(stream)
            torch.cuda.synchronize(dev)
            s = st[warm:].cpu().numpy()
            out = {"mode": a.mode, "rows": rows, "tier": bench.TIER_NAMES[int(s[0, 3]) >> 16],
                   "ms_per_query": e0.elapsed_time(e1) / n_q, "all_proven": bool((s[:, 1] == 1).all()),
                   "refined_rows_per_query": refined(1) / n_q}
            if hasattr(ctx, "coscan_offsets"):
                out["last_offsets"] = ctx.coscan_offsets(4)
            print(json.dumps(out), flush=True)
        os.environ.pop("STB_SCAN_TIER", None)
        del corpus
        torch.cuda.synchronize(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-root", default=None, help="a built checkout of the parent commit (mode full)")
    ap.add_argument("--extra", action="append", default=[], help="NAME=PATH: another co-scan build to time")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--rows2", type=int, default=1_000_000)
    ap.add_argument("--tiers", default="q8,h16,f32")
    ap.add_argument("--topk", type=int, default=10)
    ap.add_argument("--queries", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--mode", default="coscan", help=argparse.SUPPRESS)
    ap.add_argument("--root", default=ROOT, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        sys.path.insert(0, os.path.abspath(a.root))     # bench.py and the bindings of the tree being timed
        return worker(a)

    own = os.path.join(ROOT, "semtools_b200", "lib", "libsemtools_b200.so")
    modes = []
    if a.parent_root:
        plib = os.path.join(a.parent_root, "semtools_b200", "lib", "libsemtools_b200.so")
        modes.append(("full", a.parent_root, plib))
    modes.append(("coscan", ROOT, own))
    for e in a.extra:
        name, path = e.split("=", 1)
        modes.append((name, ROOT, path))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    results = []
    for r in range(a.rounds):
        for name, root, lib in modes:
            e = {k: v for k, v in os.environ.items() if k != "STB_SCAN_TIER"}
            e["STB_LIB_PATH"] = os.path.abspath(lib)
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--mode", name, "--rows", str(a.rows),
                   "--rows2", str(a.rows2), "--tiers", a.tiers, "--topk", str(a.topk), "--queries", str(a.queries),
                   "--warmup", str(a.warmup), "--root", os.path.abspath(root)]
            p = subprocess.run(cmd, env=e, capture_output=True, text=True, cwd=root)
            if p.returncode != 0:
                print(json.dumps({"mode": name, "round": r, "error": p.stderr[-2000:]}), flush=True)
                continue
            for line in p.stdout.splitlines():
                if line.startswith("{"):
                    rec = json.loads(line)
                    rec["round"] = r
                    results.append(rec)
                    print(json.dumps(rec), flush=True)
    summary = {}
    for rec in results:
        key = f'{rec["rows"]}/{rec["tier"]}/{rec["mode"]}'
        summary.setdefault(key, []).append(round(rec["ms_per_query"], 4))
    out = {"card": card, "queries": a.queries, "rounds": a.rounds, "ms_per_query": summary,
           "refined_rows_per_query": {f'{r["rows"]}/{r["mode"]}': round(r["refined_rows_per_query"])
                                      for r in results if r["tier"] == "q8"}}
    print(json.dumps(out), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            for rec in results:
                f.write(json.dumps(rec) + "\n")
            f.write(json.dumps(out) + "\n")


if __name__ == "__main__":
    main()

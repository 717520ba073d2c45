"""What the q8 tier's 4-bit prefilter reads: rows refined from the int8 codes per query and the bytes a
query really moves (136 B/row of nibble plane + {s, rho}, plus 260 B per refined row for its codes and
scale), next to the 260 B/row bench.py books for the q8 tier.  Same corpus and queries as bench.py's
headline.  Needs a GPU; prints one JSON line (and writes it to --out if given).

    python scripts/q4_probe.py [--rows 10000000] [--topk 10] [--queries 64] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--topk", type=int, default=10)
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import bench
    from semtools_b200 import capi

    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    ctx = capi.Context(0, stream.cuda_stream)
    corpus, _, _ = bench.fill_shard(torch, dev, capi, ctx, a.rows, 1, 0)
    corpus.prepare(1)
    qs = torch.from_numpy(bench.gen_queries(a.queries)).to(dev)
    hits = torch.zeros((a.queries, a.topk, 2), dtype=torch.float64, device=dev)
    st = torch.zeros((a.queries, 4), dtype=torch.int32, device=dev)
    cnt = ctypes.c_uint64(0)

    def refined(reset):
        capi._check(capi.lib().stb_debug_q4_refined(ctx._h, reset, ctypes.byref(cnt)))
        return int(cnt.value)

    refined(1)
    per_q = []
    for i in range(a.queries):
        corpus.search_topk_dev(qs[i].data_ptr(), a.topk, hits[i].data_ptr(), st[i].data_ptr())
        per_q.append(refined(1))
    s = st.cpu().numpy()
    per_q = sorted(per_q)
    med = per_q[len(per_q) // 2]
    out = {
        "gpu": torch.cuda.get_device_name(dev), "rows": a.rows, "top_k": a.topk, "queries": a.queries,
        "tier": bench.TIER_NAMES[int(s[0, 3]) >> 16], "all_proven": bool((s[:, 1] == 1).all()),
        "refined_rows_per_query": {"min": per_q[0], "median": med, "max": per_q[-1]},
        "refined_fraction_median": med / a.rows,
        "true_bytes_per_query_median": 136 * a.rows + 260 * med,
        "bench_booked_bytes_per_query": bench.TIER_BYTES["q8"] * a.rows,
    }
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

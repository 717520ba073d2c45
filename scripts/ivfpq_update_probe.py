"""K5 update probe: what stb_ivfpq_update / stb_ivfpq_remove cost against the plain corpus calls and a rebuild,
and what keeping an index current without retraining does to recall and q/s.

python scripts/ivfpq_update_probe.py [rows] [nlist] [nprobe] [rerank]
Defaults: the data of scripts/ivfpq_extend_probe.py (4M clustered rows, rows/100 centres, spread 0.6), nlist 4096,
nprobe 64, rerank 512, top_k 10, 1024 queries.  Two corpora hold the same rows, both with their q8 and 16-bit copies
built; one carries an index.  Each call is timed with a host clock around it and a synchronise, on the indexed corpus
(stb_ivfpq_*) and on the plain one (stb_corpus_*), with the same arguments:
  update of 16384 and of 262144 rows (values drawn around shifted centres), removal of one 16384-row document near
  the front, removal of 1 % of the rows in 400 ranges.
Then a mixed sequence brings the total to 20 % of the rows replaced and 10 % removed; the maintained index is
compared with a fresh build on the final rows (its time is the destroy + rebuild alternative): recall@10 against
the exact search, and batched q/s.  Half the queries come from the original centres, half from the shifted ones.
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
nlist = int(sys.argv[2]) if len(sys.argv) > 2 else 4096
nprobe = int(sys.argv[3]) if len(sys.argv) > 3 else 64
rerank = int(sys.argv[4]) if len(sys.argv) > 4 else 512
top_k, n_centers, spread, nq = 10, max(rows // 100, 1000), 0.6, 1024


def emit(**kw):
    print(json.dumps(kw), flush=True)


hw = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                    capture_output=True, text=True).stdout.strip()
emit(hardware=hw)

dev = torch.device("cuda:0")
ctx = capi.Context(0)
g = torch.Generator(device=dev); g.manual_seed(11)
centers = torch.randn((n_centers, 256), generator=g, device=dev); centers /= centers.norm(dim=1, keepdim=True)
shifted = centers + 0.5 * torch.randn((n_centers, 256), generator=g, device=dev)
shifted /= shifted.norm(dim=1, keepdim=True)
rng = np.random.default_rng(12)


def draw(cs, n):
    i = torch.randint(0, n_centers, (n,), generator=g, device=dev)
    x = cs[i] + spread / 16.0 * torch.randn((n, 256), generator=g, device=dev)
    return x / x.norm(dim=1, keepdim=True)


X = torch.empty((rows, 256), dtype=torch.float32, device=dev)
for i in range(0, rows, 1_000_000):
    X[i:i + min(1_000_000, rows - i)] = draw(centers, min(1_000_000, rows - i))
q = torch.cat([draw(centers, nq // 2), draw(shifted, nq - nq // 2)]).contiguous()
qh = q.cpu().numpy()
torch.cuda.synchronize()


def corpus():
    c = capi.Corpus(ctx, rows)
    c.append_dev(X.data_ptr(), rows)
    c.prepare(3)
    return c


def timed(fn):
    ctx.sync()
    t0 = time.perf_counter()
    out = fn()
    ctx.sync()
    return out, time.perf_counter() - t0


def build(c):
    return timed(lambda: capi.IvfPq(c, nlist=nlist, train_rows=262144, iters=8))


emit(shape=dict(rows=rows, nlist=nlist, nprobe=nprobe, top_k=top_k, rerank=rerank, nq=nq))
c_idx, c_plain = corpus(), corpus()
index, t_build = build(c_idx)
emit(config="build", rows=rows, s=t_build, stats=index.stats())
del X
torch.cuda.empty_cache()
n = rows
replaced = removed = 0


def update(m):
    global replaced
    ids = np.sort(rng.choice(n, m, replace=False)).astype(np.uint64)
    vals = draw(shifted, m).cpu().numpy()
    _, t_i = timed(lambda: index.update(ids, vals))
    _, t_c = timed(lambda: c_plain.update(ids, vals))
    replaced += m
    return t_i, t_c


def remove(ranges):
    global n, removed
    ranges = np.asarray(ranges, np.uint64)
    _, t_i = timed(lambda: index.remove(ranges))
    _, t_c = timed(lambda: c_plain.remove(ranges))
    k = int((ranges[:, 1] - ranges[:, 0]).sum())
    n -= k
    removed += k
    return t_i, t_c


def spaced_ranges(count, length):
    starts = np.sort(rng.choice(n // length - 1, count, replace=False)) * length + length // 2
    return np.stack([starts, starts + length], axis=1)


for m in (16384, 262144):
    t_i, t_c = update(m)
    emit(config=f"update {m} rows", ivfpq_update_s=t_i, corpus_update_s=t_c, rebuild_s=t_build, stats=index.stats())
t_i, t_c = remove([[1000, 1000 + 16384]])
emit(config="remove one 16384-row document near the front", ivfpq_remove_s=t_i, corpus_remove_s=t_c, rebuild_s=t_build,
     stats=index.stats())
one_pct = rows // 100
t_i, t_c = remove(spaced_ranges(400, one_pct // 400))
emit(config=f"remove 1 % of the rows in 400 ranges of {one_pct // 400}", ivfpq_remove_s=t_i, corpus_remove_s=t_c,
     rebuild_s=t_build, stats=index.stats())
# the rest of the mixed sequence: 20 % of the rows replaced, 10 % removed in all
t_mixed = 0.0
while replaced < rows // 5:
    t_mixed += update(min(262144, rows // 5 - replaced))[0]
rest = rows // 10 - removed
t_mixed += remove(spaced_ranges(1000, rest // 1000))[0]
emit(config="mixed sequence", replaced=replaced, removed=removed, rows=n, ivfpq_calls_s=t_mixed, stats=index.stats())
assert np.array_equal(c_idx.read(0, 4096).view(np.uint32), c_plain.read(0, 4096).view(np.uint32))

fresh, t_fresh = build(c_plain)
emit(config="fresh build on the final rows (destroy + rebuild)", s=t_fresh, stats=fresh.stats())
exact = c_plain.search_batch(qh, top_k=top_k)
lib_stream = torch.cuda.ExternalStream(ctx.stream) if ctx.stream else torch.cuda.default_stream()
hits = torch.empty((nq, top_k, 2), dtype=torch.float64, device=dev)
status = torch.empty((nq, 2), dtype=torch.int32, device=dev)
for name, ix in [("maintained", index), ("fresh build", fresh)]:
    got, cnt, scanned = ix.search_batch(qh, nprobe=nprobe, top_k=top_k, rerank=rerank)
    rec = np.array([len(set(got[i, : cnt[i]]["row"].tolist()) & set(exact[i]["row"].tolist())) / top_k for i in range(nq)])
    ix.search_batch_dev(q.data_ptr(), nq, nprobe, top_k, rerank, hits.data_ptr(), status.data_ptr()); ctx.sync()
    reps = 20
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(lib_stream)
    for _ in range(reps):
        ix.search_batch_dev(q.data_ptr(), nq, nprobe, top_k, rerank, hits.data_ptr(), status.data_ptr())
    b.record(lib_stream); ctx.sync(); b.synchronize()
    ms = a.elapsed_time(b) / reps
    emit(index=name, recall_at_10=float(rec.mean()), recall_original_centres=float(rec[: nq // 2].mean()),
         recall_shifted_centres=float(rec[nq // 2:].mean()), codes_scanned_per_query=float(np.mean(scanned)),
         max_list=ix.stats()["max_list"], batch_ms=ms, batch_qps=nq / ms * 1e3)
index.close(); fresh.close()
c_idx.close(); c_plain.close()

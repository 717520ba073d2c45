"""K5 persistence probe: what stb_ivfpq_save and stb_ivfpq_load cost against the build they replace.

python scripts/ivfpq_persist_probe.py [sizes]          sizes: comma-separated row counts, default 4000000,40000000
Data: clustered unit rows as scripts/ivfpq_batch_probe.py makes them (rows/100 centres, at most 100000, spread 0.6),
generated on the GPU in chunks of 1M rows and appended from HBM; nlist 4096, train_rows 262144, iters 8.  For each
size: the build, the save and the load, each timed with a host clock around the call and a synchronise; the load
also split by stb_debug_ivfpq_load_ms into reading the file and uploading its sections vs the GPU verification
(section checksums, the lists pass, the rows pass).  The file goes to a temporary directory and is removed; the
load reads it back right after the save, so from the page cache (dropping the cache is a system setting, not
something this probe changes).  Then a batch of 1024 queries (nprobe 64, top_k 10, rerank 512) must return
identical hits from the built and the loaded index.  Prints one JSON line per measurement."""
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from semtools_b200 import capi  # noqa: E402

sizes = [int(s) for s in (sys.argv[1] if len(sys.argv) > 1 else "4000000,40000000").split(",")]
nlist, nprobe, top_k, rerank, nq, spread = 4096, 64, 10, 512, 1024, 0.6


def emit(**kw):
    print(json.dumps(kw), flush=True)


hw = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                    capture_output=True, text=True).stdout.strip()
emit(hardware=hw)
dev = torch.device("cuda:0")
ctx = capi.Context(0)


def timed(fn):
    ctx.sync()
    t0 = time.perf_counter()
    out = fn()
    ctx.sync()
    return out, time.perf_counter() - t0


for rows in sizes:
    n_centers = min(max(rows // 100, 1000), 100_000)
    g = torch.Generator(device=dev); g.manual_seed(17)
    centers = torch.randn((n_centers, 256), generator=g, device=dev); centers /= centers.norm(dim=1, keepdim=True)
    c = capi.Corpus(ctx, rows)
    for i in range(0, rows, 1_000_000):
        n = min(1_000_000, rows - i)
        x = centers[torch.randint(0, n_centers, (n,), generator=g, device=dev)] + spread / 16.0 * torch.randn((n, 256), generator=g, device=dev)
        x = (x / x.norm(dim=1, keepdim=True)).contiguous()
        torch.cuda.synchronize()
        c.append_dev(x.data_ptr(), n)
        del x
    q = centers[torch.randint(0, n_centers, (nq,), generator=g, device=dev)] + spread / 16.0 * torch.randn((nq, 256), generator=g, device=dev)
    qh = (q / q.norm(dim=1, keepdim=True)).cpu().numpy()
    del centers, q
    torch.cuda.empty_cache()
    emit(shape=dict(rows=rows, nlist=nlist, centres=n_centers, nprobe=nprobe, top_k=top_k, rerank=rerank, nq=nq))
    built, t_build = timed(lambda: capi.IvfPq(c, nlist=nlist, train_rows=262144, iters=8))
    emit(config="build", rows=rows, s=round(t_build, 4), stats=built.stats())
    tmp = tempfile.mkdtemp(prefix="ivfpq_persist_")
    try:
        path = os.path.join(tmp, "index.stbivf")
        _, t_save = timed(lambda: built.save(path))
        size = os.path.getsize(path)
        emit(config="save", rows=rows, s=round(t_save, 4), file_bytes=size, GB_s=round(size / t_save / 1e9, 3))
        loaded, t_load = timed(lambda: capi.IvfPq.load(c, path))
        ms_read, ms_verify = loaded.load_ms()
        emit(config="load", rows=rows, s=round(t_load, 4), read_upload_ms=round(ms_read, 2), verify_ms=round(ms_verify, 2),
             file_from="page cache", vs_build=round(t_build / t_load, 1))
        same = loaded.stats() == built.stats()
        want = built.search_batch(qh, nprobe=nprobe, top_k=top_k, rerank=rerank)
        got = loaded.search_batch(qh, nprobe=nprobe, top_k=top_k, rerank=rerank)
        same_hits = all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(want, got))
        emit(config="check", rows=rows, stats_equal=same, batch_hits_identical=bool(same_hits), queries=nq)
        loaded.close()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    built.close(); c.close()
    torch.cuda.empty_cache()

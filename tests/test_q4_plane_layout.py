"""The q8 tier's nibble plane is stored in 32-row tiles (row_encode.cuh: stb_q4_plane_offset): chunk m of row r
at (r // 32) * 4096 + m * 512 + (r % 32) * 16.  CPU: the debug copy's gather (stb_q4_plane_gather) is the inverse
of that interleave.  GPU: through the debug copy, the maintained plane equals a fresh build after every kind of
change that moves rows across tile boundaries: a row count that is not a multiple of 32, appends that grow into a
new tile, a regrowth of the copy, updates and removals."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import unit_rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"

HARNESS = r"""
#include "row_encode.cuh"
extern "C" void gather(const uint8_t *tiles, uint64_t first, uint64_t n, uint8_t *out) { stb_q4_plane_gather(tiles, first, n, out); }
extern "C" uint64_t offset(uint64_t row, int m) { return stb_q4_plane_offset(row, m); }
extern "C" uint64_t plane_bytes(uint64_t rows) { return stb_q4_plane_bytes(rows); }
"""


def interleave(rows):
    """numpy statement of the layout: rows [n][128] -> ceil(n / 32) tiles of 4096 B"""
    n = len(rows)
    tiles = np.zeros(((n + 31) // 32) * 4096, dtype=np.uint8)
    for r in range(n):
        for m in range(8):
            o = (r // 32) * 4096 + m * 512 + (r % 32) * 16
            tiles[o:o + 16] = rows[r, 16 * m:16 * m + 16]
    return tiles


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("needs nvcc")
    d = tmp_path_factory.mktemp("q4plane")
    (d / "h.cu").write_text(HARNESS)
    so = d / "h.so"
    subprocess.run([NVCC, "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-I", os.path.join(ROOT, "semtools_b200", "csrc"),
                    "-o", str(so), str(d / "h.cu")], check=True, capture_output=True)
    L = ctypes.CDLL(str(so))
    L.gather.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_void_p]
    L.offset.argtypes = [ctypes.c_uint64, ctypes.c_int]
    L.offset.restype = ctypes.c_uint64
    L.plane_bytes.argtypes = [ctypes.c_uint64]
    L.plane_bytes.restype = ctypes.c_uint64
    return L


def test_gather_inverts_the_interleave(harness):
    rng = np.random.default_rng(1)
    n = 133
    rows = rng.integers(0, 256, (n, 128), dtype=np.uint8)
    tiles = interleave(rows)
    assert harness.plane_bytes(n) == len(tiles) and harness.plane_bytes(0) == 0 and harness.plane_bytes(32) == 4096
    for first, cnt in ((0, n), (0, 1), (31, 2), (32, 32), (37, 60), (95, 38), (n - 1, 1), (5, 0)):
        src = np.ascontiguousarray(tiles[(first // 32) * 4096:])
        out = np.zeros((cnt, 128), dtype=np.uint8)
        harness.gather(src.ctypes.data, first, cnt, out.ctypes.data)
        assert np.array_equal(out, rows[first:first + cnt]), (first, cnt)
    for r in (0, 31, 32, 1000, 2 ** 32 - 3):
        for m in (0, 7):
            assert harness.offset(r, m) == (r // 32) * 4096 + m * 512 + (r % 32) * 16


def _check_plane(ctx, c, model):
    from semtools_b200 import capi
    got, cov = c.debug_copy(capi.STB_COPY_Q8_PLANE)
    assert cov == len(model)
    fresh = capi.Corpus(ctx, max(len(model), 1))
    fresh.append(model)
    fresh.prepare(1)
    want = fresh.debug_copy(capi.STB_COPY_Q8_PLANE)[0]
    assert np.array_equal(got, want)
    # a window that starts and ends inside tiles
    if len(model) > 70:
        assert np.array_equal(c.debug_copy(capi.STB_COPY_Q8_PLANE, 33, 37)[0], want[33:70])
    fresh.close()


@pytest.mark.gpu
def test_maintained_plane_equals_a_fresh_build(ctx):
    from semtools_b200 import capi
    rng = np.random.default_rng(2)
    model = unit_rows(rng, 1000)                                      # 31 whole tiles + 8 rows
    c = capi.Corpus(ctx, 1000)
    c.append(model)
    c.prepare(1)
    _check_plane(ctx, c, model)
    tail = unit_rows(rng, 500)                                        # past the capacity: the copy regrows
    c.append(tail)
    model = np.concatenate([model, tail])
    c.prepare(1)
    _check_plane(ctx, c, model)
    tail = unit_rows(rng, 30)                                         # 1500 = 46 tiles + 28: into tile 47
    c.append(tail)
    model = np.concatenate([model, tail])
    c.prepare(1)
    _check_plane(ctx, c, model)
    idx = np.array([0, 31, 32, 999, 1000, 1499, 1529], dtype=np.uint64)
    new = unit_rows(rng, len(idx))
    c.update(idx, new)
    model[idx.astype(np.int64)] = new
    _check_plane(ctx, c, model)
    ranges = np.array([[3, 4], [40, 75], [1200, 1203]], dtype=np.uint64)   # later rows move 1, 36, 39 rows back
    c.remove(ranges)
    keep = np.ones(len(model), dtype=bool)
    for b, e in ranges.astype(np.int64):
        keep[b:e] = False
    model = np.ascontiguousarray(model[keep])
    _check_plane(ctx, c, model)
    for q in model[[5, 700, len(model) - 1]]:                         # the scan reads the plane it keeps
        import oracle
        r, d = oracle.search_rows(model, q, top_k=10)
        hits = c.search(q, top_k=10)
        assert hits["row"].tolist() == [int(x) for x in r] and np.array_equal(hits["distance"], d)
    assert c.tier_stats()["q8"]["proven"] >= 1
    c.close()

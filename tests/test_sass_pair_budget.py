"""K1's pairs (scan_topk.cu: "pairs") need the join kernel to run beside two q8 scan CTAs on one SM, read from the
shipped library with cuobjdump (no GPU needed): the q8 top-k scan stays within its 120-register budget without
spills, and what two of its CTAs leave of an SM's registers, shared memory and threads holds the join kernel."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "semtools_b200", "lib", "libsemtools_b200.so")
pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(LIB), reason="needs cuobjdump and the built library")

# H100 (sm_90) per-SM limits; a warp takes its registers from one of 4 sub-partitions of 16K, in units of 256
SMSP_REGS, SM_SMEM, SM_THREADS = 16384, 228 * 1024, 2048
SCAN_THREADS, JOIN_THREADS = 256, 32


def warp_regs(r):
    return -(-r * 32 // 256) * 256


def resources():
    out = subprocess.run(["cuobjdump", "--dump-resource-usage", LIB], capture_output=True, text=True, errors="ignore",
                         timeout=600).stdout
    return {n: (int(r), int(st), int(sh)) for n, r, st, sh in
            re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", out)}


def test_join_kernel_fits_beside_two_q8_scan_ctas():
    fns = resources()
    q8 = {n: v for n, v in fns.items() if "stb_scan_topk_kernel_q8" in n}
    join = [v for n, v in fns.items() if "stb_pair_join_kernel" in n]
    assert len(q8) == 2 and len(join) == 1, (q8, join)
    assert all(r <= 120 and st == 0 for r, st, _ in q8.values()), q8        # 120 registers, no spill stack
    jr, jst, jsh = join[0]
    assert jst == 0, join
    for r, _, sh in q8.values():
        # two CTAs of 8 warps: 4 scan warps on each sub-partition, and the join's warp on one of them
        assert 4 * warp_regs(r) + warp_regs(jr) <= SMSP_REGS, (r, jr)
        assert 2 * (sh + 1024) + jsh + 1024 <= SM_SMEM, (sh, jsh)          # + the 1 KiB each CTA reserves
        assert 2 * SCAN_THREADS + JOIN_THREADS <= SM_THREADS

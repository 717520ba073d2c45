"""What the shipped library must contain, read with cuobjdump (no GPU needed): only sm_90a code objects,
the Hopper instructions the design rests on, and the register budgets the occupancy of the hot kernels
depends on (scripts/sass_summary.py prints the same information for a reader)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "semtools_b200", "lib", "libsemtools_b200.so")
pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(LIB), reason="needs cuobjdump and the built library")


def _run(*args):
    return subprocess.run(["cuobjdump", *args, LIB], capture_output=True, text=True, errors="ignore", timeout=600).stdout


def test_library_ships_sm_90a_code_only():
    elfs = re.findall(r"ELF file\s+\d+: (\S+)", _run("-lelf"))
    assert elfs and all(".sm_90a." in e for e in elfs), elfs
    assert "PTX file" not in _run("-lptx")                      # no PTX for a JIT to fall back on: sm_90a or nothing


def test_resource_usage_of_the_hot_kernels():
    """K1 runs 2 CTAs of 256 threads per SM (tile tickets assume it): <= 128 registers, no spills to speak of.
    K3 was retuned to 3 CTAs/SM (<= 80 registers)."""
    out = _run("--dump-resource-usage")
    fns = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", out)
    assert len(fns) >= 40
    scan = [(n, int(r), int(st)) for n, r, st, _ in fns if "stb_scan_topk_kernel" in n]
    assert len(scan) >= 14                                        # f32 / h16 / q8 x list widths x range walk
    assert all(r <= 128 and st <= 32 for _, r, st in scan), scan
    embed = [int(r) for n, r, _, _ in fns if "stb_embed_kernel" in n]
    assert embed and max(embed) <= 80, embed


def test_resource_usage_of_the_gemm_kernels():
    """K2's GEMM holds a 64x256 accumulator in 128 registers per consumer thread at 1 CTA/SM: every
    instantiation (shadow: 4 + 2 + 2, q8: 4 + 2) stays at <= 168 registers with nothing on the stack."""
    out = _run("--dump-resource-usage")
    fns = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", out)
    gemm = [(n, int(r), int(st)) for n, r, st, _ in fns if "stb_batch_gemm_kernel" in n]
    assert len(gemm) == 14, gemm
    assert all(r <= 168 and st == 0 for _, r, st in gemm), gemm


def test_hopper_instructions_are_where_the_design_says():
    sass = _run("-sass")
    per_fn, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1); per_fn[cur] = ""
        elif cur:
            per_fn[cur] += line + "\n"
    gemm = "".join(v for k, v in per_fn.items() if "stb_batch_gemm" in k)
    assert "HGMMA.64x256x16.F32" in gemm and "UBLKCP" in gemm and "SYNCS" in gemm   # wgmma m64n256k16, cp.async.bulk, mbarrier
    assert "HMMA" not in gemm.replace("HGMMA", "")                               # no legacy mma.sync in the tensor path
    assert "IGMMA.64x256x32.S8.S8" in gemm and "UTMALDG" in gemm                  # the q8 copy: s8 wgmma, TMA tensor loads
    q8 = [v for k, v in per_fn.items() if "stb_scan_topk_kernel" in k and "IDP.4A" in v]
    assert q8                                                                    # the int8 tier scans with dp4a
    k1 = [v for k, v in per_fn.items() if "stb_scan_topk_kernel" in k]
    assert all(re.search(r"ACQBULK|PREEXIT", v) for v in k1)                     # griddepcontrol (PDL) in every K1 variant
    assert all("LDG.E.128" in v for v in k1)                                     # 16-byte coalesced loads in the scan

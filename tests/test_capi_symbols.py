"""CPU suite, part 2: the C-ABI library loads and exports every symbol the header
declares, and refuses to compute without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import numpy as np
import pytest

from semtools_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "semtools_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(stb_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    L = ctypes.CDLL(capi.LIB_PATH)
    syms = header_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(L, s), f"{s} declared in the header but not exported"
    assert sorted(capi.SYMBOLS) == syms, "capi.SYMBOLS out of sync with the header"


def test_host_only_entry_points():
    assert capi.lib().stb_version() >= 100
    assert capi.fnv1a64(b"") == 0xCBF29CE484222325
    assert capi.fnv1a64(b"foobar") == 0x85944171F73967E8
    import oracle
    for p, n in [("/test/doc1.txt", 0), ("a/ü.md", 7), ("x", -1)]:
        assert capi.line_id(p, n) == oracle.line_id(p, n)
    f16, eps = capi.batch_params()                      # default build: fp16 shadow, EPS 0.0012
    assert (f16, eps) in ((False, 0.0080), (True, 0.0012))


def test_product_does_not_import_oracle():
    import subprocess, sys
    code = ("import sys; import semtools_b200; "
            "bad=[m for m in sys.modules if m.split('.')[0]=='oracle']; print(bad); sys.exit(1 if bad else 0)")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    for dirpath, _, files in os.walk(os.path.join(ROOT, "semtools_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
                assert "oracle/" not in src.replace("nothing in this directory may\n// include, link or call anything under oracle/", "") \
                    or f in ("common.cuh", "embed_pool.cu", "scan_topk.cu", "semtools_b200.h"), f


@pytest.mark.skipif(capi.device_count() > 0, reason="GPU present")
def test_no_gpu_means_loud_failure_not_cpu_fallback():
    with pytest.raises(capi.StbError) as e:
        capi.Context(0)
    assert e.value.status == capi.STB_ERR_CUDA
    assert "no CPU path" in str(e.value)


def test_header_is_plain_c_and_the_library_links_from_c(tmp_path):
    """The drop-in boundary is a C ABI: include/semtools_b200.h must compile as C99 (pedantic, no warnings)
    and a C program must link against the shared library and call it (host-only entry points: no GPU here)."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    src = tmp_path / "use_abi.c"
    src.write_text('#include <stdio.h>\n#include <string.h>\n#include "semtools_b200.h"\n'
                   'int main(void) {\n'
                   '  const char *s = "hello";\n'
                   '  stb_hit h; h.distance = 0.5; h.row = 7;\n'
                   '  printf("%d %llu %llu %d\\n", stb_version(), (unsigned long long)stb_fnv1a64((const uint8_t *)s, strlen(s)),\n'
                   '         (unsigned long long)stb_line_id((const uint8_t *)"a.txt", 5, 3), (int)sizeof(h));\n'
                   '  return 0;\n}\n')
    exe = tmp_path / "use_abi"
    lib_dir = os.path.dirname(capi.LIB_PATH)
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src),
                        "-L", lib_dir, "-lsemtools_b200", f"-Wl,-rpath,{lib_dir}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    version, fnv, lid, hit_size = r.stdout.split()
    assert int(version) == capi.lib().stb_version() and int(fnv) == capi.fnv1a64(b"hello") == 0xA430D84680AABD0B
    assert int(lid) == capi.line_id("a.txt", 3) and int(hit_size) == 16

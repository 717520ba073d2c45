"""CPU: every device, page-locked and device-mapped host buffer of the library has one owner, StbBuf
(csrc/common.cuh).

Outside that type no source allocates or frees CUDA memory by hand."""
import collections
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "semtools_b200", "csrc")

CALL = re.compile(r"\b(cuda(?:Malloc\w*|HostAlloc|Free\w*))\s*\(")
# (file, call) -> occurrences allowed outside StbBuf
ALLOWED = {}


def code_only(text):
    """The source without comments and string or character literals (which may name the calls)."""
    tok = re.compile(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'', re.S)
    return tok.sub(lambda m: "\n" * m.group(0).count("\n") if m.group(0).startswith("/") else '""', text)


def buffer_type_span(text):
    m = re.search(r"^struct StbBuf \{.*?^\};", text, flags=re.M | re.S)
    assert m, "common.cuh no longer defines struct StbBuf"
    return m.span()


def calls_outside_buffer_type():
    found = collections.Counter()
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh"))):
        name = os.path.basename(path)
        text = code_only(open(path).read())
        if name == "common.cuh":
            b, e = buffer_type_span(text)
            inside = {m.group(1) for m in CALL.finditer(text[b:e])}
            assert {"cudaMalloc", "cudaMallocHost", "cudaHostAlloc", "cudaFree", "cudaFreeHost"} <= inside
            text = text[:b] + text[e:]
        for m in CALL.finditer(text):
            found[(name, m.group(1))] += 1
    return found


def test_no_cuda_memory_is_allocated_or_freed_outside_the_buffer_type():
    found = calls_outside_buffer_type()
    extra = {k: v for k, v in found.items() if v > ALLOWED.get(k, 0)}
    assert not extra, f"allocate or free through StbBuf (common.cuh), not by hand: {extra}"
    assert found == ALLOWED, f"the allowlist is stale: {dict(found)}"

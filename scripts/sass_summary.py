#!/usr/bin/env python3
"""Per-kernel SASS mnemonic counts of the shipped library (a reader's view of tests/test_sass_contract.py),
and the q8 top-k prefilter's tile bodies, the pair's included: instructions per 32-row tile and their opcode mix
    python scripts/sass_summary.py [lib.so]"""
import collections, re, subprocess, sys
lib = sys.argv[1] if len(sys.argv) > 1 else "semtools_b200/lib/libsemtools_b200.so"
sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, errors="ignore").stdout
pat = {"HGMMA (wgmma.mma_async)": r"\bHGMMA", "WARPGROUP (wgmma fence / wait)": r"\bWARPGROUP", "UBLKCP (cp.async.bulk)": r"\bUBLKCP",
       "SYNCS (mbarrier)": r"\bSYNCS", "ACQBULK/PREEXIT (griddepcontrol, PDL)": r"\b(ACQBULK|PREEXIT)",
       "IDP.4A (dp4a)": r"\bIDP\.4A", "LDG.E.128": r"LDG\.E\.(NA\.)?128|LDG\.E\.128", "HMMA (legacy mma.sync)": r"\bHMMA",
       "DFMA (f64 re-rank)": r"\bDFMA", "ATOMG/RED (global atomics)": r"\b(ATOMG|RED)\b"}
cur, cnt, code = None, collections.OrderedDict(), {}
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1); cnt[cur] = collections.Counter(); code[cur] = []; continue
    if cur:
        for k, r in pat.items():
            if re.search(r, line):
                cnt[cur][k] += 1
        m = re.search(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", line)
        if m:
            code[cur].append((int(m.group(1), 16), m.group(2)))
print("# per-kernel SASS mnemonic counts of", lib, "(cuobjdump -sass; all code objects sm_90a)\n")
tot = collections.Counter()
names = {}
for fn, c in cnt.items():
    names[fn] = re.sub(r"\(.*", "", subprocess.run(["c++filt", fn], capture_output=True, text=True).stdout.strip())
    if not c:
        continue
    print(names[fn][:90])
    print("    " + ", ".join(f"{k}: {c[k]}" for k in pat if c[k]))
    tot.update(c)
print("\nTOTAL  " + ", ".join(f"{k}: {tot[k]}" for k in pat))


def tile_bodies(ins):
    """The prefilter's tile bodies: from the head of the innermost loop around a ballot (VOTE.ANY with a register
    result: the refine-queue vote) to the first conditional branch after it (the queue-full test).  A pair's host
    has three: its own query's, the pair's (both queries' accumulators on one set of plane loads: two votes) and
    the guest-only wrap's."""
    at = {a: i for i, (a, _) in enumerate(ins)}
    seen = set()
    for vote, (_, t) in enumerate(ins):
        if not re.match(r"VOTE\.ANY R", t):
            continue
        head = None
        for i, (a, tt) in enumerate(ins):
            m = re.match(r"(@!?U?P\w+ )?BRA (0x[0-9a-f]+)", tt)
            if m and i > vote and at.get(int(m.group(2), 16), i) <= vote:
                h = at[int(m.group(2), 16)]
                head = h if head is None or h > head else head
        end = next((i for i in range(vote, len(ins)) if re.match(r"@!?P\w+ BRA ", ins[i][1])), None)
        if head is None or end is None or head in seen:
            continue
        seen.add(head)
        yield ins[head:end + 1]


print("\n# q8 top-k prefilter tile bodies (32 rows per warp)")
for fn, ins in code.items():
    if not re.search(r"stb_scan_topk_kernel_q8<\d+, \d+, \d+, \d+>", names.get(fn, "")):
        continue
    found = False
    for body in tile_bodies(ins):
        mix = collections.Counter()
        for _, t in body:
            op = re.sub(r"^@!?U?P\w+ ", "", t).split()[0]
            mix["IDP.4A" if op.startswith("IDP.4A") else op.split(".")[0]] += 1
        if mix["IDP.4A"] < 128 or mix["LOP3"] < 64:   # not a plane tile (lists, sorts, the int8 refine)
            continue
        found = True
        kind = "pair (two queries)" if mix["IDP.4A"] >= 256 else "one query"
        print(f"{names[fn]} [{kind}]: {len(body)} instructions ({len(body) / 32:.1f} per row)")
        print("    " + ", ".join(f"{k}: {v}" for k, v in mix.most_common()))
    if not found:
        print(names[fn], ": tile body not found")

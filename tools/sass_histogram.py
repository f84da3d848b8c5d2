#!/usr/bin/env python3
"""SASS opcode histogram per kernel of libb200ops.so (cuobjdump -sass), written to profiles/<round>_sass_opcodes.txt.
Evidence for what the kernels are made of: HGMMA (wgmma), UBLKCP / SYNCS (TMA bulk copies + mbarriers),
IDP.4A (dp4a) ... — the PTX names never appear in SASS (B200_PROFILING.md)."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = os.path.join(ROOT, "llama-box_b200", "libb200ops.so")
out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "r2_sass_opcodes.txt")
txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
kern, hist = None, collections.OrderedDict()
for ln in txt.splitlines():
    m = re.match(r"\s*Function : (\S+)", ln)
    if m:
        kern = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        kern = kern.replace("(anonymous namespace)::", "")       # the wide path's kernels live in unnamed namespaces
        kern = re.sub(r"\(.*", "", kern)
        hist.setdefault(kern, collections.Counter())
        continue
    m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*(?:\.[A-Z0-9_]+)*)", ln)
    if m and kern:
        hist[kern][m.group(1)] += 1
KEY = ("HGMMA", "UTCHMMA", "UTCIMMA", "UTCQMMA", "LDTM", "STTM", "UTCBAR", "UTCATOMSWS", "UBLKCP", "UTMALDG", "SYNCS", "IDP", "HFMA2", "HMUL2", "HADD2", "FFMA", "LDG", "LDS", "STS", "STG", "SHFL", "BAR", "MUFU", "DFMA", "DADD")
with open(out, "w") as f:
    f.write("# SASS opcode histogram per kernel of llama-box_b200/libb200ops.so (cuobjdump -sass, sm_90a); tools/sass_histogram.py\n")
    f.write("# columns: total instructions | selected opcode families (prefix match)\n")
    agg = collections.defaultdict(collections.Counter)
    for k, c in hist.items():
        base = re.sub(r"<.*", "", k)                       # fold template instances
        agg[base].update(c)
    for k, c in sorted(agg.items(), key=lambda kv: -sum(kv[1].values())):
        fam = collections.Counter()
        for op, n in c.items():
            for p in KEY:
                if op == p or op.startswith(p + ".") or (p in ("IDP", "SYNCS", "LDG", "LDS", "STS", "STG", "BAR", "MUFU") and op.startswith(p)):
                    fam[p] += n
        f.write(f"{k:40s} {sum(c.values()):8d} | " + " ".join(f"{p}={fam[p]}" for p in KEY if fam[p]) + "\n")
        top = ", ".join(f"{op}:{n}" for op, n in c.most_common(12))
        f.write(f"{'':40s} top: {top}\n")
print("wrote", out)

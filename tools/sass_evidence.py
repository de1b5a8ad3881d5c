#!/usr/bin/env python
"""tools/sass_evidence.py -- which Hopper-class (sm_90a) instructions the shipped library contains, per kernel.

    python tools/sass_evidence.py

Counts, in `cuobjdump -sass graphgan_b200/libgraphgan_b200.so`: UBLKCP (cp.async.bulk, the TMA engine's 1-D bulk copy),
SYNCS.* (mbarrier init / arrive.expect_tx / try_wait), UTMALDG/UTMASTG (tensor-map TMA; none: the streams here are 1-D),
HGMMA (wgmma; none by design: there is no dense contraction on this path), plus the classic LDG.E.128 / ATOMS / REDG."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(ROOT, "graphgan_b200", "libgraphgan_b200.so")
sass = subprocess.run(["cuobjdump", "-sass", lib], stdout=subprocess.PIPE, text=True, check=True).stdout
pat = {"UBLKCP": r"\bUBLKCP", "SYNCS (mbarrier)": r"\bSYNCS", "UTMALDG/UTMASTG": r"\bUTMA(LDG|STG)", "HGMMA (wgmma)": r"\bHGMMA",
       "LDG.E.128": r"\bLDG\.E\.128", "LDGSTS": r"\bLDGSTS", "ATOMS": r"\bATOMS", "REDG/ATOMG": r"\b(REDG|ATOMG)", "FENCE.VIEW.ASYNC": r"\bFENCE\.VIEW\.ASYNC"}
per = collections.OrderedDict()
name = None
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        name = subprocess.run(["c++filt", m.group(1)], stdout=subprocess.PIPE, text=True).stdout.strip()
        name = re.sub(r"\(anonymous namespace\)::", "", name)
        name = name.split("(")[0]
        per[name] = collections.Counter()
        continue
    if name is None:
        continue
    if re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
        per[name]["instructions"] += 1
        for k, p in pat.items():
            if re.search(p, line):
                per[name][k] += 1
cols = ["instructions"] + list(pat)
print("# SASS evidence: %s (cuobjdump -sass), sm_90a" % os.path.relpath(lib, ROOT))
print("| kernel | " + " | ".join(cols) + " |")
print("|---|" + "---|" * len(cols))
tot = collections.Counter()
for n, c in per.items():
    tot.update(c)
    print("| `%s` | " % n + " | ".join(str(c[k]) for k in cols) + " |")
print("| **total** | " + " | ".join(str(tot[k]) for k in cols) + " |")

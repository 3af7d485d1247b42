#!/usr/bin/env python3
"""SASS census of the built extension: per kernel, how many of each instruction class that matters here (wgmma = IGMMA /
HGMMA, WARPGROUP.*; TMA bulk copies = UBLKCP; mbarrier = SYNCS; fences; shuffles; global loads / stores).
  python scripts/sass_census.py [blackbird_b200/_bb*.so] > profiles/sass_census.txt"""
import collections
import glob
import re
import subprocess
import sys

KEEP = ["IGMMA", "HGMMA", "WARPGROUP", "UBLKCP", "UTMALDG", "UTMASTG", "SYNCS", "UTMACMDFLUSH",
        "IMAD", "IDP", "SHFL", "LDS", "LDG", "STG", "ATOMG", "REDG", "MEMBAR", "CCTL", "FENCE"]


def main() -> int:
    so = sys.argv[1] if len(sys.argv) > 1 else sorted(glob.glob("blackbird_b200/_bb*.so"))[0]
    txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    demangle = subprocess.run(["c++filt"], input=txt, capture_output=True, text=True).stdout
    print(f"SASS census of {so} (cuobjdump -sass, sm_90a).  Columns = instruction counts per kernel.\n")
    cur, counts = None, collections.OrderedDict()
    for line in demangle.splitlines():
        m = re.match(r"\s*Function : (.*)", line)
        if m:
            cur = m.group(1).strip()
            counts[cur] = collections.Counter()
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m and cur:
            op = m.group(1)
            counts[cur]["total"] += 1
            for k in KEEP:
                if op.split(".")[0] == k or op.startswith(k + "."):
                    counts[cur][k] += 1
    for fn, c in counts.items():
        print(fn[:110])
        print("    total=%d  " % c["total"] + "  ".join(f"{k}={c[k]}" for k in KEEP if c[k]))
        print()
    return 0


if __name__ == "__main__":
    sys.exit(main())

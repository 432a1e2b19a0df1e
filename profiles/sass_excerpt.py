#!/usr/bin/env python
"""Counts, per kernel of the shipped library, the SASS instructions that prove the path:
    python profiles/sass_excerpt.py [lib.so]
UTMALDG (TMA box loads), UBLKCP (bulk copies), UTMAPF / UBLKPF (L2 prefetch), SYNCS (mbarriers), IDP.2A (two s16 x u8
MACs), I2IP (saturate + pack), I2F.U8 (byte-select conversion), ELECT."""
import re
import subprocess
import sys
from collections import Counter

lib = sys.argv[1] if len(sys.argv) > 1 else "transform360_b200/lib/libTransform360.so"
sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
want = re.compile(r"\b(UTMALDG[\w.]*|UBLKCP[\w.]*|UTMAPF[\w.]*|UBLKPF[\w.]*|SYNCS[\w.]*|IDP\.2A[\w.]*|I2IP[\w.]*|ELECT|I2F\.U8)\b")
counts, fn = Counter(), None
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        fn = m.group(1)
        continue
    if fn and re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
        m = want.search(line)
        if m:
            counts[(fn, m.group(1))] += 1
names = sorted({f for f, _ in counts})
demangled = dict(zip(names, subprocess.run(["c++filt"] + names, capture_output=True, text=True).stdout.splitlines()))
for (f, op), n in sorted(counts.items(), key=lambda kv: (demangled[kv[0][0]], kv[0][1])):
    print(f"{n:5d}  {demangled[f].replace('t360::(anonymous namespace)::', '')}  {op}")

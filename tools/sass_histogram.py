"""SASS opcode histogram of the kernels in dig_b200/libdig3d.so (on sm_90a: wgmma -> HGMMA, cp.async.bulk -> UBLKCP,
mbarrier -> SYNCS, setmaxnreg -> USETMAXREG).  Needs no GPU:

    python tools/sass_histogram.py [regex over demangled kernel names]
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "dig_b200", "libdig3d.so")
pat = re.compile(sys.argv[1] if len(sys.argv) > 1 else r"h16|_tc_kernel|gather_warp|linear_tc")
KEY = ("UTCHMMA", "UTCQMMA", "UTCBAR", "LDTM", "STTM", "UBLKCP", "UTMALDG", "SYNCS", "USETMAXREG", "HMMA", "MUFU", "FFMA2", "FMUL2", "FADD2",
       "F2FP", "LDL", "STL", "ATOMS", "RED", "ATOMG")
out = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True).stdout
name, hist = None, None
kernels = []
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        if name is not None:
            kernels.append((name, hist))
        name, hist = m.group(1), collections.Counter()
        continue
    m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)", line)
    if m and name is not None:
        hist[m.group(1)] += 1
if name is not None:
    kernels.append((name, hist))
print(f"# cuobjdump -sass {os.path.relpath(SO, ROOT)} -- opcode histograms (static instruction counts)")
for mangled, hist in kernels:
    dem = subprocess.run(["c++filt", mangled], capture_output=True, text=True).stdout.strip()
    short = dem.split("(")[0]
    if not pat.search(short):
        continue
    total = sum(hist.values())
    print(f"\n{short}   [{total} instructions]")
    print("  key: " + ", ".join(f"{k} {hist[k]}" for k in KEY if hist.get(k)))
    print("  top: " + ", ".join(f"{k} {v}" for k, v in hist.most_common(14)))

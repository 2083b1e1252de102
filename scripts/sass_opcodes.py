#!/usr/bin/env python
"""Opcode histogram of every kernel in librtx.so (cuobjdump -sass): the
evidence that the TMA bulk-copy path (UBLKCP / SYNCS / UTMACMDFLUSH), the
mbarrier waits and the FP64 / FP32 pipes are what the kernels use.
    python scripts/sass_opcodes.py > sass_opcodes.txt"""
import collections, os, re, subprocess
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(ROOT, "rayopt_b200", "librtx.so")
out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
demangle = lambda n: subprocess.run(["cu++filt", n], capture_output=True, text=True).stdout.strip() or n
kern, hist = None, collections.OrderedDict()
arch = re.search(r"arch = (sm_\w+)", out)
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        kern = demangle(m.group(1))
        hist[kern] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_]+)", line)
    if m and kern:
        hist[kern][m.group(1).split(".")[0]] += 1
KEY = ["UBLKCP", "SYNCS", "UTMACMDFLUSH", "FENCE", "BAR", "DFMA", "DMUL", "DADD", "FFMA", "FMUL", "FADD",
       "MUFU", "LDS", "STS", "LDG", "STG", "VOTE", "SHFL", "ATOM", "ATOMG", "RED", "REDG"]
print("# %s (%s): static SASS opcode counts per kernel" % (os.path.basename(lib), arch.group(1) if arch else "?"))
print("# kernel | total | " + " ".join(KEY))
tot = collections.Counter()
for k, c in hist.items():
    tot.update(c)
    print("%s | %d | %s" % (k.replace("rtx::", "").rsplit("(", 1)[0].replace("(bool)", ""), sum(c.values()), " ".join("%s=%d" % (o, c[o]) for o in KEY if c[o])))
print("# all kernels: " + " ".join("%s=%d" % (o, tot[o]) for o in KEY))
print("# tensor-core / tensor-map opcodes (none expected: elementwise FP64/FP32, 1-D bulk copies): "
      + " ".join("%s=%d" % (o, tot[o]) for o in ("UTCMMA", "UTCHMMA", "HMMA", "UTMALDG", "UTMASTG")))

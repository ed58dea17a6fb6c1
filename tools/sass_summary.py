"""SASS evidence: per kernel of libriqn_b200.so, how many tensor-core / TMA instructions it contains (`cuobjdump -sass`;
the PTX names never appear in SASS: wgmma.mma_async = HGMMA, TMA load / store = UTMALDG / UTMASTG, cp.async.bulk
(non-tensor) = UBLKCP).  Usage: python tools/sass_summary.py"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(ROOT, "rainbow_iqn_apex_b200", "libriqn_b200.so")
out = subprocess.run(["cuobjdump", "-sass", lib], stdout=subprocess.PIPE, text=True, check=True).stdout
MNEM = ("HGMMA", "UTMALDG", "UTMASTG", "UBLKCP", "HMMA", "REDG", "ATOMG")
counts, cur = collections.OrderedDict(), None
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        counts[cur] = collections.Counter()
        continue
    if cur is None:
        continue
    for k in MNEM:
        if re.search(r"\b%s\b|\b%s\." % (k, k), line):
            counts[cur][k] += 1
demangled = subprocess.run(["c++filt"], input="\n".join(counts), stdout=subprocess.PIPE, text=True).stdout.splitlines()
print("# cuobjdump -sass rainbow_iqn_apex_b200/libriqn_b200.so  (sm_90a); instruction counts per kernel")
print("# %-78s %s" % ("kernel", " ".join("%10s" % k for k in MNEM)))
tot = collections.Counter()
for (name, c), d in zip(counts.items(), demangled):
    d = re.sub(r"\(.*", "", d).replace("void ", "").replace("(int)", "")
    if sum(c.values()) == 0:
        continue
    print("%-80s %s" % (d[:80], " ".join("%10d" % c[k] for k in MNEM)))
    tot.update(c)
print("%-80s %s" % ("TOTAL", " ".join("%10d" % tot[k] for k in MNEM)))
sys.exit(0)

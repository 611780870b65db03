"""Opcode census of the shipped library: per kernel, how many wgmma / mma.sync / TMA / mbarrier instructions its SASS
holds (`cuobjdump -sass yolosharp_b200/lib/libyolob200.so`).  python tools/sass_summary.py"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = os.path.join(ROOT, "yolosharp_b200", "lib", "libyolob200.so")
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
WATCH = ["HGMMA", "UTMALDG", "UTMASTG", "UBLKCP", "UTCBAR", "UTCCP", "SYNCS", "ELECT", "HMMA", "IMMA",
         "FFMA", "HFMA2", "MUFU", "LDG", "STG", "LDS", "STS", "ATOM", "RED", "SHFL", "BAR"]
per = collections.OrderedDict()
cur = None
arch = set()
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        cur = per.setdefault(re.sub(r"\(.*", "", name), collections.Counter())
        continue
    m = re.search(r"arch = (sm_\w+)", line)
    if m:
        arch.add(m.group(1))
    if cur is None:
        continue
    m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)", line)
    if m:
        op = m.group(1)
        cur["_total"] += 1
        for w in WATCH:
            if op.startswith(w):
                cur[w] += 1
                break
tot = collections.Counter()
for c in per.values():
    tot.update(c)
print(f"# {os.path.relpath(so, ROOT)}: arch {sorted(arch)}, {len(per)} kernels, {tot['_total']} SASS instructions")
print("# whole library: " + "  ".join(f"{w} {tot[w]}" for w in WATCH if tot[w]))
print("# kernels that use the tensor cores / TMA:")
cols = ["HGMMA", "HMMA", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS"]
print(f"{'kernel':58s} " + " ".join(f"{c:>8s}" for c in cols) + "    total")
for name, c in per.items():
    if any(c[k] for k in cols[:5]):
        print(f"{name[:58]:58s} " + " ".join(f"{c[k]:8d}" for k in cols) + f" {c['_total']:8d}")
print("# (HGMMA = wgmma.mma_async, HMMA = mma.sync (TF32 weight gradient), UTMALDG = cp.async.bulk.tensor load,")
print("#  UBLKCP = cp.async.bulk, SYNCS = mbarrier try_wait / arrive)")

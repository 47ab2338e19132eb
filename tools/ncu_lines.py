#!/usr/bin/env python3
"""Attribute the executed instructions of one kernel of an .ncu-rep to CUDA source lines (no GPU needed): SASS page of the
report + `nvdisasm -g` line info of the cubin inside libb200orb.so that holds the kernel.
usage: ncu_lines.py rep.ncu-rep kernel-regex mangled-substring [source-file]"""
import collections
import csv
import os
import re
import subprocess
import sys
import tempfile

rep, kre, mangled = sys.argv[1], sys.argv[2], sys.argv[3]
srcfile = sys.argv[4] if len(sys.argv) > 4 else None
root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
tmp = tempfile.mkdtemp()
subprocess.run(["cuobjdump", "-xelf", "all", os.path.join(root, "orb_slam2_ssd_semantic_b200", "libb200orb.so")], cwd=tmp,
               capture_output=True)
# one cubin per module of the library: disassemble the one that holds the kernel
for cubin in sorted(f for f in os.listdir(tmp) if f.endswith(".cubin")):
    dis = subprocess.run(["nvdisasm", "-g", "-c", os.path.join(tmp, cubin)], capture_output=True, text=True).stdout.splitlines()
    start = next((i for i, l in enumerate(dis) if l.startswith(".text.") and mangled in l), None)
    if start is not None:
        break
else:
    sys.exit("no cubin of libb200orb.so holds a kernel matching " + mangled)
cur, off2line = None, {}
for l in dis[start + 1:]:
    if l.startswith("//-----") and "text." in l:
        break
    m = re.search(r'//## File "(.*?)", line (\d+)', l)
    if m:
        cur = (os.path.basename(m.group(1)), int(m.group(2)))
        continue
    m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(\S+)", l)
    if m:
        off2line[int(m.group(1), 16)] = (cur, m.group(2))
out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--kernel-name", "regex:" + kre], capture_output=True,
                     text=True).stdout
rows = list(csv.reader(out.splitlines()))
hdr = next(r for r in rows if r and r[0] == "Address")
ie = hdr.index("Instructions Executed")
byline, byop, tot, base = collections.Counter(), collections.Counter(), 0, None
ninst = 0
for r in rows:
    if not r or r[0] in ("Address", "Kernel Name"):
        if r and r[0] == "Kernel Name":
            base = None
            ninst += 1
        continue
    a = int(r[0], 16)
    if base is None:
        base = a
    n = int(r[ie])
    tot += n
    ln, op = off2line.get(a - base, (None, "?"))
    byline[ln] += n
    byop[op.split(".")[0]] += n
print("kernel instances in report: %d, total warp instructions %d" % (ninst, tot))
print("opcodes:", ", ".join("%s %.1f%%" % (k, 100 * v / tot) for k, v in byop.most_common(14)))
cache = {}
for ln, v in byline.most_common(40):
    text = ""
    if ln:
        f = ln[0]
        if f not in cache:
            p = os.path.join(root, "orb_slam2_ssd_semantic_b200", "csrc", f)
            if not os.path.exists(p):
                p = os.path.join(root, "include", f)
            cache[f] = open(p).read().splitlines() if os.path.exists(p) else []
        text = cache[f][ln[1] - 1].strip()[:105] if len(cache[f]) >= ln[1] else ""
    print("%5.1f%%  %s:%s  %s" % (100 * v / tot, ln[0] if ln else "?", ln[1] if ln else "", text))

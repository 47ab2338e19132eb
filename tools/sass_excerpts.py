#!/usr/bin/env python3
"""Writes profiles/rNN_sass_excerpts.txt from the built library (no GPU needed): static instruction counts and opcode mix of
the hot kernels, proof lines for what the cubin does / does not contain (TMA, tensor ops), and a few excerpts.
usage: python tools/sass_excerpts.py profiles/r02_sass_excerpts.txt"""
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
out_path = sys.argv[1]
tmp = tempfile.mkdtemp()
subprocess.run(["cuobjdump", "-xelf", "all", os.path.join(ROOT, "orb_slam2_ssd_semantic_b200", "libb200orb.so")], cwd=tmp, capture_output=True)
# one cubin per module of the library: the disassembly of all of them, one after the other
dis = [l for cubin in sorted(f for f in os.listdir(tmp) if f.endswith(".cubin"))
       for l in subprocess.run(["nvdisasm", "-c", os.path.join(tmp, cubin)], capture_output=True, text=True).stdout.splitlines()]
kernels = [("k_fast_cells<48>", "k_fast_cellsILi48E"), ("k_orient_desc", "k_orient_descENS"),
           ("k_quadtree", "10k_quadtreeENS"), ("k_match_last_fused", "k_match_last_fused"),
           ("k_blur7_strip", "k_blur7_strip"), ("k_resize_g", "k_resize_g"), ("k_ocm_scan_keys", "k_ocm_scan_keys"),
           ("k_ocm_bin", "k_ocm_binE"), ("k_dynm_plane_filter", "k_dynm_plane_filter"),
           ("k_dynm_erode<true>", "k_dynm_erodeILb1")]
out = ["# SASS of libb200orb.so (sm_90a): `cuobjdump -xelf all` + `nvdisasm -c` of the library built from this tree by",
       "# csrc/Makefile (nvcc 12.9, -O3 --fmad=false -lineinfo).  Static instruction counts and opcode mix per hot kernel, excerpts."]
tot = collections.Counter()
for l in dis:
    m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(@!?U?P\d\s+)?(\S+)", l)
    if m:
        tot[m.group(3).split(".")[0].rstrip(";")] += 1
out.append("# all cubins: %d instructions.  UTMALDG %d, UTMASTG %d, UTCMMA / tcgen05 %d, HMMA %d, IMMA %d, LDGSTS %d (no TMA, no tensor"
           % (sum(tot.values()), tot["UTMALDG"], tot["UTMASTG"], tot["UTCMMA"], tot["HMMA"], tot["IMMA"], tot["LDGSTS"]))
out.append("# ops: integer / bitwise byte work on 31..43-px tiles at 4-byte alignment, DESIGN.md section 4);  VIMNMX3 %d, VIMNMX %d, POPC %d,"
           % (tot["VIMNMX3"], tot["VIMNMX"], tot["POPC"]))
out.append("# REDUX %d, IDP %d, PRMT %d, VOTE %d, SHFL %d, MATCH %d, ATOMS %d, ATOMG %d, RED %d."
           % (tot["REDUX"], tot["IDP"], tot["PRMT"], tot["VOTE"], tot["SHFL"], tot["MATCH"], tot["ATOMS"], tot["ATOMG"], tot["RED"]))
out.append("")
bodies = {}
for name, mang in kernels:
    try:
        start = next(i for i, l in enumerate(dis) if l.startswith(".text.") and mang in l)
    except StopIteration:
        continue
    c, body = collections.Counter(), []
    for l in dis[start + 1:]:
        if l.startswith(".text."):
            break
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?);", l)
        if m:
            ins = m.group(2)
            body.append(ins)
            c[re.sub(r"^@!?U?P\d\s+", "", ins).split()[0].split(".")[0]] += 1
    bodies[name] = body
    out.append("%-24s %5d instr: %s" % (name, sum(c.values()), ", ".join("%s %d" % kv for kv in c.most_common(12))))
out.append("")


def excerpt(name, pat, before, after, title):
    b = bodies.get(name)
    if not b:
        return
    i = next((i for i, x in enumerate(b) if re.search(pat, x)), None)
    if i is None:
        return
    out.append("## " + title)
    out.extend("    " + x for x in b[max(0, i - before):i + after])
    out.append("")


excerpt("k_fast_cells<48>", r"VIMNMX3\.S16x2", 22, 40,
        "k_fast_cells<48>: exact FAST score of one queued pixel -- LDS.U8 ring loads, IMAD packing (bright | dark in s16x2), VIMNMX3.S16x2 min / max tree")
excerpt("k_orient_desc", r"LDS\.128", 4, 34,
        "k_orient_desc: steered BRIEF -- LDS.128 pattern fetch, FMUL / FADD / F2I rotation, IMAD + LDG.U8 gathers, VOTE")
excerpt("k_resize_g", r"IDP\.2A", 10, 16, "k_resize_g: PRMT + IDP.2A horizontal pass on funnel-shifted source windows")
with open(out_path, "w") as f:
    f.write("\n".join(out) + "\n")
print("\n".join(out[:22]))

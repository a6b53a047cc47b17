#!/usr/bin/env python
"""sass_k2path.py <obj> <func-substr>: static per-opcode count of one iteration of a blend kernel's entry loop on the
k = 2 hierarchy path (the innermost loop around the MUFU.RSQ of pair_hier_alpha, minus the general-k block), e.g.

  python tools/sass_k2path.py hierarchical-3d-gaussians_b200/build/render_backward.o \\
      _ZN5h3dgs22render_backward_kernelILb1ELb0EE

Needs cuobjdump on PATH; no GPU."""
import re, subprocess, sys, collections
obj, fn = sys.argv[1], sys.argv[2]
txt = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
funcs = re.split(r"\n\s*Function : ", txt)
body = [f for f in funcs if fn in f.split("\n")[0]]
assert len(body) == 1, [f.split("\n")[0] for f in body]
ins = []
for line in body[0].split("\n"):
    m = re.match(r"\s+/\*([0-9a-f]{4,5})\*/\s+(.*?)\s*;", line)
    if m:
        ins.append((int(m.group(1), 16), m.group(2)))
def tgt(t):
    m = re.search(r"BRA(?:\.U)?(?:\.ANY)?\s+(?:!?U?P\d,\s*)?(?:`\()?.*?0x([0-9a-f]+)", t)
    return int(m.group(1), 16) if m and "BRA" in t else None
ri = next(i for i, (a, t) in enumerate(ins) if "MUFU.RSQ" in t)
# loop: first backward branch after the RSQ whose target is before it
hi = next(i for i in range(ri, len(ins)) if tgt(ins[i][1]) is not None and tgt(ins[i][1]) <= ins[ri][0])
lo = next(i for i, (a, t) in enumerate(ins) if a >= tgt(ins[hi][1]))
# k = 2 block start: the block containing the RSQ starts after the last unconditional BRA before it
k2s = max(i for i in range(lo, ri) if ins[i][1].startswith("BRA")) + 1
# the branch to it
br = max(i for i in range(lo, k2s) if tgt(ins[i][1]) == ins[k2s][0] and ins[i][1].startswith("@"))
path = ins[lo:br + 1] + ins[k2s:hi + 1]
cls = collections.Counter()
for a, t in path:
    op = t.split()[1] if t.startswith("@") else t.split()[0]
    cls[op.split(".")[0]] += 1
print(f"{fn}: loop {hi + 1 - lo}, k=2 path {len(path)}:", dict(cls.most_common()))

#!/usr/bin/env python
"""Development aid (CPU, emulation build): loop statistics of the blend kernels on a 1/16-scale config #3 frame --
warp iterations, no-taker exits, pixel-entries actually blended, per-group iterations.
usage: python tools/emu_loop_stats.py [leaves=94000]"""
import ctypes as C
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "hierarchical-3d-gaussians_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "emul")):
    sys.path.insert(0, p)
from build_emu import build  # noqa: E402
from emu_api import Emu  # noqa: E402
from h3dgs import synth  # noqa: E402
from oracle import oracle  # noqa: E402

leaves_n = int(sys.argv[1]) if len(sys.argv) > 1 else 94000
W, H = 480, 270
cam = synth.make_camera(W, H)
lv = synth.cloud_v1(leaves_n, cam, sh_degree=3, zmin=2.0, zmax=60.0, seed=0, scale_k=1.0)
z = lv["means3D"][:, 2:3]
lv["scales"] = (4 * 2.4e-3 * np.sqrt(2.0 * z) * np.exp(0.5 * np.random.default_rng(7).standard_normal((z.shape[0], 3)))).astype(np.float32)
h = synth.build_hierarchy(lv)
thr = synth.tau_threshold(6.0, cam)
n, ri, pi, ni = oracle.expand_to_size(h["nodes"], h["boxes"], thr, cam.camera_center)
ts, kids = oracle.get_interpolation_weights(ni, thr, h["nodes"], h["boxes"], cam.camera_center)
emu = Emu(build(tempfile.mkdtemp(prefix="h3dgs_emu_stats")))
emu.L.h3dgs_emu_stats.restype = C.POINTER(C.c_longlong)
st = emu.L.h3dgs_emu_stats()
bg = np.zeros(3, np.float32)
for i in range(16):
    st[i] = 0
a, keep = emu.args(cam, bg, h, ts=ts, kids=kids, ridx=ri, pidx=pi)
fw = emu.forward(a, keep)
g = emu.backward(a, fw, synth.l1_grad(fw["color"]))
s = [st[i] for i in range(16)]
V = int((fw["radii"] > 0).sum())
print(f"cut {n} V {V} D {fw['D']} (D/V {fw['D'] / V:.2f}, mean tile list {fw['D'] / (((W + 15) // 16) * ((H + 15) // 16)):.0f}); t<1 on {float((ts < 1).mean()):.2f} of the cut")
print(f"  forward : {s[8]} warp iterations, {s[9]} pixel-entries blended -> {s[9] / max(s[8], 1):.1f} of 64 pixels per iteration")
print(f"  backward: {s[0]} warp iterations, {s[1]} ({s[1] / max(s[0], 1):.2%}) leave at the no-taker vote, {s[2]} pixel-entries -> {s[2] / max(s[0] - s[1], 1):.1f} of 64 per full iteration; "
      f"group-iterations {s[3]}, of which {s[4]} without a taker")

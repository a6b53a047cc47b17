#!/usr/bin/env python
"""Time of the hierarchy creator (h3dgs.hier_build.build_hierarchy, csrc/hier_build.cu) on seeded clouds:

  sfm1m, sfm1.5m, sfm4m   1M, 1.5M (config #3's leaf count) and 4M Gaussians placed like an SfM reconstruction
                          (tools/bench_knn.py sfm_like), trained-looking attributes: log-normal scales, random
                          rotations, opacities in (0.05, 1), degree-3 SH.

Per cloud: median of --reps builds timed with CUDA events on the current stream after --warmup builds, and the tree
depth (height of the root).  Then the command-line creator at 1.5M (a PLY in save_ply's layout in a temporary
directory), wall time split into PLY read, build and .hier write.  For information only: on config #3's leaves in front
of a 1080p camera (cloud_v1's own scales), the cut size and the PSNR of the tau = 1, 3, 6, 15 px renders against the target-0 (all leaves)
render, for the built hierarchy and for synth.build_hierarchy.  Prints the GPU name and power limit read in the same run,
then one JSON line per measurement.  Writes only under a temporary directory.

  python tools/bench_hier_build.py [--reps 10] [--warmup 2] [--sizes 1000000,1500000,4000000] [--no-cli] [--no-quality]"""
import argparse
import json
import math
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "hierarchical-3d-gaussians_b200")
sys.path.insert(0, os.path.join(ROOT, "tools"))


def cloud(n, seed):
    """-> dict(xyz, shs [n,16,3], opacities [n] activated, log_scales, rotations) float32"""
    from bench_knn import sfm_like
    rs = np.random.default_rng(seed + 100)
    return dict(xyz=sfm_like(n, seed=seed), shs=(0.3 * rs.standard_normal((n, 16, 3))).astype(np.float32),
                opacities=rs.uniform(0.05, 1.0, n).astype(np.float32),
                log_scales=(math.log(0.01) + 0.7 * rs.standard_normal((n, 3))).astype(np.float32),
                rotations=rs.standard_normal((n, 4)).astype(np.float32))


def _build_args(c):
    import torch
    t = {k: torch.from_numpy(v).cuda() for k, v in c.items()}
    return t["xyz"], t["shs"], t["opacities"], t["log_scales"], t["rotations"]


def time_build(c, reps, warmup):
    import torch
    from h3dgs.hier_build import build_hierarchy
    args = _build_args(c)
    for _ in range(warmup):
        h = build_hierarchy(*args)
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        h = build_hierarchy(*args)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    nodes = h["nodes"].cpu().numpy()
    return dict(gpu_ms_median=float(np.median(ms)), gpu_ms_min=float(np.min(ms)), gpu_ms_max=float(np.max(ms)),
                reps=reps, depth=int(nodes[0, 0]), nodes=int(nodes.shape[0]))


def time_cli(c):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    from test_hier_build_cpu import write_ply
    from h3dgs import hier_build
    from gaussian_hierarchy.hier_io import write_hierarchy
    with tempfile.TemporaryDirectory() as d:
        ply = os.path.join(d, "point_cloud.ply")
        logit = np.log(c["opacities"] / (1 - c["opacities"])).astype(np.float32)
        write_ply(ply, c["xyz"], c["shs"], logit, c["log_scales"], c["rotations"])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        g = hier_build.read_ply(ply)
        t1 = time.perf_counter()
        t = {k: torch.from_numpy(v).cuda() for k, v in g.items()}
        h = hier_build.build_hierarchy(t["xyz"], t["shs"], torch.sigmoid(t["opacities"]), t["log_scales"], t["rotations"])
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        write_hierarchy(os.path.join(d, "hierarchy.hier"), h["xyz"], h["shs"], h["opacities"], h["log_scales"],
                        h["rotations"], h["nodes"], h["boxes"])
        t3 = time.perf_counter()
    return dict(read_s=t1 - t0, build_s=t2 - t1, write_s=t3 - t2, total_s=t3 - t0)


def quality():
    """cut size and PSNR vs the target-0 render, built hierarchy vs synth.build_hierarchy, on config #3's leaves"""
    import torch
    from h3dgs import pipeline, synth
    from h3dgs.hier_build import build_hierarchy
    cam = synth.make_camera(1920, 1080)
    # cloud_v1's own scales: bench.py's scale_k = 1.0 leaves are too large to render all at once (target 0)
    leaves = synth.cloud_v1(1_500_000, cam, sh_degree=3, zmin=2.0, zmax=60.0, seed=0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    h = build_hierarchy(t(leaves["means3D"]), t(leaves["shs"]), t(leaves["opacities"][:, 0]),
                        t(np.log(leaves["scales"])), t(leaves["rotations"]))
    h = {k: v.cpu().numpy() for k, v in h.items()}
    q = h["rotations"] / np.linalg.norm(h["rotations"], axis=1, keepdims=True)
    built = dict(means3D=h["xyz"], scales=np.exp(h["log_scales"]), rotations=q.astype(np.float32),
                 opacities=np.abs(h["opacities"]), shs=h["shs"], nodes=h["nodes"], boxes=h["boxes"])
    dcam = pipeline.DeviceCamera(cam)
    bg = torch.zeros(3, device="cuda")
    out = []
    for name, arrays in (("built", built), ("synth", synth.build_hierarchy(leaves))):
        scene = pipeline.Scene(arrays, requires_grad=False)
        with torch.no_grad():
            ref = pipeline.render_hier(scene, dcam, bg, 0.0)[0].clamp(0, 1)
            for tau in (1.0, 3.0, 6.0, 15.0):
                img, _, n = pipeline.render_hier(scene, dcam, bg, synth.tau_threshold(tau, cam))
                mse = float(((img.clamp(0, 1) - ref) ** 2).mean())
                out.append(dict(hierarchy=name, tau=tau, cut=int(n), psnr_vs_target0=10 * math.log10(1 / max(mse, 1e-20))))
        del scene
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sizes", default="1000000,1500000,4000000")
    ap.add_argument("--no-cli", action="store_true")
    ap.add_argument("--no-quality", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_hier_build.py needs a CUDA device: there is no CPU fallback for this path")
    sys.path.insert(0, PKG)
    from bench_knn import gpu_conditions
    torch.cuda.set_device(0)
    print(json.dumps(gpu_conditions()), flush=True)
    for i, n in enumerate(int(s) for s in args.sizes.split(",")):
        r = time_build(cloud(n, i), args.reps, args.warmup)
        print(json.dumps(dict(cloud=f"sfm{n / 1e6:g}m", gaussians=n, **r)), flush=True)
        torch.cuda.empty_cache()
    if not args.no_cli:
        print(json.dumps(dict(cli="creator", gaussians=1_500_000, **time_cli(cloud(1_500_000, 1)))), flush=True)
    if not args.no_quality:
        for r in quality():
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()

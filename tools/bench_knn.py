#!/usr/bin/env python
"""Time of simple_knn._C.distCUDA2 (csrc/knn.cu) on three seeded clouds of the sizes GaussianModel.create_from_pcd sees:

  cube1m    1M points uniform in a cube;
  sfm4m     4M points shaped like an SfM reconstruction: Gaussian blobs with heavy-tailed sizes and weights, plus 1 %
            outliers spread over a box twice the scene's size;
  coarse2m  the coarse stage's input: 2M SfM-like points plus 100 000 skybox points, placed as create_from_pcd places
            them -- a cap of a sphere around the centre of the scene's bounding box, of radius 10x its half-diagonal,
            azimuth uniform, polar angle arccos(1 - 1.4 u) for u uniform in [0, 1).

Per cloud: median of --reps calls timed with CUDA events on the current stream, after --warmup calls; for context, the
host time of scipy cKDTree (build + k=4 query, every core).  Prints the GPU name and power limit read in the same run,
then one JSON line per cloud.  Writes nothing.

  python tools/bench_knn.py [--reps 20] [--warmup 3] [--clouds cube1m,sfm4m,coarse2m]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "hierarchical-3d-gaussians_b200")


def uniform_cube(n, seed=0):
    return np.random.default_rng(seed).uniform(-1.0, 1.0, (n, 3)).astype(np.float32)


def sfm_like(n, seed=1, blobs=4000):
    rs = np.random.default_rng(seed)
    centres = rs.uniform(-50.0, 50.0, (blobs, 3)) * np.array([1.0, 1.0, 0.3])
    sigma = np.minimum(0.02 * (1.0 + rs.pareto(1.2, blobs)), 10.0)          # heavy-tailed blob sizes
    weight = rs.lognormal(0.0, 1.5, blobs)                                   # and uneven point counts
    n_out = n // 100
    which = rs.choice(blobs, n - n_out, p=weight / weight.sum())
    pts = centres[which] + sigma[which, None] * rs.standard_normal((n - n_out, 3))
    outliers = rs.uniform(-100.0, 100.0, (n_out, 3))
    pts = np.concatenate([pts, outliers])
    return pts[rs.permutation(n)].astype(np.float32)


def with_skybox(pts, n_sky, seed=2):
    rs = np.random.default_rng(seed)
    lo, hi = pts.min(axis=0).astype(np.float64), pts.max(axis=0).astype(np.float64)
    mean = 0.5 * (lo + hi)
    radius = 10.0 * np.linalg.norm(hi - mean)
    theta = 2.0 * np.pi * rs.uniform(0.0, 1.0, n_sky)
    phi = np.arccos(1.0 - 1.4 * rs.uniform(0.0, 1.0, n_sky))
    sky = mean + radius * np.stack([np.cos(theta) * np.sin(phi), np.sin(theta) * np.sin(phi), np.cos(phi)], axis=1)
    return np.concatenate([sky.astype(np.float32), pts])                    # skybox first, as create_from_pcd


CLOUDS = {
    "cube1m": lambda: uniform_cube(1_000_000),
    "sfm4m": lambda: sfm_like(4_000_000),
    "coarse2m": lambda: with_skybox(sfm_like(2_000_000, seed=3), 100_000),
}


def gpu_conditions():
    import torch
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(0), "power_limit": r.stdout.strip().split(",")[-1].strip() if r.returncode == 0 else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--clouds", default=",".join(CLOUDS))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_knn.py needs a CUDA device: there is no CPU fallback for this path")
    sys.path.insert(0, PKG)
    from scipy.spatial import cKDTree
    from simple_knn._C import distCUDA2
    torch.cuda.set_device(0)
    print(json.dumps(gpu_conditions()), flush=True)
    for name in args.clouds.split(","):
        pts = CLOUDS[name]()
        x = torch.from_numpy(pts).cuda()
        for _ in range(args.warmup):
            distCUDA2(x)
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            distCUDA2(x)
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
        t0 = time.perf_counter()
        cKDTree(pts).query(pts, k=4, workers=-1)
        host_s = time.perf_counter() - t0
        print(json.dumps({"cloud": name, "points": int(pts.shape[0]), "gpu_ms_median": float(np.median(ms)),
                          "gpu_ms_min": float(np.min(ms)), "gpu_ms_max": float(np.max(ms)), "reps": args.reps,
                          "ckdtree_k4_host_s": host_s, "host_cores": os.cpu_count()}), flush=True)


if __name__ == "__main__":
    main()

"""Times the hierarchy merger (h3dgs.hier_merge.merge_hierarchies, csrc/hier_merge.cu) on seeded chunk scenes: 4 chunks
of 1.5 M Gaussians on a 2 x 2 grid and 16 chunks of 1 M on a 4 x 4 grid, every chunk's cloud spilling 25 % of the cell
width past its cell and built by the creator.  Prints the GPU, its power limit, the median CUDA-event time of the merge
after warm-up, and the command-line merger's wall time split into read, merge and write.  Writes only under a
temporary directory.

    python tools/bench_hier_merge.py [--reps 5] [--warmup 2] [--no-cli]"""
import argparse
import io
import os
import subprocess
import sys
import tempfile
from contextlib import redirect_stdout

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "hierarchical-3d-gaussians_b200"))

WORKLOADS = {"2x2x1.5m": (2, 1_500_000), "4x4x1m": (4, 1_000_000)}
CELL = 50.0


def cells_of(n):
    return np.array([[(i - (n - 1) / 2) * CELL, (j - (n - 1) / 2) * CELL, CELL, CELL] for j in range(n) for i in range(n)],
                    np.float32)


def chunk_cloud(cell, P, seed, spill=0.25):
    """a trained chunk's cloud: uniform over its cell widened by `spill` of the width on every side, SfM-like scales.
    tests/hier_merge_ref.py has a chunk_cloud of the same shape for the unit tests' small cells (4-wide, z in [-1, 1],
    the creator tests' scales); this one is sized for 50-wide cells of a million Gaussians, with a deeper z range and
    larger scales, and stays here so that the tool does not import the test suite."""
    g = np.random.default_rng(seed)
    cx, cy, ex, ey = (float(v) for v in cell)
    xyz = np.stack([g.uniform(cx - (0.5 + spill) * ex, cx + (0.5 + spill) * ex, P),
                    g.uniform(cy - (0.5 + spill) * ey, cy + (0.5 + spill) * ey, P), g.uniform(-5.0, 15.0, P)], 1)
    return dict(xyz=xyz.astype(np.float32), shs=(0.3 * g.standard_normal((P, 16, 3))).astype(np.float32),
                opacities=g.uniform(0.05, 1.0, P).astype(np.float32),
                log_scales=(-3.0 + 0.5 * g.standard_normal((P, 3))).astype(np.float32),
                rotations=g.standard_normal((P, 4)).astype(np.float32))


def scene(name):
    """-> (chunks as dicts of CUDA tensors in the load_hierarchy layout, cells)"""
    import torch
    from h3dgs.hier_build import build_hierarchy
    n, P = WORKLOADS[name]
    cells = cells_of(n)
    chunks = []
    for k, cell in enumerate(cells):
        c = {key: torch.from_numpy(v).cuda() for key, v in chunk_cloud(cell, P, 100 * n + k).items()}
        h = build_hierarchy(c["xyz"], c["shs"], c["opacities"], c["log_scales"], c["rotations"])
        chunks.append({key: h[key] for key in ("xyz", "shs", "opacities", "log_scales", "rotations", "nodes", "boxes")})
    return chunks, cells


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                                   # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-cli", action="store_true")
    a = ap.parse_args()
    import torch
    from h3dgs.hier_merge import merge_hierarchies
    from gaussian_hierarchy import merger
    from gaussian_hierarchy.hier_io import write_hierarchy
    print(f"gpu: {torch.cuda.get_device_name()} | nvidia-smi name, power limit: {gpu_info()}")
    for name in WORKLOADS:
        chunks, cells = scene(name)
        for _ in range(a.warmup):
            h = merge_hierarchies(chunks, cells)
        times = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            h = merge_hierarchies(chunks, cells)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        t = np.array(times)
        nodes_in = sum(int(c["nodes"].shape[0]) for c in chunks)
        print(f"{name}: {len(chunks)} chunks, {nodes_in} nodes in -> {h['items']} pieces, {h['nodes'].shape[0]} nodes, "
              f"{h['xyz'].shape[0]} rows | merge {np.median(t):.1f} ms (min {t.min():.1f}, max {t.max():.1f}, {a.reps} runs)")
        if a.no_cli:
            continue
        with tempfile.TemporaryDirectory() as d:
            names = []
            for k, (c, cell) in enumerate(zip(chunks, cells)):
                nm = f"{k % int(np.sqrt(len(chunks)))}_{k // int(np.sqrt(len(chunks)))}"
                names.append(nm)
                os.makedirs(os.path.join(d, "trained_chunks", nm))
                os.makedirs(os.path.join(d, "chunks", nm))
                write_hierarchy(os.path.join(d, "trained_chunks", nm, "hierarchy.hier_opt"), c["xyz"], c["shs"],
                                c["opacities"], c["log_scales"], c["rotations"], c["nodes"], c["boxes"])
                with open(os.path.join(d, "chunks", nm, "center.txt"), "w") as f:
                    f.write(" ".join(map(str, np.array([cell[0], cell[1], 0.0], np.float64))))
                with open(os.path.join(d, "chunks", nm, "extent.txt"), "w") as f:
                    f.write(" ".join(map(str, np.array([cell[2], cell[3], 2e12], np.float64))))
            buf = io.StringIO()
            with redirect_stdout(buf):
                rc = merger.main([os.path.join(d, "trained_chunks"), "0", os.path.join(d, "chunks"),
                                  os.path.join(d, "merged.hier")] + names)
            print(f"{name}: CLI (rc {rc}): {buf.getvalue().strip()}")
        del chunks, h
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

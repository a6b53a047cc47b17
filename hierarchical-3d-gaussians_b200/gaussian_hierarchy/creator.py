"""The GaussianHierarchyCreator stage of scripts/full_train.py:185-200, on this repository's kernels:

    python -m gaussian_hierarchy.creator <point_cloud.ply> <chunk dir> <output dir> [<scaffold dir>]

reads the chunk's trained point cloud (GaussianModel.save_ply), drops the skybox rows train_single put in front
(scene/gaussian_model.py:235-239; their count is the first line of <scaffold dir>/pc_info.txt, and create_from_hier
appends them again from the scaffold, :355-383), activates opacity with sigmoid, builds the hierarchy on the GPU
(h3dgs.hier_build.build_hierarchy) and writes <output dir>/hierarchy.hier.  <chunk dir> is accepted for argument parity
and not read."""
import os
import sys
import time

import numpy as np
import torch

from h3dgs import hier_build
from gaussian_hierarchy.hier_io import write_hierarchy


def _device():
    """where the build runs (the CPU suite patches this to drive an emulation build)"""
    return torch.device("cuda")


def skybox_points(scaffold_dir):
    with open(os.path.join(scaffold_dir, "pc_info.txt")) as f:
        return int(f.readline())


def main(argv=None):
    argv = sys.argv[1:] if argv is None else list(argv)
    if len(argv) not in (3, 4):
        print(__doc__.strip().splitlines()[2].strip(), file=sys.stderr)
        return 2
    ply, _chunk_dir, out_dir = argv[:3]
    t0 = time.perf_counter()
    g = hier_build.read_ply(ply)
    skip = skybox_points(argv[3]) if len(argv) == 4 else 0
    P = g["xyz"].shape[0] - skip
    if skip < 0 or P < 1:
        raise ValueError(f"{ply}: {g['xyz'].shape[0]} Gaussians, {skip} of them skybox: nothing to build from")
    dev = _device()
    t = lambda k: torch.from_numpy(np.ascontiguousarray(g[k][skip:])).to(dev)
    t1 = time.perf_counter()
    h = hier_build.build_hierarchy(t("xyz"), t("shs"), torch.sigmoid(t("opacities")), t("log_scales"), t("rotations"))
    t2 = time.perf_counter()
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "hierarchy.hier")
    write_hierarchy(path, h["xyz"], h["shs"], h["opacities"], h["log_scales"], h["rotations"], h["nodes"], h["boxes"])
    t3 = time.perf_counter()
    print(f"hierarchy: {P} Gaussians ({skip} skybox rows dropped) -> {2 * P - 1} nodes, {path} "
          f"(read {t1 - t0:.2f} s, build {t2 - t1:.2f} s, write {t3 - t2:.2f} s)")
    return 0


if __name__ == "__main__":
    sys.exit(main())

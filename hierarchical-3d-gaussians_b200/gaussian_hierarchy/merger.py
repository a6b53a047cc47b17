"""The GaussianHierarchyMerger stage of scripts/full_train.py:241-264, on this repository's kernels:

    python -m gaussian_hierarchy.merger <trained_chunks dir> <n> <chunks dir> <output .hier> <chunk name>...

reads every named chunk's post-optimised hierarchy (<trained_chunks dir>/<name>/hierarchy.hier_opt) and its cell
(<chunks dir>/<name>/center.txt and extent.txt, as preprocess/make_chunk.py writes them), merges them on the GPU
(h3dgs.hier_merge.merge_hierarchies: each chunk keeps the leaf Gaussians its cell owns; include/h3dgs.h) and writes
one float32 .hier file.  What upstream reads from the second argument is not known (full_train.py passes "0"): it must
be an integer and is otherwise not read."""
import os
import sys
import time

import numpy as np
import torch

from h3dgs import hier_merge
from gaussian_hierarchy.hier_io import load_hierarchy, write_hierarchy


def _device():
    """where the merge runs (the CPU suite patches this to drive an emulation build)"""
    return torch.device("cuda")


def _usage():
    print(__doc__.strip().splitlines()[2].strip(), file=sys.stderr)
    return 2


def main(argv=None):
    argv = sys.argv[1:] if argv is None else list(argv)
    if len(argv) < 5:
        return _usage()
    trained, n, chunks_dir, out_path, names = argv[0], argv[1], argv[2], argv[3], argv[4:]
    try:
        int(n)
    except ValueError:
        print(f"GaussianHierarchyMerger: the second argument must be an integer, got {n!r}", file=sys.stderr)
        return 2
    paths = []
    for name in names:
        p = (os.path.join(trained, name, "hierarchy.hier_opt"), os.path.join(chunks_dir, name, "center.txt"),
             os.path.join(chunks_dir, name, "extent.txt"))
        for f in p:
            if not os.path.isfile(f):
                print(f"GaussianHierarchyMerger: missing {f}", file=sys.stderr)
                return 1
        paths.append(p)
    t0 = time.perf_counter()
    dev = _device()
    chunks, cells = [], []
    for hier, center, extent in paths:
        xyz, shs, opac, ls, rots, nodes, boxes = load_hierarchy(hier)
        chunks.append({k: v.to(dev) for k, v in dict(xyz=xyz, shs=shs, opacities=opac, log_scales=ls, rotations=rots,
                                                       nodes=nodes, boxes=boxes).items()})
        cells.append(hier_merge.read_cell(center, extent))
    t1 = time.perf_counter()
    h = hier_merge.merge_hierarchies(chunks, np.stack(cells))
    t2 = time.perf_counter()
    d = os.path.dirname(out_path)
    if d:
        os.makedirs(d, exist_ok=True)
    write_hierarchy(out_path, h["xyz"], h["shs"], h["opacities"], h["log_scales"], h["rotations"], h["nodes"], h["boxes"])
    t3 = time.perf_counter()
    rows_in = sum(int(c["xyz"].shape[0]) for c in chunks)
    nodes_in = sum(int(c["nodes"].shape[0]) for c in chunks)
    print(f"merged {len(chunks)} chunks: {nodes_in} nodes, {rows_in} rows -> {h['items']} pieces, "
          f"{h['nodes'].shape[0]} nodes, {h['xyz'].shape[0]} rows, {out_path} "
          f"(read {t1 - t0:.2f} s, merge {t2 - t1:.2f} s, write {t3 - t2:.2f} s)")
    return 0


if __name__ == "__main__":
    sys.exit(main())

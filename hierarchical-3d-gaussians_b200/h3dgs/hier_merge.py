"""The hierarchy merger on libh3dgs.so (csrc/hier_merge.cu, sm_90a): `merge_hierarchies` joins chunk hierarchies into
one, each chunk keeping the leaf Gaussians its cell owns, in the arrays `gaussian_hierarchy._C.write_hierarchy` takes
(rule: include/h3dgs.h h3dgs_merge_hierarchies).  `read_cell` reads a chunk's center.txt / extent.txt.
No CPU fallback; raises if the library is missing or a call fails."""
import ctypes as C

import numpy as np
import torch

from h3dgs import _lib

_scratch = {}
_OUT = ("xyz", "shs", "opacities", "log_scales", "rotations", "nodes", "boxes", "source_chunk", "source_row")


def _on_device(t):
    """the library takes device pointers (the CPU suite patches this to drive an emulation build)"""
    return t.is_cuda


def read_cell(center_txt, extent_txt):
    """(cx, cy, ex, ey) of a chunk: the first two numbers of make_chunk.py's center.txt and extent.txt (full widths),
    parsed as Python floats and then rounded to float32"""
    vals = []
    for path in (center_txt, extent_txt):
        with open(path) as f:
            w = f.read().split()
        if len(w) < 2:
            raise ValueError(f"{path}: expected at least two numbers, found {len(w)}")
        vals += [float(w[0]), float(w[1])]
    return np.array(vals, np.float32)


def merge_hierarchies(chunks, cells):
    """chunks: K >= 1 dicts of tensors on one CUDA device in the load_hierarchy layout: xyz [M,3], shs [M,16,3],
    opacities [M] or [M,1] (activated), log_scales [M,3], rotations [M,4] (float32), nodes [N,7] (int32, chunk-local
    indices), boxes [N,2,4] (float32).  cells: [K,4] (cx, cy, ex, ey) per chunk.  -> dict with xyz, shs, opacities
    [RO,1], log_scales, rotations, nodes, boxes, source_chunk and source_row (int32: the chunk and its row of every
    output row, -1 for a merged row), on the input's device.  Runs on the current stream and synchronises it (an
    offline step)."""
    K = len(chunks)
    if K < 1:
        raise ValueError("merge_hierarchies: needs at least one chunk")
    cells = np.ascontiguousarray(np.asarray(cells, np.float32).reshape(K, 4))
    dev = chunks[0]["xyz"].device
    parts = {k: [] for k in ("xyz", "shs", "opacities", "log_scales", "rotations", "nodes", "boxes")}
    n_off, r_off = [0], [0]
    for i, c in enumerate(chunks):
        M, N = int(c["xyz"].shape[0]), int(c["nodes"].shape[0])
        want = dict(xyz=(M, 3), shs=(M, 16, 3), opacities=(M,), log_scales=(M, 3), rotations=(M, 4), nodes=(N, 7),
                    boxes=(N, 2, 4))
        for k, shape in want.items():
            t = c[k].reshape(M) if k == "opacities" and c[k].numel() == M else c[k]
            dtype = torch.int32 if k == "nodes" else torch.float32
            if tuple(t.shape) != shape or t.dtype != dtype:
                raise ValueError(f"merge_hierarchies: chunk {i}: {k} is {tuple(t.shape)} {t.dtype}, expected {shape} {dtype}")
            if not _on_device(t) or t.device != dev:
                raise RuntimeError("merge_hierarchies: inputs must be CUDA tensors on one device")
            parts[k].append(t)
        n_off.append(n_off[-1] + N)
        r_off.append(r_off[-1] + M)
    cat = {k: torch.cat(v).contiguous() if len(v) > 1 else v[0].contiguous() for k, v in parts.items()}
    L = _lib.lib()
    need = L.h3dgs_merge_hierarchies_scratch_bytes(K, n_off[-1], r_off[-1])
    if need == 0:
        raise ValueError(f"merge_hierarchies: {n_off[-1]} nodes and {r_off[-1]} rows are out of range")
    key = (dev.index,)
    s = _scratch.get(key)
    if s is None or s.numel() < need:
        _scratch.pop(key, None)                  # release the old block before allocating the larger one
        s = torch.empty((need,), dtype=torch.uint8, device=dev)
        _scratch[key] = s
    bufs = {}

    def alloc(_user, which, nbytes):
        dtype = torch.uint8 if which == 9 else (torch.int32 if which in (5, 7, 8) else torch.float32)
        n = max(int(nbytes), 1) if which == 9 else int(nbytes) // 4
        bufs[which] = torch.empty((max(n, 1),), dtype=dtype, device=dev)
        return bufs[which].data_ptr()
    cb = _lib.ALLOC_FN(alloc)
    noff = np.array(n_off, np.int64)
    roff = np.array(r_off, np.int64)
    counts = np.zeros(3, np.int64)
    with torch.cuda.device(dev):
        _lib.check(L.h3dgs_merge_hierarchies(
            K, noff.ctypes.data, roff.ctypes.data, cells.ctypes.data, cat["xyz"].data_ptr(), cat["shs"].data_ptr(),
            cat["opacities"].data_ptr(), cat["log_scales"].data_ptr(), cat["rotations"].data_ptr(),
            cat["nodes"].data_ptr(), cat["boxes"].data_ptr(), cb, None, counts.ctypes.data, s.data_ptr(),
            torch.cuda.current_stream().cuda_stream))
    NO, RO, R = (int(v) for v in counts)
    shapes = dict(xyz=(RO, 3), shs=(RO, 16, 3), opacities=(RO, 1), log_scales=(RO, 3), rotations=(RO, 4), nodes=(NO, 7),
                  boxes=(NO, 2, 4), source_chunk=(RO,), source_row=(RO,))
    out = {k: bufs[i][:int(np.prod(shapes[k]))].view(shapes[k]) for i, k in enumerate(_OUT)}
    out["items"] = R
    return out

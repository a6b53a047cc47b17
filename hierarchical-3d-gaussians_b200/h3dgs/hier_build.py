"""The hierarchy creator on libh3dgs.so (csrc/hier_build.cu, sm_90a): `build_hierarchy` turns trained Gaussians into the
arrays `gaussian_hierarchy._C.write_hierarchy` takes (rule: include/h3dgs.h h3dgs_build_hierarchy), and `read_ply`
reads the point clouds GaussianModel.save_ply writes (scene/gaussian_model.py:491-508).
No CPU fallback; raises if the library is missing or a call fails."""
import numpy as np
import torch

from h3dgs import _lib

_scratch = {}


def _on_device(t):
    """the library takes device pointers (the CPU suite patches this to drive an emulation build)"""
    return t.is_cuda


def build_hierarchy(xyz, shs, opacities, log_scales, rotations):
    """xyz [P,3], shs [P,K,3] (K = 1, 4, 9 or 16; zero-padded to 16), activated opacities [P] or [P,1], log_scales [P,3],
    rotations [P,4] wxyz: float32 tensors on one CUDA device.  -> dict with xyz, shs [N,16,3], opacities [N,1],
    log_scales, rotations, nodes [N,7] int32, boxes [N,2,4] and source [N] int32 (input row of a leaf, -1 for a merged
    row), N = 2P - 1, on the input's device.  Runs on the current stream and synchronises it (an offline step)."""
    P = int(xyz.shape[0])
    if P < 1:
        raise ValueError("build_hierarchy: needs at least one Gaussian")
    opacities = opacities.reshape(P)
    K = int(shs.shape[1]) if shs.dim() == 3 else -1
    shapes = ((xyz, (P, 3)), (log_scales, (P, 3)), (rotations, (P, 4)), (opacities, (P,)))
    if K not in (1, 4, 9, 16) or tuple(shs.shape) != (P, K, 3) or any(tuple(t.shape) != s for t, s in shapes):
        raise ValueError("build_hierarchy: expected xyz [P,3], shs [P,K,3] with K in 1, 4, 9, 16, opacities [P], "
                         "log_scales [P,3], rotations [P,4]")
    ins = (xyz, shs, opacities, log_scales, rotations)
    if any(not _on_device(t) or t.dtype != torch.float32 or t.device != xyz.device for t in ins):
        raise RuntimeError("build_hierarchy: inputs must be float32 CUDA tensors on one device")
    dev = xyz.device
    if K < 16:                                   # the filler of GaussianModel.create_from_hier
        shs = torch.cat((shs, torch.zeros((P, 16 - K, 3), dtype=torch.float32, device=dev)), 1)
    xyz, shs, opacities, log_scales, rotations = (t.contiguous() for t in (xyz, shs, opacities, log_scales, rotations))
    N = 2 * P - 1
    f = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
    out = dict(xyz=f(N, 3), shs=f(N, 16, 3), opacities=f(N, 1), log_scales=f(N, 3), rotations=f(N, 4),
               nodes=torch.empty((N, 7), dtype=torch.int32, device=dev), boxes=f(N, 2, 4),
               source=torch.empty((N,), dtype=torch.int32, device=dev))
    L = _lib.lib()
    need = L.h3dgs_build_hierarchy_scratch_bytes(P)
    if need == 0:
        raise ValueError(f"build_hierarchy: P = {P} is out of range")
    key = (dev.index,)
    s = _scratch.get(key)
    if s is None or s.numel() < need:
        _scratch.pop(key, None)                  # release the old block before allocating the larger one
        s = torch.empty((need,), dtype=torch.uint8, device=dev)
        _scratch[key] = s
    with torch.cuda.device(dev):
        _lib.check(L.h3dgs_build_hierarchy(
            P, xyz.data_ptr(), log_scales.data_ptr(), rotations.data_ptr(), opacities.data_ptr(), shs.data_ptr(),
            out["xyz"].data_ptr(), out["shs"].data_ptr(), out["opacities"].data_ptr(), out["log_scales"].data_ptr(),
            out["rotations"].data_ptr(), out["nodes"].data_ptr(), out["boxes"].data_ptr(), out["source"].data_ptr(),
            s.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return out


_PLY_TYPES = {"float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8", "uchar": "u1", "uint8": "u1",
              "char": "i1", "int8": "i1", "short": "<i2", "int16": "<i2", "ushort": "<u2", "uint16": "<u2",
              "int": "<i4", "int32": "<i4", "uint": "<u4", "uint32": "<u4"}


def read_ply(path):
    """A binary little-endian PLY of GaussianModel.save_ply (properties found by name; 0, 9, 24 or 45 f_rest_*) ->
    dict of float32 arrays: xyz [P,3], shs [P,K,3] (K = 1 + f_rest / 3, coefficient-major as get_features),
    opacities [P] (raw logits, as stored), log_scales [P,3], rotations [P,4] (as stored)."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        props, P, fmt, in_vertex = [], None, None, False
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: no end_header")
            w = line.decode("ascii", "replace").split()
            if not w or w[0] in ("comment", "obj_info"):
                continue
            if w[0] == "end_header":
                break
            if w[0] == "format":
                fmt = w[1]
            elif w[0] == "element":
                in_vertex = w[1] == "vertex"
                if in_vertex:
                    P = int(w[2])
                elif P is None:
                    raise ValueError(f"{path}: an element before 'vertex' is not supported")
            elif w[0] == "property" and in_vertex:
                if w[1] == "list" or w[1] not in _PLY_TYPES:
                    raise ValueError(f"{path}: unsupported vertex property {' '.join(w[1:])}")
                props.append((w[2], _PLY_TYPES[w[1]]))
        if fmt != "binary_little_endian":
            raise ValueError(f"{path}: format {fmt}, expected binary_little_endian")
        if P is None:
            raise ValueError(f"{path}: no vertex element")
        dt = np.dtype(props)
        data = np.fromfile(f, dtype=dt, count=P)
        if data.shape[0] != P:
            raise ValueError(f"{path}: {data.shape[0]} of {P} vertices present")
    names = set(dt.names)
    need = ["x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2", "opacity"] + [f"scale_{i}" for i in range(3)] + \
        [f"rot_{i}" for i in range(4)]
    missing = [n for n in need if n not in names]
    if missing:
        raise ValueError(f"{path}: missing properties {missing}")
    R = sum(1 for n in names if n.startswith("f_rest_"))
    if R not in (0, 9, 24, 45) or any(f"f_rest_{i}" not in names for i in range(R)):
        raise ValueError(f"{path}: {R} f_rest_* properties, expected 0, 9, 24 or 45 numbered from 0")
    col = lambda ns: np.stack([data[n].astype(np.float32) for n in ns], 1)
    K = 1 + R // 3
    shs = np.zeros((P, K, 3), np.float32)
    shs[:, 0] = col([f"f_dc_{i}" for i in range(3)])
    if R:      # save_ply flattens features_rest.transpose(1, 2): channel-major
        shs[:, 1:] = col([f"f_rest_{i}" for i in range(R)]).reshape(P, 3, K - 1).transpose(0, 2, 1)
    return dict(xyz=col("xyz"), shs=shs, opacities=data["opacity"].astype(np.float32),
                log_scales=col([f"scale_{i}" for i in range(3)]), rotations=col([f"rot_{i}" for i in range(4)]))

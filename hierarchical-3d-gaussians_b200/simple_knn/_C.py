"""`simple_knn._C`: distCUDA2 on libh3dgs.so (csrc/knn.cu, sm_90a), the signature of the reference's call site
(scene/gaussian_model.py:192: `distCUDA2(torch.from_numpy(points).float().cuda())`).
No CPU fallback; raises if the library is missing or a call fails."""
import torch

from h3dgs import _lib

_scratch = {}


def _on_device(t):
    """the library takes device pointers (the CPU suite patches this to drive an emulation build)"""
    return t.is_cuda


def distCUDA2(points):
    """points: float32 CUDA tensor [P, 3] -> float32 tensor [P] on the same device: the mean of the squared distances
    from each point to its three nearest other points (exact; see include/h3dgs.h h3dgs_dist_knn3)."""
    if not _on_device(points) or points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] != 3:
        raise RuntimeError("distCUDA2: points must be a float32 CUDA tensor of shape [P, 3]")
    L = _lib.lib()
    points = points.contiguous()
    P = int(points.shape[0])
    out = torch.empty((P,), dtype=torch.float32, device=points.device)
    if P == 0:
        return out
    need = L.h3dgs_knn_scratch_bytes(P)
    key = (points.device.index, )
    s = _scratch.get(key)
    if s is None or s.numel() < need:
        s = torch.empty((need,), dtype=torch.uint8, device=points.device)
        _scratch[key] = s
    with torch.cuda.device(points.device):
        _lib.check(L.h3dgs_dist_knn3(P, points.data_ptr(), out.data_ptr(), s.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream))
    return out

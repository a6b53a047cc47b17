"""Sparse Adam on libh3dgs.so (SURVEY.md 8f-4): the reference's `scene/OurAdam.py` `Adam.step(relevant)`
(train_single.py:170-178) as one in-place kernel per parameter tensor instead of gather / ~10 elementwise
kernels / three scatters.  Same constructor defaults, `step(relevant)` signature and state keys
(`step`, `exp_avg`, `exp_avg_sq`).  amsgrad / weight_decay / maximize / capturable are not supported
(the reference's call sites never set them).  No CPU fallback."""
import os

import torch
from torch.optim.optimizer import Optimizer

from . import _lib


class Adam(Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False):
        if weight_decay != 0 or amsgrad:
            raise NotImplementedError("sparse Adam: weight_decay / amsgrad are not supported")
        if not 0.0 <= lr or not 0.0 <= eps or not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError("invalid Adam hyper-parameter")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=0, amsgrad=False))

    @torch.no_grad()
    def step(self, relevant, closure=None):
        """relevant: int64 CUDA tensor of row indices to update (scene/OurAdam.py:116).  1-D: the rows must be UNIQUE and
        in range -- what train_single's call site produces (`(grad != 0).nonzero().flatten()`, train_single.py:170-174):
        the kernel updates rows in place, so a duplicate index is a data race (the reference's gather / scatter would be
        last-write-wins) and an index >= rows an out-of-bounds write.  H3DGS_DEBUG_CHECKS=1 verifies both (one sync).
        [R,2]: train_coarse's unflattened `(opacity.grad != 0).nonzero()` (train_coarse.py:136-137).  Indexing with it
        selects the rows of column 0 and, through column 1 (all zeros), row 0; OurAdam updates exactly that row set, so
        here the rows of column 0 other than 0 are updated, and row 0 once when R > 0 -- no host synchronisation.
        An EMPTY index (R == 0, 1-D or [0,2]) is OurAdam's dense step: every row of every parameter is updated
        (scene/OurAdam.py:214-228 -> _single_tensor_adam2), as the reference does when no gradient is non-zero."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        L = _lib.lib()
        relevant = relevant.to(torch.int64)
        pairs = relevant.dim() == 2
        if pairs:
            if relevant.shape[0]:
                rows = relevant[:, 0]
                relevant = torch.cat((rows.masked_fill(rows == 0, -1), rows.new_zeros(1)))     # -1: skipped by the kernel
            else:
                relevant = relevant.new_zeros(0)
        relevant = relevant.contiguous()
        R = int(relevant.numel())
        debug = os.environ.get("H3DGS_DEBUG_CHECKS") == "1"
        for group in self.param_groups:
            b1, b2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
                    raise RuntimeError("sparse Adam needs contiguous float32 CUDA parameters (no CPU fallback)")
                if relevant.device != p.device:
                    raise RuntimeError(f"relevant lives on {relevant.device}, the parameter on {p.device}")
                kept = relevant[relevant >= 0] if (debug and pairs) else relevant
                if debug and R and (int(kept.min()) < 0 or int(kept.max()) >= p.shape[0] or
                                    int(torch.unique(kept).numel()) != kept.numel()):
                    raise RuntimeError("sparse Adam: relevant must hold unique row indices in [0, rows)")
                st = self.state[p]
                if len(st) == 0:
                    st["step"] = torch.tensor(0.0)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["step"] += 1                       # every call, whatever the rows (scene/OurAdam.py:277)
                width = p.numel() // p.shape[0]
                g = p.grad.contiguous()
                # R == 0: the dense step over every row (a NULL index)
                rows, idx = (R, relevant.data_ptr()) if R else (p.shape[0], None)
                with torch.cuda.device(p.device):
                    _lib.check(L.h3dgs_sparse_adam(rows, width, idx, p.data_ptr(), g.data_ptr(),
                                                   st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(),
                                                   float(group["lr"]), float(b1), float(b2), float(group["eps"]),
                                                   int(st["step"].item()), torch.cuda.current_stream().cuda_stream))
        return loss

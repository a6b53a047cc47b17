"""Sync-free step of train_post's objective (hierarchy post-optimisation), replayed from CUDA graphs.

GraphedStep's loss is mean |image - gt|.  The loop body train_post.py:91-142 optimises something else:

    y    = image.permute(1,2,0) @ E[:3,:3] + E[:3,3]      render_post with use_trained_exp (E = the image's exposure)
    a    = clamp(y, 0, 1) * alpha_mask                    render_post :285, train_post.py:135-137
    loss = (1-l) mean|a - gt| + l (1 - SSIM(a, gt))       l = lambda_dssim (0.2)

GraphedPostStep keeps GraphedStep's graph A (LOD cut with the threshold on the device, skybox rows, capacity-mode forward)
and replaces the loss half of graph B by csrc/loss.cu's post-loss kernels: exposure, clamp and mask are applied while the
SSIM tile is staged, and the backward chains through mask, clamp and exposure in the kernel that convolves the derivative
maps, so dL/dimage is written once.  One device thread then stores [loss, L1, SSIM, rows, D, longest tile list, binning
overflow, row overflow].  Camera, target, mask, exposure and LOD threshold are device-resident inputs that change between
replays; nothing in the step returns to the host.

A frame that does not fit the capacities is flagged, renders the background only and contributes zero gradients, as in
GraphedStep; the caller re-runs it through pipeline.post_step, the exact path with the same kernels.  Gradients are with
respect to the activated Scene tensors; the optimizer and the skybox / anchor gradient zeroing of train_post.py:167-181
stay the caller's.  One GPU only: the SSIM window reaches across the tile-row shards of the sharded forms.
"""
import ctypes as C

import torch

from . import _lib
from .graphstep import GraphedStep, _ptr
from .loss import _coefficients


class GraphedPostStep(GraphedStep):
    """scene: pipeline.Scene with a hierarchy.  Fixed per instance: W, H, tanfovx, tanfovy, lambda_dssim, and whether an
    exposure and an alpha mask are applied.  Changing between replays: set_camera, set_threshold, the target and its mask
    (upload_target(src, stream, mask) into one of two slots, or step(gt=, mask=)), and the exposure (step(exposure=)).

    The arithmetic is the one of pipeline.post_step: image and radii are bit-identical whenever the frame fits, dL/dimage
    too, and the Gaussian gradients equal up to the order of the backward's atomic sums."""

    def __init__(self, scene, W, H, tanfovx, tanfovy, bg, threshold, lambda_dssim=0.2, exposure=False, mask=False,
                 sh_degree=3, row_capacity=None, bin_capacity=1 << 22, sort_capacity=4096, world=1, capture=True):
        if int(world) != 1:
            raise ValueError("GraphedPostStep runs on one GPU: the SSIM window reaches across the tile-row shards")
        super().__init__(scene, W, H, tanfovx, tanfovy, bg, threshold, sh_degree=sh_degree, row_capacity=row_capacity,
                         bin_capacity=bin_capacity, sort_capacity=sort_capacity, capture=False)
        dev, H, W = self.dev, self.H, self.W
        self.lambda_dssim = float(lambda_dssim)
        self._identity = torch.eye(3, 4, device=dev)
        self.exposure = self._identity.clone() if exposure else None
        # one mask per target slot: a mask travels with its target
        self.mask_bufs = [torch.ones((H, W), device=dev), torch.ones((H, W), device=dev)] if mask else [None, None]
        self.mask = self.mask_bufs[0]
        self.sums = torch.zeros(2, dtype=torch.float64, device=dev)
        self.maps = torch.zeros((3, 3, H, W), dtype=torch.float32, device=dev)
        self.status_dev = torch.zeros(8, dtype=torch.float64, device=dev)
        # the weights of sign(a - gt) and of the SSIM-sum gradient for loss.backward(), formed as post_loss's backward
        # forms them, so that the graphed dL/dimage equals the eager one bit for bit
        one, zero = torch.ones((), device=dev), torch.zeros((), device=dev)
        self.coeffs = _coefficients(one, zero, zero, self.lambda_dssim, float(3 * H * W))
        if capture:
            self.capture()

    def _part_b(self, slot=0):
        """The objective against target slot `slot` and its mask, its gradient, the backward, the status words."""
        L, st = self.L, self._stream()
        gt, M = self.gt_bufs[slot], self.mask_bufs[slot]
        _lib.check(L.h3dgs_post_loss_forward(self.H, self.W, self.image.data_ptr(), gt.data_ptr(), _ptr(self.exposure),
                                             _ptr(M), self.sums.data_ptr(), self.maps.data_ptr(), st))
        _lib.check(L.h3dgs_post_loss_backward(self.H, self.W, self.image.data_ptr(), gt.data_ptr(), _ptr(self.exposure),
                                              _ptr(M), self.maps.data_ptr(), self.coeffs.data_ptr(), self.dcolor.data_ptr(), st))
        g = self.grads
        outs = (g["means3D"].data_ptr(), self.d_means2D.data_ptr(), g["shs"].data_ptr(), None, g["opacities"].data_ptr(),
                g["scales"].data_ptr(), g["rotations"].data_ptr(), None)
        state = (self.radii.data_ptr(), self._bufs[0].data_ptr(), self._bufs[1].data_ptr(), self._bufs[2].data_ptr(),
                 self.bin_capacity, self.dcolor.data_ptr(), None)
        _lib.check(L.h3dgs_rasterize_backward(C.byref(self.args), *state, *outs, self.accum.data_ptr(), 3, st))
        _lib.check(L.h3dgs_post_step_status(self.sums.data_ptr(), 1.0 / self.image.numel(), self.lambda_dssim,
                                            self.count.data_ptr(), self.S, self.P, self.scan_info().data_ptr(),
                                            self.status_dev.data_ptr(), st))

    def _set_mask(self, slot, mask):
        if self.mask_bufs[slot] is None:
            if mask is not None:
                raise ValueError("this step was built without a mask (mask=False)")
            return
        if mask is None:
            self.mask_bufs[slot].fill_(1.0)               # no alpha mask: ones, as the reference's loader falls back to
        else:
            self.mask_bufs[slot].copy_(mask.reshape(self.H, self.W), non_blocking=True)

    def upload_target(self, src, stream, mask=None):
        """Copy the NEXT step's target and its alpha mask ([1,H,W] or [H,W]; None = ones) into one of the two target slots
        on `stream`, after the last step that read that slot has finished; returns the event to hand to step() as
        gt_ready (step() also picks the slot up by itself)."""
        slot = self._upload_slot
        self._upload_slot ^= 1
        with torch.cuda.stream(stream):
            stream.wait_event(self._slot_done[slot])
            self.gt_bufs[slot].copy_(src, non_blocking=True)
            self._set_mask(slot, mask)
            ready = torch.cuda.Event()
            ready.record(stream)
        self._pending = (slot, ready)
        return ready

    def step(self, cam=None, gt=None, mask=None, exposure=None, gt_ready=None):
        """cam, gt (+ its mask; None = ones): optional new inputs, copied into the static buffers (the target into slot
        0).  exposure: this step's [3,4] (or larger: its top 3x4 block) exposure; None = identity, as render_post does for
        an image without one.  gt_ready: the event upload_target() returned."""
        if mask is not None and gt is None:
            raise ValueError("a mask travels with its target: pass gt with it, or upload both with upload_target")
        if self.exposure is not None:
            self.exposure.copy_(self._identity if exposure is None else exposure[:3, :4], non_blocking=True)
        elif exposure is not None:
            raise ValueError("this step was built without an exposure (exposure=False)")
        if gt is not None:
            self._set_mask(0, mask)
        return super().step(cam, gt, gt_ready)

    def status(self):
        """One 64-byte read-back: loss, L1, SSIM, rows needed, D, longest tile list, overflow flag."""
        s = self.status_dev.cpu()
        return dict(loss=float(s[0]), l1=float(s[1]), ssim=float(s[2]), rows=int(s[3]), D=int(s[4]),
                    longest_list=int(s[5]), overflow=bool(s[6] != 0 or s[7] != 0))

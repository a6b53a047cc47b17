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
import torch

from . import _lib
from .graphstep import GraphedStep


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
        self._init_post_loss(lambda_dssim, exposure, mask)
        self.status_dev = torch.zeros(8, dtype=torch.float64, device=self.dev)
        if capture:
            self.capture()

    def _part_b(self, slot=0):
        """The objective against target slot `slot` and its mask, its gradient, the backward, the status words."""
        self._post_loss(slot)
        self._backward(3)
        _lib.check(self.L.h3dgs_post_step_status(self.sums.data_ptr(), 1.0 / self.image.numel(), self.lambda_dssim,
                                                 self.count.data_ptr(), self.S, self.P, self.scan_info().data_ptr(),
                                                 self.status_dev.data_ptr(), self._stream()))

    def step(self, cam=None, gt=None, mask=None, exposure=None, gt_ready=None):
        """cam, gt (+ its mask; None = ones): optional new inputs, copied into the static buffers (the target into slot
        0).  exposure: this step's [3,4] (or larger: its top 3x4 block) exposure; None = identity, as render_post does for
        an image without one.  gt_ready: the event upload_target() returned."""
        if mask is not None and gt is None:
            raise ValueError("a mask travels with its target: pass gt with it, or upload both with upload_target")
        self._set_exposure(exposure)
        if gt is not None:
            self._set_mask(0, mask)
        return super().step(cam, gt, gt_ready)

    def status(self):
        """One 64-byte read-back: loss, L1, SSIM, rows needed, D, longest tile list, overflow flag."""
        s = self.status_dev.cpu()
        return dict(loss=float(s[0]), l1=float(s[1]), ssim=float(s[2]), rows=int(s[3]), D=int(s[4]),
                    longest_list=int(s[5]), overflow=bool(s[6] != 0 or s[7] != 0))

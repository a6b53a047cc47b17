"""Sync-free step of train_single's objective on a flat chunk, replayed from CUDA graphs.

The loop body train_single.py:94-148 is, per step:

    image, radii, invdepth = rasterizer(do_depth=True, bg = this step's random background)
    y     = image.permute(1,2,0) @ E[:3,:3] + E[:3,3]      E = the image's TRAINED exposure          render() :115-117
    a     = clamp(y, 0, 1) * alpha_mask                                                               :118, train_single.py:102-104
    photo = (1-l) mean|a - gt| + l (1 - SSIM(a, gt))                                                  :106-108
    loss  = photo + w mean|(invdepth - mono_invdepth) * depth_mask|      w = depth_l1_weight(iteration)   :111-117
    loss.backward()
    max_radii2D / xyz_gradient_accum / denom updated for the rows with radii > 0                      :147-148

GraphedSingleStep runs it as graph A = the capacity-mode forward with the inverse depth (all N rows, no LOD cut) and
graph B = csrc/loss.cu's post-loss forward, its backward with the exposure gradient, the inverse-depth L1 kernel, the
rasterizer backward fed with dL/dimage and dL/dinvdepth, the densification statistics kernel and one device thread that
stores [loss, photo, L1, SSIM, depth L1, D, longest tile list, overflow] and the fp32 exposure gradient.  Camera,
background, exposure, depth weight and the two slots of {target, alpha mask, mono inverse depth, depth mask} are
device-resident inputs that change between replays; nothing in the step returns to the host.

A frame that does not fit the capacities is flagged, renders the background only, contributes zero gradients (the
exposure's included) and leaves the statistics as they were; the caller re-runs it through pipeline.single_step, the
exact path with the same kernels.  Gradients are with respect to the activated Scene tensors.  The optimizers (sparse
Adam over the rows with a gradient, the exposure's Adam), densify_and_prune, reset_opacity and the big-Gaussian
rescale of train_single.py:150-186 stay the caller's.  One GPU only: the SSIM window reaches across tile-row shards.
"""
import torch

from . import _lib
from ._lib import ptr
from .graphstep import GraphedBase
from .pipeline import DensifyStats


class GraphedSingleStep(GraphedBase):
    """scene: a flat pipeline.Scene.  Fixed per instance: W, H, tanfovx, tanfovy, lambda_dssim, and what the objective
    contains: exposure (a trained exposure, with its gradient in exposure_grad), mask (an alpha mask), depth (the
    inverse-depth term) and stats (the densification statistics; True for zeros, or a pipeline.DensifyStats of the
    scene's row count to carry on from).  Changing between replays: set_camera, set_background, set_depth_weight, the
    exposure (step(exposure=)) and the target with its mask and depth maps (upload_target(src, stream, mask,
    mono_invdepth, depth_mask) into one of two slots, or step(gt=, ...)).

    The row count N and the active SH degree are launch constants inside the graphs.  N changes at every
    densify_and_prune and the degree at every oneupSHdegree (train_single.py:91-92, 150-151): construct a new step
    then, handing it the statistics to carry over (tools/bench_single_step.py reports what a construction with its
    capture costs, against the 100-300 steps between two densifications).  capture()'s eager warm-up step does not
    count in the statistics.  The reference keeps them only while iteration < densify_until_iter (train_single.py:145):
    from then on use a step built with stats=False.

    The arithmetic is the one of pipeline.single_step: image, inverse depth and radii are bit-identical whenever the
    frame fits, dL/dimage and dL/dinvdepth too, the statistics too, and the Gaussian gradients equal up to the order of
    the backward's atomic sums."""

    def __init__(self, scene, W, H, tanfovx, tanfovy, lambda_dssim=0.2, exposure=True, mask=False, depth=True, stats=True,
                 sh_degree=3, bin_capacity=1 << 22, sort_capacity=4096, world=1, capture=True):
        if int(world) != 1:
            raise ValueError("GraphedSingleStep runs on one GPU: the SSIM window reaches across the tile-row shards")
        if scene.hier:
            raise ValueError("GraphedSingleStep trains a flat scene (train_single.py); a hierarchy goes through GraphedPostStep")
        super().__init__(scene, W, H, sh_degree, None, bin_capacity, sort_capacity)
        dev, H, W, N, f = self.dev, self.H, self.W, self.N, self._zeros
        # inputs that change between replays, and what travels with a target, one per slot
        self.bg, self.depth_weight = f(3), f(1)
        self._init_post_loss(lambda_dssim, exposure, mask)
        self.mono_bufs = [f(H, W), f(H, W)] if depth else [None, None]
        self.depth_mask_bufs = [f(H, W), f(H, W)] if depth else [None, None]
        # outputs
        self.image, self.invdepth = f(3, H, W), f(1, H, W)
        self.dinvdepth = f(H, W) if depth else None
        self.depth_sum = torch.zeros(1, dtype=torch.float64, device=dev) if depth else None
        self.exposure_grad64 = torch.zeros((3, 4), dtype=torch.float64, device=dev) if exposure else None
        self.exposure_grad = f(3, 4) if exposure else None
        self.status_dev = torch.zeros(8, dtype=torch.float64, device=dev)
        self._init_grads(N)
        if isinstance(stats, DensifyStats):
            if stats.denom.shape[0] != N:
                raise ValueError(f"the statistics hold {stats.denom.shape[0]} rows, the scene {N}")
            self.stats = stats
        else:
            self.stats = DensifyStats(N, dev) if stats else None
        self._count_stats = True
        self.args = self._raster_args(tanfovx, tanfovy, do_depth=1)
        if capture:
            self.capture()

    def _warm_up(self):
        """capture()'s eager step runs on whatever the buffers hold -- a camera set beforehand against a zero target,
        say: it must not count in statistics that are carried across steps and across rebuilt instances"""
        self._count_stats = False
        try:
            super()._warm_up()
        finally:
            self._count_stats = True

    # ---- the two halves of the step (eager or under capture) ------------------------------
    def _part_a(self):
        """capacity-mode forward of all N rows, with the inverse depth"""
        self._forward(self.image, self.invdepth)

    def _part_b(self, slot=0):
        """The objective against slot `slot`, its gradients, the backward, the statistics, the status words."""
        L, st, H, W = self.L, self._stream(), self.H, self.W
        self._post_loss(slot, self.exposure_grad64)
        if self.dinvdepth is not None:
            _lib.check(L.h3dgs_invdepth_l1_grad(H, W, self.invdepth.data_ptr(), self.mono_bufs[slot].data_ptr(),
                                                self.depth_mask_bufs[slot].data_ptr(), self.depth_weight.data_ptr(),
                                                self.dinvdepth.data_ptr(), self.depth_sum.data_ptr(), st))
        self._backward(3)
        info = self.scan_info().data_ptr()
        if self.stats is not None and self._count_stats:
            s = self.stats
            _lib.check(L.h3dgs_densify_stats(self.P, self.radii.data_ptr(), self.d_means2D.data_ptr(), s.max_radii2D.data_ptr(),
                                             s.xyz_gradient_accum.data_ptr(), s.denom.data_ptr(), info, st))
        _lib.check(L.h3dgs_single_step_status(self.sums.data_ptr(), ptr(self.depth_sum), self.depth_weight.data_ptr(),
                                              1.0 / (3 * H * W), 1.0 / (H * W), self.lambda_dssim, info,
                                              ptr(self.exposure_grad64), ptr(self.exposure_grad), self.status_dev.data_ptr(), st))

    # ---- driving --------------------------------------------------------------------------
    def set_background(self, bg):
        """this step's background (train_single.py:60 draws one per step)"""
        self.bg.copy_(bg.reshape(3), non_blocking=True)

    def set_depth_weight(self, weight):
        """depth_l1_weight(iteration) for the next step; 0 switches the depth term off (its gradient is then zero)"""
        if self.dinvdepth is None:
            raise ValueError("this step was built without the depth term (depth=False)")
        self.depth_weight.fill_(float(weight))

    def _fill_slot(self, slot, src, mask=None, mono_invdepth=None, depth_mask=None):
        """upload_target(src, stream, mask, mono_invdepth, depth_mask): the NEXT step's target, its alpha mask ([1,H,W] or
        [H,W]; None = ones), and its mono inverse depth with the depth mask (None = ones).  mono_invdepth None is a view
        whose depth is unreliable (train_single.py:111): its depth mask is zero, so the term and its gradient are."""
        self.gt_bufs[slot].copy_(src, non_blocking=True)
        self._fill_maps(slot, mask, mono_invdepth, depth_mask)

    def _fill_maps(self, slot, mask, mono_invdepth, depth_mask):
        H, W = self.H, self.W
        self._set_mask(slot, mask)
        if self.dinvdepth is None:
            if mono_invdepth is not None:
                raise ValueError("this step was built without the depth term (depth=False)")
        elif mono_invdepth is None:
            self.depth_mask_bufs[slot].zero_()
        else:
            self.mono_bufs[slot].copy_(mono_invdepth.reshape(H, W), non_blocking=True)
            if depth_mask is None:
                self.depth_mask_bufs[slot].fill_(1.0)
            else:
                self.depth_mask_bufs[slot].copy_(depth_mask.reshape(H, W), non_blocking=True)

    def step(self, cam=None, gt=None, mask=None, mono_invdepth=None, depth_mask=None, exposure=None, bg=None,
             depth_weight=None, gt_ready=None):
        """cam, bg, depth_weight: optional new inputs.  gt with its mask and depth maps: copied into slot 0 (otherwise the
        slot of the last upload_target() is read).  exposure: this step's [3,4] (or larger: its top 3x4 block) exposure;
        None = identity.  gt_ready: the event upload_target() returned."""
        if gt is None and (mask is not None or mono_invdepth is not None or depth_mask is not None):
            raise ValueError("mask and depth maps travel with their target: pass gt with them, or upload them with upload_target")
        self._set_exposure(exposure)
        if bg is not None:
            self.set_background(bg)
        if depth_weight is not None:
            self.set_depth_weight(depth_weight)
        if gt is not None:
            self._fill_maps(0, mask, mono_invdepth, depth_mask)
        return super().step(cam, gt, gt_ready)

    def status(self):
        """One 64-byte read-back: loss, photometric loss, L1, SSIM, pure depth L1, D, longest tile list, overflow flag."""
        s = self.status_dev.cpu()
        return dict(loss=float(s[0]), photo=float(s[1]), l1=float(s[2]), ssim=float(s[3]), depth_l1=float(s[4]),
                    D=int(s[5]), longest_list=int(s[6]), overflow=bool(s[7] != 0))

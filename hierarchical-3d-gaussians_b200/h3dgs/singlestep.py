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
exact path with the same kernels.  Gradients are with respect to the activated Scene tensors.  One GPU only: the SSIM
window reaches across tile-row shards.

Without a state, the optimizers, densify_and_prune, reset_opacity and the big-Gaussian rescale of
train_single.py:150-186 stay the caller's.  With a SingleState, graph B ends with csrc/single_param.cu's parameter step
(the exposure's Adam, the skybox lock, the flattened relevance, OurAdam with this iteration's xyz lr, the rescale past
the scaffold, the activations the next forward reads), the frame's exposure is the state's row of the image named by a
device word, and the learning rates are device words: the whole iteration then replays without a host sync between
two densifications.  SingleState.densify_and_prune and reset_opacity (csrc/densify.cu) grow, shrink and reset the
state itself, so the loop needs the GaussianModel only for saves and checkpoints (INTEGRATION.md).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import ptr
from .coarsestep import CoarseState
from .graphstep import GraphedBase
from .pipeline import DensifyStats


def rescale_threshold(cameras_extent, scale_big_gauss=True):
    """train_single.py:182 compares a float32 tensor with the Python float cameras_extent * 0.02: in float32.  Without
    the rescale (--skip_scale_big_gauss) +inf, which no exp(scaling) exceeds"""
    return float(np.float32(float(cameras_extent) * 0.02)) if scale_big_gauss else float("inf")


class SingleState(CoarseState):
    """What train_single's optimizers hold, on the device: GaussianModel's six stored tensors with their OurAdam moments
    and step count and the group hyper-parameters (CoarseState), the exposures _exposure [n_images,3,4] with their
    torch.optim.Adam moments and step count, skybox_points, skybox_locked, scaffold_points (None = 0: the rescale
    covers every row), whether the big-Gaussian rescale runs (scale_big_gauss = not --skip_scale_big_gauss), and the
    densification statistics (stats: a pipeline.DensifyStats; state.max_radii2D is its max_radii2D).

    Device words the host fills without a sync: lrs = [xyz lr, exposure lr] (set_learning_rates, every iteration) and
    image_index (set_image: the frame's row of the exposures).  exposure_grad [3,4] is the exact path's last dL/dE.
    percent_dense (training_setup's, None until it is known) sets densify_and_prune's clone / split size threshold."""

    def __init__(self, params, skybox_points, lrs, exposure, betas=(0.9, 0.999), eps=1e-15, exp_avg=None, exp_avg_sq=None,
                 step=0, stats=None, skybox_locked=False, scaffold_points=None, scale_big_gauss=True, exposure_lr=0.0,
                 exposure_exp_avg=None, exposure_exp_avg_sq=None, exposure_step=0, exposure_betas=(0.9, 0.999),
                 exposure_eps=1e-8, percent_dense=None):
        super().__init__(params, skybox_points, lrs, betas, eps, exp_avg, exp_avg_sq, step)
        dev, N = self.dev, self.N
        if stats is None:
            stats = DensifyStats(N, dev)
        if stats.denom.shape[0] != N or stats.max_radii2D.shape[0] != N:
            raise ValueError(f"the statistics hold {stats.denom.shape[0]} rows, the state {N}")
        self.stats = stats
        self.max_radii2D = stats.max_radii2D
        self.skybox_locked = bool(skybox_locked)
        self.scaffold_points = 0 if scaffold_points is None else int(scaffold_points)
        self.scale_big_gauss = bool(scale_big_gauss)
        self.exposure = exposure.detach().float().contiguous().clone().to(dev)
        if self.exposure.dim() != 3 or tuple(self.exposure.shape[1:]) != (3, 4):
            raise ValueError(f"exposure must be [n_images, 3, 4], not {tuple(self.exposure.shape)}")
        self.n_images = self.exposure.shape[0]
        mom = lambda t: torch.zeros_like(self.exposure) if t is None else t.detach().float().contiguous().clone().to(dev)
        self.exposure_exp_avg, self.exposure_exp_avg_sq = mom(exposure_exp_avg), mom(exposure_exp_avg_sq)
        self.exposure_step = torch.full((1,), int(exposure_step), dtype=torch.int64, device=dev)
        self.exposure_betas = (float(exposure_betas[0]), float(exposure_betas[1]))
        self.exposure_eps = float(exposure_eps)
        self.lrs = torch.tensor([float(self.lr[0]), float(exposure_lr)], dtype=torch.float64, device=dev)
        self.image_index = torch.zeros(1, dtype=torch.int32, device=dev)
        self.exposure_grad = torch.zeros((3, 4), device=dev)
        self.scratch = torch.zeros(_lib.SINGLE_SCRATCH_BYTES, dtype=torch.uint8, device=dev)
        self.percent_dense = None if percent_dense is None else float(percent_dense)

    # ---- per-iteration inputs (no host sync) ----------------------------------------------
    def set_learning_rates(self, xyz_lr, exposure_lr):
        """update_learning_rate(iteration): xyz_scheduler_args(iteration) and exposure_scheduler_args(iteration)"""
        self.lrs[0].fill_(float(xyz_lr))
        self.lrs[1].fill_(float(exposure_lr))

    def set_image(self, index):
        """the frame's image: its row of the exposures (GaussianModel.exposure_mapping[image_name])"""
        index = int(index)
        if not 0 <= index < self.n_images:
            raise ValueError(f"image index {index} outside the {self.n_images} exposures")
        self.image_index.fill_(index)

    # ---- GaussianModel / optimizers interchange --------------------------------------------
    @classmethod
    def from_model(cls, gaussians, scale_big_gauss=True):
        """from a GaussianModel after training_setup (OurAdam and exposure_optimizer with their state if they have any),
        with its densification statistics; scale_big_gauss = not args.skip_scale_big_gauss"""
        params, lrs, betas, eps, m, v, step = cls._model_groups(gaussians)
        N, dev = params[0].shape[0], params[0].device
        stats = DensifyStats(N, dev)
        for name in ("max_radii2D", "xyz_gradient_accum", "denom"):
            t = getattr(gaussians, name, None)
            if t is not None and t.numel() == N:
                getattr(stats, name).copy_(t.detach().reshape(getattr(stats, name).shape))
        eo = gaussians.exposure_optimizer
        g = eo.param_groups[0]
        st = eo.state.get(gaussians._exposure, {})
        return cls(params, gaussians.skybox_points, lrs, gaussians._exposure, betas, eps, m, v, step, stats,
                   gaussians.skybox_locked, gaussians.scaffold_points, scale_big_gauss, g["lr"], st.get("exp_avg"),
                   st.get("exp_avg_sq"), int(float(st["step"])) if "step" in st else 0, tuple(g["betas"]), g["eps"],
                   getattr(gaussians, "percent_dense", None))

    def copy_to_model(self, gaussians):
        """the parameters, both optimizers' state, the exposures and the statistics (xyz_gradient_accum and denom [N,1],
        max_radii2D [N]) into a GaussianModel (before scene.save, capture(), densify_and_prune or reset_opacity)"""
        super().copy_to_model(gaussians)
        eo = gaussians.exposure_optimizer
        with torch.no_grad():
            gaussians._exposure.data.copy_(self.exposure)
            eo.state[gaussians._exposure] = dict(step=torch.tensor(float(self.exposure_step.item())),
                                                 exp_avg=self.exposure_exp_avg.clone(), exp_avg_sq=self.exposure_exp_avg_sq.clone())
            gaussians.xyz_gradient_accum = self.stats.xyz_gradient_accum.clone()
            gaussians.denom = self.stats.denom.clone()

    # ---- densify_and_prune / reset_opacity (csrc/densify.cu) -------------------------------
    def _densify_args(self):
        a = _lib.DensifyArgs()
        a.N, a.sh_coeffs, a.scaffold_points, a.skybox_points = self.N, self.sh_coeffs, self.scaffold_points, self.skybox_points
        for k in range(6):
            a.params[k], a.exp_avg[k], a.exp_avg_sq[k] = ptr(self.params[k]), ptr(self.exp_avg[k]), ptr(self.exp_avg_sq[k])
        return a

    def _launch_densify(self, args, mode):
        with torch.cuda.device(self.dev):
            _lib.check(_lib.lib().h3dgs_densify(C.byref(args), mode, torch.cuda.current_stream(self.dev).cuda_stream))

    def densify_and_prune(self, max_grad, min_opacity, extent, generator=None, normals=None):
        """GaussianModel.densify_and_prune(max_grad, min_opacity, extent) on the state -> the new row count N'.

        Rows are decided from stats.xyz_gradient_accum and stats.max_radii2D and written once, in the reference's final
        order [kept originals | clones | first split copies | second split copies]; new rows have zero moments, both
        step counts and the exposures are kept, and the statistics restart at zero with N' rows (state.stats and
        state.max_radii2D are new tensors: build the next step on them).  One host sync: the 16-byte count word, which
        sizes the new tensors.  The split copies' standard normals z [2S,3] are drawn as
        torch.empty((2S, 3)).normal_(generator=generator), the draw torch.normal(zeros, stds) makes before scaling, so
        the default generator gives the reference's samples; normals= supplies them instead (tests).  max_grad must be
        > 0 and min_opacity <= 0.15, as in train_single (0.0002 and 0.005): then no clone splits and no new row is
        pruned, which the single-pass layout relies on."""
        if self.percent_dense is None:
            raise ValueError("percent_dense is unknown: build the state with from_model after training_setup, or pass it")
        max_grad, min_opacity = float(np.float32(max_grad)), float(np.float32(min_opacity))
        if not max_grad > 0.0 or not min_opacity <= float(np.float32(0.15)):
            raise ValueError(f"densify_and_prune needs max_grad > 0 and min_opacity <= 0.15, not {max_grad}, {min_opacity}")
        if generator is not None and normals is not None:
            raise ValueError("pass either a generator or the normals, not both")
        if generator is not None and torch.device(generator.device) != self.dev:
            raise ValueError(f"the generator is on {generator.device}, the state on {self.dev}")
        N, dev = self.N, self.dev
        nbytes = int(_lib.lib().h3dgs_densify_scratch_bytes(N))
        if nbytes == 0:
            raise ValueError(f"{N} rows are too many to densify (3N must fit int32)")
        flags = torch.empty(max(N, 1), dtype=torch.uint8, device=dev)
        scratch = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
        off = (-scratch.data_ptr()) % 256
        a = self._densify_args()
        a.max_grad, a.min_opacity = max_grad, min_opacity
        a.size_threshold = float(np.float32(self.percent_dense * float(extent)))
        a.xyz_gradient_accum, a.max_radii2D = self.stats.xyz_gradient_accum.data_ptr(), self.stats.max_radii2D.data_ptr()
        a.flags, a.scratch = flags.data_ptr(), scratch.data_ptr() + off
        self._launch_densify(a, _lib.DENSIFY_COUNT)
        K, Cn, S, N2 = (int(x) for x in scratch[off:off + 16].view(torch.int32).cpu())
        if N2 < 0:
            raise RuntimeError(f"densify_and_prune would make {K + Cn + 2 * S} rows, more than int32 indexes")
        if normals is None:
            normals = torch.empty((2 * S, 3), device=dev).normal_(generator=generator)
        elif tuple(normals.shape) != (2 * S, 3) or normals.dtype != torch.float32 or normals.device != dev:
            raise ValueError(f"normals must be float32 [{2 * S}, 3] on {dev}, not {normals.dtype} {tuple(normals.shape)} "
                             f"on {normals.device}")
        normals = normals.contiguous()
        new = [torch.empty((N2,) + tuple(p.shape[1:]), device=dev) for p in self.params]
        m = [torch.empty_like(p) for p in new]
        v = [torch.empty_like(p) for p in new]
        a.out_rows, a.split_rows, a.normals = N2, S, ptr(normals)
        for k in range(6):
            a.out_params[k], a.out_exp_avg[k], a.out_exp_avg_sq[k] = ptr(new[k]), ptr(m[k]), ptr(v[k])
        self._launch_densify(a, _lib.DENSIFY_WRITE)
        self.params, self.exp_avg, self.exp_avg_sq, self.N = new, m, v, N2
        self.stats = DensifyStats(N2, dev)
        self.max_radii2D = self.stats.max_radii2D
        self.counts = dict(kept=K, cloned=Cn, split=S)
        return N2

    def reset_opacity(self):
        """GaussianModel.reset_opacity in place: opacity = inverse_sigmoid(min(sigmoid(opacity), 0.01)) on the rows past
        skybox_points, both opacity moments zero on every row; step counts and everything else unchanged.  The activated
        rows are stale afterwards: make a new scene (make_scene) or activate the old one."""
        self._launch_densify(self._densify_args(), _lib.DENSIFY_RESET_OPACITY)

    # ---- the parameter kernel --------------------------------------------------------------
    def _single_args(self, scene, cameras_extent=0.0, grads=None, exposure_grad=None, scan_info=None, exposure_row=None):
        a = _lib.SingleArgs()
        a.gauss = self._args(scene, 0.0, grads, scan_info)
        a.gauss.rescale_threshold = rescale_threshold(cameras_extent, self.scale_big_gauss)
        a.skybox_locked, a.scaffold_points, a.n_images = int(self.skybox_locked), self.scaffold_points, self.n_images
        a.lrs = self.lrs.data_ptr()
        a.exposure, a.exposure_exp_avg = self.exposure.data_ptr(), self.exposure_exp_avg.data_ptr()
        a.exposure_exp_avg_sq, a.exposure_step = self.exposure_exp_avg_sq.data_ptr(), self.exposure_step.data_ptr()
        (a.exposure_beta1, a.exposure_beta2), a.exposure_eps = self.exposure_betas, self.exposure_eps
        a.exposure_grad = ptr(self.exposure_grad if exposure_grad is None else exposure_grad)
        a.image_index, a.exposure_row = self.image_index.data_ptr(), ptr(exposure_row)
        return a

    def _launch_single(self, args, mode):
        with torch.cuda.device(self.dev):
            _lib.check(_lib.lib().h3dgs_single_param_step(C.byref(args), mode, torch.cuda.current_stream(self.dev).cuda_stream))

    def exposure_row(self, out=None):
        """the frame's exposure [3,4]: exposures[image_index], read on the device"""
        out = torch.empty((3, 4), device=self.dev) if out is None else out
        self._launch_single(self._single_args(self._null_scene(), exposure_row=out), _lib.SINGLE_EXPOSURE_ROW)
        return out

    def _null_scene(self):
        from types import SimpleNamespace
        return SimpleNamespace(means3D=None, shs=None, opacities=None, scales=None, rotations=None)

    def param_step(self, scene, grads, cameras_extent, exposure_grad=None, scan_info=None):
        """train_single.py:159-186 on a Gaussian-step iteration: the exposure's Adam with exposure_grad (default: the
        state's, which the exact path writes) at image_index, then the lock, relevance, OurAdam, the rescale and the
        activations of scene (the activated rows, refreshed) from the rasterizer's activated gradients `grads`"""
        self._launch_single(self._single_args(scene, cameras_extent, grads, exposure_grad, scan_info), _lib.SINGLE_STEP)

    def no_gaussian_step(self, scene, cameras_extent, exposure_grad=None):
        """train_single.py:159-186 on a densify or opacity-reset iteration, after densify_and_prune / reset_opacity (the
        new parameters carry no gradient, so OurAdam takes no step and does not count one): the exposure's Adam, then
        the rescale of the densified rows and their activations"""
        self._launch_single(self._single_args(scene, cameras_extent, None, exposure_grad), _lib.SINGLE_NO_GAUSSIAN_STEP)


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
    the backward's atomic sums.

    state (a SingleState; scene = state.make_scene()) with cameras_extent: graph B ends with the state's parameter step,
    the exposure is the state's row of the image step(image=) names, and stats=True means state.stats.  The instance
    holds the row count and the SH degree: build a new one on the same state at oneupSHdegree and after every
    densify_and_prune or reset_opacity (INTEGRATION.md).  An overflowed frame changes no state; re-run it through
    pipeline.single_step(state=).  capture()'s warm-up changes no state."""

    def __init__(self, scene, W, H, tanfovx, tanfovy, lambda_dssim=0.2, exposure=True, mask=False, depth=True, stats=True,
                 sh_degree=3, bin_capacity=1 << 22, sort_capacity=4096, world=1, capture=True, state=None,
                 cameras_extent=None):
        if int(world) != 1:
            raise ValueError("GraphedSingleStep runs on one GPU: the SSIM window reaches across the tile-row shards")
        if scene.hier:
            raise ValueError("GraphedSingleStep trains a flat scene (train_single.py); a hierarchy goes through GraphedPostStep")
        if state is not None:
            if not exposure:
                raise ValueError("a state trains the exposures: build the step with exposure=True")
            if cameras_extent is None:
                raise ValueError("a state's parameter step needs cameras_extent (the rescale threshold)")
            if scene.means3D.shape[0] != state.N or scene.shs.shape[1] != state.sh_coeffs:
                raise ValueError("the scene's rows do not match the state (build it with state.make_scene())")
            if not 0 <= int(sh_degree) or (int(sh_degree) + 1) ** 2 > state.sh_coeffs:
                raise ValueError(f"SH degree {sh_degree} needs more than the state's {state.sh_coeffs} coefficients")
            if stats is True:
                stats = state.stats
        self.state, self.cameras_extent = state, cameras_extent
        self._sargs = self._row_args = None
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

    def _update(self):
        """whether part B ends with the state's parameter step: with a state, outside capture()'s warm-up"""
        return self.state is not None and self._count_stats

    # ---- the two halves of the step (eager or under capture) ------------------------------
    def _part_a(self):
        """capacity-mode forward of all N rows, with the inverse depth"""
        self._forward(self.image, self.invdepth)

    def _part_b(self, slot=0):
        """The objective against slot `slot`, its gradients, the backward, the statistics, the status words."""
        L, st, H, W = self.L, self._stream(), self.H, self.W
        if self.state is not None:
            if self._row_args is None:
                self._row_args = self.state._single_args(self.state._null_scene(), exposure_row=self.exposure)
            _lib.check(L.h3dgs_single_param_step(C.byref(self._row_args), _lib.SINGLE_EXPOSURE_ROW, st))
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
        if self._update():
            if self._sargs is None:
                self._sargs = self.state._single_args(self.scene, self.cameras_extent, self.grads, self.exposure_grad,
                                                      self.scan_info())
            _lib.check(L.h3dgs_single_param_step(C.byref(self._sargs), _lib.SINGLE_STEP, st))

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
             depth_weight=None, gt_ready=None, image=None):
        """cam, bg, depth_weight: optional new inputs.  gt with its mask and depth maps: copied into slot 0 (otherwise the
        slot of the last upload_target() is read).  exposure: this step's [3,4] (or larger: its top 3x4 block) exposure;
        None = identity.  With a state, image (or state.set_image) names the frame's exposure row instead, and the
        learning rates are state.set_learning_rates'.  gt_ready: the event upload_target() returned."""
        if gt is None and (mask is not None or mono_invdepth is not None or depth_mask is not None):
            raise ValueError("mask and depth maps travel with their target: pass gt with them, or upload them with upload_target")
        if self.state is None:
            if image is not None:
                raise ValueError("image names a row of a state's exposures: this step has no state")
            self._set_exposure(exposure)
        elif exposure is not None:
            raise ValueError("with a state the exposure is the state's row of the frame's image: pass image=")
        elif image is not None:
            self.state.set_image(image)
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

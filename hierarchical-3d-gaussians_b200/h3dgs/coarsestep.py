"""Sync-free iteration of train_coarse (train_coarse.py:86-145), parameter update included, replayed from CUDA graphs.

The loop body is, per iteration:

    image = render_coarse(... sh_degree = active degree, bg = this iteration's random background)   (no exposure, no clamp)
    a     = image * alpha_mask                                                      train_coarse.py:113-116
    loss  = (1-l) mean|a - gt| + l (1 - SSIM(a, gt));  loss.backward()
    max_radii2D[vis] = max(max_radii2D[vis], radii)                                 :125
    _scaling.grad[:skybox_points] = 0;  OurAdam.step((_opacity.grad != 0).nonzero())     :135-138 (xyz lr 0)
    big-Gaussian rescale of the rows past the skybox                                :141-145

The model never changes size (no densification) and has one optimizer, so the whole iteration lives on the device:
graph A = the capacity-mode forward of all N rows; graph B = csrc/loss.cu's coarse-loss pair, the rasterizer backward,
max_radii2D (h3dgs_densify_stats without the other two statistics), csrc/coarse_param.cu's parameter step (activation
backward, skybox lock, relevance, Adam, rescale, the activations the next forward reads) and one status thread.
Camera, background and the target with its mask change between replays; nothing returns to the host.

CoarseState holds GaussianModel's six stored tensors, their OurAdam moments, the device step count, skybox_points,
max_radii2D and the group hyper-parameters; it is built from and copied back to a GaussianModel and its optimizer, so
that scene.save and checkpoints work as in the reference.  The active SH degree is a launch constant: at the switch
(iteration 1000, GaussianModel(1)) build a new GraphedCoarseStep on the same state and scene.

A frame that does not fit the capacities is flagged and changes nothing (no parameter, moment, step count,
max_radii2D or activated row); the caller re-runs it through pipeline.coarse_step, the exact path with the same
kernels.  One GPU only: the SSIM window reaches across the tile-row shards of the sharded forms.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import ptr
from .graphstep import GraphedBase

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")        # training_setup's group order
_MODEL_ATTRS = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")


def rescale_threshold(cameras_extent):
    """train_coarse.py:142 compares a float32 tensor with the Python float cameras_extent * 0.1: in float32"""
    return float(np.float32(float(cameras_extent) * 0.1))


class CoarseState:
    """GaussianModel's stored tensors (xyz [N,3], features_dc [N,1,3], features_rest [N,K,3], opacity [N,1], scaling
    [N,3], rotation [N,4]), their exp_avg / exp_avg_sq, the step count (a device int64, OurAdam's state["step"] of all
    six), skybox_points, max_radii2D [N] and per group lr / betas / eps (training_setup's groups; train_coarse sets the
    xyz group's lr to 0, train_coarse.py:55-57).  The device tensors are updated in place by the step."""

    def __init__(self, params, skybox_points, lrs, betas=(0.9, 0.999), eps=1e-15, exp_avg=None, exp_avg_sq=None, step=0,
                 max_radii2D=None):
        if len(params) != 6:
            raise ValueError("params: the six stored tensors in training_setup's order " + str(GROUPS))
        self.params = [p.detach().float().contiguous().clone() for p in params]
        dev = self.dev = self.params[0].device
        N = self.N = self.params[0].shape[0]
        shapes = [(N, 3), (N, 1, 3), None, (N, 1), (N, 3), (N, 4)]
        for p, s, g in zip(self.params, shapes, GROUPS):
            if (s is not None and tuple(p.shape) != s) or p.shape[0] != N or p.device != dev:
                raise ValueError(f"{g}: shape {tuple(p.shape)} on {p.device}")
        if self.params[2].dim() != 3 or self.params[2].shape[2] != 3:
            raise ValueError("features_rest must be [N, K, 3]")
        self.sh_coeffs = 1 + self.params[2].shape[1]
        self.skybox_points = int(skybox_points)
        self.exp_avg = [torch.zeros_like(p) for p in self.params] if exp_avg is None else [m.detach().float().contiguous().clone() for m in exp_avg]
        self.exp_avg_sq = [torch.zeros_like(p) for p in self.params] if exp_avg_sq is None else [v.detach().float().contiguous().clone() for v in exp_avg_sq]
        for m, v, p in zip(self.exp_avg, self.exp_avg_sq, self.params):
            if m.shape != p.shape or v.shape != p.shape:
                raise ValueError("moments must have their parameter's shape")
        self.step = torch.full((1,), int(step), dtype=torch.int64, device=dev)
        self.max_radii2D = torch.zeros(N, device=dev) if max_radii2D is None else max_radii2D.detach().float().contiguous().clone().to(dev)
        self.lr = [float(x) for x in lrs]
        bs = [tuple(betas)] * 6 if np.ndim(betas[0]) == 0 else [tuple(b) for b in betas]
        self.betas = [(float(a), float(b)) for a, b in bs]
        self.eps = [float(eps)] * 6 if np.ndim(eps) == 0 else [float(e) for e in eps]
        self.scratch = torch.zeros(_lib.COARSE_SCRATCH_BYTES, dtype=torch.uint8, device=dev)

    # ---- GaussianModel / OurAdam interchange ----------------------------------------------
    @staticmethod
    def _model_groups(gaussians):
        """-> (params, lrs, betas, eps, exp_avg or None, exp_avg_sq or None, step) of a GaussianModel and its OurAdam"""
        params = [getattr(gaussians, a) for a in _MODEL_ATTRS]
        opt = gaussians.optimizer
        groups = {g["name"]: g for g in opt.param_groups}
        gs = [groups[n] for n in GROUPS]
        st = [opt.state.get(g["params"][0], {}) for g in gs]
        have = all(len(s) for s in st)
        steps = {int(float(s["step"])) for s in st} if have else {0}
        if len(steps) != 1:
            raise ValueError(f"the six groups have taken different step counts {sorted(steps)}")
        return (params, [g["lr"] for g in gs], [tuple(g["betas"]) for g in gs], [g["eps"] for g in gs],
                [s["exp_avg"] for s in st] if have else None, [s["exp_avg_sq"] for s in st] if have else None, steps.pop())

    @classmethod
    def from_model(cls, gaussians):
        """from a GaussianModel after training_setup (and the xyz lr set to 0), with its OurAdam's state if it has any"""
        params, lrs, betas, eps, m, v, step = cls._model_groups(gaussians)
        return cls(params, gaussians.skybox_points, lrs, betas, eps, m, v, step,
                   getattr(gaussians, "max_radii2D", None) if getattr(gaussians, "max_radii2D", None) is not None and
                   gaussians.max_radii2D.numel() == params[0].shape[0] else None)

    def optimizer_state(self):
        """-> [{step, exp_avg, exp_avg_sq}] per group, shaped as OurAdam keeps its state (step a CPU float tensor)"""
        step = float(self.step.item())
        return [dict(step=torch.tensor(step), exp_avg=m.clone(), exp_avg_sq=v.clone()) for m, v in zip(self.exp_avg, self.exp_avg_sq)]

    def copy_to_model(self, gaussians):
        """the parameters, max_radii2D and the optimizer state into a GaussianModel (before scene.save or capture()).
        When the row count differs from the model's (the state was densified on the device), each group gets a new
        Parameter, bound in the optimizer group, its state and the model attribute, as densify_and_prune rebinds them"""
        opt = gaussians.optimizer
        groups = {g["name"]: g for g in opt.param_groups}
        with torch.no_grad():
            for a, n, p, s in zip(_MODEL_ATTRS, GROUPS, self.params, self.optimizer_state()):
                t = getattr(gaussians, a)
                if t.shape == p.shape:
                    t.data.copy_(p)
                else:
                    opt.state.pop(groups[n]["params"][0], None)
                    t = torch.nn.Parameter(p.to(t.device, copy=True))
                    groups[n]["params"][0] = t
                    setattr(gaussians, a, t)
                opt.state[groups[n]["params"][0]] = {k: (v.to(t.device) if k != "step" else v) for k, v in s.items()}
            gaussians.max_radii2D = self.max_radii2D.clone()

    # ---- the parameter kernel --------------------------------------------------------------
    def _args(self, scene, cameras_extent, grads=None, scan_info=None):
        a = _lib.CoarseArgs()
        a.N, a.sh_coeffs, a.skybox_points = self.N, self.sh_coeffs, self.skybox_points
        a.rescale_threshold = rescale_threshold(cameras_extent)
        for k in range(6):
            a.params[k] = ptr(self.params[k])
            a.exp_avg[k], a.exp_avg_sq[k] = ptr(self.exp_avg[k]), ptr(self.exp_avg_sq[k])
            a.lr[k], (a.beta1[k], a.beta2[k]), a.eps[k] = self.lr[k], self.betas[k], self.eps[k]
        a.step, a.scratch = self.step.data_ptr(), self.scratch.data_ptr()
        if grads is not None:
            a.grad_means3D, a.grad_shs, a.grad_opacities = ptr(grads["means3D"]), ptr(grads["shs"]), ptr(grads["opacities"])
            a.grad_scales, a.grad_rotations = ptr(grads["scales"]), ptr(grads["rotations"])
        a.means3D, a.shs, a.opacities = ptr(scene.means3D), ptr(scene.shs), ptr(scene.opacities)
        a.scales, a.rotations = ptr(scene.scales), ptr(scene.rotations)
        a.scan_info = ptr(scan_info)
        return a

    def _launch(self, args, mode):
        with torch.cuda.device(self.dev):
            _lib.check(_lib.lib().h3dgs_coarse_param_step(C.byref(args), mode, torch.cuda.current_stream(self.dev).cuda_stream))

    def make_scene(self, requires_grad=True):
        """a flat pipeline.Scene of the activated rows (means3D, shs [N,K+1,3], opacities [N,1], scales, rotations),
        filled from the stored tensors by the kernel's activation mode"""
        from .pipeline import Scene
        N, dev = self.N, self.dev
        z = lambda *s: torch.zeros(s, device=dev)
        scene = Scene(dict(means3D=z(N, 3), shs=z(N, self.sh_coeffs, 3), opacities=z(N, 1), scales=z(N, 3),
                           rotations=z(N, 4), skybox_points=self.skybox_points), device=dev, requires_grad=requires_grad)
        self.activate(scene)
        return scene

    def activate(self, scene):
        """scene's activated rows from the stored tensors (GaussianModel's get_xyz / get_features / get_opacity /
        get_scaling / get_rotation)"""
        self._launch(self._args(scene, 0.0), _lib.COARSE_ACTIVATE)

    def param_step(self, scene, grads, cameras_extent, scan_info=None):
        """train_coarse.py:135-145 from the activated gradients `grads` (dict of the rasterizer's full-size
        gradients: means3D, shs, opacities, scales, rotations), and scene's activated rows refreshed"""
        self._launch(self._args(scene, cameras_extent, grads, scan_info), _lib.COARSE_STEP)

    def update_max_radii(self, radii, scan_info=None):
        """train_coarse.py:125: max_radii2D of the rows with radii > 0 (h3dgs_densify_stats, max_radii2D only)"""
        with torch.cuda.device(self.dev):
            _lib.check(_lib.lib().h3dgs_densify_stats(self.N, radii.data_ptr(), None, self.max_radii2D.data_ptr(), None,
                                                     None, ptr(scan_info), torch.cuda.current_stream(self.dev).cuda_stream))


class GraphedCoarseStep(GraphedBase):
    """state: a CoarseState; scene: its make_scene() (the activated rows the forward reads and the step rewrites).
    Fixed per instance: W, H, tanfovx, tanfovy, lambda_dssim, cameras_extent (the rescale threshold), the active SH
    degree, and whether an alpha mask is applied.  Changing between replays: set_camera, set_background and the target
    with its mask (upload_target(src, stream, mask) into one of two slots, or step(gt=, mask=)).

    The arithmetic is the one of pipeline.coarse_step: image, loss and radii are bit-identical whenever the frame fits,
    dL/dimage too, the Gaussian gradients equal up to the order of the backward's atomic sums, and the parameter step
    is the same kernel.  capture()'s eager warm-up step changes no state."""

    def __init__(self, state, scene, W, H, tanfovx, tanfovy, cameras_extent, lambda_dssim=0.2, mask=False, sh_degree=0,
                 bin_capacity=1 << 22, sort_capacity=4096, capture=True):
        if scene.hier:
            raise ValueError("GraphedCoarseStep trains a flat scene (train_coarse.py)")
        if scene.means3D.shape[0] != state.N or scene.shs.shape[1] != state.sh_coeffs:
            raise ValueError("the scene's rows do not match the state (build it with state.make_scene())")
        if not 0 <= int(sh_degree) or (int(sh_degree) + 1) ** 2 > state.sh_coeffs:
            raise ValueError(f"SH degree {sh_degree} needs more than the state's {state.sh_coeffs} coefficients")
        super().__init__(scene, W, H, sh_degree, None, bin_capacity, sort_capacity)
        self.state, self.cameras_extent = state, float(cameras_extent)
        self.bg = self._zeros(3)
        self._init_post_loss(lambda_dssim, False, mask)
        self.image = self._zeros(3, self.H, self.W)
        self.status_dev = torch.zeros(6, dtype=torch.float64, device=self.dev)
        self._init_grads(self.N)
        self.args = self._raster_args(tanfovx, tanfovy)
        self._update = True
        self._cargs = None
        if capture:
            self.capture()

    def _warm_up(self):
        """capture()'s eager step runs on whatever the buffers hold: it must not touch the state"""
        self._update = False
        try:
            super()._warm_up()
        finally:
            self._update = True

    def _part_a(self):
        """capacity-mode forward of all N rows"""
        self._forward(self.image)

    def _part_b(self, slot=0):
        """The objective against slot `slot`, the backward, max_radii2D, the parameter step, the status words."""
        L, st, H, W = self.L, self._stream(), self.H, self.W
        img, gt, m = self.image.data_ptr(), self.gt_bufs[slot].data_ptr(), ptr(self.mask_bufs[slot])
        _lib.check(L.h3dgs_coarse_loss_forward(H, W, img, gt, m, self.sums.data_ptr(), self.maps.data_ptr(), st))
        _lib.check(L.h3dgs_coarse_loss_backward(H, W, img, gt, m, self.maps.data_ptr(), self.coeffs.data_ptr(),
                                                self.dcolor.data_ptr(), st))
        self._backward(3)
        info = self.scan_info()
        if self._update:
            self.state.update_max_radii(self.radii, info)
            if self._cargs is None:
                self._cargs = self.state._args(self.scene, self.cameras_extent, self.grads, info)
            _lib.check(L.h3dgs_coarse_param_step(C.byref(self._cargs), _lib.COARSE_STEP, st))
        _lib.check(L.h3dgs_coarse_step_status(self.sums.data_ptr(), 1.0 / (3 * H * W), self.lambda_dssim, info.data_ptr(),
                                              self.status_dev.data_ptr(), st))

    def set_background(self, bg):
        """this iteration's background (train_coarse.py:61 draws one per iteration)"""
        self.bg.copy_(bg.reshape(3), non_blocking=True)

    def step(self, cam=None, gt=None, mask=None, bg=None, gt_ready=None):
        """cam, bg, gt (+ its mask; None = ones): optional new inputs, copied into the static buffers (the target into
        slot 0).  gt_ready: the event upload_target() returned."""
        if mask is not None and gt is None:
            raise ValueError("a mask travels with its target: pass gt with it, or upload both with upload_target")
        if bg is not None:
            self.set_background(bg)
        if gt is not None:
            self._set_mask(0, mask)
        return super().step(cam, gt, gt_ready)

    def status(self):
        """One 48-byte read-back: loss, L1, SSIM, D, longest tile list, overflow flag."""
        s = self.status_dev.cpu()
        return dict(loss=float(s[0]), l1=float(s[1]), ssim=float(s[2]), D=int(s[3]), longest_list=int(s[4]),
                    overflow=bool(s[5] != 0))

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
respect to the activated Scene tensors.  One GPU only: the SSIM window reaches across the tile-row shards of the sharded
forms.

Without a state, the optimizer and the skybox / anchor gradient zeroing of train_post.py:167-181 stay the caller's.  With
a PostState, graph B ends with csrc/post_param.cu's parameter step: the activations' backward of a create_from_hier
model (abs, exp, F.normalize), the locks, torch.optim.Adam's dense step with the xyz lr of a device word, and the
activated rows the next forward reads.  train_post neither densifies nor changes the SH degree (the maximum from the
start), so the graphs are captured once for the whole run.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import ptr
from .coarsestep import CoarseState
from .graphstep import GraphedStep


class PostState(CoarseState):
    """What train_post's optimizer holds, on the device: GaussianModel's six stored tensors (create_from_hier's: 16 SH
    coefficients, opacity through abs), their torch.optim.Adam moments and step count and the group hyper-parameters
    (CoarseState), the hierarchy's nodes and boxes, skybox_points (the LAST rows), skybox_locked and the anchors
    (gaussians.anchors: row indices, duplicates allowed, negative ones counted from the end as torch's indexing does).

    The rows whose six gradients train_post.py:167-181 zeroes are turned into one uint8 mask `locked` here, once: the
    anchors, and the skybox tail when skybox_locked.  The xyz lr is a device double (set_learning_rate, every
    iteration); the other five lrs are the groups' constants."""

    def __init__(self, params, skybox_points, lrs, nodes, boxes, betas=(0.9, 0.999), eps=1e-15, exp_avg=None,
                 exp_avg_sq=None, step=0, skybox_locked=True, anchors=None):
        super().__init__(params, skybox_points, lrs, betas, eps, exp_avg, exp_avg_sq, step)
        dev, N, S = self.dev, self.N, self.skybox_points
        if not 0 <= S <= N:
            raise ValueError(f"skybox_points {S} outside [0, {N}]")
        self.nodes, self.boxes = nodes.to(dev), boxes.to(dev)
        self.skybox_locked = bool(skybox_locked)
        a = torch.zeros(0, dtype=torch.int64) if anchors is None else torch.as_tensor(anchors).detach().reshape(-1).long().cpu()
        if a.numel() and (int(a.min()) < -N or int(a.max()) >= N):
            raise ValueError(f"an anchor lies outside the {N} rows: [{int(a.min())}, {int(a.max())}]")
        self.anchors = a
        mask = torch.zeros(N, dtype=torch.uint8)
        mask[a] = 1
        if S and self.skybox_locked:
            mask[N - S:] = 1
        self.locked = mask.to(dev) if bool(mask.any()) else None
        self.lrs = torch.tensor([float(self.lr[0])], dtype=torch.float64, device=dev)
        self.scratch = torch.zeros(_lib.POST_SCRATCH_BYTES, dtype=torch.uint8, device=dev)

    def set_learning_rate(self, xyz_lr):
        """update_learning_rate(iteration): xyz_scheduler_args(iteration), read by the next step on the device"""
        self.lrs.fill_(float(xyz_lr))

    # ---- GaussianModel / optimizer interchange ---------------------------------------------
    @classmethod
    def from_model(cls, gaussians):
        """from a GaussianModel made by create_from_hier after training_setup(our_adam=False), with its torch.optim.Adam
        state if it has any.  Refused: OurAdam (training_setup's default), and an Adam whose options leave the default
        non-capturable foreach step (amsgrad, weight_decay, maximize, capturable, fused)"""
        opt = gaussians.optimizer
        if not isinstance(opt, torch.optim.Adam):
            raise ValueError(f"train_post's optimizer is torch.optim.Adam (training_setup(our_adam=False)), not {type(opt).__name__}")
        for g in opt.param_groups:
            if g.get("amsgrad") or g.get("weight_decay") or g.get("maximize") or g.get("capturable") or g.get("fused"):
                raise ValueError(f"group {g.get('name')}: only Adam's default step (no amsgrad, weight_decay, maximize, "
                                 "capturable or fused) is reproduced")
        params, lrs, betas, eps, m, v, step = cls._model_groups(gaussians)
        return cls(params, gaussians.skybox_points, lrs, gaussians.nodes, gaussians.boxes, betas, eps, m, v, step,
                   getattr(gaussians, "skybox_locked", True), getattr(gaussians, "anchors", None))

    # copy_to_model (CoarseState's): the parameters and the optimizer state into the GaussianModel, before scene.save
    # (save_hier) or capture()

    # ---- the parameter kernel --------------------------------------------------------------
    def _post_args(self, scene, grads=None, scan_info=None, count=None, extra_rows=0, row_capacity=0):
        a = _lib.PostArgs()
        a.gauss = self._args(scene, 0.0, grads, scan_info)
        a.lrs, a.locked, a.count = self.lrs.data_ptr(), ptr(self.locked), ptr(count)
        a.extra_rows, a.row_capacity = int(extra_rows), int(row_capacity)
        return a

    def _launch_post(self, args, mode):
        with torch.cuda.device(self.dev):
            _lib.check(_lib.lib().h3dgs_post_param_step(C.byref(args), mode, torch.cuda.current_stream(self.dev).cuda_stream))

    def make_scene(self, requires_grad=True):
        """a hierarchy pipeline.Scene of the activated rows (means3D, shs [N,16,3], opacities [N,1], scales, rotations)
        with the model's nodes and boxes, filled from the stored tensors by the kernel's activation mode"""
        from .pipeline import Scene
        N, dev = self.N, self.dev
        z = lambda *s: torch.zeros(s, device=dev)
        scene = Scene(dict(means3D=z(N, 3), shs=z(N, self.sh_coeffs, 3), opacities=z(N, 1), scales=z(N, 3),
                           rotations=z(N, 4), skybox_points=self.skybox_points, nodes=self.nodes, boxes=self.boxes),
                      device=dev, requires_grad=requires_grad)
        self.activate(scene)
        return scene

    def activate(self, scene):
        """scene's activated rows from the stored tensors: get_xyz, get_features, abs(_opacity), exp(_scaling),
        F.normalize(_rotation)"""
        self._launch_post(self._post_args(scene), _lib.POST_ACTIVATE)

    def param_step(self, scene, grads=None, scan_info=None, count=None, extra_rows=0, row_capacity=0):
        """train_post.py:167-192 from the activated gradients `grads` (dict of the rasterizer's full-size gradients:
        means3D, shs, opacities, scales, rotations; None = the .grad of scene's tensors, as pipeline.post_step(update=False)
        leaves them): the activations' backward, the locks, the dense Adam step, and scene's activated rows refreshed.
        scan_info / count with extra_rows and row_capacity: a capacity-mode frame's flags (an overflowed frame changes
        nothing); None = the exact path"""
        if grads is None:
            grads = {k: getattr(scene, k).grad.contiguous() for k in ("means3D", "shs", "opacities", "scales", "rotations")}
        self._launch_post(self._post_args(scene, grads, scan_info, count, extra_rows, row_capacity), _lib.POST_STEP)


class GraphedPostStep(GraphedStep):
    """scene: pipeline.Scene with a hierarchy.  Fixed per instance: W, H, tanfovx, tanfovy, lambda_dssim, and whether an
    exposure and an alpha mask are applied.  Changing between replays: set_camera, set_threshold, the target and its mask
    (upload_target(src, stream, mask) into one of two slots, or step(gt=, mask=)), and the exposure (step(exposure=)).

    The arithmetic is the one of pipeline.post_step: image and radii are bit-identical whenever the frame fits, dL/dimage
    too, and the Gaussian gradients equal up to the order of the backward's atomic sums.

    state (a PostState; scene = state.make_scene()): graph B ends with the state's parameter step, whose xyz lr is
    state.set_learning_rate's.  An overflowed frame (binning or rows) changes no state; re-run it through
    pipeline.post_step(state=).  capture()'s warm-up changes no state.  cull: the view-culled cut (GraphedLodCut)."""

    def __init__(self, scene, W, H, tanfovx, tanfovy, bg, threshold, lambda_dssim=0.2, exposure=False, mask=False,
                 sh_degree=3, row_capacity=None, bin_capacity=1 << 22, sort_capacity=4096, world=1, capture=True,
                 state=None, cull=False):
        if int(world) != 1:
            raise ValueError("GraphedPostStep runs on one GPU: the SSIM window reaches across the tile-row shards")
        if state is not None:
            if scene.means3D.shape[0] != state.N or scene.shs.shape[1] != state.sh_coeffs:
                raise ValueError("the scene's rows do not match the state (build it with state.make_scene())")
            if not 0 <= int(sh_degree) or (int(sh_degree) + 1) ** 2 > state.sh_coeffs:
                raise ValueError(f"SH degree {sh_degree} needs more than the state's {state.sh_coeffs} coefficients")
        self.state, self._update, self._pargs = state, state is not None, None
        super().__init__(scene, W, H, tanfovx, tanfovy, bg, threshold, sh_degree=sh_degree, row_capacity=row_capacity,
                         bin_capacity=bin_capacity, sort_capacity=sort_capacity, capture=False, cull=cull)
        self._init_post_loss(lambda_dssim, exposure, mask)
        self.status_dev = torch.zeros(8, dtype=torch.float64, device=self.dev)
        if capture:
            self.capture()

    def _warm_up(self):
        """capture()'s eager step runs on whatever the buffers hold: it must not touch the state"""
        update, self._update = self._update, False
        try:
            super()._warm_up()
        finally:
            self._update = update

    def _part_b(self, slot=0):
        """The objective against target slot `slot` and its mask, its gradient, the backward, the status words, and
        with a state its parameter step."""
        self._post_loss(slot)
        self._backward(3)
        _lib.check(self.L.h3dgs_post_step_status(self.sums.data_ptr(), 1.0 / self.image.numel(), self.lambda_dssim,
                                                 self.count.data_ptr(), self.S, self.P, self.scan_info().data_ptr(),
                                                 self.status_dev.data_ptr(), self._stream()))
        if self._update:
            if self._pargs is None:
                self._pargs = self.state._post_args(self.scene, self.grads, self.scan_info(), self.count, self.S, self.P)
            _lib.check(self.L.h3dgs_post_param_step(C.byref(self._pargs), _lib.POST_STEP, self._stream()))

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

"""One training-style step of the hot path on synthetic data, through the same public
API the reference's scripts use:

  expand_to_size -> get_interpolation_weights        (train_post.py:91-113)
  gather cut rows + lerp with parents (PyTorch ops)  (gaussian_renderer/__init__.py:199-234)
  GaussianRasterizer(settings)(...)                  (gaussian_renderer/__init__.py:247-277)
  L1 loss -> backward                                (train_post.py:134-142, lambda_dssim term omitted:
                                                      SSIM is outside the path, SURVEY.md 8d)

Used by bench.py and the GPU tests; nothing here touches oracle/.
"""

import torch

from . import _lib
from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
from gaussian_hierarchy._C import expand_to_size, get_interpolation_weights


class Scene:
    """Device-resident Gaussians (already-activated values are the leaves, i.e. what
    GaussianModel.get_* would return) plus, for hierarchy scenes, nodes/boxes and the
    caller-preallocated LOD scratch of train_post.py:59-63."""

    def __init__(self, arrays, device="cuda", requires_grad=True):
        t = lambda a: a.to(device) if torch.is_tensor(a) else torch.tensor(a, device=device)
        self.device = device
        self.means3D = t(arrays["means3D"]).requires_grad_(requires_grad)
        self.scales = t(arrays["scales"]).requires_grad_(requires_grad)
        self.rotations = t(arrays["rotations"]).requires_grad_(requires_grad)
        self.opacities = t(arrays["opacities"]).requires_grad_(requires_grad)
        self.shs = t(arrays["shs"]).requires_grad_(requires_grad)
        self.hier = "nodes" in arrays
        N = self.means3D.shape[0]
        # skybox rows sit after the hierarchy rows and are rendered on every step
        # (gaussian_renderer/__init__.py:220-234); the LOD scratch covers them (train_post.py:59-63)
        self.skybox_points = int(arrays.get("skybox_points", 0))
        self.skybox_inds = torch.arange(N - self.skybox_points, N, dtype=torch.int32, device=device)
        if self.hier:
            self.nodes = t(arrays["nodes"])
            self.boxes = t(arrays["boxes"])
            z = lambda dt: torch.zeros(N, dtype=dt, device=device)
            self.render_indices, self.parent_indices, self.nodes_for_render = z(torch.int32), z(torch.int32), z(torch.int32)
            self.interpolation_weights, self.num_siblings = z(torch.float32), z(torch.int32)
        self.empty_i = torch.empty(0, dtype=torch.int32, device=device)
        self.empty_f = torch.empty(0, dtype=torch.float32, device=device)

    def params(self):
        return [self.means3D, self.scales, self.rotations, self.opacities, self.shs]

    def zero_grad(self):
        for p in self.params():
            p.grad = None


class DeviceCamera:
    def __init__(self, cam, device="cuda"):
        self.W, self.H = cam.W, cam.H
        self.tanfovx, self.tanfovy = cam.tanfovx, cam.tanfovy
        self.viewmatrix = torch.tensor(cam.world_view_transform, device=device)
        self.projmatrix = torch.tensor(cam.full_proj_transform, device=device)
        self.campos = torch.tensor(cam.camera_center, device=device)
        self.campos_cpu = torch.tensor(cam.camera_center)


def lod_cut(scene, cam, threshold):
    """-> number of cut Gaussians; fills scene.render_indices/parent_indices/interpolation_weights/num_siblings."""
    zeros3 = torch.zeros(3)
    n = expand_to_size(scene.nodes, scene.boxes, threshold, cam.campos, zeros3, scene.render_indices,
                       scene.parent_indices, scene.nodes_for_render)
    get_interpolation_weights(scene.nodes_for_render[:n], threshold, scene.nodes, scene.boxes, cam.campos_cpu, zeros3,
                              scene.interpolation_weights, scene.num_siblings)
    return n


def interpolate_cut(scene, n):
    """The gather + parent lerp of render_post (interp_python=True), in PyTorch ops so
    autograd scatters the gradients back to the full-size leaves; skybox rows are appended
    un-interpolated (:220-229)."""
    idx = scene.render_indices[:n].long()
    par = scene.parent_indices[:n].long()
    par = torch.where(par < 0, idx, par)             # the root has no parent: t == 1 there
    t = scene.interpolation_weights[:n].unsqueeze(1)
    u = 1.0 - t
    means = t * scene.means3D[idx] + u * scene.means3D[par]
    scales = t * scene.scales[idx] + u * scene.scales[par]
    shs = t.unsqueeze(2) * scene.shs[idx] + u.unsqueeze(2) * scene.shs[par]
    q_c = scene.rotations[idx]
    q_p = scene.rotations[par]
    sign = torch.where((q_c * q_p).sum(1, keepdim=True) < 0, -1.0, 1.0)     # quaternion sign alignment
    rots = t * q_c + u * (q_p * sign)
    opac = t * scene.opacities[idx] + u * scene.opacities[par]
    if scene.skybox_points:
        sky = scene.skybox_inds.long()
        means, scales, rots = torch.cat((means, scene.means3D[sky])), torch.cat((scales, scene.scales[sky])), torch.cat((rots, scene.rotations[sky]))
        opac, shs = torch.cat((opac, scene.opacities[sky])), torch.cat((shs, scene.shs[sky]))
    return means.contiguous(), scales.contiguous(), rots.contiguous(), opac.contiguous(), shs.contiguous()


def make_settings(scene, cam, bg, sh_degree, ts=None, kids=None, do_depth=False, debug=False, ridx=None, pidx=None):
    return GaussianRasterizationSettings(
        image_height=cam.H, image_width=cam.W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=bg, scale_modifier=1.0,
        viewmatrix=cam.viewmatrix, projmatrix=cam.projmatrix, sh_degree=sh_degree, campos=cam.campos,
        prefiltered=False, debug=debug, render_indices=ridx if ridx is not None else scene.empty_i,
        parent_indices=pidx if pidx is not None else scene.empty_i,
        interpolation_weights=ts if ts is not None else scene.empty_f,
        num_node_kids=kids if kids is not None else scene.empty_i, do_depth=do_depth)


def _skybox_weights(scene, n):
    """t = 1, kids = 1 for the skybox rows that follow the cut (gaussian_renderer/__init__.py:232-234)."""
    S = scene.skybox_points
    if S:
        scene.interpolation_weights[n:n + S] = 1.0
        scene.num_siblings[n:n + S] = 1


def render_flat(scene, cam, bg, sh_degree=3, do_depth=False, means2D=None):
    """`render()` of the reference minus exposure/clamp (flat chunk training, config #2) -> (img, radii), and with
    do_depth=True (as render() sets it, :57) -> (img, radii, invdepth [1,H,W]).  means2D: the caller's [N,3] sink for the
    screen-space gradient (render()'s viewspace_points); None makes one."""
    rs = make_settings(scene, cam, bg, sh_degree, do_depth=do_depth)
    if means2D is None:
        means2D = torch.zeros_like(scene.means3D, requires_grad=scene.means3D.requires_grad)
    img, radii, invdepth = GaussianRasterizer(rs)(means3D=scene.means3D, means2D=means2D, shs=scene.shs, colors_precomp=None,
                                                  opacities=scene.opacities, scales=scene.scales, rotations=scene.rotations,
                                                  cov3D_precomp=None)
    return (img, radii, invdepth) if do_depth else (img, radii)


def render_hier(scene, cam, bg, threshold, sh_degree=3):
    """`render_post()` of the reference (hierarchy post-optimisation, config #3)."""
    n = lod_cut(scene, cam, threshold)
    means, scales, rots, opac, shs = interpolate_cut(scene, n)
    ts = scene.interpolation_weights
    if scene.skybox_points:
        # a copy, as in render_post (:232): autograd holds a view of the cut's weights for the lerp backward
        ts = ts.clone()
        ts[n:n + scene.skybox_points] = 1.0
        scene.num_siblings[n:n + scene.skybox_points] = 1
    rs = make_settings(scene, cam, bg, sh_degree, ts=ts, kids=scene.num_siblings)
    means2D = torch.zeros_like(means, requires_grad=means.requires_grad)
    img, radii, _ = GaussianRasterizer(rs)(means3D=means, means2D=means2D, shs=shs, colors_precomp=None,
                                           opacities=opac, scales=scales, rotations=rots, cov3D_precomp=None)
    return img, radii, n


def cull_mask(scene, cam, out=None):
    """The view cull's row mask (h3dgs_lod_cull_mask) -> uint8 [rows] on the device: 1 for every hierarchy row the
    rasterizer could draw from `cam` at some lerp weight, whatever the threshold; skybox rows are not written."""
    L = _lib.lib()
    if out is None:
        out = torch.zeros(scene.means3D.shape[0], dtype=torch.uint8, device=scene.means3D.device)
    _lib.check(L.h3dgs_lod_cull_mask(scene.nodes.shape[0], scene.nodes.data_ptr(), scene.means3D.data_ptr(),
                                     scene.scales.data_ptr(), scene.rotations.data_ptr(), 1.0, cam.viewmatrix.data_ptr(),
                                     cam.projmatrix.data_ptr(), cam.W, cam.H, float(cam.tanfovx), float(cam.tanfovy),
                                     out.data_ptr(), torch.cuda.current_stream(out.device).cuda_stream))
    return out


def _culled_cut(scene, cam, threshold):
    """the cut under the view cull's mask (h3dgs_lod_cut_masked), weights included -> n; one synchronising read"""
    L = _lib.lib()
    N, dev = scene.nodes.shape[0], scene.nodes.device
    mask = cull_mask(scene, cam)
    count = torch.zeros(1, dtype=torch.int32, device=dev)
    scratch = torch.empty(int(L.h3dgs_expand_scratch_bytes(N)), dtype=torch.uint8, device=dev)
    _lib.check(L.h3dgs_lod_cut_masked(N, scene.nodes.data_ptr(), scene.boxes.data_ptr(), float(threshold), None,
                                      cam.campos.data_ptr(), mask.data_ptr(), scene.render_indices.data_ptr(),
                                      scene.parent_indices.data_ptr(), scene.nodes_for_render.data_ptr(),
                                      scene.interpolation_weights.data_ptr(), scene.num_siblings.data_ptr(),
                                      count.data_ptr(), scratch.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
    return int(count.item())


def fused_cut(scene, cam, threshold, cull=False):
    """LOD cut for the fused form -> (n cut rows, P rows to rasterize): the skybox rows follow the
    cut in render_indices/parent_indices as their own parents with t = 1, kids = 1.
    cull: keep only the cut rows that can reach cam's image (cull_mask); the image is the same."""
    n = _culled_cut(scene, cam, threshold) if cull else lod_cut(scene, cam, threshold)
    S = scene.skybox_points
    if S:
        scene.render_indices[n:n + S] = scene.skybox_inds
        scene.parent_indices[n:n + S] = scene.skybox_inds
        _skybox_weights(scene, n)
    return n, n + S


def render_hier_fused(scene, cam, bg, threshold, sh_degree=3, cull=False):
    """Same result as render_hier, but the cut gather + parent lerp (and the gradient scatter in
    backward) run inside K1/K9 through the settings' render_indices/parent_indices fields instead
    of ~25 PyTorch kernels with full-size temporaries (SURVEY.md 8f-1).  Skybox rows are appended to
    the cut as indices that are their own parent with t = 1 (x = 1*x exactly, as in render_post).
    cull: the view-culled cut (fused_cut); the image is bit-identical, n counts the culled cut's rows."""
    n, P = fused_cut(scene, cam, threshold, cull)
    rs = make_settings(scene, cam, bg, sh_degree, ts=scene.interpolation_weights, kids=scene.num_siblings,
                       ridx=scene.render_indices[:P], pidx=scene.parent_indices[:P])
    means2D = torch.zeros((P, 3), device=scene.means3D.device, requires_grad=scene.means3D.requires_grad)
    img, radii, _ = GaussianRasterizer(rs)(means3D=scene.means3D, means2D=means2D, shs=scene.shs, colors_precomp=None,
                                           opacities=scene.opacities, scales=scene.scales, rotations=scene.rotations,
                                           cov3D_precomp=None)
    return img, radii, n


def budget_threshold(scene, cam, budget, floor, cull=False):
    """The finest LOD threshold whose cut holds at most `budget` rows (skybox rows not counted), no finer than `floor`
    -> (threshold, rows of the cut there, met).  When even the coarsest cut (at the largest finite node size) exceeds
    the budget, that threshold comes back with met = False.  cull: count only the rows that can reach cam's image
    (cull_mask), the rows the culled cut keeps.  One synchronising read; sync-free forms use GraphedRender(budget=...)."""
    L = _lib.lib()
    N, dev = scene.nodes.shape[0], scene.nodes.device
    scratch = torch.empty(int(L.h3dgs_lod_budget_scratch_bytes(N)), dtype=torch.uint8, device=dev)
    thr = torch.empty(1, dtype=torch.float32, device=dev)
    info = torch.empty(4, dtype=torch.int32, device=dev)
    mask = cull_mask(scene, cam) if cull else None
    _lib.check(L.h3dgs_lod_budget_masked(N, scene.nodes.data_ptr(), scene.boxes.data_ptr(), cam.campos.data_ptr(),
                                         _lib.ptr(mask), float(floor), None, int(budget), None, thr.data_ptr(),
                                         info.data_ptr(), scratch.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
    t, i = thr.cpu(), info.cpu()
    return float(t[0]), int(i[0]), not bool(i[1])


def render_hier_budget(scene, cam, bg, budget, floor, sh_degree=3, cull=False):
    """render_hier_fused at budget_threshold(scene, cam, budget, floor, cull) -> (img, radii, n, threshold, met)"""
    threshold, _, met = budget_threshold(scene, cam, budget, floor, cull)
    img, radii, n = render_hier_fused(scene, cam, bg, threshold, sh_degree, cull)
    return img, radii, n, threshold, met


def l1_step(scene, cam, bg, gt, threshold=None, sh_degree=3, fused=True, gt_ready=None):
    """forward + L1 loss + backward; returns the loss tensor (device) and bookkeeping.
    gt_ready: optional CUDA event after which `gt` (uploaded on another stream) may be read."""
    scene.zero_grad()
    if scene.hier:
        img, radii, n = (render_hier_fused if fused else render_hier)(scene, cam, bg, threshold, sh_degree)
    else:
        img, radii = render_flat(scene, cam, bg, sh_degree)
        n = scene.means3D.shape[0]
    if gt_ready is not None:
        torch.cuda.current_stream().wait_event(gt_ready)
    loss = (img - gt).abs().mean()
    loss.backward()
    return loss, radii, n


def post_step(scene, cam, bg, gt, threshold, lambda_dssim=0.2, exposure=None, mask=None, sh_degree=3, state=None,
              update=True):
    """One step of train_post's loop body (train_post.py:91-142) on the exact path: render_hier_fused, then the objective
    (exposure, clamp, alpha mask, (1-l) L1 + l (1 - SSIM): h3dgs.loss.post_loss), then backward.  Gradients land in the
    scene's tensors.  Also the path that re-runs a frame h3dgs.poststep.GraphedPostStep flagged as overflowed.

    state: a h3dgs.poststep.PostState (scene = state.make_scene()).  With update=True the iteration then ends with the
    state's parameter step (train_post.py:167-192: the locks, the dense Adam step with state.set_learning_rate's xyz lr),
    which also refreshes the scene's activated rows.  update=False leaves the state as it is (a saving iteration, whose
    step follows scene.save, and the last iteration, which takes none).
    -> ((loss, l1, ssim) device scalars, radii, n cut rows)"""
    from .loss import post_loss
    scene.zero_grad()
    img, radii, n = render_hier_fused(scene, cam, bg, threshold, sh_degree)
    loss, l1, ssim = post_loss(img, gt, lambda_dssim, exposure, mask)
    loss.backward()
    if state is not None and update:
        state.param_step(scene)
    return (loss, l1, ssim), radii, n


class DensifyStats:
    """The three per-Gaussian tensors train_single's densification reads (scene/gaussian_model.py: max_radii2D [N],
    xyz_gradient_accum [N,1], denom [N,1]), zero for a new model."""

    def __init__(self, N, device="cuda"):
        self.max_radii2D = torch.zeros(N, device=device)
        self.xyz_gradient_accum = torch.zeros((N, 1), device=device)
        self.denom = torch.zeros((N, 1), device=device)

    def update(self, radii, d_means2D, scan_info=None):
        """train_single.py:147-148 in one kernel (h3dgs_densify_stats).  scan_info: the state word of a capacity-mode
        frame (an overflowed frame then changes nothing); None = the exact mode."""
        from . import _lib
        P = self.denom.shape[0]
        if radii.shape != (P,) or radii.dtype != torch.int32 or not radii.is_contiguous():
            raise ValueError(f"radii must be a contiguous int32 [{P}] (the statistics hold {P} rows), not {radii.dtype} {tuple(radii.shape)}")
        if d_means2D.shape != (P, 3) or d_means2D.dtype != torch.float32 or not d_means2D.is_contiguous():
            raise ValueError(f"d_means2D must be a contiguous float32 [{P}, 3], not {d_means2D.dtype} {tuple(d_means2D.shape)}")
        with torch.cuda.device(radii.device):
            _lib.check(_lib.lib().h3dgs_densify_stats(radii.shape[0], radii.data_ptr(), d_means2D.data_ptr(),
                                                     self.max_radii2D.data_ptr(), self.xyz_gradient_accum.data_ptr(),
                                                     self.denom.data_ptr(), None if scan_info is None else scan_info.data_ptr(),
                                                     torch.cuda.current_stream().cuda_stream))


def single_step(scene, cam, bg, gt, lambda_dssim=0.2, exposure=None, mask=None, mono_invdepth=None, depth_mask=None,
                depth_weight=0.0, stats=None, sh_degree=3, state=None, cameras_extent=None, update=True):
    """One step of train_single's loop body (train_single.py:94-148) on a flat scene, on the exact path: render() with
    do_depth, the objective (h3dgs.loss.single_loss: exposure, clamp, alpha mask, (1-l) L1 + l (1 - SSIM), plus
    depth_weight times the inverse-depth L1 when mono_invdepth is given and the weight is not 0), backward, and the
    densification statistics into `stats` (a DensifyStats; None skips them).  Gradients land in the scene's tensors and,
    when `exposure` requires grad, in exposure.grad.  Also the path that re-runs a frame
    h3dgs.singlestep.GraphedSingleStep flagged as overflowed.

    state: a h3dgs.singlestep.SingleState (scene = state.make_scene()).  The exposure is then the state's row of the
    image state.set_image() named, its gradient lands in state.exposure_grad, and with update=True the iteration ends
    with the state's parameter step (train_single.py:159-186, rescale threshold from cameras_extent), which also
    refreshes the scene's activated rows.  update=False leaves the state as it is (save, checkpoint, densify and reset
    iterations, and the last one).
    -> ((loss, photo, l1, ssim, depth_l1) device scalars, radii, means2D with its .grad)"""
    from .loss import single_loss
    if scene.hier:
        raise ValueError("single_step trains a flat scene (train_single.py); a hierarchy goes through post_step")
    if state is not None:
        if exposure is not None:
            raise ValueError("with a state the exposure is the state's row of the frame's image (state.set_image)")
        if update and cameras_extent is None:
            raise ValueError("the parameter step needs cameras_extent (the rescale threshold)")
        exposure = state.exposure_row().requires_grad_(True)
    scene.zero_grad()
    means2D = torch.zeros_like(scene.means3D, requires_grad=True)
    img, radii, invdepth = render_flat(scene, cam, bg, sh_degree, do_depth=True, means2D=means2D)
    out = single_loss(img, invdepth, gt, lambda_dssim, exposure, mask, mono_invdepth, depth_mask, depth_weight)
    out[0].backward()
    if stats is not None:
        stats.update(radii, means2D.grad)
    if state is not None:
        state.exposure_grad.copy_(exposure.grad)
        if update:
            grads = dict(means3D=scene.means3D.grad, shs=scene.shs.grad, opacities=scene.opacities.grad,
                         scales=scene.scales.grad, rotations=scene.rotations.grad)
            state.param_step(scene, {k: v.contiguous() for k, v in grads.items()}, cameras_extent)
    return out, radii, means2D


def coarse_step(state, scene, cam, bg, gt, cameras_extent, lambda_dssim=0.2, mask=None, sh_degree=0, update=True):
    """One iteration of train_coarse's loop body (train_coarse.py:97-145) on the exact path: render_coarse (render_flat
    of the activated rows in `scene`, state.make_scene()), the objective (h3dgs.loss.coarse_loss: alpha mask, (1-l) L1
    + l (1 - SSIM), no clamp), backward, max_radii2D, then with update=True the parameter step of
    h3dgs.coarsestep.CoarseState (skybox lock, relevance, Adam, rescale) on the gradients that landed in the scene's
    tensors, which also refreshes the activated rows.  update=False leaves the state as it is (the reference's last
    iteration, train_coarse.py:134).  Also the path that re-runs a frame h3dgs.coarsestep.GraphedCoarseStep flagged as
    overflowed.  -> ((loss, l1, ssim) device scalars, radii)"""
    from .loss import coarse_loss
    if scene.hier:
        raise ValueError("coarse_step trains a flat scene (train_coarse.py)")
    scene.zero_grad()
    img, radii = render_flat(scene, cam, bg, sh_degree)
    out = coarse_loss(img, gt, lambda_dssim, mask)
    out[0].backward()
    state.update_max_radii(radii)
    if update:
        grads = dict(means3D=scene.means3D.grad, shs=scene.shs.grad, opacities=scene.opacities.grad, scales=scene.scales.grad,
                     rotations=scene.rotations.grad)
        state.param_step(scene, {k: v.contiguous() for k, v in grads.items()}, cameras_extent)
    return out, radii


def fov_threshold(tau, cam):
    """render_hierarchy.py:55-56"""
    return (2 * (tau + 0.5)) * cam.tanfovx / (0.5 * cam.W)

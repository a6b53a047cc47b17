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


def render_flat(scene, cam, bg, sh_degree=3):
    """`render()` of the reference minus exposure/clamp (flat chunk training, config #2)."""
    rs = make_settings(scene, cam, bg, sh_degree)
    means2D = torch.zeros_like(scene.means3D, requires_grad=scene.means3D.requires_grad)
    img, radii, _ = GaussianRasterizer(rs)(means3D=scene.means3D, means2D=means2D, shs=scene.shs, colors_precomp=None,
                                           opacities=scene.opacities, scales=scene.scales, rotations=scene.rotations,
                                           cov3D_precomp=None)
    return img, radii


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


def fused_cut(scene, cam, threshold):
    """LOD cut for the fused form -> (n cut rows, P rows to rasterize): the skybox rows follow the
    cut in render_indices/parent_indices as their own parents with t = 1, kids = 1."""
    n = lod_cut(scene, cam, threshold)
    S = scene.skybox_points
    if S:
        scene.render_indices[n:n + S] = scene.skybox_inds
        scene.parent_indices[n:n + S] = scene.skybox_inds
        _skybox_weights(scene, n)
    return n, n + S


def render_hier_fused(scene, cam, bg, threshold, sh_degree=3):
    """Same result as render_hier, but the cut gather + parent lerp (and the gradient scatter in
    backward) run inside K1/K9 through the settings' render_indices/parent_indices fields instead
    of ~25 PyTorch kernels with full-size temporaries (SURVEY.md 8f-1).  Skybox rows are appended to
    the cut as indices that are their own parent with t = 1 (x = 1*x exactly, as in render_post)."""
    n, P = fused_cut(scene, cam, threshold)
    rs = make_settings(scene, cam, bg, sh_degree, ts=scene.interpolation_weights, kids=scene.num_siblings,
                       ridx=scene.render_indices[:P], pidx=scene.parent_indices[:P])
    means2D = torch.zeros((P, 3), device=scene.means3D.device, requires_grad=scene.means3D.requires_grad)
    img, radii, _ = GaussianRasterizer(rs)(means3D=scene.means3D, means2D=means2D, shs=scene.shs, colors_precomp=None,
                                           opacities=scene.opacities, scales=scene.scales, rotations=scene.rotations,
                                           cov3D_precomp=None)
    return img, radii, n


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


def post_step(scene, cam, bg, gt, threshold, lambda_dssim=0.2, exposure=None, mask=None, sh_degree=3):
    """One step of train_post's loop body (train_post.py:91-142) on the exact path: render_hier_fused, then the objective
    (exposure, clamp, alpha mask, (1-l) L1 + l (1 - SSIM): h3dgs.loss.post_loss), then backward.  Gradients land in the
    scene's tensors.  Also the path that re-runs a frame h3dgs.poststep.GraphedPostStep flagged as overflowed.
    -> ((loss, l1, ssim) device scalars, radii, n cut rows)"""
    from .loss import post_loss
    scene.zero_grad()
    img, radii, n = render_hier_fused(scene, cam, bg, threshold, sh_degree)
    loss, l1, ssim = post_loss(img, gt, lambda_dssim, exposure, mask)
    loss.backward()
    return (loss, l1, ssim), radii, n


def fov_threshold(tau, cam):
    """render_hierarchy.py:55-56"""
    return (2 * (tau + 0.5)) * cam.tanfovx / (0.5 * cam.W)

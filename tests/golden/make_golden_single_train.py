"""Generates tests/golden/single_train.npz by EXECUTING the reference's own code on the CPU: GaussianModel(3) (its
activations, training_setup's six groups with OurAdam, exposure_optimizer = torch.optim.Adam([_exposure]), the lr
schedulers, oneupSHdegree, densify_and_prune, reset_opacity, scaling_inverse_activation), render()
(gaussian_renderer/__init__.py:21-125, use_trained_exp=True) with a CAPTURING fake rasterizer, the reference's
utils/loss_utils l1_loss and ssim, and train_single.py:85-186 restated verbatim (train_single.py itself needs a dataset,
a GPU and a viewer socket) over six consecutive iterations, 999..1004, four images with their own exposures:

  999    SH degree 0, skybox locked, image 0, the exposure lr inside its delay phase, irrelevant rows, an opacity
         gradient that underflows in sigmoid_backward;
  1000   oneupSHdegree (degree 1), skybox unlocked, image 1, violators of the rescale at and one ulp around the threshold,
         big rows below scaffold_points left alone;
  1001   no relevant row: OurAdam's dense step (scene/OurAdam.py:214-228, _single_tensor_adam2), skybox locked;
  1002   densify_and_prune (clones, splits and prunes): OurAdam takes no step and counts none, the exposure's step and
         the rescale run on the densified rows;
  1003   a full step on the densified rows, the exposure lr past its delay phase;
  1004   reset_opacity alone: no Gaussian step, the exposure's step and the rescale.  It is the last iteration of the
         fixture: the reference does not zero the other five gradients after a reset alone (INTEGRATION.md).

The xyz scheduler of training_setup has no delay phase (get_expon_lr_func without lr_delay_steps); the exposure's has
one, here exposure_lr_delay_steps = 1002 so that both sides of it are in the fixture.  The fake rasterizer returns
raw + (sum over the activated inputs x of sum(x * K_x)) * P (coefficients above the active degree get no gradient, as
the rasterizer's); its radii are seeded.  Needs a checkout of the reference, named by H3DGS_REFERENCE.

  tests/test_single_train_cpu.py    tests/single_train_ref.py and the kernels (emulation build) == this fixture
  tests/test_gpu_single_train.py    the kernels on the device == this fixture
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "hierarchical-3d-gaussians_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "emul")):
    sys.path.insert(0, p)

import refharness                                    # noqa: E402
from fake_device import cuda_names_mean_cpu          # noqa: E402
from h3dgs import synth                              # noqa: E402

H, W, N, SKY, SCAFFOLD, NIMG = 19, 23, 80, 6, 10, 4
LAMBDA, EXTENT = 0.2, 8.0                            # the rescale threshold is EXTENT * 0.02
# iteration -> (skybox_locked, image, dense step)
PLAN = {999: (True, 0, False), 1000: (False, 1, False), 1001: (True, 2, True), 1002: (False, 3, False),
        1003: (False, 0, False), 1004: (False, 1, False)}
NAMES = ("means3D", "shs", "opacities", "scales", "rotations")
ATTRS = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")


class Capture(torch.nn.Module):
    """Stands in for diff_gaussian_rasterization.GaussianRasterizer."""
    raw = pattern = radii = K = None
    inputs = {}

    def __init__(self, raster_settings):
        super().__init__()
        Capture.settings = raster_settings

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None):
        xs = dict(means3D=means3D, shs=shs, opacities=opacities, scales=scales, rotations=rotations)
        s = 0.0
        for k, x in xs.items():
            if x.requires_grad and not x.is_leaf:
                x.retain_grad()
            s = s + (x * Capture.K[k]).sum()
        s = s + (means2D * Capture.K["means2D"]).sum()
        Capture.inputs = xs
        return Capture.raw + s * Capture.pattern, Capture.radii, torch.zeros((1, H, W))


def main():
    assert refharness.have_reference()
    with cuda_names_mean_cpu():
        gr = refharness.import_reference_renderer()
        gr.GaussianRasterizer = Capture
        from scene.gaussian_model import GaussianModel
        from scene import OurAdam
        from utils.loss_utils import l1_loss, ssim
        if not hasattr(OurAdam.Adam, "_cuda_graph_capture_health_check"):      # a private hook newer torch renamed
            OurAdam.Adam._cuda_graph_capture_health_check = lambda self: None
        torch.manual_seed(5)                                                # densify_and_split's samples
        rng = np.random.default_rng(23)
        f32 = lambda a: np.asarray(a, np.float32)
        q = lambda a: (np.round(a * 256.0) / 256.0).astype(np.float32)
        cam = synth.make_camera(W, H)
        gaussians = GaussianModel(3)
        xyz = f32(rng.normal(0, 2, (N, 3)))
        dc = f32(rng.normal(0, 0.5, (N, 1, 3)))
        rest = f32(rng.normal(0, 0.05, (N, 15, 3)))
        op = f32(np.full((N, 1), np.log(0.3 / 0.7)))
        op[:SKY] = 0.7
        op[SKY + 1, 0] = 30.0                        # sigmoid ~ 1: (g * (1 - y)) * y underflows for a tiny g
        op[N - 4:] = np.log(0.002 / 0.998)           # pruned by densify_and_prune (opacity < 0.005)
        sc = f32(rng.normal(-4.5, 0.6, (N, 3)))
        sc[40:50] = -1.8                             # split candidates: max scale > percent_dense * extent = 0.08
        rot = f32(rng.normal(0, 1, (N, 4)))
        thr = np.float32(EXTENT * 0.02)
        # violators at and one ulp around the threshold, on rows that get no gradient in iteration 1000 (torch's exp)
        s = torch.tensor([float(np.log(np.float64(thr)))], dtype=torch.float32)
        while torch.exp(s).item() > thr:
            s = torch.nextafter(s, torch.tensor([-np.inf]))
        while torch.exp(torch.nextafter(s, torch.tensor([np.inf]))).item() <= thr:
            s = torch.nextafter(s, torch.tensor([np.inf]))
        edges = (SCAFFOLD + 2, SCAFFOLD + 3, SCAFFOLD + 4)
        for r, v in zip(edges, (torch.nextafter(s, torch.tensor([-np.inf])), s, torch.nextafter(s, torch.tensor([np.inf])))):
            sc[r] = [float(v), -7.0, -7.0]
        sc[SCAFFOLD + 10:SCAFFOLD + 16] = -1.5       # big Gaussians with gradients
        sc[:SCAFFOLD] = -1.0                         # big skybox and scaffold rows are never rescaled
        P = lambda a: torch.nn.Parameter(torch.tensor(a))
        gaussians._xyz, gaussians._features_dc, gaussians._features_rest = P(xyz), P(dc), P(rest)
        gaussians._opacity, gaussians._scaling, gaussians._rotation = P(op), P(sc), P(rot)
        ex0 = torch.eye(3, 4)[None].repeat(NIMG, 1, 1) + torch.tensor(f32(rng.normal(0, 0.03, (NIMG, 3, 4))))
        gaussians._exposure = torch.nn.Parameter(ex0)
        gaussians.exposure_mapping = {f"img{i}": i for i in range(NIMG)}
        gaussians.pretrained_exposures = None
        gaussians.skybox_points = SKY
        gaussians.scaffold_points = SCAFFOLD
        gaussians.spatial_lr_scale = 1.0
        gaussians.max_radii2D = torch.zeros(N)
        opt = types.SimpleNamespace(percent_dense=0.01, position_lr_init=0.00002, position_lr_final=0.0000002,
                                    position_lr_delay_mult=0.01, position_lr_max_steps=30_000, feature_lr=0.0025,
                                    opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001, exposure_lr_init=0.001,
                                    exposure_lr_final=0.0001, exposure_lr_delay_steps=1002, exposure_lr_delay_mult=0.001,
                                    iterations=30_000, lambda_dssim=LAMBDA, densify_until_iter=15_000,
                                    densify_from_iter=500, densification_interval=501, opacity_reset_interval=1004,
                                    densify_grad_threshold=0.002)
        gaussians.training_setup(opt)
        out = {f"init_{a}": getattr(gaussians, a).detach().numpy().copy() for a in ATTRS}
        out["init_exposure"] = gaussians._exposure.detach().numpy().copy()
        vcam = refharness.StubCamera(cam, device="cpu")
        vcam.alpha_mask, vcam.depth_reliable = None, False
        pipe = refharness.Pipe()
        for c, iteration in enumerate(sorted(PLAN)):
            locked, image, dense = PLAN[iteration]
            gaussians.skybox_locked = locked
            n = gaussians._xyz.shape[0]
            K = {k: torch.tensor(f32(rng.normal(0, 1, shp)))
                 for k, shp in (("means3D", (n, 3)), ("shs", (n, 16, 3)), ("opacities", (n, 1)), ("scales", (n, 3)),
                                ("rotations", (n, 4)), ("means2D", (n, 3)))}
            K["opacities"][rng.uniform(size=n) < 0.4] = 0.0          # irrelevant rows
            K["opacities"][0] = 0.0                                  # the flattened index does not add row 0
            if iteration == 1000:
                for r in edges:
                    for v in K.values():
                        v[r] = 0.0
            K["opacities"][SKY + 1] = 1e-30                          # the underflow row
            if dense:
                K["opacities"].zero_()                               # no relevant row at all
            Capture.K = K
            Capture.raw = torch.tensor(q(rng.uniform(0.1, 0.8, (3, H, W))), requires_grad=True)
            Capture.pattern = torch.tensor(f32(rng.normal(0, 1e-3, (3, H, W))))
            Capture.radii = torch.tensor((rng.integers(0, 30, n) * (rng.uniform(size=n) > 0.2)).astype(np.int32))
            gt_image = torch.tensor(q(rng.uniform(0, 1, (3, H, W))))
            vcam.image_name = f"img{image}"
            viewpoint_cam = vcam
            background = torch.tensor(f32(rng.uniform(0, 1, 3)))
            # ---- train_single.py:85-186 ----
            gaussians.update_learning_rate(iteration)
            if iteration % 1000 == 0:
                gaussians.oneupSHdegree()
            deg = gaussians.active_sh_degree
            K["shs"][:, (deg + 1) ** 2:] = 0.0                      # the rasterizer's gradient above the active degree
            render_pkg = gr.render(viewpoint_cam, gaussians, pipe, background, indices=None, use_trained_exp=True)
            image_t, invDepth, viewspace_point_tensor, visibility_filter, radii = render_pkg["render"], render_pkg["depth"], render_pkg["viewspace_points"], render_pkg["visibility_filter"], render_pkg["radii"]
            Ll1 = l1_loss(image_t, gt_image)
            Lssim = (1.0 - ssim(image_t, gt_image))
            photo_loss = (1.0 - opt.lambda_dssim) * Ll1 + opt.lambda_dssim * Lssim
            loss = photo_loss.clone()
            loss.backward()
            rec = {}
            with torch.no_grad():
                act = {k: Capture.inputs[k].detach().numpy().copy() for k in NAMES}
                act_grad = {k: Capture.inputs[k].grad.numpy().copy() for k in NAMES}
                exposure_grad = gaussians._exposure.grad.numpy().copy()
                xyz_lr = [g["lr"] for g in gaussians.optimizer.param_groups if g["name"] == "xyz"][0]
                exp_lr = gaussians.exposure_optimizer.param_groups[0]["lr"]
                if iteration < opt.densify_until_iter:
                    gaussians.max_radii2D[visibility_filter] = torch.max(gaussians.max_radii2D[visibility_filter], radii)
                    gaussians.add_densification_stats(viewspace_point_tensor, visibility_filter)
                    densify = iteration > opt.densify_from_iter and iteration % opt.densification_interval == 0
                    if densify:
                        gaussians.densify_and_prune(opt.densify_grad_threshold, 0.005, EXTENT)
                    reset = iteration % opt.opacity_reset_interval == 0
                    if reset:
                        gaussians.reset_opacity()
                    if densify or reset:
                        st = lambda a: gaussians.optimizer.state[getattr(gaussians, a)]
                        rec.update({f"c{c}_dens{a}": getattr(gaussians, a).detach().numpy().copy() for a in ATTRS})
                        rec.update({f"c{c}_densm{a}": st(a)["exp_avg"].numpy().copy() for a in ATTRS})
                        rec.update({f"c{c}_densv{a}": st(a)["exp_avg_sq"].numpy().copy() for a in ATTRS})
                        rec[f"c{c}_n_after_densify"] = np.int32(gaussians._xyz.shape[0])
                if iteration < opt.iterations:
                    gaussians.exposure_optimizer.step()
                    gaussians.exposure_optimizer.zero_grad(set_to_none=True)
                    if gaussians._xyz.grad is not None and gaussians.skybox_locked:
                        gaussians._xyz.grad[:gaussians.skybox_points, :] = 0
                        gaussians._rotation.grad[:gaussians.skybox_points, :] = 0
                        gaussians._features_dc.grad[:gaussians.skybox_points, :, :] = 0
                        gaussians._features_rest.grad[:gaussians.skybox_points, :, :] = 0
                        gaussians._opacity.grad[:gaussians.skybox_points, :] = 0
                        gaussians._scaling.grad[:gaussians.skybox_points, :] = 0
                    gstep = gaussians._opacity.grad is not None
                    if gstep:
                        stored_grad = {a: getattr(gaussians, a).grad.numpy().copy() for a in ATTRS}
                        relevant = (gaussians._opacity.grad.flatten() != 0).nonzero()
                        relevant = relevant.flatten().long()
                        gaussians.optimizer.step(relevant)
                        gaussians.optimizer.zero_grad(set_to_none=True)
                    else:
                        stored_grad = {a: np.zeros_like(getattr(gaussians, a).detach().numpy()) for a in ATTRS}
                        relevant = torch.zeros(0, dtype=torch.long)
                    post_adam = {a: getattr(gaussians, a).detach().numpy().copy() for a in ATTRS}
                vals, _ = gaussians.get_scaling.max(dim=1)
                violators = vals > EXTENT * 0.02
                if gaussians.scaffold_points is not None:
                    violators[:gaussians.scaffold_points] = False
                gaussians._scaling[violators] = gaussians.scaling_inverse_activation(gaussians.get_scaling[violators] * 0.8)
            g = lambda a: gaussians.optimizer.state[getattr(gaussians, a)]
            es = gaussians.exposure_optimizer.state[gaussians._exposure]
            out.update(rec)
            out.update({f"c{c}_iteration": np.int32(iteration), f"c{c}_locked": np.int32(locked), f"c{c}_image": np.int32(image),
                        f"c{c}_degree": np.int32(deg), f"c{c}_gstep": np.int32(gstep), f"c{c}_xyz_lr": np.float64(xyz_lr),
                        f"c{c}_exp_lr": np.float64(exp_lr), f"c{c}_relevant": relevant.numpy(),
                        f"c{c}_exposure_grad": exposure_grad, f"c{c}_exposure": gaussians._exposure.detach().numpy().copy(),
                        f"c{c}_exposure_m": es["exp_avg"].numpy().copy(), f"c{c}_exposure_v": es["exp_avg_sq"].numpy().copy(),
                        f"c{c}_exposure_step": np.int64(float(es["step"])), f"c{c}_loss": np.float64(loss.item())})
            out.update({f"c{c}_act_{k}": v for k, v in act.items()})
            out.update({f"c{c}_actgrad_{k}": v for k, v in act_grad.items()})
            out.update({f"c{c}_grad{a}": v for a, v in stored_grad.items()})
            out.update({f"c{c}_adam{a}": v for a, v in post_adam.items()})
            out.update({f"c{c}_after{a}": getattr(gaussians, a).detach().numpy().copy() for a in ATTRS})
            out.update({f"c{c}_m{a}": g(a)["exp_avg"].numpy().copy() for a in ATTRS})
            out.update({f"c{c}_v{a}": g(a)["exp_avg_sq"].numpy().copy() for a in ATTRS})
            out[f"c{c}_step"] = np.int64(float(g("_xyz")["step"]))
            print(f"iteration {iteration}: degree {deg} locked={locked} image={image} N={gaussians._xyz.shape[0]} "
                  f"gstep={gstep} R={relevant.shape[0]} step={int(out[f'c{c}_step'])} exposure step={int(out[f'c{c}_exposure_step'])} "
                  f"violators={int(violators.sum())} xyz_lr={xyz_lr:.3e} exp_lr={exp_lr:.3e}")
        lrs = [g_["lr"] for g_ in gaussians.optimizer.param_groups]
        np.savez_compressed(os.path.join(HERE, "single_train.npz"), iterations=np.int32(len(PLAN)), lam=np.float64(LAMBDA),
                            extent=np.float64(EXTENT), skybox=np.int32(SKY), scaffold=np.int32(SCAFFOLD),
                            n_images=np.int32(NIMG), lrs=np.float64(lrs), edges=np.int32(edges), **out)


if __name__ == "__main__":
    main()

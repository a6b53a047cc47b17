"""Generates tests/golden/coarse_iteration.npz by EXECUTING the reference's own code on the CPU: GaussianModel(1) (its
activations, training_setup's six groups with OurAdam, oneupSHdegree, scaling_inverse_activation), render_coarse
(gaussian_renderer/__init__.py:296-407) with a CAPTURING fake rasterizer, the reference's utils/loss_utils l1_loss and
ssim, and train_coarse.py:97-145 restated verbatim (train_coarse.py itself needs a dataset, a GPU and a viewer socket)
over four consecutive iterations, 999..1002:

  it 0   SH degree 0, no mask, image values above 1, irrelevant rows, an opacity gradient that underflows in
         sigmoid_backward although the activated gradient is not 0;
  it 1   oneupSHdegree (degree 1), binary mask, violators of the rescale at and one ulp around the threshold;
  it 2   no relevant row: OurAdam's dense step (scene/OurAdam.py:214-228, _single_tensor_adam2);
  it 3   fractional mask; row 0 (a skybox row without a gradient of its own) carries momentum from its updates.

The fake rasterizer returns raw + (sum over the activated inputs x of sum(x * K_x)) * P: a seeded raw image as a leaf
that requires grad, and a seeded coupling that gives every activated input the gradient K_x * <dL/dimage, P>; its radii
are seeded.  Rows with K_opacity = 0 are irrelevant.  Needs a checkout of the reference, named by H3DGS_REFERENCE.

  tests/test_coarse_step_cpu.py    tests/coarse_ref.py, the kernels (emulation build) and the loss pair == this fixture
  tests/test_gpu_coarse_step.py    the kernels, the loss pair and h3dgs.optim.Adam with the [R,2] index == this fixture
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

H, W, N, SKY = 19, 23, 64, 6
LAMBDA, EXTENT = 0.2, 8.0                            # arguments/__init__.py; the threshold is EXTENT * 0.1
MASKS = ["none", "binary", "none", "fractional"]
NAMES = ("means3D", "shs", "opacities", "scales", "rotations")


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
        rng = np.random.default_rng(17)
        f32 = lambda a: np.asarray(a, np.float32)
        q = lambda a: (np.round(a * 256.0) / 256.0).astype(np.float32)
        cam = synth.make_camera(W, H)
        gaussians = GaussianModel(1)
        xyz = f32(rng.normal(0, 2, (N, 3)))
        dc = f32(rng.normal(0, 0.5, (N, 1, 3)))
        rest = np.zeros((N, 3, 3), np.float32)
        op = f32(np.full((N, 1), np.log(0.02 / 0.98)))
        op[:SKY] = 0.7
        op[SKY + 1, 0] = 30.0                        # sigmoid ~ 1: (g * (1 - y)) * y underflows for a tiny g
        sc = f32(rng.normal(-3.5, 0.6, (N, 3)))
        rot = f32(rng.normal(0, 1, (N, 4)))
        thr = np.float32(EXTENT * 0.1)
        # violators at and one ulp around the threshold, on rows that never get a gradient (their scaling stays put
        # until the dense step of it 2): the largest s with exp(s) <= thr (torch's exp), one below, one above
        s = torch.tensor([float(np.log(np.float64(thr)))], dtype=torch.float32)
        while torch.exp(s).item() > thr:
            s = torch.nextafter(s, torch.tensor([-np.inf]))
        while torch.exp(torch.nextafter(s, torch.tensor([np.inf]))).item() <= thr:
            s = torch.nextafter(s, torch.tensor([np.inf]))
        edges = (SKY + 2, SKY + 3, SKY + 4)
        for r, v in zip(edges, (torch.nextafter(s, torch.tensor([-np.inf])), s, torch.nextafter(s, torch.tensor([np.inf])))):
            sc[r] = [float(v), -5.0, -5.0]
        sc[SKY + 10:SKY + 16] = -1.0                 # big Gaussians with gradients
        sc[:3] = 0.0                                 # big skybox rows are never rescaled
        P = lambda a: torch.nn.Parameter(torch.tensor(a))
        gaussians._xyz, gaussians._features_dc, gaussians._features_rest = P(xyz), P(dc), P(rest)
        gaussians._opacity, gaussians._scaling, gaussians._rotation = P(op), P(sc), P(rot)
        gaussians._exposure = torch.nn.Parameter(torch.eye(3, 4)[None])
        gaussians.skybox_points = SKY
        gaussians.spatial_lr_scale = 1.0
        gaussians.max_radii2D = torch.zeros(N)
        opt = types.SimpleNamespace(percent_dense=0.01, position_lr_init=0.00002, position_lr_final=0.0000002,
                                    position_lr_delay_mult=0.01, position_lr_max_steps=30_000, feature_lr=0.0025,
                                    opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001, exposure_lr_init=0.001,
                                    exposure_lr_final=0.0001, exposure_lr_delay_steps=5000, exposure_lr_delay_mult=0.001,
                                    iterations=30_000, lambda_dssim=LAMBDA)
        gaussians.training_setup(opt)
        for param_group in gaussians.optimizer.param_groups:           # train_coarse.py:55-57
            if param_group["name"] == "xyz":
                param_group["lr"] = 0.0
        attrs = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")
        out = {f"init_{a}": getattr(gaussians, a).detach().numpy().copy() for a in attrs}
        vcam = refharness.StubCamera(cam, device="cpu")
        pipe = refharness.Pipe()
        for it, msk in enumerate(MASKS):
            iteration = 999 + it
            K = {k: torch.tensor(f32(rng.normal(0, 1, shp)))
                 for k, shp in (("means3D", (N, 3)), ("shs", (N, 4, 3)), ("opacities", (N, 1)), ("scales", (N, 3)),
                                ("rotations", (N, 4)), ("means2D", (N, 3)))}
            K["opacities"][rng.uniform(size=N) < 0.4] = 0.0          # irrelevant rows
            K["opacities"][0] = 0.0                                  # row 0 moves only through the zero column
            for r in edges:
                for v in K.values():
                    v[r] = 0.0
            K["opacities"][SKY + 1] = 1e-30                          # the underflow row
            if it == 2:
                K["opacities"].zero_()                               # no relevant row at all
            Capture.K = K
            Capture.raw = torch.tensor(q(rng.uniform(-0.2, 1.4, (3, H, W))), requires_grad=True)
            Capture.pattern = torch.tensor(f32(rng.normal(0, 1e-2, (3, H, W))))
            Capture.radii = torch.tensor((rng.integers(0, 30, N) * (rng.uniform(size=N) > 0.3)).astype(np.int32))
            gt_image = torch.tensor(q(rng.uniform(0, 1, (3, H, W))))
            if msk == "none":
                mask = None
            elif msk == "binary":
                mask = torch.tensor((rng.uniform(size=(1, H, W)) > 0.3).astype(np.float32))
            else:
                mask = torch.tensor(q((rng.uniform(size=(1, H, W)) > 0.3) * rng.uniform(0.2, 1.0, (1, H, W))))
            vcam.alpha_mask = mask
            viewpoint_cam = vcam
            background = torch.tensor(f32(rng.uniform(0, 1, 3)))
            # ---- train_coarse.py:97-145 ----
            if iteration % 1000 == 0:
                gaussians.oneupSHdegree()
            render_pkg = gr.render_coarse(viewpoint_cam, gaussians, pipe, background, indices=None)
            image, viewspace_point_tensor, visibility_filter, radii = render_pkg["render"], render_pkg["viewspace_points"], render_pkg["visibility_filter"], render_pkg["radii"]
            if viewpoint_cam.alpha_mask is not None:
                alpha_mask = viewpoint_cam.alpha_mask.cuda().float()
                Ll1 = l1_loss(image * alpha_mask, gt_image)
                loss = (1.0 - opt.lambda_dssim) * Ll1 + opt.lambda_dssim * (1.0 - ssim(image * alpha_mask, gt_image))
            else:
                Ll1 = l1_loss(image, gt_image)
                loss = (1.0 - opt.lambda_dssim) * Ll1 + opt.lambda_dssim * (1.0 - ssim(image, gt_image))
            loss.backward()
            gaussians.max_radii2D[visibility_filter] = torch.max(gaussians.max_radii2D[visibility_filter], radii)
            with torch.no_grad():
                act = {k: Capture.inputs[k].detach().numpy().copy() for k in NAMES}
                act_grad = {k: Capture.inputs[k].grad.numpy().copy() for k in NAMES}
                gaussians._scaling.grad[:gaussians.skybox_points, :] = 0
                relevant = (gaussians._opacity.grad != 0).nonzero()
                stored_grad = {a: getattr(gaussians, a).grad.numpy().copy() for a in attrs}
                gaussians.optimizer.step(relevant)
                post_adam = {a: getattr(gaussians, a).detach().numpy().copy() for a in attrs}
                gaussians.optimizer.zero_grad(set_to_none=True)
                with torch.no_grad():
                    vals, _ = gaussians.get_scaling.max(dim=1)
                    violators = vals > EXTENT * 0.1
                    violators[:gaussians.skybox_points] = False
                    gaussians._scaling[violators] = gaussians.scaling_inverse_activation(gaussians.get_scaling[violators] * 0.8)
            g = lambda a: gaussians.optimizer.state[getattr(gaussians, a)]
            out.update({f"c{it}_raw": Capture.raw.detach().numpy(), f"c{it}_pattern": Capture.pattern.numpy(),
                        f"c{it}_gt": gt_image.numpy(), f"c{it}_mask": np.ones((H, W), np.float32) if mask is None else mask.numpy()[0],
                        f"c{it}_has_mask": np.int32(mask is not None), f"c{it}_bg": background.numpy(),
                        f"c{it}_radii": Capture.radii.numpy(), f"c{it}_degree": np.int32(gaussians.active_sh_degree),
                        f"c{it}_loss": np.float64(loss.item()), f"c{it}_l1": np.float64(Ll1.item()),
                        f"c{it}_dimage": Capture.raw.grad.numpy().copy(), f"c{it}_image": image.detach().numpy().copy(), f"c{it}_relevant": relevant.numpy(),
                        f"c{it}_max_radii2D": gaussians.max_radii2D.numpy().copy()})
            out.update({f"c{it}_act_{k}": v for k, v in act.items()})
            out.update({f"c{it}_actgrad_{k}": v for k, v in act_grad.items()})
            out.update({f"c{it}_grad{a}": v for a, v in stored_grad.items()})
            out.update({f"c{it}_adam{a}": v for a, v in post_adam.items()})
            out.update({f"c{it}_after{a}": getattr(gaussians, a).detach().numpy().copy() for a in attrs})
            out.update({f"c{it}_m{a}": g(a)["exp_avg"].numpy().copy() for a in attrs})
            out.update({f"c{it}_v{a}": g(a)["exp_avg_sq"].numpy().copy() for a in attrs})
            out[f"c{it}_step"] = np.int64(float(g("_xyz")["step"]))
            print(f"iteration {iteration}: degree {gaussians.active_sh_degree} mask={msk} R={relevant.shape[0]} "
                  f"loss={loss.item():.7f} violators={int(violators.sum())}")
        lrs = [g_["lr"] for g_ in gaussians.optimizer.param_groups]
        np.savez_compressed(os.path.join(HERE, "coarse_iteration.npz"), iterations=np.int32(len(MASKS)), lam=np.float64(LAMBDA),
                            extent=np.float64(EXTENT), skybox=np.int32(SKY), lrs=np.float64(lrs), edges=np.int32(edges), **out)


if __name__ == "__main__":
    main()

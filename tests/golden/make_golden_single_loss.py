"""Generates tests/golden/single_loss.npz by EXECUTING the reference's own code on the CPU: render()
(gaussian_renderer/__init__.py:20-135, with use_trained_exp=True, so :115-118 apply the exposure and the clamp) with a
CAPTURING fake rasterizer that returns a seeded raw image and inverse depth as leaves that require grad, the model's
`_exposure` an nn.Parameter read through the reference's own get_exposure_from_name, then train_single.py's loss lines
(:101-117, around the reference's utils/loss_utils.l1_loss and ssim), loss.backward(), and the statistics lines
(train_single.py:147 and the reference's own GaussianModel.add_densification_stats).  The fake rasterizer couples the
zero means2D linearly into the image (image + sum(means2D * K), K seeded), which leaves the image as it is and gives
viewspace_points a gradient for the statistics.  train_single.py itself needs a dataset and a GPU, so its lines are
restated here.  Needs a checkout of the reference, named by H3DGS_REFERENCE.

  tests/test_single_loss_cpu.py    the kernels (emulation build) and h3dgs.loss.single_loss == this fixture
  tests/test_gpu_single_step.py    the kernels (nvcc build) == this fixture
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "hierarchical-3d-gaussians_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "emul")):
    sys.path.insert(0, p)

import refharness                                    # noqa: E402
from fake_device import cuda_names_mean_cpu          # noqa: E402
from h3dgs import synth                              # noqa: E402

# (exposure, alpha mask, depth term) per case
CASES = [("identity", "none", True), ("on", "binary", True), ("offset", "fractional", True), ("offset", "half", False),
         ("on", "none", True), ("offset", "binary", True)]
H, W, N = 21, 27, 50
LAMBDA = 0.2                                         # arguments/__init__.py
WEIGHTS = [1.0, 0.37, 0.05, 0.0, 0.0, 0.8]          # depth_l1_weight(iteration) of the case (0: the term is absent)


class Capture(torch.nn.Module):
    """Stands in for diff_gaussian_rasterization.GaussianRasterizer."""
    image = invdepth = radii = coupling = None

    def __init__(self, raster_settings):
        super().__init__()
        assert raster_settings.do_depth

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None):
        return Capture.image + (means2D * Capture.coupling).sum(), Capture.radii, Capture.invdepth * 1.0


def main():
    assert refharness.have_reference()
    with cuda_names_mean_cpu():
        gr = refharness.import_reference_renderer()
        gr.GaussianRasterizer = Capture
        from scene.gaussian_model import GaussianModel
        from utils.loss_utils import l1_loss, ssim
        cam = synth.make_camera(W, H)
        leaves = synth.cloud_v1(N, cam, zmin=2.0, zmax=30.0, seed=3, scale_k=1.0)
        pc = refharness.StubModel(leaves, device="cpu", requires_grad=False)
        pc.get_exposure_from_name = lambda name: GaussianModel.get_exposure_from_name(pc, name)
        vcam = refharness.StubCamera(cam, device="cpu")
        pc.exposure_mapping = {vcam.image_name: 1}
        rng = np.random.default_rng(41)
        q = lambda a: (np.round(a * 256.0) / 256.0).astype(np.float32)
        out = {}
        # the statistics run on through the cases, as they do through training steps
        pc.max_radii2D = torch.zeros(N)
        pc.xyz_gradient_accum = torch.zeros((N, 1))
        pc.denom = torch.zeros((N, 1))
        for i, (exp, msk, depth) in enumerate(CASES):
            raw = q(rng.uniform(-0.2, 1.2, (3, H, W)))
            gt_raw = q(rng.uniform(-0.1, 1.1, (3, H, W)))
            E = np.eye(3, 4, dtype=np.float32)
            if exp != "identity":
                E[:, :3] = np.eye(3, dtype=np.float32) * 0.9 + rng.uniform(-0.15, 0.15, (3, 3)).astype(np.float32)
                E[:, 3] = rng.uniform(-0.05, 0.05, 3).astype(np.float32) if exp == "on" else (0.35, -0.3, 0.05)
            if msk == "none":
                mask = None
            elif msk == "binary":
                mask = (rng.uniform(size=(1, H, W)) > 0.3).astype(np.float32)
            elif msk == "half":
                mask = np.ones((1, H, W), np.float32)
                mask[..., : W // 2] = 0.0
            else:
                mask = q((rng.uniform(size=(1, H, W)) > 0.3) * rng.uniform(0.2, 1.0, (1, H, W)))
            invd = q(rng.uniform(0.0, 2.0, (1, H, W)))
            mono = q(rng.uniform(0.0, 2.0, (1, H, W)))
            same = rng.uniform(size=(1, H, W)) < 0.1
            mono[same] = invd[same]
            dmask = (rng.uniform(size=(1, H, W)) > 0.25).astype(np.float32)
            radii = (rng.integers(0, 40, N) * (rng.uniform(size=N) > 0.4)).astype(np.int32)
            gt_image = torch.tensor(gt_raw).clamp(0.0, 1.0)                   # cameras.py:62
            if mask is not None:
                gt_image *= torch.tensor(mask)                                 # :66-67
            Capture.image = torch.tensor(raw, requires_grad=True)
            Capture.invdepth = torch.tensor(invd, requires_grad=True)
            Capture.radii = torch.tensor(radii)
            Capture.coupling = torch.tensor(rng.uniform(-3.0, 3.0, (N, 3)).astype(np.float32))
            pc._exposure = torch.nn.Parameter(torch.stack([torch.eye(3, 4), torch.tensor(E)]))      # gaussian_model.py:259-260
            viewpoint_cam = vcam
            viewpoint_cam.alpha_mask = None if mask is None else torch.tensor(mask)
            viewpoint_cam.depth_reliable = depth
            weight = WEIGHTS[i]
            # ---- train_single.py:97-123 ----
            render_pkg = gr.render(viewpoint_cam, pc, refharness.Pipe(), torch.zeros(3), indices=None, use_trained_exp=True)
            image, invDepth, viewspace_point_tensor, visibility_filter, radii_v = render_pkg["render"], render_pkg["depth"], render_pkg["viewspace_points"], render_pkg["visibility_filter"], render_pkg["radii"]
            if viewpoint_cam.alpha_mask is not None:
                alpha_mask = viewpoint_cam.alpha_mask
                image *= alpha_mask
            Ll1 = l1_loss(image, gt_image)
            Lssim = (1.0 - ssim(image, gt_image))
            photo_loss = (1.0 - LAMBDA) * Ll1 + LAMBDA * Lssim
            loss = photo_loss.clone()
            Ll1depth_pure = torch.zeros(())
            if weight > 0 and viewpoint_cam.depth_reliable:
                mono_invdepth = torch.tensor(mono)
                depth_mask = torch.tensor(dmask)
                Ll1depth_pure = torch.abs((invDepth - mono_invdepth) * depth_mask).mean()
                Ll1depth = weight * Ll1depth_pure
                loss += Ll1depth
            loss.backward()
            # ---- train_single.py:147-148 ----
            with torch.no_grad():
                pc.max_radii2D[visibility_filter] = torch.max(pc.max_radii2D[visibility_filter], radii_v)
                GaussianModel.add_densification_stats(pc, viewspace_point_tensor, visibility_filter)
            dinv = Capture.invdepth.grad
            out.update({f"c{i}_raw": raw, f"c{i}_gt": gt_image.numpy(), f"c{i}_E": E,
                        f"c{i}_mask": np.ones((H, W), np.float32) if mask is None else mask[0],
                        f"c{i}_flags": np.array([mask is not None, weight > 0 and depth], np.int32),
                        f"c{i}_invdepth": invd[0], f"c{i}_mono": mono[0], f"c{i}_dmask": dmask[0], f"c{i}_weight": np.float64(weight),
                        f"c{i}_radii": radii, f"c{i}_dmeans2D": viewspace_point_tensor.grad.numpy().astype(np.float32),
                        f"c{i}_loss": np.float64(loss.item()), f"c{i}_photo": np.float64(photo_loss.item()),
                        f"c{i}_l1": np.float64(Ll1.item()), f"c{i}_depth": np.float64(Ll1depth_pure.item()),
                        f"c{i}_grad": Capture.image.grad.numpy().astype(np.float32),
                        f"c{i}_dinv": (torch.zeros(1, H, W) if dinv is None else dinv).numpy()[0].astype(np.float32),
                        f"c{i}_dE": pc._exposure.grad.numpy()[1].astype(np.float32),
                        f"c{i}_max_radii2D": pc.max_radii2D.numpy().copy(), f"c{i}_accum": pc.xyz_gradient_accum.numpy().copy(),
                        f"c{i}_denom": pc.denom.numpy().copy()})
            assert float(pc._exposure.grad[0].abs().sum()) == 0.0
            print(f"case {i}: exposure={exp} mask={msk} depth={depth} w={weight} loss={loss.item():.7f} depth={Ll1depth_pure.item():.7f}")
        np.savez_compressed(os.path.join(HERE, "single_loss.npz"), cases=np.int32(len(CASES)), lam=np.float64(LAMBDA), **out)


if __name__ == "__main__":
    main()

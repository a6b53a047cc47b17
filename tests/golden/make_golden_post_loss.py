"""Generates tests/golden/post_loss.npz by EXECUTING the reference's own code on the CPU: render_post()
(gaussian_renderer/__init__.py:138-292) with a CAPTURING fake rasterizer that returns a seeded raw image as a leaf that
requires grad -- with use_trained_exp=True and a `pretrained_exposures` entry where a case has an exposure, which pins
the direction of the exposure matrix and the clamp after it -- followed by train_post.py's loss lines (:134-137: the
image times the alpha mask, (1 - lambda) l1_loss + lambda (1 - ssim)) around the reference's own utils/loss_utils.l1_loss
and ssim, and loss.backward().  The stored gradient is dL/d(raw image), through the reference's exposure and clamp.  The
target is what scene/cameras.py:62-67 leaves: clamped, then multiplied by the mask.  train_post.py itself needs a dataset
and a GPU, so its two loss lines are restated here.  Needs a checkout of the reference, named by H3DGS_REFERENCE.

  tests/test_post_loss_cpu.py     the post-loss kernels (emulation build) == this fixture
  tests/test_gpu_post_step.py     the post-loss kernels (nvcc build) == this fixture
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
from fake_device import cuda_names_mean_cpu          # noqa: E402  (device="cuda" in the reference lands on the CPU)
from h3dgs import synth                              # noqa: E402

# (exposure: none / on / offset driving pixels below 0 and above 1, mask: ones / binary / train_test_exp half /
# fractional / zero) per case; H x W odd so that the tiles are ragged
CASES = [("none", "ones"), ("on", "ones"), ("offset", "ones"), ("none", "binary"), ("on", "half"), ("offset", "fractional"),
         ("on", "zero"), ("offset", "binary")]
H, W = 21, 27
LAMBDA = 0.2                                         # arguments/__init__.py:98


class Capture(torch.nn.Module):
    """Stands in for diff_gaussian_rasterization.GaussianRasterizer: returns the seeded raw image of the case."""
    image = None

    def __init__(self, raster_settings):
        super().__init__()
        self.rs = raster_settings

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None):
        return Capture.image * 1.0, torch.ones(means3D.shape[0], dtype=torch.int32), torch.zeros(1, H, W)


def main():
    assert refharness.have_reference()
    with cuda_names_mean_cpu():
        gr = refharness.import_reference_renderer()
        gr.GaussianRasterizer = Capture               # the module-level name render_post() looks up
        from utils.loss_utils import l1_loss, ssim
        cam = synth.make_camera(W, H)
        leaves = synth.cloud_v1(50, cam, zmin=2.0, zmax=30.0, seed=3, scale_k=1.0)
        pc = refharness.StubModel(leaves, device="cpu", requires_grad=False)
        vcam = refharness.StubCamera(cam, device="cpu")
        rng = np.random.default_rng(29)
        out = {}
        for i, (exp, msk) in enumerate(CASES):
            # multiples of 1/256 (exact in fp32; with no exposure, some land exactly on 0 and 1, where the clamp passes)
            q = lambda a: (np.round(a * 256.0) / 256.0).astype(np.float32)
            raw = q(rng.uniform(-0.2, 1.2, (3, H, W)))
            gt_raw = q(rng.uniform(-0.1, 1.1, (3, H, W)))
            E = np.zeros((3, 4), np.float32)
            if exp != "none":
                # a non-symmetric 3x4 affine colour transform: a transposed application would give other numbers
                E[:, :3] = np.eye(3, dtype=np.float32) * 0.9 + rng.uniform(-0.15, 0.15, (3, 3)).astype(np.float32)
                E[:, 3] = rng.uniform(-0.05, 0.05, 3).astype(np.float32) if exp == "on" else (0.35, -0.3, 0.05)
            if msk == "ones":
                mask = np.ones((1, H, W), np.float32)
            elif msk == "binary":
                mask = (rng.uniform(size=(1, H, W)) > 0.3).astype(np.float32)
            elif msk == "half":                                                # cameras.py:56-60 (a test view, train_test_exp)
                mask = np.ones((1, H, W), np.float32)
                mask[..., : W // 2] = 0.0
            elif msk == "fractional":
                mask = q((rng.uniform(size=(1, H, W)) > 0.3) * rng.uniform(0.2, 1.0, (1, H, W)))
            else:
                mask = np.zeros((1, H, W), np.float32)
            alpha_mask = torch.tensor(mask)
            gt_image = torch.tensor(gt_raw).clamp(0.0, 1.0)                  # cameras.py:62
            gt_image *= alpha_mask                                             # :66-67
            Capture.image = torch.tensor(raw, requires_grad=True)
            pc.pretrained_exposures = {vcam.image_name: torch.tensor(E)} if exp != "none" else None
            image = gr.render_post(vcam, pc, refharness.Pipe(), torch.zeros(3), use_trained_exp=True)["render"]
            Ll1 = l1_loss(image * alpha_mask, gt_image)                        # train_post.py:135-136
            loss = (1.0 - LAMBDA) * Ll1 + LAMBDA * (1.0 - ssim(image * alpha_mask, gt_image))
            loss.backward()
            out.update({f"c{i}_raw": raw, f"c{i}_gt": gt_image.numpy(), f"c{i}_E": E, f"c{i}_mask": mask[0],
                        f"c{i}_flags": np.array([exp != "none", msk != "ones"], np.int32),
                        f"c{i}_loss": np.float64(loss.item()), f"c{i}_l1": np.float64(Ll1.item()),
                        f"c{i}_grad": Capture.image.grad.numpy().astype(np.float32)})
            print(f"case {i}: exposure={exp} mask={msk} loss={loss.item():.7f} l1={Ll1.item():.7f}")
        np.savez_compressed(os.path.join(HERE, "post_loss.npz"), cases=np.int32(len(CASES)), lam=np.float64(LAMBDA), **out)


if __name__ == "__main__":
    main()

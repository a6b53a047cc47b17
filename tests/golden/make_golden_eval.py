"""Generates tests/golden/eval_metrics.npz by EXECUTING the reference's own code on the CPU: render_post()
(gaussian_renderer/__init__.py:138-292) with a CAPTURING fake rasterizer that returns a seeded raw image -- with
use_trained_exp=True and a `pretrained_exposures` entry where a case has an exposure, which pins the direction of the
exposure matrix and the clamp after it -- followed by the evaluation lines of render_hierarchy.py:94-112 (clamp of the
target, train_test_exp half-width crop, alpha mask) and the reference's own psnr (utils/image_utils.py) and ssim
(utils/loss_utils.py).  render_hierarchy.py itself imports torchvision and lpips, so its dozen evaluation lines are
restated here around those calls.  Needs a checkout of the reference, named by H3DGS_REFERENCE, and no GPU.

  tests/test_eval_metrics_golden_cpu.py   the metrics kernel (emulation build) == this fixture
  tests/test_gpu_evaluate.py              the metrics kernel (nvcc build) == this fixture
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

# (exposure, mask, train_test_exp crop, one channel exact) per case; H x W odd so that tiles and the crop are ragged.
# An exact channel is only exact without exposure: the 3x3 product may round differently from torch's matmul by an ulp.
CASES = [(False, False, False, False), (True, False, False, False), (False, True, False, False), (False, False, True, False),
         (True, True, True, False), (True, True, False, False), (False, True, True, False), (False, False, False, True),
         (False, True, True, True)]
H, W = 29, 43


class Capture(torch.nn.Module):
    """Stands in for diff_gaussian_rasterization.GaussianRasterizer: returns the seeded raw image of the case."""
    image = None

    def __init__(self, raster_settings):
        super().__init__()
        self.rs = raster_settings

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None):
        return Capture.image.clone(), torch.ones(means3D.shape[0], dtype=torch.int32), torch.zeros(1, H, W)


def main():
    assert refharness.have_reference()
    with cuda_names_mean_cpu():
        gr = refharness.import_reference_renderer()
        gr.GaussianRasterizer = Capture               # the module-level name render_post() looks up
        from utils.image_utils import psnr
        from utils.loss_utils import ssim
        cam = synth.make_camera(W, H)
        leaves = synth.cloud_v1(50, cam, zmin=2.0, zmax=30.0, seed=3, scale_k=1.0)
        pc = refharness.StubModel(leaves, device="cpu", requires_grad=False)
        vcam = refharness.StubCamera(cam, device="cpu")
        rng = np.random.default_rng(17)
        out = {}
        for i, (exp, msk, crop, exact) in enumerate(CASES):
            # raw renders and targets reach a little beyond [0, 1] on both sides, so that both clamps act
            # (multiples of 1/256: exact in fp32, and the fixture compresses)
            q = lambda a: (np.round(a * 256.0) / 256.0).astype(np.float32)
            raw = q(rng.uniform(-0.15, 1.15, (3, H, W)))
            gt = q(rng.uniform(-0.1, 1.1, (3, H, W)))
            E = np.zeros((3, 4), np.float32)
            if exp:
                # a non-symmetric 3x4 affine colour transform: a transposed application would give other numbers
                E[:, :3] = np.eye(3, dtype=np.float32) * 0.9 + rng.uniform(-0.15, 0.15, (3, 3)).astype(np.float32)
                E[:, 3] = rng.uniform(-0.05, 0.05, 3).astype(np.float32)
            mask = q((rng.uniform(size=(1, H, W)) > 0.3) * rng.uniform(0.5, 1.0, (1, H, W)))
            Capture.image = torch.tensor(raw)
            pc.pretrained_exposures = {vcam.image_name: torch.tensor(E)} if exp else None
            with torch.no_grad():
                image = gr.render_post(vcam, pc, refharness.Pipe(), torch.zeros(3), use_trained_exp=exp)["render"]
                image = torch.clamp(image, 0.0, 1.0)                              # render_hierarchy.py:82-92
                if exact:
                    gt[0] = image[0].numpy()                                      # channel 0 exact: PSNR inf there
                gt_image = torch.clamp(torch.tensor(gt), 0.0, 1.0)                # :94
                alpha_mask = torch.tensor(mask) if msk else torch.ones(1, H, W)   # :96 (no mask = all ones)
                if crop:                                                          # :98-101
                    image = image[..., image.shape[-1] // 2:]
                    gt_image = gt_image[..., gt_image.shape[-1] // 2:]
                    alpha_mask = alpha_mask[..., alpha_mask.shape[-1] // 2:]
                saved = image.clone()                                             # what :104 saves
                image *= alpha_mask                                               # :109-112
                gt_image *= alpha_mask
                p = psnr(image, gt_image).mean().double()
                s = ssim(image, gt_image).mean().double()
            out.update({f"c{i}_raw": raw, f"c{i}_gt": gt, f"c{i}_E": E, f"c{i}_mask": mask[0],
                        f"c{i}_flags": np.array([exp, msk, crop, exact], np.int32), f"c{i}_image": saved.numpy(),
                        f"c{i}_psnr": np.float64(p), f"c{i}_ssim": np.float64(s)})
            print(f"case {i}: exp={exp} mask={msk} crop={crop} exact={exact} psnr={float(p):.6f} ssim={float(s):.6f}")
        np.savez_compressed(os.path.join(HERE, "eval_metrics.npz"), cases=np.int32(len(CASES)), **out)


if __name__ == "__main__":
    main()

"""Generates tests/golden/lpips.npz by EXECUTING the reference's own lpipsPyTorch.LPIPS('vgg') on the CPU, with two
monkeypatches so that nothing is downloaded: torchvision.models.vgg16 builds the network with seeded random weights, and
torch.hub.load_state_dict_from_url returns seeded linear weights under the upstream key names (lin{k}.model.1.weight).
Both come from tests/lpips_ref.seeded_state_dicts(SEED); the fixture keeps the seed and a checksum of the weights, not
the 59 MB of weights.  The inputs of each case are preprocessed as render_hierarchy.py:94-113 does (clamp, the
train_test_exp crop, the alpha mask) when the case says so, and passed unbatched [3,H,W], as there.
Needs a checkout of the reference, named by H3DGS_REFERENCE, and no GPU.

  tests/test_lpips_cpu.py     the float64 restatement and the emulation build of csrc/lpips.cu == this fixture
  tests/test_gpu_lpips.py     the nvcc build == this fixture, within the end-to-end budget
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import lpips_ref                                      # noqa: E402

SEED = 20240
# name, H, W, preprocess (clamp + mask/crop as render_hierarchy.py), mask, crop, identical pair
CASES = [("odd_37x53", 37, 53, False, False, False, False), ("min_16x16", 16, 16, False, False, False, False),
         ("odd_17x33", 17, 33, False, False, False, False), ("even_64x48", 64, 48, False, False, False, False),
         ("masked_37x53", 37, 53, True, True, False, False), ("crop_masked_33x70", 33, 70, True, True, True, False),
         ("identical_40x40", 40, 40, True, False, False, True)]
TOO_SMALL = (15, 40)


def main():
    ref = os.environ.get("H3DGS_REFERENCE")
    if not ref:
        sys.exit("set H3DGS_REFERENCE to a checkout of the reference")
    sys.path.insert(0, ref)
    import torchvision
    vgg_sd, lin_sd = lpips_ref.seeded_state_dicts(SEED)

    build = torchvision.models.vgg16

    def vgg16(*args, **kwargs):
        net = build(weights=None)
        net.features.load_state_dict({k[len("features."):]: v for k, v in vgg_sd.items()})
        return net
    torchvision.models.vgg16 = vgg16
    torch.hub.load_state_dict_from_url = lambda *a, **k: {k2: v.clone() for k2, v in lin_sd.items()}
    from lpipsPyTorch.modules.lpips import LPIPS
    crit = LPIPS("vgg", "0.1")

    rng = np.random.default_rng(SEED)
    out = dict(seed=np.int64(SEED), checksum=np.array(lpips_ref.checksum(vgg_sd, lin_sd)),
               names=np.array([c[0] for c in CASES]))
    for name, H, W, prep, use_mask, crop, same in CASES:
        x = rng.uniform(-0.1, 1.1, (3, H, W)).astype(np.float32)
        y = x.copy() if same else np.clip(x + rng.normal(0, 0.15, x.shape), -0.1, 1.1).astype(np.float32)
        mask = (rng.uniform(size=(H, W)) > 0.25).astype(np.float32) if use_mask else None
        tx, ty = torch.from_numpy(x), torch.from_numpy(y)
        tm = None if mask is None else torch.from_numpy(mask)
        if prep:
            tx, ty = lpips_ref.preprocess(tx, tm, crop), lpips_ref.preprocess(ty, tm, crop)
        # LPIPS.forward, with the per-tap means kept
        with torch.no_grad():
            fx, fy = crit.net(tx), crit.net(ty)
            taps = [float(l((a - b) ** 2).mean()) for a, b, l in zip(fx, fy, crit.lin)]
            value = crit(tx, ty)
        assert tuple(value.shape) == (1, 1, 1, 1)
        out[f"{name}_x"], out[f"{name}_y"] = x, y
        if mask is not None:
            out[f"{name}_mask"] = mask
        out[f"{name}_flags"] = np.array([prep, use_mask, crop, same])
        out[f"{name}_taps"] = np.array(taps, np.float64)
        out[f"{name}_value"] = np.float64(value.item())
    H, W = TOO_SMALL
    x = torch.from_numpy(rng.uniform(0, 1, (3, H, W)).astype(np.float32))
    try:
        crit(x, x)
        err = ""
    except Exception as e:                      # the reference raises inside the network (a zero-size pooling level)
        err = f"{type(e).__name__}: {e}"
    out["too_small_shape"] = np.array(TOO_SMALL)
    out["too_small_error"] = np.array(err)
    np.savez_compressed(os.path.join(HERE, "lpips.npz"), **out)
    print({n: float(out[f"{n}_value"]) for n in out["names"]}, err)


if __name__ == "__main__":
    main()

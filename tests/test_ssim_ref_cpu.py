"""CPU: tests/ssim_ref.py, the float64 restatement of the fused L1 + SSIM loss and of the evaluation metrics with a
per-element fp32 error budget, pinned three ways -- float64 torch autograd of the reference's own formulation (grouped
conv2d, 121 taps), the fp32 golden fixtures the reference produced, and fp32 evaluations in two association orders that
must stay within the budget -- and then csrc/loss.cu and csrc/metrics.cu themselves, run on the emulation build."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "emul"))

import ssim_ref as S  # noqa: E402

SMALL_SHAPES = [(1, 1, 1), (3, 1, 17), (3, 17, 1), (1, 5, 7), (3, 11, 11), (3, 16, 16), (3, 17, 33), (4, 31, 47)]
EMU_SHAPES = [(1, 1, 1), (3, 1, 17), (3, 17, 1), (1, 5, 7), (3, 11, 11), (3, 16, 16), (3, 17, 33)]


# ---- the float64 restatement against torch float64 autograd -----------------------------------------------------------
def _torch_loss64(img, gt, lam):
    """the reference's formulation (utils/loss_utils.py) in float64, with the exact outer product of the fp32 weights"""
    import torch
    import torch.nn.functional as F
    w1 = torch.tensor(S.window_fp32().astype(np.float64))
    Cn = img.shape[0]
    win = torch.outer(w1, w1)[None, None].expand(Cn, 1, 11, 11).contiguous()
    a = torch.tensor(img, dtype=torch.float64, requires_grad=True)
    b = torch.tensor(gt, dtype=torch.float64)
    x, y = a[None], b[None]
    mu1, mu2 = F.conv2d(x, win, padding=5, groups=Cn), F.conv2d(y, win, padding=5, groups=Cn)
    s1 = F.conv2d(x * x, win, padding=5, groups=Cn) - mu1 * mu1
    s2 = F.conv2d(y * y, win, padding=5, groups=Cn) - mu2 * mu2
    s12 = F.conv2d(x * y, win, padding=5, groups=Cn) - mu1 * mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    ssim = (((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s1 + s2 + C2))).mean()
    l1 = (a - b).abs().mean()
    loss = (1 - lam) * l1 + lam * (1 - ssim)
    loss.backward()
    return loss.item(), l1.item(), ssim.item(), a.grad.numpy()


@pytest.mark.parametrize("shape", SMALL_SHAPES)
@pytest.mark.parametrize("kind", ["random", "flat", "unclamped", "corners"])
def test_restatement_matches_float64_autograd(shape, kind):
    img, gt = S.make_contents(kind, *shape, seed=1)
    lam = 0.2
    r = S.loss_reference(img, gt, lam)
    loss, l1, ssim, grad = _torch_loss64(img, gt, lam)
    assert abs(r["loss"] - loss) <= 1e-12 * r["loss_mag"]
    assert abs(r["l1"] - l1) <= 1e-12 * max(r["l1_mag"], 1e-300)
    assert abs(r["ssim"] - ssim) <= 1e-12 * r["ssim_mag"]
    # sign(0) has no derivative: torch's abs' gives 0 at a == b, as loss.cu does
    assert np.all(np.abs(r["grad"] - grad) <= 1e-12 * r["grad_mag"] + 1e-300)


def _torch_metrics64(img, gt, E, mask, x0):
    """render_hierarchy.py's evaluation lines in float64: exposure (right-multiplied, offset column), clamps, crop, mask,
    psnr (utils/image_utils.py, then the mean) and ssim (utils/loss_utils.py)"""
    import torch
    import torch.nn.functional as F
    im = torch.tensor(img, dtype=torch.float64)
    if E is not None:
        Et = torch.tensor(E, dtype=torch.float64)
        im = torch.matmul(im.permute(1, 2, 0), Et[:3, :3]).permute(2, 0, 1) + Et[:3, 3, None, None]
    im = torch.clamp(im, 0.0, 1.0)
    g = torch.clamp(torch.tensor(gt, dtype=torch.float64), 0.0, 1.0)
    m = torch.ones((1,) + img.shape[1:], dtype=torch.float64) if mask is None else torch.tensor(mask, dtype=torch.float64)[None]
    im, g, m = im[..., x0:], g[..., x0:], m[..., x0:]
    out = im.clone()
    im, g = im * m, g * m
    mse = ((im - g) ** 2).view(3, -1).mean(1, keepdim=True)
    psnr = (20 * torch.log10(1.0 / torch.sqrt(mse))).mean()
    w1 = torch.tensor(S.window_fp32().astype(np.float64))
    win = torch.outer(w1, w1)[None, None].expand(3, 1, 11, 11).contiguous()
    x, y = im[None], g[None]
    mu1, mu2 = F.conv2d(x, win, padding=5, groups=3), F.conv2d(y, win, padding=5, groups=3)
    s1 = F.conv2d(x * x, win, padding=5, groups=3) - mu1 * mu1
    s2 = F.conv2d(y * y, win, padding=5, groups=3) - mu2 * mu2
    s12 = F.conv2d(x * y, win, padding=5, groups=3) - mu1 * mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    ssim = (((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s1 + s2 + C2))).mean()
    return out.numpy(), float(psnr), float(ssim)


def metric_inputs(H, W, exposure, mask, seed=0):
    """raw render and target reaching past [0, 1]; a non-symmetric exposure whose offsets push values past 1 and below 0;
    mask None / "binary" / "fractional" """
    rng = np.random.default_rng(seed)
    img = rng.uniform(-0.2, 1.2, (3, H, W)).astype(np.float32)
    gt = rng.uniform(-0.1, 1.1, (3, H, W)).astype(np.float32)
    E = None
    if exposure:
        E = np.zeros((3, 4), np.float32)
        E[:, :3] = np.eye(3) * 0.9 + rng.uniform(-0.2, 0.2, (3, 3))
        E[:, 3] = (0.3, -0.3, 0.05)
    M = None
    if mask == "binary":
        M = (rng.uniform(size=(H, W)) > 0.3).astype(np.float32)
    elif mask == "fractional":
        M = ((rng.uniform(size=(H, W)) > 0.3) * rng.uniform(0.2, 1.0, (H, W))).astype(np.float32)
    return img, gt, E, M


@pytest.mark.parametrize("hwx", [(1, 1, 0), (17, 33, 0), (17, 33, 17), (29, 43, 21)])
@pytest.mark.parametrize("exposure", [False, True])
@pytest.mark.parametrize("mask", [None, "binary", "fractional"])
def test_metrics_restatement_matches_float64_torch(hwx, exposure, mask):
    H, W, x0 = hwx
    img, gt, E, M = metric_inputs(H, W, exposure, mask)
    r = S.metrics_reference(img, gt, E, M, x0)
    out, psnr, ssim = _torch_metrics64(img, gt, E, M, x0)
    assert np.all(np.abs(r["out_img"] - out) <= 1e-12)
    assert abs(r["psnr"] - psnr) <= 1e-12 * abs(psnr) or (np.isinf(psnr) and r["psnr"] == psnr)
    assert abs(r["ssim"] - ssim) <= 1e-12 * r["ssim_mag"]


# ---- the restatement against the reference's fp32 golden fixtures -----------------------------------------------------
@pytest.mark.parametrize("name", ["a", "b", "c"])
def test_restatement_matches_loss_golden(golden_dir, name):
    z = np.load(os.path.join(golden_dir, f"loss_{name}.npz"))
    r = S.loss_reference(z["img"], z["gt"], float(z["lam"]))
    assert abs(r["l1"] - float(z["l1"])) < 1e-6 and abs(r["ssim"] - float(z["ssim"])) < 2e-6
    assert abs(r["loss"] - float(z["loss"])) < 1e-6
    assert np.abs(r["grad"] - z["grad"]).max() < 1e-5 * np.abs(z["grad"]).max()


@pytest.mark.parametrize("i", range(9))
def test_restatement_matches_eval_metrics_golden(golden_dir, i):
    z = np.load(os.path.join(golden_dir, "eval_metrics.npz"))
    exp, msk, crop, _ = (bool(v) for v in z[f"c{i}_flags"])
    raw = z[f"c{i}_raw"]
    x0 = raw.shape[2] // 2 if crop else 0
    r = S.metrics_reference(raw, z[f"c{i}_gt"], z[f"c{i}_E"] if exp else None, z[f"c{i}_mask"] if msk else None, x0)
    assert np.abs(r["out_img"] - z[f"c{i}_image"]).max() <= 1e-6
    pr = float(z[f"c{i}_psnr"])
    if np.isinf(pr):
        assert np.isinf(r["psnr"]) and r["psnr"] > 0
    else:
        assert abs(r["psnr"] - pr) <= 1e-4
    assert abs(r["ssim"] - float(z[f"c{i}_ssim"])) <= 1e-5 * abs(float(z[f"c{i}_ssim"]))


# ---- the budget bounds other fp32 association orders ------------------------------------------------------------------
_WORST = {}


@pytest.mark.parametrize("shape", SMALL_SHAPES + [(3, 64, 48)])
@pytest.mark.parametrize("kind", S.CONTENTS)
@pytest.mark.parametrize("order", ["separable", "2d"])
def test_budget_bounds_fp32_orders(shape, kind, order):
    img, gt = S.make_contents(kind, *shape, seed=2)
    lam = 0.2
    r = S.loss_reference(img, gt, lam)
    k0, k1 = S.loss_coefficients(lam, img.size)
    s, _, g = S.loss_fp32(img, gt, k0, k1, order)
    rs, _ = S.compare(s, r["maps"]["s"].v, S.U * np.broadcast_to(r["maps"]["s"].e, s.shape))
    rg, _ = S.compare(g, r["grad"], r["grad_tol"])
    worst = _WORST.setdefault(order, [0.0, 0.0])
    worst[0], worst[1] = max(worst[0], rs), max(worst[1], rg)
    print(f"\n{order} {shape} {kind}: ssim map {rs:.3g}, grad {rg:.3g}; worst so far {worst}")
    assert rs <= 1.0 and rg <= 1.0


def test_division_check_raises_rather_than_under_bounds():
    B = S.E(np.array([1e-3]), e=np.array([0.06 * 1e-3 / S.U]))
    with pytest.raises(S.DivisionTooInexact):
        S._check_division(B, "B2")
    S._check_division(S.E(np.array([1e-3]), e=np.array([0.04 * 1e-3 / S.U])), "B2")


# ---- the kernels on the emulation build -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """the emulation build of the library's sources (loss.cu among them) plus metrics.cu"""
    from unittest import mock
    import build_emu
    from emu_api import Emu
    with mock.patch.object(build_emu, "SOURCES", build_emu.SOURCES + ["metrics.cu"]):
        return Emu(build_emu.build(str(tmp_path_factory.mktemp("h3dgs_emu_ssim"))))


def loss_kernel_emu(emu, img, gt, k0, k1):
    """forward + backward through the C-ABI -> (sums [2], grad)"""
    from emu_api import aligned, f32, ptr
    Cn, H, W = img.shape
    a, b = f32(img), f32(gt)
    sums = aligned(16, np.float64, (2,))
    maps = aligned(3 * Cn * H * W * 4, np.float32, (3, Cn, H, W))
    emu.check(emu.L.h3dgs_l1_ssim_forward(Cn, H, W, ptr(a), ptr(b), ptr(sums), ptr(maps), None))
    coeffs = f32(np.array([k0, k1], np.float32))
    grad = aligned(Cn * H * W * 4, np.float32, (Cn, H, W))
    emu.check(emu.L.h3dgs_l1_ssim_backward(Cn, H, W, ptr(a), ptr(b), ptr(maps), ptr(coeffs), ptr(grad), None))
    return sums.copy(), grad.copy()


@pytest.mark.parametrize("shape", EMU_SHAPES)
@pytest.mark.parametrize("kind", ["random", "flat", "equal_ulp", "saturated", "unclamped", "corners"])
def test_loss_kernel_on_emulator_within_budget(emu, shape, kind):
    img, gt = S.make_contents(kind, *shape, seed=3)
    lam = 0.2
    r = S.loss_reference(img, gt, lam)
    n = float(img.size)
    k0, k1 = S.loss_coefficients(lam, n)
    sums, grad = loss_kernel_emu(emu, img, gt, k0, k1)
    # the coefficients went in as fp32 roundings of k0, k1: the budget carries four roundings for each
    rl1 = abs(sums[0] / n - r["l1"]) / max(r["l1_sum_tol"], 1e-300) if sums[0] / n != r["l1"] else 0.0
    rss = abs(sums[1] / n - r["ssim"]) / r["ssim_sum_tol"]
    rg, _ = S.compare(grad, r["grad"], r["grad_tol"])
    print(f"\n{shape} {kind}: l1 {rl1:.3g}, ssim {rss:.3g}, grad {rg:.3g}")
    assert np.all(np.isfinite(grad)) and np.isfinite(sums).all()
    assert rl1 <= 1.0 and rss <= 1.0 and rg <= 1.0


def metrics_kernel_emu(emu, img, gt, E, M, x0):
    from emu_api import aligned, f32, ptr
    from h3dgs import _lib
    _, H, W = img.shape
    out = aligned(3 * H * (W - x0) * 4, np.float32, (3, H, W - x0))
    sums = aligned(32, np.float64, (4,))
    counter = aligned(4, np.int32, (1,))
    results = aligned(_lib.EVAL_ROW * 8, np.float64, (1, _lib.EVAL_ROW))
    keep = [f32(img), f32(gt), None if E is None else f32(E), None if M is None else f32(M)]
    emu.check(emu.L.h3dgs_eval_metrics(H, W, ptr(keep[0]), ptr(keep[1]), ptr(keep[2]), ptr(keep[3]), x0, ptr(out),
                                       ptr(sums), None, 0, 0, None, ptr(counter), ptr(results), 1, None))
    return out.copy(), sums.copy(), results[0].copy()


def check_metrics(r, out, sums, row):
    """ratios to the budget of out_img, the four sums, psnr and ssim (inf where a channel is exact)"""
    ro, _ = S.compare(out, r["out_img"], r["out_img_tol"])
    rsum = 0.0
    for k in range(4):
        d = abs(sums[k] - r["sums"][k])
        rsum = max(rsum, 0.0 if d == 0 else d / r["sums_tol"][k])
    exact = r["sums"][:3] == 0
    if exact.any():
        assert np.isinf(row[0]) and row[0] > 0 and np.all(sums[:3][exact] == 0)
        rp = 0.0
    else:
        rp = abs(row[0] - r["psnr"]) / r["psnr_tol"] if row[0] != r["psnr"] else 0.0
    rs = abs(row[1] - r["ssim"]) / r["ssim_tol"] if row[1] != r["ssim"] else 0.0
    return dict(out_img=ro, sums=rsum, psnr=rp, ssim=rs)


@pytest.mark.parametrize("hwx", [(1, 1, 0), (17, 33, 0), (17, 33, 16), (17, 33, 17), (17, 33, 32)])
@pytest.mark.parametrize("exposure", [False, True])
@pytest.mark.parametrize("mask", [None, "binary", "fractional"])
def test_metrics_kernel_on_emulator_within_budget(emu, hwx, exposure, mask):
    H, W, x0 = hwx
    img, gt, E, M = metric_inputs(H, W, exposure, mask, seed=4)
    r = S.metrics_reference(img, gt, E, M, x0)
    out, sums, row = metrics_kernel_emu(emu, img, gt, E, M, x0)
    ratios = check_metrics(r, out, sums, row)
    print(f"\n{hwx} exposure={exposure} mask={mask}: {ratios}")
    assert all(v <= 1.0 for v in ratios.values()), ratios

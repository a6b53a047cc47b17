"""CPU: train_post's objective (exposure, clamp, alpha mask, L1 + SSIM) as csrc/loss.cu's post-loss kernels evaluate it.
tests/post_loss_ref.py restates it; the restatement is pinned against float64 torch autograd of the reference's own
composition (matmul from the right, clamp, mask, grouped conv2d SSIM), and then the kernels, run on the emulation build,
must stay within its per-element budget, take the same clamp decisions, equal h3dgs_l1_ssim_* bit for bit without
exposure and mask, and match tests/golden/post_loss.npz, which the reference's render_post and loss lines produced."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "emul"))

import post_loss_ref as R  # noqa: E402
import ssim_ref as S  # noqa: E402

SHAPES = [(1, 1), (1, 17), (17, 1), (11, 11), (16, 16), (17, 33)]


# ---- torch's clamp backward, and the float64 composition ---------------------------------------------------------------
def test_torch_clamp_backward_passes_both_ends():
    """what the kernels' [0 <= y <= 1] restates: torch's clamp(0, 1) passes the gradient at exactly 0 and 1"""
    import torch
    f = np.float32
    vals = [f(0), f(1), np.nextafter(f(0), f(1)), np.nextafter(f(0), f(-1)), np.nextafter(f(1), f(0)),
            np.nextafter(f(1), f(2)), f(-0.5), f(1.5)]
    for dt in (torch.float32, torch.float64):
        x = torch.tensor(np.array(vals, np.float64), dtype=dt, requires_grad=True)
        x.clamp(0, 1).sum().backward()
        assert x.grad.tolist() == [1, 1, 1, 0, 1, 0, 0, 0]
    y = np.array(vals, np.float32)
    assert ((y >= 0) & (y <= 1)).tolist() == [True, True, True, False, True, False, False, False]


def _ssim64(x, y, Cn=3):
    import torch
    import torch.nn.functional as F
    w1 = torch.tensor(S.window_fp32().astype(np.float64))
    win = torch.outer(w1, w1)[None, None].expand(Cn, 1, 11, 11).contiguous()
    x, y = x[None], y[None]
    mu1, mu2 = F.conv2d(x, win, padding=5, groups=Cn), F.conv2d(y, win, padding=5, groups=Cn)
    s1 = F.conv2d(x * x, win, padding=5, groups=Cn) - mu1 * mu1
    s2 = F.conv2d(y * y, win, padding=5, groups=Cn) - mu2 * mu2
    s12 = F.conv2d(x * y, win, padding=5, groups=Cn) - mu1 * mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    return (((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s1 + s2 + C2))).mean()


def _torch_post64(img, gt, lam, Ex, M):
    """render_post's exposure and clamp and train_post's loss lines in float64 autograd.  The values of y and a are
    replaced (straight through, gradient unchanged) by the kernels' fp32 y and a, so that the clamp decides on the same
    numbers and the float64 SSIM sees the kernels' a; every derivative is torch's own."""
    import torch
    im = torch.tensor(img, dtype=torch.float64, requires_grad=True)
    y = im
    if Ex is not None:
        Et = torch.tensor(Ex, dtype=torch.float64)
        y = torch.matmul(im.permute(1, 2, 0), Et[:3, :3]).permute(2, 0, 1) + Et[:3, 3, None, None]
    y32, a32, _ = R.staged(img, Ex, M)
    y = y + (torch.tensor(y32, dtype=torch.float64) - y).detach()
    a = torch.clamp(y, 0.0, 1.0)
    if M is not None:
        a = a * torch.tensor(M, dtype=torch.float64)[None]
    a = a + (torch.tensor(a32, dtype=torch.float64) - a).detach()
    g = torch.tensor(gt, dtype=torch.float64)
    l1 = (a - g).abs().mean()
    ssim = _ssim64(a, g)
    loss = (1.0 - lam) * l1 + lam * (1.0 - ssim)
    loss.backward()
    return loss.item(), l1.item(), ssim.item(), im.grad.numpy()


@pytest.mark.parametrize("exposure", R.EXPOSURES)
def test_exposed_fp32_is_the_right_multiplied_exposure(exposure):
    """the pinned fp32 order is within its three roundings of float64 torch.matmul from the right (a transposed or
    left-multiplied exposure is O(0.1) away)"""
    import torch
    img, _, Ex, _ = R.make_inputs(13, 21, exposure, "none", seed=1)
    y32 = R.exposed_fp32(img, Ex)
    if Ex is None:
        assert np.array_equal(y32, img)
        return
    im, Et = torch.tensor(img, dtype=torch.float64), torch.tensor(Ex, dtype=torch.float64)
    y64 = (torch.matmul(im.permute(1, 2, 0), Et[:3, :3]).permute(2, 0, 1) + Et[:3, 3, None, None]).numpy()
    mag = np.stack([sum(np.abs(img[k].astype(np.float64) * float(Ex[k, c])) for k in range(3)) + abs(float(Ex[c, 3]))
                    for c in range(3)])
    assert np.all(np.abs(y32 - y64) <= 3 * S.U * mag * (1 + 1e-6))
    assert np.abs(np.matmul(img.transpose(1, 2, 0), Ex[:3, :3].T).transpose(2, 0, 1) - y64).max() > 1e-2


@pytest.mark.parametrize("shape", [(1, 1), (11, 11), (17, 33)])
@pytest.mark.parametrize("exposure", R.EXPOSURES)
@pytest.mark.parametrize("mask", R.MASKS)
def test_restatement_matches_float64_autograd(shape, exposure, mask):
    img, gt, Ex, M = R.make_inputs(*shape, exposure, mask, seed=2)
    lam = 0.2
    r = R.post_reference(img, gt, lam, Ex, M)
    loss, l1, ssim, grad = _torch_post64(img, gt, lam, Ex, M)
    assert abs(r["loss"] - loss) <= 1e-12 * r["loss_mag"]
    assert abs(r["l1"] - l1) <= 1e-12 * max(r["l1_mag"], 1e-300)
    assert abs(r["ssim"] - ssim) <= 1e-12 * r["ssim_mag"]
    assert np.all(np.abs(r["grad"] - grad) <= 1e-12 * r["grad_mag"] + 1e-300)


@pytest.mark.parametrize("exposure", R.EXPOSURES)
def test_clamp_edge_inputs_hit_the_edges(exposure):
    img, gt, Ex = R.clamp_edge_inputs(9, 11, exposure)
    y = R.exposed_fp32(img, Ex)
    f = np.float32
    for t in (f(0), f(1)):
        assert (y == t).sum() >= 1, (exposure, t)
        assert ((y < t) & (y > t - 1e-6)).sum() >= 1 and ((y > t) & (y < t + 1e-6)).sum() >= 1
    if Ex is None:
        for t in (np.nextafter(f(0), f(-1)), np.nextafter(f(1), f(2)), np.nextafter(f(0), f(1)), np.nextafter(f(1), f(0))):
            assert (y == t).sum() >= 1


# ---- the kernels on the emulation build --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    import build_emu
    from emu_api import Emu
    return Emu(build_emu.build(str(tmp_path_factory.mktemp("h3dgs_emu_post"))))


def post_kernel_emu(emu, img, gt, Ex, M, k0, k1):
    """h3dgs_post_loss_forward + _backward -> (sums [2], maps, grad)"""
    from emu_api import aligned, f32, ptr
    _, H, W = img.shape
    keep = [f32(img), f32(gt), None if Ex is None else f32(Ex), None if M is None else f32(M.reshape(H, W))]
    sums = aligned(16, np.float64, (2,))
    maps = aligned(9 * H * W * 4, np.float32, (3, 3, H, W))
    emu.check(emu.L.h3dgs_post_loss_forward(H, W, ptr(keep[0]), ptr(keep[1]), ptr(keep[2]), ptr(keep[3]), ptr(sums),
                                            ptr(maps), None))
    coeffs = f32(np.array([k0, k1], np.float32))
    grad = aligned(3 * H * W * 4, np.float32, (3, H, W))
    emu.check(emu.L.h3dgs_post_loss_backward(H, W, ptr(keep[0]), ptr(keep[1]), ptr(keep[2]), ptr(keep[3]), ptr(maps),
                                             ptr(coeffs), ptr(grad), None))
    return sums.copy(), maps.copy(), grad.copy()


def check_post(r, sums, grad, n):
    """ratios to the budget of L1, SSIM and dL/dimg"""
    rl1 = abs(sums[0] / n - r["l1"]) / max(r["l1_sum_tol"], 1e-300) if sums[0] / n != r["l1"] else 0.0
    rss = abs(sums[1] / n - r["ssim"]) / r["ssim_sum_tol"] if sums[1] / n != r["ssim"] else 0.0
    rg, _ = R.compare(grad, r["grad"], r["grad_tol"])
    assert np.all(np.isfinite(grad)) and np.isfinite(sums).all()
    return dict(l1=rl1, ssim=rss, grad=rg)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("exposure", R.EXPOSURES)
@pytest.mark.parametrize("mask", ["none", "binary", "half", "fractional", "zero"])
def test_post_kernel_on_emulator_within_budget(emu, shape, exposure, mask):
    img, gt, Ex, M = R.make_inputs(*shape, exposure, mask, seed=3)
    lam = 0.2
    r = R.post_reference(img, gt, lam, Ex, M)
    n = float(img.size)
    k0, k1 = S.loss_coefficients(lam, n)
    sums, _, grad = post_kernel_emu(emu, img, gt, Ex, M, k0, k1)
    ratios = check_post(r, sums, grad, n)
    print(f"\n{shape} {exposure} {mask}: {ratios}")
    assert all(v <= 1.0 for v in ratios.values()), ratios


@pytest.mark.parametrize("content", ["saturated", "flat"])
@pytest.mark.parametrize("lam", [0.0, 0.2, 1.0])
def test_post_kernel_on_emulator_contents_and_lambdas(emu, content, lam):
    img, gt, Ex, M = R.make_inputs(17, 33, "offset", "binary", content, seed=4)
    r = R.post_reference(img, gt, lam, Ex, M)
    n = float(img.size)
    k0, k1 = S.loss_coefficients(lam, n)
    sums, _, grad = post_kernel_emu(emu, img, gt, Ex, M, k0, k1)
    ratios = check_post(r, sums, grad, n)
    assert all(v <= 1.0 for v in ratios.values()), ratios


@pytest.mark.parametrize("exposure", R.EXPOSURES)
@pytest.mark.parametrize("mask", ["none", "fractional"])
def test_post_kernel_clamp_decisions_at_the_edges(emu, exposure, mask):
    """y exactly at 0 and 1 and one ulp either side: the kernels decide as the restatement (a wrong decision moves a
    gradient by |dL/da|, far outside the budget); without exposure the decision is visible directly: dL/dimg is 0
    exactly where the clamp blocks, and nonzero where it passes and mask * dL/da is"""
    img, gt, Ex = R.clamp_edge_inputs(17, 19, exposure, seed=5)
    M = R.make_mask(mask, 17, 19, np.random.default_rng(6))
    if M is not None:
        M[0:2] = 1.0                                           # the edge pixels stay unmasked
    lam = 0.2
    r = R.post_reference(img, gt, lam, Ex, M)
    n = float(img.size)
    k0, k1 = S.loss_coefficients(lam, n)
    sums, _, grad = post_kernel_emu(emu, img, gt, Ex, M, k0, k1)
    ratios = check_post(r, sums, grad, n)
    assert all(v <= 1.0 for v in ratios.values()), ratios
    if Ex is None:
        live = np.abs(r["grad_a"]) > 2 * np.abs(r["grad_tol"]) + 1e-30
        if M is not None:
            live &= M[None] != 0
        assert np.all(grad[~r["keep"]] == 0.0)
        assert np.all(grad[r["keep"] & live] != 0.0)


@pytest.mark.parametrize("shape", [(1, 1), (16, 16), (17, 33)])
@pytest.mark.parametrize("content", ["in_range", "unclamped"])
def test_without_exposure_and_mask_equals_l1_ssim_bitwise(emu, shape, content):
    """no exposure, no mask: the post loss is the fused L1 + SSIM loss of clamp(img), bit for bit, and its gradient that
    loss's gradient where 0 <= img <= 1 and 0 elsewhere"""
    from emu_api import aligned, f32, ptr
    H, W = shape
    rng = np.random.default_rng(7)
    lo, hi = (0.0, 1.0) if content == "in_range" else (-0.3, 1.3)
    img = rng.uniform(lo, hi, (3, H, W)).astype(np.float32)
    if content == "in_range":
        img.reshape(-1)[:2] = (0.0, 1.0)
    gt = rng.uniform(0, 1, (3, H, W)).astype(np.float32)
    k0, k1 = S.loss_coefficients(0.2, float(img.size))
    sums, maps, grad = post_kernel_emu(emu, img, gt, None, None, k0, k1)
    a = f32(np.clip(img, 0, 1))
    b = f32(gt)
    sums2 = aligned(16, np.float64, (2,))
    maps2 = aligned(9 * H * W * 4, np.float32, (3, 3, H, W))
    emu.check(emu.L.h3dgs_l1_ssim_forward(3, H, W, ptr(a), ptr(b), ptr(sums2), ptr(maps2), None))
    coeffs = f32(np.array([k0, k1], np.float32))
    grad2 = aligned(3 * H * W * 4, np.float32, (3, H, W))
    emu.check(emu.L.h3dgs_l1_ssim_backward(3, H, W, ptr(a), ptr(b), ptr(maps2), ptr(coeffs), ptr(grad2), None))
    assert np.array_equal(sums.view(np.uint64), sums2.view(np.uint64))
    assert np.array_equal(maps.view(np.uint32), maps2.view(np.uint32))
    ref = np.where((img >= 0) & (img <= 1), grad2, np.float32(0))
    assert np.array_equal(grad.view(np.uint32), ref.view(np.uint32))


# ---- against the reference's own render_post and loss lines -------------------------------------------------------------
def _golden_cases(golden_dir):
    z = np.load(os.path.join(golden_dir, "post_loss.npz"))
    return z, int(z["cases"])


@pytest.mark.parametrize("i", range(8))
def test_post_kernel_matches_the_reference(emu, golden_dir, i):
    z, n_cases = _golden_cases(golden_dir)
    assert i < n_cases
    exp, msk = (bool(v) for v in z[f"c{i}_flags"])
    raw, gt = z[f"c{i}_raw"], z[f"c{i}_gt"]
    Ex = z[f"c{i}_E"] if exp else None
    M = z[f"c{i}_mask"]
    lam = float(z["lam"])
    n = float(raw.size)
    k0, k1 = S.loss_coefficients(lam, n)
    sums, _, grad = post_kernel_emu(emu, raw, gt, Ex, M, k0, k1)
    l1, ssim = sums[0] / n, sums[1] / n
    loss = (1 - lam) * l1 + lam * (1 - ssim)
    assert abs(l1 - float(z[f"c{i}_l1"])) < 1e-6
    assert abs(loss - float(z[f"c{i}_loss"])) < 1e-6
    ref = z[f"c{i}_grad"]
    assert np.abs(grad - ref).max() <= 1e-5 * max(np.abs(ref).max(), 1e-30)
    # the restatement agrees with the reference too (its own decisions, clamp included)
    r = R.post_reference(raw, gt, lam, Ex, M)
    assert np.abs(r["grad"] - ref).max() <= 1e-5 * max(np.abs(ref).max(), 1e-30)

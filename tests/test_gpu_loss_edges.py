"""GPU: the fused L1 + SSIM loss (csrc/loss.cu), the evaluation metrics (csrc/metrics.cu) and the bench step's L1 loss
(csrc/l1_loss.cu), element by element against the float64 restatement of tests/ssim_ref.py and its derived fp32 budget,
at frames smaller than the window's halo, single rows and columns, the 16-pixel tile edge +-1 and 1080p; on flat,
nearly equal, saturated and unclamped contents; for every way the three outputs can be differentiated; inside a CUDA
graph capture that makes the loss's first call; and, for the metrics, the crop and mask invariants."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import ssim_ref as S  # noqa: E402

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1, 1), (3, 1, 17), (3, 17, 1), (1, 5, 7), (3, 11, 11), (3, 16, 16), (3, 17, 33), (4, 31, 47), (3, 64, 48),
          (3, 270, 480)]
_WORST = {}
_PARTS = {}


def _report(key, **ratios):
    w = _WORST.setdefault(key, {})
    for k, v in ratios.items():
        w[k] = max(w.get(k, 0.0), v)
    print(f"\n[{key}] " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items()) + "; worst " +
          ", ".join(f"{k} {v:.3g}" for k, v in w.items()))


def _parts(shape, kind):
    key = (shape, kind)
    if key not in _PARTS:
        _PARTS.clear()
        img, gt = S.make_contents(kind, *shape, seed=5)
        _PARTS[key] = (img, gt, S.loss_parts(img, gt))
    return _PARTS[key]


def _scalar_ratio(got, ref, tol):
    d = abs(float(got) - ref)
    if not np.isfinite(float(got)):
        return np.inf
    return 0.0 if d == 0 else d / tol


def _run(img, gt, lam, use="loss", make=None):
    """fused_l1_ssim on the device, differentiated as `use` says -> (loss, l1, ssim, grad) as numpy"""
    import torch
    from h3dgs.loss import fused_l1_ssim
    x = torch.tensor(img, device="cuda") if make is None else make(img)
    x.requires_grad_(True)
    g = torch.tensor(gt, device="cuda")
    if tuple(x.shape) != tuple(g.shape):
        g = g.reshape(x.shape)
    loss, l1, ssim = fused_l1_ssim(x, g, lam)
    obj = {"loss": lambda: loss, "l1": lambda: l1, "ssim": lambda: ssim, "loss+0.3ssim": lambda: loss + 0.3 * ssim,
           "3.7loss": lambda: 3.7 * loss}[use]()
    obj.backward()
    return float(loss), float(l1), float(ssim), x.grad


UPSTREAM = {"loss": (1.0, 0.0, 0.0), "l1": (0.0, 1.0, 0.0), "ssim": (0.0, 0.0, 1.0), "loss+0.3ssim": (1.0, 0.0, 0.3),
            "3.7loss": (3.7, 0.0, 0.0)}


def _check(img, gt, lam, use, grad, loss, l1, ssim, key, parts=None):
    gl, g1, gs = UPSTREAM[use]
    r = S.loss_reference(img, gt, lam, g_loss=gl, g_l1=g1, g_ssim=gs, parts=parts)
    g = grad.detach().reshape(img.shape).cpu().numpy()
    assert np.all(np.isfinite(g))
    rg, _ = S.compare(g, r["grad"], r["grad_tol"])
    rl = _scalar_ratio(loss, r["loss"], r["loss_tol"])
    r1 = _scalar_ratio(l1, r["l1"], r["l1_tol"])
    rs = _scalar_ratio(ssim, r["ssim"], r["ssim_tol"])
    _report(key, grad=rg, loss=rl, l1=r1, ssim=rs)
    assert rg <= 1.0 and rl <= 1.0 and r1 <= 1.0 and rs <= 1.0, (rg, rl, r1, rs)


@pytest.mark.parametrize("lam", [0.0, 0.2, 1.0])
@pytest.mark.parametrize("kind", S.CONTENTS)
@pytest.mark.parametrize("shape", SHAPES)
def test_loss_within_budget(shape, kind, lam):
    img, gt, parts = _parts(shape, kind)
    loss, l1, ssim, grad = _run(img, gt, lam)
    _check(img, gt, lam, "loss", grad, loss, l1, ssim, f"{shape}", parts)


def test_loss_full_hd_within_budget():
    img, gt = S.make_contents("random", 3, 1080, 1920, seed=6)
    loss, l1, ssim, grad = _run(img, gt, 0.2)
    _check(img, gt, 0.2, "loss", grad, loss, l1, ssim, "1080p")


@pytest.mark.parametrize("kind", ["random", "equal", "equal_ulp", "saturated", "corners"])
@pytest.mark.parametrize("shape", [(3, 17, 33), (4, 31, 47), (3, 64, 48)])
def test_lambda_zero_gradient_is_the_sign_bitwise_and_repeats(shape, kind):
    import torch
    from h3dgs.loss import fused_l1_ssim
    img, gt = S.make_contents(kind, *shape, seed=7)
    img[0, 0, 0], gt[0, 0, 0] = np.float32(0.0), np.float32(-0.0)       # +0 vs -0: equal, no gradient
    x = torch.tensor(img, device="cuda", requires_grad=True)
    g = torch.tensor(gt, device="cuda")
    loss = fused_l1_ssim(x, g, 0.0)[0]
    loss.backward(retain_graph=True)
    first = x.grad.clone()
    x.grad = None
    loss.backward()
    assert torch.equal(first.view(torch.int32), x.grad.view(torch.int32))
    # the coefficient as loss.py forms it in fp32: (g_loss (1 - 0) + 0) / N
    one = torch.ones((), dtype=torch.float32)
    coeff = float(((one * (1.0 - 0.0) + torch.zeros(())) / float(img.size)).item())
    sgn = np.sign(img.astype(np.float64) - gt.astype(np.float64)).astype(np.float32)
    want = (np.float32(coeff) * sgn).astype(np.float32)
    want[sgn == 0] = 0.0
    got = first.cpu().numpy()
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("use", list(UPSTREAM))
def test_every_backward_use(use):
    img, gt = S.make_contents("flat", 3, 37, 53, seed=8)
    loss, l1, ssim, grad = _run(img, gt, 0.2, use)
    _check(img, gt, 0.2, use, grad, loss, l1, ssim, f"use {use}")


def _batched(img):
    import torch
    return torch.tensor(img, device="cuda")[None].clone()


def _right_half(img):
    import torch
    big = torch.rand((img.shape[0], img.shape[1], 2 * img.shape[2]), device="cuda")
    big[..., img.shape[2]:] = torch.tensor(img, device="cuda")
    return big[..., img.shape[2]:].detach()


def _permuted(img):
    import torch
    return torch.tensor(np.ascontiguousarray(img.transpose(1, 2, 0)), device="cuda").permute(2, 0, 1)


@pytest.mark.parametrize("layout", ["batched", "right_half", "permuted"])
def test_input_layouts(layout):
    import torch
    from h3dgs.loss import fused_l1_ssim
    img, gt = S.make_contents("random", 3, 33, 40, seed=9)
    make = {"batched": _batched, "right_half": _right_half, "permuted": _permuted}[layout]
    x = make(img).requires_grad_(True)
    assert layout == "batched" or not x.is_contiguous()
    g = torch.tensor(gt, device="cuda").reshape(x.shape)
    loss, l1, ssim = fused_l1_ssim(x, g, 0.2)
    loss.backward()
    assert x.grad.shape == x.shape
    _check(img, gt, 0.2, "loss", x.grad, float(loss), float(l1), float(ssim), f"layout {layout}")


_CAPTURE = r"""
import sys
import numpy as np
import torch
sys.path[:0] = [sys.argv[2], sys.argv[2] + "/hierarchical-3d-gaussians_b200"]
from h3dgs.loss import fused_l1_ssim
z = np.load(sys.argv[1])
x = torch.zeros(z["img0"].shape, device="cuda", requires_grad=True)
g = torch.zeros(z["img0"].shape, device="cuda")
with torch.no_grad():
    x.copy_(torch.tensor(z["img0"])); g.copy_(torch.tensor(z["gt0"]))
torch.cuda.synchronize()
graph = torch.cuda.CUDAGraph()
with torch.cuda.graph(graph):                       # the first call of the loss in this process
    loss = fused_l1_ssim(x, g, 0.2)[0]
    grad, = torch.autograd.grad(loss, x)
with torch.no_grad():
    x.copy_(torch.tensor(z["img"])); g.copy_(torch.tensor(z["gt"]))
graph.replay()
torch.cuda.synchronize()
gl, gg = loss.item(), grad.cpu().numpy()
x2 = torch.tensor(z["img"], device="cuda", requires_grad=True)
l2 = fused_l1_ssim(x2, torch.tensor(z["gt"], device="cuda"), 0.2)[0]
l2.backward()
np.savez(sys.argv[1] + ".out.npz", graph_loss=gl, graph_grad=gg, eager_loss=l2.item(), eager_grad=x2.grad.cpu().numpy())
"""


def test_first_call_inside_a_graph_capture(tmp_path):
    img0, gt0 = S.make_contents("random", 3, 45, 70, seed=10)
    img, gt = S.make_contents("flat", 3, 45, 70, seed=11)
    path = str(tmp_path / "capture.npz")
    np.savez(path, img0=img0, gt0=gt0, img=img, gt=gt)
    r = subprocess.run([sys.executable, "-c", _CAPTURE, path, ROOT], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    z = np.load(path + ".out.npz")
    assert np.array_equal(z["graph_grad"].view(np.int32), z["eager_grad"].view(np.int32))
    ref = S.loss_reference(img, gt, 0.2)
    rl = _scalar_ratio(float(z["graph_loss"]), ref["loss"], ref["loss_tol"])
    rg, _ = S.compare(z["graph_grad"], ref["grad"], ref["grad_tol"])
    _report("capture", loss=rl, grad=rg)
    assert rl <= 1.0 and rg <= 1.0


# ---- metrics.cu --------------------------------------------------------------------------------------------------------
def _metrics(img, gt, E, M, x0):
    """h3dgs_eval_metrics through h3dgs.evaluate._metrics -> (out_img, sums, row) as numpy"""
    import torch
    from h3dgs import _lib
    from h3dgs.evaluate import _metrics as run
    _, H, W = img.shape
    t = lambda a: None if a is None else torch.tensor(np.ascontiguousarray(a), device="cuda")
    out = torch.zeros((3, H, W - x0), device="cuda")
    sums = torch.zeros(4, dtype=torch.float64, device="cuda")
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    results = torch.zeros((1, _lib.EVAL_ROW), dtype=torch.float64, device="cuda")
    run(_lib.lib(), H, W, t(img), t(gt), t(E), t(M), x0, out, sums, counter, results,
        torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out.cpu().numpy(), sums.cpu().numpy(), results[0].cpu().numpy()


METRIC_CASES = [(1, 1, 0), (17, 33, 0), (17, 33, 16), (17, 33, 17), (17, 33, 32), (64, 48, 24), (270, 480, 240)]


@pytest.mark.parametrize("mask", [None, "binary", "fractional"])
@pytest.mark.parametrize("exposure", [False, True])
@pytest.mark.parametrize("hwx", METRIC_CASES)
def test_metrics_within_budget_and_invariant(hwx, exposure, mask):
    from test_ssim_ref_cpu import check_metrics, metric_inputs
    H, W, x0 = hwx
    img, gt, E, M = metric_inputs(H, W, exposure, mask, seed=12)
    r = S.metrics_reference(img, gt, E, M, x0)
    out, sums, row = _metrics(img, gt, E, M, x0)
    ratios = check_metrics(r, out, sums, row)
    _report(f"metrics {hwx}", **ratios)
    assert all(v <= 1.0 for v in ratios.values()), ratios
    rng = np.random.default_rng(13)
    img2, gt2 = img.copy(), gt.copy()
    img2[..., :x0] = rng.uniform(-1, 2, img2[..., :x0].shape)                 # left of the crop
    gt2[..., :x0] = rng.uniform(-1, 2, gt2[..., :x0].shape)
    if M is not None:
        off = np.broadcast_to(M == 0, img.shape)                              # masked out
        img2[off] = rng.uniform(-1, 2, int(off.sum()))
        gt2[off] = rng.uniform(-1, 2, int(off.sum()))
    out2, sums2, row2 = _metrics(img2, gt2, E, M, x0)
    # the per-tile partial sums are bitwise the same; only the order of their double atomics varies from run to run
    n_cta = 3 * ((W - x0 + 15) // 16) * ((H + 15) // 16)
    assert np.all(np.abs(sums2 - sums) <= n_cta * 2.0 ** -52 * np.abs(sums))
    assert np.all(np.abs(row2[:2] - row[:2]) <= n_cta * 2.0 ** -50 * np.abs(row[:2]))
    if M is None:
        assert np.array_equal(out2.view(np.int32), out.view(np.int32))


@pytest.mark.parametrize("hwx", [(17, 33, 16), (17, 33, 17), (64, 48, 24)])
def test_metrics_crop_edge_and_exact_channel(hwx):
    H, W, x0 = hwx
    rng = np.random.default_rng(14)
    img = rng.uniform(0, 1, (3, H, W)).astype(np.float32)
    gt = img.copy()
    _, sums, row = _metrics(img, gt, None, None, x0)
    assert np.all(sums[:3] == 0) and np.isinf(row[0]) and row[0] > 0
    left = gt.copy()
    left[1, H // 2, x0 - 1] += 0.5                                            # one column left of the crop: not counted
    _, sums, row = _metrics(img, left, None, None, x0)
    assert np.all(sums[:3] == 0) and np.isinf(row[0])
    at = gt.copy()
    at[1, H // 2, x0] += 0.5                                                  # the crop's first column: counted
    _, sums, row = _metrics(img, at, None, None, x0)
    assert sums[0] == 0 and sums[2] == 0 and sums[1] > 0


# ---- l1_loss.cu ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shard", [(1, 0), (3, 1), (3, 2)])
@pytest.mark.parametrize("W", [64, 65, 66, 67])
def test_l1_loss_grad(W, shard):
    import torch
    from h3dgs import _lib
    C_, H = 3, 70
    rng = np.random.default_rng(15 + W)
    img = rng.uniform(-0.2, 1.2, (C_, H, W)).astype(np.float32)
    gt = rng.uniform(-0.2, 1.2, (C_, H, W)).astype(np.float32)
    eq = rng.uniform(size=img.shape) < 0.2
    gt[eq] = img[eq]
    img[0, 0, :4], gt[0, 0, :4] = (0.0, -0.0, 0.0, -0.0), (-0.0, 0.0, 0.0, -0.0)
    scale = np.float32(1.0 / img.size)
    a, b = torch.tensor(img, device="cuda"), torch.tensor(gt, device="cuda")
    grad = torch.full(img.shape, 7.0, device="cuda")
    loss = torch.zeros(1, dtype=torch.float64, device="cuda")
    sc, si = shard
    _lib.check(_lib.lib().h3dgs_l1_loss_grad(C_, H, W, a.data_ptr(), b.data_ptr(), float(scale), sc, si, grad.data_ptr(),
                                             loss.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    g = grad.cpu().numpy()
    own = ((np.arange(H) >> 4) % sc == si)[None, :, None] if sc > 1 else np.ones((1, H, 1), bool)
    own = np.broadcast_to(own, img.shape)
    assert np.all(g[~own] == 7.0)
    d = img.astype(np.float64) - gt.astype(np.float64)
    want = np.where(d > 0, scale, np.where(d < 0, -scale, np.float32(0.0))).astype(np.float32)
    assert np.array_equal(g[own].view(np.int32), want[own].view(np.int32))
    ad = np.abs(d[own])
    n = ad.size
    assert abs(float(loss.item()) - ad.sum()) <= n * S.U * ad.sum()

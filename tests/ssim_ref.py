"""Float64 restatement of the fused L1 + SSIM loss (csrc/loss.cu) and of the evaluation metrics (csrc/metrics.cu), with
a per-element error budget for their fp32 evaluation.

LOSS.  utils/loss_utils.py: l1_loss = mean |img - gt|; ssim with an 11-tap Gaussian window, sigma 1.5, zero padding
(conv2d padding=5, groups = channels), C1 = 0.01^2, C2 = 0.03^2, size_average=True; combined as train_post.py does:
loss = (1 - lambda) L1 + lambda (1 - SSIM).  The gradient with respect to img is the closed form loss.cu documents:
  d(sum s)/d img = G*(ds/dmu1) + 2 img G*(ds/dE11) + gt G*(ds/dE12),
  ds/dmu1 = 2 mu2 (A2 - A1) / (B1 B2) - s (2 mu1 / B1 - 2 mu1 / B2), ds/dE11 = -s / B2, ds/dE12 = 2 A1 / (B1 B2),
weighted by k0 = (g_loss (1 - lambda) + g_l1) / N for sign(img - gt) and k1 = (g_ssim - g_loss lambda) / N for the SSIM
sum, as h3dgs/loss.py forms them.

METRICS.  render_hierarchy.py's evaluation as metrics.cu states it: exposure applied from the right with its offset
column (out[c] = sum_k img[k] E[k][c] + E[c][3]), clamp of both images to [0, 1], the train_test_exp crop (columns
x0..W-1, SSIM's zero padding at the crop border), the alpha mask applied to both images after the clamp, PSNR per
channel (-10 log10 mse) averaged over the three channels, and SSIM averaged over the cropped frame.

WEIGHTS.  `window_fp32` reproduces the kernels' fp32 1-D weights bit for bit: exp in double, rounded to float, summed in
float in order, each divided in float.  Everything after that is float64.  The reference's 2-D window is the fp32
rounding of the outer product w w^T; the separable form here uses the exact products (exact in float64), so the two
windows differ by at most one fp32 rounding per 2-D weight.

ERROR BUDGET.  Values carry chain_ref.E: a float64 value, its magnitude chain a (the formula on absolute values, the
scale of the float64 comparisons) and a running bound e of the error of an fp32 evaluation, in units of U = 2^-24.
How each operation adds to the bound:
  - inputs (img, gt, exposure, mask, the weights as the kernels hold them) are exact; C1 and C2 carry three roundings
    (0.01f, its square, and the rounding of the square);
  - each convolution pass is one flat sum of 11 products: a tap adds one rounding per product (two for w a a, w a b)
    and the sum adds U m per addition, m the sum of |terms|, in whatever order the terms are associated;
  - the variance subtractions s1 = E11 - mu1^2, s2, s12, and A1, A2, B1 = mu1^2 + mu2^2 + C1, B2 = s1 + s2 + C2 are
    flat sums whose m carries the magnitudes of everything they cancel: this is where a flat, nearly equal pair of
    images loses its digits, and B2 ~ C2 = 9e-4 divides them;
  - s, the three derivative maps ds/dmu1, ds/dE11, ds/dE12: one rounding per product and per reciprocal; a division
    a / b adds (e_a + |a / b| e_b) / |b| + |a / b|, which is first order in U e_b / |b|.  Every B1 and B2 divided by
    is checked to have U e_B / |B| <= 0.05, and `DivisionTooInexact` is raised otherwise, so the bound never silently
    under-bounds;
  - the convolution of the three maps with the window: two passes as above;
  - the final c0 + 2 a c1 + b c2: a flat sum of three terms (the doubling is exact);
  - the L1 term k0 sign(a - b) is exact apart from the fp32 rounding of k0 in loss.py: four roundings (1 - lambda,
    the product, the sum, the division), and k1 carries four as well;
  - the scalar outputs: each CTA sums its 256 per-pixel values with an fp32 tree of 8 levels (8 U sum |values|), the
    CTA sums go to a double by atomics (n_cta 2^-53 sum |values|), and the returned scalars are rounded to fp32 once.
  The metrics kernel sums the squared errors and the SSIM values in double: d = a - b is one fp32 rounding, d^2 and
  the sums are double.
The kernels contract some products into FMAs, which only removes roundings.
"""
import math

import numpy as np

from chain_ref import E, U, _sum, compare  # noqa: F401  (compare: re-exported for the tests)

RADIUS, TAPS = 5, 11
C1_64, C2_64 = 0.01 ** 2, 0.03 ** 2
CTA_LEVELS = 8                   # 256 values per CTA: 5 shuffle levels + 3 across the 8 warps
TILE = 16


class DivisionTooInexact(ValueError):
    """a denominator's error bound is not small against its value: the first-order division bound would not hold"""


def window_fp32():
    """the kernels' 1-D weights, bit for bit (make_window in metrics.cu / loss.cu)"""
    w = np.array([np.float32(math.exp(-float((x - RADIUS) * (x - RADIUS)) / (2.0 * 1.5 * 1.5))) for x in range(TAPS)],
                 np.float32)
    s = np.float32(0.0)
    for x in range(TAPS):
        s = np.float32(s + w[x])
    return (w / s).astype(np.float32)


def _shift(x, d, axis):
    """y[i] = x[i + d] along axis, 0 outside"""
    x = np.asarray(x)
    out = np.zeros_like(x)
    n = x.shape[axis]
    if abs(d) >= n:
        return out
    src, dst = [slice(None)] * x.ndim, [slice(None)] * x.ndim
    if d >= 0:
        src[axis], dst[axis] = slice(d, n), slice(0, n - d)
    else:
        src[axis], dst[axis] = slice(0, n + d), slice(-d, n)
    out[tuple(dst)] = x[tuple(src)]
    return out


def _shift_e(x, d, axis):
    e = np.broadcast_to(np.asarray(x.e, np.float64), x.v.shape)
    return E(_shift(x.v, d, axis), _shift(x.a, d, axis), _shift(x.m, d, axis), _shift(e, d, axis))


def _twice(x):
    """2 x: exact in fp32"""
    return E(2.0 * x.v, 2.0 * x.a, 2.0 * x.m, 2.0 * x.e)


def _const_sq(v):
    return E(v, e=3.0 * abs(v))


def _conv(factors, w):
    """the window applied to the product of `factors` (E maps [..., H, W]), zero padded: a horizontal then a vertical
    pass, each one flat sum of 11 products"""
    h = None
    for k in range(TAPS):
        t = E(float(w[k]))
        for f in factors:
            t = t * _shift_e(f, k - RADIUS, -1)
        h = t if h is None else h + t
    o = None
    for k in range(TAPS):
        t = E(float(w[k])) * _shift_e(h, k - RADIUS, -2)
        o = t if o is None else o + t
    return o


def _check_division(B, name):
    r = U * np.asarray(B.e) / np.abs(B.v)
    if np.any(r > 0.05):
        raise DivisionTooInexact(f"{name}: U e / |B| reaches {float(r.max()):.3g} (> 0.05)")


def _diff(a, b):
    """a - b as one fp32 rounding of the (inexact) operands"""
    v = a.v - b.v
    return E(v, a.a + b.a, None, a.e + b.e + np.abs(v))


def ssim_terms(a, b, w, order="loss"):
    """-> dict of E maps: s (the SSIM map), and for order "loss" the three derivative maps dm, d11, d12.
    order "loss": s = A1 A2 (1/B1) (1/B2) as loss.cu; order "metrics": s = (A1 A2) / (B1 B2) as metrics.cu."""
    mu1, mu2 = _conv([a], w), _conv([b], w)
    e11, e22, e12 = _conv([a, a], w), _conv([b, b], w), _conv([a, b], w)
    C1, C2 = _const_sq(C1_64), _const_sq(C2_64)
    mu1sq, mu2sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1, s2, s12 = e11 - mu1sq, e22 - mu2sq, e12 - mu12
    A1, A2 = _twice(mu12) + C1, _twice(s12) + C2
    B1, B2 = mu1sq + mu2sq + C1, s1 + s2 + C2
    _check_division(B1, "B1")
    _check_division(B2, "B2")
    out = dict(mu1=mu1, mu2=mu2)
    if order == "metrics":
        B12 = B1 * B2
        _check_division(B12, "B1 B2")
        out["s"] = (A1 * A2) / B12
        return out
    iB1, iB2 = 1.0 / B1, 1.0 / B2
    s = A1 * A2 * iB1 * iB2
    out["s"] = s
    out["dm"] = _twice(mu2) * (A2 - A1) * iB1 * iB2 - s * (_twice(mu1) * iB1 - _twice(mu1) * iB2)
    out["d11"] = -(s * iB2)
    out["d12"] = _twice(A1) * iB1 * iB2
    return out


def loss_coefficients(lam, n, g_loss=1.0, g_l1=0.0, g_ssim=0.0):
    """(k0, k1): the weights of sign(img - gt) and of the SSIM-sum gradient, in float64"""
    return (g_loss * (1.0 - lam) + g_l1) / n, (g_ssim - g_loss * lam) / n


def _cta_counts(H, W):
    return ((W + TILE - 1) // TILE) * ((H + TILE - 1) // TILE)


def loss_parts(img, gt):
    """the lambda-independent part of `loss_reference`: the SSIM and L1 maps, and the SSIM-sum gradient map
    c0 + 2 a c1 + b c2, as E"""
    img = np.asarray(img, np.float32).astype(np.float64)
    gt = np.asarray(gt, np.float32).astype(np.float64)
    w = window_fp32()
    a, b = E(img), E(gt)
    t = ssim_terms(a, b, w, "loss")
    c0, c1, c2 = _conv([t["dm"]], w), _conv([t["d11"]], w), _conv([t["d12"]], w)
    t["S"] = c0 + _twice(a) * c1 + b * c2
    t["l1"] = _diff(a, b)
    t["img"], t["gt"] = img, gt
    return t


def loss_reference(img, gt, lam, g_loss=1.0, g_l1=0.0, g_ssim=0.0, need_grad=True, parts=None):
    """img, gt: [C,H,W] fp32.  -> dict with, for each of loss / l1 / ssim (scalars) and grad ([C,H,W]): the float64
    value `<k>`, its magnitude chain `<k>_mag` and its absolute fp32 budget `<k>_tol`.  g_loss, g_l1, g_ssim: the
    upstream gradients of the three outputs.  parts: `loss_parts(img, gt)`, when already computed."""
    t = loss_parts(img, gt) if parts is None else parts
    img, gt = t["img"], t["gt"]
    Cn, H, W = img.shape
    n = float(img.size)
    s = t["s"]
    d = t["l1"]
    l1p = E(np.abs(d.v), d.a, None, d.e)
    n_cta = Cn * _cta_counts(H, W)
    out = {}
    for key, p in (("l1", l1p), ("ssim", s)):
        tot = float(np.sum(p.v))
        mag = float(np.sum(p.a))
        absum = float(np.sum(np.abs(p.v)))
        err = U * float(np.sum(p.e)) + U * CTA_LEVELS * absum + n_cta * 2.0 ** -53 * absum
        out[key], out[key + "_mag"], out[key + "_sum_tol"] = tot / n, mag / n, err / n
    out["loss"] = (1.0 - lam) * out["l1"] + lam * (1.0 - out["ssim"])
    out["loss_mag"] = (1.0 - lam) * out["l1_mag"] + lam * (1.0 + out["ssim_mag"])
    out["loss_tol"] = (1.0 - lam) * out["l1_sum_tol"] + lam * out["ssim_sum_tol"] + U * abs(out["loss"])
    for key in ("l1", "ssim"):
        out[key + "_tol"] = out[key + "_sum_tol"] + U * abs(out[key])
    if not need_grad:
        return out
    k0, k1 = loss_coefficients(lam, n, g_loss, g_l1, g_ssim)
    S = t["S"]
    sgn = np.sign(img - gt)
    L = E(k0 * sgn, abs(k0) * np.abs(sgn), None, 4.0 * abs(k0) * np.abs(sgn))
    K1 = E(k1, e=4.0 * abs(k1))
    g = L + K1 * S
    out["grad"], out["grad_mag"], out["grad_tol"] = g.v, g.a, U * np.broadcast_to(g.e, g.v.shape)
    out["maps"] = dict(s=s, dm=t["dm"], d11=t["d11"], d12=t["d12"])
    return out


def _clamp01(x):
    v = np.clip(x.v, 0.0, 1.0)
    return E(v, np.minimum(x.a, 1.0), None, x.e)


def metrics_reference(img, gt, exposure=None, mask=None, x0=0):
    """img, gt: [3,H,W] fp32; exposure [3,4] or None; mask [H,W] or None; x0 the first kept column.
    -> dict: out_img [3,H,W-x0] (exposed, clamped, cropped, before the mask) with out_img_tol; sums [4] (per-channel
    squared error, SSIM map sum) with sums_tol; psnr, ssim (the result row's first two words) with their tolerances."""
    img = np.asarray(img, np.float32).astype(np.float64)[..., x0:]
    gt = np.asarray(gt, np.float32).astype(np.float64)[..., x0:]
    _, H, Wc = img.shape
    n = float(H * Wc)
    w = window_fp32()
    if exposure is not None:
        Ex = np.asarray(exposure, np.float32).astype(np.float64).reshape(3, 4)
        chans = []
        for c in range(3):
            chans.append(_sum([E(img[k]) * E(Ex[k, c]) for k in range(3)] + [E(np.full((H, Wc), Ex[c, 3]))]))
        a = E(np.stack([x.v for x in chans]), np.stack([x.a for x in chans]), np.stack([x.m for x in chans]),
              np.stack([np.broadcast_to(x.e, (H, Wc)) for x in chans]))
    else:
        a = E(img)
    a, b = _clamp01(a), _clamp01(E(gt))
    out = dict(out_img=a.v.copy(), out_img_tol=U * np.broadcast_to(a.e, a.v.shape))
    if mask is not None:
        m = E(np.asarray(mask, np.float32).astype(np.float64)[None, :, x0:])
        a, b = a * m, b * m
    s = ssim_terms(a, b, w, "metrics")["s"]
    d = _diff(a, b)
    de = np.broadcast_to(d.e, d.v.shape)
    sums, tol = np.zeros(4), np.zeros(4)
    for c in range(3):
        se = d.v[c] ** 2
        sums[c] = se.sum()
        tol[c] = U * float(np.sum(2.0 * np.abs(d.v[c]) * de[c] + U * de[c] ** 2)) + 2.0 ** -52 * n * sums[c]
    sums[3] = s.v.sum()
    tol[3] = U * float(np.sum(s.e)) + 2.0 ** -52 * 3 * n * float(np.sum(np.abs(s.v)))
    out["sums"], out["sums_tol"] = sums, tol
    with np.errstate(divide="ignore", invalid="ignore"):
        psnr_c = -10.0 * np.log10(sums[:3] / n)
        psnr_tol_c = 10.0 / math.log(10.0) * tol[:3] / sums[:3]
    out["psnr_channels"] = psnr_c
    out["psnr"] = float(psnr_c.mean())
    out["psnr_tol"] = float(psnr_tol_c.sum() / 3.0)
    out["ssim"] = sums[3] / (3.0 * n)
    out["ssim_tol"] = tol[3] / (3.0 * n)
    out["ssim_mag"] = float(np.sum(s.a)) / (3.0 * n)
    return out


# ---- fp32 evaluations of the same formula in other association orders (numpy float32, every operation rounded) ------
def _conv_fp32(x, w, order):
    """x: [C,H,W] float32.  "separable": an 11-tap horizontal pass then a vertical one, each summed left to right;
    "2d": the 121 products with the fp32-rounded outer-product weights, summed row by row, left to right"""
    f = np.float32
    if order == "separable":
        h = np.zeros_like(x)
        for k in range(TAPS):
            h = (h + f(w[k]) * _shift(x, k - RADIUS, -1)).astype(f)
        o = np.zeros_like(x)
        for k in range(TAPS):
            o = (o + f(w[k]) * _shift(h, k - RADIUS, -2)).astype(f)
        return o
    w2 = np.outer(w, w).astype(f)
    o = np.zeros_like(x)
    for i in range(TAPS):
        xi = _shift(x, i - RADIUS, -2)
        for j in range(TAPS):
            o = (o + w2[i, j] * _shift(xi, j - RADIUS, -1)).astype(f)
    return o


def loss_fp32(img, gt, k0, k1, order="separable"):
    """the forward maps and the gradient in numpy float32 -> (ssim map, l1 map, grad)"""
    f = np.float32
    a, b = np.asarray(img, f), np.asarray(gt, f)
    w = window_fp32()
    mu1, mu2 = _conv_fp32(a, w, order), _conv_fp32(b, w, order)
    e11, e22, e12 = _conv_fp32(a * a, w, order), _conv_fp32(b * b, w, order), _conv_fp32(a * b, w, order)
    C1, C2 = f(f(0.01) * f(0.01)), f(f(0.03) * f(0.03))
    s1, s2, s12 = e11 - mu1 * mu1, e22 - mu2 * mu2, e12 - mu1 * mu2
    A1, A2 = f(2) * mu1 * mu2 + C1, f(2) * s12 + C2
    B1, B2 = mu1 * mu1 + mu2 * mu2 + C1, s1 + s2 + C2
    iB1, iB2 = f(1) / B1, f(1) / B2
    s = A1 * A2 * iB1 * iB2
    dm = f(2) * mu2 * (A2 - A1) * iB1 * iB2 - s * (f(2) * mu1 * iB1 - f(2) * mu1 * iB2)
    d11 = -s * iB2
    d12 = f(2) * A1 * iB1 * iB2
    c0, c1, c2 = _conv_fp32(dm, w, order), _conv_fp32(d11, w, order), _conv_fp32(d12, w, order)
    sgn = np.sign(a - b).astype(f)
    g = f(k0) * sgn + f(k1) * (c0 + f(2) * a * c1 + b * c2)
    return s.astype(f), np.abs(a - b), g.astype(f)


# ---- test contents ---------------------------------------------------------------------------------------------------
CONTENTS = ["random", "flat", "equal", "equal_ulp", "saturated", "unclamped", "corners"]


def corner_pixels(H, W):
    """tile corners (15,15), (16,16), the frame's first and last pixel, and 5 and 6 pixels from each border"""
    pts = [(15, 15), (16, 16), (0, 0), (H - 1, W - 1)]
    for k in (5, 6):
        pts += [(k, W // 2), (H - 1 - k, W // 2), (H // 2, k), (H // 2, W - 1 - k)]
    return sorted({(y, x) for y, x in pts if 0 <= y < H and 0 <= x < W})


def make_contents(kind, C, H, W, seed=0):
    """-> (img, gt) float32 [C,H,W]"""
    rng = np.random.default_rng(seed)
    f = np.float32

    def flat():
        by, bx = max(1, H // 3 + 1), max(1, W // 4 + 1)
        levels = rng.uniform(0.05, 0.95, (C, (H + by - 1) // by, (W + bx - 1) // bx))
        return np.repeat(np.repeat(levels, by, 1), bx, 2)[:, :H, :W]
    if kind == "random":
        gt = rng.uniform(0, 1, (C, H, W))
        img = np.clip(gt * 0.7 + 0.3 * rng.uniform(0, 1, (C, H, W)), 0, 1)
    elif kind == "flat":
        base = flat()
        img = base + 1e-3 * rng.standard_normal((C, H, W))
        gt = base + 1e-3 * rng.standard_normal((C, H, W))
    elif kind in ("equal", "equal_ulp"):
        img = (flat() + 1e-3 * rng.standard_normal((C, H, W))).astype(f)
        gt = img.copy()
        if kind == "equal_ulp":
            for i, (y, x) in enumerate(corner_pixels(H, W)):
                c = i % C
                gt[c, y, x] = np.nextafter(gt[c, y, x], f(2) if i % 2 == 0 else f(-2))
        return img.astype(f), gt.astype(f)
    elif kind == "saturated":
        img, gt = rng.uniform(0, 1, (C, H, W)), rng.uniform(0, 1, (C, H, W))
        img[:, : H // 2, : W // 2] = 0.0
        gt[:, : H // 2, : W // 3] = 0.0
        img[:, H // 2:, W // 2:] = 1.0
        gt[:, H // 3:, W // 2:] = 1.0
    elif kind == "unclamped":
        img, gt = rng.uniform(-0.25, 1.5, (C, H, W)), rng.uniform(-0.25, 1.5, (C, H, W))
    elif kind == "corners":
        gt = flat()
        img = gt.copy()
        for i, (y, x) in enumerate(corner_pixels(H, W)):
            img[i % C, y, x] += 0.25 if i % 2 == 0 else -0.125
    else:
        raise ValueError(kind)
    return img.astype(f), gt.astype(f)

"""Float64 restatement of train_post's objective as csrc/loss.cu's post-loss kernels evaluate it, with a per-element fp32
error budget, on top of tests/ssim_ref.py.

OBJECTIVE.  render_post (gaussian_renderer/__init__.py:279-285) with use_trained_exp and train_post.py:135-137:
  y = image.permute(1,2,0) @ E[:3,:3] + E[:3,3]   (y_c = sum_k img_k E[k][c] + E[c][3]; no exposure: y = img)
  a = clamp(y, 0, 1) * mask
  loss = (1 - lambda) mean|a - gt| + lambda (1 - SSIM(a, gt)), gt used as it is (the loader clamped and masked it).

WHAT IS EXACT.  The kernels round y in a pinned order, ((img_0 E[0][c] + img_1 E[1][c]) + img_2 E[2][c]) + E[c][3], each
product and sum once (`exposed_fp32` does the same in numpy, bit for bit); the clamp is exact; a = clamp(y) * mask is one
fp32 rounding, reproduced by numpy too.  So the kernels' a is known exactly, the clamp decision [0 <= y <= 1] (torch's
clamp backward passes both ends) is known exactly, and ssim_ref.loss_reference applies to a as it is.

BUDGET of dL/dimg.  ssim_ref's budget of dL/da, then (chain_ref.E arithmetic) the product with the mask (one rounding),
the exact 0/1 of the clamp, and the exposure transpose dL/dimg_k = (E[k][0] g_0 + E[k][1] g_1) + E[k][2] g_2: three
rounded products and two rounded sums.
"""
import numpy as np

import ssim_ref as S
from chain_ref import E, U, _sum, compare  # noqa: F401  (compare: re-exported for the tests)


def exposure_block(exposure):
    return None if exposure is None else np.asarray(exposure, np.float32)[:3, :4]


def exposed_fp32(img, exposure):
    """the kernels' y [3,H,W], bit for bit"""
    img = np.asarray(img, np.float32)
    Ex = exposure_block(exposure)
    if Ex is None:
        return img.copy()
    out = np.empty_like(img)
    for c in range(3):
        out[c] = ((img[0] * Ex[0, c] + img[1] * Ex[1, c]) + img[2] * Ex[2, c]) + Ex[c, 3]
    return out


def staged(img, exposure, mask):
    """-> (y, a, keep): the exposed image, the clamped and masked image the loss sees (fp32, as the kernels hold it) and
    the clamp's pass mask 0 <= y <= 1"""
    y = exposed_fp32(img, exposure)
    a = np.clip(y, np.float32(0), np.float32(1))
    if mask is not None:
        a = (a * np.asarray(mask, np.float32).reshape(y.shape[1:])[None]).astype(np.float32)
    return y, a.astype(np.float32), (y >= 0) & (y <= 1)


def _chan(x, c, shape):
    return E(x.v[c], np.broadcast_to(x.a, shape)[c], np.broadcast_to(x.m, shape)[c], np.broadcast_to(x.e, shape)[c])


def post_reference(img, gt, lam, exposure=None, mask=None, g_loss=1.0, g_l1=0.0, g_ssim=0.0):
    """img (raw render), gt: [3,H,W] fp32; exposure [3,4]+ or None; mask [H,W] / [1,H,W] or None.
    -> ssim_ref.loss_reference's dict for a (loss, l1, ssim with _mag and _tol), with grad / grad_mag / grad_tol
    replaced by the gradient to img, plus y, a, keep"""
    y, a, keep = staged(img, exposure, mask)
    r = S.loss_reference(a, gt, lam, g_loss, g_l1, g_ssim)
    shape = a.shape
    g = E(r["grad"], r["grad_mag"], None, r["grad_tol"] / U)
    if mask is not None:
        g = g * E(np.broadcast_to(np.asarray(mask, np.float32).reshape(shape[1:])[None], shape).astype(np.float64))
    g = g.mask(keep)
    Ex = exposure_block(exposure)
    if Ex is not None:
        gc = [_chan(g, c, shape) for c in range(3)]
        rows = [_sum([E(float(Ex[k, c])) * gc[c] for c in range(3)]) for k in range(3)]
        g = E(np.stack([x.v for x in rows]), np.stack([x.a for x in rows]), np.stack([x.m for x in rows]),
              np.stack([np.broadcast_to(x.e, shape[1:]) for x in rows]))
    r["grad_a"] = r["grad"]
    r["grad"], r["grad_mag"], r["grad_tol"] = g.v, g.a, U * np.broadcast_to(g.e, shape)
    r["y"], r["a"], r["keep"] = y, a, keep
    return r


# ---- test inputs -----------------------------------------------------------------------------------------------------
EXPOSURES = ["none", "on", "offset"]
MASKS = ["none", "ones", "binary", "half", "fractional", "zero"]


def make_exposure(kind, rng):
    """None; a non-symmetric 3x4 colour transform; the same with offsets that push pixels below 0 and above 1"""
    if kind == "none":
        return None
    Ex = np.zeros((3, 4), np.float32)
    Ex[:, :3] = np.eye(3) * 0.9 + rng.uniform(-0.15, 0.15, (3, 3))
    Ex[:, 3] = rng.uniform(-0.05, 0.05, 3) if kind == "on" else (0.35, -0.3, 0.05)
    return Ex


def make_mask(kind, H, W, rng):
    """all ones, binary, train_test_exp's half (cameras.py:56-60 zeroes one half), fractional, all zero"""
    if kind == "none":
        return None
    if kind == "ones":
        return np.ones((H, W), np.float32)
    if kind == "binary":
        return (rng.uniform(size=(H, W)) > 0.3).astype(np.float32)
    if kind == "half":
        m = np.ones((H, W), np.float32)
        m[:, : W // 2] = 0.0
        return m
    if kind == "fractional":
        return ((rng.uniform(size=(H, W)) > 0.3) * rng.uniform(0.2, 1.0, (H, W))).astype(np.float32)
    if kind == "zero":
        return np.zeros((H, W), np.float32)
    raise ValueError(kind)


def make_inputs(H, W, exposure, mask, content="random", seed=0):
    """-> (img, gt, E, M): a raw render reaching past [0, 1], and the target as the loader leaves it (clamped, masked)"""
    rng = np.random.default_rng(seed)
    if content == "random":
        img = rng.uniform(-0.2, 1.2, (3, H, W))
        gt = rng.uniform(-0.1, 1.1, (3, H, W))
    elif content == "saturated":
        img = rng.uniform(0, 1, (3, H, W))
        img[:, : H // 2, : W // 2] = -0.25
        img[:, H // 2:, W // 2:] = 1.5
        gt = rng.uniform(0, 1, (3, H, W))
        gt[:, H // 3:, W // 2:] = 1.0
    elif content == "flat":
        base = rng.uniform(0.2, 0.8, (3, 1, 1))
        img = base + 1e-3 * rng.standard_normal((3, H, W))
        gt = base + 1e-3 * rng.standard_normal((3, H, W))
    else:
        raise ValueError(content)
    Ex = make_exposure(exposure, rng)
    M = make_mask(mask, H, W, rng)
    gt = np.clip(gt.astype(np.float32), 0, 1)
    if M is not None:
        gt = gt * M[None]
    return img.astype(np.float32), gt.astype(np.float32), Ex, M


def clamp_edge_inputs(H, W, exposure, seed=0):
    """raw renders whose y lands exactly on 0 and 1 and on the nearest values either side of them (pixels of the first
    rows).  Without exposure that is 0, 1 and one ulp around each; with an exposure img_0 is solved for the edge and then
    img_1 = img_2 = 0 and img_0 walked by ulps: y exactly at the edge (where the pinned fp32 order reaches it), and the nearest y below and above."""
    img, gt, Ex, _ = make_inputs(H, W, exposure, "none", seed=seed)
    f = np.float32
    labels = [(f(0), "exact"), (f(1), "exact"), (f(0), "below"), (f(0), "above"), (f(1), "below"), (f(1), "above")]
    pix = [(y, x) for y in range(H) for x in range(W)][: 4 * len(labels)]
    for i, (py, px) in enumerate(pix):
        t, side = labels[i % len(labels)]
        c = (i // len(labels)) % 3
        if Ex is None:
            img[c, py, px] = t if side == "exact" else np.nextafter(t, f(-1) if side == "below" else f(2))
            continue
        # img_1 = img_2 = 0: the products are exact zeros, and fl(img_0 E[0][c]) + E[c][3] can reach the edge exactly
        img[1, py, px] = img[2, py, px] = 0.0
        v0 = f((float(t) - float(Ex[c, 3])) / float(Ex[0, c]))
        vs = [v0]
        for _ in range(96):
            vs = [np.nextafter(vs[0], f(-np.inf))] + vs + [np.nextafter(vs[-1], f(np.inf))]
        pick = None
        for v in vs:
            img[0, py, px] = v
            yv = exposed_fp32(img[:, py:py + 1, px:px + 1], Ex)[c, 0, 0]
            if side == "exact" and yv == t:
                pick = v
            elif side == "below" and yv < t and (pick is None or yv > best):
                pick, best = v, yv
            elif side == "above" and yv > t and (pick is None or yv < best):
                pick, best = v, yv
        img[0, py, px] = v0 if pick is None else pick
    return img, gt, Ex

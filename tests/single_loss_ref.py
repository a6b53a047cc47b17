"""Float64 restatement of what train_single's objective adds to train_post's (tests/post_loss_ref.py): the gradient to a
trained exposure, the inverse-depth L1 term, and the densification statistics -- as csrc/loss.cu and csrc/l1_loss.cu
evaluate them, each with its fp32 budget.

EXPOSURE GRADIENT.  y_c = sum_k img_k E[k][c] + E[c][3], so dL/dE[k][c] = sum_p img_k dL/dy_c and dL/dE[c][3] = sum_p
dL/dy_c.  dL/dy is what the post-loss backward holds before the exposure transpose: post_loss_ref.post_reference applied
to y itself without an exposure gives exactly that (same a, same clamp decision), with its per-pixel budget t_c.  The
kernel rounds each product img_k g_c once (U), sums 32 lanes by a butterfly of five fp32 additions (5 U of the absolute
sum, first order) and continues in fp64:
    tol[k][c] = sum_p |img_k| t_c + 6 U sum_p |img_k g_c|,     tol[c][3] = sum_p t_c + 5 U sum_p |g_c|.

DEPTH TERM.  t = fl(fl(d - m) k) and dL/dd = fl(fl(fl(w / HW) sign(t)) k) are single fp32 operations: numpy reproduces
them bit for bit.  The sum of |t| is accumulated per thread in fp32 over its grid-stride visits, then over the CTA (3 + 5
butterfly levels twice): (visits + 13) U of the absolute sum.

STATISTICS.  max, sqrt(fl(fl(x x) + fl(y y))) and +1 are single fp32 operations: exact in numpy.
"""
import numpy as np

import post_loss_ref as R
from chain_ref import U

F = np.float32


def exposure_grad_reference(img, gt, lam, exposure=None, mask=None):
    """-> dict(dE [3,4] float64, dE_tol [3,4], g = dL/dy [3,H,W], post = post_reference of (img, exposure))"""
    img = np.asarray(img, F)
    y = R.exposed_fp32(img, exposure)
    ry = R.post_reference(y, gt, lam, None, mask)
    g, t = ry["grad"], ry["grad_tol"]
    x = img.astype(np.float64)
    dE, tol = np.zeros((3, 4)), np.zeros((3, 4))
    for c in range(3):
        for k in range(3):
            terms = x[k] * g[c]
            dE[k, c] = terms.sum()
            tol[k, c] = (np.abs(x[k]) * t[c]).sum() + 6 * U * np.abs(terms).sum()
        dE[c, 3] = g[c].sum()
        tol[c, 3] = t[c].sum() + 5 * U * np.abs(g[c]).sum()
    return dict(dE=dE, dE_tol=tol * (1 + 1e-6) + 1e-300, g=g, loss=ry)


def depth_reference(invdepth, mono, depth_mask, weight):
    """-> dict(sum = sum |t| float64, sum_tol, pure = the mean, grad fp32 [H,W] exactly as the kernel writes it)"""
    d, m, k = (np.asarray(a, F).reshape(-1) for a in (invdepth, mono, depth_mask))
    t = ((d - m).astype(F) * k).astype(F)
    n = t.size
    scale = F(F(weight) / F(n))
    grad = ((np.sign(t).astype(F) * scale).astype(F) * k).astype(F)
    tot = np.abs(t.astype(np.float64)).sum()
    vec = 4 if n % 4 == 0 else 1
    threads = min(-(-(n // vec) // 256), 132 * 16) * 256
    visits = -(-(n // vec) // threads) * vec
    return dict(sum=tot, sum_tol=(visits + 13) * U * tot + 1e-300, pure=tot / n, grad=grad.reshape(np.shape(invdepth)[-2:]))


def stats_reference(radii, d_means2D, max_radii2D, xyz_gradient_accum, denom):
    """train_single.py:147 and gaussian_model.py:687-689 -> the three updated arrays (fp32, exact)"""
    radii = np.asarray(radii)
    g = np.asarray(d_means2D, F)
    vis = radii > 0
    norm = np.sqrt(((g[:, 0] * g[:, 0]).astype(F) + (g[:, 1] * g[:, 1]).astype(F)).astype(F)).astype(F)
    mr = np.asarray(max_radii2D, F).copy()
    acc = np.asarray(xyz_gradient_accum, F).reshape(-1).copy()
    den = np.asarray(denom, F).reshape(-1).copy()
    mr[vis] = np.maximum(mr[vis], radii[vis].astype(F))
    acc[vis] = np.maximum(norm[vis], acc[vis])
    den[vis] += F(1)
    return mr, acc.reshape(np.shape(xyz_gradient_accum)), den.reshape(np.shape(denom))


def make_depth_inputs(H, W, kind="random", seed=0):
    """-> (invdepth, mono, depth_mask) [H,W]: some pixels with d == m exactly, a binary mask with holes ("zero": all zero)"""
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.0, 2.0, (H, W)).astype(F)
    m = rng.uniform(0.0, 2.0, (H, W)).astype(F)
    same = rng.uniform(size=(H, W)) < 0.1
    m[same] = d[same]
    k = (rng.uniform(size=(H, W)) > 0.25).astype(F) if kind != "zero" else np.zeros((H, W), F)
    return d, m, k

"""TEST INFRASTRUCTURE.  GaussianModel.densify_and_prune and reset_opacity (scene/gaussian_model.py:510-514, 543-685)
restated in numpy fp32, one operation per rounded result, in csrc/densify.cu's order:

  g = xyz_gradient_accum (NaN -> 0), r = max_radii2D, o = sigmoid(opacity) = 1 / (1 + exp(-x)), p = pow(o, 0.2f),
  m = max(exp(scaling)) (NaN propagating);
  clone  (sqrt(g * g) * r) * p >= max_grad and o > 0.15f and m <= float32(percent_dense * extent)
  split  (g * r) * p >= max_grad           and o > 0.15f and m >  float32(percent_dense * extent)
  keep   not split and not o < min_opacity;  rows < scaffold_points are kept and nothing else
  order  [kept originals | clones | first split copies | second split copies]; new rows have zero moments
  split  xyz + ((R[c,0] s0 + R[c,1] s1) + R[c,2] s2), s = z * exp(scaling) + 0, R = build_rotation(stored q);
         scaling log(exp(scaling) * (1.0f / 1.6f))
  reset  rows >= skybox_points: log(x / (1 - x)), x = min(sigmoid(o), 0.01f) (NaN propagating); both opacity moments 0

exp, log and pow come from a math backend: HOST (the C library's expf / logf / powf, which the emulation build calls)
or torch_math(device) (torch's exp / log / pow on that device: on the H100, the CUDA library's, which the kernels
call).  Everything else is IEEE fp32 and the same everywhere."""
import ctypes as C
import ctypes.util

import numpy as np

F = np.float32
GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")


class _Host:
    def __init__(self):
        m = C.CDLL(ctypes.util.find_library("m"))
        for n in ("expf", "logf"):
            getattr(m, n).restype, getattr(m, n).argtypes = C.c_float, [C.c_float]
        m.powf.restype, m.powf.argtypes = C.c_float, [C.c_float, C.c_float]
        self._exp = np.vectorize(lambda x: m.expf(float(x)), otypes=[F])
        self._log = np.vectorize(lambda x: m.logf(float(x)), otypes=[F])
        self._pow = np.vectorize(lambda x: m.powf(float(x), float(F(0.2))), otypes=[F])

    def exp(self, x):
        x = np.asarray(x, F)
        return self._exp(x).reshape(x.shape) if x.size else x.copy()

    def log(self, x):
        x = np.asarray(x, F)
        return self._log(x).reshape(x.shape) if x.size else x.copy()

    def pow02(self, x):
        x = np.asarray(x, F)
        return self._pow(x).reshape(x.shape) if x.size else x.copy()


HOST = _Host()


class torch_math:
    """exp / log / pow(x, 0.2) of torch on `device` (on the H100: the CUDA library's expf / logf / powf)"""

    def __init__(self, device):
        import torch
        self.torch, self.device = torch, device

    def _run(self, fn, x):
        t = self.torch
        x = np.asarray(x, F)
        return fn(t.from_numpy(np.ascontiguousarray(x)).to(self.device)).cpu().numpy()

    def exp(self, x):
        return self._run(self.torch.exp, x)

    def log(self, x):
        return self._run(self.torch.log, x)

    def pow02(self, x):
        return self._run(lambda t: self.torch.pow(t, 0.2), x)


def sigmoid(x, M):
    x = np.asarray(x, F)
    return (F(1) / (F(1) + M.exp(-x))).astype(F)


def max_nan(e):
    """torch.max(dim=1): the largest of the row, NaN when any is NaN"""
    mx = e.max(axis=1)
    mx[np.isnan(e).any(axis=1)] = F(np.nan)
    return mx


def decide(params, gacc, radii, scaffold, max_grad, min_opacity, size_threshold, M=HOST):
    """-> flags uint8 [N]: keep | clone << 1 | split << 2"""
    with np.errstate(all="ignore"):
        g = np.asarray(gacc, F).reshape(-1).copy()
        g[np.isnan(g)] = 0
        r = np.asarray(radii, F).reshape(-1)
        o = sigmoid(params[3].reshape(-1), M)
        p = M.pow02(o)
        mx = max_nan(M.exp(params[4]))
        bright = o > F(0.15)
        gn = np.sqrt(g * g)
        clone = ((gn * r) * p >= F(max_grad)) & bright & (mx <= F(size_threshold))
        split = ((g * r) * p >= F(max_grad)) & bright & (mx > F(size_threshold))
        keep = ~split & ~(o < F(min_opacity))
    keep[:scaffold] = True
    clone[:scaffold] = False
    split[:scaffold] = False
    return (keep.astype(np.uint8) | (clone.astype(np.uint8) << 1) | (split.astype(np.uint8) << 2)).astype(np.uint8)


def build_rotation(q):
    """utils/general_utils.py:82-103, element by element"""
    q = np.asarray(q, F)
    n = np.sqrt(((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]) + q[:, 3] * q[:, 3])
    w, x, y, z = (q[:, k] / n for k in range(4))
    two, one = F(2), F(1)
    R = np.empty((q.shape[0], 3, 3), F)
    R[:, 0, 0] = one - two * (y * y + z * z)
    R[:, 0, 1] = two * (x * y - w * z)
    R[:, 0, 2] = two * (x * z + w * y)
    R[:, 1, 0] = two * (x * y + w * z)
    R[:, 1, 1] = one - two * (x * x + z * z)
    R[:, 1, 2] = two * (y * z - w * x)
    R[:, 2, 0] = two * (x * z - w * y)
    R[:, 2, 1] = two * (y * z + w * x)
    R[:, 2, 2] = one - two * (x * x + y * y)
    return R


def split_xyz(xyz, R, z, e):
    """xyz + R (z * e + 0), the product summed column by column; also -> the summands' magnitudes sum_j |R_cj s_j|"""
    s = (np.asarray(z, F) * e + F(0)).astype(F)
    t = [R[:, :, j] * s[:, j:j + 1] for j in range(3)]
    return (((t[0] + t[1]) + t[2]) + xyz).astype(F), (np.abs(t[0]) + np.abs(t[1]) + np.abs(t[2])).astype(F)


def densify(params, exp_avg, exp_avg_sq, gacc, radii, scaffold, max_grad, min_opacity, size_threshold, normals, M=HOST):
    """params / moments: the six groups (numpy fp32, GaussianModel's shapes).  normals [2S,3].
    -> dict(params, exp_avg, exp_avg_sq (new lists), flags, counts (K, C, S, N'), mag [2S,3]: sum_j |R_cj s_j| of each
    split position)"""
    flags = decide(params, gacc, radii, scaffold, max_grad, min_opacity, size_threshold, M)
    keep, clone, split = (flags & 1) != 0, (flags & 2) != 0, (flags & 4) != 0
    K, Cn, S = int(keep.sum()), int(clone.sum()), int(split.sum())
    normals = np.asarray(normals, F).reshape(2 * S, 3)
    with np.errstate(all="ignore"):
        e = M.exp(params[4][split])
        R = build_rotation(params[5][split])
        x1, m1 = split_xyz(params[0][split], R, normals[:S], e)
        x2, m2 = split_xyz(params[0][split], R, normals[S:], e)
        sc = M.log((e * (F(1) / F(1.6))).astype(F))
    out_p, out_m, out_v = [], [], []
    for k in range(6):
        p = params[k]
        if k == 0:
            new = [x1, x2]
        elif k == 4:
            new = [sc, sc]
        else:
            new = [p[split], p[split]]
        out_p.append(np.concatenate([p[keep], p[clone]] + new).astype(F))
        z = lambda n: np.zeros((n,) + p.shape[1:], F)
        out_m.append(np.concatenate([exp_avg[k][keep], z(Cn + 2 * S)]).astype(F))
        out_v.append(np.concatenate([exp_avg_sq[k][keep], z(Cn + 2 * S)]).astype(F))
    return dict(params=out_p, exp_avg=out_m, exp_avg_sq=out_v, flags=flags, counts=(K, Cn, S, K + Cn + 2 * S),
                mag=np.concatenate([m1, m2]).astype(F))


def reset_opacity(params, exp_avg, exp_avg_sq, skybox, M=HOST):
    """-> (opacity, exp_avg opacity, exp_avg_sq opacity) after reset_opacity"""
    o = params[3].copy()
    with np.errstate(all="ignore"):
        x = sigmoid(o[skybox:], M)
        x = np.where(np.isnan(x) | (x < F(0.01)), x, F(0.01)).astype(F)
        o[skybox:] = M.log((x / (F(1) - x)).astype(F))
    return o, np.zeros_like(exp_avg[3]), np.zeros_like(exp_avg_sq[3])


def ulps(a, b):
    """distance in fp32 units in the last place (NaN == NaN)"""
    a, b = np.asarray(a, F).ravel(), np.asarray(b, F).ravel()
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    d = np.abs(ia - ib)
    d[np.isnan(a) & np.isnan(b)] = 0
    return d


def position_budget(got, want, mag):
    """|got - want| allowed between two evaluations of xyz + R s that differ only in the order (and contraction) of
    the three-term product: each is within 3 u sum_j |R_cj s_j| + u |result| of the exact value (u = 2^-24), so they
    are within twice that of each other"""
    u = F(2.0 ** -24)
    return 2 * (3 * u * mag + u * np.maximum(np.abs(got), np.abs(want))) + np.finfo(F).tiny


# ---- cases ------------------------------------------------------------------------------------------------------
def random_state(N, seed, K=15):
    """six stored groups and their moments, as train_single keeps them mid-run"""
    rng = np.random.default_rng(seed)
    p = [rng.normal(0, 2, (N, 3)), rng.normal(0, 0.5, (N, 1, 3)), rng.normal(0, 0.05, (N, K, 3)),
         rng.normal(0, 2, (N, 1)), rng.normal(-4.0, 1.0, (N, 3)), rng.normal(0, 1, (N, 4))]
    p = [x.astype(F) for x in p]
    m = [rng.normal(0, 1e-3, x.shape).astype(F) for x in p]
    v = [np.abs(rng.normal(0, 1e-6, x.shape)).astype(F) for x in p]
    return p, m, v


def random_stats(N, seed, frac=0.05):
    """statistics so that a few percent of the rows pass the gradient test (threshold 2e-4, radii up to 40)"""
    rng = np.random.default_rng(seed)
    g = np.abs(rng.normal(0, 2e-6, (N, 1))).astype(F)
    hot = rng.random(N) < frac
    g[hot, 0] = rng.uniform(1e-5, 1e-4, int(hot.sum())).astype(F)
    r = rng.integers(0, 40, N).astype(F)
    return g, r

"""TEST INFRASTRUCTURE.  train_coarse's parameter side (train_coarse.py:127-145 with GaussianModel's activations and
scene/OurAdam.py's non-capturable step) restated in torch, one operation per rounded result, so that it runs on CPU or
CUDA tensors and reproduces csrc/coarse_param.cu's order:

  the activations' backward from the activated gradients (identity; shs split into dc / rest; sigmoid_backward
  (g * (1 - y)) * y; exp's g * y; F.normalize's backward), _scaling.grad[:S] = 0, relevant = (_opacity.grad !=
  0).nonzero() -- [R,2], so the row set is relevant[:,0] and row 0 whenever R > 0, every row (OurAdam's dense step)
  when R == 0 --, Adam on that row set with the
  bias corrections in Python floats, then the big-Gaussian rescale, then the activations.

Every Adam operation takes full-size tensor operands (torch's alpha / value forms may fuse a multiply into an add, and
its kernels with a scalar operand take other paths, division by a scalar as a product with the reciprocal among them),
as csrc/adam.cuh rounds each on its own."""
import math

import numpy as np
import torch

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")


def sqrt32(x):
    """the correctly rounded fp32 root (torch's vectorised CPU sqrt is not; the fp64 root rounds to the right float)"""
    return torch.sqrt(x.double()).float()


def quat_norm(q):
    """|q| summed in the kernel's order ((q0^2 + q1^2) + q2^2) + q3^2, and the clamp_min(1e-12) divisor"""
    s = q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]
    s = s + q[:, 2] * q[:, 2]
    s = s + q[:, 3] * q[:, 3]
    n = sqrt32(s)[:, None]
    return n, n.clamp_min(1e-12)


def activate(params):
    """GaussianModel's get_xyz / get_features / get_opacity / get_scaling / get_rotation"""
    xyz, dc, rest, op, sc, rot = params
    _, d = quat_norm(rot)
    return dict(means3D=xyz.clone(), shs=torch.cat((dc, rest), 1), opacities=torch.sigmoid(op), scales=torch.exp(sc),
                rotations=rot / d)


def stored_grads(params, act, grads, skybox):
    """dL/d of the six stored tensors from the activated gradients (act: the forward's activated rows)"""
    xyz, dc, rest, op, sc, rot = params
    y = act["opacities"]
    g_op = grads["opacities"] * (1.0 - y)
    g_op = g_op * y
    g_sc = grads["scales"] * act["scales"]
    g_sc[:skybox] = 0
    g = grads["rotations"]
    n, d = quat_norm(rot)
    t = (-g) * ((rot / d) / d)
    gd = ((t[:, 0:1] + t[:, 1:2]) + t[:, 2:3]) + t[:, 3:4]
    gd = torch.where(n >= 1e-12, gd, torch.zeros_like(gd))
    s = torch.where(n == 0, torch.zeros_like(gd), gd / n)
    g_rot = g / d + rot * s
    K = dc.shape[1]
    return [grads["means3D"].clone(), grads["shs"][:, :K].clone(), grads["shs"][:, K:].clone(), g_op, g_sc, g_rot]


def bias_corrections(lr, beta1, beta2, step):
    """OurAdam's Python floats (step = the count after the increment), rounded to fp32 where they meet the tensors"""
    bc1, bc2 = 1 - beta1 ** step, 1 - beta2 ** step
    return np.float32(lr / bc1), np.float32(math.sqrt(bc2))


def adam_rows(p, g, m, v, rows, lr, beta1, beta2, eps, step):
    """adam.cuh on the listed rows, in place"""
    step_size, bc2_sqrt = bias_corrections(lr, beta1, beta2, step)
    gr = g[rows]
    f = lambda x: torch.full_like(gr, float(np.float32(x)))         # full operands: no scalar fast path of torch's
    mm = m[rows] * f(beta1) + f(1.0 - beta1) * gr
    vv = v[rows] * f(beta2) + f(1.0 - beta2) * (gr * gr)
    denom = sqrt32(vv) / f(bc2_sqrt) + f(eps)
    p[rows] = p[rows] + f(-step_size) * (mm / denom)
    m[rows] = mm
    v[rows] = vv


def param_step(state, act, grads, threshold):
    """one train_coarse optimizer step + rescale on state (dict: params [6], exp_avg [6], exp_avg_sq [6], step int,
    skybox, lr [6], betas [6], eps [6]), in place; -> (relevant [R,2], the new activated rows)"""
    params = state["params"]
    S = state["skybox"]
    sg = stored_grads(params, act, grads, S)
    relevant = (sg[3] != 0).nonzero()
    state["step"] += 1
    # OurAdam's row set: relevant[:,0] and row 0 when R > 0; every row (its dense step) when R == 0
    rows = torch.unique(torch.cat((relevant[:, 0], relevant.new_zeros(1)))) if relevant.shape[0] else \
        torch.arange(params[0].shape[0], device=params[0].device)
    for k in range(6):
        b1, b2 = state["betas"][k]
        adam_rows(params[k], sg[k], state["exp_avg"][k], state["exp_avg_sq"][k], rows, state["lr"][k], b1, b2,
                  state["eps"][k], state["step"])
    sc = params[4]
    e = torch.exp(sc)
    vals = e.max(dim=1).values
    viol = vals > float(np.float32(threshold))
    viol[:S] = False
    sc[viol] = torch.log(e[viol] * 0.8)
    return relevant, activate(params)


def random_state(N, skybox, seed, device="cpu", K=3):
    """a GaussianModel-shaped state with skybox rows first, mid-training moments and a step count of 7"""
    g = np.random.default_rng(seed)
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device=device)
    params = [t(g.normal(0, 2, (N, 3))), t(g.normal(0, 0.5, (N, 1, 3))), t(g.normal(0, 0.1, (N, K, 3))),
              t(g.normal(-2, 1.5, (N, 1))), t(g.normal(-3, 1.0, (N, 3))), t(g.normal(0, 1, (N, 4)))]
    exp_avg = [t(g.normal(0, 1e-3, p.shape)) for p in params]
    exp_avg_sq = [t(g.uniform(0, 1e-5, p.shape)) for p in params]
    return dict(params=params, exp_avg=exp_avg, exp_avg_sq=exp_avg_sq, step=7, skybox=skybox,
                lr=[0.0, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001], betas=[(0.9, 0.999)] * 6, eps=[1e-15] * 6)


def random_grads(N, seed, device="cpu", K=3, zero_frac=0.4):
    """activated gradients; a fraction of the rows is untouched by the frame (all zero), as the backward leaves them"""
    g = np.random.default_rng(seed)
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device=device)
    out = dict(means3D=t(g.normal(0, 1e-2, (N, 3))), shs=t(g.normal(0, 1e-2, (N, K + 1, 3))),
               opacities=t(g.normal(0, 1e-2, (N, 1))), scales=t(g.normal(0, 1e-2, (N, 3))),
               rotations=t(g.normal(0, 1e-2, (N, 4))))
    off = torch.tensor(g.uniform(size=N) < zero_frac, device=device)
    for v in out.values():
        v[off] = 0
    return out


def clone_state(st):
    c = dict(st)
    for k in ("params", "exp_avg", "exp_avg_sq"):
        c[k] = [x.clone() for x in st[k]]
    return c


# ---- the reference's own iteration (tests/golden/coarse_iteration.npz) -----------------------------------------------------
ATTRS = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")


def golden_start(z, c):
    """the state before iteration c of the fixture (the reference's stored tensors, OurAdam's moments and step count)"""
    def t(key):
        return torch.tensor(z[key])
    if c == 0:
        params = [t(f"init_{a}") for a in ATTRS]
        m = [torch.zeros_like(p) for p in params]
        v = [torch.zeros_like(p) for p in params]
        step = 0
    else:
        params = [t(f"c{c - 1}_after{a}") for a in ATTRS]
        m = [t(f"c{c - 1}_m{a}") for a in ATTRS]
        v = [t(f"c{c - 1}_v{a}") for a in ATTRS]
        step = int(z[f"c{c - 1}_step"])
    lrs = [float(x) for x in z["lrs"]]
    return dict(params=params, exp_avg=m, exp_avg_sq=v, step=step, skybox=int(z["skybox"]), lr=lrs,
                betas=[(0.9, 0.999)] * 6, eps=[1e-15] * 6)


def golden_inputs(z, c):
    """the activated rows the reference rendered in iteration c and their gradients"""
    names = ("means3D", "shs", "opacities", "scales", "rotations")
    return ({k: torch.tensor(z[f"c{c}_act_{k}"]) for k in names}, {k: torch.tensor(z[f"c{c}_actgrad_{k}"]) for k in names})


def rotation_grad_tol(z, c, rot):
    """F.normalize's backward g / d + q (sum_j -g_j q_j / d^3) / |q| cancels: its error is bounded by the size of its
    terms, about 2 |g| / d, times a few ulp -- 2^-19 * max_j |g_j| / d per row"""
    g = np.abs(z[f"c{c}_actgrad_rotations"]).max(axis=1, keepdims=True).astype(np.float64)
    d = np.maximum(np.linalg.norm(np.asarray(rot, np.float64), axis=1, keepdims=True), 1e-12)
    return 2.0 ** -19 * g / d


def golden_violations(z, c, before, params, m, v, skip_rows=()):
    """-> list of (what, worst ratio) over the budget of one iteration against the reference's OurAdam and rescale.

    The reference's CPU ops fuse a multiply into an add (add_(alpha=), addcmul_(value=), addcdiv_(value=)) and divide by
    the Python-float bias correction through its reciprocal, where csrc/adam.cuh rounds every operation: about 8
    roundings placed differently, so the update u = step_size * m / denom differs by at most 8 * 2^-24 |u| < 2^-20 |u|
    and each moment by 2^-22 of its terms (0.9 |m_old| + 0.1 |g| and 0.999 v_old + 0.001 g^2).  The rotation's stored
    gradient is F.normalize's backward, whose 4-term sum torch orders freely (rotation_grad_tol), and a
    rescaled scaling passes through exp / log of two libraries (4 ulp).  Decisions -- relevance, the row set, which rows
    are rescaled -- must be the reference's exactly.  skip_rows: rows left out (the threshold-edge rows on a platform
    whose exp is not the fixture's)."""
    bad = []
    ulp = lambda x: np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)
    S = int(z["skybox"])
    adam4 = z[f"c{c}_adam_scaling"]
    resc = np.any(z[f"c{c}_after_scaling"] != adam4, axis=1)
    resc[:S] = False
    for k, a in enumerate(ATTRS):
        g = z[f"c{c}_grad{a}"].astype(np.float64)
        m0, v0 = before["exp_avg"][k].numpy().astype(np.float64), before["exp_avg_sq"][k].numpy().astype(np.float64)
        gtol = rotation_grad_tol(z, c, before["params"][5].numpy()) if k == 5 else 0.0
        tm = 2.0 ** -22 * (0.9 * np.abs(m0) + 0.1 * np.abs(g)) + 0.1 * gtol + ulp(z[f"c{c}_m{a}"])
        tv = 2.0 ** -22 * (0.999 * v0 + 0.001 * g * g) + 0.001 * 2 * np.abs(g) * gtol + ulp(z[f"c{c}_v{a}"])
        u = np.abs(z[f"c{c}_adam{a}"].astype(np.float64) - before["params"][k].numpy())
        tp = 2.0 ** -20 * u + 2 * ulp(z[f"c{c}_after{a}"])
        if k == 4:
            tp = tp + 4 * ulp(z[f"c{c}_after{a}"]) * resc[:, None]
        for what, got, want, tol in (("m", m[k], z[f"c{c}_m{a}"], tm), ("v", v[k], z[f"c{c}_v{a}"], tv),
                                     ("param", params[k], z[f"c{c}_after{a}"], tp)):
            d = np.abs(np.asarray(got, np.float64) - want.astype(np.float64))
            if len(skip_rows):
                d[list(skip_rows)] = 0
            r = float((d / np.maximum(tol, 1e-45)).max())
            if r > 1.0:
                bad.append((f"{a} {what}", r))
    return bad

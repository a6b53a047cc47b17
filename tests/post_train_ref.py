"""TEST INFRASTRUCTURE.  train_post's parameter side (train_post.py:85, 167-192 with create_from_hier's activations and
torch.optim.Adam's default CUDA path) restated in torch and numpy, one operation per rounded result, in
csrc/post_param.cu's order:

  the activations' backward from the activated gradients (identity; shs split into dc / rest; abs's g * sign(o);
  exp's g * y; F.normalize's backward); all six stored gradients zeroed on the locked rows (the anchors, and the last
  skybox_points rows when skybox_locked); torch.optim.Adam on EVERY element (a dense step) with this iteration's xyz lr;
  the activations xyz, cat(dc, rest), abs(o), exp(s), q / max(|q|, 1e-12).

The Adam arithmetic is torch's foreach CUDA path (m = lerp(m, g, 1 - beta1), v = v beta2 then + (1 - beta2) g g,
p + step_size m / (sqrt(v) / bc2_sqrt + eps)), its fused multiply-adds formed in extended precision as
tests/single_train_ref.py forms them."""
import numpy as np
import torch

import coarse_ref as CR
from single_train_ref import exposure_bias, fma

F = np.float32
LRS = [1.6e-4, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]       # train_post's groups (OptimizationParams defaults)


def locked_mask(N, skybox, skybox_locked, anchors):
    """the rows train_post.py:167-181 zeroes: the anchors (torch indexing: duplicates, negatives from the end) and the
    skybox tail"""
    m = torch.zeros(N, dtype=torch.bool)
    if len(anchors):
        m[torch.as_tensor(anchors, dtype=torch.long)] = True
    if skybox and skybox_locked:
        m[N - skybox:] = True
    return m


def activate(params):
    """create_from_hier's get_xyz / get_features / get_opacity (abs) / get_scaling / get_rotation"""
    xyz, dc, rest, op, sc, rot = params
    _, d = CR.quat_norm(rot)
    return dict(means3D=xyz.clone(), shs=torch.cat((dc, rest), 1), opacities=torch.abs(op), scales=torch.exp(sc),
                rotations=rot / d)


def stored_grads(params, act, grads, locked):
    """dL/d of the six stored tensors, the locked rows' zeroed (locked: bool [N] or None)"""
    sg = CR.stored_grads(params, act, grads, 0)
    sg[3] = grads["opacities"] * torch.sign(params[3])                  # abs_backward: grad * self.sgn()
    if locked is not None:
        for g in sg:
            g[locked.to(g.device)] = 0
    return sg


def torch_adam(p, g, m, v, lr, beta1, beta2, eps, t):
    """torch.optim.Adam's foreach CUDA step of one tensor (numpy fp32, in place); t = the count after the increment"""
    w = F(1.0 - beta1)
    m1 = fma(w, g - m, m) if abs(w) < F(0.5) else fma(m - g, F(1) - w, g)
    v1 = fma(F(1.0 - beta2), g * g, v * F(beta2))
    ss, bs = exposure_bias(lr, beta1, beta2, t)
    den = np.sqrt(v1) / bs + F(eps)
    p[...] = fma(ss, m1 / den, p)
    m[...] = m1
    v[...] = v1


def param_step(state, act, grads, xyz_lr, locked):
    """one train_post optimizer step on state (coarse_ref's dict of torch CPU tensors), in place -> the new activated rows"""
    sg = stored_grads(state["params"], act, grads, locked)
    state["step"] += 1
    for k in range(6):
        p, m, v = (state[n][k].numpy() for n in ("params", "exp_avg", "exp_avg_sq"))
        b1, b2 = state["betas"][k]
        torch_adam(p, sg[k].numpy().astype(F), m, v, xyz_lr if k == 0 else state["lr"][k], b1, b2, state["eps"][k],
                   state["step"])
    return activate(state["params"])


def random_post_state(N, skybox, seed, K=15):
    """coarse_ref.random_state with SH degree 3 rows, train_post's lrs and stored opacities of both signs, some exactly
    +0 and -0"""
    st = CR.random_state(N, skybox, seed, "cpu", K)
    st["lr"] = list(LRS)
    g = np.random.default_rng(seed + 500)
    op = g.normal(0, 0.4, (N, 1)).astype(F)
    op[g.uniform(size=N) < 0.05] = 0.0
    op[g.uniform(size=N) < 0.05] = -0.0
    st["params"][3] = torch.tensor(op)
    return st


# ---- the reference's own iterations (tests/golden/post_train.npz) --------------------------------------------------------
ATTRS = CR.ATTRS


def golden_start(z, c):
    """the state before iteration c's optimizer step: the reference's stored tensors, its torch.optim.Adam moments and
    step count, the skybox size and whether it is locked in iteration c"""
    t = lambda key: torch.tensor(z[key])
    if c == 0:
        params = [t(f"init_{a}") for a in ATTRS]
        m, v = [torch.zeros_like(p) for p in params], [torch.zeros_like(p) for p in params]
    else:
        params = [t(f"c{c - 1}_after{a}") for a in ATTRS]
        m, v = [t(f"c{c - 1}_m{a}") for a in ATTRS], [t(f"c{c - 1}_v{a}") for a in ATTRS]
    return dict(params=params, exp_avg=m, exp_avg_sq=v, step=int(z[f"c{c - 1}_step"]) if c else 0,
                skybox=int(z["skybox"]), lr=[float(x) for x in z["lrs"]], betas=[(0.9, 0.999)] * 6, eps=[1e-15] * 6,
                skybox_locked=bool(z[f"c{c}_locked"]))


def golden_locked(z, c):
    N = z["init__xyz"].shape[0]
    return locked_mask(N, int(z["skybox"]), bool(z[f"c{c}_locked"]), [int(a) for a in z["anchors"]])


def golden_violations(z, c, before, params, m, v):
    """-> list of (what, worst ratio) over the budget of iteration c against the reference's torch.optim.Adam on the CPU
    (its single-tensor path: lerp, addcmul_(value=), addcdiv_(value=)), whose roundings are placed differently from the
    foreach CUDA arithmetic restated here -- the budget of coarse_ref.golden_violations: the update within 2^-20 of
    itself, each moment within 2^-22 of its terms, the rotation's stored gradient within F.normalize's reordering"""
    return CR.golden_violations(z, c, before, params, m, v)

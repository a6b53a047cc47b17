"""TEST INFRASTRUCTURE.  train_single's parameter side (train_single.py:85-88, 157-186 with GaussianModel's activations,
scene/OurAdam.py's non-capturable step and torch.optim.Adam on the exposures) restated in torch and numpy, one operation
per rounded result, in csrc/single_param.cu's order.  Where the rules agree with train_coarse's it is tests/coarse_ref.py:

  the activations' backward; with skybox_locked all six stored gradients of rows < skybox_points = 0; relevant =
  (_opacity.grad.flatten() != 0).nonzero() -- exactly those rows, every row (OurAdam's dense step) when there is none
  --; Adam on that row set with this iteration's xyz lr; the rescale of rows >= scaffold_points whose largest exp(s)
  exceeds float32(extent * 0.02); the activations.

The exposure's Adam is torch's foreach CUDA arithmetic (m = lerp(m, g, 1 - beta1), v = v beta2 then + (1 - beta2) g g,
p + step_size m / (sqrt(v) / bc2_sqrt + eps)), with its fused multiply-adds formed exactly in extended precision."""
import numpy as np
import torch

import coarse_ref as CR

F = np.float32


def gaussian_step(state, act, grads, threshold, xyz_lr):
    """one OurAdam step + rescale on state (coarse_ref's dict, plus skybox_locked and scaffold), in place;
    -> (relevant [R], the new activated rows)"""
    params = state["params"]
    S = state["skybox"]
    sg = CR.stored_grads(params, act, grads, 0)
    if state["skybox_locked"]:
        for g in sg:
            g[:S] = 0
    relevant = (sg[3].flatten() != 0).nonzero().flatten()
    state["step"] += 1
    rows = relevant if relevant.shape[0] else torch.arange(params[0].shape[0], device=params[0].device)
    lrs = [xyz_lr] + list(state["lr"][1:])
    for k in range(6):
        b1, b2 = state["betas"][k]
        CR.adam_rows(params[k], sg[k], state["exp_avg"][k], state["exp_avg_sq"][k], rows, lrs[k], b1, b2,
                     state["eps"][k], state["step"])
    rescale(params, threshold, state["scaffold"])
    return relevant, CR.activate(params)


def rescale(params, threshold, scaffold):
    """train_single.py:180-186: vals = get_scaling.max(dim=1); violators = vals > threshold (in float32);
    violators[:scaffold_points] = False; _scaling[violators] = log(get_scaling[violators] * 0.8)"""
    sc = params[4]
    e = torch.exp(sc)
    viol = e.max(dim=1).values > float(F(threshold))
    viol[:scaffold] = False
    sc[viol] = torch.log(e[viol] * 0.8)


def fma(a, b, c):
    """fp32 fused multiply-add: the product is exact in long double, one rounding (to fp32, past a 64-bit one)"""
    ld = np.longdouble
    return (np.asarray(a, F).astype(ld) * np.asarray(b, F).astype(ld) + np.asarray(c, F).astype(ld)).astype(F)


def exposure_bias(lr, beta1, beta2, t):
    """torch.optim.Adam's Python floats of step count t: step_size = -(lr / bc1), bc2_sqrt = bc2 ** 0.5, as fp32"""
    bc1, bc2 = 1 - beta1 ** float(t), 1 - beta2 ** float(t)
    return F((lr / bc1) * -1), F(bc2 ** 0.5)


def exposure_adam(ex, m, v, grad_row, image, lr, t, beta1=0.9, beta2=0.999, eps=1e-8):
    """one torch.optim.Adam step of the whole [n,3,4] exposure tensor (numpy fp32, in place); the gradient is grad_row
    at row `image` and zero elsewhere; t = the step count after the increment"""
    g = np.zeros_like(ex)
    g[image] = grad_row
    w = F(1.0 - beta1)
    m1 = fma(w, g - m, m) if abs(w) < F(0.5) else fma(m - g, F(1) - w, g)
    v1 = fma(F(1.0 - beta2), g * g, v * F(beta2))
    ss, bs = exposure_bias(lr, beta1, beta2, t)
    den = np.sqrt(v1) / bs + F(eps)
    ex[...] = fma(ss, m1 / den, ex)
    m[...] = m1
    v[...] = v1


def random_single_state(N, skybox, seed, skybox_locked=True, scaffold=0, n_images=4, device="cpu", K=15):
    """coarse_ref.random_state with SH degree 3 rows, the lock and scaffold settings, train_single's lrs and exposures
    in mid-training"""
    st = CR.random_state(N, skybox, seed, device, K)
    st["lr"] = [1.6e-4, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]
    st["skybox_locked"], st["scaffold"] = skybox_locked, scaffold
    g = np.random.default_rng(seed + 1000)
    ex = np.tile(np.eye(3, 4, dtype=F), (n_images, 1, 1)) + g.normal(0, 0.05, (n_images, 3, 4)).astype(F)
    st["exposure"] = ex
    st["exposure_m"] = g.normal(0, 1e-3, ex.shape).astype(F)
    st["exposure_v"] = g.uniform(0, 1e-5, ex.shape).astype(F)
    st["exposure_step"] = 7
    return st


def clone_single(st):
    c = CR.clone_state(st)
    for k in ("exposure", "exposure_m", "exposure_v"):
        c[k] = st[k].copy()
    return c


# ---- the reference's own iterations (tests/golden/single_train.npz) ------------------------------------------------------
ATTRS = CR.ATTRS


def golden_start(z, c):
    """the state before iteration c's optimizer steps: the reference's stored tensors, OurAdam's moments and step
    count (after densify_and_prune / reset_opacity when iteration c ran them), and the exposures with their Adam state"""
    t = lambda key: torch.tensor(z[key])
    if f"c{c}_dens_xyz" in z:
        params = [t(f"c{c}_dens{a}") for a in ATTRS]
        m, v = [t(f"c{c}_densm{a}") for a in ATTRS], [t(f"c{c}_densv{a}") for a in ATTRS]
    elif c == 0:
        params = [t(f"init_{a}") for a in ATTRS]
        m, v = [torch.zeros_like(p) for p in params], [torch.zeros_like(p) for p in params]
    else:
        params = [t(f"c{c - 1}_after{a}") for a in ATTRS]
        m, v = [t(f"c{c - 1}_m{a}") for a in ATTRS], [t(f"c{c - 1}_v{a}") for a in ATTRS]
    step = int(z[f"c{c - 1}_step"]) if c else 0
    if c == 0:
        ex = z["init_exposure"].copy()
        em, ev, es = np.zeros_like(ex), np.zeros_like(ex), 0
    else:
        ex, em, ev = (z[f"c{c - 1}_exposure{k}"].copy() for k in ("", "_m", "_v"))
        es = int(z[f"c{c - 1}_exposure_step"])
    return dict(params=params, exp_avg=m, exp_avg_sq=v, step=step, skybox=int(z["skybox"]),
                lr=[float(x) for x in z["lrs"]], betas=[(0.9, 0.999)] * 6, eps=[1e-15] * 6,
                skybox_locked=bool(z[f"c{c}_locked"]), scaffold=int(z["scaffold"]), exposure=ex, exposure_m=em,
                exposure_v=ev, exposure_step=es)


def golden_frame(z, c):
    """-> (image, xyz lr, exposure lr, the frame's fp32 exposure gradient row, whether OurAdam stepped, threshold)"""
    image = int(z[f"c{c}_image"])
    return (image, float(z[f"c{c}_xyz_lr"]), float(z[f"c{c}_exp_lr"]), z[f"c{c}_exposure_grad"][image].copy(),
            bool(z[f"c{c}_gstep"]), float(z["extent"]) * 0.02)


def golden_iteration(z, c, st):
    """the restatement of iteration c on st, in place -> relevant (None without a Gaussian step)"""
    image, xyz_lr, exp_lr, eg, gstep, thr = golden_frame(z, c)
    st["exposure_step"] += 1
    exposure_adam(st["exposure"], st["exposure_m"], st["exposure_v"], eg, image, exp_lr, st["exposure_step"])
    if not gstep:
        rescale(st["params"], thr, st["scaffold"])
        return None
    act, grads = CR.golden_inputs(z, c)
    relevant, _ = gaussian_step(st, act, grads, thr, xyz_lr)
    return relevant


def _ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


def golden_exposure_violations(z, c, before, ex, m, v):
    """torch.optim.Adam on the CPU (the fixture's: single-tensor path) against the foreach CUDA arithmetic: about 8
    roundings placed differently, so the update differs by at most 2^-20 of itself and each moment by 2^-22 of its terms"""
    image = int(z[f"c{c}_image"])
    g = np.zeros_like(before["exposure"], np.float64)
    g[image] = z[f"c{c}_exposure_grad"][image]
    m0, v0 = before["exposure_m"].astype(np.float64), before["exposure_v"].astype(np.float64)
    want = {k: z[f"c{c}_exposure{k}"] for k in ("", "_m", "_v")}
    tol = {"_m": 2.0 ** -22 * (0.9 * np.abs(m0) + 0.1 * np.abs(g)) + _ulp(want["_m"]),
           "_v": 2.0 ** -22 * (0.999 * v0 + 0.001 * g * g) + _ulp(want["_v"]),
           "": 2.0 ** -20 * np.abs(want[""].astype(np.float64) - before["exposure"]) + 2 * _ulp(want[""])}
    bad = []
    for k, got in (("", ex), ("_m", m), ("_v", v)):
        r = float((np.abs(np.asarray(got, np.float64) - want[k]) / np.maximum(tol[k], 1e-45)).max())
        if r > 1.0:
            bad.append((f"exposure{k}", r))
    return bad


def golden_no_step_violations(z, c, before, params, m, v, skip_rows=()):
    """an iteration without OurAdam's step: moments and every stored tensor but the scaling as densify_and_prune /
    reset_opacity left them, the scaling after the rescale within the 4 ulp of two libraries' exp / log"""
    bad = []
    for k, a in enumerate(ATTRS):
        for what, got, want in (("m", m[k], before["exp_avg"][k].numpy()), ("v", v[k], before["exp_avg_sq"][k].numpy())):
            if not np.array_equal(np.asarray(got), want):
                bad.append((f"{a} {what}", 1e9))
        got, want = np.asarray(params[k], np.float64), z[f"c{c}_after{a}"].astype(np.float64)
        tol = 4 * _ulp(want) if k == 4 else 0 * want
        d = np.abs(got - want)
        if len(skip_rows):
            d[list(skip_rows)] = 0
        if np.any(d > tol):
            bad.append((f"{a} param", float(d.max())))
    return bad

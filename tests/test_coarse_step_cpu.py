"""CPU: train_coarse's objective and parameter step on the emulation build (the library's kernels compiled for the host).

  * the coarse-loss pair equals h3dgs_l1_ssim_forward / _backward bit for bit with a mask of ones and img in [0, 1],
    equals the post-loss pair (no exposure, same mask) wherever no value is clamped, and passes the gradient for y > 1;
  * h3dgs_coarse_param_step against tests/coarse_ref.py: skybox rows first, zero / underflowing / NaN opacity
    gradients, row 0's update whenever any row is relevant, OurAdam's dense step when no row is, violators at and one ulp around
    the threshold, an overflowed frame; stored rows, moments and decisions bit for bit, the rows that pass through
    expf / logf / F.normalize within a stated ulp budget (the host's libm and the restatement's exp / log / sqrt
    reductions are not the device's);
  * the bias corrections of the prologue against the host's doubles;
  * densify_stats with NULL xyz_gradient_accum / denom touches max_radii2D only."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "emul"))

import coarse_ref as CR  # noqa: E402

F = np.float32
# the intrinsics coarse_param.cu uses beyond what the emulator header provides
_SHIM = """#include <math.h>
static inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
static inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
static inline float __fsqrt_rn(float a) { volatile float r = sqrtf(a); return r; }
"""


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    import build_emu
    from emu_api import Emu
    out = str(tmp_path_factory.mktemp("h3dgs_emu_coarse"))
    build_emu.build(out)
    src = os.path.join(out, "hierarchical-3d-gaussians_b200", "csrc")
    with open(os.path.join(out, "shim.h"), "w") as f:
        f.write(_SHIM)
    flags = ["-std=c++17", "-O1", "-fPIC", "-ffp-contract=off", "-fno-strict-aliasing", "-w", "-D__CUDACC__",
             "-DH3_PAIR_HOST_EMU", "-DH3_HOST_EMU", "-I", src, "-include", os.path.join(out, "shim.h")]
    obj = os.path.join(out, "coarse_param.o")
    r = subprocess.run(["/usr/bin/g++"] + flags + ["-c", os.path.join(src, "coarse_param.cpp"), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[:4000]
    objs = [os.path.join(out, s.replace(".cu", ".o")) for s in build_emu.SOURCES] + [os.path.join(out, "simt_emu.o"), obj]
    so = os.path.join(out, "libh3dgs_emu_coarse.so")
    r = subprocess.run(["/usr/bin/g++", "-shared", "-o", so] + objs + ["-lm", "-lpthread"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[:4000]
    return Emu(so)


def _expf(x):
    import ctypes.util
    libm = C.CDLL(ctypes.util.find_library("m"))
    libm.expf.restype, libm.expf.argtypes = C.c_float, [C.c_float]
    return F(libm.expf(float(x)))


def ulps(a, b):
    """distance in fp32 ulps (same-sign finite values; NaN == NaN counts as 0)"""
    a, b = np.asarray(a, F).ravel(), np.asarray(b, F).ravel()
    both_nan = np.isnan(a) & np.isnan(b)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    d = np.abs(ia - ib)
    d[both_nan] = 0
    return d


# ---- the loss pair ------------------------------------------------------------------------------------------------------
def _loss_emu(emu, fn, img, gt, mask, k=(0.3, -0.01)):
    from emu_api import aligned, f32, ptr
    _, H, W = img.shape
    keep = [f32(img), f32(gt), None if mask is None else f32(mask)]
    sums = aligned(16, np.float64, (2,))
    maps = aligned(9 * H * W * 4, F, (3, 3, H, W))
    coeffs = f32(np.array(k, F))
    grad = aligned(3 * H * W * 4, F, (3, H, W))
    L = emu.L
    if fn == "coarse":
        emu.check(L.h3dgs_coarse_loss_forward(H, W, ptr(keep[0]), ptr(keep[1]), ptr(keep[2]), ptr(sums), ptr(maps), None))
        emu.check(L.h3dgs_coarse_loss_backward(H, W, ptr(keep[0]), ptr(keep[1]), ptr(keep[2]), ptr(maps), ptr(coeffs), ptr(grad), None))
    elif fn == "post":
        emu.check(L.h3dgs_post_loss_forward(H, W, ptr(keep[0]), ptr(keep[1]), None, ptr(keep[2]), ptr(sums), ptr(maps), None))
        emu.check(L.h3dgs_post_loss_backward(H, W, ptr(keep[0]), ptr(keep[1]), None, ptr(keep[2]), ptr(maps), ptr(coeffs), ptr(grad), None))
    else:
        emu.check(L.h3dgs_l1_ssim_forward(3, H, W, ptr(keep[0]), ptr(keep[1]), ptr(sums), ptr(maps), None))
        emu.check(L.h3dgs_l1_ssim_backward(3, H, W, ptr(keep[0]), ptr(keep[1]), ptr(maps), ptr(coeffs), ptr(grad), None))
    return sums.copy(), grad.copy()


@pytest.mark.parametrize("shape", [(1, 1), (17, 33), (40, 23)])
def test_coarse_loss_with_ones_is_l1_ssim(emu, shape):
    g = np.random.default_rng(3)
    img, gt = g.uniform(0, 1, (3,) + shape).astype(F), g.uniform(0, 1, (3,) + shape).astype(F)
    a = _loss_emu(emu, "coarse", img, gt, np.ones(shape, F))
    b = _loss_emu(emu, "l1ssim", img, gt, None)
    c = _loss_emu(emu, "coarse", img, gt, None)
    for x in (a, c):
        assert np.array_equal(x[0], b[0]) and np.array_equal(x[1].view(np.int32), b[1].view(np.int32))


@pytest.mark.parametrize("mask", ["binary", "fractional"])
def test_coarse_loss_is_post_loss_unclamped(emu, mask):
    g = np.random.default_rng(5)
    H, W = 29, 35
    img, gt = g.uniform(-0.3, 1.4, (3, H, W)).astype(F), g.uniform(0, 1, (3, H, W)).astype(F)
    M = (g.uniform(size=(H, W)) > 0.3).astype(F)
    if mask == "fractional":
        M *= g.uniform(0.2, 1.0, (H, W)).astype(F)
    inside = (img >= 0) & (img <= 1)
    cs, cg = _loss_emu(emu, "coarse", img, gt, M)
    ps, pg = _loss_emu(emu, "post", np.clip(img, 0, 1), gt, M)
    # on the clamped copy the staged values agree everywhere, so the SSIM maps and sums do; the gradient differs only
    # where the coarse image is outside [0, 1]
    ps2, _ = _loss_emu(emu, "post", img, gt, M)
    assert np.array_equal(ps, ps2)
    cs_clip, cg_clip = _loss_emu(emu, "coarse", np.clip(img, 0, 1), gt, M)
    assert np.array_equal(cs_clip, ps) and np.array_equal(cg_clip[inside].view(np.int32), pg[inside].view(np.int32))
    # above 1 (and below 0) the gradient passes: mask * (k0 sign + k1 ...) is non-zero where the mask is
    out = ~inside & (M[None] > 0)
    assert out.sum() > 50 and np.count_nonzero(cg[out]) >= 0.95 * out.sum()
    assert not np.array_equal(cs, ps)


# ---- the parameter step -------------------------------------------------------------------------------------------------
class _EmuState:
    """host arrays of one coarse state and scene, and the h3dgs_coarse_args pointing at them"""

    def __init__(self, st, act, grads, threshold, scan_info=None):
        from emu_api import aligned, f32
        from h3dgs import _lib
        self.p = [f32(x.numpy()) for x in st["params"]]
        self.m = [f32(x.numpy()) for x in st["exp_avg"]]
        self.v = [f32(x.numpy()) for x in st["exp_avg_sq"]]
        self.act = {k: f32(v.numpy()) for k, v in act.items()}
        self.g = {k: f32(v.numpy()) for k, v in grads.items()}
        self.step = aligned(8, np.int64, (1,))
        self.step[0] = st["step"]
        self.scratch = aligned(64)
        self.info = None if scan_info is None else np.array(scan_info, np.uint32)
        a = self.a = _lib.CoarseArgs()
        N = a.N = st["params"][0].shape[0]
        a.sh_coeffs, a.skybox_points, a.rescale_threshold = st["params"][2].shape[1] + 1, st["skybox"], float(F(threshold))
        for k in range(6):
            a.params[k], a.exp_avg[k], a.exp_avg_sq[k] = self.p[k].ctypes.data, self.m[k].ctypes.data, self.v[k].ctypes.data
            a.lr[k], (a.beta1[k], a.beta2[k]), a.eps[k] = st["lr"][k], st["betas"][k], st["eps"][k]
        a.step, a.scratch = self.step.ctypes.data, self.scratch.ctypes.data
        for k in ("means3D", "shs", "opacities", "scales", "rotations"):
            setattr(a, "grad_" + k, self.g[k].ctypes.data)
            setattr(a, k, self.act[k].ctypes.data)
        a.scan_info = None if self.info is None else self.info.ctypes.data
        assert N > 0

    def run(self, emu, mode):
        emu.check(emu.L.h3dgs_coarse_param_step(C.byref(self.a), mode, None))


def _case(N, S, seed, special=True):
    import torch
    st = CR.random_state(N, S, seed)
    act = CR.activate(st["params"])
    grads = CR.random_grads(N, seed + 1)
    thr = 0.05
    if special:
        op = st["params"][3]
        # underflow: a tiny activated gradient on an almost saturated opacity; the stored product is 0 in fp32
        op[S + 5, 0] = 30.0
        grads["opacities"][S + 5, 0] = 1e-30
        grads["opacities"][S + 6, 0] = float("nan")
        # violators at and one ulp around the threshold (rows past the skybox), decided on exp of the updated scaling:
        # rows S+7..S+9 get no Adam update (their gradients are zero), so their stored scaling is what exp reads
        for r in (S + 7, S + 8, S + 9):
            for v in grads.values():
                v[r] = 0
        t = F(thr)
        # the scaling whose exp (the kernel's expf: here the host's libm) is the largest float at or below the threshold,
        # then the next one up: exp lands just below / on and just above it
        s = F(np.log(np.float64(t)))
        while _expf(s) > t:
            s = np.nextafter(s, F(-np.inf))
        while _expf(np.nextafter(s, F(np.inf))) <= t:
            s = np.nextafter(s, F(np.inf))
        for r, val in zip((S + 7, S + 8, S + 9), (np.nextafter(s, F(-np.inf)), s, np.nextafter(s, F(np.inf)))):
            st["params"][4][r] = torch.tensor([float(val), -9.0, -9.0])
        st["params"][4][S + 10:S + 40] = 0.5          # a block of big Gaussians
        st["params"][4][:4] = 0.5                     # big skybox rows are never rescaled
        # row 0 is a skybox row without a gradient of its own
        for v in grads.values():
            v[0] = 0
        act = CR.activate(st["params"])
    return st, act, grads, thr


@pytest.mark.parametrize("N,S,seed", [(1, 0, 1), (37, 4, 2), (300, 12, 3), (1000, 100, 4)])
def test_param_step_matches_restatement(emu, N, S, seed):
    import torch
    st, act, grads, thr = _case(N, S, seed, special=N >= 100)
    es = _EmuState(st, act, grads, thr)
    ref = CR.clone_state(st)
    relevant, act_ref = CR.param_step(ref, {k: v.clone() for k, v in act.items()}, grads, thr)
    es.run(emu, 0)
    assert int(es.step[0]) == ref["step"]
    if N >= 100:
        assert relevant.shape[0] > 0 and 0 not in relevant[:, 0].tolist()
        assert S + 5 not in relevant[:, 0].tolist() and S + 6 in relevant[:, 0].tolist()
    for k in range(6):
        exact = k != 5              # the rotation's gradient goes through F.normalize's backward (division, sqrt)
        for name, got, want in (("param", es.p[k], ref["params"][k]), ("exp_avg", es.m[k], ref["exp_avg"][k]),
                                ("exp_avg_sq", es.v[k], ref["exp_avg_sq"][k])):
            d = ulps(got, want.numpy())
            if k == 4 and name == "param":
                d = d.reshape(N, 3)[np.arange(N) != S + 9]     # row S+9's decision rests on the last ulp of exp (below)
                # the rescale's log(exp(s) * 0.8): host libm against torch's vectorised exp / log
                assert d.max() <= 2, (k, name, d.max())
            elif exact:
                assert d.max() == 0, (CR.GROUPS[k], name, d.max())
            else:
                assert d.max() <= 4, (CR.GROUPS[k], name, d.max())
    # untouched rows stay exactly as they were
    rows = set(relevant[:, 0].tolist()) | ({0} if relevant.shape[0] else set())
    still = np.array([i for i in range(N) if i not in rows], np.int64)
    if still.size:
        for k in range(6):
            assert np.array_equal(es.m[k][still], st["exp_avg"][k].numpy()[still])
    # the activated rows
    assert np.array_equal(es.act["means3D"], act_ref["means3D"].numpy())
    assert np.array_equal(es.act["shs"], act_ref["shs"].numpy())
    # exp of a rescaled scaling carries the 1-2 ulp of the host's log(exp(s) * 0.8f) times |s|
    for k, budget in (("opacities", 2), ("scales", 4), ("rotations", 4)):
        assert ulps(es.act[k], act_ref[k].numpy()).max() <= budget, k
    if N >= 100:
        # the threshold decisions: at and below it no rescale, one ulp above it rescales
        sc, sc0, scr = es.p[4], st["params"][4].numpy(), ref["params"][4].numpy()
        e7, e8, e9 = S + 7, S + 8, S + 9
        assert sc[e7, 0] == sc0[e7, 0] and sc[e8, 0] == sc0[e8, 0] and sc[e9, 0] != sc0[e9, 0]
        assert np.array_equal(sc[:4], sc0[:4]) or 0 in rows
        edge = np.isin(np.arange(N), (e7, e8, e9))
        assert np.array_equal((sc != sc0)[~edge], (scr != sc0)[~edge])

def test_no_relevant_row_takes_the_dense_step(emu):
    """an empty index sends OurAdam to its dense step (scene/OurAdam.py:214-228, _single_tensor_adam2): every row's
    moments decay and every row with momentum moves, though no opacity gradient is non-zero"""
    st, act, grads, thr = _case(50, 5, 9, special=False)
    grads["opacities"].zero_()
    es = _EmuState(st, act, grads, thr)
    ref = CR.clone_state(st)
    relevant, _ = CR.param_step(ref, {k: v.clone() for k, v in act.items()}, grads, thr)
    assert relevant.shape[0] == 0
    es.run(emu, 0)
    assert int(es.step[0]) == st["step"] + 1
    for k in range(6):
        assert not np.array_equal(es.m[k], st["exp_avg"][k].numpy())              # every row's moments decayed
        for got, want in ((es.m[k], ref["exp_avg"][k]), (es.v[k], ref["exp_avg_sq"][k]), (es.p[k], ref["params"][k])):
            assert ulps(got, want.numpy()).max() <= (4 if k >= 4 else 0), CR.GROUPS[k]
    moved = np.any(es.p[3] != st["params"][3].numpy(), axis=1)
    assert moved.all()                                                            # opacity moves by momentum alone


def test_overflowed_frame_changes_nothing(emu):
    st, act, grads, thr = _case(300, 12, 3)
    es = _EmuState(st, act, grads, thr, scan_info=[10, 5, 1])
    before = [x.copy() for x in es.p + es.m + es.v + list(es.act.values())]
    es.run(emu, 0)
    after = es.p + es.m + es.v + list(es.act.values())
    assert int(es.step[0]) == st["step"]
    assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(before, after))


def test_activation_mode_fills_the_scene(emu):
    import torch
    st, _, grads, thr = _case(200, 10, 11, special=False)
    act_ref = CR.activate(st["params"])
    zero = {k: torch.zeros_like(v) for k, v in act_ref.items()}
    es = _EmuState(st, zero, grads, thr)
    es.run(emu, 1)
    assert np.array_equal(es.act["means3D"], act_ref["means3D"].numpy()) and np.array_equal(es.act["shs"], act_ref["shs"].numpy())
    for k in ("opacities", "scales", "rotations"):
        assert ulps(es.act[k], act_ref[k].numpy()).max() <= 4, k


@pytest.mark.parametrize("step0", [0, 1, 999, 29_999])
def test_bias_corrections_are_the_host_doubles(emu, step0):
    st, act, grads, thr = _case(3, 0, 1, special=False)
    st["step"] = step0
    st["lr"] = [0.0, 0.0025, 0.000125, 0.05, 0.005, 0.001]
    es = _EmuState(st, act, grads, thr)
    es.run(emu, 2)
    sc = es.scratch[:48].view(F)
    for k in range(6):
        want = CR.bias_corrections(st["lr"][k], 0.9, 0.999, step0 + 1)
        assert sc[k] == want[0] and sc[6 + k] == want[1]
    assert int(es.step[0]) == step0


def test_densify_stats_max_radii_only(emu):
    from emu_api import aligned, f32, i32, ptr
    g = np.random.default_rng(2)
    P = 300
    radii = i32((g.integers(0, 30, P) * (g.uniform(size=P) > 0.4)).astype(np.int32))
    mr0 = g.uniform(0, 20, P).astype(F)
    mr = f32(mr0)
    emu.check(emu.L.h3dgs_densify_stats(P, ptr(radii), None, ptr(mr), None, None, None, None))
    vis = radii > 0
    assert np.array_equal(mr[vis], np.maximum(mr0[vis], radii[vis].astype(F))) and np.array_equal(mr[~vis], mr0[~vis])
    dm = f32(np.zeros((P, 3), F))
    assert emu.L.h3dgs_densify_stats(P, ptr(radii), ptr(dm), ptr(mr), ptr(f32(np.zeros(P, F))), None, None, None) < 0


# ---- against the reference's own GaussianModel, OurAdam and render_coarse (tests/golden/coarse_iteration.npz) ---------------
def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "coarse_iteration.npz"))


@pytest.mark.parametrize("c", range(4))
def test_restatement_is_the_reference_iteration(golden_dir, c):
    z = _golden(golden_dir)
    st = CR.golden_start(z, c)
    before = CR.clone_state(st)
    act, grads = CR.golden_inputs(z, c)
    relevant, _ = CR.param_step(st, act, grads, float(z["extent"]) * 0.1)
    assert np.array_equal(relevant.numpy(), z[f"c{c}_relevant"]) and st["step"] == int(z[f"c{c}_step"])
    # the stored gradients the reference's autograd formed (sigmoid / exp backward exactly, normalize's within ulp)
    sg = CR.stored_grads(before["params"], act, grads, int(z["skybox"]))
    for k, a in enumerate(CR.ATTRS):
        want = z[f"c{c}_grad{a}"]
        if k == 5:
            assert np.all(np.abs(sg[k].numpy() - want) <= CR.rotation_grad_tol(z, c, before["params"][5].numpy())), a
        else:
            assert np.array_equal(sg[k].numpy(), want), a
    bad = CR.golden_violations(z, c, before, [p.numpy() for p in st["params"]], [m.numpy() for m in st["exp_avg"]],
                               [v.numpy() for v in st["exp_avg_sq"]])
    assert not bad, bad


@pytest.mark.parametrize("c", range(4))
def test_kernel_is_the_reference_iteration(emu, golden_dir, c):
    z = _golden(golden_dir)
    st = CR.golden_start(z, c)
    act, grads = CR.golden_inputs(z, c)
    es = _EmuState(st, act, grads, float(z["extent"]) * 0.1)
    es.run(emu, 0)
    assert int(es.step[0]) == int(z[f"c{c}_step"])
    bad = CR.golden_violations(z, c, st, es.p, es.m, es.v)
    assert not bad, bad
    # the rows OurAdam left alone are untouched bit for bit, and the dense step of iteration 2 touched every row
    rows = z[f"c{c}_relevant"][:, 0]
    touched = np.zeros(len(es.m[3]), bool)
    if len(rows):
        touched[rows] = True
        touched[0] = True
    else:
        touched[:] = True
    assert np.array_equal(np.any(es.m[3] != st["exp_avg"][3].numpy(), axis=1), touched & np.any(es.m[3] != 0, axis=1) | (touched & np.any(st["exp_avg"][3].numpy() != 0, axis=1)))


@pytest.mark.parametrize("c", range(4))
def test_loss_pair_is_the_reference_objective(emu, golden_dir, c):
    z = _golden(golden_dir)
    img, gt = z[f"c{c}_image"], z[f"c{c}_gt"]
    M = z[f"c{c}_mask"] if int(z[f"c{c}_has_mask"]) else None
    lam, n = float(z["lam"]), float(img.size)
    assert img.max() > 1.0
    k0, k1 = F((1.0 - lam) / n), F(-lam / n)
    sums, grad = _loss_emu(emu, "coarse", img, gt, M, (k0, k1))
    l1, ssim = sums[0] / n, sums[1] / n
    assert abs(l1 - float(z[f"c{c}_l1"])) < 1e-6 and abs((1 - lam) * l1 + lam * (1 - ssim) - float(z[f"c{c}_loss"])) < 1e-6
    ref = z[f"c{c}_dimage"]
    assert np.abs(grad - ref).max() <= 1e-5 * np.abs(ref).max()

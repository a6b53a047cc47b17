"""CPU: train_single's parameter step (csrc/single_param.cu) on the emulation build, against tests/single_train_ref.py.

  * the full step: the skybox lock of all six stored gradients (locked and unlocked), the flattened relevance (no row 0
    of its own, zero / underflowing / NaN opacity gradients), this iteration's xyz lr from the device word, scaffold rows
    left alone by the rescale, violators at and one ulp around the threshold, the exposure's Adam on every image row;
    stored rows, moments, exposures and step counts bit for bit, the rows that pass through expf / logf / F.normalize
    within the ulp budget of tests/test_coarse_step_cpu.py (host libm against torch's CPU exp / log / sqrt);
  * OurAdam's dense step when no row is relevant;
  * the no-Gaussian-step mode: the exposure's Adam and the rescale, no Gaussian moment or step count touched;
  * the exposure row the forward reads;
  * an overflowed frame changes no byte of state;
  * the bias corrections of the prologue against the host's doubles."""
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
import single_train_ref as SR  # noqa: E402

F = np.float32
NAMES = ("means3D", "shs", "opacities", "scales", "rotations")
_SHIM = """#include <math.h>
static inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
static inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
static inline float __fsqrt_rn(float a) { volatile float r = sqrtf(a); return r; }
"""


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    import build_emu
    from emu_api import Emu
    out = str(tmp_path_factory.mktemp("h3dgs_emu_single"))
    build_emu.build(out)
    src = os.path.join(out, "hierarchical-3d-gaussians_b200", "csrc")
    with open(os.path.join(out, "shim.h"), "w") as f:
        f.write(_SHIM)
    flags = ["-std=c++17", "-O1", "-fPIC", "-ffp-contract=off", "-fno-strict-aliasing", "-w", "-D__CUDACC__",
             "-DH3_PAIR_HOST_EMU", "-DH3_HOST_EMU", "-I", src, "-include", os.path.join(out, "shim.h")]
    objs = [os.path.join(out, s.replace(".cu", ".o")) for s in build_emu.SOURCES] + [os.path.join(out, "simt_emu.o")]
    for name in ("coarse_param", "single_param"):
        obj = os.path.join(out, name + ".o")
        r = subprocess.run(["/usr/bin/g++"] + flags + ["-c", os.path.join(src, name + ".cpp"), "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[:4000]
        objs.append(obj)
    so = os.path.join(out, "libh3dgs_emu_single.so")
    r = subprocess.run(["/usr/bin/g++", "-shared", "-o", so] + objs + ["-lm", "-lpthread"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[:4000]
    return Emu(so)


def _expf(x):
    import ctypes.util
    libm = C.CDLL(ctypes.util.find_library("m"))
    libm.expf.restype, libm.expf.argtypes = C.c_float, [C.c_float]
    return F(libm.expf(float(x)))


def ulps(a, b):
    a, b = np.asarray(a, F).ravel(), np.asarray(b, F).ravel()
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    d = np.abs(ia - ib)
    d[np.isnan(a) & np.isnan(b)] = 0
    return d


class _EmuState:
    """host arrays of one single state and scene, and the h3dgs_single_args pointing at them"""

    def __init__(self, st, act, grads, threshold, xyz_lr, exposure_lr, image, exposure_grad, scan_info=None):
        from emu_api import aligned, f32
        from h3dgs import _lib
        self.p = [f32(x.numpy()) for x in st["params"]]
        self.m = [f32(x.numpy()) for x in st["exp_avg"]]
        self.v = [f32(x.numpy()) for x in st["exp_avg_sq"]]
        self.act = {k: f32(v.numpy()) for k, v in act.items()}
        self.g = {k: f32(v.numpy()) for k, v in grads.items()}
        self.step = aligned(8, np.int64, (1,))
        self.step[0] = st["step"]
        self.estep = aligned(8, np.int64, (1,))
        self.estep[0] = st["exposure_step"]
        self.ex, self.em, self.ev = f32(st["exposure"]), f32(st["exposure_m"]), f32(st["exposure_v"])
        self.egrad = f32(exposure_grad)
        self.row = f32(np.zeros((3, 4), F))
        self.lrs = aligned(16, np.float64, (2,))
        self.lrs[:] = (xyz_lr, exposure_lr)
        self.image = aligned(4, np.int32, (1,))
        self.image[0] = image
        self.scratch = aligned(64)
        self.info = None if scan_info is None else np.array(scan_info, np.uint32)
        s = self.s = _lib.SingleArgs()
        a = s.gauss
        a.N = st["params"][0].shape[0]
        a.sh_coeffs, a.skybox_points, a.rescale_threshold = st["params"][2].shape[1] + 1, st["skybox"], float(F(threshold))
        for k in range(6):
            a.params[k], a.exp_avg[k], a.exp_avg_sq[k] = self.p[k].ctypes.data, self.m[k].ctypes.data, self.v[k].ctypes.data
            a.lr[k], (a.beta1[k], a.beta2[k]), a.eps[k] = (st["lr"][k] if k else -1.0), st["betas"][k], st["eps"][k]
        a.step, a.scratch = self.step.ctypes.data, self.scratch.ctypes.data
        for k in NAMES:
            setattr(a, "grad_" + k, self.g[k].ctypes.data)
            setattr(a, k, self.act[k].ctypes.data)
        a.scan_info = None if self.info is None else self.info.ctypes.data
        s.skybox_locked, s.scaffold_points, s.n_images = int(st["skybox_locked"]), st["scaffold"], st["exposure"].shape[0]
        s.lrs, s.exposure, s.exposure_exp_avg, s.exposure_exp_avg_sq = (self.lrs.ctypes.data, self.ex.ctypes.data,
                                                                        self.em.ctypes.data, self.ev.ctypes.data)
        s.exposure_step, s.exposure_beta1, s.exposure_beta2, s.exposure_eps = self.estep.ctypes.data, 0.9, 0.999, 1e-8
        s.exposure_grad, s.image_index, s.exposure_row = self.egrad.ctypes.data, self.image.ctypes.data, self.row.ctypes.data

    def run(self, emu, mode):
        emu.check(emu.L.h3dgs_single_param_step(C.byref(self.s), mode, None))

    def everything(self):
        return self.p + self.m + self.v + list(self.act.values()) + [self.step, self.estep, self.ex, self.em, self.ev]


THR = 0.05
XYZ_LR, EXP_LR = 1.3e-4, 7e-4


def _case(N, S, seed, locked=True, scaffold=0, special=True):
    import torch
    st = SR.random_single_state(N, S, seed, skybox_locked=locked, scaffold=scaffold)
    grads = CR.random_grads(N, seed + 1, K=15)
    if special:
        op = st["params"][3]
        op[S + 5, 0] = 30.0                               # the stored opacity gradient underflows to 0: not relevant
        grads["opacities"][S + 5, 0] = 1e-30
        grads["opacities"][S + 6, 0] = float("nan")       # NaN != 0: relevant
        for r in (S + 7, S + 8, S + 9):                   # violators at / around the threshold, no Adam update
            for v in grads.values():
                v[r] = 0
        t = F(THR)
        s = F(np.log(np.float64(t)))
        while _expf(s) > t:
            s = np.nextafter(s, F(-np.inf))
        while _expf(np.nextafter(s, F(np.inf))) <= t:
            s = np.nextafter(s, F(np.inf))
        for r, val in zip((S + 7, S + 8, S + 9), (np.nextafter(s, F(-np.inf)), s, np.nextafter(s, F(np.inf)))):
            st["params"][4][r] = torch.tensor([float(val), -9.0, -9.0])
        st["params"][4][S + 10:S + 40] = 0.5              # big Gaussians
        st["params"][4][:4] = 0.5                         # big rows below the scaffold (when there is one)
        for v in grads.values():
            v[0] = 0                                      # row 0 has no gradient: the flattened index does not list it
    act = CR.activate(st["params"])
    eg = np.random.default_rng(seed + 2).normal(0, 1e-2, (3, 4)).astype(F)
    return st, act, grads, eg


def _reference(st, act, grads, eg, image, mode=0):
    ref = SR.clone_single(st)
    relevant = None
    a = {k: v.clone() for k, v in act.items()}
    ref["exposure_step"] += 1
    SR.exposure_adam(ref["exposure"], ref["exposure_m"], ref["exposure_v"], eg, image, EXP_LR, ref["exposure_step"])
    if mode == 0:
        relevant, a = SR.gaussian_step(ref, a, grads, THR, XYZ_LR)
    else:
        SR.rescale(ref["params"], THR, ref["scaffold"])
        a = CR.activate(ref["params"])
    return ref, relevant, a


def _compare(es, st, ref, act_ref, N, S, special):
    for k in range(6):
        for name, got, want in (("param", es.p[k], ref["params"][k]), ("exp_avg", es.m[k], ref["exp_avg"][k]),
                                ("exp_avg_sq", es.v[k], ref["exp_avg_sq"][k])):
            d = ulps(got, want.numpy())
            if k == 4 and name == "param":
                if special:
                    d = d.reshape(N, 3)[np.arange(N) != S + 9]
                # log(exp(s) * 0.8): the host's expf / logf and torch's CPU exp / log each within 1 ulp of the true
                # value: up to 2 ulp apart in log, plus exp's difference carried through the product
                assert d.max() <= 3, (name, d.max())
            else:
                assert d.max() <= (4 if k == 5 else 0), (CR.GROUPS[k], name, d.max())
    assert int(es.step[0]) == ref["step"] and int(es.estep[0]) == ref["exposure_step"]
    for x, y in ((es.ex, ref["exposure"]), (es.em, ref["exposure_m"]), (es.ev, ref["exposure_v"])):
        assert np.array_equal(x.view(np.int32), y.view(np.int32))
    assert np.array_equal(es.act["means3D"], act_ref["means3D"].numpy()) and np.array_equal(es.act["shs"], act_ref["shs"].numpy())
    for k, budget in (("opacities", 2), ("rotations", 4)):
        assert ulps(es.act[k], act_ref[k].numpy()).max() <= budget, k
    # exp of a rescaled scaling carries the 2 ulp of the host's log(exp(s) * 0.8f), relative 2 |s| 2^-23: 2 |s| ulp of exp
    s_ref = np.abs(ref["params"][4].numpy()).ravel()
    assert np.all(ulps(es.act["scales"], act_ref["scales"].numpy()) <= 4 + 2 * np.ceil(s_ref)), "scales"


@pytest.mark.parametrize("N,S,seed,locked,scaffold", [(1, 0, 1, True, 0), (40, 4, 2, False, 0), (300, 12, 3, True, 0),
                                                      (300, 12, 4, False, 0), (1000, 100, 5, True, 60)])
def test_step_matches_restatement(emu, N, S, seed, locked, scaffold):
    special = N >= 100
    st, act, grads, eg = _case(N, S, seed, locked, scaffold, special)
    image = seed % 4
    es = _EmuState(st, act, grads, THR, XYZ_LR, EXP_LR, image, eg)
    ref, relevant, act_ref = _reference(st, act, grads, eg, image)
    es.run(emu, 0)
    _compare(es, st, ref, act_ref, N, S, special)
    rel = set(relevant.tolist())
    if special:
        assert 0 not in rel and S + 5 not in rel and S + 6 in rel
        assert all(r >= S for r in rel) if locked else any(r < S for r in rel)
        # untouched rows keep their moments: the flattened index adds no row 0
        assert np.array_equal(es.m[3][0], st["exp_avg"][3].numpy()[0])
        sc, sc0 = es.p[4], st["params"][4].numpy()
        assert sc[S + 7, 0] == sc0[S + 7, 0] and sc[S + 8, 0] == sc0[S + 8, 0] and sc[S + 9, 0] != sc0[S + 9, 0]
        # rows below the scaffold are never rescaled; above it the big rows are
        if scaffold:
            assert np.array_equal(sc[:4], sc0[:4]) and np.all(sc[S + 10:S + 40] < sc0[S + 10:S + 40])
    # every exposure row moved, the image's with its gradient, the others as their moments decay
    assert np.all(np.any(es.ex != st["exposure"], axis=(1, 2)))


def test_no_relevant_row_takes_the_dense_step(emu):
    st, act, grads, eg = _case(50, 5, 9, special=False)
    grads["opacities"].zero_()
    es = _EmuState(st, act, grads, THR, XYZ_LR, EXP_LR, 1, eg)
    ref, relevant, act_ref = _reference(st, act, grads, eg, 1)
    assert relevant.shape[0] == 0
    es.run(emu, 0)
    _compare(es, st, ref, act_ref, 50, 5, False)
    assert np.all(np.any(es.m[3] != st["exp_avg"][3].numpy(), axis=1))         # every row's moments decayed


def test_skybox_lock_zeroes_all_six_gradients(emu):
    """a locked row with gradients everywhere: on a dense step it moves by momentum alone, as with zero gradients"""
    st, act, grads, eg = _case(64, 16, 12, locked=True, special=False)
    grads["opacities"][16:] = 0                              # dense step; the locked rows carry gradients
    es = _EmuState(st, act, grads, THR, XYZ_LR, EXP_LR, 0, eg)
    zero = {k: v.clone() for k, v in grads.items()}
    for v in zero.values():
        v[:16] = 0
    es0 = _EmuState(st, act, zero, THR, XYZ_LR, EXP_LR, 0, eg)
    es.run(emu, 0)
    es0.run(emu, 0)
    for a, b in zip(es.everything(), es0.everything()):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_no_gaussian_step_mode(emu):
    st, act, grads, eg = _case(300, 12, 3, scaffold=20)
    es = _EmuState(st, act, grads, THR, XYZ_LR, EXP_LR, 2, eg)
    ref, _, act_ref = _reference(st, act, grads, eg, 2, mode=1)
    es.run(emu, 1)
    assert int(es.step[0]) == st["step"] and int(es.estep[0]) == st["exposure_step"] + 1
    for k in range(6):
        assert np.array_equal(es.m[k], st["exp_avg"][k].numpy()) and np.array_equal(es.v[k], st["exp_avg_sq"][k].numpy())
        if k != 4:
            assert np.array_equal(es.p[k], st["params"][k].numpy())
    for x, y in ((es.ex, ref["exposure"]), (es.em, ref["exposure_m"]), (es.ev, ref["exposure_v"])):
        assert np.array_equal(x.view(np.int32), y.view(np.int32))
    d = ulps(es.p[4], ref["params"][4].numpy()).reshape(300, 3)
    assert d[np.arange(300) != 12 + 9].max() <= 2
    assert np.all(es.p[4][22:52] < st["params"][4].numpy()[22:52])        # big rows past the scaffold were rescaled
    # only the rescaled rows' activations were rewritten
    changed = np.any(es.p[4] != st["params"][4].numpy(), axis=1)
    assert np.array_equal(np.any(es.act["scales"] != act["scales"].numpy(), axis=1), changed)


def test_exposure_row(emu):
    st, act, grads, eg = _case(8, 0, 4, special=False)
    for image in range(4):
        es = _EmuState(st, act, grads, THR, XYZ_LR, EXP_LR, image, eg)
        before = [x.copy() for x in es.everything()]
        es.run(emu, 2)
        assert np.array_equal(es.row, st["exposure"][image])
        assert all(np.array_equal(a, b) for a, b in zip(before, es.everything()))


def test_overflowed_frame_changes_nothing(emu):
    st, act, grads, eg = _case(300, 12, 3)
    for mode in (0, 1):
        es = _EmuState(st, act, grads, THR, XYZ_LR, EXP_LR, 1, eg, scan_info=[10, 5, 1])
        before = [x.copy() for x in es.everything()]
        es.run(emu, mode)
        assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(before, es.everything()))


@pytest.mark.parametrize("step0", [0, 1, 999, 29_999])
def test_bias_corrections_are_the_host_doubles(emu, step0):
    st, act, grads, eg = _case(3, 0, 1, special=False)
    st["step"], st["exposure_step"] = step0, step0 + 3
    es = _EmuState(st, act, grads, THR, XYZ_LR, EXP_LR, 0, eg)
    es.run(emu, 3)
    sc = es.scratch[:60].view(F)
    for k in range(6):
        want = CR.bias_corrections(XYZ_LR if k == 0 else st["lr"][k], 0.9, 0.999, step0 + 1)
        assert sc[k] == want[0] and sc[6 + k] == want[1], k
    assert (sc[13], sc[14]) == SR.exposure_bias(EXP_LR, 0.9, 0.999, step0 + 4)
    assert int(es.step[0]) == step0 and int(es.estep[0]) == step0 + 3


# ---- against the reference's own GaussianModel, OurAdam, exposure_optimizer and render() (tests/golden/single_train.npz)
def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "single_train.npz"))


def _check_golden(z, c, before, p, m, v, ex, em, ev, step, estep, skip_rows=()):
    gstep = bool(z[f"c{c}_gstep"])
    assert step == int(z[f"c{c}_step"]) and estep == int(z[f"c{c}_exposure_step"])
    if gstep:
        bad = CR.golden_violations(z, c, before, p, m, v, skip_rows=skip_rows)
    else:
        bad = SR.golden_no_step_violations(z, c, before, p, m, v, skip_rows=skip_rows)
    bad += SR.golden_exposure_violations(z, c, before, ex, em, ev)
    assert not bad, bad


@pytest.mark.parametrize("c", range(6))
def test_restatement_is_the_reference_iteration(golden_dir, c):
    z = _golden(golden_dir)
    st = SR.golden_start(z, c)
    before = SR.clone_single(st)
    relevant = SR.golden_iteration(z, c, st)
    if relevant is not None:
        # the flattened index of the reference, and the stored gradients its autograd and lock formed
        assert np.array_equal(relevant.numpy(), z[f"c{c}_relevant"])
        act, grads = CR.golden_inputs(z, c)
        sg = CR.stored_grads(before["params"], act, grads, 0)
        if before["skybox_locked"]:
            for g in sg:
                g[:before["skybox"]] = 0
        for k, a in enumerate(CR.ATTRS):
            want = z[f"c{c}_grad{a}"]
            if k == 5:
                assert np.all(np.abs(sg[k].numpy() - want) <= CR.rotation_grad_tol(z, c, before["params"][5].numpy())), a
            else:
                assert np.array_equal(sg[k].numpy(), want), a
    _check_golden(z, c, before, [x.numpy() for x in st["params"]], [x.numpy() for x in st["exp_avg"]],
                  [x.numpy() for x in st["exp_avg_sq"]], st["exposure"], st["exposure_m"], st["exposure_v"], st["step"],
                  st["exposure_step"])


def test_golden_covers_the_listed_iterations(golden_dir):
    z = _golden(golden_dir)
    its = range(int(z["iterations"]))
    degrees = [int(z[f"c{c}_degree"]) for c in its]
    assert degrees[0] == 0 and degrees[-1] == 1                                   # the degree step at 1000
    assert {bool(z[f"c{c}_locked"]) for c in its} == {True, False}
    gsteps = [bool(z[f"c{c}_gstep"]) for c in its]
    assert gsteps.count(False) == 2                                               # densify, reset
    assert any(g and len(z[f"c{c}_relevant"]) == 0 for c, g in zip(its, gsteps))  # a dense step
    assert len({int(z[f"c{c}_image"]) for c in its}) >= 3
    assert int(z["c2_step"]) == int(z["c3_step"]) and int(z["c2_exposure_step"]) + 1 == int(z["c3_exposure_step"])
    assert z["c3_after_xyz"].shape[0] != z["c2_after_xyz"].shape[0]               # densify_and_prune changed N


@pytest.mark.parametrize("c", range(6))
def test_kernel_is_the_reference_iteration(emu, golden_dir, c):
    import torch
    z = _golden(golden_dir)
    st = SR.golden_start(z, c)
    image, xyz_lr, exp_lr, eg, gstep, thr = SR.golden_frame(z, c)
    if gstep:
        act, grads = CR.golden_inputs(z, c)
    else:
        act = CR.activate(st["params"])
        grads = {k: torch.zeros_like(v) for k, v in act.items()}
    es = _EmuState(st, act, grads, thr, xyz_lr, exp_lr, image, eg)
    es.run(emu, 0 if gstep else 1)
    # the threshold-edge rows were placed with torch's CPU exp; the emulation build decides with the host's expf
    _check_golden(z, c, st, es.p, es.m, es.v, es.ex, es.em, es.ev, int(es.step[0]), int(es.estep[0]),
                  skip_rows=[int(r) for r in z["edges"]])

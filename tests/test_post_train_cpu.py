"""CPU: train_post's parameter step (csrc/post_param.cu) on the emulation build, against tests/post_train_ref.py.

  * the step: abs's backward on stored opacities of both signs and exactly +-0 (NaN gradients included), the locks
    (anchors with duplicates, negative indices and a skybox row; the skybox tail locked and not; no lock at all), the
    dense Adam step that moves rows without a gradient on their moments alone, this iteration's xyz lr from the device
    word; stored rows, moments and step count bit for bit, the rotation group and the activations through expf /
    F.normalize within the ulp budget of tests/test_single_train_cpu.py; N = 1 and N > 2^16;
  * a locked row with gradients steps exactly as one without;
  * the activation mode;
  * a binning overflow and a row overflow (the cut plus the skybox rows past the row capacity) change no byte of state,
    a cut that just fits steps;
  * the bias corrections of the prologue against the host's doubles;
  * PostState's lock mask: anchors in range, duplicates, negatives, skybox tail, and out-of-range anchors refused;
  * against the reference's own create_from_hier model, torch.optim.Adam, render_post and train_post lines
    (tests/golden/post_train.npz): the fixture covers what it claims, the restatement's stored gradients are the
    reference's autograd and lock lines', and the restatement and the kernel land on the reference's state within the
    derived budget of post_train_ref.golden_violations."""
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
import post_train_ref as PR  # noqa: E402
import single_train_ref as SR  # noqa: E402

F = np.float32
NAMES = ("means3D", "shs", "opacities", "scales", "rotations")
_SHIM = """#include <math.h>
static inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
static inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
static inline float __fsqrt_rn(float a) { volatile float r = sqrtf(a); return r; }
"""
XYZ_LR = 1.3e-4


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    import build_emu
    from emu_api import Emu
    out = str(tmp_path_factory.mktemp("h3dgs_emu_post"))
    build_emu.build(out)
    src = os.path.join(out, "hierarchical-3d-gaussians_b200", "csrc")
    with open(os.path.join(out, "shim.h"), "w") as f:
        f.write(_SHIM)
    flags = ["-std=c++17", "-O1", "-fPIC", "-ffp-contract=off", "-fno-strict-aliasing", "-w", "-D__CUDACC__",
             "-DH3_PAIR_HOST_EMU", "-DH3_HOST_EMU", "-I", src, "-include", os.path.join(out, "shim.h")]
    objs = [os.path.join(out, s.replace(".cu", ".o")) for s in build_emu.SOURCES] + [os.path.join(out, "simt_emu.o")]
    obj = os.path.join(out, "post_param.o")
    r = subprocess.run(["/usr/bin/g++"] + flags + ["-c", os.path.join(src, "post_param.cpp"), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[:4000]
    so = os.path.join(out, "libh3dgs_emu_post.so")
    r = subprocess.run(["/usr/bin/g++", "-shared", "-o", so] + objs + [obj, "-lm", "-lpthread"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[:4000]
    return Emu(so)


def ulps(a, b):
    a, b = np.asarray(a, F).ravel(), np.asarray(b, F).ravel()
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    d = np.abs(ia - ib)
    d[np.isnan(a) & np.isnan(b)] = 0
    return d


class _EmuPost:
    """host arrays of one post state and scene, and the h3dgs_post_args pointing at them"""

    def __init__(self, st, act, grads, xyz_lr, locked=None, scan_info=None, count=None, extra_rows=0, row_capacity=0):
        from emu_api import aligned, f32
        from h3dgs import _lib
        self.p = [f32(x.numpy()) for x in st["params"]]
        self.m = [f32(x.numpy()) for x in st["exp_avg"]]
        self.v = [f32(x.numpy()) for x in st["exp_avg_sq"]]
        self.act = {k: f32(v.numpy()) for k, v in act.items()}
        self.g = {k: f32(v.numpy()) for k, v in grads.items()}
        self.step = aligned(8, np.int64, (1,))
        self.step[0] = st["step"]
        self.lrs = aligned(8, np.float64, (1,))
        self.lrs[0] = xyz_lr
        self.scratch = aligned(64)
        self.locked = None if locked is None else np.ascontiguousarray(locked.numpy().astype(np.uint8))
        self.info = None if scan_info is None else np.array(scan_info, np.uint32)
        self.count = None if count is None else np.array([count], np.int32)
        s = self.s = _lib.PostArgs()
        a = s.gauss
        a.N, a.sh_coeffs, a.skybox_points = st["params"][0].shape[0], st["params"][2].shape[1] + 1, st["skybox"]
        for k in range(6):
            a.params[k], a.exp_avg[k], a.exp_avg_sq[k] = self.p[k].ctypes.data, self.m[k].ctypes.data, self.v[k].ctypes.data
            a.lr[k], (a.beta1[k], a.beta2[k]), a.eps[k] = (st["lr"][k] if k else -1.0), st["betas"][k], st["eps"][k]
        a.step, a.scratch = self.step.ctypes.data, self.scratch.ctypes.data
        for k in NAMES:
            setattr(a, "grad_" + k, self.g[k].ctypes.data)
            setattr(a, k, self.act[k].ctypes.data)
        a.scan_info = None if self.info is None else self.info.ctypes.data
        s.lrs = self.lrs.ctypes.data
        s.locked = None if self.locked is None else self.locked.ctypes.data
        s.count = None if self.count is None else self.count.ctypes.data
        s.extra_rows, s.row_capacity = extra_rows, row_capacity

    def run(self, emu, mode):
        emu.check(emu.L.h3dgs_post_param_step(C.byref(self.s), mode, None))

    def everything(self):
        return self.p + self.m + self.v + list(self.act.values()) + [self.step]


def _case(N, S, seed):
    st = PR.random_post_state(N, S, seed)
    grads = CR.random_grads(N, seed + 1, K=15)
    if N > 10:
        grads["opacities"][3, 0] = float("nan")                           # sign(o) of a NaN gradient: NaN or 0 * NaN
        st["params"][3][4, 0] = float("nan")                             # sign(NaN) = 0: the gradient is +-0
        st["params"][5][5] = 0.0                                          # |q| = 0: F.normalize's clamp
    act = PR.activate(st["params"])
    return st, act, grads


def _compare(es, ref, act_ref):
    for k in range(6):
        for name, got, want in (("param", es.p[k], ref["params"][k]), ("exp_avg", es.m[k], ref["exp_avg"][k]),
                                ("exp_avg_sq", es.v[k], ref["exp_avg_sq"][k])):
            # the rotation group's gradient is F.normalize's backward (host libm's sqrt against torch's CPU ops)
            assert ulps(got, want.numpy()).max() <= (4 if k == 5 else 0), (CR.GROUPS[k], name)
    assert int(es.step[0]) == ref["step"]
    for k in ("means3D", "shs", "opacities"):
        assert np.array_equal(es.act[k].view(np.int32), act_ref[k].numpy().view(np.int32)), k
    # expf of the host against torch's CPU exp, each within 1 ulp; the normalize within the rotation budget
    assert ulps(es.act["scales"], act_ref["scales"].numpy()).max() <= 2
    assert ulps(es.act["rotations"], act_ref["rotations"].numpy()).max() <= 4


@pytest.mark.parametrize("N,S,locked_sky,anchors,seed", [
    (1, 0, True, [], 1),                                     # one row, no skybox, no anchor: no mask at all
    (300, 12, True, [3, 3, 299, -2, 40], 2),                 # duplicates, a skybox row, a negative index
    (300, 12, False, [7], 3),                                # the skybox unlocked
    (400, 0, True, [], 4),                                   # no skybox, nothing locked
    (70_000, 100, True, [0, 65_536, 69_999, 65_536], 5)])   # more rows than 2^16
def test_step_matches_restatement(emu, N, S, locked_sky, anchors, seed):
    st, act, grads = _case(N, S, seed)
    mask = PR.locked_mask(N, S, locked_sky, anchors)
    es = _EmuPost(st, act, grads, XYZ_LR, mask if bool(mask.any()) else None)
    ref = CR.clone_state(st)
    act_ref = PR.param_step(ref, act, grads, XYZ_LR, mask)
    es.run(emu, 0)
    _compare(es, ref, act_ref)
    # the dense step: rows without a gradient move on their moments alone, as do the locked ones
    still = np.all(grads["means3D"].numpy() == 0, axis=1)
    if still.any():
        r = int(np.nonzero(still)[0][0])
        assert np.any(es.p[0][r] != st["params"][0].numpy()[r]) and np.any(es.m[0][r] != st["exp_avg"][0].numpy()[r])
    # abs folds negative stored opacities back
    assert np.all(es.act["opacities"][~np.isnan(es.act["opacities"])] >= 0)


def test_locked_row_steps_as_a_row_without_gradients(emu):
    N, S = 64, 16
    st, act, grads = _case(N, S, 12)
    mask = PR.locked_mask(N, S, True, [20, 33])
    es = _EmuPost(st, act, grads, XYZ_LR, mask)
    zero = {k: v.clone() for k, v in grads.items()}
    for v in zero.values():
        v[mask] = 0
    es0 = _EmuPost(st, act, zero, XYZ_LR, None)
    es.run(emu, 0)
    es0.run(emu, 0)
    for a, b in zip(es.everything(), es0.everything()):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_activate_mode(emu):
    st, act, grads = _case(300, 10, 6)
    blank = {k: np.zeros_like(v) for k, v in act.items()}
    import torch
    es = _EmuPost(st, {k: torch.tensor(v) for k, v in blank.items()}, grads, XYZ_LR)
    es.s.gauss.step = es.s.gauss.scratch = None
    es.s.lrs = None
    es.run(emu, 1)
    for k in ("means3D", "shs", "opacities"):
        assert np.array_equal(es.act[k].view(np.int32), act[k].numpy().view(np.int32)), k
    assert ulps(es.act["scales"], act["scales"].numpy()).max() <= 1
    assert ulps(es.act["rotations"], act["rotations"].numpy()).max() <= 4
    for a, b in zip(es.p + es.m + es.v, st["params"] + st["exp_avg"] + st["exp_avg_sq"]):
        assert np.array_equal(a.view(np.uint8), b.numpy().view(np.uint8))


@pytest.mark.parametrize("kind", ["bin", "rows"])
def test_overflowed_frame_changes_nothing(emu, kind):
    N, S = 300, 12
    st, act, grads = _case(N, S, 3)
    kw = dict(scan_info=[10, 5, 1]) if kind == "bin" else dict(scan_info=[10, 5, 0], count=200, extra_rows=S, row_capacity=211)
    es = _EmuPost(st, act, grads, XYZ_LR, PR.locked_mask(N, S, True, [1]), **kw)
    before = [x.copy() for x in es.everything()]
    es.run(emu, 0)
    assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(before, es.everything()))
    if kind == "rows":
        # the same frame with the cut that just fits: it steps
        es = _EmuPost(st, act, grads, XYZ_LR, None, scan_info=[10, 5, 0], count=200, extra_rows=S, row_capacity=212)
        es.run(emu, 0)
        assert int(es.step[0]) == st["step"] + 1 and not np.array_equal(es.p[3], before[3])


@pytest.mark.parametrize("step0", [0, 1, 999, 29_999])
def test_bias_corrections_are_the_host_doubles(emu, step0):
    st, act, grads = _case(3, 0, 1)
    st["step"] = step0
    es = _EmuPost(st, act, grads, XYZ_LR)
    es.run(emu, 2)
    sc = es.scratch[:48].view(F)
    for k in range(6):
        want = SR.exposure_bias(XYZ_LR if k == 0 else st["lr"][k], 0.9, 0.999, step0 + 1)
        assert sc[k] == want[0] and sc[6 + k] == want[1], k
    assert int(es.step[0]) == step0


def _state(N, S, locked_sky, anchors):
    import torch
    from h3dgs.poststep import PostState
    st = PR.random_post_state(N, S, 9)
    return PostState(st["params"], S, st["lr"], torch.zeros((N, 2), dtype=torch.int32), torch.zeros((N, 2, 4)),
                     skybox_locked=locked_sky, anchors=anchors)


@pytest.mark.parametrize("N,S,locked_sky,anchors", [(10, 0, True, []), (10, 3, True, []), (10, 3, False, [2, 2, -1]),
                                                    (10, 0, False, None), (10, 4, True, [0, 9])])
def test_lock_mask(N, S, locked_sky, anchors):
    s = _state(N, S, locked_sky, anchors)
    want = PR.locked_mask(N, S, locked_sky, anchors or [])
    if not bool(want.any()):
        assert s.locked is None
    else:
        assert np.array_equal(s.locked.numpy().astype(bool), want.numpy())


@pytest.mark.parametrize("anchors", [[10], [-11], [0, 3, 12]])
def test_out_of_range_anchor_is_refused(anchors):
    with pytest.raises(ValueError):
        _state(10, 2, True, anchors)


# ---- against the reference's own create_from_hier, torch.optim.Adam, render_post and train_post lines ------------------
def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "post_train.npz"))


def test_golden_covers_the_listed_iterations(golden_dir):
    z = _golden(golden_dir)
    its = range(int(z["iterations"]))
    N, S, P = z["init__xyz"].shape[0], int(z["skybox"]), int(z["hier_rows"])
    assert N == P + S and S > 0
    assert {bool(z[f"c{c}_locked"]) for c in its} == {True, False}
    a = [int(x) for x in z["anchors"]]
    assert len(set(a)) < len(a) and any(x >= P for x in a)                     # a duplicate and a skybox row
    op = z["init__opacity"].ravel()
    assert (op < 0).any() and ((op == 0) & ~np.signbit(op)).any() and ((op == 0) & np.signbit(op)).any()
    assert len({float(z[f"c{c}_xyz_lr"]) for c in its}) == len(its)           # a changing xyz lr
    assert 2 in {int(z[f"c{c}_image"]) for c in its}                          # img2 has no exposure
    for c in its:
        ri, pi = set(z[f"c{c}_render_indices"].tolist()), set(z[f"c{c}_parent_indices"].tolist())
        g = np.abs(z[f"c{c}_actgrad_opacities"]).ravel()
        # a parent outside the cut receives lerp gradients; a row in neither has none and still moves (dense step)
        assert any(g[r] > 0 for r in pi - ri)
        idle = [r for r in range(P) if r not in ri and r not in pi]
        assert all(g[r] == 0 for r in idle)
        if c:
            # idle rows with moments from earlier cuts move on them alone
            before, m0 = z[f"c{c - 1}_after_xyz"], z[f"c{c - 1}_m_xyz"]
            coasting = [r for r in idle if np.all(m0[r] != 0)]
            assert coasting and all(np.all(z[f"c{c}_after_xyz"][r] != before[r]) for r in coasting)


@pytest.mark.parametrize("c", range(4))
def test_restatement_is_the_reference_iteration(golden_dir, c):
    import torch
    z = _golden(golden_dir)
    st = PR.golden_start(z, c)
    before = CR.clone_state(st)
    act, grads = CR.golden_inputs(z, c)
    mask = PR.golden_locked(z, c)
    # the stored gradients the reference's autograd (abs, exp, normalize, cat) and lock lines formed
    sg = PR.stored_grads(before["params"], act, grads, mask)
    for k, a in enumerate(CR.ATTRS):
        want = z[f"c{c}_grad{a}"]
        if k == 5:
            assert np.all(np.abs(sg[k].numpy() - want) <= CR.rotation_grad_tol(z, c, before["params"][5].numpy())), a
        else:
            assert np.array_equal(sg[k].numpy().view(np.int32), want.view(np.int32)), a
    # the activated rows render_post read are the restatement's activations of the stored tensors
    act_ref = PR.activate(before["params"])
    for k in ("means3D", "shs", "opacities", "scales"):
        assert np.array_equal(act_ref[k].numpy(), z[f"c{c}_act_{k}"]), k
    PR.param_step(st, act, grads, float(z[f"c{c}_xyz_lr"]), mask)
    assert st["step"] == int(z[f"c{c}_step"])
    bad = PR.golden_violations(z, c, before, [x.numpy() for x in st["params"]], [x.numpy() for x in st["exp_avg"]],
                               [x.numpy() for x in st["exp_avg_sq"]])
    assert not bad, bad


@pytest.mark.parametrize("c", range(4))
def test_kernel_is_the_reference_iteration(emu, golden_dir, c):
    z = _golden(golden_dir)
    st = PR.golden_start(z, c)
    act, grads = CR.golden_inputs(z, c)
    es = _EmuPost(st, act, grads, float(z[f"c{c}_xyz_lr"]), PR.golden_locked(z, c))
    es.run(emu, 0)
    assert int(es.step[0]) == int(z[f"c{c}_step"])
    bad = PR.golden_violations(z, c, st, es.p, es.m, es.v)
    assert not bad, bad

"""CPU: train_single's densify_and_prune and reset_opacity (csrc/densify.cu, SingleState.densify_and_prune /
reset_opacity) on the emulation build, against tests/densify_ref.py, and both against the reference's own
GaussianModel (tests/golden/densify.npz).

  * the restatement reproduces the fixture: row order, flags, counts, moments and statistics exactly; rows through exp /
    log / pow within the host-libm ulp budget of test_single_train_cpu.py; split positions within the budget of a
    reordered three-term product (the fixture's CPU bmm);
  * the kernels through SingleState match the restatement bit for bit (the emulation build calls the same libm), on
    the fixture's cases and on random states, with an under- and an overflowing sqrt(g * g);
  * reset_opacity changes only the opacity past the skybox and zeroes both opacity moments;
  * argument errors raise."""
import ctypes as C
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "emul"))

import densify_ref as D  # noqa: E402

F = np.float32
_SHIM = """#include <math.h>
#include <stdint.h>
static inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
static inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
static inline float __fsqrt_rn(float a) { volatile float r = sqrtf(a); return r; }
"""
CASES = ("edges", "no_split", "no_clone", "no_prune", "all_pruned")


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    import build_emu
    out = str(tmp_path_factory.mktemp("h3dgs_emu_densify"))
    build_emu.build(out)
    src = os.path.join(out, "hierarchical-3d-gaussians_b200", "csrc")
    with open(os.path.join(out, "shim.h"), "w") as f:
        f.write(_SHIM)
    flags = ["-std=c++17", "-O1", "-fPIC", "-ffp-contract=off", "-fno-strict-aliasing", "-w", "-D__CUDACC__",
             "-DH3_PAIR_HOST_EMU", "-DH3_HOST_EMU", "-I", src, "-include", os.path.join(out, "shim.h")]
    objs = [os.path.join(out, s.replace(".cu", ".o")) for s in build_emu.SOURCES] + [os.path.join(out, "simt_emu.o")]
    obj = os.path.join(out, "densify.o")
    r = subprocess.run(["/usr/bin/g++"] + flags + ["-c", os.path.join(src, "densify.cpp"), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[:4000]
    so = os.path.join(out, "libh3dgs_emu_densify.so")
    r = subprocess.run(["/usr/bin/g++", "-shared", "-o", so] + objs + [obj, "-lm", "-lpthread"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[:4000]
    return so


@pytest.fixture
def emu(emu_so):
    from fake_device import cpu_as_device
    with cpu_as_device(emu_so) as L:
        yield L


@pytest.fixture(scope="module")
def z(golden_dir):
    return np.load(os.path.join(golden_dir, "densify.npz"))


def _inputs(z, name):
    p = [z[f"{name}_p{k}"] for k in range(6)]
    m = [z[f"{name}_m{k}"] for k in range(6)]
    v = [z[f"{name}_v{k}"] for k in range(6)]
    return p, m, v


def _state(p, m, v, g=None, r=None, scaffold=0, skybox=0, percent_dense=0.01, step=7):
    from h3dgs.pipeline import DensifyStats
    from h3dgs.singlestep import SingleState
    N = p[0].shape[0]
    stats = DensifyStats(N, "cpu")
    if g is not None:
        stats.xyz_gradient_accum.copy_(torch.tensor(np.asarray(g, F)).reshape(N, 1))
        stats.max_radii2D.copy_(torch.tensor(np.asarray(r, F)))
        stats.denom.fill_(1.0)
    t = lambda a: [torch.tensor(np.asarray(x, F)) for x in a]
    return SingleState(t(p), skybox, [0.0] * 6, torch.eye(3, 4)[None].repeat(2, 1, 1), exp_avg=t(m), exp_avg_sq=t(v),
                       step=step, stats=stats, scaffold_points=scaffold, exposure_step=5, percent_dense=percent_dense)


def _check_against(st, ref, exact=True):
    """the state after the kernel against the restatement's result"""
    K, Cn, S, N2 = ref["counts"]
    assert st.N == N2 and st.counts == dict(kept=K, cloned=Cn, split=S)
    for k in range(6):
        for got, want in ((st.params[k], ref["params"][k]), (st.exp_avg[k], ref["exp_avg"][k]),
                          (st.exp_avg_sq[k], ref["exp_avg_sq"][k])):
            got = got.numpy()
            assert got.shape == want.shape
            if exact:
                assert np.array_equal(got.view(np.int32), want.view(np.int32)), D.GROUPS[k]
    for t in (st.stats.max_radii2D, st.stats.xyz_gradient_accum, st.stats.denom):
        assert t.shape[0] == N2 and not t.any()
    assert st.max_radii2D is st.stats.max_radii2D


# ---- the restatement against the reference ---------------------------------------------------------------------
def _golden_violations(z, name, out):
    """out: dict(params, exp_avg, exp_avg_sq) -> list of what differs from the fixture beyond its budget"""
    bad = []
    Ks = [z[f"{name}_out_p{k}"].shape[0] for k in range(6)]
    if any(o.shape[0] != Ks[0] for o in out["params"]):
        return [f"rows {[o.shape[0] for o in out['params']]} != {Ks}"]
    N2 = Ks[0]
    S = z[f"{name}_normals"].shape[0] // 2 if f"{name}_normals" in z else 0
    split0 = N2 - 2 * S
    for k in range(6):
        for key, got in (("p", out["params"][k]), ("m", out["exp_avg"][k]), ("v", out["exp_avg_sq"][k])):
            want = z[f"{name}_out_{key}{k}"]
            if key == "p" and k == 0 and S:
                mag = out["mag"] if "mag" in out else None
                w, g_ = want[split0:], got[split0:]
                if not np.array_equal(got[:split0].view(np.int32), want[:split0].view(np.int32)):
                    bad.append("xyz of the rows before the split copies")
                if np.any(np.abs(g_ - w) > D.position_budget(g_, w, mag)):
                    bad.append(f"split positions: {np.abs(g_ - w).max()}")
            elif key == "p" and k == 4 and S:
                # log(exp(s) * (1 / 1.6f)) against the CPU's log(exp(s) / 1.6f): the reciprocal's rounding (relative
                # 2^-24) and each side's exp and log within 1 ulp: at most 3 ulp of log plus 2 |s| ulp carried
                d = D.ulps(got[split0:], want[split0:]).reshape(-1, 3)
                lim = 3 + 2 * np.ceil(np.abs(want[split0:]))
                if np.any(d > lim) or not np.array_equal(got[:split0].view(np.int32), want[:split0].view(np.int32)):
                    bad.append(f"split scalings: {d.max()} ulp")
            elif not np.array_equal(got.view(np.int32), want.view(np.int32)):
                bad.append(f"{key}{k}: {D.ulps(got, want).max()} ulp")
    return bad


def _ref(z, name, normals=None, M=D.HOST):
    p, m, v = _inputs(z, name)
    T = F(float(z["percent_dense"]) * float(z["extent"]))
    return D.densify(p, m, v, z[f"{name}_gacc"], z[f"{name}_radii"], int(z[f"{name}_scaffold"]), float(z["max_grad"]),
                     float(z["min_opacity"]), T, z[f"{name}_normals"] if normals is None else normals, M)


@pytest.mark.parametrize("name", CASES)
def test_restatement_is_the_reference(z, name):
    out = _ref(z, name)
    assert not _golden_violations(z, name, out)
    # densify_and_prune leaves every statistic zero at the new size, and takes no optimizer step
    N2 = out["counts"][3]
    for s in ("max_radii2D", "xyz_gradient_accum", "denom"):
        assert z[f"{name}_out_{s}"].shape[0] == N2 and not z[f"{name}_out_{s}"].any()
    assert all(float(z[f"{name}_out_step{k}"]) == 7.0 for k in range(6))


def test_fixture_covers_the_cases(z):
    out = {n: _ref(z, n) for n in CASES}
    K, Cn, S, N2 = out["edges"]["counts"]
    f = out["edges"]["flags"]
    assert S > 0 and Cn > 0 and K + S < z["edges_p0"].shape[0]                  # something of each, and a prune
    assert list(f[:3]) == [1, 1, 1] and f[3] == 3 and f[4] == 4 and f[5] == 0   # scaffold; skybox rows past it
    assert list(f[6:9]) == [1, 3, 3] and list(f[9:12]) == [1, 4, 4]            # one ulp below, at, above max_grad
    assert f[12] == 1 and f[13] == 3 and f[14] == 1 and f[15] == 0             # 0.15 and the 0.005 edge
    assert f[16] == 3 and f[17] == 4                                            # max scaling at and above the threshold
    assert f[18] == 1 and f[19] == 1 and f[20] == 1                             # NaN accumulator, scaling, opacity
    assert out["no_split"]["counts"][2] == 0 and out["no_split"]["counts"][1] > 0
    assert out["no_clone"]["counts"][1] == 0 and out["no_clone"]["counts"][2] > 0
    K, Cn, S, _ = out["no_prune"]["counts"]
    assert K + S == z["no_prune_p0"].shape[0] and S > 0 and Cn > 0
    assert out["all_pruned"]["counts"] == (4, 0, 0, 4)


@pytest.mark.parametrize("name", ("reset_sky", "reset_none"))
def test_reset_restatement_is_the_reference(z, name):
    p, m, v = _inputs(z, name)
    o, mo, vo = D.reset_opacity(p, m, v, int(z[f"{name}_skybox"]))
    want = z[f"{name}_out_p3"]
    sky = int(z[f"{name}_skybox"])
    assert np.array_equal(o[:sky].view(np.int32), want[:sky].view(np.int32))
    # log(x / (1 - x)) of the host's sigmoid against torch's CPU one: within 2 ulp of sigmoid, carried through log
    assert D.ulps(o, want).max() <= 4
    assert not z[f"{name}_out_m3"].any() and not z[f"{name}_out_v3"].any() and not mo.any() and not vo.any()
    for k in (0, 1, 2, 4, 5):
        assert np.array_equal(z[f"{name}_out_p{k}"], p[k]) and np.array_equal(z[f"{name}_out_m{k}"], m[k])


# ---- the kernels against the restatement and the reference ---------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_kernel_is_the_restatement_and_the_reference(emu, z, name):
    p, m, v = _inputs(z, name)
    st = _state(p, m, v, z[f"{name}_gacc"], z[f"{name}_radii"], int(z[f"{name}_scaffold"]), int(z[f"{name}_skybox"]),
                float(z["percent_dense"]))
    N2 = st.densify_and_prune(float(z["max_grad"]), float(z["min_opacity"]), float(z["extent"]),
                              normals=torch.tensor(z[f"{name}_normals"]))
    ref = _ref(z, name)
    assert N2 == ref["counts"][3]
    _check_against(st, ref)
    got = dict(params=[t.numpy() for t in st.params], exp_avg=[t.numpy() for t in st.exp_avg],
               exp_avg_sq=[t.numpy() for t in st.exp_avg_sq], mag=ref["mag"])
    assert not _golden_violations(z, name, got)
    assert int(st.step) == 7 and int(st.exposure_step) == 5


@pytest.mark.parametrize("N,seed,scaffold,K", [(1, 1, 0, 15), (257, 2, 0, 15), (1000, 3, 50, 15), (600, 4, 10, 3),
                                               (300, 5, 0, 0)])
def test_kernel_is_the_restatement_on_random_states(emu, N, seed, scaffold, K):
    p, m, v = D.random_state(N, seed, K=K)
    g, r = D.random_stats(N, seed + 7, frac=0.2)
    if N > 100:
        g[10, 0], r[10], p[3][10, 0], p[4][10] = 1e-25, 1e26, 5.0, -6.0      # sqrt(g * g) underflows: no clone
        g[11, 0], r[11], p[3][11, 0], p[4][11] = 1e25, 1e-20, 5.0, -6.0      # sqrt(g * g) overflows: clone
        g[12, 0], r[12], p[3][12, 0], p[4][12] = -1.0, 10.0, 5.0, -1.0       # a negative g splits only through |g|
        g[13, 0], r[13], p[3][13, 0], p[4][13] = -1.0, 10.0, 5.0, -6.0
    st = _state(p, m, v, g, r, scaffold, 0)
    flags = D.decide(p, g, r, scaffold, 2e-4, 0.005, F(0.01 * 8.0))
    S = int(((flags & 4) != 0).sum())
    normals = np.random.default_rng(seed).normal(0, 1, (2 * S, 3)).astype(F)
    ref = D.densify(p, m, v, g, r, scaffold, 2e-4, 0.005, F(0.01 * 8.0), normals)
    st.densify_and_prune(2e-4, 0.005, 8.0, normals=torch.tensor(normals))
    _check_against(st, ref)
    if N > 100 and scaffold <= 10:
        assert flags[10] & 2 == 0 and flags[11] & 2 and flags[12] == 1 and flags[13] == 3


@pytest.mark.parametrize("name", ("reset_sky", "reset_none"))
def test_reset_kernel(emu, z, name):
    p, m, v = _inputs(z, name)
    sky = int(z[f"{name}_skybox"])
    st = _state(p, m, v, skybox=sky)
    before = [t.clone() for t in st.params + st.exp_avg + st.exp_avg_sq]
    st.reset_opacity()
    o, mo, vo = D.reset_opacity(p, m, v, sky)
    assert np.array_equal(st.params[3].numpy().view(np.int32), o.view(np.int32))
    assert not st.exp_avg[3].any() and not st.exp_avg_sq[3].any()
    assert D.ulps(st.params[3].numpy(), z[f"{name}_out_p3"]).max() <= 4
    after = st.params + st.exp_avg + st.exp_avg_sq
    for i, (a, b) in enumerate(zip(before, after)):
        if i % 6 != 3:
            assert torch.equal(a, b)
    assert int(st.step) == 7 and st.N == p[0].shape[0]


def test_drawn_normals_have_the_split_count(emu, z):
    """without normals= the state draws [2S, 3] from the generator, consuming it as torch.normal(zeros, stds) does"""
    p, m, v = _inputs(z, "edges")
    args = (z["edges_gacc"], z["edges_radii"], int(z["edges_scaffold"]), int(z["edges_skybox"]))
    st = _state(p, m, v, *args)
    gen = torch.Generator().manual_seed(4)
    st.densify_and_prune(2e-4, 0.005, 8.0, generator=gen)
    S = st.counts["split"]
    g2 = torch.Generator().manual_seed(4)
    stds = torch.rand((2 * S, 3), generator=torch.Generator().manual_seed(1)) + 0.5
    samples = torch.normal(torch.zeros(2 * S, 3), stds, generator=g2)
    assert torch.equal(gen.get_state(), g2.get_state())
    zs = torch.empty((2 * S, 3)).normal_(generator=torch.Generator().manual_seed(4))
    assert torch.equal(samples, zs * stds + 0)
    ref = D.densify(p, m, v, *args[:3], 2e-4, 0.005, F(0.08), zs.numpy())
    _check_against(st, ref)


# ---- the hand-back to a GaussianModel after the row count changed --------------------------------------------------
def _model_like(st):
    """a GaussianModel-shaped object of st's row count: six Parameters in OurAdam-shaped named groups, the exposures
    with a torch.optim.Adam, and the attributes from_model reads"""
    from h3dgs.optim import Adam
    attrs = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")
    model = types.SimpleNamespace(skybox_points=st.skybox_points, skybox_locked=st.skybox_locked,
                                  scaffold_points=st.scaffold_points, percent_dense=st.percent_dense)
    for a, p in zip(attrs, st.params):
        setattr(model, a, torch.nn.Parameter(torch.zeros_like(p)))
    model.optimizer = Adam([{"params": [getattr(model, a)], "lr": lr, "name": n} for a, lr, n in
                            zip(attrs, st.lr, D.GROUPS)], lr=0.0, eps=1e-15)
    model._exposure = torch.nn.Parameter(torch.zeros_like(st.exposure))
    model.exposure_optimizer = torch.optim.Adam([model._exposure])
    return model, attrs


def test_copy_to_model_after_densify_round_trips(emu, z):
    """the loop keeps one state and hands it to its GaussianModel for saves and checkpoints: after a densify the
    model's six Parameters are rebound (groups, optimizer state and attributes agree, N' rows everywhere capture()
    reads), and from_model gives the state back"""
    from h3dgs.singlestep import SingleState
    p, m, v = _inputs(z, "edges")
    st = _state(p, m, v, z["edges_gacc"], z["edges_radii"], int(z["edges_scaffold"]), int(z["edges_skybox"]))
    model, attrs = _model_like(st)
    st.copy_to_model(model)                                  # the model at the starting row count
    old = [getattr(model, a) for a in attrs]
    N2 = st.densify_and_prune(2e-4, 0.005, 8.0, normals=torch.tensor(z["edges_normals"]))
    assert N2 != p[0].shape[0]
    st.copy_to_model(model)
    opt = model.optimizer
    assert len(opt.state) == 6
    for a, g, o in zip(attrs, opt.param_groups, old):
        t = getattr(model, a)
        assert g["params"][0] is t and t is not o and isinstance(t, torch.nn.Parameter) and t.shape[0] == N2
        assert opt.state[t]["exp_avg"].shape == t.shape and opt.state[t]["exp_avg_sq"].shape == t.shape
    sd = opt.state_dict()                                    # capture()'s optimizer entry
    assert all(s["exp_avg"].shape[0] == N2 for s in sd["state"].values())
    for name in ("max_radii2D", "xyz_gradient_accum", "denom"):
        assert getattr(model, name).shape[0] == N2
    back = SingleState.from_model(model)
    assert back.N == N2 and back.percent_dense == st.percent_dense
    for k in range(6):
        for a, b in ((back.params[k], st.params[k]), (back.exp_avg[k], st.exp_avg[k]), (back.exp_avg_sq[k], st.exp_avg_sq[k])):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert int(back.step) == int(st.step) == 7 and int(back.exposure_step) == int(st.exposure_step)
    assert torch.equal(back.exposure, st.exposure)
    for name in ("max_radii2D", "xyz_gradient_accum", "denom"):
        assert torch.equal(getattr(back.stats, name), getattr(st.stats, name))
    # an unchanged row count still copies in place: the Parameters keep their identity
    kept = [getattr(model, a) for a in attrs]
    st.copy_to_model(model)
    assert all(getattr(model, a) is t for a, t in zip(attrs, kept))


# ---- argument errors -------------------------------------------------------------------------------------------
def test_argument_errors(emu, z):
    p, m, v = _inputs(z, "edges")
    args = (z["edges_gacc"], z["edges_radii"], 3, 6)
    st = _state(p, m, v, *args)
    with pytest.raises(ValueError):
        st.densify_and_prune(0.0, 0.005, 8.0)
    with pytest.raises(ValueError):
        st.densify_and_prune(2e-4, 0.2, 8.0)
    with pytest.raises(ValueError):
        st.densify_and_prune(2e-4, 0.005, 8.0, normals=torch.zeros((1, 3)))
    with pytest.raises(ValueError):
        st.densify_and_prune(2e-4, 0.005, 8.0, generator=torch.Generator(), normals=torch.zeros((0, 3)))
    st_none = _state(p, m, v, *args, percent_dense=None)
    with pytest.raises(ValueError):
        st_none.densify_and_prune(2e-4, 0.005, 8.0)
    assert st.N == p[0].shape[0]                            # nothing was swapped by a refused call
    from h3dgs import _lib
    a = _lib.DensifyArgs()
    with pytest.raises(RuntimeError):                      # no tensors
        _lib.check(emu.h3dgs_densify(C.byref(a), _lib.DENSIFY_RESET_OPACITY, None))
    with pytest.raises(RuntimeError):
        _lib.check(emu.h3dgs_densify(C.byref(a), 7, None))
    a = st._densify_args()
    a.max_grad, a.min_opacity = 2e-4, 0.005
    with pytest.raises(RuntimeError):                      # no statistics, flags or scratch
        _lib.check(emu.h3dgs_densify(C.byref(a), _lib.DENSIFY_COUNT, None))
    a.N = 1 << 30
    with pytest.raises(RuntimeError):                      # 3N does not fit int32
        _lib.check(emu.h3dgs_densify(C.byref(a), _lib.DENSIFY_RESET_OPACITY, None))
    assert emu.h3dgs_densify_scratch_bytes(1 << 30) == 0 and emu.h3dgs_densify_scratch_bytes(1000) > 12000

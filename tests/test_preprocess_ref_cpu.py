"""CPU: tests/preprocess_ref.py (the float64 restatement of the preprocess forward, K1 + K1b) pinned by independent means,
and the kernels' emulation build (tests/emul/) held to it on the edge families: near plane, frustum clamp, lambda floor,
radius ceiling, tile rect (borders, multiples of 16, five image sizes), huge splats (saturating conversions), degenerate
covariances, SH colour at its clamp, the fused gather, tile shards, and rows that do not project to finite values.
Every case asserts the binning invariants (preprocess_ref.check_invariants); every family must reach the decision it is
named for.  oracle.c, an fp32 evaluation in K1's order, goes through the same checker, and must equal the kernels bit
for bit in every integer artefact."""
import os
import sys

import numpy as np
import pytest

import preprocess_ref as pr

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emul"))
BG = np.zeros(3, np.float32)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    from build_emu import build
    from emu_api import Emu
    return Emu(build(str(tmp_path_factory.mktemp("h3dgs_emu"))))


def run_emu(emu, cam, sc, deg, mod=1.0, shard=(1, 0)):
    n = np.asarray(sc["means3D"]).shape[0]
    full = dict(sc)
    a, keep = emu.args(cam, BG, full, sh_degree=deg, ts=sc.get("ts"), kids=sc.get("kids"), ridx=sc.get("ridx"),
                       pidx=sc.get("pidx"), shard=shard, colors=sc.get("colors"), cov=sc.get("cov3D"))
    a.scale_modifier = mod
    fw = emu.forward(a, keep)
    st = emu.state(a, fw)
    # K1's per-row outputs inside the geometry buffer
    import ctypes as C
    from h3dgs import _lib
    v, b = _lib.StateView(), fw["bufs"]
    emu.check(emu.L.h3dgs_state_layout(a.P, a.image_width, a.image_height, fw["D"], b[0].ctypes.data, b[1].ctypes.data,
                                       b[2].ctypes.data, C.byref(v)))
    geom = lambda p, dt, n: b[0][p - b[0].ctypes.data:p - b[0].ctypes.data + n * np.dtype(dt).itemsize].view(dt)
    st.update(depths=geom(v.depths, np.float32, a.P), tiles_touched=geom(v.tiles_touched, np.uint32, a.P),
              records=geom(v.records, np.float32, 12 * a.P).reshape(a.P, 12))
    return dict(radii=fw["radii"].copy(), D=fw["D"], color=fw["color"].copy(), records=st["records"].copy(),
                depths=st["depths"].copy(), tiles_touched=st["tiles_touched"].copy(), ranges=st["ranges"].copy(),
                point_list=st.get("point_list", np.zeros(0, np.uint32)).copy(),
                keys_sorted=st.get("keys_sorted", np.zeros(0, np.uint64)).copy())


def run_oracle(cam, sc, deg, mod=1.0):
    """oracle.c's forward in the layout `check` takes"""
    from oracle import oracle
    f = oracle.rasterize_forward(sc["means3D"], sc.get("shs"), sc.get("colors"), sc["opacities"], sc.get("scales"),
                                 sc.get("rotations"), sc.get("cov3D"), cam.world_view_transform, cam.full_proj_transform,
                                 cam.camera_center, BG, cam.W, cam.H, cam.tanfovx, cam.tanfovy, sh_degree=deg, scale_modifier=mod)
    P = f["radii"].size
    kb = np.ones(P, np.uint32) | (f["clamped"].astype(np.uint32) << np.array([20, 21, 22], np.uint32)).sum(1).astype(np.uint32)
    with np.errstate(all="ignore"):
        rec = np.concatenate([f["xy"], f["conic_opacity"], np.ones((P, 1), np.float32), kb.view(np.float32)[:, None], f["rgb"],
                              (np.float32(1) / f["depths"])[:, None]], 1).astype(np.float32)
    return dict(radii=f["radii"], D=f["num_rendered"], records=rec, depths=f["depths"], tiles_touched=f["tiles_touched"],
                ranges=f["ranges"], point_list=f["point_list"], keys_sorted=f["keys"], color=f["color"])


def same_integers(a, b):
    for k in ("radii", "tiles_touched", "ranges", "point_list", "keys_sorted"):
        assert np.array_equal(np.asarray(a[k]).astype(np.int64).reshape(-1), np.asarray(b[k]).astype(np.int64).reshape(-1)), k
    assert a["D"] == b["D"]


def hold(emu, family, with_oracle=True):
    cases, named = family
    total = {}
    for lab, cam, sc, deg, mod in cases:
        R = pr.reference(sc, cam, deg, mod)
        out = run_emu(emu, cam, sc, deg, mod)
        rep = pr.check(R, out, name=lab)
        if with_oracle and sc.get("ridx") is None:
            o = run_oracle(cam, sc, deg, mod)
            pr.check(pr.reference(sc, cam, deg, mod), o, name=lab + " (oracle.c)")
            same_integers(out, o)
        for k, v in rep["undecided"].items():
            total[k] = total.get(k, 0) + v
        total["decided"] = total.get("decided", 0) + rep["decided"]
    for n in named:
        assert total.get(n, 0) > 0, f"the family never reaches the decision {n}: {total}"
    assert total["decided"] > 0 or not named                # (at a radius of 2^31 no ceiling is decided)
    return total


# ---- the reference itself ------------------------------------------------------------------------------------------------
def test_ref_matches_the_reference_projects_own_python(golden_dir):
    """cov3d.npz (build_covariance_from_scaling_rotation), sh_deg0..3.npz (eval_sh + 0.5, clamp) and camera.npz (the view
    and projection matrices the cameras here are built from)"""
    from h3dgs import synth
    z = np.load(os.path.join(golden_dir, "camera.npz"))
    cam = synth.make_camera(64, 48, fovx_deg=float(np.degrees(z["fovx_0"])), R=z["R_0"], T=z["T_0"], primx=float(z["primx_0"]),
                            primy=float(z["primy_0"]))
    assert np.allclose(cam.world_view_transform, z["wv_0"], atol=1e-6)
    for deg in range(4):
        g = np.load(os.path.join(golden_dir, f"sh_deg{deg}.npz"))
        n = g["xyz"].shape[0]
        from types import SimpleNamespace
        c = SimpleNamespace(W=64, H=48, world_view_transform=np.eye(4, dtype=np.float32), full_proj_transform=np.eye(4, dtype=np.float32),
                            camera_center=g["campos"], tanfovx=0.5, tanfovy=0.4)
        sc = dict(means3D=g["xyz"], shs=g["feats"], opacities=np.ones((n, 1), np.float32), scales=np.ones((n, 3), np.float32),
                  rotations=np.tile(np.array([1, 0, 0, 0], np.float32), (n, 1)))
        R = pr.reference(sc, c, deg)
        for ch in range(3):
            r = R.rgb[ch]
            dcd = np.abs(r.v) > 4 * pr.U * r.e
            assert np.array_equal((r.v < 0)[dcd], g["clamped"][dcd, ch])
            assert (np.abs(np.maximum(r.v, 0) - g["colors"][:, ch]) <= 2 * pr.U * r.e + 1e-7).all()
    g = np.load(os.path.join(golden_dir, "cov3d.npz"))
    # build_covariance_from_scaling_rotation normalises the quaternion; the renderer receives it normalised
    q = g["rotations"].astype(np.float64)
    q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    n = q.shape[0]
    sc = dict(means3D=np.tile(np.array([0.1, 0.2, 3.0], np.float32), (n, 1)), shs=np.zeros((n, 1, 3), np.float32),
              opacities=np.ones((n, 1), np.float32), scales=g["scales"], rotations=q)
    R = pr.reference(sc, c, 0)
    for k in range(6):
        assert (np.abs(R.cov6[k].v - g["cov6"][:, k]) <= 8 * pr.U * R.cov6[k].e + 1e-6 * np.abs(g["cov6"]).max(1)).all(), k


@pytest.mark.parametrize("seed", [1, 2])
def test_ref_matches_torch_splat_and_oracle_on_random_scenes(seed):
    import torch
    from oracle import torch_splat
    from util import make_scene
    cam, sc, *_ = make_scene(600, 160, 96, seed=seed)
    R = pr.reference(sc, cam, 3)
    D = lambda a: torch.tensor(np.asarray(a, np.float64))
    p = torch_splat.project(D(sc["means3D"]), D(sc["shs"]), None, D(sc["opacities"]), D(sc["scales"]), D(sc["rotations"]), None,
                            D(cam.world_view_transform), D(cam.full_proj_transform), D(cam.camera_center), cam.W, cam.H,
                            pr.F(cam.tanfovx), pr.F(cam.tanfovy), 3, 1.0)
    b = R.variants[0]
    vis = p["visible"].numpy().astype(bool)
    assert vis.sum() > 300
    for k, ref in (("ix", p["px"]), ("iy", p["py"]), ("depth", p["depth"]), ("conx", p["conic"][:, 0]), ("cony", p["conic"][:, 1]),
                   ("conz", p["conic"][:, 2])):
        d = np.abs(b[k].v - ref.numpy())[vis]
        assert (d <= 3e-7 * (1 + np.abs(ref.numpy()[vis]))).all(), k   # torch_splat holds 0.3 / 1.3 / 1e-7 in double, not as fp32 constants
    assert np.array_equal(pr.f2i_sat(np.ceil(b["radf"].v))[vis], p["radii"].numpy()[vis])
    rep = pr.check(R, run_oracle(cam, sc, 3), name=f"oracle.c seed {seed}")
    assert rep["decided"] > 0.9 * rep["rows"] and rep["worst"] <= 1.0


def test_budget_is_not_slack(emu):
    """a perturbation of a few budgets in one float of one row is reported"""
    cases, _ = pr.family_degenerate()
    lab, cam, sc, deg, mod = cases[0]
    R = pr.reference(sc, cam, deg, mod)
    out = run_emu(emu, cam, sc, deg, mod)
    rep = pr.check(R, out, name=lab)
    assert 0.0 < rep["worst"] <= 1.0
    i = int(np.nonzero(out["radii"] > 0)[0][3])
    for col, k in ((2, "conx"), (3, "cony"), (4, "conz"), (11, "invz")):
        o = dict(out, records=out["records"].copy())
        o["records"][i, col] += np.float32(6 * pr.U * R.variants[0][k].e[i])
        with pytest.raises(AssertionError):
            pr.check(pr.reference(sc, cam, deg, mod), o, name="perturbed")


# ---- the families on the emulation build ------------------------------------------------------------------------------------
@pytest.mark.parametrize("fam", ["near", "clamp", "floor", "radius", "huge", "degenerate", "gather"])
def test_family(emu, fam):
    hold(emu, getattr(pr, "family_" + fam)())


def test_family_rect(emu):
    tot = hold(emu, pr.family_rect(pr.SIZES[:4]))
    print(tot)


@pytest.mark.parametrize("deg,M", [(0, 1), (1, 4), (2, 9), (3, 16), (1, 16), (2, 16)])
def test_family_sh(emu, deg, M):
    hold(emu, pr.family_sh(deg, M))


def test_whole_screen_coverage_and_saturated_radius(emu):
    for lab, cam, sc, deg, mod in pr.family_huge()[0]:
        out = run_emu(emu, cam, sc, deg, mod)
        T = ((cam.W + 15) // 16) * ((cam.H + 15) // 16)
        assert (out["tiles_touched"] == T).sum() >= 12 and (out["radii"] == pr.INT_MAX).any()


def test_precomputed_colours_are_copied_unclamped(emu):
    cases, _ = pr.family_degenerate()
    lab, cam, sc, deg, mod = cases[0]
    sc = dict(sc)
    sc.pop("shs")
    sc["colors"] = np.random.default_rng(1).uniform(-2, 3, (sc["means3D"].shape[0], 3)).astype(np.float32)
    pr.check(pr.reference(sc, cam, 0, mod), run_emu(emu, cam, sc, 0, mod), name="colors_precomp")


@pytest.mark.parametrize("count", [1, 2, 3, 4, 8])
def test_family_shards(emu, count):
    """tiles_touched = owned rows x columns (explicit count), summing over the shards to the unsharded value; the
    scanned ranges' lengths are the per-tile counts of the rects"""
    for lab, cam, sc, deg, mod in pr.family_rect(pr.SIZES[1:3])[0] + pr.family_huge()[0]:
        R = pr.reference(sc, cam, deg, mod)
        whole = run_emu(emu, cam, sc, deg, mod)
        tot = np.zeros(R.P, np.int64)
        for idx in range(count):
            out = run_emu(emu, cam, sc, deg, mod, shard=(count, idx))
            pr.check(pr.reference(sc, cam, deg, mod), out, shard=(count, idx), name=f"{lab} shard {idx}/{count}")
            assert np.array_equal(out["radii"], whole["radii"])
            tot += out["tiles_touched"]
        assert np.array_equal(tot, whole["tiles_touched"].astype(np.int64))


@pytest.mark.parametrize("which", pr.NONFINITE_INPUTS)
def test_rows_that_do_not_project_are_invisible(emu, which):
    """NaN / +-inf in one input, every third row: a row whose depth, centre, conic or radius is not finite is invisible,
    and every other row, the ranges, the point list and the image are those of the scene without the poisoned rows."""
    cam, bad_sc, sc, bad = pr.family_nonfinite(which)
    deg = 0 if which == "colors" else 3
    out = run_emu(emu, cam, bad_sc, deg)
    R = pr.reference(bad_sc, cam, deg)
    pr.check(R, out, name=f"non-finite {which}")
    good = np.setdiff1d(np.arange(R.P), bad)
    if which in ("opacities", "shs", "colors"):
        # the row still projects: it stays visible and its record holds the value (a NaN SH colour becomes 0, no flag);
        # what the blend makes of it is the blend's matter
        assert (out["radii"][bad] > 0).all()
        return
    assert R.nonfinite[bad].sum() + (out["radii"][bad] == 0).sum() >= bad.size and not out["radii"][bad].any()
    clean = run_emu(emu, cam, {k: v[good] for k, v in sc.items()}, deg)
    assert np.array_equal(out["radii"][good], clean["radii"]) and out["D"] == clean["D"]
    assert np.array_equal(out["records"][good][clean["radii"] > 0].view(np.uint32), clean["records"][clean["radii"] > 0].view(np.uint32))
    assert np.array_equal(out["ranges"], clean["ranges"]) and np.array_equal(good[clean["point_list"]], out["point_list"])
    assert np.array_equal(out["color"].view(np.uint32), clean["color"].view(np.uint32))

"""GPU: the preprocess forward (preprocess_kernel: K1, preprocess_color_kernel: K1b) and what the binning makes of it, per
Gaussian against the float64 restatement of tests/preprocess_ref.py at the edges where K1's decisions flip: the families
of preprocess_ref (near plane, frustum clamp, lambda floor, radius ceiling, tile rect at five image sizes, huge splats,
degenerate covariances, SH colour at its clamp, the fused gather, tile shards, rows that do not project to finite values),
through _C.rasterize_gaussians and _C.state_view.  Every case asserts the binning invariants; every family must reach the
decision it is named for.  The per-case counts (rows decided, rows on each decision, worst |kernel - f64| / budget) are
printed (run with -s)."""
import numpy as np
import pytest

import preprocess_ref as pr

pytestmark = pytest.mark.gpu


def run(cam, sc, deg, mod=1.0, shard=(1, 0)):
    import torch
    from diff_gaussian_rasterization import _C
    t = lambda a, dt=torch.float32: None if a is None else torch.tensor(np.asarray(a), device="cuda", dtype=dt)
    m, op, sh, col = t(sc["means3D"]), t(sc["opacities"]), t(sc.get("shs")), t(sc.get("colors"))
    s, r, cov = t(sc.get("scales")), t(sc.get("rotations")), t(sc.get("cov3D"))
    ridx, pidx, ts, kids = t(sc.get("ridx"), torch.int32), t(sc.get("pidx"), torch.int32), t(sc.get("ts")), t(sc.get("kids"), torch.int32)
    f = _C.rasterize_gaussians(t(np.zeros(3)), m, col, op, s, r, float(mod), cov, t(cam.world_view_transform),
                               t(cam.full_proj_transform), cam.tanfovx, cam.tanfovy, cam.H, cam.W, sh, deg, t(cam.camera_center),
                               False, False, ridx, pidx, ts, kids, False, shard=shard)
    n, color, radii, gb, bb, ib, _ = f
    P = radii.numel()
    st = _C.state_view(P, cam.W, cam.H, n, gb, bb, ib)
    g = lambda k: st[k].cpu().numpy().copy() if k in st else np.zeros(0, np.int64)
    return dict(radii=radii.cpu().numpy().copy(), D=int(n), color=color.cpu().numpy().copy(), records=g("records"), depths=g("depths"),
                tiles_touched=g("tiles_touched"), ranges=g("ranges"), point_list=g("point_list"), keys_sorted=g("keys_sorted"))


def hold(family):
    cases, named = family
    total = {"decided": 0}
    for lab, cam, sc, deg, mod in cases:
        rep = pr.check(pr.reference(sc, cam, deg, mod), run(cam, sc, deg, mod), name=lab)
        for k, v in rep["undecided"].items():
            total[k] = total.get(k, 0) + v
        total["decided"] += rep["decided"]
    for n in named:
        assert total.get(n, 0) > 0, f"the family never reaches the decision {n}: {total}"
    assert total["decided"] > 0 or not named


@pytest.mark.parametrize("fam", ["near", "clamp", "floor", "radius", "rect", "huge", "degenerate", "gather"])
def test_family(fam):
    hold(getattr(pr, "family_" + fam)())


@pytest.mark.parametrize("deg,M", [(0, 1), (1, 4), (2, 9), (3, 16), (1, 16), (2, 16)])
def test_family_sh(deg, M):
    hold(pr.family_sh(deg, M))


def test_whole_screen_coverage_and_saturated_radius():
    for lab, cam, sc, deg, mod in pr.family_huge()[0]:
        out = run(cam, sc, deg, mod)
        T = ((cam.W + 15) // 16) * ((cam.H + 15) // 16)
        assert (out["tiles_touched"] == T).sum() >= 12 and (out["radii"] == pr.INT_MAX).any()


def test_precomputed_colours_are_copied_unclamped():
    lab, cam, sc, deg, mod = pr.family_degenerate()[0][0]
    sc = dict(sc)
    sc.pop("shs")
    sc["colors"] = np.random.default_rng(1).uniform(-2, 3, (sc["means3D"].shape[0], 3)).astype(np.float32)
    pr.check(pr.reference(sc, cam, 0, mod), run(cam, sc, 0, mod), name="colors_precomp")


@pytest.mark.parametrize("count", [1, 2, 3, 4, 8])
def test_family_shards(count):
    for lab, cam, sc, deg, mod in pr.family_rect(pr.SIZES[1:3])[0] + pr.family_huge()[0]:
        whole = run(cam, sc, deg, mod)
        tot = np.zeros(whole["radii"].size, np.int64)
        for idx in range(count):
            out = run(cam, sc, deg, mod, shard=(count, idx))
            pr.check(pr.reference(sc, cam, deg, mod), out, shard=(count, idx), name=f"{lab} shard {idx}/{count}")
            assert np.array_equal(out["radii"], whole["radii"])
            tot += out["tiles_touched"]
        assert np.array_equal(tot, whole["tiles_touched"].astype(np.int64))


@pytest.mark.parametrize("which", pr.NONFINITE_INPUTS)
def test_rows_that_do_not_project_are_invisible(which):
    """NaN / +-inf in one input, every third row (the emulation build runs this under AddressSanitizer first,
    tests/emul/asan_check.py): such a row is invisible, and every other row, the ranges, the point list and the image are
    those of the scene without the poisoned rows.  A NaN opacity or colour leaves the row visible."""
    cam, bad_sc, sc, bad = pr.family_nonfinite(which)
    deg = 0 if which == "colors" else 3
    out = run(cam, bad_sc, deg)
    R = pr.reference(bad_sc, cam, deg)
    pr.check(R, out, name=f"non-finite {which}")
    good = np.setdiff1d(np.arange(R.P), bad)
    if which in ("opacities", "shs", "colors"):
        assert (out["radii"][bad] > 0).all()
        return
    assert not out["radii"][bad].any()
    clean = run(cam, {k: v[good] for k, v in sc.items()}, deg)
    vis = clean["radii"] > 0
    assert np.array_equal(out["radii"][good], clean["radii"]) and out["D"] == clean["D"]
    assert np.array_equal(out["records"][good][vis].view(np.uint32), clean["records"][vis].view(np.uint32))
    assert np.array_equal(out["ranges"], clean["ranges"]) and np.array_equal(good[clean["point_list"]], out["point_list"])
    assert np.array_equal(out["color"].view(np.uint32), clean["color"].view(np.uint32))

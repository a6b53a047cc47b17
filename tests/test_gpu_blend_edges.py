"""GPU: the blend kernels (render_forward.cu, render_backward.cu, pair_math.cuh) per pixel and per Gaussian against a
float64 blend of their own 2D records (tests/blend_ref.py), on scenes built to sit at the kernels' decision edges.

Every case renders through the public _C entry points, reads K1's records and the tile lists out of the state buffers,
and gets the blend's [P][10] per-Gaussian sums from the backward's first phase (rasterize_gaussians_backward(...,
phases=1)).  Then, outside the pixels that have a pair within the decision margin of blend_ref:
  - n_contrib equals the float64 last contributor exactly (the taken set is the same);
  - colour, inverse depth and final T, per pixel, and each of the 10 sums, per element, differ from float64 by no more
    than their error budget: the per-pair relative error of fp32 + MUFU arithmetic (ex2.approx / lg2.approx ~2^-22,
    rcp.approx + one Newton step ~1 ulp, the exponent's ulps on the magnitude of its terms, the hierarchy weight's
    branches <= 4e-6, the transmittance's error accumulated along the pixel's list) times the pair's absolute term,
    plus n U times the absolute-sum scale for the n-term fp32 sum (blend_ref.py states the derivation term by term).

The measured maxima of |kernel - float64| / budget are printed per case (run with -s); each must stay <= 1."""
import math

import numpy as np
import pytest

from blend_ref import blend_reference, compare, hier_weight, ALPHA_CAP, ALPHA_SKIP, T_STOP, U

pytestmark = pytest.mark.gpu

FOVX = 60.0


def _cam(W, H):
    from h3dgs import synth
    return synth.make_camera(W, H, fovx_deg=FOVX)


def _place(cam, u, v, z):
    """world position whose projection lands on pixel (u, v) at depth z (identity view)"""
    return [((2 * u + 1) / cam.W - 1) * z * cam.tanfovx, ((2 * v + 1) / cam.H - 1) * z * cam.tanfovy, z]


def _cov(cam, z, sx, sy, rho=0.0):
    """3D covariance whose screen-space covariance at depth z is [[sx^2, rho sx sy], [., sy^2]] pixels^2 (before the
    0.3 dilation); the depth variance is negligible"""
    f = cam.W / (2 * cam.tanfovx)
    k = (z / f) ** 2
    return [sx * sx * k, rho * sx * sy * k, 0.0, sy * sy * k, 0.0, 1e-10]


class Scene:
    def __init__(self, cam):
        self.cam = cam
        self.means, self.covs, self.op, self.rgb = [], [], [], []
        self.ts, self.kids = [], []

    def add(self, u, v, z, sx, sy, rho=0.0, op=0.5, t=1.0, k=1, rgb=None, rng=None):
        self.means.append(_place(self.cam, u, v, z))
        self.covs.append(_cov(self.cam, z, sx, sy, rho))
        self.op.append(op)
        self.rgb.append(rgb if rgb is not None else (rng.uniform(0, 1, 3) if rng is not None else [0.5, 0.5, 0.5]))
        self.ts.append(t)
        self.kids.append(k)
        return len(self.op) - 1


def _render(sc, bg, hier, do_depth, gcol, gdep, op=None):
    """forward + backward phase 1 through _C -> (color, invdepth, state dict, accum [P][10]) as numpy"""
    import torch
    from diff_gaussian_rasterization import _C
    cam = sc.cam
    dev = "cuda"
    f = lambda a: torch.tensor(np.asarray(a, np.float32), device=dev)
    m, cov, rgb = f(sc.means), f(sc.covs), f(sc.rgb)
    opac = f(np.asarray(sc.op if op is None else op, np.float32).reshape(-1, 1))
    ts = f(sc.ts) if hier else None
    kids = torch.tensor(np.asarray(sc.kids, np.int64).astype(np.int32), device=dev) if hier else None
    vm, pm, cp = f(cam.world_view_transform), f(cam.full_proj_transform), f(cam.camera_center)
    bgt = f(bg)
    n, color, radii, gb, bb, ib, invd = _C.rasterize_gaussians(bgt, m, rgb, opac, None, None, 1.0, cov, vm, pm, cam.tanfovx,
                                                               cam.tanfovy, cam.H, cam.W, None, 0, cp, False, False, None,
                                                               None, ts, kids, do_depth)
    P = m.shape[0]
    sv = _C.state_view(P, cam.W, cam.H, n, gb, bb, ib)
    st = {k: v.cpu().numpy().copy() for k, v in sv.items()}
    st["radii"] = radii.cpu().numpy()
    accum = np.zeros((P, 10), np.float32)
    if n:
        scratch = _C.rasterize_gaussians_backward(bgt, m, radii, rgb, opac, None, None, 1.0, cov, vm, pm, cam.tanfovx,
                                                  cam.tanfovy, f(gcol), f(gdep) if do_depth else None, None, 0, cp, gb, n,
                                                  bb, ib, False, None, None, ts, kids, do_depth, cam.H, cam.W, phases=1)
        accum = scratch.view(torch.float32)[: P * 10].view(P, 10).cpu().numpy().copy()
    return color.cpu().numpy(), (invd.cpu().numpy()[0] if do_depth else None), st, accum


def _grads(cam, seed):
    g = np.random.default_rng(seed)
    return (g.standard_normal((3, cam.H, cam.W)) / 64).astype(np.float32), (g.standard_normal((cam.H, cam.W)) / 64).astype(np.float32)


def run_case(name, sc, hier=False, do_depth=False, bg=(0.1, 0.4, 0.9), op=None, seed=0,
             max_near_pixels=1e-3, max_near_gauss=0.05):
    """Render `sc` and check it against blend_ref.
    Returns (reference dict, records, (color, invdepth, state, accum))."""
    cam = sc.cam
    bg = np.asarray(bg, np.float32)
    gcol, gdep = _grads(cam, seed)
    run = _render(sc, bg, hier, do_depth, gcol, gdep, op)
    color, invd, st, accum = run
    vis = st["radii"] > 0
    rec = st["records"].copy()
    rec[~vis] = 0                      # rows K1 did not write (culled) are never listed
    kids = np.asarray(sc.kids, np.int64)
    if hier:       # K1 keeps the count in 20 bits: k <= 1 as 1, larger counts saturated, never wrapped
        assert np.array_equal(rec[vis, 7].view(np.uint32) & 0xFFFFF, np.clip(kids, 1, 2 ** 20 - 1)[vis])
    ref = blend_reference(rec, st["ranges"], st.get("point_list", np.zeros(0, np.int64)), cam.W, cam.H, bg, gcol,
                          gdep if do_depth else None, hier=hier, do_depth=do_depth, kids=kids)
    keep = ~ref["near_pixel"]
    near_share = float(ref["near_pixel"].mean())
    used = ref["npix"] > 0
    gshare = float(ref["near_gauss"][used].mean()) if used.any() else 0.0
    assert near_share <= max_near_pixels, (name, near_share, ref["near_kind"])
    assert gshare <= max_near_gauss, (name, gshare, ref["near_kind"])
    rows = ~ref["near_gauss"]
    report = {}
    nc = st["n_contrib"].astype(np.int64)
    bad = (nc != ref["n_contrib"]) & keep
    assert not bad.any(), (name, "n_contrib", int(bad.sum()), np.argwhere(bad)[:5].tolist())
    checks = [("color", color, ref["color"], ref["color_tol"][None], keep[None]),
              ("final_T", st["final_T"], ref["final_T"], ref["final_T_tol"], keep)]
    if do_depth:
        checks.append(("invdepth", invd, ref["invdepth"], ref["invdepth_tol"], keep))
    cols = list(range(9)) + ([9] if do_depth else [])
    for c in cols:
        checks.append((f"accum[{c}]", accum[:, c], ref["accum"][:, c], ref["accum_tol"][:, c], rows))
    for what, got, want, tol, mask in checks:
        r, cnt = compare(got, want, tol, mask)
        report[what] = r
        assert r <= 1.0, (name, what, r)
    if not do_depth:
        assert np.all(accum[:, 9] == 0)
    print(f"\n[{name}] max |kernel - f64| / budget: " + " ".join(f"{k}={v:.3g}" for k, v in report.items()) +
          f"  excluded: {near_share:.2e} of pixels, {gshare:.2e} of Gaussians {ref['near_kind']}")
    return ref, rec, run


def _gauss_at(rec, i, u, v):
    """float64 G of record i at pixel (u, v)"""
    x, y, cx, cy, cz = (float(a) for a in rec[i, :5])
    dx, dy = x - u, y - v
    return math.exp(-0.5 * (cx * dx * dx + cz * dy * dy) - cy * dx * dy)


def _base_alpha_for(target, t, k):
    """the base alpha whose hierarchy weight (t, k) is `target` (bisection in float64)"""
    lo_, hi_ = 0.0, ALPHA_CAP
    for _ in range(200):
        mid = 0.5 * (lo_ + hi_)
        if hier_weight(np.array(mid), np.array(t), np.array(k))[0] < target:
            lo_ = mid
        else:
            hi_ = mid
    return 0.5 * (lo_ + hi_)


# ---- hierarchy weight over its whole range -----------------------------------------------------------------------------
SWEEP_KIDS = [0, 1, 2, 3, 4, 7, 16, 17, 64, 255, 1000, 4095, 4096, 4097, 65535, 65536, 2 ** 20 - 1, 2 ** 20, 2 ** 20 + 2, -1]


@pytest.mark.parametrize("t", [0.0, 2.0 ** -24, 0.5, 1.0 - 2.0 ** -24, 1.0])
@pytest.mark.parametrize("do_depth", [False, True])
def test_hierarchy_weight_sweep(t, do_depth):
    """One 6-row band per num_node_kids value; in each, two long Gaussians (from the left and the right edge, slightly
    different widths so their alphas interleave) whose base alpha falls from the 0.99 cap to below 1/255 across the
    image: every band crosses alpha = 1/16 (the series / MUFU switch) and the 1/255 cut many times."""
    cam = _cam(160, 120)
    rng = np.random.default_rng(1)
    sc = Scene(cam)
    for b, k in enumerate(SWEEP_KIDS):
        v = 6 * b + 2.5
        sc.add(0, v, 3.0 + 0.01 * b, 45.0, 2.5, op=1.2, t=t, k=k, rng=rng)
        sc.add(cam.W - 1, v + 0.5, 4.0 + 0.01 * b, 47.3, 2.3, op=1.1, t=t, k=k, rng=rng)
    ref, rec, run = run_case(f"sweep t={t:.9g} depth={do_depth}", sc, hier=True, do_depth=do_depth, seed=2)
    # the bands do blend where they should: the identity counts everywhere, the others as far as their weight allows
    nc = ref["n_contrib"]
    assert (nc > 0).mean() > 0.5
    if t < 1:
        # k = 2^20 + 2 is a large count, not k = 2: at t = 0 nothing of its band passes 1/255
        b = SWEEP_KIDS.index(2 ** 20 + 2)
        two = SWEEP_KIDS.index(2)
        own = lambda band: ref["accum"][2 * band:2 * band + 2, 6:9]
        assert np.abs(own(two)).sum() > 0
        if t == 0.0:
            assert np.all(own(b) == 0) and np.all(run[3][2 * b:2 * b + 2] == 0)


# ---- the alpha = 1/255 cut ---------------------------------------------------------------------------------------------
SKIP_MODES = [(1.0, 1), (0.3, 2), (0.0, 7), (0.0, 300), (0.5, 40)]


@pytest.mark.parametrize("hier", [False, True])
def test_skip_threshold_both_sides(hier):
    """Isolated Gaussians, each tuned so that its alpha (after the hierarchy weight) at one chosen pixel is
    1/255 (1 +- 1e-3): taken on the + side, skipped on the - side."""
    cam = _cam(160, 120)
    rng = np.random.default_rng(3)
    sc = Scene(cam)
    targets = []
    i = 0
    for gy in range(10):
        for gx_ in range(13):
            t, k = SKIP_MODES[i % len(SKIP_MODES)] if hier else (1.0, 1)
            u, v = 6 + 12 * gx_, 6 + 12 * gy
            j = sc.add(u + 0.3, v - 0.2, 2.0 + 0.05 * i, 1.5, 1.3, rho=0.3, op=0.5, t=t, k=k, rng=rng)
            targets.append((j, u + 2, v + 1, t, k, 1 if i % 2 == 0 else -1))
            i += 1
    gcol, gdep = _grads(cam, 0)
    _, _, st, _ = _render(sc, np.zeros(3, np.float32), hier, False, gcol, gdep)
    op = np.array(sc.op, np.float64)
    for j, u, v, t, k, s in targets:
        a = _base_alpha_for(ALPHA_SKIP * (1 + s * 1e-3), t, k) if hier else ALPHA_SKIP * (1 + s * 1e-3)
        op[j] = a / _gauss_at(st["records"], j, u, v)
    ref, rec, run = run_case(f"skip hier={hier}", sc, hier=hier, op=op, seed=4)
    for j, u, v, t, k, s in targets:
        assert not ref["near_pixel"][v, u]
        assert (ref["n_contrib"][v, u] > 0) == (s > 0), (j, t, k, s)          # the scene is what it claims to be


# ---- the T < 1e-4 stop, at the TMA batch edges -------------------------------------------------------------------------
@pytest.mark.parametrize("stop_at,n", [(255, 300), (256, 300), (299, 300)])
@pytest.mark.parametrize("side", [-1, 1])
def test_stop_threshold_at_batch_edges(stop_at, n, side):
    """A stack of n small Gaussians over one pixel; there the transmittance in front of entry `stop_at` is 2e-4 and that
    entry brings T (1 - alpha) to 1e-4 (1 + side 1e-3): the list stops there (side -1) or goes on (side +1).  stop_at =
    255 / 256 are the last entry of the first 256-entry TMA batch and the first of the second, 299 the last of the list.
    (Small, so that the neighbouring pixels cross 1e-4 at other entries, if at all, and far from their margin.)"""
    cam = _cam(64, 48)
    rng = np.random.default_rng(5)
    u0, v0 = 20, 13
    sc = Scene(cam)
    for j in range(n):
        sc.add(u0 + 0.1, v0 - 0.1, 2.0 + 0.01 * j, 2.5, 2.2, op=0.05, rng=rng)
    gcol, gdep = _grads(cam, 0)
    _, _, st, _ = _render(sc, np.zeros(3, np.float32), False, False, gcol, gdep)
    G = np.array([_gauss_at(st["records"], j, u0, v0) for j in range(n)])
    a_front = 1 - (2e-4) ** (1.0 / stop_at)
    op = np.full(n, 0.3)
    op[:stop_at] = a_front / G[:stop_at]
    Tb = np.prod(1 - np.float32(op[:stop_at]).astype(np.float64) * G[:stop_at])
    op[stop_at] = (1 - T_STOP * (1 + side * 1e-3) / Tb) / G[stop_at]
    ref, rec, run = run_case(f"stop at {stop_at}/{n} side {side}", sc, op=op, seed=6)
    assert not ref["near_pixel"][v0, u0]
    if side < 0:
        assert ref["n_contrib"][v0, u0] == stop_at                 # entry stop_at (0-based) ends the list, unblended
    else:
        assert ref["n_contrib"][v0, u0] == stop_at + 1             # blended; the next entry (alpha 0.3) stops
    assert run[2]["n_contrib"][v0, u0] == ref["n_contrib"][v0, u0]


# ---- the 0.99 cap, opacity above 1 -------------------------------------------------------------------------------------
def test_alpha_cap_both_sides():
    """Isolated Gaussians with opacity above 1 whose opacity G at one pixel is 0.99 (1 +- 1e-3).  The cap is not
    differentiated (the published backward): above it the pixel still passes G dL/dalpha to the opacity, continuous
    across the cap -- so blend_ref and the kernel must agree on both sides, and the capped pixels' sums are not 0."""
    cam = _cam(160, 120)
    rng = np.random.default_rng(7)
    sc = Scene(cam)
    targets = []
    for i in range(60):
        u, v = 8 + 16 * (i % 10), 8 + 20 * (i // 10)
        j = sc.add(u - 0.2, v + 0.1, 2.0 + 0.05 * i, 2.0, 1.7, rho=-0.2, op=1.3, rng=rng)
        targets.append((j, u + 1, v, 1 if i % 2 == 0 else -1))
    gcol, gdep = _grads(cam, 0)
    _, _, st, _ = _render(sc, np.zeros(3, np.float32), False, False, gcol, gdep)
    op = np.array(sc.op, np.float64)
    for j, u, v, s in targets:
        op[j] = ALPHA_CAP * (1 + s * 1e-3) / _gauss_at(st["records"], j, u, v)
    assert op.min() > 1.0
    ref, rec, run = run_case("cap", sc, op=op, seed=8)
    for j, u, v, s in targets:
        assert not ref["near_pixel"][v, u] and ref["n_contrib"][v, u] > 0
        assert run[3][j, 5] != 0 and ref["accum"][j, 5] != 0


# ---- image borders, tiny images, off-screen means, needles -------------------------------------------------------------
@pytest.mark.parametrize("W,H", [(13, 9), (64, 47), (160, 119)])
@pytest.mark.parametrize("hier", [False, True])
def test_borders_offscreen_and_needles(W, H, hier):
    """Odd H (the second pixel of a thread outside the image), images below one tile, Gaussians centred off screen
    (the 1.3 tan(fov) clamp of the projection is active), and thin needle-shaped conics centred in a 4x4 block, so that
    their reach mask covers only a few of the tile's blocks."""
    cam = _cam(W, H)
    rng = np.random.default_rng(W * 1000 + H)
    sc = Scene(cam)
    P = int(np.clip(W * H // 25, 40, 300))         # a few layers per pixel, not hundreds
    for i in range(P):
        kind = i % 4
        t = float(rng.choice([1.0, 0.0, rng.uniform()])) if hier else 1.0
        k = int(rng.choice([1, 2, 3, 5, 17, 70000])) if hier else 1
        z = rng.uniform(2, 8)
        if kind == 0:          # off screen: beyond 1.3 tan(fov), wide enough to reach in
            u = (W - 1 + rng.uniform(0.16, 0.22) * W) if rng.uniform() < 0.5 else -rng.uniform(0.16, 0.22) * W
            v = rng.uniform(-0.2, 1.2) * H
            sc.add(u, v, z, rng.uniform(0.12, 0.25) * W, rng.uniform(0.12, 0.25) * W, rho=rng.uniform(-0.5, 0.5),
                   op=rng.uniform(0.3, 1.3), t=t, k=k, rng=rng)
        elif kind == 1:        # needle centred in a 4x4 block (0.9 x 0.05 px before the 0.3 px^2 dilation)
            u, v = 4 * rng.integers(0, max(W // 4, 1)) + 1.5, 4 * rng.integers(0, max(H // 4, 1)) + 1.5
            sc.add(u, v, z, 0.9, 0.05, rho=rng.choice([-0.9, 0.9]), op=rng.uniform(0.2, 1.0), t=t, k=k, rng=rng)
        else:                  # ordinary, some large
            sc.add(rng.uniform(-3, W + 3), rng.uniform(-3, H + 3), z, rng.uniform(0.5, 6), rng.uniform(0.5, 6),
                   rho=rng.uniform(-0.8, 0.8), op=rng.uniform(0.05, 1.2), t=t, k=k, rng=rng)
    ref, rec, run = run_case(f"borders {W}x{H} hier={hier}", sc, hier=hier, do_depth=hier, seed=9,
                             max_near_gauss=0.1)
    st = run[2]
    assert (ref["n_contrib"] > 0).mean() > 0.5
    # the clamp is active for some visible off-screen means
    xv = np.array(sc.means)[:, 0] / np.array(sc.means)[:, 2]
    assert ((np.abs(xv) > 1.3 * cam.tanfovx) & (st["radii"] > 0)).any()
    needles = np.arange(1, P, 4)
    assert (st["radii"][needles] > 0).any()


# ---- the public gradients, per row, against torch_splat ----------------------------------------------------------------
def _public_run(cam, sc, bg, gcol, gdep, ts, kids, do_depth, colors, cov):
    """forward + backward through _C -> (public gradients dict, accum [P][10], state dict) as numpy"""
    import torch
    from diff_gaussian_rasterization import _C
    f = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    m, op = f(sc["means3D"]), f(sc["opacities"])
    sh, rgb = (None, f(colors)) if colors is not None else (f(sc["shs"]), None)
    s, r, cv = (None, None, f(cov)) if cov is not None else (f(sc["scales"]), f(sc["rotations"]), None)
    tt = f(ts) if ts is not None else None
    kk = torch.tensor(kids, device="cuda") if kids is not None else None
    vm, pm, cp = f(cam.world_view_transform), f(cam.full_proj_transform), f(cam.camera_center)
    deg = 3 if sh is not None else 0
    n, color, radii, gb, bb, ib, invd = _C.rasterize_gaussians(f(bg), m, rgb, op, s, r, 1.0, cv, vm, pm, cam.tanfovx,
                                                               cam.tanfovy, cam.H, cam.W, sh, deg, cp, False, False, None,
                                                               None, tt, kk, do_depth)
    args = (f(bg), m, radii, rgb, op, s, r, 1.0, cv, vm, pm, cam.tanfovx, cam.tanfovy, f(gcol), f(gdep) if do_depth else None,
            sh, deg, cp, gb, n, bb, ib, False, None, None, tt, kk, do_depth, cam.H, cam.W)
    # both phases into one scratch, which keeps the [P][10] sums that the public gradients were made from (a second
    # replay would add them in another order)
    scratch = _C.rasterize_gaussians_backward(*args, phases=1)
    d2, dcol, dop, dm3, dcov, dsh, dsc, drot = _C.rasterize_gaussians_backward(*args, scratch=scratch)
    P = m.shape[0]
    accum = scratch.view(torch.float32)[: P * 10].view(P, 10)
    sv = _C.state_view(P, cam.W, cam.H, n, gb, bb, ib)
    st = {k: v.cpu().numpy().copy() for k, v in sv.items()}
    st["radii"] = radii.cpu().numpy()
    c = lambda x: x.cpu().numpy().reshape(P, -1) if (x is not None and x.numel()) else None
    g = dict(means3D=c(dm3), opacities=c(dop), shs=c(dsh), colors=c(dcol), scales=c(dsc), rotations=c(drot), cov3D=c(dcov))
    return {k: v for k, v in g.items() if v is not None}, c(d2), accum.cpu().numpy().astype(np.float64), st


@pytest.mark.parametrize("mode,do_depth", [("flat", False), ("flat", True), ("hier", True), ("precomp", False)])
def test_public_gradients_per_row(mode, do_depth):
    """Every returned gradient ROW against torch_splat's float64 autograd (oracle/torch_splat.py), each element with its
    own bar instead of the norm-wise 1e-5 max|b| of the parity tests, so a Gaussian whose gradient is far below the
    largest row is checked as strictly as that row.  The scenes are test_gpu_parity's kinds (flat, inverse depth,
    hierarchy weight, precomputed colour and covariance), at a size torch_splat's dense [pixels x Gaussians] blend handles.

    With J_c the float64 Jacobian of the 2D record entry c (x, y, conic, opacity, rgb, 1/z) of a row by that row's
    parameters (torch_splat.project), the public gradient is sum_c J_c dL/d(entry c).  Two bars, per element:
      - the chain rule of the preprocess backward, on the kernel's own [P][10] sums S:
            |g - sum_c J_c f_c S_c| <= 2^-9 sum_c |J_c f_c S_c|      (f_c: the accumulator's constant factors)
        -- fp32 through the 2D-covariance inversion and the cov3D / scale / rotation chain.  The published conic
        backward forms differences such as det - a c (= -b^2) in fp32, whose rounding is relative to a c, not to the
        small exact value that enters J; on these scenes the scales reach ~3.4e-4 of sum_c |J_c f_c S_c| (measured on an H100);
      - against torch_splat, the blend's own budget (blend_ref's accum_tol) carried through |J|, plus what K1's fp32
        projection of x, y and the conic moves (2^-10 of the absolute-sum scale accum_abs carried through |J|).
    Rows that receive gradient from a pixel with a near-decision pair (blend_ref near_gauss) are left out; the share is
    asserted small.  dL/dmeans2D is S_0 0.5 W, S_1 0.5 H to one rounding."""
    import torch
    from oracle import torch_splat
    from util import make_scene
    W, H, P = 128, 96, 1000
    cam, sc, ts, kids, bg = make_scene(P, W, H, mode="hier" if mode == "hier" else "flat", seed=21)
    colors = cov = None
    if mode == "precomp":
        colors = np.random.default_rng(0).uniform(0, 1, (P, 3)).astype(np.float32)
        T64 = lambda a: torch.tensor(a, dtype=torch.float64)
        S = torch_splat.build_cov3d(T64(sc["scales"]), T64(sc["rotations"]), 1.0)
        cov = S.reshape(P, 9)[:, [0, 1, 2, 4, 5, 8]].numpy().astype(np.float32)
    g = np.random.default_rng(22)
    gcol = (g.standard_normal((3, H, W)) / (H * W)).astype(np.float32)
    gdep = (g.standard_normal((H, W)) / (H * W)).astype(np.float32)
    pub, d2, accum, st = _public_run(cam, sc, bg, gcol, gdep, ts, kids, do_depth, colors, cov)

    # float64: torch_splat's projection and blend, differentiated by autograd
    T = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)
    prm = dict(means3D=T(sc["means3D"]), opacities=T(sc["opacities"]))
    if colors is not None:
        prm["colors"] = T(colors)
    else:
        prm["shs"] = T(sc["shs"])
    if cov is not None:
        prm["cov3D"] = T(cov)
    else:
        prm["scales"], prm["rotations"] = T(sc["scales"]), T(sc["rotations"])
    D = lambda a: torch.tensor(np.asarray(a, np.float64))
    pr = torch_splat.project(prm["means3D"], prm.get("shs"), prm.get("colors"), prm["opacities"], prm.get("scales"),
                             prm.get("rotations"), prm.get("cov3D"), D(cam.world_view_transform),
                             D(cam.full_proj_transform), D(cam.camera_center), W, H, cam.tanfovx, cam.tanfovy,
                             3 if colors is None else 0, 1.0)
    assert np.array_equal(pr["radii"].numpy(), st["radii"])          # the same Gaussians on the same tiles
    color, invd = torch_splat.blend2d(pr["px"], pr["py"], pr["conic"], pr["opacities"], pr["rgb"], pr["depth"],
                                      pr["visible"], pr["rect"], D(bg), W, H, D(ts) if ts is not None else None,
                                      D(kids) if kids is not None else None, do_depth)
    loss = (color * D(gcol)).sum() + ((invd[0] * D(gdep)).sum() if do_depth else 0.0)
    names = list(prm)
    ref = dict(zip(names, (x.numpy().reshape(P, -1) for x in torch.autograd.grad(loss, [prm[k] for k in names],
                                                                                    retain_graph=True))))
    entries = [pr["px"], pr["py"], pr["conic"][:, 0], pr["conic"][:, 1], pr["conic"][:, 2], pr["opacities"],
               pr["rgb"][:, 0], pr["rgb"][:, 1], pr["rgb"][:, 2], 1.0 / pr["depth"]]
    fac = np.array([1.0, 1.0, -0.5, -1.0, -0.5, 1.0, 1.0, 1.0, 1.0, 1.0])
    J = []          # J[c][name]: [P][n] d entry_c / d parameters, row by row (rows are independent)
    for e in entries:
        gs = torch.autograd.grad(e.sum(), [prm[k] for k in names], retain_graph=True, allow_unused=True)
        J.append({k: (np.zeros((P, prm[k][0].numel())) if x is None else x.numpy().reshape(P, -1)) for k, x in zip(names, gs)})

    vis = st["radii"] > 0
    rec = st["records"].copy()
    rec[~vis] = 0
    br = blend_reference(rec, st["ranges"], st.get("point_list", np.zeros(0, np.int64)), W, H, bg, gcol,
                         gdep if do_depth else None, hier=ts is not None, do_depth=do_depth, kids=kids)
    used = br["npix"] > 0
    assert used.sum() > 300 and br["near_gauss"][used].mean() < 0.02, br["near_kind"]
    rows = used & ~br["near_gauss"]
    cols = range(10 if do_depth else 9)
    # dL/dmeans2D: the first two sums times 0.5 W, 0.5 H
    for c, k in ((0, 0.5 * W), (1, 0.5 * H)):
        assert np.all(np.abs(d2[:, c] - accum[:, c] * k) <= U * np.abs(accum[:, c] * k))
    worst = {}
    for k in names:
        got = pub[k].astype(np.float64)
        chain = sum(J[c][k] * (fac[c] * accum[:, c:c + 1]) for c in cols)
        chain_abs = sum(np.abs(J[c][k] * (fac[c] * accum[:, c:c + 1])) for c in cols)
        r1, n1 = compare(got, chain, 2.0 ** -9 * chain_abs + 1e-30, rows[:, None])
        budget = sum(np.abs(J[c][k]) * np.abs(fac[c]) * (br["accum_tol"][:, c:c + 1] + 2.0 ** -10 * br["accum_abs"][:, c:c + 1])
                     for c in cols) + 2.0 ** -9 * chain_abs + 1e-30
        r2, n2 = compare(got, ref[k], budget, rows[:, None])
        worst[k] = (r1, r2)
        assert r1 <= 1.0, (mode, k, "chain rule", r1)
        assert r2 <= 1.0, (mode, k, "torch_splat", r2)
        assert n2 >= 0.5 * used.sum() * got.shape[1]
    print(f"\n[public {mode} depth={do_depth}] max |kernel - ref| / bar (chain rule, torch_splat): " +
          " ".join(f"{k}=({a:.3g}, {b:.3g})" for k, (a, b) in worst.items()) +
          f"  rows excluded: {br['near_gauss'][used].mean():.2e}")

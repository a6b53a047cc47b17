"""GPU: the preprocess backward (preprocess_backward_kernel: K8 + K9a + K9c, sh_backward_kernel: K9b) per Gaussian against
the float64 chain rule of tests/chain_ref.py, apart from the blend: each case runs the forward through
_C.rasterize_gaussians, reads K1's radii and records (_C.state_view), writes a chosen [P][10] into the backward's scratch
and runs only the chain-rule phase (rasterize_gaussians_backward(..., phases=2), no image gradients, as h3dgs/dist.py
does).  So the sums are exactly known, and every element of every returned tensor is held to its own budget (chain_ref:
kappa U m, derived term by term) instead of a fraction of the tensor's largest element.  Also asserted:
  - dL/dmeans2D, dL/dcolors (precomputed) and, outside scatter mode, dL/dopacities are bit-exact (a copy or one fp32
    multiply); culled rows, source rows outside the cut and SH coefficients beyond the degree are exact zeros;
  - the backward takes the forward's decisions: the SH clamp flags K1 stored (kbits 20-22) and the frustum clamp as
    K1's fp32 evaluation decides it (chain_ref.frustum_clamp_fp32);
  - two calls outside scatter mode are bitwise identical; a row block leaves the other rows zero and is bitwise the full
    call inside.
The cameras are rotated about a non-axis direction and translated 10 and 1000 units, so a transposed view index or a
wrong translation term changes the numbers.  The measured maxima of |kernel - float64| / budget are printed per case
(run with -s); each must stay <= 1."""
import numpy as np
import pytest

from chain_ref import (chain_reference, compare, fma_ratio_fp32, frustum_clamp_fp32, gather_fp32, general_camera,
                       random_accum, random_rows, view_xyz_fp32, world_from_view)

pytestmark = pytest.mark.gpu

W, H = 160, 100


def _t(a, dtype=None):
    import torch
    if a is None:
        return None
    a = np.asarray(a)
    return torch.tensor(a, device="cuda", dtype=dtype if dtype is not None else (torch.int32 if a.dtype.kind == "i" else torch.float32))


def run_backward(cam, sc, accum, deg, do_depth=False, mod=1.0, grad_rows=(0, 0), forward=None, debug=False):
    """forward (or the given one) + the chain-rule phase on `accum` -> (gradients dict, radii, records, forward, K1's
    view-space z); debug: the backward's serial path"""
    import torch
    from diff_gaussian_rasterization import _C
    from h3dgs import _lib
    f32 = lambda a: _t(None if a is None else np.asarray(a, np.float32))
    m, op = f32(sc["means3D"]), f32(sc["opacities"])
    sh, col = f32(sc.get("shs")), f32(sc.get("colors"))
    s, r, cov = f32(sc.get("scales")), f32(sc.get("rotations")), f32(sc.get("cov3D"))
    ridx, pidx, ts = _t(sc.get("ridx")), _t(sc.get("pidx")), f32(sc.get("ts"))
    kids = None if ts is None else torch.ones(ts.numel(), dtype=torch.int32, device="cuda")
    vm, pm, cp = f32(cam.world_view_transform), f32(cam.full_proj_transform), f32(cam.camera_center)
    bg = f32(np.zeros(3))
    if forward is None:
        forward = _C.rasterize_gaussians(bg, m, col, op, s, r, mod, cov, vm, pm, cam.tanfovx, cam.tanfovy, H, W, sh, deg,
                                         cp, False, False, ridx, pidx, ts, kids, do_depth)
    n, _color, radii, gb, bb, ib, _ = forward
    P = radii.numel()
    scratch = torch.zeros((_lib.lib().h3dgs_backward_scratch_bytes(P),), dtype=torch.uint8, device="cuda")
    scratch.view(torch.float32)[: P * 10] = f32(accum).reshape(-1)
    g = _C.rasterize_gaussians_backward(bg, m, radii, col, op, s, r, mod, cov, vm, pm, cam.tanfovx, cam.tanfovy, None, None,
                                        sh, deg, cp, gb, n, bb, ib, debug, ridx, pidx, ts, kids, do_depth, H, W, phases=2,
                                        scratch=scratch, grad_rows=grad_rows)
    names = ("means2D", "colors", "opacities", "means3D", "cov3D", "shs", "scales", "rotations")
    out = {k: v.cpu().numpy().copy() for k, v in zip(names, g) if v is not None and v.numel()}
    st = _C.state_view(P, W, H, n, gb, bb, ib)
    return out, radii.cpu().numpy(), st["records"].cpu().numpy().copy(), forward, st["depths"].cpu().numpy().copy()


def chain_ref_for(cam, sc, accum, deg, do_depth, mod, radii, kb):
    """chain_ref's reference for one run, with the forward's decisions: radii, the SH clamp flags of kbits `kb` and the
    frustum clamp as K1 evaluates it -> (ref dict, fclamp, tx/tz, ty/tz)"""
    scatter = sc.get("ridx") is not None
    means = (gather_fp32(sc["means3D"], sc.get("scales"), sc.get("rotations"), sc.get("shs"), sc["ridx"], sc["pidx"],
                         sc["ts"])["means3D"] if scatter else sc["means3D"])
    fcl, rx, ry = frustum_clamp_fp32(cam.world_view_transform, means, cam.tanfovx, cam.tanfovy)
    shc = np.stack([(kb >> (20 + ch)) & 1 for ch in range(3)], 1).astype(bool)
    ref = chain_reference(sc["means3D"], sc["opacities"], sc.get("scales"), sc.get("rotations"), sc.get("shs"),
                          sc.get("colors"), sc.get("cov3D"), mod, cam.world_view_transform, cam.full_proj_transform,
                          cam.camera_center, W, H, cam.tanfovx, cam.tanfovy, deg, radii, accum, shc, fcl,
                          np.stack([np.sign(rx), np.sign(ry)], 1), do_depth, sc.get("ridx"), sc.get("pidx"), sc.get("ts"))
    return ref, fcl, rx, ry


def check_case(name, cam, sc, accum, deg=3, do_depth=False, mod=1.0, min_visible=0.5, debug=False, keep=None):
    """run the case, compare every returned element with chain_ref; -> (report, radii, kbits, fclamp, K1 ratios, got).
    keep: a dict that receives the reference ('ref') and the forward ('forward')"""
    got, radii, rec, fwd, depth = run_backward(cam, sc, accum, deg, do_depth, mod, debug=debug)
    vis = radii > 0
    assert vis.mean() >= min_visible, (name, vis.mean())
    kb = rec[:, 7].view(np.uint32)
    scatter = sc.get("ridx") is not None
    ref, fcl, rx, ry = chain_ref_for(cam, sc, accum, deg, do_depth, mod, radii, kb)
    means = (gather_fp32(sc["means3D"], sc.get("scales"), sc.get("rotations"), sc.get("shs"), sc["ridx"], sc["pidx"],
                         sc["ts"])["means3D"] if scatter else sc["means3D"])
    # K1 evaluates the view transform in the order frustum_clamp_fp32 (and the backward) assume: its stored depth is the
    # same fp32 value bit for bit, so a change of K1's order fails here as well as a change of the backward's
    vz = view_xyz_fp32(cam.world_view_transform, means)[2]
    assert np.array_equal(depth[vis].view(np.uint32), vz[vis].view(np.uint32)), name
    if keep is not None:
        keep.update(ref=ref, forward=fwd)
    report = {}
    assert set(got) == set(ref), (name, sorted(got), sorted(ref))
    for k, (r, tol, _) in ref.items():
        assert np.isfinite(got[k]).all(), (name, k, "non-finite gradient", np.argwhere(~np.isfinite(got[k]))[:5].tolist())
        worst, cnt = compare(got[k], r, tol)
        report[k] = worst
        if not worst <= 1.0:
            bad = np.argwhere(np.abs(got[k].reshape(r.shape) - r) > tol)[:5]
            raise AssertionError((name, k, worst, [(tuple(b), float(got[k].reshape(r.shape)[tuple(b)]),
                                                    float(r[tuple(b)]), float(tol[tuple(b)])) for b in bad]))
    if not scatter:
        again, *_ = run_backward(cam, sc, accum, deg, do_depth, mod, forward=fwd)
        for k in got:
            assert np.array_equal(got[k].view(np.uint32), again[k].view(np.uint32)), (name, k)
    print(f"\n[{name}] max |kernel - f64| / budget: " + " ".join(f"{k}={v:.3g}" for k, v in report.items()))
    return report, radii, kb, fcl, (rx, ry), got


def place(cam, ratios_x, ratios_y, z):
    """fp32 world means at view-space (rx z, ry z, z)"""
    pv = np.stack([np.asarray(ratios_x) * z, np.asarray(ratios_y) * z, z], 1)
    return world_from_view(cam, pv).astype(np.float32)


def base_scene(rng, n, M=16, scale_of_z=0.02, z=None):
    z = rng.uniform(2.0, 12.0, n) if z is None else z
    scales, rots, opac, shs = random_rows(rng, n, M)
    scales = (scales / scales.mean(1, keepdims=True) * scale_of_z * z[:, None]).astype(np.float32)
    return z, dict(scales=scales, rotations=rots, opacities=opac, shs=shs)


TRANS = {10: (6.0, -5.0, 5.83), 1000: (610.0, -520.0, 598.0)}


# ---- the frustum clamp at its edge ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("dist", [10, 1000])
def test_frustum_clamp_edge(dist):
    """Gaussians whose K1 tx/tz (ty/tz) sits at +-limx (1 + k 2^-23), k in [-512, 512], on both axes, both signs and in
    the corners, wide enough to reach into the image.  Near the edge an FMA-contracted evaluation of the view-space mean
    decides the clamp otherwise than K1 for some rows (the scene must contain such rows); the backward must mask the
    gradient as K1 decided."""
    cam = general_camera(W, H, TRANS[dist])
    rng = np.random.default_rng(dist)
    lx, ly = 1.3 * np.float32(cam.tanfovx), 1.3 * np.float32(cam.tanfovy)
    ks = np.arange(-512, 513, 4)
    rows_x, rows_y = [], []
    for sx, sy in ((1, None), (-1, None), (None, 1), (None, -1), (1, 1), (1, -1), (-1, 1), (-1, -1)):
        for k in ks:
            e = 1 + k * 2.0 ** -23
            rows_x.append(sx * lx * e if sx is not None else rng.uniform(-0.8, 0.8) * cam.tanfovx)
            rows_y.append(sy * ly * e if sy is not None else rng.uniform(-0.8, 0.8) * cam.tanfovy)
    n = len(rows_x)
    z, sc = base_scene(rng, n, scale_of_z=0.2)
    sc["means3D"] = place(cam, rows_x, rows_y, z)
    accum = random_accum(np.random.default_rng(7), n)
    rep, radii, kb, fcl, (rx, ry), _ = check_case(f"clamp edge {dist}", cam, sc, accum, min_visible=1.0)
    # the scene is at the edge: both decisions on each axis, and rows where the FMA-ordered evaluation decides otherwise
    near = (np.abs(np.abs(rx) / np.float32(lx) - 1) < 2.0 ** -12) | (np.abs(np.abs(ry) / np.float32(ly) - 1) < 2.0 ** -12)
    assert near.sum() > n // 4 and fcl[near].any() and (~fcl[near]).any()
    fx, fy = fma_ratio_fp32(cam.world_view_transform, sc["means3D"])
    fma_cl = np.stack([(fx < -lx) | (fx > lx), (fy < -ly) | (fy > ly)], 1)
    differ = (fma_cl != fcl).any(1)
    print(f"  rows whose FMA-ordered clamp decision differs from K1's: {int(differ.sum())} of {n}")
    if dist == 1000:
        assert differ.sum() >= 10


# ---- near plane ------------------------------------------------------------------------------------------------------------
def nudge_to_vz(cam, means, target):
    """move each fp32 mean by a few ulp in two coordinates until K1's fp32 view-space z is exactly `target` [n]"""
    means = np.array(means, np.float32)
    v = np.asarray(cam.world_view_transform, np.float32).reshape(16)
    j1, j2 = np.argsort(-np.abs(v[[2, 6, 10]]))[:2]       # the two coordinates that move vz the most
    b1, b2 = (means[:, j].view(np.int32).astype(np.int64) for j in (j1, j2))
    done = np.zeros(len(means), bool)
    for k1 in sorted(range(-48, 49), key=abs):
        for k2 in sorted(range(-48, 49), key=abs):
            cand = means.copy()
            cand[:, j1] = (b1 + k1).astype(np.int32).view(np.float32)
            cand[:, j2] = (b2 + k2).astype(np.int32).view(np.float32)
            hit = ~done & (view_xyz_fp32(v, cand)[2] == target)
            means[hit] = cand[hit]
            done |= hit
    assert done.all(), (~done).sum()
    return means


def test_near_plane():
    """K1's fp32 vz exactly 0.2 (culled: the test is vz > 0.2), 0.2 + 1 ... 16 ulp (kept), 0.21 and 0.3.  The camera is
    rotated and close to the origin, so the world coordinates are small enough for their ulps to place vz ulp by ulp."""
    cam = general_camera(W, H, (0.05, -0.03, 0.02))
    rng = np.random.default_rng(3)
    near = np.float32(0.2)
    targets = [near] + [(near.view(np.int32) + k).view(np.float32) for k in (1, 2, 3, 5, 8, 16)] + [np.float32(0.21),
                                                                                                    np.float32(0.3)]
    zt = np.repeat(np.array(targets, np.float32), 12)
    n = zt.size
    z = zt.astype(np.float64)
    _, sc = base_scene(rng, n, scale_of_z=0.02, z=z)
    sc["means3D"] = nudge_to_vz(cam, place(cam, rng.uniform(-0.9, 0.9, n) * cam.tanfovx,
                                           rng.uniform(-0.9, 0.9, n) * cam.tanfovy, z), zt)
    accum = random_accum(np.random.default_rng(8), n)
    _, radii, *_ = check_case("near plane", cam, sc, accum, do_depth=True, min_visible=0.8)
    assert (radii[zt == near] == 0).all() and (radii[zt > near] > 0).all()


# ---- covariance extremes -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dist", [10, 1000])
@pytest.mark.parametrize("mod", [0.37, 1.0, 2.5])
def test_covariance_extremes(mod, dist):
    """dilation-dominated (screen variance far below the 0.3 px^2 dilation: where the 1e-7 of the inverse's gradient
    matters), needles (short, and long on screen: where a c - b^2 cancels, and fp64 is needed) and pancakes (scale ratios to 1e-4, and one zero scale), nearly isotropic (cancellation in the
    rotation gradient), screen-covering; quaternions of norm 0.3 / 1 / 3 and with zero components.  (1000 units from the
    origin, the fp32 view-space mean alone carries ~1e-5 relative error, as much as the 1e-7 term moves a gradient: the
    camera 10 units away is the one that resolves it.)"""
    cam = general_camera(W, H, TRANS[dist])
    rng = np.random.default_rng(int(mod * 100) + dist)
    kinds = ["dilation", "needle", "long", "pancake", "zero", "iso", "cover"]
    per = 40
    n = per * len(kinds)
    z, sc = base_scene(rng, n)
    s = np.empty((n, 3))
    for i, kd in enumerate(kinds):
        sl = slice(i * per, (i + 1) * per)
        zz = z[sl, None]
        ratio = 10.0 ** rng.uniform(-4, -1, (per, 1))
        s[sl] = {"dilation": lambda: 1e-5 * zz * np.ones((per, 3)),
                 "needle": lambda: 0.03 * zz * np.hstack([np.ones((per, 1)), ratio, ratio]),
                 # screen-long needles: a nearly rank-one 2D covariance, denom = a c - b^2 far below a c
                 "long": lambda: rng.uniform(0.2, 0.6, (per, 1)) * zz * np.hstack([np.ones((per, 1)), ratio, ratio]),
                 "pancake": lambda: 0.03 * zz * np.hstack([np.ones((per, 2)), ratio]),
                 "zero": lambda: 0.03 * zz * np.hstack([np.ones((per, 2)), np.zeros((per, 1))]),
                 "iso": lambda: 0.02 * zz * (1 + 1e-4 * rng.standard_normal((per, 3))),
                 "cover": lambda: 1.5 * zz * np.ones((per, 3)) * rng.uniform(0.5, 1, (per, 3))}[kd]()
    sc["scales"] = (s / mod).astype(np.float32)
    q = sc["rotations"].astype(np.float64)
    q[0::3] *= 0.3
    q[1::3] *= 3.0
    q[5::7, 1:3] = 0.0           # zero components
    q[6::11, 0] = 0.0
    sc["rotations"] = q.astype(np.float32)
    sc["means3D"] = place(cam, rng.uniform(-1.0, 1.0, n) * cam.tanfovx, rng.uniform(-1.0, 1.0, n) * cam.tanfovy, z)
    accum = random_accum(np.random.default_rng(9), n)
    check_case(f"covariance {dist} mod={mod}", cam, sc, accum, mod=mod, do_depth=True, min_visible=0.9)
    for col in (2, 3, 4):           # one conic column at a time
        check_case(f"covariance {dist} mod={mod} S{col} only", cam, sc, random_accum(np.random.default_rng(col), n, single=col),
                   mod=mod, min_visible=0.9)


def test_precomputed_inputs():
    """the cov3D_precomp and colors_precomp paths"""
    cam = general_camera(W, H, TRANS[10])
    rng = np.random.default_rng(12)
    n = 200
    z, sc = base_scene(rng, n)
    sc["means3D"] = place(cam, rng.uniform(-1.5, 1.5, n) * cam.tanfovx, rng.uniform(-1.5, 1.5, n) * cam.tanfovy, z)
    s, q = sc.pop("scales").astype(np.float64), sc.pop("rotations").astype(np.float64)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    r, x, y, w = q.T
    R = np.stack([1 - 2 * (y * y + w * w), 2 * (x * y - r * w), 2 * (x * w + r * y), 2 * (x * y + r * w),
                  1 - 2 * (x * x + w * w), 2 * (y * w - r * x), 2 * (x * w - r * y), 2 * (y * w + r * x),
                  1 - 2 * (x * x + y * y)], 1).reshape(n, 3, 3)
    S = R @ (s[:, :, None] ** 2 * np.transpose(R, (0, 2, 1)))
    sc["cov3D"] = S.reshape(n, 9)[:, [0, 1, 2, 4, 5, 8]].astype(np.float32)
    sc.pop("shs")
    sc["colors"] = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    check_case("precomputed", cam, sc, random_accum(np.random.default_rng(13), n), deg=0, do_depth=True, min_visible=0.7)


# ---- SH ----------------------------------------------------------------------------------------------------------------
def _look_camera(d, dist):
    """a camera whose view direction is the world direction d, at `dist` from the origin"""
    d = np.asarray(d, np.float64) / np.linalg.norm(d)
    a = np.array([0.3, 0.9, 0.1]) if abs(d[1]) < 0.9 else np.array([0.9, 0.1, 0.3])
    x = np.cross(a, d)
    x /= np.linalg.norm(x)
    y = np.cross(d, x)
    from h3dgs import synth
    R = np.stack([x, y, d], 1)                  # view z axis = d
    return synth.make_camera(W, H, R=R, T=np.array([0.7, -0.4, dist]))


DIRS = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1), (1, 1, 1), (-1, 1, -1)]


@pytest.mark.parametrize("deg,M", [(0, 1), (1, 4), (2, 9), (3, 16), (0, 16), (1, 16), (2, 16), (1, 9)])
def test_sh_degrees_directions_and_colour_clamp(deg, M):
    """M = 9 takes the scalar path and M = 16 the float4 path; degree below M's degree leaves the higher coefficients
    exact zeros.  View directions exactly along the +- axes and diagonals (a Gaussian on the camera's axis), and colours
    just below and just above 0 per channel: the backward follows the forward's clamp flags."""
    from oracle import torch_splat
    import torch
    rng = np.random.default_rng(deg * 10 + M)
    for d in DIRS:
        cam = _look_camera(d, 40.0)
        n = 24
        rx = np.r_[0.0, 0.0, rng.uniform(-0.9, 0.9, n - 2)] * cam.tanfovx
        ry = np.r_[0.0, 0.0, rng.uniform(-0.9, 0.9, n - 2)] * cam.tanfovy
        z, sc = base_scene(rng, n, M=M)
        sc["means3D"] = place(cam, rx, ry, z)
        # colours at +-1e-6 around 0: DC term set from the float64 rest of the SH sum
        cen = cam.camera_center.astype(np.float64)
        dirs = sc["means3D"].astype(np.float64) - cen
        dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
        sh = sc["shs"].astype(np.float64)
        sh[:, 0] = 0
        rest = torch_splat.eval_sh(deg, torch.tensor(sh[:, : (deg + 1) ** 2]), torch.tensor(dirs)).numpy()
        side = rng.choice([-1.0, 1.0], (n, 3)) * np.where(rng.uniform(size=(n, 3)) < 0.7, 1e-6, 0.3)
        sc["shs"][:, 0] = ((side - 0.5 - rest) / torch_splat.C0).astype(np.float32)
        rep, radii, kb, *_ = check_case(f"sh deg={deg} M={M} dir={d}", cam, sc, random_accum(rng, n), deg=deg,
                                        min_visible=1.0)
        flags = np.stack([(kb >> (20 + ch)) & 1 for ch in range(3)], 1).astype(bool)
        clear = np.abs(side) > 1e-3
        assert np.array_equal(flags[clear], side[clear] < 0)
        assert flags.any() and (~flags).any()


# ---- depth -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("do_depth", [False, True])
def test_depth_sum(do_depth):
    """with do_depth the S9 sum reaches dL/dmean3D; without it a non-zero S9 changes nothing"""
    cam = general_camera(W, H, TRANS[1000])
    rng = np.random.default_rng(14)
    n = 200
    z, sc = base_scene(rng, n)
    sc["means3D"] = place(cam, rng.uniform(-1, 1, n) * cam.tanfovx, rng.uniform(-1, 1, n) * cam.tanfovy, z)
    a = random_accum(rng, n)
    check_case(f"depth={do_depth}", cam, sc, a, do_depth=do_depth)
    b = a.copy()
    b[:, 9] = 0
    g1, *_ = run_backward(cam, sc, a, 3, do_depth)
    g0, *_ = run_backward(cam, sc, b, 3, do_depth)
    same = np.array_equal(g1["means3D"].view(np.uint32), g0["means3D"].view(np.uint32))
    assert same != do_depth


# ---- scatter mode ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dist", [10, 1000])
def test_scatter(dist):
    """the fused gather and the t / (1 - t) scatter: t in {0, 1, 0.5, random}; parent_indices = -1; one parent shared by
    1 - 64 children; quaternion dots < 0, = 0 and > 0; cut rows behind the camera (culled); source rows outside the cut"""
    cam = general_camera(W, H, TRANS[dist])
    rng = np.random.default_rng(dist + 1)
    groups = [1, 2, 5, 17, 64]
    P = sum(groups) + 40
    ND = 12                                       # parents of one child each: the quaternion-dot cases
    N = P + len(groups) + ND + 30                 # the last 30 source rows are in no cut
    z, sc = base_scene(rng, N)
    sc["means3D"] = place(cam, rng.uniform(-1, 1, N) * cam.tanfovx, rng.uniform(-1, 1, N) * cam.tanfovy, z)
    ridx = rng.permutation(P).astype(np.int32)
    pidx = np.full(P, -1, np.int32)
    o = 0
    for gi, gsz in enumerate(groups):
        pidx[o:o + gsz] = P + gi
        o += gsz
    pidx[o:o + 20] = rng.integers(0, P, 20)        # parents that are themselves rendered children
    o += 20
    own = np.arange(o, o + ND)                     # rows with a parent of their own
    pidx[own] = P + len(groups) + np.arange(ND)
    ts = rng.choice([0.0, 1.0, 0.5], P).astype(np.float32)
    ts[::3] = rng.uniform(0, 1, ts[::3].size).astype(np.float32)
    ts[own] = rng.uniform(0.1, 0.9, ND).astype(np.float32)
    # parents close to their children
    par = pidx >= 0
    sc["means3D"][pidx[par]] = sc["means3D"][ridx[par]] + rng.uniform(-0.05, 0.05, (par.sum(), 3)).astype(np.float32)
    # own parents: quaternion dots < 0, exactly 0 (q_p = (x, -r, z, -y) for q_c = (r, x, y, z): the fp32 products cancel
    # pairwise) and > 0
    q = sc["rotations"]
    for j, row in enumerate(own):
        c, p = ridx[row], pidx[row]
        q[p] = [-q[c] + np.float32(0.01), np.array([q[c][1], -q[c][0], q[c][3], -q[c][2]], np.float32),
                q[c] + np.float32(0.01)][j % 3]
    # a few cut rows behind the camera
    back = ridx[-5:]
    sc["means3D"][back] = place(cam, [0.0] * 5, [0.0] * 5, np.full(5, -3.0))
    sc.update(ridx=ridx, pidx=pidx, ts=ts)
    accum = random_accum(rng, P)
    rep, radii, _, _, _, got = check_case(f"scatter {dist}", cam, sc, accum, do_depth=True, min_visible=0.8)
    assert (radii[-5:] == 0).all()
    g = gather_fp32(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], ridx, pidx, ts)
    lerped = g["lerp"] & (radii > 0)
    assert (lerped & (g["dot"] < 0)).any() and (lerped & (g["dot"] == 0)).any() and (lerped & (g["dot"] > 0)).any()
    outside = np.setdiff1d(np.arange(N), np.r_[ridx, pidx[par]])
    assert outside.size >= 30
    for k in ("means3D", "opacities", "shs", "scales", "rotations"):
        assert not got[k].reshape(N, -1)[outside].any(), k


# ---- row blocks --------------------------------------------------------------------------------------------------------
def test_row_blocks():
    """grad_rows = [a, b): rows outside stay zero, rows inside are bitwise the full call's (clamped rows included)"""
    cam = general_camera(W, H, TRANS[1000])
    rng = np.random.default_rng(15)
    n = 300
    z, sc = base_scene(rng, n, scale_of_z=0.12)
    # include clamped rows
    sc["means3D"] = place(cam, rng.uniform(-1.6, 1.6, n) * cam.tanfovx, rng.uniform(-1.6, 1.6, n) * cam.tanfovy, z)
    accum = random_accum(rng, n)
    full, radii, _, fwd, _ = run_backward(cam, sc, accum, 3, True)
    for a, b in ((0, 128), (100, 229), (250, 300)):
        blk, *_ = run_backward(cam, sc, accum, 3, True, grad_rows=(a, b), forward=fwd)
        for k in full:
            x, y = blk[k].reshape(n, -1), full[k].reshape(n, -1)
            assert np.array_equal(x[a:b].view(np.uint32), y[a:b].view(np.uint32)), (k, a, b)
            assert not x[:a].any() and not x[b:].any(), (k, a, b)
    fcl = frustum_clamp_fp32(cam.world_view_transform, sc["means3D"], cam.tanfovx, cam.tanfovy)[0]
    assert fcl[radii > 0].any()

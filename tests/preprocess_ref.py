"""Float64 restatement of the preprocess forward (K1: projection, conic, radius, tile rect; K1b: SH colour) with a running
fp32 error bound per value and a margin per decision, and the checker that holds a run of the kernels to it.

Written from DESIGN.md §7 and include/h3dgs.h.  The value-with-bound arithmetic (`E`), the fp32 fused gather, the general
cameras and `compare` are those of tests/chain_ref.py.  Constants the kernels hold in fp32 (0.2, 1.3, 0.3, 0.1, 1e-7) enter
as their fp32 values, exactly; the SH constants carry one rounding (chain_ref._sh_basis).

Per row the reference gives depth, pixel centre, conic, lerped opacity, 1 / z and RGB as E values, and for every decision
K1 / K1b take the float64 quantity, its threshold and its bound:
    near      vz > 0.2                      clampx/y  |tx/tz| against 1.3 tan(fov) (the clamped value feeds J02 / J12)
    det       det != 0                      floor     mid^2 - det against 0.1
    ceil      3 sqrt(lambda) against the next integer      rect x0/y0/x1/y1  the truncated tile coordinate
    sh0..2    colour + 0.5 against 0
A decision whose margin exceeds its bound is decided.  `check` compares a run row by row:
  - a decided row's integer outputs are exact and its floats are inside their budgets;
  - an undecided row must equal the reference evaluated with its undecided float decisions (clamp, floor) forced one way
    or the other -- every float output and the radius from the same evaluation -- its radius must lie between the ceilings
    of the bound's two ends, and each rect edge between the truncations of its bound's two ends;
  - whatever the branch, the row's outputs agree with each other: the rect recomputed in fp32 from the stored centre and
    radius is the set of tiles the row appears in, `tiles_touched` is its (owned) area, radius 0 <=> no tile <=> no entry.
Rows that do not project to finite values in float64 must be invisible.  Rows whose intermediates leave [1e-37, 1e37]
(fp32 overflow / denormals, where a relative bound means nothing) are not predicted: they must be invisible or hold finite
outputs, and obey the consistency rules.  float -> int conversions saturate, NaN -> 0 (`f2i_sat`)."""
import itertools

import numpy as np

from chain_ref import E, U, _sh_basis, _sum, gather_fp32

F = lambda x: float(np.float32(x))
NEAR, FOV, DIL, FLOOR, WEPS = F(0.2), F(1.3), F(0.3), F(0.1), F(1e-7)
TILE = 16
KIDS_MASK = (1 << 20) - 1
INT_MAX, INT_MIN = 2 ** 31 - 1, -2 ** 31
FLOATS = ("depth", "ix", "iy", "conx", "cony", "conz", "invz")
REC = dict(ix=0, iy=1, conx=2, cony=3, conz=4, opac=5, t=6, kbits=7, r=8, g=9, b=10, invz=11)


def f2i_sat(x):
    """float -> int toward zero, saturating, NaN -> 0"""
    x = np.asarray(x, np.float64)
    return np.clip(np.trunc(np.where(np.isnan(x), 0.0, x)), INT_MIN, INT_MAX).astype(np.int64)


def rect_fp32(ix, iy, rad, W, H):
    """the tile rect [x0, y0, x1, y1) as DESIGN.md §7 states it, in fp32 from a stored centre and radius"""
    f = np.float32
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    r = np.asarray(rad, np.int64).astype(f)
    out = []
    with np.errstate(all="ignore"):
        for p, g in ((np.asarray(ix, f), gx), (np.asarray(iy, f), gy)):
            out.append((np.clip(f2i_sat((p - r) / f(TILE)), 0, g), np.clip(f2i_sat((((p + r) + f(TILE)) - f(1)) / f(TILE)), 0, g)))
    return out[0][0], out[1][0], out[0][1], out[1][1]


def owned_rows(y0, y1, shard):
    """explicit count of tile rows y in [y0, y1) with y % count == index"""
    cnt, idx = shard
    return np.array([sum(1 for y in range(a, b) if y % cnt == idx) for a, b in zip(y0, y1)], np.int64)


def _sel(c, a, b):
    return E(np.where(c, a.v, b.v), np.where(c, a.a, b.a), np.where(c, a.m, b.m), np.where(c, a.e, b.e))


class Ref:
    pass


def reference(sc, cam, deg=3, mod=1.0):
    """sc: means3D, opacities, scales + rotations or cov3D, shs or colors, optionally ridx / pidx / ts / kids (fp32 / int32
    arrays as the renderer takes them).  -> Ref"""
    f32 = np.float32
    W, H = cam.W, cam.H
    scat = sc.get("ridx") is not None
    N = np.asarray(sc["means3D"]).shape[0]
    if scat:
        ridx = np.asarray(sc["ridx"], np.int64)
        tail = ridx < 0
        safe = np.where(tail, 0, ridx)
        with np.errstate(all="ignore"):
            g = gather_fp32(sc["means3D"], sc.get("scales"), sc.get("rotations"), sc.get("shs"), safe, sc["pidx"], sc["ts"])
            o = np.asarray(sc["opacities"], f32).reshape(-1)
            opac = np.where(g["lerp"], g["t"] * o[g["c"]] + g["u"] * o[g["p"]], o[g["c"]])
        P = ridx.size
    else:
        P, ar = N, np.arange(N)
        tail = np.zeros(P, bool)
        g = dict(c=ar, means3D=np.asarray(sc["means3D"], f32), lerp=np.zeros(P, bool), dot=None,
                 scales=None if sc.get("scales") is None else np.asarray(sc["scales"], f32),
                 rotations=None if sc.get("rotations") is None else np.asarray(sc["rotations"], f32),
                 shs=None if sc.get("shs") is None else np.asarray(sc["shs"], f32))
        opac = np.asarray(sc["opacities"], f32).reshape(-1)
    ex = lambda a: E(np.asarray(a, np.float64))
    v = [ex(f32(x)) for x in np.asarray(cam.world_view_transform, f32).reshape(16)]
    q = [ex(f32(x)) for x in np.asarray(cam.full_proj_transform, f32).reshape(16)]
    tanx, tany = F(cam.tanfovx), F(cam.tanfovy)
    m = [ex(g["means3D"][:, k]) for k in range(3)]
    R = Ref()
    R.P, R.W, R.H, R.tail, R.gather, R.opac = P, W, H, tail, g, opac
    R.dec = {}
    big = np.zeros(P)
    small = np.full(P, np.inf)

    def track(*xs):
        nonlocal big, small
        for x in xs:
            a = np.abs(x.v)
            big = np.maximum(big, a)

    with np.errstate(all="ignore"):
        t = [v[r] * m[0] + v[4 + r] * m[1] + v[8 + r] * m[2] + v[12 + r] for r in range(3)]
        tz = t[2]
        R.dec["near"] = (tz.v - NEAR, U * tz.e)
        hx, hy, hw = (q[r] * m[0] + q[4 + r] * m[1] + q[8 + r] * m[2] + q[12 + r] for r in (0, 1, 3))
        pw = 1 / (hw + WEPS)
        ndx, ndy = hx * pw, hy * pw
        ix = ((ndx + 1.0) * float(W) - 1.0) * 0.5
        iy = ((ndy + 1.0) * float(H) - 1.0) * 0.5
        track(hw + WEPS, pw)
        small = np.minimum(np.abs((hw + WEPS).v), np.abs(tz.v))              # the divisors
        if sc.get("cov3D") is None:
            md = ex(f32(mod))
            s = [md * ex(g["scales"][:, k]) for k in range(3)]
            r_, x_, y_, z_ = (ex(g["rotations"][:, k]) for k in range(4))
            Rm = [[1 - 2 * (y_ * y_ + z_ * z_), 2 * (x_ * y_ - r_ * z_), 2 * (x_ * z_ + r_ * y_)],
                  [2 * (x_ * y_ + r_ * z_), 1 - 2 * (x_ * x_ + z_ * z_), 2 * (y_ * z_ - r_ * x_)],
                  [2 * (x_ * z_ - r_ * y_), 2 * (y_ * z_ + r_ * x_), 1 - 2 * (x_ * x_ + y_ * y_)]]
            Mm = [[s[k] * Rm[j][k] for j in range(3)] for k in range(3)]
            V6 = [_sum([Mm[k][a] * Mm[k][b] for k in range(3)]) for a, b in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))]
            track(*[Mm[k][j] for k in range(3) for j in range(3)])
        else:
            cv = np.asarray(sc["cov3D"], f32)[g["c"]]
            V6 = [ex(cv[:, k]) for k in range(6)]
        track(*V6)
        R.cov6 = V6
        lim = [ex(FOV) * ex(tanx), ex(FOV) * ex(tany)]
        ratio = [t[0] / tz, t[1] / tz]
        for k, n in ((0, "clampx"), (1, "clampy")):
            R.dec[n] = (np.abs(ratio[k].v) - lim[k].v, U * (ratio[k].e + lim[k].e))
        disc_dec = None
        R.variants = []
        for force in itertools.product((False, True), repeat=3):
            # force[k]: take the other branch of (clampx, clampy, floor) on the rows where that decision is undecided
            txy = []
            for k, n in ((0, "clampx"), (1, "clampy")):
                mg, bd = R.dec[n]
                cl = (mg > 0) ^ (force[k] & ~(np.abs(mg) > bd))
                bound = E(np.sign(ratio[k].v)) * lim[k] * tz
                txy.append(_sel(cl, bound, ratio[k] * tz))
            fx, fy = ex(W) / (2 * ex(tanx)), ex(H) / (2 * ex(tany))
            J00, J02 = fx / tz, -(fx * txy[0]) / (tz * tz)
            J11, J12 = fy / tz, -(fy * txy[1]) / (tz * tz)
            A = [[J00 * v[4 * c] + J02 * v[4 * c + 2] for c in range(3)], [J11 * v[4 * c + 1] + J12 * v[4 * c + 2] for c in range(3)]]
            Vm = [[V6[0], V6[1], V6[2]], [V6[1], V6[3], V6[4]], [V6[2], V6[4], V6[5]]]
            AV = [[A[r][0] * Vm[0][c] + A[r][1] * Vm[1][c] + A[r][2] * Vm[2][c] for c in range(3)] for r in range(2)]
            ca = (AV[0][0] * A[0][0] + AV[0][1] * A[0][1] + AV[0][2] * A[0][2]) + DIL
            cb = AV[0][0] * A[1][0] + AV[0][1] * A[1][1] + AV[0][2] * A[1][2]
            cc = (AV[1][0] * A[1][0] + AV[1][1] * A[1][1] + AV[1][2] * A[1][2]) + DIL
            det = ca * cc - cb * cb
            mid = 0.5 * (ca + cc)
            disc = mid * mid - det
            if disc_dec is None:
                disc_dec = (disc.v - FLOOR, U * disc.e)
                R.dec["det"] = (np.abs(det.v), U * det.e)
                R.dec["floor"] = disc_dec
                small = np.minimum(small, np.abs(det.v))
                track(*A[0], *A[1], *AV[0], *AV[1], ca * cc, cb * cb, mid * mid, tz * tz, fx * txy[0], fy * txy[1])
            fl = (disc_dec[0] > 0) ^ (force[2] & ~(np.abs(disc_dec[0]) > disc_dec[1]))
            sq = _sel(fl & ~np.isnan(disc.v), disc, E(np.full(P, FLOOR))).sqrt()
            radf = 3.0 * (mid + sq).sqrt()
            var = dict(depth=tz, ix=ix, iy=iy, conx=cc / det, cony=-cb / det, conz=ca / det, invz=1 / tz, radf=radf)
            # admissible where every forced decision really is undecided
            ok = np.ones(P, bool)
            for k, n in enumerate(("clampx", "clampy", "floor")):
                if force[k]:
                    ok &= ~(np.abs(R.dec[n][0]) > R.dec[n][1])
            var["ok"] = ok
            R.variants.append(var)
        base = R.variants[0]
        R.dec["ceil"] = (np.abs(base["radf"].v - np.round(base["radf"].v)), U * base["radf"].e)
        R.nonfinite = ~np.all([np.isfinite(base[k].v) for k in FLOATS + ("radf",)], 0) & ~tail
        fin = [base[k] for k in FLOATS + ("radf",)] + [det]
        track(*[x for x in fin])
        R.suspect = ~R.nonfinite & ~tail & ~((big < 1e37) & (small > 1e-37)) & (tz.v > 0)

        # ---- colour ----
        R.colors = None if sc.get("colors") is None else np.asarray(sc["colors"], f32)[g["c"]]
        R.rgb = None
        if R.colors is None:
            cp = [ex(f32(x)) for x in np.asarray(cam.camera_center, f32)]
            d0 = [m[k] - cp[k] for k in range(3)]
            ln = (d0[0] * d0[0] + d0[1] * d0[1] + d0[2] * d0[2]).sqrt()
            basis = _sh_basis(deg, d0[0] / ln, d0[1] / ln, d0[2] / ln)
            R.rgb = []
            for ch in range(3):
                r = _sum([B * ex(g["shs"][:, k, ch]) for k, (B, *_) in enumerate(basis)]) + 0.5
                R.dec[f"sh{ch}"] = (r.v, U * r.e)
                R.rgb.append(r)
    k = np.ones(P, np.int64) if sc.get("kids") is None else np.asarray(sc["kids"], np.int64)
    R.kids = np.where(k <= 1, 1, np.minimum(k, KIDS_MASK))
    R.ts = np.ones(P, f32) if sc.get("ts") is None else np.asarray(sc["ts"], f32)[:P]
    return R


def undecided(R, name):
    mg, bd = R.dec[name]
    return ~(np.abs(mg) > bd) & ~R.tail & ~R.nonfinite & ~R.suspect & ~np.isnan(mg)


def tiles_of_rows(out, P, gx):
    """from the sorted lists: per row the number of entries and the bounding tile rect it appears in"""
    cnt = np.zeros(P, np.int64)
    x0 = np.full(P, 1 << 30); y0 = np.full(P, 1 << 30); x1 = np.full(P, -1); y1 = np.full(P, -1)
    if out["D"]:
        pl = np.asarray(out["point_list"]).astype(np.int64)
        tile = (np.asarray(out["keys_sorted"]).view(np.uint64) >> np.uint64(32)).astype(np.int64)
        np.add.at(cnt, pl, 1)
        np.minimum.at(x0, pl, tile % gx); np.maximum.at(x1, pl, tile % gx)
        np.minimum.at(y0, pl, tile // gx); np.maximum.at(y1, pl, tile // gx)
    return cnt, x0, y0, x1 + 1, y1 + 1


def check_invariants(out, P, W, H, shard=(1, 0)):
    """radii > 0 <=> tiles_touched > 0 (unsharded), sum tiles_touched = D = sum of range lengths, every point_list entry
    < P and visible, every tile's keys non-decreasing and of that tile.  -> per-row observed (count, x0, y0, x1, y1)"""
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    radii, tt = np.asarray(out["radii"]).astype(np.int64), np.asarray(out["tiles_touched"]).astype(np.int64)
    rng = np.asarray(out["ranges"]).astype(np.int64).reshape(gx * gy, 2)
    D = int(out["D"])
    assert (radii >= 0).all()
    if shard[0] == 1:
        assert np.array_equal(radii > 0, tt > 0), np.nonzero((radii > 0) != (tt > 0))[0][:8]
    else:
        assert not tt[radii <= 0].any()
    lens = rng[:, 1] - rng[:, 0]
    assert (lens >= 0).all() and tt.sum() == D == lens.sum(), (int(tt.sum()), D, int(lens.sum()))
    if D:
        pl = np.asarray(out["point_list"]).astype(np.int64)
        keys = np.asarray(out["keys_sorted"]).view(np.uint64)
        assert (pl >= 0).all() and (pl < P).all() and (radii[pl] > 0).all()
        tile = (keys >> np.uint64(32)).astype(np.int64)
        for tl in np.nonzero(lens)[0]:
            a, b = rng[tl]
            assert (tile[a:b] == tl).all() and (np.diff(keys[a:b].astype(np.int64)) >= 0).all(), int(tl)
    obs = tiles_of_rows(out, P, gx)
    assert np.array_equal(obs[0], tt), "tiles_touched is not the number of list entries of the row"
    return obs, lens


def check(R, out, shard=(1, 0), name=""):
    """hold one run of the kernels (out: radii, records [P][12] fp32, depths, tiles_touched, ranges, point_list,
    keys_sorted, D) to the reference.  -> report: rows decided, rows undecided per decision, worst |kernel - f64| / budget"""
    P, W, H = R.P, R.W, R.H
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    (cnt, ox0, oy0, ox1, oy1), lens = check_invariants(out, P, W, H, shard)
    radii = np.asarray(out["radii"]).astype(np.int64)
    rec = np.asarray(out["records"], np.float32).reshape(P, 12)
    vis = radii > 0
    und = {n: undecided(R, n) for n in R.dec}
    predicted = ~R.tail & ~R.nonfinite & ~R.suspect

    # ---- rows that must be invisible ----
    assert not vis[R.tail].any(), "a tail row (render_indices < 0) is visible"
    assert not vis[R.nonfinite].any(), (name, "rows that do not project to finite values are visible",
                                        np.nonzero(vis & R.nonfinite)[0][:8])
    got = dict(depth=np.asarray(out["depths"], np.float32), **{k: rec[:, REC[k]] for k in FLOATS[1:]})
    for k in FLOATS:
        assert np.isfinite(got[k][vis]).all(), (name, k, "a visible row stores a non-finite value")

    # ---- visibility before the rect ----
    near, det = R.dec["near"], R.dec["det"]
    must_cull = predicted & (((near[0] <= 0) & ~und["near"]) | ((det[0] == 0) & ~und["det"]))
    assert not vis[must_cull].any(), (name, "culled rows are visible", np.nonzero(vis & must_cull)[0][:8])
    may_cull = und["near"] | und["det"] | must_cull | ~predicted

    # ---- floats and radius of the visible rows: one admissible evaluation fits them all ----
    rows = vis & predicted
    fits = np.zeros(P, bool)
    worst = np.zeros(P)
    with np.errstate(all="ignore"):
        for var in R.variants:
            okv = var["ok"].copy()
            w = np.zeros(P)
            for k in FLOATS:
                r = np.abs(got[k].astype(np.float64) - var[k].v) / (U * var[k].e)
                r = np.where(got[k].astype(np.float64) == var[k].v, 0.0, r)
                w = np.maximum(w, np.where(np.isnan(r), np.inf, r))
            rf, rb = var["radf"].v, U * var["radf"].e
            okr = (radii >= f2i_sat(np.ceil(rf - rb))) & (radii <= f2i_sat(np.ceil(rf + rb)))
            good = okv & (w <= 1.0) & okr
            worst = np.where(good & ~fits, w, worst)
            fits |= good
    bad = rows & ~fits
    if bad.any():
        i = int(np.nonzero(bad)[0][0])
        v0 = R.variants[0]
        raise AssertionError((name, "row outside every admissible evaluation", i, int(radii[i]), float(v0["radf"].v[i]),
                              {k: (float(got[k][i]), float(v0[k].v[i]), float(U * v0[k].e[i])) for k in FLOATS}))
    dec_float = rows & ~und["clampx"] & ~und["clampy"] & ~und["floor"] & ~und["ceil"]
    assert np.array_equal(radii[dec_float], f2i_sat(np.ceil(R.variants[0]["radf"].v))[dec_float]), (name, "radius of decided rows")

    # ---- the rect: from the stored centre and radius (consistency), and against the float64 centre (margins) ----
    x0, y0, x1, y1 = rect_fp32(rec[:, 0], rec[:, 1], radii, W, H)
    area = (x1 - x0) * (y1 - y0)
    assert (area[vis] > 0).all(), (name, "a visible row with an empty rect")
    seen = vis & (cnt > 0)                                  # a shard sees the columns, and only its own tile rows
    assert np.array_equal(ox0[seen], x0[seen]) and np.array_equal(ox1[seen], x1[seen]), (name, "columns of the emitted entries")
    if shard[0] == 1:
        assert np.array_equal(oy0[vis], y0[vis]) and np.array_equal(oy1[vis], y1[vis]), (name, "tile rows of the emitted entries")
    own = owned_rows(y0, y1, shard) * (x1 - x0) if shard[0] > 1 else area
    assert np.array_equal(np.where(vis, own, 0), np.asarray(out["tiles_touched"]).astype(np.int64)), (name, "tiles_touched")
    per_tile = np.zeros((gy, gx), np.int64)
    for i in np.nonzero(vis)[0]:
        ys = [y for y in range(y0[i], y1[i]) if y % shard[0] == shard[1]]
        per_tile[ys, x0[i]:x1[i]] += 1
    assert np.array_equal(per_tile.reshape(-1), lens), (name, "per-tile list lengths")
    base = R.variants[0]
    rr = radii.astype(np.float64)
    edges = {}
    with np.errstate(all="ignore"):
        for nm, c, sgn, gmax, kern in (("x0", base["ix"], -1, gx, x0), ("y0", base["iy"], -1, gy, y0), ("x1", base["ix"], 1, gx, x1),
                                       ("y1", base["iy"], 1, gy, y1)):
            arg = (c.v + sgn * rr + (15.0 if sgn > 0 else 0.0)) / TILE
            bd = U * (c.e + 3 * (np.abs(c.v) + rr + 16)) / TILE
            lo, hi = np.clip(f2i_sat(arg - bd), 0, gmax), np.clip(f2i_sat(arg + bd), 0, gmax)
            ok = (kern >= lo) & (kern <= hi)
            assert ok[rows].all(), (name, nm, "edge outside the truncations of its bound", np.nonzero(rows & ~ok)[0][:8])
            edges[nm] = rows & (lo != hi)
            R.dec[nm] = (np.abs(arg - np.round(arg)), bd)
            # rows the rect may cull: an empty rect inside the bounds
        # an invisible predicted row needs a reason: a cull it may take, or a rect that may be empty
        rad0 = f2i_sat(np.ceil(base["radf"].v))
        ex0, ey0, ex1, ey1 = rect_fp32(base["ix"].v, base["iy"].v, rad0, W, H)
        near_edge = np.zeros(P, bool)
        for c, g, r in ((base["ix"], gx, rad0), (base["iy"], gy, rad0)):
            for arg in ((c.v - r) / TILE, (c.v + r + 15) / TILE):
                bd = U * (c.e + 3 * (np.abs(c.v) + r + 16)) / TILE + 1e-300
                near_edge |= (f2i_sat(arg - bd) != f2i_sat(arg + bd))
        empty_ok = ((ex1 - ex0) * (ey1 - ey0) == 0) | near_edge | und["ceil"]
    unexplained = predicted & ~vis & ~may_cull & ~empty_ok
    assert not unexplained.any(), (name, "rows invisible without a reason", np.nonzero(unexplained)[0][:8])

    # ---- opacity (the fp32 lerp, bit for bit), t, kids, colour and its flags ----
    eq = lambda a, b: np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))
    assert eq(rec[vis, REC["opac"]], R.opac[vis]), (name, "opacity is not the two-products-one-sum lerp")
    assert eq(rec[vis, REC["t"]], R.ts[vis]), (name, "t")
    kb = rec[:, REC["kbits"]].view(np.uint32).astype(np.int64)
    assert np.array_equal(kb[vis] & KIDS_MASK, R.kids[vis]), (name, "kids field")
    assert not (kb[vis] >> 23).any()
    flags = np.stack([(kb >> (20 + ch)) & 1 for ch in range(3)], 1).astype(bool)
    worst_rgb = 0.0
    if R.colors is not None:
        assert eq(rec[vis, 8:11], R.colors[vis]) and not flags[vis].any(), (name, "precomputed colours are copied, no flag")
    else:
        for ch in range(3):
            r = R.rgb[ch]
            u = ~(np.abs(r.v) > U * r.e)
            sel = vis & np.isfinite(r.v)
            dcd = sel & ~u
            assert np.array_equal(flags[dcd, ch], r.v[dcd] < 0), (name, f"clamp flag of channel {ch}")
            g = rec[:, 8 + ch].astype(np.float64)
            want = np.where(flags[:, ch], 0.0, r.v)                      # the kernel's own branch, value from that branch
            with np.errstate(all="ignore"):
                d = np.abs(g - want) / (U * r.e)
            d = np.where(g == want, 0.0, d)
            assert (g[sel & flags[:, ch]] == 0).all(), (name, "a flagged channel is not 0")
            assert (d[sel] <= 1.0).all(), (name, f"rgb channel {ch}", float(d[sel].max()), int(np.nonzero(sel)[0][np.argmax(d[sel])]))
            worst_rgb = max(worst_rgb, float(d[sel].max()) if sel.any() else 0.0)
            und[f"sh{ch}"] = vis & u & np.isfinite(r.v)
            nanrow = vis & ~np.isfinite(r.v)
            # a NaN colour (NaN SH on a projectable row): fmaxf(NaN, 0) = 0 and no flag
            assert not flags[nanrow & np.isnan(r.v), ch].any() and (g[nanrow & np.isnan(r.v)] == 0).all()
    und.update(edges)
    anyu = np.zeros(P, bool)
    for n, mk in und.items():
        anyu |= mk
    rep = dict(rows=P, visible=int(vis.sum()), decided=int((predicted & ~anyu).sum()), nonfinite=int(R.nonfinite.sum()),
               unpredicted=int(R.suspect.sum()), worst=float(worst[rows].max()) if rows.any() else 0.0, worst_rgb=worst_rgb,
               undecided={n: int(mk.sum()) for n, mk in und.items() if mk.any()})
    print(f"\n[{name}] " + " ".join(f"{k}={v}" for k, v in rep.items()))
    return rep


# ---- edge families (shared by the CPU and GPU tests): each -> list of (label, cam, sc, deg, mod) --------------------------
from chain_ref import general_camera, random_rows, world_from_view  # noqa: E402

TRANS = {10: (6.0, -5.0, 5.83), 1000: (610.0, -520.0, 598.0)}
ULPS = (0, 1, -1, 2, -2, 512, -512)


def place(cam, rx, ry, z):
    z = np.asarray(z, np.float64)
    return world_from_view(cam, np.stack([np.asarray(rx) * z, np.asarray(ry) * z, z], 1)).astype(np.float32)


def rows(rng, n, cam, z=None, scale_of_z=0.02, M=16, spread=0.9):
    z = rng.uniform(2.0, 12.0, n) if z is None else np.asarray(z, np.float64)
    s, q, o, sh = random_rows(rng, n, M)
    s = (s / s.mean(1, keepdims=True) * scale_of_z * z[:, None]).astype(np.float32)
    return dict(means3D=place(cam, rng.uniform(-spread, spread, n) * cam.tanfovx, rng.uniform(-spread, spread, n) * cam.tanfovy, z),
                scales=s, rotations=q, opacities=o, shs=sh), z


def ndc_ratio(cam, ix, W):
    """view-space x / z of pixel centre ix (centred principal point)"""
    return ((2.0 * np.asarray(ix, np.float64) + 1.0) / W - 1.0)


def bisect_scale(cam, sc, margin, lo=1e-3, hi=1e3, deg=0):
    """per row the factor on sc['scales'] at which margin(Ref) changes sign, by bisection in the float64 reference"""
    n = sc["scales"].shape[0]
    a, b = np.full(n, lo), np.full(n, hi)
    base = sc["scales"].astype(np.float64)
    ev = lambda f: margin(reference(dict(sc, scales=(base * f[:, None]).astype(np.float32)), cam, deg))
    sa = ev(a) > 0
    for _ in range(40):
        mid = np.sqrt(a * b)
        up = (ev(mid) > 0) == sa
        a, b = np.where(up, mid, a), np.where(up, b, mid)
    return np.sqrt(a * b)


def family_near():
    cam = general_camera(160, 100, (0.05, -0.03, 0.02))
    rng = np.random.default_rng(3)
    z = np.concatenate([np.float32(0.2).astype(np.float64) * (1 + k * 2.0 ** -23) * np.ones(24) for k in ULPS] + [np.full(12, 0.21), np.full(12, 0.19)])
    sc, _ = rows(rng, z.size, cam, z=z)
    return [("near", cam, sc, 3, 1.0)], ("near",)


def family_clamp():
    out = []
    for dist in (10, 1000):
        cam = general_camera(160, 100, TRANS[dist], primx=0.5 if dist == 10 else 0.37, primy=0.5 if dist == 10 else 0.64)
        rng = np.random.default_rng(dist)
        lx, ly = F(1.3) * F(cam.tanfovx), F(1.3) * F(cam.tanfovy)
        rx, ry = [], []
        for sx, sy in ((1, None), (-1, None), (None, 1), (None, -1), (1, 1), (1, -1), (-1, 1), (-1, -1)):
            for k in list(range(-16, 17, 2)) + [-512, 512]:
                e = 1 + k * 2.0 ** -23
                rx.append(sx * lx * e if sx else rng.uniform(-0.8, 0.8) * cam.tanfovx)
                ry.append(sy * ly * e if sy else rng.uniform(-0.8, 0.8) * cam.tanfovy)
        sc, z = rows(rng, len(rx), cam, scale_of_z=0.2)
        sc["means3D"] = place(cam, rx, ry, z)
        out.append((f"clamp {dist}", cam, sc, 3, 1.0))
    return out, ("clampx", "clampy")


def family_floor():
    cam = general_camera(160, 100, TRANS[10], primx=0.37, primy=0.64)
    rng = np.random.default_rng(5)
    n = 40
    sc, z = rows(rng, n, cam, scale_of_z=1e-5)                      # cov2D = 0.3 I: floor active, radius 3
    sw, z2 = rows(rng, n, cam)
    sw["scales"] = (np.array([1.0, 1e-4, 1e-4]) * z2[:, None] * 0.01).astype(np.float32)
    f = bisect_scale(cam, sw, lambda R: R.dec["floor"][0])
    parts = [sc]
    for k in ULPS:
        parts.append(dict(sw, scales=(sw["scales"].astype(np.float64) * f[:, None] * (1 + k * 2.0 ** -22)).astype(np.float32)))
    return [("floor", cam, {k: np.concatenate([p[k] for p in parts]) for k in sc}, 3, 1.0)], ("floor",)


def family_radius():
    cam = general_camera(160, 100, TRANS[10], primx=0.37, primy=0.64)
    rng = np.random.default_rng(6)
    sw, z = rows(rng, 60, cam, scale_of_z=0.03)
    target = np.ceil(reference(sw, cam, 0).variants[0]["radf"].v) + 0.0
    f = bisect_scale(cam, sw, lambda R: R.variants[0]["radf"].v - target, lo=0.5, hi=4.0)
    parts = [dict(sw, scales=(sw["scales"].astype(np.float64) * f[:, None] * (1 + k * 2.0 ** -23)).astype(np.float32))
             for k in (0, 1, -1, 2, -2, 64, -64, 4096, -4096)]
    return [("radius", cam, {k: np.concatenate([p[k] for p in parts]) for k in sw}, 3, 1.0)], ("ceil",)


SIZES = ((8, 8), (15, 33), (336, 250), (1920, 1080), (3840, 2160))


def family_rect(sizes=SIZES):
    """isotropic splats of radius 3 (floor active) with ix -+ 3 on multiples of 16 and neighbours, just off and just
    touching each border"""
    out = []
    for (W, H) in sizes:
        cam = general_camera(W, H, (0.0, 0.0, 0.0), angle_deg=0.0)
        rng = np.random.default_rng(W)
        px, py = [], []
        tiles = sorted({0, 1, (W // 16) // 2, W // 16})
        for tx in tiles:
            for d in (-0.01, -1e-4, 0.0, 1e-4, 0.01):
                px += [16 * tx + 3 + d, 16 * tx - 3 + d - 15 + 16]; py += [rng.uniform(0, H - 1)] * 2
        for d in (-1.0, -0.01, 0.0, 0.01, 1.0):                      # off / touching the four borders
            px += [-3 + d, W - 1 + 3 + d + 0.0, rng.uniform(0, W - 1), rng.uniform(0, W - 1), -19 + d, W + 20 + d]
            py += [rng.uniform(0, H - 1), rng.uniform(0, H - 1), -3 + d, H - 1 + 3 + d, rng.uniform(0, H - 1), -25 + d]
        tys = sorted({0, 1, H // 16})
        for ty in tys:
            for d in (-0.01, 0.0, 0.01):
                py += [16 * ty + 3 + d, 16 * ty - 2 + d]; px += [rng.uniform(0, W - 1)] * 2
        n = len(px)
        z = rng.uniform(2.0, 6.0, n)
        sc, _ = rows(rng, n, cam, z=z, scale_of_z=1e-6)
        sc["means3D"] = place(cam, ndc_ratio(cam, px, W) * cam.tanfovx, ndc_ratio(cam, py, H) * cam.tanfovy, z)
        out.append((f"rect {W}x{H}", cam, sc, 0, 1.0))
    return out, ("x0", "y0", "x1", "y1")


def family_huge(sizes=((160, 100), (336, 250))):
    out = []
    for (W, H) in sizes:
        cam = general_camera(W, H, TRANS[10])
        rng = np.random.default_rng(W + 1)
        n = 48
        sc, z = rows(rng, n, cam)
        fx = W / (2 * cam.tanfovx)
        k = np.arange(n) % 4
        px_sigma = np.where(k == 0, 2.0 ** 31 / 3 * rng.uniform(1.0, 2.0, n), np.where(k == 1, 2.0 ** 29, np.where(k == 2, 5e4, 2.0 ** 31 / 3)))
        sc["scales"] = (px_sigma * z / fx)[:, None].astype(np.float32) * np.ones((1, 3), np.float32)
        rx = np.where(k == 3, rng.choice([-1, 1], n) * 10.0 ** rng.uniform(8.5, 10, n), rng.uniform(-0.9, 0.9, n) * cam.tanfovx)
        sc["means3D"] = place(cam, rx, rng.uniform(-0.9, 0.9, n) * cam.tanfovy, z)
        out.append((f"huge {W}x{H}", cam, sc, 1, 1.0))
    return out, ()


def family_degenerate():
    out = []
    for dist, mod in ((10, 1.0), (1000, 1.0), (10, 0.0)):
        cam = general_camera(160, 100, TRANS[dist], primx=0.37, primy=0.64)
        rng = np.random.default_rng(dist + 7)
        n = 90
        sc, z = rows(rng, n, cam, scale_of_z=0.05)
        k = np.arange(n) % 9
        s = sc["scales"]
        s[k == 0, 0] = 0; s[k == 1, :2] = 0; s[k == 2] = 0
        nd = k == 3                                                     # needles: det cancels
        s[nd] = (rng.uniform(0.2, 0.6, (nd.sum(), 1)) * z[nd, None] * np.array([1.0, 1e-4, 1e-4])).astype(np.float32)
        q = sc["rotations"]
        q[k == 4] *= 3.0; q[k == 5] *= 0.3; q[k == 6] = 0.0
        out.append((f"degenerate {dist} mod={mod}", cam, sc, 3, mod))
    cam = general_camera(160, 100, TRANS[10])
    rng = np.random.default_rng(17)
    n = 60
    sc, z = rows(rng, n, cam)
    a = rng.standard_normal((n, 3)) * 0.05 * z[:, None]
    k = np.arange(n) % 4
    cov = np.zeros((n, 6))
    r1 = np.stack([a[:, 0] * a[:, 0], a[:, 0] * a[:, 1], a[:, 0] * a[:, 2], a[:, 1] * a[:, 1], a[:, 1] * a[:, 2], a[:, 2] * a[:, 2]], 1)
    cov[k == 1] = r1[k == 1]
    cov[k == 2] = -r1[k == 2] * 30                                    # not positive semidefinite
    cov[k == 3] = r1[k == 3] + np.array([1e-3, 0, 0, 1e-3, 0, 1e-3])
    sc.pop("scales"); sc.pop("rotations")
    sc["cov3D"] = cov.astype(np.float32)
    out.append(("cov3D zero / rank 1 / not PSD", cam, sc, 3, 1.0))
    return out, ()


DIRS = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1), (1, 1, 1), (-1, 1, -1), (1, -1, 0), (0, 1, 1)]


def look_camera(d, dist, W=160, H=100):
    from h3dgs import synth
    d = np.asarray(d, np.float64) / np.linalg.norm(d)
    a = np.array([0.3, 0.9, 0.1]) if abs(d[1]) < 0.9 else np.array([0.9, 0.1, 0.3])
    x = np.cross(a, d); x /= np.linalg.norm(x)
    return synth.make_camera(W, H, R=np.stack([x, np.cross(d, x), d], 1), T=np.array([0.0, 0.0, dist]))


def family_sh(deg, M):
    out = []
    rng = np.random.default_rng(deg * 10 + M)
    for d in DIRS:
        cam = look_camera(d, 40.0)
        n = 30
        sc, z = rows(rng, n, cam, M=M)
        rx = np.r_[0.0, 0.0, rng.uniform(-0.9, 0.9, n - 2)] * cam.tanfovx
        ry = np.r_[0.0, 0.0, rng.uniform(-0.9, 0.9, n - 2)] * cam.tanfovy
        sc["means3D"] = place(cam, rx, ry, z)
        if M > 1:
            sc["shs"][10:20, 1:] *= 300.0                              # cancelling coefficients of opposite sign
        sc["shs"][:, 0] = 0
        rest = np.stack([r.v for r in reference(sc, cam, deg).rgb], 1)          # 0.5 + the rest of the sum
        tiny = np.array([0.0, 1e-7, -1e-7, 1e-6, -1e-6, 3e-5, -3e-5])
        side = np.where(rng.uniform(size=(n, 3)) < 0.7, rng.choice(tiny, (n, 3)), rng.choice([-0.3, 0.3], (n, 3)))
        side[10:20] = rng.choice([-30.0, 30.0, 1e-3, -1e-3], (10, 3))
        sc["shs"][:, 0] = ((side - rest) / 0.28209479177387814).astype(np.float32)
        out.append((f"sh deg={deg} M={M} dir={d}", cam, sc, deg, 1.0))
    return out, ("sh0", "sh1", "sh2")


KIDS = [-2 ** 31, -1, 0, 1, 2, 65535, 65536, 2 ** 20 - 1, 2 ** 20, 2 ** 31 - 1]


def family_gather():
    out = []
    for dist in (10, 1000):
        cam = general_camera(160, 100, TRANS[dist])
        rng = np.random.default_rng(dist + 2)
        N = 260
        sc, z = rows(rng, N, cam)
        P = 200
        ridx = rng.integers(0, 120, P).astype(np.int32)                # several cut rows share a source row
        pidx = rng.integers(120, N, P).astype(np.int32)
        pidx[::7] = -1
        pidx[1::11] = ridx[1::11]                                      # child = parent
        ridx[-9:] = -1                                                 # the tail of a device-side cut
        ts = rng.choice(np.array([0.0, 2.0 ** -24, 0.5, 1 - 2.0 ** -24, 1.0], np.float32), P)
        ts[::5] = rng.uniform(0, 1, ts[::5].size).astype(np.float32)
        par = (pidx >= 0) & (ridx >= 0)
        sc["means3D"][pidx[par]] = sc["means3D"][ridx[par]] + rng.uniform(-0.05, 0.05, (par.sum(), 3)).astype(np.float32)
        q = sc["rotations"]
        for j in np.nonzero(par)[0][:90]:
            c, p = ridx[j], pidx[j]
            tiny = np.float32(1e-30)
            orth = np.array([q[c][1], -q[c][0], q[c][3], -q[c][2]], np.float32)   # fp32 dot exactly 0
            q[p] = [-q[c], orth, orth + tiny * q[c], orth - tiny * q[c], -q[c] + np.float32(0.01), q[c] + np.float32(0.01)][j % 6]
        kids = np.array([KIDS[j % len(KIDS)] for j in range(P)], np.int64).astype(np.int32)
        sc.update(ridx=ridx, pidx=pidx, ts=ts, kids=kids)
        out.append((f"gather {dist}", cam, sc, 3, 1.0))
    return out, ()


BAD = (np.nan, np.inf, -np.inf)
NONFINITE_INPUTS = ("means3D", "scales", "rotations", "opacities", "shs", "cov3D", "colors")


def family_nonfinite(which):
    """one input at a time holds NaN / +-inf in every third row; -> (cases, index of the poisoned rows, clean scene)"""
    cam = general_camera(160, 100, TRANS[10])
    rng = np.random.default_rng(23)
    n = 120
    sc, z = rows(rng, n, cam, scale_of_z=0.05)
    sc["opacities"] = np.full((n, 1), 0.9, np.float32)
    if which == "cov3D":
        s = sc.pop("scales").astype(np.float64) ** 2
        sc.pop("rotations")
        sc["cov3D"] = np.stack([s[:, 0], 0 * z, 0 * z, s[:, 1], 0 * z, s[:, 2]], 1).astype(np.float32)
    if which == "colors":
        sc.pop("shs")
        sc["colors"] = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    bad = np.arange(1, n, 3)
    poisoned = {k: np.array(v) for k, v in sc.items()}
    a = poisoned[which].reshape(n, -1)
    for j, i in enumerate(bad):
        a[i, j % a.shape[1]] = BAD[j % 3]
    return cam, poisoned, sc, bad

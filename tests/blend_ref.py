"""Float64 restatement of the blend stage (K6 forward, K7 backward replay) over the kernel's OWN 2D records.

The inputs are what K1 wrote -- the unsorted per-Gaussian records ([P][12] fp32: x, y, conic.xyz, opacity, t, kbits, rgb,
invdepth; `_C.state_view(...)["records"]`) -- and the tile lists (ranges, point_list), so the blend kernels are checked
apart from preprocess: any difference is the blend stage's.  Every value is computed in float64 from the fp32 inputs
with the published formulas, written out here directly (expm1 / log1p for the hierarchy weight, cumulative products for
the transmittance); nothing is taken over from csrc/pair_math.cuh.

Besides the outputs it returns, per element, the ERROR BUDGET of an fp32 implementation (`blend_reference` docstring),
and classifies every (pixel, entry) pair by its distance to the four decisions a blend takes:
  power = 0,  alpha' = 1/255 (skip),  T (1 - alpha') = 1e-4 (stop),  opacity G = 0.99 (cap).
A pixel with a pair within the margin of one of them may legitimately decide otherwise in fp32; such pixels, and the
Gaussians that receive gradient from them, are left out of the strict comparisons (`near_pixel`, `near_gauss`).

num_node_kids follows the documented rule (include/h3dgs.h): k <= 1 is the identity, counts above 65535 act as 65535.
"""
import numpy as np

ALPHA_CAP = float(np.float32(0.99))          # the kernels compare against the fp32 constants
ALPHA_SKIP = float(np.float32(1.0 / 255.0))
T_STOP = float(np.float32(1e-4))
KIDS_MAX = 65535
TILE = 16
U = 2.0 ** -24                               # fp32 unit roundoff
MARGIN = 1e-5                                # smallest relative decision margin
PAIRS_PER_CHUNK = 1 << 17

# ---- error analysis (fp32 + MUFU), relative errors -------------------------------------------------------------------
# exponent: power = (C d + B) d + A in fp32 carries a few ulp of the magnitude of its terms, mag = |A| + |B d| + |C d^2|
#   -> G = ex2.approx(power log2 e): relative error <= 4 U mag + 2^-22 (ex2.approx) + U (the log2 e product).
# hierarchy weight (k > 1, t < 1): series branches < 2e-7, MUFU.LG2 ~2^-22 absolute on log2(1-a) >= 0.093 in magnitude
#   (a >= 1/16) -> 2e-6, and 1 - MUFU.EX2 for a result >= 0.06 -> 2^-22 / 0.06 = 4e-6:  EPS_HIER = 4e-6.
# transmittance: every taken entry multiplies (forward) or divides (backward: rcp.approx + one Newton step, ~1 ulp) T
#   by 1 - alpha, whose relative error is U + eps_alpha alpha / (1 - alpha); these add up along the pixel's list.
EPS_EX2 = 2.0 ** -22
EPS_HIER = 4e-6


def kids_rule(k):
    k = np.asarray(k, np.int64)
    return np.where(k <= 1, 1, np.minimum(k, KIDS_MAX))


def hier_weight(ab, t, k):
    """alpha' = t a + (1-t)(1 - (1-a)^(1/k)) and d alpha'/d a, float64; identity for k <= 1 or t >= 1."""
    k = kids_rule(k).astype(np.float64)
    act = (k > 1) & (t < 1)
    kk = np.where(act, k, 2.0)
    omr = -np.expm1(np.log1p(-ab) / kk)
    al = np.where(act, t * ab + (1 - t) * omr, ab)
    dadb = np.where(act, t + (1 - t) / kk * np.exp((1.0 / kk - 1.0) * np.log1p(-ab)), 1.0)
    return al, dadb, act


def blend_reference(records, ranges, point_list, W, H, bg, dL_dcolor=None, dL_dinvdepth=None, hier=False, do_depth=False,
                    kids=None):
    """records [P][12] fp32, ranges [tiles][2], point_list [D]; bg [3]; dL_dcolor [3,H,W]; dL_dinvdepth [H,W] (do_depth);
    kids [P]: the num_node_kids the renderer was given (default: the count K1 stored in the records' kbits).

    Returns a dict of float64 arrays:
      color [3,H,W], invdepth [H,W], final_T [H,W], n_contrib [H,W] (int64: 1-based list position of the last
      contributor), and their budgets color_tol [H,W], final_T_tol [H,W]: the largest |fp32 - exact| an implementation
      with the error analysis above may show (per pixel: sum_i w_i |c_i| e_i + T |bg| e_T);
      accum [P][10] (the blend's per-Gaussian sums in the accumulator layout of csrc/common.cuh, before the constant
      factors 0.5 W, 0.5 H, -0.5), accum_abs [P][10] (the sum of the absolute per-pixel terms: the scale that fp32
      summation error is bounded by), accum_tol [P][10] (the per-element budget: per-pair relative error times the
      pair's absolute term, plus n U accum_abs for the n-term fp32 sum);
      near_pixel [H,W], near_gauss [P] (bool): the exclusion sets; near_kind: counts per decision kind.
    """
    rec = np.asarray(records, np.float64)
    P = rec.shape[0]
    ranges = np.asarray(ranges, np.int64).reshape(-1, 2)
    point_list = np.asarray(point_list, np.int64)
    kbits = np.asarray(records, np.float32)[:, 7].view(np.uint32).astype(np.int64)
    # the count as the documented rule makes it from the caller's k, or from what K1 stored (bits 0..19)
    kids = kids_rule(kbits & 0xFFFFF if kids is None else kids)
    bg = np.asarray(bg, np.float64)
    gx = (W + TILE - 1) // TILE
    out = dict(color=np.zeros((3, H, W)), invdepth=np.zeros((H, W)), final_T=np.ones((H, W)),
               n_contrib=np.zeros((H, W), np.int64),
               color_tol=np.full((H, W), 1e-30), final_T_tol=np.full((H, W), 1e-30), invdepth_tol=np.full((H, W), 1e-30),
               accum=np.zeros((P, 10)), accum_abs=np.zeros((P, 10)), accum_tol=np.zeros((P, 10)),
               near_pixel=np.zeros((H, W), bool), near_gauss=np.zeros(P, bool),
               near_kind=dict(power=0, skip=0, stop=0, cap=0))
    npix_of = np.zeros(P)                      # pixels each Gaussian's sums collect (the fp32 sum's length)
    backward = dL_dcolor is not None
    if backward:
        gcol = np.asarray(dL_dcolor, np.float64).reshape(3, H, W)
        gdep = np.asarray(dL_dinvdepth, np.float64).reshape(H, W) if (do_depth and dL_dinvdepth is not None) else None
    for tile in range(ranges.shape[0]):
        tx, ty = tile % gx, tile // gx
        ys_t, xs_t = np.meshgrid(np.arange(ty * TILE, min(ty * TILE + TILE, H)), np.arange(tx * TILE, min(tx * TILE + TILE, W)),
                                 indexing="ij")
        ys_t, xs_t = ys_t.ravel(), xs_t.ravel()
        s, e = ranges[tile]
        if ys_t.size == 0:
            continue
        if e <= s:
            for c in range(3):
                out["color"][c, ys_t, xs_t] = bg[c]
            continue
        ids = point_list[s:e]
        # the tile's pixels in chunks of about PAIRS_PER_CHUNK (pixel, entry) pairs: a deep list does not hold its ~40
        # [pixels x entries] float64 arrays for all 256 pixels at once.  Per pixel the decisions are the same and the
        # values differ by the float64 rounding of the matrix products only; the per-Gaussian sums add the chunks'
        # partial sums in another order.
        step = int(np.clip(PAIRS_PER_CHUNK // ids.size, 1, ys_t.size))
        for c0 in range(0, ys_t.size, step):
            ys, xs = ys_t[c0:c0 + step], xs_t[c0:c0 + step]
            _blend_pixels(out, rec, ids, xs, ys, kids, bg, hier, npix_of, gcol if backward else None,
                          gdep if backward else None)
    # the per-Gaussian sums are fp32 additions of up to npix terms (span reductions, then atomics in any order)
    out["accum_tol"] = 2 * out["accum_tol"] + (8 + npix_of)[:, None] * U * out["accum_abs"] + 1e-30
    out["npix"] = npix_of
    return out


def _blend_pixels(out, rec, ids, xs, ys, kids, bg, hier, npix_of, gcol, gdep):
    """blend_reference's work for the pixels (xs, ys) of one tile over its list ids, written into `out`"""
    R = rec[ids]
    x, y, cx, cy, cz, op, t, rgb, invd = R[:, 0], R[:, 1], R[:, 2], R[:, 3], R[:, 4], R[:, 5], R[:, 6], R[:, 8:11], R[:, 11]
    dx = x[None] - xs[:, None]
    dy = y[None] - ys[:, None]
    power = -0.5 * (cx * dx * dx + cz * dy * dy) - cy * dx * dy
    mag = 0.5 * (np.abs(cx) * dx * dx + np.abs(cz) * dy * dy) + np.abs(cy * dx * dy)
    G = np.exp(power)
    araw = op * G
    ab = np.minimum(ALPHA_CAP, araw)
    if hier:
        al, dadb, act = hier_weight(ab, t[None], kids[ids][None])
    else:
        al, dadb, act = ab, np.ones_like(ab), np.zeros_like(ab, bool)
    eps_a = 4 * U * mag + EPS_EX2 + 3 * U + np.where(act, EPS_HIER, 0.0)
    valid = (power <= 0) & (al >= ALPHA_SKIP)
    aeff = np.where(valid, al, 0.0)
    Tall = np.cumprod(1 - aeff, axis=1)
    contrib = valid & (Tall >= T_STOP)
    a_c = np.where(contrib, al, 0.0)
    Tafter = np.cumprod(1 - a_c, axis=1)
    Tbefore = np.concatenate([np.ones((xs.size, 1)), Tafter[:, :-1]], 1)
    Tfin = Tafter[:, -1]
    n = ids.size
    pos = np.arange(1, n + 1)
    last = np.where(contrib, pos[None], 0).max(1)
    w = a_c * Tbefore
    # T's relative error in front of each entry, and at the end
    tstep = np.where(contrib, U + eps_a * a_c / (1 - a_c), 0.0)
    kap_before = np.concatenate([np.zeros((xs.size, 1)), np.cumsum(tstep, 1)[:, :-1]], 1)
    kap = tstep.sum(1)
    # decisions: pairs up to the stopping entry (or the end of the list) are the ones that matter
    stop_pos = np.where((valid & ~contrib).any(1), np.argmax(valid & ~contrib, 1), n - 1)
    rel = pos[None] - 1 <= stop_pos[:, None]
    m = np.maximum(MARGIN, 4 * eps_a)
    near_pw = rel & (power != 0) & (np.abs(power) <= MARGIN * mag)
    near_sk = rel & (power <= 0) & (np.abs(al - ALPHA_SKIP) <= m * ALPHA_SKIP)
    near_cap = rel & (power <= 0) & (np.abs(araw - ALPHA_CAP) <= m * ALPHA_CAP)
    mT = np.maximum(MARGIN, 4 * (kap_before + eps_a * al / np.maximum(1 - al, 1e-3)))
    near_st = rel & valid & (np.abs(Tbefore * (1 - al) - T_STOP) <= mT * T_STOP)
    near = near_pw | near_sk | near_cap | near_st
    for kname, arr in (("power", near_pw), ("skip", near_sk), ("cap", near_cap), ("stop", near_st)):
        out["near_kind"][kname] += int(arr.any(1).sum())
    npx = near.any(1)
    out["near_pixel"][ys[npx], xs[npx]] = True
    if npx.any():
        hit = (valid | near_sk)[npx].any(0)
        out["near_gauss"][ids[hit]] = True

    e_pair = 2 * kap[:, None] + 2 * eps_a + 16 * U           # relative error budget of one pair's terms
    col = w @ rgb + Tfin[:, None] * bg[None]
    out["color"][:, ys, xs] = col.T
    out["color_tol"][ys, xs] = 2 * ((w * e_pair) @ np.abs(rgb).max(1) + Tfin * np.abs(bg).max() * (kap + U)) + 1e-12
    out["final_T"][ys, xs] = Tfin
    out["final_T_tol"][ys, xs] = 2 * Tfin * (kap + U) + 1e-30
    out["invdepth"][ys, xs] = w @ invd
    out["invdepth_tol"][ys, xs] = 2 * ((w * e_pair) @ np.abs(invd)) + 1e-12
    out["n_contrib"][ys, xs] = last
    if gcol is None:
        return
    gc = gcol[:, ys, xs].T                                   # [m][3]
    cg = rgb @ gc.T                                          # [n][m] -> transposed below
    cg = cg.T
    cg_abs = np.abs(rgb) @ np.abs(gc).T
    cg_abs = cg_abs.T
    if gdep is not None:
        gd = gdep[ys, xs]
        cg = cg + invd[None] * gd[:, None]
        cg_abs = cg_abs + np.abs(invd)[None] * np.abs(gd)[:, None]
    bgd = gc @ bg
    wcg = w * cg
    behind = np.cumsum(wcg[:, ::-1], 1)[:, ::-1] - wcg        # sum over the contributors behind each entry
    behind_abs = np.cumsum((w * cg_abs)[:, ::-1], 1)[:, ::-1] - w * cg_abs
    om = np.where(contrib, 1 - a_c, 1.0)
    dL_da = np.where(contrib, Tbefore * cg - (behind + Tfin[:, None] * bgd[:, None]) / om, 0.0)
    dL_da_abs = np.where(contrib, Tbefore * cg_abs + (behind_abs + Tfin[:, None] * np.abs(bgd)[:, None]) / om, 0.0)
    dL_dab, dL_dab_abs = dL_da * dadb, dL_da_abs * np.abs(dadb)
    p, p_abs = G * dL_dab, G * dL_dab_abs
    o = op[None]
    terms = [
        (o * p * -(cx * dx + cy * dy), o * p_abs * (np.abs(cx * dx) + np.abs(cy * dy))),
        (o * p * -(cy * dx + cz * dy), o * p_abs * (np.abs(cy * dx) + np.abs(cz * dy))),
        (o * p * dx * dx, o * p_abs * dx * dx),
        (o * p * dx * dy, o * p_abs * np.abs(dx * dy)),
        (o * p * dy * dy, o * p_abs * dy * dy),
        (p, p_abs),
    ]
    for c in range(3):
        terms.append((w * gc[:, c:c + 1], w * np.abs(gc[:, c:c + 1])))
    if gdep is not None:
        terms.append((w * gd[:, None], w * np.abs(gd[:, None])))
    npix = contrib.sum(0)
    np.add.at(npix_of, ids, npix)
    for col_i, (v, va) in enumerate(terms):
        np.add.at(out["accum"][:, col_i], ids, v.sum(0))
        np.add.at(out["accum_abs"][:, col_i], ids, va.sum(0))
        np.add.at(out["accum_tol"][:, col_i], ids, (va * e_pair).sum(0))


def compare(got, want, tol, mask=None):
    """max of |got - want| / tol over the unmasked elements (<= 1 passes) and how many elements were compared."""
    got = np.asarray(got, np.float64); want = np.asarray(want, np.float64); tol = np.broadcast_to(tol, want.shape)
    keep = np.ones(want.shape, bool) if mask is None else np.broadcast_to(mask, want.shape)
    if not keep.any():
        return 0.0, 0
    r = np.abs(got - want)[keep] / tol[keep]
    return float(r.max()), int(keep.sum())

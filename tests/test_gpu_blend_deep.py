"""GPU: the blend kernels (render_forward.cu, render_backward.cu) and the tile sort (binning.cu, api.cu) on DEEP tile
lists, per pixel and per Gaussian against tests/blend_ref.py's float64 blend, with the criteria of
test_gpu_blend_edges.run_case (n_contrib exact, each value inside its derived budget).  Depth is where the
kernels' batch logic runs: many 256-entry TMA batches (the forward's double buffer and its mbarrier phases, the
backward's back-to-front walk that starts with the partial batch), every size class of the tile sort and the global radix
sort beyond 8192 entries, stops in late batches, and tile_max_contrib cutting a list beyond 512.

Deep random scenes would not do: with thousands of (pixel, entry) pairs per pixel almost every pixel has one within
blend_ref's decision margin, and the Gaussians it takes are left out.  These scenes are free of near decisions by
construction:
  - isotropic Gaussians whose means sit on pixel centres, so at a pixel q = c (dx^2 + dy^2) only takes values near c times
    a sum of two squares.  Each opacity is set from the kernel's own fp32 record (centre, conic) so that the 1/255 cut,
    q = 2 ln(o / a*) with a* the base alpha whose hierarchy weight is 1/255 (a* = 1/255 without the weight), falls
    midway between two consecutive values of q that occur;
  - alphas stay at or below 0.97, away from the 0.99 cap;
  - a stop is a wall: a tiny Gaussian of alpha 0.97 at its centre pixel behind darkeners that bring the transmittance in
    front of it to 5e-4, so T (1 - alpha) drops from 5e-4 to 1.5e-5 at the wall, and no other pixel comes near 1e-4.
blend_ref's classification is the judge: every case asserts that no pixel is near a decision, that at least 95 % of the
listed Gaussians are compared, and that the budget, which grows with the list, still says something (its median over the
value).  The tile lists are checked apart from blend_ref, which consumes them: per tile, point_list is numpy's stable sort
by (depth bits, index) of the rows whose fp32 rect (preprocess_ref.rect_fp32) touches the tile."""
import numpy as np
import pytest

from blend_ref import ALPHA_SKIP, ALPHA_CAP, TILE, hier_weight
from preprocess_ref import rect_fp32
from test_gpu_blend_edges import Scene, _cam, _grads, _render, run_case

pytestmark = pytest.mark.gpu

BATCH = 256                       # entries per TMA batch of both blend kernels
LENGTHS = (1, 128, 129, 256, 257, 511, 512, 513, 1024, 1025, 2048, 4097, 8192)   # every sort class and batch boundary
RADIX = 8200                      # above the shared-memory sort's 8192: the frame goes through the global radix sort
TINY = 0.05                       # px; the 0.3 px^2 dilation dominates: radius 3
INNER = tuple(range(4, 12))       # offsets in a tile at which a tiny Gaussian touches no other (a pixel of fp32 slack)
O_MAX = 0.9                       # largest opacity the snap may choose (walls excepted)
WALL_ALPHA = 0.97
T_WALL = 5e-4                     # transmittance in front of a wall
N_DARK = 8                        # darkeners per wall, the last one directly in front of it
VARIANTS = {"flat": (False, False), "depth": (False, True), "hier": (True, True)}


class Deep:
    """a Scene whose rows carry a target opacity and a role (bg, medium, wall, dark, ghost, end)"""

    def __init__(self, W, H, hier, seed):
        self.sc = Scene(_cam(W, H))
        self.hier = hier
        self.rng = np.random.default_rng(seed)
        self.target, self.role = [], []

    def add(self, u, v, z, sigma, o, role):
        t, k = 1.0, 1
        if self.hier:
            r = self.rng
            if role in ("bg", "medium"):
                t = [0.0, 0.5, float(r.uniform())][r.integers(3)]
                k = int(r.choice([2, 17, 70000]))
            else:                 # walls, darkeners, ghosts and ends keep their alpha: the weight's identity cases
                t, k = (1.0, int(r.choice([2, 17, 70000]))) if r.uniform() < 0.5 else (float(r.uniform()), int(r.choice([0, 1])))
        self.target.append(o)
        self.role.append(role)
        return self.sc.add(u, v, z, sigma, sigma, op=o, t=t, k=k, rng=self.rng)


def _a_star(ts, kids, hier):
    """per row the base alpha whose hierarchy weight is 1/255 (NaN: the weight stays below 1/255 up to the cap)"""
    n = len(ts)
    if not hier:
        return np.full(n, ALPHA_SKIP)
    t, k = np.asarray(ts, np.float64), np.asarray(kids, np.int64)
    lo, hi = np.zeros(n), np.full(n, ALPHA_CAP)
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        below = hier_weight(mid, t, k)[0] < ALPHA_SKIP
        lo, hi = np.where(below, mid, lo), np.where(below, hi, mid)
    never = hier_weight(np.full(n, ALPHA_CAP), t, k)[0] < ALPHA_SKIP * 1.01
    return np.where(never, np.nan, 0.5 * (lo + hi))


def _q(rec, i, W, H):
    """float64 q = -2 power of record i at every pixel that q <= 12 could reach, and the conic's small eigenvalue"""
    x, y, cx, cy, cz = (float(a) for a in rec[i, :5])
    lam = 0.5 * (cx + cz) - np.hypot(0.5 * (cx - cz), cy)
    r = int(np.sqrt(12.0 / lam)) + 2
    us = np.arange(max(0, int(x) - r), min(W, int(x) + r + 2))
    vs = np.arange(max(0, int(y) - r), min(H, int(y) + r + 2))
    dx, dy = x - us[None, :], y - vs[:, None]
    return np.sort((cx * dx * dx + cz * dy * dy + 2 * cy * dx * dy).ravel()), lam


def _snap(rec, i, W, H, o_target, a_star):
    """the opacity nearest o_target (<= O_MAX) whose 1/255 cut lies midway between two consecutive values of q"""
    q, lam = _q(rec, i, W, H)
    cut = np.nonzero(np.diff(q) > 0.25 * lam)[0]              # clusters: q of one sum of two squares
    lo_edge = np.r_[q[0] - lam, q[cut]]                        # below the first cluster: nothing is taken
    hi_edge = np.r_[q[0], q[cut + 1]]
    o = a_star * np.exp(0.25 * (lo_edge + hi_edge))
    o = o[o <= O_MAX]
    return float(o[np.argmin(np.abs(np.log(o / o_target)))])


def _alpha_at(rec, op, ids, u, v, hier, ts, kids):
    """float64 alpha' of the entries ids at pixel (u, v), 0 where not taken (power > 0 or below 1/255)"""
    x, y, cx, cy, cz = (rec[ids, c].astype(np.float64) for c in range(5))
    dx, dy = x - u, y - v
    power = -0.5 * (cx * dx * dx + cz * dy * dy) - cy * dx * dy
    ab = np.minimum(ALPHA_CAP, np.float32(op[ids]).astype(np.float64) * np.exp(power))
    al = hier_weight(ab, ts[ids], kids[ids])[0] if hier else ab
    return np.where((power <= 0) & (al >= ALPHA_SKIP), al, 0.0)


def _opacities(d, st, walls=()):
    """snap every row's opacity from the first render's records; walls [(tile, p, u, v)]: the wall at 1-based list
    position p of its tile gets alpha 0.97 at (u, v), the N_DARK darkeners in front of it bring T there to T_WALL"""
    cam, sc = d.sc.cam, d.sc
    rec = st["records"]
    ts, kids = np.asarray(sc.ts, np.float64), np.asarray(sc.kids, np.int64)
    a_star = _a_star(ts, kids, d.hier)
    op = np.array(d.target, np.float64)
    for i, role in enumerate(d.role):
        if role in ("bg", "medium", "ghost", "end") and np.isfinite(a_star[i]):
            op[i] = _snap(rec, i, cam.W, cam.H, op[i], a_star[i])
    G = lambda i, u, v: np.exp(-0.5 * _q_at(rec, i, u, v))
    for tile, p, u, v in walls:
        s, _ = st["ranges"][tile]
        ids = st["point_list"][s:s + p].astype(np.int64)           # the list up to the wall
        assert d.role[ids[-1]] == "wall" and all(d.role[j] == "dark" for j in ids[-1 - N_DARK:-1])
        T_rest = np.prod(1 - _alpha_at(rec, op, ids[:-1 - N_DARK], u, v, d.hier, ts, kids))
        a_d = 1 - (T_WALL / T_rest) ** (1.0 / N_DARK)
        assert 0.05 < a_d < 0.8, (tile, p, T_rest)
        for j in ids[-1 - N_DARK:-1]:
            op[j] = a_d / G(j, u, v)
        op[ids[-1]] = WALL_ALPHA / G(ids[-1], u, v)
    return op


def _q_at(rec, i, u, v):
    x, y, cx, cy, cz = (float(a) for a in rec[i, :5])
    dx, dy = x - u, y - v
    return cx * dx * dx + cz * dy * dy + 2 * cy * dx * dy


def _check_lists(st, W, H):
    """per tile: point_list = stable sort by (depth bits, index) of the rows whose fp32 rect touches the tile, and
    keys_sorted = (tile << 32) | depth bits"""
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    radii = st["radii"]
    vis = radii > 0
    x0, y0, x1, y1 = rect_fp32(st["records"][:, 0], st["records"][:, 1], radii, W, H)
    dbits = st["depths"].view(np.uint32)
    pl = st["point_list"].astype(np.int64)
    keys = st["keys_sorted"].view(np.uint64)
    for tile in range(gx * gy):
        tx, ty = tile % gx, tile // gx
        rows = np.nonzero(vis & (x0 <= tx) & (tx < x1) & (y0 <= ty) & (ty < y1))[0]
        want = rows[np.lexsort((rows, dbits[rows]))]
        s, e = (int(a) for a in st["ranges"][tile])
        assert e - s == rows.size, (tile, e - s, rows.size)
        assert np.array_equal(pl[s:e], want), (tile, "point_list", int(np.argmax(pl[s:e] != want)))
        assert np.array_equal(keys[s:e], (np.uint64(tile) << np.uint64(32)) | dbits[want].astype(np.uint64)), (tile, "keys")


def _run(name, d, variant, walls=()):
    """tune the opacities from a first render, then run_case; check the lists, the exclusions and the budget's bars"""
    hier, do_depth = VARIANTS[variant]
    cam = d.sc.cam
    gcol, gdep = _grads(cam, 0)
    _, _, st0, _ = _render(d.sc, np.zeros(3, np.float32), hier, False, gcol, gdep)
    _check_lists(st0, cam.W, cam.H)          # the walls are placed by list position
    op = _opacities(d, st0, walls)
    assert op.max() <= WALL_ALPHA * 1.001
    ref, rec, run = run_case(f"{name} {variant}", d.sc, hier=hier, do_depth=do_depth, op=op, seed=11,
                             max_near_pixels=0.0, max_near_gauss=0.0)
    st = run[2]
    _check_lists(st, cam.W, cam.H)
    assert np.array_equal(st["point_list"], st0["point_list"])
    # the construction holds: no pixel near a decision, (nearly) every listed Gaussian compared
    assert not ref["near_pixel"].any(), ref["near_kind"]
    listed = np.unique(st["point_list"])
    compared = float((~ref["near_gauss"][listed]).mean())
    assert compared >= 0.95
    # the budget still says something at this depth (measured medians: colour 1.2e-7, sums up to 1.2e-4)
    keep = ~ref["near_pixel"]
    cmag = np.abs(ref["color"]).max(0)
    col_rel = float(np.median((ref["color_tol"] / cmag)[keep & (cmag > 0)]))
    rows = ~ref["near_gauss"] & (ref["npix"] > 0)
    aa, at = ref["accum_abs"][rows], ref["accum_tol"][rows]
    acc_rel = float(np.median(at[aa > 0] / aa[aa > 0]))
    assert col_rel <= 1e-5 and acc_rel <= 1e-3, (col_rel, acc_rel)
    lens = np.diff(st["ranges"].astype(np.int64), axis=1).ravel()
    print(f"[{name} {variant}] lists up to {lens.max()} entries, {compared:.1%} of {listed.size} listed Gaussians "
          f"compared, up to {int(ref['npix'].max())} pixels per Gaussian; median budget / value: colour {col_rel:.2e}, "
          f"sums {acc_rel:.2e}")
    return ref, run, lens


def _fill_tile(d, tx, ty, n, depths, rng):
    """n tiny Gaussians inside tile (tx, ty): two thirds taken at their centre pixel only, the rest at distance <= 1"""
    for _ in range(n):
        u, v = TILE * tx + int(rng.choice(INNER)), TILE * ty + int(rng.choice(INNER))
        d.add(u, v, float(rng.choice(depths)), TINY, 0.009 if rng.uniform() < 2 / 3 else 0.045, "bg")


# ---- every size class of the tile sort and every batch boundary ----------------------------------------------------------
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_every_sort_class_and_batch_boundary(variant):
    """One 160 x 64 frame whose tiles hold 1, 128, 129, 256, 257, 511, 512, 513, 1024, 1025, 2048, 4097 and 8192
    entries: every register-sort class and the shared-memory network of the tile sort, and 1 to 32 TMA batches.  The deep
    tiles also lie under medium Gaussians (sigma 4 to 12 px) whose sums collect thousands of pixels.  Depths come from 40
    values, so the (depth, index) order decides among equal depths."""
    hier = VARIANTS[variant][0]
    d = Deep(160, 64, hier, seed=31)
    rng = np.random.default_rng(32)
    depths = 2.0 + 0.05 * np.arange(40)
    for u, v, s in ((120, 40, 12), (128, 24, 12), (112, 30, 8), (136, 48, 8), (100, 20, 4), (144, 40, 4)):
        d.add(u, v, float(rng.choice(depths)), s, 0.3, "medium")
    # the medium Gaussians' tiles, from their own fp32 rects
    gcol, gdep = _grads(d.sc.cam, 0)
    _, _, stm, _ = _render(d.sc, np.zeros(3, np.float32), hier, False, gcol, gdep)
    gx = 10
    mx0, my0, mx1, my1 = rect_fp32(stm["records"][:, 0], stm["records"][:, 1], stm["radii"], 160, 64)
    under = lambda tx, ty: int(((mx0 <= tx) & (tx < mx1) & (my0 <= ty) & (ty < my1) & (stm["radii"] > 0)).sum())
    place = dict(zip(LENGTHS, [(0, 0), (0, 1), (0, 2), (0, 3), (1, 0), (1, 1), (1, 2), (1, 3), (5, 1), (6, 1), (7, 1), (8, 1),
                               (9, 1)]))
    for n, (tx, ty) in place.items():
        assert n >= under(tx, ty)
        _fill_tile(d, tx, ty, n - under(tx, ty), depths, rng)
    ref, run, lens = _run("sort classes", d, variant)
    for n, (tx, ty) in place.items():
        assert lens[ty * gx + tx] == n, (n, int(lens[ty * gx + tx]))
    assert lens.max() == 8192
    # Gaussians whose sums collect thousands of pixels, pixels that take hundreds of entries
    assert ref["npix"].max() > 1000
    assert ref["n_contrib"].max() > 4 * BATCH
    dep = run[2]["depths"][run[2]["radii"] > 0]
    assert np.unique(dep).size <= 40 < dep.size


# ---- the global radix sort beyond 8192 entries ---------------------------------------------------------------------------
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_radix_sort_hand_over(variant):
    """A tile of 8200 entries, beyond the shared-memory sort: the whole frame is binned by the global radix sort, whose
    stable order over (tile, depth) must equal the per-tile sort's (depth, index)."""
    d = Deep(48, 32, VARIANTS[variant][0], seed=41)
    rng = np.random.default_rng(42)
    depths = 2.0 + 0.05 * np.arange(30)
    for (tx, ty), n in (((1, 0), RADIX), ((0, 1), 300), ((2, 1), 1), ((0, 0), 129)):
        _fill_tile(d, tx, ty, n, depths, rng)
    ref, run, lens = _run("radix", d, variant)
    assert lens.max() == RADIX and sorted(lens[lens > 0]) == [1, 129, 300, RADIX]
    assert ref["n_contrib"].max() > 16 * BATCH


# ---- stops at the batch edges, stops in different batches, tile_max_contrib cuts -----------------------------------------
# per tile: (list length, [(1-based wall position, pixel offset in the tile)], last entry anyone takes or None)
WALL_TILES = [
    (1100, [(255, (4, 4)), (511, (11, 4)), (767, (4, 11)), (1023, (11, 11))], None),
    (1100, [(256, (4, 4)), (512, (11, 4)), (768, (4, 11)), (1024, (11, 11))], None),
    (1100, [(257, (4, 4)), (513, (11, 4)), (769, (4, 11)), (1025, (11, 11))], None),
    (700, [(300, (8, 8)), (700, (4, 11))], None),                    # a wall as the last entry
    (600, [(100, (4, 4)), (400, (11, 11))], 512),
    (640, [(250, (11, 4)), (300, (4, 11))], 513),
    (900, [(256, (8, 4)), (600, (4, 8))], 700),
    (1100, [(513, (4, 4)), (900, (11, 8))], 1024),
    (1200, [(257, (11, 11)), (1000, (8, 11))], 1025),
]


def _wall_sequence(n, walls, last, rng):
    """the tile's list, front to back: walls with their darkeners; behind `last` only ghosts (taken at their centre pixel
    alone, which a wall has stopped by then); background everywhere else, centred off the wall pixels"""
    seq = [None] * n
    for p, pix in walls:
        seq[p - 1] = ("wall", pix)
        for j in range(p - 1 - N_DARK, p - 1):
            assert seq[j] is None
            seq[j] = ("dark", pix)
    if last is not None:
        assert max(p for p, _ in walls) < last
        for j in range(last, n):
            seq[j] = ("ghost", walls[j % len(walls)][1])
    wall_pix = {pix for _, pix in walls}
    free = [(a, b) for a in INNER for b in INNER if (a, b) not in wall_pix]
    end = (n if last is None else last) - 1
    if seq[end] is None:          # the last entry any pixel takes: background that every variant takes at its centre
        seq[end] = ("end", free[rng.integers(len(free))])
    for j in range(n):
        if seq[j] is None:
            seq[j] = ("bg", free[rng.integers(len(free))])
    return seq


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_walls_at_batch_edges_and_cuts(variant):
    """Walls at 1-based list positions 256k - 1, 256k and 256k + 1 (k = 1..4) and at the last entry, each in another
    8x8 quadrant of its tile, so that warps and groups of one tile stop in different batches; the pixels without a wall
    never stop.  In the last five tiles nothing behind entry 512, 513, 700, 1024 or 1025 is taken by any pixel, so
    tile_max_contrib cuts the backward's list at a batch edge, just past one, or mid-batch.  The list order is fixed by
    depth, three entries per depth value (the index decides among them)."""
    d = Deep(80, 32, VARIANTS[variant][0], seed=51)
    rng = np.random.default_rng(52)
    gx = 5
    seqs = [_wall_sequence(n, walls, last, rng) for n, walls, last in WALL_TILES]
    opac = dict(bg=None, wall=WALL_ALPHA, dark=0.5, ghost=0.009, end=0.045)
    for j in range(max(len(s) for s in seqs)):              # rows of all tiles interleaved, indices rise along each list
        for t, seq in enumerate(seqs):
            if j < len(seq):
                role, (a, b) = seq[j]
                o = opac[role] if role != "bg" else (0.009 if rng.uniform() < 1 / 3 else 0.045)
                d.add(TILE * (t % gx) + a, TILE * (t // gx) + b, 2.0 + 0.004 * (j // 3), TINY, o, role)
    walls = [(t, p, TILE * (t % gx) + a, TILE * (t // gx) + b) for t, (_, ws, _) in enumerate(WALL_TILES) for p, (a, b) in ws]
    ref, run, lens = _run("walls", d, variant, walls=walls)
    st = run[2]
    assert [int(lens[t]) for t in range(len(WALL_TILES))] == [n for n, _, _ in WALL_TILES]
    positions = sorted(p for _, p, _, _ in walls)
    assert {256 * k + e for k in range(1, 5) for e in (-1, 0, 1)} <= set(positions)
    wall_mask = np.zeros(ref["final_T"].shape, bool)
    for t, p, u, v in walls:
        # the wall stops the pixel: its last contributor is the darkener directly in front of it
        assert ref["n_contrib"][v, u] == p - 1 and st["n_contrib"][v, u] == p - 1, (t, p, int(st["n_contrib"][v, u]))
        assert 2.5e-4 <= ref["final_T"][v, u] <= 1e-3
        wall_mask[v, u] = True
    assert (ref["final_T"][~wall_mask] > 2e-4).all()                  # nothing else comes near the stop
    for t, (n, _, last) in enumerate(WALL_TILES):
        tx, ty = t % gx, t // gx
        blk = (slice(TILE * ty, TILE * ty + TILE), slice(TILE * tx, TILE * tx + TILE))
        want = n if last is None else last
        assert ref["n_contrib"][blk].max() == want and st["n_contrib"][blk].max() == want, (t, want)

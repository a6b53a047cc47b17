"""GPU: the block reach mask the record gather stores in the sorted records (binning.cu: tile_sort_gather_kernel and, past
the tile sort's capacity, gather_records_kernel; csrc/reach_mask.cuh::block_mask16), against tests/reach_ref.py's
float64 judge.  Both blend kernels skip every 4x4 block whose bit is clear, so the mask decides pixels.

Every case renders through _C.rasterize_gaussians and reads sorted_records, point_list, keys_sorted and ranges with
_C.state_view.  Per entry j (tile = keys_sorted[j] >> 32):
  - copy: words 0..6 and 8..11 of sorted_records[j] equal records[point_list[j]] bit for bit; the low 16 bits of word 7
    are min(kbits & 0xFFFFF, 65535), the high 16 bits the mask;
  - conservative: the judge's needed blocks (a pixel taken, or within blend_ref's decision margin) are all marked;
  - tight: marked blocks that are neither touched by the float64 ellipse nor needed stay <= 2 % of the marked blocks
    of the regular records per family, and the fallback 0xFFFF (a full mask where fewer than half of the blocks are
    touched or needed) appears only on degenerate records;
  - degenerate records: a listed conic that is not positive definite gets 0xFFFF whenever its opacity can be taken;
    a NaN opacity gets 0 or 0xFFFF.  K1 lists indefinite conics (it only rejects det = 0) and keeps rows with a NaN
    opacity visible; rows whose mean or conic is not finite do not project and are never listed, so the gather cannot
    see them -- block_mask16's answer for those is checked on the host (tests/emul/reach_mask_test.cpp).
On the needle and 1/255 scenes the consequence is checked end to end as well: n_contrib and the image equal
blend_ref's float64 blend (within its budget) on every pixel where neither the judge nor blend_ref finds a pair near a
decision.
Per family the entries, needed / marked / untouched blocks and any misses are printed (-s)."""
import numpy as np
import pytest

from blend_ref import ALPHA_SKIP, blend_reference, compare
from reach_ref import degenerate, judge
from test_gpu_blend_edges import Scene, _cam, _place

pytestmark = pytest.mark.gpu

KIDS_MAX = 65535


def _frame(sc, hier=False, shard=(1, 0), bg=(0.1, 0.4, 0.9)):
    import torch
    from diff_gaussian_rasterization import _C
    cam = sc.cam
    f = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    m, cov, rgb = f(sc.means), f(sc.covs), f(sc.rgb)
    opac = f(np.asarray(sc.op, np.float32).reshape(-1, 1))
    ts = f(sc.ts) if hier else None
    kids = torch.tensor(np.asarray(sc.kids, np.int64).astype(np.int32), device="cuda") if hier else None
    n, color, radii, gb, bb, ib, _ = _C.rasterize_gaussians(f(bg), m, rgb, opac, None, None, 1.0, cov,
                                                            f(cam.world_view_transform), f(cam.full_proj_transform),
                                                            cam.tanfovx, cam.tanfovy, cam.H, cam.W, None, 0,
                                                            f(cam.camera_center), False, False, None, None, ts, kids,
                                                            False, shard=shard)
    st = {k: v.cpu().numpy().copy() for k, v in _C.state_view(m.shape[0], cam.W, cam.H, n, gb, bb, ib).items()}
    st["radii"], st["color"], st["D"] = radii.cpu().numpy(), color.cpu().numpy(), n
    return st


def check_masks(name, sc, st, hier=False, tight=0.02):
    """the copy, conservative and tight checks over every entry of the frame; returns the judge's output"""
    cam = sc.cam
    gx = (cam.W + 15) // 16
    D = st["D"]
    assert D > 0, name
    rec, srt, pl = st["records"], st["sorted_records"], st["point_list"].astype(np.int64)
    tiles = (st["keys_sorted"].view(np.uint64) >> np.uint64(32)).astype(np.int64)
    src = rec[pl].view(np.uint32)
    got = srt.view(np.uint32)
    words = [0, 1, 2, 3, 4, 5, 6, 8, 9, 10, 11]
    assert np.array_equal(got[:, words], src[:, words]), (name, "record copy")
    assert np.array_equal(got[:, 7] & 0xFFFF, np.minimum(src[:, 7] & 0xFFFFF, KIDS_MAX)), (name, "kids")
    mask = (got[:, 7] >> 16).astype(np.int64)
    # every entry lies in its tile's range
    rg = st["ranges"].astype(np.int64)
    j = np.arange(D)
    assert np.all((rg[tiles, 0] <= j) & (j < rg[tiles, 1])), (name, "ranges")
    J = judge(rec[pl], tiles, gx, hier=hier)
    need, touch = J["needed"], J["touched"]
    miss = need & ~mask
    bad = np.nonzero(miss)[0]
    pop = lambda v: int(np.unpackbits(np.atleast_1d(np.asarray(v, ">u2")).view(np.uint8)).sum())
    deg = degenerate(rec[pl])
    marked, untouched = pop(mask[~deg]), pop((mask & ~touch & ~need)[~deg])
    print(f"\n[{name}] entries {D}  blocks needed {pop(need)}, on regular records marked {marked} untouched {untouched}  "
          f"misses {bad.size} entries / {pop(miss)} blocks  0xFFFF {int((mask == 0xFFFF).sum())} ({int(deg.sum())} degenerate)")
    assert bad.size == 0, (name, [(int(k), int(pl[k]), int(tiles[k]), f"need {need[k]:04x} mask {mask[k]:04x}",
                                   rec[pl[k], :6].tolist()) for k in bad[:5]])
    assert untouched <= tight * max(marked, 1), (name, untouched, marked)
    # the fallback: a full mask on an entry that reaches fewer than half of the tile's blocks
    few = np.unpackbits(np.asarray(touch | need, ">u2").view(np.uint8).reshape(-1, 2), axis=1).sum(1) < 8
    full = (mask == 0xFFFF) & few
    assert not (full & ~deg).any(), (name, "0xFFFF on a regular conic", np.nonzero(full & ~deg)[0][:5].tolist())
    # degenerate records: the fallback whenever the opacity can be taken; a NaN opacity is hidden (0) or falls back
    o = rec[pl, 5]
    assert np.all(mask[deg & (o >= np.float32(ALPHA_SKIP))] == 0xFFFF), (name, "degenerate conic without the fallback")
    assert np.all(np.isin(mask[np.isnan(o)], (0, 0xFFFF))), (name, "NaN opacity")
    return J, tiles


def check_blend(name, sc, st, J, tiles, bg=(0.1, 0.4, 0.9)):
    """n_contrib exactly and the image within blend_ref's budget on every pixel no listed entry is near at"""
    cam = sc.cam
    gx = (cam.W + 15) // 16
    vis = st["radii"] > 0
    rec = st["records"].copy()
    rec[~vis] = 0
    ref = blend_reference(rec, st["ranges"], st["point_list"], cam.W, cam.H, np.asarray(bg, np.float32))
    near = np.zeros((cam.H + 16, cam.W + 16), bool)
    k, p = np.nonzero(J["near"])
    near[16 * (tiles[k] // gx) + p // 16, 16 * (tiles[k] % gx) + p % 16] = True
    keep = ~near[:cam.H, :cam.W] & ~ref["near_pixel"]
    assert keep.any(), name
    bad = (st["n_contrib"].astype(np.int64) != ref["n_contrib"]) & keep
    assert not bad.any(), (name, "n_contrib", int(bad.sum()), np.argwhere(bad)[:5].tolist())
    r, cnt = compare(st["color"], ref["color"], ref["color_tol"][None], keep[None])
    print(f"[{name}] blend: {int(keep.sum())} pixels compared, {int((~keep).sum())} near; max |kernel - f64| / budget {r:.3g}")
    assert r <= 1.0, (name, "color", r)
    return ref


# ---- random scenes --------------------------------------------------------------------------------------------------------
def _cloud(W, H, P, seed, hier=False, op_max=1.0):
    from util import make_scene
    cam, d, ts, kids, _ = make_scene(P, W, H, seed=seed, mode="hier" if hier else "flat")
    sc = Scene(cam)
    rng = np.random.default_rng(seed + 1)
    S = d["scales"].astype(np.float64)
    q = d["rotations"].astype(np.float64)
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    r, x, y, z = q.T
    R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                  2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                  2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    M = R * S[:, None, :]
    Sig = M @ M.transpose(0, 2, 1)
    sc.means = d["means3D"].tolist()
    sc.covs = Sig.reshape(-1, 9)[:, [0, 1, 2, 4, 5, 8]].tolist()
    sc.op = (rng.uniform(0.004, op_max, P)).tolist()
    sc.rgb = rng.uniform(0, 1, (P, 3)).tolist()
    sc.ts = (ts if ts is not None else np.ones(P)).tolist()
    sc.kids = (kids if kids is not None else np.ones(P, np.int64)).tolist()
    return sc


def test_random_1080p():
    sc = _cloud(1920, 1080, 20000, seed=11)
    check_masks("random 1080p", sc, _frame(sc))


@pytest.mark.parametrize("shard", [(2, 0), (2, 1), (3, 2)])
def test_tile_shards(shard):
    """the tile row of a shard's CTA is (blockIdx.x / gx) shard_count + shard_index"""
    sc = _cloud(640, 360, 3000, seed=12)
    st = _frame(sc, shard=shard)
    tiles = (st["keys_sorted"].view(np.uint64) >> np.uint64(32)).astype(np.int64)
    assert np.all((tiles // 40) % shard[0] == shard[1])
    check_masks(f"shard {shard}", sc, st)


def test_hierarchy_opacity_and_kids():
    """abs-activated opacities up to 1.4 in hierarchy mode; num_node_kids up to and beyond the 16-bit field"""
    sc = _cloud(640, 360, 4000, seed=13, hier=True, op_max=1.4)
    rng = np.random.default_rng(14)
    sc.kids = rng.choice([0, 1, 2, 7, 65535, 65536, 70000, 2 ** 20 - 1, 2 ** 20 + 2], len(sc.op)).tolist()
    st = _frame(sc, hier=True)
    kb = st["records"][st["point_list"], 7].view(np.uint32) & 0xFFFFF
    assert (kb > KIDS_MAX).any() and (np.asarray(sc.op) > 1).any()
    check_masks("hierarchy o <= 1.4", sc, st, hier=True)


def test_means_off_the_tile():
    """large Gaussians centred off screen and off their tiles, so the band offsets reach the -8 / 24 clamps"""
    cam = _cam(320, 192)
    sc = Scene(cam)
    rng = np.random.default_rng(15)
    for i in range(300):
        u = rng.choice([-1, 1]) * rng.uniform(0.02, 0.25) * cam.W + (cam.W if i % 2 else 0)
        v = rng.uniform(-0.2, 1.2) * cam.H
        sc.add(u, v, rng.uniform(2, 8), rng.uniform(2, 60), rng.uniform(2, 60), rho=rng.uniform(-0.9, 0.9),
               op=rng.uniform(0.01, 1.0), rng=rng)
    check_masks("off the tile", sc, _frame(sc))


def test_degenerate_records():
    """indefinite conics (screen covariances [[sx^2, rho sx sy], [., sy^2]] with |rho| > 1: K1 lists them, since it only
    rejects det = 0), at opacities on both sides of 1/255, and regular conics with a NaN opacity, among regular rows"""
    cam = _cam(320, 192)
    sc = Scene(cam)
    rng = np.random.default_rng(17)
    kinds = []
    for i in range(240):
        k = i % 4
        u, v, z = rng.uniform(-10, cam.W + 10), rng.uniform(-10, cam.H + 10), rng.uniform(2, 8)
        sx, sy = rng.uniform(1, 20), rng.uniform(1, 20)
        if k == 0:                                   # indefinite, opacity that can be taken
            sc.add(u, v, z, sx, sy, rho=rng.choice([-1, 1]) * rng.uniform(1.5, 4), op=rng.uniform(0.01, 1.0), rng=rng)
        elif k == 1:                                 # indefinite, opacity below fp32(1/255): nothing to take
            sc.add(u, v, z, sx, sy, rho=rng.choice([-1, 1]) * rng.uniform(1.5, 4), op=rng.uniform(0.0, 0.0039), rng=rng)
        elif k == 2:                                 # NaN opacity
            sc.add(u, v, z, sx, sy, rho=rng.uniform(-0.8, 0.8), op=float("nan"), rng=rng)
        else:
            sc.add(u, v, z, sx, sy, rho=rng.uniform(-0.8, 0.8), op=rng.uniform(0.01, 1.0), rng=rng)
        kinds.append(k)
    st = _frame(sc)
    kinds = np.asarray(kinds)
    listed = np.zeros(len(kinds), bool)
    listed[st["point_list"]] = True
    rec = st["records"]
    assert (listed & (kinds == 0)).sum() > 20 and (listed & (kinds == 1)).any() and (listed & (kinds == 2)).sum() > 20
    assert degenerate(rec[listed & (kinds == 0)]).all() and not degenerate(rec[listed & (kinds == 3)]).any()
    check_masks("degenerate", sc, st)


# ---- needles --------------------------------------------------------------------------------------------------------------
def _edge_on(cam, u, v, z, sigma_px, theta, thin=1e-4):
    """3D covariance of a flat Gaussian (scales s, s, thin s) at pixel (u, v), depth z, seen edge-on: its plane holds the
    view ray and the image direction theta, so it projects to a needle sigma_px long at the dilation floor across"""
    p = np.array(_place(cam, u, v, z), np.float64)
    ray = p / np.linalg.norm(p)
    a = np.array([np.cos(theta), np.sin(theta), 0.0])
    a_perp = a - (a @ ray) * ray                  # J a_perp = J a: the projection drops the ray component
    f = cam.W / (2 * cam.tanfovx)
    s = sigma_px * z / f
    nrm = np.cross(ray, a_perp / np.linalg.norm(a_perp))
    Sig = s * s * (np.outer(a_perp, a_perp) + np.outer(ray, ray)) + (thin * s) ** 2 * np.outer(nrm, nrm)
    return Sig[[0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].tolist()


def test_needles():
    """Gaussians seen edge-on at all angles, sigma_long 50 .. 600 px: conics with condition numbers up to ~1e6; every
    tile of their rects is listed and judged"""
    cam = _cam(1920, 1080)
    sc = Scene(cam)
    rng = np.random.default_rng(16)
    for i in range(48):
        u, v, z = rng.uniform(200, 1720), rng.uniform(150, 930), rng.uniform(3, 9)
        sc.add(u, v, z, 1.0, 1.0, op=rng.uniform(0.05, 0.9), rng=rng)
        sc.covs[-1] = _edge_on(cam, u, v, z, 50 * 12 ** rng.uniform(), rng.uniform(0, np.pi))
    st = _frame(sc)
    rec = st["records"][st["radii"] > 0].astype(np.float64)
    det = rec[:, 2] * rec[:, 4] - rec[:, 3] ** 2
    assert (rec[:, 2] * rec[:, 4] / det).max() > 1e5
    J, tiles = check_masks("needles", sc, st)
    check_blend("needles", sc, st, J, tiles)


# ---- opacity at 1/255 --------------------------------------------------------------------------------------------------------
O255 = np.float32(1.0 / 255.0)
OPS = [np.nextafter(O255, np.float32(0)), O255, np.nextafter(O255, np.float32(1))]


@pytest.mark.parametrize("W,H", [(161, 97), (167, 107), (161, 107)])
def test_opacity_at_one_over_255(W, H):
    """means exactly on a pixel centre (on the optical axis of an odd-sized image: (W - 1) / 2 in fp32 exactly) -- a
    tile corner (80, 48) at 161 x 97, inside a tile (83, 53) at 167 x 107, on a tile's left edge (80, 53) at 161 x 107 --
    and a fraction of a pixel off it,
    at opacities prev / fp32 / next of 1/255.  At the centre G = ex2(0) = 1 exactly, so the blend takes fp32(1/255)."""
    cam = _cam(W, H)
    sc = Scene(cam)
    rng = np.random.default_rng(W)
    u0, v0 = (W - 1) / 2, (H - 1) / 2
    for i in range(60):
        off = 0.0 if i < 30 else rng.choice([-1, 1]) * 10.0 ** rng.uniform(-6, -3)
        s = rng.uniform(0.3, 6)
        sc.add(u0 + off, v0 - off * rng.uniform(), 2.0 + 0.05 * i, s, s * rng.uniform(0.3, 1), rho=rng.uniform(-0.5, 0.5),
               op=float(OPS[i % 3]), rng=rng)
    st = _frame(sc)
    rec = st["records"]
    on = (rec[:, 0] == np.float32(u0)) & (rec[:, 1] == np.float32(v0)) & (rec[:, 5] == O255)
    assert on.sum() >= 8, int(on.sum())
    J, tiles = check_masks(f"1/255 {W}x{H}", sc, st)
    ref = check_blend(f"1/255 {W}x{H}", sc, st, J, tiles)
    # the centre pixel takes every fp32(1/255) entry centred on it (a decision the judge leaves out as near)
    cx, cy = int(u0), int(v0)
    assert st["n_contrib"][cy, cx] == ref["n_contrib"][cy, cx] > 0


# ---- the tile sort's size classes and the radix hand-over -------------------------------------------------------------------
def test_sort_classes_and_radix():
    """tiles of every size class of the tile sort (<= 128, 256, 512, 1024, the shared-memory network) in one frame, and a
    tile past its capacity in another, which is binned by the radix sort and gathered by gather_records_kernel"""
    from test_gpu_blend_deep import Deep, _fill_tile
    for name, W, H, tiles in (("sort classes", 160, 64, (((0, 0), 100), ((1, 0), 200), ((2, 0), 400), ((3, 0), 900),
                                                          ((4, 1), 3000), ((5, 2), 1))),
                              ("radix", 48, 32, (((1, 0), 8200), ((0, 1), 300), ((2, 1), 1), ((0, 0), 129)))):
        d = Deep(W, H, False, seed=51)
        rng = np.random.default_rng(52)
        for (tx, ty), n in tiles:
            _fill_tile(d, tx, ty, n, 2.0 + 0.05 * np.arange(30), rng)
        # a few larger Gaussians across tiles, whose masks are not a single block
        for i in range(20):
            d.sc.add(rng.uniform(0, W), rng.uniform(0, H), 1.5, rng.uniform(1, 8), rng.uniform(1, 8), rho=0.3, op=0.5, rng=rng)
        st = _frame(d.sc)
        lens = st["ranges"][:, 1].astype(np.int64) - st["ranges"][:, 0]
        assert (lens.max() > 8192) == (name == "radix")
        check_masks(name, d.sc, st)

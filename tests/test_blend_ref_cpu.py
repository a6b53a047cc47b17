"""CPU: the float64 blend reference of the blend-kernel tests (tests/blend_ref.py) against torch_splat's dense blend
(oracle/torch_splat.py::blend2d, differentiated by autograd) on the same 2D Gaussians.  Both get identical inputs --
fp32 values held in float64 -- so they agree to float64 rounding everywhere except at pixels with a pair on a decision
threshold, which blend_ref reports and the comparison leaves out."""
import numpy as np
import pytest
import torch

import blend_ref
from blend_ref import blend_reference, TILE
from oracle import torch_splat


def _scene(P, W, H, seed, hier):
    g = np.random.default_rng(seed)
    f32 = lambda a: np.asarray(a, np.float32)
    px = f32(g.uniform(-6, W + 6, P)); py = f32(g.uniform(-6, H + 6, P))
    sx, sy = g.uniform(0.6, 7, P), g.uniform(0.6, 7, P)
    big = g.uniform(size=P) < 0.1
    sx[big] *= 5; sy[big] *= 5
    rho = g.uniform(-0.85, 0.85, P)
    a = sx * sx + 0.3; c = sy * sy + 0.3; b = rho * sx * sy
    det = a * c - b * b
    conic = f32(np.stack([c / det, -b / det, a / det], 1))
    op = f32(np.where(g.uniform(size=P) < 0.2, g.uniform(0.9, 1.4, P), g.uniform(0.02, 0.9, P)))
    rgb = f32(g.uniform(0, 1, (P, 3)))
    invd = f32(g.uniform(0.05, 0.5, P))
    invd[:10] = invd[10]                                   # equal depths: ties keep index order
    ts = f32(np.where(g.uniform(size=P) < 0.3, 1.0, g.uniform(0, 1, P)))
    ts[:5] = 0.0
    kids = g.choice(np.array([-1, 1, 2, 2, 3, 4, 7, 16, 17, 255, 4097, 65535], np.int32), P)
    if not hier:
        ts = kids = None
    mid = 0.5 * (a + c)
    lam = mid + np.sqrt(np.maximum(mid * mid - det, 0.1))
    rad = np.ceil(3 * np.sqrt(lam))
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    rminx = np.clip(np.trunc((px - rad) / TILE), 0, gx); rmaxx = np.clip(np.trunc((px + rad + TILE - 1) / TILE), 0, gx)
    rminy = np.clip(np.trunc((py - rad) / TILE), 0, gy); rmaxy = np.clip(np.trunc((py + rad + TILE - 1) / TILE), 0, gy)
    visible = (rmaxx - rminx) * (rmaxy - rminy) > 0
    return dict(px=px, py=py, conic=conic, op=op, rgb=rgb, invd=invd, ts=ts, kids=kids, visible=visible,
                rect=(rminx, rmaxx, rminy, rmaxy))


def _projected_scene(P, W, H, seed, hier):
    """2D Gaussians from torch_splat's float64 projection of a synthetic 3D cloud, rounded to fp32 as K1 stores them"""
    from util import make_scene
    cam, sc, ts, kids, bg = make_scene(P, W, H, mode="hier" if hier else "flat", seed=seed, zmin=1.5, zmax=6.0,
                                       scale_k=3e-2)
    sc["opacities"] = sc["opacities"] * np.float32(1.6)          # some above 1 and pixels that terminate
    D = lambda a: torch.tensor(np.asarray(a, np.float64))
    pr = torch_splat.project(D(sc["means3D"]), D(sc["shs"]), None, D(sc["opacities"]), D(sc["scales"]),
                             D(sc["rotations"]), None, D(cam.world_view_transform), D(cam.full_proj_transform),
                             D(cam.camera_center), W, H, cam.tanfovx, cam.tanfovy, 3, 1.0)
    f32 = lambda a: np.asarray(a.detach().numpy(), np.float32)
    px, py, rad = f32(pr["px"]), f32(pr["py"]), pr["radii"].numpy().astype(np.float64)
    visible = pr["visible"].numpy()
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    rminx = np.clip(np.trunc((px - rad) / TILE), 0, gx); rmaxx = np.clip(np.trunc((px + rad + TILE - 1) / TILE), 0, gx)
    rminy = np.clip(np.trunc((py - rad) / TILE), 0, gy); rmaxy = np.clip(np.trunc((py + rad + TILE - 1) / TILE), 0, gy)
    visible &= (rmaxx - rminx) * (rmaxy - rminy) > 0
    invd = f32(1.0 / pr["depth"])
    invd[~visible] = 1.0
    return dict(px=px, py=py, conic=f32(pr["conic"]), op=f32(pr["opacities"]), rgb=f32(pr["rgb"]), invd=invd,
                ts=ts, kids=kids, visible=visible, rect=(rminx, rmaxx, rminy, rmaxy))


def _tile_lists(s, W, H):
    """ranges / point_list as the binning stage lays them out: tile-major, depth (view z) ascending, ties by index."""
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    rminx, rmaxx, rminy, rmaxy = s["rect"]
    depth = (1.0 / s["invd"].astype(np.float64)).astype(np.float32)
    order = np.argsort(depth, kind="stable")
    ranges, pl = np.zeros((gx * gy, 2), np.int64), []
    for tile in range(gx * gy):
        tx, ty = tile % gx, tile // gx
        ins = [i for i in order if s["visible"][i] and rminx[i] <= tx < rmaxx[i] and rminy[i] <= ty < rmaxy[i]]
        ranges[tile] = (len(pl), len(pl) + len(ins))
        pl += ins
    return ranges, np.array(pl, np.int64), depth


@pytest.mark.parametrize("source", ["2d", "projected"])
@pytest.mark.parametrize("hier,do_depth,W,H,seed", [(False, False, 40, 30, 1), (False, True, 37, 19, 2), (True, False, 40, 30, 3),
                                                    (True, True, 45, 33, 4)])
def test_blend_reference_matches_torch_splat(hier, do_depth, W, H, seed, source, monkeypatch):
    """source "2d": 2D Gaussians drawn directly (opacities above 1, needles, every kids value of the GPU tests);
    "projected": the 2D records of a 3D cloud through torch_splat's own float64 projection."""
    # torch_splat states the thresholds in float64, the kernels (and so blend_ref) as fp32 constants; and both sides
    # compute in float64 here, so the decision margins shrink from the fp32 + MUFU budget to float64 rounding
    for name, v in (("ALPHA_CAP", 0.99), ("ALPHA_SKIP", 1.0 / 255.0), ("T_STOP", 1e-4), ("U", 2.0 ** -53),
                    ("EPS_EX2", 0.0), ("EPS_HIER", 0.0), ("MARGIN", 1e-12)):
        monkeypatch.setattr(blend_ref, name, v)
    P = 160
    s = _scene(P, W, H, seed, hier) if source == "2d" else _projected_scene(P, W, H, seed, hier)
    ranges, pl, depth = _tile_lists(s, W, H)
    rec = np.zeros((P, 12), np.float32)
    rec[:, 0], rec[:, 1], rec[:, 2:5], rec[:, 5] = s["px"], s["py"], s["conic"], s["op"]
    rec[:, 6] = s["ts"] if hier else 1.0
    rec[:, 7] = (np.maximum(s["kids"], 1) if hier else np.ones(P, np.int32)).astype(np.uint32).view(np.float32)
    rec[:, 8:11], rec[:, 11] = s["rgb"], s["invd"]
    bg = np.array([0.2, 0.5, 0.7], np.float32)
    g = np.random.default_rng(seed + 100)
    gcol = g.standard_normal((3, H, W)); gdep = g.standard_normal((H, W))
    ref = blend_reference(rec, ranges, pl, W, H, bg, gcol, gdep if do_depth else None, hier=hier, do_depth=do_depth)

    t = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)
    px, py, conic, op, rgb = t(s["px"]), t(s["py"]), t(s["conic"]), t(s["op"]), t(s["rgb"])
    dep = t(1.0 / s["invd"].astype(np.float64))
    rect = tuple(torch.tensor(r) for r in s["rect"])
    ts = torch.tensor(s["ts"], dtype=torch.float64) if hier else None
    kids = torch.tensor(s["kids"], dtype=torch.float64) if hier else None
    color, invd = torch_splat.blend2d(
        px, py, conic, op, rgb, dep, torch.tensor(s["visible"]), rect, torch.tensor(bg, dtype=torch.float64), W, H,
        ts, kids, do_depth)
    loss = (color * torch.tensor(gcol)).sum() + ((invd[0] * torch.tensor(gdep)).sum() if do_depth else 0)
    loss.backward()

    keep = ~ref["near_pixel"]
    assert keep.mean() > 0.999, ref["near_kind"]
    assert (ref["n_contrib"] > 0).mean() > 0.5 and (ref["final_T"] < 1e-2).any()      # the scene blends and terminates
    scale = np.abs(ref["color"]).max()
    assert np.abs(color.detach().numpy() - ref["color"])[:, keep].max() <= 1e-10 * scale
    if do_depth:
        assert np.abs(invd.detach().numpy()[0] - ref["invdepth"])[keep].max() <= 1e-10 * np.abs(ref["invdepth"]).max()
    rows = ~ref["near_gauss"] & s["visible"]
    assert ref["near_gauss"][s["visible"]].mean() < 0.02, ref["near_kind"]
    A = ref["accum"]
    # d loss / d(2D record) in terms of the accumulator columns (their constant factors are the preprocess backward's)
    pairs = [(px.grad, A[:, 0]), (py.grad, A[:, 1]), (conic.grad[:, 0], -0.5 * A[:, 2]), (conic.grad[:, 1], -A[:, 3]),
             (conic.grad[:, 2], -0.5 * A[:, 4]), (op.grad, A[:, 5])] + [(rgb.grad[:, c], A[:, 6 + c]) for c in range(3)]
    if do_depth:
        pairs.append((dep.grad * -(dep.detach() ** 2), A[:, 9]))      # d/d(1/z) = -z^2 d/dz
    else:
        assert np.all(A[:, 9] == 0)
    absA = ref["accum_abs"]
    cols = [0, 1, 2, 3, 4, 5, 6, 7, 8] + ([9] if do_depth else [])
    for (gt, a), c in zip(pairs, cols):
        d = np.abs(gt.numpy() - a)[rows]
        assert (d <= 1e-9 * absA[rows, c] + 1e-300).all(), (c, float((d / (absA[rows, c] + 1e-300)).max()))
    # the abs-sum scale bounds the sum, and every visible Gaussian that is taken somewhere has a non-zero scale
    assert (np.abs(A) <= absA * (1 + 1e-12) + 1e-300).all()

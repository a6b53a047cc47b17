"""CPU: the library's own kernels -- the .cu sources compiled with g++ against a small SIMT emulator
(tests/emul/: fibers for the threads of a block, rendezvous for barriers and warp collectives, memcpy for
the TMA staging) -- driven through the same C-ABI calls as on the GPU and compared with the oracle on
small scenes.  This is how kernel changes are checked before any GPU time is spent; it is test
infrastructure: the product library is built by nvcc only and has no CPU path."""
import os
import sys

import numpy as np
import pytest

from h3dgs import synth
from util import make_scene, oracle_run, rel_err

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emul"))


def image_close(a, b, what="color", max_flips=6):
    """assert_image_close for the small emulated frames: an alpha within fp32 rounding of the 1/255 skip
    threshold may flip a contribution in or out (the emulator rounds like neither the GPU's contracted
    FMAs nor the oracle); a handful of such pixels, each bounded by one contribution, is not a defect."""
    d = np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64))
    scale = max(np.abs(b).max(), 1e-30)
    bad = d > 1e-5 * scale
    assert bad.sum() <= max_flips, (what, int(bad.sum()), float(d.max()))
    assert d.max() < 1.5 / 255 * max(scale, 1.0), (what, float(d.max()))


def grad_close(a, b, name, tol=1e-5, max_rows=12):
    """assert_grad_close with the same allowance: the few rows a flipped pixel feeds (a cut row and its
    parent in scatter mode) may move by one pixel's worth of a 1/255 contribution."""
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    scale = max(np.abs(b).max(), 1e-30)
    d = np.abs(a - b).reshape(a.shape[0], -1).max(1)
    bad = d > tol * scale
    assert bad.sum() <= max_rows, (name, int(bad.sum()), float(d.max() / scale))
    assert d.max() < 5e-3 * scale, (name, float(d.max() / scale))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    from build_emu import build
    from emu_api import Emu
    return Emu(build(str(tmp_path_factory.mktemp("h3dgs_emu"))))


def _check(emu, cam, sc, bg, ts=None, kids=None, do_depth=False, sh_degree=3, colors=None, cov=None, tol=1e-5):
    f, b, gcol, gdep = oracle_run(cam, sc, bg, ts, kids, do_depth=do_depth, sh_degree=sh_degree, colors=colors, cov=cov)
    a, keep = emu.args(cam, bg, sc, sh_degree=sh_degree, ts=ts, kids=kids, do_depth=do_depth, colors=colors, cov=cov)
    fw = emu.forward(a, keep)
    st = emu.state(a, fw)
    assert fw["D"] == f["num_rendered"]
    assert np.array_equal(fw["radii"], f["radii"])
    if fw["D"]:
        assert np.array_equal(st["point_list"], f["point_list"])
        assert np.array_equal(st["keys_sorted"], f["keys"])
    assert np.array_equal(st["ranges"], f["ranges"].reshape(-1, 2))
    image_close(fw["color"], f["color"])
    image_close(st["final_T"], f["final_T"].reshape(-1), "final_T")
    assert (st["n_contrib"] != f["n_contrib"].reshape(-1)).mean() < 2e-3
    if do_depth:
        image_close(fw["invdepth"], f["invdepth"], "invdepth")
    g = emu.backward(a, fw, gcol, gdep if do_depth else None)
    for k in ("means3D", "means2D", "sh", "colors_precomp", "opacities", "scales", "rotations", "cov3Ds_precomp"):
        if g.get(k) is not None and b.get(k) is not None:
            grad_close(g[k], b[k], k, tol=tol)
    return f, fw, st, g


@pytest.mark.parametrize("mode,do_depth", [("flat", False), ("flat", True), ("hier", False), ("hier", True)])
def test_forward_backward_parity(emu, mode, do_depth):
    cam, sc, ts, kids, bg = make_scene(3000, 256, 192, mode=mode, seed=42)
    _check(emu, cam, sc, bg, ts, kids, do_depth=do_depth)


@pytest.mark.parametrize("deg,K", [(0, 1), (1, 4), (2, 9), (1, 16)])
def test_sh_degrees_and_layouts(emu, deg, K):
    cam, sc, ts, kids, bg = make_scene(1500, 160, 96, sh_degree=int(np.sqrt(K)) - 1, seed=7)
    _check(emu, cam, sc, bg, sh_degree=deg)


def test_precomputed_colour_and_covariance(emu):
    from oracle import oracle
    cam, sc, ts, kids, bg = make_scene(1500, 160, 96, seed=9)
    colors = np.random.default_rng(1).uniform(0, 1, (1500, 3)).astype(np.float32)
    f0 = oracle_run(cam, sc, bg, backward=False)[0]
    _check(emu, cam, sc, bg, colors=colors, cov=f0["cov3Ds"])


@pytest.mark.parametrize("W,H", [(8, 8), (15, 33), (100, 50)])
def test_odd_image_sizes(emu, W, H):
    cam, sc, ts, kids, bg = make_scene(300, W, H, seed=3, scale_k=2e-2)
    _check(emu, cam, sc, bg)


def test_deep_tiles_and_early_termination(emu):
    cam, sc, ts, kids, bg = make_scene(6000, 96, 64, seed=11, scale_k=3e-2, zmax=6.0)
    sc["opacities"] = np.clip(sc["opacities"] * 1.5, 0, 0.99).astype(np.float32)
    f, fw, st, g = _check(emu, cam, sc, bg)
    lens = st["ranges"][:, 1] - st["ranges"][:, 0]
    assert lens.max() > 600                                   # several TMA batches per tile
    assert (f["final_T"] < 1e-3).mean() > 0.2                 # early termination is exercised


def test_tile_shards_equal_the_whole_frame(emu):
    cam, sc, ts, kids, bg = make_scene(2500, 160, 112, mode="hier", seed=5)
    f, b, gcol, gdep = oracle_run(cam, sc, bg, ts, kids)
    a, keep = emu.args(cam, bg, sc, ts=ts, kids=kids)
    full = emu.forward(a, keep)
    gy = (cam.H + 15) // 16
    img = np.zeros_like(full["color"])
    acc = None
    for r in range(3):
        a_s, keep_s = emu.args(cam, bg, sc, ts=ts, kids=kids, shard=(3, r))
        fw = emu.forward(a_s, keep_s)
        rows = (gy + 3 - 1 - r) // 3
        packed = fw["color"].reshape(-1)[: rows * 3 * 16 * cam.W].reshape(rows, 3, 16, cam.W)
        for k in range(rows):
            y0 = (k * 3 + r) * 16
            h = min(16, cam.H - y0)
            img[:, y0:y0 + h] = packed[k, :, :h]
        g = emu.backward(a_s, fw, gcol)
        acc = {k: v.copy() for k, v in g.items() if v is not None} if acc is None else \
            {k: acc[k] + g[k] for k in acc}
    assert np.array_equal(img, full["color"])                  # same per-tile arithmetic
    for k in ("means3D", "sh", "opacities", "scales", "rotations"):
        grad_close(acc[k], b[k], k)


def test_sharded_frame_with_row_blocks(emu):
    """the multi-GPU schedule on one CPU: every shard renders its tile rows (the forward knows its gradient
    row block and skips foreign SH colours), phase 1 fills each shard's [P][10] sums, their total is what the
    reduce-scatter delivers, phase 2 finishes each shard's own row block."""
    cam, sc, ts, kids, bg = make_scene(2500, 160, 112, mode="hier", seed=8)
    f, b, gcol, gdep = oracle_run(cam, sc, bg, ts, kids)
    P, G = 2500, 3
    chunk = (P + G - 1) // G
    rows = [(min(r * chunk, P), min((r + 1) * chunk, P)) for r in range(G)]
    shards = []
    for r in range(G):
        a, keep = emu.args(cam, bg, sc, ts=ts, kids=kids, shard=(G, r), grad_rows=rows[r])
        fw = emu.forward(a, keep)
        g1 = emu.backward(a, fw, gcol, phases=1)
        shards.append((a, keep, fw, g1["scratch"].view(np.float32)[: P * 10].copy()))
    total = sum(s[3].astype(np.float64) for s in shards).astype(np.float32)
    out = {k: np.zeros_like(b[k]) for k in ("means3D", "sh", "opacities", "scales", "rotations", "means2D")}
    for r, (a, keep, fw, _) in enumerate(shards):
        from emu_api import aligned
        scratch = aligned(emu.L.h3dgs_backward_scratch_bytes(P))
        scratch.view(np.float32)[: P * 10] = total
        g2 = emu.backward(a, fw, gcol, phases=2, scratch=scratch)
        lo, hi = rows[r]
        for k in out:
            out[k][lo:hi] = g2[k][lo:hi]
    for k in out:
        grad_close(out[k], b[k], k)


def test_fused_cut_gather_and_scatter(emu):
    from oracle import oracle
    cam = synth.make_camera(160, 112)
    leaves = synth.cloud_v1(1500, cam, zmin=2.0, zmax=30.0, seed=2, scale_k=1.0)
    z = leaves["means3D"][:, 2:3]
    leaves["scales"] = (8e-3 * np.sqrt(2 * z) * np.ones((1, 3))).astype(np.float32)
    h = synth.build_hierarchy(leaves)
    thr = synth.tau_threshold(6.0, cam)
    n, ri, pi, ni = oracle.expand_to_size(h["nodes"], h["boxes"], thr, cam.camera_center)
    ts, kids = oracle.get_interpolation_weights(ni, thr, h["nodes"], h["boxes"], cam.camera_center)
    assert (ts < 1).mean() > 0.05
    bg = np.array([0.3, 0.2, 0.1], np.float32)
    f = oracle.rasterize_forward(h["means3D"], h["shs"], None, h["opacities"], h["scales"], h["rotations"], None,
                                 cam.world_view_transform, cam.full_proj_transform, cam.camera_center, bg, cam.W, cam.H,
                                 cam.tanfovx, cam.tanfovy, ts=ts, kids=kids, render_indices=ri, parent_indices=pi)
    gcol = synth.l1_grad(f["color"])
    b = oracle.rasterize_backward(f, gcol)
    a, keep = emu.args(cam, bg, h, ts=ts, kids=kids, ridx=ri, pidx=pi)
    fw = emu.forward(a, keep)
    assert np.array_equal(fw["radii"], f["radii"])
    image_close(fw["color"], f["color"])
    g = emu.backward(a, fw, gcol)
    for k in ("means3D", "sh", "opacities", "scales", "rotations", "means2D"):
        grad_close(g[k], b[k], k)


def test_device_lod_cut_and_skipped_rows(emu):
    """h3dgs_lod_cut = expand_to_size + get_interpolation_weights; rows after the cut are marked -1 and
    the rasterizer handed P = capacity skips them (the sync-free step)."""
    import ctypes as C
    from emu_api import aligned, f32, i32, ptr
    from oracle import oracle
    cam = synth.make_camera(160, 112)
    leaves = synth.cloud_v1(1200, cam, zmin=2.0, zmax=30.0, seed=4, scale_k=1.0)
    z = leaves["means3D"][:, 2:3]
    leaves["scales"] = (8e-3 * np.sqrt(2 * z) * np.ones((1, 3))).astype(np.float32)
    h = synth.build_hierarchy(leaves)
    N = h["nodes"].shape[0]
    thr = synth.tau_threshold(6.0, cam)
    n, ri, pi, ni = oracle.expand_to_size(h["nodes"], h["boxes"], thr, cam.camera_center)
    ts, kids = oracle.get_interpolation_weights(ni, thr, h["nodes"], h["boxes"], cam.camera_center)
    L = emu.L
    nodes, boxes, vp, thr_dev = i32(h["nodes"]), f32(h["boxes"]), f32(cam.camera_center), f32([thr])
    r2, p2, n2, k2 = (aligned(N * 4, np.int32, (N,)) for _ in range(4))
    t2 = aligned(N * 4, np.float32, (N,))
    count = aligned(4, np.int32, (1,))
    scratch = aligned(L.h3dgs_expand_scratch_bytes(N))
    emu.check(L.h3dgs_lod_cut(N, ptr(nodes), ptr(boxes), -1.0, ptr(thr_dev), ptr(vp), ptr(r2), ptr(p2), ptr(n2), ptr(t2),
                              ptr(k2), ptr(count), ptr(scratch), None))
    assert int(count[0]) == n
    assert np.array_equal(r2[:n], ri) and np.array_equal(p2[:n], pi) and np.array_equal(n2[:n], ni)
    assert np.array_equal(t2[:n].view(np.uint32), ts.view(np.uint32)) and np.array_equal(k2[:n], kids)
    assert (r2[n:] == -1).all()
    # the two-call API on the same library gives the same
    r3, p3, n3 = (aligned(N * 4, np.int32, (N,)) for _ in range(3))
    got = L.h3dgs_expand_to_size(N, ptr(nodes), ptr(boxes), thr, ptr(vp), 0.0, 0.0, 0.0, ptr(r3), ptr(p3), ptr(n3), ptr(scratch), None)
    assert got == n and np.array_equal(r3[:n], ri)
    # capacity-sized rasterization over the marked index array == exact rasterization of the cut
    bg = np.array([0.1, 0.2, 0.3], np.float32)
    a0, keep0 = emu.args(cam, bg, h, ts=ts, kids=kids, ridx=ri, pidx=pi)
    exact = emu.forward(a0, keep0)
    a1, keep1 = emu.args(cam, bg, h, ts=t2, kids=k2, ridx=r2, pidx=p2, P=N, bin_capacity=exact["D"] + 10, sort_capacity=4096)
    cap = emu.forward(a1, keep1)
    st = emu.state(a1, cap)
    assert list(st["scan_info"]) == [exact["D"], st["scan_info"][1], 0]
    assert np.array_equal(cap["color"], exact["color"])
    assert np.array_equal(cap["radii"][:n], exact["radii"]) and (cap["radii"][n:] == 0).all()
    gcol = synth.l1_grad(exact["color"])
    g0, g1 = emu.backward(a0, exact, gcol), emu.backward(a1, cap, gcol)
    for k in ("means3D", "sh", "opacities", "scales", "rotations"):
        assert rel_err(g1[k], g0[k]) < 1e-6, k
    # a frame that does not fit: flagged, background only, zero gradients
    for kw in (dict(bin_capacity=exact["D"] // 2, sort_capacity=4096), dict(bin_capacity=exact["D"] + 10, sort_capacity=32)):
        a2, keep2 = emu.args(cam, bg, h, ts=t2, kids=k2, ridx=r2, pidx=p2, P=N, **kw)
        ov = emu.forward(a2, keep2)
        s2 = emu.state(a2, ov)
        assert s2["scan_info"][2] == 1 and s2["scan_info"][0] == exact["D"]
        assert np.array_equal(ov["color"], np.broadcast_to(bg.reshape(3, 1, 1), ov["color"].shape))
        g2 = emu.backward(a2, ov, gcol)
        assert all(float(np.abs(v).sum()) == 0.0 for k, v in g2.items() if v is not None and k != "means2D")


def test_equal_depths_and_long_lists_fall_back_to_the_global_sort(emu):
    cam, sc, ts, kids, bg = make_scene(16000, 48, 48, seed=13, scale_k=6e-2, zmax=4.0)
    sc["means3D"][:, 2] = np.round(sc["means3D"][:, 2] * 4) / 4       # many equal depths: order must follow the index
    f, fw, st, g = _check(emu, cam, sc, bg, tol=5e-5)
    assert (st["ranges"][:, 1] - st["ranges"][:, 0]).max() > 8192    # longer than the shared-memory sort handles


def test_register_sort_size_classes_with_equal_depths(emu):
    """tile lists of 33 .. ~700 entries: every size class of the in-register sort (1, 2, 4, 8 keys per thread), with
    many equal depths, so the (depth bits, index) order -- the stable order of the reference's global sort -- is
    checked through the lane exchanges, the in-thread stages and the cross-warp stages alike"""
    n = 14000
    cam, sc, ts, kids, bg = make_scene(n, 160, 128, seed=17, scale_k=1.5e-2, zmax=8.0)
    x = sc["means3D"][:, 0] / sc["means3D"][:, 2]
    ramp = (x - x.min()) / (x.max() - x.min())
    keep = np.random.default_rng(1).uniform(size=n) < 0.03 + 0.97 * ramp ** 2       # dense right, sparse left
    sc = {k: v[keep] for k, v in sc.items()}
    sc["means3D"][:, 2] = np.round(sc["means3D"][:, 2] * 4) / 4
    f = oracle_run(cam, sc, bg, backward=False)[0]
    lens = f["ranges"].reshape(-1, 2)[:, 1] - f["ranges"].reshape(-1, 2)[:, 0]
    assert all(((lens > lo) & (lens <= hi)).any() for lo, hi in [(0, 128), (128, 256), (256, 512), (512, 1024)])
    a, keepalive = emu.args(cam, bg, sc)
    fw = emu.forward(a, keepalive)
    st = emu.state(a, fw)
    assert fw["D"] == f["num_rendered"]
    assert np.array_equal(st["keys_sorted"], f["keys"])
    assert np.array_equal(st["point_list"], f["point_list"])
    image_close(fw["color"], f["color"])


def test_random_scenes_functional(emu):
    """a small fuzz over sizes, modes, depth, opacities above one and needle-shaped Gaussians.  The bar here is
    functional (no lost or doubled contributions, no crash, no deadlock): on ill-conditioned scenes the fp32
    oracle itself is 3e-5 away from a double-precision blend, so the 1e-5 parity bar does not apply."""
    rng = np.random.default_rng(20)
    for it in range(10):
        P = int(rng.choice([1, 7, 64, 500, 2000]))
        W, H = int(rng.integers(1, 160)), int(rng.integers(1, 120))
        mode = str(rng.choice(["flat", "hier"]))
        cam, sc, ts, kids, bg = make_scene(P, W, H, mode=mode, seed=int(rng.integers(0, 10**6)),
                                           scale_k=float(10 ** rng.uniform(-3, -1.2)), zmax=float(rng.uniform(4, 40)))
        if rng.uniform() < 0.3:
            sc["opacities"] = (sc["opacities"] * rng.uniform(0.5, 3.0)).astype(np.float32)
        if rng.uniform() < 0.3:
            sc["scales"] = (sc["scales"] * np.array([1.0, 8.0, 0.2], np.float32)).astype(np.float32)
        f, b, gcol, gdep = oracle_run(cam, sc, bg, ts, kids, do_depth=True)
        a, keep = emu.args(cam, bg, sc, ts=ts, kids=kids, do_depth=True)
        fw = emu.forward(a, keep)
        assert fw["D"] == f["num_rendered"] and np.array_equal(fw["radii"], f["radii"])
        scale = max(np.abs(f["color"]).max(), 1.0)
        d = np.abs(fw["color"] - f["color"])
        assert (d > 1e-4 * scale).sum() <= 6 and d.max() < 1.5 / 255 * scale, (it, float(d.max()))
        g = emu.backward(a, fw, gcol, gdep)
        for k in ("means3D", "sh", "opacities", "scales", "rotations"):
            grad_close(g[k], b[k], k, tol=2e-4)


@pytest.mark.parametrize("W,shard", [(64, (1, 0)), (50, (1, 0)), (64, (3, 1))])
def test_fused_l1_loss_and_gradient(emu, W, shard):
    """csrc/l1_loss.cu under emulation: loss sum and sign gradient vs numpy, float4 and scalar streams, tile-row shard."""
    import ctypes as C
    H = 40
    g = np.random.default_rng(0)
    img = g.uniform(0, 1, (3, H, W)).astype(np.float32); gt = g.uniform(0, 1, (3, H, W)).astype(np.float32)
    gt[0, 3, 5] = img[0, 3, 5]                                  # sign(0) = 0
    out = np.full((3, H, W), 7.0, np.float32); s = np.zeros(1, np.float64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = emu.L.h3dgs_l1_loss_grad(3, H, W, p(img), p(gt), C.c_float(0.25), shard[0], shard[1], p(out), p(s), None)
    assert rc == 0
    rows = np.arange(H)
    own = ((rows // 16) % shard[0]) == shard[1]
    d = (img - gt)[:, own]
    assert abs(s[0] - np.abs(d.astype(np.float64)).sum()) < 1e-3
    assert np.array_equal(out[:, own], np.sign(d) * np.float32(0.25))
    assert np.all(out[:, ~own] == 7.0)


def test_split_phases_fill_the_scatter_outputs_beside_the_replay(emu):
    """scatter mode, backward in two calls: phases 1|4 (replay + zero-fill of the full-size gradients) then 2|8 (chain rule,
    outputs already zero) gives what the single call (3) gives; the outputs are poisoned first, so a missing fill shows."""
    from oracle import oracle
    cam = synth.make_camera(128, 96)
    leaves = synth.cloud_v1(900, cam, zmin=2.0, zmax=30.0, seed=4, scale_k=1.0)
    z = leaves["means3D"][:, 2:3]
    leaves["scales"] = (8e-3 * np.sqrt(2 * z) * np.ones((1, 3))).astype(np.float32)
    h = synth.build_hierarchy(leaves)
    thr = synth.tau_threshold(6.0, cam)
    n, ri, pi, ni = oracle.expand_to_size(h["nodes"], h["boxes"], thr, cam.camera_center)
    ts, kids = oracle.get_interpolation_weights(ni, thr, h["nodes"], h["boxes"], cam.camera_center)
    bg = np.array([0.3, 0.2, 0.1], np.float32)
    a, keep = emu.args(cam, bg, h, ts=ts, kids=kids, ridx=ri, pidx=pi)
    fw = emu.forward(a, keep)
    gcol = synth.l1_grad(fw["color"])
    whole = emu.backward(a, fw, gcol)
    first = emu.backward(a, fw, gcol, phases=1 | 4)
    assert all(not np.asarray(first[k]).any() for k in ("means3D", "sh", "opacities", "scales", "rotations"))
    for k in ("means3D", "sh", "opacities", "scales", "rotations"):
        first[k][...] += 0.0                                     # the arrays the second call continues with
    second = emu.backward(a, fw, gcol, phases=2 | 8, scratch=first["scratch"], outs=first)
    for k in ("means3D", "sh", "opacities", "scales", "rotations", "means2D"):
        assert np.allclose(second[k], whole[k], rtol=1e-5, atol=1e-9), k
    # without the fill flag of the first call and with "already zero" claimed, stale contents would survive: the fill matters
    stale = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in first.items()}
    stale["means3D"][...] = 3.0
    third = emu.backward(a, fw, gcol, phases=2 | 8, scratch=first["scratch"], outs=stale)
    assert not np.allclose(third["means3D"], whole["means3D"])


@pytest.mark.parametrize("G", [2, 4])
def test_peer_l1_kernel_forwards_the_rendered_rows(emu, G):
    """h3dgs_l1_loss_grad_peer with peer_images: every "rank" holds only ITS tile rows of the frame; its L1 pass copies
    them into the images of the other ranks (the fused all-gather of the peer-mode step) while it evaluates the loss of
    those rows -- afterwards every image is the whole frame, every loss sum the loss of the whole frame."""
    import ctypes as C
    H, W = 70, 64
    g = np.random.default_rng(3)
    frame = g.uniform(0, 1, (3, H, W)).astype(np.float32); gt = g.uniform(0, 1, (3, H, W)).astype(np.float32)
    rows = np.arange(H)
    images = []
    for r in range(G):
        own = ((rows // 16) % G) == r
        img = np.full((3, H, W), np.nan, np.float32)            # what a rank has not rendered is not there
        img[:, own] = frame[:, own]
        images.append(img)
    sums = [np.zeros(1, np.float64) for _ in range(G)]
    outs = [np.zeros((3, H, W), np.float32) for _ in range(G)]
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    for r in range(G):
        ls = (C.c_void_p * G)(*[s_.ctypes.data for s_ in sums])
        ims = (C.c_void_p * G)(*[im.ctypes.data for im in images])
        rc = emu.L.h3dgs_l1_loss_grad_peer(3, H, W, p(images[r]), p(gt), C.c_float(0.5), G, r, p(outs[r]), G, ls, ims, None)
        assert rc == 0, emu.L.h3dgs_last_error()
    for r in range(G):
        assert np.array_equal(images[r], frame)
        assert abs(sums[r][0] - np.abs((frame - gt).astype(np.float64)).sum()) < 1e-2
        own = ((rows // 16) % G) == r
        assert np.array_equal(outs[r][:, own], np.sign((frame - gt)[:, own]) * np.float32(0.5))


@pytest.mark.parametrize("G", [2, 4])
def test_peer_mode_fused_collectives_schedule(emu, G):
    """Peer mode (h3dgs_raster_args.peer_count) on one CPU: G "ranks" run one after the other with numpy arrays standing in
    for peer memory.  Forward: every rank stores the pixels of ITS tile rows into the image of EVERY rank -> all G images
    equal the unsharded one bit for bit.  Backward phase 1: each rank leaves the (tile, Gaussian) sums of ITS tiles in its
    own accumulator and pushes the rows other ranks own (block-cyclic, 2^5 rows) into the owners' staging areas; phase 2 of
    the owner adds the staged rows of the ranks whose tile rows the Gaussian touches (the rank mask K1 wrote) and finishes
    exactly the owned rows.  Fused gather/scatter
    (render_indices) on top."""
    from oracle import oracle
    from emu_api import aligned, ptr
    cam = synth.make_camera(160, 112)
    leaves = synth.cloud_v1(1500, cam, zmin=2.0, zmax=30.0, seed=2, scale_k=1.0)
    z = leaves["means3D"][:, 2:3]
    leaves["scales"] = (8e-3 * np.sqrt(2 * z) * np.ones((1, 3))).astype(np.float32)
    h = synth.build_hierarchy(leaves)
    thr = synth.tau_threshold(6.0, cam)
    n, ri, pi, ni = oracle.expand_to_size(h["nodes"], h["boxes"], thr, cam.camera_center)
    ts, kids = oracle.get_interpolation_weights(ni, thr, h["nodes"], h["boxes"], cam.camera_center)
    bg = np.array([0.3, 0.2, 0.1], np.float32)
    f = oracle.rasterize_forward(h["means3D"], h["shs"], None, h["opacities"], h["scales"], h["rotations"], None,
                                 cam.world_view_transform, cam.full_proj_transform, cam.camera_center, bg, cam.W, cam.H,
                                 cam.tanfovx, cam.tanfovy, ts=ts, kids=kids, render_indices=ri, parent_indices=pi)
    gcol = synth.l1_grad(f["color"])
    b = oracle.rasterize_backward(f, gcol)
    a0, keep0 = emu.args(cam, bg, h, ts=ts, kids=kids, ridx=ri, pidx=pi)
    whole = emu.forward(a0, keep0)
    P, SHIFT = n, 5
    images = [aligned(3 * cam.H * cam.W * 4, np.float32, (3, cam.H, cam.W)) for _ in range(G)]
    accums = [aligned(emu.L.h3dgs_backward_scratch_bytes(P)) for _ in range(G)]
    stages = [aligned(G * P * 40) for _ in range(G)]            # [source rank][P][10] floats on every rank, never zeroed
    for st_ in stages:
        st_.view(np.float32)[:] = np.nan                        # a row that is read without having been pushed this step would show
    ranks = []
    for r in range(G):
        a, keep = emu.args(cam, bg, h, ts=ts, kids=kids, ridx=ri, pidx=pi, shard=(G, r))
        a.peer_count, a.grad_cyclic_log2 = G, SHIFT
        for k in range(G):
            a.peer_image[k], a.peer_stage[k] = ptr(images[k]), ptr(stages[k])
        ranks.append((a, keep, emu.forward(a, keep)))
    for img in images:
        assert np.array_equal(img, whole["color"])
    for a, keep, fw in ranks:                                    # phase 1 everywhere ("barrier"), then phase 2
        emu.backward(a, fw, gcol, phases=1, scratch=accums[a.shard_index])
    rows = np.arange(P)
    owner = (rows >> SHIFT) % G
    parts = [accums[r].view(np.float32)[: P * 10].reshape(P, 10).copy() for r in range(G)]
    assert all(p_.any() for p_ in parts)
    touched = np.stack([np.abs(p_).sum(1) > 0 for p_ in parts])            # [G, P]: a small Gaussian reaches few ranks' tile rows
    assert touched.sum(0).mean() < 0.75 * G
    total = {k: np.zeros(b[k].shape, np.float64) for k in ("means3D", "sh", "opacities", "scales", "rotations")}
    m2d = np.zeros((P, 3), np.float32)
    for a, keep, fw in ranks:
        g2 = emu.backward(a, fw, gcol, phases=2, scratch=accums[a.shard_index])
        for k in total:
            total[k] += g2[k]
        own = owner == a.shard_index
        assert not g2["means2D"][~own].any()
        m2d[own] = g2["means2D"][own]
    for k in total:
        grad_close(total[k].astype(np.float32), b[k], k)
    grad_close(m2d, b["means2D"], "means2D")


@pytest.mark.parametrize("tau,misalign,agg_only", [(0.0, False, False), (6.0, False, False), (60.0, False, False), (6.0, True, False),
                                                   (6.0, False, True)])
def test_single_pass_cut_over_many_tiles(emu, tau, misalign, agg_only, monkeypatch):
    """lod_cut_fused_kernel with 600+ tiles of 1024 nodes; indices, parents, nodes, weights (bit-exact) and kids against the
    oracle.  agg_only: the emulator runs the CTAs one after the other, so every predecessor would already show its inclusive
    prefix; the switch keeps all tiles but every 300th at "aggregate only", and the look-back has to add up to 299
    aggregates over ten windows of 32 status words."""
    if agg_only:
        monkeypatch.setenv("H3DGS_EMU_CUT_AGG_ONLY", "1")
    from emu_api import aligned, f32, i32, ptr
    from oracle import oracle
    cam = synth.make_camera(320, 200)
    leaves = synth.cloud_v1(310000 if agg_only else 41000, cam, zmin=2.0, zmax=40.0, seed=11, scale_k=1.0)
    z = leaves["means3D"][:, 2:3]
    leaves["scales"] = (4e-3 * np.sqrt(2 * z) * np.ones((1, 3))).astype(np.float32)
    h = synth.build_hierarchy(leaves)
    N = h["nodes"].shape[0]
    assert N > (600 if agg_only else 80) * 1024
    thr = synth.tau_threshold(tau, cam)
    n, ri, pi, ni = oracle.expand_to_size(h["nodes"], h["boxes"], thr, cam.camera_center)
    ts, kids = oracle.get_interpolation_weights(ni, thr, h["nodes"], h["boxes"], cam.camera_center)
    L = emu.L
    nodes, boxes, vp = i32(h["nodes"]), f32(h["boxes"]), f32(cam.camera_center)
    assert nodes.ctypes.data % 16 == 0 and boxes.ctypes.data % 16 == 0        # whole tiles arrive by bulk copy (TMA wrappers) ...
    if misalign:                                                              # ... views that are not 16-B aligned by plain loads
        buf = np.zeros(nodes.size + 4, np.int32)
        off = 1 + (-(buf.ctypes.data // 4) % 4)
        buf[off:off + nodes.size] = nodes.ravel()
        nodes = buf[off:off + nodes.size].reshape(nodes.shape)
        assert nodes.ctypes.data % 16 == 4
    r2, p2, n2, k2 = (aligned(N * 4, np.int32, (N,)) for _ in range(4))
    t2 = aligned(N * 4, np.float32, (N,))
    count = aligned(4, np.int32, (1,))
    scratch = aligned(L.h3dgs_expand_scratch_bytes(N))
    emu.check(L.h3dgs_lod_cut(N, ptr(nodes), ptr(boxes), thr, None, ptr(vp), ptr(r2), ptr(p2), ptr(n2), ptr(t2), ptr(k2),
                                  ptr(count), ptr(scratch), None))
    assert int(count[0]) == n > 0
    assert np.array_equal(r2[:n], ri) and np.array_equal(p2[:n], pi) and np.array_equal(n2[:n], ni)
    assert np.array_equal(t2[:n].view(np.uint32), ts.view(np.uint32)) and np.array_equal(k2[:n], kids)
    assert (r2[n:] == -1).all()


def test_prefiltered_flag_traps_on_a_culled_point(emu):
    """prefiltered=True is the caller's promise that nothing lies behind the near plane; the reference's kernel traps
    when the promise is broken -- here the forward returns an error instead of rendering."""
    cam, sc, ts, kids, bg = make_scene(300, 64, 48, seed=5)
    a, keep = emu.args(cam, bg, sc)
    a.prefiltered = 1
    fw = emu.forward(a, keep)                     # every point of this scene is in front of the camera
    assert fw["D"] > 0
    sc2 = dict(sc); sc2["means3D"] = sc["means3D"].copy(); sc2["means3D"][7, 2] = -1.0
    a2, keep2 = emu.args(cam, bg, sc2)
    a2.prefiltered = 1
    with pytest.raises(RuntimeError, match="filtered although prefiltered"):
        emu.forward(a2, keep2)
    a2.prefiltered = 0
    assert emu.forward(a2, keep2)["radii"][7] == 0


def test_tile_scan_over_more_than_one_pass(emu):
    """9000 tiles: the single-CTA tile scan needs two passes of 1024 x 8 tiles; ranges and keys against the oracle."""
    cam, sc, ts, kids, bg = make_scene(400, 1600, 1440, seed=13)
    f, b, gcol, gdep = oracle_run(cam, sc, bg, backward=False)
    a, keep = emu.args(cam, bg, sc)
    fw = emu.forward(a, keep)
    st = emu.state(a, fw)
    assert fw["D"] == f["num_rendered"] > 0
    assert np.array_equal(st["ranges"], f["ranges"]) and np.array_equal(st["keys_sorted"], f["keys"])
    assert np.array_equal(st["point_list"], f["point_list"])

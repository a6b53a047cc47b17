"""GPU: the view cull of the LOD cut (csrc/lod_cull.cu; the row mask of h3dgs_lod_cut_masked / h3dgs_lod_budget_masked;
pipeline's cull=, GraphedRender / GraphedPostStep(cull=True), evaluate_hierarchy(cull=True)).

  * the mask kernel equals the numpy restatement (tests/lod_cull_ref.py) bit for bit, on the CPU suite's hierarchies and
    on a 3 M-node hierarchy and a surround scene;
  * at tau 0, 3, 6 and 15 the culled frame's image and inverse depth are bit-identical to the unculled frame's, every
    row with a positive radius in the unculled frame is kept, and D is equal -- from the bench views and cameras inside
    the scene;
  * GraphedRender(cull=True) equals the eager culled frame; evaluate_hierarchy(cull=True) the unculled sweep;
  * GraphedPostStep with a PostState, culled against unculled over 30 iterations: the first loss bit for bit, then the
    losses and parameters within the graphed-vs-exact tolerances;
  * the culled budget: visible rows <= B, the next finer candidate exceeds B, non-increasing in B, never coarser than
    the unculled budget's threshold;
  * without cull the graphs hold the launches they held before."""
import numpy as np
import pytest

import lod_budget_ref as bref
import lod_cull_ref as ref
from h3dgs import synth

pytestmark = pytest.mark.gpu

CAM = synth.make_camera(480, 270)
TAUS = (0.0, 3.0, 6.0, 15.0)


def _bits(x):
    return int(np.asarray(x, np.float32).view(np.uint32))


def _dev_mask(h, cam, smod=1.0):
    import torch
    from h3dgs import _lib
    t = lambda a, dt=torch.float32: torch.tensor(np.asarray(a), dtype=dt, device="cuda")
    # the inputs stay referenced until the kernel has read them (a temporary's memory goes back to the allocator at once)
    nodes, mu, sc, ro = t(h["nodes"], torch.int32), t(h["means3D"]), t(h["scales"]), t(h["rotations"])
    view, proj = t(cam.world_view_transform), t(cam.full_proj_transform)
    out = torch.full((h["means3D"].shape[0],), 0xAB, dtype=torch.uint8, device="cuda")
    _lib.check(_lib.lib().h3dgs_lod_cull_mask(h["nodes"].shape[0], nodes.data_ptr(), mu.data_ptr(), sc.data_ptr(),
                                              ro.data_ptr(), smod, view.data_ptr(), proj.data_ptr(), cam.W, cam.H,
                                              cam.tanfovx, cam.tanfovy, out.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream))
    return out.cpu().numpy()


@pytest.mark.parametrize("name", [n for n, _ in ref.scenes(CAM)])
def test_kernel_equals_the_restatement(name):
    h = dict(ref.scenes(CAM))[name]
    for cname, cam in ref.cameras(h).items():
        for smod in ((1.0, 0.5, 3.0) if cname == "default" else (1.0,)):
            want, written = ref.mask(h, cam, smod)
            got = _dev_mask(h, cam, smod)
            assert np.array_equal(got[written], want[written]), (name, cname, smod)
            assert (got[~written] == 0xAB).all()


def test_edge_rows_kernel_equals_the_restatement():
    for cam in (synth.make_camera(160, 100), synth.make_camera(480, 270, primx=0.4)):
        h = ref.pair_hierarchy(*ref.edge_pairs(cam)[:6])
        want, written = ref.mask(h, cam)
        assert np.array_equal(_dev_mask(h, cam)[written], want[written])


def _surround_scene(n_leaves=60_000, skybox=0):
    from h3dgs import pipeline
    h = ref.surround_hierarchy(n_leaves, seed=9)
    if skybox:
        h = synth.append_skybox(h, skybox)
    return h, pipeline.Scene(h, requires_grad=False)


def _front_scene(skybox=0):
    from h3dgs import pipeline
    cam = synth.make_camera(480, 270)
    lv = synth.cloud_v1(9000, cam, zmin=2.0, zmax=40.0, seed=3, scale_k=1.0)
    z = lv["means3D"][:, 2:3]
    lv["scales"] = (4e-3 * np.sqrt(2.0 * z) * np.exp(0.4 * np.random.default_rng(1).standard_normal((z.shape[0], 3)))).astype(np.float32)
    h = synth.build_hierarchy(lv)
    if skybox:
        h = synth.append_skybox(h, skybox)
    return h, pipeline.Scene(h, requires_grad=False)


def _views(W=480, H=270):
    """the bench views (the default camera and yawed, shifted ones) and cameras inside the scene"""
    rs = np.random.default_rng(2)
    out = [synth.make_camera(W, H)] + [synth.yaw_camera(W, H, float(rs.uniform(-15, 15)), rs.uniform(-0.5, 0.5, 3))
                                       for _ in range(2)]
    out += [synth.yaw_camera(W, H, 120.0, [0.5, 0.2, -3.0]), synth.yaw_camera(W, H, -70.0, [0.0, -0.3, 8.0])]
    return out


def _render(scene, dcam, thr, cull):
    """render_hier_fused with the inverse depth -> (img, radii, invdepth, n, D)"""
    import torch
    from diff_gaussian_rasterization import GaussianRasterizer, _C
    from h3dgs import pipeline
    n, P = pipeline.fused_cut(scene, dcam, thr, cull)
    rs = pipeline.make_settings(scene, dcam, torch.zeros(3, device="cuda"), 3, ts=scene.interpolation_weights,
                                kids=scene.num_siblings, ridx=scene.render_indices[:P], pidx=scene.parent_indices[:P],
                                do_depth=True)
    means2D = torch.zeros((P, 3), device="cuda")
    with torch.no_grad():
        img, radii, invd = GaussianRasterizer(rs)(means3D=scene.means3D, means2D=means2D, shs=scene.shs,
                                                  colors_precomp=None, opacities=scene.opacities, scales=scene.scales,
                                                  rotations=scene.rotations, cov3D_precomp=None)
    return img.clone(), radii.clone(), invd.clone(), n, int(_C.last_num_rendered()), \
        scene.render_indices[:n].clone()


@pytest.mark.parametrize("which", ["front", "surround"])
def test_culled_frame_is_the_unculled_frame(which):
    import torch
    from h3dgs import pipeline
    h, scene = (_front_scene if which == "front" else _surround_scene)(skybox=40)
    fewer = 0
    for cam in _views():
        dcam = pipeline.DeviceCamera(cam)
        m = _dev_mask(h, cam)
        for tau in TAUS:
            thr = pipeline.fov_threshold(tau, dcam)
            img0, rad0, inv0, n0, D0, ri0 = _render(scene, dcam, thr, False)
            img1, rad1, inv1, n1, D1, ri1 = _render(scene, dcam, thr, True)
            assert torch.equal(img0, img1) and torch.equal(inv0, inv1), (which, tau)
            assert D0 == D1 and n1 <= n0
            drawn = ri0[rad0[:n0] > 0].cpu().numpy()
            assert (m[drawn] == 1).all(), (which, tau)
            assert np.array_equal(ri1.cpu().numpy(), ri0.cpu().numpy()[m[ri0.cpu().numpy()] == 1])
            fewer += n1 < n0
    if which == "surround":
        assert fewer > 0


def test_large_hierarchy_mask_and_frames():
    """the 3 M-node hierarchy of the budget tests: the kernel against the restatement, and culled frames"""
    import torch
    from h3dgs import pipeline
    from h3dgs.hier_build import build_hierarchy
    g = torch.Generator(device="cuda").manual_seed(5)
    P = 1_500_000
    u = lambda *s: torch.rand(*s, device="cuda", generator=g)
    xyz = torch.stack([u(P) * 80 - 40, u(P) * 20 - 10, u(P) * 120 + 2], 1)
    hb = build_hierarchy(xyz, torch.randn(P, 16, 3, device="cuda", generator=g) * 0.3, u(P) * 0.9 + 0.05,
                         torch.randn(P, 3, device="cuda", generator=g) * 0.5 - 3.5, torch.randn(P, 4, device="cuda", generator=g))
    arrays = dict(means3D=hb["xyz"], scales=hb["log_scales"].exp(), rotations=hb["rotations"], opacities=hb["opacities"],
                  shs=hb["shs"], nodes=hb["nodes"], boxes=hb["boxes"])
    h = {k: v.cpu().numpy() for k, v in arrays.items()}
    scene = pipeline.Scene(arrays, requires_grad=False)
    for cam in (synth.make_camera(1280, 720), synth.yaw_camera(1280, 720, 150.0, [0.0, 0.0, -60.0])):
        want, written = ref.mask(h, cam)
        got = _dev_mask(h, cam)
        assert np.array_equal(got[written], want[written])
        dcam = pipeline.DeviceCamera(cam)
        for tau in (3.0, 15.0):
            thr = pipeline.fov_threshold(tau, dcam)
            a, b = _render(scene, dcam, thr, False), _render(scene, dcam, thr, True)
            assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2]) and a[4] == b[4]


def test_graphed_render_equals_the_eager_culled_frame():
    import torch
    from h3dgs import pipeline
    from h3dgs.evaluate import GraphedRender
    h, scene = _surround_scene(skybox=30)
    bg = torch.zeros(3, device="cuda")
    N = scene.means3D.shape[0]
    cam = _views()[0]
    gr = GraphedRender(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, 0.01, row_capacity=N, bin_capacity=1 << 21,
                       cull=True)
    g0 = GraphedRender(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, 0.01, row_capacity=N, bin_capacity=1 << 21)
    assert gr.launches_per_frame == g0.launches_per_frame + 1 and g0.cull_mask is None
    for c in _views():
        dcam = pipeline.DeviceCamera(c)
        for tau in TAUS:
            thr = pipeline.fov_threshold(tau, dcam)
            for g in (gr, g0):
                g.set_camera(dcam)
                g.set_threshold(thr)
                g.frame()
            with torch.no_grad():
                img, _, n = pipeline.render_hier_fused(scene, dcam, bg, thr, cull=True)
            k = int(gr.counter.item()) - 1
            assert torch.equal(gr.image, img) and torch.equal(g0.image, img)
            assert int(gr.count.item()) == n and gr.results[k, 3].item() == n + scene.skybox_points
            assert n <= int(g0.count.item())


def test_evaluate_hierarchy_culled_equals_unculled():
    import torch
    from h3dgs import pipeline
    from h3dgs.evaluate import evaluate_hierarchy
    h, scene = _surround_scene(skybox=30)
    dcams = [pipeline.DeviceCamera(c) for c in _views()]
    g = torch.Generator(device="cpu").manual_seed(4)
    targets = []
    for c in dcams:
        with torch.no_grad():
            img = pipeline.render_hier_fused(scene, c, torch.zeros(3, device="cuda"), pipeline.fov_threshold(0.0, c))[0]
        targets.append((img + 0.03 * torch.randn(img.shape, generator=g).cuda()).contiguous())
    a = evaluate_hierarchy(scene, dcams, targets, list(TAUS))
    b = evaluate_hierarchy(scene, dcams, targets, list(TAUS), cull=True)
    for tau in TAUS:
        assert abs(a["psnr"][tau] - b["psnr"][tau]) <= 1e-9 * abs(a["psnr"][tau])
        assert abs(a["ssim"][tau] - b["ssim"][tau]) <= 1e-9 * abs(a["ssim"][tau])
    assert (b["rows"][..., 3] <= a["rows"][..., 3]).all() and (b["rows"][..., 3] < a["rows"][..., 3]).any()


def test_post_step_culled_tracks_unculled():
    import torch
    import test_gpu_post_train as tp
    from h3dgs.pipeline import DeviceCamera
    from h3dgs.poststep import GraphedPostStep
    cam, h = tp._hier()
    bg = torch.tensor([0.2, 0.1, 0.3], device="cuda")
    states = [tp._new_state(h), tp._new_state(h)]
    forms = []
    for s, cull in zip(states, (False, True)):
        sc = s.make_scene(requires_grad=False)
        gs = GraphedPostStep(sc, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, 0.01, exposure=True, mask=True,
                             bin_capacity=1 << 21, capture=False, state=s, cull=cull)
        gs.set_camera(DeviceCamera(cam))
        gs.capture()
        forms.append(gs)
    for it in range(30):
        st = [tp._graphed(s, gs, cam, it) for s, gs in zip(states, forms)]
        assert not st[0]["overflow"] and not st[1]["overflow"]
        assert st[1]["rows"] <= st[0]["rows"]
        if it == 0:
            assert st[0]["loss"] == st[1]["loss"]
            assert torch.equal(forms[0].image, forms[1].image)
        else:
            assert abs(st[0]["loss"] - st[1]["loss"]) <= 1e-4 * abs(st[0]["loss"]), it
    torch.cuda.synchronize()
    sa, sb = states
    for k in range(6):
        lr = tp._lr(0) if k == 0 else sa.lr[k]
        d = (sa.params[k] - sb.params[k]).abs()
        assert float(d.max()) <= 30 * 3.2 * lr, k
        near = d <= 1e-3 * sb.params[k].abs() + 1e-5
        assert float(near.float().mean()) >= 0.995, k


def test_culled_budget_fits_and_is_never_coarser():
    import torch
    from h3dgs import pipeline
    h, scene = _surround_scene()
    for cam in _views():
        dcam = pipeline.DeviceCamera(cam)
        floor = pipeline.fov_threshold(0.0, dcam)
        m = _dev_mask(h, cam)
        vis = ref.visible_nodes(h["nodes"], m)
        size = bref.hg.node_sizes(h["boxes"], np.asarray(cam.camera_center, np.float32))
        r0 = pipeline.budget_threshold(scene, dcam, 10 ** 9, floor, cull=True)[1]
        prev = None
        for frac in (2.0, 1.0, 0.5, 0.2, 0.05, 0.01, 0.0):
            B = int(r0 * frac)
            t, rows, met = pipeline.budget_threshold(scene, dcam, B, floor, cull=True)
            t0, _, _ = pipeline.budget_threshold(scene, dcam, B, floor)
            assert rows == bref.rows(vis, size, np.float32(t))
            assert np.float32(t) <= np.float32(t0)                   # never coarser than the unculled budget's
            if met:
                assert rows <= B
                if np.float32(t) != np.float32(floor):
                    lo = np.float32(np.nextafter(np.float32(t), np.float32(-np.inf)))
                    below = size[(size >= np.float32(floor)) & (size < lo)]
                    finer = np.float32(np.nextafter(below.max(), np.float32(np.inf))) if below.size else np.float32(floor)
                    assert bref.rows(vis, size, finer) > B
            if prev is not None:
                assert np.float32(t) >= prev                         # budgets shrink: never finer
            prev = np.float32(t)
            img, _, n, t2, _ = pipeline.render_hier_budget(scene, dcam, torch.zeros(3, device="cuda"), B, floor, cull=True)
            assert _bits(t2) == _bits(t) and n == rows


def test_without_cull_the_graphs_are_unchanged():
    import torch
    from h3dgs import pipeline
    from h3dgs.evaluate import GraphedRender
    from h3dgs.graphstep import GraphedStep
    h, scene = _front_scene(30)
    cam = CAM
    bg = torch.zeros(3, device="cuda")
    thr = pipeline.fov_threshold(3.0, cam)
    gr = GraphedRender(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, bin_capacity=1 << 20)
    gc = GraphedRender(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, bin_capacity=1 << 20, cull=True)
    gb = GraphedRender(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, bin_capacity=1 << 20, budget=1000)
    gbc = GraphedRender(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, bin_capacity=1 << 20, budget=1000, cull=True)
    assert gr.cull_mask is None and gb.cull_mask is None
    # the cull adds its one mask launch, nothing else
    assert gc.launches_per_frame == gr.launches_per_frame + 1 and gbc.launches_per_frame == gb.launches_per_frame + 1
    gs = GraphedStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, bin_capacity=1 << 20, capture=False)
    assert gs.cull_mask is None
    with pytest.raises(ValueError):
        GraphedStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, world=2, capture=False, cull=True)
    from h3dgs.dist import TileSharder
    with pytest.raises(ValueError):
        TileSharder(2, 0, "cuda").render(scene, pipeline.DeviceCamera(cam), bg, thr, cull=True)

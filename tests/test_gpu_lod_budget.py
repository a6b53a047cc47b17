"""GPU: the LOD budget (csrc/lod_budget.cu, pipeline.budget_threshold, GraphedRender(budget=), evaluate_hierarchy's
budget sweep).

  * the kernel equals the numpy restatement (tests/lod_budget_ref.py) bit for bit on the CPU suite's hierarchies;
  * on a 3 M-node hierarchy from the device creator: the cut at the chosen threshold fits, the next finer candidate
    does not, the reported rows are the cut's count, the threshold is non-increasing in the budget, and repeated and
    graph-replayed calls are bit-identical;
  * an ample budget renders exactly the tau-mode frame at the floor;
  * the budget sweep equals per-frame budget_threshold + the exact path + the metrics kernel, never synchronises the
    host, never overflows its rows when the budget is met, and re-runs bin/sort overflows at the frame's own threshold;
  * without budget= the graphs hold the launches they held before."""
import numpy as np
import pytest

import lod_budget_ref as ref
from h3dgs import synth

pytestmark = pytest.mark.gpu

CAM = synth.make_camera(480, 270)


def _bits(x):
    return int(np.asarray(x, np.float32).view(np.uint32))


def _budget_call(nodes, boxes, vp, floor, budget, scratch=None, out=None):
    import torch
    from h3dgs import _lib
    L = _lib.lib()
    N = nodes.shape[0]
    if scratch is None:
        scratch = torch.empty(int(L.h3dgs_lod_budget_scratch_bytes(N)), dtype=torch.uint8, device="cuda")
    thr, info = out if out is not None else (torch.empty(1, device="cuda"), torch.empty(4, dtype=torch.int32, device="cuda"))
    _lib.check(L.h3dgs_lod_budget(N, nodes.data_ptr(), boxes.data_ptr(), vp.data_ptr(), float(floor), None, int(budget), None,
                                  thr.data_ptr(), info.data_ptr(), scratch.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return thr, info


@pytest.mark.parametrize("name", [n for n, _ in ref.scenes(CAM)])
def test_kernel_equals_the_restatement(name):
    import torch
    h = dict(ref.scenes(CAM))[name]
    nodes, boxes = torch.tensor(h["nodes"], device="cuda"), torch.tensor(h["boxes"], device="cuda")
    for vp in ref.views(h, CAM).values():
        v = torch.tensor(vp, device="cuda")
        for floor in ref.floors(h, vp, CAM):
            tab = ref.table(h["nodes"], h["boxes"], vp, floor)
            for B in ref.budgets(h["nodes"], tab, floor, limit=40):
                want = ref.select(h["nodes"], h["boxes"], vp, floor, B, tab)
                thr, info = _budget_call(nodes, boxes, v, floor, B)
                i = info.cpu().numpy()
                assert _bits(thr.cpu().numpy()[0]) == _bits(want["threshold"]), (name, floor, B)
                assert [int(x) for x in i] == [want["rows"], want["unmet"], want["kept"], want["total"]], (name, floor, B)


@pytest.fixture(scope="module")
def big():
    """a 3 M-node hierarchy from the device creator (1.5 M leaves in front of the camera), viewpoints near and far"""
    import torch
    from h3dgs.hier_build import build_hierarchy
    g = torch.Generator(device="cuda").manual_seed(5)
    P = 1_500_000
    u = lambda *s: torch.rand(*s, device="cuda", generator=g)
    xyz = torch.stack([u(P) * 80 - 40, u(P) * 20 - 10, u(P) * 120 + 2], 1)
    hb = build_hierarchy(xyz, torch.randn(P, 16, 3, device="cuda", generator=g) * 0.3, u(P) * 0.9 + 0.05,
                         torch.randn(P, 3, device="cuda", generator=g) * 0.5 - 3.5, torch.randn(P, 4, device="cuda", generator=g))
    vps = [torch.tensor(v, dtype=torch.float32, device="cuda") for v in ([0.0, 0.0, 0.0], [0.0, 0.0, 60.0], [35.0, 5.0, 110.0])]
    return hb["nodes"].contiguous(), hb["boxes"].contiguous(), vps


def _cut_count(nodes, boxes, vp, thr):
    import torch
    from h3dgs import _lib
    L = _lib.lib()
    N = nodes.shape[0]
    z = lambda dt: torch.empty(N, dtype=dt, device="cuda")
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    scratch = torch.empty(int(L.h3dgs_expand_scratch_bytes(N)), dtype=torch.uint8, device="cuda")
    _lib.check(L.h3dgs_lod_cut(N, nodes.data_ptr(), boxes.data_ptr(), float(thr), None, vp.data_ptr(),
                               *(z(torch.int32).data_ptr() for _ in range(3)), z(torch.float32).data_ptr(),
                               z(torch.int32).data_ptr(), count.data_ptr(), scratch.data_ptr(),
                               torch.cuda.current_stream().cuda_stream))
    return int(count.item())


def test_large_hierarchy_cut_fits_and_is_the_finest(big):
    import torch
    nodes, boxes, vps = big
    assert nodes.shape[0] == 3_000_000 - 1
    floor = np.float32(synth.tau_threshold(0.0, CAM))
    for vp in vps:
        r_floor = _cut_count(nodes, boxes, vp, floor)
        size = _sizes(boxes, vp)
        prev, seen = None, set()
        for frac in (2.0, 1.0, 0.5, 0.2, 0.05, 0.01, 1e-4, 0.0):
            B = int(r_floor * frac)
            thr, info = _budget_call(nodes, boxes, vp, floor, B)
            t = np.float32(thr.item())
            rows, unmet, _, total = (int(x) for x in info.cpu())
            assert total == r_floor and rows == _cut_count(nodes, boxes, vp, t)
            if not unmet:
                assert rows <= B
                if t != floor:
                    # the next finer candidate: nextafter of the largest size below t*'s predecessor, or the floor
                    lo = np.float32(np.nextafter(t, np.float32(-np.inf)))
                    below = size[(size >= floor) & (size < lo)]
                    finer = np.float32(np.nextafter(below.max(), np.float32(np.inf))) if below.size else floor
                    assert _cut_count(nodes, boxes, vp, finer) > B
            seen.add("floor" if t == floor else "unmet" if unmet else "inner")
            if prev is not None:
                assert t >= prev                      # budgets shrink here: the threshold never gets finer
            prev = t
        assert "inner" in seen and "floor" in seen


def _sizes(boxes, vp):
    """node sizes as the kernels compute them (hier_general.node_sizes, the oracle's node_size restated)"""
    return ref.hg.node_sizes(boxes.cpu().numpy(), vp.cpu().numpy())


def test_large_hierarchy_repeated_and_graphed_calls_are_bit_identical(big):
    import torch
    from h3dgs import _lib
    nodes, boxes, vps = big
    L = _lib.lib()
    N = nodes.shape[0]
    scratch = torch.empty(int(L.h3dgs_lod_budget_scratch_bytes(N)), dtype=torch.uint8, device="cuda")
    floor_dev = torch.full((1,), float(synth.tau_threshold(0.0, CAM)), device="cuda")
    budget_dev = torch.zeros(1, dtype=torch.int32, device="cuda")
    vp = vps[0].clone()
    thr, info = torch.empty(1, device="cuda"), torch.empty(4, dtype=torch.int32, device="cuda")

    def launch():
        _lib.check(L.h3dgs_lod_budget(N, nodes.data_ptr(), boxes.data_ptr(), vp.data_ptr(), -1.0, floor_dev.data_ptr(), 0,
                                      budget_dev.data_ptr(), thr.data_ptr(), info.data_ptr(), scratch.data_ptr(),
                                      torch.cuda.current_stream().cuda_stream))
    eager = {}
    for vi in range(len(vps)):
        vp.copy_(vps[vi])
        for B in (0, 50_000, 400_000, 2_000_000):
            budget_dev.fill_(B)
            outs = set()
            for _ in range(3):
                launch()
                outs.add((_bits(thr.item()), tuple(info.cpu().tolist())))
            assert len(outs) == 1
            eager[(vi, B)] = outs.pop()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        launch()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        launch()
    for (vi, B), want in eager.items():
        vp.copy_(vps[vi])
        budget_dev.fill_(B)
        thr.fill_(-1)
        graph.replay()
        assert (_bits(thr.item()), tuple(info.cpu().tolist())) == want


def _scene(skybox=0):
    from h3dgs import pipeline
    cam = synth.make_camera(480, 270)
    lv = synth.cloud_v1(9000, cam, zmin=2.0, zmax=40.0, seed=3, scale_k=1.0)
    z = lv["means3D"][:, 2:3]
    lv["scales"] = (4e-3 * np.sqrt(2.0 * z) * np.exp(0.4 * np.random.default_rng(1).standard_normal((z.shape[0], 3)))).astype(np.float32)
    h = synth.build_hierarchy(lv)
    if skybox:
        h = synth.append_skybox(h, skybox)
    return cam, pipeline.Scene(h, requires_grad=False)


def _cams(W, H, n=3):
    rs = np.random.default_rng(2)
    return [synth.make_camera(W, H)] + [synth.yaw_camera(W, H, float(rs.uniform(-15, 15)), rs.uniform(-0.5, 0.5, 3))
                                        for _ in range(n - 1)]


@pytest.mark.parametrize("skybox", [0, 200])
def test_ample_budget_renders_the_tau_mode_frame(skybox):
    import torch
    from h3dgs import pipeline
    from h3dgs.evaluate import GraphedRender
    cam, scene = _scene(skybox)
    bg = torch.tensor([0.2, 0.1, 0.3], device="cuda")
    N = scene.means3D.shape[0]
    kw = dict(row_capacity=N, bin_capacity=1 << 20, sort_capacity=4096)
    floor = pipeline.fov_threshold(3.0, cam)
    tau_mode = GraphedRender(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, floor, **kw)
    budget_mode = GraphedRender(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, floor, budget=N, **kw)
    assert budget_mode.launches_per_frame > tau_mode.launches_per_frame
    for c in _cams(cam.W, cam.H):
        dcam = pipeline.DeviceCamera(c)
        for gr in (tau_mode, budget_mode):
            gr.set_camera(dcam)
            gr.set_threshold(pipeline.fov_threshold(3.0, dcam))
            gr.frame()
        k = int(tau_mode.counter.item()) - 1
        assert torch.equal(tau_mode.image, budget_mode.image) and torch.equal(tau_mode.radii, budget_mode.radii)
        # the metrics' per-block double sums are added with atomics: equal to their last bits, the status words exactly
        assert torch.equal(tau_mode.results[k, 2:], budget_mode.results[k, 2:])
        assert torch.allclose(tau_mode.results[k, :2], budget_mode.results[k, :2], rtol=1e-12, atol=0)
        t, rows, unmet = budget_mode.budget_values[k].tolist()
        assert _bits(t) == _bits(pipeline.fov_threshold(3.0, dcam)) and unmet == 0
        assert rows + skybox == budget_mode.results[k, 3].item()


def test_without_budget_the_graphs_are_unchanged():
    import torch
    from h3dgs import pipeline
    from h3dgs.evaluate import GraphedRender
    from h3dgs.graphstep import GraphedStep
    cam, scene = _scene(30)
    bg = torch.zeros(3, device="cuda")
    thr = pipeline.fov_threshold(3.0, cam)
    gr = GraphedRender(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, bin_capacity=1 << 20)
    gb = GraphedRender(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, bin_capacity=1 << 20, budget=1000)
    assert gr.budget_dev is None and not hasattr(gr, "budget_values")
    # the budget adds its own launches (memset, keys, sort, scan, select, finish) and the record copy, nothing else
    assert gb.launches_per_frame > gr.launches_per_frame
    gb_n = gb.launches_per_frame
    gs = GraphedStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, bin_capacity=1 << 20, capture=False)
    assert gs.budget_dev is None and gb_n > 0
    with pytest.raises(ValueError):
        gr.set_budget(10)


def _sweep_inputs(skybox=30):
    import torch
    from h3dgs import pipeline
    cam, scene = _scene(skybox)
    bg = torch.zeros(3, device="cuda")
    dcams = [pipeline.DeviceCamera(c) for c in _cams(cam.W, cam.H)]
    g = torch.Generator(device="cpu").manual_seed(4)
    targets = []
    for c in dcams:
        with torch.no_grad():
            img = pipeline.render_hier_fused(scene, c, bg, pipeline.fov_threshold(0.0, c))[0]
        targets.append((img + 0.03 * torch.randn(img.shape, generator=g).cuda()).contiguous())
    return cam, scene, bg, dcams, targets


def test_budget_sweep_equals_per_frame_budget_renders():
    import torch
    from h3dgs import _lib, pipeline
    from h3dgs.evaluate import HierarchyEvaluator, _metrics
    cam, scene, bg, dcams, targets = _sweep_inputs()
    n0 = pipeline.budget_threshold(scene, dcams[0], 10 ** 9, pipeline.fov_threshold(1.0, dcams[0]))[1]
    budgets = [n0 * 2, n0, n0 // 2, n0 // 5, n0 // 50, 0]
    ev = HierarchyEvaluator(scene, dcams, targets, None, budgets=budgets, tau_floor=1.0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ev.enqueue()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    res = ev.finish()
    assert set(res["psnr"]) == set(budgets) and res["budget_rows"].shape == (len(budgets), len(dcams), 4)
    r = ev._render_of(dcams[0])
    for bi, B in enumerate(budgets):
        for ci, c in enumerate(dcams):
            t, tau, rows, unmet = res["budget_rows"][bi, ci]
            want_t, want_rows, met = pipeline.budget_threshold(scene, c, B, pipeline.fov_threshold(1.0, c))
            assert _bits(t) == _bits(want_t) and rows == want_rows and unmet == (not met), (B, ci)
            assert abs(pipeline.fov_threshold(tau, c) - t) <= 1e-6 * t
            if met and B + scene.skybox_points <= scene.means3D.shape[0]:
                assert all(f[2][3] <= r.P for f in res["flagged"] if (f[0], f[1]) == (bi, ci))    # no row overflow
            with torch.no_grad():
                img, _, n, t2, _ = pipeline.render_hier_budget(scene, c, bg, B, pipeline.fov_threshold(1.0, c))
            assert _bits(t2) == _bits(t) and n == rows
            counter = torch.zeros(1, dtype=torch.int32, device="cuda")
            row = torch.zeros((1, _lib.EVAL_ROW), dtype=torch.float64, device="cuda")
            _metrics(r.L, c.H, c.W, img.contiguous(), targets[ci], None, None, 0, None, r.sums, counter, row,
                     torch.cuda.current_stream().cuda_stream, extra_rows=n + scene.skybox_points)
            assert np.allclose(res["rows"][bi, ci, :2], row[0, :2].cpu().numpy(), rtol=1e-12, atol=0), (B, ci)
    assert any(res["budget_rows"][-1, :, 3])            # budget 0: unmet, rendered at the coarsest cut
    assert res["budget_rows"][0, 0, 2] == n0            # the largest budget: the floor's cut


def test_budget_sweep_reruns_overflows_at_the_frames_own_threshold():
    import torch
    from h3dgs import pipeline
    from h3dgs.evaluate import HierarchyEvaluator
    cam, scene, bg, dcams, targets = _sweep_inputs()
    n0 = pipeline.budget_threshold(scene, dcams[0], 10 ** 9, pipeline.fov_threshold(0.0, dcams[0]))[1]
    budgets = [n0, n0 // 4]
    N = scene.means3D.shape[0]
    small = HierarchyEvaluator(scene, dcams, targets, None, budgets=budgets,
                               capacities=dict(row_capacity=N, bin_capacity=2000, sort_capacity=32))
    small.enqueue()
    got = small.finish()
    ample = HierarchyEvaluator(scene, dcams, targets, None, budgets=budgets,
                               capacities=dict(row_capacity=N, bin_capacity=1 << 21, sort_capacity=8192))
    ample.enqueue()
    want = ample.finish()
    assert got["rerun"] > 0 and want["rerun"] == 0
    assert np.array_equal(got["budget_rows"], want["budget_rows"])
    assert np.allclose(got["rows"][..., :2], want["rows"][..., :2], rtol=1e-12, atol=0)

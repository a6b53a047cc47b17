"""GPU: the LOD cut and the hierarchy step on general hierarchies (tests/hier_general.py): nodes holding several
Gaussians, fan-out 1..16, rows in a shuffled block order, leaves with a merged Gaussian, interior nodes with leaf
Gaussians of their own.

  * the cut (two-call API and h3dgs_lod_cut with the threshold on the device) bit for bit against the oracle, over
    sizes from one node to ~300 k (a single tile, the bulk-copy path on the last tile, more than 32 tiles), viewpoints
    outside, inside the root, inside a deep leaf and on a box face, tau thresholds and thresholds that tie a node's
    size, and a nodes view at a 28-byte offset;
  * boxes that are not 16-byte aligned are refused before anything is enqueued;
  * pipeline.l1_step (fused and unfused) against the oracle composition, per tensor and per row on the rows that
    many cut rows lerp towards and on rows that are rendered and lerp partners at once;
  * GraphedStep (eager and captured) and GraphedRender against the exact path, and their refusal of a hierarchy
    with more nodes than Gaussian rows."""
import numpy as np
import pytest

import hier_general as hg
from h3dgs import synth
from util import rel_err

pytestmark = pytest.mark.gpu

SIZES = [1, 2, 5, 1023, 1024, 1025, 4096, 32 * 1024 + 4, 300 * 1024 + 3]
TAUS = [0.0, 3.0, 6.0, 15.0, 200.0]
POISON = 12345


def _cases(h, cam):
    for name, vp in hg.viewpoints(h, cam).items():
        root = hg.node_sizes(h["boxes"][:1], vp)[0]
        above = [np.float32(2) * root] if root < hg.FLT_MAX else []
        for thr in [np.float32(synth.tau_threshold(t, cam)) for t in TAUS] + hg.tie_thresholds(h, vp) + above:
            yield name, vp, np.float32(thr)


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("N", SIZES)
def test_cut_bit_exact_on_general_trees(N):
    import torch
    from gaussian_hierarchy._C import expand_to_size, get_interpolation_weights
    from h3dgs import _lib
    from oracle import oracle
    cam = synth.make_camera(480, 270)
    h = hg.dense_hierarchy(N, N, cam, sh_degree=0)
    assert h["nodes"].shape[0] == N
    R = h["means3D"].shape[0]
    cap = max(N, R) + 16                                  # the cut emits up to R rows and marks [n, N) with -1
    L = _lib.lib()
    stream = torch.cuda.current_stream().cuda_stream
    nodes, boxes = torch.tensor(h["nodes"], device="cuda"), torch.tensor(h["boxes"], device="cuda")
    buf = torch.zeros(N * 7 + 8, dtype=torch.int32, device="cuda")      # the same nodes at a 28-byte offset
    buf[7:7 + N * 7] = nodes.view(-1)
    nodes_off = buf[7:7 + N * 7].view(N, 7)
    assert nodes_off.data_ptr() % 16 == 12
    scratch = torch.empty(int(L.h3dgs_expand_scratch_bytes(N)), dtype=torch.uint8, device="cuda")
    pz = lambda dt: torch.full((cap,), POISON, dtype=dt, device="cuda")
    checked = 0
    for name, vp, thr in _cases(h, cam):
        n, ri, pi, ni = oracle.expand_to_size(h["nodes"], h["boxes"], thr, vp)
        ts, kids = oracle.get_interpolation_weights(ni, thr, h["nodes"], h["boxes"], vp)
        vpd = torch.tensor(vp, device="cuda")
        what = (name, float(thr))
        # the two-call API of train_post.py
        r, p, nn_ = pz(torch.int32), pz(torch.int32), pz(torch.int32)
        assert expand_to_size(nodes, boxes, float(thr), vpd, torch.zeros(3), r, p, nn_) == n, what
        t, k = pz(torch.float32), pz(torch.int32)
        get_interpolation_weights(nn_[:n], float(thr), nodes, boxes, torch.tensor(vp), torch.zeros(3), t, k)
        got = [x.cpu().numpy() for x in (r, p, nn_, t, k)]
        assert np.array_equal(got[0][:n], ri) and np.array_equal(got[1][:n], pi) and np.array_equal(got[2][:n], ni), what
        assert np.array_equal(_bits(got[3][:n]), _bits(ts)) and np.array_equal(got[4][:n], kids), what
        assert all((g[n:] == POISON).all() for g in got), what
        # the device cut, threshold read on the device, both nodes views
        for nd in (nodes, nodes_off):
            r, p, nn_, t, k = pz(torch.int32), pz(torch.int32), pz(torch.int32), pz(torch.float32), pz(torch.int32)
            count = torch.full((1,), -7, dtype=torch.int32, device="cuda")
            thr_dev = torch.full((1,), float(thr), dtype=torch.float32, device="cuda")
            _lib.check(L.h3dgs_lod_cut(N, nd.data_ptr(), boxes.data_ptr(), -1.0, thr_dev.data_ptr(), vpd.data_ptr(), r.data_ptr(),
                                       p.data_ptr(), nn_.data_ptr(), t.data_ptr(), k.data_ptr(), count.data_ptr(),
                                       scratch.data_ptr(), stream))
            got = [x.cpu().numpy() for x in (r, p, nn_, t, k)]
            assert int(count.item()) == n, what
            assert np.array_equal(got[0][:n], ri) and np.array_equal(got[1][:n], pi) and np.array_equal(got[2][:n], ni), what
            assert np.array_equal(_bits(got[3][:n]), _bits(ts)) and np.array_equal(got[4][:n], kids), what
            assert (got[0][n:N] == -1).all() and (got[0][max(n, N):] == POISON).all(), what
            assert all((g[n:] == POISON).all() for g in got[1:]), what
        checked += n > 0
    assert checked > 0


def test_misaligned_boxes_are_refused():
    """every cut path reads boxes as float4: a view that is not 16-byte aligned is an argument error, returned before
    any kernel is launched (the outputs keep their contents)"""
    import torch
    from gaussian_hierarchy._C import expand_to_size, get_interpolation_weights
    from h3dgs import _lib
    cam = synth.make_camera(480, 270)
    h = hg.dense_hierarchy(9, 1025, cam, sh_degree=0)
    N = 1025
    L = _lib.lib()
    nodes = torch.tensor(h["nodes"], device="cuda")
    buf = torch.zeros(N * 8 + 4, device="cuda")
    buf[1:1 + N * 8] = torch.tensor(h["boxes"]).view(-1)
    boxes = buf[1:1 + N * 8].view(N, 2, 4)
    assert boxes.data_ptr() % 16 == 4 and boxes.is_contiguous()
    vp = torch.tensor(cam.camera_center, device="cuda")
    r = torch.full((4 * N,), 7, dtype=torch.int32, device="cuda")
    p, nn_, k = torch.zeros_like(r), torch.zeros_like(r), torch.zeros_like(r)
    t = torch.zeros(4 * N, device="cuda")
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        expand_to_size(nodes, boxes, 0.01, vp, torch.zeros(3), r, p, nn_)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        get_interpolation_weights(torch.arange(10, dtype=torch.int32, device="cuda"), 0.01, nodes, boxes, vp.cpu(),
                                  torch.zeros(3), t, k)
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    scratch = torch.empty(int(L.h3dgs_expand_scratch_bytes(N)), dtype=torch.uint8, device="cuda")
    rc = L.h3dgs_lod_cut(N, nodes.data_ptr(), boxes.data_ptr(), 0.01, None, vp.data_ptr(), r.data_ptr(), p.data_ptr(),
                         nn_.data_ptr(), t.data_ptr(), k.data_ptr(), count.data_ptr(), scratch.data_ptr(),
                         torch.cuda.current_stream().cuda_stream)
    assert rc == -1 and b"16-byte aligned" in L.h3dgs_last_error()
    torch.cuda.synchronize()
    assert bool((r == 7).all()) and not bool(t.any())


def _step_scene(tau, skybox=200):
    cam = synth.make_camera(480, 270)
    h = hg.dense_hierarchy(21, 4096, cam)
    if skybox:
        h = synth.append_skybox(h, skybox)
    return cam, h, synth.tau_threshold(tau, cam)


def _row_close(g, ref, rows, name):
    """per row: max |g - ref| within 1e-3 of the row's own magnitude plus 5e-6 of the tensor's"""
    g = np.asarray(g, np.float64).reshape(g.shape[0], -1)[rows]
    ref2 = np.asarray(ref, np.float64).reshape(ref.shape[0], -1)
    scale = np.abs(ref2).max()
    ref2 = ref2[rows]
    d = np.abs(g - ref2).max(1)
    lim = 1e-3 * np.abs(ref2).max(1) + 5e-6 * scale
    assert (d <= lim).all(), (name, rows[d > lim][:5], float((d / np.maximum(lim, 1e-30)).max()))


@pytest.mark.parametrize("tau", [6.0, 15.0])
def test_hierarchy_step_on_a_general_tree(tau):
    import torch
    from h3dgs import pipeline
    from oracle import oracle
    from test_gpu_pipeline import _oracle_hier_step
    cam, h, thr = _step_scene(tau)
    S = h["skybox_points"]
    gt = np.random.default_rng(2).uniform(0, 1, (3, cam.H, cam.W)).astype(np.float32)
    n_ref, f, gref = _oracle_hier_step(h, cam, thr, gt)
    _, ri, pi, ni = oracle.expand_to_size(h["nodes"], h["boxes"], thr, cam.camera_center)
    ts, kids = oracle.get_interpolation_weights(ni, thr, h["nodes"], h["boxes"], cam.camera_center)
    part = (ts > 0) & (ts < 1) & (pi >= 0)
    assert part.any() and (kids[part] > 2).any()
    lerp_count = np.bincount(pi[part], minlength=h["means3D"].shape[0])
    many = np.nonzero(lerp_count >= 4)[0]                          # parent rows of four or more lerp scatters
    both = np.intersect1d(ri, pi[part])                            # rendered rows that are lerp partners too
    if tau == 15.0:
        assert many.size > 0 and both.size > 0
    rows = np.union1d(many, both)
    scene = pipeline.Scene(h)
    dcam = pipeline.DeviceCamera(cam)
    bg0, gtd = torch.zeros(3, device="cuda"), torch.tensor(gt, device="cuda")
    imgs = {}
    for fused in (False, True):
        loss, radii, n = pipeline.l1_step(scene, dcam, bg0, gtd, thr, fused=fused)
        assert n == n_ref and radii.shape[0] == n + S
        assert np.array_equal(radii.cpu().numpy(), f["radii"])
        assert abs(loss.item() - np.abs(f["color"] - gt).mean()) < 1e-6
        for name, p in [("means3D", scene.means3D), ("scales", scene.scales), ("shs", scene.shs),
                        ("opacities", scene.opacities), ("rotations", scene.rotations)]:
            g = p.grad.cpu().numpy()
            e = rel_err(g, gref[name])
            assert e < 2e-5, (fused, name, e)
            if rows.size:
                _row_close(g, gref[name], rows, (fused, name))
        with torch.no_grad():
            imgs[fused] = (pipeline.render_hier_fused if fused else pipeline.render_hier)(scene, dcam, bg0, thr)[0]
    assert torch.equal(imgs[False], imgs[True])


@pytest.mark.parametrize("capture", [False, True])
def test_sync_free_step_on_a_general_tree(capture):
    import torch
    from h3dgs import pipeline
    from h3dgs.graphstep import GraphedStep
    from test_gpu_graphstep import _cams, _exact_step
    cam, h, thr = _step_scene(15.0)
    S = h["skybox_points"]
    assert h["means3D"].shape[0] - S > h["nodes"].shape[0]          # R > N_nodes
    scene = pipeline.Scene(h)
    bg = torch.tensor([0.2, 0.1, 0.3], device="cuda")
    cams = _cams(cam.W, cam.H)
    g = torch.Generator(device="cpu").manual_seed(5)
    gts = [torch.rand((3, cam.H, cam.W), generator=g).cuda() for _ in cams]
    dcams = [pipeline.DeviceCamera(c) for c in cams]
    gs = GraphedStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, bin_capacity=1 << 20, sort_capacity=4096,
                     capture=False)
    gs.set_camera(dcams[0]); gs.gt.copy_(gts[0])
    if capture:
        gs.capture()
    for v, tau in ((0, 15.0), (1, 15.0), (2, 6.0), (0, 3.0)):
        t = synth.tau_threshold(tau, cam)
        loss, radii, n, grads, img, D = _exact_step(scene, dcams[v], bg, gts[v], t)
        gs.set_threshold(t)
        gs.step(dcams[v], gts[v])
        st = gs.status()
        assert not st["overflow"] and st["rows"] == n + S and st["D"] == D
        assert abs(st["loss"] - loss) < 1e-7
        assert torch.equal(gs.image, img)
        assert torch.equal(gs.radii[:n + S], radii) and bool((gs.radii[n + S:] == 0).all())
        for k, ref in grads.items():
            e = rel_err(gs.grads[k].cpu().numpy(), ref.cpu().numpy())
            assert e < 5e-6, (v, k, e)


def test_graphed_render_on_a_general_tree():
    import torch
    from h3dgs import pipeline
    from h3dgs.evaluate import GraphedRender
    from test_gpu_graphstep import _cams
    cam, h, _ = _step_scene(0.0)
    S = h["skybox_points"]
    scene = pipeline.Scene(h, requires_grad=False)
    bg = torch.tensor([0.2, 0.1, 0.3], device="cuda")
    gr = GraphedRender(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, pipeline.fov_threshold(0.0, cam),
                       bin_capacity=1 << 20, sort_capacity=4096)
    k = 0
    for dcam in [pipeline.DeviceCamera(c) for c in _cams(cam.W, cam.H)]:
        for tau in TAUS[:4]:
            thr = pipeline.fov_threshold(tau, dcam)
            with torch.no_grad():
                img, radii, n = pipeline.render_hier_fused(scene, dcam, bg, thr)
            gr.set_camera(dcam)
            gr.set_threshold(thr)
            gr.frame()
            k += 1
            assert torch.equal(gr.image, img), tau
            row = gr.results[k - 1].cpu().numpy()
            assert row[2] == 0.0 and row[3] == n + S and torch.equal(gr.radii[:n + S], radii)


def test_sync_free_paths_refuse_more_nodes_than_rows():
    """h3dgs_lod_cut marks one index entry per node; a hierarchy whose nodes outnumber its Gaussian rows (nodes that hold
    no Gaussian) would overrun the row-sized index arrays, so both sync-free paths refuse it up front"""
    import torch
    from h3dgs import pipeline
    from h3dgs.evaluate import GraphedRender
    from h3dgs.graphstep import GraphedStep
    cam = synth.make_camera(480, 270)
    h = hg.dense_hierarchy(3, 2000, cam, empty_p=0.7, leaf_leafs=(1, 1), leaf_merged_p=0.0, interior_merged=(1, 1),
                           interior_leafs_p=0.0)
    assert h["nodes"].shape[0] > h["means3D"].shape[0]
    scene = pipeline.Scene(h, requires_grad=False)
    bg = torch.zeros(3, device="cuda")
    thr = synth.tau_threshold(6.0, cam)
    for cls in (GraphedStep, GraphedRender):
        with pytest.raises(ValueError, match="nodes"):
            cls(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, capture=False)
    # the exact path sizes nothing by the node count and still renders the cut
    with torch.no_grad():
        img, radii, n = pipeline.render_hier_fused(scene, pipeline.DeviceCamera(cam), bg, thr)
    assert 0 < n <= h["means3D"].shape[0] and bool(torch.isfinite(img).all())

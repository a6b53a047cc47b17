"""CPU: the LOD cut on general hierarchies (tests/hier_general.py) -- nodes holding several Gaussians, fan-out 1..16,
rows in a shuffled block order, leaves with a merged Gaussian, interior nodes with leaf Gaussians -- against an
independent numpy statement of the cut and a path-by-path invariant; then the library's own cut and fused
gather/scatter kernels, built against the SIMT emulator (tests/emul/), against the oracle."""
import os
import sys

import numpy as np
import pytest

import hier_general as hg
from h3dgs import synth

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emul"))

SIZES = [1, 2, 5, 1023, 1024, 1025, 4096, 32 * 1024 + 4]
TAUS = [0.0, 3.0, 6.0, 15.0, 200.0]
CAM = synth.make_camera(480, 270)

_trees = {}
POISON = 12345


def tree(N, **kw):
    key = (N, tuple(sorted(kw.items())))
    if key not in _trees:
        _trees[key] = hg.dense_hierarchy(N, N, CAM, **kw)
    return _trees[key]


def cases(h, taus=TAUS):
    """(viewpoint name, viewpoint, threshold) over every viewpoint, the tau thresholds, the tie thresholds and one
    threshold above the root's size (when it is finite)"""
    for name, vp in hg.viewpoints(h, CAM).items():
        root = hg.node_sizes(h["boxes"][:1], vp)[0]
        above = [np.float32(2) * root] if root < hg.FLT_MAX else []
        for thr in [np.float32(synth.tau_threshold(t, CAM)) for t in taus] + hg.tie_thresholds(h, vp) + above:
            yield name, vp, np.float32(thr)


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def test_generator_covers_what_the_cut_tests_rely_on():
    h = tree(4096)
    nodes = h["nodes"]
    N, R = nodes.shape[0], h["means3D"].shape[0]
    depth, parent, start, cl, cm, first, nk = nodes.T
    assert (start != np.arange(N)).mean() > 0.9 and R != N
    assert ((cl + cm) > 1).any() and (cm[nk == 0] > 0).any() and (cl[nk > 0] > 0).any()
    assert (nk > 2).any() and (nk == 1).any() and (nk >= 12).any()
    lvl = np.zeros(N, np.int64)
    for n in range(1, N):
        lvl[n] = lvl[parent[n]] + 1
    assert len(set(lvl[nk == 0])) > 2 and (depth[nk == 0] == 0).all()   # leaves at different heights
    has = parent >= 0
    assert all(depth[n] == 1 + depth[first[n]:first[n] + nk[n]].max() for n in np.nonzero(nk)[0])
    assert (start[parent[has]] != parent[has]).mean() > 0.9            # the parent's first Gaussian is not its id
    ids = np.arange(N)
    assert all(np.array_equal(parent[first[n]:first[n] + nk[n]], np.full(nk[n], n)) for n in ids[nk > 0])   # contiguous
    sky = synth.append_skybox(h, 7)
    assert sky["means3D"].shape[0] == R + 7 and sky["skybox_points"] == 7
    # nested boxes, min.w = the largest extent
    b = h["boxes"]
    assert (b[has, 0, :3] >= b[parent[has], 0, :3]).all() and (b[has, 1, :3] <= b[parent[has], 1, :3]).all()
    assert np.array_equal(b[:, 0, 3], (b[:, 1, :3] - b[:, 0, :3]).max(1))
    # at tau 15 the cut holds interior nodes, 0 < t < 1 rows under parents of more than two children, and parent rows
    # that four or more rows lerp towards; coarse nodes with leaf Gaussians are rendered and are lerp partners at once
    thr = synth.tau_threshold(15.0, CAM)
    n, ri, pi, ni = hg.cut(nodes, b, thr, CAM.camera_center)
    t, k = hg.weights(ni, thr, nodes, b, CAM.camera_center)
    part = (t > 0) & (t < 1)
    assert (part & (k > 2)).sum() > 20 and (depth[ni] > 0).any()
    assert np.bincount(pi[part]).max() >= 4
    assert np.isin(pi[part], ri).any()
    # the empty-node knob: more nodes than Gaussian rows
    e = hg.dense_hierarchy(3, 2000, CAM, empty_p=0.7, leaf_leafs=(1, 1), leaf_merged_p=0.0, interior_merged=(1, 1),
                           interior_leafs_p=0.0)
    assert e["nodes"].shape[0] > e["means3D"].shape[0]


@pytest.mark.parametrize("N", SIZES)
def test_oracle_equals_the_numpy_statement(N):
    from oracle import oracle
    h = tree(N)
    assert h["nodes"].shape[0] == N
    for name, vp, thr in cases(h):
        n, ri, pi, ni = oracle.expand_to_size(h["nodes"], h["boxes"], thr, vp)
        m = hg.cut(h["nodes"], h["boxes"], thr, vp)
        assert n == m[0], (name, thr)
        for a, b in zip((ri, pi, ni), m[1:]):
            assert np.array_equal(a, b), (name, thr)
        ts, kids = oracle.get_interpolation_weights(ni, thr, h["nodes"], h["boxes"], vp)
        t2, k2 = hg.weights(ni, thr, h["nodes"], h["boxes"], vp)
        assert np.array_equal(bits(ts), bits(t2)) and np.array_equal(kids, k2), (name, thr)


@pytest.mark.parametrize("N", [2, 5, 1025, 4096])
def test_cut_invariant_holds(N):
    from oracle import oracle
    h = tree(N)
    seen = set()
    for name, vp, thr in cases(h):
        n, ri, pi, ni = oracle.expand_to_size(h["nodes"], h["boxes"], thr, vp)
        hg.check_cut_invariant(h["nodes"], h["boxes"], thr, vp, ri, ni)
        size = hg.node_sizes(h["boxes"], vp)
        seen.add(("root below target", bool(size[0] < thr)))
        if size[0] < thr:
            assert n == 0                       # a root already below the target selects nothing
    if N > 5:
        assert seen == {("root below target", False), ("root below target", True)}


@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    from build_emu import build
    from emu_api import Emu
    return Emu(build(str(tmp_path_factory.mktemp("h3dgs_emu_general"))))


def _emu_cut(emu, h, thr, vp, nodes=None, device_threshold=True):
    from emu_api import aligned, f32, i32, ptr
    L = emu.L
    N = h["nodes"].shape[0]
    cap = max(N, h["means3D"].shape[0]) + 16                 # the cut emits up to R rows; -1 marks [n, N)
    nodes = i32(h["nodes"]) if nodes is None else nodes
    boxes, vpa, thr_dev = f32(h["boxes"]), f32(vp), f32([thr])
    r, p, nn, k = (aligned(cap * 4, np.int32, (cap,)) for _ in range(4))
    for a in (r, p, nn, k):
        a[:] = POISON
    t = aligned(cap * 4, np.float32, (cap,))
    t[:] = POISON
    count = aligned(4, np.int32, (1,))
    scratch = aligned(L.h3dgs_expand_scratch_bytes(N))
    emu.check(L.h3dgs_lod_cut(N, ptr(nodes), ptr(boxes), -1.0 if device_threshold else float(thr),
                              ptr(thr_dev) if device_threshold else None, ptr(vpa), ptr(r), ptr(p), ptr(nn), ptr(t), ptr(k),
                              ptr(count), ptr(scratch), None))
    return int(count[0]), r, p, nn, t, k


def _check_against_oracle(got, h, thr, vp, what):
    from oracle import oracle
    n, ri, pi, ni = oracle.expand_to_size(h["nodes"], h["boxes"], thr, vp)
    ts, kids = oracle.get_interpolation_weights(ni, thr, h["nodes"], h["boxes"], vp)
    c, r, p, nn, t, k = got
    assert c == n, what
    assert np.array_equal(r[:n], ri), what
    assert np.array_equal(p[:n], pi), what
    assert np.array_equal(nn[:n], ni), what
    assert np.array_equal(bits(t[:n]), bits(ts)), what
    assert np.array_equal(k[:n], kids), what
    N = h["nodes"].shape[0]
    assert (r[n:N] == -1).all(), what
    assert (r[max(n, N):] == POISON).all() and all((a[n:] == POISON).all() for a in (p, nn, t, k)), what   # nothing else written
    return n


@pytest.mark.parametrize("N", SIZES)
def test_emulated_device_cut_equals_the_oracle(emu_lib, N):
    """h3dgs_lod_cut (threshold on the device for the tau cases, by value for the ties) bit for bit, the -1 tail included"""
    h = tree(N)
    taus = TAUS if N <= 4096 else [6.0, 200.0]
    for name, vp, thr in cases(h, taus):
        _check_against_oracle(_emu_cut(emu_lib, h, thr, vp, device_threshold=name != "face"), h, thr, vp, (name, thr))


def test_emulated_two_call_api_equals_the_oracle(emu_lib):
    from emu_api import aligned, f32, i32, ptr
    from oracle import oracle
    L = emu_lib.L
    for N in (5, 1025, 4096):
        h = tree(N)
        nodes, boxes = i32(h["nodes"]), f32(h["boxes"])
        scratch = aligned(L.h3dgs_expand_scratch_bytes(N))
        for name, vp, thr in cases(h):
            n, ri, pi, ni = oracle.expand_to_size(h["nodes"], h["boxes"], thr, vp)
            ts, kids = oracle.get_interpolation_weights(ni, thr, h["nodes"], h["boxes"], vp)
            cap = max(N, h["means3D"].shape[0])
            r, p, nn = (aligned(cap * 4, np.int32, (cap,)) for _ in range(3))
            vpa = f32(vp)
            got = emu_lib.check(L.h3dgs_expand_to_size(N, ptr(nodes), ptr(boxes), float(thr), ptr(vpa), 0.0, 0.0, 0.0,
                                                       ptr(r), ptr(p), ptr(nn), ptr(scratch), None))
            assert got == n and np.array_equal(r[:n], ri) and np.array_equal(p[:n], pi) and np.array_equal(nn[:n], ni)
            if n == 0:
                continue
            t, k, idx = aligned(n * 4, np.float32, (n,)), aligned(n * 4, np.int32, (n,)), i32(ni)
            emu_lib.check(L.h3dgs_get_interpolation_weights(n, ptr(idx), float(thr), ptr(nodes), ptr(boxes),
                                                            float(vp[0]), float(vp[1]), float(vp[2]), 0.0, 0.0, 0.0,
                                                            ptr(t), ptr(k), None))
            assert np.array_equal(bits(t), bits(ts)) and np.array_equal(k, kids), (name, thr)


@pytest.mark.parametrize("agg_only", [False, True])
def test_emulated_cut_with_unaligned_nodes_and_many_tiles(emu_lib, agg_only, monkeypatch):
    """a nodes view at a 28-byte offset (plain loads on every tile); ~300 k nodes, and with agg_only the look-back adds
    up aggregates over several windows of 32 status words"""
    if agg_only:
        monkeypatch.setenv("H3DGS_EMU_CUT_AGG_ONLY", "1")
    from emu_api import aligned
    N = 300 * 1024 + 3 if agg_only else 4096
    h = tree(N, sh_degree=0)
    buf = aligned((N * 7 + 8) * 4, np.int32, (N * 7 + 8,))
    buf[7:7 + N * 7] = h["nodes"].ravel()
    nodes = buf[7:7 + N * 7].reshape(N, 7)
    assert nodes.ctypes.data % 16 == 12
    for tau in (6.0, 15.0):
        thr = np.float32(synth.tau_threshold(tau, CAM))
        n = _check_against_oracle(_emu_cut(emu_lib, h, thr, CAM.camera_center, nodes=nodes), h, thr, CAM.camera_center, tau)
        assert n > 0


def test_misaligned_boxes_are_refused(emu_lib):
    """boxes are read as float4 on every path: a view that is not 16-byte aligned is an argument error, reported before
    anything runs (the outputs stay untouched)"""
    from emu_api import aligned, f32, i32, ptr
    L = emu_lib.L
    h = tree(1025)
    N = 1025
    buf = aligned((N * 8 + 4) * 4, np.float32, (N * 8 + 4,))
    buf[1:1 + N * 8] = h["boxes"].ravel()
    boxes = buf[1:1 + N * 8]
    nodes, vp, thr_dev = i32(h["nodes"]), f32(CAM.camera_center), f32([0.01])
    r, p, nn, k = (aligned(N * 4, np.int32, (N,)) for _ in range(4))
    r[:] = 7
    t = aligned(N * 4, np.float32, (N,))
    count = aligned(4, np.int32, (1,))
    scratch = aligned(L.h3dgs_expand_scratch_bytes(N))
    rc = L.h3dgs_lod_cut(N, ptr(nodes), ptr(boxes), 0.01, ptr(thr_dev), ptr(vp), ptr(r), ptr(p), ptr(nn), ptr(t), ptr(k),
                         ptr(count), ptr(scratch), None)
    assert rc == -1 and b"16-byte aligned" in L.h3dgs_last_error() and (r == 7).all()
    rc = L.h3dgs_expand_to_size(N, ptr(nodes), ptr(boxes), 0.01, ptr(vp), 0.0, 0.0, 0.0, ptr(r), ptr(p), ptr(nn), ptr(scratch), None)
    assert rc == -1 and b"16-byte aligned" in L.h3dgs_last_error() and (r == 7).all()
    idx = i32(np.arange(10))
    rc = L.h3dgs_get_interpolation_weights(10, ptr(idx), 0.01, ptr(nodes), ptr(boxes), 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, ptr(t),
                                           ptr(k), None)
    assert rc == -1 and b"16-byte aligned" in L.h3dgs_last_error() and not t.any()


@pytest.mark.parametrize("tau", [6.0, 15.0])
def test_emulated_fused_gather_and_scatter_on_a_general_tree(emu_lib, tau):
    """K1 gathers and lerps rows through render_indices / parent_indices, K9 scatters t*g and (1-t)*g back: here with
    parent rows that four or more cut rows lerp towards and rows that are rendered and lerp partners at once"""
    from oracle import oracle
    from test_emu_kernels_cpu import grad_close, image_close
    cam = synth.make_camera(160, 112)
    h = hg.dense_hierarchy(11, 1500, cam)
    thr = synth.tau_threshold(tau, cam)
    n, ri, pi, ni = oracle.expand_to_size(h["nodes"], h["boxes"], thr, cam.camera_center)
    ts, kids = oracle.get_interpolation_weights(ni, thr, h["nodes"], h["boxes"], cam.camera_center)
    part = (ts > 0) & (ts < 1)
    assert part.any() and (kids[part] > 2).any()
    if tau == 15.0:
        assert np.bincount(pi[part]).max() >= 4 and np.isin(pi[part], ri).any()
    bg = np.array([0.3, 0.2, 0.1], np.float32)
    f = oracle.rasterize_forward(h["means3D"], h["shs"], None, h["opacities"], h["scales"], h["rotations"], None,
                                 cam.world_view_transform, cam.full_proj_transform, cam.camera_center, bg, cam.W, cam.H,
                                 cam.tanfovx, cam.tanfovy, ts=ts, kids=kids, render_indices=ri, parent_indices=pi)
    gcol = synth.l1_grad(f["color"])
    b = oracle.rasterize_backward(f, gcol)
    a, keep = emu_lib.args(cam, bg, h, ts=ts, kids=kids, ridx=ri, pidx=pi)
    fw = emu_lib.forward(a, keep)
    assert np.array_equal(fw["radii"], f["radii"]) and (f["radii"] > 0).mean() > 0.5
    image_close(fw["color"], f["color"])
    g = emu_lib.backward(a, fw, gcol)
    for k in ("means3D", "sh", "opacities", "scales", "rotations", "means2D"):
        grad_close(g[k], b[k], k)

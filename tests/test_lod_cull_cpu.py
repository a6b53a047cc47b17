"""CPU: the view cull of the LOD cut (csrc/lod_cull.cu, and the row mask in hierarchy.cu's cut and lod_budget.cu's
budget), built against the SIMT emulator (tests/emul/).

  * the mask kernel equals the numpy restatement (tests/lod_cull_ref.py) bit for bit on creator-built, general,
    surrounding, single-node and odd-row hierarchies, from the default, yawed, off-centre, far and inside cameras, at
    scale modifiers 1, 0.5 and 3;
  * conservativeness: every row the real preprocess kernel (K1) draws with a positive radius, lerped with its partner
    at t = 0, 1, random and the near-plane crossing, is kept -- on the hierarchies and on edge rows built at the cull's
    decision edges (near plane +- ulps, rect edges +- 1 px at the four borders, needles, partners behind the camera,
    |q| up to 2, zero scales);
  * the masked cut equals the oracle's cut filtered by the mask (same order, same fields);
  * the masked budget equals the budget restatement on the visible counts: threshold, rows and unmet flag;
  * an all-ones mask gives the unmasked cut and budget bit for bit."""
import os
import sys
from unittest import mock

import numpy as np
import pytest

import lod_budget_ref as bref
import lod_cull_ref as ref
from h3dgs import synth

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emul"))

CAM = synth.make_camera(480, 270)
SCENES = dict(ref.scenes(CAM))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """the emulation build of the library's sources plus lod_budget.cu and lod_cull.cu"""
    import build_emu
    from emu_api import Emu
    with mock.patch.object(build_emu, "SOURCES", build_emu.SOURCES + ["lod_budget.cu", "lod_cull.cu"]):
        return Emu(build_emu.build(str(tmp_path_factory.mktemp("h3dgs_emu_lod_cull"))))


def emu_mask(emu, h, cam, smod=1.0):
    from emu_api import aligned, f32, i32, ptr
    R = h["means3D"].shape[0]
    nd, mu, sc, ro = i32(h["nodes"]), f32(h["means3D"]), f32(h["scales"]), f32(h["rotations"])
    view, proj = f32(cam.world_view_transform), f32(cam.full_proj_transform)
    out = aligned(R, np.uint8)
    out[:] = 0xAB                                         # rows of no node keep what they held
    emu.check(emu.L.h3dgs_lod_cull_mask(h["nodes"].shape[0], ptr(nd), ptr(mu), ptr(sc), ptr(ro), smod, ptr(view),
                                        ptr(proj), cam.W, cam.H, cam.tanfovx, cam.tanfovy, ptr(out), None))
    return out.copy()


def emu_cut(emu, nodes, boxes, t, vp, mask=None):
    from emu_api import aligned, f32, i32, ptr
    L = emu.L
    N = nodes.shape[0]
    nd, bx, v = i32(nodes), f32(boxes), f32(vp)
    m = i32(np.zeros(1)) if mask is None else aligned(mask.size, np.uint8)
    if mask is not None:
        m[:] = mask
    R = max(N, int(nodes[:, 3].astype(np.int64).sum() + nodes[:, 4].sum()), 1)     # rows: a node may hold several
    outs = [aligned(4 * R, np.int32) for _ in range(3)] + [aligned(4 * R, np.float32), aligned(4 * R, np.int32)]
    count = aligned(4, np.int32)
    scratch = aligned(L.h3dgs_expand_scratch_bytes(N))
    if mask is None:
        emu.check(L.h3dgs_lod_cut(N, ptr(nd), ptr(bx), float(t), None, ptr(v), *(ptr(o) for o in outs), ptr(count),
                                  ptr(scratch), None))
    else:
        emu.check(L.h3dgs_lod_cut_masked(N, ptr(nd), ptr(bx), float(t), None, ptr(v), ptr(m), *(ptr(o) for o in outs),
                                         ptr(count), ptr(scratch), None))
    n = int(count[0])
    return n, [o[:n].copy() for o in outs]


def emu_budget(emu, nodes, boxes, vp, floor, budget, mask=None):
    from emu_api import aligned, f32, i32, ptr
    L = emu.L
    N = nodes.shape[0]
    nd, bx, v = i32(nodes), f32(boxes), f32(vp)
    thr, info = aligned(4, np.float32, (1,)), aligned(16, np.int32, (4,))
    scratch = aligned(L.h3dgs_lod_budget_scratch_bytes(N))
    scratch[:] = 0xAB
    m = None
    if mask is not None:
        m = aligned(mask.size, np.uint8)
        m[:] = mask
        emu.check(L.h3dgs_lod_budget_masked(N, ptr(nd), ptr(bx), ptr(v), ptr(m), float(floor), None, int(budget), None,
                                            ptr(thr), ptr(info), ptr(scratch), None))
    else:
        emu.check(L.h3dgs_lod_budget(N, ptr(nd), ptr(bx), ptr(v), float(floor), None, int(budget), None, ptr(thr),
                                     ptr(info), ptr(scratch), None))
    return dict(threshold=thr[0], rows=int(info[0]), unmet=int(info[1]), kept=int(info[2]), total=int(info[3]))


def bits(x):
    return int(np.asarray(x, np.float32).view(np.uint32))


@pytest.mark.parametrize("name", list(SCENES))
def test_mask_kernel_equals_the_restatement(emu, name):
    h = SCENES[name]
    seen = set()
    for cname, cam in ref.cameras(h).items():
        for smod in ((1.0, 0.5, 3.0) if cname in ("default", "inside") else (1.0,)):
            got = emu_mask(emu, h, cam, smod)
            want, written = ref.mask(h, cam, smod)
            assert np.array_equal(got[written], want[written]), (name, cname, smod, np.nonzero(got[written] != want[written])[0][:10])
            assert (got[~written] == 0xAB).all()
            seen |= set(int(x) for x in want[written])
    if name in ("creator", "general300", "surround", "odd"):
        assert seen == {0, 1}


def run_k1(emu, h, cam, rows, partner, ts, smod=1.0):
    """K1 (through the emulated forward) on rows lerped with their partners at weights ts -> radii"""
    from emu_api import f32
    import preprocess_ref as pr
    sc = dict(means3D=h["means3D"], scales=h["scales"], rotations=h["rotations"], opacities=h["opacities"],
              shs=h["shs"][:, :1])
    a, keep = emu.args(cam, np.zeros(3, np.float32), sc, sh_degree=0, ts=ts, kids=np.ones(rows.size, np.int32),
                       ridx=rows.astype(np.int32), pidx=partner.astype(np.int32))
    a.scale_modifier = smod
    fw = emu.forward(a, keep)
    return fw["radii"]


def _check_conservative(emu, h, cam, smod=1.0, seed=0):
    rows, partner = ref.pairs(h["nodes"])
    m, _ = ref.mask(h, cam, smod)
    assert np.array_equal(emu_mask(emu, h, cam, smod)[rows], m[rows])
    rng = np.random.default_rng(seed)
    drawn = np.zeros(rows.size, bool)
    for t in ref.t_values(h, rows, partner, cam, rng):
        rad = run_k1(emu, h, cam, rows, partner, t, smod)
        hit = rad > 0
        bad = np.nonzero(hit & (m[rows] == 0))[0]
        assert bad.size == 0, ("a drawn row was culled", rows[bad[:5]], t[bad[:5]], rad[bad[:5]])
        drawn |= hit
    return m[rows].astype(bool), drawn


@pytest.mark.parametrize("name", ["creator", "general300", "surround", "single", "odd"])
def test_every_drawn_row_is_kept(emu, name):
    h = SCENES[name]
    cams = ref.cameras(h, W=160, H=100)
    for cname in ("default", "yaw0", "behind", "offcentre", "far10", "inside"):
        for smod in ((1.0, 3.0) if cname in ("default", "inside") else (1.0,)):
            _check_conservative(emu, h, cams[cname], smod)


def test_edge_rows_are_kept_when_drawn(emu):
    cam = synth.make_camera(160, 100)
    A, sa, qa, B, sb, qb, fam = ref.edge_pairs(cam)
    h = ref.pair_hierarchy(A, sa, qa, B, sb, qb)
    kept, drawn = _check_conservative(emu, h, cam)
    rows, _ = ref.pairs(h["nodes"])
    child = (rows % 2) == 1                                  # the rows whose partner is the other row of the pair
    fam_of = fam[rows[child] // 2]
    for f in set(fam):
        k, d = kept[child][fam_of == f], drawn[child][fam_of == f]
        assert d.any() or f in ("near", "far_side_rev"), f   # every family reaches the drawn side ...
    # ... and the edges reach the culled side: rows just outside the rect edges and behind the near plane are dropped
    assert (~kept[child][fam_of == "rect"]).sum() > 0
    assert (~kept[child][fam_of == "near"]).sum() > 0 and kept[child][fam_of == "near"].sum() > 0
    # edge rows off-centre and at scale_modifier != 1
    for c2, smod in ((synth.make_camera(160, 100, primx=0.35, primy=0.6), 1.0), (cam, 2.5), (cam, 0.4)):
        _check_conservative(emu, h, c2, smod)


@pytest.mark.parametrize("name", ["creator", "general300", "surround", "single", "odd"])
def test_masked_cut_is_the_oracle_cut_filtered(emu, name):
    from oracle import oracle
    h = SCENES[name]
    nodes, boxes = h["nodes"], h["boxes"]
    for cname, cam in list(ref.cameras(h).items())[:6]:
        m, _ = ref.mask(h, cam)
        vp = np.asarray(cam.camera_center, np.float32)
        for tau in (0.0, 3.0, 6.0, 15.0):
            t = np.float32(synth.tau_threshold(tau, cam))
            n0, ri0, pi0, ni0 = oracle.expand_to_size(nodes, boxes, t, vp)[:4]
            ts0, kids0 = oracle.get_interpolation_weights(ni0[:n0], t, nodes, boxes, vp)[:2]
            keep = m[ri0[:n0]] == 1
            n, (ri, pi, ni, ts, kids) = emu_cut(emu, nodes, boxes, t, vp, m)
            assert n == int(keep.sum())
            assert np.array_equal(ri, ri0[:n0][keep]) and np.array_equal(pi, pi0[:n0][keep])
            assert np.array_equal(ni, ni0[:n0][keep])
            assert np.array_equal(ts.view(np.uint32), np.asarray(ts0[:n0], np.float32)[keep].view(np.uint32))
            assert np.array_equal(kids, np.asarray(kids0[:n0])[keep])
            assert n == bref.rows(ref.visible_nodes(nodes, m), bref.hg.node_sizes(boxes, vp), t)


@pytest.mark.parametrize("name", ["creator", "general300", "surround", "odd"])
def test_masked_budget_equals_the_restatement_on_visible_counts(emu, name):
    h = SCENES[name]
    nodes, boxes = h["nodes"], h["boxes"]
    outcomes = set()
    for cname, cam in list(ref.cameras(h).items())[:5]:
        m, _ = ref.mask(h, cam)
        vis = ref.visible_nodes(nodes, m)
        vp = np.asarray(cam.camera_center, np.float32)
        for floor in bref.floors(h, vp, CAM)[:3]:
            tab = bref.table(vis, boxes, vp, floor)
            for B in bref.budgets(vis, tab, floor, limit=10):
                want = bref.select(vis, boxes, vp, floor, B, tab)
                got = emu_budget(emu, nodes, boxes, vp, floor, B, m)
                assert bits(got["threshold"]) == bits(want["threshold"]), (name, cname, floor, B)
                assert [got[k] for k in ("rows", "unmet", "kept", "total")] == \
                    [want[k] for k in ("rows", "unmet", "kept", "total")], (name, cname, floor, B)
                unculled = emu_budget(emu, nodes, boxes, vp, floor, B)
                assert got["threshold"] <= unculled["threshold"]      # never coarser than without the cull
                outcomes.add("floor" if bits(want["threshold"]) == bits(floor) else "unmet" if want["unmet"] else "inner")
    assert outcomes >= {"floor", "inner"}


@pytest.mark.parametrize("name", ["creator", "general300", "odd"])
def test_all_ones_mask_is_the_unmasked_cut_and_budget(emu, name):
    h = SCENES[name]
    nodes, boxes = h["nodes"], h["boxes"]
    ones = np.ones(h["means3D"].shape[0], np.uint8)
    vp = np.asarray(CAM.camera_center, np.float32)
    for tau in (0.0, 6.0):
        t = np.float32(synth.tau_threshold(tau, CAM))
        n0, o0 = emu_cut(emu, nodes, boxes, t, vp)
        n1, o1 = emu_cut(emu, nodes, boxes, t, vp, ones)
        assert n0 == n1 and all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(o0, o1))
    for floor in bref.floors(h, vp, CAM)[:3]:
        tab = bref.table(nodes, boxes, vp, floor)
        for B in bref.budgets(nodes, tab, floor, limit=6):
            a, b = emu_budget(emu, nodes, boxes, vp, floor, B), emu_budget(emu, nodes, boxes, vp, floor, B, ones)
            assert bits(a["threshold"]) == bits(b["threshold"]) and \
                [a[k] for k in ("rows", "unmet", "kept", "total")] == [b[k] for k in ("rows", "unmet", "kept", "total")]


def test_argument_checks(emu):
    from emu_api import aligned, f32, i32, ptr
    L = emu.L
    h = SCENES["general5"]
    nd, mu, sc, ro = i32(h["nodes"]), f32(h["means3D"]), f32(h["scales"]), f32(h["rotations"])
    view, proj = f32(CAM.world_view_transform), f32(CAM.full_proj_transform)
    out = aligned(h["means3D"].shape[0], np.uint8)
    args = [h["nodes"].shape[0], ptr(nd), ptr(mu), ptr(sc), ptr(ro), 1.0, ptr(view), ptr(proj), 480, 270, CAM.tanfovx,
            CAM.tanfovy, ptr(out), None]

    def call(**kw):
        a = list(args)
        for i, val in kw.items():
            a[int(i[1:])] = val
        return L.h3dgs_lod_cull_mask(*a)
    assert call() == 0
    assert call(a0=0) < 0 and b"empty" in L.h3dgs_last_error()
    for i in (1, 2, 3, 4, 6, 7, 12):
        assert call(**{f"a{i}": None}) < 0 and b"NULL" in L.h3dgs_last_error()
    assert call(a8=0) < 0 and call(a11=0.0) < 0

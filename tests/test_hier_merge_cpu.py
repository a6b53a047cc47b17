"""CPU: the hierarchy merger (csrc/hier_merge.cu, emulation build) against the numpy restatement of
tests/hier_merge_ref.py: nodes, sources and copied rows exactly, top boxes the union of their children, top merged rows
within the creator's tolerance; on creator-built chunks, general hierarchies, chunks that own nothing, shared borders,
the outer ring, a hole, trailing unclaimed rows and W = 0 items.  Also the identity merge, structural invariants and
the LOD cut on merged trees, repeatability, argument checks and the command-line merger."""
import contextlib
import os
import sys
from unittest import mock

import numpy as np
import pytest

import hier_build_ref as hb
import hier_general as hg
import hier_merge_ref as ref
from h3dgs import synth

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emul"))

OUT = ("xyz", "shs", "opacities", "log_scales", "rotations", "nodes", "boxes", "source_chunk", "source_row")
F = np.float32


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """the emulation build of the library's sources plus hier_build.cu and hier_merge.cu"""
    import build_emu
    from emu_api import Emu
    with mock.patch.object(build_emu, "SOURCES", build_emu.SOURCES + ["hier_build.cu", "hier_merge.cu"]):
        return Emu(build_emu.build(str(tmp_path_factory.mktemp("h3dgs_emu_hier_merge"))))


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def run(emu, chunks, cells, check=True):
    """the C-ABI on the emulation build -> dict of the nine outputs (+ R), or (rc, outputs, allocation log)"""
    from emu_api import aligned, f32, i32, ptr
    from h3dgs import _lib
    K = len(chunks)
    cat = lambda k, dt: np.ascontiguousarray(np.concatenate([np.asarray(c[k], dt).reshape((c[k].shape[0], -1)) for c in chunks]))
    xyz, shs, op, ls, rot = (f32(cat(k, F)) for k in ("xyz", "shs", "opacities", "log_scales", "rotations"))
    nodes, boxes = i32(cat("nodes", np.int32)), f32(cat("boxes", F))
    noff = np.concatenate([[0], np.cumsum([c["nodes"].shape[0] for c in chunks])]).astype(np.int64)
    roff = np.concatenate([[0], np.cumsum([c["xyz"].shape[0] for c in chunks])]).astype(np.int64)
    cl = np.ascontiguousarray(np.asarray(cells, F).reshape(K, 4))
    scratch = aligned(max(emu.L.h3dgs_merge_hierarchies_scratch_bytes(K, int(noff[-1]), int(roff[-1])), 1))
    bufs, log = {}, []

    def alloc(_u, which, nbytes):
        log.append(which)
        bufs[which] = aligned(max(int(nbytes), 4))
        return bufs[which].ctypes.data
    cb = _lib.ALLOC_FN(alloc)
    counts = np.zeros(3, np.int64)
    rc = emu.L.h3dgs_merge_hierarchies(K, noff.ctypes.data, roff.ctypes.data, cl.ctypes.data, ptr(xyz), ptr(shs), ptr(op),
                                       ptr(ls), ptr(rot), ptr(nodes), ptr(boxes), cb, None, counts.ctypes.data,
                                       ptr(scratch), None)
    if not check:
        return rc, counts, log
    emu.check(rc)
    NO, RO, R = (int(v) for v in counts)
    shapes = dict(xyz=(RO, 3), shs=(RO, 16, 3), opacities=(RO,), log_scales=(RO, 3), rotations=(RO, 4), nodes=(NO, 7),
                  boxes=(NO, 2, 4), source_chunk=(RO,), source_row=(RO,))
    dts = dict(nodes=np.int32, source_chunk=np.int32, source_row=np.int32)
    out = {k: bufs[i].view(dts.get(k, F))[:int(np.prod(shapes[k]))].reshape(shapes[k]).copy() for i, k in enumerate(OUT)}
    out["R"] = R
    return out


def check_against_ref(got, chunks, cells):
    """the comparison every merge goes through (the GPU suite imports it)"""
    r = ref.merge(chunks, cells)
    assert got["R"] == r["R"]
    assert np.array_equal(got["nodes"], r["nodes"])
    assert np.array_equal(got["source_chunk"], r["source_chunk"]) and np.array_equal(got["source_row"], r["source_row"])
    copied = r["source_chunk"] >= 0
    for k in ("xyz", "shs", "opacities", "log_scales", "rotations"):
        assert np.array_equal(bits(got[k][copied]), bits(r[k][copied])), k
    b, rb = got["boxes"], r["boxes"]
    T, top, single = r["T"], r["top_interior"], r["single"]
    other = np.setdiff1d(np.arange(b.shape[0]), top)
    exact = np.setdiff1d(other, single)
    assert np.array_equal(bits(b[exact]), bits(rb[exact]))
    if single.size:
        ulp = np.spacing(np.abs(rb[single][:, :, :3]))
        assert (np.abs(b[single][:, :, :3] - rb[single][:, :, :3]) <= ulp).all()
    nodes = got["nodes"]
    ca, cb = nodes[top, 5], nodes[top, 5] + 1
    assert np.array_equal(b[top, 0, :3], np.minimum(b[ca, 0, :3], b[cb, 0, :3]))
    assert np.array_equal(b[top, 1, :3], np.maximum(b[ca, 1, :3], b[cb, 1, :3]))
    assert np.array_equal(bits(b[top, 0, 3]), bits((b[top, 1, :3] - b[top, 0, :3]).max(1))) and (b[top, 1, 3] == 0).all()
    if top.size == 0:
        return r
    rows = nodes[top, 2]
    allxyz = np.concatenate([c["xyz"] for c in chunks])
    ext = max(float((allxyz.max(0) - allxyz.min(0)).max()), 1e-30)
    rx = r["xyz"][rows]
    assert np.abs(got["xyz"][rows] - rx).max() <= 1e-6 * ext + np.spacing(np.abs(rx)).max()
    cg = hb.cov_of(got["log_scales"][rows], got["rotations"][rows])
    cr = r["top_cov"][top]
    rel = np.linalg.norm(cg - cr, axis=(1, 2)) / np.linalg.norm(cr, axis=(1, 2))
    assert rel.max() < 1e-5, rel.max()
    o, ro = got["opacities"][rows].astype(np.float64), r["opacities"][rows].astype(np.float64)
    assert (np.abs(o - ro) <= 1e-5 * np.abs(ro) + 1e-30).all()
    sh, rsh = got["shs"][rows].astype(np.float64), r["shs"][rows].astype(np.float64)
    assert (np.abs(sh - rsh) <= 1e-5 * (np.abs(rsh).max(axis=(1, 2), keepdims=True) + 1e-30)).all()
    return r


# ---------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------
def creator_chunk(emu_or_fn, cell, P, seed, **kw):
    """a chunk cloud built by the creator -> dict in the merger's input layout"""
    c = ref.chunk_cloud(cell, P, seed, **kw)
    h = emu_or_fn(c)
    return dict(xyz=h["xyz"], shs=h["shs"], opacities=np.asarray(h["opacities"]).reshape(-1), log_scales=h["log_scales"],
                rotations=h["rotations"], nodes=h["nodes"], boxes=h["boxes"])


def _build(emu):
    from test_hier_build_cpu import run as build_run
    return lambda c: build_run(emu, c)


def general_chunk(seed, n_nodes, trailing=0):
    cam = synth.make_camera(320, 180)
    h = hg.general_hierarchy(np.random.default_rng(seed), n_nodes, cam, empty_p=0.1)
    out = dict(xyz=h["means3D"], shs=h["shs"], opacities=h["opacities"][:, 0], log_scales=np.log(h["scales"]).astype(F),
               rotations=h["rotations"], nodes=h["nodes"], boxes=h["boxes"])
    if trailing:
        g = np.random.default_rng(seed + 1)
        sky = hb.cloud(trailing, seed + 2)
        sky["xyz"][:, :2] = g.uniform(-50, 50, (trailing, 2))
        for k in ("xyz", "shs", "opacities", "log_scales", "rotations"):
            out[k] = np.concatenate([out[k], sky[k].reshape((trailing,) + out[k].shape[1:])]).astype(F)
    return out


def general_cells(chunks, nx, ny):
    xy = np.concatenate([c["xyz"][:, :2] for c in chunks])
    lo, hi = xy.min(0), xy.max(0)
    w = (hi - lo) / [nx, ny]
    return np.array([[lo[0] + (i + 0.5) * w[0], lo[1] + (j + 0.5) * w[1], w[0] * 0.8, w[1] * 0.8]
                     for j in range(ny) for i in range(nx)], F)


def tiny_chunk(xy, nodes, seed=77):
    """a hand-written chunk: one row per (x, y), the given node table, every box spanning [-10, 10]^3"""
    c = hb.cloud(len(xy), seed)
    c["xyz"][:, :2] = np.asarray(xy, F)
    nodes = np.asarray(nodes, np.int32)
    boxes = np.zeros((nodes.shape[0], 2, 4), F)
    boxes[:, 0, :3], boxes[:, 1, :3], boxes[:, 0, 3] = -10.0, 10.0, 20.0
    return dict(c, nodes=nodes, boxes=boxes)


def cases(build):
    c = {}
    for K, (nx, ny) in ((1, (1, 1)), (2, (2, 1)), (3, (3, 1)), (4, (2, 2))):
        cells = ref.grid_cells(nx, ny)
        c[f"creator{K}"] = ([creator_chunk(build, cells[k], 300 + 37 * k, 10 * K + k) for k in range(K)], cells)
    gch = [general_chunk(s, 400, trailing=7 * (s % 2)) for s in (1, 2, 3)]
    c["general"] = (gch, general_cells(gch, 3, 1))
    cells = ref.grid_cells(2, 1)
    inside = creator_chunk(build, np.array([-2.0, 0.0, 1.0, 1.0], F), 120, 5, spill=0.0)        # entirely in chunk 0's cell
    c["owns_nothing"] = ([creator_chunk(build, cells[0], 200, 6), creator_chunk(build, cells[1], 200, 7), inside],
                         np.concatenate([cells, [[0.0, 40.0, 4.0, 4.0]]]).astype(F))
    bc = ref.chunk_cloud(cells[0], 256, 8, spill=0.5)
    bc["xyz"][:64, 0] = 0.0                                    # exactly on the shared border x = 0
    bc["xyz"][64:96, 0] = -30.0                                # beyond the outer ring
    b2 = ref.chunk_cloud(cells[1], 256, 9, spill=0.5)
    b2["xyz"][:64, 0] = 0.0
    c["border_and_ring"] = ([_built(build, bc), _built(build, b2)], cells)
    hole = ref.grid_cells(3, 3, skip={(1, 1)})
    c["hole"] = ([creator_chunk(build, hole[k], 150, 40 + k, spill=0.6) for k in range(len(hole))], hole)
    z = [ref.chunk_cloud(cc, 100, 50 + k) for k, cc in enumerate(cells)]
    z[1]["opacities"][:] = 0
    c["zero_weight"] = ([_built(build, x) for x in z], cells)
    # row 0 of chunk 0 is an owned leaf Gaussian of an impure node: a one-Gaussian item made from global row 0
    root = tiny_chunk([[-1.0, 0.0], [1.0, 0.0]], [[0, -1, 0, 2, 0, 0, 0]])
    c["row0_single"] = ([root, creator_chunk(build, cells[1], 200, 60)], cells)
    return c


def _built(build, cloud):
    h = build(cloud)
    return dict(xyz=h["xyz"], shs=h["shs"], opacities=np.asarray(h["opacities"]).reshape(-1), log_scales=h["log_scales"],
                rotations=h["rotations"], nodes=h["nodes"], boxes=h["boxes"])


@pytest.fixture(scope="module")
def CASES(emu):
    return cases(_build(emu))


NAMES = ["creator1", "creator2", "creator3", "creator4", "general", "owns_nothing", "border_and_ring", "hole", "zero_weight",
         "row0_single"]


@pytest.mark.parametrize("name", NAMES)
def test_matches_the_restatement(emu, CASES, name):
    chunks, cells = CASES[name]
    got = run(emu, chunks, cells)
    check_invariants(got, chunks, cells)
    check_against_ref(got, chunks, cells)


def check_invariants(got, chunks, cells):
    """every owned leaf Gaussian exactly once, no unowned one; links consistent, siblings contiguous, boxes nested"""
    owned = set()
    for c, ch in enumerate(chunks):
        nd = ch["nodes"]
        rows = np.concatenate([np.arange(nd[n, 2], nd[n, 2] + nd[n, 3]) for n in range(nd.shape[0])]).astype(np.int64)
        own = ref.owners(ch["xyz"][rows, :2], cells) == c
        owned |= {(c, int(r)) for r in rows[own]}
    nodes = got["nodes"]
    NO, RO = nodes.shape[0], got["xyz"].shape[0]
    leafrows = [(int(got["source_chunk"][nodes[o, 2] + q]), int(got["source_row"][nodes[o, 2] + q]))
                for o in range(NO) for q in range(nodes[o, 3])]
    assert len(leafrows) == len(set(leafrows)) and set(leafrows) == owned
    assert nodes[0, 1] == -1 and (nodes[1:, 1] >= 0).all()
    for o in range(NO):
        s, cc = nodes[o, 5], nodes[o, 6]
        assert (nodes[s:s + cc, 1] == o).all()
        if cc:
            assert (got["boxes"][s:s + cc, 0, :3] >= got["boxes"][o, 0, :3]).all()
            assert (got["boxes"][s:s + cc, 1, :3] <= got["boxes"][o, 1, :3]).all()
    assert np.bincount(nodes[1:, 1], minlength=NO).tolist() == nodes[:, 6].tolist()
    cnt = nodes[:, 3] + nodes[:, 4]
    assert cnt.sum() == RO and np.array_equal(nodes[cnt > 0, 2], (np.cumsum(cnt) - cnt)[cnt > 0])


def test_identity_merge(emu):
    """one chunk whose cell covers everything, rows in node order, node 0 the root: the input minus its trailing rows"""
    ch = general_chunk(11, 300, trailing=0)
    nodes = ch["nodes"].copy()
    cnt = nodes[:, 3] + nodes[:, 4]
    newstart = np.cumsum(cnt) - cnt
    rows = np.concatenate([np.arange(nodes[n, 2], nodes[n, 2] + cnt[n]) for n in range(nodes.shape[0])]).astype(np.int64)
    c = {k: ch[k][rows] for k in ("xyz", "shs", "opacities", "log_scales", "rotations")}
    nodes[:, 2] = np.where(cnt > 0, newstart, np.minimum(newstart, len(rows) - 1))
    c.update(nodes=nodes, boxes=ch["boxes"])
    M = len(rows)
    sky = hb.cloud(9, 3)
    full = {k: np.concatenate([c[k], sky[k].reshape((9,) + c[k].shape[1:]).astype(F)]) for k in ("xyz", "shs", "opacities",
                                                                                               "log_scales", "rotations")}
    full.update(nodes=nodes, boxes=ch["boxes"])
    got = run(emu, [full], [[0.0, 0.0, 1e6, 1e6]])
    assert got["R"] == 1 and np.array_equal(got["nodes"], nodes)
    for k in ("xyz", "shs", "opacities", "log_scales", "rotations"):
        assert np.array_equal(bits(got[k]), bits(c[k][:M])), k
    assert np.array_equal(bits(got["boxes"]), bits(ch["boxes"]))
    assert (got["source_chunk"] == 0).all() and np.array_equal(got["source_row"], np.arange(M))


def test_lod_cut_on_a_merged_hierarchy(emu, CASES):
    chunks, cells = CASES["general"]
    got = run(emu, chunks, cells)
    cam = synth.make_camera(320, 180)
    h = dict(nodes=got["nodes"], boxes=got["boxes"])
    for vname, vp in hg.viewpoints(h, cam).items():
        for tau in (0.0, 3.0, 15.0):
            thr = synth.tau_threshold(tau, cam)
            n, ri, pi, ni = hg.cut(got["nodes"], got["boxes"], thr, vp)
            hg.check_cut_invariant(got["nodes"], got["boxes"], thr, vp, ri, ni)
            if tau == 0.0:                                  # exactly the owned leaf Gaussians
                leaf_rows = np.concatenate([np.arange(s, s + k) for s, k in zip(got["nodes"][:, 2], got["nodes"][:, 3])])
                assert np.array_equal(np.sort(ri), np.sort(leaf_rows)), vname


def test_two_runs_give_identical_bytes(emu, CASES):
    chunks, cells = CASES["creator4"]
    a, b = run(emu, chunks, cells), run(emu, chunks, cells)
    for k in OUT:
        assert a[k].tobytes() == b[k].tobytes(), k


def test_bad_arguments(emu, CASES):
    chunks, cells = CASES["creator2"]
    L = emu.L
    assert L.h3dgs_merge_hierarchies_scratch_bytes(0, 1, 1) == 0 and L.h3dgs_merge_hierarchies_scratch_bytes(1, 1 << 30, 1 << 30) == 0

    def expect_einval(chs, cl, what):
        rc, counts, log = run(emu, chs, cl, check=False)
        assert rc == -1 and log == [] and not counts.any(), what
        return L.h3dgs_last_error().decode()

    def edit(k, fn):
        chs = [dict(c) for c in chunks]
        chs[1] = dict(chs[1])
        chs[1][k] = chs[1][k].copy()
        fn(chs[1][k])
        return chs
    assert "node table" in expect_einval(edit("nodes", lambda a: a.__setitem__((5, 1), 10 ** 6)), cells, "parent out of range")
    assert "node table" in expect_einval(edit("nodes", lambda a: a.__setitem__((3, 1), 4)), cells, "parent disagrees")
    assert "node table" in expect_einval(edit("nodes", lambda a: a.__setitem__((7, 2), a[8, 2])), cells, "row claimed twice")
    # parent cycles whose links are otherwise consistent (each node is its parent's only child), of length 2 and 3,
    # beside a valid root
    two = tiny_chunk(np.zeros((3, 2)), [[0, -1, 0, 1, 0, 0, 0], [0, 2, 1, 1, 0, 2, 1], [0, 1, 2, 1, 0, 1, 1]])
    three = tiny_chunk(np.zeros((4, 2)), [[0, -1, 0, 1, 0, 0, 0], [0, 3, 1, 1, 0, 2, 1], [0, 1, 2, 1, 0, 3, 1],
                                          [0, 2, 3, 1, 0, 1, 1]])
    for cyc in (two, three):
        assert "parent chain" in expect_einval([cyc], np.array([[0.0, 0.0, 4.0, 4.0]], F), "cycle")
        assert "parent chain" in expect_einval([chunks[0], cyc], cells, "cycle in the second chunk")
    for k, row, val in (("xyz", 3, np.nan), ("log_scales", 4, 300.5), ("opacities", 5, -1.0), ("rotations", 6, np.inf)):
        leafrow = int(chunks[1]["nodes"][chunks[1]["nodes"][:, 3] > 0][row, 2])
        assert "leaf Gaussian" in expect_einval(edit(k, lambda a: a.reshape(a.shape[0], -1).__setitem__((leafrow, 0), val)),
                                                cells, k)
    for bad in (0.0, -1.0, np.inf, np.nan):
        cl = cells.copy(); cl[1, 2] = bad
        assert "extent" in expect_einval(chunks, cl, bad)
    # each chunk's Gaussians lie in the other's cell: nothing is kept
    build = _build(emu)
    a, b = (creator_chunk(build, cells[k], 60, 90 + k, spill=0.0) for k in (0, 1))
    assert "owns" in expect_einval([a, b], cells[::-1].copy(), "nothing owned")


# ---------------------------------------------------------------------------------------------------------------
# the Python API and the command-line merger
# ---------------------------------------------------------------------------------------------------------------
def _emu_patches(emu):
    import torch
    from h3dgs import _lib, hier_merge
    from gaussian_hierarchy import merger
    return [mock.patch.object(_lib, "_lib", emu.L), mock.patch.object(hier_merge, "_on_device", lambda t: True),
            mock.patch.object(merger, "_device", lambda: torch.device("cpu")),
            mock.patch.object(torch.cuda, "device", lambda *_a: mock.MagicMock()),
            mock.patch.object(torch.cuda, "current_stream", lambda *a, **k: mock.Mock(cuda_stream=0))]


def _torch_chunks(chunks):
    import torch
    return [{k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in c.items()} for c in chunks]


def test_python_merge_on_the_emulation_build(emu, CASES):
    from h3dgs.hier_merge import merge_hierarchies
    chunks, cells = CASES["creator3"]
    direct = run(emu, chunks, cells)
    with contextlib.ExitStack() as st:
        for p in _emu_patches(emu):
            st.enter_context(p)
        h = merge_hierarchies(_torch_chunks(chunks), cells)
    for k in OUT:
        assert np.array_equal(h[k].numpy().reshape(direct[k].shape).view(np.uint8), direct[k].view(np.uint8)), k
    assert h["opacities"].shape == (direct["xyz"].shape[0], 1) and h["items"] == direct["R"]


def write_chunk_dirs(root, chunks, cells, names, sky=5):
    """a full_train tree: <root>/trained_chunks/<name>/hierarchy.hier_opt (skybox rows after the hierarchy's) and
    <root>/chunks/<name>/{center,extent}.txt as make_chunk.py writes them"""
    from gaussian_hierarchy.hier_io import write_hierarchy
    for c, (ch, cell, name) in enumerate(zip(chunks, cells, names)):
        d = root / "trained_chunks" / name
        d.mkdir(parents=True)
        s = hb.cloud(sky, 70 + c)
        s["xyz"] *= 100.0
        cat = lambda k: np.concatenate([ch[k].reshape(ch[k].shape[0], -1), s[k].reshape(sky, -1)]).astype(F)
        write_hierarchy(str(d / "hierarchy.hier_opt"), cat("xyz"), cat("shs").reshape(-1, 16, 3), cat("opacities"),
                        cat("log_scales"), cat("rotations"), ch["nodes"], ch["boxes"])
        cd = root / "chunks" / name
        cd.mkdir(parents=True)
        center = np.array([cell[0], cell[1], 0.5])
        extent = np.array([cell[2], cell[3], 2e12])
        (cd / "center.txt").write_text(' '.join(map(str, center)))
        (cd / "extent.txt").write_text(' '.join(map(str, extent)))


def test_merger_cli_with_full_train_argv(emu, CASES, tmp_path):
    from gaussian_hierarchy import merger
    from gaussian_hierarchy._C import load_hierarchy
    chunks, cells = CASES["creator2"]
    names = ["0_0", "1_0"]
    write_chunk_dirs(tmp_path, chunks, cells, names)
    out = tmp_path / "out" / "merged.hier"
    with contextlib.ExitStack() as st:
        for p in _emu_patches(emu):
            st.enter_context(p)
        assert merger.main([str(tmp_path / "trained_chunks"), "0", str(tmp_path / "chunks"), str(out)] + names) == 0
        want = run(emu, chunks, cells)
        assert merger.main([str(tmp_path / "trained_chunks"), "x", str(tmp_path / "chunks"), str(out)] + names) == 2
        assert merger.main([str(tmp_path / "trained_chunks"), "0", str(tmp_path / "chunks"), str(out), "0_0", "9_9"]) == 1
        assert merger.main(["only", "three", "args"]) == 2
    xyz, shs, opac, ls, rots, nodes, boxes = load_hierarchy(str(out))
    assert np.array_equal(nodes.numpy(), want["nodes"]) and np.array_equal(bits(boxes.numpy()), bits(want["boxes"]))
    for k, v in (("xyz", xyz), ("shs", shs), ("log_scales", ls), ("rotations", rots)):
        assert np.array_equal(bits(v.numpy()), bits(want[k])), k
    assert np.array_equal(bits(opac.numpy()[:, 0]), bits(want["opacities"]))


def test_read_cell_parses_make_chunk_text(tmp_path):
    from h3dgs.hier_merge import read_cell
    (tmp_path / "c.txt").write_text(' '.join(map(str, np.array([0.1, -2.5, 3.0]))))
    (tmp_path / "e.txt").write_text(' '.join(map(str, np.array([50.0, 49.99999, 2e12]))))
    got = read_cell(str(tmp_path / "c.txt"), str(tmp_path / "e.txt"))
    assert got.dtype == np.float32 and np.array_equal(got, np.array([0.1, -2.5, 50.0, 49.99999], np.float32))

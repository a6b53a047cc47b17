"""GPU: the edges of the SH backward's own-row stores in scatter mode with float4 rows (3 M a multiple of 4):
sh_backward_rows_kernel (a warp takes 32 rendered rows; an own row is stored when sh_row_count_kernel counted one
writer, else reduced; a run of consecutive siblings reduces each parent piece once) and the per-device row-count buffer
of csrc/api.cu (never freed, replaced by a larger one outside a capture only; a capture that finds it too small gets
none and its graph reduces every row).  A store is right only if the count is: a count of 1 on a row with two writers
overwrites the other writer's reduction, which no image or loss comparison sees.  So every case here is checked per
full-size row:
  - every gradient within chain_ref's per-element float64 budget (dL/dSH and dL/dmeans3D with its view-direction term
    included), through test_gpu_scatter_edges' reference of the scatter;
  - every row that exactly one visible rendered row writes (as its own row, never as a lerped parent) bit-identical
    in dL/dSH and dL/dmeans3D between the storing schedule (one call) and the reducing one (debug);
  - SH coefficients past the active degree, and rows no visible rendered row reaches, +0.0 bit for bit.
Scenes: `run_scene`, which places sibling runs at chosen lanes and lengths (runs starting at lanes 0, 1, 30 and 31,
runs of 32, 33, 64, 65 and 129 rows across warp and CTA boundaries, runs broken by a culled row or a t = 1 row and
resumed with the same parent, parent_indices = -1 with t < 1, own rows that are another warp's lerped parent, own rows
referenced as a parent with t = 1, own rows with t = 0, P a multiple of neither 32 nor 128), and
test_gpu_scatter_edges.cut_scene; every float4 layout (deg, M) on both; row blocks of the one-call schedule whose
edges cut a warp and a sibling run; and the row-count buffer's states -- a capture that finds it too small, a graph
captured before the buffer was replaced and replayed after, a smaller call after a larger one -- in a fresh process,
so that the library's per-device state is known.  The `case_*` functions and the eager buffer states also run on the
emulation build (test_sh_rows_edges_cpu.py)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from chain_ref import compare, gather_fp32, general_camera, random_accum, random_rows
from test_gpu_chain_edges import TRANS, W, H, chain_ref_for, place
import test_gpu_scatter_edges as se
from test_gpu_sh_backward_rows import writers

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FULL = se.FULL
# every layout the float4 kernel takes: 3 M % 4 == 0 and (deg + 1)^2 <= M
FLOAT4_LAYOUTS = [(d, M) for M in (4, 8, 12, 16) for d in range(4) if (d + 1) ** 2 <= M]
BLOCK_EDGES = (37, 150, 151)                       # row-block edges inside a warp and inside a sibling run of run_scene


# ---- the run-geometry scene ------------------------------------------------------------------------------------------
FILL = ("plain", "uniq", "self", "self0", "uniq0", "plain_self")


def run_layout():
    """the rendered rows in order: dicts with `kind` and, for siblings, the run's `key`.  Kinds: sib (lerped with the
    run's parent), back (a sibling behind the camera: culled), t1 (a sibling with t = 1: not lerped), plain (t = 1, a
    parent nothing else reaches), uniq (its own parent), uniq0 (its own parent, t = 0), self (parent_indices = -1,
    t < 1), self0 (parent_indices = -1, t = 0), plain_self (parent_indices = -1, t = 1), xref (lerped with another
    rendered row's node row `tgt`), xref1 (parent is another rendered row's node row, t = 1)"""
    L, nruns = [], [0]

    def fill(n):
        for _ in range(n):
            L.append(dict(kind=FILL[len(L) % len(FILL)]))

    def fill_to(lane):
        fill((lane - len(L)) % 32)

    def run(n, back=(), one=()):
        key = nruns[0]
        nruns[0] += 1
        for j in range(n):
            L.append(dict(kind="back" if j in back else "t1" if j in one else "sib", key=key))

    run(32)                    # [0, 32): lanes 0 .. 31 of warp 0
    fill(1)
    run(64)                    # [33, 97): from lane 1 across warps 1 | 2; row 37 (a block edge) inside
    fill_to(30)
    run(65)                    # [126, 191): from lane 30 across the CTA boundary at 128; rows 150, 151 inside
    fill_to(31)                # (already there)
    run(33)                    # [191, 224): from lane 31
    run(129)                   # [224, 353): from lane 0, across the CTA boundary at 256
    fill(5)
    run(11, back=(5,))         # broken by a culled row, resumed with the same parent
    fill(3)
    run(9, one=(4,))           # broken by a t = 1 row, resumed
    fill_to(30)
    run(2)                     # lanes 30, 31
    fill_to(31)
    run(3)                     # from lane 31 into the next warp
    fill_to(29)
    run(5, one=(2,))           # the t = 1 row at lane 31, resumed in the next warp
    fill_to(30)
    run(5, back=(1,))          # the culled row at lane 31, resumed in the next warp
    tail = len(L)
    fill(611 - len(L))         # P = 611: a multiple of neither 32 nor 128
    # own rows that are also lerped parents: early rows take own rows of late CTAs and late rows take early ones (their
    # reductions and the own row's writer run in different warps and CTAs), the last pair within a warp; own rows that
    # are a parent with t = 1 (one writer: stored)
    early = [i for i in range(97, 126) if L[i]["kind"] in FILL]
    for i, tgt in zip(early[::3], (300, 340, 380, 565, 575, 590, 600, 605, 610)):
        L[i] = dict(kind="xref", tgt=tgt)
    late = [i for i in range(tail, 611) if L[i]["kind"] in FILL and i not in (565, 575, 590, 600, 605, 610)]
    for i, tgt in zip(late[::4], (5, 20, 31, 40, 127, 128, 150, 500)):
        L[i] = dict(kind="xref", tgt=tgt)
    for i, tgt in zip(early[1::3], (60, 230, 270)):
        L[i] = dict(kind="xref1", tgt=tgt)
    return L


def run_scene(deg, M, seed):
    """run_layout's rows as a cut over N source rows: rendered rows [0, P) take distinct node rows ridx (a permutation
    of [0, P)); each run one parent row at the mean of its visible siblings, each uniq / plain row a parent row of its
    own; the last 30 source rows are in no cut.  -> cam, sc, info (row sets by kind)"""
    rng = np.random.default_rng(seed)
    cam = general_camera(W, H, TRANS[10])
    L = run_layout()
    P = len(L)
    nruns = 1 + max(r["key"] for r in L if "key" in r)
    own_par = [i for i, r in enumerate(L) if r["kind"] in ("plain", "uniq", "uniq0")]
    N = P + nruns + len(own_par) + 30
    z = rng.uniform(3.0, 10.0, N)
    s, q, o, sh = random_rows(rng, N, M)
    s = (s / s.mean(1, keepdims=True) * 0.02 * z[:, None]).astype(np.float32)
    means = place(cam, rng.uniform(-0.8, 0.8, N) * cam.tanfovx, rng.uniform(-0.8, 0.8, N) * cam.tanfovy, z)
    ridx = rng.permutation(P).astype(np.int32)
    pidx = np.full(P, -1, np.int32)
    ts = rng.uniform(0.05, 0.95, P).astype(np.float32)
    kind = np.array([r["kind"] for r in L])
    sib = np.isin(kind, ("sib", "back", "t1"))
    key = np.array([r.get("key", -1) for r in L])
    pidx[sib] = P + key[sib]
    pidx[own_par] = P + nruns + np.arange(len(own_par))
    for i, r in enumerate(L):
        if "tgt" in r:
            pidx[i] = ridx[r["tgt"]]
    # t at the edges among the siblings: 0 (the own row gets +0), 2^-24 and 1 - 2^-24 (u = 2^-24: still lerped)
    edges = np.flatnonzero(kind == "sib")[::7]
    ts[edges] = np.resize(np.array([0.0, 2.0 ** -24, 1 - 2.0 ** -24], np.float32), edges.size)
    ts[np.isin(kind, ("plain", "plain_self", "t1", "xref1"))] = 1.0
    ts[np.isin(kind, ("self0", "uniq0"))] = 0.0
    ts[kind == "back"] = np.float32(0.95)
    back = np.flatnonzero(kind == "back")
    means[ridx[back]] = place(cam, [0.0] * back.size, [0.0] * back.size, np.full(back.size, -3.0))
    for k in range(nruns):
        kids = np.flatnonzero((key == k) & (kind != "back"))
        means[P + k] = means[ridx[kids]].mean(0)
    means[pidx[own_par]] = means[ridx[own_par]] + rng.uniform(-0.05, 0.05, (len(own_par), 3)).astype(np.float32)
    sc = dict(means3D=means, scales=s, rotations=q, opacities=o, shs=sh, ridx=ridx, pidx=pidx, ts=ts,
              kids=np.ones(P, np.int32))
    info = {k: np.flatnonzero(kind == k) for k in set(kind)}
    info["unused"] = np.arange(N - 30, N)
    return cam, sc, info


def sibling_runs(sc, radii):
    """the runs as the kernel sees them in a whole-frame call: consecutive visible lerped rows with one parent ->
    (per-row parent or -1, [(first row, length)])"""
    g = gather_fp32(sc["means3D"], None, None, None, sc["ridx"], sc["pidx"], sc["ts"])
    sp = np.where((np.asarray(radii) > 0) & g["lerp"], g["p"], -1)
    runs, i = [], 0
    while i < sp.size:
        j = i + 1
        while j < sp.size and sp[j] == sp[i]:
            j += 1
        if sp[i] >= 0:
            runs.append((i, j - i))
        i = j
    return sp, runs


def check_geometry(name, sc, radii):
    """every situation run_scene is built for occurs in the emitted arrays with the forward's visibility"""
    P = len(sc["ridx"])
    vis = np.asarray(radii) > 0
    g = gather_fp32(sc["means3D"], None, None, None, sc["ridx"], sc["pidx"], sc["ts"])
    sp, runs = sibling_runs(sc, radii)
    sib = [(i, n) for i, n in runs if n >= 2]
    assert {0, 1, 30, 31} <= {i % 32 for i, _ in sib}, (name, "run starts", sorted({i % 32 for i, _ in sib}))
    assert {32, 33, 64, 65, 129} <= {n for _, n in sib}, (name, "run lengths", sorted({n for _, n in sib}))
    assert any(i // 32 != (i + n - 1) // 32 for i, n in sib) and any(i // 128 != (i + n - 1) // 128 for i, n in sib)
    assert any(i % 32 + n == 32 for i, n in sib), name                              # a run that ends at lane 31
    pidx = np.asarray(sc["pidx"])
    mid = np.arange(1, P - 1)
    resumed = (sp[mid - 1] >= 0) & (sp[mid - 1] == sp[mid + 1]) & (pidx[mid] == sp[mid - 1])
    assert (resumed & ~vis[mid] & g["lerp"][mid]).any(), (name, "a run broken by a culled row and resumed")
    assert (resumed & vis[mid] & (g["t"][mid] == 1)).any(), (name, "a run broken by a t = 1 row and resumed")
    selfp = vis & g["lerp"] & (pidx < 0)
    assert selfp.sum() >= 10 and (selfp & (g["t"] == 0)).any(), name              # parent_indices = -1, t < 1 (and 0)
    n, both = writers(sc, radii)
    assert (n[g["c"][selfp]] >= 2).all(), name                                     # own row and parent: never stored
    row_of = {int(c): i for i, c in enumerate(g["c"]) if vis[i]}
    lerped = np.flatnonzero(vis & g["lerp"] & (pidx >= 0))
    pairs = [(i, row_of[int(g["p"][i])]) for i in lerped if int(g["p"][i]) in row_of]   # (row, whose own row it lerps)
    assert sum(i // 128 != j // 128 for i, j in pairs) >= 10 and any(i // 32 == j // 32 for i, j in pairs), name
    t1ref = vis & (g["t"] == 1) & (pidx >= 0) & np.isin(pidx, g["c"][vis])
    assert (t1ref & (n[np.maximum(pidx, 0)] == 1)).sum() >= 3, (name, "a single-writer own row referenced with t = 1")
    stored0 = vis & g["lerp"] & (g["t"] == 0) & (pidx >= 0) & (n[g["c"]] == 1)
    assert stored0.sum() >= 5, (name, "stored own rows with t = 0")
    assert P % 32 and P % 128 and both.size >= 10


# ---- running and checking one backward -------------------------------------------------------------------------------
def upload(cam, sc):
    import torch
    from test_gpu_chain_edges import _t
    f = lambda a: _t(np.asarray(a, np.float32))
    dv = {k: f(sc[k]) for k in FULL + ("ts",)}
    dv.update(ridx=_t(sc["ridx"]), pidx=_t(sc["pidx"]), kids=_t(sc["kids"]), bg=f(np.zeros(3)),
              vm=f(cam.world_view_transform), pm=f(cam.full_proj_transform), cp=f(cam.camera_center))
    assert all(v.data_ptr() % 16 == 0 for v in dv.values() if isinstance(v, torch.Tensor))
    return dv


def forward(cam, dv, deg):
    """-> (the forward's tuple, radii, K1's kbits per rendered row)"""
    from diff_gaussian_rasterization import _C
    fwd = _C.rasterize_gaussians(dv["bg"], dv["means3D"], None, dv["opacities"], dv["scales"], dv["rotations"], 1.0,
                                 None, dv["vm"], dv["pm"], cam.tanfovx, cam.tanfovy, H, W, dv["shs"], deg, dv["cp"],
                                 False, False, dv["ridx"], dv["pidx"], dv["ts"], dv["kids"], False)
    n, _c, radii, gb, bb, ib, _ = fwd
    st = _C.state_view(radii.numel(), W, H, n, gb, bb, ib)
    return fwd, radii.cpu().numpy(), st["records"].cpu().numpy()[:, 7].copy().view(np.uint32)


def call(cam, dv, deg, fwd, phases, gcol=None, scratch=None, debug=False, grad_rows=(0, 0)):
    """one h3dgs_rasterize_backward through _C (no host synchronisation: capturable) -> the gradient tensors by name"""
    from diff_gaussian_rasterization import _C
    n, _c, radii, gb, bb, ib, _ = fwd
    g = _C.rasterize_gaussians_backward(dv["bg"], dv["means3D"], radii, None, dv["opacities"], dv["scales"],
                                        dv["rotations"], 1.0, None, dv["vm"], dv["pm"], cam.tanfovx, cam.tanfovy, gcol,
                                        None, dv["shs"], deg, dv["cp"], gb, n, bb, ib, debug, dv["ridx"], dv["pidx"],
                                        dv["ts"], dv["kids"], False, H, W, phases=phases, scratch=scratch,
                                        grad_rows=grad_rows)
    names = ("means2D", "colors", "opacities", "means3D", "cov3D", "shs", "scales", "rotations")
    return {k: v for k, v in zip(names, g) if v is not None and v.numel()}


def new_scratch(P, accum=None):
    import torch
    from h3dgs import _lib
    s = torch.zeros((_lib.lib().h3dgs_backward_scratch_bytes(P),), dtype=torch.uint8, device="cuda")
    if accum is not None:
        s.view(torch.float32)[: P * 10] = torch.tensor(np.asarray(accum, np.float32).reshape(-1), device="cuda")
    return s


def host(out, scratch, P):
    import torch
    return ({k: v.cpu().numpy().copy() for k, v in out.items()},
            scratch.view(torch.float32)[: P * 10].view(P, 10).cpu().numpy().copy())


def backward(cam, dv, deg, fwd, phases, gcol=None, accum=None, debug=False, grad_rows=(0, 0)):
    """phases 3: the replay from dL/dcolor `gcol` and the chain rule in one call; phases 2: the chain rule on the sums
    `accum` -> (gradients, the [P][10] sums the chain rule read)"""
    from test_gpu_chain_edges import _t
    P = fwd[2].numel()
    scratch = new_scratch(P, accum)
    out = call(cam, dv, deg, fwd, phases, None if gcol is None else _t(gcol), scratch, debug, grad_rows)
    return host(out, scratch, P)


def check_rows(name, cam, sc, deg, got, accum, radii, kb, src=None):
    """every element of every gradient within chain_ref's budget, +0.0 where the budget and the reference are 0, on
    rows no visible rendered row reaches and on coefficients past the degree.  src: `sc` sits at these rows of the
    full-size gradients, and every other row must be +0.0 -> chain_ref's reference"""
    ref = chain_ref_for(cam, sc, accum, deg, False, 1.0, radii, kb)[0]
    if src is not None:
        other = np.ones(len(got["means3D"]), bool)
        other[src] = False
        for k in FULL:
            assert not got[k][other].view(np.uint32).any(), (name, k, "a row outside the cut is not +0.0")
        got = {k: (v[src] if k in FULL else v) for k, v in got.items()}
    assert set(got) == set(ref), (name, sorted(got), sorted(ref))
    for k, (r, tol, _) in ref.items():
        assert np.isfinite(got[k]).all(), (name, k, "non-finite gradient")
        w, _n = compare(got[k], r, tol)
        if not w <= 1.0:
            bad = np.argwhere(np.abs(got[k].reshape(r.shape) - r) > tol)[:5]
            raise AssertionError((name, k, w, [(tuple(b), float(got[k].reshape(r.shape)[tuple(b)]), float(r[tuple(b)]),
                                                float(tol[tuple(b)])) for b in bad]))
    se.exact_zeros(name, got, ref)
    N = len(sc["means3D"])
    rows, _g = se.reached(sc, radii)
    dead = np.setdiff1d(np.arange(N), rows)
    for k in FULL:
        assert not got[k][dead].view(np.uint32).any(), (name, k, "a row no visible rendered row reaches is not +0.0")
    beyond = got["shs"].reshape(N, -1, 3)[:, (deg + 1) ** 2:]
    assert not beyond.view(np.uint32).any(), (name, "coefficients past the degree are not +0.0")
    se.summary(name, ref, got, rows.size, dead.size)
    return ref


def same_single_writer_rows(name, sc, radii, a, b, src=None):
    """rows exactly one visible rendered row writes: bit-identical dL/dSH and dL/dmeans3D in `a` and `b` (a stored row
    is what one reduction into the zero line gives; dL/dmeans3D takes two commuting terms) -> (writers, those rows)"""
    n, _both = writers(sc, radii)
    one = np.flatnonzero(n == 1)
    for k in ("shs", "means3D"):
        x, y = (a[k], b[k]) if src is None else (a[k][src], b[k][src])
        x, y = x.reshape(n.size, -1)[one], y.reshape(n.size, -1)[one]
        bad = np.flatnonzero((x.view(np.uint32) != y.view(np.uint32)).any(1))
        assert bad.size == 0, (name, k, "single-writer rows differ: stores vs reductions", one[bad][:5].tolist())
    return n, one


def frame(name, cam, sc, deg, dv, fwd, radii, kb, seed, src=None):
    """the one-call backward (phases 3: zero-fill, row counts, replay, stores) and the debug backward (reductions only)
    on the one call's sums, each per row against chain_ref, and the single-writer rows of the two bit for bit"""
    gcol = (np.random.default_rng(seed).standard_normal((3, H, W)) / (H * W)).astype(np.float32)
    one, accum = backward(cam, dv, deg, fwd, 3, gcol=gcol)
    vis = radii > 0
    assert (np.abs(accum[vis]).sum(1) > 0).mean() > 0.5, name                   # the replay reached the visible rows
    red, _ = backward(cam, dv, deg, fwd, 2, accum=accum, debug=True)
    check_rows(name + " (one call)", cam, sc, deg, one, accum, radii, kb, src)
    check_rows(name + " (debug: reductions only)", cam, sc, deg, red, accum, radii, kb, src)
    n, single = same_single_writer_rows(name, sc, radii, one, red, src)
    shs = one["shs"] if src is None else one["shs"][src]
    assert single.size > 50 and (n > 2).any() and shs.reshape(n.size, -1)[single].any(), (name, single.size)
    return one, accum


# ---- families --------------------------------------------------------------------------------------------------------
def case_layout(deg, M, scene="runs", seed=None):
    """one float4 layout on run_scene or cut_scene: the one-call and debug schedules per full-size row"""
    seed = seed if seed is not None else 1000 + 10 * deg + M
    name = f"sh rows {scene} deg={deg} M={M}"
    cam, sc, info = run_scene(deg, M, seed) if scene == "runs" else se.cut_scene(deg, M, seed)
    dv = upload(cam, sc)
    fwd, radii, kb = forward(cam, dv, deg)
    assert (radii > 0).mean() >= 0.8, (name, (radii > 0).mean())
    if scene == "runs":
        check_geometry(name, sc, radii)
        assert (radii[info["back"]] == 0).all()
    else:
        assert (radii[info["back"]] == 0).all() and any((radii[kids] > 0).sum() >= 33 for _p, kids in info["fans"])
    frame(name, cam, sc, deg, dv, fwd, radii, kb, seed)


def case_row_blocks(deg, M, seed=None):
    """grad_rows = [a, b) with edges at 37, 150, 151 (inside a warp and inside a sibling run): the counts are over all
    rows, the kernels run over the block.  Each block, in its own zero-filled outputs, equals the reference of its own
    rows (+0.0 on every row none of them reaches), its single-writer rows are bit-identical to the debug schedule's,
    and the sum over the blocks equals the whole frame's reference.  The chain rule runs on one set of sums (phases 2)
    so that the blocks and the whole frame share them"""
    seed = seed if seed is not None else 2000 + 10 * deg + M
    cam, sc, info = run_scene(deg, M, seed)
    dv = upload(cam, sc)
    fwd, radii, kb = forward(cam, dv, deg)
    P = radii.size
    sp, _runs = sibling_runs(sc, radii)
    for a in BLOCK_EDGES:
        assert a % 32 and sp[a - 1] >= 0 and sp[a - 1] == sp[a], (a, "a block edge inside a warp and a sibling run")
    accum = random_accum(np.random.default_rng(seed), P)
    whole, _ = backward(cam, dv, deg, fwd, 2, accum=accum)
    ref_all = check_rows(f"whole frame deg={deg} M={M}", cam, sc, deg, whole, accum, radii, kb)
    total = {k: np.zeros(v.shape) for k, v in whole.items()}
    bounds = (0,) + BLOCK_EDGES + (P,)
    for a, b in zip(bounds[:-1], bounds[1:]):
        name = f"row block [{a}, {b}) deg={deg} M={M}"
        mine = np.zeros_like(radii)
        mine[a:b] = radii[a:b]
        blk, _ = backward(cam, dv, deg, fwd, 2, accum=accum, grad_rows=(a, b))
        red, _ = backward(cam, dv, deg, fwd, 2, accum=accum, grad_rows=(a, b), debug=True)
        check_rows(name, cam, sc, deg, blk, accum, mine, kb)
        check_rows(name + " (debug)", cam, sc, deg, red, accum, mine, kb)
        same_single_writer_rows(name, sc, mine, blk, red)
        for k in total:
            total[k] += blk[k].astype(np.float64)
    for k, (r, tol, _) in ref_all.items():
        w, _n = compare(total[k], r, tol)
        assert w <= 1.0, ("sum of the row blocks", deg, M, k, w)


# ---- the row-count buffer's states (one fresh process) ---------------------------------------------------------------
class _MemsetParams(C.Structure):                  # CUDA_MEMSET_NODE_PARAMS (cuda.h)
    _fields_ = [("dst", C.c_uint64), ("pitch", C.c_size_t), ("value", C.c_uint), ("elementSize", C.c_uint),
                ("width", C.c_size_t), ("height", C.c_size_t)]


def graph_memsets(graph):
    """(destination, bytes) of every memset node of a graph captured with torch.cuda.CUDAGraph(keep_graph=True)"""
    cu = C.CDLL("libcuda.so.1")
    h = C.c_void_p(graph.raw_cuda_graph())
    n = C.c_size_t(0)
    assert cu.cuGraphGetNodes(h, None, C.byref(n)) == 0
    nodes = (C.c_void_p * n.value)()
    assert cu.cuGraphGetNodes(h, nodes, C.byref(n)) == 0
    out = []
    for node in nodes:
        ty = C.c_int(-1)
        assert cu.cuGraphNodeGetType(C.c_void_p(node), C.byref(ty)) == 0
        if ty.value == 2:                                                       # CU_GRAPH_NODE_TYPE_MEMSET
            p = _MemsetParams()
            assert cu.cuGraphMemsetNodeGetParams(C.c_void_p(node), C.byref(p)) == 0
            out.append((int(p.dst), int(p.elementSize) * int(p.width) * int(p.height)))
    return out


def count_memsets(graph, tensors):
    """the graph's memsets of memory none of `tensors` holds: the zeroing of the row-count buffer, if it has one"""
    spans = [(t.data_ptr(), t.data_ptr() + t.numel() * t.element_size()) for t in tensors]
    ms = graph_memsets(graph)
    assert any(d == tensors[0].data_ptr() for d, _b in ms), "the graph's zero-fill of dL/dmeans3D was not found"
    return [(d, b) for d, b in ms if not any(lo <= d < hi for lo, hi in spans)]


def embed(small, N, rng):
    """the cut `small` with its source rows spread over N source rows (the others 0.25 and in no cut) -> (sc, rows)"""
    Ns = len(small["means3D"])
    src = np.sort(rng.choice(N, Ns, replace=False))
    big = {}
    for k in FULL:
        a = np.full((N,) + small[k].shape[1:], 0.25, np.float32)
        a[src] = small[k]
        big[k] = a
    big.update(ridx=src[small["ridx"]].astype(np.int32), ts=small["ts"], kids=small["kids"],
               pidx=np.where(small["pidx"] < 0, -1, src[np.maximum(small["pidx"], 0)]).astype(np.int32))
    return big, src


def buffer_states(emu_so=None):
    """run in a fresh process (the row-count buffer starts unallocated); emu_so: on the emulation build, the eager
    states only"""
    if emu_so:
        sys.path.insert(0, os.path.join(HERE, "emul"))
        from fake_device import cpu_as_device, cuda_names_mean_cpu
        with cpu_as_device(emu_so), cuda_names_mean_cpu():
            _buffer_states(False)
    else:
        _buffer_states(True)


def _buffer_states(capture, deg=3, M=16, seed=91):
    import torch
    cam, small, _info = run_scene(deg, M, seed)
    Ns = len(small["means3D"])
    N1, N2, N3 = (300_000, 200_000, 400_000) if capture else (6_000, 4_000, 8_000)
    rng = np.random.default_rng(seed)
    scenes = {N: embed(small, N, rng) for N in (N1, N2, N3)}
    dv_s = upload(cam, small)
    fwd_s, radii, kb = forward(cam, dv_s, deg)
    check_geometry("buffer states", small, radii)
    n_w, _both = writers(small, radii)
    frame(f"warm-up, N={Ns}", cam, small, deg, dv_s, fwd_s, radii, kb, seed)   # the buffer now holds Ns rows
    print(f"state: eager at N={Ns}")
    run = {}
    for N, (sc, src) in scenes.items():
        dv = upload(cam, sc)
        fwd, r, _kb = forward(cam, dv, deg)
        assert np.array_equal(r, radii)
        run[N] = (sc, src, dv, fwd)

    def replay(name, graph, outs, scratch, N):
        graph.replay()
        got, accum = host(outs, scratch, radii.size)
        _sc, src, dv, fwd = run[N]
        check_rows(name, cam, small, deg, got, accum, radii, kb, src)
        red, _ = backward(cam, dv, deg, fwd, 2, accum=accum, debug=True)
        same_single_writer_rows(name, small, radii, got, red, src)
        return got

    def capture_at(N, phases, gcol=None, scratch=None):
        _sc, _src, dv, fwd = run[N]
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph(keep_graph=True)
        with torch.cuda.graph(g):
            outs = call(cam, dv, deg, fwd, phases, gcol, scratch)
        g.instantiate()
        counts = count_memsets(g, [outs[k] for k in FULL] + [scratch])
        return g, outs, counts

    if capture:
        from test_gpu_chain_edges import _t
        # (a) the one-call backward (replay included) captured at N1 > Ns: the buffer is too small, the graph zeroes no
        # count buffer and reduces every row
        gcol = _t((np.random.default_rng(seed + 1).standard_normal((3, H, W)) / (H * W)).astype(np.float32))
        scr_a = new_scratch(radii.size)
        g_a, outs_a, counts = capture_at(N1, 3, gcol, scr_a)
        assert counts == [], ("a capture that found the buffer too small zeroes a count buffer", counts)
        for k in range(2):
            replay(f"(a) replay {k} of the capture at N={N1} > {Ns}", g_a, outs_a, scr_a, N1)
        print(f"state a: captured at N={N1} with the buffer at {Ns} rows: no counts, replays checked")
        # (b) eager at N1 (the buffer is replaced), a capture at N2 < N1 (it is reused), eager at N3 > N1 (replaced
        # again), the N2 graph replayed.  The chain rule on fixed sums (phases 2), so the replays compare bit for bit
        _sc, src1, dv1, fwd1 = run[N1]
        frame(f"(b) eager at N={N1}", cam, small, deg, dv1, fwd1, radii, kb, seed + 2, src1)
        accum_b = random_accum(np.random.default_rng(seed + 3), radii.size)
        scr_b = new_scratch(radii.size, accum_b)
        g_b, outs_b, counts_b = capture_at(N2, 2, None, scr_b)
        assert len(counts_b) == 1 and counts_b[0][1] == N2 * 4, ("the N2 capture counts into the N1 buffer", counts_b)
        before = replay(f"(b) the N={N2} graph before the buffer is replaced", g_b, outs_b, scr_b, N2)
        _sc, src3, dv3, fwd3 = run[N3]
        frame(f"(b) eager at N={N3}", cam, small, deg, dv3, fwd3, radii, kb, seed + 4, src3)
        g_c, _outs_c, counts_c = capture_at(N2, 2, None, new_scratch(radii.size, accum_b))
        assert len(counts_c) == 1 and counts_c[0][0] != counts_b[0][0], ("the buffer was replaced", counts_b, counts_c)
        del g_c
        after = replay(f"(b) the N={N2} graph after the buffer is replaced", g_b, outs_b, scr_b, N2)
        # rows whose sum does not depend on the order of the atomics: one writer (dL/dmeans3D: two terms), two for
        # dL/dSH
        src2 = run[N2][1]
        for k in FULL:
            keep = n_w <= (2 if k == "shs" else 1)
            x, y = before[k][src2][keep], after[k][src2][keep]
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), ("(b) replay after the reallocation", k)
        assert np.array_equal(before["means2D"].view(np.uint32), after["means2D"].view(np.uint32))
        print(f"state b: graph at N={N2} counted into the N={N1} buffer, replayed bit-identically after the N={N3} one")
    else:
        _sc, src1, dv1, fwd1 = run[N1]
        frame(f"eager at N={N1}", cam, small, deg, dv1, fwd1, radii, kb, seed + 2, src1)
    # (c) an eager call at a smaller N after larger ones: counts zeroed over [0, N) only
    _sc, src2, dv2, fwd2 = run[N2]
    frame(f"(c) eager at N={N2} after N={N3 if capture else N1}", cam, small, deg, dv2, fwd2, radii, kb, seed + 5, src2)
    frame(f"(c) eager at N={Ns}", cam, small, deg, dv_s, fwd_s, radii, kb, seed + 6)
    print("state c: smaller eager calls after larger ones")


_SUB = r"""
import sys
sys.path[:0] = [sys.argv[1], sys.argv[2], sys.argv[2] + "/hierarchical-3d-gaussians_b200"]
import test_gpu_sh_rows_edges as t
t.buffer_states(*sys.argv[3:])
"""


def run_buffer_states(emu_so=None, timeout=900):
    """buffer_states in a fresh Python process, which must exit normally -> its output"""
    r = subprocess.run([sys.executable, "-c", _SUB, HERE, ROOT] + ([emu_so] if emu_so else []), cwd=ROOT,
                       capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-4000:]
    return r.stdout


# ---- the GPU tests ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg,M", FLOAT4_LAYOUTS)
@pytest.mark.parametrize("scene", ["runs", "cut"])
def test_layout(scene, deg, M):
    case_layout(deg, M, scene)


@pytest.mark.parametrize("deg,M", [(3, 16), (1, 8), (2, 12), (0, 4)])
def test_row_blocks(deg, M):
    case_row_blocks(deg, M)


def test_row_count_buffer_states():
    out = run_buffer_states()
    for s in ("state: eager", "state a:", "state b:", "state c:"):
        assert s in out, out[-3000:]
    print(out)

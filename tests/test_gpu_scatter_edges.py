"""GPU: the hierarchy cut's fused gather (K1, K1b: each rendered row lerped from its node's row and its parent's) and the
backward's t / (1 - t) scatter into the full-size gradient rows (preprocess_backward_kernel, sh_backward_kernel:
red.global.add into rows the library zero-fills beside the replay), per rendered row against preprocess_ref and per
full-size row against chain_ref's float64 statement of the scatter (chain_ref.scatter_terms / scatter_tol):
    row r  =  sum_{i: c_i = r} t_i g_i  +  sum_{i: p_i = r, u_i != 0} u_i s_i g_i,     u_i = fp32(1 - t_i),
with g_i chain_ref's per-row gradient, s_i the quaternion sign (rotations only) and a budget built from its parts: each
term's chain_ref budget scaled by its weight, one rounding of each product, and (n_r - 1) U sum |terms| for the n_r-term
fp32 atomic sum in an unspecified order.  Rows no visible rendered row reaches, rows reached by exact zeros only (t = 0)
and SH coefficients beyond the active degree have budget 0 and must hold exactly +0.0, bit for bit.

Families: every SH layout (both the scalar path, 3M % 4 != 0, and the float4 path of both SH kernels, degrees below the
layout's), the weights t in {0, 1, 2^-24, 1 - 2^-24, 0.5, random} and parent_indices = -1, fan-in 1 .. 4096 onto one
parent, parents that are rendered rows and chains of them, quaternion dots < 0, = 0, > 0, lerped colours on the clamp at
0, scale_modifier != 1 with do_depth, h3dgs_lod_cut's own tail (render_indices = -1), row blocks, three backward
schedules (one call, the serial debug path, the split 1|4 then 2|8 of h3dgs/graphstep.py, once at a source size where
the 0.7 GB fill outlasts the replay) and the public API against blend_ref -> chain_ref.  The functions `case_*` are also
run on the emulation build by test_scatter_edges_cpu.py; each prints the rows it compared and excluded and the largest
|kernel - f64| / budget (run with -s)."""
import ctypes as C

import numpy as np
import pytest

import preprocess_ref as pr
from chain_ref import C0, U, compare, gather_fp32, general_camera, random_accum, random_rows
from test_gpu_chain_edges import TRANS, W, H, chain_ref_for, check_case, place, run_backward

pytestmark = pytest.mark.gpu

LAYOUTS = [(0, 1), (1, 4), (0, 4), (1, 8), (2, 9), (1, 9), (2, 12), (3, 16), (0, 16), (1, 16), (2, 16)]
T_EDGES = np.array([0.0, 1.0, 2.0 ** -24, 1 - 2.0 ** -24, 0.5], np.float32)
FULL = ("means3D", "opacities", "shs", "scales", "rotations")


# ---- the cut -------------------------------------------------------------------------------------------------------------
def cut_scene(deg, M, seed, fans=(1, 2, 33, 64), dist=10, n_free=60, n_back=5, clamp=True):
    """A cut over N source rows.  Rendered rows [0, P) take distinct node rows ridx (a permutation of [0, P)); the
    parents: one source row per fan-in group (its children), rows of other rendered rows (`rendpar`), chains
    a -> b -> c -> root of rendered rows, one own parent per row with the three quaternion-dot cases (`own`),
    parent_indices = -1 with t < 1 (`self`), and rows behind the camera whose node rows nothing else reaches (`back`).
    The last 30 source rows are in no cut.  Lerped colours of the `own` and `self` rows sit at the clamp at 0.
    -> cam, sc (with kids), info (the row sets)"""
    rng = np.random.default_rng(seed)
    cam = general_camera(W, H, TRANS[dist])
    G = len(fans)
    n_rp, n_chain, n_own, n_self = 20, 8, 12, 24
    P = sum(fans) + n_rp + 4 * n_chain + n_own + n_self + n_free + n_back
    N = P + G + n_own + 30
    z = rng.uniform(2.0, 12.0, N)
    s, q, o, sh = random_rows(rng, N, M)
    s = (s / s.mean(1, keepdims=True) * 0.02 * z[:, None]).astype(np.float32)
    rx, ry = rng.uniform(-1, 1, N) * cam.tanfovx, rng.uniform(-1, 1, N) * cam.tanfovy
    rx[:2] = ry[:2] = 0.0                                         # on the camera's axis
    means = place(cam, rx, ry, z)
    ridx = rng.permutation(P).astype(np.int32)
    pidx = np.full(P, -1, np.int32)
    ts = rng.choice(T_EDGES, P)
    ts[::3] = rng.uniform(0, 1, ts[::3].size).astype(np.float32)
    info, o_ = {}, 0
    seg = lambda name, n: info.__setitem__(name, np.arange(o_, o_ + n))
    info["fans"] = []
    for gi, f in enumerate(fans):
        info["fans"].append((P + gi, np.arange(o_, o_ + f)))
        pidx[o_:o_ + f] = P + gi
        ts[o_:o_ + f][ts[o_:o_ + f] == 1] = np.float32(0.25)       # every child reaches the shared parent
        o_ += f
    seg("rendpar", n_rp)
    others = np.setdiff1d(np.arange(P), info["rendpar"])
    pidx[info["rendpar"]] = ridx[rng.choice(others, n_rp)]
    o_ += n_rp
    seg("chain", 4 * n_chain)
    for k in range(n_chain):
        a = o_ + 4 * k
        pidx[a:a + 3] = ridx[a + 1:a + 4]                         # row a's parent is row a+1's node, ...
        ts[a:a + 4] = rng.uniform(0.1, 0.9, 4).astype(np.float32)
    o_ += 4 * n_chain
    seg("own", n_own)
    pidx[info["own"]] = P + G + np.arange(n_own)
    ts[info["own"]] = rng.uniform(0.1, 0.9, n_own).astype(np.float32)
    o_ += n_own
    seg("self", n_self)
    ts[info["self"]] = np.resize(np.array([0.0, 2.0 ** -24, 0.5, 1 - 2.0 ** -24], np.float32), n_self)
    ts[info["self"][::4]] = rng.uniform(0, 1, n_self // 4).astype(np.float32)
    o_ += n_self + n_free
    seg("back", n_back)
    # parents close to their children; own parents with quaternion dots < 0, exactly 0 (q_p = (x, -r, z, -y) for
    # q_c = (r, x, y, z): the fp32 products cancel pairwise) and > 0
    par = pidx >= 0
    near = means[ridx[par]] + rng.uniform(-0.05, 0.05, (par.sum(), 3)).astype(np.float32)
    sole = np.isin(pidx[par], ridx, invert=True)                 # do not move rendered rows
    means[pidx[par][sole]] = near[sole]
    for j, row in enumerate(info["own"]):
        c, p = ridx[row], pidx[row]
        q[p] = [-q[c] + np.float32(0.01), np.array([q[c][1], -q[c][0], q[c][3], -q[c][2]], np.float32),
                q[c] + np.float32(0.01)][j % 3]
    means[ridx[info["back"]]] = place(cam, [0.0] * n_back, [0.0] * n_back, np.full(n_back, -3.0))
    sc = dict(means3D=means, scales=s, rotations=q, opacities=o, shs=sh, ridx=ridx, pidx=pidx, ts=ts,
              kids=np.ones(P, np.int32))
    if clamp:
        # lerped colours at +-1e-6 .. 3e-5 around 0 (and some far off): the DC coefficient of node and parent from the
        # float64 rest of the lerped SH sum; rows whose parent is their own
        rows_ = np.r_[info["own"], info["self"]]
        sc["shs"][ridx[rows_], 0] = 0
        sc["shs"][np.where(pidx[rows_] < 0, ridx[rows_], pidx[rows_]), 0] = 0
        rest = np.stack([r.v for r in pr.reference(sc, cam, deg).rgb], 1)[rows_]
        tiny = np.array([1e-7, -1e-7, 1e-6, -1e-6, 3e-5, -3e-5, 0.3, -0.3])
        dc = ((rng.choice(tiny, (rows_.size, 3)) - rest) / C0).astype(np.float32)
        sc["shs"][ridx[rows_], 0] = dc
        sc["shs"][np.where(pidx[rows_] < 0, ridx[rows_], pidx[rows_]), 0] = dc
        info["clamp"] = rows_
    info["unused"] = np.arange(N - 30, N)
    return cam, sc, info


# ---- checks ----------------------------------------------------------------------------------------------------------------
def forward_rows(name, cam, sc, deg, mod=1.0):
    """the forward per rendered row against preprocess_ref -> its report"""
    from test_gpu_preprocess_edges import run
    out = run(cam, sc, deg, mod)
    rep = pr.check(pr.reference(sc, cam, deg, mod), out, name=name + " forward")
    tail = np.asarray(sc["ridx"]) < 0
    assert not out["radii"][tail].any() and not out["tiles_touched"][tail].any(), name
    return rep, out


def exact_zeros(name, got, ref):
    """elements with budget 0 and value 0 hold +0.0 bit for bit -> number of such full-size elements"""
    n = 0
    for k, (r, tol, _) in ref.items():
        z = (tol == 0) & (r == 0)
        g = np.ascontiguousarray(got[k], np.float32).reshape(r.shape)
        bad = z & (g.view(np.uint32) != 0)
        assert not bad.any(), (name, k, "not +0.0", np.argwhere(bad)[:5].tolist(), g[bad][:5].tolist())
        n += int(z.sum()) if k in FULL else 0
    return n


def reached(sc, radii):
    """full-size rows some visible rendered row reaches (node, or parent where the lerp is taken)"""
    g = gather_fp32(sc["means3D"], None, None, None, np.where(np.asarray(sc["ridx"]) < 0, 0, sc["ridx"]), sc["pidx"], sc["ts"])
    vis = np.asarray(radii) > 0
    return np.unique(np.r_[g["c"][vis], g["p"][vis & g["lerp"]]]), g


def summary(name, ref, got, rows, excluded=0):
    worst = {k: compare(got[k], r, tol)[0] for k, (r, tol, _) in ref.items() if k in FULL}
    print(f"\n[{name}] full-size rows compared: {rows}, excluded: {excluded}; max |kernel - f64| / budget: "
          + " ".join(f"{k}={v:.3g}" for k, v in worst.items()))
    return worst


def check_full(name, cam, sc, deg, accum, do_depth=True, mod=1.0, min_visible=0.8, debug=False):
    """check_case (every element of every gradient within chain_ref's budget) plus the exact zeros -> (got, ref, radii)"""
    keep = {}
    _, radii, kb, *_rest, got = check_case(name, cam, sc, accum, deg=deg, do_depth=do_depth, mod=mod,
                                           min_visible=min_visible, debug=debug, keep=keep)
    nz = exact_zeros(name, got, keep["ref"])
    rows, _g = reached(sc, radii)
    summary(name, keep["ref"], got, rows.size)
    assert rows.size > 0 and nz > 0, name
    return got, keep["ref"], radii, kb


# ---- families ----------------------------------------------------------------------------------------------------------------
def case_layout(deg, M, dist=10, fans=(1, 2, 33, 64), seed=None):
    """the forward per rendered row and the backward per full-size row on one cut of every kind of row"""
    name = f"scatter deg={deg} M={M} dist={dist} fans={max(fans)}"
    cam, sc, info = cut_scene(deg, M, (seed if seed is not None else 100 * deg + M + dist), fans=fans, dist=dist)
    rep, out = forward_rows(name, cam, sc, deg)
    radii = out["radii"]
    assert (radii[info["back"]] == 0).all()
    kb = out["records"][:, 7].view(np.uint32)
    flags = np.stack([(kb >> (20 + ch)) & 1 for ch in range(3)], 1).astype(bool)
    cl = info["clamp"][radii[info["clamp"]] > 0]
    assert flags[cl].any() and (~flags[cl]).any(), name           # lerped colours on both sides of the clamp
    accum = random_accum(np.random.default_rng(seed or 7), len(sc["ridx"]))
    got, ref, radii, _ = check_full(name, cam, sc, deg, accum)
    # coverage: every weight edge, the lerp decision for t = 1 - 2^-24 and parent_indices = -1, all three quaternion
    # dots, every fan-in, parents that are rendered rows, chains; node rows with t = 0 and nothing else are +0.0
    g = gather_fp32(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], sc["ridx"], sc["pidx"], sc["ts"])
    vis = radii > 0
    for t in T_EDGES:
        assert (vis & (g["t"] == t)).any(), (name, float(t))
    assert (vis & g["lerp"] & (g["t"] == np.float32(1 - 2.0 ** -24))).any() and not (g["lerp"] & (g["t"] == 1)).any()
    assert (vis[info["self"]] & g["lerp"][info["self"]]).sum() >= 10
    for cmp in (np.less, np.equal, np.greater):
        assert (vis & g["lerp"] & cmp(g["dot"], 0)).any(), (name, cmp)
    for parent, kids in info["fans"]:
        on = vis[kids] & g["lerp"][kids]
        assert on.sum() >= 0.7 * kids.size, (name, parent, on.sum())
    assert (vis & g["lerp"])[info["rendpar"]].any() and (vis & g["lerp"])[info["chain"]].sum() >= 10
    zero_only = np.setdiff1d(g["c"][vis & (g["t"] == 0)], np.r_[g["c"][vis & (g["t"] != 0)], g["p"][vis & g["lerp"]]])
    assert zero_only.size > 0 and not got["means3D"][zero_only].view(np.uint32).any(), name
    culled_only = np.setdiff1d(sc["ridx"][~vis], reached(sc, radii)[0])
    assert culled_only.size >= len(info["back"]) and not got["shs"].reshape(len(sc["means3D"]), -1)[culled_only].any()
    assert not got["rotations"][info["unused"]].any()
    if deg < {1: 0, 4: 1, 8: 1, 9: 2, 12: 2, 16: 3}[M]:
        beyond = got["shs"][:, (deg + 1) ** 2:]
        assert not beyond.view(np.uint32).any(), name             # coefficients beyond the active degree: +0.0
    return rep


def case_modifier_depth(deg=3, M=16):
    """scale_modifier != 1 and do_depth, in scatter mode"""
    cam, sc, info = cut_scene(deg, M, 77, dist=1000)
    name = f"scatter mod=0.37 depth deg={deg} M={M}"
    forward_rows(name, cam, sc, deg, mod=0.37)
    accum = random_accum(np.random.default_rng(78), len(sc["ridx"]))
    check_full(name, cam, sc, deg, accum, do_depth=True, mod=0.37)


def case_device_cut_tail(leaves=1500, deg=3, tau=6.0):
    """h3dgs_lod_cut's own cut: the rows after the count hold render_indices = -1.  The forward gives them radius 0 and
    no tiles; the backward writes nothing for them"""
    import torch
    from h3dgs import _lib, synth
    cam = synth.make_camera(W, H)
    lv = synth.cloud_v1(leaves, cam, zmin=2.0, zmax=40.0, seed=3, scale_k=1.0)
    z = lv["means3D"][:, 2:3]
    lv["scales"] = (1.2e-2 * np.sqrt(2.0 * z) * np.exp(0.4 * np.random.default_rng(1).standard_normal(z.shape[:1] + (3,)))).astype(np.float32)
    h = synth.build_hierarchy(lv)
    N = h["nodes"].shape[0]
    L = _lib.lib()
    dv = lambda a, dt=torch.float32: torch.tensor(np.asarray(a), dtype=dt, device="cuda")
    ridx, pidx, nfr, kids = (torch.zeros(N, dtype=torch.int32, device="cuda") for _ in range(4))
    ts, count = torch.zeros(N, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    thr = synth.tau_threshold(tau, cam)
    thr_dev = dv([thr])
    nodes, boxes, cp = dv(h["nodes"], torch.int32), dv(h["boxes"]), dv(cam.camera_center)
    scratch = torch.empty(int(L.h3dgs_expand_scratch_bytes(N)), dtype=torch.uint8, device="cuda")
    _lib.check(L.h3dgs_lod_cut(N, nodes.data_ptr(), boxes.data_ptr(), thr, thr_dev.data_ptr(), cp.data_ptr(),
                               ridx.data_ptr(), pidx.data_ptr(), nfr.data_ptr(), ts.data_ptr(), kids.data_ptr(),
                               count.data_ptr(), scratch.data_ptr(), torch.cuda.current_stream().cuda_stream))
    n = int(count.cpu()[0])
    r = ridx.cpu().numpy()
    assert 0 < n < N and (r[n:] == -1).all() and (r[:n] >= 0).all()
    sc = {k: np.asarray(h[k], np.float32) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    sc.update(ridx=r, pidx=pidx.cpu().numpy(), ts=ts.cpu().numpy(), kids=kids.cpu().numpy())
    name = f"device cut tail n={n} of {N}"
    forward_rows(name, cam, sc, deg)
    accum = random_accum(np.random.default_rng(32), N)
    got, ref, radii, _ = check_full(name, cam, sc, deg, accum, min_visible=0.2 * n / N)
    assert not radii[n:].any()
    g = gather_fp32(sc["means3D"], None, None, None, r[:n], sc["pidx"][:n], sc["ts"][:n])
    assert g["lerp"][radii[:n] > 0].sum() > 50                    # the cut lerps
    return n, N


def case_row_blocks(deg=3, M=16, bounds=(0, 37, 150, 151, None)):
    """grad_rows = [a, b) in scatter mode: each block's output equals the reference of its own rows (exactly +0.0 on the
    rows they do not reach), and the sum over the blocks equals the whole call within the whole call's budget"""
    cam, sc, info = cut_scene(deg, M, 55)
    P = len(sc["ridx"])
    bounds = [P if b is None else b for b in bounds]
    accum = random_accum(np.random.default_rng(56), P)
    whole, radii, rec, fwd, _ = run_backward(cam, sc, accum, deg, True)
    kb = rec[:, 7].view(np.uint32)
    ref_all = chain_ref_for(cam, sc, accum, deg, True, 1.0, radii, kb)[0]
    total = {k: np.zeros(v.shape) for k, v in whole.items()}
    for a, b in zip(bounds[:-1], bounds[1:]):
        blk, *_ = run_backward(cam, sc, accum, deg, True, grad_rows=(a, b), forward=fwd)
        mine = np.zeros(P, radii.dtype)
        mine[a:b] = radii[a:b]
        ref = chain_ref_for(cam, sc, accum, deg, True, 1.0, mine, kb)[0]
        name = f"row block [{a}, {b})"
        for k, (r, tol, _) in ref.items():
            w, _n = compare(blk[k], r, tol)
            assert w <= 1.0, (name, k, w)
        exact_zeros(name, blk, ref)
        for k in total:
            total[k] += blk[k].astype(np.float64)
    for k, (r, tol, _) in ref_all.items():
        w, _n = compare(total[k], r, tol)
        assert w <= 1.0, ("sum of the row blocks", k, w)
    rows, _g = reached(sc, radii)
    summary("row blocks, summed", ref_all, total, rows.size)


def split_backward(cam, sc, deg, gcol, forward, mod=1.0, do_depth=False):
    """the split schedule through the C-ABI as h3dgs/graphstep.py issues it: phases 1 | 4 (replay; the zero-fill of
    the full-size rows on the side stream beside it), then 2 | 8 (the chain rule; no second fill).  The outputs start
    as NaN.  -> (gradients dict, the [P][10] sums the replay made)"""
    import torch
    from diff_gaussian_rasterization import _C
    from h3dgs import _lib
    f = lambda a: None if a is None else torch.tensor(np.asarray(a, np.float32), device="cuda")
    i = lambda a: torch.tensor(np.asarray(a, np.int32), device="cuda")
    n, _col, radii, gb, bb, ib, _ = forward
    N, M = sc["means3D"].shape[0], sc["shs"].shape[1]
    P = len(sc["ridx"])
    m, sh, op, s, r = f(sc["means3D"]), f(sc["shs"]), f(sc["opacities"]), f(sc["scales"]), f(sc["rotations"])
    ts, kids, ridx, pidx = f(sc["ts"]), i(sc["kids"]), i(sc["ridx"]), i(sc["pidx"])
    bg, vm, pm, cp = f(np.zeros(3)), f(cam.world_view_transform), f(cam.full_proj_transform), f(cam.camera_center)
    a = _C._make_args(P, m, sh, None, op, s, r, None, bg, vm, pm, cp, cam.tanfovx, cam.tanfovy, cam.H, cam.W, deg, mod,
                      False, False, ts, kids, do_depth, (1, 0), ridx, pidx, N)
    nan = lambda *shape: torch.full(shape, float("nan"), dtype=torch.float32, device="cuda")
    out = dict(means3D=nan(N, 3), means2D=nan(P, 3), shs=nan(N, M, 3), opacities=nan(N, 1), scales=nan(N, 3),
               rotations=nan(N, 4))
    L = _lib.lib()
    scratch = torch.zeros((L.h3dgs_backward_scratch_bytes(P),), dtype=torch.uint8, device="cuda")
    g = f(gcol)
    st = torch.cuda.current_stream().cuda_stream
    for phases in (1 | 4, 2 | 8):
        _lib.check(L.h3dgs_rasterize_backward(C.byref(a), radii.data_ptr(), gb.data_ptr(), bb.data_ptr(), ib.data_ptr(),
                                              int(n), g.data_ptr(), None, out["means3D"].data_ptr(),
                                              out["means2D"].data_ptr(), out["shs"].data_ptr(), None,
                                              out["opacities"].data_ptr(), out["scales"].data_ptr(),
                                              out["rotations"].data_ptr(), None, scratch.data_ptr(), phases, st))
    accum = scratch.view(torch.float32)[: P * 10].view(P, 10).cpu().numpy().copy()
    return {k: v.cpu().numpy() for k, v in out.items()}, accum


def case_schedules(deg=3, M=16, seed=61):
    """one frame, three backward schedules, each per full-size row against the reference (never against each other):
    one call (the SH and covariance kernels concurrently), debug (serial) and the split 1|4 then 2|8"""
    cam, sc, info = cut_scene(deg, M, seed)
    P = len(sc["ridx"])
    gcol = (np.random.default_rng(seed).standard_normal((3, H, W)) / (H * W)).astype(np.float32)
    _, radii, rec, fwd, _ = run_backward(cam, sc, np.zeros((P, 10), np.float32), deg)
    split, accum = split_backward(cam, sc, deg, gcol, fwd)
    assert (np.abs(accum[radii > 0]).sum(1) > 0).mean() > 0.5          # the replay reached most visible rows
    kb = rec[:, 7].view(np.uint32)
    ref = chain_ref_for(cam, sc, accum, deg, False, 1.0, radii, kb)[0]
    for k, (r, tol, _) in ref.items():
        w, _n = compare(split[k], r, tol)
        assert w <= 1.0, ("split 1|4, 2|8", k, w)
    exact_zeros("split", split, ref)
    rows, _g = reached(sc, radii)
    summary(f"schedule split deg={deg} M={M}", ref, split, rows.size)
    for debug in (False, True):
        check_full(f"schedule {'debug (serial)' if debug else 'one call'} deg={deg} M={M}", cam, sc, deg, accum,
                   do_depth=False, debug=debug)


def case_split_big_source(N=3_000_000, P=3000, deg=3, M=16):
    """the split schedule with num_source at config #3's size (3 M rows: a 0.7 GB fill) and a small cut, so the fill
    outlasts the replay.  The reference is taken on the rows the cut references; every other row is +0.0"""
    rng = np.random.default_rng(71)
    cam, small, info = cut_scene(deg, M, 71)
    Ps, Ns = len(small["ridx"]), small["means3D"].shape[0]
    src = np.sort(rng.choice(N, Ns, replace=False))             # where the small scene's rows live in the big one
    big = {}
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        a = np.empty((N,) + small[k].shape[1:], np.float32)
        a[...] = np.float32(0.25)
        a[src] = small[k]
        big[k] = a
    big.update(ridx=src[small["ridx"]].astype(np.int32), pidx=np.where(small["pidx"] < 0, -1, src[np.maximum(small["pidx"], 0)]).astype(np.int32),
               ts=small["ts"], kids=small["kids"])
    gcol = (rng.standard_normal((3, H, W)) / (H * W)).astype(np.float32)
    _, radii, rec, fwd, _ = run_backward(cam, small, np.zeros((Ps, 10), np.float32), deg, forward=None)
    from diff_gaussian_rasterization import _C
    import torch
    f = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    i = lambda a: torch.tensor(np.asarray(a, np.int32), device="cuda")
    fwd_big = _C.rasterize_gaussians(f(np.zeros(3)), f(big["means3D"]), None, f(big["opacities"]), f(big["scales"]),
                                     f(big["rotations"]), 1.0, None, f(cam.world_view_transform),
                                     f(cam.full_proj_transform), cam.tanfovx, cam.tanfovy, H, W, f(big["shs"]), deg,
                                     f(cam.camera_center), False, False, i(big["ridx"]), i(big["pidx"]), f(big["ts"]),
                                     i(big["kids"]), False)
    assert np.array_equal(fwd_big[2].cpu().numpy(), radii)
    got, accum = split_backward(cam, big, deg, gcol, fwd_big)
    kb = rec[:, 7].view(np.uint32)
    ref = chain_ref_for(cam, small, accum, deg, False, 1.0, radii, kb)[0]
    other = np.ones(N, bool)
    other[src] = False
    for k in FULL:
        r, tol, _ = ref[k]
        g = got[k]
        w, _n = compare(g[src], r, tol)
        assert w <= 1.0, ("split, 3 M source rows", k, w)
        assert not g[other].view(np.uint32).any(), ("split, 3 M source rows: a row outside the cut is not +0.0", k)
    exact_zeros("split 3M", {k: got[k][src] if k in FULL else got[k] for k in got}, ref)
    rows, _g = reached(small, radii)
    summary(f"split schedule, {N} source rows", ref, {k: got[k][src] for k in FULL}, rows.size)


def case_composition(deg, M, seed=None):
    """the public API (GaussianRasterizer with the hierarchy arguments, the whole backward from a random dL/dcolor)
    against blend_ref's sums -> chain_ref -> the scatter.  The budget adds the sums' own (accum_tol, and their rounding
    to fp32) carried through the magnitude chain of chain_ref; full-size rows that a rendered row of blend_ref's
    near_gauss set reaches are left out"""
    import torch
    from blend_ref import blend_reference
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer, _C
    seed = seed if seed is not None else 300 + 10 * deg + M
    cam, sc, info = cut_scene(deg, M, seed, fans=(1, 2, 33), n_free=120)
    P, N = len(sc["ridx"]), sc["means3D"].shape[0]
    rng = np.random.default_rng(seed)
    gcol = (rng.standard_normal((3, H, W)) / (H * W)).astype(np.float32)
    f = lambda a, rg=False: torch.tensor(np.asarray(a, np.float32), device="cuda", requires_grad=rg)
    i = lambda a: torch.tensor(np.asarray(a, np.int32), device="cuda")
    prm = {k: f(sc[k], True) for k in FULL}
    bg = f(np.zeros(3))
    rs = GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=bg,
                                       scale_modifier=1.0, viewmatrix=f(cam.world_view_transform),
                                       projmatrix=f(cam.full_proj_transform), sh_degree=deg, campos=f(cam.camera_center),
                                       prefiltered=False, debug=False, render_indices=i(sc["ridx"]),
                                       parent_indices=i(sc["pidx"]), interpolation_weights=f(sc["ts"]),
                                       num_node_kids=i(sc["kids"]), do_depth=False)
    means2D = torch.zeros((P, 3), dtype=torch.float32, device="cuda", requires_grad=True)
    img, radii_t, *_ = GaussianRasterizer(rs)(means3D=prm["means3D"], means2D=means2D, shs=prm["shs"], colors_precomp=None,
                                               opacities=prm["opacities"], scales=prm["scales"], rotations=prm["rotations"],
                                               cov3D_precomp=None)
    (img * f(gcol)).sum().backward()
    got = {k: prm[k].grad.cpu().numpy() for k in FULL}
    radii = radii_t.cpu().numpy()
    # the forward's state (records, tile lists) from the same call through _C
    n, _c, radii2, gb, bb, ib, _ = _C.rasterize_gaussians(bg, prm["means3D"].detach(), None, prm["opacities"].detach(),
                                                          prm["scales"].detach(), prm["rotations"].detach(), 1.0, None,
                                                          rs.viewmatrix, rs.projmatrix, cam.tanfovx, cam.tanfovy, H, W,
                                                          prm["shs"].detach(), deg, rs.campos, False, False, rs.render_indices,
                                                          rs.parent_indices, rs.interpolation_weights, rs.num_node_kids, False)
    assert np.array_equal(radii2.cpu().numpy(), radii)
    st = {k: v.cpu().numpy() for k, v in _C.state_view(P, W, H, n, gb, bb, ib).items()}
    rec = st["records"].copy()
    rec[radii <= 0] = 0
    br = blend_reference(rec, st["ranges"], st.get("point_list", np.zeros(0, np.int64)), W, H, np.zeros(3), gcol,
                         hier=True, kids=sc["kids"])
    kb = st["records"][:, 7].view(np.uint32)
    acc32 = br["accum"].astype(np.float32)
    ref = chain_ref_for(cam, sc, acc32, deg, False, 1.0, radii, kb)[0]
    # the sums' own error (blend_ref's budget plus their rounding to fp32), carried through chain_ref's magnitude chain
    # (the same formula on absolute values: chain_ref is linear in the sums)
    dacc = (br["accum_tol"] + U * np.abs(br["accum"])) * (1 + 2.0 ** -20)
    prop = chain_ref_for(cam, sc, dacc.astype(np.float32), deg, False, 1.0, radii, kb)[0]
    rows, g = reached(sc, radii)
    vis = radii > 0
    near = vis & br["near_gauss"]
    bad_rows = np.unique(np.r_[g["c"][near], g["p"][near & g["lerp"]]])
    keep = np.ones(N, bool)
    keep[bad_rows] = False
    compared = np.intersect1d(rows, np.nonzero(keep)[0]).size
    assert compared >= 0.9 * rows.size, (deg, M, compared, rows.size)
    worst = {}
    for k in FULL:
        r, tol, _ = ref[k]
        budget = tol + prop[k][2] + 1e-30
        worst[k], _n = compare(got[k], r, budget, keep)
        assert worst[k] <= 1.0, (deg, M, k, worst[k])
    print(f"\n[composition deg={deg} M={M}] full-size rows compared: {compared}, excluded: {rows.size - compared}; "
          "max |kernel - ref| / budget: " + " ".join(f"{k}={v:.3g}" for k, v in worst.items()))


# ---- the GPU tests -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg,M", LAYOUTS)
def test_layout(deg, M):
    case_layout(deg, M)


@pytest.mark.parametrize("deg,M", [(0, 1), (2, 9), (3, 16)])
def test_layout_far_camera(deg, M):
    case_layout(deg, M, dist=1000)


def test_fan_in():
    """one parent shared by 1, 2, 33, 512 and 4096 rendered children: the atomic-order part of the budget"""
    case_layout(3, 16, fans=(1, 2, 33, 512, 4096))
    case_layout(1, 9, fans=(1, 2, 33, 512, 4096))


def test_modifier_and_depth():
    case_modifier_depth()
    case_modifier_depth(2, 9)


def test_device_cut_tail():
    case_device_cut_tail()


@pytest.mark.parametrize("deg,M", [(3, 16), (2, 9)])
def test_row_blocks(deg, M):
    case_row_blocks(deg, M)


@pytest.mark.parametrize("deg,M", [(3, 16), (1, 9)])
def test_schedules(deg, M):
    case_schedules(deg, M)


def test_split_schedule_config3_source_size():
    case_split_big_source()


@pytest.mark.parametrize("deg,M", LAYOUTS)
def test_composition(deg, M):
    case_composition(deg, M)

"""numpy restatement of the view cull's row mask (csrc/lod_cull.cu, include/h3dgs.h h3dgs_lod_cull_mask), float64
operation by operation from the float32 inputs, in the kernel's order, so that the two agree bit for bit; and the
hierarchies, cameras and edge rows the CPU and GPU tests of the cull share.

A row is kept unless no lerp weight t in [0, 1] with its partner row (the parent node's start row, the row itself for a
root) can give it a positive radius and a non-empty tile rect in K1; DESIGN.md §3.9 derives the bound."""
import numpy as np

import hier_general as hg
import preprocess_ref as pr
from h3dgs import synth

f64 = np.float64
REL, COV, EIG, CAMR, FLOOR_ROOT = 2.0 ** -16, 2.0 ** -12, 2.0 ** -9, 2.0 ** -20, 0.3163
NEAR, DILATION, FOV_CLAMP, W_EPS = (f64(np.float32(x)) for x in (0.2, 0.3, 1.3, 1e-7))
TILE = 16


def _row_dot(m, r, x, y, z):
    return ((m[r] * x + m[r + 4] * y) + m[r + 8] * z) + m[r + 12]


def _row_abs(m, r, x, y, z):
    return ((np.abs(m[r]) * x + np.abs(m[r + 4]) * y) + np.abs(m[r + 8]) * z) + np.abs(m[r + 12])


def _qn2(q):
    q = q.astype(f64)
    return ((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]) + q[:, 3] * q[:, 3]


def keep(a, sa, qa, b, sb, qb, view, proj, W, H, tanx, tany, smod=1.0):
    """per pair: True when K1 could draw the row (a, sa, qa) lerped with its partner (b, sb, qb) for some t in [0, 1]"""
    m = np.asarray(view, np.float32).reshape(16).astype(f64)
    q = np.asarray(proj, np.float32).reshape(16).astype(f64)
    tanx, tany = f64(np.float32(tanx)), f64(np.float32(tany))
    fx = f64(W) / (2.0 * tanx) * (1.0 + CAMR)
    fy = f64(H) / (2.0 * tany) * (1.0 + CAMR)
    limx, limy = FOV_CLAMP * tanx * (1.0 + CAMR), FOV_CLAMP * tany * (1.0 + CAMR)
    wf2 = f64(0.0)
    for k in range(3):
        for j in range(3):
            wf2 = wf2 + m[4 * k + j] * m[4 * k + j]
    ex, ey = f64(TILE * ((W + TILE - 1) // TILE)), f64(TILE * ((H + TILE - 1) // TILE))
    smod = np.abs(f64(np.float32(smod)))
    with np.errstate(all="ignore"):
        fin = np.ones(a.shape[0], bool)
        for arr in (a, b, sa, sb, qa, qb):
            fin &= np.isfinite(arr).all(1)
        A, B = a.astype(f64), b.astype(f64)
        ax, ay, az, bx, by, bz = A[:, 0], A[:, 1], A[:, 2], B[:, 0], B[:, 1], B[:, 2]
        Ax, Ay, Az = np.fmax(np.abs(ax), np.abs(bx)), np.fmax(np.abs(ay), np.abs(by)), np.fmax(np.abs(az), np.abs(bz))
        za, zb = _row_dot(m, 2, ax, ay, az), _row_dot(m, 2, bx, by, bz)
        dz = REL * _row_abs(m, 2, Ax, Ay, Az)
        behind = np.fmax(za, zb) + dz <= NEAR
        zc = NEAR - dz
        ca, cb = za < zc, ~(za < zc) & (zb < zc)
        t0 = (zc - zb) / (za - zb)
        t1 = (zc - za) / (zb - za)
        e0 = [np.where(ca, bc + t0 * (ac - bc), ac) for ac, bc in ((ax, bx), (ay, by), (az, bz))]
        e1 = [np.where(cb, ac + t1 * (bc - ac), bc) for ac, bc in ((ax, bx), (ay, by), (az, bz))]
        z0, z1 = np.where(ca, zc, za), np.where(cb, zc, zb)
        z_lo = np.fmax(NEAR, np.fmin(z0, z1) - dz)
        Sx, Sy, Sw = _row_abs(q, 0, Ax, Ay, Az), _row_abs(q, 1, Ax, Ay, Az), _row_abs(q, 3, Ax, Ay, Az)
        d0, d1 = _row_dot(q, 3, *e0) + W_EPS, _row_dot(q, 3, *e1) + W_EPS
        d_lo = np.fmin(d0, d1) - REL * Sw
        unbounded = ~(d_lo > 0.0)
        nx0, nx1 = _row_dot(q, 0, *e0) / d0, _row_dot(q, 0, *e1) / d1
        ny0, ny1 = _row_dot(q, 1, *e0) / d0, _row_dot(q, 1, *e1) / d1
        nxm, nym = np.fmax(np.abs(nx0), np.abs(nx1)), np.fmax(np.abs(ny0), np.abs(ny1))
        px = REL * (((Sx + nxm * Sw) / d_lo + nxm) + 1.0)
        py = REL * (((Sy + nym * Sw) / d_lo + nym) + 1.0)
        ix_lo, ix_hi = ((np.fmin(nx0, nx1) - px + 1.0) * W - 1.0) * 0.5, ((np.fmax(nx0, nx1) + px + 1.0) * W - 1.0) * 0.5
        iy_lo, iy_hi = ((np.fmin(ny0, ny1) - py + 1.0) * H - 1.0) * 0.5, ((np.fmax(ny0, ny1) + py + 1.0) * H - 1.0) * 0.5
        SA, SB = np.abs(sa.astype(f64)), np.abs(sb.astype(f64))
        smax = np.fmax(np.fmax(SA[:, 0], SA[:, 1]), SA[:, 2])
        smax = np.fmax(smax, np.fmax(np.fmax(SB[:, 0], SB[:, 1]), SB[:, 2]))
        smax = smod * smax
        Q2 = np.fmax(_qn2(qa), _qn2(qb))
        Rn = np.fmax(1.0, 2.0 * Q2 - 1.0) + COV * (1.0 + Q2)
        lam_v = ((smax * smax) * (Rn * Rn)) * (1.0 + COV)
        J2 = ((fx * fx) * (1.0 + limx * limx) + (fy * fy) * (1.0 + limy * limy)) / (z_lo * z_lo)
        lam = (J2 * wf2) * lam_v
        L = (lam * (1.0 + COV) + DILATION) * (1.0 + EIG) + FLOOR_ROOT
        rad = 3.0 * np.sqrt(L) * (1.0 + COV) + 1.0
        gxp = 1.0 + REL * (np.fmax(np.abs(ix_lo), np.abs(ix_hi)) + rad + W)
        gyp = 1.0 + REL * (np.fmax(np.abs(iy_lo), np.abs(iy_hi)) + rad + H)
        off = (ix_hi + rad + gxp < 1.0) | (iy_hi + rad + gyp < 1.0) | (ix_lo - rad - gxp >= ex) | (iy_lo - rad - gyp >= ey)
    return ~fin | (~behind & (unbounded | ~off))


def pairs(nodes):
    """(row, partner row) of every row of every node, in node order"""
    nodes = np.asarray(nodes, np.int64)
    parent, start, n = nodes[:, 1], nodes[:, 2], nodes[:, 3] + nodes[:, 4]
    n = np.maximum(n, 0)
    ni = np.repeat(np.arange(nodes.shape[0]), n)
    rows = start[ni] + (np.arange(ni.size) - np.repeat(np.cumsum(n) - n, n))
    par = parent[ni]
    partner = np.where(par >= 0, start[np.maximum(par, 0)], rows)
    return rows, partner


def mask(h, cam, smod=1.0):
    """-> (mask uint8 [rows], written bool [rows]): h3dgs_lod_cull_mask for the camera (rows of no node: not written)"""
    R = h["means3D"].shape[0]
    rows, partner = pairs(h["nodes"])
    k = keep(h["means3D"][rows], h["scales"][rows], h["rotations"][rows], h["means3D"][partner], h["scales"][partner],
             h["rotations"][partner], cam.world_view_transform, cam.full_proj_transform, cam.W, cam.H, cam.tanfovx,
             cam.tanfovy, smod)
    out, written = np.zeros(R, np.uint8), np.zeros(R, bool)
    out[rows], written[rows] = k, True
    return out, written


def visible_nodes(nodes, m):
    """nodes with count_leafs / count_merged replaced by the node's masked leaf and merged rows (vl, vm): the cut and the
    budget under the mask are the unmasked ones of this hierarchy"""
    nodes = np.array(nodes, np.int32, copy=True)
    c = np.concatenate([[0], np.cumsum(m.astype(np.int64))])
    s, cl, cm = nodes[:, 2].astype(np.int64), nodes[:, 3].astype(np.int64), nodes[:, 4].astype(np.int64)
    ok = (cl + cm) > 0
    vl = np.where(ok, c[np.clip(s + cl, 0, m.size)] - c[np.clip(s, 0, m.size)], 0)
    vm = np.where(ok, c[np.clip(s + cl + cm, 0, m.size)] - c[np.clip(s + cl, 0, m.size)], 0)
    nodes[:, 3], nodes[:, 4] = vl, vm
    return nodes


# ---------------------------------------------------------------------------------------------------------------
# hierarchies, cameras and edge rows
# ---------------------------------------------------------------------------------------------------------------
def _identity_quat(n):
    q = np.zeros((n, 4), np.float32)
    q[:, 0] = 1
    return q


def single_node():
    return dict(means3D=np.array([[0.0, 0.0, 4.0]], np.float32), scales=np.full((1, 3), 0.05, np.float32),
                rotations=_identity_quat(1), opacities=np.full((1, 1), 0.8, np.float32),
                shs=np.zeros((1, 16, 3), np.float32), nodes=np.array([[0, -1, 0, 1, 0, 0, 0]], np.int32),
                boxes=np.array([[[-0.2, -0.2, 3.8, 0.4], [0.2, 0.2, 4.2, 0.0]]], np.float32))


def odd_rows(h, seed=0):
    """h with some rows not finite (NaN or inf in a mean, a scale or a rotation), zero scales, and unnormalised
    rotations up to |q| = 2"""
    rng = np.random.default_rng(seed)
    h = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in h.items()}
    R = h["means3D"].shape[0]
    pick = lambda k: rng.choice(R, size=min(k, R), replace=False)
    h["means3D"][pick(3), rng.integers(0, 3)] = np.nan
    h["means3D"][pick(2), 2] = np.inf
    h["scales"][pick(3), 1] = np.inf
    h["rotations"][pick(2), 0] = np.nan
    h["scales"][pick(max(R // 10, 1))] = 0.0
    z = pick(max(R // 5, 1))
    h["rotations"][z] *= rng.uniform(1.0, 2.0, (z.size, 1)).astype(np.float32)
    return h


def scenes(cam):
    """(name, hierarchy with Gaussian rows): creator-built, general (tests/hier_general.py), single-node, odd rows"""
    out = [("creator", synth.build_hierarchy(synth.cloud_v1(200, cam, zmin=2.0, zmax=30.0, seed=21)))]
    for n in (2, 5, 300):
        out.append((f"general{n}", hg.dense_hierarchy(n, n, cam)))
    out.append(("surround", surround_hierarchy(600, seed=4)))
    out.append(("single", single_node()))
    out.append(("odd", odd_rows(hg.dense_hierarchy(7, 400, cam), 1)))
    return out


def surround_hierarchy(n_leaves, seed=0, radius=30.0, sh_degree=3):
    """leaves on every side of the origin (a shell 1 .. radius units out, all directions), as a creator-built hierarchy:
    a camera near the origin sees only part of it"""
    rng = np.random.default_rng(seed)
    d = rng.standard_normal((n_leaves, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    r = rng.uniform(1.0, radius, (n_leaves, 1))
    xyz = (d * r).astype(np.float32)
    K = (sh_degree + 1) ** 2
    q = rng.standard_normal((n_leaves, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    leaves = dict(means3D=xyz, scales=(0.01 * r * np.exp(0.4 * rng.standard_normal((n_leaves, 3)))).astype(np.float32),
                  rotations=q.astype(np.float32), opacities=rng.uniform(0.2, 0.9, (n_leaves, 1)).astype(np.float32),
                  shs=(0.3 * rng.standard_normal((n_leaves, K, 3))).astype(np.float32))
    return synth.build_hierarchy(leaves)


def cameras(h, W=480, H=270):
    """the default camera, yawed and shifted ones, an off-centre principal point, cameras 10 and 1000 units from the
    origin, and one inside the boxes (at the centre of a mid-level node's box)"""
    rs = np.random.default_rng(2)
    out = dict(default=synth.make_camera(W, H))
    for k in range(2):
        out[f"yaw{k}"] = synth.yaw_camera(W, H, float(rs.uniform(-40, 40)), rs.uniform(-0.5, 0.5, 3))
    out["behind"] = synth.yaw_camera(W, H, 180.0, [0.0, 0.0, 2.0])
    out["offcentre"] = synth.make_camera(W, H, primx=0.3, primy=0.65)
    out["far10"] = synth.yaw_camera(W, H, 20.0, [0.0, 0.0, 10.0])
    out["far1000"] = synth.yaw_camera(W, H, -10.0, [3.0, -2.0, 1000.0], zfar=5000.0)
    b = h["boxes"]
    mid = int(np.argmax(h["nodes"][:, 6] > 0) if b.shape[0] == 1 else b.shape[0] // 3)
    c = ((b[mid, 0, :3].astype(np.float64) + b[mid, 1, :3]) / 2)
    out["inside"] = synth.yaw_camera(W, H, 35.0, -np.array([[np.cos(0.61), 0, -np.sin(0.61)], [0, 1, 0],
                                                            [np.sin(0.61), 0, np.cos(0.61)]]) @ c)
    return out


def edge_pairs(cam, seed=0):
    """(row means, scales, rotations; partner means, scales, rotations; family names) at the decision edges of the
    cull: centres at the near plane +- ulps, rect edges +- 1 px at each of the four borders, needles, a partner on the
    far side of the camera, |q| up to 2 and zero scales"""
    rng = np.random.default_rng(seed)
    fam, A, B = [], [], []
    W, H = cam.W, cam.H
    tx, ty = cam.tanfovx, cam.tanfovy

    def add(name, a, b):
        fam.extend([name] * a.shape[0]); A.append(a); B.append(b)

    # near plane: both endpoints at view z = near +- k ulp (and one side well in front / behind)
    z = np.float32(0.2)
    ks = np.arange(-6, 7)
    zs = np.array([np.float32(z) + np.float32(k) * np.spacing(z) for k in ks], np.float64)
    # ... and just behind the cull's own margin (2^-16 of the depth's scale, here ~0.2): the culled side of the edge
    zs = np.concatenate([zs, 0.2 * (1.0 - 2.0 ** -np.arange(10.0, 17.0))])
    rx, ry = rng.uniform(-0.5, 0.5, zs.size) * tx, rng.uniform(-0.5, 0.5, zs.size) * ty
    a = pr.place(cam, rx, ry, zs)
    add("near", a, a)
    add("near_cross", a, pr.place(cam, rx, ry, np.full(zs.size, -1.5)))
    add("near_front", pr.place(cam, rx, ry, np.full(zs.size, 0.19)), pr.place(cam, rx, ry, np.full(zs.size, 0.21)))
    # rect edges: a pixel centre one radius-ish outside each border, +- 1 px, at a few depths
    for zz in (0.5, 3.0, 20.0):
        for d in np.arange(-6.0, 6.5, 0.5):
            for side in range(4):
                ix = {0: -d, 1: TILE * ((W + TILE - 1) // TILE) + d, 2: W / 2, 3: W / 2}[side]
                iy = {0: H / 2, 1: H / 2, 2: -d, 3: TILE * ((H + TILE - 1) // TILE) + d}[side]
                p = pr.place(cam, [pr.ndc_ratio(cam, ix, W) * tx], [pr.ndc_ratio(cam, iy, H) * ty], [zz])
                add("rect", p, p)
    # needles: one long axis, rotated, near the borders
    n = 40
    rxn = rng.choice([-1.0, 1.0], n) * rng.uniform(1.0, 1.6, n) * tx
    ryn = rng.uniform(-1.2, 1.2, n) * ty
    a = pr.place(cam, rxn, ryn, rng.uniform(0.5, 8.0, n))
    add("needle", a, a)
    # partners on the far side of the camera
    m = 40
    a = pr.place(cam, rng.uniform(-1.5, 1.5, m) * tx, rng.uniform(-1.5, 1.5, m) * ty, rng.uniform(0.3, 5.0, m))
    bb = pr.place(cam, rng.uniform(-3, 3, m), rng.uniform(-3, 3, m), -rng.uniform(0.1, 5.0, m))
    add("far_side", a, bb)
    add("far_side_rev", bb, a)
    A, B = np.concatenate(A).astype(np.float32), np.concatenate(B).astype(np.float32)
    N = A.shape[0]
    fam = np.array(fam)
    sa = (np.exp(rng.uniform(-6, -1, (N, 3)))).astype(np.float32)
    sb = (np.exp(rng.uniform(-6, -1, (N, 3)))).astype(np.float32)
    nd = fam == "needle"
    sa[nd] = np.array([0.4, 1e-4, 1e-4], np.float32)
    sb[nd] = np.array([0.6, 2e-4, 1e-4], np.float32)
    qa, qb = rng.standard_normal((N, 4)), rng.standard_normal((N, 4))
    qa /= np.linalg.norm(qa, axis=1, keepdims=True)
    qb /= np.linalg.norm(qb, axis=1, keepdims=True)
    big = rng.uniform(size=N) < 0.25
    qa[big] *= rng.uniform(1.0, 2.0, (big.sum(), 1))
    zero = rng.uniform(size=N) < 0.1
    sa[zero] = 0.0
    sb[zero & (rng.uniform(size=N) < 0.5)] = 0.0
    return A, sa, qa.astype(np.float32), B, sb, qb.astype(np.float32), fam


def pair_hierarchy(A, sa, qa, B, sb, qb):
    """one two-node tree per pair: the root holds the partner row, its one child the row -- the child's partner is the
    root's start row, as the cut pairs them"""
    n = A.shape[0]
    K = 16
    means = np.empty((2 * n, 3), np.float32); scales = np.empty((2 * n, 3), np.float32); rots = np.empty((2 * n, 4), np.float32)
    means[0::2], means[1::2] = B, A
    scales[0::2], scales[1::2] = sb, sa
    rots[0::2], rots[1::2] = qb, qa
    nodes = np.zeros((2 * n, 7), np.int32)
    k = np.arange(n)
    nodes[0::2] = np.stack([np.ones(n), -np.ones(n), 2 * k, np.zeros(n), np.ones(n), 2 * k + 1, np.ones(n)], 1)
    nodes[1::2] = np.stack([np.zeros(n), 2 * k, 2 * k + 1, np.ones(n), np.zeros(n), np.zeros(n), np.zeros(n)], 1)
    return dict(means3D=means, scales=scales, rotations=rots, opacities=np.full((2 * n, 1), 0.9, np.float32),
                shs=np.zeros((2 * n, K, 3), np.float32), nodes=nodes,
                boxes=np.zeros((2 * n, 2, 4), np.float32))


def t_values(h, rows, partner, cam, rng, n_random=2):
    """lerp weights per pair: 0, 1, random ones, and the two sides of the near plane crossing when the segment crosses"""
    m = np.asarray(cam.world_view_transform, np.float64).reshape(16)
    za = _row_dot(m, 2, *h["means3D"][rows].astype(np.float64).T)
    zb = _row_dot(m, 2, *h["means3D"][partner].astype(np.float64).T)
    with np.errstate(all="ignore"):
        tc = (f64(NEAR) - zb) / (za - zb)
    ts = [np.zeros(rows.size), np.ones(rows.size)] + [rng.uniform(size=rows.size) for _ in range(n_random)]
    ok = np.isfinite(tc) & (tc > 0) & (tc < 1)
    for d in (-1e-6, 1e-6, 1e-3):
        ts.append(np.where(ok, np.clip(tc + d, 0, 1), rng.uniform(size=rows.size)))
    return [t.astype(np.float32) for t in ts]

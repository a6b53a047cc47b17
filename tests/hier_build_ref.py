"""The hierarchy creator restated from include/h3dgs.h (h3dgs_build_hierarchy) in numpy, by different means than the
kernel: the fp32 Morton quantisation, a TOP-DOWN radix split of the augmented keys (the kernel builds the same unique
tree bottom-up, Karras-style), BFS numbering level by level, and every merged node's statistics computed directly from
its leaf set in float64 (the kernel combines two children).  Also the test clouds."""
import numpy as np

EIG_FLOOR = 1e-24


def morton(xyz):
    """63-bit keys: 21 bits per axis, x highest; q = min(2097151, (uint32)((x - lo) * s)) in fp32"""
    xyz = np.asarray(xyz, np.float32)
    lo, hi = xyz.min(0), xyz.max(0)
    with np.errstate(divide="ignore"):
        s = np.where(hi == lo, np.float32(0), np.float32(2097152.0) / (hi - lo)).astype(np.float32)
    t = (xyz - lo) * s                                   # float32, each operation rounded
    q = np.minimum(t, np.float32(2097151)).astype(np.uint64)
    key = np.zeros(len(xyz), np.uint64)
    for b in range(21):
        for a in range(3):
            key |= ((q[:, a] >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b + 2 - a)
    return key


def _bit_length(x):
    """bit_length of uint64 values (0 -> 0)"""
    x = x.astype(np.uint64)
    out = np.zeros(x.shape, np.int64)
    for b in range(63, -1, -1):
        hit = (out == 0) & (((x >> np.uint64(b)) & np.uint64(1)) == 1)
        out[hit] = b + 1
    return out


def topology(xyz):
    """-> (order: sorted position -> input index, lo [N], hi [N] sorted ranges, parent [N], first_child [N], level [N])
    in BFS order"""
    key = morton(xyz)
    order = np.argsort(key, kind="stable")
    k = key[order]
    P = len(k)
    lo, hi, parent, child, level = [0], [P], [-1], [0], [0]
    cur = np.array([0])
    while cur.size:
        a, b = np.array(lo)[cur], np.array(hi)[cur]
        inner = cur[b - a > 1]
        if inner.size == 0:
            break
        a, b = np.array(lo)[inner], np.array(hi)[inner]
        x = k[a] ^ k[b - 1]
        m = np.empty(inner.size, np.int64)
        byk = x != 0
        if byk.any():                                     # split at the highest differing key bit
            bit = _bit_length(x[byk]) - 1
            pre = (k[b[byk] - 1] >> bit.astype(np.uint64)) << bit.astype(np.uint64)
            m[byk] = np.searchsorted(k, pre, "left")
        if (~byk).any():                                  # equal keys: the highest differing bit of the positions
            y = (a[~byk] ^ (b[~byk] - 1)).astype(np.uint64)
            bit = (_bit_length(y) - 1).astype(np.uint64)
            m[~byk] = (((b[~byk] - 1).astype(np.uint64) >> bit) << bit).astype(np.int64)
        assert ((m > a) & (m < b)).all()
        nxt = len(lo)
        new = []
        for j, n in enumerate(inner):
            child[n] = nxt + 2 * j
            lv = level[n] + 1
            lo += [int(a[j]), int(m[j])]; hi += [int(m[j]), int(b[j])]
            parent += [int(n), int(n)]; child += [0, 0]; level += [lv, lv]
            new += [nxt + 2 * j, nxt + 2 * j + 1]
        cur = np.array(new)
    N = len(lo)
    assert N == 2 * P - 1
    return order, np.array(lo), np.array(hi), np.array(parent), np.array(child), np.array(level)


def _R(q):
    q = np.asarray(q, np.float64)
    n = np.linalg.norm(q, axis=1, keepdims=True)
    q = np.where(n > 0, q / np.where(n > 0, n, 1), np.array([1.0, 0, 0, 0]))
    r, x, y, z = q.T
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                     np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                     np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], 1)


def leaf_moments(log_scales, rotations, opacities):
    s = np.exp(np.asarray(log_scales, np.float64))
    R = _R(rotations)
    cov = np.einsum("nik,nk,njk->nij", R, s * s, R)
    A = s[:, 0] * s[:, 1] + s[:, 0] * s[:, 2] + s[:, 1] * s[:, 2]
    return cov, np.asarray(opacities, np.float64).reshape(-1) * A


def build(xyz, shs, opacities, log_scales, rotations):
    """-> dict(xyz, shs, opacities [N], log_scales, rotations, nodes, boxes, source, cov [N,3,3] float64 (the moment-
    matched covariance of every node; a leaf's own), W [N]).  Merged log_scales / rotations are left NaN: any
    eigendecomposition of cov is valid, so the tests compare cov instead."""
    xyz, shs = np.asarray(xyz, np.float32), np.asarray(shs, np.float32)
    opacities = np.asarray(opacities, np.float32).reshape(-1)
    log_scales, rotations = np.asarray(log_scales, np.float32), np.asarray(rotations, np.float32)
    P = len(xyz)
    order, lo, hi, parent, child, level = topology(xyz)
    N = 2 * P - 1
    leaf = hi - lo == 1
    source = np.where(leaf, order[np.minimum(lo, P - 1)], -1).astype(np.int32)
    height = np.zeros(N, np.int64)
    for lv in range(level.max(), 0, -1):
        at = np.nonzero(level == lv)[0]
        np.maximum.at(height, parent[at], height[at] + 1)
    nodes = np.stack([height, parent, np.arange(N), leaf, ~leaf, np.where(leaf, 0, child), np.where(leaf, 0, 2)], 1)

    # statistics of every node straight from its leaf set (sorted positions lo .. hi), one BFS level at a time
    covl, wl = leaf_moments(log_scales, rotations, opacities)
    mu_s, cov_s, w_s = xyz.astype(np.float64)[order], covl[order], wl[order]
    sh_s = shs.astype(np.float64)[order].reshape(P, -1)
    W = np.zeros(N); mu = np.zeros((N, 3)); cov = np.zeros((N, 3, 3)); sh = np.zeros((N, sh_s.shape[1]))
    for lv in range(level.max() + 1):
        at = np.nonzero(level == lv)[0]
        cnt = hi[at] - lo[at]
        seg = np.repeat(np.arange(at.size), cnt)
        pos = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt) + np.repeat(lo[at], cnt)
        w = w_s[pos]
        sw = np.bincount(seg, w, at.size)
        safe = np.where(sw > 0, sw, 1.0)
        m = np.stack([np.bincount(seg, w * mu_s[pos, a], at.size) for a in range(3)], 1) / safe[:, None]
        d = mu_s[pos] - m[seg]
        c = cov_s[pos] + d[:, :, None] * d[:, None, :]
        C = np.stack([np.bincount(seg, w * c[:, i, j], at.size) for i in range(3) for j in range(3)], 1).reshape(-1, 3, 3)
        S = np.stack([np.bincount(seg, w * sh_s[pos, e], at.size) for e in range(sh_s.shape[1])], 1)
        W[at], mu[at], cov[at], sh[at] = sw, m, C / safe[:, None, None], S / safe[:, None]
    li = np.nonzero(leaf)[0]                              # a leaf's moments are its own, whatever its weight
    mu[li], cov[li], sh[li] = xyz[source[li]], covl[source[li]], shs.reshape(P, -1)[source[li]]
    # W = 0: the unweighted mean of the two children's moments, deepest first
    for lv in range(level.max(), -1, -1):
        for n in np.nonzero((level == lv) & ~leaf & (W == 0))[0]:
            a, b = child[n], child[n] + 1
            mu[n] = (mu[a] + mu[b]) / 2
            da, db = mu[a] - mu[n], mu[b] - mu[n]
            cov[n] = ((cov[a] + np.outer(da, da)) + (cov[b] + np.outer(db, db))) / 2
            sh[n] = (sh[a] + sh[b]) / 2
    lam = np.maximum(np.linalg.eigvalsh(cov), EIG_FLOOR)
    sg = np.sqrt(lam)
    A = sg[:, 0] * sg[:, 1] + sg[:, 0] * sg[:, 2] + sg[:, 1] * sg[:, 2]

    out = dict(xyz=mu.astype(np.float32), shs=sh.reshape(N, -1, 3).astype(np.float32),
               opacities=(W / A).astype(np.float32), log_scales=np.full((N, 3), np.nan, np.float32),
               rotations=np.full((N, 4), np.nan, np.float32), nodes=nodes.astype(np.int32), source=source, cov=cov, W=W)
    li = np.nonzero(leaf)[0]
    for k, a in (("xyz", xyz), ("shs", shs), ("opacities", opacities), ("log_scales", log_scales), ("rotations", rotations)):
        out[k][li] = a[source[li]]
    # boxes: leaf mu +- 3 sqrt(diag Sigma_i) rounded to fp32, interior the union of the children
    bmin = np.zeros((N, 3), np.float32); bmax = np.zeros((N, 3), np.float32)
    ext = 3.0 * np.sqrt(np.diagonal(covl, 0, 1, 2))[source[li]]
    bmin[li] = (xyz[source[li]].astype(np.float64) - ext).astype(np.float32)
    bmax[li] = (xyz[source[li]].astype(np.float64) + ext).astype(np.float32)
    for lv in range(level.max(), -1, -1):
        at = np.nonzero((level == lv) & ~leaf)[0]
        bmin[at] = np.minimum(bmin[child[at]], bmin[child[at] + 1]); bmax[at] = np.maximum(bmax[child[at]], bmax[child[at] + 1])
    boxes = np.zeros((N, 2, 4), np.float32)
    boxes[:, 0, :3], boxes[:, 1, :3] = bmin, bmax
    boxes[:, 0, 3] = (bmax - bmin).max(1)
    out["boxes"] = boxes
    return out


def cov_of(log_scales, rotations):
    """covariance rebuilt from a row's (log_scale, rotation)"""
    s = np.exp(np.asarray(log_scales, np.float64))
    R = _R(rotations)
    return np.einsum("nik,nk,njk->nij", R, s * s, R)


# ---------------------------------------------------------------------------------------------------------------
# clouds
# ---------------------------------------------------------------------------------------------------------------
def cloud(P, seed=0, sh_coeffs=16, xyz=None, scale=-4.0):
    g = np.random.default_rng(seed)
    if xyz is None:
        xyz = g.uniform(-5, 5, (P, 3))
    q = g.standard_normal((P, 4)) * g.uniform(0.5, 2.0, (P, 1))         # any norm
    return dict(xyz=np.asarray(xyz, np.float32), shs=g.standard_normal((P, sh_coeffs, 3)).astype(np.float32),
                opacities=g.uniform(0.01, 1.0, P).astype(np.float32),
                log_scales=(scale + 0.5 * g.standard_normal((P, 3))).astype(np.float32), rotations=q.astype(np.float32))


def cases():
    g = np.random.default_rng(7)
    c = {f"P{P}": cloud(P, seed=P) for P in (1, 2, 3, 17, 1000)}
    c["identical"] = cloud(64, 1, xyz=np.tile([[1.5, -2.0, 3.25]], (64, 1)))
    base = g.uniform(-1, 1, (50, 3))
    c["duplicates"] = cloud(300, 2, xyz=base[g.integers(0, 50, 300)])
    t = g.uniform(-3, 3, 500)
    c["collinear"] = cloud(500, 3, xyz=np.stack([t, 2 * t + 1, -t], 1))
    uv = g.uniform(-3, 3, (700, 2))
    c["planar"] = cloud(700, 4, xyz=np.stack([uv[:, 0], uv[:, 1], 0.5 * uv[:, 0] - uv[:, 1] + 2], 1))
    c["two_clusters"] = cloud(600, 5, xyz=np.concatenate([g.normal(0, 0.1, (300, 3)), g.normal(1e4, 0.1, (300, 3))]))
    z = cloud(200, 6, sh_coeffs=4)
    z["opacities"][:] = 0
    c["zero_opacity"] = z
    c["sampled_large"] = sampled_large()[0]
    return c


def sampled_large(n=20000, seed=11):
    """many small Gaussians sampled from one large one -> (cloud, mean, covariance of the large one)"""
    g = np.random.default_rng(seed)
    mean = np.array([1.0, -2.0, 0.5])
    A = g.standard_normal((3, 3))
    cov = A @ A.T + 0.5 * np.eye(3)
    xyz = g.multivariate_normal(mean, cov, n)
    c = cloud(n, seed + 1, xyz=xyz, scale=-7.0)
    c["opacities"][:] = 0.5
    c["log_scales"][:] = -7.0                   # equal weights: the root moments are the sample moments
    return c, mean, cov

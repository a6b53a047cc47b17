"""The hierarchy merger restated from include/h3dgs.h (h3dgs_merge_hierarchies) in numpy, by different means than the
kernel: explicit per-subtree sets of leaf Gaussians (built by recursion over the children lists, not by parent walks
or pointer jumping), purity and item moments as direct sums over those sets, and the top tree from
tests/hier_build_ref.py (top-down radix split, per-node sums over each node's item set).  Also the test scenes."""
import numpy as np

import hier_build_ref as hb

F = np.float32


def owners(xy, cells):
    """the owning chunk of every point: the smallest (k1, k2, j), fp32, every operation rounded"""
    xy = np.asarray(xy, F)
    cells = np.asarray(cells, F).reshape(-1, 4)
    best = np.zeros(len(xy), np.int64)
    b1 = np.full(len(xy), np.inf, F)
    b2 = np.full(len(xy), np.inf, F)
    for j, (cx, cy, ex, ey) in enumerate(cells):
        ax, ay = np.abs(xy[:, 0] - cx), np.abs(xy[:, 1] - cy)
        ox = np.maximum(ax - F(0.5) * ex, F(0))
        oy = np.maximum(ay - F(0.5) * ey, F(0))
        k1 = ox * ox + oy * oy
        k2 = np.maximum(ax / ex, ay / ey)
        better = (k1 < b1) | ((k1 == b1) & (k2 < b2)) if j else np.ones(len(xy), bool)
        best[better], b1[better], b2[better] = j, k1[better], k2[better]
    return best


def _subtree_sets(nodes):
    """-> list of sorted arrays: the leaf Gaussian rows (chunk-local) in every node's subtree"""
    N = nodes.shape[0]
    out = [None] * N
    roots = [n for n in range(N) if nodes[n, 1] == -1]
    for r in roots:
        stack = [(r, False)]
        while stack:
            n, done = stack.pop()
            s, cc = int(nodes[n, 5]), int(nodes[n, 6])
            if not done:
                stack.append((n, True))
                stack.extend((k, False) for k in range(s, s + cc))
                continue
            own = np.arange(nodes[n, 2], nodes[n, 2] + nodes[n, 3], dtype=np.int64)
            out[n] = np.sort(np.concatenate([own] + [out[k] for k in range(s, s + cc)]))
    return out


def _descendants(nodes, n):
    out, stack = [], [n]
    while stack:
        m = stack.pop()
        out.append(m)
        stack.extend(range(int(nodes[m, 5]), int(nodes[m, 5] + nodes[m, 6])))
    return out


def item_moments(xyz, shs, opac, ls, rot):
    """W, mu, cov, sh of one set of Gaussians (the creator's formulas, direct sums; W = 0: the unweighted mean)"""
    cov, w = hb.leaf_moments(ls, rot, opac)
    x = xyz.astype(np.float64)
    sh = shs.reshape(len(x), -1).astype(np.float64)
    W = w.sum()
    f = w if W > 0 else np.ones_like(w)
    D = f.sum()
    mu = (f[:, None] * x).sum(0) / D
    d = x - mu
    C = (f[:, None, None] * (cov + d[:, :, None] * d[:, None, :])).sum(0) / D
    return W, mu, C, (f[:, None] * sh).sum(0) / D


def merge(chunks, cells):
    """chunks: dicts of numpy arrays (xyz, shs [M,16,3], opacities [M], log_scales, rotations, nodes, boxes).
    -> dict(xyz, shs, opacities, log_scales, rotations, nodes, boxes, source_chunk, source_row, R, T, top_cov [T,3,3],
    top_W [T], top_interior and single (the output nodes that are top interior nodes / one-Gaussian items)); merged top rows' log_scales / rotations are NaN (compare top_cov)."""
    cells = np.asarray(cells, F).reshape(-1, 4)
    whole, single = [], []
    kept_nonroot = []   # (chunk, node)
    for c, ch in enumerate(chunks):
        nodes = ch["nodes"]
        N = nodes.shape[0]
        sets = _subtree_sets(nodes)
        own_leaf = np.zeros(ch["xyz"].shape[0], bool)
        leaf_rows = np.concatenate([np.arange(nodes[n, 2], nodes[n, 2] + nodes[n, 3]) for n in range(N)]).astype(np.int64) \
            if N else np.zeros(0, np.int64)
        owner = owners(ch["xyz"][leaf_rows, :2], cells)
        own_leaf[leaf_rows[owner == c]] = True
        pure = np.array([own_leaf[sets[n]].all() for n in range(N)])
        has = np.array([sets[n].size > 0 for n in range(N)])
        for n in range(N):
            p = nodes[n, 1]
            if pure[n] and has[n] and (p == -1 or not pure[p]):
                whole.append((c, n))
                kept_nonroot += [(c, m) for m in _descendants(nodes, n) if m != n]
            if not pure[n]:
                single += [(c, int(r)) for r in range(nodes[n, 2], nodes[n, 2] + nodes[n, 3]) if own_leaf[r]]
    kept_nonroot.sort()
    single.sort()
    items = [("w", c, n) for c, n in whole] + [("s", c, r) for c, r in single]
    R = len(items)
    assert R > 0
    # item moments, positions, boxes, depths
    Wi, mui, covi, shi = np.zeros(R), np.zeros((R, 3)), np.zeros((R, 3, 3)), np.zeros((R, 48))
    boxi, depthi = np.zeros((R, 2, 4), F), np.zeros(R, np.int64)
    for i, (kind, c, k) in enumerate(items):
        ch = chunks[c]
        rows = _subtree_sets(ch["nodes"])[k] if kind == "w" else np.array([k])
        Wi[i], mui[i], covi[i], shi[i] = item_moments(ch["xyz"][rows], ch["shs"][rows], ch["opacities"][rows],
                                                      ch["log_scales"][rows], ch["rotations"][rows])
        if kind == "w":
            boxi[i], depthi[i] = ch["boxes"][k], ch["nodes"][k, 0]
        else:
            cv, _ = hb.leaf_moments(ch["log_scales"][[k]], ch["rotations"][[k]], ch["opacities"][[k]])
            ext = 3.0 * np.sqrt(np.diagonal(cv[0]))
            x = ch["xyz"][k].astype(np.float64)
            boxi[i, 0, :3], boxi[i, 1, :3] = (x - ext).astype(F), (x + ext).astype(F)
            boxi[i, 0, 3] = (boxi[i, 1, :3] - boxi[i, 0, :3]).max()
    pos = mui.astype(F)
    # the top tree
    order, lo, hi, parent, child, level = hb.topology(pos)
    T = 2 * R - 1
    leaf = hi - lo == 1
    slot_item = np.where(leaf, order[np.minimum(lo, R - 1)], -1)
    depth = np.zeros(T, np.int64)
    depth[leaf] = depthi[slot_item[leaf]]
    for lv in range(level.max(), -1, -1):
        at = np.nonzero((level == lv) & ~leaf)[0]
        depth[at] = 1 + np.maximum(depth[child[at]], depth[child[at] + 1])
    W, mu, cov, sh = np.zeros(T), np.zeros((T, 3)), np.zeros((T, 3, 3)), np.zeros((T, 48))
    for p in range(T):
        its = order[lo[p]:hi[p]]
        w = Wi[its]
        W[p] = w.sum()
        if W[p] > 0:
            mu[p] = (w[:, None] * mui[its]).sum(0) / W[p]
            d = mui[its] - mu[p]
            cov[p] = (w[:, None, None] * (covi[its] + d[:, :, None] * d[:, None, :])).sum(0) / W[p]
            sh[p] = (w[:, None] * shi[its]).sum(0) / W[p]
    for lv in range(level.max(), -1, -1):                # W = 0: the unweighted mean of the two children, deepest first
        for p in np.nonzero(level == lv)[0]:
            if leaf[p]:
                i = slot_item[p]
                mu[p], cov[p], sh[p] = mui[i], covi[i], shi[i]
            elif W[p] == 0:
                a, b = child[p], child[p] + 1
                mu[p] = (mu[a] + mu[b]) / 2
                da, db = mu[a] - mu[p], mu[b] - mu[p]
                cov[p] = ((cov[a] + np.outer(da, da)) + (cov[b] + np.outer(db, db))) / 2
                sh[p] = (sh[a] + sh[b]) / 2
    tbox = np.zeros((T, 2, 4), F)
    tbox[leaf] = boxi[slot_item[leaf]]
    for lv in range(level.max(), -1, -1):
        at = np.nonzero((level == lv) & ~leaf)[0]
        tbox[at, 0, :3] = np.minimum(tbox[child[at], 0, :3], tbox[child[at] + 1, 0, :3])
        tbox[at, 1, :3] = np.maximum(tbox[child[at], 1, :3], tbox[child[at] + 1, 1, :3])
        tbox[at, 0, 3] = (tbox[at, 1, :3] - tbox[at, 0, :3]).max(1)
        tbox[at, 1, 3] = 0
    # output nodes: the top tree, then the kept non-root nodes
    out_of = {}
    for p in np.nonzero(leaf)[0]:
        kind, c, k = items[slot_item[p]]
        if kind == "w":
            out_of[(c, k)] = int(p)
    for j, key in enumerate(kept_nonroot):
        out_of[key] = T + j
    NO = T + len(kept_nonroot)
    single = np.array([p for p in np.nonzero(leaf)[0] if items[slot_item[p]][0] == "s"], np.int64)
    src = []            # per output node: ("top", p) | ("single", c, r) | ("node", c, n)
    for p in range(T):
        if not leaf[p]:
            src.append(("top", p))
        else:
            kind, c, k = items[slot_item[p]]
            src.append(("single", c, k) if kind == "s" else ("node", c, k))
    src += [("node", c, n) for c, n in kept_nonroot]
    cnt = np.array([1 if s[0] != "node" else int(chunks[s[1]]["nodes"][s[2], 3] + chunks[s[1]]["nodes"][s[2], 4]) for s in src])
    starts = np.cumsum(cnt) - cnt
    RO = int(cnt.sum())
    starts = np.where(cnt > 0, starts, np.minimum(starts, RO - 1))
    nodes = np.zeros((NO, 7), np.int64)
    boxes = np.zeros((NO, 2, 4), F)
    sc_, sr_ = np.full(RO, -1, np.int32), np.full(RO, -1, np.int32)
    rows = {k: np.zeros((RO,) + s, F) for k, s in (("xyz", (3,)), ("shs", (16, 3)), ("opacities", ()), ("log_scales", (3,)),
                                                   ("rotations", (4,)))}
    for o, s in enumerate(src):
        st = starts[o]
        if s[0] == "top":
            p = s[1]
            nodes[o] = [depth[p], parent[p], st, 0, 1, child[p], 2]
            boxes[o] = tbox[p]
            rows["xyz"][st] = mu[p].astype(F)
            rows["shs"][st] = sh[p].reshape(16, 3).astype(F)
            lam = np.sqrt(np.maximum(np.linalg.eigvalsh(cov[p]), hb.EIG_FLOOR))
            rows["opacities"][st] = F(W[p] / (lam[0] * lam[1] + lam[0] * lam[2] + lam[1] * lam[2]))
            rows["log_scales"][st] = np.nan
            rows["rotations"][st] = np.nan
        elif s[0] == "single":
            _, c, r = s
            nodes[o] = [0, parent[o], st, 1, 0, 0, 0]
            boxes[o] = tbox[o]
            sc_[st], sr_[st] = c, r
        else:
            _, c, n = s
            nd = chunks[c]["nodes"][n]
            par = parent[o] if o < T else out_of[(c, int(nd[1]))]
            nodes[o] = [nd[0], par, st, nd[3], nd[4], out_of[(c, int(nd[5]))] if nd[6] > 0 else 0, nd[6]]
            boxes[o] = chunks[c]["boxes"][n]
            k = int(nd[3] + nd[4])
            sc_[st:st + k], sr_[st:st + k] = c, np.arange(nd[2], nd[2] + k)
    for k in rows:
        for c, ch in enumerate(chunks):
            sel = sc_ == c
            rows[k][sel] = ch[k][sr_[sel]]
    out = dict(rows, nodes=nodes.astype(np.int32), boxes=boxes, source_chunk=sc_, source_row=sr_, R=R, T=T,
               top_cov=cov, top_W=W, top_interior=np.nonzero(~leaf)[0], single=single)
    return out


# ---------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------
def grid_cells(nx, ny, size=4.0, skip=()):
    """cells of an nx x ny grid of size x size chunks centred on the origin, row-major; `skip` drops (i, j) cells"""
    out = []
    for j in range(ny):
        for i in range(nx):
            if (i, j) not in skip:
                out.append([(i - (nx - 1) / 2) * size, (j - (ny - 1) / 2) * size, size, size])
    return np.array(out, F)


def chunk_cloud(cell, P, seed, spill=0.25, sh_coeffs=16):
    """a chunk's trained cloud: uniform over its cell widened by `spill` of the width on every side"""
    g = np.random.default_rng(seed)
    cx, cy, ex, ey = (float(v) for v in cell)
    xyz = np.stack([g.uniform(cx - (0.5 + spill) * ex, cx + (0.5 + spill) * ex, P),
                    g.uniform(cy - (0.5 + spill) * ey, cy + (0.5 + spill) * ey, P), g.uniform(-1.0, 1.0, P)], 1)
    return hb.cloud(P, seed=seed + 1000, sh_coeffs=sh_coeffs, xyz=xyz)

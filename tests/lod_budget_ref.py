"""numpy restatement of the LOD budget (csrc/lod_budget.cu, include/h3dgs.h h3dgs_lod_budget), brute force.

R(t) is the cut's row count at threshold t, from the per-node predicate of the cut (sizes from hier_general.node_sizes,
the restatement of the oracle's node_size).  The threshold a budget B selects is the smallest float32 t in
[floor, t_max], t_max = max(floor, the largest finite size), with R(t) <= B; R is constant between consecutive distinct
sizes, so it is the smallest feasible one of the candidates floor and nextafter(s, +inf) for each size s in
[floor, t_max).  When none is feasible the answer is t_max and the budget is unmet."""
import numpy as np

import hier_general as hg


def rows_per_node(nodes, size, t):
    """the cut's rows of every node at threshold t"""
    t = np.float32(t)
    depth, parent, _, cl, cm = (nodes[:, i].astype(np.int64) for i in range(5))
    has = parent >= 0
    q = np.where(has, size[np.maximum(parent, 0)], np.float32(np.nan))
    coarse = size >= t
    mid = ~coarse & has & (q >= t)
    return np.where(coarse, cl, np.where(mid, cl + np.where(depth != 0, cm, 0), 0))


def rows(nodes, size, t):
    return int(rows_per_node(nodes, size, t).sum())


def rows_by_keys(nodes, size, t):
    """the same count as a sum of step weights w [t <= key] over node sizes (the derivation the kernel computes): a node
    with a non-empty middle interval puts -[d != 0] cm at its size and cl + [d != 0] cm at its parent's, any other node
    cl at its own size"""
    t = np.float32(t)
    depth, parent, _, cl, cm = (nodes[:, i].astype(np.int64) for i in range(5))
    has = parent >= 0
    q = np.where(has, size[np.maximum(parent, 0)], np.float32(np.nan))
    cmd = np.where(depth != 0, cm, 0)
    split = has & ~(size >= q) & ~np.isnan(q)
    own = np.where(split, -cmd, cl)
    return int((own * (t <= size)).sum() + ((cl + cmd) * (split & (t <= q))).sum())


def t_max(size, floor):
    floor = np.float32(floor)
    fin = size[np.isfinite(size) & (size >= floor)]
    return np.float32(fin.max() + np.float32(0)) if fin.size else floor


def candidates(size, floor):
    """floor, then nextafter(s, +inf) for each distinct finite size s in [floor, t_max), ascending"""
    floor = np.float32(floor)
    tm = t_max(size, floor)
    s = np.unique(size[np.isfinite(size) & (size >= floor) & (size < tm)])
    nxt = np.nextafter(s, np.float32(np.inf)).astype(np.float32)
    return [floor] + [np.float32(x) for x in nxt]


def table(nodes, boxes, viewpoint, floor):
    """-> (candidates, R at each, sizes)"""
    size = hg.node_sizes(boxes, viewpoint)
    cands = candidates(size, floor)
    return cands, np.array([rows(nodes, size, t) for t in cands], np.int64), size


def select(nodes, boxes, viewpoint, floor, budget, tab=None):
    """-> dict(threshold, rows, unmet, kept, total): what h3dgs_lod_budget writes (tab: table() of the same inputs)"""
    cands, r, size = tab if tab is not None else table(nodes, boxes, viewpoint, floor)
    floor = np.float32(floor)
    kept, total = int((size >= floor).sum()), int(r[0])
    ok = np.nonzero(r <= budget)[0]
    if ok.size:
        return dict(threshold=cands[ok[0]], rows=int(r[ok[0]]), unmet=0, kept=kept, total=total)
    tm = t_max(size, floor)
    return dict(threshold=tm, rows=rows(nodes, size, tm), unmet=1, kept=kept, total=total)


def budgets(nodes, tab, floor, limit=None):
    """0, every R(candidate) and one either side, one above R(floor), and R(t_max) - 1 (unmet when positive); with
    limit, an even sample of the ones around R(candidate), the others always kept"""
    cands, r, size = tab
    r_max = rows(nodes, size, t_max(size, floor))
    special = {0, int(r[0]) + 7, r_max - 1, r_max}
    near = set()
    for x in set(int(v) for v in r):
        near |= {x - 1, x, x + 1}
    near = sorted(near - special)
    if limit and len(near) > limit:
        near = [near[i] for i in np.unique(np.linspace(0, len(near) - 1, limit).round().astype(int))]
    return sorted(b for b in special | set(near) if b >= 0)


# ---------------------------------------------------------------------------------------------------------------
# the hierarchies, viewpoints and floors the CPU and GPU tests share
# ---------------------------------------------------------------------------------------------------------------
def odd_sizes(h, seed=0):
    """h with boxes whose sizes are NaN (NaN extent), +inf and -inf (zero distance is impossible outside a box, so a
    +-inf extent), negative, zero, and duplicated (copies of other nodes' boxes)"""
    rng = np.random.default_rng(seed)
    b = h["boxes"].copy()
    N = b.shape[0]
    pick = lambda k: rng.choice(np.arange(1, N), size=min(k, N - 1), replace=False)
    for val, k in ((np.nan, 6), (np.inf, 4), (-np.inf, 3), (-0.5, 4), (0.0, 4), (-0.0, 3)):
        b[pick(k), 0, 3] = np.float32(val)
    dst, src = pick(N // 5), pick(N // 5)
    b[dst] = b[src]
    return dict(h, boxes=b)


def scenes(cam):
    """(name, hierarchy dict with nodes and boxes) -- creator-built, general (tests/hier_general.py), single-node, and
    with odd sizes"""
    from h3dgs import synth
    out = [("creator", synth.build_hierarchy(synth.cloud_v1(200, cam, zmin=2.0, zmax=30.0, seed=21)))]
    for n in (2, 5, 300, 1025):
        out.append((f"general{n}", hg.dense_hierarchy(n, n, cam)))
    single = dict(nodes=np.array([[0, -1, 0, 1, 0, 0, 0]], np.int32),
                  boxes=np.array([[[-0.2, -0.2, 4.0, 0.4], [0.2, 0.2, 4.4, 0.0]]], np.float32))
    out.append(("single", single))
    out.append(("odd", odd_sizes(hg.dense_hierarchy(7, 600, cam), 1)))
    out.append(("odd_creator", odd_sizes(out[0][1], 2)))
    return out


def views(h, cam):
    """the viewpoints of hier_general (outside, inside the root, inside a deep leaf, on a face); the camera and a point
    inside the box for a single node"""
    if h["nodes"].shape[0] == 1:
        return dict(outside=np.asarray(cam.camera_center, np.float32), root=np.array([0, 0, 4.2], np.float32))
    return hg.viewpoints(h, cam)


def floors(h, vp, cam):
    """0, -0, the thresholds of tau 0 and 6, and a node's own size (a floor tied with a key)"""
    from h3dgs import synth
    size = hg.node_sizes(h["boxes"], vp)
    fin = size[np.isfinite(size) & (size > 0)]
    out = [np.float32(0.0), np.float32(-0.0), np.float32(synth.tau_threshold(0.0, cam)),
           np.float32(synth.tau_threshold(6.0, cam))]
    if fin.size:
        out.append(np.float32(np.sort(fin)[fin.size // 3]))
    return out

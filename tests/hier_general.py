"""General hierarchies for the LOD-cut tests, and an independent numpy statement of the cut.

synth.build_hierarchy makes a complete binary tree whose Gaussian row equals the node id, with one Gaussian per
node.  Hierarchies read from .hier files need not look like that: a node may hold several Gaussians (count_leafs
leaf Gaussians followed by count_merged merged ones), fan-out varies, and a node's block of rows sits anywhere.
general_hierarchy builds trees of that kind (same dict layout as synth.build_hierarchy, so synth.append_skybox
works on them); cut / weights / check_cut_invariant restate the cut from include/h3dgs.h and the predicate in
csrc/hierarchy.cu's header comment, in float32 with the kernel's order of operations, so that they can be
compared with the kernel and the oracle bit for bit."""
import random
from collections import deque

import numpy as np

from h3dgs import synth

FLT_MAX = np.float32(np.finfo(np.float32).max)


def _structure(rng, n_nodes, leaf_p, wide_p):
    """BFS-numbered tree with exactly n_nodes nodes: children of a node are contiguous, fan-out 1..8 (1 = a chain
    link) and now and then 12..16; a node becomes a leaf with probability leaf_p, so leaves sit at different heights."""
    r = random.Random(int(rng.integers(1 << 62)))
    parent = np.full(n_nodes, -1, np.int64)
    first = np.zeros(n_nodes, np.int64)
    nkids = np.zeros(n_nodes, np.int64)
    level = np.zeros(n_nodes, np.int64)
    queue, nxt = deque([0]), 1
    while queue:
        n = queue.popleft()
        left = n_nodes - nxt
        if left == 0 or (queue and r.random() < leaf_p):
            continue
        f = r.randint(12, 16) if r.random() < wide_p else r.choice((1, 1, 2, 2, 3, 3, 4, 4, 5, 6, 7, 8))
        f = min(f, left)
        first[n], nkids[n] = nxt, f
        parent[nxt:nxt + f], level[nxt:nxt + f] = n, level[n] + 1
        queue.extend(range(nxt, nxt + f))
        nxt += f
    assert nxt == n_nodes
    return parent, first, nkids, level


def _preorder(first, nkids):
    out, stack = [], [0]
    while stack:
        n = stack.pop()
        out.append(n)
        stack.extend(range(first[n] + nkids[n] - 1, first[n] - 1, -1))
    return np.array(out, np.int64)


def general_hierarchy(rng, n_nodes, cam, leaf_p=0.3, wide_p=0.03, leaf_leafs=(1, 4), leaf_merged_p=0.25,
                      interior_merged=(1, 2), interior_leafs_p=0.08, empty_p=0.0, sh_degree=3, zmax=40.0, leaf_scale=4e-3, spread=1.15):
    """-> dict(means3D, scales, rotations, opacities, shs [R,...], nodes [n_nodes,7] i32, boxes [n_nodes,2,4] f32).

    Leaves hold leaf_leafs[0]..leaf_leafs[1] leaf Gaussians (from synth.cloud_v1, Morton-sorted and dealt out in
    depth-first order, so a subtree covers a compact region) and, with probability leaf_merged_p, one merged Gaussian
    as well (count_merged = 1: the entry the cut's depth != 0 gate skips).  Interior nodes hold interior_merged merged
    Gaussians and, with probability interior_leafs_p, 1..3 leaf Gaussians of their own.  With empty_p > 0 that share
    of the interior nodes below the root holds no Gaussian at all (their start is a valid row but means nothing).
    A node's rows are the block [start, start + count_leafs + count_merged), leaf Gaussians first; the blocks are
    stored in a shuffled order, so start is unrelated to the node id.  Boxes are nested (a parent's box is the
    union of its children's and of its own Gaussians' 3-sigma boxes), min.w is the largest extent: node sizes never
    increase from a parent to a child."""
    parent, first, nkids, level = _structure(rng, n_nodes, leaf_p, wide_p)
    N = n_nodes
    leaf = nkids == 0
    interior = ~leaf
    cl = np.zeros(N, np.int64)
    cm = np.zeros(N, np.int64)
    cl[leaf] = rng.integers(leaf_leafs[0], leaf_leafs[1] + 1, leaf.sum())
    cm[leaf] = rng.uniform(size=leaf.sum()) < leaf_merged_p
    cm[interior] = rng.integers(interior_merged[0], interior_merged[1] + 1, interior.sum())
    own = interior & (rng.uniform(size=N) < interior_leafs_p)
    cl[own] = rng.integers(1, 4, own.sum())
    if empty_p > 0:
        empty = interior & (rng.uniform(size=N) < empty_p)
        empty[0] = False
        cl[empty] = cm[empty] = 0
    # depth: 0 at leaves, else 1 + the maximum over the children (deepest level first)
    depth = np.zeros(N, np.int64)
    levels = [np.nonzero(level == d)[0] for d in range(int(level.max()) + 1)]
    for lv in reversed(levels[1:]):
        np.maximum.at(depth, parent[lv], depth[lv] + 1)

    # leaf Gaussians: cloud_v1, Morton-sorted, dealt out in preorder
    L = int(cl.sum())
    cloud = synth.cloud_v1(L, cam, sh_degree=sh_degree, zmin=2.0, zmax=zmax, seed=int(rng.integers(1 << 30)), scale_k=1.0,
                         spread=spread)
    z = cloud["means3D"][:, 2:3]
    cloud["scales"] = (leaf_scale * np.sqrt(2.0 * z) * np.exp(0.4 * rng.standard_normal((L, 3)))).astype(np.float32)
    order = np.argsort(synth._morton(cloud["means3D"]), kind="stable")
    cloud = {k: v[order] for k, v in cloud.items()}
    pre = _preorder(first, nkids)
    leaf_off = np.zeros(N, np.int64)
    leaf_off[pre] = np.cumsum(cl[pre]) - cl[pre]

    # subtree statistics over the leaf Gaussians below (and in) each node -> the merged Gaussians
    owner = np.repeat(pre, cl[pre])                                    # node of every cloud Gaussian
    K = cloud["shs"].shape[1]
    cnt = np.bincount(owner, minlength=N).astype(np.float64)
    s_mean = np.zeros((N, 3)); np.add.at(s_mean, owner, cloud["means3D"].astype(np.float64))
    s_op = np.zeros(N); np.add.at(s_op, owner, cloud["opacities"][:, 0].astype(np.float64))
    s_sh = np.zeros((N, K, 3)); np.add.at(s_sh, owner, cloud["shs"].astype(np.float64))
    lo = np.full((N, 3), np.inf); np.minimum.at(lo, owner, cloud["means3D"].astype(np.float64))
    hi = np.full((N, 3), -np.inf); np.maximum.at(hi, owner, cloud["means3D"].astype(np.float64))
    smax = np.zeros(N); np.maximum.at(smax, owner, cloud["scales"].max(1).astype(np.float64))
    for lv in reversed(levels[1:]):
        p = parent[lv]
        np.add.at(cnt, p, cnt[lv]); np.add.at(s_mean, p, s_mean[lv]); np.add.at(s_op, p, s_op[lv]); np.add.at(s_sh, p, s_sh[lv])
        np.minimum.at(lo, p, lo[lv]); np.maximum.at(hi, p, hi[lv]); np.maximum.at(smax, p, smax[lv])
    mnode = np.repeat(np.arange(N), cm)                                # node of every merged Gaussian
    mk = np.arange(mnode.size) - np.repeat(np.cumsum(cm) - cm, cm)     # its index inside the node
    c = cnt[mnode][:, None]
    span = (hi - lo)[mnode]
    merged = dict(means3D=s_mean[mnode] / c + 0.15 * mk[:, None] * span,
                  scales=np.maximum(0.1 * span, 1.5 * smax[mnode][:, None]) * np.ones((1, 3)),
                  rotations=np.tile([1.0, 0.0, 0.0, 0.0], (mnode.size, 1)),
                  opacities=np.minimum(0.95, 1.1 * s_op[mnode] / cnt[mnode])[:, None],
                  shs=s_sh[mnode] / c[:, :, None])

    # blocks in a shuffled order; leaf Gaussians first, then the merged ones
    count = cl + cm
    R = int(count.sum())
    place = rng.permutation(N)
    start = np.zeros(N, np.int64)
    start[place] = np.cumsum(count[place]) - count[place]
    start = np.minimum(start, R - 1)                                   # an empty node at the very end still points at a row
    row_node = np.repeat(place, count[place])
    within = np.arange(R) - start[row_node]
    is_leafg = within < cl[row_node]
    moff = np.cumsum(cm) - cm
    src_leaf = leaf_off[row_node] + within
    src_merged = moff[row_node] + within - cl[row_node]
    out = {}
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        a = cloud[k].astype(np.float64)
        b = merged[k].reshape((-1,) + a.shape[1:])
        sel = is_leafg.reshape((-1,) + (1,) * (a.ndim - 1))
        out[k] = np.where(sel, a[np.where(is_leafg, src_leaf, 0)],
                          b[np.where(is_leafg, 0, src_merged)] if b.shape[0] else 0.0).astype(np.float32)

    # nested boxes: own Gaussians' 3-sigma boxes, then the union over the children (deepest level first)
    ext = 3.0 * out["scales"].max(1, keepdims=True).astype(np.float64)
    bmin = np.full((N, 3), np.inf); np.minimum.at(bmin, row_node, out["means3D"] - ext)
    bmax = np.full((N, 3), -np.inf); np.maximum.at(bmax, row_node, out["means3D"] + ext)
    for lv in reversed(levels[1:]):
        np.minimum.at(bmin, parent[lv], bmin[lv]); np.maximum.at(bmax, parent[lv], bmax[lv])
    boxes = np.zeros((N, 2, 4), np.float32)
    boxes[:, 0, :3] = bmin; boxes[:, 1, :3] = bmax
    boxes[:, 0, 3] = (boxes[:, 1, :3] - boxes[:, 0, :3]).max(1)
    nodes = np.stack([depth, parent, start, cl, cm, np.where(leaf, 0, first), nkids], 1).astype(np.int32)
    out.update(nodes=nodes, boxes=boxes)
    return out


# ---------------------------------------------------------------------------------------------------------------
# the cut, restated (include/h3dgs.h; csrc/hierarchy.cu header comment), float32 throughout
# ---------------------------------------------------------------------------------------------------------------
def node_sizes(boxes, viewpoint):
    """min.w / distance from the viewpoint to the box, FLT_MAX when the viewpoint is inside (faces included).
    Operation order of the kernel: (cx*cx + cy*cy) + cz*cz, sqrt, division -- each correctly rounded in float32."""
    v = np.asarray(viewpoint, np.float32).reshape(1, 3)
    mn, mx = boxes[:, 0, :3], boxes[:, 1, :3]
    inside = ((v >= mn) & (v <= mx)).all(1)
    c = np.maximum(mn, np.minimum(mx, v)) - v
    d2 = (c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1]) + c[:, 2] * c[:, 2]
    with np.errstate(divide="ignore"):
        size = boxes[:, 0, 3] / np.sqrt(d2)
    return np.where(inside, FLT_MAX, size).astype(np.float32)


def cut(nodes, boxes, target, viewpoint):
    """expand_to_size -> (n, render_indices, parent_indices, nodes_for_render).  A node emits its count_leafs leaf
    Gaussians when it is at least as coarse as the target; a node finer than the target whose parent is not emits
    count_leafs + count_merged (count_merged only when it is not a leaf).  Rows come in node order."""
    target = np.float32(target)
    size = node_sizes(boxes, viewpoint)
    depth, parent, start, cl, cm = (nodes[:, i].astype(np.int64) for i in range(5))
    has_parent = parent >= 0
    psize = np.where(has_parent, size[np.maximum(parent, 0)], np.float32(0))
    coarse = size >= target
    on_cut = ~coarse & has_parent & (psize >= target)
    count = np.where(coarse, cl, np.where(on_cut, cl + np.where(depth != 0, cm, 0), 0))
    ni = np.repeat(np.arange(nodes.shape[0]), count)
    q = np.arange(ni.size) - np.repeat(np.cumsum(count) - count, count)
    ri = start[ni] + q
    pg = np.where(has_parent, start[np.maximum(parent, 0)], -1)
    return int(ni.size), ri.astype(np.int32), pg[ni].astype(np.int32), ni.astype(np.int32)


def weights(node_indices, target, nodes, boxes, viewpoint):
    """get_interpolation_weights -> (t, kids): t = 1 without a parent or when the parent is coarser than twice the
    target, else max(0, 1 - max(0, target - s0) / (psize - s0)) with s0 = max(psize / 2, size) (1 when that span
    is empty); kids = the parent's count_children (1 without a parent)."""
    target = np.float32(target)
    ni = np.asarray(node_indices, np.int64)
    size = node_sizes(boxes, viewpoint)
    parent = nodes[ni, 1].astype(np.int64)
    has_parent = parent >= 0
    ps = np.where(has_parent, size[np.maximum(parent, 0)], np.float32(0))
    s = size[ni]
    s0 = np.maximum(np.float32(0.5) * ps, s)
    diff = ps - s0
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.maximum(np.float32(1) - np.maximum(np.float32(0), target - s0) / diff, np.float32(0))
    t = np.where(~has_parent | (ps > np.float32(2) * target) | (diff <= 0), np.float32(1), t).astype(np.float32)
    kids = np.where(has_parent, nodes[np.maximum(parent, 0), 6], 1).astype(np.int32)
    return t, kids


def check_cut_invariant(nodes, boxes, target, viewpoint, ri, ni):
    """The cut stated path by path, independent of any implementation.  Sizes never increase from a parent to a
    child (asserted), so a root-to-leaf path crosses the target at most once.  On a path whose root is at or above
    the target exactly one node is selected -- the first one below the target, or the leaf if there is none -- and
    emits its rows; the nodes above it emit their leaf Gaussians (count_leafs) and the nodes below it nothing.  A
    path whose root is already below the target selects nothing.  Rows come in node order, start .. start+count-1."""
    target = np.float32(target)
    size = node_sizes(boxes, viewpoint)
    N = nodes.shape[0]
    depth, parent, start, cl, cm, _, nkids = (nodes[:, i].astype(np.int64) for i in range(7))
    has_parent = parent >= 0
    assert (size[has_parent] <= size[parent[has_parent]]).all(), "boxes are not nested"
    ni = np.asarray(ni, np.int64)
    assert (np.diff(ni) >= 0).all(), "rows are not in node order"
    got = np.bincount(ni, minlength=N)
    q = np.arange(ni.size) - np.repeat(np.cumsum(got) - got, got)
    assert np.array_equal(np.asarray(ri, np.int64), start[ni] + q)
    want = np.full(N, -1, np.int64)
    for leafnode in np.nonzero(nkids == 0)[0]:
        path = [int(leafnode)]
        while parent[path[-1]] >= 0:
            path.append(int(parent[path[-1]]))
        path.reverse()
        if size[path[0]] < target:
            exp = [0] * len(path)
        else:
            below = [i for i, n in enumerate(path) if size[n] < target]
            s = below[0] if below else len(path) - 1
            exp = [int(cl[n]) for n in path[:s]]
            n = path[s]
            exp.append(int(cl[n] + (cm[n] if depth[n] != 0 else 0)) if size[n] < target else int(cl[n]))
            exp += [0] * (len(path) - s - 1)
        for n, e in zip(path, exp):
            assert want[n] in (-1, e), ("paths disagree", n)
            want[n] = e
    assert (want >= 0).all()
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, ("emitted rows per node differ", bad[:10], got[bad[:10]], want[bad[:10]])


# ---------------------------------------------------------------------------------------------------------------
# scenes, viewpoints and thresholds the tests share
# ---------------------------------------------------------------------------------------------------------------
def dense_hierarchy(seed, n_nodes, cam, **kw):
    """a compact cloud in front of the camera whose cut lands inside the tree (0 < t < 1 rows at tau 6 .. 15)"""
    kw = dict(dict(zmax=10.0, leaf_scale=3e-3, spread=0.5), **kw)
    return general_hierarchy(np.random.default_rng(seed), n_nodes, cam, **kw)


def viewpoints(h, cam):
    """outside every box (the camera), inside the root box, inside a deepest leaf's box, on a face of a mid-level box"""
    nodes, boxes = h["nodes"], h["boxes"]
    N = nodes.shape[0]
    center = lambda n: ((boxes[n, 0, :3].astype(np.float64) + boxes[n, 1, :3]) / 2).astype(np.float32)
    lvl = np.zeros(N, np.int64)
    for n in range(1, N):
        lvl[n] = lvl[nodes[n, 1]] + 1
    leaves = np.nonzero(nodes[:, 6] == 0)[0]
    deep = int(leaves[np.argmax(lvl[leaves])])
    mid = int(np.argmin(np.abs(lvl - lvl.max() // 2) + (nodes[:, 6] == 0) * N))
    face = center(mid)
    face[0] = boxes[mid, 0, 0]                                 # exactly on the min-x face
    return dict(outside=np.asarray(cam.camera_center, np.float32), root=center(0), leaf=center(deep), face=face)


def tie_thresholds(h, vp):
    """thresholds equal to the float32 size of a node on a finite path (size >= target and psize >= target ties) and
    to half its parent's size (psize > 2 * target tie)"""
    size = node_sizes(h["boxes"], vp)
    parent = h["nodes"][:, 1]
    ok = np.nonzero((parent >= 0) & (size < FLT_MAX))[0]
    ok = ok[size[parent[ok]] < FLT_MAX]
    if ok.size == 0:
        return []
    n = int(ok[ok.size // 2])
    ps = size[parent[n]]
    return [size[n], ps, np.float32(0.5) * ps]

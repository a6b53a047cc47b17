"""GPU: the hierarchy creator (csrc/hier_build.cu on the H100) -- the CPU suite's cases against the numpy restatement;
the benchmark clouds at full size (structural invariants, repeat-call identity, output on the input's device); target
size 0 renders exactly what the flat cloud renders; a post-optimisation loop on a built hierarchy reduces the loss; the
command-line creator end to end."""
import os
import sys

import numpy as np
import pytest

import hier_build_ref as ref
from test_hier_build_cpu import CASES, bits, built_scene, check_against_ref, write_ply

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def build_np(c):
    import torch
    from h3dgs.hier_build import build_hierarchy
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in c.items()}
    h = build_hierarchy(t["xyz"], t["shs"], t["opacities"], t["log_scales"], t["rotations"])
    out = {k: v.cpu().numpy() for k, v in h.items()}
    out["opacities"] = out["opacities"][:, 0]
    return out


@pytest.mark.parametrize("name", list(CASES) + ["P65537"])
def test_matches_the_restatement(name):
    c = CASES[name] if name in CASES else ref.cloud(65537, seed=3)
    check_against_ref(build_np(c), c)


def check_structure(h, c):
    """vectorised invariants of a built hierarchy of P input rows"""
    P = c["xyz"].shape[0]
    N = 2 * P - 1
    nodes, boxes, src = h["nodes"], h["boxes"], h["source"]
    assert nodes.shape == (N, 7) and h["xyz"].shape == (N, 3) and boxes.shape == (N, 2, 4)
    leaf = nodes[:, 6] == 0
    assert leaf.sum() == P and np.array_equal(np.sort(src[leaf]), np.arange(P)) and (src[~leaf] == -1).all()
    assert np.array_equal(nodes[:, 2], np.arange(N)) and nodes[0, 1] == -1
    assert np.array_equal(nodes[:, 3], leaf.astype(np.int32)) and np.array_equal(nodes[:, 4], (~leaf).astype(np.int32))
    inner = np.nonzero(~leaf)[0]
    assert (nodes[inner, 6] == 2).all() and (nodes[leaf, 5] == 0).all()
    a, b = nodes[inner, 5], nodes[inner, 5] + 1
    assert (a > inner).all() and (nodes[a, 1] == inner).all() and (nodes[b, 1] == inner).all()
    assert np.array_equal(np.sort(np.concatenate([a, b])), np.arange(1, N))            # every node but the root once
    assert (np.diff(a) > 0).all()                                                       # BFS: children in parent order
    assert np.array_equal(nodes[inner, 0], 1 + np.maximum(nodes[a, 0], nodes[b, 0])) and (nodes[leaf, 0] == 0).all()
    assert (boxes[inner, 0, :3] == np.minimum(boxes[a, 0, :3], boxes[b, 0, :3])).all()
    assert (boxes[inner, 1, :3] == np.maximum(boxes[a, 1, :3], boxes[b, 1, :3])).all()
    s = src[leaf]
    for k in ("xyz", "log_scales", "rotations", "opacities"):
        assert np.array_equal(bits(h[k][leaf]), bits(c[k][s])), k
    assert np.isfinite(h["xyz"]).all() and np.isfinite(h["log_scales"]).all() and np.isfinite(h["opacities"]).all()


def bench_cloud(n, seed):
    import bench_hier_build
    return bench_hier_build.cloud(n, seed)


@pytest.mark.parametrize("n,seed", [(1_000_000, 0), (1_500_000, 1), (4_000_000, 2)])
def test_bench_clouds(n, seed):
    import torch
    from h3dgs.hier_build import build_hierarchy
    c = bench_cloud(n, seed)
    t = {k: torch.from_numpy(v).cuda() for k, v in c.items()}
    h1 = build_hierarchy(t["xyz"], t["shs"], t["opacities"], t["log_scales"], t["rotations"])
    assert all(v.device == t["xyz"].device for v in h1.values())
    h1 = {k: v.cpu().numpy() for k, v in h1.items()}
    h2 = build_hierarchy(t["xyz"], t["shs"], t["opacities"], t["log_scales"], t["rotations"])
    for k, v in h2.items():
        assert v.cpu().numpy().tobytes() == h1[k].tobytes(), k
    h1["opacities"] = h1["opacities"][:, 0]
    check_structure(h1, c)


def test_target_zero_renders_the_flat_cloud():
    """at target size 0 every node emits its leaf Gaussians with t = 1: the render_post flow draws the input cloud"""
    import torch
    from h3dgs import pipeline, synth
    rng = np.random.default_rng(3)
    src = None

    def with_distinct_depths(c):
        nonlocal src
        c = dict(c)
        c["xyz"] = c["xyz"].copy()
        c["xyz"][:, 2] = (2.0 + 28.0 * rng.permutation(len(c["xyz"])) / len(c["xyz"])).astype(np.float32)
        src = c
        return build_np(c)
    cam, h = built_scene(with_distinct_depths, n=3000, seed=4)
    flat = dict(means3D=src["xyz"], scales=np.exp(src["log_scales"]), rotations=src["rotations"],
                opacities=src["opacities"][:, None], shs=src["shs"])
    dcam = pipeline.DeviceCamera(cam)
    bg = torch.zeros(3, device="cuda")
    with torch.no_grad():
        img_h, _, n = pipeline.render_hier(pipeline.Scene(h, requires_grad=False), dcam, bg, 0.0)
        img_f, _ = pipeline.render_flat(pipeline.Scene(flat, requires_grad=False), dcam, bg)
    assert n == 3000
    assert img_f.abs().sum() > 0
    assert torch.equal(img_h, img_f)


def _post_scene():
    from h3dgs import synth
    cam = synth.make_camera(320, 180)
    leaves = synth.cloud_v1(6000, cam, zmin=2.0, zmax=30.0, seed=5, scale_k=1.0)
    z = leaves["means3D"][:, 2:3]
    scales = (8e-3 * np.sqrt(2.0 * z) * np.ones((1, 3))).astype(np.float32)
    got = build_np(dict(xyz=leaves["means3D"], shs=leaves["shs"], opacities=leaves["opacities"][:, 0],
                        log_scales=np.log(scales), rotations=leaves["rotations"]))
    q = got["rotations"] / np.linalg.norm(got["rotations"], axis=1, keepdims=True)
    h = dict(means3D=got["xyz"], scales=np.exp(got["log_scales"]), rotations=q.astype(np.float32),
             opacities=np.abs(got["opacities"])[:, None], shs=got["shs"], nodes=got["nodes"], boxes=got["boxes"])
    return cam, h


def test_post_optimisation_on_a_built_hierarchy_reduces_the_loss():
    import torch
    from h3dgs import pipeline, synth
    cam, h = _post_scene()
    thr = synth.tau_threshold(6.0, cam)
    dcam = pipeline.DeviceCamera(cam)
    bg = torch.zeros(3, device="cuda")
    with torch.no_grad():
        gt = pipeline.render_hier_fused(pipeline.Scene(h, requires_grad=False), dcam, bg, thr)[0].clone()
    g = np.random.default_rng(0)
    h2 = dict(h)
    h2["shs"] = (h["shs"] + 0.15 * g.standard_normal(h["shs"].shape)).astype(np.float32)
    h2["opacities"] = np.clip(h["opacities"] * g.uniform(0.6, 1.0, h["opacities"].shape), 0.01, None).astype(np.float32)
    scene = pipeline.Scene(h2)
    opt = torch.optim.Adam([{"params": [scene.shs], "lr": 2e-2}, {"params": [scene.opacities], "lr": 1e-2}])
    losses = []
    for _ in range(40):
        loss, _, n = pipeline.l1_step(scene, dcam, bg, gt, thr)
        losses.append(loss.item())
        opt.step()
    assert 0 < n < h["nodes"].shape[0]
    assert np.isfinite(losses).all() and losses[-1] < 0.5 * losses[0], (losses[0], losses[-1])


@pytest.mark.parametrize("capture", [False, True])
def test_graphed_step_on_a_built_hierarchy(capture):
    """GraphedStep (N nodes = N rows, so its row guard passes) renders what the exact fused path renders"""
    import torch
    from h3dgs import pipeline, synth
    from h3dgs.graphstep import GraphedStep
    cam, h = _post_scene()
    thr = synth.tau_threshold(6.0, cam)
    dcam = pipeline.DeviceCamera(cam)
    bg = torch.zeros(3, device="cuda")
    gt = torch.rand((3, cam.H, cam.W), generator=torch.Generator().manual_seed(1)).cuda()
    scene = pipeline.Scene(h)
    with torch.no_grad():
        img, _, n = pipeline.render_hier_fused(scene, dcam, bg, thr)
        loss = float((img - gt).abs().mean())
    gs = GraphedStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, bin_capacity=1 << 20, sort_capacity=4096,
                     capture=False)
    gs.set_camera(dcam); gs.gt.copy_(gt)
    if capture:
        gs.capture()
    for _ in range(2):
        gs.step(dcam, gt)
        st = gs.status()
        assert not st["overflow"] and st["rows"] == n and 0 < n < h["nodes"].shape[0]
        assert abs(st["loss"] - loss) < 1e-6 and torch.equal(gs.image, img)
        assert all(bool(torch.isfinite(g).all()) for g in gs.grads.values())


def test_creator_cli_end_to_end(tmp_path):
    import subprocess
    import torch
    from gaussian_hierarchy._C import load_hierarchy, expand_to_size
    S, P = 100, 20000
    c = ref.cloud(S + P, seed=12)
    logit = np.random.default_rng(2).standard_normal(S + P).astype(np.float32)
    ply = tmp_path / "point_cloud.ply"
    write_ply(ply, c["xyz"], c["shs"], logit, c["log_scales"], c["rotations"])
    scaffold = tmp_path / "scaffold"
    scaffold.mkdir()
    (scaffold / "pc_info.txt").write_text(f"{S}\n")
    exe = os.path.join(ROOT, "hierarchical-3d-gaussians_b200", "bin", "GaussianHierarchyCreator")
    r = subprocess.run([exe, str(ply), str(tmp_path / "chunk"), str(tmp_path / "out"), str(scaffold)],
                       capture_output=True, text=True, env=dict(os.environ, PYTHON=sys.executable))
    assert r.returncode == 0, r.stdout + r.stderr
    xyz, shs, opac, ls, rots, nodes, boxes = load_hierarchy(str(tmp_path / "out" / "hierarchy.hier"))
    N = 2 * P - 1
    assert xyz.shape[0] == N == nodes.shape[0]
    tail = {k: v[S:] for k, v in c.items()}
    tail["opacities"] = torch.sigmoid(torch.from_numpy(logit[S:]).cuda()).cpu().numpy()     # as the creator computes it
    want = build_np(tail)
    assert np.array_equal(nodes.numpy(), want["nodes"]) and np.array_equal(bits(xyz.numpy()), bits(want["xyz"]))
    nd, bx = nodes.cuda(), boxes.cuda()
    z = lambda: torch.zeros(N, dtype=torch.int32, device="cuda")
    n = expand_to_size(nd, bx, 0.0, torch.zeros(3, device="cuda") + 100.0, torch.zeros(3), z(), z(), z())
    assert n == P

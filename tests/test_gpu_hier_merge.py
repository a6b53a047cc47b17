"""GPU: the hierarchy merger (csrc/hier_merge.cu on the H100) -- the CPU suite's cases against the numpy restatement;
the two benchmark workloads at full size (invariants, repeat-call identity, outputs on the input's device); at target
size 0 the merged hierarchy renders exactly the owned leaf Gaussians; GraphedStep agrees with the exact fused path on a
merged hierarchy; the command-line merger end to end."""
import os
import sys

import numpy as np
import pytest

import hier_merge_ref as ref
from test_hier_merge_cpu import NAMES, OUT, bits, cases, check_against_ref, check_invariants, write_chunk_dirs

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def build_np(c):
    from test_gpu_hier_build import build_np as b
    return b(c)


def merge_np(chunks, cells):
    import torch
    from h3dgs.hier_merge import merge_hierarchies
    t = [{k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in c.items()} for c in chunks]
    h = merge_hierarchies(t, cells)
    out = {k: h[k].cpu().numpy() for k in OUT}
    out["opacities"] = out["opacities"][:, 0]
    out["R"] = h["items"]
    return out


@pytest.fixture(scope="module")
def CASES():
    return cases(build_np)


@pytest.mark.parametrize("name", NAMES)
def test_matches_the_restatement(CASES, name):
    chunks, cells = CASES[name]
    got = merge_np(chunks, cells)
    check_invariants(got, chunks, cells)
    check_against_ref(got, chunks, cells)


def check_structure(h, chunks, cells):
    """vectorised invariants of a merge of creator-built chunks (one row per node, start = i)"""
    nodes, sc, sr = h["nodes"], h["source_chunk"], h["source_row"]
    NO = nodes.shape[0]
    assert h["xyz"].shape[0] == NO and np.array_equal(nodes[:, 2], np.arange(NO)) and nodes[0, 1] == -1
    assert np.array_equal(np.bincount(nodes[1:, 1], minlength=NO), nodes[:, 6])
    inner = np.nonzero(nodes[:, 6] > 0)[0]
    first = nodes[inner, 5]
    assert (nodes[first, 1] == inner).all() and (nodes[first + nodes[inner, 6] - 1, 1] == inner).all()
    kid = np.nonzero(nodes[:, 1] >= 0)[0]
    b = h["boxes"]
    assert (b[kid, 0, :3] >= b[nodes[kid, 1], 0, :3]).all() and (b[kid, 1, :3] <= b[nodes[kid, 1], 1, :3]).all()
    leaf = nodes[:, 3] == 1
    want = []
    for c, ch in enumerate(chunks):
        rows = np.nonzero(ch["nodes"][:, 3] == 1)[0]            # creator-built: leaf row = leaf node
        own = ref.owners(ch["xyz"][rows, :2], cells) == c
        want.append(c * (1 << 32) + rows[own].astype(np.int64))
    want = np.sort(np.concatenate(want))
    got = np.sort(sc[leaf].astype(np.int64) * (1 << 32) + sr[leaf])
    assert np.array_equal(got, want)
    for c, ch in enumerate(chunks):
        sel = sc == c
        for k in ("xyz", "log_scales", "rotations"):
            assert np.array_equal(bits(h[k][sel]), bits(ch[k][sr[sel]])), k
    assert np.isfinite(h["xyz"]).all() and np.isfinite(h["opacities"]).all()


@pytest.mark.parametrize("name", ["2x2x1.5m", "4x4x1m"])
def test_bench_workloads(name):
    import torch
    import bench_hier_merge
    from h3dgs.hier_merge import merge_hierarchies
    chunks, cells = bench_hier_merge.scene(name)
    h1 = merge_hierarchies(chunks, cells)
    assert all(h1[k].device == chunks[0]["xyz"].device for k in OUT)
    a = {k: h1[k].cpu().numpy() for k in OUT}
    del h1
    h2 = merge_hierarchies(chunks, cells)
    for k in OUT:
        assert h2[k].cpu().numpy().tobytes() == a[k].tobytes(), k
    del h2
    a["opacities"] = a["opacities"][:, 0]
    npc = [{k: v.cpu().numpy().reshape(v.shape[0], -1) if k == "opacities" else v.cpu().numpy() for k, v in c.items()}
           for c in chunks]
    for c in npc:
        c["opacities"] = c["opacities"][:, 0]
    check_structure(a, npc, cells)
    torch.cuda.empty_cache()


def _merged_scene(seed=4, n=1500):
    """two creator-built chunks of a scene in front of synth's camera, distinct depths -> (cam, merged hierarchy, the
    leaf Gaussians of the input chunks that the ownership rule keeps, as a flat cloud)"""
    from h3dgs import synth
    cam = synth.make_camera(640, 360)
    rng = np.random.default_rng(seed)
    leaves = synth.cloud_v1(2 * n, cam, zmin=2.0, zmax=30.0, seed=seed)
    xyz = leaves["means3D"].copy()
    xyz[:, 2] = (2.0 + 28.0 * rng.permutation(2 * n) / (2 * n)).astype(np.float32)
    xm = float(np.median(xyz[:, 0]))
    span = float(xyz[:, 0].max() - xyz[:, 0].min()) + 1.0
    ysp = float(xyz[:, 1].max() - xyz[:, 1].min()) + 1.0
    yc = float(xyz[:, 1].mean())
    cells = np.array([[xm - span / 2, yc, span, ysp], [xm + span / 2, yc, span, ysp]], np.float32)
    chunks = []
    for k in range(2):
        sel = xyz[:, 0] < xm + 0.1 * span if k == 0 else xyz[:, 0] > xm - 0.1 * span     # overlapping chunk clouds
        c = dict(xyz=xyz[sel], shs=leaves["shs"][sel], opacities=leaves["opacities"][sel, 0],
                 log_scales=np.log(leaves["scales"][sel]), rotations=leaves["rotations"][sel])
        h = build_np(c)
        chunks.append({kk: h[kk] for kk in ("xyz", "shs", "opacities", "log_scales", "rotations", "nodes", "boxes")})
    m = merge_np(chunks, cells)
    owned = []                                   # the inputs' owned leaf Gaussians, by the ownership rule
    for k, ch in enumerate(chunks):
        rows = np.concatenate([np.arange(s, s + c) for s, c in zip(ch["nodes"][:, 2], ch["nodes"][:, 3])]).astype(np.int64)
        owned.append({kk: ch[kk][rows[ref.owners(ch["xyz"][rows, :2], cells) == k]]
                      for kk in ("xyz", "shs", "opacities", "log_scales", "rotations")})
    o = {kk: np.concatenate([x[kk] for x in owned]) for kk in owned[0]}
    flat = dict(means3D=o["xyz"], scales=np.exp(o["log_scales"]), rotations=o["rotations"],
                opacities=o["opacities"].reshape(-1, 1), shs=o["shs"])
    h = dict(means3D=m["xyz"], scales=np.exp(m["log_scales"]), rotations=m["rotations"],
             opacities=np.abs(m["opacities"])[:, None], shs=m["shs"], nodes=m["nodes"], boxes=m["boxes"])
    return cam, h, flat


def test_target_zero_renders_the_owned_leaf_gaussians():
    import torch
    from h3dgs import pipeline
    cam, h, flat = _merged_scene()
    dcam = pipeline.DeviceCamera(cam)
    bg = torch.zeros(3, device="cuda")
    with torch.no_grad():
        img_h, _, n = pipeline.render_hier(pipeline.Scene(h, requires_grad=False), dcam, bg, 0.0)
        img_f, _ = pipeline.render_flat(pipeline.Scene(flat, requires_grad=False), dcam, bg)
    assert n == flat["means3D"].shape[0] and img_f.abs().sum() > 0
    assert torch.equal(img_h, img_f)


def test_graphed_step_on_a_merged_hierarchy():
    """GraphedStep (one row per node, so its row guard passes) renders what the exact fused path renders at tau 6"""
    import torch
    from h3dgs import pipeline, synth
    from h3dgs.graphstep import GraphedStep
    cam, h, _ = _merged_scene(seed=5)
    q = h["rotations"] / np.linalg.norm(h["rotations"], axis=1, keepdims=True)
    h = dict(h, rotations=q.astype(np.float32))
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
    for _ in range(2):
        gs.step(dcam, gt)
        st = gs.status()
        assert not st["overflow"] and st["rows"] == n and 0 < n
        assert abs(st["loss"] - loss) < 1e-6 and torch.equal(gs.image, img)


def test_merger_cli_end_to_end(tmp_path, CASES):
    import subprocess
    import torch
    from gaussian_hierarchy._C import load_hierarchy, expand_to_size
    chunks, cells = CASES["creator4"]
    names = ["0_0", "1_0", "0_1", "1_1"]
    write_chunk_dirs(tmp_path, chunks, cells, names)
    exe = os.path.join(ROOT, "hierarchical-3d-gaussians_b200", "bin", "GaussianHierarchyMerger")
    out = tmp_path / "output" / "merged.hier"
    r = subprocess.run([exe, str(tmp_path / "trained_chunks"), "0", str(tmp_path / "chunks"), str(out)] + names,
                       capture_output=True, text=True, env=dict(os.environ, PYTHON=sys.executable))
    assert r.returncode == 0, r.stdout + r.stderr
    xyz, shs, opac, ls, rots, nodes, boxes = load_hierarchy(str(out))
    want = merge_np(chunks, cells)
    assert np.array_equal(nodes.numpy(), want["nodes"]) and np.array_equal(bits(xyz.numpy()), bits(want["xyz"]))
    N = nodes.shape[0]
    z = lambda: torch.zeros(N, dtype=torch.int32, device="cuda")
    n = expand_to_size(nodes.cuda(), boxes.cuda(), 0.0, torch.zeros(3, device="cuda") + 100.0, torch.zeros(3), z(), z(), z())
    assert n == int(want["nodes"][:, 3].sum())
    r = subprocess.run([exe, str(tmp_path / "trained_chunks"), "0", str(tmp_path / "chunks"), str(out), "0_0", "7_7"],
                       capture_output=True, text=True, env=dict(os.environ, PYTHON=sys.executable))
    assert r.returncode != 0 and "7_7" in r.stderr

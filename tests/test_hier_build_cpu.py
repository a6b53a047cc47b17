"""CPU: the hierarchy creator (csrc/hier_build.cu, emulation build) against the numpy restatement of
tests/hier_build_ref.py: topology, node fields, sources and leaf rows exactly, boxes within one fp32 ulp with exact
nesting, merged rows within tolerance; moment matching on a large Gaussian sampled by small ones; the LOD cut on built
hierarchies against tests/hier_general.py; repeatability and argument checks; read_ply; the command-line creator."""
import os
import sys
from unittest import mock

import numpy as np
import pytest

import hier_build_ref as ref
import hier_general as hg
from h3dgs import synth

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emul"))

CASES = ref.cases()


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """the emulation build of the library's sources plus hier_build.cu"""
    import build_emu
    from emu_api import Emu
    with mock.patch.object(build_emu, "SOURCES", build_emu.SOURCES + ["hier_build.cu"]):
        return Emu(build_emu.build(str(tmp_path_factory.mktemp("h3dgs_emu_hier_build"))))


def _pad16(shs):
    return np.concatenate([shs, np.zeros((shs.shape[0], 16 - shs.shape[1], 3), np.float32)], 1)


def run(emu, c, check=True):
    from emu_api import aligned, f32, ptr
    P = int(c["xyz"].shape[0])
    N = 2 * P - 1
    ins = [f32(c["xyz"]), f32(c["log_scales"]), f32(c["rotations"]), f32(c["opacities"]), f32(_pad16(c["shs"]))]
    out = dict(xyz=aligned(N * 12, np.float32, (N, 3)), shs=aligned(N * 192, np.float32, (N, 16, 3)),
               opacities=aligned(N * 4, np.float32, (N,)), log_scales=aligned(N * 12, np.float32, (N, 3)),
               rotations=aligned(N * 16, np.float32, (N, 4)), nodes=aligned(N * 28, np.int32, (N, 7)),
               boxes=aligned(N * 32, np.float32, (N, 2, 4)), source=aligned(N * 4, np.int32, (N,)))
    scratch = aligned(emu.L.h3dgs_build_hierarchy_scratch_bytes(P))
    rc = emu.L.h3dgs_build_hierarchy(P, *(ptr(a) for a in ins), *(ptr(out[k]) for k in
                                     ("xyz", "shs", "opacities", "log_scales", "rotations", "nodes", "boxes", "source")),
                                     ptr(scratch), None)
    if check:
        emu.check(rc)
        return out
    return rc, out


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def check_against_ref(got, c):
    """the comparison every built hierarchy goes through (the GPU suite imports it)"""
    r = ref.build(c["xyz"], _pad16(c["shs"]), c["opacities"], c["log_scales"], c["rotations"])
    P = c["xyz"].shape[0]
    N = 2 * P - 1
    assert np.array_equal(got["nodes"], r["nodes"])
    assert np.array_equal(got["source"], r["source"])
    leaf = r["source"] >= 0
    for k in ("xyz", "shs", "opacities", "log_scales", "rotations"):
        assert np.array_equal(bits(got[k][leaf]), bits(r[k][leaf])), k
    # boxes: within one ulp of the restatement; interior boxes exactly the union of the kernel's own children
    b, rb = got["boxes"], r["boxes"]
    ulp = np.spacing(np.abs(rb[:, :, :3]))
    assert (np.abs(b[:, :, :3] - rb[:, :, :3]) <= ulp).all()
    nodes = got["nodes"]
    inner = np.nonzero(nodes[:, 6] == 2)[0]
    ca, cb = nodes[inner, 5], nodes[inner, 5] + 1
    assert np.array_equal(b[inner, 0, :3], np.minimum(b[ca, 0, :3], b[cb, 0, :3]))
    assert np.array_equal(b[inner, 1, :3], np.maximum(b[ca, 1, :3], b[cb, 1, :3]))
    assert np.array_equal(bits(b[:, 0, 3]), bits((b[:, 1, :3] - b[:, 0, :3]).max(1)))
    assert (b[:, 1, 3] == 0).all()
    if inner.size == 0:
        return r
    # merged rows
    ext = max(float((c["xyz"].max(0) - c["xyz"].min(0)).max()), 1e-30)
    assert np.abs(got["xyz"][inner] - r["xyz"][inner]).max() <= 1e-6 * ext + np.spacing(np.abs(r["xyz"][inner])).max()
    cg = ref.cov_of(got["log_scales"][inner], got["rotations"][inner])
    cr = r["cov"][inner]
    rel = np.linalg.norm(cg - cr, axis=(1, 2)) / np.linalg.norm(cr, axis=(1, 2))
    assert rel.max() < 1e-5, rel.max()
    o, ro = got["opacities"][inner].astype(np.float64), r["opacities"][inner].astype(np.float64)
    assert (np.abs(o - ro) <= 1e-5 * np.abs(ro) + 1e-30).all()
    sh, rsh = got["shs"][inner].astype(np.float64), r["shs"][inner].astype(np.float64)
    scale = np.abs(rsh).max(axis=(1, 2), keepdims=True) + 1e-30
    assert (np.abs(sh - rsh) <= 1e-5 * scale).all()
    assert (np.diff(got["log_scales"][inner], axis=1) <= 0).all()                # descending
    q = got["rotations"][inner].astype(np.float64)
    assert np.abs(np.linalg.norm(q, axis=1) - 1).max() < 1e-6 and (q[:, 0] >= 0).all()
    assert N == nodes.shape[0]
    return r


@pytest.mark.parametrize("name", list(CASES))
def test_matches_the_restatement(emu, name):
    check_against_ref(run(emu, CASES[name]), CASES[name])


def test_65537_gaussians(emu):
    c = ref.cloud(65537, seed=3)
    check_against_ref(run(emu, c), c)


def test_zero_opacity_gives_zero_merged_opacity(emu):
    got = run(emu, CASES["zero_opacity"])
    assert (got["opacities"][got["source"] < 0] == 0).all()


def test_moment_matching_recovers_the_sampled_gaussian(emu):
    c, mean, cov = ref.sampled_large()
    got = run(emu, c)
    n = c["xyz"].shape[0]
    assert (np.abs(got["xyz"][0] - mean) < 5 * np.sqrt(np.diag(cov) / n)).all()
    c0 = ref.cov_of(got["log_scales"][:1], got["rotations"][:1])[0]
    assert np.linalg.norm(c0 - cov) / np.linalg.norm(cov) < 0.05


def test_two_runs_give_identical_bytes(emu):
    c = CASES["P1000"]
    a, b = run(emu, c), run(emu, c)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k


def built_scene(emu_or_fn, n=3000, seed=21):
    """a cloud in front of synth's camera, built -> dict in synth.build_hierarchy's layout (activated values)"""
    cam = synth.make_camera(640, 360)
    leaves = synth.cloud_v1(n, cam, zmin=2.0, zmax=30.0, seed=seed)
    c = dict(xyz=leaves["means3D"], shs=leaves["shs"], opacities=leaves["opacities"][:, 0],
             log_scales=np.log(leaves["scales"]), rotations=leaves["rotations"])
    got = emu_or_fn(c)
    return cam, dict(means3D=got["xyz"], scales=np.exp(got["log_scales"]), rotations=got["rotations"],
                     opacities=np.abs(got["opacities"]).reshape(-1, 1), shs=got["shs"], nodes=got["nodes"], boxes=got["boxes"])


def test_lod_cut_on_a_built_hierarchy(emu):
    from emu_api import aligned, f32, i32, ptr
    cam, h = built_scene(lambda c: run(emu, c))
    L = emu.L
    N = h["nodes"].shape[0]
    nodes, boxes = i32(h["nodes"]), f32(h["boxes"])
    scratch = aligned(L.h3dgs_expand_scratch_bytes(N))
    for vname, vp in hg.viewpoints(h, cam).items():
        for tau in (0.0, 3.0, 6.0, 15.0):
            thr = synth.tau_threshold(tau, cam)
            n, ri, pi, ni = hg.cut(h["nodes"], h["boxes"], thr, vp)
            hg.check_cut_invariant(h["nodes"], h["boxes"], thr, vp, ri, ni)
            r, p, nn = (aligned(N * 4, np.int32, (N,)) for _ in range(3))
            vpa, idx = f32(vp), i32(ni)                  # kept alive across the calls
            got = emu.check(L.h3dgs_expand_to_size(N, ptr(nodes), ptr(boxes), float(thr), ptr(vpa), 0.0, 0.0, 0.0,
                                                   ptr(r), ptr(p), ptr(nn), ptr(scratch), None))
            assert got == n and np.array_equal(r[:n], ri) and np.array_equal(p[:n], pi) and np.array_equal(nn[:n], ni), (vname, tau)
            ts, kids = hg.weights(ni, thr, h["nodes"], h["boxes"], vp)
            t, k = aligned(N * 4, np.float32, (N,)), aligned(N * 4, np.int32, (N,))
            if n:
                emu.check(L.h3dgs_get_interpolation_weights(n, ptr(idx), float(thr), ptr(nodes), ptr(boxes),
                                                            float(vp[0]), float(vp[1]), float(vp[2]), 0.0, 0.0, 0.0,
                                                            ptr(t), ptr(k), None))
            assert np.array_equal(bits(t[:n]), bits(ts)) and np.array_equal(k[:n], kids), (vname, tau)


def test_bad_arguments(emu):
    from emu_api import aligned, ptr
    L = emu.L
    assert L.h3dgs_build_hierarchy_scratch_bytes(0) == 0 and L.h3dgs_build_hierarchy_scratch_bytes((1 << 30) + 1) == 0
    c = CASES["P17"]
    for field, row, val in (("xyz", 3, np.nan), ("xyz", 0, np.inf), ("log_scales", 5, np.inf), ("log_scales", 16, np.nan),
                            ("opacities", 2, -0.25), ("opacities", 7, np.nan), ("opacities", 9, np.inf),
                            ("rotations", 4, np.nan), ("rotations", 11, -np.inf), ("log_scales", 6, 300.5)):
        bad = {k: v.copy() for k, v in c.items()}
        bad[field].reshape(17, -1)[row, 0] = val
        rc, out = run(emu, bad, check=False)
        assert rc == -1, (field, val)
        assert b"non-finite" in L.h3dgs_last_error()
        assert not out["nodes"].any() and not out["xyz"].any()
    z = aligned(64)
    assert L.h3dgs_build_hierarchy(0, *([ptr(z)] * 14), None) == -1
    assert L.h3dgs_build_hierarchy((1 << 30) + 1, *([ptr(z)] * 14), None) == -1
    assert L.h3dgs_build_hierarchy(2, *([ptr(z)] * 5), None, *([ptr(z)] * 8), None) == -1


# ---------------------------------------------------------------------------------------------------------------
# read_ply and the command-line creator
# ---------------------------------------------------------------------------------------------------------------
def write_ply(path, xyz, shs, logit_opacities, log_scales, rotations):
    """the file GaussianModel.save_ply writes (scene/gaussian_model.py:491-508), property for property"""
    P, K = shs.shape[:2]
    names = ["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(3)] + \
        [f"f_rest_{i}" for i in range(3 * (K - 1))] + ["opacity"] + [f"scale_{i}" for i in range(3)] + [f"rot_{i}" for i in range(4)]
    rest = shs[:, 1:].transpose(0, 2, 1).reshape(P, -1)
    cols = np.concatenate([xyz, np.zeros_like(xyz), shs[:, 0], rest, logit_opacities.reshape(P, 1), log_scales, rotations], 1)
    el = np.empty(P, dtype=[(n, "<f4") for n in names])
    for i, n in enumerate(names):
        el[n] = cols[:, i]
    head = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % P + "".join(f"property float {n}\n" for n in names) + "end_header\n"
    with open(path, "wb") as f:
        f.write(head.encode())
        f.write(el.tobytes())


@pytest.mark.parametrize("K", [1, 4, 9, 16])
def test_read_ply_round_trip(tmp_path, K):
    from h3dgs.hier_build import read_ply
    c = ref.cloud(37, seed=K, sh_coeffs=K)
    logit = np.random.default_rng(K).standard_normal(37).astype(np.float32)
    write_ply(tmp_path / "pc.ply", c["xyz"], c["shs"], logit, c["log_scales"], c["rotations"])
    g = read_ply(str(tmp_path / "pc.ply"))
    for k, v in (("xyz", c["xyz"]), ("shs", c["shs"]), ("opacities", logit), ("log_scales", c["log_scales"]),
                 ("rotations", c["rotations"])):
        assert g[k].dtype == np.float32 and np.array_equal(bits(g[k]), bits(v)), k


def test_read_ply_rejects_what_it_cannot_read(tmp_path):
    from h3dgs.hier_build import read_ply
    p = tmp_path / "a.ply"
    p.write_bytes(b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nend_header\n0\n")
    with pytest.raises(ValueError, match="binary_little_endian"):
        read_ply(str(p))
    p.write_bytes(b"ply\nformat binary_little_endian 1.0\nelement vertex 1\nproperty float x\nend_header\n" + bytes(4))
    with pytest.raises(ValueError, match="missing"):
        read_ply(str(p))


def _emu_patches(emu):
    import torch
    from h3dgs import _lib, hier_build
    from gaussian_hierarchy import creator
    return [mock.patch.object(_lib, "_lib", emu.L), mock.patch.object(hier_build, "_on_device", lambda t: True),
            mock.patch.object(creator, "_device", lambda: torch.device("cpu")),
            mock.patch.object(torch.cuda, "device", lambda *_a: mock.MagicMock()),
            mock.patch.object(torch.cuda, "current_stream", lambda *a, **k: mock.Mock(cuda_stream=0))]


def test_python_build_hierarchy_on_the_emulation_build(emu):
    import contextlib
    import torch
    from h3dgs.hier_build import build_hierarchy
    c = CASES["P1000"]
    with contextlib.ExitStack() as st:
        for p in _emu_patches(emu):
            st.enter_context(p)
        t = {k: torch.from_numpy(v) for k, v in c.items()}
        h = build_hierarchy(t["xyz"], t["shs"], t["opacities"], t["log_scales"], t["rotations"])
        direct = run(emu, c)
        for k in direct:
            assert np.array_equal(h[k].numpy().reshape(direct[k].shape).view(np.uint8), direct[k].view(np.uint8)), k
        assert h["opacities"].shape == (1999, 1) and h["shs"].shape == (1999, 16, 3)
        wide = torch.zeros((1000, 5))
        wide[:, 1:4] = t["xyz"]
        h2 = build_hierarchy(wide[:, 1:4], t["shs"][:, :4], t["opacities"][:, None], t["log_scales"], t["rotations"])
        assert (h2["shs"][:, 4:] == 0).all() and torch.equal(h2["nodes"], h["nodes"])
        with pytest.raises(ValueError):
            build_hierarchy(t["xyz"], t["shs"][:, :5], t["opacities"], t["log_scales"], t["rotations"])
        with pytest.raises(RuntimeError, match="non-finite"):
            bad = t["opacities"].clone(); bad[3] = -1
            build_hierarchy(t["xyz"], t["shs"], bad, t["log_scales"], t["rotations"])
    with pytest.raises(RuntimeError):
        build_hierarchy(t["xyz"], t["shs"], t["opacities"], t["log_scales"], t["rotations"])      # CPU tensors


def test_creator_cli_with_full_train_argv(emu, tmp_path):
    import contextlib
    import torch
    from gaussian_hierarchy import creator
    from gaussian_hierarchy._C import load_hierarchy
    S, P = 40, 600
    c = ref.cloud(S + P, seed=9)
    c["xyz"][:S] *= 100.0                               # the skybox rows train_single puts in front
    logit = np.random.default_rng(1).standard_normal(S + P).astype(np.float32)
    chunk = tmp_path / "trained_chunk"
    (chunk / "point_cloud" / "iteration_30000").mkdir(parents=True)
    ply = chunk / "point_cloud" / "iteration_30000" / "point_cloud.ply"
    write_ply(ply, c["xyz"], c["shs"], logit, c["log_scales"], c["rotations"])
    scaffold = tmp_path / "scaffold" / "point_cloud" / "iteration_30000"
    scaffold.mkdir(parents=True)
    (scaffold / "pc_info.txt").write_text(f"{S}\n")
    with contextlib.ExitStack() as st:
        for p in _emu_patches(emu):
            st.enter_context(p)
        assert creator.main([str(ply), str(tmp_path / "source_chunk"), str(chunk), str(scaffold)]) == 0
        xyz, shs, opac, ls, rots, nodes, boxes = load_hierarchy(str(chunk / "hierarchy.hier"))
        tail = {k: v[S:] for k, v in c.items()}
        tail["opacities"] = torch.sigmoid(torch.from_numpy(logit[S:])).numpy()
        want = run(emu, tail)
    N = 2 * P - 1
    assert xyz.shape == (N, 3) and nodes.shape == (N, 7) and opac.shape == (N, 1)
    assert np.array_equal(nodes.numpy(), want["nodes"]) and np.array_equal(bits(xyz.numpy()), bits(want["xyz"]))
    assert np.array_equal(bits(opac.numpy()[:, 0]), bits(want["opacities"])) and np.array_equal(bits(boxes.numpy()), bits(want["boxes"]))
    assert np.array_equal(bits(shs.numpy()), bits(want["shs"])) and np.array_equal(bits(rots.numpy()), bits(want["rotations"]))
    assert creator.main(["only", "two"]) == 2

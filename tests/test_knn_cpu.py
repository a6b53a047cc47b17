"""CPU: the exact 3-nearest-neighbour kernel (csrc/knn.cu, emulation build) bit for bit against the restatement of
tests/knn_ref.py on clouds that stress an exact search; permutation invariance; non-finite rows ignored; the drop-in
simple_knn._C.distCUDA2 (strided input, argument checks) on the emulation build; and the import of simple_knn from the
package directory the way the reference's scene/gaussian_model.py:21 does it."""
import os
import subprocess
import sys
from unittest import mock

import numpy as np
import pytest

import knn_ref

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PKG = os.path.join(ROOT, "hierarchical-3d-gaussians_b200")
sys.path.insert(0, os.path.join(HERE, "emul"))

CASES = knn_ref.cases()


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """the emulation build of the library's sources plus knn.cu"""
    import build_emu
    from emu_api import Emu
    with mock.patch.object(build_emu, "SOURCES", build_emu.SOURCES + ["knn.cu"]):
        return Emu(build_emu.build(str(tmp_path_factory.mktemp("h3dgs_emu_knn"))))


def _run(emu, pts):
    from emu_api import aligned, f32, ptr
    P = int(pts.shape[0])
    x = f32(pts) if P else None
    out = aligned(max(P, 1) * 4, np.float32, (max(P, 1),))
    out[:] = -1.0
    scratch = aligned(emu.L.h3dgs_knn_scratch_bytes(P)) if P else None
    emu.check(emu.L.h3dgs_dist_knn3(P, ptr(x), ptr(out), ptr(scratch), None))
    return out[:P].copy()


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("name", list(CASES))
def test_matches_the_restatement_bit_for_bit(emu, name):
    pts = CASES[name]
    got, ref = _run(emu, pts), knn_ref.dist_knn3(pts)
    assert _same_bits(got, ref), (name, np.flatnonzero(got.view(np.uint32) != ref.view(np.uint32))[:10])


def test_fewer_than_three_other_points(emu):
    fm = np.float32(np.finfo(np.float32).max)
    assert _run(emu, CASES["cube0"]).shape == (0,)
    assert np.all(np.isposinf(_run(emu, CASES["cube1"]))) and np.all(np.isposinf(_run(emu, CASES["cube2"])))
    p = np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0]], np.float32)
    assert _same_bits(_run(emu, p), np.array([((np.float32(1) + np.float32(4)) + fm) / np.float32(3),
                                              ((np.float32(1) + np.float32(5)) + fm) / np.float32(3),
                                              ((np.float32(4) + np.float32(5)) + fm) / np.float32(3)], np.float32))


@pytest.mark.parametrize("name", ["cube4097", "duplicates", "lattice", "scene_skybox"])
def test_permuting_the_input_permutes_the_output(emu, name):
    pts = CASES[name]
    perm = np.random.default_rng(5).permutation(len(pts))
    assert _same_bits(_run(emu, pts[perm]), _run(emu, pts)[perm])


@pytest.mark.parametrize("name", ["cube1025", "plane", "duplicates", "scene_skybox"])
def test_non_finite_rows_are_ignored(emu, name):
    pts = CASES[name]
    mixed, finite = knn_ref.with_non_finite(pts)
    got = _run(emu, mixed)
    assert _same_bits(got[finite], _run(emu, mixed[finite]))


def test_only_non_finite_rows_do_not_fault(emu):
    mixed, finite = knn_ref.with_non_finite(np.zeros((0, 3), np.float32))
    assert not finite.any()
    assert _run(emu, mixed).shape == (len(mixed),)


def test_bad_arguments(emu):
    from emu_api import aligned, f32, ptr
    x, out = f32(CASES["cube33"]), aligned(33 * 4, np.float32, (33,))
    s = aligned(emu.L.h3dgs_knn_scratch_bytes(33))
    assert emu.L.h3dgs_dist_knn3(-1, ptr(x), ptr(out), ptr(s), None) == -1
    assert emu.L.h3dgs_dist_knn3(33, None, ptr(out), ptr(s), None) == -1
    assert emu.L.h3dgs_dist_knn3(33, ptr(x), None, ptr(s), None) == -1
    assert emu.L.h3dgs_dist_knn3(33, ptr(x), ptr(out), None, None) == -1
    assert emu.L.h3dgs_dist_knn3(0, None, None, None, None) == 0
    with pytest.raises(RuntimeError, match="bad arguments"):
        emu.check(emu.L.h3dgs_dist_knn3(-1, None, None, None, None))


def test_dropin_distCUDA2_on_the_emulation_build(emu):
    import torch
    from h3dgs import _lib
    import simple_knn._C as kc
    pts = torch.from_numpy(CASES["cube1025"])
    with mock.patch.object(_lib, "_lib", emu.L), mock.patch.object(kc, "_on_device", lambda t: True), \
            mock.patch.object(torch.cuda, "device", lambda *_a: mock.MagicMock()), \
            mock.patch.object(torch.cuda, "current_stream", lambda *a, **k: mock.Mock(cuda_stream=0)):
        d = kc.distCUDA2(pts)
        assert d.shape == (1025,) and d.dtype == torch.float32
        assert _same_bits(d.numpy(), knn_ref.dist_knn3(CASES["cube1025"]))
        wide = torch.zeros((1025, 5))
        wide[:, 1:4] = pts
        assert not wide[:, 1:4].is_contiguous()
        assert _same_bits(kc.distCUDA2(wide[:, 1:4]).numpy(), d.numpy())
        assert kc.distCUDA2(torch.zeros((0, 3))).shape == (0,)
        scales = torch.log(torch.sqrt(torch.clamp_min(kc.distCUDA2(pts), 1e-7)))[..., None].repeat(1, 3)
        assert scales.shape == (1025, 3)
        for bad in (pts.double(), pts[:, :2].contiguous(), pts.reshape(-1)):
            with pytest.raises(RuntimeError):
                kc.distCUDA2(bad)
    with pytest.raises(RuntimeError):
        kc.distCUDA2(pts)                    # a CPU tensor, with the real device check


SCRIPT = r'''
import inspect, sys
from simple_knn._C import distCUDA2
import simple_knn
assert inspect.getsourcefile(distCUDA2).startswith(sys.argv[1]), inspect.getsourcefile(distCUDA2)
assert inspect.getsourcefile(simple_knn).startswith(sys.argv[1]), inspect.getsourcefile(simple_knn)
print("ok")
'''


def test_reference_import_resolves_into_this_package():
    env = dict(os.environ, PYTHONPATH=PKG)
    r = subprocess.run([sys.executable, "-c", SCRIPT, PKG], capture_output=True, text=True, env=env, cwd=PKG)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr

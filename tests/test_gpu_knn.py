"""GPU: simple_knn._C.distCUDA2 (csrc/knn.cu, nvcc build) bit for bit against the restatement of tests/knn_ref.py, on
the CPU suite's clouds and on the three clouds of tools/bench_knn.py at full size (1M, 4M, 2.1M points); repeat calls
identical; no host synchronisation; argument checks; the output on the input's device; the call site's shape."""
import importlib.util
import os

import numpy as np
import pytest

import knn_ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = knn_ref.cases()


def _bench_clouds():
    spec = importlib.util.spec_from_file_location("bench_knn", os.path.join(ROOT, "tools", "bench_knn.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m.CLOUDS


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _dist(pts, device="cuda"):
    import torch
    from simple_knn._C import distCUDA2
    return distCUDA2(torch.from_numpy(pts).to(device)).cpu().numpy()


@pytest.mark.parametrize("name", list(CASES))
def test_matches_the_restatement(name):
    pts = CASES[name]
    assert _same_bits(_dist(pts), knn_ref.dist_knn3(pts))


def test_non_finite_rows_are_ignored():
    mixed, finite = knn_ref.with_non_finite(CASES["scene_skybox"])
    assert _same_bits(_dist(mixed)[finite], _dist(mixed[finite]))


@pytest.mark.parametrize("name", ["cube1m", "sfm4m", "coarse2m"])
def test_bench_clouds_at_full_size(name):
    import torch
    from simple_knn._C import distCUDA2
    pts = _bench_clouds()[name]()
    x = torch.from_numpy(pts).cuda()
    a = distCUDA2(x)
    b = distCUDA2(x)
    a, b = a.cpu().numpy(), b.cpu().numpy()
    assert _same_bits(a, b)
    assert _same_bits(a, knn_ref.dist_knn3(pts))


def test_no_host_synchronisation():
    import torch
    from simple_knn._C import distCUDA2
    x = torch.from_numpy(CASES["scene_skybox"]).cuda()
    ref = distCUDA2(x)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = distCUDA2(x)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(out.view(torch.int32), ref.view(torch.int32))


def test_argument_checks_and_call_site_shape():
    import torch
    from simple_knn._C import distCUDA2
    x = torch.from_numpy(CASES["cube4097"])
    for bad in (x, x.double().cuda(), x[:, :2].cuda()):
        with pytest.raises(RuntimeError):
            distCUDA2(bad)
    d = distCUDA2(x.cuda())
    assert d.shape == (4097,) and d.dtype == torch.float32 and d.device == torch.device("cuda", 0)
    scales = torch.log(torch.sqrt(torch.clamp_min(distCUDA2(x.cuda()), 1e-7)))[..., None].repeat(1, 3)
    assert scales.shape == (4097, 3)
    wide = torch.zeros((4097, 5), device="cuda")
    wide[:, 1:4] = x.cuda()
    assert _same_bits(distCUDA2(wide[:, 1:4]).cpu().numpy(), d.cpu().numpy())


def test_output_on_the_input_device():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs a second GPU")
    from simple_knn._C import distCUDA2
    pts = CASES["scene_skybox"]
    out = distCUDA2(torch.from_numpy(pts).to("cuda:1"))
    assert out.device == torch.device("cuda", 1)
    assert _same_bits(out.cpu().numpy(), _dist(pts, "cuda:0"))

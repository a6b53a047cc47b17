"""CPU: the families of tests/test_gpu_scatter_edges.py (the hierarchy cut's gather per rendered row, the t / (1 - t)
scatter per full-size row, against preprocess_ref and chain_ref) on the emulation build of the kernels (tests/emul/),
driven through the same Python layer with the emulation build standing in for libh3dgs.so (tests/emul/fake_device.py).
The split schedule at config #3's source size needs the GPU; here the split schedule runs on the small cut.  Also here:
the 16-byte alignment of the rows that the kernels read and write as float4, refused by the C-ABI and copied by _C."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emul"))

import test_gpu_scatter_edges as se  # noqa: E402


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    from build_emu import build
    return build(str(tmp_path_factory.mktemp("h3dgs_emu_scatter")))


@pytest.fixture
def on_emu(emu_so):
    from fake_device import cpu_as_device, cuda_names_mean_cpu
    with cpu_as_device(emu_so) as L, cuda_names_mean_cpu():
        yield L


@pytest.mark.parametrize("deg,M", se.LAYOUTS)
def test_layout(on_emu, deg, M):
    se.case_layout(deg, M)


@pytest.mark.parametrize("deg,M", [(0, 1), (2, 9), (3, 16)])
def test_layout_far_camera(on_emu, deg, M):
    se.case_layout(deg, M, dist=1000)


def test_fan_in(on_emu):
    se.case_layout(1, 9, fans=(1, 2, 33, 512, 4096))


def test_modifier_and_depth(on_emu):
    se.case_modifier_depth(2, 9)


def test_device_cut_tail(on_emu):
    se.case_device_cut_tail(leaves=800)


@pytest.mark.parametrize("deg,M", [(3, 16), (2, 9)])
def test_row_blocks(on_emu, deg, M):
    se.case_row_blocks(deg, M)


@pytest.mark.parametrize("deg,M", [(3, 16), (1, 9)])
def test_schedules(on_emu, deg, M):
    se.case_schedules(deg, M)


@pytest.mark.parametrize("deg,M", [(1, 9), (3, 16)])
def test_composition(on_emu, deg, M):
    se.case_composition(deg, M)


# ---- rows read and written as float4 must be 16-byte aligned --------------------------------------------------------------
def _odd_view(a):
    """a copy of `a` at a 4-byte (not 16-byte) offset"""
    from emu_api import aligned
    a = np.asarray(a, np.float32)
    buf = aligned(a.nbytes + 16, np.float32)
    v = buf[1:1 + a.size].reshape(a.shape)
    v[...] = a
    assert v.ctypes.data % 16 == 4
    return v


@pytest.mark.parametrize("M", [16, 9])
def test_cabi_refuses_misaligned_float4_rows(emu_so, M):
    """the forward and the backward refuse rotations, shs (when 3 M % 4 == 0), dL_drotations and dL_dsh (likewise) at a
    4-byte offset with H3DGS_EINVAL before any launch; shs of a scalar layout may sit at any float offset"""
    from emu_api import Emu, f32
    emu = Emu(emu_so)
    cam, sc, info = se.cut_scene(3 if M == 16 else 2, M, 5, fans=(1, 2), n_free=10, clamp=False)
    bg = np.zeros(3, np.float32)
    kw = dict(sh_degree=3 if M == 16 else 2, ts=sc["ts"], kids=sc["kids"], ridx=sc["ridx"], pidx=sc["pidx"])
    a, keep = emu.args(cam, bg, sc, **kw)
    good = emu.forward(a, keep)
    n0 = emu.L.h3dgs_launch_count()
    for field, src in (("rotations", sc["rotations"]), ("shs", sc["shs"])):
        b, keep_b = emu.args(cam, bg, sc, **kw)
        odd = _odd_view(src)
        setattr(b, field, odd.ctypes.data)
        if field == "shs" and (3 * M) % 4:
            out = emu.forward(b, keep_b)                       # the scalar path reads any float offset
            assert np.array_equal(out["radii"], good["radii"])
            continue
        with pytest.raises(RuntimeError, match=f"{field} must be 16-byte aligned"):
            emu.forward(b, keep_b)
        assert emu.L.h3dgs_launch_count() == n0, field
    # the backward's float4 reductions into dL_drotations and dL_dsh
    N = sc["means3D"].shape[0]
    P = a.P
    for name in ("rotations", "sh"):
        outs = dict(means3D=np.zeros((N, 3), np.float32), means2D=np.zeros((P, 3), np.float32),
                    sh=np.zeros((N, M, 3), np.float32), colors_precomp=None, opacities=np.zeros((N, 1), np.float32),
                    scales=np.zeros((N, 3), np.float32), rotations=np.zeros((N, 4), np.float32), cov3Ds_precomp=None)
        outs = {k: (None if v is None else _odd_view(v) if k == name else f32(v)) for k, v in outs.items()}
        gcol = np.zeros((3, cam.H, cam.W), np.float32)
        n1 = emu.L.h3dgs_launch_count()
        if name == "sh" and (3 * M) % 4:
            emu.backward(a, good, gcol, outs=outs)
            continue
        with pytest.raises(RuntimeError, match=f"dL_d{'rotations' if name == 'rotations' else 'sh'} must be 16-byte aligned"):
            emu.backward(a, good, gcol, outs=outs)
        assert emu.L.h3dgs_launch_count() == n1, name


def test_python_layer_copies_misaligned_views(on_emu):
    """_C hands the library 16-byte aligned rows: a contiguous view at an odd float offset is copied, an aligned tensor
    is passed as it is; a render from such views equals the render from aligned tensors"""
    import torch
    from diff_gaussian_rasterization import _C
    base = torch.arange(4 * 33 + 1, dtype=torch.float32)
    view = base[1:].view(33, 4)
    assert view.is_contiguous() and view.data_ptr() % 16 == 4
    out = _C._f32c(view, "rotations")
    assert out.data_ptr() % 16 == 0 and torch.equal(out, view)
    al = torch.zeros(33, 4)
    assert _C._f32c(al, "rotations").data_ptr() == al.data_ptr()
    cam, sc, info = se.cut_scene(3, 16, 6, fans=(1, 2), n_free=10, clamp=False)
    t = lambda a, dt=torch.float32: torch.tensor(np.asarray(a), dtype=dt)

    def odd(a):
        a = torch.tensor(np.asarray(a, np.float32))
        buf = torch.zeros(a.numel() + 4)
        v = buf[1:1 + a.numel()].view(a.shape)
        v.copy_(a)
        return v
    args = lambda rot, sh: (t(np.zeros(3)), t(sc["means3D"]), None, t(sc["opacities"]), t(sc["scales"]), rot, 1.0, None,
                            t(cam.world_view_transform), t(cam.full_proj_transform), cam.tanfovx, cam.tanfovy, cam.H, cam.W,
                            sh, 3, t(cam.camera_center), False, False, t(sc["ridx"], torch.int32), t(sc["pidx"], torch.int32),
                            t(sc["ts"]), t(sc["kids"], torch.int32), False)
    a = _C.rasterize_gaussians(*args(t(sc["rotations"]), t(sc["shs"])))
    b = _C.rasterize_gaussians(*args(odd(sc["rotations"]), odd(sc["shs"])))
    assert torch.equal(a[2], b[2]) and torch.equal(a[1], b[1])

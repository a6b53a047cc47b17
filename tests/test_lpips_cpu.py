"""CPU: LPIPS with the VGG16 network.

  * the float64 restatement (tests/lpips_ref.py) against tests/golden/lpips.npz, which the reference's own
    lpipsPyTorch.LPIPS('vgg') computed on seeded weights (tests/golden/make_golden_lpips.py);
  * LpipsVGG's loader against malformed state dicts;
  * csrc/lpips.cu on the emulation build: conv layers against float64 within the per-layer budget, the head on its own
    taps within the head budget, an identical pair giving exactly 0, and the golden's value."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emul"))

import lpips_ref  # noqa: E402


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "lpips.npz"))


@pytest.fixture(scope="module")
def weights(golden):
    vgg, lin = lpips_ref.seeded_state_dicts(int(golden["seed"]))
    assert lpips_ref.checksum(vgg, lin) == str(golden["checksum"]), "the seeded weights differ from the fixture's"
    return vgg, lin


def _inputs(z, name):
    prep, use_mask, crop, _ = (bool(v) for v in z[f"{name}_flags"])
    x, y = torch.from_numpy(z[f"{name}_x"]), torch.from_numpy(z[f"{name}_y"])
    mask = torch.from_numpy(z[f"{name}_mask"]) if use_mask else None
    if prep:
        x, y = lpips_ref.preprocess(x, mask, crop), lpips_ref.preprocess(y, mask, crop)
    return x, y


def test_restatement_matches_the_reference(golden, weights):
    """fp32 budget: the reference ran 13 fp32 convolutions of up to 4608 terms on the CPU; its per-tap means agree with
    float64 to 1e-4 relative (plus 1e-9 for the identical pair's zeros)"""
    for name in golden["names"]:
        taps, value = lpips_ref.lpips(*_inputs(golden, str(name)), *weights)
        ref = golden[f"{name}_taps"]
        assert np.all(np.abs(np.array(taps) - ref) <= 1e-4 * np.abs(ref) + 1e-9), (name, taps, ref)
        assert abs(value - float(golden[f"{name}_value"])) <= 1e-4 * abs(value) + 1e-9, name
        if golden[f"{name}_flags"][3]:
            assert value == 0.0 and float(golden[f"{name}_value"]) == 0.0


def test_too_small_raises_as_the_reference_does(golden, weights):
    H, W = (int(v) for v in golden["too_small_shape"])
    assert str(golden["too_small_error"])            # the reference raised
    with pytest.raises(ValueError):
        lpips_ref.lpips(torch.zeros(3, H, W), torch.zeros(3, H, W), *weights)


def test_loader_rejects_malformed_state_dicts(weights):
    from h3dgs.lpips import checked_weights
    vgg, lin = weights
    convs, biases, lins = checked_weights(vgg, lin)
    assert len(convs) == 13 and len(biases) == 13 and [t.numel() for t in lins] == list(lpips_ref.TAP_CHANNELS)
    bare = {k[len("features."):]: v for k, v in vgg.items()}              # vgg16().features.state_dict() keys
    assert all(torch.equal(a, b) for a, b in zip(checked_weights(bare, lin)[0], convs))
    cases = [("features.5.weight", None, "features.5.weight"),
             ("features.28.bias", torch.zeros(511), "features.28.bias"),
             ("features.0.weight", torch.zeros(64, 3, 3), "features.0.weight"),
             ("features.2.weight", torch.zeros(64, 64, 3, 3, dtype=torch.int32), "features.2.weight"),
             ("lin3.model.1.weight", None, "lin3.model.1.weight"),
             ("lin0.model.1.weight", torch.zeros(1, 65, 1, 1), "lin0.model.1.weight"),
             ("lin4.model.1.weight", "not a tensor", "lin4.model.1.weight")]
    for key, val, named in cases:
        v2, l2 = dict(vgg), dict(lin)
        sd = v2 if key.startswith("features") else l2
        if val is None:
            del sd[key]
        else:
            sd[key] = val
        with pytest.raises(ValueError, match=named.replace(".", r"\.")):
            checked_weights(v2, l2)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """the emulation build of the library's sources plus lpips.cu, with csrc/mma.cuh (inline PTX) replaced by its
    emulator twin tests/emul/mma_emu.cuh, as the build replaces tma.cuh by tma_emu.cuh"""
    from unittest import mock
    import build_emu
    from emu_api import Emu
    with open(os.path.join(HERE, "emul", "mma_emu.cuh")) as f:
        twin = f.read()
    rewrite = build_emu.rewrite

    def rewrite_with_twin(text):
        return twin if "mma.sync.aligned.m16n8k8" in text else rewrite(text)
    with mock.patch.object(build_emu, "SOURCES", build_emu.SOURCES + ["lpips.cu"]), \
            mock.patch.object(build_emu, "rewrite", rewrite_with_twin):
        return Emu(build_emu.build(str(tmp_path_factory.mktemp("h3dgs_emu_lpips"))))


@pytest.fixture(scope="module")
def packed(emu, weights):
    from h3dgs.lpips import checked_weights, pack
    return pack(emu.L, *checked_weights(*weights))


def _nhwc_input(x):
    """[3,H,W] -> the network input the library builds: [H][W][8], z-scored, channels 3..7 zero"""
    z = lpips_ref.z_score(x).float()
    out = torch.zeros(x.shape[1], x.shape[2], 8)
    out[..., :3] = z.permute(1, 2, 0)
    return out


def _conv(emu, packed, layer, x):
    from emu_api import aligned, f32, ptr
    H, W, _ = x.shape
    co = lpips_ref.CONV_CHANNELS[layer][1]
    out = aligned(H * W * co * 4, np.float32, (H, W, co))
    xin = f32(x.numpy())                         # kept alive across the call
    emu.check(emu.L.h3dgs_lpips_conv(layer, H, W, ptr(xin), packed.data_ptr(), ptr(out), None))
    return torch.from_numpy(out.copy())


def _check_layer(vgg, layer, x, ours):
    """ours [H,W,C_out] against float64 on the same input x [H,W,C_in] -> the largest fraction of the budget used"""
    i = lpips_ref.CONV_INDICES[layer]
    ci = lpips_ref.CONV_CHANNELS[layer][0]
    ref, bound = lpips_ref.conv_layer(x[..., :ci].permute(2, 0, 1), vgg[f"features.{i}.weight"], vgg[f"features.{i}.bias"],
                                      with_bound=True)
    K = 9 * max(ci, 8)
    err = (ours.permute(2, 0, 1).double() - ref).abs()
    budget = lpips_ref.layer_budget(K, bound)
    assert bool((err <= budget).all()), (layer, float(err.max()), float((err / budget).max()))
    return float((err / budget).max())


def test_emulated_conv_layers_within_budget(emu, packed, weights, golden):
    vgg, _ = weights
    x = _nhwc_input(torch.from_numpy(golden["odd_17x33_x"]))
    y0 = _conv(emu, packed, 0, x)
    _check_layer(vgg, 0, x, y0)
    _check_layer(vgg, 1, y0, _conv(emu, packed, 1, y0))
    g = torch.Generator().manual_seed(5)
    for layer, (H, W) in ((2, (9, 17)), (7, (5, 19)), (12, (3, 4))):      # odd and non-tile-multiple sizes
        xin = torch.relu(torch.randn((H, W, lpips_ref.CONV_CHANNELS[layer][0]), generator=g))
        _check_layer(vgg, layer, xin, _conv(emu, packed, layer, xin))


def _emu_lpips(emu, packed, x, y, H, W):
    from emu_api import aligned, f32, ptr
    a, t, p = C.c_int64(), C.c_int64(), C.c_int64()
    emu.check(emu.L.h3dgs_lpips_scratch_floats(H, W, C.byref(a), C.byref(t), C.byref(p)))
    act, taps = aligned(a.value * 4, np.float32), aligned(t.value * 4, np.float32)
    parts, out = aligned(p.value * 8, np.float64), aligned(8, np.float64)
    xa, ya = f32(x.numpy()), f32(y.numpy())      # kept alive across the calls
    emu.check(emu.L.h3dgs_lpips_features(H, W, 0, ptr(ya), None, None, 0, packed.data_ptr(), ptr(act),
                                         ptr(taps), None))
    ty = torch.from_numpy(taps.copy())
    emu.check(emu.L.h3dgs_lpips_features(H, W, 0, ptr(xa), None, None, 0, packed.data_ptr(), ptr(act),
                                         ptr(taps), None))
    tx = torch.from_numpy(taps.copy())
    taps[:] = ty.numpy()
    emu.check(emu.L.h3dgs_lpips_distance(H, W, 0, ptr(xa), None, None, 0, packed.data_ptr(), ptr(act),
                                         ptr(taps), ptr(parts), None, ptr(out), 1, None))
    return lpips_ref.split_taps(tx, H, W), lpips_ref.split_taps(ty, H, W), float(out[0])


def test_emulated_pair_head_and_golden(emu, packed, weights, golden):
    vgg, lin = weights
    x, y = _inputs(golden, "min_16x16")
    tx, ty, value = _emu_lpips(emu, packed, x, y, 16, 16)
    head = lpips_ref.head(tx, ty, lin)
    assert abs(value - sum(head)) <= sum(lpips_ref.head_bound(tx, ty, lin)), (value, sum(head))
    # the whole value against the reference's: TF32 network, well inside 2 % of the value here
    assert abs(value - float(golden["min_16x16_value"])) <= 2e-2 * float(golden["min_16x16_value"])
    # an identical pair: exactly zero
    _, _, same = _emu_lpips(emu, packed, x, x.clone(), 16, 16)
    assert same == 0.0

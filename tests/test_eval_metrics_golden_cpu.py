"""CPU: the evaluation metrics kernel (csrc/metrics.cu, emulation build) against tests/golden/eval_metrics.npz, which the
reference's own render_post / psnr / ssim computed (tests/golden/make_golden_eval.py): exposure direction, clamps, the
train_test_exp crop with SSIM's zero padding at the crop border, the alpha mask, PSNR = inf on an exact channel."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emul"))

from h3dgs import _lib  # noqa: E402


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """the emulation build of the library's sources plus metrics.cu (the evaluation kernels)"""
    from unittest import mock
    import build_emu
    from emu_api import Emu
    with mock.patch.object(build_emu, "SOURCES", build_emu.SOURCES + ["metrics.cu"]):
        return Emu(build_emu.build(str(tmp_path_factory.mktemp("h3dgs_emu_eval"))))


def _run(emu, z, i, status=None):
    from emu_api import aligned, f32, ptr
    exp, msk, crop, _ = (bool(v) for v in z[f"c{i}_flags"])
    raw, gt = f32(z[f"c{i}_raw"]), f32(z[f"c{i}_gt"])
    _, H, W = raw.shape
    x0 = W // 2 if crop else 0
    E = f32(z[f"c{i}_E"]) if exp else None
    mask = f32(z[f"c{i}_mask"]) if msk else None
    out = aligned(3 * H * (W - x0) * 4, np.float32, (3, H, W - x0))
    sums = aligned(32, np.float64, (4,))
    counter = aligned(4, np.int32, (1,))
    results = aligned(2 * _lib.EVAL_ROW * 8, np.float64, (2, _lib.EVAL_ROW))
    count, extra, cap, scan = status if status is not None else (None, 0, 0, None)
    emu.check(emu.L.h3dgs_eval_metrics(H, W, ptr(raw), ptr(gt), ptr(E), ptr(mask), x0, ptr(out), ptr(sums), ptr(count),
                                       extra, cap, ptr(scan), ptr(counter), ptr(results), 2, None))
    return out, results, counter


@pytest.mark.parametrize("i", range(9))
def test_metrics_kernel_matches_the_reference(emu, golden_dir, i):
    z = np.load(os.path.join(golden_dir, "eval_metrics.npz"))
    out, results, counter = _run(emu, z, i)
    assert int(counter[0]) == 1
    ref_img = z[f"c{i}_image"]
    assert out.shape == ref_img.shape
    assert np.abs(out - ref_img).max() <= 1e-6
    p, s = results[0, 0], results[0, 1]
    pr, sr = float(z[f"c{i}_psnr"]), float(z[f"c{i}_ssim"])
    if np.isinf(pr):
        assert np.isinf(p) and p > 0
    else:
        assert abs(p - pr) <= 1e-4, (p, pr)
    assert abs(s - sr) <= 1e-5 * abs(sr), (s, sr)
    assert results[0, 2] == 0.0 and results[0, 3] == 0.0


def test_status_words_and_slots(emu, golden_dir):
    from emu_api import aligned
    z = np.load(os.path.join(golden_dir, "eval_metrics.npz"))
    count = aligned(4, np.int32, (1,)); count[0] = 90
    scan = aligned(16, np.uint32, (4,)); scan[:3] = (1234, 77, 0)
    _, results, _ = _run(emu, z, 0, status=(count, 10, 100, scan))
    assert list(results[0, 2:]) == [0.0, 100.0, 1234.0, 77.0]
    _, results, _ = _run(emu, z, 0, status=(count, 11, 100, scan))      # 101 rows > 100: a row overflow
    assert results[0, 2] == 1.0 and results[0, 3] == 101.0
    scan[2] = 1                                                          # binning overflow
    _, results, _ = _run(emu, z, 0, status=(count, 0, 100, scan))
    assert results[0, 2] == 1.0


def test_rows_go_to_consecutive_slots_and_stop_at_the_end(emu, golden_dir):
    from emu_api import aligned, f32, ptr
    z = np.load(os.path.join(golden_dir, "eval_metrics.npz"))
    raw, gt = f32(z["c0_raw"]), f32(z["c0_gt"])
    _, H, W = raw.shape
    sums = aligned(32, np.float64, (4,))
    counter = aligned(4, np.int32, (1,))
    results = aligned(4 * _lib.EVAL_ROW * 8, np.float64, (4, _lib.EVAL_ROW))
    results[3] = -7.0
    for _ in range(4):      # max_rows = 3: the fourth call is counted, not stored
        emu.check(emu.L.h3dgs_eval_metrics(H, W, ptr(raw), ptr(gt), None, None, 0, None, ptr(sums), None, 0, 0, None,
                                           ptr(counter), ptr(results), 3, None))
    assert int(counter[0]) == 4
    assert np.all(results[:3, 0] == results[0, 0]) and np.all(results[3] == -7.0)
    with pytest.raises(RuntimeError, match="bad arguments"):
        emu.check(emu.L.h3dgs_eval_metrics(H, W, ptr(raw), ptr(gt), None, None, W, None, ptr(sums), None, 0, 0, None,
                                           ptr(counter), ptr(results), 3, None))

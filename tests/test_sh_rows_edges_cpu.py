"""CPU: tests/test_gpu_sh_rows_edges.py's cases (the SH backward's own-row stores per full-size row across every float4
layout, run_scene's run geometry, row blocks, and the row-count buffer's eager states) on the emulation build of the
kernels (tests/emul/).  The captured states need CUDA graphs and stay on the GPU."""
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emul"))

import test_gpu_sh_rows_edges as sr  # noqa: E402


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    from build_emu import build
    return build(str(tmp_path_factory.mktemp("h3dgs_emu_sh_rows_edges")))


@pytest.fixture
def on_emu(emu_so):
    from fake_device import cpu_as_device, cuda_names_mean_cpu
    with cpu_as_device(emu_so) as L, cuda_names_mean_cpu():
        yield L


@pytest.mark.parametrize("deg,M", sr.FLOAT4_LAYOUTS)
@pytest.mark.parametrize("scene", ["runs", "cut"])
def test_layout(on_emu, scene, deg, M):
    sr.case_layout(deg, M, scene)


@pytest.mark.parametrize("deg,M", [(3, 16), (1, 8)])
def test_row_blocks(on_emu, deg, M):
    sr.case_row_blocks(deg, M)


def test_row_count_buffer_eager_states(emu_so):
    out = sr.run_buffer_states(emu_so)
    for s in ("state: eager", "state c:"):
        assert s in out, out[-3000:]

"""CPU: tests/test_gpu_sh_backward_rows.py's cases (the SH backward's own-row stores against its reductions and against
chain_ref) on the emulation build of the kernels (tests/emul/)."""
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emul"))

import test_gpu_sh_backward_rows as sr  # noqa: E402


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    from build_emu import build
    return build(str(tmp_path_factory.mktemp("h3dgs_emu_sh_rows")))


@pytest.fixture
def on_emu(emu_so):
    from fake_device import cpu_as_device, cuda_names_mean_cpu
    with cpu_as_device(emu_so) as L, cuda_names_mean_cpu():
        yield L


@pytest.mark.parametrize("deg,M", [(3, 16), (1, 4), (2, 12)])
def test_store_equals_reduce(on_emu, deg, M):
    sr.case_store_equals_reduce(deg, M)

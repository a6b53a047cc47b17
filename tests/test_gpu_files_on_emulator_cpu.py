"""CPU: the GPU test files themselves -- the same parity tests the H100 runs, with their own criteria -- executed
against the emulation build of the kernels (H3DGS_EMULATE=1, tests/conftest.py, tests/emul/): the product's Python
layer runs unchanged on CPU tensors and the kernels run under the SIMT emulator.  The 1080p / 4K frames are left to
the GPU (they pass here too, in minutes); NCCL and the optimizer kernel are out of the emulator's reach.  The fused
L1 + SSIM loss kernels (csrc/loss.cu) run on the emulation build in tests/test_ssim_ref_cpu.py."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_gpu_parity_files_pass_on_the_emulator():
    env = dict(os.environ, H3DGS_EMULATE="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_parity.py", "tests/test_gpu_hierarchy.py",
                        "tests/test_gpu_pipeline.py", "tests/test_gpu_blend_edges.py",
                        "tests/test_gpu_chain_edges.py", "tests/test_gpu_preprocess_edges.py", "-q", "-p", "no:cacheprovider",
                        "-k", "not 3840 and not full_size and not config2"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = r.stdout[-1500:]
    assert r.returncode == 0, tail + r.stderr[-1500:]
    m = re.search(r"(\d+) passed", tail)
    assert m and int(m.group(1)) >= 70 and "failed" not in tail, tail


def test_gpu_blend_deep_passes_on_the_emulator():
    """The deep tile lists (every tile-sort class up to 8192 entries, the radix sort beyond, walls at every batch edge)
    in their flat and hierarchy variants; the inverse-depth variants only add the tenth sum and are left to the GPU."""
    env = dict(os.environ, H3DGS_EMULATE="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_blend_deep.py", "-q", "-p", "no:cacheprovider",
                        "-k", "not depth"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    tail = r.stdout[-1500:]
    assert r.returncode == 0, tail + r.stderr[-1500:]
    m = re.search(r"(\d+) passed", tail)
    assert m and int(m.group(1)) >= 6 and "failed" not in tail, tail

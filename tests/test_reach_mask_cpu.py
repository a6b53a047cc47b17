"""CPU: csrc/reach_mask.cuh::block_mask16 (the 4x4-block reach mask the record gather stores and both blend kernels
cull by), compiled for the host, against a brute-force per-pixel evaluation in three families -- 200 000 random projected
Gaussians x tile positions, needles (Gaussians seen edge-on, sigma_long 50 .. 600 px) over every tile they can reach, and
opacities at prev / fp32 / next of 1/255 with means on pixel centres, tile corners and edges: no pixel with
alpha >= 1/255 outside a marked block, and < 2 % of the marked blocks untouched, per family.  Conics that are not
positive definite and non-finite means or conics get the fallback 0xFFFF, a NaN opacity 0."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_block_reach_mask_is_conservative_and_tight(tmp_path):
    exe = str(tmp_path / "reach_mask_test")
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "emul", "reach_mask_test.cpp"),
                    "-lm"], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr

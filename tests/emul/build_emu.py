"""TEST INFRASTRUCTURE ONLY.  Builds libh3dgs_emu.so: the library's own .cu sources, compiled with g++
against the SIMT emulator (simt_emu.h), exporting the same C-ABI as libh3dgs.so but running on the CPU.
The sources are COPIED to a scratch directory and only mechanically rewritten there (launch syntax,
CUDA includes, dynamic shared memory, the TMA wrappers); nothing of this is part of the product."""
import os
import re
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "hierarchical-3d-gaussians_b200", "csrc")
SOURCES = ["api.cu", "preprocess.cu", "binning.cu", "render_forward.cu", "render_backward.cu", "preprocess_backward.cu",
           "hierarchy.cu", "l1_loss.cu", "loss.cu"]

_LAUNCH = re.compile(r"((?:\b[\w:]+)(?:<[^<>;()]*>)?)\s*<<<(.*?)>>>\s*\(", re.S)


def rewrite(text):
    text = text.replace("#include <cuda_runtime.h>", '#include "simt_emu.h"')
    text = re.sub(r"#include <cub/cub.cuh>\n", "", text)
    text = re.sub(r"extern\s+__shared__\s+(\w+)\s+(\w+)\[\];", r"\1* \2 = (\1*)simt::g_dyn_smem;", text)
    text = re.sub(r"__device__\s+__constant__", "static const", text)
    text = _LAUNCH.sub(lambda m: f"SIMT_LAUNCH(({m.group(1)}), {m.group(2)})(", text)
    # the three MUFU wrappers written in inline PTX
    text = re.sub(r'asm\("ex2\.approx\.ftz\.f32 %0, %1;" : "=f"\((\w+)\) : "f"\((.*?)\)\);', r"\1 = exp2f(\2);", text)
    text = re.sub(r'asm\("lg2\.approx\.ftz\.f32 %0, %1;" : "=f"\((\w+)\) : "f"\((.*?)\)\);', r"\1 = log2f(\2);", text)
    text = re.sub(r'asm\("rcp\.approx\.ftz\.f32 %0, %1;" : "=f"\((\w+)\) : "f"\((.*?)\)\);', r"\1 = 1.0f / (\2);", text)
    return text


def build(out_dir):
    """-> path of libh3dgs_emu.so (built under out_dir)"""
    src_dir = os.path.join(out_dir, "hierarchical-3d-gaussians_b200", "csrc")
    os.makedirs(src_dir, exist_ok=True)
    os.makedirs(os.path.join(out_dir, "include"), exist_ok=True)
    shutil.copy(os.path.join(ROOT, "include", "h3dgs.h"), os.path.join(out_dir, "include", "h3dgs.h"))
    for f in os.listdir(CSRC):
        if f.endswith((".cu", ".cuh")) and f != "tma.cuh":
            with open(os.path.join(CSRC, f)) as fh:
                text = rewrite(fh.read())
            with open(os.path.join(src_dir, f.replace(".cu", ".cpp") if f.endswith(".cu") else f), "w") as fh:
                fh.write(text)
    shutil.copy(os.path.join(HERE, "tma_emu.cuh"), os.path.join(src_dir, "tma.cuh"))
    for f in ("simt_emu.h", "simt_emu.cpp"):
        shutil.copy(os.path.join(HERE, f), os.path.join(src_dir, f))
    flags = ["-std=c++17", "-O1", "-g", "-fPIC", "-ffp-contract=off", "-fno-strict-aliasing", "-w", "-D__CUDACC__",
             "-DH3_PAIR_HOST_EMU", "-DH3_HOST_EMU", "-I", src_dir]
    objs = []
    for f in [s.replace(".cu", ".cpp") for s in SOURCES] + ["simt_emu.cpp"]:
        obj = os.path.join(out_dir, f.replace(".cpp", ".o"))
        r = subprocess.run(["/usr/bin/g++"] + flags + ["-c", os.path.join(src_dir, f), "-o", obj], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"g++ failed for {f}:\n{r.stderr[:6000]}")
        objs.append(obj)
    so = os.path.join(out_dir, "libh3dgs_emu.so")
    r = subprocess.run(["/usr/bin/g++", "-shared", "-o", so] + objs + ["-lm", "-lpthread"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stderr[:6000])
    return so


if __name__ == "__main__":
    import sys
    print(build(sys.argv[1] if len(sys.argv) > 1 else "/tmp/h3dgs_emu"))

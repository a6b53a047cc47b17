"""TEST INFRASTRUCTURE ONLY.  A memcheck for the kernels without a GPU: build the emulation library with
AddressSanitizer (heap and globals -- `__shared__` arrays are globals in the emulator; stack instrumentation is off
because the fibers switch stacks by hand), preload libasan so that numpy's buffers get red zones too, and run a set
of scenes through the blend kernels, the sharded schedule, the fused cut gather, the device-side LOD cut /
capacity mode, and the preprocess edge families with non-finite inputs and huge splats (tests/preprocess_ref.py).  Usage:   python tests/emul/asan_check.py          (re-executes itself under LD_PRELOAD)
A deliberately short output buffer is reported as heap-buffer-overflow (checked by --negative-control)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = "/tmp/h3dgs_emu_asan"


def build():
    sys.path.insert(0, HERE)
    import build_emu
    build_emu.build(OUT)
    src = os.path.join(OUT, "hierarchical-3d-gaussians_b200", "csrc")
    flags = ["-std=c++17", "-O1", "-g", "-fPIC", "-ffp-contract=off", "-fno-strict-aliasing", "-w", "-D__CUDACC__",
             "-DH3_PAIR_HOST_EMU", "-DH3_HOST_EMU", "-I", src, "-fsanitize=address", "--param", "asan-stack=0", "-fno-omit-frame-pointer"]
    objs = []
    for f in [s.replace(".cu", ".cpp") for s in build_emu.SOURCES] + ["simt_emu.cpp"]:
        o = os.path.join(OUT, f.replace(".cpp", ".asan.o"))
        subprocess.run(["/usr/bin/g++"] + flags + ["-c", os.path.join(src, f), "-o", o], check=True)
        objs.append(o)
    so = os.path.join(OUT, "libh3dgs_emu_asan.so")
    subprocess.run(["/usr/bin/g++", "-shared", "-fsanitize=address", "-o", so] + objs + ["-lm"], check=True)
    return so


def run_cases(so, negative):
    for p in (ROOT, os.path.join(ROOT, "hierarchical-3d-gaussians_b200"), os.path.join(ROOT, "tests"), HERE):
        sys.path.insert(0, p)
    import ctypes as C
    import numpy as np
    from emu_api import Emu
    from util import make_scene
    emu = Emu(so)
    if negative:
        from h3dgs import _lib
        cam, sc, ts, kids, bg = make_scene(1000, 64, 48, seed=1)
        a, keep = emu.args(cam, bg, sc)
        bufs = [None] * 3

        def alloc(_u, which, n):
            bufs[which] = np.zeros(int(n), np.uint8)
            return bufs[which].ctypes.data
        cb = _lib.ALLOC_FN(alloc)
        color, radii, n = np.zeros(3 * cam.H * cam.W, np.float32), np.zeros(1000 - 64, np.int32), C.c_int64(0)
        emu.L.h3dgs_rasterize_forward(C.byref(a), cb, None, color.ctypes.data, radii.ctypes.data, None, C.byref(n), None)
        print("negative control: NOT reported")
        return
    import test_emu_kernels_cpu as T
    import preprocess_ref as PR
    import test_preprocess_ref_cpu as TP
    n = 0
    # rows that do not project to finite values (NaN / inf in each input) and huge splats (saturated radius and rect):
    # the binning must never be handed a counted tile that no row fills
    for which in PR.NONFINITE_INPUTS:
        TP.test_rows_that_do_not_project_are_invisible(emu, which)
        n += 1
    TP.hold(emu, PR.family_huge())
    TP.hold(emu, PR.family_degenerate())
    n += 2
    print(f"asan: {n} non-finite / huge / degenerate cases done", flush=True)
    for (P, W, H, kw, depth) in [(3000, 256, 192, dict(mode="hier", seed=42), True), (1500, 160, 96, dict(seed=7), False),
                                 (300, 15, 33, dict(seed=3, scale_k=2e-2), False),
                                 (6000, 96, 64, dict(seed=11, scale_k=3e-2, zmax=6.0), False),
                                 (16000, 48, 48, dict(seed=13, scale_k=6e-2, zmax=4.0), False)]:
        cam, sc, ts, kids, bg = make_scene(P, W, H, **kw)
        T._check(emu, cam, sc, bg, ts, kids, do_depth=depth, tol=5e-5)
        n += 1
    for t in (T.test_tile_shards_equal_the_whole_frame, T.test_sharded_frame_with_row_blocks,
              T.test_fused_cut_gather_and_scatter, T.test_device_lod_cut_and_skipped_rows):
        t(emu)
        n += 1
    for G in (2, 4):                                   # peer mode: rank mask, push into the staging areas, gather in K9
        T.test_peer_mode_fused_collectives_schedule(emu, G)
        n += 1
    # round 2: the in-register tile sort over all size classes, the TMA-staged single-pass cut (bulk and plain-load paths),
    # the L1 kernel's image forwarding, the split-phase zero-fill
    T.test_register_sort_size_classes_with_equal_depths(emu)
    for tau, mis in ((6.0, False), (6.0, True)):
        T.test_single_pass_cut_over_many_tiles.__wrapped__(emu, tau, mis, False, None) if hasattr(T.test_single_pass_cut_over_many_tiles, "__wrapped__") \
            else T.test_single_pass_cut_over_many_tiles(emu, tau, mis, False, None)
    for G in (2, 4):
        T.test_peer_l1_kernel_forwards_the_rendered_rows(emu, G)
    T.test_split_phases_fill_the_scatter_outputs_beside_the_replay(emu)
    n += 6
    print(f"asan check complete: {n} cases, no report")


if __name__ == "__main__":
    if os.environ.get("H3DGS_ASAN_CHILD") != "1":
        so = build()
        libasan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
        env = dict(os.environ, LD_PRELOAD=libasan, ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0", H3DGS_ASAN_CHILD="1")
        r = subprocess.run([sys.executable, os.path.abspath(__file__)] + sys.argv[1:], env=env)
        sys.exit(0 if (r.returncode == 0) != ("--negative-control" in sys.argv) else 1)
    run_cases(os.path.join(OUT, "libh3dgs_emu_asan.so"), "--negative-control" in sys.argv)

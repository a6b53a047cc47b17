#!/usr/bin/env python
"""Cost of the LOD budget (csrc/lod_budget.cu) on bench.py's hier3m workload (config #3: 3 M nodes, 1920x1080), one GPU:

  pass    device time of h3dgs_lod_budget next to h3dgs_lod_cut's at the threshold it picks, per view and budget, and
          at two floors (tau 0 and tau 6): the floor decides how many nodes are kept as keys, while the sort runs over
          all N pairs either way (its length is a launch constant of a capturable call);
  sweep   evaluator frames/s of a budget sweep (HierarchyEvaluator(budgets=..., tau_floor=0)) against the tau sweep
          (taus 0, 3, 6, 15), the same number of frames per view.

  python tools/bench_lod_budget.py [--reps 50] [--sweeps 3] [--warmup 1]

Prints one JSON line with the GPU name and power limit.  Writes nothing into the tree (the workload cache goes to the
temporary directory, as for bench.py)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (workloads; puts the package on sys.path)

TAUS = [0.0, 3.0, 6.0, 15.0]
BUDGETS = [2_000_000, 1_000_000, 500_000, 200_000]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--sweeps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_lod_budget.py needs a CUDA device: there is no CPU fallback for this path")
    dev = "cuda:0"
    torch.cuda.set_device(0)
    arrays, cams = bench.build_workload("hier3m", device=dev)
    from h3dgs import _lib, pipeline
    from h3dgs.evaluate import HierarchyEvaluator
    L = _lib.lib()
    scene = pipeline.Scene(arrays, device=dev, requires_grad=False)
    dcams = [pipeline.DeviceCamera(c, device=dev) for c in cams]
    N = scene.nodes.shape[0]
    stream = torch.cuda.current_stream().cuda_stream
    scratch = torch.empty(int(L.h3dgs_lod_budget_scratch_bytes(N)), dtype=torch.uint8, device=dev)
    cut_scratch = torch.empty(int(L.h3dgs_expand_scratch_bytes(N)), dtype=torch.uint8, device=dev)
    thr = torch.empty(1, device=dev)
    info = torch.empty(4, dtype=torch.int32, device=dev)
    count = torch.empty(1, dtype=torch.int32, device=dev)

    def budget(c, floor, B):
        _lib.check(L.h3dgs_lod_budget(N, scene.nodes.data_ptr(), scene.boxes.data_ptr(), c.campos.data_ptr(), floor, None, B,
                                      None, thr.data_ptr(), info.data_ptr(), scratch.data_ptr(), stream))

    def cut(c):
        _lib.check(L.h3dgs_lod_cut(N, scene.nodes.data_ptr(), scene.boxes.data_ptr(), 0.0, thr.data_ptr(), c.campos.data_ptr(),
                                   scene.render_indices.data_ptr(), scene.parent_indices.data_ptr(),
                                   scene.nodes_for_render.data_ptr(), scene.interpolation_weights.data_ptr(),
                                   scene.num_siblings.data_ptr(), count.data_ptr(), cut_scratch.data_ptr(), stream))

    def device_ms(fn):
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.reps

    passes = []
    for vi, c in enumerate(dcams):
        for tau_floor in (0.0, 6.0):
            floor = pipeline.fov_threshold(tau_floor, c)
            for B in BUDGETS:
                ms_budget = device_ms(lambda: budget(c, floor, B))
                t, (rows, unmet, kept, total) = thr.item(), info.tolist()
                ms_cut = device_ms(lambda: cut(c))
                assert int(count.item()) == rows
                passes.append(dict(view=vi, tau_floor=tau_floor, budget=B, threshold=t, rows=rows, unmet=unmet,
                                   rows_at_floor=total, kept_fraction=kept / N, budget_ms=ms_budget, cut_ms=ms_cut))

    g = torch.Generator(device="cpu").manual_seed(5)
    gts = [torch.rand((3, c.H, c.W), generator=g).to(dev) for c in dcams]
    ev_tau = HierarchyEvaluator(scene, dcams, gts, TAUS)
    ev_budget = HierarchyEvaluator(scene, dcams, gts, None, budgets=BUDGETS, tau_floor=0.0)

    def sweep(ev):
        ev.enqueue()
        return ev.finish()

    def timed(ev):
        for _ in range(args.warmup):
            sweep(ev)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(max(args.sweeps, 1)):
            res = sweep(ev)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), res
    ms_t, res_t = timed(ev_tau)
    ms_b, res_b = timed(ev_budget)
    frames = len(dcams) * len(TAUS)
    n = max(args.sweeps, 1)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:    # pragma: no cover
        q = f"unavailable: {e}"
    print(json.dumps({
        "workload": bench.WORKLOADS["hier3m"], "nodes": N, "reps": args.reps, "passes": passes,
        "budget_ms_mean": sum(p["budget_ms"] for p in passes) / len(passes),
        "cut_ms_mean": sum(p["cut_ms"] for p in passes) / len(passes),
        "sweep_fps_tau": n * frames / (ms_t * 1e-3), "sweep_fps_budget": n * frames / (ms_b * 1e-3),
        "rerun_tau": res_t["rerun"], "rerun_budget": res_b["rerun"],
        "budget_sweep": {str(B): {"psnr": res_b["psnr"][B], "ssim": res_b["ssim"][B],
                                  "mean_rows": float(res_b["budget_rows"][i, :, 2].mean()),
                                  "mean_tau": float(res_b["budget_rows"][i, :, 1].mean()),
                                  "unmet_views": int(res_b["budget_rows"][i, :, 3].sum())} for i, B in enumerate(BUDGETS)},
        "tau_sweep": {str(t): {"psnr": res_t["psnr"][t], "ssim": res_t["ssim"][t]} for t in TAUS},
        "gpu": q}))


if __name__ == "__main__":
    main()

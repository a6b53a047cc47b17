#!/usr/bin/env python
"""Frames/s of render_hierarchy.py's evaluation sweep on bench.py's workloads (one GPU): every view at
tau in {0, 3, 6, 15}, PSNR + SSIM, no mask, no exposure, black background.  Two forms, whole sweeps timed:

  value   h3dgs.evaluate.HierarchyEvaluator: one graph replay per frame, one read-back per sweep (frames that overflow
          the learned capacities are re-run through the exact path inside the timed region);
  dropin  the drop-in flow as render_hierarchy.py runs it, mirrored with our own code: pipeline.render_hier (two host
          round trips, the PyTorch gather / lerp) + clamps + mask product + PyTorch PSNR + h3dgs.loss.ssim, accumulated on
          the device and read once per tau (the script's print).  Its per-frame torch.cuda.empty_cache() is left out.

  python tools/bench_eval.py [--workload hier3m] [--sweeps 5] [--warmup 2]

Prints one JSON line, with the GPU name, power limit and the SM clocks sampled during the run.  Writes nothing into the
tree (the workload cache goes to the temporary directory, as for bench.py)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (workloads and the clock sampler; puts the package on sys.path)

TAUS = [0.0, 3.0, 6.0, 15.0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="hier3m", choices=[k for k in bench.WORKLOADS if k != "flat1m"])
    ap.add_argument("--sweeps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py needs a CUDA device: there is no CPU fallback for this path")
    dev = "cuda:0"
    torch.cuda.set_device(0)
    W, H = bench.RESOLUTION.get(args.workload, (bench.W, bench.H))
    bench.W, bench.H = W, H
    arrays, cams = bench.build_workload(args.workload, device=dev)
    from h3dgs import pipeline
    from h3dgs.evaluate import HierarchyEvaluator
    from h3dgs.loss import ssim
    scene = pipeline.Scene(arrays, device=dev, requires_grad=False)
    dcams = [pipeline.DeviceCamera(c, device=dev) for c in cams]
    g = torch.Generator(device="cpu").manual_seed(5)
    gts = [torch.rand((3, H, W), generator=g).to(dev) for _ in cams]
    bg = torch.zeros(3, device=dev)
    ones = torch.ones((1, H, W), device=dev)

    def dropin_sweep():
        out = {}
        for tau in TAUS:
            ps, ss = 0.0, 0.0
            for c, gt in zip(dcams, gts):
                with torch.no_grad():
                    image = torch.clamp(pipeline.render_hier(scene, c, bg, pipeline.fov_threshold(tau, c))[0].clamp(0, 1), 0.0, 1.0)
                    t = torch.clamp(gt, 0.0, 1.0)
                    image = image * ones
                    t = t * ones
                    mse = ((image - t) ** 2).view(3, -1).mean(1, keepdim=True)
                    ps = ps + (20 * torch.log10(1.0 / torch.sqrt(mse))).mean().double()
                    ss = ss + ssim(image, t).mean().double()
            out[tau] = (float(ps) / len(dcams), float(ss) / len(dcams))
        return out

    ev = HierarchyEvaluator(scene, dcams, gts, TAUS)
    r0 = next(iter(ev.renders.values()))
    caps = {"row_capacity": r0.P, "bin_capacity": r0.bin_capacity, "sort_capacity": r0.sort_capacity}

    def graphed_sweep():
        ev.enqueue()
        res = ev.finish()
        need = [dict(tau=TAUS[ti], view=ci, rows=int(r[3]), D=int(r[4]), longest_list=int(r[5])) for ti, ci, r in res["flagged"]]
        return {t: (res["psnr"][t], res["ssim"][t]) for t in TAUS}, (res["rerun"], need)

    def timed(fn, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            r = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), r

    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(1.0)
    for _ in range(args.warmup):
        graphed_sweep()
        dropin_sweep()
    frames = len(dcams) * len(TAUS)
    n = max(args.sweeps, 1)
    ms_g, (g_metrics, (rerun, need)) = timed(graphed_sweep, n)
    ms_d, d_metrics = timed(dropin_sweep, n)
    clocks = sampler.stop()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:    # pragma: no cover
        q = f"unavailable: {e}"
    fps_g, fps_d = n * frames / (ms_g * 1e-3), n * frames / (ms_d * 1e-3)
    print(json.dumps({
        "metric": f"render_hierarchy tau-sweep frames/s (PSNR + SSIM, tau in {TAUS}) @{W}x{H}", "workload": bench.WORKLOADS[args.workload],
        "value": fps_g, "unit": "frames/s", "value_dropin": fps_d, "speedup_vs_dropin": fps_g / fps_d,
        "ms_per_frame": ms_g / (n * frames), "ms_per_frame_dropin": ms_d / (n * frames), "sweeps_timed": n,
        "frames_per_sweep": frames, "rerun_frames_per_sweep": rerun, "rerun_needed": need, "capacities": caps,
        "max_psnr_diff_db": max(abs(g_metrics[t][0] - d_metrics[t][0]) for t in TAUS),
        "max_ssim_diff": max(abs(g_metrics[t][1] - d_metrics[t][1]) for t in TAUS),
        "per_tau": {str(t): {"psnr": g_metrics[t][0], "ssim": g_metrics[t][1]} for t in TAUS},
        "gpu": q, "clocks": clocks}))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""LPIPS (VGG16) on the GPU: csrc/lpips.cu against torch's cuDNN TF32 convolutions, with seeded weights (the timings do
not depend on the weights' values; nothing is downloaded).

  layers  per conv layer at the levels of a 1920x1080 frame: kernel time (CUDA events over --reps launches), FLOP from
          the shapes (2 H W 9 C_in C_out), achieved TFLOP/s and its share of the 495 TFLOP/s TF32 dense data-sheet figure,
          next to torch.nn.functional.conv2d on the same shapes (channels-last fp32, cudnn.allow_tf32 on);
  pair    one LPIPS pair at 1920x1080: LpipsVGG against the same network in torch (TF32, channels-last, weights loaded
          once -- the reference's lpips() also rebuilds VGG16 and reloads both files on every call, not counted here);
  sweep   render_hierarchy.py's tau sweep on bench.py's hier3m workload, frames/s: the evaluator without LPIPS, with
          lpips=net, and the drop-in way -- the evaluator's kept images, then the torch network on each (image, target)
          pair, 2 feature passes per frame.

  python tools/bench_lpips.py [--reps 20] [--sweeps 3] [--warmup 1]

Prints one JSON line with the GPU name, power limit and the SM clocks sampled during the run.  Writes nothing into the
tree (the workload cache goes to the temporary directory, as for bench.py)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402  (workloads and the clock sampler; puts the package on sys.path)
import lpips_ref  # noqa: E402  (the seeded weights and the network's shapes)

TAUS = [0.0, 3.0, 6.0, 15.0]
TF32_PEAK = 495e12          # H100 SXM data sheet, TF32 dense


def _timed(fn, n):
    import torch
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sweeps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch
    import torch.nn.functional as F
    if not torch.cuda.is_available():
        raise SystemExit("bench_lpips.py needs a CUDA device: there is no CPU fallback for this path")
    torch.cuda.set_device(0)
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    from h3dgs import _lib
    from h3dgs.lpips import LpipsVGG
    vgg, lin = lpips_ref.seeded_state_dicts(1)
    net = LpipsVGG.from_state_dicts(vgg, lin)
    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(1.0)

    # ---- per layer ----
    layers, H, W = [], 1080, 1920
    for l, (ci, co) in enumerate(lpips_ref.CONV_CHANNELS):
        if l in lpips_ref.POOL_BEFORE:
            H, W = H // 2, W // 2
        x = torch.rand((H, W, max(ci, 8)), device="cuda")
        y = torch.empty((H, W, co), device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        ours = lambda: _lib.check(net.L.h3dgs_lpips_conv(l, H, W, x.data_ptr(), net.weights.data_ptr(), y.data_ptr(), st))
        xt = x[..., :ci].permute(2, 0, 1)[None].contiguous(memory_format=torch.channels_last)
        w = vgg[f"features.{lpips_ref.CONV_INDICES[l]}.weight"].cuda().contiguous(memory_format=torch.channels_last)
        b = vgg[f"features.{lpips_ref.CONV_INDICES[l]}.bias"].cuda()
        theirs = lambda: F.relu(F.conv2d(xt, w, b, padding=1))
        for fn in (ours, theirs):
            _timed(fn, 3)
        ms, _ = _timed(ours, args.reps)
        ms_t, _ = _timed(theirs, args.reps)
        flop = 2.0 * H * W * 9 * ci * co
        layers.append(dict(layer=l, H=H, W=W, C_in=ci, C_out=co, gflop=flop / 1e9, ms=ms, tflops=flop / ms / 1e9,
                           share_of_tf32_peak=flop / ms / 1e-3 / TF32_PEAK, ms_cudnn=ms_t, tflops_cudnn=flop / ms_t / 1e9))
        del x, y, xt
    torch.cuda.empty_cache()
    total_flop = sum(r["gflop"] for r in layers) * 1e9
    ms_conv, ms_conv_t = sum(r["ms"] for r in layers), sum(r["ms_cudnn"] for r in layers)

    # ---- one pair at 1920x1080 ----
    g = torch.Generator().manual_seed(3)
    xa = torch.rand((3, 1080, 1920), generator=g).cuda()
    xb = (xa + 0.05 * torch.randn((3, 1080, 1920), generator=g).cuda()).clamp(0, 1)
    ws = [(vgg[f"features.{i}.weight"].cuda().contiguous(memory_format=torch.channels_last), vgg[f"features.{i}.bias"].cuda())
          for i in lpips_ref.CONV_INDICES]
    ls = [lin[f"lin{k}.model.1.weight"].cuda() for k in range(5)]
    mean, std = lpips_ref.MEAN.cuda()[None, :, None, None], lpips_ref.STD.cuda()[None, :, None, None]

    def feats(x):
        x = ((x[None] - mean) / std).contiguous(memory_format=torch.channels_last)
        out = []
        for l, (w, b) in enumerate(ws):
            if l in lpips_ref.POOL_BEFORE:
                x = F.max_pool2d(x, 2)
            x = F.relu(F.conv2d(x, w, b, padding=1))
            if l in lpips_ref.TAP_AFTER:
                out.append(x / (torch.sqrt((x * x).sum(1, keepdim=True)) + 1e-10))
        return out

    def torch_lpips(x, y):
        with torch.no_grad():
            res = [F.conv2d((a - b) ** 2, l).mean((2, 3), True) for a, b, l in zip(feats(x), feats(y), ls)]
            return torch.sum(torch.cat(res, 0), 0, True)

    for fn in (lambda: net(xa, xb), lambda: torch_lpips(xa, xb)):
        _timed(fn, 2)
    ms_pair, v_ours = _timed(lambda: net(xa, xb), max(args.reps // 4, 3))
    ms_pair_t, v_t = _timed(lambda: torch_lpips(xa, xb), max(args.reps // 4, 3))
    pair = dict(ms=ms_pair, ms_torch_tf32=ms_pair_t, speedup=ms_pair_t / ms_pair, value=float(v_ours),
                value_torch_tf32=float(v_t))
    del xa, xb
    torch.cuda.empty_cache()

    # ---- the tau sweep ----
    bench.W, bench.H = 1920, 1080
    arrays, cams = bench.build_workload("hier3m", device="cuda:0")
    from h3dgs import pipeline
    from h3dgs.evaluate import HierarchyEvaluator
    scene = pipeline.Scene(arrays, device="cuda:0", requires_grad=False)
    dcams = [pipeline.DeviceCamera(c, device="cuda:0") for c in cams]
    g = torch.Generator(device="cpu").manual_seed(5)
    gts = [torch.rand((3, 1080, 1920), generator=g).cuda() for _ in cams]
    plain = HierarchyEvaluator(scene, dcams, gts, TAUS)
    caps = {"row_capacity": next(iter(plain.renders.values())).P,
            "bin_capacity": next(iter(plain.renders.values())).bin_capacity,
            "sort_capacity": next(iter(plain.renders.values())).sort_capacity}
    with_lp = HierarchyEvaluator(scene, dcams, gts, TAUS, capacities=caps, lpips=net)
    kept = HierarchyEvaluator(scene, dcams, gts, TAUS, capacities=caps, keep_images=True)

    def sweep(ev):
        def run():
            ev.enqueue()
            return ev.finish()
        return run

    def dropin():
        res = sweep(kept)()
        vals = [[torch_lpips(res["images"][ti][ci], gts[ci].clamp(0, 1)) for ci in range(len(dcams))] for ti in range(len(TAUS))]
        return {t: float(torch.cat([v.reshape(1) for v in vals[ti]]).double().mean()) for ti, t in enumerate(TAUS)}

    forms = dict(plain=sweep(plain), lpips=sweep(with_lp), dropin=dropin)
    for _ in range(args.warmup):
        for fn in forms.values():
            fn()
    n = max(args.sweeps, 1)
    frames = len(dcams) * len(TAUS)
    ms_sweep, out = {}, {}
    for k, fn in forms.items():
        ms_sweep[k], out[k] = _timed(fn, n)
    clocks = sampler.stop()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:    # pragma: no cover
        q = f"unavailable: {e}"
    print(json.dumps({
        "metric": "LPIPS-VGG16 on sm_90a: per-layer TFLOP/s, one 1920x1080 pair, hier3m tau-sweep frames/s",
        "layers": layers, "conv_stack_ms": ms_conv, "conv_stack_ms_cudnn": ms_conv_t,
        "conv_stack_tflops": total_flop / ms_conv / 1e9, "conv_stack_tflops_cudnn": total_flop / ms_conv_t / 1e9,
        "pair_1080p": pair,
        "sweep": {"frames_per_sweep": frames, "feature_passes_per_camera": {"ours": len(TAUS) + 1, "dropin": 2 * len(TAUS)},
                  "frames_per_s_plain": frames / (ms_sweep["plain"] * 1e-3),
                  "frames_per_s_lpips": frames / (ms_sweep["lpips"] * 1e-3),
                  "frames_per_s_dropin_torch_lpips": frames / (ms_sweep["dropin"] * 1e-3),
                  "rerun_frames": out["lpips"]["rerun"],
                  "lpips_per_tau": out["lpips"]["lpips"], "lpips_per_tau_dropin": out["dropin"]},
        "gpu": q, "clocks": clocks}))


if __name__ == "__main__":
    main()

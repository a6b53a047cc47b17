#!/usr/bin/env python
"""Milliseconds per step of train_post's loop body (train_post.py:91-142: LOD cut, render_post with the image's exposure,
clamp, alpha mask, 0.8 L1 + 0.2 (1 - SSIM), backward; no optimizer) on bench.py's config #3 workload (3M-node hierarchy,
1920x1080, SH-3, tau = 6 px), one GPU, every view with its own exposure and binary mask.  Three forms, CUDA events
around whole runs of steps:

  dropin   pipeline.render_hier (the PyTorch gather / lerp of render_post, two host round trips), torch exposure matmul,
           clamp and mask product, and the reference's conv2d SSIM (tools/config4_train_post.conv_ssim);
  exact    pipeline.post_step: fused gather / lerp, h3dgs.loss.post_loss (exposure, clamp, mask and L1 + SSIM in one
           kernel forward and one backward);
  graphed  h3dgs.poststep.GraphedPostStep: one replay of graph A + graph B per step, status read back once per run;
           frames that overflow the capacities are re-run through the exact path inside the timed region.

It also times the loss alone at 1080p (CUDA events over 50 forward + backward calls): the two post-loss kernels against
torch's exposure / clamp / mask ops plus the fused L1 + SSIM pair they replace.

  python tools/bench_post_step.py [--steps 40] [--warmup 8]

Prints one JSON line with the GPU name and power limit read in the same run.  Writes nothing into the tree."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402  (workloads; puts the package on sys.path)

LAMBDA = 0.2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_post_step.py needs a CUDA device: there is no CPU fallback for this path")
    from config4_train_post import conv_ssim
    from diff_gaussian_rasterization import _C
    from h3dgs import pipeline
    from h3dgs.loss import fused_l1_ssim, post_loss
    from h3dgs.poststep import GraphedPostStep
    dev = "cuda:0"
    torch.cuda.set_device(0)
    W, H = bench.W, bench.H
    arrays, cams = bench.build_workload("hier3m", device=dev)
    scene = pipeline.Scene(arrays, device=dev)
    dcams = [pipeline.DeviceCamera(c, device=dev) for c in cams]
    thr = [pipeline.fov_threshold(bench.TAU, c) for c in cams]
    bg = torch.zeros(3, device=dev)
    rng = np.random.default_rng(5)
    exps, masks, gts = [], [], []
    for _ in cams:
        E = np.zeros((4, 4), np.float32)                 # pretrained_exposures hold 4x4 matrices; the top 3x4 block acts
        E[:3, :3] = np.eye(3) * 0.9 + rng.uniform(-0.1, 0.1, (3, 3))
        E[:3, 3] = rng.uniform(-0.05, 0.05, 3)
        E[3, 3] = 1.0
        M = torch.tensor((rng.uniform(size=(1, H, W)) > 0.1).astype(np.float32), device=dev)
        exps.append(torch.tensor(E, device=dev))
        masks.append(M)
        gts.append((torch.rand((3, H, W), device=dev) * M).contiguous())
    V = len(cams)

    def dropin(i):
        v = i % V
        scene.zero_grad()
        img = pipeline.render_hier(scene, dcams[v], bg, thr[v])[0]
        E = exps[v]
        img = torch.matmul(img.permute(1, 2, 0), E[:3, :3]).permute(2, 0, 1) + E[:3, 3, None, None]
        img = img.clamp(0, 1) * masks[v]
        loss = (1.0 - LAMBDA) * (img - gts[v]).abs().mean() + LAMBDA * (1.0 - conv_ssim(img, gts[v]))
        loss.backward()
        return loss

    def exact(i):
        v = i % V
        return pipeline.post_step(scene, dcams[v], bg, gts[v], thr[v], LAMBDA, exps[v], masks[v])[0][0]

    # capacities from one exact pass over the views (rows x 1.25, D x 1.5), as the evaluator learns them
    rows = D = 0
    for v in range(V):
        with torch.no_grad():
            n = pipeline.render_hier_fused(scene, dcams[v], bg, thr[v])[2]
        rows, D = max(rows, n + scene.skybox_points), max(D, _C.last_num_rendered())
    caps = dict(row_capacity=min(int(rows * 1.25) + 1, scene.means3D.shape[0]), bin_capacity=int(D * 1.5) + 1,
                sort_capacity=4096)
    gs = GraphedPostStep(scene, W, H, cams[0].tanfovx, cams[0].tanfovy, bg, thr[0], LAMBDA, exposure=True, mask=True,
                         capture=False, **caps)
    gs.set_camera(dcams[0])
    gs.gt.copy_(gts[0])
    gs.capture()
    status = torch.zeros((max(args.steps, args.warmup), 8), dtype=torch.float64, device=dev)
    side = torch.cuda.Stream()

    def graphed_run(n):
        """n steps; each target and mask uploaded on a side stream into the slot the step after next reads"""
        side.wait_stream(torch.cuda.current_stream())
        ready = gs.upload_target(gts[0], side, masks[0])
        for i in range(n):
            v = i % V
            gs.set_camera(dcams[v])
            gs.set_threshold(thr[v])
            gs.step(exposure=exps[v], gt_ready=ready)
            status[i].copy_(gs.status_dev)
            if i + 1 < n:
                ready = gs.upload_target(gts[(i + 1) % V], side, masks[(i + 1) % V])
        flagged = [i for i, s in enumerate(status[:n].cpu().numpy()) if s[6] or s[7]]
        for i in flagged:
            exact(i)
        return len(flagged)

    def timed(fn, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn(n)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n, out

    loop = lambda f: (lambda n: [f(i) for i in range(n)])
    for f in (loop(dropin), loop(exact), graphed_run):
        f(args.warmup)
    ms = {}
    for rep in range(2):                                 # alternated: two runs of each form
        for name, f in (("dropin", loop(dropin)), ("exact", loop(exact)), ("graphed", graphed_run)):
            t, out = timed(f, args.steps)
            ms.setdefault(name, []).append(t)
            if name == "graphed":
                rerun = out

    # the loss alone at 1080p: post-loss kernel pair vs torch exposure / clamp / mask + the fused L1 + SSIM pair
    x = torch.rand((3, H, W), device=dev) * 1.2 - 0.1
    E, M, gt = exps[0], masks[0], gts[0]

    def new_loss(n):
        for _ in range(n):
            xi = x.detach().requires_grad_(True)
            post_loss(xi, gt, LAMBDA, E, M)[0].backward()

    def old_loss(n):
        for _ in range(n):
            xi = x.detach().requires_grad_(True)
            a = (torch.matmul(xi.permute(1, 2, 0), E[:3, :3]).permute(2, 0, 1) + E[:3, 3, None, None]).clamp(0, 1) * M
            fused_l1_ssim(a, gt, LAMBDA)[0].backward()

    new_loss(10); old_loss(10)
    loss_ms = {"post_loss_kernels": timed(new_loss, 50)[0], "torch_ops_plus_l1_ssim": timed(old_loss, 50)[0]}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:    # pragma: no cover
        q = f"unavailable: {e}"
    best = {k: min(v) for k, v in ms.items()}
    print(json.dumps({
        "metric": f"train_post loop body ms/step (exposure, clamp, mask, 0.8 L1 + 0.2 (1 - SSIM), backward) @{W}x{H}",
        "workload": bench.WORKLOADS["hier3m"], "ms_per_step": best, "runs": ms, "steps_timed": args.steps,
        "speedup_graphed_vs_dropin": best["dropin"] / best["graphed"], "speedup_graphed_vs_exact": best["exact"] / best["graphed"],
        "graphed_rerun_frames": rerun, "capacities": caps, "loss_ms_per_fwd_bwd_1080p": loss_ms, "gpu": q}))


if __name__ == "__main__":
    main()

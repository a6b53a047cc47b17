#!/usr/bin/env python
"""Milliseconds per step of train_single's loop body (train_single.py:94-148: render() with the inverse depth and a
random background, the image's trained exposure, clamp, alpha mask, 0.8 L1 + 0.2 (1 - SSIM), the inverse-depth L1,
backward, densification statistics; no optimizer) on bench.py's config #2 workload (1M flat Gaussians, 1920x1080,
SH-3), one GPU, every view with its own exposure, binary mask, mono inverse depth and depth mask.  Three forms, CUDA
events around whole runs of steps:

  dropin   the drop-in rasterizer, torch exposure matmul, clamp, mask product, the reference's conv2d SSIM, torch depth
           term, autograd, and the indexed torch updates of the statistics;
  exact    pipeline.single_step: h3dgs.loss.single_loss and the statistics kernel;
  graphed  h3dgs.singlestep.GraphedSingleStep: one replay of graph A + graph B per step, status read back once per run;
           frames that overflow the capacities are re-run through the exact path inside the timed region.

It also times, at 1080p over 50 calls each: the loss side alone (the three kernels against torch ops + the fused L1 +
SSIM pair + torch depth term), the statistics kernel against the torch lines it replaces, and what constructing and
capturing a GraphedSingleStep costs (a new one is needed whenever the row count or the SH degree changes).

  python tools/bench_single_step.py [--steps 40] [--warmup 8]

Prints one JSON line with the GPU name and power limit read in the same run.  Writes nothing into the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

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
        raise SystemExit("bench_single_step.py needs a CUDA device: there is no CPU fallback for this path")
    from config4_train_post import conv_ssim
    from diff_gaussian_rasterization import _C
    from h3dgs import pipeline
    from h3dgs.loss import fused_l1_ssim, single_loss
    from h3dgs.singlestep import GraphedSingleStep
    dev = "cuda:0"
    torch.cuda.set_device(0)
    W, H = bench.W, bench.H
    arrays, cams = bench.build_workload("flat1m", device=dev)
    scene = pipeline.Scene(arrays, device=dev)
    N = scene.means3D.shape[0]
    dcams = [pipeline.DeviceCamera(c, device=dev) for c in cams]
    rng = np.random.default_rng(5)
    exps, masks, gts, monos, dmasks = [], [], [], [], []
    for _ in cams:
        E = np.eye(3, 4, dtype=np.float32) * 0.9
        E[:, :3] += rng.uniform(-0.1, 0.1, (3, 3))
        E[:, 3] = rng.uniform(-0.05, 0.05, 3)
        M = torch.tensor((rng.uniform(size=(1, H, W)) > 0.1).astype(np.float32), device=dev)
        exps.append(torch.tensor(E, device=dev, requires_grad=True))
        masks.append(M)
        gts.append((torch.rand((3, H, W), device=dev) * M).contiguous())
        monos.append(torch.rand((1, H, W), device=dev))
        dmasks.append((torch.rand((1, H, W), device=dev) > 0.2).float())
    V = len(cams)
    bgs = torch.rand((max(args.steps, args.warmup), 3), device=dev)          # train_single.py:60, drawn ahead
    weight = 0.5

    def torch_stats(st, radii, g):
        vis = (radii > 0).nonzero().flatten()
        st.max_radii2D[vis] = torch.max(st.max_radii2D[vis], radii[vis])
        st.xyz_gradient_accum[vis] = torch.max(torch.norm(g[vis, :2], dim=-1, keepdim=True), st.xyz_gradient_accum[vis])
        st.denom[vis] += 1

    stats_d, stats_e = pipeline.DensifyStats(N, dev), pipeline.DensifyStats(N, dev)

    def dropin(i):
        v = i % V
        scene.zero_grad()
        E = exps[v]
        E.grad = None
        m2d = torch.zeros_like(scene.means3D, requires_grad=True)
        img, radii, inv = pipeline.render_flat(scene, dcams[v], bgs[i], do_depth=True, means2D=m2d)
        img = torch.matmul(img.permute(1, 2, 0), E[:3, :3]).permute(2, 0, 1) + E[:3, 3, None, None]
        img = img.clamp(0, 1) * masks[v]
        loss = (1.0 - LAMBDA) * (img - gts[v]).abs().mean() + LAMBDA * (1.0 - conv_ssim(img, gts[v]))
        loss = loss + weight * torch.abs((inv - monos[v]) * dmasks[v]).mean()
        loss.backward()
        with torch.no_grad():
            torch_stats(stats_d, radii, m2d.grad)
        return loss

    def exact(i):
        v = i % V
        exps[v].grad = None
        return pipeline.single_step(scene, dcams[v], bgs[i], gts[v], LAMBDA, exps[v], masks[v], monos[v], dmasks[v], weight, stats_e)[0][0]

    # capacity from one exact pass over the views (D x 1.5)
    D = 0
    for v in range(V):
        with torch.no_grad():
            pipeline.render_flat(scene, dcams[v], bgs[0])
        D = max(D, _C.last_num_rendered())
    caps = dict(bin_capacity=int(D * 1.5) + 1, sort_capacity=4096)

    def construct():
        g = GraphedSingleStep(scene, W, H, cams[0].tanfovx, cams[0].tanfovy, LAMBDA, mask=True, capture=False, **caps)
        g.set_camera(dcams[0])
        g.set_depth_weight(weight)
        g.capture()
        return g

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gs = construct()
    torch.cuda.synchronize()
    first_ms = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    gs = construct()                                         # the library and torch are warm: what a rebuild costs in training
    torch.cuda.synchronize()
    rebuild_ms = (time.perf_counter() - t0) * 1e3
    status = torch.zeros((max(args.steps, args.warmup), 8), dtype=torch.float64, device=dev)
    side = torch.cuda.Stream()

    def graphed_run(n):
        side.wait_stream(torch.cuda.current_stream())
        ready = gs.upload_target(gts[0], side, masks[0], monos[0], dmasks[0])
        for i in range(n):
            v = i % V
            gs.set_camera(dcams[v])
            gs.set_background(bgs[i])
            gs.step(exposure=exps[v], gt_ready=ready)
            status[i].copy_(gs.status_dev)
            if i + 1 < n:
                u = (i + 1) % V
                ready = gs.upload_target(gts[u], side, masks[u], monos[u], dmasks[u])
        flagged = [i for i, s in enumerate(status[:n].cpu().numpy()) if s[7]]
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

    # the loss side alone at 1080p
    x = torch.rand((3, H, W), device=dev) * 1.2 - 0.1
    d = torch.rand((1, H, W), device=dev)
    E, M, gt, mono, dm = exps[0], masks[0], gts[0], monos[0], dmasks[0]

    def new_loss(n):
        for _ in range(n):
            E.grad = None
            xi, di = x.detach().requires_grad_(True), d.detach().requires_grad_(True)
            single_loss(xi, di, gt, LAMBDA, E, M, mono, dm, weight)[0].backward()

    def old_loss(n):
        for _ in range(n):
            E.grad = None
            xi, di = x.detach().requires_grad_(True), d.detach().requires_grad_(True)
            a = (torch.matmul(xi.permute(1, 2, 0), E[:3, :3]).permute(2, 0, 1) + E[:3, 3, None, None]).clamp(0, 1) * M
            (fused_l1_ssim(a, gt, LAMBDA)[0] + weight * torch.abs((di - mono) * dm).mean()).backward()

    new_loss(10); old_loss(10)
    loss_ms = {"single_loss_kernels": timed(new_loss, 50)[0], "torch_ops_plus_l1_ssim": timed(old_loss, 50)[0]}

    # the statistics alone: 1M rows, the visibility of view 0
    with torch.no_grad():
        radii = pipeline.render_flat(scene, dcams[0], bgs[0])[1]
    g2 = torch.randn((N, 3), device=dev) * 1e-3
    st = pipeline.DensifyStats(N, dev)
    k_fn = lambda n: [st.update(radii, g2) for _ in range(n)]
    t_fn = lambda n: [torch_stats(st, radii, g2) for _ in range(n)]
    k_fn(5); t_fn(5)
    stats_ms = {"densify_stats_kernel": timed(k_fn, 50)[0], "torch_lines": timed(t_fn, 50)[0]}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:    # pragma: no cover
        q = f"unavailable: {e}"
    best = {k: min(v) for k, v in ms.items()}
    print(json.dumps({
        "metric": f"train_single loop body ms/step (exposure with gradient, clamp, mask, 0.8 L1 + 0.2 (1 - SSIM), inverse-depth L1, "
                  f"backward, densification statistics) @{W}x{H}",
        "workload": bench.WORKLOADS["flat1m"], "ms_per_step": best, "runs": ms, "steps_timed": args.steps,
        "speedup_graphed_vs_dropin": best["dropin"] / best["graphed"], "speedup_graphed_vs_exact": best["exact"] / best["graphed"],
        "graphed_rerun_frames": rerun, "capacities": caps, "launches_per_graphed_step": gs.launches_per_step,
        "loss_ms_per_fwd_bwd_1080p": loss_ms, "stats_ms_1m_rows": stats_ms,
        "construct_and_capture_ms": {"first": first_ms, "rebuild": rebuild_ms}, "gpu": q}))


if __name__ == "__main__":
    main()

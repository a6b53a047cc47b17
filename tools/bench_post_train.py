#!/usr/bin/env python
"""Milliseconds per WHOLE iteration of train_post's loop body (train_post.py:69-192: the xyz lr, the LOD cut at the
threshold train_post.py:73-74 draws, render_post with the image's pretrained exposure, clamp, alpha mask, 0.8 L1 + 0.2
(1 - SSIM), backward, the skybox and anchor locks, torch.optim.Adam's dense step over every row) on bench.py's config #3
hierarchy (3M nodes, 1920x1080, SH-3) with a 20 000-row skybox tail and 3 000 anchors, one GPU, 8 views each with its
own exposure and binary mask.  Three forms, CUDA events around whole runs of iterations:

  caller    GraphedPostStep without a state, then the caller's side in torch: the activations' backward by autograd
            through abs / exp / normalize / cat, the lock lines, torch.optim.Adam over the six groups and the
            re-activation into the rendered tensors;
  exact     pipeline.post_step(state=): the same kernels eagerly, parameter step included;
  graphed   GraphedPostStep(state=): one replay of graph A + graph B per iteration and its 64-byte status read, a frame
            that overflowed the capacities re-run through the exact path before the next iteration, inside the timed
            region.

It also times the parameter step alone (csrc/post_param.cu's launches, replayed 20 times from one CUDA graph) with its
achieved GB/s from the algorithmic bytes: each of a row's 59 stored floats reads its value, two moments and its
activated gradient and writes its value, two moments and its activated value (32 bytes); the three scalings also read
their activated value (12 bytes); the lock mask is one byte per row: 1 901 bytes per SH-3 row.

  python tools/bench_post_train.py [--iters 24] [--warmup 8]

Prints one JSON line with the GPU's name and power limit read in the same run.  Writes nothing into the tree."""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402  (workloads; puts the package on sys.path)

LAMBDA, SKY, ANCHORS = 0.2, 20_000, 3_000
LRS = [1.6e-4, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]             # arguments/__init__.py (spatial_lr_scale 1)


def gpu_conditions():
    import torch
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    f = [x.strip() for x in r.stdout.strip().split(",")] if r.returncode == 0 else [None, None]
    return {"gpu": torch.cuda.get_device_name(0), "power_limit": f[1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_post_train.py needs a CUDA device: there is no CPU fallback for this path")
    import torch.nn.functional as Fn
    from diff_gaussian_rasterization import _C
    from h3dgs import _lib, pipeline, synth
    from h3dgs.poststep import GraphedPostStep, PostState
    dev = "cuda:0"
    torch.cuda.set_device(0)
    W, H = bench.W, bench.H
    arrays, cams = bench.build_workload("hier3m")
    arrays = synth.append_skybox(arrays, SKY)
    V = len(cams)
    t = lambda a: torch.as_tensor(np.asarray(a, np.float32), device=dev)
    shs = t(arrays["shs"])
    params = [t(arrays["means3D"]), shs[:, :1].contiguous(), shs[:, 1:].contiguous(), t(arrays["opacities"]).reshape(-1, 1),
              torch.log(t(arrays["scales"])), t(arrays["rotations"])]
    N = params[0].shape[0]
    nodes, boxes = torch.as_tensor(arrays["nodes"], device=dev), torch.as_tensor(arrays["boxes"], device=dev)
    rng = np.random.default_rng(5)
    anchors = torch.tensor(rng.choice(N, ANCHORS, replace=False), dtype=torch.int64, device=dev)
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
    dcams = [pipeline.DeviceCamera(c, device=dev) for c in cams]
    n_it = max(args.iters, args.warmup)
    # train_post.py:73-74: limit = 2^(u (log2 0.1 - log2 0.005) + log2 0.005), the cut's threshold
    us = np.random.default_rng(11).uniform(size=n_it)
    thr = [2.0 ** (u * (math.log2(0.1) - math.log2(0.005)) + math.log2(0.005)) for u in us]
    lr_of = lambda i: LRS[0] * 0.999 ** i
    bg = torch.zeros(3, device=dev)
    new_state = lambda: PostState(params, SKY, LRS, nodes, boxes, skybox_locked=True, anchors=anchors)

    # capacities from one exact pass over the iterations' (view, threshold) pairs (rows x 1.25, D x 1.5)
    probe = new_state().make_scene(requires_grad=False)
    rows = D = 0
    for i in range(n_it):
        with torch.no_grad():
            n = pipeline.render_hier_fused(probe, dcams[i % V], bg, thr[i])[2]
        rows, D = max(rows, n + SKY), max(D, _C.last_num_rendered())
    caps = dict(row_capacity=min(int(rows * 1.25) + 1, N), bin_capacity=int(D * 1.5) + 1, sort_capacity=4096)
    del probe

    # ---- caller: the graphed objective, then the optimizer in torch ---------------------------------------------------
    attrs = [torch.nn.Parameter(p.clone()) for p in params]
    opt = torch.optim.Adam([{"params": [p], "lr": lr} for p, lr in zip(attrs, LRS)], lr=0.0, eps=1e-15)
    with torch.no_grad():
        cs = pipeline.Scene(dict(means3D=attrs[0].detach().clone(), shs=torch.cat((attrs[1], attrs[2]), 1),
                                 opacities=torch.abs(attrs[3]), scales=torch.exp(attrs[4]), rotations=Fn.normalize(attrs[5]),
                                 skybox_points=SKY, nodes=nodes, boxes=boxes), device=dev, requires_grad=False)
    g_plain = GraphedPostStep(cs, W, H, cams[0].tanfovx, cams[0].tanfovy, bg, thr[0], LAMBDA, exposure=True, mask=True,
                              capture=False, **caps)
    g_plain.set_camera(dcams[0])
    g_plain.capture()

    def caller(i):
        v = i % V
        opt.param_groups[0]["lr"] = lr_of(i)
        g_plain.set_camera(dcams[v])
        g_plain.set_threshold(thr[i])
        g_plain.step(gt=gts[v], mask=masks[v], exposure=exps[v])
        gr = g_plain.grads
        with torch.enable_grad():
            act = [attrs[0] * 1.0, torch.cat((attrs[1], attrs[2]), 1), torch.abs(attrs[3]), torch.exp(attrs[4]),
                   Fn.normalize(attrs[5])]
            torch.autograd.backward(act, [gr["means3D"], gr["shs"], gr["opacities"], gr["scales"], gr["rotations"]])
        with torch.no_grad():
            for p in attrs:
                p.grad[-SKY:] = 0
                p.grad[anchors] = 0
            opt.step()
            opt.zero_grad(set_to_none=True)
            cs.means3D.copy_(attrs[0]); cs.shs.copy_(torch.cat((attrs[1], attrs[2]), 1))
            cs.opacities.copy_(torch.abs(attrs[3])); cs.scales.copy_(torch.exp(attrs[4]))
            cs.rotations.copy_(Fn.normalize(attrs[5]))

    # ---- exact and graphed with a state ------------------------------------------------------------------------------
    se = new_state()
    sce = se.make_scene()

    def exact_on(state, scene, i):
        v = i % V
        state.set_learning_rate(lr_of(i))
        return pipeline.post_step(scene, dcams[v], bg, gts[v], thr[i], LAMBDA, exps[v], masks[v], state=state)

    sg = new_state()
    scg = sg.make_scene(requires_grad=False)
    gs = GraphedPostStep(scg, W, H, cams[0].tanfovx, cams[0].tanfovy, bg, thr[0], LAMBDA, exposure=True, mask=True,
                         capture=False, state=sg, **caps)
    gs.set_camera(dcams[0])
    gs.capture()
    side = torch.cuda.Stream()

    def graphed(n):
        """INTEGRATION.md's loop: the status read every iteration, an overflowed frame re-run exactly before the next"""
        side.wait_stream(torch.cuda.current_stream())
        ready = gs.upload_target(gts[0], side, masks[0])
        reruns = 0
        for i in range(n):
            v = i % V
            sg.set_learning_rate(lr_of(i))
            gs.set_camera(dcams[v])
            gs.set_threshold(thr[i])
            gs.step(exposure=exps[v], gt_ready=ready)
            if i + 1 < n:
                u = (i + 1) % V
                ready = gs.upload_target(gts[u], side, masks[u])
            if gs.status()["overflow"]:
                reruns += 1
                exact = sg.make_scene()
                exact_on(sg, exact, i)
                sg.activate(scg)
        return reruns

    def timed(fn, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn(n)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n, out

    loop = lambda f: (lambda n: [f(i) for i in range(n)])
    forms = [("caller", loop(caller)), ("exact", loop(lambda i: exact_on(se, sce, i))), ("graphed", graphed)]
    ms, errors, reruns = {}, {}, []
    for name, f in forms:
        try:
            f(args.warmup)
        except Exception as e:                                # a form that cannot run is reported, not timed
            errors[name] = repr(e)[:200]
    for rep in range(2):                                      # alternated: two runs of each form
        for name, f in forms:
            if name in errors:
                continue
            t_ms, out = timed(f, args.iters)
            ms.setdefault(name, []).append(t_ms)
            if name == "graphed":
                reruns.append(out)

    # the parameter step alone, 20 replays of its launches in one graph (exact mode: no overflow gate)
    import ctypes as C
    pa = sg._post_args(scg, gs.grads)
    L = _lib.lib()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _lib.check(L.h3dgs_post_param_step(C.byref(pa), _lib.POST_STEP, s.cuda_stream))
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(20):
            _lib.check(L.h3dgs_post_param_step(C.byref(pa), _lib.POST_STEP, torch.cuda.current_stream().cuda_stream))
    graph.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    param_ms = e0.elapsed_time(e1) / 100
    floats = 3 + 3 + 45 + 1 + 3 + 4
    row_bytes = floats * 32 + 3 * 4 + 1
    gbs = N * row_bytes / (param_ms * 1e-3) / 1e9

    out = dict(workload="hier3m+skybox", W=W, H=H, N=N, skybox=SKY, anchors=ANCHORS, views=V, iters=args.iters,
               row_capacity=caps["row_capacity"], bin_capacity=caps["bin_capacity"],
               ms_per_iteration={k: (round(min(v), 3) if v else "not measured") for k, v in
                                 (("caller", ms.get("caller")), ("exact", ms.get("exact")), ("graphed", ms.get("graphed")))},
               runs=ms, errors=errors, graphed_overflow_reruns=reruns, param_step_ms=round(param_ms, 4),
               param_step_bytes=N * row_bytes, param_step_gbs=round(gbs, 1), **gpu_conditions())
    print(json.dumps(out))


if __name__ == "__main__":
    main()

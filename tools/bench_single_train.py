#!/usr/bin/env python
"""Milliseconds per WHOLE iteration of train_single's loop body (train_single.py:85-186 between densifications: the
lrs, render() with the inverse depth, the image's trained exposure, clamp, alpha mask, 0.8 L1 + 0.2 (1 - SSIM), the
inverse-depth L1, backward, densification statistics, torch.optim.Adam on the exposures, the skybox lock, OurAdam on
the flattened index, the big-Gaussian rescale) on bench.py's config #2 workload (1M flat Gaussians, 1920x1080, SH-3),
one GPU, 8 views each with its own exposure, binary mask, mono inverse depth and depth mask.  Three forms, CUDA events
around whole runs of iterations:

  caller    GraphedSingleStep without a state, then the caller's side in torch as INTEGRATION.md described it before
            the state existed: the activations' backward by autograd, the lock lines, (grad != 0).nonzero() (a host
            sync), h3dgs.optim.Adam over the six groups, torch.optim.Adam on the exposures, the rescale lines and the
            re-activation into the rendered tensors;
  exact     pipeline.single_step(state=): the same kernels eagerly, parameter step included;
  graphed   GraphedSingleStep(state=): one replay of graph A + graph B per iteration and its 64-byte status read (the
            one host sync left), a frame that overflowed the capacities re-run through the exact path before the next
            iteration, inside the timed region.

It also times the parameter step alone (csrc/single_param.cu's launches, replayed 20 times from one CUDA graph) with
its achieved GB/s from the algorithmic bytes: every row reads its opacity gradient and activated opacity and its
stored scaling (5 floats); a relevant row also reads its 59 stored floats, 118 moments and 59 activated gradients and
writes 59 stored floats, 118 moments and 59 activated floats (472 more).

  python tools/bench_single_train.py [--iters 24] [--warmup 8]

Prints one JSON line with the GPU's name and power limit read in the same run.  Writes nothing into the tree."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402  (workloads; puts the package on sys.path)

LAMBDA, WEIGHT, EXTENT, SKY = 0.2, 0.5, 40.0, 20_000
LRS = [1.6e-4 * 40.0, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]      # arguments/__init__.py, xyz scaled by the extent


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
        raise SystemExit("bench_single_train.py needs a CUDA device: there is no CPU fallback for this path")
    from diff_gaussian_rasterization import _C
    from h3dgs import _lib, pipeline
    from h3dgs.optim import Adam
    from h3dgs.singlestep import GraphedSingleStep, SingleState
    dev = "cuda:0"
    torch.cuda.set_device(0)
    W, H = bench.W, bench.H
    arrays, cams = bench.build_workload("flat1m", device=dev)
    V = len(cams)
    t = lambda a: torch.as_tensor(np.asarray(a, np.float32), device=dev)
    shs = t(arrays["shs"])
    op = t(arrays["opacities"]).reshape(-1, 1).clamp(1e-4, 1 - 1e-4)
    params = [t(arrays["means3D"]), shs[:, :1].contiguous(), shs[:, 1:].contiguous(), torch.log(op / (1 - op)),
              torch.log(t(arrays["scales"])), t(arrays["rotations"])]
    N = params[0].shape[0]
    rng = np.random.default_rng(5)
    exposure = torch.tensor(np.stack([np.eye(3, 4) * 0.9 + np.pad(rng.uniform(-0.1, 0.1, (3, 3)), ((0, 0), (0, 1)))
                                      for _ in range(V)]).astype(np.float32), device=dev)
    masks, gts, monos, dmasks = [], [], [], []
    for _ in cams:
        M = torch.tensor((rng.uniform(size=(1, H, W)) > 0.1).astype(np.float32), device=dev)
        masks.append(M)
        gts.append((torch.rand((3, H, W), device=dev) * M).contiguous())
        monos.append(torch.rand((1, H, W), device=dev))
        dmasks.append((torch.rand((1, H, W), device=dev) > 0.2).float())
    dcams = [pipeline.DeviceCamera(c, device=dev) for c in cams]
    n_it = max(args.iters, args.warmup)
    bgs = torch.rand((n_it, 3), device=dev)
    lr_of = lambda i: (LRS[0] * 0.999 ** i, 1e-3 * 0.999 ** i)
    new_state = lambda: SingleState(params, SKY, LRS, exposure, skybox_locked=True, scaffold_points=SKY)

    D = 0
    probe = new_state().make_scene(requires_grad=False)
    for v in range(V):
        with torch.no_grad():
            pipeline.render_flat(probe, dcams[v], bgs[0])
        D = max(D, _C.last_num_rendered())
    caps = dict(bin_capacity=int(D * 1.5) + 1, sort_capacity=4096)
    del probe

    # ---- caller: the graphed objective, then the optimizers in torch ---------------------------------------------------
    attrs = [torch.nn.Parameter(p.clone()) for p in params]
    ex_param = torch.nn.Parameter(exposure.clone())
    opt = Adam([{"params": [p], "lr": lr} for p, lr in zip(attrs, LRS)], lr=0.0, eps=1e-15)
    ex_opt = torch.optim.Adam([ex_param])
    with torch.no_grad():
        cs = pipeline.Scene(dict(means3D=attrs[0].detach().clone(), shs=torch.cat((attrs[1], attrs[2]), 1), opacities=torch.sigmoid(attrs[3]),
                                 scales=torch.exp(attrs[4]), rotations=torch.nn.functional.normalize(attrs[5]),
                                 skybox_points=SKY), device=dev, requires_grad=False)
    g_plain = GraphedSingleStep(cs, W, H, cams[0].tanfovx, cams[0].tanfovy, LAMBDA, mask=True, capture=False, **caps)
    g_plain.set_depth_weight(WEIGHT)
    g_plain.set_camera(dcams[0])
    g_plain.capture()

    def caller(i):
        v = i % V
        xyz_lr, ex_lr = lr_of(i)
        opt.param_groups[0]["lr"] = xyz_lr
        ex_opt.param_groups[0]["lr"] = ex_lr
        g_plain.set_camera(dcams[v])
        g_plain.step(gt=gts[v], mask=masks[v], mono_invdepth=monos[v], depth_mask=dmasks[v], exposure=ex_param[v],
                     bg=bgs[i])
        gr = g_plain.grads
        with torch.enable_grad():
            act = [attrs[0] * 1.0, torch.cat((attrs[1], attrs[2]), 1), torch.sigmoid(attrs[3]), torch.exp(attrs[4]),
                   torch.nn.functional.normalize(attrs[5])]
            torch.autograd.backward(act, [gr["means3D"], gr["shs"], gr["opacities"], gr["scales"], gr["rotations"]])
        with torch.no_grad():
            ex_param.grad = torch.zeros_like(ex_param)
            ex_param.grad[v] = g_plain.exposure_grad
            ex_opt.step()
            ex_opt.zero_grad(set_to_none=True)
            for p in attrs:
                p.grad[:SKY] = 0
            relevant = (attrs[3].grad.flatten() != 0).nonzero().flatten()
            opt.step(relevant)
            opt.zero_grad(set_to_none=True)
            vals, _ = torch.exp(attrs[4]).max(dim=1)
            viol = vals > EXTENT * 0.02
            viol[:SKY] = False
            attrs[4][viol] = torch.log(torch.exp(attrs[4])[viol] * 0.8)
            cs.means3D.copy_(attrs[0]); cs.shs.copy_(torch.cat((attrs[1], attrs[2]), 1))
            cs.opacities.copy_(torch.sigmoid(attrs[3])); cs.scales.copy_(torch.exp(attrs[4]))
            cs.rotations.copy_(torch.nn.functional.normalize(attrs[5]))

    # ---- exact and graphed with a state ------------------------------------------------------------------------------
    se = new_state()
    sce = se.make_scene()

    def exact_on(state, scene, i):
        v = i % V
        state.set_learning_rates(*lr_of(i))
        state.set_image(v)
        return pipeline.single_step(scene, dcams[v], bgs[i], gts[v], LAMBDA, None, masks[v], monos[v], dmasks[v], WEIGHT,
                                    state.stats, state=state, cameras_extent=EXTENT)

    sg = new_state()
    scg = sg.make_scene(requires_grad=False)
    gs = GraphedSingleStep(scg, W, H, cams[0].tanfovx, cams[0].tanfovy, LAMBDA, mask=True, capture=False, state=sg,
                           cameras_extent=EXTENT, **caps)
    gs.set_depth_weight(WEIGHT)
    gs.set_camera(dcams[0])
    gs.capture()
    side = torch.cuda.Stream()

    def graphed(n):
        """INTEGRATION.md's loop: the status read every iteration, an overflowed frame re-run exactly before the next"""
        side.wait_stream(torch.cuda.current_stream())
        ready = gs.upload_target(gts[0], side, masks[0], monos[0], dmasks[0])
        reruns = 0
        for i in range(n):
            v = i % V
            sg.set_learning_rates(*lr_of(i))
            gs.set_camera(dcams[v])
            gs.set_background(bgs[i])
            gs.step(gt_ready=ready, image=v)
            if i + 1 < n:
                u = (i + 1) % V
                ready = gs.upload_target(gts[u], side, masks[u], monos[u], dmasks[u])
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

    # the parameter step alone, 20 replays of its launches in one graph
    import ctypes as C
    sa = sg._single_args(scg, EXTENT, gs.grads, gs.exposure_grad)
    L = _lib.lib()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _lib.check(L.h3dgs_single_param_step(C.byref(sa), _lib.SINGLE_STEP, s.cuda_stream))
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(20):
            _lib.check(L.h3dgs_single_param_step(C.byref(sa), _lib.SINGLE_STEP, torch.cuda.current_stream().cuda_stream))
    graph.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    param_ms = e0.elapsed_time(e1) / 100
    g_op = gs.grads["opacities"].flatten() * (1 - scg.opacities.flatten()) * scg.opacities.flatten()
    R = int((g_op != 0).sum())
    R = R if R else N
    gbs = (N * 5 + R * 472) * 4 / (param_ms * 1e-3) / 1e9

    out = dict(workload="flat1m", W=W, H=H, N=N, views=V, iters=args.iters,
               ms_per_iteration={k: (round(min(v), 3) if k in ms else "not measured") for k, v in
                                 (("caller", ms.get("caller")), ("exact", ms.get("exact")), ("graphed", ms.get("graphed")))},
               runs=ms, errors=errors, graphed_overflow_reruns=reruns, param_step_ms=round(param_ms, 4),
               param_step_relevant_rows=R, param_step_gbs=round(gbs, 1), **gpu_conditions())
    print(json.dumps(out))


if __name__ == "__main__":
    main()

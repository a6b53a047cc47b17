#!/usr/bin/env python
"""Milliseconds per iteration of train_coarse's loop body (train_coarse.py:97-145: render_coarse with a random
background, alpha mask, 0.8 L1 + 0.2 (1 - SSIM), backward, max_radii2D, the skybox scaling lock, OurAdam on
(_opacity.grad != 0).nonzero() with the xyz lr at 0, the big-Gaussian rescale) on a scaffold-sized cloud: 2M SfM-like
points after 100 000 skybox rows (tools/bench_knn.py's coarse2m), laid out as create_from_pcd does (scales from
distCUDA2, identity rotations, opacity 0.02 and 0.7 on the skybox), SH degree 1, 1920x1080, 8 views.  Four forms, CUDA
events around whole runs of iterations:

  ref_debug   the reference flow on the drop-in packages: torch activations, GaussianRasterizer with debug=True as
              render_coarse hard-wires it, the reference-form conv2d SSIM, autograd, the indexed max_radii2D update,
              OurAdam's gather / update / scatter with the unflattened index, the rescale lines;
  ref         the same with debug=False;
  exact       pipeline.coarse_step (the coarse-loss kernels and csrc/coarse_param.cu, eagerly);
  graphed     h3dgs.coarsestep.GraphedCoarseStep, one replay of graph A + graph B per iteration, the status read back
              every iteration (a host synchronisation) to re-run an overflowed frame through the exact path inside the
              timed region.

It also times the parameter step's three launches alone, replayed 20 times from one CUDA graph (no host work between
them), and reports its achieved GB/s from the algorithmic bytes of the
shapes: every row reads its opacity gradient, activated opacity and stored scaling (5 floats); a relevant row also
reads its 23 stored floats, 46 moments and 23 activated gradients and writes 23 stored floats, 46 moments and 23
activated floats (181 more).

  python tools/bench_coarse_step.py [--iters 16] [--warmup 8]

Prints one JSON line with the GPU's name, power limit and SM clock read in the same run.  Writes nothing into the tree."""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "hierarchical-3d-gaussians_b200"))

W, H, VIEWS, SKY, LAMBDA, EXTENT = 1920, 1080, 8, 100_000, 0.2, 60.0
LRS = [0.0, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]          # arguments/__init__.py, xyz forced to 0 (:55-57)


def gpu_conditions():
    import torch
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    f = [x.strip() for x in r.stdout.strip().split(",")] if r.returncode == 0 else [None, None, None]
    return {"gpu": torch.cuda.get_device_name(0), "power_limit": f[1], "sm_clock": f[2]}


def scaffold(dev):
    """create_from_pcd's stored tensors for the coarse2m cloud (scene/gaussian_model.py:146-210)"""
    import numpy as np
    import torch
    from bench_knn import CLOUDS
    from simple_knn._C import distCUDA2
    xyz = torch.tensor(CLOUDS["coarse2m"](), device=dev)
    N = xyz.shape[0]
    rs = np.random.default_rng(4)
    color = torch.tensor(rs.uniform(0, 1, (N, 3)).astype(np.float32), device=dev)
    color[:SKY] = torch.tensor([0.7, 0.8, 0.95], device=dev)
    dc = ((color - 0.5) / 0.28209479177387814)[:, None, :].contiguous()
    rest = torch.zeros((N, 3, 3), device=dev)
    dist2 = torch.clamp_min(distCUDA2(xyz), 1e-7)
    dist2[:SKY] *= 10
    dist2[SKY:] = torch.clamp_max(dist2[SKY:], 10)
    scales = torch.log(torch.sqrt(dist2))[..., None].repeat(1, 3)
    rots = torch.zeros((N, 4), device=dev)
    rots[:, 0] = 1
    p = torch.full((N, 1), 0.02, device=dev)
    op = torch.log(p / (1 - p))
    op[:SKY] = 0.7
    return [xyz, dc, rest, op, scales, rots]


def cameras(dev):
    """8 views from the middle of the cloud, 45 degrees apart, far plane past the skybox sphere"""
    from h3dgs import pipeline, synth
    return [pipeline.DeviceCamera(synth.yaw_camera(W, H, 45.0 * k, (0.0, 0.0, 0.0), zfar=5000.0), device=dev)
            for k in range(VIEWS)]


def timed(fn, iters, warmup):
    import torch
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(iters):
        fn(i)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=16)
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_coarse_step.py needs a CUDA device: there is no CPU fallback for this path")
    from config4_train_post import conv_ssim
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    from h3dgs import pipeline
    from h3dgs.coarsestep import CoarseState, GraphedCoarseStep
    dev = "cuda:0"
    torch.cuda.set_device(0)
    stored = scaffold(dev)
    N = stored[0].shape[0]
    cams = cameras(dev)
    g = torch.Generator(device=dev).manual_seed(9)
    gts = [torch.rand((3, H, W), device=dev, generator=g) for _ in range(VIEWS)]
    masks = [(torch.rand((1, H, W), device=dev, generator=g) > 0.05).float() for _ in range(VIEWS)]
    bgs = [torch.rand(3, device=dev, generator=g) for _ in range(VIEWS)]
    out = {"workload": f"coarse2m scaffold: N={N} ({SKY} skybox rows first), {W}x{H}, SH degree 1, {VIEWS} views, binary mask"}
    out.update(gpu_conditions())

    # ---- the reference flow on the packages -----------------------------------------------------------------------
    params = [torch.nn.Parameter(t.clone()) for t in stored]
    moments = [[torch.zeros_like(t), torch.zeros_like(t)] for t in stored]
    steps = [0] * 6
    max_radii = torch.zeros(N, device=dev)
    thr = EXTENT * 0.1

    def our_adam(relevant):
        """scene/OurAdam.py:_single_tensor_adam, non-capturable, with train_coarse's unflattened index"""
        for i, p in enumerate(params):
            steps[i] += 1
            if relevant.shape[0] == 0:
                continue
            grad, ea, es, prm = p.grad[relevant], moments[i][0][relevant], moments[i][1][relevant], p.data[relevant]
            ea.mul_(0.9).add_(grad, alpha=0.1)
            es.mul_(0.999).addcmul_(grad, grad, value=0.001)
            bc1, bc2 = 1 - 0.9 ** steps[i], 1 - 0.999 ** steps[i]
            denom = (es.sqrt() / math.sqrt(bc2)).add_(1e-15)
            prm.addcdiv_(ea, denom, value=-LRS[i] / bc1)
            moments[i][0][relevant], moments[i][1][relevant], p.data[relevant] = ea, es, prm

    def ref_iter(k, debug):
        cam = cams[k % VIEWS]
        xyz, dc, rest, op, sc, rot = params
        ss = torch.zeros_like(xyz, requires_grad=True) + 0
        e = torch.empty(0, device=dev)
        ei = e.int()
        rs = GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
                                           bg=bgs[k % VIEWS], scale_modifier=1.0, viewmatrix=cam.viewmatrix,
                                           projmatrix=cam.projmatrix, sh_degree=1, campos=cam.campos, prefiltered=False,
                                           debug=debug, do_depth=False, render_indices=ei, parent_indices=ei,
                                           interpolation_weights=e, num_node_kids=ei)
        img, radii, _ = GaussianRasterizer(rs)(means3D=xyz, means2D=ss, shs=torch.cat((dc, rest), 1), colors_precomp=None,
                                               opacities=torch.sigmoid(op), scales=torch.exp(sc),
                                               rotations=torch.nn.functional.normalize(rot), cov3D_precomp=None)
        a = img * masks[k % VIEWS]
        loss = (1.0 - LAMBDA) * torch.abs(a - gts[k % VIEWS]).mean() + LAMBDA * (1.0 - conv_ssim(a, gts[k % VIEWS]))
        loss.backward()
        vis = radii > 0
        max_radii[vis] = torch.max(max_radii[vis], radii[vis].float())
        with torch.no_grad():
            sc.grad[:SKY, :] = 0
            our_adam((op.grad != 0).nonzero())
            for p in params:
                p.grad = None
            vals, _ = torch.exp(sc).max(dim=1)
            viol = vals > thr
            viol[:SKY] = False
            sc[viol] = torch.log(torch.exp(sc[viol]) * 0.8)

    out["ref_debug_ms"] = timed(lambda k: ref_iter(k, True), args.iters, args.warmup)
    out["ref_ms"] = timed(lambda k: ref_iter(k, False), args.iters, args.warmup)
    del params, moments

    # ---- exact and graphed -------------------------------------------------------------------------------------------
    st = CoarseState(stored, SKY, LRS, eps=1e-15)
    scene = st.make_scene()
    out["exact_ms"] = timed(lambda k: pipeline.coarse_step(st, scene, cams[k % VIEWS], bgs[k % VIEWS], gts[k % VIEWS], EXTENT,
                                                           LAMBDA, masks[k % VIEWS], sh_degree=1), args.iters, args.warmup)
    sg = CoarseState(stored, SKY, LRS, eps=1e-15)
    sceneg = sg.make_scene(requires_grad=False)
    gs = GraphedCoarseStep(sg, sceneg, W, H, cams[0].tanfovx, cams[0].tanfovy, EXTENT, LAMBDA, mask=True, sh_degree=1,
                           bin_capacity=1 << 25, sort_capacity=8192, capture=False)
    gs.set_camera(cams[0])
    gs.capture()
    reruns = [0]
    side = torch.cuda.Stream()

    def graphed(k):
        ev = gs.upload_target(gts[k % VIEWS], side, masks[k % VIEWS])
        gs.step(cam=cams[k % VIEWS], bg=bgs[k % VIEWS], gt_ready=ev)
        if gs.status()["overflow"]:
            reruns[0] += 1
            sceneg.means3D.requires_grad_(True); sceneg.shs.requires_grad_(True); sceneg.opacities.requires_grad_(True)
            sceneg.scales.requires_grad_(True); sceneg.rotations.requires_grad_(True)
            pipeline.coarse_step(sg, sceneg, cams[k % VIEWS], bgs[k % VIEWS], gts[k % VIEWS], EXTENT, LAMBDA,
                                 masks[k % VIEWS], sh_degree=1)
            for t in (sceneg.means3D, sceneg.shs, sceneg.opacities, sceneg.scales, sceneg.rotations):
                t.requires_grad_(False)
                t.grad = None

    out["graphed_ms"] = timed(graphed, args.iters, args.warmup)
    out["graphed_overflow_reruns"] = reruns[0]
    out["graphed_status"] = gs.status()

    # ---- the parameter kernel alone ------------------------------------------------------------------------------
    grads = gs.grads
    R = int((((grads["opacities"] * (1 - sceneg.opacities)) * sceneg.opacities) != 0).sum())
    import ctypes as C
    from h3dgs import _lib
    cargs = sg._args(sceneg, EXTENT, grads)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _lib.check(_lib.lib().h3dgs_coarse_param_step(C.byref(cargs), _lib.COARSE_STEP, s.cuda_stream))
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(20):
            _lib.check(_lib.lib().h3dgs_coarse_param_step(C.byref(cargs), _lib.COARSE_STEP,
                                                         torch.cuda.current_stream().cuda_stream))
    kernel_ms = timed(lambda k: graph.replay(), 5, 2) / 20
    nbytes = 4 * (5 * N + 181 * R)
    out.update(param_kernel_ms=kernel_ms, param_kernel_relevant_rows=R, param_kernel_bytes=nbytes,
               param_kernel_GBps=nbytes / (kernel_ms * 1e-3) / 1e9)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

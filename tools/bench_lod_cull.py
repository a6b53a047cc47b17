#!/usr/bin/env python
"""The view cull of the LOD cut (csrc/lod_cull.cu) on bench.py's hier3m workload (config #3: 3 M nodes, 1920x1080) and on
a surround scene (1 M leaves on every side of the camera, built with the device creator), one GPU, per view:

  rows     the cut's rows at tau 6, the culled cut's rows, and V (rows K1 draws); culled / V shows how tight the bound is;
  passes   device time of the mask pass, of the cut with and without a mask, and of the budget with and without;
  frames   GraphedRender frame time at tau 6 and GraphedPostStep step time, cull off and on, the arms alternated;
  budget   at a fixed B: the chosen threshold, the rows drawn and the PSNR against the tau 0 frame, with and without cull.

  python tools/bench_lod_cull.py [--reps 30] [--budget 400000] [--rounds 3]

Prints one JSON line with the GPU name and power limit.  Writes nothing into the tree."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (workloads; puts the package on sys.path)


def surround(device, P=1_000_000, radius=60.0, seed=3):
    """leaves in a shell 1 .. radius units around the origin, every direction, sqrt-of-distance sizes as hier3m's"""
    import torch
    from h3dgs.hier_build import build_hierarchy
    g = torch.Generator(device=device).manual_seed(seed)
    d = torch.randn(P, 3, device=device, generator=g)
    d = d / d.norm(dim=1, keepdim=True)
    r = 1.0 + (radius - 1.0) * torch.rand(P, 1, device=device, generator=g)
    xyz = d * r
    log_s = (torch.log(2.4e-3 * torch.sqrt(2.0 * r)) + 0.5 * torch.randn(P, 3, device=device, generator=g))
    q = torch.randn(P, 4, device=device, generator=g)
    hb = build_hierarchy(xyz, 0.3 * torch.randn(P, 16, 3, device=device, generator=g),
                         0.05 + 0.9 * torch.rand(P, device=device, generator=g), log_s, q / q.norm(dim=1, keepdim=True))
    return dict(means3D=hb["xyz"], scales=hb["log_scales"].exp(), rotations=hb["rotations"], opacities=hb["opacities"],
                shs=hb["shs"], nodes=hb["nodes"], boxes=hb["boxes"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--budget", type=int, default=400_000)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_lod_cull.py needs a CUDA device: there is no CPU fallback for this path")
    dev = "cuda:0"
    torch.cuda.set_device(0)
    from h3dgs import _lib, pipeline, synth
    from h3dgs.evaluate import GraphedRender
    from h3dgs.poststep import GraphedPostStep
    L = _lib.lib()
    stream = torch.cuda.current_stream().cuda_stream

    def device_ms(fn, reps=args.reps):
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    arrays3m, cams = bench.build_workload("hier3m", device=dev)
    W, H = cams[0].W, cams[0].H
    surround_cams = [synth.make_camera(W, H), synth.yaw_camera(W, H, 90.0, [0.0, 0.0, 0.0]),
                     synth.yaw_camera(W, H, 200.0, [5.0, 1.0, 10.0])]
    out = {}
    for wname, arrays, views in (("hier3m", arrays3m, cams), ("surround1m", surround(dev), surround_cams)):
        scene = pipeline.Scene(arrays, device=dev, requires_grad=False)
        N = scene.nodes.shape[0]
        R = scene.means3D.shape[0]
        mask = torch.zeros(R, dtype=torch.uint8, device=dev)
        cut_scratch = torch.empty(int(L.h3dgs_expand_scratch_bytes(N)), dtype=torch.uint8, device=dev)
        b_scratch = torch.empty(int(L.h3dgs_lod_budget_scratch_bytes(N)), dtype=torch.uint8, device=dev)
        count = torch.zeros(1, dtype=torch.int32, device=dev)
        thr_dev = torch.empty(1, device=dev)
        info = torch.empty(4, dtype=torch.int32, device=dev)
        bg = torch.zeros(3, device=dev)
        per_view = []
        for vi, c in enumerate(views):
            dcam = pipeline.DeviceCamera(c, device=dev)
            thr = pipeline.fov_threshold(6.0, dcam)
            floor = pipeline.fov_threshold(0.0, dcam)

            def mask_pass():
                _lib.check(L.h3dgs_lod_cull_mask(N, scene.nodes.data_ptr(), scene.means3D.data_ptr(), scene.scales.data_ptr(),
                                                 scene.rotations.data_ptr(), 1.0, dcam.viewmatrix.data_ptr(),
                                                 dcam.projmatrix.data_ptr(), W, H, float(dcam.tanfovx),
                                                 float(dcam.tanfovy), mask.data_ptr(), stream))

            def cut(m):
                _lib.check(L.h3dgs_lod_cut_masked(N, scene.nodes.data_ptr(), scene.boxes.data_ptr(), thr, None,
                                                  dcam.campos.data_ptr(), _lib.ptr(m), scene.render_indices.data_ptr(),
                                                  scene.parent_indices.data_ptr(), scene.nodes_for_render.data_ptr(),
                                                  scene.interpolation_weights.data_ptr(), scene.num_siblings.data_ptr(),
                                                  count.data_ptr(), cut_scratch.data_ptr(), stream))

            def budget(m):
                _lib.check(L.h3dgs_lod_budget_masked(N, scene.nodes.data_ptr(), scene.boxes.data_ptr(),
                                                     dcam.campos.data_ptr(), _lib.ptr(m), floor, None, args.budget, None,
                                                     thr_dev.data_ptr(), info.data_ptr(), b_scratch.data_ptr(), stream))
            mask_pass()
            ms = dict(mask=[], cut_nomask=[], cut_mask=[], budget_nomask=[], budget_mask=[])
            for _ in range(args.rounds):               # the arms alternate
                ms["mask"].append(device_ms(mask_pass))
                ms["cut_nomask"].append(device_ms(lambda: cut(None)))
                ms["cut_mask"].append(device_ms(lambda: cut(mask)))
                ms["budget_nomask"].append(device_ms(lambda: budget(None)))
                ms["budget_mask"].append(device_ms(lambda: budget(mask)))
            with torch.no_grad():
                img0, rad0, n0 = pipeline.render_hier_fused(scene, dcam, bg, thr)
                V = int((rad0[:n0] > 0).sum())
                _, _, n1 = pipeline.render_hier_fused(scene, dcam, bg, thr, cull=True)
                ref_img = pipeline.render_hier_fused(scene, dcam, bg, floor)[0].clone()
                fixed = {}
                for cull in (False, True):
                    img, rad, n, t, met = pipeline.render_hier_budget(scene, dcam, bg, args.budget, floor, cull=cull)
                    mse = float(((img - ref_img) ** 2).mean())
                    fixed["cull" if cull else "nocull"] = dict(threshold=t, tau=t * (0.5 * W) / (2 * float(dcam.tanfovx)) - 0.5,
                                                               rows=n, drawn=int((rad[:n] > 0).sum()), met=met,
                                                               psnr_vs_tau0=float(10 * np.log10(1.0 / max(mse, 1e-20))))
            per_view.append(dict(view=vi, cut_rows=n0, culled_rows=n1, V=V, culled_over_V=n1 / max(V, 1),
                                 dropped_fraction=1 - n1 / max(n0, 1),
                                 ms={k: float(np.median(v)) for k, v in ms.items()}, fixed_budget=fixed))
        # frames: GraphedRender at tau 6 and GraphedPostStep, cull off / on alternated
        c0 = pipeline.DeviceCamera(views[0], device=dev)
        thr = pipeline.fov_threshold(6.0, c0)
        forms = {}
        for cull in (False, True):
            gr = GraphedRender(scene, W, H, c0.tanfovx, c0.tanfovy, bg, thr, row_capacity=R, bin_capacity=1 << 25,
                               cull=cull, max_frames=4096)
            gr.set_camera(c0)
            gs = GraphedPostStep(scene, W, H, c0.tanfovx, c0.tanfovy, bg, thr, row_capacity=R, bin_capacity=1 << 25,
                                 capture=False, cull=cull)
            gs.set_camera(c0)
            gs.capture()
            forms[cull] = (gr, gs)
        gt = torch.rand((3, H, W), device=dev)
        frame_ms = {False: [], True: []}
        step_ms = {False: [], True: []}
        for _ in range(args.rounds):
            for cull in (False, True):
                gr, gs = forms[cull]
                gr.counter.zero_()
                frame_ms[cull].append(device_ms(gr.frame, reps=10))
                step_ms[cull].append(device_ms(lambda: gs.step(gt=gt), reps=10))
        status = {str(c): forms[c][1].status() for c in (False, True)}
        out[wname] = dict(nodes=N, views=per_view,
                          graphed_render_ms={"off": float(np.median(frame_ms[False])), "on": float(np.median(frame_ms[True]))},
                          post_step_ms={"off": float(np.median(step_ms[False])), "on": float(np.median(step_ms[True]))},
                          post_step_status=status)
        del forms, scene
        torch.cuda.empty_cache()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:    # pragma: no cover
        q = f"unavailable: {e}"
    print(json.dumps(dict(budget=args.budget, reps=args.reps, rounds=args.rounds, results=out, gpu=q)))


if __name__ == "__main__":
    main()

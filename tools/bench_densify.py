"""train_single's densify_and_prune on config #2's 1 M-row SH-3 state: the device densify (csrc/densify.cu through
SingleState.densify_and_prune) against the hand-over it replaces (copy_to_model, a torch densify_and_prune on the model
and from_model).

The statistics are seeded so that a few percent of the rows clone, split and prune (tests/densify_ref.py's
random_stats: 5 % of the rows with a large accumulated gradient; 3 % of the rows are given a scaling past
percent_dense * extent and 1 % an opacity below min_opacity).  Timed on the same card in one run:
  device_ms      SingleState.densify_and_prune end to end (decide, scan, the 16-byte count read, allocation, the normals
                 draw, the write pass), a host clock around a synchronise;
  write_ms       the write pass alone (h3dgs_densify WRITE: row pass + f_rest pass), CUDA events, with its achieved GB/s
                 from the algorithmic bytes: each written row's 59 floats and 118 moments written once, each source row
                 read once (a kept row's moments too);
  handover_ms    copy_to_model, the torch formulation below (the reference's mask gathers and cats on GaussianModel-shaped
                 tensors and their OurAdam state), and from_model, a host clock around a synchronise.
Prints one JSON line with the GPU's name and power limit read in the same run.  Writes nothing into the tree."""
import argparse
import json
import os
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402  (workloads; puts the package on sys.path)

EXTENT, SKY, MAX_GRAD, MIN_OPACITY, PERCENT_DENSE = 40.0, 20_000, 2e-4, 0.005, 0.01
ATTRS = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")
GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")


def gpu_conditions():
    import torch
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    f = [x.strip() for x in r.stdout.strip().split(",")] if r.returncode == 0 else [None, None]
    return {"gpu": torch.cuda.get_device_name(0), "power_limit": f[1]}


def torch_densify_and_prune(model, max_grad, min_opacity, extent):
    """scene/gaussian_model.py:543-685's data movement on a GaussianModel-shaped object: clone, split (appended), the
    split originals pruned, then the opacity prune, each group's parameter and OurAdam moments gathered and cat'ed"""
    import torch
    opt = model.optimizer

    def replace(fn):
        for g in opt.param_groups:
            p = g["params"][0]
            s = opt.state.pop(p)
            newp = torch.nn.Parameter(fn(p.detach(), g["name"], False))
            s["exp_avg"], s["exp_avg_sq"] = fn(s["exp_avg"], g["name"], True), fn(s["exp_avg_sq"], g["name"], True)
            g["params"][0] = newp
            opt.state[newp] = s
            setattr(model, ATTRS[GROUPS.index(g["name"])], newp)

    grads = model.xyz_gradient_accum
    grads[grads.isnan()] = 0.0
    op = torch.sigmoid(model._opacity).flatten()
    sc = torch.exp(model._scaling).max(dim=1).values
    gate = torch.pow(op, 1 / 5.0)
    sel = (torch.norm(grads, dim=-1) * model.max_radii2D * gate >= max_grad) & (op > 0.15) & (sc <= PERCENT_DENSE * extent)
    sel[:model.scaffold_points] = False
    replace(lambda t, n, mom: torch.cat((t, torch.zeros_like(t[sel]) if mom else t[sel])))
    n0 = sel.shape[0]
    model.max_radii2D = torch.cat((model.max_radii2D, torch.zeros(int(sel.sum()), device="cuda")))
    pg = torch.zeros(model._xyz.shape[0], device="cuda")
    pg[:n0] = grads.squeeze()
    op = torch.sigmoid(model._opacity).flatten()
    e = torch.exp(model._scaling)
    sp = (pg * model.max_radii2D * torch.pow(op, 1 / 5.0) >= max_grad) & (op > 0.15) & (e.max(dim=1).values > PERCENT_DENSE * extent)
    sp[:model.scaffold_points] = False
    stds = e[sp].repeat(2, 1)
    samples = torch.normal(mean=torch.zeros_like(stds), std=stds)
    q = torch.nn.functional.normalize(model._rotation[sp])
    r, x, y, z = q.unbind(1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3).repeat(2, 1, 1)
    new = {"xyz": torch.bmm(R, samples.unsqueeze(-1)).squeeze(-1) + model._xyz[sp].repeat(2, 1),
           "scaling": torch.log(e[sp].repeat(2, 1) / (0.8 * 2))}
    replace(lambda t, n, mom: torch.cat((t, torch.zeros_like(t[sp].repeat(2, *[1] * (t.dim() - 1))) if mom else
                                        new.get(n, t[sp].repeat(2, *[1] * (t.dim() - 1))))))
    keep = ~torch.cat((sp, torch.zeros(2 * int(sp.sum()), dtype=torch.bool, device="cuda")))
    replace(lambda t, n, mom: t[keep])
    prune = (torch.sigmoid(model._opacity) < min_opacity).squeeze()
    prune[:model.scaffold_points] = False
    replace(lambda t, n, mom: t[~prune])
    N2 = model._xyz.shape[0]
    model.xyz_gradient_accum = torch.zeros((N2, 1), device="cuda")
    model.denom = torch.zeros((N2, 1), device="cuda")
    model.max_radii2D = torch.zeros(N2, device="cuda")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import ctypes as C
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_densify.py needs a CUDA device: there is no CPU fallback for this path")
    import densify_ref
    from h3dgs import _lib
    from h3dgs.optim import Adam
    from h3dgs.singlestep import SingleState
    dev = "cuda:0"
    torch.cuda.set_device(0)
    arrays, _ = bench.build_workload("flat1m", device=dev)
    t = lambda a: torch.as_tensor(np.asarray(a, np.float32), device=dev)
    shs = t(arrays["shs"])
    op = t(arrays["opacities"]).reshape(-1, 1).clamp(1e-4, 1 - 1e-4)
    params = [t(arrays["means3D"]), shs[:, :1].contiguous(), shs[:, 1:].contiguous(), torch.log(op / (1 - op)),
              torch.log(t(arrays["scales"])), t(arrays["rotations"])]
    N = params[0].shape[0]
    g, r = densify_ref.random_stats(N, 3)
    rng = np.random.default_rng(4)
    big, faint = rng.random(N) < 0.03, rng.random(N) < 0.01
    params[4][torch.tensor(big, device=dev), 0] = float(np.log(0.6))
    params[3][torch.tensor(faint, device=dev)] = -6.0
    moments = [[torch.tensor(rng.normal(0, s, tuple(p.shape)).astype(np.float32), device=dev).abs() for p in params]
               for s in (1e-3, 1e-6)]
    lrs = [1.6e-4, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]
    exposure = torch.eye(3, 4, device=dev).repeat(4, 1, 1)

    def new_state():
        s = SingleState(params, SKY, lrs, exposure, exp_avg=moments[0], exp_avg_sq=moments[1], step=100,
                        scaffold_points=SKY, percent_dense=PERCENT_DENSE)
        s.stats.xyz_gradient_accum.copy_(torch.tensor(g, device=dev))
        s.stats.max_radii2D.copy_(torch.tensor(r, device=dev))
        return s

    def model_of(s):
        m = types.SimpleNamespace(skybox_points=SKY, skybox_locked=False, scaffold_points=SKY, percent_dense=PERCENT_DENSE)
        for a, p in zip(ATTRS, s.params):
            setattr(m, a, torch.nn.Parameter(torch.zeros_like(p)))
        m.optimizer = Adam([{"params": [getattr(m, a)], "lr": lr, "name": n} for a, lr, n in zip(ATTRS, lrs, GROUPS)],
                           lr=0.0, eps=1e-15)
        m._exposure = torch.nn.Parameter(torch.zeros_like(s.exposure))
        m.exposure_optimizer = torch.optim.Adam([m._exposure])
        return m

    # ---- device densify, end to end ------------------------------------------------------------------------------
    dev_ms, counts = [], None
    for i in range(args.warmup + args.repeats):
        s = new_state()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s.densify_and_prune(MAX_GRAD, MIN_OPACITY, EXTENT)
        torch.cuda.synchronize()
        if i >= args.warmup:
            dev_ms.append((time.perf_counter() - t0) * 1e3)
        counts = s.counts
        n_out = s.N

    # ---- the write pass alone --------------------------------------------------------------------------------------
    s = new_state()
    K, Cn, S = counts["kept"], counts["cloned"], counts["split"]
    nbytes = int(_lib.lib().h3dgs_densify_scratch_bytes(N))
    flags = torch.empty(N, dtype=torch.uint8, device=dev)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)     # the caching allocator aligns to 512 bytes
    a = s._densify_args()
    a.max_grad, a.min_opacity = MAX_GRAD, MIN_OPACITY
    a.size_threshold = float(np.float32(PERCENT_DENSE * EXTENT))
    a.xyz_gradient_accum, a.max_radii2D = s.stats.xyz_gradient_accum.data_ptr(), s.stats.max_radii2D.data_ptr()
    a.flags, a.scratch = flags.data_ptr(), scratch.data_ptr()
    s._launch_densify(a, _lib.DENSIFY_COUNT)
    normals = torch.randn((2 * S, 3), device=dev)
    out = [torch.empty((n_out,) + tuple(p.shape[1:]), device=dev) for p in s.params for _ in range(3)]
    a.out_rows, a.split_rows, a.normals = n_out, S, normals.data_ptr()
    for k in range(6):
        a.out_params[k], a.out_exp_avg[k], a.out_exp_avg_sq[k] = out[3 * k].data_ptr(), out[3 * k + 1].data_ptr(), out[3 * k + 2].data_ptr()
    L, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        _lib.check(L.h3dgs_densify(C.byref(a), _lib.DENSIFY_WRITE, st))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 20
    e0.record()
    for _ in range(reps):
        L.h3dgs_densify(C.byref(a), _lib.DENSIFY_WRITE, st)
    e1.record()
    torch.cuda.synchronize()
    write_ms = e0.elapsed_time(e1) / reps
    row = 59 * 4
    write_bytes = (N * row + K * 2 * row) + n_out * 3 * row + N                 # reads (+ kept moments), writes, flags

    # ---- the hand-over it replaces -----------------------------------------------------------------------------------
    ho_ms, n_torch = [], None
    for i in range(args.warmup + args.repeats):
        s = new_state()
        m = model_of(s)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s.copy_to_model(m)
        m.max_radii2D = s.stats.max_radii2D.clone()
        torch_densify_and_prune(m, MAX_GRAD, MIN_OPACITY, EXTENT)
        s2 = SingleState.from_model(m)
        torch.cuda.synchronize()
        if i >= args.warmup:
            ho_ms.append((time.perf_counter() - t0) * 1e3)
        n_torch = s2.N
    med = lambda x: float(np.median(x))
    print(json.dumps(dict(tool="bench_densify", workload="flat1m", N=N, n_out=n_out, n_out_torch=n_torch, kept=K,
                          cloned=Cn, split=S, pruned=N - K - S, device_ms=med(dev_ms), device_ms_min=min(dev_ms),
                          write_ms=write_ms, write_GBps=write_bytes / write_ms / 1e6, handover_ms=med(ho_ms),
                          handover_ms_min=min(ho_ms), **gpu_conditions())))


if __name__ == "__main__":
    main()

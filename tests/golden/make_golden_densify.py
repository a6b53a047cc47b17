"""Generates tests/golden/densify.npz by EXECUTING the reference's own GaussianModel.densify_and_prune and reset_opacity
(scene/gaussian_model.py:510-514, 543-685) on the CPU, through the fake_device harness (device="cuda" lands on the CPU),
on GaussianModel(3) states with OurAdam moments and densification statistics set by hand.  torch.normal is wrapped so
that the standard normals densify_and_split draws are recorded: it draws them as torch does (normal_(0, 1), then
mul_(std).add_(mean)).

Cases (inputs, the normals drawn, and the model and moments after the call):
  edges     gradients at and one ulp either side of max_grad (clone and split), opacity at 0.15 and just above, at the
            0.005 prune edge, the largest scaling at percent_dense * extent and one ulp above, a NaN accumulator, a NaN
            scaling, a NaN opacity, scaffold rows with large gradients, skybox rows past the scaffold, random rows
  no_split  S = 0;  no_clone  C = 0;  no_prune  nothing pruned;  all_pruned  every row past the scaffold pruned
  reset_sky / reset_none   reset_opacity with 6 skybox rows and with none
Needs a checkout of the reference, named by H3DGS_REFERENCE.

  tests/test_densify_cpu.py   tests/densify_ref.py and the kernels (emulation build) == this fixture
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "hierarchical-3d-gaussians_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "emul")):
    sys.path.insert(0, p)

import refharness                                    # noqa: E402
import densify_ref as D                              # noqa: E402
from fake_device import cuda_names_mean_cpu          # noqa: E402

F = np.float32
ATTRS = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")
MAX_GRAD, MIN_OPACITY, EXTENT, PERCENT_DENSE = 0.0002, 0.005, 8.0, 0.01


def _edge(target, f, x0, below=False):
    """the fp32 x where torch's f(x) reaches F(target): f(x) == target, or with below the largest x with f(x) < target"""
    x = torch.tensor([x0], dtype=torch.float32)
    up, down = torch.tensor([np.inf]), torch.tensor([-np.inf])
    while f(x).item() >= F(target):
        x = torch.nextafter(x, down)
    while f(torch.nextafter(x, up)).item() < F(target):
        x = torch.nextafter(x, up)
    if below:
        return F(x.item())
    x = torch.nextafter(x, up)
    assert f(x).item() == F(target), target
    return F(x.item())


def case_edges(rng):
    N, scaffold, skybox = 48, 3, 6
    p, m, v = D.random_state(N, 101)
    g, r = D.random_stats(N, 102, frac=0.3)
    hot = lambda i, s: (g.__setitem__((i, 0), 1.0), r.__setitem__(i, 10.0), p[3].__setitem__((i, 0), 3.0),
                        p[4].__setitem__(i, s))
    small, big = F(-6.0), F(-1.0)
    for i in range(3):                                   # the scaffold: large gradients, never densified or pruned
        hot(i, big if i else small)
    p[3][2, 0] = -9.0
    hot(3, small)                                        # skybox rows past the scaffold densify like any other
    hot(4, big)
    p[3][5, 0] = -9.0
    t = F(MAX_GRAD)
    for k, s in enumerate((small, big)):                 # o = sigmoid(20) = 1, pow(1, 0.2) = 1, r = 1: the product is g
        for j, gv in enumerate((np.nextafter(t, F(-1)), t, np.nextafter(t, F(1)))):
            i = 6 + 3 * k + j
            g[i, 0], r[i], p[3][i, 0], p[4][i] = gv, 1.0, 20.0, s
    o15 = _edge(0.15, torch.sigmoid, float(np.log(0.15 / 0.85)))
    hot(12, small); p[3][12, 0] = o15                                  # o == 0.15: not > 0.15
    hot(13, small); p[3][13, 0] = np.nextafter(o15, F(1))
    o005 = _edge(0.005, torch.sigmoid, float(np.log(0.005 / 0.995)), below=True)
    p[3][14, 0] = np.nextafter(o005, F(1))                              # sigmoid >= 0.005: kept
    p[3][15, 0] = o005                                                  # sigmoid < 0.005: pruned
    sT = _edge(F(PERCENT_DENSE * EXTENT), torch.exp, float(np.log(PERCENT_DENSE * EXTENT)))
    hot(16, [sT, -7.0, -7.0])                                           # max exp(s) == threshold: clone
    hot(17, [np.nextafter(sT, F(1)), -7.0, -7.0])                       # one ulp above: split
    hot(18, small); g[18, 0] = np.nan                                   # NaN accumulator counts as 0
    hot(19, big); p[4][19, 1] = np.nan                                  # NaN scaling: neither test holds
    hot(20, small); p[3][20, 0] = np.nan                                # NaN opacity: kept, never densified
    return p, m, v, g, r, scaffold, skybox


def case_filtered(seed, kind):
    N, scaffold, skybox = 40, 4, 2
    p, m, v = D.random_state(N, seed)
    g, r = D.random_stats(N, seed + 1, frac=0.4)
    r[:] = np.maximum(r, 20)
    if kind == "no_split":
        p[4][:] = np.minimum(p[4], F(-4.0))
    elif kind == "no_clone":
        p[4][:, 0] = np.maximum(p[4][:, 0], F(-1.5))
    elif kind == "no_prune":
        p[3][:] = np.abs(p[3]) + 0.5
    elif kind == "all_pruned":
        p[3][scaffold:] = -8.0
    return p, m, v, g, r, scaffold, skybox


def model(GaussianModel, p, m, v, g, r, scaffold, skybox):
    gm = GaussianModel(3)
    P = lambda a: torch.nn.Parameter(torch.tensor(a))
    gm._xyz, gm._features_dc, gm._features_rest = P(p[0]), P(p[1]), P(p[2])
    gm._opacity, gm._scaling, gm._rotation = P(p[3]), P(p[4]), P(p[5])
    gm._exposure = torch.nn.Parameter(torch.eye(3, 4)[None].repeat(2, 1, 1))
    gm.exposure_mapping = {"a": 0, "b": 1}
    gm.pretrained_exposures = None
    gm.skybox_points, gm.scaffold_points, gm.spatial_lr_scale = skybox, scaffold, 1.0
    opt = types.SimpleNamespace(percent_dense=PERCENT_DENSE, position_lr_init=0.00002, position_lr_final=0.0000002,
                                position_lr_delay_mult=0.01, position_lr_max_steps=30_000, feature_lr=0.0025,
                                opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001, exposure_lr_init=0.001,
                                exposure_lr_final=0.0001, exposure_lr_delay_steps=0, exposure_lr_delay_mult=0.0,
                                iterations=30_000)
    gm.training_setup(opt)
    for a, mk, vk in zip(ATTRS, m, v):
        t = getattr(gm, a)
        gm.optimizer.state[t] = dict(step=torch.tensor(7.0), exp_avg=torch.tensor(mk), exp_avg_sq=torch.tensor(vk))
    gm.xyz_gradient_accum = torch.tensor(g).reshape(-1, 1)
    gm.denom = torch.ones((p[0].shape[0], 1))
    gm.max_radii2D = torch.tensor(r)
    return gm


def record(out, name, gm):
    st = lambda a: gm.optimizer.state[getattr(gm, a)]
    for k, a in enumerate(ATTRS):
        out[f"{name}_out_p{k}"] = getattr(gm, a).detach().numpy().copy()
        out[f"{name}_out_m{k}"] = st(a)["exp_avg"].numpy().copy()
        out[f"{name}_out_v{k}"] = st(a)["exp_avg_sq"].numpy().copy()
        out[f"{name}_out_step{k}"] = np.float64(float(st(a)["step"]))
    out[f"{name}_out_max_radii2D"] = gm.max_radii2D.numpy().copy()
    out[f"{name}_out_xyz_gradient_accum"] = gm.xyz_gradient_accum.numpy().copy()
    out[f"{name}_out_denom"] = gm.denom.numpy().copy()


def main():
    assert refharness.have_reference()
    out = {}
    drawn = []
    real_normal = torch.normal

    def normal(mean, std, *a, **k):
        z = torch.empty(torch.broadcast_shapes(mean.shape, std.shape)).normal_(0, 1)
        drawn.append(z.clone())
        return z.mul_(std).add_(mean)
    with cuda_names_mean_cpu():
        refharness.import_reference_renderer()
        from scene.gaussian_model import GaussianModel
        torch.manual_seed(11)
        rng = np.random.default_rng(3)
        cases = [("edges", case_edges(rng))] + [(k, case_filtered(200 + 10 * i, k)) for i, k in
                                                 enumerate(("no_split", "no_clone", "no_prune", "all_pruned"))]
        for name, (p, m, v, g, r, scaffold, skybox) in cases:
            for k in range(6):
                out[f"{name}_p{k}"], out[f"{name}_m{k}"], out[f"{name}_v{k}"] = p[k], m[k], v[k]
            out[f"{name}_gacc"], out[f"{name}_radii"] = g.copy(), r.copy()
            out[f"{name}_scaffold"], out[f"{name}_skybox"] = np.int32(scaffold), np.int32(skybox)
            gm = model(GaussianModel, p, m, v, g.copy(), r, scaffold, skybox)
            drawn.clear()
            torch.normal = normal
            try:
                gm.densify_and_prune(MAX_GRAD, MIN_OPACITY, EXTENT)
            finally:
                torch.normal = real_normal
            assert len(drawn) == 1
            out[f"{name}_normals"] = drawn[0].numpy().copy()
            record(out, name, gm)
            print(f"{name}: N {p[0].shape[0]} -> {gm._xyz.shape[0]}, {drawn[0].shape[0] // 2} split")
        for name, skybox in (("reset_sky", 6), ("reset_none", 0)):
            p, m, v, g, r, _, _ = case_filtered(300 + skybox, "no_prune")
            p[3][:, 0] = np.linspace(-9, 9, p[3].shape[0]).astype(F)
            p[3][7, 0], p[3][1, 0] = np.nan, np.nan                         # NaN past and inside the skybox
            for k in range(6):
                out[f"{name}_p{k}"], out[f"{name}_m{k}"], out[f"{name}_v{k}"] = p[k], m[k], v[k]
            out[f"{name}_skybox"] = np.int32(skybox)
            gm = model(GaussianModel, p, m, v, g, r, 0, skybox)
            gm.reset_opacity()
            record(out, name, gm)
    np.savez_compressed(os.path.join(HERE, "densify.npz"), max_grad=np.float64(MAX_GRAD),
                        min_opacity=np.float64(MIN_OPACITY), extent=np.float64(EXTENT),
                        percent_dense=np.float64(PERCENT_DENSE), **out)


if __name__ == "__main__":
    main()

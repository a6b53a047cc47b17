"""H100: train_single's densify_and_prune and reset_opacity on the device state (csrc/densify.cu,
SingleState.densify_and_prune / reset_opacity) against the restatement tests/densify_ref.py with the device's exp / log
/ pow (torch's CUDA ones, which the kernels share): the fixture's case matrix and a 1 M-row state, every value bit for
bit but the split positions, which are checked within the budget of a reordered three-term product; torch's CUDA
division by the Python scalar 0.8 * 2 is the multiplication by the fp32 reciprocal the kernel uses; the drawn normals
are torch.normal's; a reset leaves every other byte of state unchanged; a graphed loop through a device densify
matches the same loop with the densify done on the host and handed over by from_model."""
import os
import sys
import types

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import densify_ref as D  # noqa: E402

pytestmark = pytest.mark.gpu
F = np.float32
CASES = ("edges", "no_split", "no_clone", "no_prune", "all_pruned")


def _z(golden_dir):
    return np.load(os.path.join(golden_dir, "densify.npz"))


def _state(p, m, v, g=None, r=None, scaffold=0, skybox=0, percent_dense=0.01):
    import torch
    from h3dgs.pipeline import DensifyStats
    from h3dgs.singlestep import SingleState
    N = p[0].shape[0]
    stats = DensifyStats(N, "cuda")
    if g is not None:
        stats.xyz_gradient_accum.copy_(torch.tensor(np.asarray(g, F)).reshape(N, 1))
        stats.max_radii2D.copy_(torch.tensor(np.asarray(r, F)))
    t = lambda a: [torch.tensor(np.asarray(x, F), device="cuda") for x in a]
    return SingleState(t(p), skybox, [0.0] * 6, torch.eye(3, 4, device="cuda")[None].repeat(2, 1, 1), exp_avg=t(m),
                       exp_avg_sq=t(v), step=7, stats=stats, scaffold_points=scaffold, percent_dense=percent_dense)


def _check(st, ref):
    K, Cn, S, N2 = ref["counts"]
    assert st.N == N2 and st.counts == dict(kept=K, cloned=Cn, split=S)
    split0 = N2 - 2 * S
    for k in range(6):
        for got, want in ((st.params[k], ref["params"][k]), (st.exp_avg[k], ref["exp_avg"][k]),
                          (st.exp_avg_sq[k], ref["exp_avg_sq"][k])):
            got = got.cpu().numpy()
            assert got.shape == want.shape
            if k == 0 and want is ref["params"][0]:
                assert np.array_equal(got[:split0].view(np.int32), want[:split0].view(np.int32))
                g_, w = got[split0:], want[split0:]
                assert np.all(np.abs(g_ - w) <= D.position_budget(g_, w, ref["mag"])), "split positions"
            else:
                assert np.array_equal(got.view(np.int32), want.view(np.int32)), (D.GROUPS[k], D.ulps(got, want).max())
    for t in (st.stats.max_radii2D, st.stats.xyz_gradient_accum, st.stats.denom):
        assert t.shape[0] == N2 and not bool(t.any())


@pytest.mark.parametrize("name", CASES)
def test_case_matrix_matches_restatement(golden_dir, name):
    import torch
    z = _z(golden_dir)
    p, m, v = ([z[f"{name}_{x}{k}"] for k in range(6)] for x in "pmv")
    st = _state(p, m, v, z[f"{name}_gacc"], z[f"{name}_radii"], int(z[f"{name}_scaffold"]), int(z[f"{name}_skybox"]))
    normals = z[f"{name}_normals"]
    st.densify_and_prune(float(z["max_grad"]), float(z["min_opacity"]), float(z["extent"]),
                         normals=torch.tensor(normals, device="cuda"))
    ref = D.densify(p, m, v, z[f"{name}_gacc"], z[f"{name}_radii"], int(z[f"{name}_scaffold"]), float(z["max_grad"]),
                    float(z["min_opacity"]), F(0.01 * 8.0), normals, D.torch_math("cuda"))
    _check(st, ref)
    # and the reference's row count
    assert st.N == z[f"{name}_out_p0"].shape[0]


def test_million_rows_match_restatement():
    import torch
    N = 1 << 20
    p, m, v = D.random_state(N, 9)
    g, r = D.random_stats(N, 10)
    M = D.torch_math("cuda")
    flags = D.decide(p, g, r, 1000, 2e-4, 0.005, F(0.08), M)
    S = int(((flags & 4) != 0).sum())
    normals = np.random.default_rng(3).normal(0, 1, (2 * S, 3)).astype(F)
    st = _state(p, m, v, g, r, 1000)
    st.densify_and_prune(2e-4, 0.005, 8.0, normals=torch.tensor(normals, device="cuda"))
    ref = D.densify(p, m, v, g, r, 1000, 2e-4, 0.005, F(0.08), normals, M)
    K, Cn, S, N2 = ref["counts"]
    assert Cn > N // 100 and S > N // 500 and K < N - N // 500          # a few percent clone, split and prune
    _check(st, ref)


def test_division_by_the_python_scalar_is_the_reciprocal_product():
    import torch
    g = torch.Generator(device="cuda").manual_seed(0)
    e = torch.exp(torch.randn(1 << 20, device="cuda", generator=g) * 3)
    inv = torch.tensor(np.float32(1) / np.float32(1.6), device="cuda")
    assert torch.equal((e / (0.8 * 2)).view(torch.int32), (e * inv).view(torch.int32))


def test_drawn_normals_are_torch_normal():
    """the state's draw with the default generator gives torch.normal(zeros, stds)'s samples from the same seed, and
    leaves the generator where torch.normal leaves it"""
    import torch
    N = 1 << 16
    p, m, v = D.random_state(N, 21)
    g, r = D.random_stats(N, 22)
    st = _state(p, m, v, g, r, 0)
    torch.cuda.manual_seed(1234)
    st.densify_and_prune(2e-4, 0.005, 8.0)
    after = torch.cuda.get_rng_state()
    S = st.counts["split"]
    assert S > 0
    split = (D.decide(p, g, r, 0, 2e-4, 0.005, F(0.08), D.torch_math("cuda")) & 4) != 0
    stds = torch.exp(torch.tensor(p[4][split], device="cuda")).repeat(2, 1)
    torch.cuda.manual_seed(1234)
    samples = torch.normal(mean=torch.zeros((2 * S, 3), device="cuda"), std=stds)
    assert torch.equal(torch.cuda.get_rng_state(), after)
    torch.cuda.manual_seed(1234)
    zs = torch.empty((2 * S, 3), device="cuda").normal_()
    assert torch.equal(samples.view(torch.int32), (zs * stds + 0).view(torch.int32))
    ref = D.densify(p, m, v, g, r, 0, 2e-4, 0.005, F(0.08), zs.cpu().numpy(), D.torch_math("cuda"))
    _check(st, ref)


def test_reset_changes_only_the_opacity_and_its_moments(golden_dir):
    import torch
    z = _z(golden_dir)
    for name in ("reset_sky", "reset_none"):
        p, m, v = ([z[f"{name}_{x}{k}"] for k in range(6)] for x in "pmv")
        sky = int(z[f"{name}_skybox"])
        st = _state(p, m, v, skybox=sky)
        everything = lambda: st.params + st.exp_avg + st.exp_avg_sq + [st.step, st.exposure, st.exposure_exp_avg,
                                                                        st.exposure_exp_avg_sq, st.exposure_step,
                                                                        st.stats.max_radii2D, st.stats.denom,
                                                                        st.stats.xyz_gradient_accum]
        before = [t.clone() for t in everything()]
        st.reset_opacity()
        o, _, _ = D.reset_opacity(p, m, v, sky, D.torch_math("cuda"))
        assert np.array_equal(st.params[3].cpu().numpy().view(np.int32), o.view(np.int32))
        assert not bool(st.exp_avg[3].any()) and not bool(st.exp_avg_sq[3].any())
        for i, (a, b) in enumerate(zip(before, everything())):
            if i not in (3, 9, 15):
                assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), i


# ---- a graphed loop through a device densify against the host hand-over -------------------------------------------
W, H, N, SKY, SCAFFOLD, NIMG, EXTENT = 320, 240, 20_000, 300, 600, 5, 30.0
NAMES = ("means3D", "shs", "opacities", "scales", "rotations")


def _model_of(state, params, m, v):
    """a GaussianModel-shaped object holding params / moments (numpy), OurAdam-shaped groups, and state's exposures"""
    import torch
    from h3dgs.optim import Adam
    attrs = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")
    model = types.SimpleNamespace(skybox_points=state.skybox_points, skybox_locked=state.skybox_locked,
                                  scaffold_points=state.scaffold_points, percent_dense=state.percent_dense)
    for a, x in zip(attrs, params):
        setattr(model, a, torch.nn.Parameter(torch.tensor(x, device="cuda")))
    model.optimizer = Adam([{"params": [getattr(model, a)], "lr": lr, "name": n} for a, lr, n in
                            zip(attrs, state.lr, D.GROUPS)], lr=0.0, eps=1e-15)
    for a, mk, vk in zip(attrs, m, v):
        model.optimizer.state[getattr(model, a)] = dict(step=torch.tensor(float(state.step.item())),
                                                        exp_avg=torch.tensor(mk, device="cuda"),
                                                        exp_avg_sq=torch.tensor(vk, device="cuda"))
    model._exposure = torch.nn.Parameter(state.exposure.clone())
    model.exposure_optimizer = torch.optim.Adam([model._exposure])
    model.exposure_optimizer.state[model._exposure] = dict(step=torch.tensor(float(state.exposure_step.item())),
                                                           exp_avg=state.exposure_exp_avg.clone(),
                                                           exp_avg_sq=state.exposure_exp_avg_sq.clone())
    return model


def test_graphed_loop_through_a_device_densify_matches_the_host_hand_over():
    import torch
    from h3dgs import synth
    from h3dgs.pipeline import DeviceCamera
    from h3dgs.singlestep import GraphedSingleStep, SingleState
    cam = synth.make_camera(W, H)
    c = synth.cloud_v1(N, cam, sh_degree=3, zmin=2.0, zmax=30.0, seed=7, scale_k=3e-3)
    t = lambda a: torch.tensor(np.asarray(a, F), device="cuda")
    op = c["opacities"].astype(np.float64)
    params = [t(c["means3D"]), t(c["shs"][:, :1]), t(c["shs"][:, 1:]), t(np.log(op / (1 - op))), t(np.log(c["scales"])),
              t(c["rotations"])]
    exposure = torch.eye(3, 4, device="cuda").repeat(NIMG, 1, 1)
    lrs = [1.6e-4, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]
    dcam = DeviceCamera(cam)

    def make_step(state):
        scene = state.make_scene(requires_grad=False)
        gs = GraphedSingleStep(scene, W, H, cam.tanfovx, cam.tanfovy, mask=True, sh_degree=1, capture=False,
                               state=state, cameras_extent=EXTENT)
        gs.set_camera(dcam)
        gs.capture()
        return gs

    def targets(k):
        g = torch.Generator(device="cuda").manual_seed(100 + k)
        return (torch.rand((3, H, W), device="cuda", generator=g), (torch.rand((1, H, W), device="cuda", generator=g) > 0.2).float(),
                torch.rand((1, H, W), device="cuda", generator=g) * 0.5, torch.ones((1, H, W), device="cuda"),
                torch.rand(3, device="cuda", generator=g))

    def everything(st, scene):
        return (st.params + st.exp_avg + st.exp_avg_sq + [st.step, st.exposure, st.exposure_exp_avg, st.exposure_exp_avg_sq,
                                                         st.exposure_step, st.stats.max_radii2D,
                                                         st.stats.xyz_gradient_accum, st.stats.denom] +
                [getattr(scene, k) for k in NAMES])

    def step(state, gs, it):
        gt, mask, mono, dmask, bg = targets(it)
        state.set_learning_rates(1.6e-4, 1e-3)
        gs.step(gt=gt, mask=mask, mono_invdepth=mono, depth_mask=dmask, bg=bg, depth_weight=0.3, image=it % NIMG)
        s = gs.status()
        assert not s["overflow"]
        return s["loss"]

    sa = SingleState(params, SKY, lrs, exposure, skybox_locked=True, scaffold_points=SCAFFOLD, percent_dense=0.01)
    ga = make_step(sa)
    for it in range(4):
        step(sa, ga, it)
    torch.cuda.synchronize()
    host = lambda ts: [x.cpu().numpy() for x in ts]
    p0, m0, v0 = host(sa.params), host(sa.exp_avg), host(sa.exp_avg_sq)
    model0 = _model_of(sa, p0, m0, v0)                             # the loop's GaussianModel, at the starting row count
    g0, r0 = sa.stats.xyz_gradient_accum.cpu().numpy(), sa.stats.max_radii2D.cpu().numpy()
    max_grad = float(np.quantile(g0[g0 > 0], 0.9))                 # a tenth of the visible rows clone or split
    M = D.torch_math("cuda")
    S = int(((D.decide(p0, g0, r0, SCAFFOLD, max_grad, 0.005, F(0.01 * EXTENT), M) & 4) != 0).sum())
    normals = np.random.default_rng(5).normal(0, 1, (2 * S, 3)).astype(F)
    # the host path: the restatement, then a GaussianModel-shaped hand-over through from_model
    ref = D.densify(p0, m0, v0, g0, r0, SCAFFOLD, max_grad, 0.005, F(0.01 * EXTENT), normals, M)
    sb = SingleState.from_model(_model_of(sa, ref["params"], ref["exp_avg"], ref["exp_avg_sq"]))
    # the device path
    sa.densify_and_prune(max_grad, 0.005, EXTENT, normals=torch.tensor(normals, device="cuda"))
    assert sa.N == sb.N and ref["counts"][1] > 0 and S > 0
    for x in (sa, sb):
        x.set_learning_rates(1.6e-4, 1e-3)
        x.set_image(1)
        x.no_gaussian_step(x.make_scene(requires_grad=False), EXTENT)
    ga, gb = make_step(sa), make_step(sb)
    torch.cuda.synchronize()
    # the two paths leave the same state, byte for byte (split positions included: the kernel and the restatement sum
    # the 3x3 product in the same order)
    for a, b in zip(everything(sa, ga.scene), everything(sb, gb.scene)):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
    # six rebuilt iterations, each from the common state: image, loss and radii bit for bit; after the step the
    # parameters differ only by the order of the backward's atomic sums, which Adam's normalisation can turn into at
    # most one step of 3.2 lr on an element whose gradient cancels, while almost every element agrees
    for it in range(4, 10):
        with torch.no_grad():
            for a, b in zip(everything(sb, gb.scene), everything(sa, ga.scene)):
                a.copy_(b)
        la, lb = step(sa, ga, it), step(sb, gb, it)
        torch.cuda.synchronize()
        assert la == lb and torch.equal(ga.image.view(torch.int32), gb.image.view(torch.int32)), it
        assert torch.equal(ga.radii, gb.radii), it
        assert int(sa.step.item()) == int(sb.step.item()) and int(sa.exposure_step.item()) == int(sb.exposure_step.item())
        for k in range(6):
            lr = 1.6e-4 if k == 0 else lrs[k]
            d = (sa.params[k] - sb.params[k]).abs()
            assert float(d.max()) <= 3.2 * lr, (it, D.GROUPS[k], float(d.max()))
            near = d <= 1e-5 * sb.params[k].abs() + 1e-7
            assert float(near.float().mean()) >= 0.995, (it, D.GROUPS[k], float(near.float().mean()))
    assert int(sa.step.item()) == 10 and int(sa.exposure_step.item()) == 11
    # the state handed back to the loop's GaussianModel (rows changed: its Parameters are rebound) and out again
    sa.copy_to_model(model0)
    back = SingleState.from_model(model0)
    assert back.N == sa.N and model0._xyz.shape[0] == sa.N
    for a, b in zip(everything(back, ga.scene)[:26], everything(sa, ga.scene)[:26]):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))

"""GPU: train_coarse's iteration on the device (csrc/loss.cu's coarse-loss pair, csrc/coarse_param.cu's parameter step,
h3dgs.loss.coarse_loss, pipeline.coarse_step, h3dgs.coarsestep.GraphedCoarseStep, h3dgs.optim.Adam with an [R,2] index).

  * the loss pair equals h3dgs_l1_ssim_forward / _backward bit for bit with a mask of ones and img in [0, 1];
  * given identical activated gradients, the parameter step against tests/coarse_ref.py in torch on the device: stored
    rows, moments and activated rows bit for bit (the same expf / logf), except F.normalize's backward and forward,
    whose 4-term sum torch may order otherwise (a few ulp);
  * the bias corrections of steps 1..30 000 equal the host's doubles rounded to fp32;
  * one iteration graphed against exact: image, fp32 loss and L1 bit for bit, parameters to the order of the
    backward's atomic sums; 30 iterations with both target slots in use; an overflowed frame changes no state byte and
    its exact re-run does; the SH degree hand-over; the state round trip through a GaussianModel-shaped object;
  * h3dgs.optim.Adam with train_coarse's [R,2] index updates relevant[:,0] and row 0 once;
  * against tests/golden/coarse_iteration.npz (the reference's own GaussianModel, OurAdam and render_coarse over four
    iterations, one of them with an empty index and OurAdam's dense step): the parameter step, the loss pair and
    h3dgs.optim.Adam with the reference's index, within the budget tests/coarse_ref.golden_violations derives."""
import os
import sys
import types

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import coarse_ref as CR  # noqa: E402
from h3dgs import synth  # noqa: E402

pytestmark = pytest.mark.gpu
F = np.float32
NAMES = ("means3D", "shs", "opacities", "scales", "rotations")


def ulps(a, b):
    a, b = np.asarray(a, F).ravel(), np.asarray(b, F).ravel()
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    d = np.abs(ia - ib)
    d[np.isnan(a) & np.isnan(b)] = 0
    return d


def _state_from(st):
    from h3dgs.coarsestep import CoarseState
    return CoarseState(st["params"], st["skybox"], st["lr"], st["betas"], st["eps"], st["exp_avg"], st["exp_avg_sq"], st["step"])


@pytest.mark.parametrize("shape", [(1, 1), (37, 53), (1080, 1920)])
def test_coarse_loss_with_ones_is_l1_ssim(shape):
    import torch
    from h3dgs.loss import coarse_loss, fused_l1_ssim
    g = torch.Generator(device="cuda").manual_seed(3)
    img = torch.rand((3,) + shape, device="cuda", generator=g)
    gt = torch.rand((3,) + shape, device="cuda", generator=g)
    x0, x1, x2 = (img.clone().requires_grad_(True) for _ in range(3))
    a = coarse_loss(x0, gt, 0.2, torch.ones(shape, device="cuda"))
    b = fused_l1_ssim(x1, gt, 0.2)
    c = coarse_loss(x2, gt, 0.2, None)
    for out, x in ((a, x0), (b, x1), (c, x2)):
        out[0].backward()
    assert torch.equal(x0.grad.view(torch.int32), x1.grad.view(torch.int32))
    assert torch.equal(x2.grad.view(torch.int32), x1.grad.view(torch.int32))
    # above 1 the gradient passes where the clamped objective would stop it
    y = (img * 1.5).requires_grad_(True)
    coarse_loss(y, gt, 0.2)[0].backward()
    over = img * 1.5 > 1
    assert int((y.grad[over] != 0).sum()) >= 0.99 * int(over.sum())


@pytest.mark.parametrize("N,S,seed", [(1, 0, 1), (1000, 100, 2), (200_000, 5000, 3)])
def test_param_step_matches_restatement(N, S, seed):
    import torch
    st = CR.random_state(N, S, seed, device="cuda")
    grads = CR.random_grads(N, seed + 1, device="cuda")
    if N > 10:
        st["params"][3][S + 5, 0] = 30.0                    # the stored opacity gradient underflows to 0
        grads["opacities"][S + 5, 0] = 1e-30
        grads["opacities"][S + 6, 0] = float("nan")
        st["params"][4][S + 10:S + 200] = -0.5 + 0.01 * torch.arange(190, device="cuda")[:, None]   # exp 0.61 .. 4.0 around the 0.6 threshold
        for v in grads.values():
            v[0] = 0
    state = _state_from(st)
    scene = state.make_scene(requires_grad=False)
    act = CR.activate(st["params"])
    for k in NAMES:
        got, want = getattr(scene, k).detach(), act[k]
        if k == "rotations":
            assert ulps(got.cpu(), want.cpu()).max() <= 2
        else:
            assert torch.equal(got.reshape(want.shape).view(torch.int32), want.view(torch.int32)), k
    ref = CR.clone_state(st)
    thr = 0.6
    relevant, act_ref = CR.param_step(ref, {k: getattr(scene, k).detach().clone().reshape(act[k].shape) for k in NAMES},
                                      grads, thr)
    state.param_step(scene, {k: v.contiguous() for k, v in grads.items()}, thr / 0.1)
    torch.cuda.synchronize()
    assert int(state.step.item()) == ref["step"]
    for k in range(6):
        for name, got, want in (("param", state.params[k], ref["params"][k]), ("exp_avg", state.exp_avg[k], ref["exp_avg"][k]),
                                ("exp_avg_sq", state.exp_avg_sq[k], ref["exp_avg_sq"][k])):
            d = ulps(got.cpu(), want.cpu())
            # the rotation group's gradient is F.normalize's backward
            assert d.max() <= (4 if k == 5 else 0), (CR.GROUPS[k], name, int(d.max()))
    for k in NAMES:
        got, want = getattr(scene, k).detach().reshape(act_ref[k].shape), act_ref[k]
        assert ulps(got.cpu(), want.cpu()).max() <= (2 if k == "rotations" else 0), k


def test_bias_corrections_of_30000_steps_are_the_host_doubles():
    import ctypes as C
    import torch
    from h3dgs import _lib
    st = CR.random_state(4, 0, 5, device="cuda")
    state = _state_from(st)
    scene = state.make_scene(requires_grad=False)
    args = state._args(scene, 1.0)
    T = 30_000
    out = torch.empty((T, 16), dtype=torch.int32, device="cuda")
    L = _lib.lib()
    s = torch.cuda.current_stream().cuda_stream
    for t in range(T):
        state.step.fill_(t)
        _lib.check(L.h3dgs_coarse_param_step(C.byref(args), _lib.COARSE_BIAS, s))
        out[t].copy_(state.scratch.view(torch.int32)[:16])
    got = out.cpu().numpy()[:, :12].view(F)
    for t in (0, 1, 9, 99, 999, 9999, 29_999):
        for k in range(6):
            want = CR.bias_corrections(st["lr"][k], 0.9, 0.999, t + 1)
            assert got[t, k] == want[0] and got[t, 6 + k] == want[1], (t, k)
    steps = np.arange(1, T + 1, dtype=np.float64)
    for k in range(6):
        ss = (st["lr"][k] / (1 - 0.9 ** steps)).astype(F)
        bc = np.sqrt(1 - 0.999 ** steps).astype(F)
        assert np.array_equal(got[:, k], ss) and np.array_equal(got[:, 6 + k], bc), k


# ---- the graphed step against the exact path ----------------------------------------------------------------------------
W, H, N, SKY = 320, 240, 20_000, 500


def _scene_state(seed=7, sh=1):
    """a scaffold-like state: skybox rows first, GaussianModel's stored tensors from a synthetic cloud"""
    import torch
    cam = synth.make_camera(W, H)
    c = synth.cloud_v1(N, cam, sh_degree=sh, zmin=2.0, zmax=30.0, seed=seed, scale_k=3e-3)
    t = lambda a: torch.tensor(np.asarray(a, F), device="cuda")
    op = c["opacities"].astype(np.float64)
    params = [t(c["means3D"]), t(c["shs"][:, :1]), t(c["shs"][:, 1:]), t(np.log(op / (1 - op))), t(np.log(c["scales"])),
              t(c["rotations"])]
    lrs = [0.0, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]
    return cam, params, lrs


def _pair(mask=False, sh_degree=0, capture=True, **kw):
    import torch
    from h3dgs.coarsestep import CoarseState, GraphedCoarseStep
    from h3dgs.pipeline import DeviceCamera
    cam, params, lrs = _scene_state()
    sa, sb = CoarseState(params, SKY, lrs, eps=1e-15), CoarseState(params, SKY, lrs, eps=1e-15)
    sca, scb = sa.make_scene(), sb.make_scene(requires_grad=False)
    dcam = DeviceCamera(cam)
    gs = GraphedCoarseStep(sb, scb, W, H, cam.tanfovx, cam.tanfovy, cameras_extent=8.0, mask=mask, sh_degree=sh_degree,
                           capture=False, **kw)
    gs.set_camera(dcam)
    if capture:
        gs.capture()
    return cam, dcam, (sa, sca), (sb, scb), gs


def _targets(k):
    import torch
    g = torch.Generator(device="cuda").manual_seed(100 + k)
    gt = torch.rand((3, H, W), device="cuda", generator=g)
    mask = (torch.rand((1, H, W), device="cuda", generator=g) > 0.2).float()
    bg = torch.rand(3, device="cuda", generator=g)
    return gt, mask, bg


def _state_close(sa, sb, rtol, atol):
    import torch
    for k in range(6):
        for a, b in ((sa.params[k], sb.params[k]), (sa.exp_avg[k], sb.exp_avg[k]), (sa.exp_avg_sq[k], sb.exp_avg_sq[k])):
            assert torch.allclose(a, b, rtol=rtol, atol=atol), (CR.GROUPS[k], float((a - b).abs().max()))
    assert torch.equal(sa.max_radii2D, sb.max_radii2D) and int(sa.step.item()) == int(sb.step.item())


def test_one_iteration_graphed_is_exact():
    import torch
    from h3dgs.pipeline import coarse_step
    cam, dcam, (sa, sca), (sb, scb), gs = _pair(mask=True)
    gt, mask, bg = _targets(0)
    (loss, l1, ssim), radii = coarse_step(sa, sca, dcam, bg, gt, 8.0, 0.2, mask, sh_degree=0)
    gs.step(gt=gt, mask=mask, bg=bg)
    torch.cuda.synchronize()
    s = gs.status()
    assert not s["overflow"] and s["D"] > 0
    assert torch.equal(radii, gs.radii)
    # the same kernels on the same image: the fp32 loss and L1 are the exact path's bit for bit
    assert np.float32(s["loss"]) == np.float32(float(loss)) and np.float32(s["l1"]) == np.float32(float(l1))
    _state_close(sa, sb, rtol=1e-4, atol=1e-7)
    for k in NAMES:
        assert torch.allclose(getattr(sca, k).detach(), getattr(scb, k), rtol=1e-4, atol=1e-7), k


def test_image_of_graphed_forward_is_exact():
    import torch
    from h3dgs.pipeline import render_flat
    cam, dcam, (sa, sca), (sb, scb), gs = _pair(capture=False)
    gt, _, bg = _targets(1)
    with torch.no_grad():
        img, radii = render_flat(sca, dcam, bg, 0)
    gs.set_background(bg)
    gs._part_a()
    torch.cuda.synchronize()
    assert torch.equal(img.view(torch.int32), gs.image.view(torch.int32)) and torch.equal(radii, gs.radii)


def test_thirty_iterations_with_both_slots_track_the_exact_path():
    import torch
    from h3dgs.pipeline import coarse_step
    cam, dcam, (sa, sca), (sb, scb), gs = _pair(mask=True)
    side = torch.cuda.Stream()
    losses = []
    for it in range(30):
        gt, mask, bg = _targets(it)
        coarse_step(sa, sca, dcam, bg, gt, 8.0, 0.2, mask, sh_degree=0)
        ev = gs.upload_target(gt, side, mask)
        gs.step(bg=bg, gt_ready=ev)
        losses.append(gs.status()["loss"])
    torch.cuda.synchronize()
    # gradients differ in the order of the backward's atomic sums (~1e-7 relative); this tolerance is a guard chosen
    # well above the drift seen, not a derived bound (a relevance flip could in principle move a row by a whole step)
    _state_close(sa, sb, rtol=1e-3, atol=1e-5)
    assert losses[-1] < losses[0]


def test_overflowed_frame_changes_nothing_and_the_exact_rerun_does():
    import torch
    from h3dgs.pipeline import coarse_step
    cam, dcam, (sa, sca), (sb, scb), gs = _pair(bin_capacity=64)
    gt, _, bg = _targets(2)
    before = [t.clone() for t in sb.params + sb.exp_avg + sb.exp_avg_sq + [sb.step, sb.max_radii2D]] + \
             [getattr(scb, k).clone() for k in NAMES]
    gs.step(gt=gt, bg=bg)
    assert gs.status()["overflow"]
    after = sb.params + sb.exp_avg + sb.exp_avg_sq + [sb.step, sb.max_radii2D] + [getattr(scb, k) for k in NAMES]
    for a, b in zip(before, after):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
    scb.means3D.requires_grad_(True); scb.shs.requires_grad_(True); scb.opacities.requires_grad_(True)
    scb.scales.requires_grad_(True); scb.rotations.requires_grad_(True)
    coarse_step(sb, scb, dcam, bg, gt, 8.0, 0.2, None, sh_degree=0)
    assert int(sb.step.item()) == 1 and not torch.equal(sb.params[3], before[3])


def test_degree_hand_over_and_state_round_trip():
    import torch
    from h3dgs.coarsestep import CoarseState, GraphedCoarseStep
    from h3dgs.optim import Adam
    cam, dcam, (sa, sca), (sb, scb), gs = _pair()
    for it in range(3):
        gt, _, bg = _targets(it)
        gs.step(gt=gt, bg=bg)
    g1 = GraphedCoarseStep(sb, scb, W, H, cam.tanfovx, cam.tanfovy, cameras_extent=8.0, sh_degree=1, capture=False)
    g1.set_camera(dcam)
    g1.capture()
    rest0 = sb.params[2].clone()
    for it in range(3):
        gt, _, bg = _targets(10 + it)
        g1.step(gt=gt, bg=bg)
    torch.cuda.synchronize()
    assert int(sb.step.item()) == 6 and not g1.status()["overflow"]
    assert not torch.equal(rest0, sb.params[2])          # degree 1 trains the rest coefficients
    # a GaussianModel-shaped object with OurAdam-shaped groups and state
    model = types.SimpleNamespace(skybox_points=SKY)
    for a, p in zip(("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation"), sb.params):
        setattr(model, a, torch.nn.Parameter(torch.zeros_like(p)))
    model.optimizer = Adam([{"params": [getattr(model, a)], "lr": lr, "name": n} for a, lr, n in
                            zip(("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation"), sb.lr,
                                ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation"))], lr=0.0, eps=1e-15)
    sb.copy_to_model(model)
    back = CoarseState.from_model(model)
    assert int(back.step.item()) == 6 and back.lr == sb.lr and back.skybox_points == SKY
    for k in range(6):
        assert torch.equal(back.params[k], sb.params[k]) and torch.equal(back.exp_avg[k], sb.exp_avg[k])
        assert torch.equal(back.exp_avg_sq[k], sb.exp_avg_sq[k])
    assert torch.equal(back.max_radii2D, sb.max_radii2D)


def test_adam_with_an_unflattened_index_updates_column_0_and_row_0_once():
    import torch
    from h3dgs.optim import Adam
    g = torch.Generator(device="cuda").manual_seed(4)
    N = 5000
    p0 = torch.randn((N, 1), device="cuda", generator=g)
    grads = [torch.randn((N, 1), device="cuda", generator=g) * (torch.rand((N, 1), device="cuda", generator=g) > 0.5)
             for _ in range(4)]
    grads[2].zero_()                                     # a step without a relevant row
    for gr in grads:
        gr[0] = 0                                        # row 0 moves by the zero column of the index alone
    pa, pb = torch.nn.Parameter(p0.clone()), torch.nn.Parameter(p0.clone())
    oa, ob = Adam([pa], lr=0.01, eps=1e-15), Adam([pb], lr=0.01, eps=1e-15)
    for gr in grads:
        pa.grad, pb.grad = gr.clone(), gr.clone()
        rel = (gr != 0).nonzero()                        # [R,2], train_coarse.py:136
        assert rel.shape[1] == 2
        oa.step(rel)
        rows = torch.unique(torch.cat((rel[:, 0], rel.new_zeros(1)))) if rel.shape[0] else rel.new_zeros(0)
        ob.step(rows)
        torch.cuda.synchronize()
        assert torch.equal(pa.view(torch.int32), pb.view(torch.int32))
        assert torch.equal(oa.state[pa]["exp_avg"], ob.state[pb]["exp_avg"])
    assert float(oa.state[pa]["step"]) == 4.0


# ---- against the reference's own GaussianModel, OurAdam and render_coarse (tests/golden/coarse_iteration.npz) ---------------
@pytest.mark.parametrize("c", range(4))
def test_param_step_is_the_reference_iteration(golden_dir, c):
    import torch
    z = np.load(os.path.join(golden_dir, "coarse_iteration.npz"))
    st = CR.golden_start(z, c)
    act, grads = CR.golden_inputs(z, c)
    dst = dict(st)
    for key in ("params", "exp_avg", "exp_avg_sq"):
        dst[key] = [t.cuda() for t in st[key]]
    state = _state_from(dst)
    scene = state.make_scene(requires_grad=False)
    for k in NAMES:                                   # the reference's activated rows are what the forward read
        getattr(scene, k).copy_(act[k].reshape(getattr(scene, k).shape))
    state.param_step(scene, {k: v.cuda().contiguous() for k, v in grads.items()}, float(z["extent"]))
    torch.cuda.synchronize()
    assert int(state.step.item()) == int(z[f"c{c}_step"])
    # the rows placed one ulp around the rescale threshold were placed with the CPU's exp; on the device the decision is
    # torch's CUDA exp's, the same expf the kernel calls
    edges = [int(r) for r in z["edges"]]
    sa = torch.tensor(z[f"c{c}_adam_scaling"], device="cuda")[edges]
    viol = (torch.exp(sa).max(dim=1).values > float(np.float32(float(z["extent"]) * 0.1))).cpu().numpy()
    moved = (state.params[4][edges].cpu().numpy() != z[f"c{c}_adam_scaling"][edges]).any(axis=1)
    assert np.array_equal(viol, moved)
    bad = CR.golden_violations(z, c, st, [p.cpu().numpy() for p in state.params], [m.cpu().numpy() for m in state.exp_avg],
                               [v.cpu().numpy() for v in state.exp_avg_sq], skip_rows=edges)
    assert not bad, bad


@pytest.mark.parametrize("c", range(4))
def test_loss_pair_is_the_reference_objective(golden_dir, c):
    import torch
    from h3dgs.loss import coarse_loss
    z = np.load(os.path.join(golden_dir, "coarse_iteration.npz"))
    img = torch.tensor(z[f"c{c}_image"], device="cuda", requires_grad=True)
    M = torch.tensor(z[f"c{c}_mask"], device="cuda") if int(z[f"c{c}_has_mask"]) else None
    loss, l1, _ = coarse_loss(img, torch.tensor(z[f"c{c}_gt"], device="cuda"), float(z["lam"]), M)
    loss.backward()
    # fp32 sums in another order than conv2d's: the budget of tests/test_single_loss_cpu.py's golden comparison
    assert abs(float(l1) - float(z[f"c{c}_l1"])) < 1e-6 and abs(float(loss) - float(z[f"c{c}_loss"])) < 1e-6
    ref = z[f"c{c}_dimage"]
    assert np.abs(img.grad.cpu().numpy() - ref).max() <= 1e-5 * np.abs(ref).max()


def test_adam_with_the_reference_index_is_ouradam(golden_dir):
    """h3dgs.optim.Adam driven with the reference's own [R,2] index (and, in iteration 2, its empty one) on the reference's
    stored gradients reproduces OurAdam's parameters within the budget of tests/coarse_ref.golden_violations"""
    import torch
    from h3dgs.optim import Adam
    z = np.load(os.path.join(golden_dir, "coarse_iteration.npz"))
    ps = [torch.nn.Parameter(torch.tensor(z[f"init_{a}"], device="cuda")) for a in CR.ATTRS]
    opt = Adam([{"params": [p], "lr": float(lr)} for p, lr in zip(ps, z["lrs"])], lr=0.0, eps=1e-15)
    for c in range(4):
        st = CR.golden_start(z, c)
        with torch.no_grad():
            for p, a in zip(ps, CR.ATTRS):            # the iteration starts from the reference's state (after its rescale)
                p.copy_(torch.tensor(z[f"c{c - 1}_after{a}"] if c else z[f"init_{a}"], device="cuda"))
        for p, a in zip(ps, CR.ATTRS):
            p.grad = torch.tensor(z[f"c{c}_grad{a}"], device="cuda")
        opt.step(torch.tensor(z[f"c{c}_relevant"], device="cuda"))
        torch.cuda.synchronize()
        for k, (p, a) in enumerate(zip(ps, CR.ATTRS)):
            got, want = p.detach().cpu().numpy().astype(np.float64), z[f"c{c}_adam{a}"].astype(np.float64)
            u = np.abs(want - st["params"][k].numpy())
            tol = 2.0 ** -20 * u + 2 * np.spacing(np.abs(want).astype(F)) + 1e-45
            assert np.all(np.abs(got - want) <= tol), (c, a)
        assert float(opt.state[ps[0]]["step"]) == float(z[f"c{c}_step"])

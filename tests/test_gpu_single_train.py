"""GPU: train_single's parameter step on the device (csrc/single_param.cu, h3dgs.singlestep.SingleState, the state path
of GraphedSingleStep and pipeline.single_step).

  * given identical activated gradients, the step against tests/single_train_ref.py: stored rows, moments, exposures
    and step counts bit for bit (the same expf / logf on the device), except F.normalize's backward and forward;
  * the exposure's Adam equals torch.optim.Adam([_exposure]) on the same GPU bit for bit over 100 steps with a changing
    lr and a changing image;
  * the bias corrections of steps 1..30 000 equal the host's doubles rounded to fp32;
  * the graphed whole iteration against the exact path over 30 iterations with both target slots, the lrs changing
    every iteration and the images cycling: images and losses bit for bit, parameters to the order of the backward's
    atomic sums; an overflowed frame changes no state byte and its exact re-run does; capture's warm-up changes no
    state; the state survives a row-count change across a hand-over."""
import os
import sys
import types

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import coarse_ref as CR  # noqa: E402
import single_train_ref as SR  # noqa: E402
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


def _state_from(st, device="cuda"):
    import torch
    from h3dgs.singlestep import SingleState
    mv = lambda xs: [x.to(device) for x in xs]
    return SingleState(mv(st["params"]), st["skybox"], st["lr"], torch.tensor(st["exposure"]), st["betas"], st["eps"],
                       mv(st["exp_avg"]), mv(st["exp_avg_sq"]), st["step"], skybox_locked=st["skybox_locked"],
                       scaffold_points=st["scaffold"], exposure_exp_avg=torch.tensor(st["exposure_m"]),
                       exposure_exp_avg_sq=torch.tensor(st["exposure_v"]), exposure_step=st["exposure_step"])


@pytest.mark.parametrize("N,S,locked,scaffold,seed", [(1, 0, True, 0, 1), (1000, 100, True, 0, 2),
                                                      (200_000, 5000, False, 20_000, 3), (50_000, 500, True, 800, 4)])
def test_param_step_matches_restatement(N, S, locked, scaffold, seed):
    import torch
    # the restatement runs on the device too: torch's CUDA exp / log are the kernel's expf / logf, which matters where
    # log(exp(s) * 0.8) cancels near 0
    st = SR.random_single_state(N, S, seed, skybox_locked=locked, scaffold=scaffold, device="cuda")
    grads = CR.random_grads(N, seed + 1, device="cuda", K=15)
    if N > 10:
        st["params"][3][S + 5, 0] = 30.0
        grads["opacities"][S + 5, 0] = 1e-30
        grads["opacities"][S + 6, 0] = float("nan")
        st["params"][4][S + 10:S + 200] = -0.5 + 0.01 * torch.arange(190, device="cuda")[:, None]   # exp 0.61 .. 4.0
        st["params"][4][:50] = 1.0
        for v in grads.values():
            v[0] = 0
    state = _state_from(st)
    scene = state.make_scene(requires_grad=False)
    xyz_lr, exp_lr, image, extent = 1.1e-4, 6e-4, seed % 4, 30.0
    thr = extent * 0.02
    eg = np.random.default_rng(seed).normal(0, 1e-2, (3, 4)).astype(F)
    state.set_learning_rates(xyz_lr, exp_lr)
    state.set_image(image)
    act = {k: getattr(scene, k).detach().clone().reshape(v.shape) for k, v in CR.activate(st["params"]).items()}
    ref = SR.clone_single(st)
    ref["exposure_step"] += 1
    SR.exposure_adam(ref["exposure"], ref["exposure_m"], ref["exposure_v"], eg, image, exp_lr, ref["exposure_step"])
    relevant, act_ref = SR.gaussian_step(ref, act, grads, thr, xyz_lr)
    state.param_step(scene, {k: v.cuda().contiguous() for k, v in grads.items()}, extent, torch.tensor(eg, device="cuda"))
    torch.cuda.synchronize()
    assert int(state.step.item()) == ref["step"] and int(state.exposure_step.item()) == ref["exposure_step"]
    for k in range(6):
        for name, got, want in (("param", state.params[k], ref["params"][k]), ("exp_avg", state.exp_avg[k], ref["exp_avg"][k]),
                                ("exp_avg_sq", state.exp_avg_sq[k], ref["exp_avg_sq"][k])):
            d = ulps(got.cpu(), want.cpu())
            # the rotation group's gradient is F.normalize's backward
            assert d.max() <= (4 if k == 5 else 0), (CR.GROUPS[k], name, int(d.max()))
    for k in NAMES:
        got, want = getattr(scene, k).detach().reshape(act_ref[k].shape), act_ref[k]
        assert ulps(got.cpu(), want.cpu()).max() <= (2 if k == "rotations" else 0), k
    for got, want in ((state.exposure, ref["exposure"]), (state.exposure_exp_avg, ref["exposure_m"]),
                      (state.exposure_exp_avg_sq, ref["exposure_v"])):
        assert np.array_equal(got.cpu().numpy().view(np.int32), want.view(np.int32))
    if N > 10:
        assert 0 not in set(relevant.tolist()) and S + 5 not in set(relevant.tolist()) and S + 6 in set(relevant.tolist())
        assert (not locked) or int(relevant.min()) >= S


def test_exposure_adam_is_torch_adam():
    """100 steps of torch.optim.Adam([_exposure]) (its default foreach CUDA path) against the kernel on the same GPU, with
    the lr changing every step, the image cycling and one step at a zero gradient: bit for bit"""
    import torch
    from h3dgs.singlestep import SingleState
    n = 7
    g = torch.Generator(device="cuda").manual_seed(11)
    ex0 = torch.eye(3, 4, device="cuda").repeat(n, 1, 1) + 0.05 * torch.randn((n, 3, 4), device="cuda", generator=g)
    param = torch.nn.Parameter(ex0.clone())
    opt = torch.optim.Adam([param])
    st = CR.random_state(2, 0, 1, device="cuda")
    state = SingleState(st["params"], 0, st["lr"], ex0)
    scene = state.make_scene(requires_grad=False)
    lr_fn = lambda it: 0.001 * (0.1 ** (it / 100)) * (0.001 + 0.999 * np.sin(0.5 * np.pi * min(it / 50, 1)))
    for it in range(100):
        image = (3 * it) % n
        eg = torch.randn((3, 4), device="cuda", generator=g) * (0.0 if it == 40 else 1e-2)
        lr = lr_fn(it + 1)
        for group in opt.param_groups:
            group["lr"] = lr
        param.grad = torch.zeros_like(param)
        param.grad[image] = eg
        opt.step()
        state.set_learning_rates(0.0, lr)
        state.set_image(image)
        state.no_gaussian_step(scene, 1.0, eg)
        torch.cuda.synchronize()
        s = opt.state[param]
        for got, want, what in ((state.exposure, param.detach(), "param"), (state.exposure_exp_avg, s["exp_avg"], "exp_avg"),
                                (state.exposure_exp_avg_sq, s["exp_avg_sq"], "exp_avg_sq")):
            d = ulps(got.cpu(), want.cpu())
            assert d.max() == 0, (it, what, int(d.max()), int((d > 0).sum()))
        assert int(state.exposure_step.item()) == int(float(s["step"]))


def test_bias_corrections_of_30000_steps_are_the_host_doubles():
    import ctypes as C
    import torch
    from h3dgs import _lib
    st = SR.random_single_state(4, 0, 5)
    state = _state_from(st)
    scene = state.make_scene(requires_grad=False)
    xyz_lr, exp_lr = 1.6e-5, 1e-3
    state.set_learning_rates(xyz_lr, exp_lr)
    args = state._single_args(scene, 1.0)
    T = 30_000
    out = torch.empty((T, 16), dtype=torch.int32, device="cuda")
    L = _lib.lib()
    s = torch.cuda.current_stream().cuda_stream
    for t in range(T):
        state.step.fill_(t)
        state.exposure_step.fill_(t)
        _lib.check(L.h3dgs_single_param_step(C.byref(args), _lib.SINGLE_BIAS, s))
        out[t].copy_(state.scratch.view(torch.int32)[:16])
    got = out.cpu().numpy().view(F)
    steps = np.arange(1, T + 1, dtype=np.float64)
    lrs = [xyz_lr] + st["lr"][1:]
    for k in range(6):
        assert np.array_equal(got[:, k], (lrs[k] / (1 - 0.9 ** steps)).astype(F)), k
        assert np.array_equal(got[:, 6 + k], np.sqrt(1 - 0.999 ** steps).astype(F)), k
    want = np.array([SR.exposure_bias(exp_lr, 0.9, 0.999, t) for t in range(1, T + 1)], F)
    assert np.array_equal(got[:, 13], want[:, 0]) and np.array_equal(got[:, 14], want[:, 1])


# ---- the graphed whole iteration against the exact path -----------------------------------------------------------------
W, H, N, SKY, SCAFFOLD, NIMG = 320, 240, 20_000, 300, 600, 5
EXTENT = 30.0


def _params(seed=7):
    import torch
    cam = synth.make_camera(W, H)
    c = synth.cloud_v1(N, cam, sh_degree=3, zmin=2.0, zmax=30.0, seed=seed, scale_k=3e-3)
    t = lambda a: torch.tensor(np.asarray(a, F), device="cuda")
    op = c["opacities"].astype(np.float64)
    params = [t(c["means3D"]), t(c["shs"][:, :1]), t(c["shs"][:, 1:]), t(np.log(op / (1 - op))), t(np.log(c["scales"])),
              t(c["rotations"])]
    params[4][SCAFFOLD:SCAFFOLD + 40] = float(np.log(0.7))      # a few big Gaussians past the scaffold (0.7 > 30 * 0.02)
    g = torch.Generator(device="cuda").manual_seed(seed)
    exposure = torch.eye(3, 4, device="cuda").repeat(NIMG, 1, 1) + 0.02 * torch.randn((NIMG, 3, 4), device="cuda", generator=g)
    return cam, params, exposure


def _new_state(params, exposure):
    from h3dgs.singlestep import SingleState
    lrs = [1.6e-4, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]
    return SingleState(params, SKY, lrs, exposure, skybox_locked=True, scaffold_points=SCAFFOLD)


def _pair(capture=True, **kw):
    from h3dgs.pipeline import DeviceCamera
    from h3dgs.singlestep import GraphedSingleStep
    cam, params, exposure = _params()
    sa, sb = _new_state(params, exposure), _new_state(params, exposure)
    sca, scb = sa.make_scene(), sb.make_scene(requires_grad=False)
    dcam = DeviceCamera(cam)
    gs = GraphedSingleStep(scb, W, H, cam.tanfovx, cam.tanfovy, mask=True, sh_degree=1, capture=False, state=sb,
                           cameras_extent=EXTENT, **kw)
    gs.set_camera(dcam)
    if capture:
        gs.capture()
    return cam, dcam, (sa, sca), (sb, scb), gs


def _targets(k):
    import torch
    g = torch.Generator(device="cuda").manual_seed(100 + k)
    gt = torch.rand((3, H, W), device="cuda", generator=g)
    mask = (torch.rand((1, H, W), device="cuda", generator=g) > 0.2).float()
    mono = torch.rand((1, H, W), device="cuda", generator=g) * 0.5
    dmask = (torch.rand((1, H, W), device="cuda", generator=g) > 0.1).float()
    bg = torch.rand(3, device="cuda", generator=g)
    return gt, mask, mono, dmask, bg


def _lrs(it):
    return 1.6e-4 * 0.99 ** it, 1e-3 * (0.5 + 0.01 * it)


def _everything(s, scene):
    return (s.params + s.exp_avg + s.exp_avg_sq + [s.step, s.exposure, s.exposure_exp_avg, s.exposure_exp_avg_sq,
                                                  s.exposure_step, s.stats.max_radii2D, s.stats.xyz_gradient_accum,
                                                  s.stats.denom] + [getattr(scene, k) for k in NAMES])


def _exact(sa, sca, dcam, it, update=True):
    from h3dgs.pipeline import single_step
    gt, mask, mono, dmask, bg = _targets(it)
    sa.set_learning_rates(*_lrs(it))
    sa.set_image(it % NIMG)
    return single_step(sca, dcam, bg, gt, 0.2, None, mask, mono, dmask, 0.3, sa.stats, 1, state=sa, cameras_extent=EXTENT,
                       update=update)


def test_thirty_iterations_graphed_track_the_exact_path():
    import torch
    cam, dcam, (sa, sca), (sb, scb), gs = _pair()
    side = torch.cuda.Stream()
    losses = []
    for it in range(30):
        gt, mask, mono, dmask, bg = _targets(it)
        out, radii, _ = _exact(sa, sca, dcam, it)
        ev = gs.upload_target(gt, side, mask, mono, dmask)
        sb.set_learning_rates(*_lrs(it))
        gs.step(bg=bg, depth_weight=0.3, gt_ready=ev, image=it % NIMG)
        s = gs.status()
        assert not s["overflow"]
        if it == 0:
            # the same rows and exposure: the same kernels give the exact path's loss and radii bit for bit; later the
            # states differ by the order of the backward's atomic sums
            assert np.float32(s["loss"]) == np.float32(float(out[0])) and torch.equal(radii, gs.radii)
        else:
            assert abs(s["loss"] - float(out[0])) <= 1e-4 * abs(float(out[0])), it
        losses.append(s["loss"])
    torch.cuda.synchronize()
    # gradients differ in the order of the backward's atomic sums (~1e-7 relative).  Adam normalises the update, so an
    # element whose gradient is tiny (a cancelling sum) can move by a different amount, up to a whole step: |m| /
    # (sqrt(v) / bc2_sqrt) <= (1 - b1) / sqrt(1 - b2) / bc1 ~ 3.2 at most, times lr, per iteration.  So: every
    # parameter within that bound over the 30 steps, and almost every element close
    def close(a, b, lr, what):
        d = (a - b).abs()
        assert float(d.max()) <= 30 * 3.2 * lr, (what, float(d.max()))
        near = d <= 1e-3 * b.abs() + 1e-5
        assert float(near.float().mean()) >= 0.995, (what, float(near.float().mean()))
    lr0 = _lrs(0)
    for k in range(6):
        close(sa.params[k], sb.params[k], lr0[0] if k == 0 else sa.lr[k], CR.GROUPS[k])
    close(sa.exposure, sb.exposure, _lrs(29)[1], "exposure")                # the largest exposure lr of the run
    assert int(sa.step.item()) == int(sb.step.item()) == 30 and int(sb.exposure_step.item()) == 30
    assert torch.equal(sa.stats.max_radii2D, sb.stats.max_radii2D) and torch.equal(sa.stats.denom, sb.stats.denom)
    assert losses[-1] < losses[0]


def _copy_state(dst, dst_scene, src, src_scene):
    import torch
    with torch.no_grad():
        for a, b in zip(dst.params + dst.exp_avg + dst.exp_avg_sq, src.params + src.exp_avg + src.exp_avg_sq):
            a.copy_(b)
        for a, b in ((dst.step, src.step), (dst.exposure, src.exposure), (dst.exposure_exp_avg, src.exposure_exp_avg),
                     (dst.exposure_exp_avg_sq, src.exposure_exp_avg_sq), (dst.exposure_step, src.exposure_step),
                     (dst.stats.max_radii2D, src.stats.max_radii2D), (dst.stats.xyz_gradient_accum, src.stats.xyz_gradient_accum),
                     (dst.stats.denom, src.stats.denom)):
            a.copy_(b)
        for k in NAMES:
            getattr(dst_scene, k).copy_(getattr(src_scene, k))


def test_each_graphed_iteration_is_the_exact_one_from_the_same_state():
    """30 iterations, the exact path restarted each time from the graphed state, so that only one step's atomic-sum order
    separates them: the gathered exposure row is the state's row of the iteration's image bit for bit, image, loss and
    radii bit for bit, the rows OurAdam stepped are the same rows, both step counts equal, and every parameter within
    the one step Adam's normalisation allows an element with a cancelling gradient (3.2 lr) while almost all agree"""
    import torch
    from h3dgs.pipeline import single_step
    cam, dcam, (sa, sca), (sb, scb), gs = _pair()
    side = torch.cuda.Stream()
    for it in range(30):
        image = (3 * it + 1) % NIMG
        _copy_state(sa, sca, sb, scb)
        pre = sb.exposure[image].clone()
        m0 = [m.clone() for m in sb.exp_avg]
        gt, mask, mono, dmask, bg = _targets(it)
        sa.set_learning_rates(*_lrs(it))
        sa.set_image(image)
        out, radii, _ = single_step(sca, dcam, bg, gt, 0.2, None, mask, mono, dmask, 0.3, sa.stats, 1, state=sa,
                                    cameras_extent=EXTENT)
        ev = gs.upload_target(gt, side, mask, mono, dmask)
        sb.set_learning_rates(*_lrs(it))
        gs.step(bg=bg, depth_weight=0.3, gt_ready=ev, image=image)
        s = gs.status()
        assert not s["overflow"]
        assert torch.equal(gs.exposure.view(torch.int32), pre.view(torch.int32)), it
        assert np.float32(s["loss"]) == np.float32(float(out[0])) and torch.equal(radii, gs.radii), it
        torch.cuda.synchronize()
        assert int(sa.step.item()) == int(sb.step.item()) and int(sa.exposure_step.item()) == int(sb.exposure_step.item())
        assert torch.allclose(sa.exposure, sb.exposure, rtol=1e-6, atol=1e-9), (it, float((sa.exposure - sb.exposure).abs().max()))
        stepped_a = torch.any((sa.exp_avg[3] != m0[3]).reshape(N, -1), dim=1)
        stepped_b = torch.any((sb.exp_avg[3] != m0[3]).reshape(N, -1), dim=1)
        assert int((stepped_a != stepped_b).sum()) <= N // 10_000 + 1, it        # a relevance flip at atomic-noise level
        for k in range(6):
            lr = _lrs(it)[0] if k == 0 else sa.lr[k]
            d = (sa.params[k] - sb.params[k]).abs()
            assert float(d.max()) <= 3.2 * lr, (it, CR.GROUPS[k], float(d.max()))
            # almost every element agrees to 1e-5: the exceptions are elements whose stored gradient cancels (most of
            # them in the rotation group, whose gradient is F.normalize's backward: 99.88 % agreed in one step on the H100)
            near = d <= 1e-5 * sb.params[k].abs() + 1e-7
            assert float(near.float().mean()) >= 0.995, (it, CR.GROUPS[k], float(near.float().mean()))


def test_first_iteration_image_is_exact():
    import torch
    from h3dgs.pipeline import render_flat
    cam, dcam, (sa, sca), (sb, scb), gs = _pair()
    gt, mask, mono, dmask, bg = _targets(0)
    with torch.no_grad():
        img, radii, inv = render_flat(sca, dcam, bg, 1, do_depth=True)
    sb.set_learning_rates(*_lrs(0))
    gs.step(gt=gt, mask=mask, mono_invdepth=mono, depth_mask=dmask, bg=bg, depth_weight=0.3, image=2)
    torch.cuda.synchronize()
    assert torch.equal(img.view(torch.int32), gs.image.view(torch.int32)) and torch.equal(radii, gs.radii)
    assert torch.equal(gs.exposure, sa.exposure[2])                    # the forward's exposure is the image's row


def test_capture_warm_up_changes_no_state():
    import torch
    cam, dcam, (sa, sca), (sb, scb), gs = _pair(capture=False)
    before = [t.clone() for t in _everything(sb, scb)]
    gs.capture()
    torch.cuda.synchronize()
    for a, b in zip(before, _everything(sb, scb)):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def test_overflowed_frame_changes_nothing_and_the_exact_rerun_does():
    import torch
    cam, dcam, (sa, sca), (sb, scb), gs = _pair(bin_capacity=64)
    gt, mask, mono, dmask, bg = _targets(2)
    before = [t.clone() for t in _everything(sb, scb)]
    gs.step(gt=gt, mask=mask, mono_invdepth=mono, depth_mask=dmask, bg=bg, depth_weight=0.3, image=1)
    assert gs.status()["overflow"]
    for a, b in zip(before, _everything(sb, scb)):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
    for k in NAMES:
        getattr(scb, k).requires_grad_(True)
    _exact(sb, scb, dcam, 2)
    assert int(sb.step.item()) == 1 and int(sb.exposure_step.item()) == 1
    assert not torch.equal(sb.params[3], before[3]) and not torch.equal(sb.exposure, before[19])


def _model_of(state):
    """a GaussianModel-shaped object with OurAdam-shaped groups and a torch.optim.Adam on the exposures"""
    import torch
    from h3dgs.optim import Adam
    attrs = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")
    model = types.SimpleNamespace(skybox_points=state.skybox_points, skybox_locked=state.skybox_locked,
                                  scaffold_points=state.scaffold_points)
    for a, p in zip(attrs, state.params):
        setattr(model, a, torch.nn.Parameter(torch.zeros_like(p)))
    model.optimizer = Adam([{"params": [getattr(model, a)], "lr": lr, "name": n} for a, lr, n in
                            zip(attrs, state.lr, CR.GROUPS)], lr=0.0, eps=1e-15)
    model._exposure = torch.nn.Parameter(torch.zeros_like(state.exposure))
    model.exposure_optimizer = torch.optim.Adam([model._exposure])
    return model


def test_state_survives_a_row_count_change_across_a_hand_over():
    """densify_and_prune's way: rows gathered (pruned) and appended (cloned) with their moments gathered and zero
    moments appended, step counts kept; then a new graphed step on the new state, handed the statistics"""
    import torch
    from h3dgs.singlestep import GraphedSingleStep, SingleState
    cam, dcam, (sa, sca), (sb, scb), gs = _pair()
    for it in range(3):
        gt, mask, mono, dmask, bg = _targets(it)
        sb.set_learning_rates(*_lrs(it))
        gs.step(gt=gt, mask=mask, mono_invdepth=mono, depth_mask=dmask, bg=bg, depth_weight=0.3, image=it % NIMG)
    model = _model_of(sb)
    sb.copy_to_model(model)
    keep = torch.ones(N, dtype=torch.bool, device="cuda")
    keep[SCAFFOLD + 100:SCAFFOLD + 400] = False
    clone = torch.arange(SCAFFOLD + 1000, SCAFFOLD + 1500, device="cuda")
    opt = model.optimizer
    with torch.no_grad():
        for g in opt.param_groups:
            p = g["params"][0]
            s = opt.state[p]
            newp = torch.nn.Parameter(torch.cat((p[keep], p[clone])))
            s2 = dict(step=s["step"], exp_avg=torch.cat((s["exp_avg"][keep], torch.zeros_like(p[clone]))),
                      exp_avg_sq=torch.cat((s["exp_avg_sq"][keep], torch.zeros_like(p[clone]))))
            del opt.state[p]
            g["params"][0] = newp
            opt.state[newp] = s2
        for a, n in zip(("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation"), CR.GROUPS):
            setattr(model, a, {g["name"]: g["params"][0] for g in opt.param_groups}[n])
        N2 = int(keep.sum()) + clone.shape[0]
        model.xyz_gradient_accum = torch.zeros((N2, 1), device="cuda")
        model.denom = torch.zeros((N2, 1), device="cuda")
        model.max_radii2D = torch.cat((model.max_radii2D[keep], torch.zeros(clone.shape[0], device="cuda")))
    s2 = SingleState.from_model(model)
    assert s2.N == N2 and int(s2.step.item()) == 3 and int(s2.exposure_step.item()) == 3
    assert torch.equal(s2.exposure, sb.exposure) and torch.equal(s2.exposure_exp_avg, sb.exposure_exp_avg)
    assert torch.equal(s2.params[3][:int(keep.sum())], sb.params[3][keep])
    assert torch.equal(s2.stats.max_radii2D, model.max_radii2D)
    sc2 = s2.make_scene(requires_grad=False)
    s2.set_learning_rates(*_lrs(3))
    s2.set_image(0)
    s2.no_gaussian_step(sc2, EXTENT, gs.exposure_grad)      # the densify iteration's exposure step and rescale
    g2 = GraphedSingleStep(sc2, W, H, cam.tanfovx, cam.tanfovy, mask=True, sh_degree=1, capture=False, state=s2,
                           cameras_extent=EXTENT)
    g2.set_camera(dcam)
    g2.capture()
    for it in range(4, 7):
        gt, mask, mono, dmask, bg = _targets(it)
        s2.set_learning_rates(*_lrs(it))
        g2.step(gt=gt, mask=mask, mono_invdepth=mono, depth_mask=dmask, bg=bg, depth_weight=0.3, image=it % NIMG)
    torch.cuda.synchronize()
    assert not g2.status()["overflow"]
    assert int(s2.step.item()) == 6 and int(s2.exposure_step.item()) == 7
    # appended rows start from zero moments and move
    assert torch.count_nonzero(s2.exp_avg[3][-clone.shape[0]:]) > 0
    # the round trip back into the model and out again
    m2 = _model_of(s2)
    s2.copy_to_model(m2)
    back = SingleState.from_model(m2)
    for k in range(6):
        assert torch.equal(back.params[k], s2.params[k]) and torch.equal(back.exp_avg[k], s2.exp_avg[k])
    assert torch.equal(back.exposure_exp_avg_sq, s2.exposure_exp_avg_sq) and int(back.exposure_step.item()) == 7
    assert torch.equal(back.stats.denom, s2.stats.denom) and torch.equal(back.stats.xyz_gradient_accum, s2.stats.xyz_gradient_accum)


# ---- against the reference's own GaussianModel, OurAdam, exposure_optimizer and render() (tests/golden/single_train.npz)
@pytest.mark.parametrize("c", range(6))
def test_param_step_is_the_reference_iteration(golden_dir, c):
    import torch
    z = np.load(os.path.join(golden_dir, "single_train.npz"))
    st = SR.golden_start(z, c)
    image, xyz_lr, exp_lr, eg, gstep, thr = SR.golden_frame(z, c)
    state = _state_from(st)
    scene = state.make_scene(requires_grad=False)
    state.set_learning_rates(xyz_lr, exp_lr)
    state.set_image(image)
    extent = float(z["extent"])
    if gstep:
        act, grads = CR.golden_inputs(z, c)
        for k in NAMES:                                   # the reference's activated rows are what the forward read
            getattr(scene, k).copy_(act[k].reshape(getattr(scene, k).shape))
        state.param_step(scene, {k: v.cuda().contiguous() for k, v in grads.items()}, extent, torch.tensor(eg, device="cuda"))
    else:
        state.no_gaussian_step(scene, extent, torch.tensor(eg, device="cuda"))
    torch.cuda.synchronize()
    assert int(state.step.item()) == int(z[f"c{c}_step"]) and int(state.exposure_step.item()) == int(z[f"c{c}_exposure_step"])
    # the rows placed one ulp around the rescale threshold were placed with the CPU's exp; on the device the decision is
    # the device expf's, checked against torch's CUDA exp
    edges = [int(r) for r in z["edges"]]
    sa = torch.tensor(z[f"c{c}_adam_scaling"], device="cuda")[edges]
    viol = (torch.exp(sa).max(dim=1).values > float(np.float32(extent * 0.02))).cpu().numpy()
    moved = (state.params[4][edges].cpu().numpy() != z[f"c{c}_adam_scaling"][edges]).any(axis=1)
    assert np.array_equal(viol, moved)
    p, m, v = ([x.cpu().numpy() for x in xs] for xs in (state.params, state.exp_avg, state.exp_avg_sq))
    if gstep:
        bad = CR.golden_violations(z, c, st, p, m, v, skip_rows=edges)
    else:
        bad = SR.golden_no_step_violations(z, c, st, p, m, v, skip_rows=edges)
    bad += SR.golden_exposure_violations(z, c, st, state.exposure.cpu().numpy(), state.exposure_exp_avg.cpu().numpy(),
                                         state.exposure_exp_avg_sq.cpu().numpy())
    assert not bad, bad


def test_a_dropped_step_is_freed_without_the_cycle_collector():
    """no reference cycle keeps a graphed step alive: dropped, it is freed at once, not whenever Python's cycle
    collector next runs (perhaps in the middle of another instance's capture)"""
    import gc
    import weakref
    import torch
    cam, dcam, (sa, sca), (sb, scb), gs = _pair()                     # constructed and captured
    torch.cuda.synchronize()
    ref = weakref.ref(gs)
    enabled = gc.isenabled()
    gc.disable()
    try:
        del gs
        assert ref() is None
    finally:
        if enabled:
            gc.enable()

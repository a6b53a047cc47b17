"""GPU: train_post's parameter step on the device (csrc/post_param.cu, h3dgs.poststep.PostState, the state path of
GraphedPostStep and pipeline.post_step).

  * given identical activated gradients, the step against tests/post_train_ref.py: stored rows, moments and the step
    count bit for bit, except F.normalize's backward and forward;
  * the six groups equal torch.optim.Adam on the same GPU bit for bit over 100 steps (rotation within the normalize's
    ulps), fed the stored gradients torch's autograd forms through abs / exp / normalize / cat and the lock lines of
    train_post.py:167-181, with a changing xyz lr; the state handed to that optimizer by copy_to_model and taken back by
    from_model;
  * against the reference's own create_from_hier model, torch.optim.Adam, render_post and train_post lines
    (tests/golden/post_train.npz): the kernel on the device within post_train_ref.golden_violations' budget;
  * the bias corrections of steps 1..30 000 equal the host's doubles rounded to fp32;
  * the graphed whole iteration against the exact path over 30 iterations, and each graphed iteration against the exact
    one from the same state; capture's warm-up, a binning overflow and a row overflow change no state byte, and the
    exact re-run of an overflowed frame steps."""
import os
import sys
import types

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import coarse_ref as CR  # noqa: E402
import post_train_ref as PR  # noqa: E402
import single_train_ref as SR  # noqa: E402
from h3dgs import synth  # noqa: E402

pytestmark = pytest.mark.gpu
F = np.float32
NAMES = ("means3D", "shs", "opacities", "scales", "rotations")
ATTRS = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")


def ulps(a, b):
    a, b = np.asarray(a, F).ravel(), np.asarray(b, F).ravel()
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    d = np.abs(ia - ib)
    d[np.isnan(a) & np.isnan(b)] = 0
    return d


def _nodes(N):
    import torch
    return torch.zeros((N, 2), dtype=torch.int32), torch.zeros((N, 2, 4))


def _state_from(st, locked_sky=True, anchors=None):
    from h3dgs.poststep import PostState
    mv = lambda xs: [x.cuda() for x in xs]
    return PostState(mv(st["params"]), st["skybox"], st["lr"], *_nodes(st["params"][0].shape[0]), st["betas"], st["eps"],
                     mv(st["exp_avg"]), mv(st["exp_avg_sq"]), st["step"], skybox_locked=locked_sky, anchors=anchors)


@pytest.mark.parametrize("N,S,anchors,seed", [(1, 0, [], 1), (1000, 100, [5, 5, 999, 12], 2),
                                              (200_000, 5000, [0, 70_000, -1], 3)])
def test_param_step_matches_restatement(N, S, anchors, seed):
    import torch
    st = PR.random_post_state(N, S, seed)
    grads = CR.random_grads(N, seed + 1, K=15)
    if N > 10:
        grads["opacities"][3, 0] = float("nan")
        st["params"][3][4, 0] = float("nan")
    state = _state_from(st, True, anchors)
    scene = state.make_scene(requires_grad=False)
    xyz_lr = 1.1e-4
    state.set_learning_rate(xyz_lr)
    # the activated rows the kernel reads are the device's (its expf)
    act = {k: getattr(scene, k).detach().cpu().clone().reshape(v.shape) for k, v in PR.activate(st["params"]).items()}
    ref = CR.clone_state(st)
    act_ref = PR.param_step(ref, act, grads, xyz_lr, PR.locked_mask(N, S, True, anchors))
    state.param_step(scene, {k: v.cuda().contiguous() for k, v in grads.items()})
    torch.cuda.synchronize()
    assert int(state.step.item()) == ref["step"]
    for k in range(6):
        for name, got, want in (("param", state.params[k], ref["params"][k]), ("exp_avg", state.exp_avg[k], ref["exp_avg"][k]),
                                ("exp_avg_sq", state.exp_avg_sq[k], ref["exp_avg_sq"][k])):
            d = ulps(got.cpu(), want)
            assert d.max() <= (4 if k == 5 else 0), (CR.GROUPS[k], name, int(d.max()))
    for k in NAMES:
        got, want = getattr(scene, k).detach().cpu().reshape(act_ref[k].shape), act_ref[k]
        # scales: the device's expf against torch's CPU exp, each within 1 ulp of the true value
        assert ulps(got, want).max() <= {"rotations": 4, "scales": 2}.get(k, 0), k
    # and against torch's CUDA exp, bit for bit
    assert torch.equal(scene.scales.view(torch.int32), torch.exp(state.params[4]).view(torch.int32))


def _model(state):
    """a create_from_hier-shaped GaussianModel with training_setup(our_adam=False)'s torch.optim.Adam"""
    import torch
    model = types.SimpleNamespace(skybox_points=state.skybox_points, skybox_locked=state.skybox_locked,
                                  anchors=state.anchors.cuda(), nodes=state.nodes, boxes=state.boxes)
    for a, p in zip(ATTRS, state.params):
        setattr(model, a, torch.nn.Parameter(torch.zeros_like(p)))
    model.optimizer = torch.optim.Adam([{"params": [getattr(model, a)], "lr": lr, "name": n} for a, lr, n in
                                        zip(ATTRS, state.lr, CR.GROUPS)], lr=0.0, eps=1e-15)
    return model


def _reference_step(model, G, xyz_lr):
    """train_post.py:85 and 165-192 on the model: autograd through get_xyz / get_features / abs / exp / F.normalize from
    the activated gradients G, the lock lines, optimizer.step()"""
    import torch
    import torch.nn.functional as Fn
    for g in model.optimizer.param_groups:
        if g["name"] == "xyz":
            g["lr"] = xyz_lr
    act = dict(means3D=model._xyz, shs=torch.cat((model._features_dc, model._features_rest), 1),
               opacities=torch.abs(model._opacity), scales=torch.exp(model._scaling), rotations=Fn.normalize(model._rotation))
    torch.autograd.backward([act[k] for k in NAMES], [G[k] for k in NAMES])
    S = model.skybox_points
    with torch.no_grad():
        params = [getattr(model, a) for a in ATTRS]
        if S != 0 and model.skybox_locked:
            for p in params:
                p.grad[-S:] = 0
        for p in params:
            p.grad[model.anchors] = 0
    model.optimizer.step()
    model.optimizer.zero_grad(set_to_none=True)


def test_six_groups_are_torch_adam_and_the_model_round_trip():
    """copy_to_model hands the state (mid-training moments, step 7) to the reference's torch.optim.Adam; 100 steps of
    that optimizer fed the stored gradients autograd forms, against the kernel fed the activated ones: every group
    but the rotation bit for bit each step; the rotation (F.normalize's backward, a different reduction) re-synchronised
    each step after agreeing to the absolute bounds below, 99 % of its elements within 16 ulp (on the H100 0.4 % of the
    moments were further off: elements whose gradient cancels).  from_model takes the state back unchanged."""
    import torch
    from h3dgs.poststep import PostState
    N, S = 5000, 300
    st = PR.random_post_state(N, S, 21)
    anchors = [3, 3, 4000, N - 1, 17]
    st["params"][3][20, 0] = float("nan")            # a NaN stored opacity: CUDA's sign(NaN) in abs's backward
    state = _state_from(st, True, anchors)
    scene = state.make_scene(requires_grad=False)
    model = _model(state)
    state.copy_to_model(model)
    g = torch.Generator(device="cuda").manual_seed(5)
    for it in range(100):
        G = {k: 1e-2 * torch.randn(getattr(scene, k).shape, device="cuda", generator=g) for k in NAMES}
        off = torch.rand(N, device="cuda", generator=g) < 0.4                    # rows outside the frame's cut
        for v in G.values():
            v[off] = 0
        if it == 50:
            G["opacities"].zero_()
        if it == 60:
            G["opacities"][21, 0] = float("nan")      # a NaN gradient on a finite stored opacity
        xyz_lr = 1.6e-4 * 0.99 ** it
        _reference_step(model, G, xyz_lr)
        state.set_learning_rate(xyz_lr)
        state.param_step(scene, G)
        torch.cuda.synchronize()
        opt = model.optimizer
        for k, a in enumerate(ATTRS):
            p = getattr(model, a)
            s = opt.state[p]
            for what, got, want, tol in (("param", state.params[k], p.detach(), 3.2 * state.lr[5]),
                                         ("exp_avg", state.exp_avg[k], s["exp_avg"], 1e-8),
                                         ("exp_avg_sq", state.exp_avg_sq[k], s["exp_avg_sq"], 1e-12)):
                d = ulps(got.cpu(), want.cpu())
                if k != 5:
                    assert d.max() == 0, (it, CR.GROUPS[k], what, int(d.max()))
                else:
                    # F.normalize's backward in another reduction order: a few ulp of the gradient, more where it
                    # cancels; Adam normalises the update, so a cancelling element can move by up to a step
                    over = (got - want).abs() - (tol + 2.0 ** -21 * want.abs())       # the bound plus 4 ulp of the value
                    assert float(over.max()) <= 0, (it, what, float(over.max()))
                    assert float((d <= 16).mean()) >= 0.99, (it, what, float((d <= 16).mean()))
            if k == 5:
                with torch.no_grad():
                    p.copy_(state.params[5])
                    s["exp_avg"].copy_(state.exp_avg[5])
                    s["exp_avg_sq"].copy_(state.exp_avg_sq[5])
            assert int(float(s["step"])) == int(state.step.item())
        # the activated rows the next forward reads are the reference's get_* of the stored tensors
        assert ulps(scene.opacities.cpu(), torch.abs(model._opacity).detach().cpu()).max() == 0
        assert ulps(scene.scales.cpu(), torch.exp(model._scaling).detach().cpu()).max() == 0
    assert bool(torch.isnan(state.params[3][20]).all()) and bool(torch.isnan(state.params[3][21]).all())
    back = PostState.from_model(model)
    assert int(back.step.item()) == int(state.step.item()) == 107
    for k in range(6):
        for a, b in ((back.params[k], state.params[k]), (back.exp_avg[k], state.exp_avg[k]),
                     (back.exp_avg_sq[k], state.exp_avg_sq[k])):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), k          # NaN rows included
    assert torch.equal(back.locked, state.locked)


def test_from_model_refuses_another_optimizer():
    import torch
    from h3dgs.optim import Adam
    from h3dgs.poststep import PostState
    st = PR.random_post_state(10, 0, 1)
    model = _model(_state_from(st))
    model.optimizer = Adam([{"params": [getattr(model, a)], "lr": 0.0, "name": n} for a, n in zip(ATTRS, CR.GROUPS)],
                           lr=0.0, eps=1e-15)
    with pytest.raises(ValueError):
        PostState.from_model(model)
    model = _model(_state_from(st))
    model.optimizer.param_groups[0]["amsgrad"] = True
    with pytest.raises(ValueError):
        PostState.from_model(model)
    assert torch.cuda.is_available()


def test_bias_corrections_of_30000_steps_are_the_host_doubles():
    import ctypes as C
    import torch
    from h3dgs import _lib
    st = PR.random_post_state(4, 0, 5)
    state = _state_from(st)
    scene = state.make_scene(requires_grad=False)
    xyz_lr = 1.6e-5
    state.set_learning_rate(xyz_lr)
    args = state._post_args(scene)
    T = 30_000
    out = torch.empty((T, 12), dtype=torch.int32, device="cuda")
    L = _lib.lib()
    s = torch.cuda.current_stream().cuda_stream
    for t in range(T):
        state.step.fill_(t)
        _lib.check(L.h3dgs_post_param_step(C.byref(args), _lib.POST_BIAS, s))
        out[t].copy_(state.scratch.view(torch.int32)[:12])
    got = out.cpu().numpy().view(F)
    lrs = [xyz_lr] + st["lr"][1:]
    for k in range(6):
        want = np.array([SR.exposure_bias(lrs[k], 0.9, 0.999, t) for t in range(1, T + 1)], F)
        assert np.array_equal(got[:, k], want[:, 0]) and np.array_equal(got[:, 6 + k], want[:, 1]), k


# ---- the graphed whole iteration against the exact path -----------------------------------------------------------------
SKY = 200
ANCHORS = [10, 10, 500, -1]


def _hier():
    cam = synth.make_camera(480, 270)
    lv = synth.cloud_v1(9000, cam, zmin=2.0, zmax=40.0, seed=3, scale_k=1.0)
    z = lv["means3D"][:, 2:3]
    lv["scales"] = (4e-3 * np.sqrt(2.0 * z) * np.exp(0.4 * np.random.default_rng(1).standard_normal((z.shape[0], 3)))).astype(F)
    return cam, synth.append_skybox(synth.build_hierarchy(lv), SKY)


def _new_state(h):
    import torch
    from h3dgs.poststep import PostState
    t = lambda a: torch.tensor(np.asarray(a, F), device="cuda")
    op = np.asarray(h["opacities"], F).copy()
    op[::7] *= -1                                                    # stored opacities of both signs: abs folds them
    params = [t(h["means3D"]), t(h["shs"][:, :1]), t(h["shs"][:, 1:]), t(op), t(np.log(h["scales"])), t(h["rotations"])]
    return PostState(params, SKY, PR.LRS, torch.tensor(h["nodes"]), torch.tensor(h["boxes"]), skybox_locked=True,
                     anchors=ANCHORS)


def _frame(cam, it):
    import torch
    rs = np.random.default_rng(300 + it)
    c = cam if it % 3 == 0 else synth.yaw_camera(cam.W, cam.H, float(rs.uniform(-15, 15)), rs.uniform(-0.5, 0.5, 3))
    g = torch.Generator(device="cuda").manual_seed(100 + it)
    gt = torch.rand((3, cam.H, cam.W), device="cuda", generator=g)
    mask = (torch.rand((1, cam.H, cam.W), device="cuda", generator=g) > 0.2).float()
    ex = None if it % 4 == 3 else torch.eye(3, 4, device="cuda") + 0.02 * torch.randn((3, 4), device="cuda", generator=g)
    # train_post.py:73-74: limit = 2^(u (log2 0.1 - log2 0.005) + log2 0.005)
    thr = 2.0 ** (float(rs.uniform()) * (np.log2(0.1) - np.log2(0.005)) + np.log2(0.005))
    return c, gt, mask, ex, thr


def _lr(it):
    return 1.6e-4 * 0.99 ** it


def _pair(capture=True, **kw):
    import torch
    from h3dgs.poststep import GraphedPostStep
    cam, h = _hier()
    sa, sb = _new_state(h), _new_state(h)
    sca, scb = sa.make_scene(), sb.make_scene(requires_grad=False)
    bg = torch.tensor([0.2, 0.1, 0.3], device="cuda")
    gs = GraphedPostStep(scb, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, 0.01, exposure=True, mask=True,
                         bin_capacity=kw.pop("bin_capacity", 1 << 21), capture=False, state=sb, **kw)
    from h3dgs.pipeline import DeviceCamera
    gs.set_camera(DeviceCamera(cam))
    if capture:
        gs.capture()
    return cam, bg, (sa, sca), (sb, scb), gs


def _everything(s, scene):
    return s.params + s.exp_avg + s.exp_avg_sq + [s.step] + [getattr(scene, k) for k in NAMES]


def _exact(s, scene, bg, cam, it, update=True):
    from h3dgs import pipeline
    c, gt, mask, ex, thr = _frame(cam, it)
    s.set_learning_rate(_lr(it))
    return pipeline.post_step(scene, pipeline.DeviceCamera(c), bg, gt, thr, 0.2, ex, mask, state=s, update=update)


def _graphed(s, gs, cam, it, side=None):
    from h3dgs import pipeline
    c, gt, mask, ex, thr = _frame(cam, it)
    s.set_learning_rate(_lr(it))
    gs.set_threshold(thr)
    if side is None:
        gs.step(pipeline.DeviceCamera(c), gt, mask=mask, exposure=ex)
    else:
        ev = gs.upload_target(gt, side, mask=mask)
        gs.step(pipeline.DeviceCamera(c), exposure=ex, gt_ready=ev)
    return gs.status()


def test_thirty_iterations_graphed_track_the_exact_path():
    import torch
    cam, bg, (sa, sca), (sb, scb), gs = _pair()
    side = torch.cuda.Stream()
    for it in range(30):
        (loss, _, _), radii, n = _exact(sa, sca, bg, cam, it)
        s = _graphed(sb, gs, cam, it, side if it % 2 else None)
        assert not s["overflow"], it
        if it == 0:
            assert np.float32(s["loss"]) == np.float32(float(loss)) and s["rows"] == n + SKY
            assert torch.equal(gs.radii[:n + SKY], radii)
        else:
            assert abs(s["loss"] - float(loss)) <= 1e-4 * abs(float(loss)), it
    torch.cuda.synchronize()
    assert int(sa.step.item()) == int(sb.step.item()) == 30
    # every row moved (the dense step), the locked ones on their moments alone
    for k in range(6):
        lr = _lr(0) if k == 0 else sa.lr[k]
        d = (sa.params[k] - sb.params[k]).abs()
        assert float(d.max()) <= 30 * 3.2 * lr, (CR.GROUPS[k], float(d.max()))
        near = d <= 1e-3 * sb.params[k].abs() + 1e-5
        assert float(near.float().mean()) >= 0.995, (CR.GROUPS[k], float(near.float().mean()))


def _copy_state(dst, dst_scene, src, src_scene):
    import torch
    with torch.no_grad():
        for a, b in zip(_everything(dst, dst_scene), _everything(src, src_scene)):
            a.copy_(b)


def test_each_graphed_iteration_is_the_exact_one_from_the_same_state():
    import torch
    cam, bg, (sa, sca), (sb, scb), gs = _pair()
    for it in range(12):
        _copy_state(sa, sca, sb, scb)
        before = [p.clone() for p in sb.params]
        (loss, _, _), radii, n = _exact(sa, sca, bg, cam, it)
        s = _graphed(sb, gs, cam, it)
        assert not s["overflow"]
        assert np.float32(s["loss"]) == np.float32(float(loss)) and torch.equal(gs.radii[:n + SKY], radii), it
        torch.cuda.synchronize()
        assert int(sa.step.item()) == int(sb.step.item()) == it + 1
        for k in range(6):
            lr = _lr(it) if k == 0 else sa.lr[k]
            d = (sa.params[k] - sb.params[k]).abs()
            assert float(d.max()) <= 3.2 * lr, (it, CR.GROUPS[k], float(d.max()))
            near = d <= 1e-5 * sb.params[k].abs() + 1e-7
            assert float(near.float().mean()) >= 0.995, (it, CR.GROUPS[k], float(near.float().mean()))
            assert bool((sb.params[k] != before[k]).any())
        # the locked rows (anchors, skybox) moved exactly as in the exact path: by their moments alone
        lk = sb.locked.bool()
        for k in range(6):
            assert torch.equal(sa.params[k][lk], sb.params[k][lk]), (it, CR.GROUPS[k])


def test_capture_warm_up_changes_no_state():
    import torch
    cam, bg, (sa, sca), (sb, scb), gs = _pair(capture=False)
    before = [t.clone() for t in _everything(sb, scb)]
    gs.capture()
    torch.cuda.synchronize()
    for a, b in zip(before, _everything(sb, scb)):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


@pytest.mark.parametrize("kind", ["bin", "rows"])
def test_overflowed_frame_changes_nothing_and_the_exact_rerun_steps(kind):
    import torch
    kw = dict(bin_capacity=64) if kind == "bin" else dict(row_capacity=SKY + 50)
    cam, bg, (sa, sca), (sb, scb), gs = _pair(**kw)
    before = [t.clone() for t in _everything(sb, scb)]
    s = _graphed(sb, gs, cam, 0)
    assert s["overflow"]
    if kind == "rows":
        # a row overflow is seen by the status kernel only: the frame rendered its first rows and has gradients
        assert s["rows"] > SKY + 50 and any(float(g.abs().sum()) > 0 for g in gs.grads.values())
    torch.cuda.synchronize()
    for a, b in zip(before, _everything(sb, scb)):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
    for k in NAMES:
        getattr(scb, k).requires_grad_(True)
    _exact(sb, scb, bg, cam, 0)
    torch.cuda.synchronize()
    assert int(sb.step.item()) == 1 and all(not torch.equal(sb.params[k], before[k]) for k in range(6))


# ---- against the reference's own create_from_hier, torch.optim.Adam, render_post and train_post lines ------------------
@pytest.mark.parametrize("c", range(4))
def test_param_step_is_the_reference_iteration(golden_dir, c):
    import torch
    from h3dgs.poststep import PostState
    z = np.load(os.path.join(golden_dir, "post_train.npz"))
    st = PR.golden_start(z, c)
    mv = lambda xs: [x.cuda() for x in xs]
    N = st["params"][0].shape[0]
    state = PostState(mv(st["params"]), st["skybox"], st["lr"], *_nodes(N), st["betas"], st["eps"], mv(st["exp_avg"]),
                      mv(st["exp_avg_sq"]), st["step"], skybox_locked=st["skybox_locked"],
                      anchors=[int(a) for a in z["anchors"]])
    assert torch.equal(state.locked.cpu().bool(), PR.golden_locked(z, c))
    scene = state.make_scene(requires_grad=False)
    act, grads = CR.golden_inputs(z, c)
    for k in NAMES:                                   # the reference's activated rows are what the forward read
        getattr(scene, k).copy_(act[k].reshape(getattr(scene, k).shape))
    state.set_learning_rate(float(z[f"c{c}_xyz_lr"]))
    state.param_step(scene, {k: v.cuda().contiguous() for k, v in grads.items()})
    torch.cuda.synchronize()
    assert int(state.step.item()) == int(z[f"c{c}_step"])
    p, m, v = ([x.cpu().numpy() for x in xs] for xs in (state.params, state.exp_avg, state.exp_avg_sq))
    bad = PR.golden_violations(z, c, st, p, m, v)
    assert not bad, bad

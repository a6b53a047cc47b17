"""GPU: train_post's objective on the device (csrc/loss.cu post-loss kernels, h3dgs.loss.post_loss, pipeline.post_step,
h3dgs.poststep.GraphedPostStep).

  * the kernels per element against tests/post_loss_ref.py's float64 restatement and its fp32 budget, from 1x1 to 1080p
    and at the tile edge +-1, on random, saturated and flat contents, lambda in {0, 0.2, 1}; at the clamp edges; bit for
    bit equal to fused_l1_ssim without exposure and mask; against the reference's own fixture; first call in a capture;
  * the graphed step against the exact path it mirrors, with camera, target, mask, exposure and threshold changing
    between steps and both target slots in use: image and radii bit-identical, status words equal, loss / L1 / SSIM
    within 1e-7, dL/dimage equal (up to the sign of zero), Gaussian gradients equal up to the order of the backward's atomic sums;
  * an overflowed frame, world > 1, and a 40-iteration Adam loop on the graphed and on the eager step."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import post_loss_ref as R  # noqa: E402
import ssim_ref as S  # noqa: E402
from h3dgs import synth  # noqa: E402
from util import rel_err  # noqa: E402

pytestmark = pytest.mark.gpu


def _t(a):
    import torch
    return None if a is None else torch.tensor(a, device="cuda")


def _run(img, gt, lam, Ex, M):
    """post_loss on the device, loss.backward() -> (loss, l1, ssim, grad numpy)"""
    import torch
    from h3dgs.loss import post_loss
    x = torch.tensor(img, device="cuda", requires_grad=True)
    loss, l1, ssim = post_loss(x, _t(gt), lam, _t(Ex), _t(M))
    loss.backward()
    return float(loss), float(l1), float(ssim), x.grad.cpu().numpy()


def _ratio(got, ref, tol):
    d = abs(float(got) - ref)
    return np.inf if not np.isfinite(float(got)) else (0.0 if d == 0 else d / tol)


def _check(img, gt, lam, Ex, M):
    r = R.post_reference(img, gt, lam, Ex, M)
    loss, l1, ssim, grad = _run(img, gt, lam, Ex, M)
    rg, _ = R.compare(grad, r["grad"], r["grad_tol"])
    ratios = dict(grad=rg, loss=_ratio(loss, r["loss"], r["loss_tol"]), l1=_ratio(l1, r["l1"], r["l1_tol"]),
                  ssim=_ratio(ssim, r["ssim"], r["ssim_tol"]))
    print(f"\n{img.shape} lam={lam}: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items()))
    assert np.all(np.isfinite(grad)) and all(v <= 1.0 for v in ratios.values()), ratios
    return r, grad


# ---- the kernels -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 1), (1, 17), (17, 1), (15, 15), (16, 16), (17, 17), (31, 33), (33, 47), (64, 48)])
@pytest.mark.parametrize("content", ["random", "saturated", "flat"])
@pytest.mark.parametrize("em", [("none", "none"), ("on", "binary"), ("offset", "fractional"), ("offset", "half")])
def test_post_loss_within_budget(shape, content, em):
    img, gt, Ex, M = R.make_inputs(*shape, em[0], em[1], content, seed=11)
    _check(img, gt, 0.2, Ex, M)


@pytest.mark.parametrize("lam", [0.0, 0.2, 1.0])
@pytest.mark.parametrize("mask", ["none", "zero", "fractional"])
def test_post_loss_lambdas(lam, mask):
    img, gt, Ex, M = R.make_inputs(45, 70, "offset", mask, seed=12)
    _check(img, gt, lam, Ex, M)


def test_post_loss_full_hd_within_budget():
    img, gt, Ex, M = R.make_inputs(1080, 1920, "offset", "binary", seed=13)
    _check(img, gt, 0.2, Ex, M)


@pytest.mark.parametrize("exposure", R.EXPOSURES)
def test_post_loss_clamp_edges(exposure):
    """y exactly at 0 and 1 and the nearest values either side: a decision other than the restatement's moves the
    gradient by |dL/da|, far outside the budget"""
    img, gt, Ex = R.clamp_edge_inputs(33, 35, exposure, seed=14)
    r, grad = _check(img, gt, 0.2, Ex, None)
    if Ex is None:
        assert np.all(grad[~r["keep"]] == 0.0)


@pytest.mark.parametrize("content", ["in_range", "unclamped"])
def test_without_exposure_and_mask_equals_fused_l1_ssim_bitwise(content):
    import torch
    from h3dgs.loss import fused_l1_ssim, post_loss
    rng = np.random.default_rng(15)
    lo, hi = (0.0, 1.0) if content == "in_range" else (-0.3, 1.3)
    img = torch.tensor(rng.uniform(lo, hi, (3, 270, 480)).astype(np.float32), device="cuda")
    gt = torch.rand((3, 270, 480), device="cuda")
    x1 = img.clone().requires_grad_(True)
    out1 = post_loss(x1, gt, 0.2)
    out1[0].backward()
    x2 = img.clamp(0, 1).requires_grad_(True)
    out2 = fused_l1_ssim(x2, gt, 0.2)
    out2[0].backward()
    for a, b in zip(out1, out2):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    want = torch.where((img >= 0) & (img <= 1), x2.grad, torch.zeros_like(img))
    assert torch.equal(x1.grad.view(torch.int32), want.view(torch.int32))


@pytest.mark.parametrize("i", range(8))
def test_post_loss_matches_the_reference(golden_dir, i):
    z = np.load(os.path.join(golden_dir, "post_loss.npz"))
    exp, _ = (bool(v) for v in z[f"c{i}_flags"])
    raw, gt, M = z[f"c{i}_raw"], z[f"c{i}_gt"], z[f"c{i}_mask"]
    Ex = z[f"c{i}_E"] if exp else None
    loss, l1, _, grad = _run(raw, gt, float(z["lam"]), Ex, M[None])          # the mask as the reference holds it
    assert abs(l1 - float(z[f"c{i}_l1"])) < 1e-6 and abs(loss - float(z[f"c{i}_loss"])) < 1e-6
    ref = z[f"c{i}_grad"]
    assert np.abs(grad - ref).max() <= 1e-5 * max(np.abs(ref).max(), 1e-30)


_CAPTURE = r"""
import sys
import numpy as np
import torch
sys.path[:0] = [sys.argv[2], sys.argv[2] + "/hierarchical-3d-gaussians_b200"]
from h3dgs.loss import post_loss
z = np.load(sys.argv[1])
x = torch.zeros(z["img0"].shape, device="cuda", requires_grad=True)
g = torch.zeros(z["img0"].shape, device="cuda")
E = torch.eye(3, 4, device="cuda")
M = torch.ones(z["img0"].shape[1:], device="cuda")
with torch.no_grad():
    x.copy_(torch.tensor(z["img0"])); g.copy_(torch.tensor(z["gt0"]))
torch.cuda.synchronize()
graph = torch.cuda.CUDAGraph()
with torch.cuda.graph(graph):                       # the first call of the post loss in this process
    loss = post_loss(x, g, 0.2, E, M)[0]
    grad, = torch.autograd.grad(loss, x)
with torch.no_grad():                               # new inputs, exposure and mask between replays
    x.copy_(torch.tensor(z["img"])); g.copy_(torch.tensor(z["gt"])); E.copy_(torch.tensor(z["E"])); M.copy_(torch.tensor(z["M"]))
graph.replay()
torch.cuda.synchronize()
gl, gg = loss.item(), grad.cpu().numpy()
x2 = torch.tensor(z["img"], device="cuda", requires_grad=True)
l2 = post_loss(x2, torch.tensor(z["gt"], device="cuda"), 0.2, torch.tensor(z["E"], device="cuda"), torch.tensor(z["M"], device="cuda"))[0]
l2.backward()
np.savez(sys.argv[1] + ".out.npz", graph_loss=gl, graph_grad=gg, eager_loss=l2.item(), eager_grad=x2.grad.cpu().numpy())
"""


def test_first_call_inside_a_graph_capture(tmp_path):
    img0, gt0, _, _ = R.make_inputs(45, 70, "none", "none", seed=16)
    img, gt, Ex, M = R.make_inputs(45, 70, "offset", "binary", seed=17)
    path = str(tmp_path / "capture.npz")
    np.savez(path, img0=img0, gt0=gt0, img=img, gt=gt, E=Ex, M=M)
    r = subprocess.run([sys.executable, "-c", _CAPTURE, path, ROOT], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    z = np.load(path + ".out.npz")
    assert np.array_equal(z["graph_grad"].view(np.int32), z["eager_grad"].view(np.int32))
    assert abs(float(z["graph_loss"]) - float(z["eager_loss"])) < 1e-7       # double atomics: order differs
    ref = R.post_reference(img, gt, 0.2, Ex, M)
    rg, _ = R.compare(z["graph_grad"], ref["grad"], ref["grad_tol"])
    assert rg <= 1.0 and _ratio(z["graph_loss"], ref["loss"], ref["loss_tol"]) <= 1.0


# ---- the graphed step against the exact path -------------------------------------------------------------------------
def _scene(skybox=0, leaves=9000, W=480, H=270, seed=3):
    cam = synth.make_camera(W, H)
    lv = synth.cloud_v1(leaves, cam, zmin=2.0, zmax=40.0, seed=seed, scale_k=1.0)
    z = lv["means3D"][:, 2:3]
    lv["scales"] = (4e-3 * np.sqrt(2.0 * z) * np.exp(0.4 * np.random.default_rng(1).standard_normal((z.shape[0], 3)))).astype(np.float32)
    h = synth.build_hierarchy(lv)
    if skybox:
        h = synth.append_skybox(h, skybox)
    return cam, h


def _cams(W, H, n=3):
    rs = np.random.default_rng(2)
    return [synth.make_camera(W, H)] + [synth.yaw_camera(W, H, float(rs.uniform(-15, 15)), rs.uniform(-0.5, 0.5, 3))
                                        for _ in range(n - 1)]


def _frame_inputs(H, W, k):
    """target (as the loader leaves it: clamped, masked), mask, exposure of frame k: masks and exposures vary, some
    frames have neither (None: ones / identity)"""
    import torch
    g = torch.Generator(device="cpu").manual_seed(100 + k)
    rng = np.random.default_rng(200 + k)
    M = [None, R.make_mask("binary", H, W, rng), R.make_mask("half", H, W, rng), R.make_mask("fractional", H, W, rng)][k % 4]
    Ex = None if k % 3 == 2 else R.make_exposure("offset" if k % 2 else "on", rng)
    gt = torch.rand((3, H, W), generator=g)
    if M is not None:
        gt = gt * torch.tensor(M)[None]
    return gt.cuda(), _t(M), _t(Ex)


def _exact_step(scene, dcam, bg, gt, thr, M, Ex):
    import torch
    from diff_gaussian_rasterization import _C
    from h3dgs import pipeline
    (loss, l1, ssim), radii, n = pipeline.post_step(scene, dcam, bg, gt, thr, 0.2, Ex, M)
    D = _C.last_num_rendered()
    grads = {k: getattr(scene, k).grad.clone() for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    with torch.no_grad():
        img = pipeline.render_hier_fused(scene, dcam, bg, thr)[0].clone()
    # dL/dimage of the same frame, for the graphed step's to equal bit for bit
    x = img.clone().requires_grad_(True)
    from h3dgs.loss import post_loss
    post_loss(x, gt, 0.2, Ex, M)[0].backward()
    return dict(loss=float(loss), l1=float(l1), ssim=float(ssim), radii=radii.clone(), n=n, grads=grads, img=img, D=D,
                dimg=x.grad)


@pytest.mark.parametrize("skybox", [0, 200])
@pytest.mark.parametrize("capture", [False, True])
def test_graphed_post_step_equals_exact_step(skybox, capture):
    import torch
    from h3dgs import pipeline
    from h3dgs.poststep import GraphedPostStep
    cam, h = _scene(skybox=skybox)
    cams = _cams(cam.W, cam.H)
    thr = synth.tau_threshold(6.0, cam)
    scene = pipeline.Scene(h)
    bg = torch.tensor([0.2, 0.1, 0.3], device="cuda")
    dcams = [pipeline.DeviceCamera(c) for c in cams]
    gs = GraphedPostStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, lambda_dssim=0.2, exposure=True,
                         mask=True, bin_capacity=1 << 20, sort_capacity=4096, capture=False)
    gt0, M0, E0 = _frame_inputs(cam.H, cam.W, 0)
    gs.set_camera(dcams[0]); gs.gt.copy_(gt0)
    if capture:
        gs.capture()
        assert gs.launches_per_step >= 10
    side = torch.cuda.Stream()
    for k, (v, tau) in enumerate([(0, 6.0), (1, 6.0), (2, 15.0), (1, 3.0), (0, 6.0), (2, 6.0)]):
        gt, M, Ex = _frame_inputs(cam.H, cam.W, k)
        t = synth.tau_threshold(tau, cam)
        ref = _exact_step(scene, dcams[v], bg, gt, t, M, Ex)
        again = _exact_step(scene, dcams[v], bg, gt, t, M, Ex)
        gs.set_threshold(t)
        if k % 2:
            gs.step(dcams[v], gt, mask=M, exposure=Ex)                   # slot 0, copied on the current stream
        else:
            side.wait_stream(torch.cuda.current_stream())
            ready = gs.upload_target(gt, side, mask=M)                   # slots 1, 0, 1: the upload path
            gs.step(dcams[v], exposure=Ex, gt_ready=ready)
        st = gs.status()
        n, P = ref["n"], ref["n"] + skybox
        assert not st["overflow"]
        assert st["rows"] == P and st["D"] == ref["D"] and 0 < st["longest_list"] <= 4096
        for key in ("loss", "l1", "ssim"):
            assert abs(st[key] - ref[key]) < 1e-7, (k, key, st[key], ref[key])
        assert torch.equal(gs.image, ref["img"])
        assert torch.equal(gs.radii[:P], ref["radii"]) and bool((gs.radii[P:] == 0).all())
        # the backward's input is the same: the Gaussian gradients can differ by the order of its atomic sums only.
        # Equal as values, not as bits: where the exact step has no exposure or mask the graph applies the identity and
        # ones, and a masked-out -0 of one path can be +0 in the other (x*1 + 0*y)
        assert torch.equal(gs.dcolor, ref["dimg"])
        for name, g in ref["grads"].items():
            # the bar of test_gpu_graphstep.py (5e-6), or four times the spread two exact steps of the same frame show:
            # the SSIM term's per-pixel gradients cancel more in the per-Gaussian sums than the L1 term's signs
            noise = rel_err(again["grads"][name].cpu().numpy(), g.cpu().numpy())
            e = rel_err(gs.grads[name].cpu().numpy(), g.cpu().numpy())
            assert e < max(5e-6, 4.0 * noise), (k, name, e, noise)


def test_overflowed_frame_is_flagged_harmless_and_rerun_exactly():
    import torch
    from h3dgs import pipeline
    from h3dgs.poststep import GraphedPostStep
    cam, h = _scene()
    thr = synth.tau_threshold(6.0, cam)
    scene = pipeline.Scene(h)
    bg = torch.tensor([0.2, 0.1, 0.3], device="cuda")
    dcam = pipeline.DeviceCamera(cam)
    gt, M, Ex = _frame_inputs(cam.H, cam.W, 1)
    ref = _exact_step(scene, dcam, bg, gt, thr, M, Ex)
    gs = GraphedPostStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, exposure=True, mask=True,
                         bin_capacity=ref["D"] // 2, sort_capacity=4096)
    gs.step(dcam, gt, mask=M, exposure=Ex)
    st = gs.status()
    assert st["overflow"] and st["D"] == ref["D"]
    assert torch.equal(gs.image, bg.view(3, 1, 1).expand_as(gs.image))
    assert all(float(g.abs().sum()) == 0.0 for g in gs.grads.values())
    # the caller re-runs the flagged frame through the exact path: it is the frame's true step
    again = _exact_step(scene, dcam, bg, gt, thr, M, Ex)
    assert again["loss"] == ref["loss"] and torch.equal(again["img"], ref["img"])
    for name, g in ref["grads"].items():
        assert rel_err(again["grads"][name].cpu().numpy(), g.cpu().numpy()) < 5e-6


def test_more_than_one_rank_raises():
    import torch
    from h3dgs import pipeline
    from h3dgs.poststep import GraphedPostStep
    cam, h = _scene(leaves=500)
    scene = pipeline.Scene(h)
    with pytest.raises(ValueError, match="one GPU"):
        GraphedPostStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, torch.zeros(3, device="cuda"),
                        synth.tau_threshold(6.0, cam), world=2, capture=False)


# ---- a post-optimisation loop on this objective ------------------------------------------------------------------------
def _loop(h, gt, M, Ex, cam, thr, graphed, iters=40):
    import torch
    from h3dgs import pipeline
    from h3dgs.poststep import GraphedPostStep
    scene = pipeline.Scene(h)
    dcam = pipeline.DeviceCamera(cam)
    bg = torch.zeros(3, device="cuda")
    opt = torch.optim.Adam([{"params": [scene.shs], "lr": 2e-2}, {"params": [scene.opacities], "lr": 1e-2}])
    losses = []
    if graphed:
        gs = GraphedPostStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, thr, exposure=True, mask=True,
                             bin_capacity=1 << 20, sort_capacity=4096, capture=False)
        gs.set_camera(dcam)
        gs.gt.copy_(gt)
        gs.capture()
    for _ in range(iters):
        if graphed:
            gs.step(gt=gt, mask=M, exposure=Ex)
            st = gs.status()
            assert not st["overflow"]
            losses.append(st["loss"])
            scene.shs.grad, scene.opacities.grad = gs.grads["shs"].clone(), gs.grads["opacities"].clone()
        else:
            (loss, _, _), _, _ = pipeline.post_step(scene, dcam, bg, gt, thr, 0.2, Ex, M)
            losses.append(float(loss))
        opt.step()
    return np.array(losses)


def test_post_optimisation_loop_graphed_and_eager():
    """train_post.py:91-192 in miniature on this objective, with an exposure and a binary mask: 40 Adam iterations reduce
    the loss by at least 20 %.  The graphed and the eager loop take the same steps up to the order of the backward's
    atomic sums, so they drift apart slowly; the bar for their final losses is derived from that drift as two eager
    loops show it: 20 times the eager-eager difference, and at least 2e-6 of the loss."""
    import torch
    from h3dgs import pipeline
    cam = synth.make_camera(320, 180)
    leaves = synth.cloud_v1(6000, cam, zmin=2.0, zmax=30.0, seed=5, scale_k=1.0)
    z = leaves["means3D"][:, 2:3]
    leaves["scales"] = (8e-3 * np.sqrt(2.0 * z) * np.ones((1, 3))).astype(np.float32)
    h = synth.build_hierarchy(leaves)
    thr = synth.tau_threshold(6.0, cam)
    dcam = pipeline.DeviceCamera(cam)
    rng = np.random.default_rng(0)
    Ex = _t(R.make_exposure("on", rng))
    M = _t(R.make_mask("binary", cam.H, cam.W, rng))
    from h3dgs.loss import exposure_block
    with torch.no_grad():
        raw = pipeline.render_hier_fused(pipeline.Scene(h, requires_grad=False), dcam, torch.zeros(3, device="cuda"), thr)[0]
        E3 = exposure_block(Ex, raw.device)
        gt = ((torch.matmul(raw.permute(1, 2, 0), E3[:3, :3]).permute(2, 0, 1) + E3[:3, 3, None, None]).clamp(0, 1) * M).contiguous()
    h2 = dict(h)
    h2["shs"] = (h["shs"] + 0.15 * rng.standard_normal(h["shs"].shape)).astype(np.float32)
    h2["opacities"] = np.clip(h["opacities"] * rng.uniform(0.6, 1.0, h["opacities"].shape), 0.01, None).astype(np.float32)
    eager = _loop(h2, gt, M, Ex, cam, thr, graphed=False)
    eager2 = _loop(h2, gt, M, Ex, cam, thr, graphed=False)
    graphed = _loop(h2, gt, M, Ex, cam, thr, graphed=True)
    assert np.isfinite(eager).all() and np.isfinite(graphed).all()
    assert eager[-1] < 0.8 * eager[0] and graphed[-1] < 0.8 * graphed[0], (eager[[0, -1]], graphed[[0, -1]])
    assert abs(graphed[0] - eager[0]) < 1e-7                         # the first step sees identical parameters
    bar = max(20.0 * abs(eager2[-1] - eager[-1]), 2e-6 * eager[-1])
    print(f"\nfinal losses eager {eager[-1]:.9f} / {eager2[-1]:.9f}, graphed {graphed[-1]:.9f}; bar {bar:.3g}")
    assert abs(graphed[-1] - eager[-1]) <= bar

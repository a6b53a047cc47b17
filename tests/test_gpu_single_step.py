"""GPU: train_single's objective on the device (the post-loss backward with the exposure gradient, the inverse-depth L1
kernel, the densification statistics kernel, h3dgs.loss.single_loss, pipeline.single_step,
h3dgs.singlestep.GraphedSingleStep).

  * a flat capacity-mode forward and backward with the inverse depth against the exact mode;
  * the kernels per element against tests/single_loss_ref.py from 1x1 to 1080p, at the tile edge +-1 and at the clamp
    edges; dL/dimage bit for bit h3dgs_post_loss_backward's; the reference's own fixture;
  * pipeline.single_step against the drop-in flow (packages + torch ops + the reference-form conv2d SSIM);
  * the graphed step against single_step with every input changing and both slots in use; an overflowed frame; a rebuilt
    step after the row count changed; carried statistics through capture(); world > 1; a 40-iteration loop with sparse Adam and the exposure's Adam."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import post_loss_ref as R  # noqa: E402
import single_loss_ref as SR  # noqa: E402
from h3dgs import synth  # noqa: E402
from util import rel_err  # noqa: E402

pytestmark = pytest.mark.gpu
F = np.float32
NAMES = ("means3D", "shs", "opacities", "scales", "rotations")


def _t(a, **k):
    import torch
    return None if a is None else torch.tensor(a, device="cuda", **k)


# ---- the kernels -------------------------------------------------------------------------------------------------------
def _run_photo(img, gt, lam, Ex, M):
    """single_loss without a depth term, exposure trained -> (out floats, dL/dimg, dL/dE), and post_loss's dL/dimg"""
    import torch
    from h3dgs.loss import post_loss, single_loss
    x = _t(img, requires_grad=True)
    E = _t(np.eye(3, 4, dtype=F) if Ex is None else Ex, requires_grad=True)
    out = single_loss(x, None, _t(gt), lam, E, _t(M))
    out[0].backward()
    x0 = _t(img, requires_grad=True)
    post_loss(x0, _t(gt), lam, _t(np.eye(3, 4, dtype=F) if Ex is None else Ex), _t(M))[0].backward()
    assert torch.equal(x.grad.view(torch.int32), x0.grad.view(torch.int32))
    return [float(v.detach()) for v in out], x.grad.cpu().numpy(), E.grad.double().cpu().numpy()


def _check_photo(img, gt, lam, Ex, M):
    r = SR.exposure_grad_reference(img, gt, lam, Ex, M)
    _, grad, dE = _run_photo(img, gt, lam, Ex, M)
    # the autograd function hands the gradient over in the exposure's fp32
    ratio = np.abs(dE - r["dE"]) / (r["dE_tol"] + SR.U * np.abs(r["dE"]))
    print(f"\n{img.shape}: dE ratio {ratio.max():.3g}")
    assert np.isfinite(dE).all() and ratio.max() <= 1.0, ratio
    return r, grad, dE


@pytest.mark.parametrize("shape", [(1, 1), (1, 17), (15, 15), (16, 16), (17, 17), (31, 33), (64, 48)])
@pytest.mark.parametrize("content", ["random", "saturated"])
@pytest.mark.parametrize("em", [("none", "none"), ("on", "binary"), ("offset", "fractional")])
def test_exposure_gradient_within_budget(shape, content, em):
    img, gt, Ex, M = R.make_inputs(*shape, em[0], em[1], content, seed=31)
    _check_photo(img, gt, 0.2, Ex, M)


def test_exposure_gradient_full_hd():
    img, gt, Ex, M = R.make_inputs(1080, 1920, "offset", "fractional", seed=32)
    _check_photo(img, gt, 0.2, Ex, M)


@pytest.mark.parametrize("exposure", R.EXPOSURES)
def test_exposure_gradient_at_the_clamp_edges(exposure):
    img, gt, Ex = R.clamp_edge_inputs(33, 35, exposure, seed=33)
    _check_photo(img, gt, 0.2, Ex, None)


def test_zero_mask_gives_zero_exposure_gradient():
    img, gt, Ex, M = R.make_inputs(45, 70, "offset", "zero", seed=34)
    _, _, dE = _check_photo(img, gt, 0.2, Ex, M)
    assert np.all(dE == 0.0)


@pytest.mark.parametrize("shape", [(1, 1), (3, 5), (16, 16), (17, 33), (270, 480), (1080, 1920)])
@pytest.mark.parametrize("kind,w", [("random", 1.0), ("random", 0.37), ("random", 0.0), ("zero", 0.8)])
def test_invdepth_kernel(shape, kind, w):
    import torch
    from h3dgs import _lib
    H, W = shape
    d, m, k = SR.make_depth_inputs(H, W, kind, seed=35)
    td, tm, tk, tw = _t(d), _t(m), _t(k), _t(np.array([w], F))
    grad = torch.full((H, W), 9.0, device="cuda")
    tot = torch.full((1,), 5.0, dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib().h3dgs_invdepth_l1_grad(H, W, td.data_ptr(), tm.data_ptr(), tk.data_ptr(), tw.data_ptr(), grad.data_ptr(),
                                                tot.data_ptr(), torch.cuda.current_stream().cuda_stream))
    r = SR.depth_reference(d, m, k, w)
    assert np.array_equal(grad.cpu().numpy(), r["grad"])
    assert abs(float(tot) - r["sum"]) <= r["sum_tol"]
    if w == 0.0 or kind == "zero":
        assert float(grad.abs().sum()) == 0.0
    else:
        assert float(grad[td == tm].abs().sum()) == 0.0
    # torch's own lines (train_single.py:115-116) agree
    x = td.clone().requires_grad_(True)
    (w * torch.abs((x - tm) * tk).mean()).backward()
    assert torch.allclose(grad, x.grad, rtol=1e-6, atol=0)


@pytest.mark.parametrize("P", [1, 257, 100000])
@pytest.mark.parametrize("flag", [None, 0, 1])
def test_densify_stats_kernel_is_the_torch_lines(P, flag):
    import torch
    from h3dgs import pipeline
    rng = np.random.default_rng(36)
    radii = _t((rng.integers(0, 50, P) * (rng.uniform(size=P) > 0.4)).astype(np.int32))
    dm = _t((rng.standard_normal((P, 3)) * 1e-3).astype(F))
    st = pipeline.DensifyStats(P)
    st.max_radii2D.copy_(_t((rng.integers(0, 60, P) * (rng.uniform(size=P) > 0.5)).astype(F)))
    st.xyz_gradient_accum.copy_(_t((np.abs(rng.standard_normal((P, 1))) * 1e-3 * (rng.uniform(size=(P, 1)) > 0.5)).astype(F)))
    st.denom.copy_(_t(rng.integers(0, 9, (P, 1)).astype(F)))
    mr, acc, den = st.max_radii2D.clone(), st.xyz_gradient_accum.clone(), st.denom.clone()
    info = None if flag is None else torch.tensor([5, 5, flag, 0], dtype=torch.int32, device="cuda")
    st.update(radii, dm, info)
    if flag != 1:
        # train_single.py:147, gaussian_model.py:688-689; the norm as elementwise torch operations, each rounded once
        vis = (radii > 0).nonzero().flatten()
        mr[vis] = torch.max(mr[vis], radii[vis])
        g = dm[vis, :2]
        acc[vis] = torch.max(torch.sqrt(g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]).unsqueeze(1), acc[vis])
        norm_acc = torch.max(torch.norm(dm[vis, :2], dim=-1, keepdim=True), st.xyz_gradient_accum.new_zeros(()))
        den[vis] += 1
        # torch.norm itself may fuse its multiply-add: within two ulps of it
        assert bool(((st.xyz_gradient_accum[vis] - torch.max(norm_acc, acc[vis])).abs() <= 5e-7 * acc[vis]).all())
    for a, b in ((st.max_radii2D, mr), (st.xyz_gradient_accum, acc), (st.denom, den)):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("i", range(6))
def test_single_loss_matches_the_reference(golden_dir, i):
    z = np.load(os.path.join(golden_dir, "single_loss.npz"))
    from h3dgs.loss import single_loss
    msk, dep = (bool(v) for v in z[f"c{i}_flags"])
    x, inv = _t(z[f"c{i}_raw"], requires_grad=True), _t(z[f"c{i}_invdepth"][None], requires_grad=True)
    E = _t(z[f"c{i}_E"], requires_grad=True)
    out = single_loss(x, inv, _t(z[f"c{i}_gt"]), float(z["lam"]), E, _t(z[f"c{i}_mask"][None]) if msk else None,
                      _t(z[f"c{i}_mono"][None]) if dep else None, _t(z[f"c{i}_dmask"][None]), float(z[f"c{i}_weight"]))
    out[0].backward()
    for key, v in zip(("loss", "photo", "l1", None, "depth"), out):
        if key:
            assert abs(float(v.detach()) - float(z[f"c{i}_{key}"])) < 1e-6, key
    for got, ref, tol in ((x.grad, z[f"c{i}_grad"], 1e-5), (inv.grad[0], z[f"c{i}_dinv"], 1e-6), (E.grad, z[f"c{i}_dE"], 2e-5)):
        assert np.abs(got.cpu().numpy() - ref).max() <= tol * max(np.abs(ref).max(), 1e-30)


# ---- flat scenes ---------------------------------------------------------------------------------------------------------
def _leaves(n=9000, W=480, H=270, seed=3):
    cam = synth.make_camera(W, H)
    lv = synth.cloud_v1(n, cam, zmin=2.0, zmax=40.0, seed=seed, scale_k=1.0)
    z = lv["means3D"][:, 2:3]
    lv["scales"] = (4e-3 * np.sqrt(2.0 * z) * np.exp(0.4 * np.random.default_rng(1).standard_normal((z.shape[0], 3)))).astype(F)
    return cam, lv


def _cams(W, H, n=3):
    rs = np.random.default_rng(2)
    return [synth.make_camera(W, H)] + [synth.yaw_camera(W, H, float(rs.uniform(-15, 15)), rs.uniform(-0.5, 0.5, 3))
                                        for _ in range(n - 1)]


def _frame(H, W, k):
    """step k's background, target (masked as the loader leaves it), mask, exposure, mono depth, depth mask and weight;
    frame 2 has no mask, frame 3 an unreliable depth, frame 4 weight 0"""
    import torch
    rng = np.random.default_rng(500 + k)
    bg = _t(rng.uniform(0, 1, 3).astype(F))
    M = [R.make_mask("binary", H, W, rng), R.make_mask("fractional", H, W, rng), None, R.make_mask("half", H, W, rng)][k % 4]
    gt = rng.uniform(0, 1, (3, H, W)).astype(F) * (1.0 if M is None else M[None])
    E = _t(R.make_exposure("offset" if k % 2 else "on", rng), requires_grad=True)
    _, m, dm = SR.make_depth_inputs(H, W, seed=600 + k)
    mono, dmask = (None, None) if k == 3 else (_t(0.05 * m), _t(dm))
    return dict(bg=bg, gt=_t(gt.astype(F)), M=_t(M), E=E, mono=mono, dmask=dmask, w=[1.0, 0.3, 0.7, 0.5, 0.0, 0.2][k % 6])


def _exact(scene, dcam, fr, stats=None):
    import torch
    from diff_gaussian_rasterization import _C
    from h3dgs import pipeline
    fr["E"].grad = None
    out, radii, m2d = pipeline.single_step(scene, dcam, fr["bg"], fr["gt"], 0.2, fr["E"], fr["M"], fr["mono"], fr["dmask"],
                                           fr["w"], stats)
    D = _C.last_num_rendered()
    grads = {k: getattr(scene, k).grad.clone() for k in NAMES}
    with torch.no_grad():
        img, _, inv = pipeline.render_flat(scene, dcam, fr["bg"], do_depth=True)
    x, v = img.clone().requires_grad_(True), inv.clone().requires_grad_(True)
    from h3dgs.loss import single_loss
    single_loss(x, v, fr["gt"], 0.2, fr["E"].detach(), fr["M"], fr["mono"], fr["dmask"], fr["w"])[0].backward()
    dinv = torch.zeros_like(inv[0]) if v.grad is None else v.grad[0]
    return dict(out=[float(o.detach()) for o in out], radii=radii.clone(), grads=grads, img=img, inv=inv, D=D, dimg=x.grad,
                dinv=dinv, dE=fr["E"].grad.clone(), m2d=m2d.grad.clone())


def test_flat_capacity_mode_with_depth_equals_exact_mode():
    """capacity mode without the LOD cut's index arrays: forward (image, inverse depth, radii) bit-identical to the exact
    mode, backward with dL/dinvdepth equal up to the order of the atomic sums"""
    import torch
    from h3dgs import pipeline
    from h3dgs.singlestep import GraphedSingleStep
    cam, lv = _leaves()
    scene = pipeline.Scene(lv)
    dcam = pipeline.DeviceCamera(cam)
    fr = _frame(cam.H, cam.W, 0)
    ref = _exact(scene, dcam, fr)
    gs = GraphedSingleStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, mask=True, bin_capacity=1 << 20, capture=False)
    gs.step(dcam, fr["gt"], mask=fr["M"], mono_invdepth=fr["mono"], depth_mask=fr["dmask"], exposure=fr["E"], bg=fr["bg"],
            depth_weight=fr["w"])
    st = gs.status()
    assert not st["overflow"] and st["D"] == ref["D"]
    assert torch.equal(gs.image, ref["img"]) and torch.equal(gs.invdepth, ref["inv"]) and torch.equal(gs.radii, ref["radii"])
    assert float(gs.dinvdepth.abs().sum()) > 0 and torch.equal(gs.dinvdepth, ref["dinv"])
    for name, g in ref["grads"].items():
        assert rel_err(gs.grads[name].cpu().numpy(), g.cpu().numpy()) < 5e-6, name


def _ssim_conv2d(a, b):
    import torch
    import torch.nn.functional as Fn
    torch.backends.cudnn.allow_tf32 = False          # the comparison is to 1e-5: full fp32 convolutions
    g = torch.tensor([np.exp(-(x - 5) ** 2 / (2 * 1.5 ** 2)) for x in range(11)], dtype=torch.float32)
    g = (g / g.sum()).unsqueeze(1)
    win = (g @ g.t())[None, None].expand(3, 1, 11, 11).contiguous().cuda()
    a, b = a[None], b[None]
    mu1, mu2 = Fn.conv2d(a, win, padding=5, groups=3), Fn.conv2d(b, win, padding=5, groups=3)
    s1 = Fn.conv2d(a * a, win, padding=5, groups=3) - mu1 * mu1
    s2 = Fn.conv2d(b * b, win, padding=5, groups=3) - mu2 * mu2
    s12 = Fn.conv2d(a * b, win, padding=5, groups=3) - mu1 * mu2
    return (((2 * mu1 * mu2 + 1e-4) * (2 * s12 + 9e-4)) / ((mu1 * mu1 + mu2 * mu2 + 1e-4) * (s1 + s2 + 9e-4))).mean()


def dropin_step(scene, dcam, fr, stats=None):
    """train_single.py:97-123, 147-148 as the reference writes it: the drop-in rasterizer, torch ops, conv2d SSIM"""
    import torch
    from h3dgs import pipeline
    scene.zero_grad()
    fr["E"].grad = None
    m2d = torch.zeros_like(scene.means3D, requires_grad=True)
    image, radii, invDepth = pipeline.render_flat(scene, dcam, fr["bg"], do_depth=True, means2D=m2d)
    E = fr["E"]
    image = torch.matmul(image.permute(1, 2, 0), E[:3, :3]).permute(2, 0, 1) + E[:3, 3, None, None]
    image = image.clamp(0, 1)
    if fr["M"] is not None:
        image = image * fr["M"][None]
    Ll1 = torch.abs(image - fr["gt"]).mean()
    photo = 0.8 * Ll1 + 0.2 * (1.0 - _ssim_conv2d(image, fr["gt"]))
    loss = photo.clone()
    if fr["w"] > 0 and fr["mono"] is not None:
        loss = loss + fr["w"] * torch.abs((invDepth - fr["mono"][None]) * fr["dmask"][None]).mean()
    loss.backward()
    if stats is not None:
        with torch.no_grad():
            vis = (radii > 0).nonzero().flatten()
            stats.max_radii2D[vis] = torch.max(stats.max_radii2D[vis], radii[vis])
            stats.xyz_gradient_accum[vis] = torch.max(torch.norm(m2d.grad[vis, :2], dim=-1, keepdim=True), stats.xyz_gradient_accum[vis])
            stats.denom[vis] += 1
    return loss


@pytest.mark.parametrize("k", [0, 1, 3, 4])
def test_single_step_equals_the_drop_in_flow(k):
    from h3dgs import pipeline
    cam, lv = _leaves()
    scene = pipeline.Scene(lv)
    dcam = pipeline.DeviceCamera(_cams(cam.W, cam.H)[k % 3])
    fr = _frame(cam.H, cam.W, k)
    s_ref, s_got = pipeline.DensifyStats(scene.means3D.shape[0]), pipeline.DensifyStats(scene.means3D.shape[0])
    loss = dropin_step(scene, dcam, fr, s_ref)
    want = {n: getattr(scene, n).grad.clone() for n in NAMES}
    wantE = fr["E"].grad.clone()
    ref = _exact(scene, dcam, fr, s_got)
    assert abs(ref["out"][0] - float(loss.detach())) < 1e-5
    for n, g in want.items():
        assert rel_err(ref["grads"][n].cpu().numpy(), g.cpu().numpy()) < 1e-5, n
    assert rel_err(ref["dE"].cpu().numpy(), wantE.cpu().numpy()) < 1e-5
    assert bool((s_got.max_radii2D == s_ref.max_radii2D).all()) and bool((s_got.denom == s_ref.denom).all())
    assert rel_err(s_got.xyz_gradient_accum.cpu().numpy(), s_ref.xyz_gradient_accum.cpu().numpy()) < 1e-5


@pytest.mark.parametrize("capture", [False, True])
def test_graphed_single_step_equals_exact_step(capture):
    import torch
    from h3dgs import pipeline
    from h3dgs.singlestep import GraphedSingleStep
    cam, lv = _leaves()
    scene = pipeline.Scene(lv)
    dcams = [pipeline.DeviceCamera(c) for c in _cams(cam.W, cam.H)]
    N = scene.means3D.shape[0]
    s_ref = pipeline.DensifyStats(N)
    gs = GraphedSingleStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, mask=True, bin_capacity=1 << 20, capture=False)
    gs.set_camera(dcams[0])
    if capture:
        gs.capture()
        assert gs.launches_per_step >= 10
    side = torch.cuda.Stream()
    for k, v in enumerate([0, 1, 2, 1, 0, 2]):
        fr = _frame(cam.H, cam.W, k)
        again = _exact(scene, dcams[v], fr)
        ref = _exact(scene, dcams[v], fr, s_ref)
        prev = [t.cpu().numpy() for t in (gs.stats.max_radii2D, gs.stats.xyz_gradient_accum, gs.stats.denom)]
        gs.set_background(fr["bg"])
        gs.set_depth_weight(fr["w"])
        if k % 2:
            gs.step(dcams[v], fr["gt"], mask=fr["M"], mono_invdepth=fr["mono"], depth_mask=fr["dmask"], exposure=fr["E"])
        else:
            side.wait_stream(torch.cuda.current_stream())
            ready = gs.upload_target(fr["gt"], side, fr["M"], fr["mono"], fr["dmask"])          # slots 0, 1, 0
            gs.step(dcams[v], exposure=fr["E"], gt_ready=ready)
        st = gs.status()
        assert not st["overflow"] and st["D"] == ref["D"] and 0 < st["longest_list"] <= 4096
        for key, val in zip(("loss", "photo", "l1", "ssim", "depth_l1"), ref["out"]):
            assert abs(st[key] - val) < 2e-7, (k, key, st[key], val)
        assert torch.equal(gs.image, ref["img"]) and torch.equal(gs.invdepth, ref["inv"]) and torch.equal(gs.radii, ref["radii"])
        assert torch.equal(gs.dcolor, ref["dimg"]) and torch.equal(gs.dinvdepth, ref["dinv"])
        # fp64 sums in another order, then one rounding to fp32
        assert rel_err(gs.exposure_grad.cpu().numpy(), ref["dE"].cpu().numpy()) < 1e-6
        for name, g in ref["grads"].items():
            noise = rel_err(again["grads"][name].cpu().numpy(), g.cpu().numpy())
            e = rel_err(gs.grads[name].cpu().numpy(), g.cpu().numpy())
            assert e < max(5e-6, 4.0 * noise), (k, name, e, noise)
        # the statistics: counts and radii identical; the gradient norms follow d_means2D, equal up to the atomic order
        assert torch.equal(gs.stats.max_radii2D, s_ref.max_radii2D) and torch.equal(gs.stats.denom, s_ref.denom)
        assert rel_err(gs.stats.xyz_gradient_accum.cpu().numpy(), s_ref.xyz_gradient_accum.cpu().numpy()) < 5e-6
        # and the kernel itself, bit for bit, on the graphed step's own d_means2D and the statistics before the step
        want = SR.stats_reference(gs.radii.cpu().numpy(), gs.d_means2D.cpu().numpy(), *prev)
        for got, w in zip((gs.stats.max_radii2D, gs.stats.xyz_gradient_accum, gs.stats.denom), want):
            assert np.array_equal(got.cpu().numpy().view(np.uint32), w.view(np.uint32)), k
    assert float(gs.stats.denom.max()) == 6.0


def test_overflowed_frame_is_flagged_harmless_and_rerun_exactly():
    import torch
    from h3dgs import pipeline
    from h3dgs.singlestep import GraphedSingleStep
    cam, lv = _leaves()
    scene = pipeline.Scene(lv)
    dcam = pipeline.DeviceCamera(cam)
    fr = _frame(cam.H, cam.W, 1)
    ref = _exact(scene, dcam, fr)
    gs = GraphedSingleStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, mask=True, bin_capacity=ref["D"] // 2)
    gs.step(dcam, fr["gt"], mask=fr["M"], mono_invdepth=fr["mono"], depth_mask=fr["dmask"], exposure=fr["E"], bg=fr["bg"],
            depth_weight=fr["w"])
    st = gs.status()
    assert st["overflow"] and st["D"] == ref["D"] and bool((gs.radii > 0).any())
    assert torch.equal(gs.image, fr["bg"].view(3, 1, 1).expand_as(gs.image))
    assert all(float(g.abs().sum()) == 0.0 for g in gs.grads.values()) and float(gs.exposure_grad.abs().sum()) == 0.0
    assert all(float(t.abs().sum()) == 0.0 for t in (gs.stats.max_radii2D, gs.stats.xyz_gradient_accum, gs.stats.denom))
    # the caller re-runs the flagged frame through the exact path, into the step's statistics
    again = _exact(scene, dcam, fr, gs.stats)
    assert again["out"][0] == ref["out"][0] and torch.equal(again["img"], ref["img"])
    for name, g in ref["grads"].items():
        assert rel_err(again["grads"][name].cpu().numpy(), g.cpu().numpy()) < 5e-6
    assert float(gs.stats.denom.sum()) == float((ref["radii"] > 0).sum())


def test_rebuilt_step_carries_the_statistics_over():
    """densify_and_prune changes the row count: a new step over the new rows continues from the statistics handed to it"""
    import torch
    from h3dgs import pipeline
    from h3dgs.singlestep import GraphedSingleStep
    cam, lv = _leaves(n=4000)
    scene = pipeline.Scene(lv)
    dcam = pipeline.DeviceCamera(cam)
    fr = _frame(cam.H, cam.W, 0)
    gs = GraphedSingleStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, mask=True, bin_capacity=1 << 20, capture=False)
    gs.step(dcam, fr["gt"], mask=fr["M"], mono_invdepth=fr["mono"], depth_mask=fr["dmask"], exposure=fr["E"], bg=fr["bg"], depth_weight=fr["w"])
    keep = torch.arange(scene.means3D.shape[0], device="cuda") % 3 != 0          # a prune mask
    lv2 = {k: (v[keep.cpu().numpy()] if isinstance(v, np.ndarray) and v.shape[:1] == keep.shape else v) for k, v in lv.items()}
    scene2 = pipeline.Scene(lv2)
    carried = pipeline.DensifyStats(int(keep.sum()))
    carried.max_radii2D.copy_(gs.stats.max_radii2D[keep]); carried.xyz_gradient_accum.copy_(gs.stats.xyz_gradient_accum[keep])
    carried.denom.copy_(gs.stats.denom[keep])
    eager = pipeline.DensifyStats(int(keep.sum()))
    for a, b in zip((eager.max_radii2D, eager.xyz_gradient_accum, eager.denom), (carried.max_radii2D, carried.xyz_gradient_accum, carried.denom)):
        a.copy_(b)
    assert float(carried.denom.sum()) > 0
    gs2 = GraphedSingleStep(scene2, cam.W, cam.H, cam.tanfovx, cam.tanfovy, mask=True, stats=carried, bin_capacity=1 << 20, capture=False)
    assert gs2.stats is carried
    fr2 = _frame(cam.H, cam.W, 1)
    gs2.step(dcam, fr2["gt"], mask=fr2["M"], mono_invdepth=fr2["mono"], depth_mask=fr2["dmask"], exposure=fr2["E"], bg=fr2["bg"], depth_weight=fr2["w"])
    _exact(scene2, dcam, fr2, eager)
    assert torch.equal(carried.denom, eager.denom) and torch.equal(carried.max_radii2D, eager.max_radii2D)
    assert float(carried.denom.max()) == 2.0
    assert rel_err(carried.xyz_gradient_accum.cpu().numpy(), eager.xyz_gradient_accum.cpu().numpy()) < 5e-6
    with pytest.raises(ValueError, match="rows"):
        GraphedSingleStep(scene2, cam.W, cam.H, cam.tanfovx, cam.tanfovy, stats=gs.stats, capture=False)


def test_capture_leaves_carried_statistics_untouched():
    """capture() runs one eager step on whatever the buffers hold -- here a camera that sees the scene, against a zero
    target: the statistics handed over to be carried on must come out of it bit for bit, and the first real step counts
    once"""
    import torch
    from h3dgs import pipeline
    from h3dgs.singlestep import GraphedSingleStep
    cam, lv = _leaves(n=4000)
    scene = pipeline.Scene(lv)
    dcam = pipeline.DeviceCamera(cam)
    N = scene.means3D.shape[0]
    rng = np.random.default_rng(7)
    carried = pipeline.DensifyStats(N)
    carried.max_radii2D.copy_(_t(rng.integers(0, 5, N).astype(F)))
    carried.xyz_gradient_accum.copy_(_t((1e-9 * rng.uniform(size=(N, 1))).astype(F)))
    carried.denom.copy_(_t(rng.integers(0, 9, (N, 1)).astype(F)))
    before = [t.clone() for t in (carried.max_radii2D, carried.xyz_gradient_accum, carried.denom)]
    gs = GraphedSingleStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, mask=True, stats=carried, bin_capacity=1 << 20,
                           capture=False)
    gs.set_camera(dcam)
    gs.capture()
    torch.cuda.synchronize()
    assert bool((gs.radii > 0).any())                                    # the warm-up frame did see Gaussians
    for a, b in zip((carried.max_radii2D, carried.xyz_gradient_accum, carried.denom), before):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    fr = _frame(cam.H, cam.W, 0)
    gs.step(dcam, fr["gt"], mask=fr["M"], mono_invdepth=fr["mono"], depth_mask=fr["dmask"], exposure=fr["E"], bg=fr["bg"], depth_weight=fr["w"])
    want = SR.stats_reference(gs.radii.cpu().numpy(), gs.d_means2D.cpu().numpy(), *[b.cpu().numpy() for b in before])
    for got, w in zip((carried.max_radii2D, carried.xyz_gradient_accum, carried.denom), want):
        assert np.array_equal(got.cpu().numpy().view(np.uint32), w.view(np.uint32))
    assert float((carried.denom - before[2]).max()) == 1.0


def test_statistics_of_another_row_count_are_refused_on_the_exact_path():
    import torch
    from h3dgs import pipeline
    cam, lv = _leaves(n=500)
    scene = pipeline.Scene(lv)
    fr = _frame(cam.H, cam.W, 0)
    with pytest.raises(ValueError, match="rows"):
        pipeline.single_step(scene, pipeline.DeviceCamera(cam), fr["bg"], fr["gt"], stats=pipeline.DensifyStats(400))
    st = pipeline.DensifyStats(500)
    with pytest.raises(ValueError, match="int32"):
        st.update(torch.zeros(500, device="cuda"), torch.zeros((500, 3), device="cuda"))
    with pytest.raises(ValueError, match="d_means2D"):
        st.update(torch.zeros(500, dtype=torch.int32, device="cuda"), torch.zeros((500, 2), device="cuda"))


def test_more_than_one_rank_and_hierarchies_are_refused():
    from h3dgs import pipeline
    from h3dgs.singlestep import GraphedSingleStep
    cam, lv = _leaves(n=500)
    with pytest.raises(ValueError, match="one GPU"):
        GraphedSingleStep(pipeline.Scene(lv), cam.W, cam.H, cam.tanfovx, cam.tanfovy, world=2, capture=False)
    with pytest.raises(ValueError, match="flat"):
        GraphedSingleStep(pipeline.Scene(synth.build_hierarchy(lv)), cam.W, cam.H, cam.tanfovx, cam.tanfovy, capture=False)


# ---- a training loop on this objective -----------------------------------------------------------------------------------
def _loop(lv, fr, cam, E0, graphed, iters=40):
    import torch
    from h3dgs import pipeline
    from h3dgs.optim import Adam
    from h3dgs.singlestep import GraphedSingleStep
    scene = pipeline.Scene(lv)
    dcam = pipeline.DeviceCamera(cam)
    E = E0.clone().requires_grad_(True)
    opt = Adam([{"params": [scene.shs], "lr": 2e-2}, {"params": [scene.opacities], "lr": 1e-2}], lr=0.0, eps=1e-15)
    eopt = torch.optim.Adam([E], lr=1e-3)
    losses = []
    if graphed:
        gs = GraphedSingleStep(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, mask=True, bin_capacity=1 << 20, capture=False)
        gs.set_camera(dcam); gs.set_background(fr["bg"]); gs.set_depth_weight(fr["w"])
        gs.capture()
    for _ in range(iters):
        if graphed:
            gs.step(gt=fr["gt"], mask=fr["M"], mono_invdepth=fr["mono"], depth_mask=fr["dmask"], exposure=E)
            st = gs.status()
            assert not st["overflow"]
            losses.append(st["loss"])
            scene.shs.grad, scene.opacities.grad, E.grad = gs.grads["shs"].clone(), gs.grads["opacities"].clone(), gs.exposure_grad.clone()
        else:
            out, _, _ = pipeline.single_step(scene, dcam, fr["bg"], fr["gt"], 0.2, E, fr["M"], fr["mono"], fr["dmask"], fr["w"])
            losses.append(float(out[0].detach()))
        eopt.step()                                                      # train_single.py:159
        relevant = (scene.opacities.grad.flatten() != 0).nonzero().flatten().long()      # :171-174
        opt.step(relevant)
        E.grad = None
    return np.array(losses), E.detach().clone()


def test_training_loop_graphed_and_eager():
    """train_single.py:94-178 in miniature: 40 iterations of sparse Adam on SH and opacity and Adam on the exposure reduce
    the loss; the graphed and the eager loop end within the drift two eager loops show (x20, at least 1e-5 of the loss)"""
    import torch
    from h3dgs import pipeline
    cam = synth.make_camera(320, 180)
    lv = synth.cloud_v1(6000, cam, zmin=2.0, zmax=30.0, seed=5, scale_k=1.0)
    z = lv["means3D"][:, 2:3]
    lv["scales"] = (8e-3 * np.sqrt(2.0 * z) * np.ones((1, 3))).astype(F)
    dcam = pipeline.DeviceCamera(cam)
    rng = np.random.default_rng(0)
    fr = _frame(cam.H, cam.W, 0)
    Et = _t(R.make_exposure("on", rng))
    with torch.no_grad():
        raw, _, inv = pipeline.render_flat(pipeline.Scene(lv, requires_grad=False), dcam, fr["bg"], do_depth=True)
        fr["gt"] = ((torch.matmul(raw.permute(1, 2, 0), Et[:3, :3]).permute(2, 0, 1) + Et[:3, 3, None, None]).clamp(0, 1) * fr["M"]).contiguous()
        # away from the rendered inverse depth: where invdepth - mono is within rounding of 0 its sign, and with it the
        # whole depth gradient of the pixel, would follow the last bit of the parameters
        fr["mono"], fr["w"] = (0.9 * inv[0]).clone(), 0.05
    lv2 = dict(lv)
    lv2["shs"] = (lv["shs"] + 0.15 * rng.standard_normal(lv["shs"].shape)).astype(F)
    lv2["opacities"] = np.clip(lv["opacities"] * rng.uniform(0.6, 1.0, lv["opacities"].shape), 0.01, None).astype(F)
    E0 = torch.eye(3, 4, device="cuda")
    eager, Ee = _loop(lv2, fr, cam, E0, False)
    eager2, _ = _loop(lv2, fr, cam, E0, False)
    graphed, Eg = _loop(lv2, fr, cam, E0, True)
    assert np.isfinite(eager).all() and np.isfinite(graphed).all()
    assert eager[-1] < 0.8 * eager[0] and graphed[-1] < 0.8 * graphed[0], (eager[[0, -1]], graphed[[0, -1]])
    assert abs(graphed[0] - eager[0]) < 2e-7
    bar = max(20.0 * abs(eager2[-1] - eager[-1]), 1e-5 * eager[-1])
    print(f"\nfinal losses eager {eager[-1]:.9f} / {eager2[-1]:.9f}, graphed {graphed[-1]:.9f}; bar {bar:.3g}")
    assert abs(graphed[-1] - eager[-1]) <= bar
    assert float((Ee - E0).abs().max()) > 1e-3 and float((Eg - Ee).abs().max()) < 1e-4

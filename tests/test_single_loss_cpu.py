"""CPU: what train_single's objective adds to train_post's, on the emulation build -- the post-loss backward with the
exposure gradient, the inverse-depth L1 kernel, the densification statistics kernel and the status words -- against
tests/single_loss_ref.py's restatement (itself pinned against float64 torch autograd with the exposure as a leaf) and
against tests/golden/single_loss.npz, which the reference's render(), train_single loss lines and
add_densification_stats produced; then h3dgs.loss.single_loss, pipeline.single_step and the sync-free
h3dgs.singlestep.GraphedSingleStep (without graph capture) on CPU tensors."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "emul"))

import post_loss_ref as R  # noqa: E402
import single_loss_ref as SR  # noqa: E402
import ssim_ref as S  # noqa: E402
from test_post_loss_cpu import _ssim64, post_kernel_emu  # noqa: E402

F = np.float32


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    import build_emu
    return build_emu.build(str(tmp_path_factory.mktemp("h3dgs_emu_single")))


@pytest.fixture(scope="module")
def emu(emu_so):
    from emu_api import Emu
    return Emu(emu_so)


# ---- the restatement against float64 autograd ---------------------------------------------------------------------------
def _torch_single64(img, gt, lam, Ex, M, invd=None, mono=None, dmask=None, w=0.0):
    """render()'s exposure and clamp and train_single's loss lines in float64 autograd with the exposure as a leaf; y and a
    take the kernels' fp32 values straight through (see test_post_loss_cpu._torch_post64)"""
    import torch
    im = torch.tensor(img, dtype=torch.float64, requires_grad=True)
    Et = torch.tensor(np.eye(3, 4) if Ex is None else Ex, dtype=torch.float64, requires_grad=True)
    y = torch.matmul(im.permute(1, 2, 0), Et[:3, :3]).permute(2, 0, 1) + Et[:3, 3, None, None]
    y32, a32, _ = R.staged(img, Ex, M)
    y = y + (torch.tensor(y32, dtype=torch.float64) - y).detach()
    a = torch.clamp(y, 0.0, 1.0)
    if M is not None:
        a = a * torch.tensor(M, dtype=torch.float64)[None]
    a = a + (torch.tensor(a32, dtype=torch.float64) - a).detach()
    g = torch.tensor(gt, dtype=torch.float64)
    loss = (1.0 - lam) * (a - g).abs().mean() + lam * (1.0 - _ssim64(a, g))
    d = None
    if invd is not None:
        d = torch.tensor(invd, dtype=torch.float64, requires_grad=True)
        loss = loss + w * torch.abs((d - torch.tensor(mono, dtype=torch.float64)) * torch.tensor(dmask, dtype=torch.float64)).mean()
    loss.backward()
    return loss.item(), im.grad.numpy(), Et.grad.numpy(), None if d is None else d.grad.numpy()


@pytest.mark.parametrize("shape", [(1, 1), (11, 11), (17, 33)])
@pytest.mark.parametrize("exposure", R.EXPOSURES)
@pytest.mark.parametrize("mask", ["none", "binary", "fractional"])
def test_restatement_matches_float64_autograd(shape, exposure, mask):
    img, gt, Ex, M = R.make_inputs(*shape, exposure, mask, seed=21)
    r = SR.exposure_grad_reference(img, gt, 0.2, Ex, M)
    _, _, dE, _ = _torch_single64(img, gt, 0.2, Ex, M)
    mag = np.abs(r["dE"]).max() + 1e-300
    assert np.all(np.abs(r["dE"] - dE) <= 1e-11 * mag)


# ---- the kernels --------------------------------------------------------------------------------------------------------
def exposure_kernel_emu(emu, img, gt, Ex, M, k0, k1):
    """h3dgs_post_loss_forward + h3dgs_post_loss_backward_exposure -> (sums, grad, dE [3,4] float64)"""
    from emu_api import aligned, f32, ptr
    _, H, W = img.shape
    keep = [f32(img), f32(gt), None if Ex is None else f32(Ex), None if M is None else f32(M.reshape(H, W))]
    sums = aligned(16, np.float64, (2,))
    maps = aligned(9 * H * W * 4, np.float32, (3, 3, H, W))
    emu.check(emu.L.h3dgs_post_loss_forward(H, W, ptr(keep[0]), ptr(keep[1]), ptr(keep[2]), ptr(keep[3]), ptr(sums),
                                            ptr(maps), None))
    coeffs = f32(np.array([k0, k1], np.float32))
    grad = aligned(3 * H * W * 4, np.float32, (3, H, W))
    dE = aligned(96, np.float64, (3, 4))
    dE[...] = 7.0                                                  # the entry point zeroes it
    emu.check(emu.L.h3dgs_post_loss_backward_exposure(H, W, ptr(keep[0]), ptr(keep[1]), ptr(keep[2]), ptr(keep[3]), ptr(maps),
                                                      ptr(coeffs), ptr(grad), ptr(dE), None))
    return sums.copy(), grad.copy(), dE.copy()


@pytest.mark.parametrize("shape", [(1, 1), (1, 17), (16, 16), (17, 33), (33, 18)])
@pytest.mark.parametrize("exposure", R.EXPOSURES)
@pytest.mark.parametrize("mask", ["none", "binary", "fractional", "zero"])
def test_exposure_gradient_within_budget_and_dimg_bitwise(emu, shape, exposure, mask):
    img, gt, Ex, M = R.make_inputs(*shape, exposure, mask, seed=22)
    k0, k1 = S.loss_coefficients(0.2, float(img.size))
    _, grad, dE = exposure_kernel_emu(emu, img, gt, Ex, M, k0, k1)
    _, _, grad0 = post_kernel_emu(emu, img, gt, Ex, M, k0, k1)
    assert np.array_equal(grad.view(np.uint32), grad0.view(np.uint32))
    r = SR.exposure_grad_reference(img, gt, 0.2, Ex, M)
    ratio = np.abs(dE - r["dE"]) / r["dE_tol"]
    assert np.isfinite(dE).all() and ratio.max() <= 1.0, ratio
    if mask == "zero":
        assert np.all(dE == 0.0)


@pytest.mark.parametrize("content", ["saturated", "flat"])
def test_exposure_gradient_contents(emu, content):
    img, gt, Ex, M = R.make_inputs(17, 33, "offset", "fractional", content, seed=23)
    k0, k1 = S.loss_coefficients(0.2, float(img.size))
    _, _, dE = exposure_kernel_emu(emu, img, gt, Ex, M, k0, k1)
    r = SR.exposure_grad_reference(img, gt, 0.2, Ex, M)
    assert (np.abs(dE - r["dE"]) / r["dE_tol"]).max() <= 1.0


def depth_kernel_emu(emu, d, m, k, w):
    from emu_api import aligned, f32, ptr
    H, W = d.shape
    keep = [f32(d), f32(m), f32(k), f32(np.array([w], F))]
    grad = aligned(H * W * 4, np.float32, (H, W))
    grad[...] = 9.0
    tot = aligned(8, np.float64, (1,))
    tot[0] = 5.0
    emu.check(emu.L.h3dgs_invdepth_l1_grad(H, W, ptr(keep[0]), ptr(keep[1]), ptr(keep[2]), ptr(keep[3]), ptr(grad), ptr(tot), None))
    return grad.copy(), float(tot[0])


@pytest.mark.parametrize("shape", [(1, 1), (3, 5), (16, 16), (17, 33), (40, 52)])
@pytest.mark.parametrize("kind,w", [("random", 1.0), ("random", 0.37), ("random", 0.0), ("zero", 0.8)])
def test_invdepth_kernel(emu, shape, kind, w):
    d, m, k = SR.make_depth_inputs(*shape, kind, seed=24)
    grad, tot = depth_kernel_emu(emu, d, m, k, w)
    r = SR.depth_reference(d, m, k, w)
    assert np.array_equal(grad, r["grad"])                         # as values: sign(t) * 0 may be -0
    assert abs(tot - r["sum"]) <= r["sum_tol"]
    if w == 0.0 or kind == "zero":
        assert np.all(grad == 0.0)
    if kind == "zero":
        assert tot == 0.0
    else:
        assert np.all(grad[(d == m)] == 0.0)


def stats_kernel_emu(emu, radii, dm, mr, acc, den, info):
    from emu_api import aligned, f32, i32, ptr
    keep = [i32(radii), f32(dm), f32(mr), f32(acc), f32(den), None if info is None else i32(np.array(info, np.int32))]
    emu.check(emu.L.h3dgs_densify_stats(len(radii), ptr(keep[0]), ptr(keep[1]), ptr(keep[2]), ptr(keep[3]), ptr(keep[4]),
                                        ptr(keep[5]), None))
    return keep[2].copy(), keep[3].copy(), keep[4].copy()


def _stats_inputs(P, seed):
    rng = np.random.default_rng(seed)
    radii = (rng.integers(-2, 50, P) * (rng.uniform(size=P) > 0.4)).astype(np.int32)
    dm = rng.standard_normal((P, 3)).astype(F) * F(1e-3)
    dm[:, 2] = 0.0
    mr = (rng.integers(0, 60, P) * (rng.uniform(size=P) > 0.5)).astype(F)
    acc = (np.abs(rng.standard_normal((P, 1))) * 1e-3 * (rng.uniform(size=(P, 1)) > 0.5)).astype(F)
    den = rng.integers(0, 9, (P, 1)).astype(F)
    return radii, dm, mr, acc, den


@pytest.mark.parametrize("P", [1, 255, 256, 257, 1000])
@pytest.mark.parametrize("info", [None, (123, 7, 0, 0)])
def test_densify_stats_kernel_bitwise(emu, P, info):
    radii, dm, mr, acc, den = _stats_inputs(P, 25)
    got = stats_kernel_emu(emu, radii, dm, mr, acc, den, info)
    want = SR.stats_reference(radii, dm, mr, acc, den)
    for g, w in zip(got, want):
        assert np.array_equal(g.view(np.uint32), w.view(np.uint32))
    assert np.array_equal(got[2][radii <= 0], den[radii <= 0])


def test_densify_stats_kernel_does_nothing_for_an_overflowed_frame(emu):
    radii, dm, mr, acc, den = _stats_inputs(700, 26)
    assert (radii > 0).sum() > 100
    got = stats_kernel_emu(emu, radii, dm, mr, acc, den, (123, 7, 1, 0))
    for g, w in zip(got, (mr, acc, den)):
        assert np.array_equal(g.view(np.uint32), w.view(np.uint32))


def test_stats_restatement_is_the_torch_lines():
    """train_single.py:147 and gaussian_model.py:687-689 as torch evaluates them on the CPU; torch.norm may fuse its
    multiply-add, so the norm is compared to within two ulps and everything else exactly"""
    import torch
    radii, dm, mr, acc, den = _stats_inputs(500, 27)
    radii = np.maximum(radii, 0)
    want = SR.stats_reference(radii, dm, mr, acc, den)
    t_mr, t_acc, t_den, g = torch.tensor(mr), torch.tensor(acc), torch.tensor(den), torch.tensor(dm)
    vis = (torch.tensor(radii) > 0).nonzero().flatten()
    t_mr[vis] = torch.max(t_mr[vis], torch.tensor(radii)[vis])
    t_acc[vis] = torch.max(torch.norm(g[vis, :2], dim=-1, keepdim=True), t_acc[vis])
    t_den[vis] += 1
    assert np.array_equal(t_mr.numpy(), want[0]) and np.array_equal(t_den.numpy(), want[2])
    assert np.all(np.abs(t_acc.numpy() - want[1]) <= 2 * np.spacing(want[1]))


def test_status_words(emu):
    from emu_api import aligned, f32, i32, ptr
    sums = aligned(16, np.float64, (2,)); sums[:] = (30.0, 240.0)
    dsum = aligned(8, np.float64, (1,)); dsum[0] = 50.0
    w = f32(np.array([0.25], F))
    info = i32(np.array([1234, 77, 0, 0], np.int32))
    dE = aligned(96, np.float64, (3, 4)); dE[...] = np.arange(12).reshape(3, 4) / 3.0
    eg = aligned(48, np.float32, (3, 4))
    out = aligned(64, np.float64, (8,))
    call = lambda: emu.check(emu.L.h3dgs_single_step_status(ptr(sums), ptr(dsum), ptr(w), 1.0 / 300, 1.0 / 100, 0.2, ptr(info),
                                                            ptr(dE), ptr(eg), ptr(out), None))
    call()
    photo = 0.8 * 0.1 + 0.2 * (1 - 0.8)
    assert np.allclose(out, [photo + 0.25 * 0.5, photo, 0.1, 0.8, 0.5, 1234, 77, 0], rtol=1e-15)
    assert np.array_equal(eg, dE.astype(F))
    info[2] = 1
    call()
    assert out[7] == 1.0 and np.all(eg == 0.0)
    emu.check(emu.L.h3dgs_single_step_status(ptr(sums), None, None, 1.0 / 300, 1.0 / 100, 0.2, ptr(info), None, None, ptr(out), None))
    assert out[0] == out[1] and out[4] == 0.0


# ---- against the reference's own lines ----------------------------------------------------------------------------------
@pytest.mark.parametrize("i", range(6))
def test_kernels_match_the_reference(emu, golden_dir, i):
    z = np.load(os.path.join(golden_dir, "single_loss.npz"))
    assert i < int(z["cases"])
    msk, dep = (bool(v) for v in z[f"c{i}_flags"])
    raw, gt, Ex = z[f"c{i}_raw"], z[f"c{i}_gt"], z[f"c{i}_E"]
    M = z[f"c{i}_mask"] if msk else None
    lam, n = float(z["lam"]), float(raw.size)
    k0, k1 = S.loss_coefficients(lam, n)
    sums, grad, dE = exposure_kernel_emu(emu, raw, gt, Ex, M, k0, k1)
    l1, ssim = sums[0] / n, sums[1] / n
    photo = (1 - lam) * l1 + lam * (1 - ssim)
    assert abs(l1 - float(z[f"c{i}_l1"])) < 1e-6 and abs(photo - float(z[f"c{i}_photo"])) < 1e-6
    ref = z[f"c{i}_grad"]
    assert np.abs(grad - ref).max() <= 1e-5 * max(np.abs(ref).max(), 1e-30)
    refE = z[f"c{i}_dE"]
    assert np.abs(dE - refE).max() <= 2e-5 * np.abs(refE).max()
    w = float(z[f"c{i}_weight"]) if dep else 0.0
    dinv, tot = depth_kernel_emu(emu, z[f"c{i}_invdepth"], z[f"c{i}_mono"], z[f"c{i}_dmask"], w)
    assert np.abs(dinv - z[f"c{i}_dinv"]).max() <= 1e-6 * max(np.abs(z[f"c{i}_dinv"]).max(), 1e-30)
    if dep:
        assert abs(tot / (n / 3) - float(z[f"c{i}_depth"])) < 1e-6
        assert abs(photo + w * tot / (n / 3) - float(z[f"c{i}_loss"])) < 1e-6
    # the statistics run on through the cases
    P = len(z[f"c{i}_radii"])
    prev = [z[f"c{i - 1}_{k}"] for k in ("max_radii2D", "accum", "denom")] if i else [np.zeros(P, F), np.zeros((P, 1), F), np.zeros((P, 1), F)]
    got = stats_kernel_emu(emu, z[f"c{i}_radii"], z[f"c{i}_dmeans2D"], *prev, None)
    assert np.array_equal(got[0], z[f"c{i}_max_radii2D"]) and np.array_equal(got[2].reshape(P, 1), z[f"c{i}_denom"])
    assert np.all(np.abs(got[1].reshape(P, 1) - z[f"c{i}_accum"]) <= 2 * np.spacing(z[f"c{i}_accum"]))


# ---- the Python layer on CPU tensors ------------------------------------------------------------------------------------
@pytest.mark.parametrize("exposure_shape", [(3, 4), (4, 4)])
def test_single_loss_autograd(emu_so, exposure_shape):
    import torch
    from fake_device import cpu_as_device
    img, gt, Ex, M = R.make_inputs(17, 33, "offset", "fractional", seed=28)
    d, m, k = SR.make_depth_inputs(17, 33, seed=29)
    loss64, gim, gE, gd = _torch_single64(img, gt, 0.2, Ex, M, d, m, k, 0.6)
    Efull = np.zeros(exposure_shape, F)
    Efull[:3, :4] = Ex
    if exposure_shape[0] == 4:
        Efull[3, 3] = 1.0
    with cpu_as_device(emu_so):
        from h3dgs.loss import single_loss
        x = torch.tensor(img, requires_grad=True)
        inv = torch.tensor(d[None], requires_grad=True)
        E = torch.tensor(Efull, requires_grad=True)
        out = single_loss(x, inv, torch.tensor(gt), 0.2, E, torch.tensor(M[None]), torch.tensor(m[None]), torch.tensor(k[None]), 0.6)
        out[0].backward()
        o = [float(v.detach()) for v in out]
        assert abs(o[0] - loss64) < 1e-6 and abs(o[0] - o[1] - 0.6 * o[4]) < 1e-6
        assert E.grad.shape == exposure_shape and np.abs(E.grad.numpy()[:3, :4] - gE).max() <= 1e-5 * np.abs(gE).max()
        if exposure_shape[0] == 4:
            assert float(E.grad[3].abs().sum()) == 0.0
        assert np.abs(x.grad.numpy() - gim).max() <= 1e-5 * np.abs(gim).max()
        assert inv.grad.shape == (1, 17, 33) and np.abs(inv.grad.numpy()[0] - gd).max() <= 1e-6 * np.abs(gd).max()
        # a frozen exposure takes the plain backward; no depth term without a mono map or with weight 0
        x2 = torch.tensor(img, requires_grad=True)
        out2 = single_loss(x2, None, torch.tensor(gt), 0.2, torch.tensor(Efull), torch.tensor(M))
        out2[0].backward()
        assert torch.equal(x2.grad, x.grad) and float(out2[4].detach()) == 0.0 and torch.equal(out2[0], out2[1])
        out3 = single_loss(x2, inv, torch.tensor(gt), 0.2, None, None, torch.tensor(m), None, 0.0)
        assert float(out3[4].detach()) == 0.0


def _flat_scene(n=1500, W=96, H=64):
    from h3dgs import synth
    cam = synth.make_camera(W, H)
    lv = synth.cloud_v1(n, cam, zmin=2.0, zmax=40.0, seed=3, scale_k=1.0)
    z = lv["means3D"][:, 2:3]
    lv["scales"] = (1.5e-2 * np.sqrt(2.0 * z) * np.exp(0.4 * np.random.default_rng(1).standard_normal((z.shape[0], 3)))).astype(F)
    return cam, lv


def test_single_step_and_sync_free_step(emu_so):
    """pipeline.single_step against its parts, and GraphedSingleStep (no capture) against single_step over steps with
    every input changing and both slots in use; then an overflowed frame"""
    import torch
    from fake_device import cpu_as_device
    from h3dgs import synth
    from util import rel_err
    cam, lv = _flat_scene()
    H, W = cam.H, cam.W
    with cpu_as_device(emu_so):
        from diff_gaussian_rasterization import _C as rc
        from h3dgs import pipeline
        from h3dgs.singlestep import GraphedSingleStep
        scene = pipeline.Scene(lv, device="cpu")
        with pytest.raises(ValueError, match="one GPU"):
            GraphedSingleStep(scene, W, H, cam.tanfovx, cam.tanfovy, world=2, capture=False)
        dcams = [pipeline.DeviceCamera(c, device="cpu") for c in
                 (cam, synth.yaw_camera(W, H, 8.0, np.array([0.2, -0.1, 0.3])))]
        ref_stats = pipeline.DensifyStats(scene.means3D.shape[0], "cpu")
        gs = None
        side = torch.cuda.Stream()
        for k in range(4):
            rng = np.random.default_rng(300 + k)
            bg = torch.tensor(rng.uniform(0, 1, 3).astype(F))
            M = torch.tensor(R.make_mask(["binary", "fractional", "none", "half"][k], H, W, rng)) if k != 2 else None
            gt = torch.tensor(rng.uniform(0, 1, (3, H, W)).astype(F)) * (1.0 if M is None else M[None])
            E = torch.tensor(R.make_exposure("offset" if k % 2 else "on", rng), requires_grad=True)
            d, m, dm = SR.make_depth_inputs(H, W, seed=400 + k)
            mono, dmask = (torch.tensor(m), torch.tensor(dm)) if k != 3 else (None, None)
            w = [1.0, 0.3, 0.0, 0.5][k]
            before = [t.clone() for t in (ref_stats.max_radii2D, ref_stats.xyz_gradient_accum, ref_stats.denom)]
            out, radii, means2D = pipeline.single_step(scene, dcams[k % 2], bg, gt, 0.2, E, M, mono, dmask, w, ref_stats)
            D = rc.last_num_rendered()
            exact = {n: getattr(scene, n).grad.clone() for n in ("means3D", "scales", "shs", "opacities", "rotations")}
            want = SR.stats_reference(radii.numpy(), means2D.grad.numpy(), *[b.numpy() for b in before])
            for got, wnt in zip((ref_stats.max_radii2D, ref_stats.xyz_gradient_accum, ref_stats.denom), want):
                assert np.array_equal(got.numpy(), wnt)
            assert float(ref_stats.denom.sum()) > 0
            if gs is None:
                gs = GraphedSingleStep(scene, W, H, cam.tanfovx, cam.tanfovy, mask=True, bin_capacity=4 * D + 1000,
                                       sort_capacity=4096, capture=False)
            gs.set_background(bg)
            gs.set_depth_weight(w)
            if k % 2:
                gs.step(dcams[k % 2], gt, mask=M, mono_invdepth=mono, depth_mask=dmask, exposure=E)
            else:
                ready = gs.upload_target(gt, side, M, mono, dmask)
                gs.step(dcams[k % 2], exposure=E, gt_ready=ready)
            st = gs.status()
            with torch.no_grad():
                img, _, inv = pipeline.render_flat(scene, dcams[k % 2], bg, do_depth=True)
            assert not st["overflow"] and st["D"] == D
            assert torch.equal(gs.image, img) and torch.equal(gs.invdepth, inv) and torch.equal(gs.radii, radii)
            for key, v in zip(("loss", "photo", "l1", "ssim", "depth_l1"), out):
                assert abs(st[key] - float(v.detach())) < 1e-6, (k, key)
            assert np.abs((gs.exposure_grad - E.grad).numpy()).max() <= 1e-6 * float(E.grad.abs().max())
            assert torch.equal(gs.d_means2D, means2D.grad)
            for n, g in exact.items():
                assert rel_err(gs.grads[n].numpy(), g.numpy()) < 2e-6, (k, n)
            for a, b in zip((gs.stats.max_radii2D, gs.stats.xyz_gradient_accum, gs.stats.denom),
                            (ref_stats.max_radii2D, ref_stats.xyz_gradient_accum, ref_stats.denom)):
                assert torch.equal(a, b)
        # a frame that does not fit: flagged, background only, zero gradients (the exposure's too), statistics untouched
        small = GraphedSingleStep(scene, W, H, cam.tanfovx, cam.tanfovy, mask=True, bin_capacity=D // 3, sort_capacity=4096,
                                  stats=pipeline.DensifyStats(scene.means3D.shape[0], "cpu"), capture=False)
        small.set_depth_weight(0.5)
        small.step(dcams[1], gt, mask=M, mono_invdepth=torch.tensor(m), exposure=E, bg=bg)
        st = small.status()
        assert st["overflow"] and bool((small.radii > 0).any())
        assert torch.equal(small.image, bg.view(3, 1, 1).expand_as(small.image))
        assert all(float(g.abs().sum()) == 0.0 for g in small.grads.values()) and float(small.exposure_grad.abs().sum()) == 0.0
        assert float(small.stats.denom.sum()) == 0.0 and float(small.stats.max_radii2D.sum()) == 0.0
        with pytest.raises(ValueError, match="rows"):
            GraphedSingleStep(scene, W, H, cam.tanfovx, cam.tanfovy, stats=pipeline.DensifyStats(7, "cpu"), capture=False)
        with pytest.raises(ValueError, match="rows"):
            pipeline.single_step(scene, dcams[0], bg, gt, stats=pipeline.DensifyStats(7, "cpu"))
        # the eager step capture() starts with sees this camera, and does not count
        carried = [t.clone() for t in (gs.stats.max_radii2D, gs.stats.xyz_gradient_accum, gs.stats.denom)]
        gs._warm_up()
        assert bool((gs.radii > 0).any()) and gs._count_stats
        for a, b in zip((gs.stats.max_radii2D, gs.stats.xyz_gradient_accum, gs.stats.denom), carried):
            assert torch.equal(a, b)

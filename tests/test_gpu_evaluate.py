"""GPU: the sync-free evaluator of render_hierarchy.py's tau sweep (h3dgs.evaluate, csrc/metrics.cu).

  * the metrics kernel (nvcc build) against the fixture the reference's own render_post / psnr / ssim computed;
  * GraphedRender's images bit-identical to pipeline.render_hier_fused (same kernels, same order), skybox rows included;
  * evaluate_hierarchy against a per-frame loop of the drop-in flow (pipeline.render_hier) + PyTorch PSNR + h3dgs.loss.ssim,
    with exposure, mask and train_test_exp on and off;
  * overflowed frames re-run through the exact path, final numbers those of an ample capacity;
  * no host synchronisation inside the sweep."""
import os

import numpy as np
import pytest

from h3dgs import synth

pytestmark = pytest.mark.gpu

TAUS = [0.0, 3.0, 6.0, 15.0]


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


@pytest.mark.parametrize("i", range(9))
def test_metrics_kernel_matches_the_reference(golden_dir, i):
    import torch
    from h3dgs import _lib
    from h3dgs.evaluate import _metrics
    z = np.load(os.path.join(golden_dir, "eval_metrics.npz"))
    exp, msk, crop, _ = (bool(v) for v in z[f"c{i}_flags"])
    t = lambda k: torch.tensor(z[f"c{i}_{k}"], device="cuda")
    raw, gt = t("raw"), t("gt")
    _, H, W = raw.shape
    x0 = W // 2 if crop else 0
    out = torch.zeros((3, H, W - x0), device="cuda")
    results = torch.zeros((1, _lib.EVAL_ROW), dtype=torch.float64, device="cuda")
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    sums = torch.zeros(4, dtype=torch.float64, device="cuda")
    _metrics(_lib.lib(), H, W, raw, gt, t("E") if exp else None, t("mask") if msk else None, x0, out, sums, counter, results,
             torch.cuda.current_stream().cuda_stream)
    assert float((out.cpu() - torch.tensor(z[f"c{i}_image"])).abs().max()) <= 1e-6
    p, s = results[0, 0].item(), results[0, 1].item()
    pr, sr = float(z[f"c{i}_psnr"]), float(z[f"c{i}_ssim"])
    assert (np.isinf(p) and p > 0) if np.isinf(pr) else abs(p - pr) <= 1e-4, (p, pr)
    assert abs(s - sr) <= 1e-5 * abs(sr), (s, sr)


@pytest.mark.parametrize("skybox", [0, 200])
def test_graphed_render_images_equal_the_fused_path(skybox):
    import torch
    from h3dgs import pipeline
    from h3dgs.evaluate import GraphedRender
    cam, h = _scene(skybox=skybox)
    scene = pipeline.Scene(h, requires_grad=False)
    bg = torch.tensor([0.2, 0.1, 0.3], device="cuda")
    dcams = [pipeline.DeviceCamera(c) for c in _cams(cam.W, cam.H)]
    gr = GraphedRender(scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, bg, pipeline.fov_threshold(0.0, cam),
                       bin_capacity=1 << 20, sort_capacity=4096)
    assert gr.launches_per_frame >= 5
    k = 0
    for dcam in dcams:
        for tau in TAUS:
            thr = pipeline.fov_threshold(tau, dcam)
            with torch.no_grad():
                img, radii, n = pipeline.render_hier_fused(scene, dcam, bg, thr)
            gr.set_camera(dcam)
            gr.set_threshold(thr)
            gr.frame()
            k += 1
            assert torch.equal(gr.image, img), (tau, float((gr.image - img).abs().max()))
            row = gr.results[k - 1].cpu().numpy()
            assert row[2] == 0.0 and row[3] == n + skybox and torch.equal(gr.radii[:n + skybox], radii)
    assert int(gr.counter.item()) == k


def _targets(scene, dcams, bg, seed=4):
    """target = a finer render (tau 0) with seeded noise, beyond [0, 1] in places"""
    import torch
    from h3dgs import pipeline
    g = torch.Generator(device="cpu").manual_seed(seed)
    out = []
    for c in dcams:
        with torch.no_grad():
            img = pipeline.render_hier_fused(scene, c, bg, pipeline.fov_threshold(0.0, c))[0]
        out.append((img + 0.03 * torch.randn(img.shape, generator=g).cuda()).contiguous())
    return out


def _reference_loop(scene, dcams, targets, taus, masks, exposures, train_test_exp, bg):
    """render_hierarchy.py:48-119 on the drop-in flow (render_post = pipeline.render_hier + exposure + clamp)"""
    import torch
    from h3dgs import pipeline
    from h3dgs.loss import ssim
    out = {}
    for tau in taus:
        ps, ss, imgs = 0.0, 0.0, []
        for ci, c in enumerate(dcams):
            with torch.no_grad():
                image = pipeline.render_hier(scene, c, bg, pipeline.fov_threshold(tau, c))[0]
                if exposures is not None and exposures[ci] is not None:
                    E = exposures[ci]
                    image = torch.matmul(image.permute(1, 2, 0), E[:3, :3]).permute(2, 0, 1) + E[:3, 3, None, None]
                image = image.clamp(0, 1)
                gt = torch.clamp(targets[ci], 0.0, 1.0)
                mask = masks[ci] if masks is not None else torch.ones((1, c.H, c.W), device="cuda")
                if train_test_exp:
                    image, gt, mask = image[..., image.shape[-1] // 2:], gt[..., gt.shape[-1] // 2:], mask[..., mask.shape[-1] // 2:]
                imgs.append(image.clone())
                image = image * mask
                gt = gt * mask
                mse = ((image - gt) ** 2).view(3, -1).mean(1, keepdim=True)
                ps += float((20 * torch.log10(1.0 / torch.sqrt(mse))).mean().double())
                ss += float(ssim(image.contiguous(), gt.contiguous()).double())
        out[tau] = (ps / len(dcams), ss / len(dcams), imgs)
    return out


@pytest.mark.parametrize("exposure,mask,tte", [(False, False, False), (True, False, False), (False, True, False),
                                               (False, False, True), (True, True, True)])
def test_evaluate_hierarchy_matches_the_drop_in_loop(exposure, mask, tte):
    import torch
    from h3dgs import pipeline
    from h3dgs.evaluate import evaluate_hierarchy
    cam, h = _scene(skybox=100)
    scene = pipeline.Scene(h, requires_grad=False)
    bg = torch.zeros(3, device="cuda")
    dcams = [pipeline.DeviceCamera(c) for c in _cams(cam.W, cam.H)]
    targets = _targets(scene, dcams, bg)
    rng = np.random.default_rng(8)
    masks = [torch.tensor((rng.uniform(size=(1, cam.H, cam.W)) > 0.2).astype(np.float32), device="cuda") for _ in dcams] if mask else None
    exposures = None
    if exposure:
        exposures = []
        for k in range(len(dcams)):
            E = np.zeros((3, 4), np.float32)
            E[:, :3] = np.eye(3) * 1.05 + rng.uniform(-0.08, 0.08, (3, 3))
            E[:, 3] = rng.uniform(-0.03, 0.03, 3)
            exposures.append(torch.tensor(E, device="cuda"))
        exposures[1] = None                         # a camera without an exposure: render_post leaves its image as it is
    ref = _reference_loop(scene, dcams, targets, TAUS, masks, exposures, tte, bg)
    res = evaluate_hierarchy(scene, dcams, targets, TAUS, masks=masks, exposures=exposures, train_test_exp=tte,
                             keep_images=True)
    assert res["rows"].shape == (len(TAUS), len(dcams), 6)
    for ti, tau in enumerate(TAUS):
        p, s, imgs = ref[tau]
        assert abs(res["psnr"][tau] - p) <= 1e-4, (tau, res["psnr"][tau], p)
        assert abs(res["ssim"][tau] - s) <= 1e-5 * abs(s), (tau, res["ssim"][tau], s)
        assert 5.0 < p < 60.0 and 0.01 < s <= 1.0
        for ci in range(len(dcams)):
            # the drop-in lerp and the fused one differ in the last bits of a few Gaussians: allow a few flipped pixels
            d = (res["images"][ti][ci] - imgs[ci]).abs()
            assert res["images"][ti][ci].shape == imgs[ci].shape and float((d > 1e-5).float().mean()) < 1e-3


def test_overflowed_frames_are_rerun_and_equal_an_ample_capacity():
    import torch
    from h3dgs import pipeline
    from h3dgs.evaluate import evaluate_hierarchy
    cam, h = _scene(skybox=50)
    scene = pipeline.Scene(h, requires_grad=False)
    bg = torch.zeros(3, device="cuda")
    dcams = [pipeline.DeviceCamera(c) for c in _cams(cam.W, cam.H)]
    targets = _targets(scene, dcams, bg)
    ample = evaluate_hierarchy(scene, dcams, targets, TAUS,
                               capacities=dict(row_capacity=scene.means3D.shape[0], bin_capacity=1 << 21, sort_capacity=8192))
    assert ample["rerun"] == 0
    learned = evaluate_hierarchy(scene, dcams, targets, TAUS)          # re-runs, if any, are exact: the same numbers
    for tau in TAUS:
        assert abs(learned["psnr"][tau] - ample["psnr"][tau]) <= 1e-9 and abs(learned["ssim"][tau] - ample["ssim"][tau]) <= 1e-12
    D = ample["rows"][..., 4]
    rows = ample["rows"][..., 3]
    for caps in (dict(row_capacity=int(np.median(rows)), bin_capacity=int(D.max()) + 1, sort_capacity=4096),
                 dict(row_capacity=int(rows.max()), bin_capacity=int(np.median(D)), sort_capacity=4096)):
        small = evaluate_hierarchy(scene, dcams, targets, TAUS, capacities=caps)
        assert 0 < small["rerun"] < len(TAUS) * len(dcams)
        for tau in TAUS:
            assert abs(small["psnr"][tau] - ample["psnr"][tau]) <= 1e-9
            assert abs(small["ssim"][tau] - ample["ssim"][tau]) <= 1e-12
        assert np.array_equal(small["rows"][..., 3], rows)


def test_the_sweep_never_synchronises_the_host():
    import torch
    from h3dgs import pipeline
    from h3dgs.evaluate import HierarchyEvaluator
    cam, h = _scene(skybox=30)
    scene = pipeline.Scene(h, requires_grad=False)
    bg = torch.zeros(3, device="cuda")
    # two camera sizes -> two graphed instances; host targets and masks (pinned by the evaluator)
    cams = _cams(cam.W, cam.H) + [synth.make_camera(320, 200)]
    dcams = [pipeline.DeviceCamera(c) for c in cams]
    targets = [t.cpu() for t in _targets(scene, dcams, bg)]
    masks = [torch.ones((1, c.H, c.W)) for c in cams]
    ev = HierarchyEvaluator(scene, dcams, targets, TAUS, masks=masks, train_test_exp=True)
    assert len(ev.renders) == 2
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ev.enqueue()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    res = ev.finish()
    assert set(res["psnr"]) == set(TAUS) and res["rows"].shape == (len(TAUS), len(cams), 6)
    assert all(np.isfinite(v) for v in res["psnr"].values())

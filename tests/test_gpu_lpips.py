"""GPU: LPIPS with the VGG16 network (csrc/lpips.cu, h3dgs.lpips, the evaluator's lpips=).

  * every conv layer on its own input against float64, within (2^-10 + 2^-21 + (K+1) 2^-23)(sum |w||x| + |b|), at odd
    sizes and at the levels of a 1920x1080 frame;
  * the head on our own taps against float64 within its budget; an identical pair gives exactly 0.0;
  * end to end over a case matrix: max |ours - f64| <= 2 max |torch TF32 cuDNN - f64| + 1e-7, the torch run being the
    same net restated here with TF32 on (the reference's own GPU arithmetic); the golden's values within that budget;
  * the evaluator form (clamp, crop, mask inside the kernels) equal to lpips() on the preprocessed pair, bit for bit;
  * determinism: two calls, and a graph replay, give the same bits;
  * errors below 16 px and on malformed weights;
  * evaluate_hierarchy(lpips=net): each frame equals net(...) on its exposed, clamped, cropped, masked pair; re-run
    frames equal an ample capacity's; the sweep never synchronises the host; lpips=None leaves the output as it was."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import lpips_ref  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def weights():
    return lpips_ref.seeded_state_dicts(20240)


@pytest.fixture(scope="module")
def net(weights):
    from h3dgs.lpips import LpipsVGG
    return LpipsVGG.from_state_dicts(*weights)


def _conv(net, layer, x):
    """our layer on x [H,W,C_in] (device) -> [H,W,C_out]"""
    import torch
    from h3dgs import _lib
    H, W, _ = x.shape
    out = torch.empty((H, W, lpips_ref.CONV_CHANNELS[layer][1]), device="cuda")
    _lib.check(net.L.h3dgs_lpips_conv(layer, H, W, x.contiguous().data_ptr(), net.weights.data_ptr(), out.data_ptr(),
                                      torch.cuda.current_stream().cuda_stream))
    return out


def _budget_used(weights, layer, x, ours):
    """the largest fraction of the per-layer budget ours [H,W,C_out] uses against float64 on x [H,W,C_in]"""
    import torch
    import torch.nn.functional as F
    vgg = weights[0]
    i, ci = lpips_ref.CONV_INDICES[layer], lpips_ref.CONV_CHANNELS[layer][0]
    w, b = vgg[f"features.{i}.weight"].cuda().double(), vgg[f"features.{i}.bias"].cuda().double()
    xin = x[..., :ci].permute(2, 0, 1)[None].double()
    ref = F.relu(F.conv2d(xin, w, b, padding=1))[0]
    bound = (F.conv2d(xin.abs(), w.abs(), padding=1) + b.abs()[:, None, None])[0]
    K = 9 * max(ci, 8)
    frac = float(((ours.permute(2, 0, 1).double() - ref).abs() / lpips_ref.layer_budget(K, bound)).max())
    del ref, bound
    torch.cuda.empty_cache()
    return frac


def _input(x):
    import torch
    z = lpips_ref.z_score(x.cpu()).float()
    out = torch.zeros(x.shape[1], x.shape[2], 8)
    out[..., :3] = z.permute(1, 2, 0)
    return out.cuda()


@pytest.mark.parametrize("layer", range(13))
def test_conv_layer_within_budget_at_odd_sizes(net, weights, layer):
    import torch
    g = torch.Generator().manual_seed(layer)
    for H, W in ((37, 53), (8, 16), (17, 5), (70, 129)):
        if layer == 0:
            x = _input(torch.rand((3, H, W), generator=g))
        else:
            x = torch.relu(torch.randn((H, W, lpips_ref.CONV_CHANNELS[layer][0]), generator=g)).cuda()
        used = _budget_used(weights, layer, x, _conv(net, layer, x))
        assert used <= 1.0, (layer, H, W, used)


def test_conv_layers_within_budget_at_1080p(net, weights):
    """the 13 layers of a 1920x1080 frame, each on the previous layer's (our) output; prints the budget used per layer"""
    import torch
    import torch.nn.functional as F
    x = _input(torch.rand((3, 1080, 1920), generator=torch.Generator().manual_seed(7)))
    used = []
    for layer in range(13):
        if layer in lpips_ref.POOL_BEFORE:
            x = F.max_pool2d(x.permute(2, 0, 1)[None], 2)[0].permute(1, 2, 0).contiguous()
        y = _conv(net, layer, x)
        used.append(_budget_used(weights, layer, x, y))
        x = y
    print("largest fraction of the per-layer budget used at 1920x1080:", [round(u, 4) for u in used])
    assert max(used) <= 1.0, used


def _taps(net, frame):
    net.features(frame)
    H, W = frame.shape[-2:]
    return lpips_ref.split_taps(net.scratch(H, W)["taps"].cpu().clone(), H, W)


def test_head_within_budget_and_identical_pair_is_zero(net, weights):
    import torch
    g = torch.Generator().manual_seed(3)
    for H, W in ((37, 53), (270, 480)):
        x = torch.rand((3, H, W), generator=g).cuda()
        y = (x + 0.1 * torch.randn((3, H, W), generator=g).cuda()).clamp(0, 1)
        tx, ty = _taps(net, x), _taps(net, y)
        value = float(net(x, y))
        ref = sum(lpips_ref.head(tx, ty, weights[1]))
        assert abs(value - ref) <= sum(lpips_ref.head_bound(tx, ty, weights[1])), (H, W, value, ref)
        assert float(net(x, x.clone())) == 0.0


def _torch_net(weights):
    """the same network in torch on the GPU, TF32 cuDNN convolutions, channels-last, weights loaded once"""
    import torch
    import torch.nn.functional as F
    vgg, lin = weights
    ws = [(vgg[f"features.{i}.weight"].cuda(), vgg[f"features.{i}.bias"].cuda()) for i in lpips_ref.CONV_INDICES]
    ls = [lin[f"lin{k}.model.1.weight"].cuda() for k in range(5)]
    mean, std = lpips_ref.MEAN.cuda()[None, :, None, None], lpips_ref.STD.cuda()[None, :, None, None]

    def feats(x):
        x = ((x[None] - mean) / std).contiguous(memory_format=torch.channels_last)
        out = []
        for l, (w, b) in enumerate(ws):
            if l in lpips_ref.POOL_BEFORE:
                x = F.max_pool2d(x, 2)
            x = F.relu(F.conv2d(x, w, b, padding=1))
            if l in lpips_ref.TAP_AFTER:
                out.append(x / (torch.sqrt((x * x).sum(1, keepdim=True)) + 1e-10))
        return out

    def run(x, y):
        with torch.no_grad():
            res = [F.conv2d((a - b) ** 2, l).mean((2, 3), True) for a, b, l in zip(feats(x), feats(y), ls)]
            return torch.sum(torch.cat(res, 0), 0, True)
    return run


def _case_matrix(golden):
    import torch
    cases = []
    for name in golden["names"]:
        prep, use_mask, crop, _ = (bool(v) for v in golden[f"{name}_flags"])
        x, y = torch.from_numpy(golden[f"{name}_x"]), torch.from_numpy(golden[f"{name}_y"])
        m = torch.from_numpy(golden[f"{name}_mask"]) if use_mask else None
        cases.append((str(name), x, y, m, crop, prep))
    g = torch.Generator().manual_seed(11)
    for H, W in ((135, 241), (270, 480)):
        x = torch.rand((3, H, W), generator=g)
        cases.append((f"rand_{H}x{W}", x, (x + 0.1 * torch.randn((3, H, W), generator=g)).clamp(0, 1), None, False, False))
    return cases


def test_end_to_end_against_float64_and_torch_tf32(net, weights, golden_dir):
    import torch
    golden = np.load(os.path.join(golden_dir, "lpips.npz"))
    torch_run = _torch_net(weights)
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        err_ours, err_torch, rows = [], [], []
        for name, x, y, m, crop, prep in _case_matrix(golden):
            if prep:
                x, y = lpips_ref.preprocess(x, m, crop), lpips_ref.preprocess(y, m, crop)
            f64 = lpips_ref.lpips(x, y, *weights)[1]
            ours = float(net(x.cuda(), y.cuda()))
            tt = float(torch_run(x.cuda(), y.cuda()))
            err_ours.append(abs(ours - f64)); err_torch.append(abs(tt - f64))
            rows.append((name, ours, tt, f64))
    finally:
        torch.backends.cudnn.allow_tf32 = old
    budget = 2 * max(err_torch) + 1e-7
    print("end to end: max |ours - f64| =", max(err_ours), " max |torch TF32 - f64| =", max(err_torch))
    assert max(err_ours) <= budget, rows
    for name in golden["names"]:
        ours = [r[1] for r in rows if r[0] == str(name)][0]
        assert abs(ours - float(golden[f"{name}_value"])) <= budget, (name, ours, float(golden[f"{name}_value"]))


def test_evaluator_form_equals_lpips_on_the_preprocessed_pair(net, golden_dir):
    import torch
    golden = np.load(os.path.join(golden_dir, "lpips.npz"))
    for name, x, y, m, crop, prep in _case_matrix(golden):
        if not prep:
            continue
        H, W = x.shape[-2:]
        x0 = W // 2 if crop else 0
        xc, yc = x.cuda(), y.cuda()
        mc = None if m is None else m.cuda().contiguous()
        out = torch.zeros(1, dtype=torch.float64, device="cuda")
        net.features(yc, x0, None, mc, clamp=True)
        net.distance(xc, out, x0, None, mc, clamp=True)
        want = net(lpips_ref.preprocess(xc, mc, crop), lpips_ref.preprocess(yc, mc, crop))
        assert torch.equal(out.view(1, 1, 1, 1), want), name


def test_same_bits_on_rerun_and_graph_replay(net):
    import torch
    g = torch.Generator().manual_seed(9)
    x, y = torch.rand((3, 67, 123), generator=g).cuda(), torch.rand((1, 3, 67, 123), generator=g).cuda()
    a, b = net(x, y), net(x, y)
    assert a.shape == (1, 1, 1, 1) and a.dtype == torch.float64 and torch.equal(a, b)
    out = torch.zeros(1, dtype=torch.float64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        net.features(y[0]); net.distance(x, out)                   # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    out.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        net.features(y[0])
        net.distance(x, out)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(1, 1, 1, 1), a)


def test_errors(net, weights):
    import torch
    from h3dgs.lpips import LpipsVGG
    for H, W in ((15, 40), (40, 15)):
        with pytest.raises(ValueError, match="16 pixels"):
            net(torch.rand((3, H, W), device="cuda"), torch.rand((3, H, W), device="cuda"))
    net(torch.rand((3, 16, 16), device="cuda"), torch.rand((3, 16, 16), device="cuda"))
    with pytest.raises(ValueError):
        net(torch.rand((3, 20, 20), device="cuda"), torch.rand((3, 20, 21), device="cuda"))
    vgg, lin = weights
    bad = dict(vgg)
    bad["features.10.weight"] = torch.zeros(256, 128, 3, 1)
    with pytest.raises(ValueError, match=r"features\.10\.weight"):
        LpipsVGG.from_state_dicts(bad, lin)
    bad = dict(lin)
    del bad["lin2.model.1.weight"]
    with pytest.raises(ValueError, match=r"lin2\.model\.1\.weight"):
        LpipsVGG.from_state_dicts(vgg, bad)


def test_from_torch_hub_names_the_missing_file(tmp_path):
    import torch
    from h3dgs.lpips import LpipsVGG
    old = torch.hub.get_dir()
    torch.hub.set_dir(str(tmp_path))
    try:
        with pytest.raises(FileNotFoundError, match="vgg16-397923af.pth"):
            LpipsVGG.from_torch_hub()
    finally:
        torch.hub.set_dir(old)


# ---- the evaluator ---------------------------------------------------------------------------------------------------
def _evaluator_inputs(exposure=False, mask=False):
    import torch
    from h3dgs import pipeline
    from test_gpu_evaluate import _cams, _scene, _targets
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
        for _ in dcams:
            E = np.zeros((3, 4), np.float32)
            E[:, :3] = np.eye(3) * 1.05 + rng.uniform(-0.08, 0.08, (3, 3))
            E[:, 3] = rng.uniform(-0.03, 0.03, 3)
            exposures.append(torch.tensor(E, device="cuda"))
        exposures[1] = None
    return cam, scene, dcams, targets, masks, exposures


TAUS = [0.0, 3.0, 6.0, 15.0]


@pytest.mark.parametrize("exposure,mask,tte", [(False, False, False), (True, True, False), (False, True, True),
                                               (True, False, True)])
def test_evaluate_hierarchy_lpips_equals_net_on_each_frame(net, exposure, mask, tte):
    import torch
    from h3dgs.evaluate import evaluate_hierarchy
    cam, scene, dcams, targets, masks, exposures = _evaluator_inputs(exposure, mask)
    res = evaluate_hierarchy(scene, dcams, targets, TAUS, masks=masks, exposures=exposures, train_test_exp=tte,
                             keep_images=True, lpips=net)
    assert res["lpips_rows"].shape == (len(TAUS), len(dcams))
    x0 = cam.W // 2 if tte else 0
    for ti, tau in enumerate(TAUS):
        for ci in range(len(dcams)):
            m = None if masks is None else masks[ci][..., x0:]
            img = res["images"][ti][ci]
            gt = targets[ci].clamp(0.0, 1.0)[..., x0:]
            if m is not None:
                img, gt = img * m, gt * m
            want = float(net(img.contiguous(), gt.contiguous()))
            assert res["lpips_rows"][ti, ci] == want, (tau, ci, res["lpips_rows"][ti, ci], want)
        assert res["lpips"][tau] == float(res["lpips_rows"][ti].mean())
        assert 0.0 < res["lpips"][tau] < 10.0


def test_rerun_frames_equal_an_ample_capacity(net):
    from h3dgs.evaluate import evaluate_hierarchy
    _, scene, dcams, targets, masks, _ = _evaluator_inputs(mask=True)
    ample = evaluate_hierarchy(scene, dcams, targets, TAUS, masks=masks, lpips=net,
                               capacities=dict(row_capacity=scene.means3D.shape[0], bin_capacity=1 << 21, sort_capacity=8192))
    assert ample["rerun"] == 0
    rows = ample["rows"][..., 3]
    small = evaluate_hierarchy(scene, dcams, targets, TAUS, masks=masks, lpips=net,
                               capacities=dict(row_capacity=int(np.median(rows)), bin_capacity=1 << 21, sort_capacity=8192))
    assert 0 < small["rerun"] < len(TAUS) * len(dcams)
    assert np.array_equal(small["lpips_rows"], ample["lpips_rows"])


def test_sweep_with_lpips_never_synchronises_the_host(net):
    import torch
    from h3dgs import pipeline, synth
    from h3dgs.evaluate import HierarchyEvaluator
    from test_gpu_evaluate import _cams, _scene, _targets
    cam, h = _scene(skybox=30)
    scene = pipeline.Scene(h, requires_grad=False)
    bg = torch.zeros(3, device="cuda")
    cams = _cams(cam.W, cam.H) + [synth.make_camera(320, 200)]
    dcams = [pipeline.DeviceCamera(c) for c in cams]
    targets = [t.cpu() for t in _targets(scene, dcams, bg)]
    masks = [torch.ones((1, c.H, c.W)) for c in cams]
    ev = HierarchyEvaluator(scene, dcams, targets, TAUS, masks=masks, train_test_exp=True, lpips=net)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ev.enqueue()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    res = ev.finish()
    assert res["lpips_rows"].shape == (len(TAUS), len(cams)) and np.isfinite(res["lpips_rows"]).all()


def test_without_lpips_the_output_is_unchanged(net):
    from h3dgs.evaluate import evaluate_hierarchy
    _, scene, dcams, targets, masks, exposures = _evaluator_inputs(exposure=True, mask=True)
    plain = evaluate_hierarchy(scene, dcams, targets, TAUS, masks=masks, exposures=exposures)
    with_lp = evaluate_hierarchy(scene, dcams, targets, TAUS, masks=masks, exposures=exposures, lpips=net)
    assert set(plain) == {"psnr", "ssim", "rows", "rerun", "flagged", "images"}
    assert set(with_lp) == set(plain) | {"lpips", "lpips_rows"}
    # the metrics pass sums with double atomics: PSNR and SSIM may differ between two sweeps in their last bits
    assert np.array_equal(plain["rows"][..., 2:], with_lp["rows"][..., 2:]) and plain["rerun"] == with_lp["rerun"]
    assert np.abs(plain["rows"][..., 0] - with_lp["rows"][..., 0]).max() <= 1e-9
    assert np.abs(plain["rows"][..., 1] - with_lp["rows"][..., 1]).max() <= 1e-12

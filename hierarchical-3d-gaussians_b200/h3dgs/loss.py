"""Fused L1 + SSIM training loss on libh3dgs.so (SURVEY.md 8f-2).

Same numbers as the reference's `utils/loss_utils.py` (`l1_loss`, `ssim` with window 11 / sigma 1.5 /
size_average=True) combined as in train_post.py:134-140:

    loss = (1 - lambda_dssim) * l1_loss(image, gt) + lambda_dssim * (1 - ssim(image, gt))

but one CUDA kernel forward and one backward instead of 5 grouped conv2d + ~20 elementwise kernels and
their autograd.  Gradients flow to `image` only (the ground truth is data); `single_loss`, train_single's objective,
also has them to the trained exposure and the inverse depth.  No CPU fallback.
"""

import torch

from . import _lib
from ._lib import ptr


def _coefficients(g_loss, g_l1, g_ssim, lam, n):
    """[k0, k1] (device fp32) from the upstream gradients of (loss, l1, ssim): d/dimg of the L1 term gets
    (g_loss (1-l) + g_l1) / N, the SSIM sum gets (-g_loss l + g_ssim) / N"""
    return torch.stack([(g_loss * (1.0 - lam) + g_l1) / n, (g_ssim - g_loss * lam) / n]).float().contiguous()


class _FusedL1SSIM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, gt, lambda_dssim):
        if not image.is_cuda:
            raise RuntimeError("fused_l1_ssim needs CUDA tensors (there is no CPU fallback)")
        img = image.detach().float().contiguous()
        ref = gt.detach().float().contiguous()
        if img.dim() == 4 and img.shape[0] == 1:
            img, ref = img[0], ref[0]
        if img.dim() != 3 or img.shape != ref.shape:
            raise RuntimeError("expected image and gt of identical shape [C,H,W]")
        Cn, H, W = img.shape
        sums = torch.empty(2, dtype=torch.float64, device=img.device)
        maps = torch.empty((3, Cn, H, W), dtype=torch.float32, device=img.device)
        with torch.cuda.device(img.device):
            _lib.check(_lib.lib().h3dgs_l1_ssim_forward(Cn, H, W, img.data_ptr(), ref.data_ptr(), sums.data_ptr(),
                                                       maps.data_ptr(), torch.cuda.current_stream().cuda_stream))
        n = float(img.numel())
        l1 = sums[0] / n
        ssim = sums[1] / n
        ctx.save_for_backward(img, ref, maps)
        ctx.lam, ctx.n, ctx.in_shape = float(lambda_dssim), n, image.shape
        loss = (1.0 - ctx.lam) * l1 + ctx.lam * (1.0 - ssim)
        return loss.float(), l1.float(), ssim.float()

    @staticmethod
    def backward(ctx, g_loss, g_l1, g_ssim):
        img, ref, maps = ctx.saved_tensors
        Cn, H, W = img.shape
        z = torch.zeros((), device=img.device)
        g_loss = z if g_loss is None else g_loss
        g_l1 = z if g_l1 is None else g_l1
        g_ssim = z if g_ssim is None else g_ssim
        coeffs = _coefficients(g_loss, g_l1, g_ssim, ctx.lam, ctx.n)
        grad = torch.empty_like(img)
        with torch.cuda.device(img.device):
            _lib.check(_lib.lib().h3dgs_l1_ssim_backward(Cn, H, W, img.data_ptr(), ref.data_ptr(), maps.data_ptr(),
                                                        coeffs.data_ptr(), grad.data_ptr(),
                                                        torch.cuda.current_stream().cuda_stream))
        return grad.view(ctx.in_shape), None, None


def fused_l1_ssim(image, gt, lambda_dssim=0.2):
    """-> (loss, l1, ssim) scalars; loss = (1-l)*L1 + l*(1-SSIM) (train_post.py:134-140)."""
    return _FusedL1SSIM.apply(image, gt, lambda_dssim)


def l1_loss(network_output, gt):
    """utils/loss_utils.py:17-18.  Images ([C,H,W] / [1,C,H,W]) go through the fused kernel; the reference's one-liner
    accepts any shape, so anything else is evaluated as it writes it.  (A loop that needs both terms should call
    fused_l1_ssim once: l1_loss + ssim each run the fused pass.)"""
    if network_output.dim() == 3 or (network_output.dim() == 4 and network_output.shape[0] == 1):
        return _FusedL1SSIM.apply(network_output, gt, 0.0)[1]
    return torch.abs(network_output - gt).mean()


def ssim(img1, img2, window_size=11, size_average=True):
    """utils/loss_utils.py:33-41 (window 11, size_average=True only)."""
    if window_size != 11 or not size_average:
        raise NotImplementedError("only window_size=11, size_average=True (the reference's call sites)")
    return _FusedL1SSIM.apply(img1, img2, 0.0)[2]


def exposure_block(exposure, device):
    """the top 3x4 block of an exposure matrix ([3,4] or larger, as pretrained_exposures holds them), contiguous fp32 on
    `device`; None stays None"""
    if exposure is None:
        return None
    return exposure.detach()[:3, :4].to(device=device, dtype=torch.float32).contiguous()


def mask_plane(mask, H, W, device):
    """an alpha mask ([1,H,W] or [H,W]) as a contiguous fp32 [H,W] on `device`; None stays None"""
    if mask is None:
        return None
    return mask.detach().reshape(H, W).to(device=device, dtype=torch.float32).contiguous()


def post_loss(image, gt, lambda_dssim=0.2, exposure=None, mask=None):
    """train_post's objective on the raw rasterizer output `image` [3,H,W] -> (loss, l1, ssim) scalars:

        a = clamp(image.permute(1,2,0) @ E[:3,:3] + E[:3,3], 0, 1) * mask       (render_post :279-285, train_post :135-137)
        loss = (1-l) * mean|a - gt| + l * (1 - SSIM(a, gt))

    `gt` is the target as the loader leaves it (clamped and masked already; it is used as it is).  exposure: [3,4] or
    larger (its top 3x4 block) or None (identity: render_post without an entry for the image); mask: [1,H,W] or [H,W] or
    None (all ones).  One CUDA kernel forward and one backward (single_loss's, without the depth term); gradient to
    `image` only (pretrained exposures are frozen, the mask is data)."""
    if image.dim() == 4 and image.shape[0] == 1:
        image, gt = image[0], gt[0]
    exposure = None if exposure is None else exposure.detach()
    loss, _, l1, ssim, _ = _SingleLoss.apply(image, None, exposure, gt, lambda_dssim, mask, None, None, 0.0)
    return loss, l1, ssim


class _SingleLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, invdepth, exposure, gt, lambda_dssim, mask, mono_invdepth, depth_mask, depth_weight):
        from diff_gaussian_rasterization._C import _on_device
        if not _on_device(image):
            raise RuntimeError("post_loss / single_loss need CUDA tensors (there is no CPU fallback)")
        img = image.detach().float().contiguous()
        ref = gt.detach().float().contiguous()
        if img.dim() != 3 or img.shape[0] != 3 or img.shape != ref.shape:
            raise RuntimeError("expected image and gt of identical shape [3,H,W]")
        _, H, W = img.shape
        dev = img.device
        E = exposure_block(exposure, dev)
        M = mask_plane(mask, H, W, dev)
        L = _lib.lib()
        sums = torch.empty(2, dtype=torch.float64, device=dev)
        maps = torch.empty((3, 3, H, W), dtype=torch.float32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        depth = mono_invdepth is not None
        with torch.cuda.device(dev):
            _lib.check(L.h3dgs_post_loss_forward(H, W, img.data_ptr(), ref.data_ptr(), ptr(E), ptr(M), sums.data_ptr(),
                                                 maps.data_ptr(), st))
            if depth:
                if invdepth is None or invdepth.numel() != H * W:
                    raise RuntimeError("the depth term needs the rasterizer's inverse depth [1,H,W] (do_depth=True)")
                inv = invdepth.detach().float().contiguous()
                mono = mask_plane(mono_invdepth, H, W, dev)
                dmask = mask_plane(depth_mask, H, W, dev) if depth_mask is not None else torch.ones((H, W), device=dev)
                w = torch.as_tensor(depth_weight, dtype=torch.float32, device=dev).reshape(())
                dsum = torch.empty(1, dtype=torch.float64, device=dev)
                dinv = torch.empty((H, W), dtype=torch.float32, device=dev)
                _lib.check(L.h3dgs_invdepth_l1_grad(H, W, inv.data_ptr(), mono.data_ptr(), dmask.data_ptr(), w.data_ptr(),
                                                    dinv.data_ptr(), dsum.data_ptr(), st))
        n = float(img.numel())
        l1, ssim = sums[0] / n, sums[1] / n
        lam = float(lambda_dssim)
        photo = (1.0 - lam) * l1 + lam * (1.0 - ssim)
        if depth:
            depth_l1 = dsum[0] / float(H * W)
            loss = photo + w.double() * depth_l1
            ctx.dinv = dinv                     # dL/dinvdepth for an upstream gradient of 1 to the loss
        else:
            depth_l1, loss, ctx.dinv = torch.zeros((), dtype=torch.float64, device=dev), photo, None
        ctx.save_for_backward(img, ref, maps)
        ctx.E, ctx.M, ctx.lam, ctx.n = E, M, lam, n
        ctx.in_shape = image.shape
        ctx.inv_shape = None if invdepth is None else invdepth.shape
        ctx.exposure_like = exposure if (exposure is not None and ctx.needs_input_grad[2]) else None
        depth_l1 = depth_l1.float()
        ctx.mark_non_differentiable(depth_l1)       # reported, as Ll1depth_pure is; its gradient travels through the loss
        return loss.float(), photo.float(), l1.float(), ssim.float(), depth_l1

    @staticmethod
    def backward(ctx, g_loss, g_photo, g_l1, g_ssim, _g_depth):
        img, ref, maps = ctx.saved_tensors
        _, H, W = img.shape
        dev = img.device
        L = _lib.lib()
        st = torch.cuda.current_stream(dev).cuda_stream
        coeffs = _coefficients(g_loss + g_photo, g_l1, g_ssim, ctx.lam, ctx.n)
        grad = torch.empty_like(img)
        g_inv = g_E = None
        with torch.cuda.device(dev):
            if ctx.exposure_like is not None:
                dE = torch.empty((3, 4), dtype=torch.float64, device=dev)
                _lib.check(L.h3dgs_post_loss_backward_exposure(H, W, img.data_ptr(), ref.data_ptr(), ptr(ctx.E), ptr(ctx.M),
                                                               maps.data_ptr(), coeffs.data_ptr(), grad.data_ptr(),
                                                               dE.data_ptr(), st))
                g_E = torch.zeros_like(ctx.exposure_like)
                g_E[:3, :4] = dE.to(g_E.dtype)
            else:
                _lib.check(L.h3dgs_post_loss_backward(H, W, img.data_ptr(), ref.data_ptr(), ptr(ctx.E), ptr(ctx.M),
                                                      maps.data_ptr(), coeffs.data_ptr(), grad.data_ptr(), st))
            if ctx.dinv is not None and ctx.needs_input_grad[1]:
                # the forward's one pass wrote the gradient with the term's sum; times 1 under loss.backward(): exact
                g_inv = (ctx.dinv * g_loss.float()).view(ctx.inv_shape)
            elif ctx.needs_input_grad[1]:
                g_inv = torch.zeros(ctx.inv_shape, dtype=torch.float32, device=dev)
        return grad.view(ctx.in_shape), g_inv, g_E, None, None, None, None, None, None


def single_loss(image, invdepth, gt, lambda_dssim=0.2, exposure=None, mask=None, mono_invdepth=None, depth_mask=None,
                depth_weight=0.0):
    """train_single's objective on the raw rasterizer outputs `image` [3,H,W] and `invdepth` [1,H,W]
    -> (loss, photo, l1, ssim, depth_l1) scalars:

        a     = clamp(image.permute(1,2,0) @ E[:3,:3] + E[:3,3], 0, 1) * mask     (render() :115-118, train_single.py:102-104)
        photo = (1-l) * mean|a - gt| + l * (1 - SSIM(a, gt))                       (train_single.py:106-108)
        depth_l1 = mean|(invdepth - mono_invdepth) * depth_mask|                   (:115, Ll1depth_pure)
        loss  = photo + depth_weight * depth_l1

    exposure: the image's trained [3,4] or [4,4] exposure (None = identity); when it requires grad it receives its
    gradient in its own shape, zero outside the top 3x4 block.  The depth term is absent when mono_invdepth is None or
    depth_weight is the number 0 (train_single.py:111: the weight schedule reached 0, or the view's depth is
    unreliable); depth_weight may be a device tensor.  Gradients go to image, invdepth and exposure; gt, the masks and
    the mono depth are data; depth_l1 is a reported value (Ll1depth_pure), not differentiable on its own.  One CUDA
    kernel forward and one backward for the photometric term, and one pass for the depth term and its gradient."""
    if mono_invdepth is not None and not torch.is_tensor(depth_weight) and float(depth_weight) == 0.0:
        mono_invdepth = None
    return _SingleLoss.apply(image, invdepth, exposure, gt, lambda_dssim, mask, mono_invdepth, depth_mask, depth_weight)


class _CoarseLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, gt, lambda_dssim, mask):
        from diff_gaussian_rasterization._C import _on_device
        if not _on_device(image):
            raise RuntimeError("coarse_loss needs CUDA tensors (there is no CPU fallback)")
        img = image.detach().float().contiguous()
        ref = gt.detach().float().contiguous()
        if img.dim() != 3 or img.shape[0] != 3 or img.shape != ref.shape:
            raise RuntimeError("expected image and gt of identical shape [3,H,W]")
        _, H, W = img.shape
        dev = img.device
        M = mask_plane(mask, H, W, dev)
        sums = torch.empty(2, dtype=torch.float64, device=dev)
        maps = torch.empty((3, 3, H, W), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().h3dgs_coarse_loss_forward(H, W, img.data_ptr(), ref.data_ptr(), ptr(M), sums.data_ptr(),
                                                           maps.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
        n = float(img.numel())
        l1, ssim = sums[0] / n, sums[1] / n
        ctx.save_for_backward(img, ref, maps)
        ctx.M, ctx.lam, ctx.n, ctx.in_shape = M, float(lambda_dssim), n, image.shape
        loss = (1.0 - ctx.lam) * l1 + ctx.lam * (1.0 - ssim)
        return loss.float(), l1.float(), ssim.float()

    @staticmethod
    def backward(ctx, g_loss, g_l1, g_ssim):
        img, ref, maps = ctx.saved_tensors
        _, H, W = img.shape
        dev = img.device
        coeffs = _coefficients(g_loss, g_l1, g_ssim, ctx.lam, ctx.n)
        grad = torch.empty_like(img)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().h3dgs_coarse_loss_backward(H, W, img.data_ptr(), ref.data_ptr(), ptr(ctx.M), maps.data_ptr(),
                                                            coeffs.data_ptr(), grad.data_ptr(),
                                                            torch.cuda.current_stream(dev).cuda_stream))
        return grad.view(ctx.in_shape), None, None, None


def coarse_loss(image, gt, lambda_dssim=0.2, mask=None):
    """train_coarse's objective on render_coarse's image [3,H,W] -> (loss, l1, ssim) scalars:

        a    = image * mask                                         (train_coarse.py:113-116; no exposure, no clamp)
        loss = (1-l) * mean|a - gt| + l * (1 - SSIM(a, gt))

    mask: [1,H,W] or [H,W] or None (the camera has no alpha mask: a = image).  One CUDA kernel forward and one backward;
    the gradient reaches `image` for every value, above 1 included (render_coarse's colours are clamped only below)."""
    if image.dim() == 4 and image.shape[0] == 1:
        image, gt = image[0], gt[0]
    return _CoarseLoss.apply(image, gt, lambda_dssim, mask)

"""Fused L1 + SSIM training loss on libh3dgs.so (SURVEY.md 8f-2).

Same numbers as the reference's `utils/loss_utils.py` (`l1_loss`, `ssim` with window 11 / sigma 1.5 /
size_average=True) combined as in train_post.py:134-140:

    loss = (1 - lambda_dssim) * l1_loss(image, gt) + lambda_dssim * (1 - ssim(image, gt))

but one CUDA kernel forward and one backward instead of 5 grouped conv2d + ~20 elementwise kernels and
their autograd.  Gradients flow to `image` only (the ground truth is data).  No CPU fallback.
"""

import torch

from . import _lib


def _ptr(t):
    return None if t is None else t.data_ptr()


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


class _PostLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, gt, lambda_dssim, exposure, mask):
        if not image.is_cuda:
            raise RuntimeError("post_loss needs CUDA tensors (there is no CPU fallback)")
        img = image.detach().float().contiguous()
        ref = gt.detach().float().contiguous()
        if img.dim() == 4 and img.shape[0] == 1:
            img, ref = img[0], ref[0]
        if img.dim() != 3 or img.shape[0] != 3 or img.shape != ref.shape:
            raise RuntimeError("expected image and gt of identical shape [3,H,W]")
        _, H, W = img.shape
        E = exposure_block(exposure, img.device)
        M = mask_plane(mask, H, W, img.device)
        sums = torch.empty(2, dtype=torch.float64, device=img.device)
        maps = torch.empty((3, 3, H, W), dtype=torch.float32, device=img.device)
        with torch.cuda.device(img.device):
            _lib.check(_lib.lib().h3dgs_post_loss_forward(H, W, img.data_ptr(), ref.data_ptr(), _ptr(E), _ptr(M),
                                                         sums.data_ptr(), maps.data_ptr(),
                                                         torch.cuda.current_stream().cuda_stream))
        n = float(img.numel())
        l1 = sums[0] / n
        ssim = sums[1] / n
        ctx.save_for_backward(img, ref, maps)
        ctx.E, ctx.M = E, M
        ctx.lam, ctx.n, ctx.in_shape = float(lambda_dssim), n, image.shape
        loss = (1.0 - ctx.lam) * l1 + ctx.lam * (1.0 - ssim)
        return loss.float(), l1.float(), ssim.float()

    @staticmethod
    def backward(ctx, g_loss, g_l1, g_ssim):
        img, ref, maps = ctx.saved_tensors
        _, H, W = img.shape
        z = torch.zeros((), device=img.device)
        g_loss = z if g_loss is None else g_loss
        g_l1 = z if g_l1 is None else g_l1
        g_ssim = z if g_ssim is None else g_ssim
        coeffs = _coefficients(g_loss, g_l1, g_ssim, ctx.lam, ctx.n)
        grad = torch.empty_like(img)
        with torch.cuda.device(img.device):
            _lib.check(_lib.lib().h3dgs_post_loss_backward(H, W, img.data_ptr(), ref.data_ptr(), _ptr(ctx.E), _ptr(ctx.M),
                                                          maps.data_ptr(), coeffs.data_ptr(), grad.data_ptr(),
                                                          torch.cuda.current_stream().cuda_stream))
        return grad.view(ctx.in_shape), None, None, None, None


def post_loss(image, gt, lambda_dssim=0.2, exposure=None, mask=None):
    """train_post's objective on the raw rasterizer output `image` [3,H,W] -> (loss, l1, ssim) scalars:

        a = clamp(image.permute(1,2,0) @ E[:3,:3] + E[:3,3], 0, 1) * mask       (render_post :279-285, train_post :135-137)
        loss = (1-l) * mean|a - gt| + l * (1 - SSIM(a, gt))

    `gt` is the target as the loader leaves it (clamped and masked already; it is used as it is).  exposure: [3,4] or
    larger (its top 3x4 block) or None (identity: render_post without an entry for the image); mask: [1,H,W] or [H,W] or
    None (all ones).  One CUDA kernel forward and one backward; gradient to `image` only (pretrained exposures are
    frozen, the mask is data)."""
    return _PostLoss.apply(image, gt, lambda_dssim, exposure, mask)

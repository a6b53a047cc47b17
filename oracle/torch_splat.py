"""Naive pure-PyTorch CPU point-splat (BASELINE.json configs[0]).

TEST INFRASTRUCTURE ONLY (see oracle.c header).  A second, independent
restatement of the same published algorithm, dense over [pixels x Gaussians] and
differentiated by torch autograd, used to (1) cross-check the hand-written
forward AND backward of oracle.c, and (2) serve as the "naive pure-PyTorch CPU
point-splat" of BASELINE.json's north_star.  PARITY UNPINNED against the real
reference (source absent); follows utils/sh_utils.py:57-112 (SH),
utils/general_utils.py:68-114 (cov3D), gaussian_renderer/__init__.py:85-89.

Only practical for small scenes (memory ~ 8 * Npix * P * ~12 bytes).
"""
import torch

C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435]
TILE = 16


def eval_sh(deg, sh, dirs):
    """sh [P,K,3], dirs [P,3] -> [P,3]  (utils/sh_utils.py:57-112, coefficient-major here)."""
    x, y, z = dirs[:, 0:1], dirs[:, 1:2], dirs[:, 2:3]
    r = C0 * sh[:, 0]
    if deg > 0:
        r = r - C1 * y * sh[:, 1] + C1 * z * sh[:, 2] - C1 * x * sh[:, 3]
        if deg > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            r = (r + C2[0] * xy * sh[:, 4] + C2[1] * yz * sh[:, 5] + C2[2] * (2.0 * zz - xx - yy) * sh[:, 6]
                 + C2[3] * xz * sh[:, 7] + C2[4] * (xx - yy) * sh[:, 8])
            if deg > 2:
                r = (r + C3[0] * y * (3 * xx - yy) * sh[:, 9] + C3[1] * xy * z * sh[:, 10]
                     + C3[2] * y * (4 * zz - xx - yy) * sh[:, 11] + C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[:, 12]
                     + C3[4] * x * (4 * zz - xx - yy) * sh[:, 13] + C3[5] * z * (xx - yy) * sh[:, 14]
                     + C3[6] * x * (xx - 3 * yy) * sh[:, 15])
    return r


def build_cov3d(scales, rots, mod):
    r, x, y, z = rots[:, 0], rots[:, 1], rots[:, 2], rots[:, 3]
    R = torch.stack([
        1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    Lm = R * (mod * scales)[:, None, :]
    return Lm @ Lm.transpose(1, 2)


def splat(means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
          viewmatrix, projmatrix, campos, bg, W, H, tanfovx, tanfovy, sh_degree=3, scale_modifier=1.0,
          ts=None, kids=None, do_depth=False):
    """All tensor args torch (any float dtype, CPU).  Returns (color[3,H,W], radii[P], invdepth[1,H,W])."""
    pr = project(means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, viewmatrix, projmatrix,
                 campos, W, H, tanfovx, tanfovy, sh_degree, scale_modifier)
    color, invd = blend2d(pr["px"], pr["py"], pr["conic"], pr["opacities"], pr["rgb"], pr["depth"], pr["visible"],
                          pr["rect"], bg, W, H, ts, kids, do_depth)
    return color, pr["radii"], invd


def project(means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
            viewmatrix, projmatrix, campos, W, H, tanfovx, tanfovy, sh_degree=3, scale_modifier=1.0):
    """The per-Gaussian half of splat: the 2D Gaussians blend2d takes (px, py, conic, opacities, rgb, depth = view z,
    visible, rect) and radii, as a dict."""
    dt = means3D.dtype
    P = means3D.shape[0]
    V = viewmatrix.reshape(4, 4).to(dt); PM = projmatrix.reshape(4, 4).to(dt)
    hom = torch.cat([means3D, torch.ones(P, 1, dtype=dt)], 1)
    pv = hom @ V
    ph = hom @ PM
    pw = 1.0 / (ph[:, 3] + 1e-7)
    ndc = ph[:, :2] * pw[:, None]
    in_front = pv[:, 2] > 0.2
    if cov3D_precomp is not None:
        c = cov3D_precomp
        Sig = torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4], c[:, 2], c[:, 4], c[:, 5]], 1).reshape(-1, 3, 3)
    else:
        Sig = build_cov3d(scales, rotations, scale_modifier)
    fx, fy = W / (2 * tanfovx), H / (2 * tanfovy)
    tz = pv[:, 2]
    tz = torch.where(in_front, tz, torch.ones_like(tz))        # avoid NaN in culled rows
    tx = torch.clamp(pv[:, 0] / tz, -1.3 * tanfovx, 1.3 * tanfovx) * tz
    ty = torch.clamp(pv[:, 1] / tz, -1.3 * tanfovy, 1.3 * tanfovy) * tz
    zero = torch.zeros_like(tz)
    J = torch.stack([fx / tz, zero, -(fx * tx) / (tz * tz), zero, fy / tz, -(fy * ty) / (tz * tz)], 1).reshape(-1, 2, 3)
    Rwv = V[:3, :3].t()
    A = J @ Rwv
    cov = A @ Sig @ A.transpose(1, 2)
    a = cov[:, 0, 0] + 0.3; b = cov[:, 0, 1]; c_ = cov[:, 1, 1] + 0.3
    det = a * c_ - b * b
    det_s = torch.where(det == 0, torch.ones_like(det), det)
    conic = torch.stack([c_ / det_s, -b / det_s, a / det_s], 1)
    mid = 0.5 * (a + c_)
    lam = mid + torch.sqrt(torch.clamp(mid * mid - det, min=0.1))
    radius = torch.ceil(3 * torch.sqrt(lam)).detach()
    px = ((ndc[:, 0] + 1) * W - 1) * 0.5
    py = ((ndc[:, 1] + 1) * H - 1) * 0.5
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    pxd, pyd = px.detach(), py.detach()
    rminx = torch.clamp(((pxd - radius) / TILE).trunc(), 0, gx); rmaxx = torch.clamp(((pxd + radius + TILE - 1) / TILE).trunc(), 0, gx)
    rminy = torch.clamp(((pyd - radius) / TILE).trunc(), 0, gy); rmaxy = torch.clamp(((pyd + radius + TILE - 1) / TILE).trunc(), 0, gy)
    visible = in_front & (det != 0) & ((rmaxx - rminx) * (rmaxy - rminy) > 0)
    radii = torch.where(visible, radius, torch.zeros_like(radius)).to(torch.int32)
    if colors_precomp is not None:
        rgb = colors_precomp
    else:
        d = means3D - campos[None].to(dt)
        d = d / d.norm(dim=1, keepdim=True)
        rgb = torch.clamp_min(eval_sh(sh_degree, shs, d) + 0.5, 0.0)
    return dict(px=px, py=py, conic=conic, opacities=opacities.reshape(-1), rgb=rgb, depth=pv[:, 2], visible=visible,
                rect=(rminx, rmaxx, rminy, rmaxy), radii=radii)


def blend2d(px, py, conic, opacities, rgb, depth, visible, rect, bg, W, H, ts=None, kids=None, do_depth=False):
    """The blend over projected 2D Gaussians: px, py [P], conic [P,3], opacities [P], rgb [P,3], depth [P] (view z),
    visible [P] bool, rect = (rminx, rmaxx, rminy, rmaxy) in tiles.  Returns (color[3,H,W], invdepth[1,H,W] or None)."""
    dt = px.dtype
    rminx, rmaxx, rminy, rmaxy = rect
    # depth order, ties by index (stable), visible only
    idx = torch.nonzero(visible).flatten()
    order = idx[torch.argsort(depth[idx].detach().float(), stable=True)]
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    pixx = xs.reshape(-1, 1).to(dt); pixy = ys.reshape(-1, 1).to(dt)
    tlx = (xs.reshape(-1, 1) // TILE).to(dt); tly = (ys.reshape(-1, 1) // TILE).to(dt)
    o = order
    in_rect = (tlx >= rminx[o][None]) & (tlx < rmaxx[o][None]) & (tly >= rminy[o][None]) & (tly < rmaxy[o][None])
    dx = px[o][None] - pixx; dy = py[o][None] - pixy
    power = -0.5 * (conic[o, 0][None] * dx * dx + conic[o, 2][None] * dy * dy) - conic[o, 1][None] * dx * dy
    G = torch.exp(torch.clamp(power, max=0.0))
    araw = opacities[o][None] * G
    alpha = araw + (torch.clamp(araw, max=0.99) - araw).detach()      # cap not differentiated (published bwd)
    if ts is not None and ts.numel() > 0:
        t = ts.reshape(-1)[o][None].to(dt); k = kids.reshape(-1)[o][None].to(dt)
        ah = t * alpha + (1 - t) * (1 - torch.pow(1 - alpha, 1.0 / k))
        alpha = torch.where((k > 1) & (t < 1), ah, alpha)
    valid = in_rect & (power.detach() <= 0) & (alpha.detach() >= 1.0 / 255.0)
    aeff = torch.where(valid, alpha, torch.zeros_like(alpha))
    T_after = torch.cumprod(1 - aeff, dim=1)
    contrib = valid & (T_after.detach() >= 1e-4)
    aeff = torch.where(contrib, alpha, torch.zeros_like(alpha))
    T_after = torch.cumprod(1 - aeff, dim=1)
    T_before = torch.cat([torch.ones(T_after.shape[0], 1, dtype=dt), T_after[:, :-1]], 1)
    w = aeff * T_before
    color = w @ rgb[o] + T_after[:, -1:] * bg[None].to(dt) if o.numel() else bg[None].to(dt).expand(H * W, 3)
    color = color.t().reshape(3, H, W)
    invd = None
    if do_depth:
        invd = (w @ (1.0 / depth[o])[:, None]).reshape(1, H, W) if o.numel() else torch.zeros(1, H, W, dtype=dt)
    return color, invd

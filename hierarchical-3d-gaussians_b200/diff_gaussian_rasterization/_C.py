"""`diff_gaussian_rasterization._C`: the op-level functions the reference's
extension module exposes (rasterize_gaussians, rasterize_gaussians_backward,
mark_visible), implemented as thin ctypes calls into libh3dgs.so.

Tensors in, tensors out; pointers cross the C-ABI as integers.  Raises on any
error -- there is no CPU or PyTorch fallback.
"""
import ctypes as C

import torch

from h3dgs import _lib


_last_num_rendered = 0


def last_num_rendered():
    """D of the most recent forward on this process (bench bookkeeping)."""
    return _last_num_rendered


def _on_device(t):
    """the library takes device pointers (the CPU suite patches this to drive an emulation build)"""
    return t.is_cuda


def _ptr(t):
    return None if (t is None or t.numel() == 0) else t.data_ptr()


def _f32c(t, name):
    if t is None or t.numel() == 0:
        return None
    if not _on_device(t):
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if t.dtype != torch.float32:
        t = t.float()
    t = t.contiguous()
    # the kernels read rotations and SH rows as float4, and the library refuses rows that are not 16-byte aligned:
    # a contiguous view at an odd float offset is copied (a fresh allocation is aligned)
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _i32c(t, name):
    if t is None or t.numel() == 0:
        return None
    if not _on_device(t):
        t = t.cuda()
    if t.dtype != torch.int32:
        t = t.int()
    return t.contiguous()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _make_args(P, means3D, sh, colors_precomp, opacities, scales, rotations, cov3D_precomp, bg, viewmatrix, projmatrix,
               campos, tanfovx, tanfovy, image_height, image_width, sh_degree, scale_modifier, prefiltered, debug,
               interpolation_weights, num_node_kids, do_depth, shard=(1, 0), render_indices=None,
               parent_indices=None, num_source=0, grad_rows=(0, 0)):
    a = _lib.RasterArgs()
    a.P = P
    a.sh_degree = int(sh_degree)
    a.sh_coeffs = int(sh.shape[1]) if sh is not None else 0
    a.image_width, a.image_height = int(image_width), int(image_height)
    a.tanfovx, a.tanfovy, a.scale_modifier = float(tanfovx), float(tanfovy), float(scale_modifier)
    a.prefiltered, a.debug, a.do_depth = int(bool(prefiltered)), int(bool(debug)), int(bool(do_depth))
    a.bg, a.viewmatrix, a.projmatrix, a.campos = _ptr(bg), _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos)
    a.means3D, a.shs, a.colors_precomp, a.opacities = _ptr(means3D), _ptr(sh), _ptr(colors_precomp), _ptr(opacities)
    a.scales, a.rotations, a.cov3D_precomp = _ptr(scales), _ptr(rotations), _ptr(cov3D_precomp)
    a.interpolation_weights, a.num_node_kids = _ptr(interpolation_weights), _ptr(num_node_kids)
    a.render_indices, a.parent_indices, a.num_source = _ptr(render_indices), _ptr(parent_indices), int(num_source)
    a.shard_count, a.shard_index = int(shard[0]), int(shard[1])
    a.grad_row_begin, a.grad_row_end = int(grad_rows[0]), int(grad_rows[1])
    return a


def _prep_inputs(means3D, sh, colors_precomp, opacities, scales, rotations, cov3D_precomp, bg, viewmatrix, projmatrix,
                 campos, interpolation_weights, num_node_kids, render_indices, parent_indices=None):
    means3D = _f32c(means3D, "means3D")
    P = 0 if means3D is None else means3D.shape[0]
    ridx = pidx = None
    if render_indices is not None and render_indices.numel() != 0:
        # in-kernel cut gather + parent lerp (every shipped call site passes empty index tensors,
        # gaussian_renderer/__init__.py:39-42, 244-245; this is the fused form of :199-218)
        ridx = _i32c(render_indices, "render_indices")
        pidx = _i32c(parent_indices, "parent_indices")
        if pidx is None or pidx.numel() < ridx.numel():
            raise RuntimeError("parent_indices must hold one entry per render index")
        P = ridx.numel()
    sh = _f32c(sh, "shs"); colors_precomp = _f32c(colors_precomp, "colors_precomp")
    opacities = _f32c(opacities, "opacities")
    scales = _f32c(scales, "scales"); rotations = _f32c(rotations, "rotations")
    cov3D_precomp = _f32c(cov3D_precomp, "cov3D_precomp")
    bg = _f32c(bg, "bg"); viewmatrix = _f32c(viewmatrix, "viewmatrix"); projmatrix = _f32c(projmatrix, "projmatrix")
    campos = _f32c(campos, "campos")
    ts = _f32c(interpolation_weights, "interpolation_weights") if (interpolation_weights is not None and interpolation_weights.numel()) else None
    if ts is not None and not _on_device(ts):
        ts = ts.cuda()
    kids = _i32c(num_node_kids, "num_node_kids") if ts is not None else None
    if ts is not None and (ts.numel() < P or kids is None or kids.numel() < P):
        raise RuntimeError("interpolation_weights / num_node_kids must hold at least P entries")
    return P, means3D, sh, colors_precomp, opacities, scales, rotations, cov3D_precomp, bg, viewmatrix, projmatrix, campos, ts, kids, ridx, pidx


def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                        viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos,
                        prefiltered, debug, render_indices=None, parent_indices=None, interpolation_weights=None,
                        num_node_kids=None, do_depth=False, shard=(1, 0), grad_rows=(0, 0)):
    """-> (num_rendered, color[3,H,W], radii[P] i32, geomBuffer, binningBuffer, imgBuffer, invdepth[1,H,W])
    grad_rows: sharded frames only -- the rendered rows whose gradients this rank will finish (lets the
    forward skip the SH colour of Gaussians no other stage of this rank reads)."""
    L = _lib.lib()
    (P, means3D, sh, colors, opacity, scales, rotations, cov3D_precomp, background, viewmatrix, projmatrix, campos,
     ts, kids, ridx, pidx) = _prep_inputs(means3D, sh, colors, opacity, scales, rotations, cov3D_precomp, background,
                                          viewmatrix, projmatrix, campos, interpolation_weights, num_node_kids,
                                          render_indices, parent_indices)
    dev = background.device
    H, W = int(image_height), int(image_width)
    a = _make_args(P, means3D, sh, colors, opacity, scales, rotations, cov3D_precomp, background, viewmatrix, projmatrix,
                   campos, tan_fovx, tan_fovy, H, W, degree, scale_modifier, prefiltered, debug, ts, kids, do_depth, shard,
                   ridx, pidx, 0 if ridx is None else means3D.shape[0], grad_rows)
    if shard[0] > 1:      # packed shard layout [owned tile rows][3][16][W]
        gy = (H + 15) // 16
        rows = (gy + shard[0] - 1 - shard[1]) // shard[0]
        color = torch.zeros((max(rows, 1), 3, 16, W), dtype=torch.float32, device=dev)
        invdepth = torch.zeros((max(rows, 1), 1, 16, W), dtype=torch.float32, device=dev) if do_depth else torch.empty((0,), dtype=torch.float32, device=dev)
    else:
        color = torch.empty((3, H, W), dtype=torch.float32, device=dev)
        invdepth = torch.empty((1, H, W), dtype=torch.float32, device=dev) if do_depth else torch.empty((0,), dtype=torch.float32, device=dev)
    radii = torch.empty((P,), dtype=torch.int32, device=dev)
    bufs = [None, None, None]

    def _alloc(_user, which, nbytes):
        t = torch.empty((max(int(nbytes), 1),), dtype=torch.uint8, device=dev)
        bufs[which] = t
        return t.data_ptr()

    cb = _lib.ALLOC_FN(_alloc)
    n = C.c_int64(0)
    with torch.cuda.device(dev):
        _lib.check(L.h3dgs_rasterize_forward(C.byref(a), cb, None, color.data_ptr(), _ptr(radii),
                                             _ptr(invdepth), C.byref(n), _stream()))
    global _last_num_rendered
    _last_num_rendered = int(n.value)
    return int(n.value), color, radii, bufs[0], bufs[1], bufs[2], invdepth


def rasterize_gaussians_backward(background, means3D, radii, colors, opacities, scales, rotations, scale_modifier,
                                 cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color,
                                 dL_dout_invdepth, sh, degree, campos, geomBuffer, num_rendered, binningBuffer,
                                 imageBuffer, debug, render_indices=None, parent_indices=None,
                                 interpolation_weights=None, num_node_kids=None, do_depth=False, image_height=None,
                                 image_width=None, shard=(1, 0), phases=3, scratch=None, grad_rows=(0, 0)):
    """-> (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations)"""
    L = _lib.lib()
    (P, means3D, sh, colors, opacities, scales, rotations, cov3D_precomp, background, viewmatrix, projmatrix, campos,
     ts, kids, ridx, pidx) = _prep_inputs(means3D, sh, colors, opacities, scales, rotations, cov3D_precomp, background,
                                          viewmatrix, projmatrix, campos, interpolation_weights, num_node_kids,
                                          render_indices, parent_indices)
    N = P if ridx is None else means3D.shape[0]          # rows of the gradient tensors
    dev = background.device
    H = int(image_height if image_height is not None else dL_dout_color.shape[1])
    W = int(image_width if image_width is not None else dL_dout_color.shape[2])
    a = _make_args(P, means3D, sh, colors, opacities, scales, rotations, cov3D_precomp, background, viewmatrix,
                   projmatrix, campos, tan_fovx, tan_fovy, H, W, degree, scale_modifier, False, debug, ts, kids,
                   do_depth, shard, ridx, pidx, 0 if ridx is None else N, grad_rows)
    g_color = _f32c(dL_dout_color, "dL_dout_color")
    g_depth = _f32c(dL_dout_invdepth, "dL_dout_invdepth") if (do_depth and dL_dout_invdepth is not None) else None
    # a row block leaves the other rows untouched: start them from zero (in scatter mode the library
    # zero-fills the full-size gradients itself, overlapped on its side stream)
    e = (lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)) if (grad_rows[1] > grad_rows[0] and ridx is None) else \
        (lambda *s: torch.empty(s, dtype=torch.float32, device=dev))
    M = sh.shape[1] if sh is not None else 0
    if phases & 2:
        d_means3D, d_opac = e(N, 3), e(N, 1)
        d_means2D = torch.zeros((P, 3), dtype=torch.float32, device=dev) if grad_rows[1] > grad_rows[0] else e(P, 3)
        d_sh = e(N, M, 3) if sh is not None else e(0)
        d_colors = e(N, 3) if colors is not None else e(0)
        d_scales = e(N, 3) if scales is not None else e(0)
        d_rots = e(N, 4) if rotations is not None else e(0)
        d_cov = e(N, 6) if cov3D_precomp is not None else e(0)
    else:
        d_means3D = d_means2D = d_opac = d_sh = d_colors = d_scales = d_rots = d_cov = None
    if scratch is None:
        scratch = torch.empty((L.h3dgs_backward_scratch_bytes(P),), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.h3dgs_rasterize_backward(C.byref(a), _ptr(radii), _ptr(geomBuffer), _ptr(binningBuffer),
                                              _ptr(imageBuffer), int(num_rendered), _ptr(g_color), _ptr(g_depth),
                                              _ptr(d_means3D), _ptr(d_means2D), _ptr(d_sh), _ptr(d_colors),
                                              _ptr(d_opac), _ptr(d_scales), _ptr(d_rots), _ptr(d_cov),
                                              scratch.data_ptr(), int(phases), _stream()))
    if phases == 1:
        return scratch
    return d_means2D, d_colors, d_opac, d_means3D, d_cov, d_sh, d_scales, d_rots


def mark_visible(means3D, viewmatrix, projmatrix):
    L = _lib.lib()
    means3D = _f32c(means3D, "means3D")
    P = means3D.shape[0]
    present = torch.empty((P,), dtype=torch.bool, device=means3D.device)
    with torch.cuda.device(means3D.device):
        _lib.check(L.h3dgs_mark_visible(P, means3D.data_ptr(), _f32c(viewmatrix, "viewmatrix").data_ptr(),
                                        _f32c(projmatrix, "projmatrix").data_ptr(), present.data_ptr(), _stream()))
    return present


def state_view(P, W, H, num_rendered, geomBuffer, binningBuffer, imageBuffer):
    """Test helper: typed torch views of the integer artefacts inside the opaque state buffers."""
    L = _lib.lib()
    v = _lib.StateView()
    _lib.check(L.h3dgs_state_layout(P, W, H, int(num_rendered), _ptr(geomBuffer), _ptr(binningBuffer),
                                    _ptr(imageBuffer), C.byref(v)))

    def view(buf, ptr, dtype, count):
        off = ptr - buf.data_ptr()
        nbytes = count * torch.empty((), dtype=dtype).element_size()
        return buf[off:off + nbytes].view(dtype)
    D = int(num_rendered)
    T = ((W + 15) // 16) * ((H + 15) // 16)
    out = dict(depths=view(geomBuffer, v.depths, torch.float32, P),
               tiles_touched=view(geomBuffer, v.tiles_touched, torch.int32, P),
               point_offsets=view(geomBuffer, v.point_offsets, torch.int32, P),
               records=view(geomBuffer, v.records, torch.float32, P * 12).view(P, 12),
               ranges=view(imageBuffer, v.ranges, torch.int32, T * 2).view(T, 2),
               final_T=view(imageBuffer, v.final_T, torch.float32, H * W).view(H, W),
               n_contrib=view(imageBuffer, v.n_contrib, torch.int32, H * W).view(H, W))
    if D > 0:
        out["keys_sorted"] = view(binningBuffer, v.keys_sorted, torch.int64, D)
        out["point_list"] = view(binningBuffer, v.point_list, torch.int32, D)
        out["sorted_records"] = view(binningBuffer, v.sorted_records, torch.float32, D * 12).view(D, 12)
    return out

"""TEST INFRASTRUCTURE ONLY.  numpy front-end to libh3dgs_emu.so (the library's kernels compiled against the
SIMT emulator, tests/emul/): the same C-ABI calls the product's Python shim makes, with host arrays."""
import ctypes as C

import numpy as np

from h3dgs import _lib


def aligned(nbytes, dtype=np.uint8, shape=None):
    """zero-filled array whose data pointer is 256-byte aligned (the library carves sub-buffers at 256 B)"""
    raw = np.zeros(int(nbytes) + 256, np.uint8)
    off = (-raw.ctypes.data) % 256
    a = raw[off:off + int(nbytes)].view(dtype)
    return a.reshape(shape) if shape is not None else a


def f32(a, shape=None):
    a = np.asarray(a, np.float32)
    out = aligned(a.nbytes, np.float32, a.shape if shape is None else shape)
    out[...] = a.reshape(out.shape)
    return out


def i32(a):
    a = np.asarray(a, np.int32)
    out = aligned(a.nbytes, np.int32, a.shape)
    out[...] = a
    return out


def ptr(a):
    return None if a is None else a.ctypes.data


class Emu:
    def __init__(self, so_path):
        self.L = _lib.bind(C.CDLL(so_path))

    def check(self, rc):
        if rc < 0:
            raise RuntimeError(f"libh3dgs_emu error {rc}: {self.L.h3dgs_last_error().decode()}")
        return rc

    def args(self, cam, bg, sc, sh_degree=3, ts=None, kids=None, do_depth=False, ridx=None, pidx=None, shard=(1, 0),
             colors=None, cov=None, bin_capacity=0, sort_capacity=0, P=None, grad_rows=(0, 0)):
        a = _lib.RasterArgs()
        keep = dict(bg=f32(bg), view=f32(cam.world_view_transform), proj=f32(cam.full_proj_transform), campos=f32(cam.camera_center),
                    means=f32(sc["means3D"]), opac=f32(sc["opacities"]),
                    shs=f32(sc["shs"]) if colors is None else None, colors=f32(colors) if colors is not None else None,
                    scales=f32(sc["scales"]) if cov is None else None, rots=f32(sc["rotations"]) if cov is None else None,
                    cov=f32(cov) if cov is not None else None, ts=f32(ts) if ts is not None else None,
                    kids=i32(kids) if kids is not None else None, ridx=i32(ridx) if ridx is not None else None,
                    pidx=i32(pidx) if pidx is not None else None)
        n_src = sc["means3D"].shape[0]
        a.P = int(P if P is not None else (len(ridx) if ridx is not None else n_src))
        a.sh_degree, a.sh_coeffs = sh_degree, (sc["shs"].shape[1] if colors is None else 0)
        a.image_width, a.image_height = cam.W, cam.H
        a.tanfovx, a.tanfovy, a.scale_modifier = cam.tanfovx, cam.tanfovy, 1.0
        a.prefiltered, a.debug, a.do_depth = 0, 0, int(do_depth)
        a.bg, a.viewmatrix, a.projmatrix, a.campos = ptr(keep["bg"]), ptr(keep["view"]), ptr(keep["proj"]), ptr(keep["campos"])
        a.means3D, a.shs, a.colors_precomp, a.opacities = ptr(keep["means"]), ptr(keep["shs"]), ptr(keep["colors"]), ptr(keep["opac"])
        a.scales, a.rotations, a.cov3D_precomp = ptr(keep["scales"]), ptr(keep["rots"]), ptr(keep["cov"])
        a.interpolation_weights, a.num_node_kids = ptr(keep["ts"]), ptr(keep["kids"])
        a.render_indices, a.parent_indices, a.num_source = ptr(keep["ridx"]), ptr(keep["pidx"]), (n_src if ridx is not None else 0)
        a.shard_count, a.shard_index = shard
        a.grad_row_begin, a.grad_row_end = int(grad_rows[0]), int(grad_rows[1])
        a.bin_capacity, a.sort_capacity = int(bin_capacity), int(sort_capacity)
        return a, keep

    def forward(self, a, keep):
        W, H, P = a.image_width, a.image_height, a.P
        bufs = [None, None, None]

        def alloc(_user, which, nbytes):
            bufs[which] = aligned(max(int(nbytes), 1))
            return bufs[which].ctypes.data
        cb = _lib.ALLOC_FN(alloc)
        color = aligned(3 * H * W * 4, np.float32, (3, H, W))
        invd = aligned(H * W * 4, np.float32, (1, H, W)) if a.do_depth else None
        radii = aligned(max(P, 1) * 4, np.int32, (max(P, 1),))
        n = C.c_int64(0)
        self.check(self.L.h3dgs_rasterize_forward(C.byref(a), cb, None, ptr(color), ptr(radii), ptr(invd), C.byref(n), None))
        return dict(color=color, radii=radii[:P], invdepth=invd, D=int(n.value), bufs=bufs, keep=keep, cb=cb)

    def state(self, a, fwd):
        v = _lib.StateView()
        b = fwd["bufs"]
        self.check(self.L.h3dgs_state_layout(a.P, a.image_width, a.image_height, fwd["D"], ptr(b[0]), ptr(b[1]), ptr(b[2]), C.byref(v)))

        def view(buf, p, dtype, count):
            off = p - buf.ctypes.data
            return buf[off:off + count * np.dtype(dtype).itemsize].view(dtype)
        D, T = fwd["D"], ((a.image_width + 15) // 16) * ((a.image_height + 15) // 16)
        out = dict(ranges=view(b[2], v.ranges, np.uint32, 2 * T).reshape(T, 2),
                   final_T=view(b[2], v.final_T, np.float32, a.image_width * a.image_height),
                   n_contrib=view(b[2], v.n_contrib, np.uint32, a.image_width * a.image_height))
        if getattr(v, "scan_info", None):
            out["scan_info"] = view(b[2], v.scan_info, np.uint32, 3)
        if D > 0:
            out["point_list"] = view(b[1], v.point_list, np.uint32, D)
            out["keys_sorted"] = view(b[1], v.keys_sorted, np.uint64, D)
            out["sorted_records"] = view(b[1], v.sorted_records, np.float32, 12 * D).reshape(D, 12)
        return out

    def backward(self, a, fwd, dL_dcolor, dL_dinvdepth=None, phases=3, scratch=None, outs=None):
        """phases / scratch as in h3dgs_rasterize_backward: 1 fills `scratch` with the [P][10] sums (returned as
        g["scratch"]), 2 consumes it; outs: the gradient arrays of an earlier call (split phases with flags 4 / 8)"""
        P = a.P
        N = a.num_source if a.render_indices else P
        M = a.sh_coeffs
        g = dict(means3D=aligned(N * 12, np.float32, (N, 3)), means2D=aligned(P * 12, np.float32, (P, 3)),
                 sh=aligned(max(N * M * 12, 4), np.float32, (N, M, 3)) if M else None,
                 colors_precomp=aligned(N * 12, np.float32, (N, 3)) if a.colors_precomp else None,
                 opacities=aligned(N * 4, np.float32, (N, 1)),
                 scales=aligned(N * 12, np.float32, (N, 3)) if a.scales else None,
                 rotations=aligned(N * 16, np.float32, (N, 4)) if a.rotations else None,
                 cov3Ds_precomp=aligned(N * 24, np.float32, (N, 6)) if a.cov3D_precomp else None)
        if outs is not None:
            g = {k: outs[k] for k in g}
        if scratch is None:
            scratch = aligned(self.L.h3dgs_backward_scratch_bytes(P))
        gcol = f32(dL_dcolor)
        gdep = f32(dL_dinvdepth) if (a.do_depth and dL_dinvdepth is not None) else None
        b = fwd["bufs"]
        self.check(self.L.h3dgs_rasterize_backward(C.byref(a), ptr(fwd["radii"]), ptr(b[0]), ptr(b[1]), ptr(b[2]), fwd["D"],
                                                   ptr(gcol), ptr(gdep), ptr(g["means3D"]), ptr(g["means2D"]), ptr(g["sh"]),
                                                   ptr(g["colors_precomp"]), ptr(g["opacities"]), ptr(g["scales"]),
                                                   ptr(g["rotations"]), ptr(g["cov3Ds_precomp"]), ptr(scratch), int(phases), None))
        g["scratch"] = scratch
        return g

"""Screen-tile-sharded multi-GPU mode (new functionality: the reference is single-GPU,
SURVEY.md 8e).  One process per GPU, torch.distributed (NCCL over NVLink/NVSwitch on
the GPU box; gloo in the CPU tests of the host logic).

Per frame, with G ranks and replicated parameters:
  * every rank runs the LOD cut, the cut gather/lerp and K1 on the whole cut (HBM-bound
    streams), but bins / sorts / blends only the 16-px tile rows y with y % G == rank;
  * forward exchange : ONE all-gather of the packed per-rank slabs [rows][3][16][W];
  * the loss is evaluated on the full image on every rank (replicated), so no second
    image exchange is needed for dL/dcolor;
  * backward exchange: ONE reduce-scatter of the [P,10] 2D-space gradient sums (40 B per
    Gaussian, taken BEFORE the per-Gaussian chain rule: 6x less traffic than reducing the
    248 B of final gradients); K8/K9 then run on each rank's own row block only, so the
    parameter gradients come out sharded by rendered row (sum over ranks = the full gradient).
G == 1 never touches torch.distributed.
"""
import torch
import torch.distributed as dist

from diff_gaussian_rasterization import _C
from . import pipeline

TILE = 16


def owned_rows(H, world, rank):
    gy = (H + TILE - 1) // TILE
    return (gy + world - 1 - rank) // world


def rows_per_rank(H, world):
    gy = (H + TILE - 1) // TILE
    return (gy + world - 1) // world


def pack_index(H, world):
    """image row -> (rank, local tile row, row-in-tile) bookkeeping used by unpack()."""
    gy = (H + TILE - 1) // TILE
    return [(y % world, y // world) for y in range(gy)]


def unpack(gathered, H, W, world):
    """gathered [world, rpr, C, 16, W] -> image [C, H, W] (tile row y lives at rank y % world, slot y // world)."""
    rpr, C = gathered.shape[1], gathered.shape[2]
    img = gathered.permute(2, 1, 0, 3, 4).reshape(C, rpr * world * TILE, W)
    return img[:, :H].contiguous()


def pack_rows(image, world, rank):
    """[C,H,W] full image -> this rank's packed slab [owned rows][C][16][W] (host-side mirror of the
    kernel's packed shard layout; used by tests and by non-kernel producers)."""
    C, H, W = image.shape
    gy = (H + TILE - 1) // TILE
    pad = torch.zeros((C, gy * TILE, W), dtype=image.dtype, device=image.device)
    pad[:, :H] = image
    rows = pad.view(C, gy, TILE, W)[:, rank::world]            # [C, owned, 16, W]
    return rows.permute(1, 0, 2, 3).contiguous()


def gather_image(packed, H, W, world, group=None):
    """ONE all-gather of the per-rank slabs -> full [C,H,W] image on every rank."""
    rpr = rows_per_rank(H, world)
    slab = packed
    if packed.shape[0] != rpr:                # ranks owning one tile row fewer pad their slab
        slab = torch.zeros((rpr,) + tuple(packed.shape[1:]), dtype=packed.dtype, device=packed.device)
        slab[:packed.shape[0]] = packed
    flat = torch.empty((world * rpr,) + tuple(slab.shape[1:]), dtype=slab.dtype, device=slab.device)
    dist.all_gather_into_tensor(flat, slab.contiguous(), group=group)
    return unpack(flat.view((world, rpr) + tuple(slab.shape[1:])), H, W, world)


def row_block(P, world, rank):
    """rendered rows [begin, end) whose gradients rank `rank` finishes (equal blocks, last ones may be short)."""
    chunk = (P + world - 1) // world
    return min(rank * chunk, P), min((rank + 1) * chunk, P)


def accum_scratch(P, world, device):
    """backward scratch holding world equal row blocks of the [P][10] sums (tail rows zero)."""
    chunk = (P + world - 1) // world
    return torch.zeros((max(world * chunk, 1) * 10,), dtype=torch.float32, device=device).view(torch.uint8)


def reduce_accum(accum_bytes, P, world, rank, group=None):
    """ONE reduction of the [P,10] fp32 2D-space gradient sums: a reduce-scatter by row block on NCCL
    (in place: every rank keeps the complete sums of ITS rows only); backends without reduce-scatter
    (gloo, CPU tests) fall back to an all-reduce, of which only the own block is consumed."""
    chunk = (P + world - 1) // world
    acc = accum_bytes.view(torch.float32)[: world * chunk * 10]
    if dist.get_backend(group) == "nccl":
        dist.reduce_scatter_tensor(acc[rank * chunk * 10:(rank + 1) * chunk * 10], acc, op=dist.ReduceOp.SUM, group=group)
    else:
        dist.all_reduce(acc, op=dist.ReduceOp.SUM, group=group)
    return accum_bytes


class _ShardedRasterize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, shs, opacities, scales, rotations, rs, world, rank, group):
        H, W = rs.image_height, rs.image_width
        n, packed, radii, gb, bb, ib, _ = _C.rasterize_gaussians(
            rs.bg, means3D, None, opacities, scales, rotations, rs.scale_modifier, None, rs.viewmatrix, rs.projmatrix,
            rs.tanfovx, rs.tanfovy, H, W, shs, rs.sh_degree, rs.campos, rs.prefiltered, rs.debug, rs.render_indices,
            rs.parent_indices, rs.interpolation_weights, rs.num_node_kids, False, shard=(world, rank),
            grad_rows=row_block(rs.render_indices.numel() if rs.render_indices.numel() else means3D.shape[0], world, rank))
        image = gather_image(packed, H, W, world, group)
        ctx.rs, ctx.n, ctx.shard, ctx.group = rs, n, (world, rank), group
        ctx.save_for_backward(means3D, shs, opacities, scales, rotations, radii, gb, bb, ib)
        ctx.mark_non_differentiable(radii)
        return image, radii

    @staticmethod
    def backward(ctx, grad_img, _grad_radii):
        rs = ctx.rs
        means3D, shs, opacities, scales, rotations, radii, gb, bb, ib = ctx.saved_tensors
        common = (rs.bg, means3D, radii, None, opacities, scales, rotations, rs.scale_modifier, None, rs.viewmatrix,
                  rs.projmatrix, rs.tanfovx, rs.tanfovy)
        tail = (shs, rs.sh_degree, rs.campos, gb, ctx.n, bb, ib, rs.debug, rs.render_indices, rs.parent_indices,
                rs.interpolation_weights, rs.num_node_kids, False, rs.image_height, rs.image_width)
        world, rank = ctx.shard
        P = radii.shape[0]
        # phase 1: per-tile replay on the owned tiles -> partial [P,10] sums
        accum = _C.rasterize_gaussians_backward(*common, grad_img.contiguous(), None, *tail, shard=ctx.shard, phases=1,
                                                scratch=accum_scratch(P, world, radii.device))
        # ONE reduce-scatter by row block; phase 2 (per-Gaussian chain rule) only on the own block:
        # the returned gradients are SHARDED by rendered row (complete for the own block, zero elsewhere)
        reduce_accum(accum, P, world, rank, ctx.group)
        (d_means2D, _dc, d_opac, d_means3D, _dcov, d_sh, d_scales, d_rots) = _C.rasterize_gaussians_backward(
            *common, None, None, *tail, shard=ctx.shard, phases=2, scratch=accum, grad_rows=row_block(P, world, rank))
        return d_means3D, d_sh, d_opac, d_scales, d_rots, None, None, None, None


class TileSharder:
    def __init__(self, world, rank, device, group=None):
        self.world, self.rank, self.device, self.group = world, rank, device, group

    def render(self, scene, cam, bg, threshold=None, sh_degree=3, cull=False):
        if cull:
            raise ValueError("cull=True runs on one GPU: the tile-sharded forms take the unculled cut")
        if scene.hier:
            # fused form: the cut gather + parent lerp run inside K1/K9 (full arrays + indices)
            n, P = pipeline.fused_cut(scene, cam, threshold)
            means, scales, rots, opac, shs = scene.means3D, scene.scales, scene.rotations, scene.opacities, scene.shs
            rs = pipeline.make_settings(scene, cam, bg, sh_degree, ts=scene.interpolation_weights, kids=scene.num_siblings,
                                        ridx=scene.render_indices[:P], pidx=scene.parent_indices[:P])
        else:
            n = scene.means3D.shape[0]
            means, scales, rots, opac, shs = scene.means3D, scene.scales, scene.rotations, scene.opacities, scene.shs
            rs = pipeline.make_settings(scene, cam, bg, sh_degree)
        img, radii = _ShardedRasterize.apply(means, shs, opac, scales, rots, rs, self.world, self.rank, self.group)
        return img, radii, n

    def l1_step(self, scene, cam, bg, gt, threshold=None, sh_degree=3, gt_ready=None, cull=False):
        scene.zero_grad()
        img, radii, n = self.render(scene, cam, bg, threshold, sh_degree, cull)
        if gt_ready is not None:
            torch.cuda.current_stream().wait_event(gt_ready)
        loss = (img - gt).abs().mean()
        loss.backward()
        return loss, radii, n

/*
 * h3dgs.h -- C-ABI of libh3dgs.so, the H100-native (sm_90a) replacement for the
 * native ops below the reference's drop-in boundary (SURVEY.md section 8b):
 *
 *   diff_gaussian_rasterization._C.rasterize_gaussians          -> h3dgs_rasterize_forward
 *   diff_gaussian_rasterization._C.rasterize_gaussians_backward -> h3dgs_rasterize_backward
 *   diff_gaussian_rasterization._C.mark_visible                 -> h3dgs_mark_visible
 *   gaussian_hierarchy._C.expand_to_size                        -> h3dgs_expand_to_size
 *   gaussian_hierarchy._C.get_interpolation_weights             -> h3dgs_get_interpolation_weights
 *   (both of the above, device-side, for a graph-captured step)  -> h3dgs_lod_cut
 *   simple_knn._C.distCUDA2                                      -> h3dgs_dist_knn3
 *   the GaussianHierarchyCreator executable                      -> h3dgs_build_hierarchy
 *   the GaussianHierarchyMerger executable                       -> h3dgs_merge_hierarchies
 *
 * The reference binds those through two pip packages whose source is absent from
 * the reference checkout (empty submodules, .gitmodules:5-13); the interface is pinned by
 * the call sites:
 *   GaussianRasterizationSettings(17 kwargs) gaussian_renderer/__init__.py:44-62, 247-265, 319-337
 *   rasterizer(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp)
 *                                            gaussian_renderer/__init__.py:105-113, 267-277, 381-389
 *   expand_to_size(nodes, boxes, thr, viewpoint(cuda), viewdir(cpu), out x3) -> int   train_post.py:91-99
 *   get_interpolation_weights(node_idx, thr, nodes, boxes, viewpoint(cpu), viewdir(cpu), out x2)
 *                                            train_post.py:104-113
 *
 * Every pointer is a DEVICE pointer unless marked [host].  No torch types cross
 * this boundary; the Python shim (hierarchical-3d-gaussians_b200/diff_gaussian_rasterization)
 * passes tensor.data_ptr() values through ctypes.  All work is enqueued on `stream`;
 * the only host synchronisations are the ones the reference API itself forces
 * (num_rendered sizing of the binning buffer; the int returned by expand_to_size) -- capacity mode
 * (h3dgs_raster_args.bin_capacity) and h3dgs_lod_cut have none.
 * Every entry point returns 0 on success, a negative H3DGS_E* code on error and
 * leaves a message retrievable with h3dgs_last_error() (thread-local).
 *
 * Threading: the reference drives this path from a single Python thread on the default stream
 * (SURVEY.md 8b) and so does the shim.  The library keeps one side stream and one pinned read-back
 * slot PER DEVICE, so calls that target the same device must not overlap in time (different devices --
 * one process or thread per GPU, as in the tile-sharded mode -- are independent).
 */
#ifndef H3DGS_H
#define H3DGS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define H3DGS_VERSION 1
#define H3DGS_TILE 16            /* 16x16-pixel tiles                                         */
#define H3DGS_MAX_PEERS 8        /* ranks of the tile-sharded mode that can share peer memory  */
#define H3DGS_IPC_HANDLE_BYTES 64

#define H3DGS_OK 0
#define H3DGS_EINVAL (-1)        /* bad argument combination (shs xor colors, scales xor cov) */
#define H3DGS_ECUDA (-2)         /* a CUDA call or kernel failed (message has the detail)     */
#define H3DGS_ENOMEM (-3)        /* the alloc callback returned NULL                          */

/* Variable-size scratch is obtained through this callback (the reference's
 * "resizeFunctional" pattern: three byte buffers kept alive by the autograd ctx
 * until backward).  `which`: 0 = geometry state (size known from P), 1 = binning
 * state (size known only after num_rendered), 2 = image state (from W,H).  Must
 * return a device pointer aligned to 256 bytes, valid on `stream`. */
typedef void* (*h3dgs_alloc_fn)(void* user, int which, size_t bytes);

typedef struct h3dgs_raster_args {
    /* sizes */
    int32_t P;              /* Gaussians handed to the rasterizer                              */
    int32_t sh_degree;      /* active degree 0..3                                              */
    int32_t sh_coeffs;      /* K_max = shs.shape[1] (1,4,9,16); 0 when colors_precomp is used  */
    int32_t image_width, image_height;
    /* per-call constants (GaussianRasterizationSettings) */
    float tanfovx, tanfovy, scale_modifier;
    int32_t prefiltered, debug, do_depth;   /* prefiltered: the caller's promise that no point is behind the near plane; a broken promise is an error (exact mode) / word 3 of scan_info (capacity mode), as the reference's kernel traps */
    const float* bg;            /* [3]                                                          */
    const float* viewmatrix;    /* [16] world->view, transposed storage (scene/cameras.py:95)   */
    const float* projmatrix;    /* [16] full projection, transposed storage (:97)               */
    const float* campos;        /* [3]                                                          */
    /* per-Gaussian inputs */
    const float* means3D;       /* [P,3]                                                        */
    const float* shs;           /* [P,K_max,3] or NULL                                          */
    const float* colors_precomp;/* [P,3] or NULL                                                */
    const float* opacities;     /* [P]                                                          */
    const float* scales;        /* [P,3] or NULL                                                */
    const float* rotations;     /* [P,4] wxyz, normalised, or NULL                              */
    const float* cov3D_precomp; /* [P,6] xx,xy,xz,yy,yz,zz or NULL                              */
    /* hierarchy extras (empty tensors at the flat call sites -> NULL) */
    const float* interpolation_weights; /* t  [>=P] or NULL                                     */
    const int32_t* num_node_kids;       /* k  [>=P] or NULL; k <= 1 (negative included) is the
                                           identity, counts above 65535 render as 65535          */
    /* In-kernel cut gather + parent lerp (GaussianRasterizationSettings.render_indices /
     * parent_indices; empty at the shipped call sites, SURVEY.md 8a note 1).  When
     * render_indices != NULL the per-Gaussian inputs above are the FULL arrays with
     * num_source rows and rendered Gaussian i (i < P) is
     *   x = t_i * x[render_indices[i]] + (1 - t_i) * x[parent_indices[i]]
     * for means, scales, SH, opacity and (sign-aligned, un-renormalised) rotations --
     * exactly the arithmetic of render_post(interp_python=True),
     * gaussian_renderer/__init__.py:199-218.  parent < 0 means "no parent" (t must be 1).
     * Backward scatters t*g / (1-t)*g into zero-filled gradients of num_source rows. */
    const int32_t* render_indices;      /* [P] or NULL                                          */
    const int32_t* parent_indices;      /* [P] or NULL                                          */
    int32_t num_source;                 /* rows of the full arrays (ignored when render_indices == NULL) */
    /* screen-tile shard for the multi-GPU mode: this call bins and renders only
     * tile rows y with (y % shard_count) == shard_index.  (1,0) = whole image. */
    int32_t shard_count, shard_index;
    /* Backward phase 2 (per-Gaussian chain rule) only for rendered rows [grad_row_begin, grad_row_end);
     * (0, 0) = all rows.  The multi-GPU mode reduce-scatters the [P][10] sums and lets every rank finish
     * only its own row block, so the final gradients come out sharded by rendered row.  When the row block
     * is also given to the FORWARD of a sharded frame, the SH colour is evaluated only for the Gaussians this
     * rank needs: those touching its tile rows and those in its row block. */
    int32_t grad_row_begin, grad_row_end;
    /* Capacity mode -- no host synchronisation, so the call can be captured in a CUDA graph.  With
     * bin_capacity > 0 the binning state is sized for bin_capacity (tile, Gaussian) entries instead of
     * num_rendered, the per-tile sort is launched for lists of at most sort_capacity entries (0 = 8192,
     * the shared-memory limit) and nothing is read back: *num_rendered = bin_capacity, which is also the
     * value to hand to backward.  A frame that needs more (D > bin_capacity, or a tile list longer than
     * sort_capacity) sets word 2 of h3dgs_state_view.scan_info; its image is the background only and its
     * backward adds nothing -- the caller re-runs it in exact mode (bin_capacity = 0).
     * In both modes a rendered row whose render_indices entry is negative is skipped (radius 0): that is
     * the tail h3dgs_lod_cut leaves after the cut when P is the capacity of the index arrays. */
    int64_t bin_capacity;
    int32_t sort_capacity;
    /* Peer mode of a tile-sharded frame (peer_count == shard_count > 1; one process per GPU on one NVLink / NVSwitch
     * box; memory from h3dgs_peer_alloc / h3dgs_peer_open): the collectives are fused into the blend kernels.
     *  forward : every finished pixel of this rank's tile rows is stored into peer_image[r] ([3,H,W], one per rank,
     *            peer_image[shard_index] = the local one, required) for every r whose pointer is not NULL -- the
     *            all-gather of rendered tiles, tile by tile; out_color is not written.  (Pixel-wise remote stores are
     *            small NVLink packets: a caller that runs h3dgs_l1_loss_grad_peer next passes only its own pointer here
     *            and lets that kernel forward the rows with coalesced stores.)
     *  backward: phase 1 leaves this rank's PARTIAL [P][10] sums (its own tiles) in `scratch` and then PUSHES, for every
     *            row it touched that another rank owns, the 40-byte partial row into that owner's staging area:
     *            peer_stage[owner] is [peer_count][P][10] floats on rank `owner`, slot [shard_index] is ours
     *            (coalesced posted stores over NVLink: consecutive rows have the same owner).  owner(row) =
     *            (row >> grad_cyclic_log2) % peer_count, i.e. blocks of 2^grad_cyclic_log2 rendered rows dealt
     *            round-robin.  Phase 2 finishes exactly the rows this rank owns: per row it adds its own partial row
     *            and the staged rows of the ranks whose tile rows the Gaussian touches (a mask K1 keeps), in rank
     *            order -- the reduce-scatter of the per-Gaussian sums, sparse (only rows that exist travel) and
     *            independent of arrival order.  Nothing in the staging areas needs zeroing.
     * The caller separates the phases with h3dgs_peer_barrier, and the next step's phase 1 from this step's phase 2
     * of the other ranks (a barrier at the start of every step does).  peer_count <= 1: off (grad_row_begin/end apply). */
    int32_t peer_count;
    int32_t grad_cyclic_log2;
    void* peer_image[H3DGS_MAX_PEERS];
    void* peer_stage[H3DGS_MAX_PEERS];
} h3dgs_raster_args;   /* NOTE: keep hierarchical-3d-gaussians_b200/h3dgs/_lib.py::RasterArgs in sync */

/* Forward: K1 preprocess -> scan -> duplicateWithKeys -> radix sort -> tile ranges
 * -> record gather -> per-tile blend.  Outputs: out_color [3,H,W], out_radii [P]
 * (int32), out_invdepth [1,H,W] (written only when do_depth).  With shard_count > 1 the
 * image outputs use the packed shard layout [owned tile row][channel][16][W] (rows
 * beyond H inside the last tile row are not written).  The three state
 * buffers obtained from `alloc` must be kept alive and passed to backward.
 * num_rendered [host] receives D = sum of tiles touched. */
int h3dgs_rasterize_forward(const h3dgs_raster_args* args, h3dgs_alloc_fn alloc, void* alloc_user,
                            float* out_color, int32_t* out_radii, float* out_invdepth,
                            int64_t* num_rendered, void* stream);

/* Backward: per-tile gradient replay -> per-Gaussian chain rule.  All dL_d*
 * outputs are fully written (zeros for culled Gaussians); NULL skips an output
 * that does not apply (dL_dsh when colors_precomp, dL_dscales/rots when cov3D_precomp...).
 * dL_dmeans2D is [P,3] with .z = 0 (consumers read [:, :2], scene/gaussian_model.py:688). */
int h3dgs_rasterize_backward(const h3dgs_raster_args* args, const int32_t* radii,
                             const void* geom_state, const void* binning_state, const void* image_state,
                             int64_t num_rendered,
                             const float* dL_dcolor /*[3,H,W]*/, const float* dL_dinvdepth /*[1,H,W] or NULL*/,
                             float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dsh, float* dL_dcolors_precomp,
                             float* dL_dopacities, float* dL_dscales, float* dL_drotations, float* dL_dcov3D,
                             void* scratch /* >= h3dgs_backward_scratch_bytes(P) device bytes */,
                             int phases /* 3 = whole backward; 1 = per-tile replay only (fills `scratch` with the
                                           [P][10] 2D-space sums); 2 = per-Gaussian chain rule only (consumes it).
                                           The multi-GPU mode exchanges `scratch` between 1 and 2.  Scatter mode
                                           (render_indices): | 4 with phase 1 = zero-fill the full-size gradient outputs
                                           now, beside the replay (they must be passed); | 8 with phase 2 = they are
                                           already zero (an earlier call filled them). */,
                             void* stream);
size_t h3dgs_backward_scratch_bytes(int32_t P);

/* Frustum visibility (near plane), one byte per Gaussian (bool tensor). */
int h3dgs_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                       uint8_t* present, void* stream);

/* Layout introspection for tests (integer artefacts must be bit-exact vs the oracle). */
typedef struct h3dgs_state_view {
    const float* depths;              /* [P] view-space z (key low 32 bits)                    */
    const uint32_t* tiles_touched;    /* [P]                                                    */
    const uint32_t* point_offsets;    /* [P] inclusive scan (filled only by the global-sort fallback)*/
    const float* records;             /* [P][12] x,y,conic.x,conic.y | conic.z,opacity,t,k-bits | r,g,b,invdepth */
    const uint64_t* keys_sorted;      /* [D] (tile << 32) | depth bits                          */
    const uint32_t* point_list;       /* [D] Gaussian index, sorted                             */
    const uint32_t* ranges;           /* [tiles][2]                                             */
    const float* final_T;             /* [H*W]                                                  */
    const uint32_t* n_contrib;        /* [H*W]                                                  */
    const uint32_t* scan_info;        /* [4] D, longest tile list, capacity overflow (0/1), prefiltered violated (0/1) */
} h3dgs_state_view;
int h3dgs_state_layout(int32_t P, int32_t W, int32_t H, int64_t num_rendered,
                       const void* geom_state, const void* binning_state, const void* image_state,
                       h3dgs_state_view* out);

/* ---- hierarchy LOD cut ---- */
/* nodes: [N,7] int32 {depth,parent,start,count_leafs,count_merged,start_children,count_children};
 * boxes: [N,2,4] float {min.xyz,size ; max.xyz,_}, 16-byte aligned (read as float4; the three cut entry points
 * return H3DGS_EINVAL otherwise, before anything is enqueued); nodes needs only int32 alignment.  viewpoint is a DEVICE pointer here
 * (train_post.py:95 passes the cuda camera_center).  Returns the number of rendered
 * Gaussians (>= 0) or a negative error code; synchronises `stream` (the reference API returns a Python int). */
int h3dgs_expand_to_size(int32_t N, const int32_t* nodes, const float* boxes, float target_size,
                         const float* viewpoint, float viewdir_x, float viewdir_y, float viewdir_z,
                         int32_t* render_indices, int32_t* parent_indices, int32_t* nodes_for_render_indices,
                         void* scratch /* >= h3dgs_expand_scratch_bytes(N) */, void* stream);
size_t h3dgs_expand_scratch_bytes(int32_t N);

/* viewpoint passed BY VALUE (train_post.py:109 passes camera_center.cpu()). */
int h3dgs_get_interpolation_weights(int32_t n, const int32_t* node_indices, float target_size,
                                    const int32_t* nodes, const float* boxes,
                                    float viewpoint_x, float viewpoint_y, float viewpoint_z,
                                    float viewdir_x, float viewdir_y, float viewdir_z,
                                    float* ts, int32_t* num_kids, void* stream);

/* Device-side LOD cut for the sync-free step: expand_to_size and get_interpolation_weights in one
 * pass with the same arithmetic, nothing returned to the host.  Outputs as the two calls above
 * (render_indices, parent_indices, nodes_for_render_indices, ts, num_kids: first n entries); in addition
 * render_indices[n .. N) = -1 (rows the rasterizer skips when handed P = N) and *count [device] = n.
 * target_size_dev, when not NULL, is a device float that overrides target_size: train_post.py:66-74 draws a
 * new threshold every step, and a value read on the device can change between replays of a captured graph.
 * scratch as for h3dgs_expand_to_size. */
int h3dgs_lod_cut(int32_t N, const int32_t* nodes, const float* boxes, float target_size, const float* target_size_dev,
                  const float* viewpoint,
                  int32_t* render_indices, int32_t* parent_indices, int32_t* nodes_for_render_indices,
                  float* ts, int32_t* num_kids, int32_t* count, void* scratch, void* stream);

/* ---- peer memory for the tile-sharded multi-GPU mode (csrc/peer.cu) ----
 * h3dgs_peer_alloc: zero-filled device allocation that can be exported to the other ranks' processes (CUDA IPC);
 * h3dgs_peer_export / h3dgs_peer_open: 64-byte handle out / mapped pointer in (the host side exchanges the handles,
 * e.g. with torch.distributed.all_gather_object).  h3dgs_peer_barrier: device-side barrier among `world` ranks, an
 * ordinary kernel on `stream` (no host synchronisation; capturable): flags = this rank's block of
 * h3dgs_peer_flag_bytes() zero-initialised peer memory, peer_flags[r] [host array of `world` device pointers] the
 * block of rank r (peer_flags[rank] == flags).  Everything enqueued on `stream` before the barrier -- including
 * stores and reductions into peer memory -- is visible to every rank's work after it. */
size_t h3dgs_peer_flag_bytes(void);
int h3dgs_peer_alloc(size_t bytes, void** ptr);
int h3dgs_peer_free(void* ptr);
int h3dgs_peer_export(const void* ptr, void* handle /* [H3DGS_IPC_HANDLE_BYTES] */);
int h3dgs_peer_open(const void* handle, void** ptr);
int h3dgs_peer_close(void* ptr);
int h3dgs_peer_barrier(int32_t world, int32_t rank, uint32_t* flags, uint32_t* const* peer_flags, void* stream);
int h3dgs_peer_barrier_status(const uint32_t* flags, void* stream);   /* 1 = a barrier timed out (a peer never arrived) */

/* ---- fused L1 + SSIM loss (SURVEY.md 8f-2; replaces utils/loss_utils.py:17-63 as used in
 * train_post.py:134-140: loss = (1-l) * L1 + l * (1 - SSIM), 11x11 Gaussian window, sigma 1.5) ----
 * forward: sums[0] = sum |img-gt|, sums[1] = sum of the SSIM map (device doubles, zeroed here);
 *          maps [3][C,H,W] (ds/dmu1, ds/dE11, ds/dE12) are written when non-NULL (needed by backward).
 * backward: dL_dimg = coeffs[0] * sign(img-gt) + coeffs[1] * d(sum ssim)/d img ; coeffs is a DEVICE
 *          pointer to two floats so that the upstream gradient never has to visit the host. */
int h3dgs_l1_ssim_forward(int32_t C, int32_t H, int32_t W, const float* img, const float* gt, double* sums,
                          float* maps, void* stream);
int h3dgs_l1_ssim_backward(int32_t C, int32_t H, int32_t W, const float* img, const float* gt, const float* maps,
                           const float* coeffs, float* dL_dimg, void* stream);

/* ---- train_post's objective (train_post.py:134-142 on render_post's exposure and clamp, gaussian_renderer/__init__.py:279-285),
 * fused into the loss kernels above.  img [3,H,W] is the raw rasterizer output, gt [3,H,W] the target as the loader leaves
 * it (already clamped and masked: it is neither clamped nor masked here), exposure a DEVICE [3][4] matrix or NULL (=
 * identity), mask a DEVICE [H,W] alpha mask or NULL (= ones).  Per pixel and channel c:
 *   y_c = exposure ? ((img_0 E[0][c] + img_1 E[1][c]) + img_2 E[2][c]) + E[c][3] : img_c    (every product and sum rounded
 *         in this order: image.permute(1,2,0) @ E[:3,:3] + E[:3,3])
 *   a_c = clamp(y_c, 0, 1) * mask
 * forward: sums[0] = sum |a - gt|, sums[1] = sum of the SSIM map of (a, gt) (device doubles, zeroed here); maps [3][3,H,W]
 *          (ds/dmu1, ds/dE11, ds/dE12 at a) are written when non-NULL (needed by backward).
 * backward: dL/dy_c = [0 <= y_c <= 1] * mask * (coeffs[0] sign(a_c - gt_c) + coeffs[1] d(sum ssim)/d a_c),
 *          dL_dimg_k = (E[k][0] dL/dy_0 + E[k][1] dL/dy_1) + E[k][2] dL/dy_2 (or dL/dy_k without exposure); coeffs is a
 *          DEVICE pointer to two floats.  There is no gradient to the exposure or the mask.
 * With exposure and mask NULL and img in [0, 1] both equal h3dgs_l1_ssim_forward / _backward with C = 3, bit for bit.
 * Nothing synchronises with the host: exposure and mask may change between replays of a CUDA graph. */
int h3dgs_post_loss_forward(int32_t H, int32_t W, const float* img, const float* gt, const float* exposure, const float* mask,
                            double* sums, float* maps, void* stream);
int h3dgs_post_loss_backward(int32_t H, int32_t W, const float* img, const float* gt, const float* exposure, const float* mask,
                             const float* maps, const float* coeffs, float* dL_dimg, void* stream);
/* Status words of the sync-free post-loss step, written by one device thread: out[0] = loss = (1 - lambda) L1 + lambda
 * (1 - SSIM), out[1] = L1 = sums[0] * inv_numel, out[2] = SSIM = sums[1] * inv_numel, out[3] = *count + extra_rows (rows
 * the cut needs), out[4..6] = scan_info[0..2] (D, longest tile list, binning overflow), out[7] = 1 when out[3] >
 * row_capacity. */
int h3dgs_post_step_status(const double* sums, double inv_numel, double lambda_dssim, const int32_t* count, int32_t extra_rows,
                           int32_t row_capacity, const uint32_t* scan_info, double* out, void* stream);

/* L1 loss and its gradient in one pass (the loss of bench.py's step; train_post.py:134-142 with lambda_dssim = 0):
 * *loss_sum [device double, zeroed here] = sum |img - gt|, dL_dimg = sign(img - gt) * scale (scale = 1 / numel for the
 * mean).  With shard_count > 1 only the 16-pixel tile rows y_tile % shard_count == shard_index are visited (loss_sum is
 * then this rank's partial sum and the other rows of dL_dimg are left untouched). */
int h3dgs_l1_loss_grad(int32_t C, int32_t H, int32_t W, const float* img, const float* gt, float scale,
                       int32_t shard_count, int32_t shard_index, float* dL_dimg, double* loss_sum, void* stream);
/* the same, adding this rank's partial sum into loss_sums[0..peer_count) [host array of device pointers, one double
 * per rank in peer memory; NOT zeroed here] so that every rank ends up with the loss of the whole frame.
 * peer_images (optional; needs shard_count == peer_count, W % 4 == 0): host array of the ranks' [C,H,W] images in peer
 * memory -- the pixels of this rank's tile rows are copied from img into peer_images[r], r != shard_index, with
 * coalesced 128-bit stores: the all-gather of the rendered tile rows, fused into the pass that reads them anyway. */
int h3dgs_l1_loss_grad_peer(int32_t C, int32_t H, int32_t W, const float* img, const float* gt, float scale,
                            int32_t shard_count, int32_t shard_index, float* dL_dimg, int32_t peer_count,
                            double* const* loss_sums, float* const* peer_images, void* stream);

/* Status words of a sync-free step, written by one device thread (no host synchronisation, capturable): out[0] =
 * *loss_sum * inv_numel, out[1] = *count + extra_rows (rows the cut needs), out[2..4] = scan_info[0..2] (D, longest tile
 * list, binning overflow), out[5] = 1 when out[1] > row_capacity; reset_loss != 0 zeroes *loss_sum afterwards. */
int h3dgs_step_status(double* loss_sum, double inv_numel, const int32_t* count, int32_t extra_rows, int32_t row_capacity,
                      const uint32_t* scan_info, int32_t reset_loss, double* out, void* stream);

/* ---- evaluation metrics of one frame (csrc/metrics.cu; render_hierarchy.py:82-113 on top of render_post) ----
 * img [3,H,W] (the raw rasterizer output), gt [3,H,W], exposure [3][4] or NULL, mask [H,W] or NULL.  In this order:
 *   a = exposure ? sum_k img[k] * exposure[k][c] + exposure[c][3] : img[c]    (image.permute(1,2,0) @ E[:3,:3] + E[:3,3])
 *   a = clamp(a, 0, 1), b = clamp(gt, 0, 1); both cropped to columns [x0, W) (x0 = W / 2 is train_test_exp, 0 = off);
 *   out_img [3,H,W-x0] (optional) = a; then a *= mask, b *= mask;
 *   psnr = mean_c 20 log10(1 / sqrt(SSE_c / (H (W-x0)))), ssim = mean of the SSIM map (11x11 Gaussian window, sigma 1.5,
 *   zero padding at the border of the cropped frame).
 * sums: 4 device doubles of scratch (zeroed here).  A single device thread then stores one row of H3DGS_EVAL_ROW doubles
 * at results + slot * H3DGS_EVAL_ROW, slot = (*counter)++ (device int; a slot >= max_rows is counted but not stored):
 *   [0] psnr  [1] ssim  [2] overflow (0/1)  [3] rows = *count + extra_rows  [4] D  [5] longest tile list
 * with the status of a capacity-mode frame: count (device int, NULL = 0) as h3dgs_lod_cut leaves it, scan_info (NULL =
 * none) as in h3dgs_state_view; overflow = scan_info[2] != 0 or (row_capacity > 0 and rows > row_capacity).
 * No host synchronisation: a sweep of frames can be enqueued or replayed from a CUDA graph and read back once. */
#define H3DGS_EVAL_ROW 6
int h3dgs_eval_metrics(int32_t H, int32_t W, const float* img, const float* gt, const float* exposure, const float* mask,
                       int32_t x0, float* out_img, double* sums, const int32_t* count, int32_t extra_rows,
                       int32_t row_capacity, const uint32_t* scan_info, int32_t* counter, double* results,
                       int32_t max_rows, void* stream);

/* ---- exact 3-nearest-neighbour distances (csrc/knn.cu; simple_knn._C.distCUDA2, scene/gaussian_model.py:21, 190-194) ----
 * points [P,3] float, mean_dist2 [P] float.  mean_dist2[i] = ((b0 + b1) + b2) / 3.0f, where b0 <= b1 <= b2 are the three
 * smallest d = (dx*dx + dy*dy) + dz*dz, dx = q.x - p.x (fp32, every operation rounded, no FMA), over the points q of OTHER
 * indices (an exact duplicate of p counts, with d = 0).  A missing neighbour (fewer than three other points) counts as
 * FLT_MAX.  Points with a non-finite coordinate are ignored by every finite point; their own rows are unspecified.
 * The result depends only on the set of points.  scratch: >= h3dgs_knn_scratch_bytes(P) device bytes, 256-byte aligned.
 * No host synchronisation.  P = 0 enqueues nothing; P < 0, or a NULL pointer with P > 0, is H3DGS_EINVAL. */
size_t h3dgs_knn_scratch_bytes(int64_t P);
int h3dgs_dist_knn3(int32_t P, const float* points, float* mean_dist2, void* scratch, void* stream);

/* ---- hierarchy creator (csrc/hier_build.cu; the GaussianHierarchyCreator stage of scripts/full_train.py:185-200) ----
 * This project's own rule (upstream's creator is not available to compare with).  Input: P >= 1 Gaussians in the .hier
 * representation: xyz [P,3], log_scales [P,3], rotations [P,4] wxyz of any norm, activated opacities [P], shs [P,16,3].
 * Output: N = 2P - 1 nodes and N Gaussian rows, row i belongs to node i: out_xyz [N,3], out_shs [N,16,3],
 * out_opacities [N], out_log_scales [N,3], out_rotations [N,4], out_nodes [N,7], out_boxes [N,2,4] (16-byte aligned),
 * out_source [N] (the input index of a leaf row, -1 for a merged row).
 *  Topology: the binary radix tree of the augmented keys (key, sorted position).  key = 63-bit Morton code, 21 bits per
 *    axis, x in the highest bit of every triple: q = min(2097151, (uint32)((x - lo) * s)), s = 2097152.0f / (hi - lo)
 *    (0 when hi == lo), lo / hi the bounding box of the positions, every operation rounded in fp32.  The keys are sorted
 *    stably (input index as the value); every internal node splits its range at the highest differing bit; every leaf
 *    holds one Gaussian.
 *  Node order: BFS, i.e. by (level from the root, first sorted position of the range): siblings are adjacent (the lower
 *    range first) and every level is a contiguous index range.
 *  Nodes: {depth = height (0 at leaves), parent (-1 at the root), start = i, count_leafs = 1 | 0, count_merged = 0 | 1,
 *    start_children (0 at a leaf), count_children = 0 | 2}.
 *  Leaf rows: bit-exact copies of input row source[i] (the rotation stays unnormalised).
 *  Merged rows, fp64: per leaf sigma = exp(log_scale), R from the normalised quaternion (a zero quaternion counts as the
 *    identity), Sigma_i = R diag(sigma^2) R^T, A_i = s1 s2 + s1 s3 + s2 s3, w_i = o_i A_i.  Per node over the leaves of its
 *    subtree: W = sum w_i, mu = sum w_i mu_i / W, Sigma = sum w_i (Sigma_i + d_i d_i^T) / W with d_i = mu_i - mu,
 *    SH = sum w_i SH_i / W; computed from the two children carrying W, which is the same formula.  W = 0: the unweighted
 *    mean of the two children's moments (mu, Sigma with the d d^T term, SH).  Eigenvalues of Sigma floored at 1e-24 give
 *    log_scale = log(sqrt(lambda)), in descending order, and opacity = W / A(sqrt(lambda)) (not clamped; W = 0 gives 0);
 *    the eigenvectors give the rotation: unit, right-handed, w >= 0.
 *  Boxes: a leaf's is mu +- 3 sqrt(diag Sigma_i) rounded to fp32, an interior node's the fp32 union of its children's
 *    (nesting is exact); min.w = largest extent (fp32 max - min), max.w = 0.
 * H3DGS_EINVAL: P < 1, P > 2^30, a NULL pointer, out_boxes not 16-byte aligned, a non-finite position, log-scale or
 * rotation component, a log-scale above 300 (its square would overflow the fp64 moments), or a negative or non-finite
 * opacity (nothing is written to the outputs then).  An offline tool: it synchronises `stream` (twice), and returns
 * after enqueueing the last merge.  The result depends only on the input.  scratch: >= h3dgs_build_hierarchy_scratch_bytes(P)
 * device bytes, 256-byte aligned (0 for P out of range): about 1 kB per input Gaussian (fp64 moments and SH of the
 * 2P - 1 nodes), so memory, not the 2^30 limit, bounds P in practice (some 70 M Gaussians on an 80 GB device). */
size_t h3dgs_build_hierarchy_scratch_bytes(int64_t P);
int h3dgs_build_hierarchy(int32_t P, const float* xyz, const float* log_scales, const float* rotations,
                          const float* opacities, const float* shs, float* out_xyz, float* out_shs, float* out_opacities,
                          float* out_log_scales, float* out_rotations, int32_t* out_nodes, float* out_boxes,
                          int32_t* out_source, void* scratch, void* stream);

/* ---- hierarchy merger (csrc/hier_merge.cu; the GaussianHierarchyMerger stage of scripts/full_train.py:241-264) ----
 * This project's own rule (upstream's merger is not available to compare with).  Input: K >= 1 chunk hierarchies in
 * the .hier representation, concatenated in argv order: rows xyz [M,3], shs [M,16,3], activated opacities [M],
 * log_scales [M,3], rotations [M,4]; nodes [N,7] {depth, parent, start, count_leafs, count_merged, start_children,
 * count_children} with chunk-local indices; boxes [N,2,4].  Chunk c owns nodes [node_offsets[c], node_offsets[c+1]) and
 * rows [row_offsets[c], row_offsets[c+1]) (host int64 arrays of K + 1, from 0, not decreasing) and a cell
 * cells[4c .. 4c+3] = (cx, cy, ex, ey) (host fp32: the x and y of its center.txt and extent.txt, full widths).
 *  Rows that no node claims are dropped (the skybox train_post appends).  A leaf Gaussian is a row a node counts in
 *    its count_leafs.
 *  Ownership: a leaf Gaussian at (x, y) belongs to the chunk j minimising the key (k1, k2, j), in fp32 without FMA:
 *    ax = |x - cx|, ox = max(ax - 0.5f * ex, 0) (y alike), k1 = ox*ox + oy*oy, k2 = max(ax / ex, ay / ey).  Chunk c
 *    keeps only the leaf Gaussians it owns; merged rows are never tested.
 *  Pieces: a node of chunk c is pure when every leaf Gaussian of its subtree is owned by c (vacuously so without
 *    any).  Items of chunk c: every maximal pure subtree holding a leaf Gaussian, kept whole (rows, boxes, all its
 *    descendants); every owned leaf Gaussian of an impure node, as a one-Gaussian item.  Impure nodes are dropped.
 *    Item order: the subtree items by global node index, then the one-Gaussian items by global row index.
 *  Top tree: the R items are the P leaves of h3dgs_build_hierarchy's tree: an item's moments (W, mu, Sigma, SH) are
 *    that function's fp64 formulas over the leaf Gaussians of the item (W = 0: their unweighted mean), its position
 *    for the Morton key is mu rounded to fp32; a subtree item keeps its input box, a one-Gaussian item gets the
 *    creator's leaf box.  Summation order (fixed, so the result is repeatable): the item's leaf Gaussians in global row
 *    order, lane l of 32 summing positions l, l + 32, ... in turn, the 32 partial sums then combined by an xor
 *    butterfly (offsets 16, 8, 4, 2, 1).  A restatement that sums in another order, or evaluates exp differently, can
 *    put mu on the other side of an fp32 rounding boundary and so change a Morton key (about 1e-9 per multi-Gaussian
 *    item); a one-Gaussian item's mu rounds to its own position.  Top interior nodes get the creator's merged row,
 *    depth 1 + the larger child depth and the union box.  R = 1: the single item is the root.
 *  Output: nodes [0, 2R - 1) are the top tree in the creator's BFS order, its leaf slots the items; then the
 *    non-root nodes of the kept subtrees, chunk by chunk, each in input order.  Rows follow node order, each node's
 *    block in its input order; a top interior node holds one merged row (count_leafs 0, count_merged 1), a one-
 *    Gaussian item one leaf row (depth 0, count_leafs 1, no children).  parent, start and start_children are
 *    renumbered (start_children 0 without children; the start of a node without rows is where its block would begin,
 *    at most the last row); count_children counts kept children; everything else in a kept node, and every kept row
 *    and box, is a bit-exact copy.  source_chunk / source_row [RO]: the input chunk and chunk-local row of every output
 *    row, -1 / -1 for a merged top row.  On creator-built inputs every node holds one row with start = its index.
 *  Sizes: the outputs are allocated through `alloc(alloc_user, which, bytes)` once their sizes are known, after the
 *    checks: which = 9 a work block (first; 256-byte aligned), then 0 xyz [RO,3], 1 shs [RO,16,3], 2 opacities [RO],
 *    3 log_scales [RO,3], 4 rotations [RO,4], 5 nodes [NO,7] int32, 6 boxes [NO,2,4], 7 source_chunk [RO] int32,
 *    8 source_row [RO] int32.  counts (host int64[3]) receives {NO, RO, R}.
 * H3DGS_EINVAL, with nothing allocated or written: a NULL pointer, K < 1, bad offsets, no node or no row, more than
 * 2^31 - 1 nodes plus rows; an inconsistent node table (an index out of range, a child whose parent disagrees, a row
 * claimed by two nodes, a parent chain longer than N); a leaf Gaussian failing h3dgs_build_hierarchy's input checks; a
 * cell with a non-finite center or an extent that is not finite and positive; no chunk owning anything; more than
 * 2^31 - 1 output nodes or rows.  Every one of these is found before the first `alloc` call.  H3DGS_ENOMEM: `alloc`
 * returned NULL.  An offline tool: it synchronises `stream`
 * several times and returns after enqueueing the last copy.  The result depends only on the input (no fp64 atomics).
 * scratch: >= h3dgs_merge_hierarchies_scratch_bytes(K, N, M) device bytes, 256-byte aligned (0 when out of range):
 * about 50 bytes per node and row; the work block is about 1.4 kB per item. */
size_t h3dgs_merge_hierarchies_scratch_bytes(int32_t K, int64_t total_nodes, int64_t total_rows);
int h3dgs_merge_hierarchies(int32_t K, const int64_t* node_offsets, const int64_t* row_offsets, const float* cells,
                            const float* xyz, const float* shs, const float* opacities, const float* log_scales,
                            const float* rotations, const int32_t* nodes, const float* boxes, h3dgs_alloc_fn alloc,
                            void* alloc_user, int64_t* counts, void* scratch, void* stream);

/* ---- sparse Adam (SURVEY.md 8f-4; replaces scene/OurAdam.py:249-337 as driven by train_single.py:170-178) ----
 * In-place Adam update of the rows listed in relevant[num_relevant] (int64 row indices) of one parameter
 * tensor viewed as [rows, width]; `step` is the 1-based step count of that tensor (the reference
 * increments it on every call, whatever the rows).  amsgrad off, weight_decay 0, minimise. */
int h3dgs_sparse_adam(int64_t num_relevant, int32_t width, const int64_t* relevant, float* param, const float* grad,
                      float* exp_avg, float* exp_avg_sq, double lr, double beta1, double beta2, double eps, int64_t step,
                      void* stream);

/* ---- per-stage device timing (bench.py roofline) ----
 * When enabled, every stage launch is bracketed by two cudaEvents recorded on the stream
 * the kernel is launched on; h3dgs_profile_read synchronises them and returns the summed
 * device time and the number of launches of that stage since the last reset. */
enum {
    H3DGS_STAGE_PREPROCESS = 0, H3DGS_STAGE_SCAN, H3DGS_STAGE_DUPLICATE, H3DGS_STAGE_SORT, H3DGS_STAGE_RANGES,
    H3DGS_STAGE_GATHER, H3DGS_STAGE_RENDER_FWD, H3DGS_STAGE_RENDER_BWD, H3DGS_STAGE_PREPROCESS_BWD,
    H3DGS_STAGE_LOD_CUT, H3DGS_STAGE_LOD_WEIGHTS, H3DGS_STAGE_PREPROCESS_COLOR, H3DGS_STAGE_SH_BACKWARD,
    H3DGS_STAGE_COUNT
};
int h3dgs_profile_enable(int on);
int h3dgs_profile_reset(void);
int h3dgs_profile_read(int stage, double* total_ms, int64_t* launches);
const char* h3dgs_stage_name(int stage);

const char* h3dgs_last_error(void);
int h3dgs_version(void);
/* number of kernel launches issued by this library since load (bench.py "gpu_launches") */
int64_t h3dgs_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* H3DGS_H */

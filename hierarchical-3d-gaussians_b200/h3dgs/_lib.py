"""ctypes binding of libh3dgs.so (include/h3dgs.h).

There is NO CPU fallback: if the library is missing or a call fails this raises.
The oracle under /oracle is never imported from here.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# H3DGS_LIBRARY: another build of the same sources (an A/B variant from build.py --variant), by file name under lib/ or by path
LIB_PATH = os.path.join(os.path.dirname(_HERE), "lib", "libh3dgs.so")
if os.environ.get("H3DGS_LIBRARY"):
    _v = os.environ["H3DGS_LIBRARY"]
    LIB_PATH = _v if os.path.isabs(_v) else os.path.join(os.path.dirname(_HERE), "lib", _v)

ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_int, C.c_size_t)

EXPORTS = [
    "h3dgs_rasterize_forward", "h3dgs_rasterize_backward", "h3dgs_backward_scratch_bytes", "h3dgs_mark_visible",
    "h3dgs_state_layout", "h3dgs_expand_to_size", "h3dgs_expand_scratch_bytes", "h3dgs_get_interpolation_weights",
    "h3dgs_lod_cut", "h3dgs_lod_budget", "h3dgs_lod_budget_scratch_bytes", "h3dgs_lod_cull_mask", "h3dgs_lod_cut_masked",
    "h3dgs_lod_budget_masked",
    "h3dgs_last_error", "h3dgs_version", "h3dgs_launch_count",
    "h3dgs_profile_enable", "h3dgs_profile_reset", "h3dgs_profile_read", "h3dgs_stage_name",
    "h3dgs_l1_ssim_forward", "h3dgs_l1_ssim_backward", "h3dgs_l1_loss_grad", "h3dgs_l1_loss_grad_peer", "h3dgs_step_status", "h3dgs_sparse_adam",
    "h3dgs_peer_flag_bytes", "h3dgs_peer_alloc", "h3dgs_peer_free", "h3dgs_peer_export", "h3dgs_peer_open", "h3dgs_peer_close",
    "h3dgs_peer_barrier", "h3dgs_peer_barrier_status", "h3dgs_eval_metrics",
    "h3dgs_knn_scratch_bytes", "h3dgs_dist_knn3", "h3dgs_build_hierarchy_scratch_bytes", "h3dgs_build_hierarchy",
    "h3dgs_merge_hierarchies_scratch_bytes", "h3dgs_merge_hierarchies",
    "h3dgs_post_loss_forward", "h3dgs_post_loss_backward", "h3dgs_post_step_status",
    "h3dgs_post_loss_backward_exposure", "h3dgs_invdepth_l1_grad", "h3dgs_densify_stats", "h3dgs_single_step_status",
    "h3dgs_coarse_loss_forward", "h3dgs_coarse_loss_backward", "h3dgs_coarse_step_status", "h3dgs_coarse_param_step",
    "h3dgs_post_param_step", "h3dgs_densify_scratch_bytes", "h3dgs_densify",
    "h3dgs_lpips_weight_floats", "h3dgs_lpips_pack_weights", "h3dgs_lpips_scratch_floats", "h3dgs_lpips_features",
    "h3dgs_lpips_distance", "h3dgs_lpips_conv",
]
MAX_PEERS = 8
IPC_HANDLE_BYTES = 64
EVAL_ROW = 6            # H3DGS_EVAL_ROW: psnr, ssim, overflow, rows, D, longest tile list
LPIPS_MIN_SIZE = 16     # H3DGS_LPIPS_MIN_SIZE


class RasterArgs(C.Structure):
    """struct h3dgs_raster_args"""
    _fields_ = [
        ("P", C.c_int32), ("sh_degree", C.c_int32), ("sh_coeffs", C.c_int32),
        ("image_width", C.c_int32), ("image_height", C.c_int32),
        ("tanfovx", C.c_float), ("tanfovy", C.c_float), ("scale_modifier", C.c_float),
        ("prefiltered", C.c_int32), ("debug", C.c_int32), ("do_depth", C.c_int32),
        ("bg", C.c_void_p), ("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p), ("campos", C.c_void_p),
        ("means3D", C.c_void_p), ("shs", C.c_void_p), ("colors_precomp", C.c_void_p), ("opacities", C.c_void_p),
        ("scales", C.c_void_p), ("rotations", C.c_void_p), ("cov3D_precomp", C.c_void_p),
        ("interpolation_weights", C.c_void_p), ("num_node_kids", C.c_void_p),
        ("render_indices", C.c_void_p), ("parent_indices", C.c_void_p), ("num_source", C.c_int32),
        ("shard_count", C.c_int32), ("shard_index", C.c_int32),
        ("grad_row_begin", C.c_int32), ("grad_row_end", C.c_int32),
        ("bin_capacity", C.c_int64), ("sort_capacity", C.c_int32),
        ("peer_count", C.c_int32), ("grad_cyclic_log2", C.c_int32),
        ("peer_image", C.c_void_p * 8), ("peer_stage", C.c_void_p * 8),
    ]


COARSE_SCRATCH_BYTES = 64     # H3DGS_COARSE_SCRATCH_BYTES
COARSE_STEP, COARSE_ACTIVATE, COARSE_BIAS = 0, 1, 2


class CoarseArgs(C.Structure):
    """struct h3dgs_coarse_args"""
    _fields_ = [
        ("N", C.c_int32), ("sh_coeffs", C.c_int32), ("skybox_points", C.c_int32), ("rescale_threshold", C.c_float),
        ("params", C.c_void_p * 6), ("exp_avg", C.c_void_p * 6), ("exp_avg_sq", C.c_void_p * 6),
        ("lr", C.c_double * 6), ("beta1", C.c_double * 6), ("beta2", C.c_double * 6), ("eps", C.c_double * 6),
        ("step", C.c_void_p), ("scratch", C.c_void_p),
        ("grad_means3D", C.c_void_p), ("grad_shs", C.c_void_p), ("grad_opacities", C.c_void_p), ("grad_scales", C.c_void_p),
        ("grad_rotations", C.c_void_p),
        ("means3D", C.c_void_p), ("shs", C.c_void_p), ("opacities", C.c_void_p), ("scales", C.c_void_p),
        ("rotations", C.c_void_p), ("scan_info", C.c_void_p),
    ]


SINGLE_SCRATCH_BYTES = 64     # H3DGS_SINGLE_SCRATCH_BYTES
SINGLE_STEP, SINGLE_NO_GAUSSIAN_STEP, SINGLE_EXPOSURE_ROW, SINGLE_BIAS = 0, 1, 2, 3


class SingleArgs(C.Structure):
    """struct h3dgs_single_args"""
    _fields_ = [
        ("gauss", CoarseArgs), ("skybox_locked", C.c_int32), ("scaffold_points", C.c_int32), ("n_images", C.c_int32),
        ("lrs", C.c_void_p), ("exposure", C.c_void_p), ("exposure_exp_avg", C.c_void_p), ("exposure_exp_avg_sq", C.c_void_p),
        ("exposure_step", C.c_void_p), ("exposure_beta1", C.c_double), ("exposure_beta2", C.c_double),
        ("exposure_eps", C.c_double), ("exposure_grad", C.c_void_p), ("image_index", C.c_void_p), ("exposure_row", C.c_void_p),
    ]


POST_SCRATCH_BYTES = 64       # H3DGS_POST_SCRATCH_BYTES
POST_STEP, POST_ACTIVATE, POST_BIAS = 0, 1, 2


class PostArgs(C.Structure):
    """struct h3dgs_post_args"""
    _fields_ = [
        ("gauss", CoarseArgs), ("lrs", C.c_void_p), ("locked", C.c_void_p), ("count", C.c_void_p),
        ("extra_rows", C.c_int32), ("row_capacity", C.c_int32),
    ]


DENSIFY_COUNT, DENSIFY_WRITE, DENSIFY_RESET_OPACITY = 0, 1, 2


class DensifyArgs(C.Structure):
    """struct h3dgs_densify_args"""
    _fields_ = [
        ("N", C.c_int32), ("sh_coeffs", C.c_int32), ("scaffold_points", C.c_int32), ("skybox_points", C.c_int32),
        ("max_grad", C.c_float), ("min_opacity", C.c_float), ("size_threshold", C.c_float),
        ("params", C.c_void_p * 6), ("exp_avg", C.c_void_p * 6), ("exp_avg_sq", C.c_void_p * 6),
        ("xyz_gradient_accum", C.c_void_p), ("max_radii2D", C.c_void_p), ("flags", C.c_void_p), ("scratch", C.c_void_p),
        ("out_rows", C.c_int64), ("split_rows", C.c_int32), ("normals", C.c_void_p),
        ("out_params", C.c_void_p * 6), ("out_exp_avg", C.c_void_p * 6), ("out_exp_avg_sq", C.c_void_p * 6),
    ]


class StateView(C.Structure):
    """struct h3dgs_state_view"""
    _fields_ = [(n, C.c_void_p) for n in ("depths", "tiles_touched", "point_offsets", "records", "keys_sorted",
                                          "point_list", "ranges", "final_T", "n_contrib", "scan_info",
                                          "sorted_records")]


_lib = None


def bind(l):
    """ctypes prototypes of include/h3dgs.h on a loaded library (libh3dgs.so; the test suite also binds its
    CPU emulation build of the same sources)."""
    l.h3dgs_last_error.restype = C.c_char_p
    l.h3dgs_launch_count.restype = C.c_int64
    l.h3dgs_backward_scratch_bytes.restype = C.c_size_t
    l.h3dgs_backward_scratch_bytes.argtypes = [C.c_int32]
    l.h3dgs_expand_scratch_bytes.restype = C.c_size_t
    l.h3dgs_expand_scratch_bytes.argtypes = [C.c_int32]
    l.h3dgs_rasterize_forward.restype = C.c_int
    l.h3dgs_rasterize_forward.argtypes = [C.POINTER(RasterArgs), ALLOC_FN, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]
    l.h3dgs_rasterize_backward.restype = C.c_int
    l.h3dgs_rasterize_backward.argtypes = [C.POINTER(RasterArgs), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_int64, C.c_void_p, C.c_void_p] + [C.c_void_p] * 8 + [C.c_void_p, C.c_int, C.c_void_p]
    l.h3dgs_mark_visible.restype = C.c_int
    l.h3dgs_mark_visible.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    l.h3dgs_state_layout.restype = C.c_int
    l.h3dgs_state_layout.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.POINTER(StateView)]
    l.h3dgs_expand_to_size.restype = C.c_int
    l.h3dgs_expand_to_size.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_float, C.c_float,
                                       C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    l.h3dgs_get_interpolation_weights.restype = C.c_int
    l.h3dgs_get_interpolation_weights.argtypes = [C.c_int32, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p] + \
        [C.c_float] * 6 + [C.c_void_p, C.c_void_p, C.c_void_p]
    l.h3dgs_l1_loss_grad.restype = C.c_int
    l.h3dgs_l1_loss_grad.argtypes = [C.c_int32] * 3 + [C.c_void_p, C.c_void_p, C.c_float, C.c_int32, C.c_int32,
                                     C.c_void_p, C.c_void_p, C.c_void_p]
    l.h3dgs_step_status.restype = C.c_int
    l.h3dgs_step_status.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    l.h3dgs_l1_loss_grad_peer.restype = C.c_int
    l.h3dgs_l1_loss_grad_peer.argtypes = [C.c_int32] * 3 + [C.c_void_p, C.c_void_p, C.c_float, C.c_int32, C.c_int32,
                                          C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p]
    if hasattr(l, "h3dgs_peer_alloc"):           # peer memory (CUDA IPC, device-side barrier): absent from the emulation build
        l.h3dgs_peer_flag_bytes.restype = C.c_size_t
        l.h3dgs_peer_alloc.restype = C.c_int
        l.h3dgs_peer_alloc.argtypes = [C.c_size_t, C.POINTER(C.c_void_p)]
        l.h3dgs_peer_free.restype = C.c_int
        l.h3dgs_peer_free.argtypes = [C.c_void_p]
        l.h3dgs_peer_export.restype = C.c_int
        l.h3dgs_peer_export.argtypes = [C.c_void_p, C.c_void_p]
        l.h3dgs_peer_open.restype = C.c_int
        l.h3dgs_peer_open.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        l.h3dgs_peer_close.restype = C.c_int
        l.h3dgs_peer_close.argtypes = [C.c_void_p]
        l.h3dgs_peer_barrier.restype = C.c_int
        l.h3dgs_peer_barrier.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p]
        l.h3dgs_peer_barrier_status.restype = C.c_int
        l.h3dgs_peer_barrier_status.argtypes = [C.c_void_p, C.c_void_p]
    l.h3dgs_lod_cut.restype = C.c_int
    l.h3dgs_lod_cut.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_float] + [C.c_void_p] * 10
    if hasattr(l, "h3dgs_lod_budget"):           # LOD budget (an emulation build has it when it compiles lod_budget.cu)
        l.h3dgs_lod_budget_scratch_bytes.restype = C.c_size_t
        l.h3dgs_lod_budget_scratch_bytes.argtypes = [C.c_int32]
        l.h3dgs_lod_budget.restype = C.c_int
        l.h3dgs_lod_budget.argtypes = [C.c_int32] + [C.c_void_p] * 3 + [C.c_float, C.c_void_p, C.c_int32] + [C.c_void_p] * 5
        l.h3dgs_lod_budget_masked.restype = C.c_int
        l.h3dgs_lod_budget_masked.argtypes = [C.c_int32] + [C.c_void_p] * 4 + [C.c_float, C.c_void_p, C.c_int32] + \
            [C.c_void_p] * 5
    l.h3dgs_lod_cut_masked.restype = C.c_int
    l.h3dgs_lod_cut_masked.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_float] + [C.c_void_p] * 11
    if hasattr(l, "h3dgs_lod_cull_mask"):        # view cull (an emulation build has it when it compiles lod_cull.cu)
        l.h3dgs_lod_cull_mask.restype = C.c_int
        l.h3dgs_lod_cull_mask.argtypes = [C.c_int32] + [C.c_void_p] * 4 + [C.c_float] + [C.c_void_p] * 2 + \
            [C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
    if hasattr(l, "h3dgs_eval_metrics"):         # evaluation metrics (an emulation build has it when it compiles metrics.cu)
        l.h3dgs_eval_metrics.restype = C.c_int
        l.h3dgs_eval_metrics.argtypes = [C.c_int32, C.c_int32] + [C.c_void_p] * 4 + [C.c_int32] + [C.c_void_p] * 3 + \
            [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    if hasattr(l, "h3dgs_lpips_distance"):       # LPIPS (an emulation build has it when it compiles lpips.cu)
        l.h3dgs_lpips_weight_floats.restype = C.c_int64
        l.h3dgs_lpips_weight_floats.argtypes = []
        l.h3dgs_lpips_pack_weights.restype = C.c_int
        l.h3dgs_lpips_pack_weights.argtypes = [C.POINTER(C.c_void_p)] * 3 + [C.c_void_p]
        l.h3dgs_lpips_scratch_floats.restype = C.c_int
        l.h3dgs_lpips_scratch_floats.argtypes = [C.c_int32, C.c_int32] + [C.POINTER(C.c_int64)] * 3
        l.h3dgs_lpips_features.restype = C.c_int
        l.h3dgs_lpips_features.argtypes = [C.c_int32] * 3 + [C.c_void_p] * 3 + [C.c_int32] + [C.c_void_p] * 4
        l.h3dgs_lpips_distance.restype = C.c_int
        l.h3dgs_lpips_distance.argtypes = [C.c_int32] * 3 + [C.c_void_p] * 3 + [C.c_int32] + [C.c_void_p] * 6 + \
            [C.c_int32, C.c_void_p]
        l.h3dgs_lpips_conv.restype = C.c_int
        l.h3dgs_lpips_conv.argtypes = [C.c_int32] * 3 + [C.c_void_p] * 4
    if hasattr(l, "h3dgs_dist_knn3"):            # 3-NN distances (an emulation build has it when it compiles knn.cu)
        l.h3dgs_knn_scratch_bytes.restype = C.c_size_t
        l.h3dgs_knn_scratch_bytes.argtypes = [C.c_int64]
        l.h3dgs_dist_knn3.restype = C.c_int
        l.h3dgs_dist_knn3.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    if hasattr(l, "h3dgs_build_hierarchy"):      # hierarchy creator (an emulation build has it when it compiles hier_build.cu)
        l.h3dgs_build_hierarchy_scratch_bytes.restype = C.c_size_t
        l.h3dgs_build_hierarchy_scratch_bytes.argtypes = [C.c_int64]
        l.h3dgs_build_hierarchy.restype = C.c_int
        l.h3dgs_build_hierarchy.argtypes = [C.c_int32] + [C.c_void_p] * 15
    if hasattr(l, "h3dgs_merge_hierarchies"):    # hierarchy merger (an emulation build has it when it compiles hier_merge.cu)
        l.h3dgs_merge_hierarchies_scratch_bytes.restype = C.c_size_t
        l.h3dgs_merge_hierarchies_scratch_bytes.argtypes = [C.c_int32, C.c_int64, C.c_int64]
        l.h3dgs_merge_hierarchies.restype = C.c_int
        l.h3dgs_merge_hierarchies.argtypes = [C.c_int32] + [C.c_void_p] * 10 + [ALLOC_FN, C.c_void_p, C.c_void_p,
                                                                                 C.c_void_p, C.c_void_p]
    if hasattr(l, "h3dgs_l1_ssim_forward"):      # fused L1 + SSIM loss (an emulation build has it when it compiles loss.cu)
        l.h3dgs_l1_ssim_forward.restype = C.c_int
        l.h3dgs_l1_ssim_forward.argtypes = [C.c_int32] * 3 + [C.c_void_p] * 5
        l.h3dgs_l1_ssim_backward.restype = C.c_int
        l.h3dgs_l1_ssim_backward.argtypes = [C.c_int32] * 3 + [C.c_void_p] * 6
        l.h3dgs_post_loss_forward.restype = C.c_int
        l.h3dgs_post_loss_forward.argtypes = [C.c_int32] * 2 + [C.c_void_p] * 7
        l.h3dgs_post_loss_backward.restype = C.c_int
        l.h3dgs_post_loss_backward.argtypes = [C.c_int32] * 2 + [C.c_void_p] * 8
        l.h3dgs_post_step_status.restype = C.c_int
        l.h3dgs_post_step_status.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_int32, C.c_int32,
                                             C.c_void_p, C.c_void_p, C.c_void_p]
        l.h3dgs_post_loss_backward_exposure.restype = C.c_int
        l.h3dgs_post_loss_backward_exposure.argtypes = [C.c_int32] * 2 + [C.c_void_p] * 9
        l.h3dgs_single_step_status.restype = C.c_int
        l.h3dgs_single_step_status.argtypes = [C.c_void_p] * 3 + [C.c_double] * 3 + [C.c_void_p] * 5
        l.h3dgs_coarse_loss_forward.restype = C.c_int
        l.h3dgs_coarse_loss_forward.argtypes = [C.c_int32] * 2 + [C.c_void_p] * 6
        l.h3dgs_coarse_loss_backward.restype = C.c_int
        l.h3dgs_coarse_loss_backward.argtypes = [C.c_int32] * 2 + [C.c_void_p] * 7
        l.h3dgs_coarse_step_status.restype = C.c_int
        l.h3dgs_coarse_step_status.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
    if hasattr(l, "h3dgs_coarse_param_step"):    # train_coarse's parameter step (an emulation build has it when it compiles coarse_param.cu)
        l.h3dgs_coarse_param_step.restype = C.c_int
        l.h3dgs_coarse_param_step.argtypes = [C.POINTER(CoarseArgs), C.c_int32, C.c_void_p]
    if hasattr(l, "h3dgs_single_param_step"):    # train_single's parameter step (likewise)
        l.h3dgs_single_param_step.restype = C.c_int
        l.h3dgs_single_param_step.argtypes = [C.POINTER(SingleArgs), C.c_int32, C.c_void_p]
    if hasattr(l, "h3dgs_post_param_step"):      # train_post's parameter step (likewise)
        l.h3dgs_post_param_step.restype = C.c_int
        l.h3dgs_post_param_step.argtypes = [C.POINTER(PostArgs), C.c_int32, C.c_void_p]
    if hasattr(l, "h3dgs_densify"):              # densify_and_prune / reset_opacity (likewise)
        l.h3dgs_densify_scratch_bytes.restype = C.c_size_t
        l.h3dgs_densify_scratch_bytes.argtypes = [C.c_int32]
        l.h3dgs_densify.restype = C.c_int
        l.h3dgs_densify.argtypes = [C.POINTER(DensifyArgs), C.c_int32, C.c_void_p]
    l.h3dgs_invdepth_l1_grad.restype = C.c_int
    l.h3dgs_invdepth_l1_grad.argtypes = [C.c_int32] * 2 + [C.c_void_p] * 7
    l.h3dgs_densify_stats.restype = C.c_int
    l.h3dgs_densify_stats.argtypes = [C.c_int32] + [C.c_void_p] * 7
    if hasattr(l, "h3dgs_sparse_adam"):          # sparse Adam (absent from the emulation build)
        l.h3dgs_sparse_adam.restype = C.c_int
        l.h3dgs_sparse_adam.argtypes = [C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_double, C.c_double, C.c_double, C.c_double, C.c_int64, C.c_void_p]
    l.h3dgs_profile_read.argtypes = [C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int64)]
    l.h3dgs_stage_name.restype = C.c_char_p
    return l


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python hierarchical-3d-gaussians_b200/build.py` "
            "(nvcc, sm_90a). There is no CPU fallback for this path.")
    l = bind(C.CDLL(LIB_PATH))
    _lib = l
    return l


def check(rc):
    if rc < 0:
        raise RuntimeError(f"libh3dgs error {rc}: {lib().h3dgs_last_error().decode()}")
    return rc


def ptr(t):
    """a tensor as a pointer argument: NULL for None and for an empty tensor"""
    return None if (t is None or t.numel() == 0) else t.data_ptr()


def launch_count():
    return int(lib().h3dgs_launch_count())


STAGES = 18


def profile_enable(on=True):
    check(lib().h3dgs_profile_enable(1 if on else 0))


def profile_reset():
    check(lib().h3dgs_profile_reset())


def profile_read():
    """-> {stage_name: (total_ms, launches)} since the last reset (synchronises the recorded events)."""
    out = {}
    for st in range(STAGES):
        ms, n = C.c_double(0), C.c_int64(0)
        check(lib().h3dgs_profile_read(st, C.byref(ms), C.byref(n)))
        out[lib().h3dgs_stage_name(st).decode()] = (ms.value, n.value)
    return out

"""ctypes binding of the C ABI declared in include/gs_b200.h.

The CUDA library is the product; there is NO CPU fallback: importing this module
raises if ``libgs_b200.so`` has not been built (``python __graft_entry__.py`` or
``csrc/build.sh``).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgs_b200.so")

BUF_GEOM, BUF_BINNING, BUF_IMAGE, BUF_SCRATCH = 0, 1, 2, 3


class View(C.Structure):
    _fields_ = [("image_height", C.c_int32), ("image_width", C.c_int32), ("tanfovx", C.c_float),
                ("tanfovy", C.c_float), ("bg", C.c_void_p), ("scale_modifier", C.c_float),
                ("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p), ("sh_degree", C.c_int32),
                ("campos", C.c_void_p), ("prefiltered", C.c_int32), ("debug", C.c_int32)]


class State(C.Structure):
    _fields_ = [("geom", C.c_void_p), ("point_list", C.c_void_p), ("tile_keys", C.c_void_p),
                ("ranges", C.c_void_p), ("n_contrib", C.c_void_p), ("final_T", C.c_void_p),
                ("num_rendered", C.c_int64), ("num_gaussians", C.c_int32), ("tiles_x", C.c_int32),
                ("tiles_y", C.c_int32), ("owned", C.c_void_p * 4)]


ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_int32, C.c_size_t)

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: the sm_90a CUDA library has not been built. "
        "Run `python __graft_entry__.py` (or comfyui-3d-pack_b200/csrc/build.sh). There is no CPU fallback.")

lib = C.CDLL(LIB_PATH)

_P = C.c_void_p
lib.gs_b200_abi_version.restype = C.c_int32
lib.gs_b200_last_error.restype = C.c_char_p
lib.gs_b200_rasterize_forward.restype = C.c_int32
lib.gs_b200_rasterize_forward.argtypes = [C.POINTER(View), C.c_int32, C.c_int32] + [_P] * 7 + [_P] * 4 + \
    [ALLOC_FN, _P, C.POINTER(State), _P]
lib.gs_b200_rasterize_backward.restype = C.c_int32
lib.gs_b200_rasterize_backward.argtypes = [C.POINTER(View), C.c_int32, C.c_int32] + [_P] * 7 + \
    [_P, C.POINTER(State)] + [_P] * 3 + [_P] * 8 + [C.c_int32, ALLOC_FN, _P, _P]
lib.gs_b200_state_free.restype = C.c_int32
lib.gs_b200_state_free.argtypes = [C.POINTER(State), _P]
lib.gs_b200_debug_sorted_keys.restype = C.c_int32
lib.gs_b200_debug_sorted_keys.argtypes = [C.POINTER(State), _P, _P]
lib.gs_b200_sort_scratch_bytes.restype = C.c_size_t
lib.gs_b200_sort_scratch_bytes.argtypes = [C.c_int64]
lib.gs_b200_sort_pairs_u32.restype = C.c_int32
lib.gs_b200_sort_pairs_u32.argtypes = [_P, _P, _P, _P, C.c_int64, C.c_int32, C.c_int32, _P, C.POINTER(C.c_int32), _P]
lib.gs_b200_knn_mean_dist2.restype = C.c_int32
lib.gs_b200_knn_mean_dist2.argtypes = [_P, C.c_int32, _P, _P]
lib.gs_b200_step_host.restype = C.c_int32
lib.gs_b200_step_host.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, _P, C.c_int32, C.c_int32] + \
    [_P] * 5 + [_P, _P, _P, C.POINTER(C.c_int64), _P]

lib.gs_b200_step_device.restype = C.c_int32
lib.gs_b200_step_device.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, _P, _P, C.c_int32, C.c_int32] + \
    [_P] * 5 + [_P, _P, _P, C.POINTER(C.c_int64), _P]
VIEW_HOOK = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_int32, C.c_void_p)
lib.gs_b200_step_device_hook.restype = C.c_int32
lib.gs_b200_step_device_hook.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, _P, _P, C.c_int32, C.c_int32] + \
    [_P] * 5 + [_P, _P, _P, _P, VIEW_HOOK, _P, C.POINTER(C.c_int64), _P]
lib.gs_b200_image_loss.restype = C.c_int32
lib.gs_b200_image_loss.argtypes = [C.c_int32, C.c_int32, _P, _P, _P, C.c_float, C.c_float, C.c_float, _P, _P, _P]
lib.gs_b200_step_device_train.restype = C.c_int32
lib.gs_b200_step_device_train.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, _P, _P, C.c_int32, C.c_int32] + \
    [_P] * 5 + [_P, _P, C.c_float, C.c_float, C.c_float, _P, _P, _P, _P, _P, C.POINTER(C.c_int64), _P]
lib.gs_b200_render_views.restype = C.c_int32
lib.gs_b200_render_views.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, _P, _P, C.c_int32, C.c_int32] + \
    [_P] * 6 + [_P, _P, C.POINTER(C.c_int64), _P]
lib.gs_b200_step_host_dev_grads.restype = C.c_int32
lib.gs_b200_step_host_dev_grads.argtypes = lib.gs_b200_step_host.argtypes
lib.gs_b200_launch_count.restype = C.c_int64
lib.gs_b200_profile_enable.restype = None
lib.gs_b200_profile_enable.argtypes = [C.c_int32]
lib.gs_b200_profile_read.restype = C.c_int32
lib.gs_b200_profile_read.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_int32)]
# ---- mesh ops (include/dr_b200.h) -------------------------------------------------------------------------
_I = C.c_int32
lib.dr_b200_rasterize_scratch_bytes.restype = C.c_size_t
lib.dr_b200_rasterize_scratch_bytes.argtypes = [_I, _I, _I, _I]
lib.dr_b200_rasterize_fwd.restype = _I
lib.dr_b200_rasterize_fwd.argtypes = [_P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P]
lib.dr_b200_rasterize_bwd.restype = _I
lib.dr_b200_rasterize_bwd.argtypes = [_P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P]
lib.dr_b200_interpolate_fwd.restype = _I
lib.dr_b200_interpolate_fwd.argtypes = [_P, _I, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P]
lib.dr_b200_interpolate_bwd.restype = _I
lib.dr_b200_interpolate_bwd.argtypes = [_P, _I, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P]
lib.dr_b200_texture_fwd.restype = _I
lib.dr_b200_texture_fwd.argtypes = [_P, _I, _I, _I, _I, _P, _I, _I, _I, _I, _P, _P]
lib.dr_b200_texture_bwd.restype = _I
lib.dr_b200_texture_bwd.argtypes = [_P, _I, _I, _I, _I, _P, _I, _I, _I, _I, _P, _P, _P, _P]
lib.dr_b200_topology_scratch_bytes.restype = C.c_size_t
lib.dr_b200_topology_scratch_bytes.argtypes = [_I]
lib.dr_b200_edge_opposites.restype = _I
lib.dr_b200_edge_opposites.argtypes = [_P, _I, _I, _P, _P, _P]
lib.dr_b200_antialias_fwd.restype = _I
lib.dr_b200_antialias_fwd.argtypes = [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P]
lib.dr_b200_antialias_bwd.restype = _I
lib.dr_b200_antialias_bwd.argtypes = [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P]
lib.dr_b200_cr_scratch_bytes.restype = C.c_size_t
lib.dr_b200_cr_scratch_bytes.argtypes = [_I, _I, _I]
lib.dr_b200_cr_rasterize.restype = _I
lib.dr_b200_cr_rasterize.argtypes = [_P, _I, _P, _I, _P, _I, _I, C.c_float, _P, _P, _P, _P]
lib.dr_b200_cr_interpolate_fwd.restype = _I
lib.dr_b200_cr_interpolate_fwd.argtypes = [_P, _I, _I, _P, _I, _P, _P, _I, _I, _I, _P, _P]
lib.dr_b200_cr_interpolate_bwd.restype = _I
lib.dr_b200_cr_interpolate_bwd.argtypes = [_P, _I, _I, _P, _I, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P]
lib.dr_b200_uvbake_scratch_bytes.restype = C.c_size_t
lib.dr_b200_uvbake_scratch_bytes.argtypes = [_I, _I]
lib.dr_b200_uvbake_rasterize.restype = _I
lib.dr_b200_uvbake_rasterize.argtypes = [_P, _I, _P, _I, _P, _I, _I, _I, _P, _P]
lib.dr_b200_uvbake_interpolate.restype = _I
lib.dr_b200_uvbake_interpolate.argtypes = [_P, _I, _P, _I, _P, _P, _I, _I, _I, _P]
UVBAKE_EXPORTS = ["dr_b200_uvbake_scratch_bytes", "dr_b200_uvbake_rasterize", "dr_b200_uvbake_interpolate"]
CR_EXPORTS = ["dr_b200_cr_scratch_bytes", "dr_b200_cr_rasterize", "dr_b200_cr_interpolate_fwd", "dr_b200_cr_interpolate_bwd"]
DR_EXPORTS = ["dr_b200_rasterize_scratch_bytes", "dr_b200_rasterize_fwd", "dr_b200_rasterize_bwd",
              "dr_b200_interpolate_fwd", "dr_b200_interpolate_bwd", "dr_b200_texture_fwd", "dr_b200_texture_bwd",
              "dr_b200_topology_scratch_bytes", "dr_b200_edge_opposites", "dr_b200_antialias_fwd", "dr_b200_antialias_bwd"]

# ---- Instant-NGP path (include/ngp_b200.h) -----------------------------------------------------------------
_L = C.c_int64
_F = C.c_float
_D = C.c_double
lib.ngp_b200_grid_encode_fwd.restype = _I
lib.ngp_b200_grid_encode_fwd.argtypes = [_P, _L, _P, _P, _I, _F, _D, _I, _P, _P]
lib.ngp_b200_grid_encode_bwd.restype = _I
lib.ngp_b200_grid_encode_bwd.argtypes = [_P, _L, _P, _I, _F, _D, _I, _P, _P, _P]
lib.ngp_b200_grid_tv_grad.restype = _I
lib.ngp_b200_grid_tv_grad.argtypes = [_P, _L, _P, _P, _I, _F, _D, _I, _F, _P, _P]
lib.ngp_b200_march_scratch_bytes.restype = C.c_size_t
lib.ngp_b200_march_scratch_bytes.argtypes = [_L, _I]
lib.ngp_b200_march_count.restype = _I
lib.ngp_b200_march_count.argtypes = [_P, _P, _L, _P, _I, _P, _F, _F, _F, _P, _P, _P, _P, _P, _P]
lib.ngp_b200_march_write.restype = _I
lib.ngp_b200_march_write.argtypes = [_P, _P, _L, _I, _P, _F, _F, _F, _P, _P, _P, _P, _P, _P, _P]
lib.ngp_b200_ray_ranges.restype = _I
lib.ngp_b200_ray_ranges.argtypes = [_P, _L, _L, _P, _P]
lib.ngp_b200_weights_fwd.restype = _I
lib.ngp_b200_weights_fwd.argtypes = [_P, _P, _P, _P, _L, _P, _P, _P, _P]
lib.ngp_b200_weights_bwd.restype = _I
lib.ngp_b200_weights_bwd.argtypes = [_P, _P, _P, _P, _L, _P, _P, _P, _P, _P, _P, _P]
lib.ngp_b200_accumulate_fwd.restype = _I
lib.ngp_b200_accumulate_fwd.argtypes = [_P, _P, _I, _P, _L, _P, _P]
lib.ngp_b200_accumulate_bwd.restype = _I
lib.ngp_b200_accumulate_bwd.argtypes = [_P, _P, _I, _P, _L, _P, _P, _P, _P]
lib.ngp_b200_mlp2_supported.restype = _I
lib.ngp_b200_mlp2_supported.argtypes = [_I, _I, _I]
lib.ngp_b200_mlp2_fwd.restype = _I
lib.ngp_b200_mlp2_fwd.argtypes = [_P, _L, _I, _I, _I, _P, _P, _P, _P]
lib.ngp_b200_mlp2_bwd.restype = _I
lib.ngp_b200_mlp2_bwd.argtypes = [_P, _L, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P]
lib.ngp_b200_mcubes_scratch_bytes.restype = C.c_size_t
lib.ngp_b200_mcubes_scratch_bytes.argtypes = [_I, _I, _I]
lib.ngp_b200_mcubes_count.restype = _I
lib.ngp_b200_mcubes_count.argtypes = [_P, _I, _I, _I, _F, _P, _P, _P]
lib.ngp_b200_mcubes_write.restype = _I
lib.ngp_b200_mcubes_write.argtypes = [_P, _I, _I, _I, _F, C.POINTER(C.c_ulonglong), _P, _P, _P, _P]
_U4 = C.POINTER(C.c_ulonglong)
lib.ngp_b200_flexicubes_scratch_bytes.restype = C.c_size_t
lib.ngp_b200_flexicubes_scratch_bytes.argtypes = [_I, _I, _I]
lib.ngp_b200_flexicubes_count.restype = _I
lib.ngp_b200_flexicubes_count.argtypes = [_P, _I, _I, _I, _P, _P, _P]
lib.ngp_b200_flexicubes_write.restype = _I
lib.ngp_b200_flexicubes_write.argtypes = [_P, _P, _P, _L, _P, _L, _P, _L, _I, _I, _I, _D, _I, _U4, _P, _P, _P, _P, _P]
lib.ngp_b200_flexicubes_backward_workspace_bytes.restype = C.c_size_t
lib.ngp_b200_flexicubes_backward_workspace_bytes.argtypes = [_U4, _I]
lib.ngp_b200_flexicubes_backward.restype = _I
lib.ngp_b200_flexicubes_backward.argtypes = [_P, _P, _P, _L, _P, _L, _P, _L, _I, _I, _I, _D, _I, _U4] + [_P] * 11
lib.ngp_b200_flexicubes_write_attrs.restype = _I
lib.ngp_b200_flexicubes_write_attrs.argtypes = [_P, _P, _P, _L, _P, _L, _P, _L, _I, _I, _I, _D, _I, _U4, _P, _P, _P,
                                                _P, _L, _I, _P, _P, _P]
lib.ngp_b200_flexicubes_backward_attrs_workspace_bytes.restype = C.c_size_t
lib.ngp_b200_flexicubes_backward_attrs_workspace_bytes.argtypes = [_U4, _I, _I]
lib.ngp_b200_flexicubes_backward_attrs.restype = _I
lib.ngp_b200_flexicubes_backward_attrs.argtypes = [_P, _P, _P, _L, _P, _L, _P, _L, _I, _I, _I, _D, _I, _U4] + \
    [_P] * 8 + [_P, _L, _I] + [_P] * 6
lib.ngp_b200_dmc_scratch_bytes.restype = C.c_size_t
lib.ngp_b200_dmc_scratch_bytes.argtypes = [_I, _I, _I]
lib.ngp_b200_dmc_count.restype = _I
lib.ngp_b200_dmc_count.argtypes = [_P, _I, _I, _I, _F, _P, _P, _P]
lib.ngp_b200_dmc_write.restype = _I
lib.ngp_b200_dmc_write.argtypes = [_P, _P, _I, _I, _I, _F, _I, _I, _U4, _P, _P, _P, _P]
lib.ngp_b200_dmc_backward_workspace_bytes.restype = C.c_size_t
lib.ngp_b200_dmc_backward_workspace_bytes.argtypes = [_I, _I, _I]
lib.ngp_b200_dmc_backward.restype = _I
lib.ngp_b200_dmc_backward.argtypes = [_P, _P, _I, _I, _I, _F, _I, _U4, _P, _P, _P, _P, _P, _P]
NGP_EXPORTS = ["ngp_b200_mlp2_supported", "ngp_b200_mlp2_fwd", "ngp_b200_mlp2_bwd","ngp_b200_grid_encode_fwd", "ngp_b200_grid_encode_bwd", "ngp_b200_grid_tv_grad", "ngp_b200_march_scratch_bytes",
               "ngp_b200_march_count", "ngp_b200_march_write", "ngp_b200_ray_ranges", "ngp_b200_weights_fwd",
               "ngp_b200_weights_bwd", "ngp_b200_accumulate_fwd", "ngp_b200_accumulate_bwd",
               "ngp_b200_mcubes_scratch_bytes", "ngp_b200_mcubes_count", "ngp_b200_mcubes_write",
               "ngp_b200_flexicubes_scratch_bytes", "ngp_b200_flexicubes_count", "ngp_b200_flexicubes_write",
               "ngp_b200_flexicubes_backward_workspace_bytes", "ngp_b200_flexicubes_backward",
               "ngp_b200_flexicubes_write_attrs", "ngp_b200_flexicubes_backward_attrs_workspace_bytes",
               "ngp_b200_flexicubes_backward_attrs", "ngp_b200_dmc_scratch_bytes", "ngp_b200_dmc_count",
               "ngp_b200_dmc_write", "ngp_b200_dmc_backward_workspace_bytes", "ngp_b200_dmc_backward"]

lib.gs_b200_activate.restype = _I
lib.gs_b200_activate.argtypes = [_I, _P, _P, _P, _P, _P, _P, _P]
lib.gs_b200_adam_step.restype = _I
lib.gs_b200_adam_step.argtypes = [_I, _I, _P, _D, _D, _F, _I, _F, _P, _P, _P, _P, _P]
lib.gs_b200_densify_stats.restype = _I
lib.gs_b200_densify_stats.argtypes = [_I, _P, _P, _P, _P, _P, _P]
lib.gs_b200_densify_scratch_bytes.restype = C.c_size_t
lib.gs_b200_densify_scratch_bytes.argtypes = [_I]
lib.gs_b200_densify_plan.restype = _I
lib.gs_b200_densify_plan.argtypes = [_I, _P, _P, _P, _P, _F, _F, _F, _F, _P, _P, _P, _P]
lib.gs_b200_densify_apply.restype = _I
lib.gs_b200_densify_apply.argtypes = [_I, _I, _P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P]
TRAIN_EXPORTS = ["gs_b200_activate", "gs_b200_adam_step", "gs_b200_densify_stats", "gs_b200_densify_scratch_bytes",
                 "gs_b200_densify_plan", "gs_b200_densify_apply"]

SCATTER_SUM, SCATTER_MEAN, SCATTER_MAX = 0, 1, 2
SCATTER_F32, SCATTER_I32, SCATTER_I64 = 0, 1, 2
SCATTER_MAX_DIMS = 8
lib.gs_b200_scatter_index_range.restype = _I
lib.gs_b200_scatter_index_range.argtypes = [_I, _P, _I, _P, _P, _P, _P]
lib.gs_b200_scatter_scratch_bytes.restype = C.c_size_t
lib.gs_b200_scatter_scratch_bytes.argtypes = [_I, _I, _I, _P, _I, _P, _L]
lib.gs_b200_scatter_forward.restype = _I
lib.gs_b200_scatter_forward.argtypes = [_I, _I, _I, _P, _I, _L, _P, _P, _P, _P, _P, _P, _I, _P, _P, _P]
lib.gs_b200_scatter_backward.restype = _I
lib.gs_b200_scatter_backward.argtypes = [_I, _I, _P, _I, _L, _P, _P, _P, _P, _P, _P, _P, _P, _P]
SCATTER_EXPORTS = ["gs_b200_scatter_index_range", "gs_b200_scatter_scratch_bytes", "gs_b200_scatter_forward",
                   "gs_b200_scatter_backward"]

NSTAGES = 9
STAGE_NAMES = ["preprocess", "depth_sort", "scan", "emit", "tile_sort", "ranges", "composite_fwd",
               "composite_bwd", "preprocess_bwd"]

lib.gs_b200_set_tile_culling.restype = _I
lib.gs_b200_set_tile_culling.argtypes = [_I]
lib.gs_b200_get_tile_culling.restype = _I
lib.gs_b200_get_tile_culling.argtypes = []
GRAD_SINK = C.CFUNCTYPE(None, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p)
lib.gs_b200_set_grad_sink.restype = _I
lib.gs_b200_set_grad_sink.argtypes = [GRAD_SINK, _P, _I]
lib.gs_b200_composite_bwd_occupancy.restype = _I
lib.gs_b200_composite_bwd_occupancy.argtypes = [C.POINTER(C.c_int32), C.POINTER(C.c_int32)]

EXPORTS = ["gs_b200_set_grad_sink", "gs_b200_composite_bwd_occupancy", "gs_b200_image_loss", "gs_b200_step_device_train", "gs_b200_step_device_hook", "gs_b200_render_views", "gs_b200_set_tile_culling", "gs_b200_get_tile_culling", "gs_b200_step_device", "gs_b200_step_host_dev_grads", "gs_b200_launch_count", "gs_b200_profile_enable", "gs_b200_profile_read",
           "gs_b200_abi_version", "gs_b200_last_error", "gs_b200_rasterize_forward", "gs_b200_rasterize_backward",
           "gs_b200_state_free", "gs_b200_debug_sorted_keys", "gs_b200_sort_scratch_bytes",
           "gs_b200_sort_pairs_u32", "gs_b200_knn_mean_dist2", "gs_b200_step_host"] + SCATTER_EXPORTS + CR_EXPORTS + \
    UVBAKE_EXPORTS


def last_error() -> str:
    return lib.gs_b200_last_error().decode("utf-8", "replace")


def check(rc: int):
    if rc != 0:
        raise RuntimeError(f"gs_b200: {last_error()}")

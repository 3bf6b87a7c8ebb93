"""Loads libmapeval_b200.so (the C-ABI of include/mapeval_b200.h) and declares its prototypes.

There is no fallback: if the shared library is missing this module raises, and if no sm_90 device is present
`me_create` fails with ME_ERR_NO_DEVICE — the product path never routes through a CPU implementation.
"""
import ctypes as C
import os

from . import _abi as A

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmapeval_b200.so")

# every symbol include/mapeval_b200.h declares (tests check the .so exports exactly these)
SYMBOLS = (
    "me_abi_version", "me_create", "me_destroy", "me_last_error", "me_set_stream", "me_set_shard", "me_synchronize",
    "me_set_cloud", "me_set_cloud_device", "me_transform", "me_voxel_downsample", "me_get_cloud", "me_icp_point_to_point", "me_icp",
    "me_set_normals", "me_estimate_normals", "me_get_normals", "me_build_grid", "me_eval_nn_accum", "me_nn_finalize",
    "me_eval_nn", "me_get_nn", "me_eval_mme_accum", "me_mme_finalize", "me_eval_mme", "me_get_entropies",
    "me_eval_awd", "me_awd_from_rows", "me_free",
    "me_eval_w2", "me_w2_from_rows", "me_w2_begin", "me_w2_w_table", "me_w2_finish_accum_device", "me_w2_block", "me_w2_fetch", "me_get_stage_times", "me_launch_count",
    "me_accum_reset", "me_eval_nn_accum_device", "me_eval_mme_accum_device", "me_accum_block", "me_accum_fetch",
    "me_set_layout", "me_layout_active", "me_voxel_begin", "me_voxel_w_table", "me_voxel_finish_accum_device", "me_accum_fetch_awd",
    "me_plan_slab_cut", "me_plan_lattice", "me_kernel_trace",
    "me_icp_begin", "me_icp_normals_slice", "me_icp_block", "me_icp_step", "me_icp_end", "me_icp_update",
    "me_copy_cloud", "me_add_gaussian_noise", "me_add_non_uniform_density", "me_add_sparse_outliers", "me_add_local_deformation",
    "me_global_registration", "me_get_features", "me_get_correspondences",
    "me_nn_curve_accum_device", "me_nn_curve_finalize", "me_nn_curve",
    "me_nn_quantile_begin", "me_nn_quantile_block", "me_nn_quantile_step", "me_nn_quantile_end", "me_nn_quantiles",
    "me_quantile_finalize",
    "me_nn_region_begin", "me_nn_region_block", "me_nn_region_end", "me_nn_regions", "me_region_finalize",
    "me_drift_begin", "me_drift_block", "me_drift_step", "me_drift_end", "me_drift",
    "me_nn_surface_begin", "me_nn_surface_normals_slice", "me_nn_surface_block", "me_nn_surface_end", "me_nn_surface",
    "me_surface_finalize",
    "me_consistency_begin", "me_consistency_block", "me_consistency_end", "me_consistency", "me_consistency_finalize",
    "me_get_consistency_points",
    "me_mom_begin", "me_mom_block", "me_mom_step", "me_mom_end", "me_mom", "me_mom_axes", "me_get_mom_points",
    "me_mom_region_begin", "me_mom_region_block", "me_mom_region_end", "me_mom_regions",
)

_lib = None


class LibraryMissing(RuntimeError):
    pass


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LibraryMissing(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` or "
            f"`make -C cloud_map_evaluation_b200/csrc`. There is no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    ctx = C.c_void_p
    dp = C.POINTER(C.c_double)
    L.me_abi_version.restype = C.c_int
    L.me_create.argtypes = [C.POINTER(A.me_options), C.POINTER(ctx)]
    L.me_destroy.argtypes = [ctx]
    L.me_destroy.restype = None
    L.me_last_error.argtypes = [ctx]
    L.me_last_error.restype = C.c_char_p
    L.me_set_stream.argtypes = [ctx, C.c_void_p]
    L.me_set_shard.argtypes = [ctx, C.c_int32, C.c_int32]
    L.me_synchronize.argtypes = [ctx]
    L.me_set_cloud.argtypes = [ctx, C.c_int, C.c_void_p, C.c_int64]
    L.me_set_cloud_device.argtypes = [ctx, C.c_int, C.c_void_p, C.c_int64]
    L.me_transform.argtypes = [ctx, C.c_int, dp]
    L.me_awd_from_rows.argtypes = [ctx, dp, C.c_int64, C.c_double, C.c_int32, dp, C.POINTER(A.me_awd_result)]
    L.me_icp_point_to_point.argtypes = [ctx, C.c_double, C.c_int32, C.c_double, C.c_double, dp, C.POINTER(A.me_icp_result)]
    L.me_icp.argtypes = [ctx, C.c_int32, C.c_double, C.c_int32, C.c_double, C.c_double, dp, C.POINTER(A.me_icp_result)]
    L.me_icp_begin.argtypes = [ctx, C.c_int32, C.c_double, C.c_int32, C.c_double, C.c_double, dp]
    L.me_icp_normals_slice.argtypes = [ctx, C.c_int, C.POINTER(dp), C.POINTER(C.c_int64), C.POINTER(C.c_int32)]
    L.me_icp_block.argtypes = [ctx, C.POINTER(dp), C.POINTER(C.c_int32)]
    L.me_icp_step.argtypes = [ctx, C.POINTER(C.c_int32)]
    L.me_icp_end.argtypes = [ctx, C.POINTER(A.me_icp_result)]
    L.me_icp_update.argtypes = [C.c_int32, dp, dp, dp]
    L.me_set_normals.argtypes = [ctx, C.c_int, dp, C.c_int64]
    L.me_estimate_normals.argtypes = [ctx, C.c_int, C.c_int32]
    L.me_get_normals.argtypes = [ctx, C.c_int, dp]
    L.me_voxel_downsample.argtypes = [ctx, C.c_int, C.c_double, C.POINTER(C.c_int64)]
    L.me_get_cloud.argtypes = [ctx, C.c_int, dp, C.c_int64, C.POINTER(C.c_int64)]
    L.me_copy_cloud.argtypes = [ctx, C.c_int, C.c_int]
    L.me_add_gaussian_noise.argtypes = [ctx, C.c_int, C.c_double, C.c_uint64]
    L.me_add_non_uniform_density.argtypes = [ctx, C.c_int, C.c_double, C.c_double, C.c_double, C.c_uint64, C.POINTER(C.c_int64)]
    L.me_add_sparse_outliers.argtypes = [ctx, C.c_int, C.c_double, C.c_double, C.c_uint64, C.POINTER(C.c_int64)]
    L.me_add_local_deformation.argtypes = [ctx, C.c_int, C.c_double, C.c_double, dp]
    L.me_global_registration.argtypes = [ctx, C.POINTER(A.me_global_reg_params), C.POINTER(A.me_global_reg_result)]
    L.me_get_features.argtypes = [ctx, C.c_int, dp, dp, C.POINTER(C.c_float), C.c_int64, C.POINTER(C.c_int64)]
    L.me_get_correspondences.argtypes = [ctx, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]
    L.me_build_grid.argtypes = [ctx, C.c_int]
    L.me_eval_nn_accum.argtypes = [ctx, C.POINTER(A.me_nn_params), C.POINTER(A.me_nn_accum), C.POINTER(A.me_nn_accum)]
    L.me_nn_finalize.argtypes = [C.POINTER(A.me_nn_params), C.POINTER(A.me_nn_accum), C.POINTER(A.me_nn_accum),
                                 C.c_int64, C.c_int64, C.POINTER(A.me_nn_result)]
    L.me_eval_nn.argtypes = [ctx, C.POINTER(A.me_nn_params), C.POINTER(A.me_nn_result)]
    L.me_get_nn.argtypes = [ctx, C.c_int, C.c_void_p, C.c_void_p]
    L.me_eval_mme_accum.argtypes = [ctx, C.c_int, C.c_double, C.c_int32, C.POINTER(A.me_mme_accum)]
    L.me_mme_finalize.argtypes = [C.POINTER(A.me_mme_accum), C.c_int64, C.POINTER(A.me_mme_result)]
    L.me_eval_mme.argtypes = [ctx, C.c_int, C.c_double, C.c_int32, C.POINTER(A.me_mme_result), C.c_void_p]
    L.me_get_entropies.argtypes = [ctx, C.c_int, C.c_void_p]
    L.me_eval_awd.argtypes = [ctx, C.c_double, C.c_int32, C.c_int32, C.POINTER(A.me_awd_result),
                              C.POINTER(C.c_int64), C.POINTER(dp)]
    L.me_accum_reset.argtypes = [ctx]
    L.me_eval_nn_accum_device.argtypes = [ctx, C.POINTER(A.me_nn_params)]
    L.me_eval_mme_accum_device.argtypes = [ctx, C.c_int, C.c_double, C.c_int32]
    L.me_accum_block.argtypes = [ctx, C.POINTER(dp), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.me_accum_fetch.argtypes = [ctx, C.POINTER(A.me_nn_accum), C.POINTER(A.me_nn_accum), C.POINTER(A.me_mme_accum),
                                 C.POINTER(A.me_mme_accum)]
    L.me_set_layout.argtypes = [ctx, C.c_int32]
    L.me_layout_active.argtypes = [ctx, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.me_plan_lattice.argtypes = [dp, dp, C.c_int64, dp, dp, C.c_int64, C.c_double, C.c_double, C.c_int64, C.c_int32,
                                  C.POINTER(A.me_lattice_plan)]
    L.me_plan_slab_cut.argtypes = [C.POINTER(C.c_uint64), C.c_int32, C.POINTER(C.c_uint64), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                   C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_double)]
    L.me_voxel_begin.argtypes = [ctx, C.c_double, C.c_int32]
    L.me_voxel_w_table.argtypes = [ctx, C.POINTER(dp), C.POINTER(C.c_int64)]
    L.me_voxel_finish_accum_device.argtypes = [ctx, C.c_int32]
    L.me_accum_fetch_awd.argtypes = [ctx, C.POINTER(A.me_awd_result)]
    L.me_eval_w2.argtypes = [ctx, C.c_double, C.c_int32, C.c_int32, C.POINTER(A.me_w2_result), C.POINTER(C.c_int64), C.POINTER(dp)]
    L.me_w2_from_rows.argtypes = [ctx, dp, C.c_int64, C.c_double, C.c_int32, dp, C.POINTER(A.me_w2_result)]
    L.me_w2_begin.argtypes = [ctx, C.c_double, C.c_int32]
    L.me_w2_w_table.argtypes = [ctx, C.POINTER(dp), C.POINTER(C.c_int64)]
    L.me_w2_finish_accum_device.argtypes = [ctx, C.c_int32]
    L.me_w2_block.argtypes = [ctx, C.POINTER(dp), C.POINTER(C.c_int32)]
    L.me_w2_fetch.argtypes = [ctx, C.POINTER(A.me_w2_result)]
    L.me_free.argtypes = [C.c_void_p]
    L.me_free.restype = None
    L.me_get_stage_times.argtypes = [ctx, dp]
    L.me_launch_count.argtypes = [ctx]
    L.me_launch_count.restype = C.c_int64
    L.me_nn_curve_accum_device.argtypes = [ctx, dp, C.c_int32, C.POINTER(dp), C.POINTER(C.c_int32)]
    L.me_nn_curve_finalize.argtypes = [C.POINTER(A.me_nn_params), C.POINTER(A.me_nn_accum), C.POINTER(A.me_nn_accum), dp, dp,
                                       C.c_int32, C.c_int64, C.c_int64, C.POINTER(A.me_curve_row)]
    L.me_nn_curve.argtypes = [ctx, dp, C.c_int32, C.POINTER(A.me_curve_row)]
    L.me_nn_quantile_begin.argtypes = [ctx, C.c_int32, dp, C.c_int32]
    L.me_nn_quantile_block.argtypes = [ctx, C.POINTER(dp), C.POINTER(C.c_int32)]
    L.me_nn_quantile_step.argtypes = [ctx, C.POINTER(C.c_int32)]
    L.me_nn_quantile_end.argtypes = [ctx, C.POINTER(A.me_quantile_result)]
    L.me_nn_quantiles.argtypes = [ctx, C.c_int32, dp, C.c_int32, C.POINTER(A.me_quantile_result)]
    L.me_quantile_finalize.argtypes = [C.c_int64, dp, C.c_int32, dp, dp]
    i64p = C.POINTER(C.c_int64)
    L.me_nn_region_begin.argtypes = [ctx, C.c_double, i64p]
    L.me_nn_region_block.argtypes = [ctx, C.POINTER(dp), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.me_nn_region_end.argtypes = [ctx, C.POINTER(A.me_region_row), C.c_int64]
    L.me_nn_regions.argtypes = [ctx, C.c_double, C.POINTER(C.POINTER(A.me_region_row)), i64p]
    L.me_region_finalize.argtypes = [C.c_int64, C.c_double, i64p, i64p, i64p, dp, C.POINTER(A.me_region_row)]
    L.me_drift_begin.argtypes = [ctx, C.c_double, C.c_double, C.c_int32, C.c_double, C.c_double, i64p]
    L.me_drift_block.argtypes = [ctx, C.POINTER(dp), C.POINTER(C.c_int32)]
    L.me_drift_step.argtypes = [ctx, C.POINTER(C.c_int32)]
    L.me_drift_end.argtypes = [ctx, C.POINTER(A.me_drift_row), C.c_int64]
    L.me_drift.argtypes = [ctx, C.c_double, C.c_double, C.c_int32, C.c_double, C.c_double, C.POINTER(C.POINTER(A.me_drift_row)), i64p]
    L.me_nn_surface_begin.argtypes = [ctx, C.c_int32]
    L.me_nn_surface_normals_slice.argtypes = [ctx, C.c_int, C.POINTER(dp), i64p, C.POINTER(C.c_int32)]
    L.me_nn_surface_block.argtypes = [ctx, C.POINTER(dp), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.me_nn_surface_end.argtypes = [ctx, C.POINTER(A.me_surface_result)]
    L.me_nn_surface.argtypes = [ctx, C.c_int32, C.POINTER(A.me_surface_result)]
    L.me_surface_finalize.argtypes = [C.POINTER(A.me_nn_params), dp, C.c_int64, C.c_int64, C.POINTER(A.me_surface_result)]
    L.me_consistency_begin.argtypes = [ctx, C.c_int, C.c_double, C.c_int32, C.c_double, i64p]
    L.me_consistency_block.argtypes = [ctx, C.POINTER(dp), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.me_consistency_end.argtypes = [ctx, C.c_void_p, C.c_int64, C.POINTER(A.me_consistency_result)]
    L.me_consistency.argtypes = [ctx, C.c_int, C.c_double, C.c_int32, C.c_double, C.POINTER(C.c_void_p), i64p,
                                 C.POINTER(A.me_consistency_result)]
    L.me_consistency_finalize.argtypes = [C.c_int64, C.c_double, i64p, i64p, C.c_int64, dp, C.c_void_p,
                                          C.POINTER(A.me_consistency_result)]
    L.me_get_consistency_points.argtypes = [ctx, C.c_int, C.c_void_p, C.c_void_p]
    L.me_mom_begin.argtypes = [ctx, C.c_int, C.c_double, C.c_int32, C.POINTER(A.me_mom_params)]
    L.me_mom_block.argtypes = [ctx, C.POINTER(dp), C.POINTER(C.c_int32)]
    L.me_mom_step.argtypes = [ctx, C.POINTER(C.c_int32)]
    L.me_mom_end.argtypes = [ctx, C.POINTER(A.me_mom_result)]
    L.me_mom.argtypes = [ctx, C.c_int, C.c_double, C.c_int32, C.POINTER(A.me_mom_params), C.POINTER(A.me_mom_result)]
    L.me_mom_axes.argtypes = [i64p, C.c_int32, C.c_double, dp, C.POINTER(C.c_int32)]
    L.me_get_mom_points.argtypes = [ctx, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.me_mom_region_begin.argtypes = [ctx, C.c_double, C.c_int64, i64p]
    L.me_mom_region_block.argtypes = [ctx, C.POINTER(dp), i64p]
    L.me_mom_region_end.argtypes = [ctx, C.c_void_p, C.c_int64]
    L.me_mom_regions.argtypes = [ctx, C.c_double, C.c_int64, C.POINTER(C.c_void_p), i64p]
    L.me_kernel_trace.argtypes = [ctx, C.POINTER(C.c_uint64), C.POINTER(C.c_int32), C.c_int32]
    if L.me_abi_version() != A.ME_ABI_VERSION:
        raise RuntimeError("libmapeval_b200.so ABI version mismatch")
    _lib = L
    return L

"""ctypes mirror of include/mapeval_b200.h (struct layouts and constants only — no library is loaded here)."""
import ctypes as C

ME_ABI_VERSION = 2

ME_OK = 0
ME_ERR_INVALID = -1
ME_ERR_NO_DEVICE = -2
ME_ERR_CUDA = -3
ME_ERR_NOMEM = -4
ME_ERR_EMPTY = -5
ME_ERR_RANGE = -6

ME_CLOUD_EST = 0
ME_CLOUD_GT = 1

ME_CUTOFF_SQDIST_LE_R = 0
ME_CUTOFF_DIST_LT_R = 1

ME_PAIRING_AS_WRITTEN = 0
ME_PAIRING_GEOMETRIC = 1

class me_lattice_plan(C.Structure):
    _fields_ = [("v", C.c_double), ("h", C.c_double), ("m", C.c_int32), ("sparse", C.c_int32), ("nvox", C.c_int32 * 3),
                ("dims", C.c_int32 * 3), ("ncells", C.c_int64)]


ME_LAYOUT_REPLICATED = 0
ME_LAYOUT_SLAB = 1
ME_ICP_POINT_TO_POINT = 0
ME_ICP_POINT_TO_PLANE = 1
ME_ICP_GENERALIZED = 2
ME_ICP_BLOCK_P2P = 17
ME_ICP_BLOCK_NE = 29

# enum me_kernel_bit: bit (1 << value) of the me_kernel_trace mask
ME_KBIT_NN_ROWS_DENSE = 0
ME_KBIT_NN_ROWS_SPARSE = 1
ME_KBIT_NN_FLAT = 2
ME_KBIT_NN_TILE = 3
ME_KBIT_NN_FAR = 4
ME_KBIT_NN_FAR_COARSE = 5
ME_KBIT_NN_BRUTE = 6
ME_KBIT_MME_FLAT1_DENSE = 7
ME_KBIT_MME_FLAT2_DENSE = 8
ME_KBIT_MME_FLAT3_DENSE = 9
ME_KBIT_MME_FLAT1_SPARSE = 10
ME_KBIT_MME_FLAT2_SPARSE = 11
ME_KBIT_MME_FLAT3_SPARSE = 12
ME_KBIT_MME_ROWS1 = 13
ME_KBIT_MME_ROWS2 = 14
ME_KBIT_MME_ROWS3 = 15
ME_KBIT_MME_PLANE = 16
ME_KBIT_MME_GENERIC = 17
ME_KBIT_MME_SOLO = 18
ME_KBIT_SCS_R5 = 19
ME_KBIT_SCS_RT_CACHED = 20
ME_KBIT_SCS_RT_UNCACHED = 21
ME_KBIT_COUNT = 22
# name -> value of every kernel bit (ME_KBIT_COUNT excluded)
KERNEL_BITS = {k: v for k, v in dict(globals()).items() if k.startswith("ME_KBIT_") and k != "ME_KBIT_COUNT"}


def kernel_bit_names(mask):
    """the ME_KBIT_* names set in a me_kernel_trace mask"""
    return {k for k, v in KERNEL_BITS.items() if mask >> v & 1}


# enum me_trace_event: data events in the trace mask, above the sweep bits
ME_TEV_BOX_REMEMBERED = 28
ME_TEV_BOX_MISSED = 29
ME_TEV_KNN_COARSE = 30
ME_TEV_MME_FP64_FINISH = 31
TRACE_EVENTS = {k: v for k, v in dict(globals()).items() if k.startswith("ME_TEV_")}


def trace_event_names(mask):
    """the ME_TEV_* names set in a me_kernel_trace mask"""
    return {k for k, v in TRACE_EVENTS.items() if mask >> v & 1}


ME_N_STAGE_TIMES = 9
STAGE_NAMES = ("grid_est", "grid_gt", "nn_est_to_gt", "nn_gt_to_est", "mme_est", "mme_gt",
               "voxel_moments", "awd", "scs")


class me_options(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("device", C.c_int32), ("rank", C.c_int32), ("world", C.c_int32),
                ("stream", C.c_void_p), ("nn_cell_size", C.c_double), ("max_grid_cells", C.c_int64),
                ("vmd_voxel_size", C.c_double)]


class me_nn_params(C.Structure):
    _fields_ = [("tau", C.c_double * 5), ("icp_max_distance", C.c_double), ("cutoff_mode", C.c_int32),
                ("pairing", C.c_int32), ("want_full_cd", C.c_int32), ("directions", C.c_int32)]


ME_MAX_WORLD = 64
ME_NN_ACCUM_I64 = 9
ME_NN_ACCUM_F64 = 13 + 3 * ME_MAX_WORLD


class me_nn_accum(C.Structure):
    _fields_ = [("n_query", C.c_int64), ("n_corr", C.c_int64), ("n_inlier", C.c_int64 * 5), ("n_ub", C.c_int64),
                ("n_far", C.c_int64),
                ("sum_d", C.c_double * 5), ("sum_d2", C.c_double * 5), ("sum_d_all", C.c_double),
                ("sum_d2_all", C.c_double), ("sum_nn_dist", C.c_double),
                ("rank_n", C.c_double * ME_MAX_WORLD), ("rank_mean", C.c_double * ME_MAX_WORLD),
                ("rank_m2", C.c_double * ME_MAX_WORLD)]


class me_dir_result(C.Structure):
    _fields_ = [("n_source", C.c_int64), ("n_corr", C.c_int64), ("n_inlier", C.c_int64 * 5), ("n_ub", C.c_int64),
                ("mean", C.c_double * 5), ("rmse", C.c_double * 5), ("fitness", C.c_double * 5),
                ("sigma", C.c_double * 5), ("sum_nn_dist", C.c_double)]


class me_nn_result(C.Structure):
    _fields_ = [("est_to_gt", me_dir_result), ("gt_to_est", me_dir_result), ("cd", C.c_double * 5),
                ("f1", C.c_double * 5), ("iou", C.c_double * 5), ("full_cd", C.c_double)]


# accuracy curve (me_nn_curve*)
ME_CURVE_MAX_LEVELS = 1024


class me_curve_dir(C.Structure):
    _fields_ = [("n_inlier", C.c_int64), ("mean", C.c_double), ("rmse", C.c_double), ("fitness", C.c_double),
                ("sigma", C.c_double)]


class me_curve_row(C.Structure):
    _fields_ = [("tau", C.c_double), ("est_to_gt", me_curve_dir), ("gt_to_est", me_curve_dir), ("cd", C.c_double),
                ("f1", C.c_double), ("iou", C.c_double)]


def curve_block_len(n_tau):
    """values of a curve block: per direction count, sum d and sum d^2 of the bins 0..K, then n_ub"""
    return 2 * (3 * (int(n_tau) + 1) + 1)


# exact distance quantiles (me_nn_quantile*)
ME_QUANTILE_MAX_PROBS = 64
ME_DIST_KEPT = 0
ME_DIST_NN = 1
# the SUM-reducible block of a selection pass: [direction][slot][digit] counts as fp64, 2 x (2 * 64 + 2) x 256
ME_QUANTILE_BLOCK = 2 * (2 * ME_QUANTILE_MAX_PROBS + 2) * 256


class me_quantile_dir(C.Structure):
    _fields_ = [("n", C.c_int64), ("min", C.c_double), ("max", C.c_double), ("rank", C.c_int64 * ME_QUANTILE_MAX_PROBS),
                ("lo", C.c_double * ME_QUANTILE_MAX_PROBS), ("hi", C.c_double * ME_QUANTILE_MAX_PROBS),
                ("value", C.c_double * ME_QUANTILE_MAX_PROBS)]


class me_quantile_result(C.Structure):
    _fields_ = [("population", C.c_int32), ("n_probs", C.c_int32), ("p", C.c_double * ME_QUANTILE_MAX_PROBS),
                ("est_to_gt", me_quantile_dir), ("gt_to_est", me_quantile_dir), ("hausdorff", C.c_double)]


# AC / COM / CD / F1 / IoU per region (me_nn_region*)
ME_REGION_MAX_REGIONS = 1 << 21
ME_REGION_SUM_FIELDS = 18      # per region and direction: n_query n_corr n_inlier[5] sum_d[5] sum_d2[5] sum_nn_dist
ME_REGION_MAX_FIELDS = 2       # per region and direction: max_d max_nn


class me_region_dir(C.Structure):
    _fields_ = [("n_query", C.c_int64), ("n_corr", C.c_int64), ("n_inlier", C.c_int64 * 5), ("sum_d", C.c_double * 5),
                ("sum_d2", C.c_double * 5), ("sum_nn_dist", C.c_double), ("max_d", C.c_double), ("max_nn", C.c_double),
                ("mean", C.c_double * 5), ("rmse", C.c_double * 5), ("fitness", C.c_double * 5), ("mean_nn", C.c_double)]


class me_region_row(C.Structure):
    _fields_ = [("index", C.c_int64 * 3), ("min", C.c_double * 3), ("max", C.c_double * 3), ("n_est", C.c_int64),
                ("n_gt", C.c_int64), ("est_to_gt", me_region_dir), ("gt_to_est", me_region_dir), ("cd", C.c_double * 5),
                ("f1", C.c_double * 5), ("iou", C.c_double * 5)]


# point-to-plane metrics and normal consistency (me_nn_surface*)
# the SUM part: both directions laid out as the NN section of the accumulator block, then per direction n_no_normal
# n_no_normal_nn n_nc sum_c; the MAX part: per direction max_e max_e_nn
ME_SURFACE_BLOCK_SUM = 2 * (ME_NN_ACCUM_I64 + ME_NN_ACCUM_F64) + 8
ME_SURFACE_BLOCK_MAX = 4


class me_surface_dir(C.Structure):
    _fields_ = [("n_no_normal", C.c_int64), ("n_no_normal_nn", C.c_int64), ("n_nc", C.c_int64),
                ("normal_consistency", C.c_double), ("max_e", C.c_double), ("max_e_nn", C.c_double)]


class me_surface_result(C.Structure):
    _fields_ = [("plane", me_nn_result), ("est_to_gt", me_surface_dir), ("gt_to_est", me_surface_dir),
                ("normal_consistency", C.c_double)]


# drift per region (me_drift*)
ME_DRIFT_CONVERGED = 0
ME_DRIFT_ITERATION_LIMIT = 1
ME_DRIFT_TOO_FEW = 2


class me_drift_row(C.Structure):
    _fields_ = [("index", C.c_int64 * 3), ("min", C.c_double * 3), ("max", C.c_double * 3), ("n_est", C.c_int64),
                ("n_corr_before", C.c_int64), ("fitness_before", C.c_double), ("rmse_before", C.c_double),
                ("n_corr", C.c_int64), ("fitness", C.c_double), ("rmse", C.c_double), ("T", C.c_double * 16),
                ("centroid", C.c_double * 3), ("shift", C.c_double * 3), ("shift_norm", C.c_double), ("angle", C.c_double),
                ("iterations", C.c_int32), ("status", C.c_int32)]


# local map consistency: mean plane variance beside MME, whole map and per region (me_consistency*)
ME_CONSISTENCY_SUM_FIELDS = 6   # per region: n_query n_valid n_pv sum_entropy sum_pv sum_sqrt_pv
ME_CONSISTENCY_MAX_FIELDS = 1   # per region: max_pv
ME_CONSISTENCY_WALK = 0         # me_consistency_kernel
CONSISTENCY_KERNEL_NAMES = {ME_CONSISTENCY_WALK: "WALK"}


class me_consistency_row(C.Structure):
    _fields_ = [("index", C.c_int64 * 3), ("min", C.c_double * 3), ("max", C.c_double * 3), ("n_points", C.c_int64),
                ("n_query", C.c_int64), ("n_valid", C.c_int64), ("n_pv", C.c_int64), ("sum_entropy", C.c_double),
                ("sum_pv", C.c_double), ("sum_sqrt_pv", C.c_double), ("mme", C.c_double), ("mpv", C.c_double),
                ("mean_plane_std", C.c_double), ("max_pv", C.c_double)]


class me_consistency_result(C.Structure):
    _fields_ = [("radius", C.c_double), ("region_size", C.c_double), ("min_neighbors", C.c_int32), ("kernel", C.c_int32),
                ("rings", C.c_int32), ("solo", C.c_int32), ("n_regions", C.c_int64), ("n_points", C.c_int64),
                ("n_query", C.c_int64), ("n_valid", C.c_int64), ("n_pv", C.c_int64), ("sum_entropy", C.c_double),
                ("sum_pv", C.c_double), ("sum_sqrt_pv", C.c_double), ("mme", C.c_double), ("mpv", C.c_double),
                ("mean_plane_std", C.c_double), ("max_pv", C.c_double)]


# the mutually orthogonal metric without a ground truth (me_mom*)
ME_MOM_CELLS_PER_EDGE = 16
ME_MOM_BINS = 6 * ME_MOM_CELLS_PER_EDGE * ME_MOM_CELLS_PER_EDGE
ME_MOM_BLOCK = 6 + 3 * 4 * 256
ME_MOM_OK, ME_MOM_NO_PLANAR, ME_MOM_NO_SECOND_AXIS, ME_MOM_SMALL_FAMILY = 0, 1, 2, 3
MOM_STATUS_NAMES = {ME_MOM_OK: "OK", ME_MOM_NO_PLANAR: "NO_PLANAR", ME_MOM_NO_SECOND_AXIS: "NO_SECOND_AXIS",
                    ME_MOM_SMALL_FAMILY: "SMALL_FAMILY"}


class me_mom_params(C.Structure):
    _fields_ = [("angle_deg", C.c_double), ("planarity", C.c_double), ("min_family", C.c_int64)]


class me_mom_result(C.Structure):
    _fields_ = [("radius", C.c_double), ("angle_deg", C.c_double), ("planarity", C.c_double), ("min_family", C.c_int64),
                ("min_neighbors", C.c_int32), ("kernel", C.c_int32), ("rings", C.c_int32), ("solo", C.c_int32),
                ("n_points", C.c_int64), ("n_query", C.c_int64), ("n_pv", C.c_int64), ("n_planar", C.c_int64),
                ("axis", C.c_double * 9), ("n", C.c_int64 * 3), ("mean", C.c_double * 3), ("median", C.c_double * 3),
                ("mom", C.c_double), ("status", C.c_int32), ("reserved", C.c_int32)]


class me_mom_region_row(C.Structure):
    _fields_ = [("index", C.c_int64 * 3), ("n_points", C.c_int64), ("n_planar", C.c_int64), ("n", C.c_int64 * 3),
                ("mean", C.c_double * 3), ("median", C.c_double * 3), ("mom", C.c_double), ("status", C.c_int32),
                ("reserved", C.c_int32)]


class me_mme_accum(C.Structure):
    _fields_ = [("n_query", C.c_int64), ("n_valid", C.c_int64), ("sum_entropy", C.c_double),
                ("min_entropy", C.c_double), ("max_entropy", C.c_double)]


class me_mme_result(C.Structure):
    _fields_ = [("mme", C.c_double), ("n_valid", C.c_int64), ("n_total", C.c_int64),
                ("min_abs_entropy", C.c_double), ("max_abs_entropy", C.c_double)]


class me_awd_result(C.Structure):
    _fields_ = [("awd", C.c_double), ("scs", C.c_double), ("n_pairs", C.c_int64), ("n_scs", C.c_int64),
                ("n_voxels_est", C.c_int64), ("n_voxels_gt", C.c_int64), ("n_active", C.c_int64),
                ("n_old", C.c_int64), ("n_new", C.c_int64)]


ME_W2_ROW_COLS = 26
ME_W2_BLOCK = 8
# the columns of a me_eval_w2 row (sigma as xx xy xz yy yz zz)
W2_ROW_COLUMNS = ("vmin_x", "vmin_y", "vmin_z", "n_gt", "n_est", "mu_est_x", "mu_est_y", "mu_est_z", "mu_gt_x", "mu_gt_y",
                  "mu_gt_z", "sig_est_xx", "sig_est_xy", "sig_est_xz", "sig_est_yy", "sig_est_yz", "sig_est_zz", "sig_gt_xx",
                  "sig_gt_xy", "sig_gt_xz", "sig_gt_yy", "sig_gt_yz", "sig_gt_zz", "offset", "shape", "w2")


class me_w2_result(C.Structure):
    _fields_ = [("aw2", C.c_double), ("mean_offset", C.c_double), ("mean_shape", C.c_double), ("scs", C.c_double),
                ("n_pairs", C.c_int64), ("n_scs", C.c_int64), ("n_voxels_est", C.c_int64), ("n_voxels_gt", C.c_int64)]


class me_icp_result(C.Structure):
    _fields_ = [("transformation", C.c_double * 16), ("fitness", C.c_double), ("inlier_rmse", C.c_double),
                ("n_corr", C.c_int64), ("iterations", C.c_int32), ("converged", C.c_int32)]


class me_global_reg_params(C.Structure):
    _fields_ = [("voxel_size", C.c_double), ("normal_knn", C.c_int32), ("feature_radius", C.c_double),
                ("feature_max_nn", C.c_int32), ("mutual_filter", C.c_int32), ("max_correspondence_distance", C.c_double),
                ("edge_ratio", C.c_double), ("n_hypotheses", C.c_int64), ("seed", C.c_uint64)]


class me_global_reg_result(C.Structure):
    _fields_ = [("T", C.c_double * 16), ("n_est_features", C.c_int64), ("n_gt_features", C.c_int64),
                ("n_correspondences", C.c_int64), ("n_valid_hypotheses", C.c_int64), ("best_hypothesis", C.c_int64),
                ("n_inliers", C.c_int64), ("inlier_rmse", C.c_double), ("stage_ms", C.c_double * 6)]


GLOBAL_REG_STAGES = ("copy_downsample", "normals", "fpfh", "matching", "ransac", "refine")


FPFH_DIM = 33


def make_global_reg_params(voxel_size, seed=0, **overrides):
    """me_global_reg_params with the defaults of the header (feature radius 10 voxels, inlier distance 1.5 voxels, ...)"""
    v = float(voxel_size)
    vals = dict(voxel_size=v, normal_knn=30, feature_radius=10.0 * v, feature_max_nn=128, mutual_filter=1,
                max_correspondence_distance=1.5 * v, edge_ratio=0.9, n_hypotheses=100000, seed=int(seed))
    unknown = set(overrides) - set(vals)
    if unknown:
        raise ValueError(f"unknown global registration parameters: {sorted(unknown)}")
    vals.update(overrides)
    p = me_global_reg_params()
    for k, x in vals.items():
        setattr(p, k, x)
    return p


def make_nn_params(tau, icp_max_distance=1.0, cutoff_mode=ME_CUTOFF_SQDIST_LE_R, pairing=ME_PAIRING_AS_WRITTEN,
                   want_full_cd=True, directions=0):
    p = me_nn_params()
    if len(tau) < 5:
        raise ValueError("accuracy_level needs 5 thresholds (map_eval_main.cpp:133-137)")
    for i in range(5):
        p.tau[i] = float(tau[i])
    p.icp_max_distance = float(icp_max_distance)
    p.cutoff_mode = int(cutoff_mode)
    p.pairing = int(pairing)
    p.want_full_cd = 1 if want_full_cd else 0
    p.directions = int(directions)
    return p


def struct_to_dict(s):
    """Recursively convert a ctypes struct into plain python (lists for arrays)."""
    out = {}
    for name, _ in s._fields_:
        v = getattr(s, name)
        if isinstance(v, C.Structure):
            out[name] = struct_to_dict(v)
        elif isinstance(v, C.Array):
            out[name] = list(v)
        else:
            out[name] = v
    return out

"""Python host mirror of the C-ABI: a thin context object used by the tests, bench.py and the multi-GPU plumbing.

Names follow the reference's members (`MapEval::computeMME`, `calculateMetricsWithInitialMatrix`, `calculateVMD`,
map_eval/src/map_eval.h:193-260) so the parity tests read like calls into the reference.  All computation happens
in libmapeval_b200.so on the GPU; this file only marshals arguments.
"""
import ctypes as C

import numpy as np

from . import _abi as A
from . import _lib


class MapEvalError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libmapeval_b200 error {code}: {msg}")
        self.code = code


def icp_update(method, block, center=None):
    """me_icp_update (host only): the 4x4 update of one ICP iteration from a reduced block (ME_ICP_BLOCK_P2P values about
    `center` for point-to-point, ME_ICP_BLOCK_NE for point-to-plane / generalized ICP)"""
    L = _lib.load()
    b = np.ascontiguousarray(block, dtype=np.float64)
    n_need = A.ME_ICP_BLOCK_P2P if method == A.ME_ICP_POINT_TO_POINT else A.ME_ICP_BLOCK_NE
    if b.size != n_need:
        raise ValueError(f"the block of method {method} has {n_need} values")
    dp = C.POINTER(C.c_double)
    c = None if center is None else np.ascontiguousarray(center, dtype=np.float64).reshape(3)
    out = np.empty(16, np.float64)
    rc = L.me_icp_update(int(method), b.ctypes.data_as(dp), c.ctypes.data_as(dp) if c is not None else None, out.ctypes.data_as(dp))
    if rc != A.ME_OK:
        raise MapEvalError(rc, "me_icp_update")
    return out.reshape(4, 4)


_CURVE_DIR = np.dtype([("n_inlier", "<i8"), ("mean", "<f8"), ("rmse", "<f8"), ("fitness", "<f8"), ("sigma", "<f8")])
# me_curve_row, field for field
_CURVE_ROW = np.dtype([("tau", "<f8"), ("est_to_gt", _CURVE_DIR), ("gt_to_est", _CURVE_DIR), ("cd", "<f8"), ("f1", "<f8"),
                       ("iou", "<f8")])
assert _CURVE_ROW.itemsize == C.sizeof(A.me_curve_row)


def _curve_levels(tau):
    t = np.ascontiguousarray(tau, dtype=np.float64).reshape(-1)
    return t, t.ctypes.data_as(C.POINTER(C.c_double))


def _curve_arrays(rows):
    """{'tau', 'cd', 'f1', 'iou': (K,) arrays, 'est_to_gt' / 'gt_to_est': {'n_inlier', 'mean', 'rmse', 'fitness', 'sigma'}}"""
    out = {k: rows[k].copy() for k in ("tau", "cd", "f1", "iou")}
    for d in ("est_to_gt", "gt_to_est"):
        out[d] = {k: rows[d][k].copy() for k in _CURVE_DIR.names}
    return out


def curve_finalize(params, e, g, block, tau, n_est, n_gt):
    """me_nn_curve_finalize (host only): the curve from a (reduced) curve block and the (reduced) accumulators of the
    me_eval_nn* call whose records it was built from; numpy arrays per field as MapEvalB200.accuracy_curve"""
    L = _lib.load()
    t, tp = _curve_levels(tau)
    b = np.ascontiguousarray(block, dtype=np.float64)
    if b.size != A.curve_block_len(t.size):
        raise ValueError(f"a curve block of {t.size} levels has {A.curve_block_len(t.size)} values")
    rows = np.zeros(t.size, _CURVE_ROW)
    rc = L.me_nn_curve_finalize(C.byref(params), C.byref(e) if e is not None else None, C.byref(g) if g is not None else None,
                                b.ctypes.data_as(C.POINTER(C.c_double)), tp, t.size, int(n_est), int(n_gt),
                                rows.ctypes.data_as(C.POINTER(A.me_curve_row)))
    if rc != A.ME_OK:
        raise MapEvalError(rc, "me_nn_curve_finalize: invalid levels, or a block and accumulators of different evaluations")
    return _curve_arrays(rows)


def _quantile_probs(p):
    q = np.ascontiguousarray(p, dtype=np.float64).reshape(-1)
    return q, q.ctypes.data_as(C.POINTER(C.c_double))


def quantile_finalize(n, p, lo_hi):
    """me_quantile_finalize (host only): the quantile values at the probabilities p of a sorted population of n values, from
    lo_hi = (K, 2) array of (x_k, x_min(k+1, n-1)), k = floor((n - 1) p) — numpy's method="linear" in its operation order"""
    L = _lib.load()
    q, qp = _quantile_probs(p)
    lh = np.ascontiguousarray(lo_hi, dtype=np.float64).reshape(-1)
    if lh.size != 2 * q.size:
        raise ValueError("lo_hi holds one (lo, hi) pair per probability")
    out = np.empty(q.size, np.float64)
    dp = C.POINTER(C.c_double)
    rc = L.me_quantile_finalize(int(n), qp, q.size, lh.ctypes.data_as(dp), out.ctypes.data_as(dp))
    if rc != A.ME_OK:
        raise MapEvalError(rc, "me_quantile_finalize: n >= 1, 1 <= K <= ME_QUANTILE_MAX_PROBS, every p finite and in [0, 1]")
    return out


def quantile_dict(res):
    """me_quantile_result -> {'est_to_gt' / 'gt_to_est': {'n', 'min', 'max', 'rank', 'lo', 'hi', 'value'}, 'p', 'hausdorff'}"""
    K = res.n_probs
    out = {"p": np.array(res.p[:K]), "hausdorff": float(res.hausdorff)}
    for name in ("est_to_gt", "gt_to_est"):
        d = getattr(res, name)
        out[name] = {"n": int(d.n), "min": float(d.min), "max": float(d.max), "rank": np.array(d.rank[:K], np.int64),
                     "lo": np.array(d.lo[:K]), "hi": np.array(d.hi[:K]), "value": np.array(d.value[:K])}
    return out


_REGION_DIR_DT = np.dtype([("n_query", "<i8"), ("n_corr", "<i8"), ("n_inlier", "<i8", 5), ("sum_d", "<f8", 5), ("sum_d2", "<f8", 5),
                           ("sum_nn_dist", "<f8"), ("max_d", "<f8"), ("max_nn", "<f8"), ("mean", "<f8", 5), ("rmse", "<f8", 5),
                           ("fitness", "<f8", 5), ("mean_nn", "<f8")])
# me_region_row as a numpy record (8-byte fields only, so no padding): the rows convert without a per-row Python step
_REGION_ROW_DT = np.dtype([("index", "<i8", 3), ("min", "<f8", 3), ("max", "<f8", 3), ("n_est", "<i8"), ("n_gt", "<i8"),
                           ("est_to_gt", _REGION_DIR_DT), ("gt_to_est", _REGION_DIR_DT), ("cd", "<f8", 5), ("f1", "<f8", 5),
                           ("iou", "<f8", 5)])
assert _REGION_ROW_DT.itemsize == C.sizeof(A.me_region_row) and _REGION_DIR_DT.names == tuple(f[0] for f in A.me_region_dir._fields_)


def region_dict(a):
    """me_region_row records (numpy, _REGION_ROW_DT) -> {'index' (n, 3) int64, 'min' / 'max' (n, 3), 'n_est', 'n_gt',
    'cd' / 'f1' / 'iou' (n, 5), 'est_to_gt' / 'gt_to_est': {field: array}}, one entry per field"""
    out = {name: np.array(a[name]) for name in ("index", "min", "max", "n_est", "n_gt", "cd", "f1", "iou")}
    for name in ("est_to_gt", "gt_to_est"):
        out[name] = {f: np.array(a[name][f]) for f in _REGION_DIR_DT.names}
    return out


def _region_rows(n):
    """zeroed records for n rows and the pointer the C-ABI takes"""
    rows = np.zeros(max(int(n), 1), _REGION_ROW_DT)
    return rows, rows.ctypes.data_as(C.POINTER(A.me_region_row))


def region_finalize(region_size, index, n_est, n_gt, block):
    """me_region_finalize (host only): the rows of n regions from a reduced host block (ME_REGION_SUM_FIELDS x 2 SUM values per
    region, then ME_REGION_MAX_FIELDS x 2 MAX values), index (n, 3) and the per-region point counts; as region_dict"""
    L = _lib.load()
    idx = np.ascontiguousarray(index, dtype=np.int64).reshape(-1, 3)
    n = idx.shape[0]
    ne = np.ascontiguousarray(n_est, dtype=np.int64).reshape(-1)
    ng = np.ascontiguousarray(n_gt, dtype=np.int64).reshape(-1)
    blk = np.ascontiguousarray(block, dtype=np.float64).reshape(-1)
    if ne.size != n or ng.size != n or blk.size != 2 * (A.ME_REGION_SUM_FIELDS + A.ME_REGION_MAX_FIELDS) * n:
        raise ValueError("one index triple, one n_est / n_gt and 2 x (ME_REGION_SUM_FIELDS + ME_REGION_MAX_FIELDS) values per region")
    rows, rows_p = _region_rows(n)
    i64 = C.POINTER(C.c_int64)
    rc = L.me_region_finalize(n, float(region_size), idx.ctypes.data_as(i64), ne.ctypes.data_as(i64), ng.ctypes.data_as(i64),
                              blk.ctypes.data_as(C.POINTER(C.c_double)), rows_p)
    if rc != A.ME_OK:
        raise MapEvalError(rc, "me_region_finalize: n >= 0, region_size finite and > 0")
    return region_dict(rows[:n])


def surface_dict(res):
    """me_surface_result -> {'cd' / 'f1' / 'iou' (5,), 'full_cd', 'normal_consistency', 'est_to_gt' / 'gt_to_est': {the
    me_dir_result fields of the point-to-plane table, then the me_surface_dir fields}}; arrays for the five levels"""
    def _v(x):
        return np.array(x[:]) if isinstance(x, C.Array) else x
    out = {name: np.array(getattr(res.plane, name)[:]) for name in ("cd", "f1", "iou")}
    out["full_cd"] = res.plane.full_cd
    out["normal_consistency"] = res.normal_consistency
    for name in ("est_to_gt", "gt_to_est"):
        p, s = getattr(res.plane, name), getattr(res, name)
        d = {f[0]: _v(getattr(p, f[0])) for f in A.me_dir_result._fields_}
        d.update({f[0]: getattr(s, f[0]) for f in A.me_surface_dir._fields_})
        out[name] = d
    return out


def surface_finalize(params, block, n_est, n_gt):
    """me_surface_finalize (host only): the point-to-plane result from a reduced host block (ME_SURFACE_BLOCK_SUM SUM values,
    then ME_SURFACE_BLOCK_MAX MAX values) with the NN evaluation's parameters and the cloud sizes; as surface_dict"""
    L = _lib.load()
    blk = np.ascontiguousarray(block, dtype=np.float64).reshape(-1)
    if blk.size != A.ME_SURFACE_BLOCK_SUM + A.ME_SURFACE_BLOCK_MAX:
        raise ValueError("ME_SURFACE_BLOCK_SUM + ME_SURFACE_BLOCK_MAX values")
    out = A.me_surface_result()
    rc = L.me_surface_finalize(C.byref(params), blk.ctypes.data_as(C.POINTER(C.c_double)), int(n_est), int(n_gt), C.byref(out))
    if rc != A.ME_OK:
        raise MapEvalError(rc, "me_surface_finalize")
    return surface_dict(out)


# me_drift_row as a numpy record (8-byte fields, then two int32: no padding)
_DRIFT_ROW_DT = np.dtype([("index", "<i8", 3), ("min", "<f8", 3), ("max", "<f8", 3), ("n_est", "<i8"), ("n_corr_before", "<i8"),
                          ("fitness_before", "<f8"), ("rmse_before", "<f8"), ("n_corr", "<i8"), ("fitness", "<f8"), ("rmse", "<f8"),
                          ("T", "<f8", 16), ("centroid", "<f8", 3), ("shift", "<f8", 3), ("shift_norm", "<f8"), ("angle", "<f8"),
                          ("iterations", "<i4"), ("status", "<i4")])
assert _DRIFT_ROW_DT.itemsize == C.sizeof(A.me_drift_row) and _DRIFT_ROW_DT.names == tuple(f[0] for f in A.me_drift_row._fields_)


def drift_dict(a):
    """me_drift_row records (numpy, _DRIFT_ROW_DT) -> {field: array}, one entry per row field, 'T' as (n, 4, 4)"""
    out = {name: np.array(a[name]) for name in _DRIFT_ROW_DT.names}
    out["T"] = out["T"].reshape(-1, 4, 4)
    return out


# me_consistency_row as a numpy record (8-byte fields only, so no padding)
_CONS_ROW_DT = np.dtype([("index", "<i8", 3), ("min", "<f8", 3), ("max", "<f8", 3), ("n_points", "<i8"), ("n_query", "<i8"),
                         ("n_valid", "<i8"), ("n_pv", "<i8"), ("sum_entropy", "<f8"), ("sum_pv", "<f8"), ("sum_sqrt_pv", "<f8"),
                         ("mme", "<f8"), ("mpv", "<f8"), ("mean_plane_std", "<f8"), ("max_pv", "<f8")])
assert _CONS_ROW_DT.itemsize == C.sizeof(A.me_consistency_row) and \
    _CONS_ROW_DT.names == tuple(f[0] for f in A.me_consistency_row._fields_)


def consistency_dict(rows, whole):
    """me_consistency_row records (numpy, _CONS_ROW_DT) and the me_consistency_result -> {'whole': {field: value}, 'kernel'
    (ME_CONSISTENCY_* name), then one array per row field: 'index' / 'min' / 'max' (n, 3), 'n_points', ..., 'max_pv'}"""
    out = {name: np.array(rows[name]) for name in _CONS_ROW_DT.names}
    out["whole"] = {f[0]: getattr(whole, f[0]) for f in A.me_consistency_result._fields_}
    out["kernel"] = A.CONSISTENCY_KERNEL_NAMES.get(whole.kernel, str(whole.kernel))
    return out


def mom_dict(res):
    """me_mom_result -> {field: value}; 'axis' (3, 3) rows a1 a2 a3, 'n' / 'mean' / 'median' (3,), 'status' its
    ME_MOM_* name"""
    out = {}
    for f in A.me_mom_result._fields_:
        if f[0] == "reserved":
            continue
        x = getattr(res, f[0])
        out[f[0]] = np.array(x[:]) if isinstance(x, C.Array) else x
    out["axis"] = out["axis"].reshape(3, 3)
    out["status"] = A.MOM_STATUS_NAMES.get(res.status, str(res.status))
    return out


# me_mom_region_row as a numpy record (8-byte fields, then two int32: no padding)
_MOM_REGION_ROW_DT = np.dtype([("index", "<i8", 3), ("n_points", "<i8"), ("n_planar", "<i8"), ("n", "<i8", 3), ("mean", "<f8", 3),
                               ("median", "<f8", 3), ("mom", "<f8"), ("status", "<i4"), ("reserved", "<i4")])
assert _MOM_REGION_ROW_DT.itemsize == C.sizeof(A.me_mom_region_row) and \
    _MOM_REGION_ROW_DT.names == tuple(f[0] for f in A.me_mom_region_row._fields_)


def mom_region_dict(rows, region_size):
    """me_mom_region_row records (numpy, _MOM_REGION_ROW_DT) at region size s -> {'index' / 'lo' / 'hi' (n, 3): the region
    floor(x / s) and its bounds index * s, (index + 1) * s; 'n_points', 'n_planar' (n,); 'n' / 'mean' / 'median' (n, 3)
    per family; 'mom' (n,); 'status' (n,) ME_MOM_* names, as mom_dict names them}"""
    s = float(region_size)
    out = {name: np.array(rows[name]) for name in ("index", "n_points", "n_planar", "n", "mean", "median", "mom")}
    out["index"] = out["index"].reshape(-1, 3)
    for name in ("n", "mean", "median"):
        out[name] = out[name].reshape(-1, 3)
    out["lo"] = out["index"].astype(np.float64) * s
    out["hi"] = (out["index"] + 1).astype(np.float64) * s
    codes = np.asarray(rows["status"]).reshape(-1)
    names = np.array([A.MOM_STATUS_NAMES[k] for k in sorted(A.MOM_STATUS_NAMES)], dtype=object)
    if len(codes) and not ((codes >= 0) & (codes < len(names))).all():
        raise ValueError("mom_region_dict: a status outside me_mom_status")
    out["status"] = names[codes]
    return out


def mom_params(angle_deg=10.0, planarity=0.5, min_family=100):
    return A.me_mom_params(float(angle_deg), float(planarity), int(min_family))


def mom_axes(hist, angle_deg=10.0, cells_per_edge=A.ME_MOM_CELLS_PER_EDGE):
    """me_mom_axes (host only): (axes (3, 3) rows a1 a2 a3, NaN where not found; status name) from an integer histogram
    of 6 cells_per_edge^2 bins"""
    L = _lib.load()
    h = np.ascontiguousarray(hist, dtype=np.int64)
    if h.shape != (6 * cells_per_edge * cells_per_edge,):
        raise ValueError("the histogram needs 6 cells_per_edge^2 bins")
    axes = np.zeros(9, np.float64)
    st = C.c_int32(0)
    rc = L.me_mom_axes(h.ctypes.data_as(C.POINTER(C.c_int64)), int(cells_per_edge), float(angle_deg),
                       axes.ctypes.data_as(C.POINTER(C.c_double)), C.byref(st))
    if rc != A.ME_OK:
        raise MapEvalError(rc, "me_mom_axes: cells_per_edge in 1..1024, angle_deg in (0, 30], counts >= 0")
    return axes.reshape(3, 3), A.MOM_STATUS_NAMES.get(st.value, str(st.value))


def consistency_finalize(region_size, index, n_points, n_total, block):
    """me_consistency_finalize (host only): the rows of n regions and the whole-map result from a reduced host block
    (ME_CONSISTENCY_SUM_FIELDS SUM values per region, then ME_CONSISTENCY_MAX_FIELDS MAX values; one region, the whole map,
    at region_size 0 with no index), the region indices (n, 3), the per-region point counts and the cloud size; as
    consistency_dict (radius, min_neighbors, kernel, rings and solo are 0)"""
    L = _lib.load()
    idx = np.ascontiguousarray(index, dtype=np.int64).reshape(-1, 3)
    n = idx.shape[0]
    npts = np.ascontiguousarray(n_points, dtype=np.int64).reshape(-1)
    blk = np.ascontiguousarray(block, dtype=np.float64).reshape(-1)
    if npts.size != n or blk.size != (A.ME_CONSISTENCY_SUM_FIELDS + A.ME_CONSISTENCY_MAX_FIELDS) * max(n, 1):
        raise ValueError("one index triple and one point count per region, and ME_CONSISTENCY_SUM_FIELDS + "
                         "ME_CONSISTENCY_MAX_FIELDS values per region (one region at region_size 0)")
    rows = np.zeros(max(n, 1), _CONS_ROW_DT)
    whole = A.me_consistency_result()
    i64 = C.POINTER(C.c_int64)
    rc = L.me_consistency_finalize(n, float(region_size), idx.ctypes.data_as(i64), npts.ctypes.data_as(i64), int(n_total),
                                   blk.ctypes.data_as(C.POINTER(C.c_double)), rows.ctypes.data_as(C.c_void_p), C.byref(whole))
    if rc != A.ME_OK:
        raise MapEvalError(rc, "me_consistency_finalize: n >= 0, region_size finite and >= 0, n = 0 exactly at region_size 0")
    return consistency_dict(rows[:n], whole)


class MapEvalB200:
    """One context = one GPU.  rank/world select this context's contiguous query range (multi-GPU sharding)."""

    def __init__(self, device=0, rank=0, world=1, stream=None, nn_cell_size=0.0, max_grid_cells=0,
                 vmd_voxel_size=0.0):
        self._L = _lib.load()
        opt = A.me_options()
        opt.abi_version = A.ME_ABI_VERSION
        opt.device, opt.rank, opt.world = int(device), int(rank), int(world)
        opt.stream = C.c_void_p(int(stream)) if stream else None
        opt.nn_cell_size = float(nn_cell_size)
        opt.max_grid_cells = int(max_grid_cells)
        opt.vmd_voxel_size = float(vmd_voxel_size)
        self._ctx = C.c_void_p()
        rc = self._L.me_create(C.byref(opt), C.byref(self._ctx))
        if rc != A.ME_OK:
            msg = self._L.me_last_error(None)
            self._ctx = None
            raise MapEvalError(rc, msg.decode() if msg else "me_create failed")
        self.n = [0, 0]
        self._keep = [None, None]   # keeps host/device buffers alive while the library may read them
        self._mom_min_family_last = None   # min_family of the last finished MOM call (mom_regions' default)
        self._mom_region_size = None
        self.rank, self.world = int(rank), int(world)

    # -- lifecycle -------------------------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_ctx", None):
            self._L.me_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _check(self, rc):
        if rc != A.ME_OK:
            msg = self._L.me_last_error(self._ctx)
            raise MapEvalError(rc, msg.decode() if msg else "")

    def _block(self, fn, *count_types, args=()):
        """(device pointer, counts...) of a device block: fn(ctx, *args, &ptr, &count...) with one count of each ctypes type"""
        ptr = C.POINTER(C.c_double)()
        counts = [t(0) for t in count_types]
        self._check(fn(self._ctx, *args, C.byref(ptr), *(C.byref(c) for c in counts)))
        return (C.cast(ptr, C.c_void_p).value, *(c.value for c in counts))

    def _take_rows(self, ptr, n, dtype):
        """a numpy copy of n library-allocated rows of dtype at ptr; the rows are freed (me_free) in every case"""
        try:
            addr = C.cast(ptr, C.c_void_p).value
            nb = n * dtype.itemsize
            return np.frombuffer((C.c_char * nb).from_address(addr), dtype).copy() if nb else np.zeros(0, dtype)
        finally:
            self._L.me_free(ptr)

    def set_stream(self, stream_ptr):
        self._check(self._L.me_set_stream(self._ctx, C.c_void_p(int(stream_ptr)) if stream_ptr else None))

    def set_shard(self, rank, world):
        self._check(self._L.me_set_shard(self._ctx, rank, world))
        self.rank, self.world = int(rank), int(world)

    def synchronize(self):
        self._check(self._L.me_synchronize(self._ctx))

    # -- clouds ----------------------------------------------------------------------------------------------
    def set_cloud(self, which, xyz):
        """xyz: (N,3) float64 numpy array (host) or a pinned torch CPU tensor's data pointer via .numpy()."""
        a = np.ascontiguousarray(xyz, dtype=np.float64)
        if a.ndim != 2 or a.shape[1] != 3:
            raise ValueError("cloud must be (N, 3)")
        self._keep[which] = a
        self.n[which] = a.shape[0]
        self._check(self._L.me_set_cloud(self._ctx, which, a.ctypes.data_as(C.c_void_p), a.shape[0]))

    def set_cloud_ptr(self, which, host_ptr, n, keepalive=None):
        self._keep[which] = keepalive
        self.n[which] = int(n)
        self._check(self._L.me_set_cloud(self._ctx, which, C.c_void_p(int(host_ptr)), int(n)))

    def set_cloud_device(self, which, device_ptr, n, keepalive=None):
        """Borrow an fp64 (N,3) device buffer (e.g. a torch.cuda tensor's data_ptr())."""
        self._keep[which] = keepalive
        self.n[which] = int(n)
        self._check(self._L.me_set_cloud_device(self._ctx, which, C.c_void_p(int(device_ptr)), int(n)))

    def transform(self, which, T):
        T = np.ascontiguousarray(T, dtype=np.float64).reshape(16)
        self._check(self._L.me_transform(self._ctx, which, T.ctypes.data_as(C.POINTER(C.c_double))))

    def performICPRegistration(self, max_correspondence_distance, T_init=None, max_iteration=30, relative_fitness=1e-6,
                               relative_rmse=1e-6, method=A.ME_ICP_POINT_TO_POINT):
        """map_eval.cpp:1366-1394: RegistrationICP with the point-to-point (method 0) or point-to-plane (1) estimation, or
        RegistrationGeneralizedICP (2, `registration_methods` of the config); the estimated cloud held by the context is
        transformed by the result.  Returns (T 4x4, me_icp_result)."""
        T = np.ascontiguousarray(np.eye(4) if T_init is None else T_init, dtype=np.float64).reshape(16)
        out = A.me_icp_result()
        self._check(self._L.me_icp(self._ctx, int(method), float(max_correspondence_distance), int(max_iteration),
                                   float(relative_fitness), float(relative_rmse),
                                   T.ctypes.data_as(C.POINTER(C.c_double)), C.byref(out)))
        self._keep[A.ME_CLOUD_EST] = None
        return np.array(list(out.transformation)).reshape(4, 4), out

    # -- registration split at its collective (multi-GPU; dist.icp_distributed runs the loop) -------------------------
    def icp_begin(self, max_correspondence_distance, T_init=None, max_iteration=30, relative_fitness=1e-6,
                  relative_rmse=1e-6, method=A.ME_ICP_GENERALIZED):
        T = np.ascontiguousarray(np.eye(4) if T_init is None else T_init, dtype=np.float64).reshape(16)
        self._check(self._L.me_icp_begin(self._ctx, int(method), float(max_correspondence_distance), int(max_iteration),
                                         float(relative_fitness), float(relative_rmse), T.ctypes.data_as(C.POINTER(C.c_double))))

    def icp_normals_slice(self, which):
        """(device pointer of the world * slice * 3 fp64 normal buffer or None, slice points, pending): pending = True when
        the caller must all-gather the buffer in place (this rank filled rows [rank * slice, (rank + 1) * slice))"""
        ptr = C.POINTER(C.c_double)()
        s, pend = C.c_int64(0), C.c_int32(0)
        self._check(self._L.me_icp_normals_slice(self._ctx, int(which), C.byref(ptr), C.byref(s), C.byref(pend)))
        return C.cast(ptr, C.c_void_p).value, s.value, bool(pend.value)

    def icp_block(self):
        """(device pointer, n_sum) of this rank's partial ICP sums (SUM-all-reduce in place); the first call sweeps"""
        return self._block(self._L.me_icp_block, C.c_int32)

    def icp_step(self):
        """reads the reduced block, updates T, moves and sweeps again; True when the loop is over"""
        done = C.c_int32(0)
        self._check(self._L.me_icp_step(self._ctx, C.byref(done)))
        return bool(done.value)

    def icp_end(self):
        """est := Transform(original, T); returns (T 4x4, me_icp_result) like performICPRegistration"""
        out = A.me_icp_result()
        self._check(self._L.me_icp_end(self._ctx, C.byref(out)))
        self._keep[A.ME_CLOUD_EST] = None
        return np.array(list(out.transformation)).reshape(4, 4), out

    def set_normals(self, which, normals):
        a = np.ascontiguousarray(normals, dtype=np.float64)
        self._check(self._L.me_set_normals(self._ctx, which, a.ctypes.data_as(C.POINTER(C.c_double)), a.shape[0]))

    def estimate_normals(self, which, knn=20):
        """PointCloud::EstimateNormals(KDTreeSearchParamKNN(knn)); returns the (N, 3) normals in caller order."""
        self._check(self._L.me_estimate_normals(self._ctx, which, int(knn)))
        return self.get_normals(which)

    def get_normals(self, which):
        """The normals of the held cloud, (N, 3) in the order of get_cloud; an error when the cloud has none."""
        out = np.empty((self.n[which], 3), np.float64)
        self._check(self._L.me_get_normals(self._ctx, which, out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    def voxel_downsample(self, which, voxel_size):
        """PointCloud::VoxelDownSample on the held cloud (map_eval.cpp:38-39); returns the new point count."""
        n = C.c_int64(0)
        self._check(self._L.me_voxel_downsample(self._ctx, which, float(voxel_size), C.byref(n)))
        self.n[which] = n.value
        self._keep[which] = None
        return n.value

    # -- simulated degradation (evaluate_noised_gt; map_eval.cpp:1745-1829): pure functions of (cloud, parameters, seed) -------
    def copy_cloud(self, src, dst):
        """dst := src (points, and normals when src holds them) in library-owned memory; also turns a borrowed ground
        truth into an owned estimate that the operators below may change."""
        self._check(self._L.me_copy_cloud(self._ctx, int(src), int(dst)))
        self.n[dst] = self.n[src]
        self._keep[dst] = None

    def add_gaussian_noise(self, which, std_dev, seed):
        """MapEval::addGaussianNoise: p += std_dev * N(0, 1) per axis, in place."""
        self._check(self._L.me_add_gaussian_noise(self._ctx, int(which), float(std_dev), int(seed)))

    def add_non_uniform_density(self, which, sparse_ratio, dense_ratio, region_size, seed):
        """MapEval::addNonUniformDensity (stable compaction); returns the new point count."""
        n = C.c_int64(0)
        self._check(self._L.me_add_non_uniform_density(self._ctx, int(which), float(sparse_ratio), float(dense_ratio),
                                                       float(region_size), int(seed), C.byref(n)))
        self.n[which] = n.value
        return n.value

    def add_sparse_outliers(self, which, outlier_ratio, outlier_range, seed):
        """MapEval::addSparseOutliers (outliers appended; the cloud loses its normals); returns the new point count."""
        n = C.c_int64(0)
        self._check(self._L.me_add_sparse_outliers(self._ctx, int(which), float(outlier_ratio), float(outlier_range), int(seed),
                                                   C.byref(n)))
        self.n[which] = n.value
        return n.value

    def add_local_deformation(self, which, radius, strength, center):
        """MapEval::addLocalDeformation: radial push inside the radius, cosine fall-off, in place."""
        c = np.ascontiguousarray(center, dtype=np.float64).reshape(3)
        self._check(self._L.me_add_local_deformation(self._ctx, int(which), float(radius), float(strength),
                                                     c.ctypes.data_as(C.POINTER(C.c_double))))

    def get_cloud(self, which):
        """The cloud currently held by the context as an (N, 3) float64 array."""
        n = C.c_int64(0)
        self._check(self._L.me_get_cloud(self._ctx, which, None, 0, C.byref(n)))
        out = np.empty((n.value, 3), np.float64)
        self._check(self._L.me_get_cloud(self._ctx, which, out.ctypes.data_as(C.POINTER(C.c_double)), n.value, C.byref(n)))
        return out

    # -- coarse global registration: the initial pose from the maps alone -----------------------------------------------
    def global_registration(self, voxel_size, seed=0, **overrides):
        """me_global_registration: FPFH features, mutual matching and RANSAC on private feature clouds down-sampled at
        voxel_size; the context's clouds are left alone.  overrides: any other field of me_global_reg_params.  Returns a
        dict of me_global_reg_result with T as a 4x4 array (est -> gt)."""
        p = A.make_global_reg_params(voxel_size, seed, **overrides)
        out = A.me_global_reg_result()
        self._check(self._L.me_global_registration(self._ctx, C.byref(p), C.byref(out)))
        r = A.struct_to_dict(out)
        r["T"] = np.array(r["T"]).reshape(4, 4)
        r["stage_ms"] = dict(zip(A.GLOBAL_REG_STAGES, r["stage_ms"]))
        return r

    def get_correspondences(self):
        """(est feature indices, gt feature indices) of the last global_registration's correspondences, in est order"""
        n = C.c_int64(0)
        self._check(self._L.me_get_correspondences(self._ctx, None, None, 0, C.byref(n)))
        ie, ig = np.empty(n.value, np.int32), np.empty(n.value, np.int32)
        self._check(self._L.me_get_correspondences(self._ctx, ie.ctypes.data_as(C.c_void_p), ig.ctypes.data_as(C.c_void_p),
                                                   n.value, C.byref(n)))
        return ie, ig

    def get_features(self, which):
        """(xyz (N, 3), oriented normals (N, 3), FPFH (N, 33) float32) of the feature cloud the last global_registration
        built from cloud `which`, in the order of the down-sampled cloud"""
        n = C.c_int64(0)
        self._check(self._L.me_get_features(self._ctx, int(which), None, None, None, 0, C.byref(n)))
        xyz, nrm = np.empty((n.value, 3), np.float64), np.empty((n.value, 3), np.float64)
        f = np.empty((n.value, A.FPFH_DIM), np.float32)
        dp = C.POINTER(C.c_double)
        self._check(self._L.me_get_features(self._ctx, int(which), xyz.ctypes.data_as(dp), nrm.ctypes.data_as(dp),
                                            f.ctypes.data_as(C.POINTER(C.c_float)), n.value, C.byref(n)))
        return xyz, nrm, f

    def build_grid(self, which):
        self._check(self._L.me_build_grid(self._ctx, which))

    # -- a1/a2/a4 ----------------------------------------------------------------------------------------------
    def eval_nn_accum(self, params):
        e, g = A.me_nn_accum(), A.me_nn_accum()
        self._check(self._L.me_eval_nn_accum(self._ctx, C.byref(params), C.byref(e), C.byref(g)))
        return e, g

    def nn_finalize(self, params, e, g):
        out = A.me_nn_result()
        rc = self._L.me_nn_finalize(C.byref(params), C.byref(e), C.byref(g), self.n[0], self.n[1], C.byref(out))
        if rc != A.ME_OK:
            raise MapEvalError(rc, "me_nn_finalize")
        return out

    def calculateMetricsWithInitialMatrix(self, params):
        """map_eval.cpp:1204-1260 (single GPU)."""
        out = A.me_nn_result()
        self._check(self._L.me_eval_nn(self._ctx, C.byref(params), C.byref(out)))
        return out

    def accuracy_curve(self, tau):
        """AC / COM / CD / F1 / IoU at every level of tau (1..ME_CURVE_MAX_LEVELS thresholds, finite, >= 0, non-decreasing)
        from the records of the last NN evaluation, without a new sweep (me_nn_curve, world 1).  Returns numpy arrays per
        field: 'tau', 'cd', 'f1', 'iou' and per direction 'est_to_gt' / 'gt_to_est' a dict of 'n_inlier', 'mean', 'rmse',
        'fitness', 'sigma'.  Multi-GPU: curve_accum_device + dist.allreduce_curve + curve_finalize."""
        t, tp = _curve_levels(tau)
        rows = np.zeros(t.size, _CURVE_ROW)
        self._check(self._L.me_nn_curve(self._ctx, tp, t.size, rows.ctypes.data_as(C.POINTER(A.me_curve_row))))
        return _curve_arrays(rows)

    def curve_accum_device(self, tau):
        """(device pointer, n) of this rank's SUM-reducible curve block at the levels tau (me_nn_curve_accum_device)"""
        t, tp = _curve_levels(tau)
        return self._block(self._L.me_nn_curve_accum_device, C.c_int32, args=(tp, t.size))

    def distance_quantiles(self, p, population=A.ME_DIST_KEPT):
        """Exact quantiles at the probabilities p (1..ME_QUANTILE_MAX_PROBS values in [0, 1]) of the distances of the last NN
        evaluation, per direction, with min, max and the Hausdorff distance (me_nn_quantiles, world 1).  population:
        ME_DIST_KEPT (the kept pairs' d) or ME_DIST_NN (every query's NN distance; needs want_full_cd).  Returns
        {'est_to_gt' / 'gt_to_est': {'n', 'min', 'max', 'rank', 'lo', 'hi', 'value'}, 'p', 'hausdorff'}.  Multi-GPU:
        dist.quantiles_distributed."""
        q, qp = _quantile_probs(p)
        out = A.me_quantile_result()
        self._check(self._L.me_nn_quantiles(self._ctx, int(population), qp, q.size, C.byref(out)))
        return quantile_dict(out)

    def quantile_begin(self, p, population=A.ME_DIST_KEPT):
        """me_nn_quantile_begin: checks the arguments and the records, runs the first selection pass"""
        q, qp = _quantile_probs(p)
        self._check(self._L.me_nn_quantile_begin(self._ctx, int(population), qp, q.size))

    def quantile_block(self):
        """(device pointer, n) of the running pass's SUM-reducible block (all-reduce it in place after synchronize())"""
        return self._block(self._L.me_nn_quantile_block, C.c_int32)

    def quantile_step(self):
        """reads the reduced block and runs the next pass; True after the last one"""
        done = C.c_int32(0)
        self._check(self._L.me_nn_quantile_step(self._ctx, C.byref(done)))
        return bool(done.value)

    def quantile_end(self):
        """the result of the selection, as distance_quantiles"""
        out = A.me_quantile_result()
        self._check(self._L.me_nn_quantile_end(self._ctx, C.byref(out)))
        return quantile_dict(out)

    def region_errors(self, region_size):
        """AC / COM / CD / F1 / IoU per occupied region floor(x / region_size) of the last NN evaluation's records, both
        directions (me_nn_regions, world 1).  Returns region_dict's dict of arrays, rows ascending by (ix, iy, iz).
        Multi-GPU: dist.regions_distributed."""
        rows = C.POINTER(A.me_region_row)()
        n = C.c_int64(0)
        self._check(self._L.me_nn_regions(self._ctx, float(region_size), C.byref(rows), C.byref(n)))
        return region_dict(self._take_rows(rows, n.value, _REGION_ROW_DT))

    def region_begin(self, region_size):
        """me_nn_region_begin: lists the occupied regions and folds this rank's records; returns the region count"""
        n = C.c_int64(0)
        self._check(self._L.me_nn_region_begin(self._ctx, float(region_size), C.byref(n)))
        return n.value

    def region_block(self):
        """(device pointer, n_sum, n_max) of the block: SUM-reduce its first n_sum values and MAX-reduce the next n_max in place
        (after synchronize())"""
        return self._block(self._L.me_nn_region_block, C.c_int32, C.c_int32)

    def region_end(self, n_regions):
        """the rows from the reduced block, as region_errors"""
        rows, rows_p = _region_rows(n_regions)
        self._check(self._L.me_nn_region_end(self._ctx, rows_p, int(n_regions)))
        return region_dict(rows[:int(n_regions)])

    def surface_metrics(self, knn=0):
        """Point-to-plane AC / COM / CD / F1 / IoU and normal consistency from the last NN evaluation's records (me_nn_surface,
        world 1): the distance of every query point to the tangent plane of its nearest neighbour, and |n_p . n_t| per pair.
        knn = 0 uses the clouds' own normals; knn in 1..64 estimates k-NN normals for a cloud without them as a working copy
        (the cloud still has none afterwards).  Returns surface_dict's dict.  Multi-GPU: dist.surface_distributed."""
        out = A.me_surface_result()
        self._check(self._L.me_nn_surface(self._ctx, int(knn), C.byref(out)))
        return surface_dict(out)

    def surface_begin(self, knn=0):
        """me_nn_surface_begin: checks the records, the normals and knn"""
        self._check(self._L.me_nn_surface_begin(self._ctx, int(knn)))

    def surface_normals_slice(self, which):
        """(device pointer of the world * slice * 3 fp64 normal buffer or None, slice points, pending): pending = True when
        the caller must all-gather the buffer in place (this rank filled rows [rank * slice, (rank + 1) * slice))"""
        ptr = C.POINTER(C.c_double)()
        s, pend = C.c_int64(0), C.c_int32(0)
        self._check(self._L.me_nn_surface_normals_slice(self._ctx, int(which), C.byref(ptr), C.byref(s), C.byref(pend)))
        return C.cast(ptr, C.c_void_p).value, s.value, bool(pend.value)

    def surface_block(self):
        """(device pointer, n_sum, n_max) of the block; the first call folds this rank's records.  SUM-reduce the first n_sum
        values and MAX-reduce the next n_max in place (after synchronize())"""
        return self._block(self._L.me_nn_surface_block, C.c_int32, C.c_int32)

    def surface_end(self):
        """the result from the reduced block, as surface_metrics"""
        out = A.me_surface_result()
        self._check(self._L.me_nn_surface_end(self._ctx, C.byref(out)))
        return surface_dict(out)

    def region_drift(self, region_size, max_correspondence_distance, max_iteration=30, relative_fitness=1e-6,
                     relative_rmse=1e-6):
        """Aligns every occupied region floor(x / region_size) of the estimated cloud to the ground truth on its own: one
        point-to-point ICP per region, all in one pass per iteration (me_drift, world 1).  Returns drift_dict's dict of
        arrays, rows ascending by (ix, iy, iz): the transform T (R x 4 x 4) that moves the region onto the ground truth, its
        centroid shift and rotation angle, and the fitness / rmse before and after.  The estimated cloud is unchanged
        afterwards.  Multi-GPU: dist.drift_distributed."""
        rows = C.POINTER(A.me_drift_row)()
        n = C.c_int64(0)
        self._check(self._L.me_drift(self._ctx, float(region_size), float(max_correspondence_distance), int(max_iteration),
                                     float(relative_fitness), float(relative_rmse), C.byref(rows), C.byref(n)))
        return drift_dict(self._take_rows(rows, n.value, _DRIFT_ROW_DT))

    def drift_begin(self, region_size, max_correspondence_distance, max_iteration=30, relative_fitness=1e-6,
                    relative_rmse=1e-6):
        """me_drift_begin: lists the regions, keeps a copy of the estimated cloud, runs the first sweep and fold; returns
        the region count"""
        n = C.c_int64(0)
        self._check(self._L.me_drift_begin(self._ctx, float(region_size), float(max_correspondence_distance),
                                           int(max_iteration), float(relative_fitness), float(relative_rmse), C.byref(n)))
        return n.value

    def drift_block(self):
        """(device pointer, n_sum) of the block, ME_ICP_BLOCK_P2P values per region: SUM-reduce it in place (after
        synchronize())"""
        return self._block(self._L.me_drift_block, C.c_int32)

    def drift_step(self):
        """reads the reduced block, updates every running region, moves and sweeps again; True when every region is done"""
        done = C.c_int32(0)
        self._check(self._L.me_drift_step(self._ctx, C.byref(done)))
        return bool(done.value)

    def drift_end(self, n_regions):
        """the rows, as region_drift; the estimated cloud is back as it was at drift_begin"""
        rows = np.zeros(max(int(n_regions), 1), _DRIFT_ROW_DT)
        self._check(self._L.me_drift_end(self._ctx, rows.ctypes.data_as(C.POINTER(A.me_drift_row)), int(n_regions)))
        return drift_dict(rows[:int(n_regions)])

    def local_consistency(self, which, radius, min_neighbors=10, region_size=0.0):
        """Local map consistency of cloud `which` without a ground truth (me_consistency, world 1): per point MME's radius
        neighbourhood, its entropy and its plane variance (the smallest eigenvalue of the neighbourhood covariance, m^2).
        Returns consistency_dict's dict: 'whole' (mme, mpv, mean_plane_std, max_pv, the counts, and which sweep ran: kernel,
        rings, solo) and one row per occupied region floor(x / region_size) when region_size > 0.  The sweep may lay the cloud
        out again (its NN records are then stale).  Multi-GPU: dist.consistency_distributed."""
        rows = C.c_void_p()
        n = C.c_int64(0)
        whole = A.me_consistency_result()
        self._check(self._L.me_consistency(self._ctx, int(which), float(radius), int(min_neighbors), float(region_size),
                                           C.byref(rows), C.byref(n), C.byref(whole)))
        return consistency_dict(self._take_rows(rows, n.value, _CONS_ROW_DT), whole)

    def consistency_begin(self, which, radius, min_neighbors=10, region_size=0.0):
        """me_consistency_begin: sweeps this rank's query range and folds it by region; returns the row count (0 at
        region_size 0)"""
        n = C.c_int64(0)
        self._check(self._L.me_consistency_begin(self._ctx, int(which), float(radius), int(min_neighbors), float(region_size),
                                                 C.byref(n)))
        return n.value

    def consistency_block(self):
        """(device pointer, n_sum, n_max) of the block: SUM-reduce its first n_sum values and MAX-reduce the next n_max in
        place (after synchronize())"""
        return self._block(self._L.me_consistency_block, C.c_int32, C.c_int32)

    def consistency_end(self, n_regions):
        """the rows and the whole-map result from the reduced block, as local_consistency"""
        rows = np.zeros(max(int(n_regions), 1), _CONS_ROW_DT)
        whole = A.me_consistency_result()
        self._check(self._L.me_consistency_end(self._ctx, rows.ctypes.data_as(C.c_void_p), int(n_regions), C.byref(whole)))
        return consistency_dict(rows[:int(n_regions)], whole)

    def get_consistency_points(self, which):
        """(entropy, plane_variance) per point of the last consistency call on cloud `which`, caller order: 0 / NaN where
        invalid (k < min_neighbors) and at points another rank evaluated"""
        n = self.n[which]
        e = np.zeros(n, np.float64)
        v = np.zeros(n, np.float64)
        self._check(self._L.me_get_consistency_points(self._ctx, int(which), e.ctypes.data_as(C.c_void_p),
                                                      v.ctypes.data_as(C.c_void_p)))
        return e, v

    def mom(self, which, radius, min_neighbors=10, angle_deg=10.0, planarity=0.5, min_family=100):
        """The mutually orthogonal metric of cloud `which` without a ground truth (me_mom, world 1): the plane thickness
        (the median plane variance, m^2) of three mutually orthogonal plane families, summed.  Returns mom_dict's dict:
        'mom' (NaN unless 'status' is 'OK'), 'axis' (3, 3), per family 'n' / 'mean' / 'median', the counts, and which sweep
        ran.  The sweep may lay the cloud out again (its NN records are then stale).  Multi-GPU: dist.mom_distributed."""
        out = A.me_mom_result()
        p = mom_params(angle_deg, planarity, min_family)
        self._check(self._L.me_mom(self._ctx, int(which), float(radius), int(min_neighbors), C.byref(p), C.byref(out)))
        self._mom_min_family_last = out.min_family
        return mom_dict(out)

    def mom_begin(self, which, radius, min_neighbors=10, angle_deg=10.0, planarity=0.5, min_family=100):
        """me_mom_begin: sweeps this rank's query range and histograms its planar normals"""
        p = mom_params(angle_deg, planarity, min_family)
        self._check(self._L.me_mom_begin(self._ctx, int(which), float(radius), int(min_neighbors), C.byref(p)))

    def mom_block(self):
        """(device pointer, n) of the running pass's block: SUM-reduce it in place (after synchronize())"""
        return self._block(self._L.me_mom_block, C.c_int32)

    def mom_step(self):
        """me_mom_step: reads the reduced block, runs the next pass; True after the last"""
        done = C.c_int32(0)
        self._check(self._L.me_mom_step(self._ctx, C.byref(done)))
        return bool(done.value)

    def mom_end(self):
        out = A.me_mom_result()
        self._check(self._L.me_mom_end(self._ctx, C.byref(out)))
        self._mom_min_family_last = out.min_family
        return mom_dict(out)

    def get_mom_points(self, which):
        """(v, lambda2, normal (n, 3), family) per point of the last MOM call on cloud `which`, caller order: NaN / -1
        where invalid and at points another rank evaluated; family 0..2 or -1"""
        n = self.n[which]
        v = np.zeros(n, np.float64)
        l2 = np.zeros(n, np.float64)
        nrm = np.zeros((n, 3), np.float64)
        fam = np.zeros(n, np.int8)
        self._check(self._L.me_get_mom_points(self._ctx, int(which), v.ctypes.data_as(C.c_void_p), l2.ctypes.data_as(C.c_void_p),
                                              nrm.ctypes.data_as(C.c_void_p), fam.ctypes.data_as(C.c_void_p)))
        return v, l2, nrm, fam

    def mom_regions(self, region_size, min_family=None):
        """The last finished MOM call broken down by region floor(x / region_size) (me_mom_regions, world 1), without a new
        sweep: per region the cloud's points, its planar points and, per family of the whole map, the count, mean and exact
        median of v; 'mom' the sum of the medians.  min_family None: the MOM call's.  Returns mom_region_dict's dict.
        Multi-GPU: dist.mom_regions_distributed."""
        rows = C.c_void_p()
        n = C.c_int64(0)
        self._check(self._L.me_mom_regions(self._ctx, float(region_size), self._mom_min_family(min_family), C.byref(rows),
                                           C.byref(n)))
        return mom_region_dict(self._take_rows(rows, n.value, _MOM_REGION_ROW_DT), region_size)

    def _mom_min_family(self, min_family):
        if min_family is not None:
            return int(min_family)
        if self._mom_min_family_last is None:
            raise MapEvalError(A.ME_ERR_INVALID, "mom_regions: min_family=None needs a MOM call on this context first")
        return self._mom_min_family_last

    def mom_region_begin(self, region_size, min_family=None):
        """me_mom_region_begin: writes this rank's points of the last finished MOM call into the block; returns the row count"""
        n = C.c_int64(0)
        self._check(self._L.me_mom_region_begin(self._ctx, float(region_size), self._mom_min_family(min_family), C.byref(n)))
        self._mom_region_size = float(region_size)
        return n.value

    def mom_region_block(self):
        """(device pointer, n) of the block [v | code], 2 n_points fp64 values: SUM-reduce it in place (after synchronize())"""
        return self._block(self._L.me_mom_region_block, C.c_int64)

    def mom_region_end(self, n_regions):
        """the rows from the reduced block, as mom_regions"""
        rows = np.zeros(max(int(n_regions), 1), _MOM_REGION_ROW_DT)
        self._check(self._L.me_mom_region_end(self._ctx, rows.ctypes.data_as(C.c_void_p), int(n_regions)))
        return mom_region_dict(rows[:int(n_regions)], self._mom_region_size)

    def get_nn(self, which_query):
        n = self.n[which_query]
        idx = np.empty(n, np.int32)
        d2 = np.empty(n, np.float64)
        self._check(self._L.me_get_nn(self._ctx, which_query, idx.ctypes.data_as(C.c_void_p),
                                      d2.ctypes.data_as(C.c_void_p)))
        return idx, d2

    # -- a5-a9 -------------------------------------------------------------------------------------------------
    def eval_mme_accum(self, which, radius, min_neighbors):
        acc = A.me_mme_accum()
        self._check(self._L.me_eval_mme_accum(self._ctx, which, float(radius), int(min_neighbors), C.byref(acc)))
        return acc

    def mme_finalize(self, acc, which):
        out = A.me_mme_result()
        rc = self._L.me_mme_finalize(C.byref(acc), self.n[which], C.byref(out))
        if rc != A.ME_OK:
            raise MapEvalError(rc, "me_mme_finalize")
        return out

    def computeMME(self, which, radius, min_neighbors, want_entropies=False):
        """map_eval.cpp:1608-1737 (min_neighbors=10) / :1438-1535 (min_neighbors=5), single GPU."""
        out = A.me_mme_result()
        ent = np.zeros(self.n[which], np.float64) if want_entropies else None
        self._check(self._L.me_eval_mme(self._ctx, which, float(radius), int(min_neighbors), C.byref(out),
                                        ent.ctypes.data_as(C.c_void_p) if want_entropies else None))
        return (out, ent) if want_entropies else out

    def get_entropies(self, which):
        ent = np.zeros(self.n[which], np.float64)
        self._check(self._L.me_get_entropies(self._ctx, which, ent.ctypes.data_as(C.c_void_p)))
        return ent

    # -- a10-a16 -----------------------------------------------------------------------------------------------
    def calculateVMD(self, voxel_size, min_points=100, scs_radius=5, want_rows=False):
        """map_eval.cpp:240-390."""
        out = A.me_awd_result()
        n_rows = C.c_int64(0)
        rows_p = C.POINTER(C.c_double)()
        self._check(self._L.me_eval_awd(self._ctx, float(voxel_size), int(min_points), int(scs_radius), C.byref(out),
                                        C.byref(n_rows), C.byref(rows_p) if want_rows else None))
        if not want_rows:
            return out
        rows = np.ctypeslib.as_array(rows_p, shape=(n_rows.value, 27)).copy() if n_rows.value > 0 \
            else np.zeros((0, 27))
        self._L.me_free(rows_p)
        return out, rows

    def awd_from_rows(self, rows27, voxel_size, scs_radius=5):
        """W per row + AWD / SCS from given voxel Gaussians (27-column voxel_errors.txt rows)."""
        rows = np.ascontiguousarray(rows27, dtype=np.float64)
        assert rows.ndim == 2 and rows.shape[1] == 27
        out = A.me_awd_result()
        w = np.empty(rows.shape[0], np.float64)
        dp = C.POINTER(C.c_double)
        self._check(self._L.me_awd_from_rows(self._ctx, rows.ctypes.data_as(dp), rows.shape[0], float(voxel_size), int(scs_radius),
                                             w.ctypes.data_as(dp), C.byref(out)))
        return out, w

    # -- the Gaussian 2-Wasserstein distance per voxel (DESIGN §3.18) -------------------------------------------------
    def voxel_w2(self, voxel_size, min_points=100, scs_radius=5, want_rows=False):
        """AW2, the mean offset and shape terms, SCS over W2 and the counts (me_w2_result); with want_rows also the
        (n_pairs, 26) rows, columns _abi.W2_ROW_COLUMNS.  Replicated layout (dist.w2_distributed shards it)."""
        out = A.me_w2_result()
        n_rows = C.c_int64(0)
        rows_p = C.POINTER(C.c_double)()
        self._check(self._L.me_eval_w2(self._ctx, float(voxel_size), int(min_points), int(scs_radius), C.byref(out),
                                       C.byref(n_rows), C.byref(rows_p) if want_rows else None))
        if not want_rows:
            return out
        rows = self._take_rows(rows_p, n_rows.value * A.ME_W2_ROW_COLS, np.dtype(np.float64))
        return out, rows.reshape(-1, A.ME_W2_ROW_COLS)

    def w2_from_rows(self, rows, voxel_size, scs_radius=5):
        """(me_w2_result, (n, 3) offset / shape / W2 per row) of given Gaussians in the 26-column layout of voxel_w2's rows"""
        rows = np.ascontiguousarray(rows, dtype=np.float64)
        assert rows.ndim == 2 and rows.shape[1] == A.ME_W2_ROW_COLS
        out = A.me_w2_result()
        w = np.empty((rows.shape[0], 3), np.float64)
        dp = C.POINTER(C.c_double)
        self._check(self._L.me_w2_from_rows(self._ctx, rows.ctypes.data_as(dp), rows.shape[0], float(voxel_size), int(scs_radius),
                                            w.ctypes.data_as(dp), C.byref(out)))
        return out, w

    def w2_begin(self, voxel_size, min_points=100):
        self._check(self._L.me_w2_begin(self._ctx, float(voxel_size), int(min_points)))

    def w2_w_table(self):
        """(device pointer, n) of the W2 table over the estimated cloud's voxels (-1 = no pair on a slab layout)"""
        return self._block(self._L.me_w2_w_table, C.c_int64)

    def w2_finish_accum_device(self, scs_radius=5):
        self._check(self._L.me_w2_finish_accum_device(self._ctx, int(scs_radius)))

    def w2_block(self):
        """(device pointer, n) of the stage's block: SUM-reduce all n values in place"""
        return self._block(self._L.me_w2_block, C.c_int32)

    def w2_fetch(self):
        out = A.me_w2_result()
        self._check(self._L.me_w2_fetch(self._ctx, C.byref(out)))
        return out

    # -- device-resident accumulators (multi-GPU passes without host round trips) ---------------------------------
    def accum_reset(self):
        self._check(self._L.me_accum_reset(self._ctx))

    def eval_nn_accum_device(self, params):
        self._check(self._L.me_eval_nn_accum_device(self._ctx, C.byref(params)))

    def eval_mme_accum_device(self, which, radius, min_neighbors):
        self._check(self._L.me_eval_mme_accum_device(self._ctx, which, float(radius), int(min_neighbors)))

    def accum_block(self):
        """(device pointer, n_sum, n_max) of the fp64 accumulator block"""
        return self._block(self._L.me_accum_block, C.c_int32, C.c_int32)

    def accum_fetch(self, want_mme=(True, False)):
        e, g = A.me_nn_accum(), A.me_nn_accum()
        mm = [A.me_mme_accum() if w else None for w in want_mme]
        self._check(self._L.me_accum_fetch(self._ctx, C.byref(e), C.byref(g), C.byref(mm[0]) if mm[0] else None,
                                           C.byref(mm[1]) if mm[1] else None))
        return e, g, [m for m in mm if m is not None]

    # -- layouts of a multi-GPU job; the voxel stage in two halves ------------------------------------------------
    def set_layout(self, layout):
        """A.ME_LAYOUT_REPLICATED (default) or A.ME_LAYOUT_SLAB: every rank lays out only the voxel layers it owns."""
        self._check(self._L.me_set_layout(self._ctx, int(layout)))

    def layout_active(self):
        """{'layout', 'axis', 'n_laid_out': [est, gt], 'n_owned': [est, gt]} once the lattices are built"""
        lay, ax = C.c_int32(0), C.c_int32(0)
        nl, no = (C.c_int64 * 2)(), (C.c_int64 * 2)()
        self._check(self._L.me_layout_active(self._ctx, C.byref(lay), C.byref(ax), nl, no))
        return {"layout": lay.value, "axis": ax.value, "n_laid_out": list(nl), "n_owned": list(no)}

    def voxel_begin(self, voxel_size, min_points=100):
        self._check(self._L.me_voxel_begin(self._ctx, float(voxel_size), int(min_points)))

    def voxel_w_table(self):
        """(device pointer, n) of the W table over the estimated cloud's voxels (-1 = no pair)"""
        return self._block(self._L.me_voxel_w_table, C.c_int64)

    def voxel_finish_accum_device(self, scs_radius=5):
        self._check(self._L.me_voxel_finish_accum_device(self._ctx, int(scs_radius)))

    def accum_fetch_awd(self):
        out = A.me_awd_result()
        self._check(self._L.me_accum_fetch_awd(self._ctx, C.byref(out)))
        return out

    # -- introspection -----------------------------------------------------------------------------------------
    def stage_times_ms(self):
        ms = (C.c_double * A.ME_N_STAGE_TIMES)()
        self._check(self._L.me_get_stage_times(self._ctx, ms))
        return dict(zip(A.STAGE_NAMES, list(ms)))

    def launch_count(self):
        return int(self._L.me_launch_count(self._ctx))

    def kernel_trace(self, reset=True, events=False):
        """(set of ME_KBIT_* names of the sweep paths run since creation or the last reset — with events=True also the
        ME_TEV_* names of the data events —, (CAP, U) of the last mme_rows_kernel or None)"""
        mask, cfg = C.c_uint64(0), C.c_int32(0)
        self._check(self._L.me_kernel_trace(self._ctx, C.byref(mask), C.byref(cfg), 1 if reset else 0))
        names = A.kernel_bit_names(mask.value) | (A.trace_event_names(mask.value) if events else set())
        return names, ((cfg.value >> 8, cfg.value & 255) if cfg.value else None)

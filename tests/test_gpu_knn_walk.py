"""The exact k-NN walk (knn_walk.cuh) on the device at every neighbour count it serves: knn_normals_kernel against the exact
normal bounds (tests/exact_reg.py) at k = 1..64 on the tie-cut scenes of tests/test_knn_walk_reference.py, on both cell
tables and 1.5 km out; the shared-memory opt-in above k = 32; the handover to the coarse blocks (ME_TEV_KNN_COARSE); the
grid-stride loop; the gathered slices and the working normals of surface_metrics; and the FPFH neighbourhoods of
global_registration against tests/fpfh_ref.py at max_nn 1..128, on the radius and past it."""

import numpy as np
import pytest

import exact_reg as X
import fpfh_ref as R
from cloud_map_evaluation_b200 import _abi as A

from test_exact_reg import FAR, normal_scenes
from test_knn_walk_reference import (FEAT_MAX_NN, FEAT_RADIUS, FEAT_V, KS, ON_RADIUS, SCENES, TIE_CUT, central, fpfh_stairs,
                                     fpfh_tolerance, stairs)

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
SPARSE = 1                          # max_grid_cells: a budget of one cell forces the sparse cell table
COARSE = "ME_TEV_KNN_COARSE"
N_TIE = 120                         # tie-cut queries checked per (scene, k), besides the central ones
N_NORMAL_SCENE = 24                 # queries per normal_scenes() scene and k
NORMAL_SCENES = normal_scenes()


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _normals(api, pts, k, max_grid_cells=0, nn_cell_size=0.0, trace=False):
    with api.MapEvalB200(max_grid_cells=max_grid_cells, nn_cell_size=nn_cell_size) as c:
        c.set_cloud(EST, pts)
        c.set_cloud(GT, pts[:8])
        c.kernel_trace(reset=True)
        got = c.estimate_normals(EST, k)
        return (got, c.kernel_trace(events=True)[0]) if trace else got


def _check(name, rows, got):
    bad = [(r["q"], X.check_normal(r, got[r["q"]])["why"]) for r in rows if not X.check_normal(r, got[r["q"]])["ok"]]
    assert not bad, (name, len(bad), bad[:5])


# ---------------------------------------------------------------------------------------------------------------
# normals against exact arithmetic at every k
# ---------------------------------------------------------------------------------------------------------------
def tie_queries(pts, k, n=N_TIE, seed=0):
    """the points whose slot k and slot k + 1 tie (where the k-th choice matters), at most n of them by a fixed seed"""
    nb = X.knn_exact(pts, np.arange(len(pts)), k + 1)
    t = np.array([len(b) > k and X.d2_kd(pts[i], pts[b[k - 1]]) == X.d2_kd(pts[i], pts[b[k]]) for i, b in enumerate(nb)])
    idx = np.flatnonzero(t)
    if len(idx) > n:
        idx = np.sort(np.random.RandomState(seed + k).choice(idx, n, replace=False))
    return idx


_ROWS = {}


def _rows(name, k):
    """exact rows once per (scene, k), shared by both tables and both origins (a dyadic lattice moved by FAR keeps every
    offset, distance and covariance: the rows are the same)"""
    if (name, k) not in _ROWS:
        if name in SCENES:
            pts = SCENES[name]
            ties = tie_queries(pts, k)
            if k in TIE_CUT[name]:
                assert len(ties) >= 16, (name, k, len(ties))
            q = np.union1d(central(pts, 40), ties)
        else:
            pts = NORMAL_SCENES[name]
            q = np.random.RandomState(k).choice(len(pts), min(N_NORMAL_SCENE, len(pts)), replace=False)
        _ROWS[name, k] = X.normals_exact(pts, q, k=k)
    return _ROWS[name, k]


@pytest.mark.parametrize("k", KS)
def test_normals_at_every_k(api, k):
    tables = [("dense", 0), ("sparse", SPARSE)]
    for name, pts in SCENES.items():
        rows = _rows(name, k)
        for origin in (0.0, FAR):
            for table, cells in tables:
                _check((name, table, "far" if origin is FAR else "origin", k), rows, _normals(api, pts + origin, k, cells))
    for name, pts in sorted(NORMAL_SCENES.items()):
        rows = _rows(name, k)
        for table, cells in tables:
            _check((name, table, k), rows, _normals(api, pts, k, cells))


# ---------------------------------------------------------------------------------------------------------------
# the shared-memory boundary: k <= 32 runs in the default 48 KiB, k >= 33 (and n < k clamped to n) opts in
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [32, 33], ids=["k32_default_smem", "k33_opt_in"])
def test_shared_memory_boundary(api, k):
    for name in ("stairs", "cubic"):
        pts = SCENES[name]
        rows = X.normals_exact(pts, k=k)                     # every point
        _check((name, k), rows, _normals(api, pts, k))


def test_fewer_points_than_k(api):
    """n = 40 at k = 64: the kernel clamps k to 40 and opts in at 40 * 1536 B"""
    pts = stairs(5, 8, seed=3)
    assert len(pts) == 40
    rows = X.normals_exact(pts, k=64)
    assert all(len(r["nb"]) == 40 for r in rows)
    _check("n40", rows, _normals(api, pts, 64))
    _check("n40_sparse", rows, _normals(api, pts, 64, SPARSE))


# ---------------------------------------------------------------------------------------------------------------
# the coarse handover
# ---------------------------------------------------------------------------------------------------------------
WIRE_N = 100_000
WIRE_A = 0.0625                     # spacing along x = the lattice cell edge: about one point per cell
WIRE_END = 100                      # queries this close to an end have neighbourhoods of their own


def wire(n=WIRE_N):
    """a thin wire along x in caller order: x = i a, a cross-section that cycles through the corners of a 1/64 x 1/32 m
    rectangle with period 4.  Its lattice at cell edge a has 10^5 cells along x and a coarse grid; 8 fine rings hold 17
    points, fewer than every k checked here, so every query goes on to the coarse blocks with a partial list.  Away from
    the ends a query's neighbourhood is its class's (i mod 4) moved along x by a multiple of 4a, exactly, and the order of
    the indices is the same, so the device must give every query of a class the same bits."""
    i = np.arange(n)
    yz = np.array([[0.0, 0.0], [1 / 64, 0.0], [1 / 64, 1 / 32], [0.0, 1 / 32]])[i % 4]
    return np.c_[i * WIRE_A, yz]


def outliers(seed=11):
    """a flat cluster with isolated points tens of metres away (test_gpu_exact_reg's big_outliers, smaller)"""
    rs = np.random.RandomState(seed)
    return np.concatenate([rs.randn(20_000, 3) * [2.0, 2.0, 0.01], rs.rand(200, 3) * 80.0 - 40.0])


@pytest.mark.parametrize("k", [20, 33, 64])
def test_coarse_handover_wire(api, k):
    pts = wire()
    got, trace = _normals(api, pts, k, nn_cell_size=WIRE_A, trace=True)
    assert COARSE in trace
    ends = np.r_[np.arange(WIRE_END), np.arange(WIRE_N - WIRE_END, WIRE_N)]
    _check(("wire ends", k), X.normals_exact(pts, ends, k=k), got)
    inner = np.arange(WIRE_END, WIRE_N - WIRE_END)
    for r in range(4):
        cls = inner[inner % 4 == r]
        distinct = np.unique(got[cls], axis=0)
        assert len(distinct) == 1, (k, r, len(distinct))
        _check(("wire class", k, r), X.normals_exact(pts, [cls[0]], k=k), got)


@pytest.mark.parametrize("k", [20, 33, 64])
def test_coarse_handover_outliers(api, k):
    pts = outliers()
    q = np.union1d(np.random.RandomState(2).choice(20_000, 200, replace=False), np.arange(20_000, len(pts)))
    rows = X.normals_exact(pts, q, k=k)
    for table, cells in (("dense", 0), ("sparse", SPARSE)):
        got, trace = _normals(api, pts, k, cells, trace=True)
        assert COARSE in trace
        _check(("outliers", table, k), rows, got)


# ---------------------------------------------------------------------------------------------------------------
# the grid-stride loop (beyond sm_count * 32 blocks of 128 queries); the same surface must not raise the coarse event
# ---------------------------------------------------------------------------------------------------------------
def big_plane(n, seed=5):
    rs = np.random.RandomState(seed)
    uv = rs.rand(n, 2) * 100.0
    c, s = np.cos(0.3), np.sin(0.3)
    p = np.stack([uv[:, 0], uv[:, 1], 1e-3 * rs.randn(n)], 1)
    return p @ np.array([[1.0, 0.0, 0.0], [0.0, c, -s], [0.0, s, c]]).T


def test_grid_stride(api):
    import torch
    limit = torch.cuda.get_device_properties(0).multi_processor_count * 32 * 128
    pts = big_plane(int(limit * 1.1) + 1)
    q = np.sort(np.random.RandomState(7).choice(len(pts), 2000, replace=False))
    for k in (20, 64):
        got, trace = _normals(api, pts, k, trace=True)
        if k == 20:
            assert COARSE not in trace                      # a surface resolves in the fine rings
        _check(("grid stride", k), X.normals_exact(pts, q, k=k), got)


# ---------------------------------------------------------------------------------------------------------------
# gathered slices and working normals at k in {1, 3, 33, 64}
# ---------------------------------------------------------------------------------------------------------------
SLICE_KS = [1, 3, 33, 64]


def _pair():
    est = stairs(60, 40, seed=1)
    gt = stairs(60, 40, seed=2) + [0.01, -0.02, 0.005]
    return est, gt


@pytest.mark.parametrize("k", SLICE_KS)
def test_surface_slices_and_working_normals(api, k):
    """the gathered surface_normals_slice of worlds 2 and 3 equal world 1's normals bit for bit, and surface_metrics(knn=k)
    on one layout gives the block of the same call after estimate_normals(k) on both clouds (icp_normals_slice always
    estimates at k = 20: test_gpu_exact_reg.py)"""
    from test_gpu_surface_metrics import _bits, _ctx, _run, _sharded
    est, gt = _pair()
    p = A.make_nn_params([0.2, 0.1, 0.05, 0.02, 0.01], 1.0, pairing=A.ME_PAIRING_GEOMETRIC)
    with _ctx(api, est, gt) as ctx:
        ctx.calculateMetricsWithInitialMatrix(p)
        blk, _ = _run(ctx, knn=k)
        n1 = (ctx.estimate_normals(EST, k), ctx.estimate_normals(GT, k))
        np.testing.assert_array_equal(_bits(_run(ctx)[0]), _bits(blk))
    for world in (2, 3):
        _, gathered = _sharded(api, est, gt, p, world, False, k)
        assert len(gathered) == 2
        for g, n in zip(gathered, n1):
            np.testing.assert_array_equal(_bits(g), _bits(n))


# ---------------------------------------------------------------------------------------------------------------
# FPFH neighbourhoods of global_registration
# ---------------------------------------------------------------------------------------------------------------
def _features(api, est, gt, **kw):
    """get_features of both clouds after global_registration (RANSAC may refuse: the features stay valid), and the
    kernel trace"""
    with api.MapEvalB200(device=0) as ctx:
        ctx.set_cloud(EST, est)
        ctx.set_cloud(GT, gt)
        ctx.kernel_trace(reset=True)
        try:
            ctx.global_registration(FEAT_V, seed=3, n_hypotheses=64, **kw)
        except api.MapEvalError:
            pass
        return [ctx.get_features(w) for w in (EST, GT)], ctx.kernel_trace(events=True)[0]


def _check_fpfh(xyz, nrm, f, radius, max_nn, sample=None):
    """f against the statement as test_fpfh compares, from the device's oriented normals; returns the neighbourhoods'
    sizes"""
    if sample is None:
        f32, f64, flagged, nb = R.features(xyz, nrm, radius, max_nn)
        got = f
    else:
        f32, f64, flagged = R.fpfh_sample(xyz, nrm, radius, max_nn, sample)
        nb = R.hybrid_neighbours(xyz, radius, max_nn, sample)
        got = f[sample]
    ok = ~flagged
    assert flagged.sum() <= max(2, len(flagged) // 200), flagged.sum()
    err = np.abs(got[ok].astype(np.float64) - f64[ok])
    assert (err <= fpfh_tolerance(f64[ok])).all(), (radius, max_nn, int((err > fpfh_tolerance(f64[ok])).sum()))
    return np.array([len(i) for i, _ in nb])


@pytest.fixture(scope="module")
def feature_scene():
    xyz = fpfh_stairs()
    return xyz, xyz[xyz[:, 0] < 0.5 * (xyz[:, 0].min() + xyz[:, 0].max())].copy()      # gt, and est = its lower half


@pytest.mark.parametrize("max_nn", FEAT_MAX_NN)
def test_fpfh_max_nn(api, feature_scene, max_nn):
    gt, est = feature_scene
    feats, _ = _features(api, est, gt, feature_radius=FEAT_RADIUS, feature_max_nn=max_nn)
    for xyz, nrm, f in feats:
        cnt = _check_fpfh(xyz, nrm, f, FEAT_RADIUS, max_nn)
        assert cnt.max() == max_nn


def test_fpfh_on_the_radius(api, feature_scene):
    """feature_radius = 2 v: the points at exactly 2 v are out; one double up they are in"""
    gt, est = feature_scene
    counts = []
    for radius in (ON_RADIUS, float(np.nextafter(ON_RADIUS, np.inf))):
        feats, _ = _features(api, est, gt, feature_radius=radius, feature_max_nn=128)
        xyz, nrm, f = feats[1]
        counts.append(_check_fpfh(xyz, nrm, f, radius, 128))
    assert counts[1].sum() > counts[0].sum()


@pytest.mark.parametrize("knn", [3, 32, 33, 64])
def test_fpfh_normal_knn(api, feature_scene, knn):
    gt, est = feature_scene
    feats, _ = _features(api, est, gt, normal_knn=knn, feature_radius=FEAT_RADIUS, feature_max_nn=64)
    for w, (xyz, nrm, f) in zip((EST, GT), feats):
        with api.MapEvalB200(device=0) as c2:
            c2.set_cloud(w, xyz)
            plain = c2.estimate_normals(w, knn)
        oriented, amb = R.orient_normals(xyz, plain)
        # the staircase's centroid lies on a lattice column: at k = 3 that column's normals are horizontal along x, and
        # their orientation is a rounding of the centroid away (excluded, counted; either sign of the estimate)
        assert amb.sum() <= (64 if knn == 3 else 0), amb.sum()
        np.testing.assert_array_equal(nrm[~amb], oriented[~amb])
        assert all(n.tolist() in (p.tolist(), (-p).tolist()) for n, p in zip(nrm[amb], plain[amb]))
        q = np.random.RandomState(knn).choice(len(xyz), 100, replace=False)
        _check(("feature normals", knn), X.normals_exact(xyz, q, k=knn), plain)
        _check_fpfh(xyz, nrm, f, FEAT_RADIUS, 64)


def test_fpfh_grid_stride(api):
    """a gt feature cloud above sm_count * 32 blocks of 64 points, a small est cloud; a sample against the statement"""
    import torch
    limit = torch.cuda.get_device_properties(0).multi_processor_count * 32 * 64
    ny = 512
    nx = -(-int(limit * 1.1) // ny)
    gt = fpfh_stairs(nx, ny, seed=9)
    est = fpfh_stairs(40, 32, seed=10)
    feats, _ = _features(api, est, gt, feature_radius=3 * FEAT_V, feature_max_nn=20)
    xyz, nrm, f = feats[1]
    assert len(xyz) > limit
    s = np.sort(np.random.RandomState(4).choice(len(xyz), 2000, replace=False))
    _check_fpfh(xyz, nrm, f, 3 * FEAT_V, 20, sample=s)

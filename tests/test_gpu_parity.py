"""GPU parity: the sm_90a path (through the C-ABI) against the CPU oracle on the same seeded inputs.

Bar (BASELINE.json north_star): integer counts bit-exact; AC/COM/CD/MME/AWD/SCS within 1e-5 relative.
The tests assert a much tighter RTOL (fp64 arithmetic on both sides; only summation order differs)."""
import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import synth

pytestmark = pytest.mark.gpu

RTOL_BAR = 1e-5     # the stated bar
RTOL = 1e-9         # what we actually hold where both sides run fp64 arithmetic (only summation order differs)
# MME: neighbours are screened on cell-relative fp32 offsets (exact fp64 decision inside the error band, so counts stay
# bit-exact) and the accepted fp32 offsets (abs. error ~1e-6 cell edges) are accumulated in fp64
RTOL_MME = 1e-7     # mean map entropy
RTOL_ENT = 1e-6     # per-point entropies


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _ctx(api, est, gt, **kw):
    ctx = api.MapEvalB200(**kw)
    ctx.set_cloud(A.ME_CLOUD_EST, est)
    ctx.set_cloud(A.ME_CLOUD_GT, gt)
    return ctx


def _cmp_dir(got, exp):
    assert got.n_source == exp.n_source
    assert got.n_corr == exp.n_corr
    assert list(got.n_inlier) == list(exp.n_inlier)
    assert got.n_ub == exp.n_ub
    for k in ("mean", "rmse", "fitness", "sigma"):
        np.testing.assert_allclose(list(getattr(got, k)), list(getattr(exp, k)), rtol=RTOL, atol=1e-300, err_msg=k)
    np.testing.assert_allclose(got.sum_nn_dist, exp.sum_nn_dist, rtol=RTOL)


def _cmp_nn(got, exp):
    _cmp_dir(got.est_to_gt, exp.est_to_gt)
    _cmp_dir(got.gt_to_est, exp.gt_to_est)
    for k in ("cd", "f1", "iou"):
        np.testing.assert_allclose(list(getattr(got, k)), list(getattr(exp, k)), rtol=RTOL, equal_nan=True, err_msg=k)
    np.testing.assert_allclose(got.full_cd, exp.full_cd, rtol=RTOL)


@pytest.mark.parametrize("pairing", [A.ME_PAIRING_AS_WRITTEN, A.ME_PAIRING_GEOMETRIC])
@pytest.mark.parametrize("cutoff", [A.ME_CUTOFF_SQDIST_LE_R, A.ME_CUTOFF_DIST_LT_R])
def test_nn_c1_config(api, O, pairing, cutoff):
    """BASELINE config C1: 100k vs 100k uniform box, AC + CD."""
    est, gt, cfg = synth.make_pair("C1")
    p = A.make_nn_params(cfg["tau"], 1.0, cutoff_mode=cutoff, pairing=pairing)
    with _ctx(api, est, gt) as ctx:
        got = ctx.calculateMetricsWithInitialMatrix(p)
        idx_e, d2_e = ctx.get_nn(A.ME_CLOUD_EST)
        idx_g, d2_g = ctx.get_nn(A.ME_CLOUD_GT)
    exp, ie, ig = O.eval_nn(est, gt, p, want_indices=True)
    _cmp_nn(got, exp)
    np.testing.assert_array_equal(idx_e, ie)
    np.testing.assert_array_equal(idx_g, ig)
    oi, od2 = O.knn1(est, gt)
    np.testing.assert_array_equal(d2_e, od2)      # squared distances are bit-identical


def test_nn_small_cutoff_and_unequal_sizes(api, O):
    side = synth.box_side_for_density(60000)
    gt = synth.uniform_box(60000, side, 11)
    est = synth.uniform_box(83211, side, 12, noise_sigma=0.02)
    for pairing in (A.ME_PAIRING_AS_WRITTEN, A.ME_PAIRING_GEOMETRIC):
        p = A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], 0.0009, pairing=pairing)   # sqrt(R) = 0.03 m
        with _ctx(api, est, gt) as ctx:
            got = ctx.calculateMetricsWithInitialMatrix(p)
        exp = O.eval_nn(est, gt, p)
        assert 0 < exp.est_to_gt.n_corr < len(est)
        _cmp_nn(got, exp)
    # as-written pairing with more est than gt points hits the reference's out-of-range lookups
    p = A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], 1.0, pairing=A.ME_PAIRING_AS_WRITTEN)
    with _ctx(api, gt, est) as ctx:   # swap roles: n_est < n_gt -> i_gt can exceed n_est
        got = ctx.calculateMetricsWithInitialMatrix(p)
    exp = O.eval_nn(gt, est, p)
    assert exp.gt_to_est.n_ub > 0
    _cmp_nn(got, exp)


def test_nn_far_queries_clusters_and_outliers(api, O):
    """Queries far from every reference point (ring-expansion kernel), clustered references, duplicates."""
    rng = np.random.RandomState(5)
    gt = np.concatenate([rng.randn(20000, 3) * 0.3 + c for c in ([0, 0, 0], [6, 1, -2], [-3, 8, 1])])
    gt = np.concatenate([gt, gt[:100]])                         # duplicated reference points
    est = np.concatenate([gt[::3] + rng.randn(len(gt[::3]), 3) * 0.01,
                          rng.rand(3000, 3) * 40 - 20,          # outliers up to ~20 m away
                          gt[:50]])                              # exact coincidences (d = 0)
    est = est.astype(np.float32).astype(np.float64)
    gt = gt.astype(np.float32).astype(np.float64)
    p = A.make_nn_params([0.5, 0.3, 0.2, 0.1, 0.05], 1.0, pairing=A.ME_PAIRING_GEOMETRIC)
    with _ctx(api, est, gt) as ctx:
        e, g = ctx.eval_nn_accum(p)
        got = ctx.nn_finalize(p, e, g)
        idx_e, d2_e = ctx.get_nn(A.ME_CLOUD_EST)
        # the ground truth's lattice stays below 257 cells per axis here, so the far kernel has no coarse-block phase to
        # enter; tests/test_gpu_kernel_paths.py ("clusters") reaches it
        assert "ME_KBIT_NN_FAR" in ctx.kernel_trace()[0]
    assert e.n_far > 1000
    exp = O.eval_nn(est, gt, p)
    _cmp_nn(got, exp)
    oi, od2 = O.knn1(est, gt)
    np.testing.assert_array_equal(d2_e, od2)
    np.testing.assert_array_equal(idx_e, oi)


def test_nn_without_full_cd_stops_at_cutoff(api, O):
    est, gt, cfg = synth.make_pair("C1", scale=0.3)
    est = np.concatenate([est, est[:500] + 30.0])               # far outliers that need no exact NN
    p = A.make_nn_params(cfg["tau"], 0.04, want_full_cd=False, pairing=A.ME_PAIRING_GEOMETRIC)
    with _ctx(api, est, gt) as ctx:
        got = ctx.calculateMetricsWithInitialMatrix(p)
    exp = O.eval_nn(est, gt, p)
    assert got.full_cd == 0.0 and exp.full_cd == 0.0
    for d in ("est_to_gt", "gt_to_est"):
        a, b = getattr(got, d), getattr(exp, d)
        assert a.n_corr == b.n_corr and list(a.n_inlier) == list(b.n_inlier)
        np.testing.assert_allclose(list(a.rmse), list(b.rmse), rtol=RTOL)


def test_transform_then_nn(api, O):
    est, gt, cfg = synth.make_pair("C1", scale=0.2)
    th = 0.01
    T = np.array([[np.cos(th), -np.sin(th), 0, 0.02], [np.sin(th), np.cos(th), 0, -0.01], [0, 0, 1, 0.005], [0, 0, 0, 1]])
    p = A.make_nn_params(cfg["tau"], 1.0, pairing=A.ME_PAIRING_GEOMETRIC)
    with _ctx(api, est, gt) as ctx:
        ctx.transform(A.ME_CLOUD_EST, T)                       # map_3d_->Transform(initial_matrix), map_eval.cpp:1206
        got = ctx.calculateMetricsWithInitialMatrix(p)
    exp = O.eval_nn(O.transform(est, T), gt, p)
    _cmp_nn(got, exp)


@pytest.mark.parametrize("min_neighbors", [10, 5])
def test_mme_parity(api, O, min_neighbors):
    est, gt, cfg = synth.make_pair("C2", scale=0.2)             # 200k points, r = 0.1 m
    with _ctx(api, est, gt) as ctx:
        got, ent = ctx.computeMME(A.ME_CLOUD_EST, cfg["nn_radius"], min_neighbors, want_entropies=True)
    exp, oent = O.eval_mme(est, cfg["nn_radius"], min_neighbors, want_entropies=True)
    assert got.n_valid == exp.n_valid and got.n_total == exp.n_total
    np.testing.assert_array_equal(ent != 0, oent != 0)
    np.testing.assert_allclose(ent, oent, rtol=RTOL_ENT, atol=0)
    np.testing.assert_allclose(got.mme, exp.mme, rtol=RTOL_MME)
    np.testing.assert_allclose(got.min_abs_entropy, exp.min_abs_entropy, rtol=RTOL_ENT)
    np.testing.assert_allclose(got.max_abs_entropy, exp.max_abs_entropy, rtol=RTOL_ENT)


@pytest.mark.parametrize("shared_lattice", [True, False])
@pytest.mark.parametrize("cells_per_radius", [1.0, 1.7, 2.6, 4.5, 11.3, 19.0])
def test_mme_radius_to_cell_ratios(api, O, cells_per_radius, shared_lattice):
    """On the shared lattice rings = 1, 2, 3 take the flat kernel (templated on the ring count), 5 and 12 rings the plane
    kernel, 19 rings the generic fp64 row walk.  By default a radius spanning more than 3 cells makes the sweep lay the
    cloud out on a lattice of its own (h = r/2); the NN sweep afterwards goes back to the shared lattice."""
    import os
    est, gt, cfg = synth.make_pair("C2", scale=0.05)
    r = cfg["nn_radius"]
    p = A.make_nn_params(cfg["tau"], 1.0, pairing=A.ME_PAIRING_GEOMETRIC)
    if shared_lattice:
        os.environ["ME_MME_SHARED_LATTICE"] = "1"
    rings = int(np.ceil(cells_per_radius - 1e-9))
    table = "SPARSE" if os.environ.get("ME_FORCE_SPARSE") else "DENSE"
    if rings <= 3:
        kernels = {f"ME_KBIT_MME_FLAT{rings}_{table}"}
    elif not shared_lattice:
        kernels = {"ME_KBIT_MME_SOLO", f"ME_KBIT_MME_FLAT2_{table}"}      # h = r / 2 on the cloud's own lattice
    else:
        kernels = {"ME_KBIT_MME_PLANE" if rings <= 15 else "ME_KBIT_MME_GENERIC"}
    try:
        with _ctx(api, est, gt, nn_cell_size=r / cells_per_radius) as ctx:
            got = ctx.computeMME(A.ME_CLOUD_EST, r, 10)
            assert ctx.kernel_trace()[0] == kernels
            nn = ctx.calculateMetricsWithInitialMatrix(p)
            ent = ctx.get_entropies(A.ME_CLOUD_EST)       # after the NN stage re-laid the cloud out
    finally:
        os.environ.pop("ME_MME_SHARED_LATTICE", None)
    exp, oent = O.eval_mme(est, r, 10, want_entropies=True)
    assert got.n_valid == exp.n_valid
    np.testing.assert_array_equal(ent != 0, oent != 0)
    np.testing.assert_allclose(ent, oent, rtol=RTOL_ENT, atol=0)
    np.testing.assert_allclose(got.mme, exp.mme, rtol=RTOL_MME)
    _cmp_nn(nn, O.eval_nn(est, gt, p))


def test_mme_neighbours_exactly_on_the_radius(api, O):
    """A regular lattice with spacing r/2 (fp32 coordinates): thousands of pairs sit exactly at, or one rounding away
    from, d2 == r2.  nanoflann keeps d2 < r2 (strict): the fp32 screen must hand every such pair to the exact fp64 test,
    so the neighbour counts (k >= 10 validity) match the CPU path bit for bit.  Large offsets stress the band too."""
    s = np.float32(0.05)
    g = np.arange(24, dtype=np.float32) * s
    pts = np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3)
    rng = np.random.RandomState(5)
    pts = pts + (rng.rand(*pts.shape) < 0.3) * rng.normal(0, 1e-7, pts.shape).astype(np.float32)   # some a hair off
    for origin in ((0.0, 0.0, 0.0), (-731.25, 1203.5, 88.125)):
        est = np.ascontiguousarray((pts + np.array(origin, dtype=np.float32)).astype(np.float32).astype(np.float64))
        r = float(np.float64(np.float32(0.1)))
        for cell in (0.05, 0.0617):
            with _ctx(api, est, est[:10], nn_cell_size=cell) as ctx:
                got, ent = ctx.computeMME(A.ME_CLOUD_EST, r, 10, want_entropies=True)
            exp, oent = O.eval_mme(est, r, 10, want_entropies=True)
            assert got.n_valid == exp.n_valid, (origin, cell)
            np.testing.assert_array_equal(ent != 0, oent != 0)
            # exact lattices give (near-)singular covariances for boundary points; compare where well conditioned
            ok = oent > -30
            np.testing.assert_allclose(ent[ok], oent[ok], rtol=1e-5, atol=0)


def test_mme_sparse_and_large_radius(api, O):
    """Radius spanning many lattice cells, surface-like data, points with too few neighbours."""
    est = synth.outdoor_scene(120000, 77, 0.01)
    with _ctx(api, est, est[:10]) as ctx:
        got, ent = ctx.computeMME(A.ME_CLOUD_EST, 0.6, 10, want_entropies=True)
    exp, oent = O.eval_mme(est, 0.6, 10, want_entropies=True)
    assert got.n_valid == exp.n_valid
    assert 0 < exp.n_valid < len(est)
    np.testing.assert_array_equal(ent != 0, oent != 0)
    np.testing.assert_allclose(ent, oent, rtol=RTOL_ENT, atol=0)
    np.testing.assert_allclose(got.mme, exp.mme, rtol=RTOL_MME)


def test_nn_ties_and_lattice_points(api, O):
    """Both clouds on regular lattices (fp32 coordinates, large world offset): many exactly equidistant candidates.
    The fp32 screen must pass every near-tie to the fp64 arg-min, whose ties go to the smaller caller index."""
    s = np.float32(0.04)
    g = np.arange(20, dtype=np.float32) * s
    a = np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3)
    off = np.array((512.5, -2048.25, 33.0), dtype=np.float32)
    gt = np.ascontiguousarray((a + off).astype(np.float32).astype(np.float64))
    est = np.ascontiguousarray((a + off + np.float32(0.02)).astype(np.float32).astype(np.float64))   # cell centres: 8-way ties
    est = np.concatenate([est, gt[::7]])                                                       # and exact coincidences
    p = A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], 1.0, pairing=A.ME_PAIRING_GEOMETRIC)
    for cell in (0.0, 0.04, 0.1):
        with _ctx(api, est, gt, nn_cell_size=cell) as ctx:
            got = ctx.calculateMetricsWithInitialMatrix(p)
            idx, d2 = ctx.get_nn(A.ME_CLOUD_EST)
        oidx, od2 = O.knn1(est, gt)
        np.testing.assert_array_equal(d2, od2)
        np.testing.assert_array_equal(idx, oidx)
        _cmp_nn(got, O.eval_nn(est, gt, p))


def _sorted_rows(rows, v):
    keys = np.rint(rows[:, 0:3] / v).astype(np.int64)
    order = np.lexsort((keys[:, 2], keys[:, 1], keys[:, 0]))
    return rows[order]


@pytest.mark.parametrize("hint", [True, False])
def test_awd_scs_parity(api, O, hint):
    est, gt, cfg = synth.make_pair("C2", scale=0.3)             # 300k points, v = 0.25 m (~195 pts / voxel)
    v = cfg["vmd_voxel_size"]
    kw = dict(vmd_voxel_size=v) if hint else {}
    with _ctx(api, est, gt, **kw) as ctx:
        if not hint:   # lattice first laid out without knowing v, then re-laid by calculateVMD
            ctx.calculateMetricsWithInitialMatrix(A.make_nn_params(cfg["tau"], 1.0))
        got, rows = ctx.calculateVMD(v, 100, 5, want_rows=True)
    exp, orows = O.eval_awd(est, gt, v, 100, 5, want_rows=True)
    for k in ("n_pairs", "n_scs", "n_voxels_est", "n_voxels_gt", "n_active", "n_old", "n_new"):
        assert getattr(got, k) == getattr(exp, k), k
    assert got.n_pairs > 100
    np.testing.assert_allclose(got.awd, exp.awd, rtol=RTOL)
    np.testing.assert_allclose(got.scs, exp.scs, rtol=RTOL)
    a, b = _sorted_rows(rows, v), _sorted_rows(orows, v)
    np.testing.assert_array_equal(a[:, [0, 1, 2, 3, 4, 5, 10, 11]], b[:, [0, 1, 2, 3, 4, 5, 10, 11]])
    np.testing.assert_allclose(a[:, 6:9], b[:, 6:9], rtol=1e-12)            # mu_est
    np.testing.assert_allclose(a[:, 18:21], b[:, 18:21], rtol=1e-12)        # mu_gt
    np.testing.assert_allclose(a[:, 9], b[:, 9], rtol=1e-8)                 # W
    np.testing.assert_allclose(a[:, 12:18], b[:, 12:18], rtol=1e-7, atol=1e-16)
    np.testing.assert_allclose(a[:, 21:27], b[:, 21:27], rtol=1e-7, atol=1e-16)


@pytest.mark.parametrize("radius,min_points", [(1, 100), (2, 40), (7, 100)])
def test_scs_other_radii_and_point_filters(api, O, radius, min_points):
    """SCS neighbourhoods other than the reference's hard-coded 5 (generic kernel; radius 7 exceeds the per-lane cache)."""
    est, gt, cfg = synth.make_pair("C2", scale=0.2)
    v = cfg["vmd_voxel_size"]
    with _ctx(api, est, gt, vmd_voxel_size=v) as ctx:
        got = ctx.calculateVMD(v, min_points, radius)
    exp = O.eval_awd(est, gt, v, min_points, radius)
    assert (got.n_pairs, got.n_scs) == (exp.n_pairs, exp.n_scs) and got.n_pairs > 50
    np.testing.assert_allclose([got.awd, got.scs], [exp.awd, exp.scs], rtol=RTOL)


def test_awd_negative_coordinates_and_no_pairs(api, O):
    est, gt, _ = synth.make_pair("C1", scale=0.5)
    est = est - 7.3
    gt = gt - 7.3
    with _ctx(api, est, gt) as ctx:
        got = ctx.calculateVMD(0.5, 100, 5)
        none = ctx.calculateVMD(0.05, 100, 5)        # no voxel reaches 100 points: 0/0 -> NaN like the reference
    exp = O.eval_awd(est, gt, 0.5, 100, 5)
    assert (got.n_pairs, got.n_active, got.n_old, got.n_new) == (exp.n_pairs, exp.n_active, exp.n_old, exp.n_new)
    np.testing.assert_allclose(got.awd, exp.awd, rtol=RTOL)
    np.testing.assert_allclose(got.scs, exp.scs, rtol=RTOL)
    assert none.n_pairs == 0 and np.isnan(none.awd) and np.isnan(none.scs)


@pytest.mark.parametrize("tile", [False, True])
@pytest.mark.parametrize("world", [2, 3, 8])
def test_shard_count_invariance(api, O, world, tile):
    """One context PER RANK (as in a multi-GPU job: every rank lays the clouds out itself, and the order of the points
    inside a lattice cell differs from rank to rank because the scatter takes its slots with atomics).  The shards are
    cell-aligned, so every point is evaluated by exactly one rank and the summed accumulators reproduce world = 1."""
    import os
    est, gt, cfg = synth.make_pair("C1", scale=0.5)
    p = A.make_nn_params(cfg["tau"], 1.0, pairing=A.ME_PAIRING_AS_WRITTEN)
    if tile:
        os.environ["ME_NN_TILE"] = "1"
    # the tile sweep needs a dense cell table; on a sparse one ME_NN_TILE falls back to the row walk
    sweep = ("ME_KBIT_NN_ROWS_SPARSE" if os.environ.get("ME_FORCE_SPARSE")
             else ("ME_KBIT_NN_TILE" if tile else "ME_KBIT_NN_ROWS_DENSE"))
    try:
        with _ctx(api, est, gt) as ctx:
            ref = ctx.calculateMetricsWithInitialMatrix(p)
            assert sweep in ctx.kernel_trace()[0]
            ref_m = ctx.eval_mme_accum(A.ME_CLOUD_EST, 0.1, 10)
        tot_e, tot_g, tot_m = A.me_nn_accum(), A.me_nn_accum(), A.me_mme_accum()
        tot_m.min_entropy, tot_m.max_entropy = np.inf, -np.inf
        for r in range(world):
            # a different point order per rank: the caller order is permuted (indices are mapped back below)
            perm_e = np.random.RandomState(100 + r).permutation(len(est))
            with _ctx(api, est[perm_e], gt, rank=r, world=world) as ctx:
                e, g = ctx.eval_nn_accum(p_geo := A.make_nn_params(cfg["tau"], 1.0, pairing=A.ME_PAIRING_GEOMETRIC))
                assert sweep in ctx.kernel_trace()[0]
                m = ctx.eval_mme_accum(A.ME_CLOUD_EST, 0.1, 10)
            for tot, part in ((tot_e, e), (tot_g, g)):
                for name, ctype in A.me_nn_accum._fields_:
                    v = getattr(part, name)
                    if hasattr(v, "__len__"):
                        for i in range(len(v)):
                            getattr(tot, name)[i] += v[i]
                    else:
                        setattr(tot, name, getattr(tot, name) + v)
            tot_m.n_query += m.n_query; tot_m.n_valid += m.n_valid; tot_m.sum_entropy += m.sum_entropy
            tot_m.min_entropy = min(tot_m.min_entropy, m.min_entropy)
            tot_m.max_entropy = max(tot_m.max_entropy, m.max_entropy)
        with _ctx(api, est, gt) as ctx:
            ref_geo = ctx.calculateMetricsWithInitialMatrix(p_geo)
            got = ctx.nn_finalize(p_geo, tot_e, tot_g)
    finally:
        os.environ.pop("ME_NN_TILE", None)
    assert tot_e.n_query == len(est) and tot_g.n_query == len(gt)
    _cmp_nn(got, ref_geo)
    assert list(ref.est_to_gt.n_inlier) == list(ref_geo.est_to_gt.n_inlier)
    assert tot_m.n_valid == ref_m.n_valid and tot_m.n_query == len(est)
    np.testing.assert_allclose(tot_m.sum_entropy, ref_m.sum_entropy, rtol=1e-12)
    assert (tot_m.min_entropy, tot_m.max_entropy) == (ref_m.min_entropy, ref_m.max_entropy)


def test_device_resident_cloud_and_errors(api):
    import torch
    est, gt, cfg = synth.make_pair("C1", scale=0.1)
    p = A.make_nn_params(cfg["tau"], 1.0)
    with _ctx(api, est, gt) as ctx:
        ref = ctx.calculateMetricsWithInitialMatrix(p)
    te, tg = torch.from_numpy(est).cuda(), torch.from_numpy(gt).cuda()
    with api.MapEvalB200(stream=torch.cuda.current_stream().cuda_stream) as ctx:
        with pytest.raises(api.MapEvalError):
            ctx.calculateMetricsWithInitialMatrix(p)             # clouds not set -> ME_ERR_EMPTY
        ctx.set_cloud_device(A.ME_CLOUD_EST, te.data_ptr(), len(est), keepalive=te)
        ctx.set_cloud_device(A.ME_CLOUD_GT, tg.data_ptr(), len(gt), keepalive=tg)
        got = ctx.calculateMetricsWithInitialMatrix(p)
        assert list(got.est_to_gt.n_inlier) == list(ref.est_to_gt.n_inlier)
        assert got.full_cd == pytest.approx(ref.full_cd, rel=1e-12)
        bad = est.copy(); bad[3, 1] = np.nan
        ctx.set_cloud(A.ME_CLOUD_EST, bad)
        with pytest.raises(api.MapEvalError):
            ctx.calculateMetricsWithInitialMatrix(p)             # non-finite coordinates are rejected
        assert ctx.launch_count() > 0


@pytest.mark.parametrize("n_est", [5001, 5002])
def test_unaligned_device_buffer_and_extreme_points(api, O, n_est):
    """Device buffers that are 8- but not 16-byte aligned, odd/even coordinate counts, and the extreme coordinates placed
    on the first and last scalars (the bbox reduction reads 16-byte pairs plus the leftover scalars)."""
    import torch
    est, gt, cfg = synth.make_pair("C1", scale=0.06)
    est = est[:n_est].copy()
    est[0, 0] = -3.5          # global min x on the leading scalar
    est[-1, 2] = 7.25         # global max z on the trailing scalar
    p = A.make_nn_params(cfg["tau"], 1.0, pairing=A.ME_PAIRING_GEOMETRIC)
    exp = O.eval_nn(est, gt, p)
    buf = torch.zeros(3 * n_est + 1, dtype=torch.float64, device="cuda")
    buf[1:] = torch.from_numpy(est.reshape(-1)).cuda()
    view = buf[1:]
    assert view.data_ptr() % 16 == 8
    tg = torch.from_numpy(gt).cuda()
    with api.MapEvalB200(stream=torch.cuda.current_stream().cuda_stream) as ctx:
        ctx.set_cloud_device(A.ME_CLOUD_EST, view.data_ptr(), n_est, keepalive=buf)
        ctx.set_cloud_device(A.ME_CLOUD_GT, tg.data_ptr(), len(gt), keepalive=tg)
        got = ctx.calculateMetricsWithInitialMatrix(p)
    _cmp_nn(got, exp)


@pytest.mark.parametrize("voxel", [0.01, 0.05, 0.3])
def test_voxel_downsample_matches_open3d_semantics(api, O, voxel):
    """me_voxel_downsample vs the oracle's restatement of PointCloud::VoxelDownSample: the same SET of output points,
    bit for bit (sums in input order, division by the count); the oracle emits in voxel order too."""
    est, gt, cfg = synth.make_pair("C2", scale=0.1)
    est = est - np.array([250.0, -1000.0, 3.0])                  # negative / large coordinates
    est = np.ascontiguousarray(np.concatenate([est, est[:500]]))  # exact duplicates share a voxel
    with _ctx(api, est, gt) as ctx:
        n = ctx.voxel_downsample(A.ME_CLOUD_EST, voxel)
        got = ctx.get_cloud(A.ME_CLOUD_EST)
        # the path runs on the down-sampled cloud afterwards
        p = A.make_nn_params(cfg["tau"], 1.0, pairing=A.ME_PAIRING_GEOMETRIC)
        nn = ctx.calculateMetricsWithInitialMatrix(p)
    exp = O.voxel_downsample(est, voxel)
    assert n == len(exp) == len(got)
    np.testing.assert_array_equal(got, exp)
    _cmp_nn(nn, O.eval_nn(exp, gt, p))


def test_voxel_downsample_errors(api):
    est, gt, cfg = synth.make_pair("C1", scale=0.01)
    with _ctx(api, est, gt) as ctx:
        with pytest.raises(api.MapEvalError):
            ctx.voxel_downsample(A.ME_CLOUD_EST, 0.0)
        with pytest.raises(api.MapEvalError):
            ctx.voxel_downsample(A.ME_CLOUD_EST, 1e-7)             # more than 2^21 voxels per axis
        assert ctx.voxel_downsample(A.ME_CLOUD_EST, 100.0) == 1    # everything in one voxel


def test_tiny_and_degenerate_clouds(api, O):
    """Ragged / degenerate inputs: single points, a handful of points, all points identical, collinear points, clouds of
    very different extent.  The reference's own guards: empty clouds end process() (map_eval.cpp:32-35); 0/0 -> NaN for
    AWD / SCS without voxel pairs (:324, :387); MME without valid points returns 0 (:1720-1724)."""
    p = A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], 1.0, pairing=A.ME_PAIRING_GEOMETRIC)
    rng = np.random.RandomState(3)
    cases = {
        "one_vs_one": (np.array([[0.1, 0.2, 0.3]]), np.array([[0.1, 0.2, 0.35]])),
        "one_vs_many": (np.array([[0.5, 0.5, 0.5]]), rng.rand(300, 3)),
        "few": (rng.rand(7, 3), rng.rand(5, 3)),
        "identical_points": (np.tile([[1.0, 2.0, 3.0]], (200, 1)), np.tile([[1.0, 2.0, 3.01]], (150, 1))),
        "collinear": (np.stack([np.linspace(0, 1, 400), np.zeros(400), np.zeros(400)], 1),
                      np.stack([np.linspace(0, 1, 300), np.full(300, 0.02), np.zeros(300)], 1)),
        "disjoint_extents": (rng.rand(500, 3) * 0.5, rng.rand(400, 3) * 0.5 + np.array([40.0, -3.0, 7.0])),
    }
    for name, (est, gt) in cases.items():
        est, gt = np.ascontiguousarray(est, dtype=np.float64), np.ascontiguousarray(gt, dtype=np.float64)
        with _ctx(api, est, gt) as ctx:
            nn = ctx.calculateMetricsWithInitialMatrix(p)
            mme, ent = ctx.computeMME(A.ME_CLOUD_EST, 0.1, 10, want_entropies=True)
            awd = ctx.calculateVMD(0.25, 100, 5)
        _cmp_nn(nn, O.eval_nn(est, gt, p))
        omme, oent = O.eval_mme(est, 0.1, 10, want_entropies=True)
        assert (mme.n_valid, mme.n_total) == (omme.n_valid, omme.n_total), name
        np.testing.assert_array_equal(ent != 0, oent != 0, err_msg=name)
        ok = oent > -25                      # (near-)singular neighbourhoods: det is a rounding-noise quantity
        np.testing.assert_allclose(ent[ok], oent[ok], rtol=1e-5, err_msg=name)
        oawd = O.eval_awd(est, gt, 0.25, 100, 5)
        assert (awd.n_pairs, awd.n_scs, awd.n_voxels_est, awd.n_voxels_gt) == \
               (oawd.n_pairs, oawd.n_scs, oawd.n_voxels_est, oawd.n_voxels_gt), name
        np.testing.assert_allclose([awd.awd, awd.scs], [oawd.awd, oawd.scs], rtol=1e-9, equal_nan=True, err_msg=name)
    # empty clouds are refused (map_eval.cpp:32-35)
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(A.ME_CLOUD_EST, np.zeros((0, 3)))
        ctx.set_cloud(A.ME_CLOUD_GT, rng.rand(10, 3))
        with pytest.raises(api.MapEvalError):
            ctx.calculateMetricsWithInitialMatrix(p)
        with pytest.raises(api.MapEvalError):
            ctx.computeMME(A.ME_CLOUD_EST, 0.1, 10)


@pytest.mark.parametrize("max_dist", [0.15, 1.0])
def test_icp_point_to_point_and_path_b(api, O, max_dist):
    """registration_methods: 0 — RegistrationICP + TransformationEstimationPointToPoint (map_eval.cpp:1366-1394), then the
    path-B metrics of calculateMetrics(reg) (:1147-1202) on the aligned cloud."""
    est, gt, cfg = synth.make_pair("C1", scale=0.3)
    th = np.deg2rad(1.5)
    Rz = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]])
    c = gt.mean(0)
    src = np.ascontiguousarray((est - c) @ Rz.T + c + np.array([0.02, -0.015, 0.01]))
    T0 = np.eye(4)
    T0[:3, 3] = [0.001, 0.0, -0.002]
    with _ctx(api, src, gt) as ctx:
        T, reg = ctx.performICPRegistration(max_dist, T0)
        aligned = ctx.get_cloud(A.ME_CLOUD_EST)
        p = A.make_nn_params(cfg["tau"], max_dist, cutoff_mode=A.ME_CUTOFF_DIST_LT_R, pairing=A.ME_PAIRING_GEOMETRIC)
        nn = ctx.calculateMetricsWithInitialMatrix(p)          # = calculateMetrics(reg) on the aligned cloud
    To, fit, rmse, nc, it = O.icp_point_to_point(src, gt, max_dist, T0)
    assert (reg.n_corr, reg.iterations) == (nc, it)
    np.testing.assert_allclose(T, To, atol=1e-10)
    np.testing.assert_allclose([reg.fitness, reg.inlier_rmse], [fit, rmse], rtol=1e-9)
    oaligned = O.transform(src, To)
    np.testing.assert_allclose(aligned, oaligned, atol=1e-9)
    # the registration improves on the initial guess
    T1, reg1 = None, None
    with _ctx(api, src, gt) as ctx:
        _, reg0 = ctx.performICPRegistration(max_dist, T0, max_iteration=0)
    assert reg.inlier_rmse <= reg0.inlier_rmse and reg0.iterations == 0
    _cmp_nn(nn, O.eval_nn(aligned, gt, p))


def test_small_lattice_budget(api, O):
    """A cell-table budget far below what the clouds would like (large sparse scenes hit this): the lattice coarsens
    (tens of points per cell), the MME radius may span less than one cell, results are unchanged."""
    est, gt, cfg = synth.make_pair("C2", scale=0.05)
    p = A.make_nn_params(cfg["tau"], 1.0, pairing=A.ME_PAIRING_GEOMETRIC)
    with _ctx(api, est, gt, max_grid_cells=2000, vmd_voxel_size=0.0) as ctx:
        nn = ctx.calculateMetricsWithInitialMatrix(p)
        mme, ent = ctx.computeMME(A.ME_CLOUD_EST, cfg["nn_radius"], 10, want_entropies=True)
    _cmp_nn(nn, O.eval_nn(est, gt, p))
    omme, oent = O.eval_mme(est, cfg["nn_radius"], 10, want_entropies=True)
    assert mme.n_valid == omme.n_valid
    np.testing.assert_allclose(ent, oent, rtol=RTOL_ENT, atol=0)


def test_device_resident_accumulators_equal_the_host_path(api, O):
    """me_eval_*_accum_device + me_accum_fetch (what bench.py and the multi-GPU pass use) = me_eval_*_accum; a *_device MME
    section survives a later me_eval_nn_accum, which writes only the NN sections of the block"""
    est, gt, cfg = synth.make_pair("C2", scale=0.1)
    p = A.make_nn_params(cfg["tau"], 1.0)
    with _ctx(api, est, gt, vmd_voxel_size=cfg["vmd_voxel_size"]) as ctx:
        m_e = ctx.eval_mme_accum(A.ME_CLOUD_EST, cfg["nn_radius"], 10)
        m_g = ctx.eval_mme_accum(A.ME_CLOUD_GT, cfg["nn_radius"], 5)
        e, g = ctx.eval_nn_accum(p)
        ctx.accum_reset()
        ctx.eval_mme_accum_device(A.ME_CLOUD_EST, cfg["nn_radius"], 10)
        ctx.eval_mme_accum_device(A.ME_CLOUD_GT, cfg["nn_radius"], 5)
        ctx.eval_nn_accum(p)
        _, _, (m_e3, m_g3) = ctx.accum_fetch(want_mme=(True, True))
        ctx.eval_nn_accum_device(p)
        ptr, n_sum, n_max = ctx.accum_block()
        assert ptr and n_sum == 2 * (A.ME_NN_ACCUM_I64 + A.ME_NN_ACCUM_F64) + 14 and n_max == 4
        e2, g2, (m_e2, m_g2) = ctx.accum_fetch(want_mme=(True, True))
    for a, b in ((e, e2), (g, g2)):
        da, db = A.struct_to_dict(a), A.struct_to_dict(b)
        for k in ("n_query", "n_corr", "n_inlier", "n_ub", "n_far"):
            assert da[k] == db[k], k
        for k in ("sum_d", "sum_d2", "sum_d_all", "sum_d2_all", "sum_nn_dist", "rank_mean", "rank_m2"):
            np.testing.assert_allclose(da[k], db[k], rtol=1e-12)
        assert da["rank_n"] == db["rank_n"] == [da["n_corr"]] + [0.0] * (A.ME_MAX_WORLD - 1)
    for a, b in ((m_e, m_e2), (m_g, m_g2), (m_e, m_e3), (m_g, m_g3)):
        assert (a.n_query, a.n_valid) == (b.n_query, b.n_valid)
        np.testing.assert_allclose([a.sum_entropy, a.min_entropy, a.max_entropy], [b.sum_entropy, b.min_entropy, b.max_entropy], rtol=1e-12)


def test_repeated_passes_over_the_same_maps_reuse_the_lattice_plan(api, O, monkeypatch):
    """The lattice plan (refined cell edge) of a cloud pair is remembered by the context: setting the same clouds again plans in
    one step.  Results are those of a fresh context, with and without the memory (ME_NO_PLAN_CACHE)."""
    est, gt, cfg = synth.make_pair("C2", scale=0.1)
    p = A.make_nn_params(cfg["tau"], 1.0)
    got = []
    for env in (None, "1"):
        if env:
            monkeypatch.setenv("ME_NO_PLAN_CACHE", env)
        with api.MapEvalB200(vmd_voxel_size=cfg["vmd_voxel_size"]) as ctx:
            for rep in range(3):
                ctx.set_cloud(A.ME_CLOUD_EST, est)
                ctx.set_cloud(A.ME_CLOUD_GT, gt if rep != 1 else gt[: len(gt) // 2])      # pass 1: another pair in between
                m = ctx.eval_mme_accum(A.ME_CLOUD_EST, cfg["nn_radius"], 10)
                e, g = ctx.eval_nn_accum(p)
                awd = ctx.calculateVMD(cfg["vmd_voxel_size"], 20, 5)
                if rep != 1:
                    got.append((A.struct_to_dict(e), A.struct_to_dict(g), (m.n_valid, m.sum_entropy), (awd.n_pairs, awd.awd, awd.scs)))
    for other in got[1:]:
        for a, b in zip(got[0][:2], other[:2]):
            for k in ("n_query", "n_corr", "n_inlier", "n_ub"):
                assert a[k] == b[k], k
            for k in ("sum_d", "sum_d2", "sum_d_all", "sum_nn_dist"):
                np.testing.assert_allclose(a[k], b[k], rtol=1e-12)
        assert got[0][2][0] == other[2][0] and got[0][3][0] == other[3][0]
        np.testing.assert_allclose([got[0][2][1], got[0][3][1], got[0][3][2]], [other[2][1], other[3][1], other[3][2]], rtol=1e-9)

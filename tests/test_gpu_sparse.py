"""The sparse cell table (occupied row segments + hash, DESIGN.md §2) against the oracle and against the dense table:
forced through a tiny cell budget on the box configs, and on a 1 km x 1 km site-scale terrain where the dense table at
the wanted cell edge would not fit the budget."""
import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import synth

pytestmark = pytest.mark.gpu

RTOL = 1e-9


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _cmp_dir(got, exp):
    assert (got.n_source, got.n_corr, got.n_ub) == (exp.n_source, exp.n_corr, exp.n_ub)
    assert list(got.n_inlier) == list(exp.n_inlier)
    for k in ("mean", "rmse", "fitness", "sigma"):
        np.testing.assert_allclose(list(getattr(got, k)), list(getattr(exp, k)), rtol=RTOL, atol=1e-300, err_msg=k)
    np.testing.assert_allclose(got.sum_nn_dist, exp.sum_nn_dist, rtol=RTOL)


def _pass(api, est, gt, cfg, p, **kw):
    with api.MapEvalB200(vmd_voxel_size=cfg["vmd_voxel_size"], **kw) as ctx:
        ctx.set_cloud(A.ME_CLOUD_EST, est)
        ctx.set_cloud(A.ME_CLOUD_GT, gt)
        mme, ent = ctx.computeMME(A.ME_CLOUD_EST, cfg["nn_radius"], 10, want_entropies=True)
        nn = ctx.calculateMetricsWithInitialMatrix(p)
        idx, d2 = ctx.get_nn(A.ME_CLOUD_EST)
        awd = ctx.calculateVMD(cfg["vmd_voxel_size"], 100, 5)
    return mme, ent, nn, idx, d2, awd


@pytest.mark.parametrize("pairing", [A.ME_PAIRING_AS_WRITTEN, A.ME_PAIRING_GEOMETRIC])
def test_forced_sparse_table_on_a_box_config(api, O, pairing):
    est, gt, cfg = synth.make_pair("C2", scale=0.2)
    p = A.make_nn_params(cfg["tau"], 1.0, pairing=pairing)
    mme, ent, nn, idx, d2, awd = _pass(api, est, gt, cfg, p, max_grid_cells=1)       # budget of one cell: always sparse
    dmme, dent, dnn, didx, dd2, dawd = _pass(api, est, gt, cfg, p)                    # dense
    np.testing.assert_array_equal(idx, didx)
    np.testing.assert_array_equal(d2, dd2)
    assert mme.n_valid == dmme.n_valid and awd.n_pairs == dawd.n_pairs
    np.testing.assert_allclose(ent, dent, rtol=1e-6, atol=1e-12)
    onn, oie, _ = O.eval_nn(est, gt, p, want_indices=True)
    _cmp_dir(nn.est_to_gt, onn.est_to_gt)
    _cmp_dir(nn.gt_to_est, onn.gt_to_est)
    np.testing.assert_array_equal(idx, oie)
    np.testing.assert_allclose(nn.full_cd, onn.full_cd, rtol=RTOL)
    omme, oent = O.eval_mme(est, cfg["nn_radius"], 10, want_entropies=True)
    assert mme.n_valid == omme.n_valid
    np.testing.assert_allclose(ent, oent, rtol=1e-6, atol=1e-12)
    oawd = O.eval_awd(est, gt, cfg["vmd_voxel_size"], 100, 5)
    assert (awd.n_pairs, awd.n_scs, awd.n_active, awd.n_old, awd.n_new) == (oawd.n_pairs, oawd.n_scs, oawd.n_active, oawd.n_old, oawd.n_new)
    np.testing.assert_allclose([awd.awd, awd.scs], [oawd.awd, oawd.scs], rtol=1e-8)


def test_sparse_table_far_queries_normals_and_shards(api, O):
    """outliers tens of metres away (ring expansion through empty segments), k-NN normals, and two ranks summing up"""
    rs = np.random.RandomState(9)
    gt = np.concatenate([rs.randn(30000, 3) * 0.4 + c for c in ([0, 0, 0], [9, 2, -3], [-5, 12, 1])])
    est = np.concatenate([gt[::2] + rs.randn(len(gt[::2]), 3) * 0.01, rs.rand(2000, 3) * 60 - 30])
    est, gt = est.astype(np.float32).astype(np.float64), gt.astype(np.float32).astype(np.float64)
    p = A.make_nn_params([0.5, 0.3, 0.2, 0.1, 0.05], 1.0, pairing=A.ME_PAIRING_GEOMETRIC)
    with api.MapEvalB200(max_grid_cells=1) as ctx:
        ctx.set_cloud(A.ME_CLOUD_EST, est)
        ctx.set_cloud(A.ME_CLOUD_GT, gt)
        e, g = ctx.eval_nn_accum(p)
        nn = ctx.nn_finalize(p, e, g)
        idx, d2 = ctx.get_nn(A.ME_CLOUD_EST)
        # the outliers lie beyond the far kernel's cell rings: its coarse-block phase (> 256 cells per axis) finds them
        assert {"ME_KBIT_NN_FAR", "ME_KBIT_NN_FAR_COARSE", "ME_KBIT_NN_ROWS_SPARSE"} <= ctx.kernel_trace()[0]
        nrm = ctx.estimate_normals(A.ME_CLOUD_GT, 20)
    assert e.n_far > 500
    oi, od2 = O.knn1(est, gt)
    np.testing.assert_array_equal(d2, od2)
    np.testing.assert_array_equal(idx, oi)
    _cmp_dir(nn.est_to_gt, O.eval_nn(est, gt, p).est_to_gt)
    onrm = O.estimate_normals_knn(gt, 20)
    assert np.mean(np.abs(np.einsum("ni,ni->n", nrm, onrm)) > 1 - 1e-6) > 0.999
    tot = None
    for r in range(2):
        with api.MapEvalB200(max_grid_cells=1, rank=r, world=2) as ctx:
            ctx.set_cloud(A.ME_CLOUD_EST, est)
            ctx.set_cloud(A.ME_CLOUD_GT, gt)
            m = ctx.eval_mme_accum(A.ME_CLOUD_EST, 0.2, 10)
            er, gr = ctx.eval_nn_accum(p)
        part = np.array([er.n_query, er.n_corr] + list(er.n_inlier) + [gr.n_query, gr.n_corr] + list(gr.n_inlier) + [m.n_query, m.n_valid])
        tot = part if tot is None else tot + part
    with api.MapEvalB200(max_grid_cells=1) as ctx:
        ctx.set_cloud(A.ME_CLOUD_EST, est)
        ctx.set_cloud(A.ME_CLOUD_GT, gt)
        m1 = ctx.eval_mme_accum(A.ME_CLOUD_EST, 0.2, 10)
    assert list(tot) == [e.n_query, e.n_corr] + list(e.n_inlier) + [g.n_query, g.n_corr] + list(g.n_inlier) + [m1.n_query, m1.n_valid]
    assert m1.n_valid == O.eval_mme(est, 0.2, 10).n_valid


def test_site_scale_terrain(api, O):
    """1 km x 1 km x 50 m terrain, 3 M vs 2 M points: with a budget of 2^20 cells the dense table would need 1 m+ cells
    (tens of points each); the sparse table keeps the wanted edge.  Every metric against the oracle."""
    cfg = dict(synth.CONFIGS["S1"], nn_radius=2.0, vmd_voxel_size=10.0)
    est = synth.site_scene(3_000_000, synth.EST_SEED, synth.EST_NOISE_SIGMA)
    gt = synth.site_scene(2_000_000, synth.GT_SEED, synth.GT_SURFACE_NOISE_SIGMA)
    p = A.make_nn_params(cfg["tau"], 1.0)
    mme, ent, nn, idx, d2, awd = _pass(api, est, gt, cfg, p, max_grid_cells=1 << 20)
    onn, oie, _ = O.eval_nn(est, gt, p, want_indices=True)
    _cmp_dir(nn.est_to_gt, onn.est_to_gt)
    _cmp_dir(nn.gt_to_est, onn.gt_to_est)
    _, od2 = O.knn1(est, gt)
    np.testing.assert_array_equal(d2, od2)
    omme, oent = O.eval_mme(est, cfg["nn_radius"], 10, want_entropies=True)
    assert mme.n_valid == omme.n_valid and mme.n_valid > 0.9 * len(est)
    np.testing.assert_allclose(mme.mme, omme.mme, rtol=1e-7)
    np.testing.assert_allclose(ent, oent, rtol=1e-6, atol=1e-6)      # entropies cross zero on this scene (r = 2 m): absolute floor
    oawd = O.eval_awd(est, gt, cfg["vmd_voxel_size"], 100, 5)
    assert awd.n_pairs == oawd.n_pairs and awd.n_pairs > 100
    np.testing.assert_allclose([awd.awd, awd.scs], [oawd.awd, oawd.scs], rtol=1e-8)

"""The simulation operators on the device (me_copy_cloud, me_add_gaussian_noise, me_add_non_uniform_density,
me_add_sparse_outliers, me_add_local_deformation) against the numpy statement tests/perturb_ref.py.

Integer structure (kept points, counts, outlier bases) is bit-exact.  Coordinates agree to 1e-14 (sigma |g| + strength)
plus one ulp: the device's fp64 log / cos differ from the host's libm by an ulp or two, nothing else differs."""
import os
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import perturb_ref as ref  # noqa: E402

pytestmark = pytest.mark.gpu

SEED = synth.EST_SEED
EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT


def _api():
    from cloud_map_evaluation_b200 import api
    return api


@pytest.fixture(scope="module")
def scene():
    """a 200 k-point box off the origin (no coordinate 0, where sin has no sign), with unit normals"""
    gt = synth.uniform_box(200_000, 2.5, synth.GT_SEED, origin=(0.123, 0.456, -0.2))
    rng = np.random.RandomState(5)
    nrm = rng.randn(len(gt), 3)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return gt, nrm


def _ctx(gt, nrm=None, **kw):
    ctx = _api().MapEvalB200(device=0, **kw)
    ctx.set_cloud(GT, gt)
    if nrm is not None:
        ctx.set_normals(GT, nrm)
    ctx.copy_cloud(GT, EST)
    return ctx


def _ulp(x):
    return np.spacing(np.abs(x))


def test_copy_cloud(scene):
    gt, nrm = scene
    with _ctx(gt, nrm) as ctx:
        assert ctx.n[EST] == len(gt)
        np.testing.assert_array_equal(ctx.get_cloud(EST), gt)
        np.testing.assert_array_equal(ctx.get_normals(EST), nrm)
        with pytest.raises(_api().MapEvalError):
            ctx.copy_cloud(GT, GT)
    with _ctx(gt) as ctx:                                        # no normals on the source: none on the copy
        with pytest.raises(_api().MapEvalError):
            ctx.get_normals(EST)


@pytest.mark.parametrize("sigma", [0.0, 0.003, 0.1])
def test_gaussian_noise(scene, sigma):
    gt, nrm = scene
    with _ctx(gt, nrm) as ctx:
        ctx.add_gaussian_noise(EST, sigma, SEED)
        dev = ctx.get_cloud(EST)
        np.testing.assert_array_equal(ctx.get_normals(EST), nrm)     # the reference moves points_ only
    exp = ref.gaussian_noise(gt, sigma, SEED)
    if sigma == 0:
        assert dev.tobytes() == gt.tobytes()
        return
    idx = np.arange(len(gt), dtype=np.uint64)
    g = np.stack([synth.gaussian(SEED, idx, 2 * a) for a in range(3)], axis=1)
    err = np.abs(dev - exp)
    assert (err <= 1e-14 * sigma * np.abs(g) + _ulp(exp)).all(), err.max()
    assert (dev != gt).mean() > 0.99


@pytest.mark.parametrize("ratios", [(0.3, 0.8, 0.5), (1.0, 1.0, 0.5), (0.0, 0.0, 0.5), (0.25, 0.9, 0.0), (0.6, 0.1, 0.07)])
def test_non_uniform_density(scene, ratios):
    gt, nrm = scene
    sparse, dense, s = ratios
    keep, xn, yn = ref.density_keep(gt, sparse, dense, s, SEED)
    tiny = ((np.abs(xn) < 1e-9) & (xn != 0)) | ((np.abs(yn) < 1e-9) & (yn != 0))
    assert tiny.sum() == 0               # where device and host sin could disagree in sign: none on this scene
    with _ctx(gt, nrm) as ctx:
        n = ctx.add_non_uniform_density(EST, sparse, dense, s, SEED)
        assert n == keep.sum() == ctx.n[EST]
        assert ctx.get_cloud(EST).tobytes() == gt[keep].tobytes()
        assert ctx.get_normals(EST).tobytes() == nrm[keep].tobytes()
    if ratios[:2] == (1.0, 1.0):
        assert n == len(gt)
    if ratios[:2] == (0.0, 0.0):
        assert n == 0


def test_sparse_outliers(scene):
    gt, nrm = scene
    N = len(gt)
    for ratio in (0.05, 0.3):
        m = ref.outlier_count(N, ratio)
        with _ctx(gt, nrm) as ctx:                               # range 0: every outlier is a copy of its base point
            assert ctx.add_sparse_outliers(EST, ratio, 0.0, SEED) == N + m == ctx.n[EST]
            dev = ctx.get_cloud(EST)
            with pytest.raises(_api().MapEvalError):
                ctx.get_normals(EST)                             # normals_ and points_ differ in size
        assert dev[:N].tobytes() == gt.tobytes()
        assert dev[N:].tobytes() == gt[ref.outlier_bases(N, m, SEED)].tobytes()
    rng = 0.5
    with _ctx(gt) as ctx:
        ctx.add_sparse_outliers(EST, 0.3, rng, SEED)
        dev = ctx.get_cloud(EST)
    exp = ref.sparse_outliers(gt, 0.3, rng, SEED)
    assert dev.shape == exp.shape and dev[:N].tobytes() == gt.tobytes()
    j = np.arange(len(exp) - N, dtype=np.uint64)
    g = np.stack([synth.gaussian(SEED, j, 8 + 2 * a) for a in range(3)], axis=1)
    err = np.abs(dev[N:] - exp[N:])
    assert (err <= 1e-14 * rng * np.abs(g) + _ulp(exp[N:])).all(), err.max()
    # (int)(N ratio) truncation, a negative ratio, an empty cloud
    with _ctx(gt[:100]) as ctx:
        assert ctx.add_sparse_outliers(EST, 0.29, rng, SEED) == 128
        assert ctx.add_sparse_outliers(EST, -0.5, rng, SEED) == 128
    with _ctx(gt[:0]) as ctx:
        assert ctx.add_sparse_outliers(EST, 0.5, rng, SEED) == 0


def test_sparse_outliers_range_errors(scene):
    gt, _ = scene
    api = _api()
    with _ctx(gt[:1000]) as ctx:
        for ratio in (2.2e6, float("inf"), float("nan")):        # N ratio >= 2^31 (or not a number)
            with pytest.raises(api.MapEvalError) as e:
                ctx.add_sparse_outliers(EST, ratio, 1.0, SEED)
            assert e.value.code == A.ME_ERR_RANGE
        with pytest.raises(api.MapEvalError) as e:               # m = 2^31 - 1001: N + m = 2^31 - 1
            ctx.add_sparse_outliers(EST, (2 ** 31 - 1001 + 0.5) / 1000, 1.0, SEED)
        assert e.value.code == A.ME_ERR_RANGE
        for bad in (-1.0, float("nan"), float("inf")):
            with pytest.raises(api.MapEvalError) as e:
                ctx.add_sparse_outliers(EST, 0.1, bad, SEED)
            assert e.value.code == A.ME_ERR_INVALID
            with pytest.raises(api.MapEvalError) as e:
                ctx.add_gaussian_noise(EST, bad, SEED)
            assert e.value.code == A.ME_ERR_INVALID
        assert ctx.n[EST] == 1000 and ctx.get_cloud(EST).tobytes() == gt[:1000].tobytes()


@pytest.mark.parametrize("radius,strength", [(0.8, 0.2), (0.3, -0.05), (0.0, 0.2), (-1.0, 0.2)])
def test_local_deformation(scene, radius, strength):
    gt, nrm = scene
    c = gt[1234] + [0.01, -0.02, 0.005]
    pts = np.concatenate([gt, [c]])                                   # a point exactly at the centre
    pn = np.concatenate([nrm, [[0.0, 0.0, 1.0]]])
    with _ctx(pts, pn) as ctx:
        ctx.add_local_deformation(EST, radius, strength, c)
        dev = ctx.get_cloud(EST)
        assert ctx.get_normals(EST).tobytes() == pn.tobytes()
    exp = ref.local_deformation(pts, radius, strength, c)
    v = pts - c
    d = np.sqrt(v[:, 0] * v[:, 0] + (v[:, 1] * v[:, 1] + v[:, 2] * v[:, 2]))
    inside = d < radius
    assert dev[~inside].tobytes() == pts[~inside].tobytes()
    assert dev[-1].tobytes() == c.tobytes()
    err = np.abs(dev - exp)
    assert (err <= 1e-14 * abs(strength) + _ulp(exp)).all(), err.max()
    if radius > 0:
        assert inside.sum() > 500 and (dev[inside] != pts[inside]).any()


def test_borrowed_clouds_are_refused(scene):
    import torch
    gt, _ = scene
    api = _api()
    d_gt = torch.from_numpy(gt).cuda()
    with api.MapEvalB200(device=0) as ctx:
        ctx.set_cloud_device(GT, d_gt.data_ptr(), len(gt), keepalive=d_gt)
        for call in (lambda: ctx.add_gaussian_noise(GT, 0.1, SEED),
                     lambda: ctx.add_non_uniform_density(GT, 0.5, 0.5, 1.0, SEED),
                     lambda: ctx.add_sparse_outliers(GT, 0.1, 1.0, SEED),
                     lambda: ctx.add_local_deformation(GT, 1.0, 0.1, gt[0])):
            with pytest.raises(api.MapEvalError) as e:
                call()
            assert e.value.code == A.ME_ERR_INVALID
        ctx.copy_cloud(GT, EST)                                       # a borrowed ground truth becomes an owned estimate
        ctx.add_gaussian_noise(EST, 0.1, SEED)
        ctx.add_sparse_outliers(EST, 0.1, 1.0, SEED)
        assert ctx.n[EST] == len(gt) + len(gt) // 10
        ctx.synchronize()
    assert d_gt.cpu().numpy().tobytes() == gt.tobytes()                # caller memory untouched


def _degrade(ctx, seed):
    """the host driver's order: deformation, density, noise, outliers"""
    c = np.array([1.0, 1.5, 0.8])
    ctx.add_local_deformation(EST, 0.7, 0.1, c)
    ctx.add_non_uniform_density(EST, 0.4, 0.9, 0.6, seed)
    ctx.add_gaussian_noise(EST, 0.01, seed)
    ctx.add_sparse_outliers(EST, 0.05, 0.3, seed)


def test_ranks_agree_and_seeds_differ(scene):
    gt, nrm = scene
    out = []
    for rank, seed in ((0, SEED), (1, SEED), (0, SEED + 1)):
        with _ctx(gt, nrm, rank=rank, world=2) as ctx:
            _degrade(ctx, seed)
            out.append(ctx.get_cloud(EST))
    assert out[0].tobytes() == out[1].tobytes()
    assert out[0].shape != out[2].shape or out[0].tobytes() != out[2].tobytes()
    # the whole chain against the numpy statement
    c = np.array([1.0, 1.5, 0.8])
    e = ref.local_deformation(gt, 0.7, 0.1, c)
    keep, _, _ = ref.density_keep(e, 0.4, 0.9, 0.6, SEED)
    e = ref.sparse_outliers(ref.gaussian_noise(e[keep], 0.01, SEED), 0.05, 0.3, SEED)
    assert out[0].shape == e.shape
    np.testing.assert_allclose(out[0], e, rtol=0, atol=1e-13)


def test_metrics_after_degradation_match_a_fresh_context(scene):
    """every metric of a degraded estimate equals the one a fresh context computes on the same points: the operators
    invalidate the lattices, plans and per-point results of the first evaluation"""
    gt, _ = scene
    cfg = synth.CONFIGS["C2"]
    p = A.make_nn_params(cfg["tau"], 1.0)
    api = _api()

    def metrics(ctx):
        nn = ctx.calculateMetricsWithInitialMatrix(p)
        mme = ctx.computeMME(EST, cfg["nn_radius"], 10)
        awd = ctx.calculateVMD(cfg["vmd_voxel_size"], 100, 5)
        return nn, mme, awd

    with _ctx(gt, vmd_voxel_size=cfg["vmd_voxel_size"]) as a:
        nn0, _, _ = metrics(a)                                        # lattices of the undegraded copy
        assert nn0.est_to_gt.n_inlier[4] == len(gt)
        _degrade(a, SEED)
        got = metrics(a)
        est = a.get_cloud(EST)
    with api.MapEvalB200(device=0, vmd_voxel_size=cfg["vmd_voxel_size"]) as b:
        b.set_cloud(EST, est)
        b.set_cloud(GT, gt)
        exp = metrics(b)
    (nn, mme, awd), (onn, omme, oawd) = got, exp
    for d in ("est_to_gt", "gt_to_est"):
        g, e = getattr(nn, d), getattr(onn, d)
        assert list(g.n_inlier) == list(e.n_inlier) and g.n_corr == e.n_corr and g.n_source == e.n_source
        for k in ("mean", "rmse", "fitness", "sigma"):
            np.testing.assert_allclose(list(getattr(g, k)), list(getattr(e, k)), rtol=1e-12, atol=1e-15, err_msg=k)
    np.testing.assert_allclose(list(nn.cd), list(onn.cd), rtol=1e-12)
    np.testing.assert_allclose(nn.full_cd, onn.full_cd, rtol=1e-12)
    assert mme.n_valid == omme.n_valid and mme.n_total == omme.n_total
    np.testing.assert_allclose(mme.mme, omme.mme, rtol=1e-12)
    assert (awd.n_pairs, awd.n_scs, awd.n_voxels_est) == (oawd.n_pairs, oawd.n_scs, oawd.n_voxels_est)
    np.testing.assert_allclose([awd.awd, awd.scs], [oawd.awd, oawd.scs], rtol=1e-12)
    assert nn.est_to_gt.n_inlier[4] < len(gt)

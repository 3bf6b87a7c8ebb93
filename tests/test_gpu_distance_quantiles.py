"""Exact distance quantiles and the Hausdorff distance (me_nn_quantile*) from the records of the last NN evaluation.

- the order statistics (lo, hi, min, max) equal np.sort of the population built from me_get_nn bit for bit, and the values
  equal np.quantile(method="linear") bit for bit, in every cut-off x pairing mode and under both populations;
- the same on equal-distance lattices, where thousands of distances tie;
- far queries (answered by nn_far_kernel) give the Hausdorff distance of a k-d tree to 1 ulp;
- sharded over 2, 3 and 8 ranks (replicated and slab layout) and on a sparse cell table the result is world 1's, bit for bit;
- its contract: determinism, stale records, want_full_cd, one direction, a cloud change mid-loop, the curve afterwards."""
import os
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import dist as mdist
from cloud_map_evaluation_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import exact_ref as X  # noqa: E402
from test_exact_ref import offset_scene  # noqa: E402

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
DIRS = ("est_to_gt", "gt_to_est")
POPS = (A.ME_DIST_KEPT, A.ME_DIST_NN)
ALL_MODES = [(m, p) for m in (A.ME_CUTOFF_SQDIST_LE_R, A.ME_CUTOFF_DIST_LT_R)
             for p in (A.ME_PAIRING_AS_WRITTEN, A.ME_PAIRING_GEOMETRIC)]
FIXED_P = [0.0, 0.5, 0.9, 0.95, 0.99, 1.0]


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _ctx(api, est, gt, **kw):
    c = api.MapEvalB200(**kw)
    c.set_cloud(EST, est)
    c.set_cloud(GT, gt)
    return c


def _populations(ctx, est, gt, R, mode, pairing):
    """{population: (est->gt distances, gt->est distances)} built in numpy from me_get_nn"""
    ie, de = ctx.get_nn(EST)
    ig, dg = ctx.get_nn(GT)
    _, k_e, _ = X.kept_pairs(est, gt, ie, de, R, mode)
    _, k_g, _ = X.kept_pairs(gt, est, ig, dg, R, mode, as_written=pairing == A.ME_PAIRING_AS_WRITTEN)
    return {A.ME_DIST_KEPT: (k_e, k_g), A.ME_DIST_NN: (np.sqrt(de[ie >= 0]), np.sqrt(dg[ig >= 0]))}


def _probs(n_min, rng, extra=0):
    p = list(FIXED_P)
    if n_min > 1:
        p.append(1.0 / (n_min - 1))
    return np.array(p + list(rng.random(extra)))


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def _check(res, pops, p):
    for d, x in zip(DIRS, pops):
        r = res[d]
        assert r["n"] == len(x), d
        if len(x) == 0:
            assert np.isnan(r["min"]) and np.isnan(r["max"]) and np.all(np.isnan(r["value"]))
            continue
        xs = np.sort(x)
        n = len(xs)
        k = np.floor((n - 1) * p).astype(np.int64)
        assert _bits(r["min"]) == _bits(xs[0]) and _bits(r["max"]) == _bits(xs[-1]), d
        assert list(r["rank"]) == list(k), d
        np.testing.assert_array_equal(_bits(r["lo"]), _bits(xs[k]))
        np.testing.assert_array_equal(_bits(r["hi"]), _bits(xs[np.minimum(k + 1, n - 1)]))
        np.testing.assert_array_equal(_bits(r["value"]), _bits(np.quantile(x, p, method="linear")))


def _same(a, b):
    for d in DIRS:
        for f in ("n", "min", "max", "rank", "lo", "hi", "value"):
            np.testing.assert_array_equal(np.asarray(a[d][f]).view(np.uint64) if f not in ("n", "rank") else a[d][f],
                                          np.asarray(b[d][f]).view(np.uint64) if f not in ("n", "rank") else b[d][f])
    assert _bits(a["hausdorff"]) == _bits(b["hausdorff"])


# ---------------------------------------------------------------------------------------------------------------
# 1. exactness against np.sort / np.quantile
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,scale", [("C1", 1.0), ("C2", 0.1)])
def test_exact_against_numpy(api, name, scale):
    est, gt, cfg = synth.make_pair(name, scale=scale)
    rng = np.random.default_rng(1)
    with _ctx(api, est, gt) as ctx:
        for mode, pairing in ALL_MODES:
            p = A.make_nn_params(cfg["tau"], 1.0, cutoff_mode=mode, pairing=pairing)
            ref = ctx.calculateMetricsWithInitialMatrix(p)
            pops = _populations(ctx, est, gt, 1.0, mode, pairing)
            for pop in POPS:
                probs = _probs(min(len(x) for x in pops[pop]), rng, extra=50)
                res = ctx.distance_quantiles(probs, pop)
                _check(res, pops[pop], probs)
                if pop == A.ME_DIST_KEPT:
                    assert (res["est_to_gt"]["n"], res["gt_to_est"]["n"]) == (ref.est_to_gt.n_corr, ref.gt_to_est.n_corr)
                    assert np.isnan(res["hausdorff"])
                else:
                    assert (res["est_to_gt"]["n"], res["gt_to_est"]["n"]) == (len(est), len(gt))
                    for d, x in zip(DIRS, pops[pop]):
                        np.testing.assert_allclose(x.sum(), getattr(ref, d).sum_nn_dist, rtol=1e-12)
                    assert res["hausdorff"] == max(res["est_to_gt"]["max"], res["gt_to_est"]["max"])


# ---------------------------------------------------------------------------------------------------------------
# 2. ties: equal-distance lattices
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("origin", [0.0, 1500.0])
def test_ties_on_equal_distance_lattices(api, origin):
    R = 0.5
    est, gt = offset_scene(n_side=24, jitter=0.0, origin=origin, seed=3)
    rng = np.random.default_rng(2)
    with _ctx(api, est, gt) as ctx:
        for mode, pairing in ((A.ME_CUTOFF_SQDIST_LE_R, A.ME_PAIRING_AS_WRITTEN), (A.ME_CUTOFF_DIST_LT_R, A.ME_PAIRING_GEOMETRIC)):
            p = A.make_nn_params([1.0, 0.1, 0.05, 0.03, 0.0], R, cutoff_mode=mode, pairing=pairing)
            ctx.calculateMetricsWithInitialMatrix(p)
            pops = _populations(ctx, est, gt, R, mode, pairing)
            x = pops[A.ME_DIST_KEPT][0]
            assert len(x) - len(np.unique(x)) > 1000           # thousands of equal distances
            for pop in POPS:
                probs = _probs(min(len(v) for v in pops[pop]), rng, extra=57)
                _check(ctx.distance_quantiles(probs, pop), pops[pop], probs)


# ---------------------------------------------------------------------------------------------------------------
# 3. far queries and the Hausdorff distance
# ---------------------------------------------------------------------------------------------------------------
def test_far_queries_and_hausdorff(api):
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(5)
    gt = rng.random((40000, 3)) * np.array([20.0, 20.0, 3.0])
    est = gt[rng.permutation(len(gt))[:30000]] + rng.normal(0, 0.01, (30000, 3))
    clusters = [np.array([45.0, 10.0, 1.0]), np.array([-30.0, -25.0, 2.0]), np.array([10.0, 60.0, 40.0])]
    est = np.concatenate([est] + [c + rng.normal(0, 0.5, (200, 3)) for c in clusters])
    R = 1.0
    p = A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], R)
    probs = np.array(FIXED_P)
    with _ctx(api, est, gt) as ctx:
        ref = ctx.calculateMetricsWithInitialMatrix(p)
        assert ref.est_to_gt.n_corr < len(est)               # the clusters lie beyond the cut-off
        pops = _populations(ctx, est, gt, R, A.ME_CUTOFF_SQDIST_LE_R, A.ME_PAIRING_AS_WRITTEN)
        res = ctx.distance_quantiles(probs, A.ME_DIST_NN)
    _check(res, pops[A.ME_DIST_NN], probs)
    assert res["est_to_gt"]["max"] > 20.0
    h_e = cKDTree(gt).query(est)[0].max()
    h_g = cKDTree(est).query(gt)[0].max()
    h = max(h_e, h_g)
    assert abs(res["hausdorff"] - h) <= np.spacing(h)
    assert abs(res["est_to_gt"]["max"] - h_e) <= np.spacing(h_e) and abs(res["gt_to_est"]["max"] - h_g) <= np.spacing(h_g)
    assert res["hausdorff"] == max(x.max() for x in pops[A.ME_DIST_NN])


# ---------------------------------------------------------------------------------------------------------------
# 4. sharded
# ---------------------------------------------------------------------------------------------------------------
def _sharded(api, est, gt, p, probs, pop, world, slab, **kw):
    """`world` contexts on cuda:0, the selection blocks SUM-reduced with torch between the passes"""
    import torch
    ctxs = [api.MapEvalB200(rank=r, world=world, vmd_voxel_size=0.1, **kw) for r in range(world)]
    try:
        for c in ctxs:
            if slab:
                c.set_layout(A.ME_LAYOUT_SLAB)
            c.set_cloud(EST, est)
            c.set_cloud(GT, gt)
            c.accum_reset()
            c.eval_nn_accum_device(p)
        if slab and any(c.layout_active()["layout"] != A.ME_LAYOUT_SLAB for c in ctxs):
            return None
        for c in ctxs:
            c.quantile_begin(probs, pop)
        done = False
        while not done:
            blocks = []
            for c in ctxs:
                ptr, n = c.quantile_block()
                assert n == A.ME_QUANTILE_BLOCK
                c.synchronize()
                blocks.append(torch.as_tensor(mdist._DeviceBlock(ptr, n), device="cuda:0"))
            total = torch.stack(blocks).sum(0)
            for b in blocks:
                b.copy_(total)
            torch.cuda.synchronize()
            flags = [c.quantile_step() for c in ctxs]
            assert len(set(flags)) == 1
            done = flags[0]
        res = [c.quantile_end() for c in ctxs]
        for r in res[1:]:
            _same(r, res[0])
        return res[0]
    finally:
        for c in ctxs:
            c.close()


def test_sharded_equals_world_one(api):
    est, gt, cfg = synth.make_pair("C1", scale=0.3)
    probs = np.concatenate([FIXED_P, np.random.default_rng(4).random(20)])
    for mode, pairing in ((A.ME_CUTOFF_SQDIST_LE_R, A.ME_PAIRING_AS_WRITTEN), (A.ME_CUTOFF_DIST_LT_R, A.ME_PAIRING_GEOMETRIC)):
        p = A.make_nn_params(cfg["tau"], 1.0, cutoff_mode=mode, pairing=pairing)
        with _ctx(api, est, gt) as ctx:
            ctx.calculateMetricsWithInitialMatrix(p)
            ref = {pop: ctx.distance_quantiles(probs, pop) for pop in POPS}
        cases = [(2, False, {}), (3, False, {}), (8, False, {}), (2, True, {}), (3, True, {}),
                 (1, False, dict(max_grid_cells=64)), (2, False, dict(max_grid_cells=64))]
        for world, slab, kw in cases:
            for pop in POPS:
                got = _sharded(api, est, gt, p, probs, pop, world, slab, **kw)
                if got is None:
                    assert os.environ.get("ME_FORCE_SPARSE"), "the slab layout did not engage on a dense cell table"
                    continue
                _same(got, ref[pop])


# ---------------------------------------------------------------------------------------------------------------
# 5. contract
# ---------------------------------------------------------------------------------------------------------------
def test_contract(api):
    est, gt, cfg = synth.make_pair("C1", scale=0.1)
    p = A.make_nn_params(cfg["tau"], 1.0)
    probs = [0.5, 0.9, 0.95, 0.99]
    levels = np.linspace(0.01, 0.2, 100)
    with _ctx(api, est, gt) as ctx:
        with pytest.raises(api.MapEvalError, match="no current NN records"):
            ctx.distance_quantiles(probs)                        # before any NN evaluation
        ctx.calculateMetricsWithInitialMatrix(p)
        curve = ctx.accuracy_curve(levels)
        # deterministic
        for pop in POPS:
            _same(ctx.distance_quantiles(probs, pop), ctx.distance_quantiles(probs, pop))
        # the curve and the records are untouched by a selection
        after = ctx.accuracy_curve(levels)
        for d in DIRS:
            for f in ("n_inlier", "mean", "rmse", "fitness", "sigma"):
                np.testing.assert_array_equal(np.asarray(after[d][f]).view(np.uint64), np.asarray(curve[d][f]).view(np.uint64))
        ctx.get_nn(EST)
        # rejected probabilities and populations
        for bad in ([], [0.5] * (A.ME_QUANTILE_MAX_PROBS + 1), [np.nan], [-1e-300], [1.0 + 1e-15], [np.inf]):
            with pytest.raises(api.MapEvalError):
                ctx.distance_quantiles(bad)
        with pytest.raises(api.MapEvalError):
            ctx.distance_quantiles(probs, 7)
        assert ctx.distance_quantiles(np.linspace(0, 1, A.ME_QUANTILE_MAX_PROBS))["est_to_gt"]["n"] > 0
        # stale after me_transform and after ICP
        ctx.transform(EST, np.eye(4))
        with pytest.raises(api.MapEvalError, match="no current NN records"):
            ctx.distance_quantiles(probs)
        ctx.calculateMetricsWithInitialMatrix(p)
        ctx.distance_quantiles(probs)
        ctx.performICPRegistration(1.0, max_iteration=2)
        with pytest.raises(api.MapEvalError, match="no current NN records"):
            ctx.distance_quantiles(probs)
        # ME_DIST_NN needs want_full_cd
        ctx.calculateMetricsWithInitialMatrix(A.make_nn_params(cfg["tau"], 1.0, want_full_cd=False))
        with pytest.raises(api.MapEvalError, match="want_full_cd"):
            ctx.distance_quantiles(probs, A.ME_DIST_NN)
        assert ctx.distance_quantiles(probs, A.ME_DIST_KEPT)["est_to_gt"]["n"] > 0
        # directions = 1: gt -> est is empty
        ctx.calculateMetricsWithInitialMatrix(A.make_nn_params(cfg["tau"], 1.0, directions=1))
        for pop in POPS:
            r = ctx.distance_quantiles(probs, pop)
            assert r["est_to_gt"]["n"] > 0 and r["gt_to_est"]["n"] == 0
            assert np.all(np.isnan(r["gt_to_est"]["value"])) and np.isnan(r["gt_to_est"]["max"]) and np.isnan(r["hausdorff"])
        # a cloud change between begin and end voids the selection
        ctx.calculateMetricsWithInitialMatrix(p)
        ctx.quantile_begin(probs)
        ctx.quantile_step()
        ctx.transform(GT, np.eye(4))
        with pytest.raises(api.MapEvalError, match="changed after me_nn_quantile_begin"):
            ctx.quantile_step()
        with pytest.raises(api.MapEvalError):
            ctx.quantile_end()
        # end before the last step
        ctx.calculateMetricsWithInitialMatrix(p)
        ctx.quantile_begin(probs)
        with pytest.raises(api.MapEvalError, match="before the last"):
            ctx.quantile_end()

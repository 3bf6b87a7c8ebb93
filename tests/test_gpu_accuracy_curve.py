"""The accuracy curve (me_nn_curve*): AC / COM / CD / F1 / IoU at K thresholds from the records of the last NN evaluation.

- at the five levels of a configuration it gives what me_eval_nn gives: counts and n_ub bit for bit, values to 1e-12;
- at 200 levels it agrees with the CPU oracle run in groups of five;
- on equal-distance lattices, with levels exactly at the distances and one ulp below them, it meets the exact reference;
- sharded over 2, 3 and 8 ranks (replicated and slab layout) and on a sparse cell table it gives the world-1 counts;
- its contract: determinism, the level limits, stale records, one direction."""
import os
import sys

import mpmath as mp
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
FIELDS = ("mean", "rmse", "fitness", "sigma")
ALL_MODES = [(m, p) for m in (A.ME_CUTOFF_SQDIST_LE_R, A.ME_CUTOFF_DIST_LT_R)
             for p in (A.ME_PAIRING_AS_WRITTEN, A.ME_PAIRING_GEOMETRIC)]


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _ctx(api, est, gt, **kw):
    c = api.MapEvalB200(**kw)
    c.set_cloud(EST, est)
    c.set_cloud(GT, gt)
    return c


def _host_block(ctx, tau):
    import torch
    ptr, n = ctx.curve_accum_device(tau)
    ctx.synchronize()
    assert n == A.curve_block_len(len(tau))
    return torch.as_tensor(mdist._DeviceBlock(ptr, n), device="cuda:0").cpu().numpy().copy()


def _n_ub(block, K):
    s = 3 * (K + 1) + 1
    return int(block[s - 1]), int(block[2 * s - 1])


def _close(a, b, rtol):
    np.testing.assert_allclose(np.asarray(a, float), np.asarray(b, float), rtol=rtol, atol=0, equal_nan=True)


# ---------------------------------------------------------------------------------------------------------------
# 1. the five levels of me_eval_nn
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,scale", [("C1", 1.0), ("C2", 0.1)])
def test_five_levels_equal_eval_nn(api, name, scale):
    est, gt, cfg = synth.make_pair(name, scale=scale)
    tau5 = np.asarray(cfg["tau"], float)
    order = np.argsort(tau5, kind="stable")
    levels = tau5[order]
    with _ctx(api, est, gt) as ctx:
        for mode, pairing in ALL_MODES:
            p = A.make_nn_params(tau5, 1.0, cutoff_mode=mode, pairing=pairing)
            ref = ctx.calculateMetricsWithInitialMatrix(p)
            cur = ctx.accuracy_curve(levels)
            blk = _host_block(ctx, levels)
            assert _n_ub(blk, 5) == (ref.est_to_gt.n_ub, ref.gt_to_est.n_ub)
            for j, k in enumerate(order):          # level j of the curve is threshold k of the configuration
                for d in DIRS:
                    r = getattr(ref, d)
                    assert cur[d]["n_inlier"][j] == r.n_inlier[k], (mode, pairing, d, k)
                    for f in FIELDS:
                        _close(cur[d][f][j], getattr(r, f)[k], 1e-12)
                for f in ("cd", "f1", "iou"):
                    _close(cur[f][j], getattr(ref, f)[k], 1e-12)


# ---------------------------------------------------------------------------------------------------------------
# 2. the oracle at 200 levels
# ---------------------------------------------------------------------------------------------------------------
def test_two_hundred_levels_against_the_oracle(api):
    from oracle import oracle as O
    est, gt, cfg = synth.make_pair("C1", scale=0.2)
    levels = np.linspace(0.0, 0.25, 200)
    p = A.make_nn_params(cfg["tau"], 1.0)
    with _ctx(api, est, gt) as ctx:
        ctx.calculateMetricsWithInitialMatrix(p)
        cur = ctx.accuracy_curve(levels)
    for g0 in range(0, 200, 5):
        q = A.make_nn_params(levels[g0:g0 + 5], 1.0)
        exp = O.eval_nn(est, gt, q)
        for j in range(5):
            for d in DIRS:
                e = getattr(exp, d)
                assert cur[d]["n_inlier"][g0 + j] == e.n_inlier[j], (d, g0 + j)
                for f in FIELDS:
                    _close(cur[d][f][g0 + j], getattr(e, f)[j], 1e-9)
            for f in ("cd", "f1", "iou"):
                _close(cur[f][g0 + j], getattr(exp, f)[j], 1e-9)


# ---------------------------------------------------------------------------------------------------------------
# 3. exact arithmetic on equal-distance lattices
# ---------------------------------------------------------------------------------------------------------------
def _pair_exact(e, g, n_est, n_gt, K):
    """cd, f1, iou per level from the exact per-direction values, in mpmath (as exact_ref.nn_result at five levels)"""
    out = dict(cd=[], f1=[], iou=[])
    with mp.workdps(X.DPS):
        for k in range(K):
            r_e, r_g, fit = e["rmse"][k], g["rmse"][k], e["fitness"][k]
            out["cd"].append(float(mp.mpf(r_e) + mp.mpf(r_g)))
            out["f1"].append(float("nan") if fit + r_e == 0 else float(2 * mp.mpf(fit) * mp.mpf(r_e) / (mp.mpf(fit) + mp.mpf(r_e))))
            inter = e["n_inlier"][k]
            out["iou"].append(X.to_float(X.Fraction(inter, n_est + n_gt - inter)))
    return out


@pytest.mark.parametrize("origin", [0.0, 1500.0])
def test_levels_at_and_below_the_distances_against_exact(api, origin):
    R = 0.5
    est, gt = offset_scene(n_side=24, jitter=0.0, origin=origin, seed=3)
    for mode, pairing in ((A.ME_CUTOFF_SQDIST_LE_R, A.ME_PAIRING_AS_WRITTEN), (A.ME_CUTOFF_DIST_LT_R, A.ME_PAIRING_GEOMETRIC)):
        p = A.make_nn_params([1.0, 0.1, 0.05, 0.03, 0.0], R, cutoff_mode=mode, pairing=pairing)
        with _ctx(api, est, gt) as ctx:
            ctx.calculateMetricsWithInitialMatrix(p)
            ie, de = ctx.get_nn(EST)
            ig, dg = ctx.get_nn(GT)
            sq_e, d_e, _ = X.kept_pairs(est, gt, ie, de, R, mode)
            sq_g, d_g, ub = X.kept_pairs(gt, est, ig, dg, R, mode, as_written=pairing == A.ME_PAIRING_AS_WRITTEN)
            dist = np.unique(np.concatenate([d_e, d_g]))
            pick = dist[np.linspace(0, len(dist) - 1, min(len(dist), 120)).astype(int)]
            levels = np.unique(np.concatenate([pick, np.nextafter(pick, 0.0), [0.0, 1.0]]))
            assert len(levels) <= A.ME_CURVE_MAX_LEVELS
            cur = ctx.accuracy_curve(levels)
            blk = _host_block(ctx, levels)
        K = len(levels)
        assert _n_ub(blk, K) == (0, ub)
        e = X.dir_stats(sq_e, d_e, len(est), levels)
        g = X.dir_stats(sq_g, d_g, len(gt), levels)
        # the levels split the distance cluster: some level has pairs exactly at it, and the one ulp below excludes them
        assert len(set(e["n_inlier"])) >= 2
        for d, ex in (("est_to_gt", e), ("gt_to_est", g)):
            assert list(cur[d]["n_inlier"]) == ex["n_inlier"], d
            mean_all = float(ex["mean_all"]) if ex["mean_all"] is not None else 0.0
            for k in range(K):
                for f in ("mean", "rmse", "fitness"):
                    assert abs(cur[d][f][k] - ex[f][k]) <= X.rel_bound(ex[f][k]), (d, f, k)
                assert abs(cur[d]["sigma"][k] - ex["sigma"][k]) <= X.sigma_bound(ex["sigma"][k], mean_all), (d, k)
        res = _pair_exact(e, g, len(est), len(gt), K)
        for f in ("cd", "f1", "iou"):
            for k in range(K):
                x, xe = cur[f][k], res[f][k]
                assert (np.isnan(x) and np.isnan(xe)) or abs(x - xe) <= X.rel_bound(xe), (f, k, x, xe)


# ---------------------------------------------------------------------------------------------------------------
# 4. sharded
# ---------------------------------------------------------------------------------------------------------------
def _sharded_curve(api, est, gt, p, levels, world, slab, **kw):
    """device accumulator blocks and curve blocks of `world` contexts on cuda:0, SUM-reduced with torch"""
    import torch
    ctxs = [api.MapEvalB200(rank=r, world=world, vmd_voxel_size=0.1, **kw) for r in range(world)]
    try:
        curves = []
        for c in ctxs:
            if slab:
                c.set_layout(A.ME_LAYOUT_SLAB)
            c.set_cloud(EST, est)
            c.set_cloud(GT, gt)
            c.accum_reset()
            c.eval_nn_accum_device(p)
            curves.append(_host_block(c, levels))
        if slab and any(c.layout_active()["layout"] != A.ME_LAYOUT_SLAB for c in ctxs):
            return None
        blocks = []
        for c in ctxs:
            ptr, n_sum, n_max = c.accum_block()
            blocks.append(torch.as_tensor(mdist._DeviceBlock(ptr, n_sum + n_max), device="cuda:0"))
        blocks[0][:n_sum].copy_(torch.stack(blocks)[:, :n_sum].sum(0))
        torch.cuda.synchronize()
        e, g, _ = ctxs[0].accum_fetch(want_mme=(False, False))
        blk = np.sum(curves, axis=0)
        return api.curve_finalize(p, e, g, blk, levels, len(est), len(gt)), _n_ub(blk, len(levels))
    finally:
        for c in ctxs:
            c.close()


def test_sharded_curves_equal_world_one(api):
    est, gt, cfg = synth.make_pair("C1", scale=0.3)
    levels = np.linspace(0.0, 0.3, 64)
    for mode, pairing in ((A.ME_CUTOFF_SQDIST_LE_R, A.ME_PAIRING_AS_WRITTEN), (A.ME_CUTOFF_DIST_LT_R, A.ME_PAIRING_GEOMETRIC)):
        p = A.make_nn_params(cfg["tau"], 1.0, cutoff_mode=mode, pairing=pairing)
        with _ctx(api, est, gt) as ctx:
            ref5 = ctx.calculateMetricsWithInitialMatrix(p)
            ref = ctx.accuracy_curve(levels)
        cases = [(2, False, {}), (3, False, {}), (8, False, {}), (2, True, {}), (3, True, {}),
                 (1, False, dict(max_grid_cells=64)), (2, False, dict(max_grid_cells=64))]
        for world, slab, kw in cases:
            out = _sharded_curve(api, est, gt, p, levels, world, slab, **kw)
            if out is None:
                assert os.environ.get("ME_FORCE_SPARSE"), "the slab layout did not engage on a dense cell table"
                continue
            got, n_ub = out
            assert n_ub == (ref5.est_to_gt.n_ub, ref5.gt_to_est.n_ub), (world, slab, kw)
            for d in DIRS:
                assert list(got[d]["n_inlier"]) == list(ref[d]["n_inlier"]), (world, slab, kw, d)
                for f in FIELDS:
                    _close(got[d][f], ref[d][f], 1e-11)
            for f in ("cd", "f1", "iou"):
                _close(got[f], ref[f], 1e-11)


# ---------------------------------------------------------------------------------------------------------------
# 5. contract
# ---------------------------------------------------------------------------------------------------------------
def test_contract(api):
    est, gt, cfg = synth.make_pair("C1", scale=0.1)
    p = A.make_nn_params(cfg["tau"], 1.0)
    levels = np.linspace(0.01, 0.2, 100)
    with _ctx(api, est, gt) as ctx:
        with pytest.raises(api.MapEvalError, match="no current NN records"):
            ctx.accuracy_curve(levels)                      # before any NN evaluation
        ref = ctx.calculateMetricsWithInitialMatrix(p)
        # deterministic
        a, b = _host_block(ctx, levels), _host_block(ctx, levels)
        assert a.tobytes() == b.tobytes()
        # K = 1 and K = ME_CURVE_MAX_LEVELS
        one = ctx.accuracy_curve([0.2])
        assert one["est_to_gt"]["n_inlier"][0] == ref.est_to_gt.n_inlier[0]
        big = ctx.accuracy_curve(np.linspace(0.0, 0.3, A.ME_CURVE_MAX_LEVELS))
        assert len(big["tau"]) == A.ME_CURVE_MAX_LEVELS and np.all(np.diff(big["est_to_gt"]["n_inlier"]) >= 0)
        # rejected levels
        for bad in ([], np.linspace(0, 1, A.ME_CURVE_MAX_LEVELS + 1), [0.1, np.nan], [-0.1, 0.2], [0.2, 0.1], [0.1, np.inf]):
            with pytest.raises(api.MapEvalError):
                ctx.accuracy_curve(bad)
            with pytest.raises(api.MapEvalError):
                ctx.curve_accum_device(bad)
        # the device path of the accumulators serves the same curve
        ctx.accum_reset()
        ctx.eval_nn_accum_device(p)
        dev = ctx.accuracy_curve(levels)
        ctx.calculateMetricsWithInitialMatrix(p)
        host = ctx.accuracy_curve(levels)
        for d in DIRS:
            assert list(dev[d]["n_inlier"]) == list(host[d]["n_inlier"])
            for f in FIELDS:
                _close(dev[d][f], host[d][f], 1e-12)
        # stale after me_transform and after ICP
        ctx.transform(EST, np.eye(4))
        with pytest.raises(api.MapEvalError, match="no current NN records"):
            ctx.accuracy_curve(levels)
        ctx.calculateMetricsWithInitialMatrix(p)
        ctx.accuracy_curve(levels)
        ctx.performICPRegistration(1.0, max_iteration=2)
        with pytest.raises(api.MapEvalError, match="no current NN records"):
            ctx.accuracy_curve(levels)
        # directions = 1: only est -> gt
        p1 = A.make_nn_params(cfg["tau"], 1.0, directions=1)
        r1 = ctx.calculateMetricsWithInitialMatrix(p1)
        c1 = ctx.accuracy_curve(cfg["tau"][::-1])
        assert list(c1["est_to_gt"]["n_inlier"]) == list(r1.est_to_gt.n_inlier)[::-1]
        assert not np.any(c1["gt_to_est"]["n_inlier"]) and not np.any(c1["gt_to_est"]["rmse"])
        blk = _host_block(ctx, levels)
        s = 3 * (len(levels) + 1) + 1
        assert blk[:s - 1].sum() > 0 and not np.any(blk[s:])

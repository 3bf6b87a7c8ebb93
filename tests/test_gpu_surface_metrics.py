"""Point-to-plane AC / COM / CD / F1 / IoU and normal consistency (me_nn_surface*) from the records of the last NN evaluation.

- a known answer: an estimate shifted in-plane and by delta along the normal of a planar ground truth has e == delta for
  every est->gt pair, exact inlier counts, and normal consistency cos(angle) for normals tilted by a known angle;
- the block and the result against the numpy statement of tests/surface_ref.py in every cut-off x pairing mode, with zero,
  NaN and non-unit normals: counts and maxima bit for bit, sums to 1e-12, sigma to 1e-9;
- relations to the point-to-point table: the same pairs under geometric pairing, and more inliers per level (e <= d);
- working k-NN normals equal me_estimate_normals' and leave the clouds without normals and generalized ICP unchanged;
- sharded over 2, 3 and 8 ranks (replicated), 2 and 3 (slab, given normals) and on a sparse cell table;
- its contract: determinism, stale records, missing normals, bad knn, slab with working normals, open ICP / drift loops, a
  cloud change mid-call, one direction, and the curve, quantiles, region table and records unchanged by a surface call;
- one C3-size case (10 M vs 10 M, knn = 20): counts and maxima against numpy."""
import os
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import dist as mdist
from cloud_map_evaluation_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import surface_ref as S  # noqa: E402

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
DIRS = ("est_to_gt", "gt_to_est")
ALL_MODES = [(m, p) for m in (A.ME_CUTOFF_SQDIST_LE_R, A.ME_CUTOFF_DIST_LT_R)
             for p in (A.ME_PAIRING_AS_WRITTEN, A.ME_PAIRING_GEOMETRIC)]
EXACT = ("n_corr", "n_inlier", "n_no_normal", "n_no_normal_nn", "n_nc", "max_e", "max_e_nn")
R = 1.0


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _ctx(api, est, gt, **kw):
    c = api.MapEvalB200(**kw)
    c.set_cloud(EST, est)
    c.set_cloud(GT, gt)
    return c


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def _device(ptr, n):
    import torch
    return torch.as_tensor(mdist._DeviceBlock(ptr, n), device="cuda:0")


def _run(ctx, knn=0):
    """the world-1 loop through the split calls: (host copy of the block, result)"""
    ctx.surface_begin(knn)
    for w in (EST, GT):
        assert not ctx.surface_normals_slice(w)[2]
    ptr, n_sum, n_max = ctx.surface_block()
    assert (n_sum, n_max) == (A.ME_SURFACE_BLOCK_SUM, A.ME_SURFACE_BLOCK_MAX)
    ctx.synchronize()
    blk = _device(ptr, n_sum + n_max).cpu().numpy().copy()
    return blk, ctx.surface_end()


def _unit(v):
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def random_normals(rng, n, bad=True):
    v = _unit(rng.normal(size=(n, 3))) * rng.choice([1.0, 0.5, 2.0, 1.7], (n, 1))
    if bad:
        v[rng.random(n) < 0.04] = 0.0
        v[rng.random(n) < 0.02, 0] = np.nan
    return v


def check_block(got, want, sums_exact=False):
    """counts, n_query and maxima bit for bit; sums to 1e-12; the moments: n exact, mean 1e-12, M2 1e-9"""
    NN, W = S.NN, A.ME_MAX_WORLD
    for q in range(2):
        b, w = got[q * NN:(q + 1) * NN], want[q * NN:(q + 1) * NN]
        np.testing.assert_array_equal(b[:9], w[:9])
        np.testing.assert_array_equal(b[S.MOM:S.MOM + W], w[S.MOM:S.MOM + W])
        for lo, hi in ((9, 22),):
            if sums_exact:
                np.testing.assert_array_equal(_bits(b[lo:hi]), _bits(w[lo:hi]))
            else:
                np.testing.assert_allclose(b[lo:hi], w[lo:hi], rtol=1e-12, atol=0)
        np.testing.assert_allclose(b[S.MOM + W:S.MOM + 2 * W], w[S.MOM + W:S.MOM + 2 * W], rtol=1e-12, atol=0)
        np.testing.assert_allclose(b[S.MOM + 2 * W:], w[S.MOM + 2 * W:], rtol=1e-9, atol=0)
    x, y = got[2 * NN:], want[2 * NN:]
    for q in range(2):
        np.testing.assert_array_equal(x[4 * q:4 * q + 3], y[4 * q:4 * q + 3])
        np.testing.assert_allclose(x[4 * q + 3], y[4 * q + 3], rtol=1e-12, atol=0)
    np.testing.assert_array_equal(_bits(got[A.ME_SURFACE_BLOCK_SUM:]), _bits(want[A.ME_SURFACE_BLOCK_SUM:]))


def check_result(got, want, sums_exact=False):
    for d in DIRS:
        for f in EXACT:
            np.testing.assert_array_equal(_bits(got[d][f]) if np.asarray(got[d][f]).dtype.kind == "f" else got[d][f],
                                          _bits(want[d][f]) if np.asarray(want[d][f]).dtype.kind == "f" else want[d][f], f"{d} {f}")
        for f, tol in (("mean", 1e-12), ("rmse", 1e-12), ("fitness", 0), ("sigma", 1e-9), ("sum_nn_dist", 1e-12),
                       ("normal_consistency", 1e-12)):
            if sums_exact or tol == 0:
                np.testing.assert_array_equal(_bits(got[d][f]), _bits(want[d][f]), f"{d} {f}")
            else:
                np.testing.assert_allclose(got[d][f], want[d][f], rtol=tol, atol=0, err_msg=f"{d} {f}")
    for f in ("cd", "f1", "iou", "full_cd", "normal_consistency"):
        np.testing.assert_allclose(got[f], want[f], rtol=0 if sums_exact else 1e-9, atol=0, err_msg=f)


# ---------------------------------------------------------------------------------------------------------------
# 1. known answer
# ---------------------------------------------------------------------------------------------------------------
def test_known_answer(api):
    """delta = 2^-7 and normal scales that are powers of two make every e exactly delta and every c the same double, fl(0.8):
    the est -> gt sums are exact, sigma is 0, and the normal consistency (the normals tilted by acos 0.8) is 0.8 to 1e-15"""
    rng = np.random.default_rng(1)
    h, delta = 0.05, 2.0 ** -7
    g = np.arange(-40, 40) * h
    xy = np.stack(np.meshgrid(g, g, indexing="ij"), -1).reshape(-1, 2) + rng.uniform(-0.1 * h, 0.1 * h, (len(g) ** 2, 2))
    gt = np.column_stack([xy, np.zeros(len(xy))])
    est = gt + np.array([0.3 * h, 0.2 * h, 0.0])
    est[:, 2] = delta
    n = len(est)
    gt_n = np.zeros_like(gt)
    gt_n[:, 2] = rng.choice([1.0, -1.0, 2.0, -0.5], len(gt))             # non-unit and flipped
    est_n = np.array([3.0, 0.0, 4.0]) * rng.choice([1.0, -2.0, 0.25], (n, 1))   # |(3, 0, 4)| = 5: tilted by acos(0.8)
    tau = [0.1, 0.05, 0.02, 0.01, 0.005]                                  # delta = 0.0078125 lies between the last two
    with _ctx(api, est, gt) as ctx:
        ctx.set_normals(EST, est_n)
        ctx.set_normals(GT, gt_n)
        p = A.make_nn_params(tau, R, pairing=A.ME_PAIRING_GEOMETRIC)
        pp = ctx.calculateMetricsWithInitialMatrix(p)
        blk, r = _run(ctx)
        e = r["est_to_gt"]
        assert e["n_corr"] == n and e["n_no_normal"] == 0 and e["max_e"] == delta and e["max_e_nn"] == delta
        assert list(e["n_inlier"]) == [n] * 4 + [0]
        # every kept e is delta: the sums are exact multiples of it
        assert list(blk[9:14]) == [n * delta] * 4 + [0.0] and list(blk[14:19]) == [n * delta * delta] * 4 + [0.0]
        assert blk[21] == n * delta                                            # sum_nn_dist: every query's e
        assert list(e["mean"][:4]) == [delta] * 4 and list(e["rmse"][:4]) == [delta] * 4
        assert e["sigma"][0] == 0.0
        for d in DIRS:
            assert r[d]["n_nc"] == r[d]["n_corr"]
            np.testing.assert_allclose(r[d]["normal_consistency"], 0.8, rtol=1e-15)
        np.testing.assert_allclose(r["normal_consistency"], 0.8, rtol=1e-15)
        np.testing.assert_allclose(r["full_cd"] - r["gt_to_est"]["sum_nn_dist"] / len(gt), delta, rtol=1e-14)
        # the point-to-point table carries the in-plane sampling term
        assert pp.est_to_gt.rmse[0] > 2.0 * e["rmse"][0] and pp.est_to_gt.n_inlier[4] == 0


# ---------------------------------------------------------------------------------------------------------------
# 2. against numpy
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,scale", [("C1", 0.3), ("C2", 0.05)])
def test_against_numpy(api, name, scale):
    est, gt, cfg = synth.make_pair(name, scale=scale)
    rng = np.random.default_rng(11)
    est_n, gt_n = random_normals(rng, len(est)), random_normals(rng, len(gt))
    with _ctx(api, est, gt) as ctx:
        ctx.set_normals(EST, est_n)
        ctx.set_normals(GT, gt_n)
        for mode, pairing in ALL_MODES:
            for full in (True, False):
                p = A.make_nn_params(cfg["tau"], R, cutoff_mode=mode, pairing=pairing, want_full_cd=full)
                ctx.calculateMetricsWithInitialMatrix(p)
                rec = (ctx.get_nn(EST), ctx.get_nn(GT))
                blk, res = _run(ctx)
                want = S.block(S.fold_both(est, gt, est_n, gt_n, rec, p))
                check_block(blk, want)
                check_result(res, S.finalize(p, want, len(est), len(gt)))
                # me_nn_finalize's path end to end: the device block through the host finalizer
                check_result(res, api.surface_finalize(p, blk, len(est), len(gt)), sums_exact=True)
                assert res["est_to_gt"]["n_no_normal"] > 0 and res["gt_to_est"]["n_nc"] < res["gt_to_est"]["n_corr"]


# ---------------------------------------------------------------------------------------------------------------
# 3. relations to the point-to-point table
# ---------------------------------------------------------------------------------------------------------------
def test_relations(api):
    est, gt, cfg = synth.make_pair("C1", scale=0.3)
    rng = np.random.default_rng(4)
    with _ctx(api, est, gt) as ctx:
        ctx.set_normals(EST, random_normals(rng, len(est), bad=False))
        ctx.set_normals(GT, random_normals(rng, len(gt), bad=False))
        for mode in (A.ME_CUTOFF_SQDIST_LE_R, A.ME_CUTOFF_DIST_LT_R):
            p = A.make_nn_params(cfg["tau"], R, cutoff_mode=mode, pairing=A.ME_PAIRING_GEOMETRIC)
            pp = ctx.calculateMetricsWithInitialMatrix(p)
            r = ctx.surface_metrics()
            for d in DIRS:
                ref = getattr(pp, d)
                assert r[d]["n_corr"] == ref.n_corr and r[d]["n_no_normal"] == 0 and r[d]["n_nc"] == ref.n_corr
                assert np.all(r[d]["n_inlier"] >= np.array(list(ref.n_inlier)))
                assert r[d]["max_e"] <= np.sqrt(R) + 1e-12


# ---------------------------------------------------------------------------------------------------------------
# 4. working normals
# ---------------------------------------------------------------------------------------------------------------
def test_working_normals(api):
    """knn = 20 gives me_estimate_normals(20)'s result: bit for bit on one layout, and to rounding on a fresh context (its
    records lie in another in-cell order); the clouds have no normals afterwards, and generalized ICP estimates its own"""
    est, gt, cfg = synth.make_pair("C1", scale=0.2)
    p = A.make_nn_params(cfg["tau"], R)
    with _ctx(api, est, gt) as ref_ctx:
        ref_ctx.calculateMetricsWithInitialMatrix(p)
        ref_ctx.estimate_normals(EST, 20)
        ref_ctx.estimate_normals(GT, 20)
        _, ref = _run(ref_ctx)
    with _ctx(api, est, gt) as icp_ctx:
        T_ref, _ = mdist.icp_distributed(icp_ctx, "cuda:0", 0.5, max_iteration=5, method=A.ME_ICP_GENERALIZED)
    with _ctx(api, est, gt) as ctx:
        ctx.calculateMetricsWithInitialMatrix(p)
        blk, res = _run(ctx, knn=20)
        check_result(res, ref)
        for w in (EST, GT):
            with pytest.raises(api.MapEvalError, match="has no normals"):
                ctx.get_normals(w)
        # the records stay fresh: a second call gives the same bits, and so do the same normals made by me_estimate_normals
        np.testing.assert_array_equal(_bits(_run(ctx, knn=20)[0]), _bits(blk))
        n_gt = ctx.estimate_normals(GT, 20)
        np.testing.assert_array_equal(_bits(_run(ctx, knn=20)[0]), _bits(blk))        # est working, gt given
        np.testing.assert_array_equal(_bits(ctx.get_normals(GT)), _bits(n_gt))
        with pytest.raises(api.MapEvalError, match="has no normals"):
            ctx.get_normals(EST)
        ctx.estimate_normals(EST, 20)
        np.testing.assert_array_equal(_bits(_run(ctx)[0]), _bits(blk))
    # working normals of another k leave nothing behind for generalized ICP, which estimates its own 20-NN normals
    with _ctx(api, est, gt) as ctx:
        ctx.calculateMetricsWithInitialMatrix(p)
        ctx.surface_metrics(knn=6)
        T, _ = mdist.icp_distributed(ctx, "cuda:0", 0.5, max_iteration=5, method=A.ME_ICP_GENERALIZED)
        np.testing.assert_allclose(T, T_ref, rtol=0, atol=1e-9)


# ---------------------------------------------------------------------------------------------------------------
# 5. sharded
# ---------------------------------------------------------------------------------------------------------------
def _sharded(api, est, gt, p, world, slab, knn, normals=None, **kw):
    """`world` contexts on cuda:0: the working normals all-gathered and the blocks SUM- / MAX-reduced with torch"""
    import torch
    ctxs = [api.MapEvalB200(rank=r, world=world, vmd_voxel_size=0.1, **kw) for r in range(world)]
    try:
        for c in ctxs:
            if slab:
                c.set_layout(A.ME_LAYOUT_SLAB)
            c.set_cloud(EST, est)
            c.set_cloud(GT, gt)
            if normals is not None:
                c.set_normals(EST, normals[0])
                c.set_normals(GT, normals[1])
            c.accum_reset()
            c.eval_nn_accum_device(p)
        if slab and any(c.layout_active()["layout"] != A.ME_LAYOUT_SLAB for c in ctxs):
            return None, None
        for c in ctxs:
            c.surface_begin(knn)
        gathered = []
        for w in (EST, GT):
            sl = [c.surface_normals_slice(w) for c in ctxs]
            if not sl[0][2]:
                continue
            s = sl[0][1]
            bufs = [_device(ptr, world * s * 3) for ptr, _, _ in sl]
            for c in ctxs:
                c.synchronize()
            for r in range(world):
                for b in bufs:
                    if b is not bufs[r]:
                        b[r * s * 3:(r + 1) * s * 3].copy_(bufs[r][r * s * 3:(r + 1) * s * 3])
            torch.cuda.synchronize()
            gathered.append(bufs[0][:len(est if w == EST else gt) * 3].cpu().numpy().reshape(-1, 3).copy())
        sums, maxs = [], []
        for c in ctxs:
            ptr, n_sum, n_max = c.surface_block()
            c.synchronize()
            t = _device(ptr, n_sum + n_max)
            sums.append(t[:n_sum])
            maxs.append(t[n_sum:])
        total, top = torch.stack(sums).sum(0), torch.stack(maxs).amax(0)
        for a, b in zip(sums, maxs):
            a.copy_(total)
            b.copy_(top)
        torch.cuda.synchronize()
        res = [c.surface_end() for c in ctxs]
        for r in res[1:]:
            check_result(r, res[0], sums_exact=True)
        return res[0], gathered
    finally:
        for c in ctxs:
            c.close()


def test_sharded_equals_world_one(api):
    est, gt, cfg = synth.make_pair("C1", scale=0.3)
    rng = np.random.default_rng(8)
    given = (random_normals(rng, len(est)), random_normals(rng, len(gt)))
    for mode, pairing in ((A.ME_CUTOFF_SQDIST_LE_R, A.ME_PAIRING_AS_WRITTEN), (A.ME_CUTOFF_DIST_LT_R, A.ME_PAIRING_GEOMETRIC)):
        p = A.make_nn_params(cfg["tau"], R, cutoff_mode=mode, pairing=pairing)
        with _ctx(api, est, gt) as ctx:
            ctx.calculateMetricsWithInitialMatrix(p)
            ref_work = ctx.surface_metrics(knn=20)
            work_n = (ctx.estimate_normals(EST, 20), ctx.estimate_normals(GT, 20))
            ctx.set_normals(EST, given[0])
            ctx.set_normals(GT, given[1])
            ref_given = ctx.surface_metrics()
        cases = [(2, False, 20, None, {}), (3, False, 20, None, {}), (8, False, 20, None, {}),
                 (2, True, 0, given, {}), (3, True, 0, given, {}),
                 (1, False, 20, None, dict(max_grid_cells=64)), (2, False, 20, None, dict(max_grid_cells=64))]
        for world, slab, knn, normals, kw in cases:
            got, gathered = _sharded(api, est, gt, p, world, slab, knn, normals, **kw)
            if got is None:
                assert os.environ.get("ME_FORCE_SPARSE"), "the slab layout did not engage on a dense cell table"
                continue
            ref = ref_given if normals is not None else ref_work
            check_result(got, ref)
            if world > 1 and knn:
                assert len(gathered) == 2
                for g, w in zip(gathered, work_n):
                    np.testing.assert_array_equal(_bits(g), _bits(w))


# ---------------------------------------------------------------------------------------------------------------
# 6. contract
# ---------------------------------------------------------------------------------------------------------------
def test_contract(api):
    est, gt, cfg = synth.make_pair("C1", scale=0.1)
    p = A.make_nn_params(cfg["tau"], R)
    levels = np.linspace(0.01, 0.2, 100)
    probs = [0.5, 0.9, 0.95, 0.99]
    rng = np.random.default_rng(2)
    with _ctx(api, est, gt) as ctx:
        with pytest.raises(api.MapEvalError, match="no current NN records"):
            ctx.surface_metrics(knn=20)                               # before any NN evaluation
        ctx.calculateMetricsWithInitialMatrix(p)
        # missing normals with knn = 0, and knn out of range
        with pytest.raises(api.MapEvalError, match="estimated cloud has no normals.*me_set_normals.*me_estimate_normals"):
            ctx.surface_metrics()
        ctx.set_normals(EST, random_normals(rng, len(est)))
        with pytest.raises(api.MapEvalError, match="ground-truth cloud has no normals"):
            ctx.surface_metrics()
        for bad in (-1, 65, 1000):
            with pytest.raises(api.MapEvalError, match="knn"):
                ctx.surface_metrics(knn=bad)
        curve = ctx.accuracy_curve(levels)
        quant = ctx.distance_quantiles(probs, A.ME_DIST_NN)
        regions = ctx.region_errors(0.5)
        rec = (ctx.get_nn(EST), ctx.get_nn(GT))
        # deterministic: two calls give the same block
        np.testing.assert_array_equal(_bits(_run(ctx, knn=10)[0]), _bits(_run(ctx, knn=10)[0]))
        # the curve, the quantiles, the region table and the records are untouched by a surface call
        after = ctx.accuracy_curve(levels)
        for d in DIRS:
            for f in ("n_inlier", "mean", "rmse", "fitness", "sigma"):
                np.testing.assert_array_equal(_bits(after[d][f]), _bits(curve[d][f]))
        q2 = ctx.distance_quantiles(probs, A.ME_DIST_NN)
        for d in DIRS:
            np.testing.assert_array_equal(_bits(q2[d]["value"]), _bits(quant[d]["value"]))
        r2 = ctx.region_errors(0.5)
        for d in DIRS:
            for f in ("n_corr", "sum_d", "sum_d2", "max_d"):
                np.testing.assert_array_equal(_bits(r2[d][f]) if r2[d][f].dtype.kind == "f" else r2[d][f],
                                              _bits(regions[d][f]) if regions[d][f].dtype.kind == "f" else regions[d][f])
        for w in (EST, GT):
            i2, e2 = ctx.get_nn(w)
            np.testing.assert_array_equal(i2, rec[w][0])
            np.testing.assert_array_equal(_bits(e2), _bits(rec[w][1]))
        # calls out of order
        with pytest.raises(api.MapEvalError, match="without an open surface call"):
            ctx.surface_block()
        ctx.surface_begin(10)
        with pytest.raises(api.MapEvalError, match="still pending"):
            ctx.surface_block()
        ctx.surface_begin(10)
        ctx.surface_normals_slice(GT)
        with pytest.raises(api.MapEvalError, match="before me_nn_surface_block"):
            ctx.surface_end()
        # a cloud change between begin and end voids the call
        ctx.surface_begin(10)
        ctx.surface_normals_slice(GT)
        ctx.surface_block()
        ctx.transform(GT, np.eye(4))
        with pytest.raises(api.MapEvalError, match="changed after me_nn_surface_begin"):
            ctx.surface_end()
        ctx.calculateMetricsWithInitialMatrix(p)
        ctx.surface_begin(10)
        ctx.transform(EST, np.eye(4))
        with pytest.raises(api.MapEvalError, match="changed after me_nn_surface_begin"):
            ctx.surface_block()
        # stale after me_set_cloud
        ctx.calculateMetricsWithInitialMatrix(p)
        ctx.surface_metrics(knn=10)
        ctx.set_cloud(GT, gt)
        with pytest.raises(api.MapEvalError, match="no current NN records"):
            ctx.surface_metrics(knn=10)
        # directions = 1: only est -> gt is filled
        ctx.calculateMetricsWithInitialMatrix(A.make_nn_params(cfg["tau"], R, directions=1))
        r = ctx.surface_metrics(knn=10)
        assert r["est_to_gt"]["n_corr"] > 0 and r["gt_to_est"]["n_corr"] == 0 and r["gt_to_est"]["n_nc"] == 0
        assert np.isnan(r["gt_to_est"]["normal_consistency"]) and np.isnan(r["normal_consistency"])
        # an open registration (closed when the context is)
        ctx.calculateMetricsWithInitialMatrix(p)
        ctx.icp_begin(0.5, max_iteration=2, method=A.ME_ICP_POINT_TO_POINT)
        with pytest.raises(api.MapEvalError, match="while a registration is open"):
            ctx.surface_metrics(knn=10)
    # an open drift loop (closed when the context is)
    with _ctx(api, est, gt) as ctx:
        ctx.calculateMetricsWithInitialMatrix(p)
        ctx.drift_begin(2.0, 0.5, 2)
        with pytest.raises(api.MapEvalError, match="while a drift loop is open"):
            ctx.surface_metrics(knn=10)


def test_slab_working_normals_are_refused(api):
    est, gt, cfg = synth.make_pair("C1", scale=0.3)
    p = A.make_nn_params(cfg["tau"], R)
    ctxs = [api.MapEvalB200(rank=r, world=2, vmd_voxel_size=0.1) for r in range(2)]
    try:
        for c in ctxs:
            c.set_layout(A.ME_LAYOUT_SLAB)
            c.set_cloud(EST, est)
            c.set_cloud(GT, gt)
            c.eval_nn_accum_device(p)
        if ctxs[0].layout_active()["layout"] != A.ME_LAYOUT_SLAB:
            assert os.environ.get("ME_FORCE_SPARSE")
            return
        with pytest.raises(api.MapEvalError, match="need the replicated layout"):
            ctxs[0].surface_begin(20)
    finally:
        for c in ctxs:
            c.close()


# ---------------------------------------------------------------------------------------------------------------
# 7. C3 size
# ---------------------------------------------------------------------------------------------------------------
def test_c3_size_against_numpy(api):
    est, gt, cfg = synth.make_pair("C3")
    p = A.make_nn_params(cfg["tau"], R, pairing=A.ME_PAIRING_GEOMETRIC)
    with _ctx(api, est, gt) as ctx:
        ctx.calculateMetricsWithInitialMatrix(p)
        blk, res = _run(ctx, knn=20)
        rec = (ctx.get_nn(EST), ctx.get_nn(GT))
        est_n, gt_n = ctx.estimate_normals(EST, 20), ctx.estimate_normals(GT, 20)   # the working normals, kept this time
    want = S.block(S.fold_both(est, gt, est_n, gt_n, rec, p))
    check_block(blk, want)
    for d in DIRS:
        assert res[d]["n_corr"] > 0.9 * len(est)

"""AC / COM / CD / F1 / IoU per region (me_nn_region*) from the records of the last NN evaluation.

- one region that holds both clouds reproduces me_eval_nn's counts bit for bit and its values to 1e-12, in every cut-off x
  pairing mode;
- at several region sizes the rows partition the global accumulators: counts exactly, sums to 1e-12;
- every row equals a numpy restatement built from me_get_nn and the clouds in caller order (counts and maxima exact, sums
  to 1e-12), and every point's region is numpy's floor(x / s), on region faces, at negative coordinates and at s = 0.1;
- sharded over 2, 3 and 8 ranks (replicated and slab layout) and on a sparse cell table: counts, n_est / n_gt and maxima
  are world 1's bit for bit, sums agree to 1e-12;
- its contract: determinism, stale records, bad region sizes, index overflow, too many regions, one direction, a cloud
  change mid-call, and the curve and quantiles unchanged by a region call."""
import os
import re
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import dist as mdist
from cloud_map_evaluation_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import exact_ref as X  # noqa: E402

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
DIRS = ("est_to_gt", "gt_to_est")
ALL_MODES = [(m, p) for m in (A.ME_CUTOFF_SQDIST_LE_R, A.ME_CUTOFF_DIST_LT_R)
             for p in (A.ME_PAIRING_AS_WRITTEN, A.ME_PAIRING_GEOMETRIC)]
COUNTS = ("n_query", "n_corr", "n_inlier")
SUMS = ("sum_d", "sum_d2", "sum_nn_dist")
MAXES = ("max_d", "max_nn")
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


def restate(est, gt, s, nn, tau, mode, pairing, want_full_cd=True):
    """numpy statement of the table from the caller-order records nn = ((idx, d2) est->gt, (idx, d2) gt->est): the occupied
    regions ascending by (ix, iy, iz), n_est / n_gt, and per direction the summed and max fields"""
    idx = np.floor(np.vstack([est, gt]) / s).astype(np.int64)
    keys, inv = np.unique(idx, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    nr = len(keys)
    reg = (inv[:len(est)], inv[len(est):])
    out = {"index": keys, "n_est": np.bincount(reg[0], minlength=nr), "n_gt": np.bincount(reg[1], minlength=nr)}
    for q, (name, query, ref) in enumerate((("est_to_gt", est, gt), ("gt_to_est", gt, est))):
        ii, d2 = nn[q]
        rq = reg[q]
        D = {"n_query": np.bincount(rq[ii != -2], minlength=nr)}
        have = ii >= 0
        dn = np.sqrt(d2[have]) if want_full_cd else np.zeros(int(have.sum()))
        D["sum_nn_dist"] = np.bincount(rq[have], weights=dn, minlength=nr)
        D["max_nn"] = np.zeros(nr)
        np.maximum.at(D["max_nn"], rq[have], dn)
        keep = have & ((d2 <= R) if mode == A.ME_CUTOFF_SQDIST_LE_R else (d2 < R * R))
        qi = np.nonzero(keep)[0]
        ri = ii[qi].astype(np.int64)
        if q == 1 and pairing == A.ME_PAIRING_AS_WRITTEN:      # (gt[nn_est], est[i_gt]); out-of-range pairs left out
            ok = (ri < len(gt)) & (qi < len(est))
            qi, ri = qi[ok], ri[ok]
            diff = gt[ri] - est[qi]
        else:
            diff = query[qi] - ref[ri]
        sq = X.sqnorm_eigen(diff)
        d = np.sqrt(sq)
        rk = rq[qi]
        D["n_corr"] = np.bincount(rk, minlength=nr)
        D["max_d"] = np.zeros(nr)
        np.maximum.at(D["max_d"], rk, d)
        D["n_inlier"] = np.stack([np.bincount(rk[d <= t], minlength=nr) for t in tau], 1)
        D["sum_d"] = np.stack([np.bincount(rk, weights=np.where(d <= t, d, 0.0), minlength=nr) for t in tau], 1)
        D["sum_d2"] = np.stack([np.bincount(rk, weights=np.where(d <= t, sq, 0.0), minlength=nr) for t in tau], 1)
        out[name] = D
    return out


def check_table(got, want, exact_sums=False):
    np.testing.assert_array_equal(got["index"], want["index"])
    np.testing.assert_array_equal(got["n_est"], want["n_est"])
    np.testing.assert_array_equal(got["n_gt"], want["n_gt"])
    for d in DIRS:
        for f in COUNTS:
            np.testing.assert_array_equal(got[d][f], want[d][f], f"{d} {f}")
        for f in MAXES:
            np.testing.assert_array_equal(_bits(got[d][f]), _bits(want[d][f]), f"{d} {f}")
        for f in SUMS:
            if exact_sums:
                np.testing.assert_array_equal(_bits(got[d][f]), _bits(want[d][f]), f"{d} {f}")
            else:
                np.testing.assert_allclose(got[d][f], want[d][f], rtol=1e-12, atol=0, err_msg=f"{d} {f}")


def _records(ctx):
    return ctx.get_nn(EST), ctx.get_nn(GT)


# ---------------------------------------------------------------------------------------------------------------
# 1. one region holds everything
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,scale", [("C1", 1.0), ("C2", 0.05)])
def test_one_region_reproduces_the_whole_map(api, name, scale):
    est, gt, cfg = synth.make_pair(name, scale=scale)
    lo = np.minimum(est.min(0), gt.min(0))
    est, gt = est - lo + 1.0, gt - lo + 1.0          # the positive octant
    s = 4.0 * float(np.maximum(est.max(0), gt.max(0)).max())
    with _ctx(api, est, gt) as ctx:
        for mode, pairing in ALL_MODES:
            p = A.make_nn_params(cfg["tau"], R, cutoff_mode=mode, pairing=pairing)
            ref = ctx.calculateMetricsWithInitialMatrix(p)
            t = ctx.region_errors(s)
            assert list(t["index"][0]) == [0, 0, 0] and len(t["n_est"]) == 1
            assert (t["n_est"][0], t["n_gt"][0]) == (len(est), len(gt))
            for d, n in zip(DIRS, (len(est), len(gt))):
                r, g = getattr(ref, d), t[d]
                assert g["n_query"][0] == n and g["n_corr"][0] == r.n_corr
                assert list(g["n_inlier"][0]) == list(r.n_inlier)
                for f in ("mean", "rmse", "fitness"):
                    np.testing.assert_allclose(g[f][0], list(getattr(r, f)), rtol=1e-12, atol=0, err_msg=f)
                np.testing.assert_allclose(g["sum_nn_dist"][0], r.sum_nn_dist, rtol=1e-12)
                np.testing.assert_allclose(g["mean_nn"][0] * g["n_query"][0], g["sum_nn_dist"][0], rtol=1e-12)
            for f in ("cd", "f1", "iou"):
                np.testing.assert_allclose(t[f][0], list(getattr(ref, f)), rtol=1e-12, atol=0, err_msg=f)


# ---------------------------------------------------------------------------------------------------------------
# 2. the rows partition the global accumulators
# ---------------------------------------------------------------------------------------------------------------
def test_partition_identity(api):
    est, gt, cfg = synth.make_pair("C1", scale=0.3)
    with _ctx(api, est, gt) as ctx:
        for mode, pairing in ALL_MODES:
            p = A.make_nn_params(cfg["tau"], R, cutoff_mode=mode, pairing=pairing)
            e, g = ctx.eval_nn_accum(p)
            for s in (0.05, 0.37, 1.0, 2.5):
                t = ctx.region_errors(s)
                assert t["n_est"].sum() == len(est) and t["n_gt"].sum() == len(gt)
                assert np.all(t["n_est"] + t["n_gt"] > 0)
                for d, acc, n in zip(DIRS, (e, g), (len(est), len(gt))):
                    r = t[d]
                    assert r["n_query"].sum() == acc.n_query == n
                    assert r["n_corr"].sum() == acc.n_corr
                    assert list(r["n_inlier"].sum(0)) == list(acc.n_inlier)
                    np.testing.assert_allclose(r["sum_d"].sum(0), list(acc.sum_d), rtol=1e-12)
                    np.testing.assert_allclose(r["sum_d2"].sum(0), list(acc.sum_d2), rtol=1e-12)
                    np.testing.assert_allclose(r["sum_nn_dist"].sum(), acc.sum_nn_dist, rtol=1e-12)


# ---------------------------------------------------------------------------------------------------------------
# 3. every row against numpy
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,scale", [("C1", 0.3), ("C2", 0.05)])
def test_rows_against_numpy(api, name, scale):
    est, gt, cfg = synth.make_pair(name, scale=scale)
    modes = [(A.ME_CUTOFF_SQDIST_LE_R, A.ME_PAIRING_GEOMETRIC), (A.ME_CUTOFF_DIST_LT_R, A.ME_PAIRING_GEOMETRIC),
             (A.ME_CUTOFF_SQDIST_LE_R, A.ME_PAIRING_AS_WRITTEN)]
    with _ctx(api, est, gt) as ctx:
        for mode, pairing in modes:
            for full in (True, False):
                p = A.make_nn_params(cfg["tau"], R, cutoff_mode=mode, pairing=pairing, want_full_cd=full)
                ctx.calculateMetricsWithInitialMatrix(p)
                nn = _records(ctx)
                for s in (0.13, 0.5, 3.0):
                    check_table(ctx.region_errors(s), restate(est, gt, s, nn, cfg["tau"], mode, pairing, want_full_cd=full))


def test_region_faces_and_negative_coordinates(api):
    """points exactly on region faces (k * s and its neighbours to the ulp), negative coordinates, s = 0.1 (not
    representable): every point's region is numpy's floor(x / s)"""
    rng = np.random.default_rng(5)
    s = 0.1
    k = np.arange(-40, 41)
    face = np.stack(np.meshgrid(k * s, k[::4] * s, [-2.0 * s, 0.0, 3.0 * s], indexing="ij"), -1).reshape(-1, 3)
    ulp = np.concatenate([np.nextafter(face, np.inf), np.nextafter(face, -np.inf)])
    gt = np.vstack([face, ulp[::3], rng.uniform(-4.0, 4.0, (20000, 3))])
    est = np.vstack([face[::2] + rng.normal(0, 0.003, (len(face[::2]), 3)), ulp[1::3], rng.uniform(-4.0, 4.0, (15000, 3))])
    # the quotient of some face points rounds across the integer: those are where a wrong division would show
    q = gt / s
    assert np.any(np.floor(q) != np.round(q)) and np.any(np.floor(q) == np.round(q))
    tau = [0.2, 0.1, 0.08, 0.05, 0.01]
    with _ctx(api, est, gt) as ctx:
        for mode, pairing in ((A.ME_CUTOFF_SQDIST_LE_R, A.ME_PAIRING_AS_WRITTEN), (A.ME_CUTOFF_DIST_LT_R, A.ME_PAIRING_GEOMETRIC)):
            p = A.make_nn_params(tau, R, cutoff_mode=mode, pairing=pairing)
            ctx.calculateMetricsWithInitialMatrix(p)
            nn = _records(ctx)
            for ss in (s, 0.3, 1.0):
                t = ctx.region_errors(ss)
                check_table(t, restate(est, gt, ss, nn, tau, mode, pairing))
                np.testing.assert_array_equal(t["min"], t["index"] * ss)
                np.testing.assert_array_equal(t["max"], (t["index"] + 1) * ss)


# ---------------------------------------------------------------------------------------------------------------
# 4. sharded
# ---------------------------------------------------------------------------------------------------------------
def _sharded(api, est, gt, p, s, world, slab, **kw):
    """`world` contexts on cuda:0, the blocks SUM- / MAX-reduced with torch"""
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
        ns = [c.region_begin(s) for c in ctxs]
        assert len(set(ns)) == 1
        sums, maxs = [], []
        for c in ctxs:
            ptr, n_sum, n_max = c.region_block()
            assert (n_sum, n_max) == (2 * A.ME_REGION_SUM_FIELDS * ns[0], 2 * A.ME_REGION_MAX_FIELDS * ns[0])
            c.synchronize()
            t = torch.as_tensor(mdist._DeviceBlock(ptr, n_sum + n_max), device="cuda:0")
            sums.append(t[:n_sum])
            maxs.append(t[n_sum:])
        total, top = torch.stack(sums).sum(0), torch.stack(maxs).amax(0)
        for a, b in zip(sums, maxs):
            a.copy_(total)
            b.copy_(top)
        torch.cuda.synchronize()
        res = [c.region_end(ns[0]) for c in ctxs]
        for r in res[1:]:
            check_table(r, res[0], exact_sums=True)
        return res[0]
    finally:
        for c in ctxs:
            c.close()


def test_sharded_equals_world_one(api):
    est, gt, cfg = synth.make_pair("C1", scale=0.3)
    for mode, pairing in ((A.ME_CUTOFF_SQDIST_LE_R, A.ME_PAIRING_AS_WRITTEN), (A.ME_CUTOFF_DIST_LT_R, A.ME_PAIRING_GEOMETRIC)):
        p = A.make_nn_params(cfg["tau"], R, cutoff_mode=mode, pairing=pairing)
        for s in (0.25, 1.5):
            with _ctx(api, est, gt) as ctx:
                ctx.calculateMetricsWithInitialMatrix(p)
                ref = ctx.region_errors(s)
            cases = [(2, False, {}), (3, False, {}), (8, False, {}), (2, True, {}), (3, True, {}),
                     (1, False, dict(max_grid_cells=64)), (2, False, dict(max_grid_cells=64))]
            for world, slab, kw in cases:
                got = _sharded(api, est, gt, p, s, world, slab, **kw)
                if got is None:
                    assert os.environ.get("ME_FORCE_SPARSE"), "the slab layout did not engage on a dense cell table"
                    continue
                check_table(got, ref, exact_sums=world == 1)


# ---------------------------------------------------------------------------------------------------------------
# 5. contract
# ---------------------------------------------------------------------------------------------------------------
def _block_bits(ctx, s):
    import torch
    n = ctx.region_begin(s)
    ptr, n_sum, n_max = ctx.region_block()
    ctx.synchronize()
    out = torch.as_tensor(mdist._DeviceBlock(ptr, n_sum + n_max), device="cuda:0").cpu().numpy().view(np.uint64).copy()
    ctx.region_end(n)
    return out


def test_contract(api):
    est, gt, cfg = synth.make_pair("C1", scale=0.1)
    p = A.make_nn_params(cfg["tau"], R)
    levels = np.linspace(0.01, 0.2, 100)
    probs = [0.5, 0.9, 0.95, 0.99]
    with _ctx(api, est, gt) as ctx:
        with pytest.raises(api.MapEvalError, match="no current NN records"):
            ctx.region_errors(0.5)                                   # before any NN evaluation
        ctx.calculateMetricsWithInitialMatrix(p)
        curve = ctx.accuracy_curve(levels)
        quant = ctx.distance_quantiles(probs, A.ME_DIST_NN)
        idx, d2 = ctx.get_nn(GT)
        # deterministic: two calls give the same block
        np.testing.assert_array_equal(_block_bits(ctx, 0.5), _block_bits(ctx, 0.5))
        # the curve, the quantiles and the records are untouched by a region call
        after = ctx.accuracy_curve(levels)
        for d in DIRS:
            for f in ("n_inlier", "mean", "rmse", "fitness", "sigma"):
                np.testing.assert_array_equal(_bits(after[d][f]), _bits(curve[d][f]))
        q2 = ctx.distance_quantiles(probs, A.ME_DIST_NN)
        for d in DIRS:
            np.testing.assert_array_equal(_bits(q2[d]["value"]), _bits(quant[d]["value"]))
        i2, e2 = ctx.get_nn(GT)
        np.testing.assert_array_equal(i2, idx)
        np.testing.assert_array_equal(_bits(e2), _bits(d2))
        # bad region sizes
        for bad in (0.0, -1.0, np.nan, np.inf, -np.inf):
            with pytest.raises(api.MapEvalError, match="region_size"):
                ctx.region_errors(bad)
        # index overflow: the message names the axis and the smallest size that fits
        with pytest.raises(api.MapEvalError, match=r"along [xyz] outside \|index\| < 2\^20") as ei:
            ctx.region_errors(1e-9)
        s_fit = float(re.search(r"smallest region_size that fits is (\S+)", str(ei.value)).group(1))
        with pytest.raises(api.MapEvalError, match=r"outside \|index\|"):
            ctx.region_errors(np.nextafter(s_fit, 0.0))
        try:
            ctx.region_errors(s_fit)
        except api.MapEvalError as e:           # it fits along every axis; it may still hold too many regions
            assert "occupied regions" in str(e)
        # stale after me_transform and after me_set_cloud
        ctx.transform(EST, np.eye(4))
        with pytest.raises(api.MapEvalError, match="no current NN records"):
            ctx.region_errors(0.5)
        ctx.calculateMetricsWithInitialMatrix(p)
        ctx.region_errors(0.5)
        ctx.set_cloud(GT, gt)
        with pytest.raises(api.MapEvalError, match="no current NN records"):
            ctx.region_errors(0.5)
        # directions = 1: only the est -> gt rows are filled
        ctx.calculateMetricsWithInitialMatrix(A.make_nn_params(cfg["tau"], R, directions=1))
        t = ctx.region_errors(0.5)
        assert t["est_to_gt"]["n_query"].sum() == len(est) and t["est_to_gt"]["n_corr"].sum() > 0
        for f in COUNTS + SUMS + MAXES:
            assert not np.any(t["gt_to_est"][f]), f
        assert np.all(np.isnan(t["gt_to_est"]["mean"])) and np.all(np.isnan(t["cd"]))
        # a cloud change between begin and end voids the table; a short row buffer is refused
        ctx.calculateMetricsWithInitialMatrix(p)
        n = ctx.region_begin(0.5)
        ctx.transform(GT, np.eye(4))
        with pytest.raises(api.MapEvalError, match="changed after me_nn_region_begin"):
            ctx.region_end(n)
        ctx.calculateMetricsWithInitialMatrix(p)
        n = ctx.region_begin(0.5)
        with pytest.raises(api.MapEvalError, match="capacity"):
            ctx.region_end(n - 1)


def test_too_many_regions_are_refused(api):
    rng = np.random.default_rng(9)
    n = (A.ME_REGION_MAX_REGIONS // 2) + 20000                  # > 2^21 points in all, each alone in its region
    est, gt = rng.uniform(0.0, 100.0, (n, 3)), rng.uniform(0.0, 100.0, (n, 3))
    with _ctx(api, est, gt) as ctx:
        ctx.calculateMetricsWithInitialMatrix(A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], R))
        with pytest.raises(api.MapEvalError, match=r"occupied regions .* at most ME_REGION_MAX_REGIONS"):
            ctx.region_errors(0.001)
        assert ctx.region_errors(5.0)["n_est"].sum() == n

"""Repeated passes on one context, and the ME_PAIRING_AS_WRITTEN fold, against fresh contexts and exact arithmetic.

A context remembers the lattice plan of a cloud pair (the refined cell edge, and the boxes it was planned for), so every
pass after the first over the same clouds takes a shorter route through the lattice build.  The passes below run on one
context: the same clouds three times, then one point moved outside the remembered box, then a ground truth of another
size, and each must return what a fresh context returns for the same clouds: the same counts and the same sums up to the
order of their terms.  The trace shows which builds took the remembered box.  A non-finite coordinate must still be
refused on a remembered plan.

The gt->est direction of ME_PAIRING_AS_WRITTEN pairs every ground-truth query i with its nearest estimated point nn and
measures gt[nn] - est[i] (the reference's swapped indices; a pair whose indices run past a cloud is counted in n_ub).
The sweep leaves that squared norm in the query's record and a streaming pass folds the records; the counts must equal a
numpy restatement of the rule exactly and the sums to 1e-12, with queries finished by the far kernel among them."""
import ctypes as C

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import synth

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _fields(s, prefix="", out=None):
    """every field of a result struct, as a flat dict of python numbers"""
    out = {} if out is None else out
    for name, _ in s._fields_:
        v = getattr(s, name)
        if isinstance(v, C.Structure):
            _fields(v, f"{prefix}{name}.", out)
        else:
            out[f"{prefix}{name}"] = list(v) if isinstance(v, C.Array) else v
    return out


def _same(a, b):
    """two flat field dicts agree: counts exactly, sums to 1e-12 (the sweeps' fp64 sums take their terms in an order
    that the atomics of the lattice build choose, so two contexts agree to the last bits only)"""
    assert a.keys() == b.keys()
    for k in a:
        if all(isinstance(v, int) for v in np.atleast_1d(a[k]).tolist()):
            assert a[k] == b[k], (k, a[k], b[k])
        else:
            np.testing.assert_allclose(np.asarray(b[k], np.float64), np.asarray(a[k], np.float64), rtol=1e-12, atol=0,
                                       equal_nan=True, err_msg=k)


def _pass(ctx, est, gt, cfg, p):
    """one full pass (MME of the estimate, NN both ways, voxel stage) with the clouds handed over again"""
    ctx.set_cloud(EST, est)
    ctx.set_cloud(GT, gt)
    out = _fields(ctx.computeMME(EST, cfg["nn_radius"], 10), "mme.")
    e, g = ctx.eval_nn_accum(p)
    _fields(e, "e.", out)
    _fields(g, "g.", out)
    _fields(ctx.calculateVMD(cfg["vmd_voxel_size"], 100, 5), "awd.", out)
    return out


def _fresh(api, est, gt, cfg, p):
    with api.MapEvalB200(vmd_voxel_size=cfg["vmd_voxel_size"]) as ctx:
        return _pass(ctx, est, gt, cfg, p)


def test_repeated_passes_equal_fresh_contexts(api):
    est, gt, cfg = synth.make_pair("C2", scale=0.05)
    p = A.make_nn_params(cfg["tau"], 1.0)
    ref = _fresh(api, est, gt, cfg, p)
    moved = est.copy()
    moved[17] = est.max(axis=0) + 0.75                     # outside the remembered box of the estimate
    smaller = np.ascontiguousarray(gt[: len(gt) * 3 // 4])   # another ground truth size: another plan
    ref_moved = _fresh(api, moved, gt, cfg, p)
    ref_smaller = _fresh(api, moved, smaller, cfg, p)
    with api.MapEvalB200(vmd_voxel_size=cfg["vmd_voxel_size"]) as ctx:
        def events():
            return ctx.kernel_trace(events=True)[0] & {"ME_TEV_BOX_REMEMBERED", "ME_TEV_BOX_MISSED"}

        _same(_pass(ctx, est, gt, cfg, p), ref)
        assert events() == set()                                   # nothing remembered yet: the boxes are measured
        for _ in range(2):
            _same(_pass(ctx, est, gt, cfg, p), ref)
            assert events() == {"ME_TEV_BOX_REMEMBERED"}
        _same(_pass(ctx, moved, gt, cfg, p), ref_moved)
        assert "ME_TEV_BOX_MISSED" in events()                     # the estimate's box moved: laid out again
        _same(_pass(ctx, moved, smaller, cfg, p), ref_smaller)
        _same(_pass(ctx, est, gt, cfg, p), ref)                    # and back to the first pair


def test_non_finite_coordinate_on_a_remembered_plan(api):
    est, gt, cfg = synth.make_pair("C2", scale=0.02)
    p = A.make_nn_params(cfg["tau"], 1.0)
    with api.MapEvalB200(vmd_voxel_size=cfg["vmd_voxel_size"]) as ctx:
        for _ in range(2):
            _pass(ctx, est, gt, cfg, p)
        bad = est.copy()
        bad[123, 1] = np.nan
        ctx.set_cloud(EST, bad)
        ctx.set_cloud(GT, gt)
        with pytest.raises(api.MapEvalError) as ei:
            ctx.computeMME(EST, cfg["nn_radius"], 10)
        assert ei.value.code == A.ME_ERR_RANGE
        with pytest.raises(api.MapEvalError) as ei:
            ctx.eval_nn_accum(p)
        assert ei.value.code == A.ME_ERR_RANGE
        # the clouds of the remembered plan still evaluate as before
        _same(_pass(ctx, est, gt, cfg, p), _fresh(api, est, gt, cfg, p))


def test_points_the_library_moves_are_measured(api):
    """me_transform, a degradation operator and the drift loop move a cloud's points without a new hand-over: the next
    build measures the box instead of laying the cloud out on the old one and again (no ME_TEV_BOX_MISSED)"""
    est, gt, cfg = synth.make_pair("C2", scale=0.05)
    p = A.make_nn_params(cfg["tau"], 1.0)
    T = np.eye(4)
    T[:3, 3] = [0.31, -0.17, 0.05]
    with api.MapEvalB200(vmd_voxel_size=cfg["vmd_voxel_size"]) as ctx:
        for _ in range(2):
            _pass(ctx, est, gt, cfg, p)
        ctx.kernel_trace()
        ctx.transform(EST, T)
        ctx.eval_nn_accum(p)
        ctx.add_gaussian_noise(GT, 0.05, 7)
        ctx.eval_nn_accum(p)
        ctx.region_drift(2.0, 0.5, max_iteration=5)
        ctx.eval_nn_accum(p)
        assert "ME_TEV_BOX_MISSED" not in ctx.kernel_trace(events=True)[0]
        _pass(ctx, est, gt, cfg, p)                               # handed over again: the last measured box is the guess
        assert "ME_TEV_BOX_MISSED" in ctx.kernel_trace(events=True)[0]


def _as_written_expected(est, gt, idx_g, d2_g, p):
    """numpy restatement of the gt->est ME_PAIRING_AS_WRITTEN statistics from the records of the sweep (caller order):
    (n_corr, n_ub, n_inlier[5], sum_d[5], sum_d2[5])"""
    kept = (idx_g >= 0) & (d2_g <= p.icp_max_distance)            # ME_CUTOFF_SQDIST_LE_R
    s = idx_g[kept].astype(np.int64)                                # source index into gt
    t = np.nonzero(kept)[0]                                         # target index into est
    ok = (s < len(gt)) & (t < len(est))
    s, t = s[ok], t[ok]
    dx, dy, dz = (gt[s, k] - est[t, k] for k in range(3))
    sq = dx * dx + (dy * dy + dz * dz)                              # Eigen's squaredNorm order
    d = np.sqrt(sq)
    inl = [d <= p.tau[k] for k in range(5)]
    return (int(ok.sum()), int((~ok).sum()), [int(m.sum()) for m in inl], [float(d[m].sum()) for m in inl],
            [float(sq[m].sum()) for m in inl])


@pytest.mark.parametrize("kernel", ["rows", "flat"])
def test_as_written_fold_with_out_of_range_indices(api, monkeypatch, kernel):
    if kernel == "flat":
        monkeypatch.setenv("ME_NN_KERNEL", "flat")
    side = synth.box_side_for_density(60000)
    est = synth.uniform_box(60000, side, 11)
    gt = synth.uniform_box(83211, side, 12, noise_sigma=0.02)      # n_gt > n_est: gt queries past n_est run out of range
    rng = np.random.RandomState(3)
    # queries several cells outside the estimate's lattice, which only the far kernel resolves: 400 beyond one of its
    # corners by 0.1 - 0.4 m per axis (within the 1 m cut-off: kept pairs) and 400 metres away; first in the cloud, so
    # that their as-written pairs are in range
    lo, hi = est.min(axis=0), est.max(axis=0)
    sign = rng.choice([-1.0, 1.0], (400, 3))
    near = np.where(sign > 0, hi, lo) + sign * rng.uniform(0.1, 0.4, (400, 3))
    far = est[rng.randint(0, len(est), 400)] + rng.choice([-1.0, 1.0], (400, 3)) * (0.6 * side)
    gt = np.ascontiguousarray(np.concatenate([near, far, gt]))
    p = A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], 1.0, pairing=A.ME_PAIRING_AS_WRITTEN)
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, est)
        ctx.set_cloud(GT, gt)
        ctx.kernel_trace()
        _, g = ctx.eval_nn_accum(p)
        idx_g, d2_g = ctx.get_nn(GT)
        trace, _ = ctx.kernel_trace()
    assert ("ME_KBIT_NN_FLAT" if kernel == "flat" else "ME_KBIT_NN_ROWS_DENSE") in trace, sorted(trace)
    assert "ME_KBIT_NN_FAR" in trace, sorted(trace)
    assert (d2_g[:400] <= p.icp_max_distance).all()               # the far kernel's queries near the corners are kept
    n_corr, n_ub, n_inl, sum_d, sum_d2 = _as_written_expected(est, gt, idx_g, d2_g, p)
    assert n_ub > 0 and n_inl[0] > 0
    assert (g.n_corr, g.n_ub, list(g.n_inlier)) == (n_corr, n_ub, n_inl)
    np.testing.assert_allclose(list(g.sum_d), sum_d, rtol=1e-12)
    np.testing.assert_allclose(list(g.sum_d2), sum_d2, rtol=1e-12)

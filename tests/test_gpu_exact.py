"""The library's NN statistics and voxel-Gaussian metrics against the exact reference of tests/exact_ref.py, with the
error bounds stated there.  The oracle is not used: every expected value is the reference's definition evaluated
without rounding.

NN scenes: a ground-truth lattice of 262 144 points and est = gt + a constant offset below h / 2, so that every distance
is the same up to a jitter of 0 .. 1e-3 of the offset; at the origin and 1.5 km out; thresholds inside the distance
cluster (mean_k != mean_all) and below it (n_inlier = 0); both cut-off modes and both pairings; world 1, then the device
accumulators of 2, 3 and 8 ranks (one context per rank on one device), then the slab layout.  On a sparse cell table
(ME_FORCE_SPARSE) the slab layout is not available and its cases skip.

Voxel scenes: surfaces at 2 and 3 m voxels with 100-2 000 points per voxel, where most Gaussians have eigenvalues above
the 1e-6 clamp; degenerate voxels; every min_points edge; coordinates on and one ulp off voxel faces, at -0.0 and at
+-1.5 km; est = gt and a permutation of it; the sparse cell table.  And the device W / SCS on given Gaussians
(me_awd_from_rows) with spectra from 1e-9 to 10 m^2, 1.5 km out."""
import os
import sys

import mpmath as mp
import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import dist as mdist

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import exact_ref as X  # noqa: E402
from test_exact_ref import _sym, check_nn, check_voxel_rows, offset_scene, surface  # noqa: E402

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
R = 0.5
MODES = ((A.ME_CUTOFF_SQDIST_LE_R, A.ME_PAIRING_AS_WRITTEN), (A.ME_CUTOFF_DIST_LT_R, A.ME_PAIRING_GEOMETRIC))


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _ctx(api, est, gt, **kw):
    c = api.MapEvalB200(**kw)
    c.set_cloud(EST, est)
    c.set_cloud(GT, gt)
    return c


def _nn_scene(jitter, origin):
    est, gt = offset_scene(n_side=64, jitter=jitter, origin=origin, seed=7)
    d = np.sqrt(X.sqnorm_eigen(est - gt))
    tau = [1.0, 0.1, float(np.median(d)), float(d.min()) * 0.999, 0.03]
    return est, gt, tau


def _world1(api, est, gt, p, mode, pairing, tau):
    """the world-1 result and the exact statistics from its per-query nearest neighbours"""
    with _ctx(api, est, gt) as ctx:
        got = ctx.calculateMetricsWithInitialMatrix(p)
        ie, de = ctx.get_nn(EST)
        ig, dg = ctx.get_nn(GT)
    e = X.dir_stats(*X.kept_pairs(est, gt, ie, de, R, mode)[:2], len(est), tau)
    g = X.dir_stats(*X.kept_pairs(gt, est, ig, dg, R, mode, as_written=pairing == A.ME_PAIRING_AS_WRITTEN)[:2], len(gt), tau)
    return got, (e, g, X.nn_result(e, g, len(est), len(gt), np.sqrt(de), np.sqrt(dg)))


@pytest.mark.parametrize("origin", [0.0, 1500.0])
@pytest.mark.parametrize("jitter", [0.0, 1e-9, 1e-7, 1e-5, 1e-3])
def test_nn_statistics_are_exact_to_the_bound(api, jitter, origin):
    est, gt, tau = _nn_scene(jitter, origin)
    for mode, pairing in MODES:
        p = A.make_nn_params(tau, R, cutoff_mode=mode, pairing=pairing)
        got, (e, g, res) = _world1(api, est, gt, p, mode, pairing, tau)
        assert e["n_inlier"][3] == 0 and e["n_corr"] == len(est)
        assert jitter == 0.0 or e["mean"][2] != e["mean"][0]
        check_nn(got, e, g, res)


def _view(ptr, n):
    import torch
    return torch.as_tensor(mdist._DeviceBlock(ptr, n), device="cuda:0")


def _device_job(api, est, gt, p, world, slab):
    """one pass through the device accumulator blocks of `world` contexts on cuda:0, SUM-reduced with torch"""
    import torch
    ctxs = [api.MapEvalB200(rank=r, world=world, vmd_voxel_size=0.5) for r in range(world)]
    try:
        for c in ctxs:
            if slab:
                c.set_layout(A.ME_LAYOUT_SLAB)
            c.set_cloud(EST, est)
            c.set_cloud(GT, gt)
            c.accum_reset()
            c.eval_nn_accum_device(p)
            c.synchronize()
        if slab and any(c.layout_active()["layout"] != A.ME_LAYOUT_SLAB for c in ctxs):
            return None
        blocks = []
        for c in ctxs:
            ptr, n_sum, n_max = c.accum_block()
            blocks.append(_view(ptr, n_sum + n_max))
        red = torch.stack(blocks)[:, :n_sum].sum(0)
        blocks[0][:n_sum].copy_(red)
        torch.cuda.synchronize()
        e, g, _ = ctxs[0].accum_fetch(want_mme=(False, False))
        return ctxs[0].nn_finalize(p, e, g)
    finally:
        for c in ctxs:
            c.close()


@pytest.mark.parametrize("origin", [0.0, 1500.0])
@pytest.mark.parametrize("jitter", [1e-9, 1e-5])
def test_nn_statistics_through_the_device_accumulators_of_many_ranks(api, jitter, origin):
    """world 2, 3 and 8 on the replicated layout, then 2 and 3 on the slab layout: the same exact values to the same
    bound, whatever the number of ranks (the moments of every rank are merged, not their sums of squares)"""
    est, gt, tau = _nn_scene(jitter, origin)
    for mode, pairing in MODES:
        p = A.make_nn_params(tau, R, cutoff_mode=mode, pairing=pairing)
        ref, exact = _world1(api, est, gt, p, mode, pairing, tau)
        for world, slab in ((2, False), (3, False), (8, False), (2, True), (3, True)):
            got = _device_job(api, est, gt, p, world, slab)
            if got is None:
                assert os.environ.get("ME_FORCE_SPARSE"), "the slab layout did not engage on a dense cell table"
                continue
            assert list(got.est_to_gt.n_inlier) == list(ref.est_to_gt.n_inlier), (world, slab)
            assert list(got.gt_to_est.n_inlier) == list(ref.gt_to_est.n_inlier), (world, slab)
            check_nn(got, *exact)


def test_world_size_beyond_the_moment_slots_is_refused(api):
    with pytest.raises(api.MapEvalError, match="ME_MAX_WORLD"):
        api.MapEvalB200(rank=0, world=A.ME_MAX_WORLD + 1)
    with api.MapEvalB200() as c:
        with pytest.raises(api.MapEvalError, match="ME_MAX_WORLD"):
            c.set_shard(0, A.ME_MAX_WORLD + 1)
        c.set_shard(A.ME_MAX_WORLD - 1, A.ME_MAX_WORLD)


# ---------------------------------------------------------------------------------------------------------------
# voxel stage
# ---------------------------------------------------------------------------------------------------------------
def _vmd(api, est, gt, v, min_points, **kw):
    with _ctx(api, est, gt, vmd_voxel_size=kw.pop("vmd", v), **kw) as ctx:
        return ctx.calculateVMD(v, min_points, 5, want_rows=True)


def _check_vmd(api, est, gt, v, min_points, sample_every=1, **kw):
    got, rows = _vmd(api, est, gt, v, min_points, **kw)
    pairs, nve, nvg = X.voxel_pairs(est, gt, v, min_points)
    assert (got.n_voxels_est, got.n_voxels_gt, got.n_pairs) == (nve, nvg, len(pairs))
    checked, above = check_voxel_rows(rows, pairs, v, range(0, len(rows), sample_every))
    return got, rows, checked, above


@pytest.mark.parametrize("v", [2.0, 3.0])
def test_surface_voxels_against_exact(api, v):
    est = surface(150000, 30.0, v, seed=1)
    gt = surface(150000, 30.0, v, seed=2, origin=(0.01, -0.02, 0.03))
    got, rows, checked, above = _check_vmd(api, est, gt, v, 100, sample_every=2)
    assert checked > 50 and above >= 0.3 * checked, (checked, above)
    # AWD is the mean of W: its error is the mean of the per-row errors, each at most bound / (W + W_ex)
    pairs, _, _ = X.voxel_pairs(est, gt, v, 100)
    keys = np.floor(rows[:, 0:3] / v + 0.5).astype(np.int64)
    w_ex, slack = [], 0.0
    for r, k in zip(rows, keys):
        n_e, mu_e, m2_e, n_g, mu_g, m2_g = pairs[tuple(int(c) for c in k)]
        w2, tr = X.wasserstein2(mu_g, X.stored_sigma(n_g, m2_g), n_g, mu_e, X.stored_sigma(n_e, m2_e), n_e)
        w_ex.append(mp.sqrt(w2))
        slack += X.w_bound(tr, r[6:9], r[18:21], v) / max(r[9] + float(w_ex[-1]), 1e-300)
    awd_ex = float(sum(w_ex) / len(w_ex))
    assert abs(got.awd - awd_ex) <= slack / len(w_ex) + X.rel_bound(awd_ex)


def _noise_voxel(rng, key, v, n):
    return (np.asarray(key) + rng.uniform(0.05, 0.95, (n, 3))) * v


def test_degenerate_voxels(api):
    """identical points, two points repeated, collinear points, an axis-aligned plane (off-diagonals exactly 0), an
    isotropic lattice (a triple eigenvalue), and an eigenvalue within 1e-9 of the clamp; each in est against a noisy gt
    voxel and the other way round"""
    v = 3.0
    rng = np.random.RandomState(5)
    c = lambda key: (np.asarray(key, float) + 0.5) * v        # noqa: E731
    t = np.arange(-5, 6, dtype=np.float64)
    g5 = np.arange(5) * 0.4 - 0.8
    lat = np.stack(np.meshgrid(g5, g5, g5, indexing="ij"), -1).reshape(-1, 3)
    pl = np.stack(np.meshgrid(g5, g5, indexing="ij"), -1).reshape(-1, 2)
    near = np.sqrt(1e-3 * (1 + 1e-9) / 110.0)           # 11 points: stored M2 / 100, then / 10: eigenvalue ~1e-6 + 1e-15
    shapes = [
        lambda k: np.tile(c(k), (150, 1)),
        lambda k: np.concatenate([np.tile(c(k) - 0.3, (75, 1)), np.tile(c(k) + [0.3, -0.2, 0.1], (75, 1))]),
        lambda k: c(k) + np.outer(np.linspace(-1, 1, 150), [0.6, 0.3, -0.2]),
        lambda k: c(k) + np.column_stack([pl, np.zeros(len(pl))]),
        lambda k: c(k) + lat,
        lambda k: c(k) + np.outer(t, [near, 0.0, 0.0]),
    ]
    est_parts, gt_parts = [], []
    for i, f in enumerate(shapes):
        ka, kb = (2 * i, 0, 0), (2 * i, 2, 0)
        est_parts += [f(ka), _noise_voxel(rng, kb, v, 150)]
        gt_parts += [_noise_voxel(rng, ka, v, 150), f(kb)]
    est, gt = np.concatenate(est_parts), np.concatenate(gt_parts)
    got, rows, checked, _ = _check_vmd(api, est, gt, v, 2)
    assert got.n_pairs == 2 * len(shapes) == checked
    # the near-clamp voxel really is near the clamp
    n, _, m2 = X.exact_moments(c((10, 0, 0)) + np.outer(t, [near, 0.0, 0.0]))
    assert abs(float(m2[0][0]) / 1000 - 1e-6) < 1e-14


@pytest.mark.parametrize("min_points", [1, 2, 10, 11, 100])
def test_min_points_edges(api, min_points):
    """voxels of exactly 1, 2, 10, 11, 100 and 150 points in both clouds: pairs exist iff both have >= min_points (the
    stored covariance switches from M2 to M2 / (n - 1)^2 between 10 and 11)"""
    v = 2.0
    rng = np.random.RandomState(min_points)
    sizes = [1, 2, 10, 11, 100, 150]
    est = np.concatenate([_noise_voxel(rng, (i, j, 0), v, n) for i, n in enumerate(sizes) for j in range(len(sizes))])
    gt = np.concatenate([_noise_voxel(rng, (i, j, 0), v, n) for j, n in enumerate(sizes) for i in range(len(sizes))])
    got, _, checked, _ = _check_vmd(api, est, gt, v, min_points)
    k = sum(n >= min_points for n in sizes)
    assert got.n_pairs == k * k == checked


@pytest.mark.parametrize("where", ["origin", "+1.5km", "-1.5km"])
def test_voxel_keys_on_faces_match_ieee_floor(api, where):
    """points exactly on k v, one ulp either side, quotients IEEE rounds up to an integer (x < k v but x / v == k), -0.0:
    the voxel counts must be numpy's floor(x / v) bit for bit"""
    from fractions import Fraction
    v = 0.2
    base = {"origin": 0.0, "+1.5km": 1500.0, "-1.5km": -1500.0}[where]
    k0 = int(np.floor(base / v))
    on = np.arange(k0 - 300, k0 + 301, dtype=np.float64) * v
    cand = np.concatenate([on, np.nextafter(on, -np.inf), np.nextafter(on, np.inf)])
    # x below k v in exact arithmetic whose quotient IEEE rounds up to k
    rounds_up = np.array([x for x in cand if Fraction(float(x)) < int(np.floor(x / v)) * Fraction(v)])
    assert len(rounds_up) > 0
    near = slice(300 - 6, 300 + 7)
    vals = np.concatenate([on[near], np.nextafter(on[near], -np.inf), np.nextafter(on[near], np.inf), rounds_up[:12],
                           [0.6, -0.0, 0.0] if where == "origin" else []])
    rng = np.random.RandomState(11)
    pts = np.stack([rng.choice(vals, 4000), rng.choice(vals, 4000), rng.choice(vals, 4000)], 1)
    est, gt = np.ascontiguousarray(pts[:2000]), np.ascontiguousarray(pts[2000:])
    _check_vmd(api, est, gt, v, 1, vmd=0.0)


def test_est_equal_to_gt_and_permuted(api):
    """W(G, G) is not 0 (the Cholesky-trace quirk) and is well conditioned; a permutation of the points changes only the
    rounding of the moments"""
    v = 3.0
    gt = surface(30000, 24.0, v, seed=3, origin=(1500.0, -1500.0, 40.0))
    got, rows, checked, above = _check_vmd(api, gt.copy(), gt, v, 100, sample_every=2)
    assert checked > 20 and above >= 0.3 * checked and (rows[:, 9] > 1e-7).mean() > 0.5
    perm = np.random.RandomState(4).permutation(len(gt))
    got2, rows2, _, _ = _check_vmd(api, np.ascontiguousarray(gt[perm]), gt, v, 100, sample_every=2)
    assert (got2.n_pairs, got2.n_voxels_est) == (got.n_pairs, got.n_voxels_est)


def test_voxel_stage_on_a_sparse_cell_table(api):
    """a cell budget far below the scene's: the voxel stage runs on the sparse table (voxel_precount_kernel)"""
    v = 3.0
    est = surface(120000, 36.0, v, seed=8)
    gt = surface(120000, 36.0, v, seed=9, origin=(0.02, 0.01, -0.01))
    _check_vmd(api, est, gt, v, 100, sample_every=3, max_grid_cells=64)


# ---------------------------------------------------------------------------------------------------------------
# device W and SCS on given Gaussians
# ---------------------------------------------------------------------------------------------------------------
def _rot(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.diag(r))


SPECTRA = [(1e-9, 1e-9, 1e-9), (10.0, 1.0, 0.1), (10.0, 10.0, 1e-9), (1e-6, 1e-6 * (1 + 1e-9), 0.5), (2.0, 2.0, 2.0),
           (1e-3, 1e-5, 1e-7), (5.0, 1e-6 * (1 - 1e-9), 1e-6 * (1 + 1e-9)), (0.3, 0.3, 1e-4)]
NS = [2, 10, 11, 100, 100000]


def _stored(rng, spec, n):
    """the upper triangle of a stored covariance whose eigenvalues are spec once W has divided it by (n - 1)"""
    Rm = _rot(rng)
    S = Rm @ np.diag(spec) @ Rm.T
    st = (S + S.T) / 2 * (n - 1)
    return st[[0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]


def test_device_wasserstein_and_scs_on_synthetic_gaussians(api):
    v = 3.0
    rng = np.random.RandomState(21)
    rows, keys = [], []
    side = 6
    for i in range(side):
        for j in range(side):
            for k in range(side):
                key = np.array([500 + i, -500 + j, 13 + k])
                n_e, n_g = NS[rng.randint(len(NS))], NS[rng.randint(len(NS))]
                s_e = SPECTRA[rng.randint(len(SPECTRA))]
                s_g = SPECTRA[rng.randint(len(SPECTRA))] if rng.rand() < 0.7 else s_e
                mu_g = (key + 0.5) * v + rng.uniform(-0.5, 0.5, 3)
                dmu = rng.choice([0.0, 1e-6, 1e-3, 0.1, 1.0]) * _rot(rng)[0]
                mu_e = mu_g + dmu
                r = np.zeros(27)
                r[0:3], r[3:6] = key * v, (key + 1) * v
                r[6:9], r[10], r[11] = mu_e, n_g, n_e
                r[12:18] = _stored(rng, s_e, n_e)
                r[18:21] = mu_g
                r[21:27] = _stored(rng, s_g, n_g)
                rows.append(r)
                keys.append(tuple(int(c) for c in key))
    rows = np.array(rows)
    with api.MapEvalB200() as ctx:
        got, w = ctx.awd_from_rows(rows, v, 5)
    w_ex, w_dev, worst = {}, {}, 0.0
    for r, key, wd in zip(rows, keys, w):
        sg, se = _sym(r[21:27]).reshape(3, 3).tolist(), _sym(r[12:18]).reshape(3, 3).tolist()
        w2, tr = X.wasserstein2(r[18:21], sg, int(r[10]), r[6:9], se, int(r[11]))
        b = X.w_bound(tr, r[6:9], r[18:21], v)
        err = abs(wd * wd - float(w2))
        worst = max(worst, err / b)
        assert err <= b, (key, wd, float(mp.sqrt(w2)), err, b)
        w_ex[key], w_dev[key] = mp.sqrt(w2), wd
    # SCS of the device's own W, in mpmath: only the SCS arithmetic is compared
    scs_dev, cnt = X.scs_exact(w_dev, 5)
    assert cnt == got.n_scs and abs(got.scs - float(scs_dev)) <= 1e-12 * abs(float(scs_dev))
    # SCS of the exact W: every neighbourhood mean is far above the W error here, so they agree to the propagated bound
    scs_ex, _ = X.scs_exact(w_ex, 5)
    rel = max(abs(w_dev[k] - float(w_ex[k])) / float(w_ex[k]) for k in w_ex if w_ex[k] > 0)
    assert abs(got.scs - float(scs_ex)) <= 4 * (1 + float(scs_ex)) * rel + 1e-12
    assert got.n_pairs == len(rows)

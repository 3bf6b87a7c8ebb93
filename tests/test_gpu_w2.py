"""The Gaussian 2-Wasserstein stage (me_eval_w2, me_w2_from_rows, the me_w2_* halves) against the exact reference of
tests/w2_ref.py, with the bound stated there: analytic clouds, thickened planes, surface scenes, degenerate voxels, given
Gaussians over a grid of spectra and point counts, every min_points edge, the sparse cell table, an exact copy and a
permutation of the ground truth, slab jobs of 2 and 3 ranks on one device, and calculateVMD left as it was."""
import math
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
import w2_ref as W  # noqa: E402
from test_exact_ref import surface  # noqa: E402

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _ctx(api, est, gt, **kw):
    c = api.MapEvalB200(**kw)
    c.set_cloud(EST, est)
    c.set_cloud(GT, gt)
    return c


def _w2(api, est, gt, v, min_points=100, **kw):
    with _ctx(api, est, gt, vmd_voxel_size=v, **kw) as ctx:
        return ctx.voxel_w2(v, min_points, 5, want_rows=True)


def _check(api, est, gt, v, min_points=100, sample_every=1, **kw):
    got, rows = _w2(api, est, gt, v, min_points, **kw)
    pairs, nve, nvg = W.voxel_pairs(est, gt, v, min_points)
    assert (got.n_pairs, got.n_voxels_est, got.n_voxels_gt) == (len(pairs), nve, nvg)
    W.check_rows(rows, est, gt, v, min_points, range(0, len(rows), sample_every))
    if len(rows):
        np.testing.assert_allclose([got.aw2, got.mean_offset, got.mean_shape], rows[:, [25, 23, 24]].mean(0), rtol=1e-12)
    return got, rows


def _voxel_points(rng, key, v, n, spread=0.3):
    c = (np.asarray(key, float) + 0.5) * v
    return c + rng.uniform(-spread, spread, (n, 3)) * v


def test_affine_clouds_follow_the_closed_form(api):
    """est = mu + s (x - mu) + delta inside the gt voxel: W2^2 = |delta|^2 + (1 - s)^2 tr Sigma_gt"""
    v = 2.0
    rng = np.random.RandomState(1)
    est_parts, gt_parts, expect = [], [], {}
    for i, (s, dn) in enumerate([(1.0, 0.0), (1.0, 0.05), (0.5, 0.0), (0.8, 0.1), (1.3, 0.02), (0.0, 0.1), (0.2, 0.0)]):
        key = (i, 1, -2)
        g = _voxel_points(rng, key, v, 300, spread=0.25)
        mu = g.mean(0)
        delta = dn * _unit(rng)
        est_parts.append(mu + s * (g - mu) + delta)
        gt_parts.append(g)
        expect[key] = (dn, abs(1 - s) * math.sqrt(np.trace(np.cov(g.T))))
    est, gt = np.concatenate(est_parts), np.concatenate(gt_parts)
    got, rows = _check(api, est, gt, v, 100)
    assert got.n_pairs == len(expect)
    for r in rows:
        o, b = expect[tuple(int(c) for c in np.floor(r[0:3] / v + 0.5))]
        # s = 0 collapses the estimate to one point: its Sigma is the rounding of the moments, whose square root (w2_ref's
        # sqrt_shift) is what b can carry beyond the closed form
        assert r[23] == pytest.approx(o, abs=1e-12) and r[24] == pytest.approx(b, rel=1e-9, abs=W.sqrt_shift(300, v, 0.0))


def _unit(rng):
    x = rng.normal(size=3)
    return x / np.linalg.norm(x)


@pytest.mark.parametrize("sig_gt,sig_est", [(0.0, 0.01), (0.01, 0.01), (0.01, 0.03), (0.02, 0.005)])
def test_thickened_planes(api, sig_gt, sig_est):
    """a planar gt voxel against the same plane with normal noise: the shape term follows |sigma_est - sigma_gt| as the
    exact reference gives it, where the offset stays at the noise's sampling error"""
    v = 2.0
    rng = np.random.RandomState(int(1000 * (sig_gt + 2 * sig_est)))
    n = 4000
    est_parts, gt_parts = [], []
    for i in range(4):
        xy = rng.uniform(0.1, 1.9, (n, 2)) + [i * v, 0.0]
        gt_parts.append(np.column_stack([xy, 1.0 + rng.normal(0, sig_gt, n) if sig_gt else np.full(n, 1.0)]))
        est_parts.append(np.column_stack([xy, 1.0 + rng.normal(0, sig_est, n)]))
    est, gt = np.concatenate(est_parts), np.concatenate(gt_parts)
    got, rows = _check(api, est, gt, v, 100)
    assert got.n_pairs == 4
    np.testing.assert_allclose(rows[:, 24], abs(sig_est - sig_gt), rtol=0.1, atol=2e-3)
    assert rows[:, 23].max() < 5 * math.hypot(sig_est, sig_gt) / math.sqrt(n) + 1e-12


@pytest.mark.parametrize("v", [2.0, 3.0])
def test_surface_voxels_against_exact(api, v):
    est = surface(150000, 30.0, v, seed=1)
    gt = surface(150000, 30.0, v, seed=2, origin=(0.01, -0.02, 0.03))
    got, rows = _check(api, est, gt, v, 100, sample_every=2)
    pairs, nve, nvg = X.voxel_pairs(est, gt, v, 100)
    assert (got.n_pairs, got.n_voxels_est, got.n_voxels_gt) == (len(pairs), nve, nvg) and got.n_pairs > 50
    # SCS over the device's own W2, in mpmath
    keys = np.floor(rows[:, 0:3] / v + 0.5).astype(np.int64)
    scs, cnt = X.scs_exact({tuple(int(c) for c in k): w for k, w in zip(keys, rows[:, 25])}, 5)
    assert cnt == got.n_scs and got.scs == pytest.approx(float(scs), rel=1e-12)


def test_degenerate_voxels(api):
    """identical points, two points repeated, collinear points, an axis-aligned plane, an isotropic lattice; each in est
    against a noisy gt voxel and the other way round, and each against itself"""
    v = 3.0
    rng = np.random.RandomState(5)
    c = lambda key: (np.asarray(key, float) + 0.5) * v        # noqa: E731
    g5 = np.arange(5) * 0.4 - 0.8
    lat = np.stack(np.meshgrid(g5, g5, g5, indexing="ij"), -1).reshape(-1, 3)
    pl = np.stack(np.meshgrid(g5, g5, indexing="ij"), -1).reshape(-1, 2)
    shapes = [
        lambda k: np.tile(c(k), (150, 1)),
        lambda k: np.concatenate([np.tile(c(k) - 0.3, (75, 1)), np.tile(c(k) + [0.3, -0.2, 0.1], (75, 1))]),
        lambda k: c(k) + np.outer(np.linspace(-1, 1, 150), [0.6, 0.3, -0.2]),
        lambda k: c(k) + np.column_stack([pl, np.zeros(len(pl))]),
        lambda k: c(k) + lat,
    ]
    est_parts, gt_parts = [], []
    for i, f in enumerate(shapes):
        ka, kb, kc = (2 * i, 0, 0), (2 * i, 2, 0), (2 * i, 4, 0)
        est_parts += [f(ka), _voxel_points(rng, kb, v, 150), f(kc)]
        gt_parts += [_voxel_points(rng, ka, v, 150), f(kb), f(kc)]
    est, gt = np.concatenate(est_parts), np.concatenate(gt_parts)
    got, rows = _check(api, est, gt, v, 2)
    assert got.n_pairs == 3 * len(shapes)
    assert np.isfinite(rows).all()
    self_rows = rows[np.floor(rows[:, 1] / v + 0.5) == 4]
    assert len(self_rows) == len(shapes)


def _spd(rng, spec):
    from test_gpu_exact import _rot
    R = _rot(rng)
    S = R @ np.diag(spec) @ R.T
    return (S + S.T) / 2


def test_w2_from_rows_over_spectra_and_counts(api):
    """given Gaussians with spectra from 1e-9 to 10 m^2 (the SPECTRA x NS grid of the AWD test), 1.5 km out"""
    from test_gpu_exact import NS, SPECTRA
    v = 3.0
    rng = np.random.RandomState(21)
    rows, keys = [], []
    side = 6
    for i in range(side):
        for j in range(side):
            for k in range(side):
                key = np.array([500 + i, -500 + j, 13 + k])
                s_e = SPECTRA[rng.randint(len(SPECTRA))]
                s_g = SPECTRA[rng.randint(len(SPECTRA))] if rng.rand() < 0.7 else s_e
                mu_g = (key + 0.5) * v + rng.uniform(-0.5, 0.5, 3)
                mu_e = mu_g + rng.choice([0.0, 1e-6, 1e-3, 0.1, 1.0]) * _unit(rng)
                Se = _spd(rng, s_e)
                Sg = Se.copy() if s_g is s_e and rng.rand() < 0.5 else _spd(rng, s_g)
                rows.append(W.to_row(key, v, NS[rng.randint(len(NS))], NS[rng.randint(len(NS))], mu_e, mu_g, Se, Sg))
                keys.append(tuple(int(c) for c in key))
    rows = np.array(rows)
    with api.MapEvalB200() as ctx:
        got, w = ctx.w2_from_rows(rows, v, 5)
    assert got.n_pairs == len(rows)
    for r, key, (o, b, w2) in zip(rows, keys, w):
        Se = np.zeros((3, 3)); Se[W.UPPER] = r[11:17]; Se = Se + np.triu(Se, 1).T
        Sg = np.zeros((3, 3)); Sg[W.UPPER] = r[17:23]; Sg = Sg + np.triu(Sg, 1).T
        o2, b2 = W.w2_exact(r[8:11], Sg.tolist(), r[5:8], Se.tolist())
        # the rows are exact doubles: only the eigen-decompositions round, by u |Sigma| per entry
        db = sum(math.sqrt(3) * min(math.sqrt(3 * e), 3 * e / math.sqrt(lm) if lm > 0 else math.inf)
                 for e, lm in ((W.C_BOUND * W.U * np.abs(S).max(), W.lambda_min(S.tolist())) for S in (Se, Sg)))
        db += W.C_BOUND * W.U * math.sqrt(np.trace(Se) + np.trace(Sg))
        bx = float(mp.sqrt(b2))
        bound = W.C_BOUND * W.U * float(mp.sqrt(o2)) * (np.abs(r[5:11]).sum() + 2 * v) + db * (2 * bx + db)
        assert abs(w2 * w2 - float(o2 + b2)) <= bound, (key, o, b, float(mp.sqrt(o2)), bx, bound)
        assert abs(b - bx) <= db
    scs, cnt = X.scs_exact({k: x for k, x in zip(keys, w[:, 2])}, 5)
    assert cnt == got.n_scs and got.scs == pytest.approx(float(scs), rel=1e-12)
    np.testing.assert_allclose([got.aw2, got.mean_offset, got.mean_shape], w[:, [2, 0, 1]].mean(0), rtol=1e-12)


@pytest.mark.parametrize("min_points", [2, 10, 100])
def test_min_points_edges(api, min_points):
    v = 2.0
    rng = np.random.RandomState(min_points)
    sizes = [1, 2, 10, 11, 100, 150]
    est = np.concatenate([_voxel_points(rng, (i, j, 0), v, n, 0.45) for i, n in enumerate(sizes) for j in range(len(sizes))])
    gt = np.concatenate([_voxel_points(rng, (i, j, 0), v, n, 0.45) for j, n in enumerate(sizes) for i in range(len(sizes))])
    got, _ = _check(api, est, gt, v, min_points)
    k = sum(n >= min_points for n in sizes)
    assert got.n_pairs == k * k


def test_refusals(api):
    est = surface(20000, 10.0, 2.0, seed=1)
    with _ctx(api, est, est.copy()) as ctx:
        for args in ((2.0, 1), (2.0, 0), (0.0, 100), (-1.0, 100)):
            with pytest.raises(api.MapEvalError) as e:
                ctx.voxel_w2(*args)
            assert e.value.code == A.ME_ERR_INVALID
        with pytest.raises(api.MapEvalError) as e:
            ctx.voxel_w2(1e-3, 100)
        assert e.value.code == A.ME_ERR_RANGE
        for fn in (ctx.w2_w_table, ctx.w2_fetch, ctx.w2_block, lambda: ctx.w2_finish_accum_device(5)):
            with pytest.raises(api.MapEvalError):
                fn()
        assert ctx.voxel_w2(2.0, 100).n_pairs > 0


def test_voxel_stage_on_a_sparse_cell_table(api):
    v = 3.0
    est = surface(120000, 36.0, v, seed=8)
    gt = surface(120000, 36.0, v, seed=9, origin=(0.02, 0.01, -0.01))
    _check(api, est, gt, v, 100, sample_every=3, max_grid_cells=64)


def test_exact_copy_and_permutation_stay_below_the_threshold(api):
    v = 3.0
    gt = surface(30000, 24.0, v, seed=3, origin=(1500.0, -1500.0, 40.0))
    perm = np.random.RandomState(4).permutation(len(gt))
    for est in (gt.copy(), np.ascontiguousarray(gt[perm])):
        got, rows = _check(api, est, gt, v, 100, sample_every=4)
        assert got.n_pairs > 20
        assert rows[:, 25].max() < W.THRESHOLD, rows[:, 25].max()


def _view(ptr, n):
    import torch
    return torch.as_tensor(mdist._DeviceBlock(ptr, n), device="cuda:0")


@pytest.mark.parametrize("world", [2, 3])
def test_slab_job_matches_world_one(api, world):
    """ranks as contexts on one device; the MAX all-reduce of the W2 table and the SUM all-reduce of the block done here"""
    import torch
    est, gt, cfg = synth.make_pair("C3", scale=0.02)
    v = cfg["vmd_voxel_size"]
    with _ctx(api, est, gt, vmd_voxel_size=v) as c:
        ref = c.voxel_w2(v, 20, 5)
        assert A.struct_to_dict(mdist.w2_distributed(c, "cuda:0", v, 20, 5)) == pytest.approx(A.struct_to_dict(ref), rel=1e-12,
                                                                                               nan_ok=True)
    ctxs = []
    try:
        for r in range(world):
            c = api.MapEvalB200(rank=r, world=world, vmd_voxel_size=v)
            c.set_layout(A.ME_LAYOUT_SLAB)
            c.set_cloud(EST, est)
            c.set_cloud(GT, gt)
            ctxs.append(c)
        for c in ctxs:
            c.w2_begin(v, 20)
            c.synchronize()
        assert all(c.layout_active()["layout"] == A.ME_LAYOUT_SLAB for c in ctxs)
        tabs = [_view(*c.w2_w_table()) for c in ctxs]
        assert int(torch.stack([(t >= 0).to(torch.int32) for t in tabs]).sum(0).max()) <= 1
        m = torch.stack(tabs).max(0).values
        for t in tabs:
            t.copy_(m)
        torch.cuda.synchronize()
        for c in ctxs:
            c.w2_finish_accum_device(5)
            c.synchronize()
        blocks = [_view(*c.w2_block()) for c in ctxs]
        red = torch.stack(blocks).sum(0)
        for b in blocks:
            b.copy_(red)
        torch.cuda.synchronize()
        outs = [c.w2_fetch() for c in ctxs]
    finally:
        for c in ctxs:
            c.close()
    for o in outs:
        for k in ("n_pairs", "n_scs", "n_voxels_est", "n_voxels_gt"):
            assert getattr(o, k) == getattr(ref, k), k
        np.testing.assert_allclose([o.aw2, o.mean_offset, o.mean_shape, o.scs], [ref.aw2, ref.mean_offset, ref.mean_shape, ref.scs],
                                   rtol=1e-11)
    assert ref.n_pairs > 50 and ref.n_scs > 0


def test_calculate_vmd_is_unchanged_by_the_stage(api):
    """calculateVMD's rows on one context are bit-identical whether or not voxel_w2 ran before it, and its counts are the
    same; its sums agree to the order of the atomic additions that form them, as between any two calls"""
    est, gt, cfg = synth.make_pair("C2", scale=0.05)
    v = cfg["vmd_voxel_size"]

    def vmd(ctx):
        res, rows = ctx.calculateVMD(v, 100, 5, want_rows=True)
        return A.struct_to_dict(res), rows[np.lexsort(rows[:, 2::-1].T)]

    with _ctx(api, est, gt, vmd_voxel_size=v) as ctx:
        runs = [vmd(ctx)]
        w = [ctx.voxel_w2(v, 100)]
        runs.append(vmd(ctx))
        w.append(ctx.voxel_w2(v, 100, want_rows=True)[0])
        runs.append(vmd(ctx))
    (a, ra), others = runs[0], runs[1:]
    assert a["n_pairs"] > 0
    for b, rb in others:
        assert ra.tobytes() == rb.tobytes()
        for k in ("n_pairs", "n_scs", "n_voxels_est", "n_voxels_gt", "n_active", "n_old", "n_new"):
            assert a[k] == b[k], k
        assert b["awd"] == pytest.approx(a["awd"], rel=1e-13) and b["scs"] == pytest.approx(a["scs"], rel=1e-13)
    assert w[0].n_pairs == w[1].n_pairs > 0
    assert w[1].aw2 == pytest.approx(w[0].aw2, rel=1e-13)

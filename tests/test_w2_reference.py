"""The exact W2 reference of tests/w2_ref.py on its own, on the CPU: closed forms of the Bures distance, symmetry, the
triangle inequality, scipy's fp64 sqrtm, and the demonstration behind w2_ref.THRESHOLD (the trace formula against the
residual form in numpy fp64 on an exact copy of a surface scene)."""
import math
import os
import sys

import mpmath as mp
import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import exact_ref as X  # noqa: E402
import w2_ref as W  # noqa: E402
from test_exact_ref import surface  # noqa: E402


def _rot(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.diag(r))


def _spd(rng, spec):
    R = _rot(rng)
    S = R @ np.diag(spec) @ R.T
    return (S + S.T) / 2


def _b(Sg, Se):
    return float(mp.sqrt(W.w2_exact([0, 0, 0], Sg.tolist(), [0, 0, 0], Se.tolist())[1]))


@pytest.mark.parametrize("s", [0.0, 0.5, 1.0, 1.7, 3.0])
def test_scaled_covariance(s):
    """Sigma_est = s^2 Sigma_gt gives b = |1 - s| sqrt(tr Sigma_gt)"""
    Sg = _spd(np.random.RandomState(1), [2.0, 0.3, 1e-3])
    assert _b(Sg, s * s * Sg) == pytest.approx(abs(1 - s) * math.sqrt(np.trace(Sg)), rel=1e-12, abs=1e-14)


def test_diagonal_covariances():
    a, b = np.array([4.0, 0.25, 1e-6]), np.array([1.0, 0.36, 0.0])
    assert _b(np.diag(a), np.diag(b)) ** 2 == pytest.approx(float(((np.sqrt(a) - np.sqrt(b)) ** 2).sum()), rel=1e-12)


def test_equal_covariances_leave_the_offset():
    rng = np.random.RandomState(2)
    S = _spd(rng, [0.5, 0.1, 0.0])
    mu_g, mu_e = rng.normal(size=3), rng.normal(size=3)
    o2, b2 = W.w2_exact(mu_g, S.tolist(), mu_e, S.tolist())
    assert float(b2) < 1e-40 and float(mp.sqrt(o2)) == pytest.approx(float(np.linalg.norm(mu_e - mu_g)), rel=1e-15)


def test_symmetric_and_a_metric():
    rng = np.random.RandomState(3)
    for _ in range(20):
        G = [(rng.normal(size=3), _spd(rng, rng.choice([1e-6, 0.01, 0.3, 2.0], 3))) for _ in range(3)]
        w = lambda i, j: float(mp.sqrt(sum(W.w2_exact(G[i][0], G[i][1].tolist(), G[j][0], G[j][1].tolist()))))  # noqa: E731
        assert w(0, 1) == pytest.approx(w(1, 0), rel=1e-30, abs=1e-30)
        assert w(0, 2) <= w(0, 1) + w(1, 2) + 1e-30


def test_against_scipy_sqrtm():
    from scipy.linalg import sqrtm
    rng = np.random.RandomState(4)
    for _ in range(20):
        Sg, Se = _spd(rng, rng.uniform(0.01, 3, 3)), _spd(rng, rng.uniform(0.01, 3, 3))
        A = np.real(sqrtm(Sg))
        b2 = np.trace(Sg) + np.trace(Se) - 2 * np.trace(np.real(sqrtm(A @ Se @ A)))
        assert _b(Sg, Se) ** 2 == pytest.approx(b2, rel=1e-10, abs=1e-13)
        assert W.b_residual64(Sg, Se) ** 2 == pytest.approx(b2, rel=1e-10, abs=1e-13)


def test_exact_gaussian_is_the_unbiased_covariance():
    pts = np.random.RandomState(5).normal(size=(50, 3))
    n, mu, S = W.exact_gaussian(pts)
    np.testing.assert_allclose(np.array([[float(x) for x in r] for r in S]), np.cov(pts.T), rtol=1e-13)
    np.testing.assert_allclose([float(x) for x in mu], pts.mean(0), rtol=1e-14)


def test_threshold_separates_the_trace_formula_from_the_residual_form():
    """On an exact copy of a surface scene (the points of each voxel summed in another order), in fp64: the trace formula's b
    exceeds THRESHOLD on a large share of the voxels, the residual form's b stays 100 times below it on every voxel.  The
    GPU tests hold an exact copy and a permutation to THRESHOLD."""
    for v in (2.0, 3.0):
        pts = surface(60000, 24.0, v, seed=3, origin=(1500.0, -1500.0, 40.0))
        groups = {k: pts[i] for k, i in X.voxel_groups(pts, v).items() if len(i) >= 100}
        keys = sorted(groups)[:120]
        bt, br = W.trace_and_residual_floors({k: groups[k] for k in keys}, v)
        assert (bt > W.THRESHOLD).mean() > 0.25 and bt.max() > 100 * W.THRESHOLD, (np.median(bt), bt.max())
        assert br.max() < W.THRESHOLD / 100, br.max()


def test_bound_holds_for_fp64_on_a_surface_voxel():
    """the W2^2 bound covers the numpy fp64 residual form on a perturbed copy"""
    v = 2.0
    rng = np.random.RandomState(6)
    gt = surface(20000, 8.0, v, seed=7)
    est = gt + rng.normal(0, 0.01, gt.shape)
    pairs, _, _ = W.voxel_pairs(est, gt, v, 100)
    for key in sorted(pairs)[:10]:
        ie, ig = pairs[key]
        ex = W.pair_exact(est[ie], gt[ig], v)
        c = (np.asarray(key) + 0.5) * v
        Se, Sg = W.fp64_sigma(est[ie], c), W.fp64_sigma(gt[ig], c)
        o = float(np.linalg.norm(est[ie].mean(0) - gt[ig].mean(0)))
        b = W.b_residual64(Sg, Se)
        assert abs(o * o + b * b - ex["w2sq"]) <= ex["bound"]

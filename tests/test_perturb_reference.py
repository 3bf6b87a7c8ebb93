"""The numpy statement of the simulation operators (tests/perturb_ref.py) against the reference's definitions
(map_eval.cpp:1745-1829): the distributions its std::mt19937 draws have, the (int) truncation of the outlier count, and
the geometry of the local deformation.  Statistical bounds are 5 sigma; the draws are seeded, so every check is
deterministic."""
import math
import os
import sys

import numpy as np
import pytest
from scipy import stats

from cloud_map_evaluation_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import perturb_ref as ref  # noqa: E402

SEED = synth.EST_SEED
N = 1_000_000


@pytest.fixture(scope="module")
def cloud():
    return synth.uniform_box(N, 4.0, synth.GT_SEED, origin=(0.123, 0.456, 0.0))


def test_uniform53_and_uniform24_share_the_hash():
    idx = np.arange(100_000, dtype=np.uint64)
    for lane in (0, 6, 7, 13):
        u53 = ref.uniform53(SEED, idx, lane)
        u24 = synth.uniform24(SEED, idx, lane).astype(np.float64)
        assert ((u53 >= 0) & (u53 < 1)).all()
        np.testing.assert_array_equal(np.floor(u53 * 2.0 ** 24) * 2.0 ** -24, u24)   # h >> 40 = (h >> 11) >> 29


def test_gaussian_noise_moments(cloud):
    """addGaussianNoise: independent N(0, sigma^2) per axis, every point"""
    sigma = 0.05
    d = ref.gaussian_noise(cloud, sigma, SEED) - cloud
    assert np.isfinite(d).all()
    for a in range(3):
        assert abs(d[:, a].mean()) < 5 * sigma / math.sqrt(N), a
        assert abs(d[:, a].var() - sigma ** 2) < 5 * sigma ** 2 * math.sqrt(2.0 / N), a
    r = np.corrcoef(d.T)
    for a, b in ((0, 1), (0, 2), (1, 2)):
        assert abs(r[a, b]) < 5 / math.sqrt(N), (a, b)
    # ... and independent of the position (the noise lanes are not the coordinates' lanes)
    assert abs(np.corrcoef(d[:, 0], cloud[:, 0])[0, 1]) < 5 / math.sqrt(N)
    np.testing.assert_array_equal(ref.gaussian_noise(cloud, 0.0, SEED), cloud)
    assert not np.array_equal(ref.gaussian_noise(cloud[:100], sigma, SEED + 1), ref.gaussian_noise(cloud[:100], sigma, SEED))


def test_non_uniform_density_keep_shares(cloud):
    """addNonUniformDensity: a point in a region where sin(x / s pi) sin(y / s pi) > 0 is kept with probability sparse,
    elsewhere with probability dense; 1 keeps everything and 0 nothing"""
    sparse, dense, s = 0.3, 0.8, 0.5
    keep, xn, yn = ref.density_keep(cloud, sparse, dense, s, SEED)
    pos = xn * yn > 0
    for mask, p in ((pos, sparse), (~pos, dense)):
        k = mask.sum()
        assert k > N // 4
        assert abs(keep[mask].sum() - p * k) < 5 * math.sqrt(k * p * (1 - p))
    # the reference's own expression, point by point on a sample
    for i in range(0, N, 9973):
        x, y = cloud[i, 0], cloud[i, 1]
        xr, yr = math.sin(x / s * math.pi), math.sin(y / s * math.pi)
        assert (xr * yr > 0) == pos[i]
    pts, nrm = ref.non_uniform_density(cloud, sparse, dense, s, SEED, normals=cloud * 2)
    np.testing.assert_array_equal(pts, cloud[keep])              # stable: caller order kept
    np.testing.assert_array_equal(nrm, 2 * cloud[keep])
    np.testing.assert_array_equal(ref.non_uniform_density(cloud, 1.0, 1.0, s, SEED), cloud)
    assert len(ref.non_uniform_density(cloud, 0.0, 0.0, s, SEED)) == 0
    # region_size 0: NaN signs, every point takes the dense ratio
    keep0, _, _ = ref.density_keep(cloud[:1000], 0.0, 1.0, 0.0, SEED)
    assert keep0.all()


def test_sparse_outliers_count_bases_and_offsets(cloud):
    """addSparseOutliers: (int)(N ratio) outliers, bases uniform over the points, offsets N(0, range^2) per axis"""
    ratio, rng = 0.2, 0.7
    m = ref.outlier_count(N, ratio)
    assert m == int(N * ratio) == 200_000
    out = ref.sparse_outliers(cloud, ratio, rng, SEED)
    assert out.shape == (N + m, 3)
    np.testing.assert_array_equal(out[:N], cloud)
    base = ref.outlier_bases(N, m, SEED)
    assert base.min() >= 0 and base.max() <= N - 1
    hist = np.bincount(base // (N // 100), minlength=100)
    assert stats.chisquare(hist).pvalue > 1e-6
    z = (out[N:] - cloud[base]) / rng
    for a in range(3):
        assert abs(z[:, a].mean()) < 5 / math.sqrt(m)
        assert abs(z[:, a].var() - 1) < 5 * math.sqrt(2.0 / m)
        assert stats.kstest(z[:, a], "norm").pvalue > 1e-6
    # static_cast<int> truncates the product as rounded in fp64
    for n, r in ((10, 0.7), (100, 0.29), (1000, 0.0015), (7, 0.999), (5, -0.5), (0, 0.3)):
        assert ref.outlier_count(n, r) == max(0, math.trunc(n * r)), (n, r)
    assert ref.outlier_count(100, 0.29) == 28            # 28.999999999999996
    with pytest.raises(OverflowError):
        ref.outlier_count(1000, 2.2e6)
    np.testing.assert_array_equal(ref.sparse_outliers(cloud[:3], 0.2, rng, SEED), cloud[:3])   # (int)(0.6) = 0


def test_local_deformation_geometry():
    """addLocalDeformation: inside the radius every point moves radially away from the centre by strength * w,
    w = 0.5 (1 + cos(pi d / r)); at d >= r nothing moves; the centre point stays"""
    c = np.array([1.0, -2.0, 0.5])
    r, strength = 1.5, 0.2
    pts = synth.uniform_box(200_000, 4.0, synth.GT_SEED) + (c - 2.0)
    pts = np.concatenate([pts, [c], c + [[r, 0, 0], [0, -r, 0], [0, 0, r]]])
    out = ref.local_deformation(pts, r, strength, c)
    v = pts - c
    d = np.sqrt(v[:, 0] ** 2 + (v[:, 1] ** 2 + v[:, 2] ** 2))
    inside = d < r
    assert inside.sum() > 10_000 and (~inside).sum() > 10_000
    np.testing.assert_array_equal(out[~inside], pts[~inside])
    np.testing.assert_array_equal(out[-4:], pts[-4:])            # centre and three points on the sphere
    mv = inside & (d > 0)
    disp = out[mv] - pts[mv]
    w = 0.5 * (1 + np.cos(np.pi * d[mv] / r))
    mag = np.linalg.norm(disp, axis=1)
    np.testing.assert_allclose(mag, strength * w, rtol=1e-9, atol=1e-15)
    cosang = np.einsum("ij,ij->i", disp, v[mv]) / (mag * d[mv])
    assert (cosang[mag > 1e-12] > 1 - 1e-9).all()                # radial, outward
    # the reference's expression point by point (Python floats are IEEE doubles)
    for i in list(range(0, len(pts) - 4, 997)) + [len(pts) - 4]:
        p = pts[i]
        dv = [p[0] - c[0], p[1] - c[1], p[2] - c[2]]
        dist = math.sqrt(dv[0] * dv[0] + (dv[1] * dv[1] + dv[2] * dv[2]))
        q = list(p)
        if dist < r:
            weight = 0.5 * (1 + math.cos(math.pi * dist / r))
            z = dv[0] * dv[0] + (dv[1] * dv[1] + dv[2] * dv[2])
            direction = [x / math.sqrt(z) for x in dv] if z > 0 else dv
            q = [q[a] + direction[a] * strength * weight for a in range(3)]
        np.testing.assert_allclose(out[i], q, rtol=0, atol=4e-16 * (abs(strength) + np.abs(p)).max())
    # radius <= 0 moves nothing
    np.testing.assert_array_equal(ref.local_deformation(pts, 0.0, strength, c), pts)
    np.testing.assert_array_equal(ref.local_deformation(pts, -1.0, strength, c), pts)

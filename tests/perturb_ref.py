"""numpy statement of the four simulation operators (me_add_gaussian_noise, me_add_non_uniform_density,
me_add_sparse_outliers, me_add_local_deformation), built on synth.py's counter-based hash.

The reference's operators (MapEval::addGaussianNoise / addNonUniformDensity / addSparseOutliers / addLocalDeformation,
map_eval.cpp:1745-1829) draw from std::random_device; here every draw is uniform24 / gaussian of synth.py at a fixed lane,
or uniform53 = (h >> 11) * 2^-53 from the same hash h.  Every function returns new arrays and leaves its input alone.
tests/test_perturb_reference.py checks these against the reference's definitions; tests/test_gpu_perturb.py checks the
device against these.
"""
import numpy as np

from cloud_map_evaluation_b200 import synth

NOISE_LANE = 0          # gaussian(seed, i, 2a): lanes 0-5
DENSITY_LANE = 6
OUTLIER_BASE_LANE = 7
OUTLIER_OFFSET_LANE = 8  # gaussian(seed, j, 8 + 2a): lanes 8-13


def _hash(seed, idx, lane):
    """the 64-bit hash synth.uniform24 takes its 24 bits from"""
    with np.errstate(over="ignore"):
        s = synth._mix(np.uint64(seed) + np.uint64(lane) * np.uint64(0xD1B54A32D192ED03))
        return synth._mix(s ^ (np.asarray(idx, dtype=np.uint64) * np.uint64(0x2545F4914F6CDD1D) + np.uint64(lane)))


def uniform53(seed, idx, lane):
    """53-bit uniform in [0, 1) as fp64 from the same hash as uniform24"""
    return (_hash(seed, idx, lane) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def gaussian_noise(xyz, std_dev, seed):
    """p_a += std_dev * gaussian(seed, i, 2a); std_dev = 0 returns the cloud unchanged"""
    out = np.array(xyz, dtype=np.float64, copy=True)
    if std_dev == 0 or len(out) == 0:
        return out
    idx = np.arange(len(out), dtype=np.uint64)
    for a in range(3):
        out[:, a] = out[:, a] + std_dev * synth.gaussian(seed, idx, NOISE_LANE + 2 * a)
    return out


def density_keep(xyz, sparse_ratio, dense_ratio, region_size, seed):
    """(keep mask, xn, yn): the reference's sin(x / region_size * M_PI) signs select the threshold"""
    xyz = np.asarray(xyz, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        xn = np.sin(xyz[:, 0] / region_size * np.pi)
        yn = np.sin(xyz[:, 1] / region_size * np.pi)
        threshold = np.where(xn * yn > 0, sparse_ratio, dense_ratio)
    # the fp32 uniform widened to fp64 before the comparison (a bare float32 array would compare in float32)
    u = synth.uniform24(seed, np.arange(len(xyz), dtype=np.uint64), DENSITY_LANE).astype(np.float64)
    return u < threshold, xn, yn


def non_uniform_density(xyz, sparse_ratio, dense_ratio, region_size, seed, normals=None):
    """stable compaction of the kept points (and of their normals)"""
    keep, _, _ = density_keep(xyz, sparse_ratio, dense_ratio, region_size, seed)
    pts = np.ascontiguousarray(np.asarray(xyz, dtype=np.float64)[keep])
    return pts if normals is None else (pts, np.ascontiguousarray(np.asarray(normals)[keep]))


def outlier_count(n, outlier_ratio):
    """static_cast<int>(points_.size() * outlier_ratio); none for a negative ratio"""
    want = float(n) * float(outlier_ratio)
    if not want < 2.0 ** 31:
        raise OverflowError("N * outlier_ratio >= 2^31")
    return int(want) if want > 0 else 0


def outlier_bases(n, m, seed):
    """base index of outlier j = min(floor(uniform53(seed, j, 7) * N), N - 1)"""
    u = uniform53(seed, np.arange(m, dtype=np.uint64), OUTLIER_BASE_LANE)
    return np.minimum(np.floor(u * float(n)), n - 1).astype(np.int64)


def sparse_outliers(xyz, outlier_ratio, outlier_range, seed):
    """the N points followed by m outliers, o_a = p_base,a + outlier_range * gaussian(seed, j, 8 + 2a)"""
    xyz = np.asarray(xyz, dtype=np.float64)
    n = len(xyz)
    m = outlier_count(n, outlier_ratio)
    if m == 0:
        return xyz.copy()
    base = outlier_bases(n, m, seed)
    j = np.arange(m, dtype=np.uint64)
    o = xyz[base].copy()
    for a in range(3):
        o[:, a] = o[:, a] + outlier_range * synth.gaussian(seed, j, OUTLIER_OFFSET_LANE + 2 * a)
    return np.ascontiguousarray(np.concatenate([xyz, o]))


def local_deformation(xyz, radius, strength, center):
    """inside the radius (strict): p += ((p - c) / d * strength) * w, w = 0.5 (1 + cos(pi d / r)), d from Eigen's
    squaredNorm x*x + (y*y + z*z); the centre itself stays (normalize() leaves a zero vector).  numpy rounds every operation
    on its own, as the device does without contraction."""
    out = np.array(xyz, dtype=np.float64, copy=True)
    c = np.asarray(center, dtype=np.float64)
    dv = out - c
    d = np.sqrt(dv[:, 0] * dv[:, 0] + (dv[:, 1] * dv[:, 1] + dv[:, 2] * dv[:, 2]))
    inside = d < radius
    moved = inside & (d > 0)
    w = 0.5 * (1.0 + np.cos(np.pi * d[moved] / radius))
    for a in range(3):
        out[moved, a] = out[moved, a] + (dv[moved, a] / d[moved] * strength) * w
    return out

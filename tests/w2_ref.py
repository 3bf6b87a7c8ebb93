"""Exact reference for the Gaussian 2-Wasserstein distance per voxel (DESIGN §3.18), on the CPU, with no use of the GPU.

Per voxel pair the rational moments of exact_ref.exact_moments give mu and the unbiased covariance Sigma = M2 / (n - 1) as
exact rationals.  The matrix square roots are taken with mpmath eigsy at DPS digits (eigenvalues clamped at 0), and
  o^2 = |mu_est - mu_gt|^2,   b^2 = tr Sigma_gt + tr Sigma_est - 2 tr((A Sigma_est A)^1/2),  A = Sigma_gt^1/2,
  W2^2 = o^2 + b^2,
where the cancellation of the trace formula costs nothing at 60 digits.

Error bound a correct fp64 implementation meets, through W2^2 (u = 2^-53, C = exact_ref.C_BOUND):
  |W2^2 - W2_ex^2| <= C u o (|mu_e|_1 + |mu_g|_1 + 2 v) + db (2 b_ex + db)
  db = sum over the two clouds of sqrt(3) min(sqrt(3 e), 3 e / sqrt(lambda_min)) + C u sqrt(tr Sigma_gt + tr Sigma_est)
  e  = C u n (3 v^2 / 4) / (n - 1)      (the bound on an entry of Sigma from fp64 moments about the voxel centre)
The offset term is the W bound of exact_ref.  For the shape term, b is a metric, so the error of b is at most the Bures
distance between each computed covariance and its exact value, which is at most |S'^1/2 - S^1/2|_F.  An entry error e
gives an operator-norm error of at most 3 e, and the square root moves by at most the square root of that in operator
norm, or by 3 e / sqrt(lambda_min) when Sigma is positive definite.  Frobenius norm adds sqrt(3).  The last term of db is
the rounding of the residual |A - B P Q^T|_F itself, relative to the size of A and B.

THRESHOLD is the largest W2 an exact copy or a permutation of the ground truth may show.  It comes from
trace_and_residual_floors: in numpy fp64, on the voxels of a surface scene with the points summed in two orders, the trace
formula leaves b up to sqrt(u tr Sigma) ~ 1e-7 m: above THRESHOLD on about 45 % of the voxels and 0 on the rest, where
its argument rounds below 0.  The residual form stays at the rounding of the moments, below THRESHOLD / 100 on every
voxel (~1e-13 m).
"""
import math
from fractions import Fraction

import mpmath as mp
import numpy as np

import exact_ref as X

U, C_BOUND, DPS = X.U, X.C_BOUND, X.DPS
THRESHOLD = 1e-10          # m; see trace_and_residual_floors
COLS = 26                  # me_eval_w2 rows: vmin[3] n_gt n_est mu_est[3] mu_gt[3] sig_est[6] sig_gt[6] offset shape w2
UPPER = ([0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2])


def exact_gaussian(pts):
    """(n, mu[3] Fractions, Sigma 3x3 Fractions = M2 / (n - 1)) of a voxel's fp64 points"""
    n, mu, m2 = X.exact_moments(pts)
    return n, mu, [[m2[a][b] / (n - 1) for b in range(3)] for a in range(3)]


def _mpmat(S):
    M = mp.matrix(3, 3)
    for r in range(3):
        for c in range(3):
            M[r, c] = X._mp(S[r][c]) if not isinstance(S, mp.matrix) else S[r, c]
    return (M + M.T) / 2


def sqrtm_psd(S):
    """S^1/2 of a symmetric 3x3 (nested lists of Fractions / floats, or mp.matrix), eigenvalues clamped at 0"""
    E, Q = mp.eigsy(_mpmat(S))
    return Q * mp.diag([mp.sqrt(max(E[i], mp.mpf(0))) for i in range(3)]) * Q.T


def w2_exact(mu_g, S_g, mu_e, S_e):
    """(o^2, b^2) as mpf at DPS digits"""
    with mp.workdps(DPS):
        A = sqrtm_psd(S_g)
        Se = _mpmat(S_e)
        inner = sqrtm_psd(A * Se * A)
        b2 = sum(_mpmat(S_g)[i, i] + Se[i, i] - 2 * inner[i, i] for i in range(3))
        o2 = sum((X._mp(mu_e[i]) - X._mp(mu_g[i])) ** 2 for i in range(3))
        return o2, max(b2, mp.mpf(0))


def lambda_min(S):
    with mp.workdps(DPS):
        E, _ = mp.eigsy(_mpmat(S))
        return float(max(min(E[i] for i in range(3)), mp.mpf(0)))


def entry_bound(n, v):
    return C_BOUND * U * n * (3 * v * v / 4) / (n - 1)


def sqrt_shift(n, v, lam_min):
    """the bound on |S'^1/2 - S^1/2|_F for an fp64 Sigma of a voxel of n points"""
    e = entry_bound(n, v)
    d = math.sqrt(3 * e)
    if lam_min > 0:
        d = min(d, 3 * e / math.sqrt(lam_min))
    return math.sqrt(3) * d


def w2_bound(o_ex, b_ex, mu_e, mu_g, tr_sum, n_e, n_g, lam_e, lam_g, v):
    """the bound on |W2^2 - W2_ex^2| (module docstring)"""
    mu_e, mu_g = np.abs(np.asarray(mu_e, np.float64)), np.abs(np.asarray(mu_g, np.float64))
    db = sqrt_shift(n_e, v, lam_e) + sqrt_shift(n_g, v, lam_g) + C_BOUND * U * math.sqrt(max(tr_sum, 0.0))
    return C_BOUND * U * o_ex * (mu_e.sum() + mu_g.sum() + 2 * v) + db * (2 * b_ex + db)


def pair_exact(est_pts, gt_pts, v):
    """everything a row of one voxel pair is checked against: dict of floats (o, b, w2 and their bound) and the exact
    Gaussians"""
    n_e, mu_e, S_e = exact_gaussian(est_pts)
    n_g, mu_g, S_g = exact_gaussian(gt_pts)
    o2, b2 = w2_exact(mu_g, S_g, mu_e, S_e)
    o, b = float(mp.sqrt(o2)), float(mp.sqrt(b2))
    tr = float(sum(S_g[i][i] + S_e[i][i] for i in range(3)))
    bound = w2_bound(o, b, [float(x) for x in mu_e], [float(x) for x in mu_g], tr, n_e, n_g, lambda_min(S_e), lambda_min(S_g), v)
    return dict(n_e=n_e, n_g=n_g, mu_e=mu_e, mu_g=mu_g, S_e=S_e, S_g=S_g, o=o, b=b, w2sq=float(o2 + b2), bound=bound)


def voxel_pairs(est, gt, v, min_points):
    """{key: (est indices, gt indices)} of the pairs of the W2 stage, and the voxel counts of both clouds"""
    ge, gg = X.voxel_groups(est, v), X.voxel_groups(gt, v)
    out = {k: (ie, gg[k]) for k, ie in ge.items() if k in gg and len(ie) >= min_points and len(gg[k]) >= min_points}
    return out, len(ge), len(gg)


def check_rows(rows, est, gt, v, min_points, sample=None):
    """rows of me_eval_w2 against the exact reference; returns the worst |W2^2 - exact| / bound"""
    pairs, _, _ = voxel_pairs(est, gt, v, min_points)
    assert len(rows) == len(pairs)
    keys = np.floor(rows[:, 0:3] / v + 0.5).astype(np.int64)
    assert len({tuple(k) for k in keys.tolist()}) == len(rows)
    worst = 0.0
    for i in (range(len(rows)) if sample is None else sample):
        r, key = rows[i], tuple(int(c) for c in keys[i])
        ie, ig = pairs[key]
        ex = pair_exact(est[ie], gt[ig], v)
        assert (int(r[3]), int(r[4])) == (ex["n_g"], ex["n_e"])
        np.testing.assert_allclose(r[5:8], [float(x) for x in ex["mu_e"]], rtol=0, atol=C_BOUND * U * (np.abs(r[5:8]).max() + v))
        np.testing.assert_allclose(r[8:11], [float(x) for x in ex["mu_g"]], rtol=0, atol=C_BOUND * U * (np.abs(r[8:11]).max() + v))
        for col, S, n in ((11, ex["S_e"], ex["n_e"]), (17, ex["S_g"], ex["n_g"])):
            np.testing.assert_allclose(r[col:col + 6], np.array([[float(x) for x in row] for row in S])[UPPER], rtol=0,
                                       atol=entry_bound(n, v))
        assert abs(r[25] - math.sqrt(r[23] * r[23] + r[24] * r[24])) <= 4 * U * r[25]
        err = abs(r[25] ** 2 - ex["w2sq"])
        assert err <= ex["bound"], (key, r[23:26], ex["o"], ex["b"], err, ex["bound"])
        worst = max(worst, err / ex["bound"] if ex["bound"] > 0 else 0.0)
    return worst


def scs_of(w_by_key, radius=5):
    return X.scs_exact(w_by_key, radius)


# ---------------------------------------------------------------------------------------------------------------
# fp64 statements of the two ways to take b, for the demonstration behind THRESHOLD
# ---------------------------------------------------------------------------------------------------------------
def fp64_sigma(pts, centre):
    """Sigma in fp64 as the library forms it: moments about the voxel centre summed in the given order, M2 / (n - 1)"""
    d = np.asarray(pts, np.float64) - centre
    n = len(d)
    s1 = np.zeros(3)
    s2 = np.zeros((3, 3))
    for p in d:                                   # a running sum in the order of the points
        s1 += p
        s2 += np.outer(p, p)
    return (s2 - np.outer(s1, s1) / n) / (n - 1)


def _sqrtm64(S):
    w, V = np.linalg.eigh((S + S.T) / 2)
    return (V * np.sqrt(np.maximum(w, 0.0))) @ V.T


def b_trace64(S_g, S_e):
    A = _sqrtm64(S_g)
    inner = _sqrtm64(A @ S_e @ A)
    return math.sqrt(max(0.0, np.trace(S_g) + np.trace(S_e) - 2 * np.trace(inner)))


def b_residual64(S_g, S_e):
    A, B = _sqrtm64(S_g), _sqrtm64(S_e)
    P, _, Qt = np.linalg.svd(B @ A)
    return float(np.linalg.norm(A - B @ (P @ Qt)))


def trace_and_residual_floors(pts_by_voxel, v, seed=0):
    """(b of the trace formula, b of the residual form) per voxel, for the voxel against a copy of itself whose points are
    summed in another order"""
    rng = np.random.RandomState(seed)
    bt, br = [], []
    for key, pts in pts_by_voxel.items():
        c = (np.asarray(key, np.float64) + 0.5) * v
        S_g = fp64_sigma(pts, c)
        S_e = fp64_sigma(pts[rng.permutation(len(pts))], c)
        bt.append(b_trace64(S_g, S_e))
        br.append(b_residual64(S_g, S_e))
    return np.array(bt), np.array(br)


def to_row(key, v, n_g, n_e, mu_e, mu_g, S_e, S_g):
    r = np.zeros(COLS)
    r[0:3] = np.asarray(key, np.float64) * v
    r[3], r[4] = n_g, n_e
    r[5:8], r[8:11] = mu_e, mu_g
    r[11:17], r[17:23] = np.asarray(S_e)[UPPER], np.asarray(S_g)[UPPER]
    return r


def fraction_matrix(S):
    return [[Fraction(float(S[a][b])) for b in range(3)] for a in range(3)]

"""Exact reference for the NN statistics and the voxel-Gaussian metrics: the reference's definitions evaluated without
rounding, on the CPU, with no use of the oracle or of the GPU.

NN statistics (map_eval.cpp:1069-1145, 1245-1253, 1398-1431).  The per-pair values the reference forms in fp64 — the
Eigen-order squared norm sq = x^2 + (y^2 + z^2) of (source - target) and d = sqrt(sq) — are fp64 operations of the
reference, not approximations, so they are reproduced in fp64 (numpy does exactly these operations).  Everything after
them is exact: the sums are integers (every double is an integer times a common power of two), the quotients are
rationals, and the square roots are taken with mpmath at 60 digits before the final rounding to fp64.  sigma is the
reference's two-pass definition, sum over ALL kept pairs of (d - mean_k)^2 over |C|.

Voxel metrics (voxel_calculator.cpp:21-56, 115-140; map_eval.cpp:240-390).  Voxel keys are the IEEE floor(x / v) (numpy
reproduces it).  The mean and the sum of squared deviations M2 of a voxel's points are exact rationals.  The stored
covariance is M2 when n <= 10 and M2 / (n - 1)^2 otherwise (buildVoxelMap divides once, computeVoxelEntropy divides the
stored matrix again).  W is computeWassersteinDistanceGaussian: a third division by (n - 1), symmetrisation, eigenvalues
clamped at 1e-6 (mpmath eigsy), the identity for n <= 1, and the trace of the Cholesky factor of L1 S2 L1^T where the Bures
term would need a matrix square root.  SCS follows from the exact W.

Error bounds a correct fp64 implementation meets (u = 2^-53, C = C_BOUND):
  mean, rmse, fitness, cd, f1, iou, full CD   |x - x_ex| <= C u |x_ex|
  sigma                                       |s - s_ex| <= 1e-10 s_ex + C u mean_all
  W                                           |W^2 - W_ex^2| <= C u (tr_sum + chol + |dmu| (|mu_e| + |mu_g| + v))
  stored covariance entries                   <= C u n (3 v^2 / 4) / divisor   (divisor 1 or (n - 1)^2)
  voxel mean                                  <= C u (|mu| + v)
The sigma bound is absolute in mean_all because sigma of a tight cluster of distances is a difference of nearly equal
quantities: an implementation that forms it from sum(d) and sum(d^2) loses u (mean / spread)^2 of it and fails here.
W is compared through W^2 because W = sqrt(max(0, .)) has an unbounded relative condition number near 0.  chol =
sum_k A_kk / L_kk + S1_kk sqrt(S2_kk) / L1_kk over the two Cholesky factorisations (L1 of the clamped S1, L of
A = L1 S2 L1^T) is their first-order sensitivity to a relative perturbation u of their inputs: with eigenvalues clamped at
1e-6 next to eigenvalues of ~10 it exceeds tr_sum by three orders, and no fp64 evaluation of the quirk does better.
"""
import math
from fractions import Fraction

import mpmath as mp
import numpy as np

U = 2.0 ** -53
C_BOUND = 1e3
DPS = 60
CLAMP = 1e-6          # the double literal of voxel_calculator.cpp:128


# ---------------------------------------------------------------------------------------------------------------
# exact arithmetic on arrays of doubles
# ---------------------------------------------------------------------------------------------------------------
def to_ints(x):
    """x (fp64 array) = ints * 2^e exactly, with one common exponent e: (list of Python ints, e)"""
    x = np.asarray(x, dtype=np.float64).ravel()
    if len(x) == 0:
        return [], 0
    m, ex = np.frexp(x)
    mi = (m * 2.0 ** 53).astype(np.int64)           # exact: |m| < 1 has at most 53 significant bits
    ex = ex.astype(np.int64) - 53
    e0 = int(ex.min())
    return [int(a) << int(b - e0) for a, b in zip(mi.tolist(), ex.tolist())], e0


def _pow2(e):
    return Fraction(2) ** e


def exact_sum(x):
    """the exact sum of an fp64 array, as a Fraction"""
    ints, e = to_ints(x)
    return sum(ints) * _pow2(e)


def to_float(q):
    """a Fraction or mpf, correctly rounded to fp64 (nan passes through)"""
    if isinstance(q, float):
        return q
    if isinstance(q, Fraction):
        return float(q)           # Fraction.__float__ rounds correctly
    return float(q)


def _sqrt(q):
    with mp.workdps(DPS):
        return mp.sqrt(mp.mpf(q.numerator) / q.denominator)


# ---------------------------------------------------------------------------------------------------------------
# NN statistics
# ---------------------------------------------------------------------------------------------------------------
def sqnorm_eigen(diff):
    """Eigen's squaredNorm of (n, 3) fp64 differences: x*x + (y*y + z*z), no fused operations"""
    diff = np.asarray(diff, dtype=np.float64)
    return diff[:, 0] * diff[:, 0] + (diff[:, 1] * diff[:, 1] + diff[:, 2] * diff[:, 2])


def kept_pairs(query, ref, nn_idx, nn_d2, R, cutoff_mode, as_written=False):
    """(sq, d, n_ub) of the kept pairs of one direction, from the per-query nearest neighbours (me_get_nn).
    cutoff_mode 0: keep iff d2 <= R; 1: keep iff d2 < R * R.  as_written (gt -> est of ME_PAIRING_AS_WRITTEN): the pair
    of gt query i with nearest est point j is (source gt[j], target est[i]) (map_eval.cpp:1233,1241,1093-1094); pairs
    whose swapped indices fall outside the clouds are dropped and counted."""
    nn_idx, nn_d2 = np.asarray(nn_idx), np.asarray(nn_d2)
    have = nn_idx >= 0
    keep = have & ((nn_d2 <= R) if cutoff_mode == 0 else (nn_d2 < R * R))
    qi = np.nonzero(keep)[0]
    ri = nn_idx[qi].astype(np.int64)
    n_ub = 0
    if as_written:          # query = gt, ref = est
        ok = (ri < len(query)) & (qi < len(ref))
        n_ub = int((~ok).sum())
        diff = query[ri[ok]] - ref[qi[ok]]
    else:
        diff = query[qi] - ref[ri]
    sq = sqnorm_eigen(diff)
    return sq, np.sqrt(sq), n_ub


def dir_stats(sq, d, n_source, tau):
    """one direction of getDiffRegResultWithCorrespondence, exact after d: dict of fp64 lists (mean, rmse, fitness,
    sigma), exact counts, and the exact mean of d over all kept pairs (mean_all, a Fraction or None)"""
    sq, d = np.asarray(sq, np.float64), np.asarray(d, np.float64)
    nc = len(d)
    D, ed = to_ints(d)
    Q, eq = to_ints(sq)
    sd, sq_scale = _pow2(ed), _pow2(eq)
    s_all = sum(D) * sd
    q_all = sum(x * x for x in D) * sd * sd             # sum of d^2 (exact), for the two-pass sigma
    out = dict(n_corr=nc, n_inlier=[], mean=[], rmse=[], fitness=[], sigma=[],
               mean_all=(s_all / nc if nc else None))
    nan = float("nan")
    for t in tau:
        m = np.nonzero(d <= t)[0]
        sk = sum(D[i] for i in m) * sd
        qk = sum(Q[i] for i in m) * sq_scale
        out["n_inlier"].append(len(m))
        out["fitness"].append(to_float(Fraction(len(m), int(n_source))))
        if nc == 0:                                       # 0/0 as in the reference
            out["mean"].append(nan); out["rmse"].append(nan); out["sigma"].append(nan)
            continue
        mean_k = sk / nc
        out["mean"].append(to_float(mean_k))
        out["rmse"].append(to_float(_sqrt(qk / nc)))
        ss = q_all - 2 * mean_k * s_all + nc * mean_k * mean_k    # sum over ALL kept pairs of (d - mean_k)^2, exact
        out["sigma"].append(to_float(_sqrt(ss / nc)))
    return out


def nn_result(e2g, g2e, n_est, n_gt, sum_nn_e=None, sum_nn_g=None):
    """cd, f1, iou (map_eval.cpp:1245-1253) and full CD (:1429) from two dir_stats, evaluated exactly in mpmath from the
    fp64 per-direction values the reference combines (rmse, fitness), which are the correctly rounded exact ones.
    sum_nn_*: fp64 arrays of sqrt(d2_nn) over all queries of each direction (full CD)."""
    out = dict(cd=[], f1=[], iou=[])
    with mp.workdps(DPS):
        for k in range(5):
            r_e, r_g, fit = e2g["rmse"][k], g2e["rmse"][k], e2g["fitness"][k]
            out["cd"].append(float(mp.mpf(r_e) + mp.mpf(r_g)) if not (np.isnan(r_e) or np.isnan(r_g)) else float("nan"))
            if np.isnan(r_e) or fit + r_e == 0:
                out["f1"].append(float("nan"))
            else:
                out["f1"].append(float(2 * mp.mpf(fit) * mp.mpf(r_e) / (mp.mpf(fit) + mp.mpf(r_e))))
            inter = e2g["n_inlier"][k]
            out["iou"].append(to_float(Fraction(inter, n_est + n_gt - inter)))
        if sum_nn_e is not None:
            out["full_cd"] = float(exact_sum(sum_nn_e) / n_est + exact_sum(sum_nn_g) / n_gt)
    return out


def sigma_bound(sigma_ex, mean_all):
    return 1e-10 * sigma_ex + C_BOUND * U * mean_all


def rel_bound(x_ex):
    return C_BOUND * U * abs(x_ex)


# ---------------------------------------------------------------------------------------------------------------
# voxel Gaussians
# ---------------------------------------------------------------------------------------------------------------
def voxel_keys(xyz, v):
    """int64 (n, 3) IEEE floor(x / v) per axis (voxel_calculator.cpp:241-245)"""
    return np.floor(np.asarray(xyz, np.float64) / v).astype(np.int64)


def voxel_groups(xyz, v):
    """{key tuple: indices of the points in it}"""
    keys = voxel_keys(xyz, v)
    uk, inv = np.unique(keys, axis=0, return_inverse=True)
    inv = inv.ravel()
    order = np.argsort(inv, kind="stable")
    bounds = np.searchsorted(inv[order], np.arange(len(uk) + 1))
    return {tuple(int(c) for c in uk[i]): order[bounds[i]:bounds[i + 1]] for i in range(len(uk))}


def exact_moments(pts):
    """(n, mu[3] Fractions, M2 3x3 Fractions) of a voxel's fp64 points"""
    pts = np.asarray(pts, np.float64)
    n = len(pts)
    ints, e = to_ints(pts)
    P = [ints[3 * i:3 * i + 3] for i in range(n)]
    s = [sum(p[a] for p in P) for a in range(3)]
    # M2 = sum (p - mu)(p - mu)^T = sum p p^T - s s^T / n, exact in integers over n
    m2 = [[Fraction(n * sum(p[a] * p[b] for p in P) - s[a] * s[b], n) * _pow2(2 * e) for b in range(3)] for a in range(3)]
    return n, [Fraction(s[a], n) * _pow2(e) for a in range(3)], m2


def stored_sigma(n, m2):
    """the covariance buildVoxelMap leaves in the voxel (3x3 Fractions)"""
    div = 1 if n <= 10 else (n - 1) ** 2
    return [[m2[a][b] / div for b in range(3)] for a in range(3)]


def _mp(q):
    return mp.mpf(q.numerator) / q.denominator if isinstance(q, Fraction) else mp.mpf(q)


def _clamped(stored, n):
    if n <= 1:
        return mp.eye(3)
    S = mp.matrix(3, 3)
    for r in range(3):
        for c in range(3):
            S[r, c] = _mp(stored[r][c]) / (n - 1)
    S = (S + S.T) / 2
    E, Q = mp.eigsy(S)
    D = mp.diag([max(E[i], mp.mpf(CLAMP)) for i in range(3)])
    return Q * D * Q.T


def _chol(A):
    L = mp.matrix(3, 3)
    for k in range(3):
        x = A[k, k] - sum(L[k, j] ** 2 for j in range(k))
        L[k, k] = mp.sqrt(x)
        for i in range(k + 1, 3):
            L[i, k] = (A[i, k] - sum(L[i, j] * L[k, j] for j in range(k))) / L[k, k]
    return L


def wasserstein2(mu_g, stored_g, n_g, mu_e, stored_e, n_e):
    """W^2 of computeWassersteinDistanceGaussian(gt_voxel, est_voxel) and the scale of its bound, tr_sum + chol (module
    docstring), as mpf at DPS digits.  mu: 3 values, stored: 3x3 (Fractions or floats) as held in the voxel, n: the
    voxel's point count."""
    with mp.workdps(DPS):
        s1, s2 = _clamped(stored_g, n_g), _clamped(stored_e, n_e)
        L1 = _chol(s1)
        a = L1 * s2 * L1.T
        La = _chol(a)
        tr_sqrt = sum(La[i, i] for i in range(3))
        tr_sum = sum(s1[i, i] + s2[i, i] for i in range(3))
        # conditioning of the two Cholesky factors: a relative perturbation u of the k-th Schur complement moves L_kk by
        # u S_k / (2 L_kk) <= u A_kk / (2 L_kk); with eigenvalues clamped at 1e-6 and up to ~10 this exceeds tr_sum by 1e3
        cond = sum(a[i, i] / La[i, i] + s1[i, i] / L1[i, i] * mp.sqrt(s2[i, i]) for i in range(3))
        dm2 = sum((_mp(mu_g[i]) - _mp(mu_e[i])) ** 2 for i in range(3))
        w2 = dm2 + tr_sum - 2 * tr_sqrt
        return max(w2, mp.mpf(0)), tr_sum + cond


def w_bound(scale, mu_e, mu_g, v):
    """the bound on |W^2 - W_ex^2|; scale = tr_sum + chol as wasserstein2 returns it"""
    mu_e, mu_g = np.asarray(mu_e, np.float64), np.asarray(mu_g, np.float64)
    dmu = float(np.linalg.norm(mu_e - mu_g))
    return C_BOUND * U * (float(scale) + dmu * (np.abs(mu_e).sum() + np.abs(mu_g).sum() + v))


def sigma_entry_bound(n, v):
    div = 1 if n <= 10 else (n - 1) ** 2
    return C_BOUND * U * n * (3 * v * v / 4) / div


def mu_bound(mu, v):
    return C_BOUND * U * (np.abs(np.asarray(mu, np.float64)) + v)


def voxel_pairs(est, gt, v, min_points):
    """the voxel pairs calculateVMD evaluates: {key: (n_e, mu_e, M2_e, n_g, mu_g, M2_g)} over keys present in both clouds
    with at least min_points points in each (map_eval.cpp:270-284), plus the voxel counts of each cloud"""
    ge, gg = voxel_groups(est, v), voxel_groups(gt, v)
    out = {}
    for k, ie in ge.items():
        ig = gg.get(k)
        if ig is None or len(ie) < min_points or len(ig) < min_points:
            continue
        out[k] = exact_moments(est[ie]) + exact_moments(gt[ig])
    return out, len(ge), len(gg)


def scs_exact(w_table, radius=5):
    """map_eval.cpp:351-387 on {key: W (mpf or float)}: (SCS as mpf, count); neighbours are the other keys of the table
    within the (2 radius + 1)^3 block"""
    keys = list(w_table)
    total, count = mp.mpf(0), 0
    with mp.workdps(DPS):
        for k in keys:
            nb = [w_table[(k[0] + dx, k[1] + dy, k[2] + dz)]
                  for dx in range(-radius, radius + 1) for dy in range(-radius, radius + 1) for dz in range(-radius, radius + 1)
                  if (dx, dy, dz) != (0, 0, 0) and (k[0] + dx, k[1] + dy, k[2] + dz) in w_table]
            if not nb:
                continue
            nb = [mp.mpf(x) for x in nb]
            mean = sum(nb) / len(nb)
            var = sum((x - mean) ** 2 for x in nb) / len(nb)
            total += mp.sqrt(var) / mean
            count += 1
        return (total / count if count else mp.nan), count


# ---------------------------------------------------------------------------------------------------------------
# mean map entropy (map_eval.cpp:1433-1436, 1438-1737)
#
# Neighbours are the reference's fp64 decisions, reproduced in fp64: d2 = ((dx dx) + dy dy) + dz dz (d2_kd, nanoflann),
# strict d2 < r^2, the query itself removed once (duplicates of it stay), valid iff k >= min_neighbors.  The centred
# covariance sum (p - pbar)(p - pbar)^T / (k - 1) of the fp64 coordinates, its determinant and its adjugate are exact
# rationals; the entropy 0.5 ln(2 pi e det) is taken with mpmath.  det <= 0 rejects the point (the isnan / isinf test of
# map_eval.cpp:1692, :1574, :1472 / :1505).
#
# B64, the bound an fp64 evaluation of the neighbourhood meets (the reference's centred product, or the library's moments
# about the query, cov = (S2 - S1 S1^T / k) / (k - 1)): every covariance entry is within
#   dC_ij = C_MME u (k + 2) (sum_p |d_pi| |d_pj| + |S1_i S1_j| / k) / (k - 1),   d_p = p - q,
# the gamma_{k+2} bound of a recursive sum of k products and the centring, with a margin of C_MME.  The permanent
# majorises the determinant's change: |det(C + D) - det C| <= per(|C| + dC) - per(|C|) = ddet.  A query is determined when
# ddet < det / 2 (its validity is then decided, and B64 = 0.5 ddet / (det - ddet) + C_BOUND u (1 + |e|)), or when
# det = ddet = 0 (an exactly flat or straight neighbourhood along the axes: rejected by every fp64 evaluation).
# C_MME is deliberately not C_BOUND: with 10^3 the bound would be 0.02 nats on a 1 um plane and could not tell an fp64
# evaluation (2e-7) from one built on fp32 offsets (5e-4).
#
# B32(E), the first-order certificate of an evaluation whose offsets carry an error of at most E per axis (the library's
# fp32-offset sweeps): with q = tr adj(C) / det = sum 1 / lambda_i and s = E sqrt(k / (k - 1)) sqrt(q),
#   rho = 2 sqrt(3) s + 3 s^2,  rho' = rho + 3 rho^2,  B32 = 0.5 |ln(1 - rho')|  (undetermined when rho' >= 1/2).
# It is rotation invariant: on a tilted plane of normal noise sigma it grows like E / sigma, where entrywise bounds grow
# like E r / sigma^2.  mme_fp32_certificate evaluates it on any covariance, the exact one or a kernel's own.
# ---------------------------------------------------------------------------------------------------------------
C_MME = 4.0
TAU_FP64 = 1e-3       # nats: a fp32-offset sweep finishes a query in fp64 when its certificate exceeds this


def d2_kd(q, p):
    """squared distances of (n, 3) fp64 differences q - p in nanoflann's order ((dx dx) + dy dy) + dz dz"""
    d = np.asarray(q, np.float64) - np.asarray(p, np.float64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def mme_neighbours(pts, r, le=False):
    """per query the indices of its neighbours: d2_kd < r^2 (or <= with le, a deliberately wrong variant), the query itself
    removed once"""
    from scipy.spatial import cKDTree
    pts = np.asarray(pts, np.float64)
    r2 = r * r
    cand = cKDTree(pts).query_ball_point(pts, r * (1 + 1e-6) + 1e-300)
    out = []
    for i, c in enumerate(cand):
        c = np.asarray(sorted(c), dtype=np.int64)
        d2 = d2_kd(pts[i], pts[c])
        c = c[(d2 <= r2) if le else (d2 < r2)]
        out.append(c[c != i])
    return out


def _permanent_growth(a, d):
    """per(a + d) - per(a) for non-negative 3x3 a, d, without cancellation"""
    tot = 0.0
    for s in ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)):
        x = [a[i][s[i]] for i in range(3)]
        y = [d[i][s[i]] for i in range(3)]
        tot += (y[0] * x[1] * x[2] + x[0] * y[1] * x[2] + x[0] * x[1] * y[2] + y[0] * y[1] * x[2] + y[0] * x[1] * y[2]
                + x[0] * y[1] * y[2] + y[0] * y[1] * y[2])
    return tot


def mme_fp32_certificate(cov, k, E):
    """B32 (module notes) of a 3x3 covariance (floats or Fractions) of k neighbours under an offset error E per axis;
    inf when undetermined (rho' >= 1/2, or det <= 0)"""
    c = [[float(cov[a][b]) for b in range(3)] for a in range(3)]
    det = float(np.linalg.det(np.array(c))) if not isinstance(cov[0][0], Fraction) else float(_det3(cov))
    adj = (c[0][0] * c[1][1] - c[0][1] ** 2) + (c[0][0] * c[2][2] - c[0][2] ** 2) + (c[1][1] * c[2][2] - c[1][2] ** 2)
    if not det > 0 or not adj > 0:
        return float("inf")
    s = E * math.sqrt(k / (k - 1) * adj / det)
    rho = 2 * math.sqrt(3) * s + 3 * s * s
    rho += 3 * rho * rho
    return 0.5 * abs(math.log1p(-rho)) if rho < 0.5 else float("inf")


def _det3(m):
    return (m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0])
            + m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]))


def mme_point(pts, i, nb, min_neighbors, ints=None, drop_query=True, divisor=None):
    """the exact entropy of query i with neighbours nb: dict(k, valid, determined, e (fp64 of the exact value, 0.0 when
    rejected), cov (3x3 Fractions or None), b64).  ints: to_ints(pts) (pass it to avoid recomputing).  drop_query=False
    and divisor='k' are deliberately wrong variants for the tests' teeth."""
    pts = np.asarray(pts, np.float64)
    k = len(nb)
    out = dict(k=k, valid=False, determined=True, e=0.0, cov=None, b64=0.0)
    if k < min_neighbors:
        return out
    if not drop_query:
        nb = np.concatenate([[i], nb])
    if ints is None:
        ints = to_ints(pts)
    I, ex = ints
    X = [I[3 * j:3 * j + 3] for j in nb]
    n = len(X)
    den = (n - 1) if divisor is None else n
    S = [sum(x[a] for x in X) for a in range(3)]
    M = [[n * sum(x[a] * x[b] for x in X) - S[a] * S[b] for b in range(3)] for a in range(3)]
    scale = _pow2(2 * ex) / (n * den)
    cov = [[Fraction(M[a][b]) * scale for b in range(3)] for a in range(3)]
    det = _det3(cov)
    # the fp64 error bound of the entries, from the offsets to the query
    d = pts[nb] - pts[i]
    ad = np.abs(d)
    s1 = d.sum(0)
    dC = C_MME * U * (n + 2) * ((ad.T @ ad) + np.abs(np.outer(s1, s1)) / n) / (n - 1)
    a = [[abs(float(cov[r][c])) for c in range(3)] for r in range(3)]
    ddet = _permanent_growth(a, dC.tolist())
    detf = float(det)
    out["cov"] = cov
    if det <= 0:
        out["determined"] = det == 0 and ddet == 0.0
        return out
    if not ddet < 0.5 * detf:
        out["determined"] = False
        return out
    with mp.workdps(DPS):
        e = 0.5 * (mp.log(2 * mp.pi * mp.e) + mp.log(det.numerator) - mp.log(det.denominator))
    ef = float(e)
    out.update(valid=True, e=ef, b64=0.5 * ddet / (detf - ddet) + C_BOUND * U * (1 + abs(ef)))
    return out


def mme_exact(pts, r, min_neighbors, E=None, nbs=None):
    """every query of the cloud: arrays k, valid, determined, e, b64 and (with E) b32 = B32(E) of the exact covariance"""
    pts = np.asarray(pts, np.float64)
    nbs = mme_neighbours(pts, r) if nbs is None else nbs
    ints = to_ints(pts)
    rows = [mme_point(pts, i, nb, min_neighbors, ints) for i, nb in enumerate(nbs)]
    res = {f: np.array([p[f] for p in rows]) for f in ("k", "valid", "determined", "e", "b64")}
    res["cov"] = [p["cov"] for p in rows]
    if E is not None:
        res["b32"] = np.array([mme_fp32_certificate(p["cov"], p["k"], E) if p["valid"] else 0.0 for p in rows])
    res["nbs"] = nbs
    return res


def mme_aggregate_bounds(ex, per_point_bound):
    """bounds of (n_valid, sum, min/max |e|) given per-point bounds over the valid determined queries: (n_undetermined,
    bound of sum_entropy, bound of min_abs / max_abs_entropy)"""
    und = int((~ex["determined"]).sum())
    v = ex["valid"] & ex["determined"]
    n = int(v.sum())
    s_b = float(per_point_bound[v].sum()) + C_BOUND * U * n * float(np.abs(ex["e"][v]).sum())
    ext_b = float(per_point_bound[v].max()) if n else 0.0
    return und, s_b, ext_b


def mme_summary(ex):
    """(n_valid, sum, min_abs, max_abs) of the exact per-point values (fp64 of exact sums)"""
    v = ex["valid"]
    e = ex["e"][v]
    s = float(sum((Fraction(x) for x in e), Fraction(0)))
    nz = e[e != 0]
    return int(v.sum()), s, (float(np.abs(nz.max())) if len(nz) else np.nan), (float(np.abs(nz.min())) if len(nz) else np.nan)


def finish_entropy_fp64(d, min_neighbors):
    """numpy statement of the library's fp64 finish (mme.cu finish_entropy): the moments of the offsets d (k, 3) about the
    query, summed in order, cov = (S2 - S1 S1^T / k) / (k - 1), Eigen's cofactor determinant; 0.0 when rejected"""
    d = np.asarray(d, np.float64)
    k = len(d)
    if k < min_neighbors or k < 2:
        return 0.0
    s1 = [np.cumsum(d[:, a])[-1] for a in range(3)]
    s2 = [[np.cumsum(d[:, a] * d[:, b])[-1] for b in range(3)] for a in range(3)]
    kd, inv = float(k), 1.0 / float(k - 1)
    c = [[(s2[a][b] - s1[a] * s1[b] / kd) * inv for b in range(3)] for a in range(3)]
    for a in range(3):
        for b in range(a):
            c[a][b] = c[b][a]
    A = c[0][0] * (c[1][1] * c[2][2] - c[1][2] * c[2][1])
    B = c[0][1] * (c[1][0] * c[2][2] - c[1][2] * c[2][0])
    Cc = c[0][2] * (c[1][0] * c[2][1] - c[1][1] * c[2][0])
    with np.errstate(all="ignore"):
        e = 0.5 * np.log(2 * np.pi * np.e * ((A - B) + Cc))
    return 0.0 if not np.isfinite(e) else float(e)


def mme_offset_error(h, rings, pts):
    """E of run_mme: the per-axis error bound of the fp32 offsets on a lattice of edge h searched at `rings` rings"""
    maxabs = float(np.abs(np.asarray(pts, np.float64)).max())
    return 1e-7 * (2.0 * rings + 6.0) * h + 4e-15 * maxabs


def fp32_offsets(pts, i, nb, h, R):
    """the flat kernel's offset rebuild of the neighbours nb of query i, emulated in float32 on a lattice of edge h (origin
    at the cell below the cloud's minimum): rel = fp32(x - cell origin), w = fp32(ix);
    dx = fma(c.w - q.w, h, c.x - q.x), dy = c.y + fma(dyc - R + R, h, -q.y), dz likewise"""
    pts = np.asarray(pts, np.float64)
    o = np.floor(pts.min(0) / h) * h
    cell = np.floor((pts - o) / h)
    rel = (pts - (o + cell * h)).astype(np.float32)
    h32 = np.float32(h)
    f32 = np.float32

    def fma(a, b, c):                       # float32 fused multiply-add: a * b is exact in fp64
        return (np.float64(a) * np.float64(b) + np.float64(c)).astype(np.float32)

    q, qc = rel[i], cell[i]
    c, cc = rel[nb], cell[nb]
    wq, wc = f32(qc[0]), cc[:, 0].astype(np.float32)
    dx = fma(wc - wq, h32, c[:, 0] - q[0])
    cy = fma((cc[:, 1] - qc[1]).astype(np.float32), h32, -q[1])
    cz = fma((cc[:, 2] - qc[2]).astype(np.float32), h32, -q[2])
    assert np.all(np.abs(cc - qc) <= R)
    dy = c[:, 1] + cy
    dz = c[:, 2] + cz
    return np.column_stack([dx, dy, dz]).astype(np.float64)

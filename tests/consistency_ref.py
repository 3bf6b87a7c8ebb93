"""The local consistency rule (DESIGN §3.15) stated in numpy and mpmath.

- finalize: me_consistency_finalize in numpy, the same operations in the same order (rows, then the whole map as the rows'
  sums in list order).
- exact_point: MME's neighbourhood (exact_ref.mme_neighbours), the exact rational covariance of the k neighbour offsets
  (exact_ref's integer statement, so C = (S2 - S1 S1^T / k) / (k - 1) without rounding), its smallest eigenvalue from
  mpmath at high precision, and a bound for the library's fp64 pipeline:
    |v_fp64 - lambda3| <= ||dC||_F + C_JACOBI u tr C
  * ||dC||_F: the entries' rounding of the fp64 moments and of the covariance expressions, the bound exact_ref derives for
    MME (C_MME u (k + 2) (|d|^T |d| + |S1 S1^T| / k) / (k - 1) per entry); by Weyl's inequality an eigenvalue moves by at
    most the spectral norm of the perturbation, which the Frobenius norm bounds.
  * the Jacobi solve (eig3_jacobi): every rotation is applied as two passes of two-term updates per entry, an exact
    similarity of a matrix within 6 u ||A||_F; a 3x3 symmetric matrix converges quadratically, so the stopping rule
    (off^2 <= 1e-34 diag^2) is met within 10 sweeps of 3 rotations from any start, and the off-diagonal it leaves moves an
    eigenvalue by at most 1e-17 ||A||_F < u ||A||_F.  30 rotations x 6 u + u < 200 u, and ||C||_F <= tr C for a
    positive semi-definite C: C_JACOBI = 200.  The clamp max(0, .) only moves v towards the exact lambda3 >= 0.
"""
import math
import os
import sys
from fractions import Fraction

import mpmath as mp
import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import exact_ref as X  # noqa: E402

SUM_F, MAX_F = 6, 1
U = 2.0 ** -53
C_JACOBI = 200.0
DPS = 60


def _means(n_valid, n_pv, se, sv, ssv, mx):
    mme = se / n_valid if n_valid > 0 else 0.0
    if n_pv > 0:
        return mme, sv / n_pv, ssv / n_pv, mx
    return mme, math.nan, math.nan, math.nan


def finalize(region_size, index, n_points, n_total, block):
    """me_consistency_finalize: (rows as a list of dicts, whole as a dict)"""
    index = np.asarray(index, np.int64).reshape(-1, 3)
    n = index.shape[0]
    blk = np.asarray(block, np.float64).reshape(-1)
    B = max(n, 1)
    mx = blk[SUM_F * B:]
    rows = []
    W = dict(n_query=0, n_valid=0, n_pv=0, sum_entropy=0.0, sum_pv=0.0, sum_sqrt_pv=0.0)
    max_v = 0.0
    for r in range(B):
        v = blk[r * SUM_F:(r + 1) * SUM_F]
        nq, nv, npv = int(v[0]), int(v[1]), int(v[2])
        W["n_query"] += nq
        W["n_valid"] += nv
        W["n_pv"] += npv
        W["sum_entropy"] += float(v[3])
        W["sum_pv"] += float(v[4])
        W["sum_sqrt_pv"] += float(v[5])
        max_v = float(np.fmax(max_v, mx[r]))
        if n == 0:
            continue
        row = dict(index=index[r].copy(), min=index[r] * float(region_size), max=(index[r] + 1) * float(region_size),
                   n_points=int(n_points[r]), n_query=nq, n_valid=nv, n_pv=npv, sum_entropy=float(v[3]), sum_pv=float(v[4]),
                   sum_sqrt_pv=float(v[5]))
        row["mme"], row["mpv"], row["mean_plane_std"], row["max_pv"] = _means(nv, npv, v[3], v[4], v[5], mx[r])
        rows.append(row)
    W["mme"], W["mpv"], W["mean_plane_std"], W["max_pv"] = _means(W["n_valid"], W["n_pv"], W["sum_entropy"], W["sum_pv"],
                                                                   W["sum_sqrt_pv"], max_v)
    W["n_points"] = int(n_total)
    return rows, W


def exact_cov(pts, i, nb):
    """the exact covariance (3x3 Fractions) of the k = len(nb) neighbour offsets of query i, or None for k < 2"""
    pts = np.asarray(pts, np.float64)
    k = len(nb)
    if k < 2:
        return None
    sel = np.concatenate([[i], np.asarray(nb, np.int64)])
    I, ex = X.to_ints(pts[sel])
    P = [I[3 * j:3 * j + 3] for j in range(len(sel))]
    q = P[0]
    D = [[p[a] - q[a] for a in range(3)] for p in P[1:]]
    S = [sum(d[a] for d in D) for a in range(3)]
    scale = Fraction(2) ** (2 * ex) / (k * (k - 1)) if ex >= 0 else Fraction(1, 2 ** (-2 * ex)) / (k * (k - 1))
    return [[Fraction(k * sum(d[a] * d[b] for d in D) - S[a] * S[b]) * scale for b in range(3)] for a in range(3)]


def smallest_eig(cov):
    """the smallest eigenvalue of an exact symmetric 3x3 matrix, as a float, from mpmath at DPS digits"""
    with mp.workdps(DPS):
        M = mp.matrix([[mp.mpf(c.numerator) / c.denominator for c in row] for row in cov])
        w = mp.eigsy(M, eigvals_only=True)
        return float(min(w[j] for j in range(3)))


def fp64_bound(pts, i, nb, cov):
    """the bound of |v_fp64 - lambda3| (module notes)"""
    pts = np.asarray(pts, np.float64)
    n = len(nb)
    d = pts[nb] - pts[i]
    ad = np.abs(d)
    s1 = d.sum(0)
    dC = X.C_MME * U * (n + 2) * ((ad.T @ ad) + np.abs(np.outer(s1, s1)) / n) / (n - 1)
    tr = float(sum(cov[a][a] for a in range(3)))
    return float(np.sqrt((dC * dC).sum())) + C_JACOBI * U * tr


def exact_points(pts, r, min_neighbors, idx=None):
    """per query (all, or the indices idx): k, lambda3 (NaN for k < m) and the bound"""
    pts = np.asarray(pts, np.float64)
    nbs = X.mme_neighbours(pts, r)
    idx = range(len(pts)) if idx is None else idx
    out = dict(i=[], k=[], lam=[], bound=[])
    for i in idx:
        nb = nbs[i]
        k = len(nb)
        out["i"].append(i)
        out["k"].append(k)
        if k < min_neighbors:
            out["lam"].append(math.nan)
            out["bound"].append(0.0)
            continue
        cov = exact_cov(pts, i, nb)
        out["lam"].append(max(0.0, smallest_eig(cov)))
        out["bound"].append(fp64_bound(pts, i, nb, cov))
    return {f: np.array(v) for f, v in out.items()}

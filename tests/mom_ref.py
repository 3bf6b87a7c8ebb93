"""The mutually orthogonal metric's rule (DESIGN §3.16) stated in numpy and mpmath.

- bins / histogram: the cube-map bin of a unit vector and the symmetric histogram (bin(n) and bin(-n) per planar normal);
- axes: me_mom_axes in the same operation order (bin centres, windowed scores, the greedy pick of a1, a2, a3);
- planar / families / fold / statement: the planarity test, the family of every planar point, the library's fold of the
  counts and sums of v (per chunk of 1024 caller-order points: lane l adds the points l, l + 32, ... in order, then an xor
  shuffle tree; the chunks merged the same way), numpy medians, and the metric;
- exact_normal: the exact eigenvector of the smallest eigenvalue of the rational covariance (consistency_ref.exact_cov) from
  mpmath, and a bound on the angle between it and the library's fp64 normal:
    sin(theta) <= eps / (gap - eps) + C_VEC u,   eps = ||dC||_F + C_JACOBI u tr C  (consistency_ref.fp64_bound)
  * Davis-Kahan's sin(theta) theorem: the eigenvector of the smallest eigenvalue of C + E lies within
    asin(||E||_2 / delta) of C's, where delta separates lambda3(C) from the other eigenvalues of C + E; by Weyl's
    inequality delta >= gap - ||E||_2, gap = lambda2 - lambda3 of the exact C.  The fp64 covariance and the Jacobi solve
    together act as a perturbation of norm at most eps (consistency_ref's derivation for v);
  * the eigenvector columns are the products of at most 30 plane rotations, each applied with two-term updates, so they are
    orthonormal to within 30 x 6 u; the normalisation adds 3 u: C_VEC = 200.
  The planarity filter guarantees gap >= (1 - rho) lambda2, which keeps the bound small on every planar point.
"""
import math
import os
import sys

import mpmath as mp
import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import consistency_ref as CR  # noqa: E402
import exact_ref as X  # noqa: E402

M = 16
BINS = 6 * M * M
U = 2.0 ** -53
C_VEC = 200.0
CHUNK = 1024


def bins(n, m=M):
    """the cube-map bin of every row of n (N, 3): a = argmax |n_a| (lowest on a tie), s = sign(n_a), b < c the other axes,
    u = n_b / |n_a|, w = n_c / |n_a|, i = min(M - 1, floor((u + 1) (M / 2))), j likewise, ((2a + [s < 0]) M + i) M + j"""
    n = np.asarray(n, np.float64).reshape(-1, 3)
    ab = np.abs(n)
    a = np.zeros(len(n), np.int64)
    mx = ab[:, 0].copy()
    for k in (1, 2):
        big = ab[:, k] > mx
        a[big] = k
        mx[big] = ab[big, k]
    rows = np.arange(len(n))
    na = n[rows, a]
    nb = np.where(a == 0, n[:, 1], n[:, 0])
    nc = np.where(a == 2, n[:, 1], n[:, 2])
    u = nb / mx
    w = nc / mx
    i = np.minimum(m - 1, np.floor((u + 1.0) * (0.5 * m)).astype(np.int64))
    j = np.minimum(m - 1, np.floor((w + 1.0) * (0.5 * m)).astype(np.int64))
    return ((2 * a + (na < 0.0)) * m + i) * m + j


def histogram(normals, m=M):
    """the symmetric histogram of the planar normals (N, 3): one count at bin(n) and one at bin(-n)"""
    normals = np.asarray(normals, np.float64).reshape(-1, 3)
    return (np.bincount(bins(normals, m), minlength=6 * m * m) + np.bincount(bins(-normals, m), minlength=6 * m * m)).astype(np.int64)


def centres(m=M):
    """the normalised face point of every bin (6 M^2, 3)"""
    b = np.arange(6 * m * m)
    j, i, face = b % m, (b // m) % m, b // (m * m)
    a = face // 2
    p = np.zeros((len(b), 3))
    p[np.arange(len(b)), a] = np.where(face & 1, -1.0, 1.0)
    ob = np.where(a == 0, 1, 0)
    oc = np.where(a == 2, 1, 2)
    p[np.arange(len(b)), ob] = -1.0 + (2 * i + 1) / float(m)
    p[np.arange(len(b)), oc] = -1.0 + (2 * j + 1) / float(m)
    nrm = np.sqrt((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2])
    return p / nrm[:, None]


def _dot(x, y):
    return (x[..., 0] * y[..., 0] + x[..., 1] * y[..., 1]) + x[..., 2] * y[..., 2]


def axes(hist, angle_deg, m=M):
    """me_mom_axes: (axes (3, 3) rows a1 a2 a3 with NaN where not found, status 'OK' / 'NO_PLANAR' / 'NO_SECOND_AXIS')"""
    h = np.asarray(hist, np.int64)
    out = np.full((3, 3), np.nan)
    rad = angle_deg * math.pi / 180.0
    cos_a, sin_a = math.cos(rad), math.sin(rad)
    C = centres(m)
    dots = _dot(C[:, None, :], C[None, :, :])
    S = ((dots >= cos_a) & (h[None, :] != 0)).astype(np.int64) @ h
    if h.sum() == 0:
        return out, "NO_PLANAR"
    b1 = int(np.argmax(S))
    a1 = C[b1]
    out[0] = a1
    ok = (S > 0) & (np.abs(_dot(C, a1[None, :])) <= sin_a)
    if not ok.any():
        return out, "NO_SECOND_AXIS"
    cand = np.flatnonzero(ok)
    b2 = int(cand[np.argmax(S[cand])])
    c2 = C[b2]
    t = _dot(c2, a1)
    d = c2 - t * a1
    a2 = d / np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
    out[1] = a2
    out[2] = [a1[1] * a2[2] - a1[2] * a2[1], a1[2] * a2[0] - a1[0] * a2[2], a1[0] * a2[1] - a1[1] * a2[0]]
    return out, "OK"


def planar(v, lambda2, rho):
    """the planar points from the per-point arrays: v finite (k >= m), lambda2 > 0 and v <= rho lambda2"""
    v = np.asarray(v, np.float64)
    l2 = np.asarray(lambda2, np.float64)
    with np.errstate(invalid="ignore"):
        return np.isfinite(v) & (l2 > 0.0) & (v <= rho * l2)


def families(normals, is_planar, ax, angle_deg):
    """family 0..2 of every planar point (the first axis with |n . a_j| >= cos(angle)), -1 otherwise"""
    n = np.asarray(normals, np.float64).reshape(-1, 3)
    cos_a = math.cos(angle_deg * math.pi / 180.0)
    fam = np.full(len(n), -1, np.int8)
    for j in (2, 1, 0):
        with np.errstate(invalid="ignore"):
            hit = is_planar & (np.abs(_dot(n, ax[j][None, :])) >= cos_a)
        fam[hit] = j
    return fam


def _tree(acc):
    """the xor shuffle tree over the last axis (32 lanes); lane 0's value"""
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[..., lane ^ o]
    return acc[..., 0]


def _lanes(x):
    """x (n_rows, L) -> per row, lane l's sequential sum of the entries l, l + 32, ..., then the tree"""
    n_rows, L = x.shape
    T = -(-L // 32)
    pad = np.zeros((n_rows, T * 32))
    pad[:, :L] = x
    acc = np.zeros((n_rows, 32))
    for t in range(T):
        acc = acc + pad[:, t * 32:(t + 1) * 32]
    return _tree(acc)


def fold(v, fam):
    """the library's fold: (n_j as int (3,), sum v_j (3,)) in its order (chunks of 1024 caller-order points, then the merge)"""
    v = np.asarray(v, np.float64)
    n = len(v)
    nch = -(-n // CHUNK)
    counts, sums = np.zeros(3, np.int64), np.zeros(3)
    for j in range(3):
        x = np.zeros(nch * CHUNK)
        x[:n] = np.where(fam == j, v, 0.0)
        part = _lanes(x.reshape(nch, CHUNK))
        sums[j] = _lanes(part[None, :])[0]
        counts[j] = int((fam == j).sum())
    return counts, sums


def statement(v, lambda2, normals, rho, angle_deg, min_family):
    """the whole rule from the per-point arrays: dict(hist, axis, status, family, n, mean, median, mom)"""
    pl = planar(v, lambda2, rho)
    h = histogram(np.asarray(normals).reshape(-1, 3)[pl])
    ax, status = axes(h, angle_deg)
    out = dict(hist=h, axis=ax, status=status, n_planar=int(pl.sum()))
    if status != "OK":
        out.update(family=np.full(len(v), -1, np.int8), n=np.zeros(3, np.int64), mean=np.full(3, np.nan),
                   median=np.full(3, np.nan), mom=math.nan)
        return out
    fam = families(normals, pl, ax, angle_deg)
    n, s = fold(v, fam)
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = np.where(n > 0, s / np.maximum(n, 1), np.nan)
    med = np.array([np.quantile(np.asarray(v)[fam == j], 0.5, method="linear") if n[j] else np.nan for j in range(3)])
    if (n < min_family).any():
        status = "SMALL_FAMILY"
    mom = med[0] + med[1] + med[2] if status == "OK" else math.nan
    out.update(family=fam, n=n, mean=mean, median=med, mom=mom, status=status)
    return out


def exact_normal(pts, i, nb):
    """(lambda2, lambda3, the unit eigenvector of lambda3, canonical sign) of the exact covariance of query i"""
    cov = CR.exact_cov(pts, i, nb)
    with mp.workdps(CR.DPS):
        Mx = mp.matrix([[mp.mpf(c.numerator) / c.denominator for c in row] for row in cov])
        w, V = mp.eigsy(Mx)
        order = sorted(range(3), key=lambda k: w[k])
        n = np.array([float(V[a, order[0]]) for a in range(3)])
        l3, l2 = float(w[order[0]]), float(w[order[1]])
    n /= np.linalg.norm(n)
    if n[int(np.argmax(np.abs(n)))] < 0:
        n = -n
    return l2, l3, n, cov


def normal_bound(pts, i, nb, cov, l2, l3):
    """the bound on sin(angle) between the fp64 normal and the exact one (module notes); inf when the gap does not cover eps"""
    eps = CR.fp64_bound(pts, i, nb, cov)
    gap = l2 - l3
    if gap <= eps:
        return math.inf, eps
    return eps / (gap - eps) + C_VEC * U, eps


def exact_points(pts, r, idx):
    """per sampled query: k, exact lambda2, lambda3, normal, the normal's sin bound and lambda2's bound (eps)"""
    pts = np.asarray(pts, np.float64)
    nbs = X.mme_neighbours(pts, r)
    out = dict(i=[], k=[], l2=[], l3=[], n=[], sin=[], eps=[])
    for i in idx:
        nb = nbs[i]
        if len(nb) < 3:
            continue
        l2, l3, n, cov = exact_normal(pts, i, nb)
        s, eps = normal_bound(pts, i, nb, cov, l2, l3)
        for f, x in zip(("i", "k", "l2", "l3", "n", "sin", "eps"), (i, len(nb), l2, l3, n, s, eps)):
            out[f].append(x)
    return {f: np.array(v) for f, v in out.items()}

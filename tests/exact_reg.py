"""Exact reference for registration (icp.cu): the k-NN normals, the ICP blocks and the updates me_icp_update takes from
them, evaluated without rounding on the CPU, with no use of the oracle or of the GPU (not collected as a test module).

Conventions of exact_ref.py: the fp64 decisions of the reference are reproduced in fp64 (d2_kd distances, the d2 < R^2
test of SearchHybrid, the tie to the smaller caller index), everything after them is exact (Fractions of the doubles,
mpmath at DPS digits for eigen-decompositions, SVDs and trigonometry), u = 2^-53.

k-NN normals (EstimateNormals(KNN k), k = min(20, n), the query included).  The covariance of the k neighbours is a
rational; lambda_0 <= lambda_1 <= lambda_2 and v_0 come from mpmath.  The kernel forms the covariance from the offsets
d = p - q to the query (cumulants about the query, knn_normals_kernel): every entry is within
  E_ij = C_NRM u (k + 2) (sum |d_i| |d_j| + |S1_i S1_j| / k) / k,   S1 = sum d,
the gamma_{k+2} bound of a k-term sum of products, the scaling and the centring, with a margin of C_NRM (exact_ref's
C_MME construction with the divisor k).  FastEigen3x3 takes the eigenvalues from acos(det / 2), whose error grows near a
double eigenvalue: with g = lambda_1 - lambda_0 its eigenvalue error is eps_s = C_EIG u lambda_2 max(1, lambda_2 / g), and
the cross products of the rows of C - (lambda_0 + eps_s) I leave a component eps_s / g along v_1.  For a device normal n:
  | |n| - 1 | <= C_EIG u;
  n^T C n - lambda_0 <= 2 E_F + C_EIG u lambda_2 + min(g, eps_s^2 / g) (E_F the Frobenius norm of E): no spectral gap is
  needed, so lines and isotropic blobs are covered;
  sin(n, v_0) <= (E_F + eps_s) / g (Davis-Kahan) where that is below SIN_DETERMINED.
An exactly diagonal covariance takes FastEigen3x3's axis branch, which returns the axis of the strictly smallest diagonal
entry and (0, 0, 1) otherwise, an eigenvector of the largest eigenvalue when a neighbourhood is collinear along z (k = 3
on a lattice): that axis is accepted as well as any normal within the bounds below.
The sign is FastEigen3x3's, a result rather than a convention (generalized ICP's Rx = I when n.x < -0.99): it must equal
that of fast_eigen3x3 below applied to the exactly rounded covariance, except where a branch decision of that statement
lies within TIE_REL of a tie.

ICP blocks.  From the moved source points, the target points and (methods 1, 2) the normals, the 17 or 29 values of
icp_accum_kernel / icp_ne_accum_kernel exactly: pairs kept by d2_kd < R^2, the point-to-point sums about c,
J = [v x n, n] and r = (v_s - v_t) . n_t for point-to-plane, and for generalized ICP gicp_cov with the Rx = I quirk,
C_s = R C(n_s) R^T and M^-1 by cofactors (each pair's terms as rationals, summed at DPS digits).  The count is exact.  The
bound of a value is C_REG u (m + 8) sum |term|: each term's fp64 error plus the gamma_m summation error over any order, with
|B| + kappa(M) |B|_max in place of |M^-1| for generalized ICP.

Updates (me_icp_update on a block, the block's doubles taken as exact).  Point-to-point: Umeyama without scaling from an
mpmath SVD of sigma = Sqp / n - qm pm^T; R is the rotation polar factor, bounded by C_REG u A / (s_2 + s_3) entrywise, with
A = s_1 + max |Sqp / n| + |qm| |pm| the scale sigma is formed at (a rank-2 sigma still has a unique R).  Point-to-plane
and generalized ICP: x = -(JTJ)^-1 JTr by exact elimination, bounded by C_REG u kappa(JTJ) |x| plus, when the block carries
a bound, its first-order effect; T = Rz Ry Rx with the translation x[3:].
"""
import math
from fractions import Fraction

import mpmath as mp
import numpy as np

from exact_ref import DPS, U, d2_kd

C_NRM = 4.0
C_EIG = 1024.0
C_REG = 64.0
SIN_DETERMINED = 1e-3     # Davis-Kahan is applied (and the sign compared) where the bound on the angle is below this
TIE_REL = 1e-6            # a branch decision of FastEigen3x3 within this relative distance of a tie exempts the sign
EPS_GICP = 1e-3           # TransformationEstimationForGeneralizedICP() default epsilon


def _F(x):
    return Fraction(float(x))


def _mpf(q):
    return mp.mpf(q.numerator) / q.denominator if isinstance(q, Fraction) else mp.mpf(q)


def gamma(m):
    return m * U / (1 - m * U)


# ---------------------------------------------------------------------------------------------------------------
# k-NN normals
# ---------------------------------------------------------------------------------------------------------------
def knn_exact(pts, queries, k, larger_index_on_tie=False):
    """per query index the k nearest caller indices by (d2_kd, index), the query included.  larger_index_on_tie is a
    deliberately wrong variant for the tests' teeth."""
    from scipy.spatial import cKDTree
    pts = np.asarray(pts, np.float64)
    k = min(k, len(pts))
    tree = cKDTree(pts)
    dk, _ = tree.query(pts[queries], k=k)
    dk = dk.reshape(len(queries), -1)[:, -1]
    out = []
    for qi, r in zip(queries, dk):
        cand = np.asarray(tree.query_ball_point(pts[qi], r * (1 + 1e-9) + 1e-300), dtype=np.int64)
        d2 = d2_kd(pts[qi], pts[cand])
        order = np.lexsort((-cand if larger_index_on_tie else cand, d2))
        out.append(cand[order[:k]])
    return out


def covariance_exact(pts, nb):
    """the covariance (1/k) sum (p - mean)(p - mean)^T of the points nb, as a 3x3 list of Fractions"""
    X = [[_F(v) for v in pts[j]] for j in nb]
    k = len(X)
    S = [sum(x[a] for x in X) for a in range(3)]
    return [[(k * sum(x[a] * x[b] for x in X) - S[a] * S[b]) / (k * k) for b in range(3)] for a in range(3)]


def covariance_bound(pts, q, nb):
    """E (3x3 floats): the entrywise bound of the kernel's covariance, moments about the query point q"""
    d = np.asarray(pts, np.float64)[nb] - np.asarray(q, np.float64)
    k = len(nb)
    ad = np.abs(d)
    s1 = d.sum(0)
    return C_NRM * U * (k + 2) * ((ad.T @ ad) + np.abs(np.outer(s1, s1)) / k) / k


def eig_exact(cov):
    """(lambda ascending (3 floats), v_0 (3 floats)) of a 3x3 Fraction matrix, in mpmath"""
    with mp.workdps(DPS):
        A = mp.matrix([[_mpf(cov[a][b]) for b in range(3)] for a in range(3)])
        E, Q = mp.eigsy(A)
        order = sorted(range(3), key=lambda i: E[i])
        return [float(E[i]) for i in order], np.array([float(Q[r, order[0]]) for r in range(3)])


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


class _Ties:
    """collects the relative distance to a tie of every branch decision"""
    def __init__(self):
        self.min_rel = math.inf

    def cmp(self, a, b):
        s = max(abs(a), abs(b))
        if s > 0:
            self.min_rel = min(self.min_rel, abs(a - b) / s)


def _evec0(A, ev, ties):
    r0, r1, r2 = [A[0] - ev, A[1], A[2]], [A[1], A[4] - ev, A[5]], [A[2], A[5], A[8] - ev]
    c = [_cross(r0, r1), _cross(r0, r2), _cross(r1, r2)]
    d = [_dot(v, v) for v in c]
    imax = 0
    if d[1] > d[imax]:
        imax = 1
    if d[2] > d[imax]:
        imax = 2
    for j in range(3):
        if j != imax:
            ties.cmp(d[j], d[imax])
    s = math.sqrt(d[imax])
    return [x / s for x in c[imax]]


def _evec1(A, e0, ev1, ties):
    ties.cmp(abs(e0[0]), abs(e0[1]))
    if abs(e0[0]) > abs(e0[1]):
        inv = 1.0 / math.sqrt(e0[0] * e0[0] + e0[2] * e0[2])
        Uv = [-e0[2] * inv, 0.0, e0[0] * inv]
    else:
        inv = 1.0 / math.sqrt(e0[1] * e0[1] + e0[2] * e0[2])
        Uv = [0.0, e0[2] * inv, -e0[1] * inv]
    V = _cross(e0, Uv)
    AU = [A[0] * Uv[0] + A[1] * Uv[1] + A[2] * Uv[2], A[1] * Uv[0] + A[4] * Uv[1] + A[5] * Uv[2],
          A[2] * Uv[0] + A[5] * Uv[1] + A[8] * Uv[2]]
    AV = [A[0] * V[0] + A[1] * V[1] + A[2] * V[2], A[1] * V[0] + A[4] * V[1] + A[5] * V[2],
          A[2] * V[0] + A[5] * V[1] + A[8] * V[2]]
    m00, m01, m11 = _dot(Uv, AU) - ev1, _dot(Uv, AV), _dot(V, AV) - ev1
    a00, a01, a11 = abs(m00), abs(m01), abs(m11)
    ties.cmp(a00, a11)
    if a00 >= a11:
        if max(a00, a01) > 0:
            ties.cmp(a00, a01)
            if a00 >= a01:
                m01 /= m00; m00 = 1 / math.sqrt(1 + m01 * m01); m01 *= m00
            else:
                m00 /= m01; m01 = 1 / math.sqrt(1 + m00 * m00); m00 *= m01
            return [m01 * Uv[j] - m00 * V[j] for j in range(3)]
        return Uv
    if max(a11, a01) > 0:
        ties.cmp(a11, a01)
        if a11 >= a01:
            m01 /= m11; m11 = 1 / math.sqrt(1 + m01 * m01); m01 *= m11
        else:
            m11 /= m01; m01 = 1 / math.sqrt(1 + m11 * m11); m11 *= m01
        return [m11 * Uv[j] - m01 * V[j] for j in range(3)]
    return Uv


def fast_eigen3x3(cov, ties=None):
    """Open3D's FastEigen3x3 (Eberly's robust 3x3 eigenvector, fast_eigen3x3_normal in icp.cu) in fp64: the normal of a
    row-major 3x3 covariance (9 floats), (0, 0, 1) for the zero matrix as knn_normals_kernel stores it.  ties (a _Ties)
    collects how close each branch decision came to a tie."""
    ties = ties if ties is not None else _Ties()
    cov = [float(x) for x in cov]
    mx = max(cov)
    if mx == 0:
        return [0.0, 0.0, 1.0]
    A = [x / mx for x in cov]
    norm = A[1] * A[1] + A[2] * A[2] + A[5] * A[5]
    ties.min_rel = min(ties.min_rel, math.sqrt(norm))          # zero off-diagonals: on the edge of the axis branch
    if norm > 0:
        q = (A[0] + A[4] + A[8]) / 3
        b00, b11, b22 = A[0] - q, A[4] - q, A[8] - q
        p = math.sqrt((b00 * b00 + b11 * b11 + b22 * b22 + norm * 2) / 6)
        c00, c01, c02 = b11 * b22 - A[5] * A[5], A[1] * b22 - A[5] * A[2], A[1] * A[5] - b11 * A[2]
        det = (b00 * c00 - A[1] * c01 + A[2] * c02) / (p * p * p)
        half_det = min(max(det * 0.5, -1.0), 1.0)
        ties.min_rel = min(ties.min_rel, abs(half_det))
        angle = math.acos(half_det) / 3.0
        tpi = 2.09439510239319549
        beta2, beta0 = math.cos(angle) * 2, math.cos(angle + tpi) * 2
        beta1 = -(beta0 + beta2)
        ev0, ev1, ev2 = q + p * beta0, q + p * beta1, q + p * beta2
        for a, b in ((ev0, ev1), (ev0, ev2), (ev1, ev2)):
            ties.cmp(a, b)
        if half_det >= 0:
            ea = _evec0(A, ev2, ties)
            if ev2 < ev0 and ev2 < ev1:
                return ea
            eb = _evec1(A, ea, ev1, ties)
            if ev1 < ev0 and ev1 < ev2:
                return eb
            return _cross(eb, ea)
        ea = _evec0(A, ev0, ties)
        if ev0 < ev1 and ev0 < ev2:
            return ea
        eb = _evec1(A, ea, ev1, ties)
        if ev1 < ev0 and ev1 < ev2:
            return eb
        return _cross(ea, eb)
    for a, b in ((0, 4), (0, 8), (4, 8)):
        ties.cmp(cov[a], cov[b])
    if cov[0] < cov[4] and cov[0] < cov[8]:
        return [1.0, 0.0, 0.0]
    if cov[4] < cov[0] and cov[4] < cov[8]:
        return [0.0, 1.0, 0.0]
    return [0.0, 0.0, 1.0]


def normals_exact(pts, queries=None, k=20, nbs=None):
    """per query: dict(nb, cov (Fractions), lam (ascending), v0, E (3x3), stmt (fast_eigen3x3 of the rounded covariance),
    tie (relative distance of its closest branch decision to a tie)).  Fewer than 3 neighbours: cov None (the kernel's
    identity covariance gives (0, 0, 1))."""
    pts = np.asarray(pts, np.float64)
    queries = np.arange(len(pts)) if queries is None else np.asarray(queries)
    nbs = knn_exact(pts, queries, k) if nbs is None else nbs
    out = []
    for qi, nb in zip(queries, nbs):
        row = dict(q=int(qi), nb=nb, cov=None, diagonal=False)       # diagonal: with a repeated smallest eigenvalue
        if len(nb) >= 3:
            cov = covariance_exact(pts, nb)
            lam, v0 = eig_exact(cov)
            t = _Ties()
            stmt = fast_eigen3x3([float(cov[a][b]) for a in range(3) for b in range(3)], t)
            if math.sqrt(_dot(stmt, stmt)) == 0.0:
                stmt = [0.0, 0.0, 1.0]
            row.update(cov=cov, lam=lam, v0=v0, E=covariance_bound(pts, pts[qi], nb),
                       diagonal=cov[0][1] == 0 and cov[0][2] == 0 and cov[1][2] == 0
                       and sorted(cov[a][a] for a in range(3))[0] == sorted(cov[a][a] for a in range(3))[1],
                       E_raw=covariance_bound(pts, np.zeros(3), nb), stmt=np.array(stmt), tie=t.min_rel)
        out.append(row)
    return out


def check_normal(row, n, raw=False):
    """the bounds of the module notes for one device normal n: dict(ok, why, sin_bound, sign_checked).  raw: the
    covariance was formed from cumulants of the raw coordinates (Open3D's ComputeCovariance, the oracle), whose entries
    are within E of the offsets from the origin instead"""
    n = np.asarray(n, np.float64)
    if row["cov"] is None:
        ok = n.tolist() == [0.0, 0.0, 1.0]
        return dict(ok=ok, why="" if ok else "fewer than 3 neighbours: not (0, 0, 1)", sin_bound=0.0, sign_checked=ok)
    if row["diagonal"] and n.tolist() == row["stmt"].tolist():
        # FastEigen3x3's axis branch on an exactly diagonal covariance with a repeated smallest eigenvalue
        return dict(ok=True, why="", sin_bound=0.0, sign_checked=False)
    lam, E = row["lam"], row["E_raw" if raw else "E"]
    l2 = max(abs(lam[2]), 0.0)
    EF = float(np.sqrt((E * E).sum()))
    if abs(float(np.linalg.norm(n)) - 1.0) > C_EIG * U:
        return dict(ok=False, why=f"|n| - 1 = {np.linalg.norm(n) - 1:.3g}", sin_bound=math.inf, sign_checked=False)
    gap = lam[1] - lam[0]
    eps_s = C_EIG * U * l2 * (max(1.0, l2 / gap) if gap > 0 else math.inf)
    with mp.workdps(DPS):
        nm = [mp.mpf(float(x)) for x in n]
        quad = sum(nm[a] * _mpf(row["cov"][a][b]) * nm[b] for a in range(3) for b in range(3)) / sum(x * x for x in nm)
        resid = float(quad - mp.mpf(lam[0]))
    rb = 2 * EF + C_EIG * U * l2 + (min(gap, eps_s * eps_s / gap) if gap > 0 else 0.0)
    if resid > rb:
        return dict(ok=False, why=f"Rayleigh residual {resid:.3g} > {rb:.3g}", sin_bound=math.inf, sign_checked=False)
    sb = (EF + eps_s) / gap if gap > 0 else math.inf
    if sb < SIN_DETERMINED:
        s = float(np.linalg.norm(np.cross(n, row["v0"]))) / float(np.linalg.norm(n))
        if s > sb * (1 + 1e-6) + 4 * U:
            return dict(ok=False, why=f"sin angle {s:.3g} > Davis-Kahan {sb:.3g}", sin_bound=sb, sign_checked=False)
    sign_checked = sb < SIN_DETERMINED and row["tie"] > TIE_REL
    if sign_checked and float(np.dot(n, row["stmt"])) <= 0:
        return dict(ok=False, why="sign differs from FastEigen3x3", sin_bound=sb, sign_checked=True)
    return dict(ok=True, why="", sin_bound=sb, sign_checked=sign_checked)


# ---------------------------------------------------------------------------------------------------------------
# ICP blocks
# ---------------------------------------------------------------------------------------------------------------
def kept_pairs(src, tgt, R):
    """(source indices, target indices, d2) of the pairs SearchHybrid(p, R, 1) keeps: the nearest target point by
    (d2_kd, index), kept iff d2 < R^2"""
    from scipy.spatial import cKDTree
    src, tgt = np.asarray(src, np.float64), np.asarray(tgt, np.float64)
    tree = cKDTree(tgt)
    d, _ = tree.query(src, k=1)
    si, ti, dd = [], [], []
    for i, r in enumerate(d):
        if not r * r < 4 * R * R:
            continue
        cand = np.asarray(tree.query_ball_point(src[i], r * (1 + 1e-9) + 1e-300), dtype=np.int64)
        d2 = d2_kd(src[i], tgt[cand])
        j = int(np.lexsort((cand, d2))[0])
        if d2[j] < R * R:
            si.append(i); ti.append(int(cand[j])); dd.append(float(d2[j]))
    return np.array(si, np.int64), np.array(ti, np.int64), np.array(dd)


def p2p_block_exact(p, q, d2, c):
    """the 17 values of icp_accum_kernel over the kept pairs (p source, q target, d2 their d2_kd): (Fractions, bounds)"""
    p, q, c = np.asarray(p, np.float64), np.asarray(q, np.float64), np.asarray(c, np.float64)
    m = len(p)
    P = [[_F(v) - _F(cc) for v, cc in zip(row, c)] for row in p]
    Q = [[_F(v) - _F(cc) for v, cc in zip(row, c)] for row in q]
    blk = [Fraction(m)]
    blk += [sum((x[a] for x in P), Fraction(0)) for a in range(3)]
    blk += [sum((x[a] for x in Q), Fraction(0)) for a in range(3)]
    blk += [sum((y[r] * x[col] for x, y in zip(P, Q)), Fraction(0)) for r in range(3) for col in range(3)]
    blk += [sum((_F(v) for v in d2), Fraction(0))]
    ap, aq = np.abs(p - c), np.abs(q - c)
    scale = np.concatenate([[0.0], ap.sum(0), aq.sum(0), (aq.T @ ap).reshape(9), [np.abs(d2).sum()]])
    return blk, C_REG * U * (m + 8) * scale


def gicp_cov_exact(x, R=None, eps=EPS_GICP, quirk=True):
    """GetRotationFromE1ToX(x) diag(eps, 1, 1) (...)^T with x as given, Rx = I when x0 < -0.99 (quirk=False drops that: a
    deliberately wrong variant), rotated by R: 3x3 Fractions"""
    x = [_F(v) for v in x]
    I3 = [[Fraction(int(a == b)) for b in range(3)] for a in range(3)]
    Q = I3
    if not (quirk and x[0] < Fraction(-99, 100)):
        f = 1 / (1 + x[0])
        Q = [[1 - f * (x[1] ** 2 + x[2] ** 2), -x[1], -x[2]],
             [x[1], 1 - f * x[1] ** 2, -f * x[1] * x[2]],
             [x[2], -f * x[1] * x[2], 1 - f * x[2] ** 2]]
    if R is not None:
        Rf = [[_F(v) for v in row] for row in R]
        Q = [[sum(Rf[a][t] * Q[t][b] for t in range(3)) for b in range(3)] for a in range(3)]
    D = [_F(eps), Fraction(1), Fraction(1)]
    return [[sum(D[t] * Q[a][t] * Q[b][t] for t in range(3)) for b in range(3)] for a in range(3)]


def _inv3(M):
    c00, c01, c02 = M[1][1] * M[2][2] - M[1][2] ** 2, M[0][2] * M[1][2] - M[0][1] * M[2][2], M[0][1] * M[1][2] - M[0][2] * M[1][1]
    c11, c12, c22 = M[0][0] * M[2][2] - M[0][2] ** 2, M[0][1] * M[0][2] - M[0][0] * M[1][2], M[0][0] * M[1][1] - M[0][1] ** 2
    det = M[0][0] * c00 + M[0][1] * c01 + M[0][2] * c02
    return [[c00 / det, c01 / det, c02 / det], [c01 / det, c11 / det, c12 / det], [c02 / det, c12 / det, c22 / det]]


def ne_block_exact(vs, vt, nt, d2, method, ns=None, R=None, cov=None):
    """the 29 values of icp_ne_accum_kernel over the kept pairs (vs moved source, vt target, nt target normals, ns source
    normals as given, R the rotation block of T): (values as Fractions / mpf, bounds).  method 1 point-to-plane, 2
    generalized ICP.  cov(n, R) replaces gicp_cov_exact (the tests' teeth)."""
    vs, vt, nt = (np.asarray(a, np.float64) for a in (vs, vt, nt))
    cov = cov or gicp_cov_exact
    m = len(vs)
    iu = [(a, b) for a in range(6) for b in range(a, 6)]
    acc = [mp.mpf(0)] * 27 if method == 2 else [Fraction(0)] * 27
    scale = np.zeros(27)
    with mp.workdps(DPS):
        for i in range(m):
            v = [_F(x) for x in vs[i]]
            d = [_F(a) - _F(b) for a, b in zip(vs[i], vt[i])]
            n = [_F(x) for x in nt[i]]
            if method == 1:
                J = _cross(v, n) + n
                r = _dot(d, n)
                terms = [J[a] * J[b] for a, b in iu] + [J[a] * r for a in range(6)]
                av, an = np.abs(vs[i]), np.abs(nt[i])
                Ja = np.concatenate([[av[1] * an[2] + av[2] * an[1], av[2] * an[0] + av[0] * an[2], av[0] * an[1] + av[1] * an[0]], an])
                ra = float(np.abs(vs[i] - vt[i]) @ an)
                scale += np.array([Ja[a] * Ja[b] for a, b in iu] + [Ja[a] * ra for a in range(6)])
                acc = [s + t for s, t in zip(acc, terms)]
            else:
                Mx = [[a + b for a, b in zip(ra_, rb_)] for ra_, rb_ in zip(cov(ns[i], R), cov(nt[i], None))]
                B = _inv3(Mx)
                A = [[0, v[2], -v[1], 1, 0, 0], [-v[2], 0, v[0], 0, 1, 0], [v[1], -v[0], 0, 0, 0, 1]]
                BA = [[sum(B[r][t] * A[t][col] for t in range(3)) for col in range(6)] for r in range(3)]
                g = [sum(B[r][t] * d[t] for t in range(3)) for r in range(3)]
                terms = [sum(A[t][a] * BA[t][b] for t in range(3)) for a, b in iu] + [sum(A[t][a] * g[t] for t in range(3)) for a in range(6)]
                acc = [s + _mpf(t) for s, t in zip(acc, terms)]
                Mf = np.array([[float(x) for x in row] for row in Mx])
                Bf = np.array([[float(x) for x in row] for row in B])
                Babs = np.abs(Bf) + np.linalg.cond(Mf) * np.abs(Bf).max()
                Aa = np.abs(np.array([[float(x) for x in row] for row in A]))
                da = np.abs(vs[i] - vt[i])
                JJ = Aa.T @ Babs @ Aa
                scale += np.concatenate([[JJ[a, b] for a, b in iu], Aa.T @ Babs @ da])
    blk = [Fraction(m)] + acc + [sum((_F(x) for x in d2), Fraction(0))]
    bound = C_REG * U * (m + 8) * np.concatenate([[0.0], scale, [np.abs(d2).sum()]])
    return blk, bound


def block_floats(blk):
    return np.array([float(x) for x in blk])


# ---------------------------------------------------------------------------------------------------------------
# updates
# ---------------------------------------------------------------------------------------------------------------
def umeyama_exact(blk, c):
    """the update me_icp_update computes from a point-to-point block (its doubles taken as exact) about c:
    (T 4x4 floats, bound 4x4 floats, singular values of sigma).  The bound is inf when s_2 + s_3 = 0."""
    b = [Fraction(float(x)) for x in blk]
    c = [Fraction(float(x)) for x in c]
    n = b[0]
    pm, qm = [b[1 + a] / n for a in range(3)], [b[4 + a] / n for a in range(3)]
    sig = [[b[7 + 3 * r + col] / n - qm[r] * pm[col] for col in range(3)] for r in range(3)]
    with mp.workdps(DPS):
        S = mp.matrix([[_mpf(sig[r][col]) for col in range(3)] for r in range(3)])
        Um, sv, Vt = mp.svd_r(S)
        d = mp.sign(mp.det(Um) * mp.det(Vt))
        D = mp.diag([1, 1, d if d != 0 else 1])
        Rm = Um * D * Vt
        src = mp.matrix([_mpf(pm[a] + c[a]) for a in range(3)])
        dst = mp.matrix([_mpf(qm[a] + c[a]) for a in range(3)])
        t = dst - Rm * src
        T = np.eye(4)
        for r in range(3):
            for col in range(3):
                T[r, col] = float(Rm[r, col])
            T[r, 3] = float(t[r])
        s = [float(sv[i]) for i in range(3)]
    A = s[0] + max(abs(float(b[7 + k] / n)) for k in range(9)) + max(map(abs, map(float, qm))) * max(map(abs, map(float, pm)))
    bR = C_REG * U * A / (s[1] + s[2]) if s[1] + s[2] > 0 else math.inf
    srcf = np.array([float(pm[a] + c[a]) for a in range(3)])
    mag = float(np.abs(srcf).sum() + np.abs([float(x) for x in qm]).sum() + 2 * np.abs([float(x) for x in c]).sum())
    bound = np.zeros((4, 4))
    bound[:3, :3] = bR
    bound[:3, 3] = bR * float(np.abs(srcf).sum()) + C_REG * U * mag
    return T, bound, s


def _solve_exact(M, rhs):
    """M x = rhs by Gaussian elimination in Fractions; None when M is singular"""
    n = len(rhs)
    A = [row[:] + [rhs[i]] for i, row in enumerate(M)]
    for col in range(n):
        piv = next((r for r in range(col, n) if A[r][col] != 0), None)
        if piv is None:
            return None
        A[col], A[piv] = A[piv], A[col]
        for r in range(col + 1, n):
            f = A[r][col] / A[col][col]
            if f:
                A[r] = [a - f * b for a, b in zip(A[r], A[col])]
    x = [Fraction(0)] * n
    for r in range(n - 1, -1, -1):
        x[r] = (A[r][n] - sum(A[r][k] * x[k] for k in range(r + 1, n))) / A[r][r]
    return x


def vec6_to_mat4(x):
    """TransformVector6dToMatrix4d in mpmath: Rz(x2) Ry(x1) Rx(x0), translation x[3:]"""
    with mp.workdps(DPS):
        a, b, g = (_mpf(v) if isinstance(v, Fraction) else mp.mpf(v) for v in x[:3])
        Rx = mp.matrix([[1, 0, 0], [0, mp.cos(a), -mp.sin(a)], [0, mp.sin(a), mp.cos(a)]])
        Ry = mp.matrix([[mp.cos(b), 0, mp.sin(b)], [0, 1, 0], [-mp.sin(b), 0, mp.cos(b)]])
        Rz = mp.matrix([[mp.cos(g), -mp.sin(g), 0], [mp.sin(g), mp.cos(g), 0], [0, 0, 1]])
        Rm = Rz * Ry * Rx
        T = np.eye(4)
        for r in range(3):
            for col in range(3):
                T[r, col] = float(Rm[r, col])
            T[r, 3] = float(_mpf(x[3 + r]) if isinstance(x[3 + r], Fraction) else x[3 + r])
    return T


def ne_update_exact(blk, blk_bound=None):
    """the update me_icp_update computes from a point-to-plane / generalized ICP block (its doubles taken as exact):
    (T 4x4, bound 4x4, x (6 floats), kappa).  blk_bound (the bound of the block's values) adds its first-order effect."""
    b = [Fraction(float(v)) for v in blk]
    JTJ = [[Fraction(0)] * 6 for _ in range(6)]
    t = 1
    for a in range(6):
        for c in range(a, 6):
            JTJ[a][c] = JTJ[c][a] = b[t]
            t += 1
    x = _solve_exact(JTJ, [-b[22 + a] for a in range(6)])
    if x is None:
        return np.eye(4), np.zeros((4, 4)), None, math.inf
    Jf = np.array([[float(v) for v in row] for row in JTJ])
    xf = np.array([float(v) for v in x])
    kappa = float(np.linalg.cond(Jf))
    bx = C_REG * U * kappa * float(np.linalg.norm(xf))
    if blk_bound is not None:
        bb = np.asarray(blk_bound, np.float64)
        dJ = np.zeros((6, 6))
        t = 1
        for a in range(6):
            for c in range(a, 6):
                dJ[a, c] = dJ[c, a] = bb[t]
                t += 1
        inv_norm = float(np.linalg.norm(np.linalg.inv(Jf), 2))
        bx += inv_norm * (float(np.linalg.norm(dJ, 2)) * float(np.linalg.norm(xf)) + float(np.linalg.norm(bb[22:28])))
    T = vec6_to_mat4(x)
    bound = np.zeros((4, 4))
    bound[:3, :3] = 3 * bx + C_REG * U
    bound[:3, 3] = bx + C_REG * U * np.abs(xf[3:])
    return T, bound, xf, kappa

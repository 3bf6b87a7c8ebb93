"""numpy statement of me_global_registration's five stages (not collected as a test module):

1. feature clouds: normals oriented towards v = centroid + (0, 0, 10 * bbox diagonal), flipped where n . (v - p) < 0;
2. FPFH: hybrid neighbourhoods (the <= max_nn nearest OTHER points with d^2 < r^2, d^2 = (dx dx + dy dy) + dz dz, ties
   to the smaller index), Open3D's ComputePairFeatures with the swap acos|a1| > acos|a2| evaluated as |a1| < |a2|, norms
   and dots in Eigen's order x*x + (y*y + z*z), 11 bins per group (clamped), SPFH increments 100 / k, FPFH = SPFH + the
   neighbours' SPFH weighted by 1 / d^2 and normalised to 100 per group, stored as fp32;
3. exact fp32 matching: squared distances summed in dimension order, every operation rounded (numpy does not fuse), ties
   to the smaller index; the mutual filter;
4. RANSAC: draws uniform53(seed, h, 16 + t) of perturb_ref, the edge check on squared lengths, the rank check (w1 > 1e-6 w0
   of the three's cross-covariance), the one-sided Jacobi SVD and
   Umeyama of svd3.cuh restated operation by operation (vectorised over hypotheses), inlier counts, the winner;
5. the refinement over the winner's inliers and n_inliers / inlier_rmse under it.

Every operation the device rounds is rounded here in the same order, with one exception: atan2 of the device and of libm
may differ in the last bit.  pair_features therefore flags the pairs whose f0, f1 or f2 lies within 1e-12 of an inner bin
edge; everywhere else the bins, and with them SPFH and FPFH, are the device's bit for bit.
"""
import numpy as np
from scipy.spatial import cKDTree

import perturb_ref

FPFH_DIM = 33
EDGE_TOL = 1e-12
LANE_DRAW = 16          # RANSAC draws: lanes 16, 17, 18
RANK_EPS = 1e-6         # a hypothesis is rejected when w1 <= RANK_EPS w0 (collinear triples)


# ---- 1. orientation -------------------------------------------------------------------------------------------------
def orient_normals(xyz, nrm, tol=1e-9):
    """(oriented normals, ambiguous mask): flip where n . (v - p) < 0; ambiguous where |n . (v - p)| <= tol |v - p|, a
    decision the rounding of the centroid could change"""
    xyz, nrm = np.asarray(xyz, np.float64), np.asarray(nrm, np.float64)
    c = xyz.mean(0)
    diag = np.sqrt(((xyz.max(0) - xyz.min(0)) ** 2).sum())
    v = c + np.array([0.0, 0.0, 10.0 * diag])
    dv = v - xyz
    d = nrm[:, 0] * dv[:, 0] + nrm[:, 1] * dv[:, 1] + nrm[:, 2] * dv[:, 2]
    out = np.where((d < 0)[:, None], -nrm, nrm)
    return out, np.abs(d) <= tol * np.linalg.norm(dv, axis=1)


# ---- 2. FPFH --------------------------------------------------------------------------------------------------------
def d2_kd(a, b):
    d = a - b
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def hybrid_neighbours(xyz, radius, max_nn, queries=None, larger_index_on_tie=False, closed=False, skip_self=True):
    """per point (or per index of queries) (indices, d2): the <= max_nn nearest other points with d2 < radius^2, sorted by
    (d2, index).  larger_index_on_tie (ties to the larger index), closed (d2 <= radius^2) and skip_self=False (the point is
    its own neighbour) are deliberately wrong variants for the tests' teeth."""
    xyz = np.asarray(xyz, np.float64)
    tree = cKDTree(xyz)
    r2 = radius * radius
    queries = np.arange(len(xyz)) if queries is None else np.asarray(queries, np.int64)
    cand = tree.query_ball_point(xyz[queries], radius * (1 + 1e-9) + 1e-12, workers=-1)
    out = []
    for i, c in zip(queries, cand):
        c = np.asarray(c, np.int64)
        if skip_self:
            c = c[c != i]
        d2 = d2_kd(xyz[i], xyz[c])
        keep = d2 <= r2 if closed else d2 < r2
        c, d2 = c[keep], d2[keep]
        o = np.lexsort((-c if larger_index_on_tie else c, d2))[:max(max_nn, 0)]
        out.append((c[o], d2[o]))
    return out


def _dot(a, b):
    return a[..., 0] * b[..., 0] + (a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2])


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def pair_features(p1, n1, p2, n2):
    """(f (m, 3), flagged (m,)) for pairs of rows: (f0, f1, f2) = (atan2(w . n2, n1 . n2), v . n2, n1 . d / |d|) in the
    frame of the swapped pair; zeros for coincident points or n1 parallel to the line"""
    p1, n1, p2, n2 = (np.atleast_2d(np.asarray(x, np.float64)) for x in (p1, n1, p2, n2))
    dp = p2 - p1
    ln = np.sqrt(_dot(dp, dp))
    with np.errstate(divide="ignore", invalid="ignore"):
        a1, a2 = _dot(n1, dp) / ln, _dot(n2, dp) / ln
        swap = np.abs(a1) < np.abs(a2)
        m1 = np.where(swap[:, None], n2, n1)
        m2 = np.where(swap[:, None], n1, n2)
        dp = np.where(swap[:, None], -dp, dp)
        f2 = np.where(swap, -a2, a1)
        v = _cross(dp, m1)
        vn = np.sqrt(_dot(v, v))
        v = v / vn[:, None]
        w = _cross(m1, v)
        f = np.stack([np.arctan2(_dot(w, m2), _dot(m1, m2)), _dot(v, m2), f2], 1)
    f[(ln == 0) | (vn == 0)] = 0.0
    return f, bin_edge_flags(f)


def _scaled(f):
    return np.stack([11.0 * (f[:, 0] + np.pi) / (2.0 * np.pi), 11.0 * (f[:, 1] + 1.0) * 0.5, 11.0 * (f[:, 2] + 1.0) * 0.5], 1)


def pair_bins(f):
    """(m, 3) bins in 0..32: floor of the scaled feature, clamped to 0..10, groups at 0, 11, 22"""
    return np.clip(np.floor(_scaled(f)), 0, 10).astype(np.int64) + np.array([0, 11, 22])


def bin_edge_flags(f):
    """pairs with a feature within EDGE_TOL of an inner bin edge (in feature units)"""
    t = _scaled(f)
    r = np.round(t)
    width = np.array([2.0 * np.pi / 11.0, 2.0 / 11.0, 2.0 / 11.0])
    return ((np.abs(t - r) * width < EDGE_TOL) & (r >= 1) & (r <= 10)).any(1)


def spfh(xyz, nrm, nbrs):
    """(SPFH (N, 33) fp64, flagged (N,)): increments of 100 / k added in neighbour order"""
    xyz, nrm = np.asarray(xyz, np.float64), np.asarray(nrm, np.float64)
    n = len(xyz)
    cnt = np.array([len(ix) for ix, _ in nbrs])
    h = np.zeros((n, FPFH_DIM))
    flagged = np.zeros(n, bool)
    src = np.repeat(np.arange(n), cnt)
    dst = np.concatenate([ix for ix, _ in nbrs]) if n else np.zeros(0, np.int64)
    rank = np.concatenate([np.arange(c) for c in cnt]) if n else np.zeros(0, np.int64)
    f, fl = pair_features(xyz[src], nrm[src], xyz[dst], nrm[dst])
    b = pair_bins(f)
    np.logical_or.at(flagged, src, fl)
    with np.errstate(divide="ignore"):
        inc = 100.0 / cnt.astype(np.float64)
    for r in range(int(cnt.max(initial=0))):      # the r-th neighbour of every point: one sequential step per point
        sel = rank == r
        for g in range(3):
            h[src[sel], b[sel, g]] += inc[src[sel]]
    return h, flagged


def fpfh(sp, nbrs, sp_flagged=None):
    """(FPFH (N, 33) fp32, FPFH fp64, flagged (N,)): point i is flagged when its SPFH or a neighbour's is"""
    n = len(sp)
    acc = np.zeros((n, FPFH_DIM))
    s = np.zeros((n, 3))
    cnt = np.array([len(ix) for ix, _ in nbrs])
    for r in range(int(cnt.max(initial=0))):
        pts = np.flatnonzero(cnt > r)
        j = np.array([nbrs[i][0][r] for i in pts], np.int64)
        d2 = np.array([nbrs[i][1][r] for i in pts])
        ok = d2 != 0.0
        pts, j, d2 = pts[ok], j[ok], d2[ok]
        val = sp[j] / d2[:, None]
        for b in range(FPFH_DIM):
            s[pts, b // 11] += val[:, b]
            acc[pts, b] += val[:, b]
    with np.errstate(divide="ignore"):
        scale = np.where(s != 0.0, 100.0 / s, 0.0)
    f64 = acc * np.repeat(scale, 11, axis=1) + sp
    flagged = np.zeros(n, bool)
    if sp_flagged is not None:
        flagged |= sp_flagged
        for i in range(n):
            if len(nbrs[i][0]) and sp_flagged[nbrs[i][0]].any():
                flagged[i] = True
    return f64.astype(np.float32), f64, flagged


def fpfh_sample(xyz, nrm, radius, max_nn, sample):
    """(FPFH fp32, FPFH fp64, flagged) of the points `sample` alone, from the neighbourhoods of the sample and of its
    neighbours: what features() gives at those rows, at a cost that does not grow with the cloud"""
    xyz = np.asarray(xyz, np.float64)
    sample = np.asarray(sample, np.int64)
    n = len(xyz)
    empty = (np.zeros(0, np.int64), np.zeros(0))
    nb_s = hybrid_neighbours(xyz, radius, max_nn, sample)
    ring = np.setdiff1d(np.unique(np.concatenate([ix for ix, _ in nb_s] + [np.zeros(0, np.int64)])), sample)
    nb_r = hybrid_neighbours(xyz, radius, max_nn, ring)
    nbrs = [empty] * n
    for i, v in zip(sample, nb_s):
        nbrs[i] = v
    for i, v in zip(ring, nb_r):
        nbrs[i] = v
    sp, fl = spfh(xyz, nrm, nbrs)
    only = [empty] * n
    for i, v in zip(sample, nb_s):
        only[i] = v
    f32, f64, ffl = fpfh(sp, only, fl)
    return f32[sample], f64[sample], ffl[sample]


def features(xyz, nrm, radius, max_nn):
    """(FPFH fp32, FPFH fp64, flagged, neighbourhoods) of a feature cloud with its (oriented) normals"""
    nb = hybrid_neighbours(xyz, radius, max_nn)
    sp, fl = spfh(xyz, nrm, nb)
    f32, f64, ffl = fpfh(sp, nb, fl)
    return f32, f64, ffl, nb


# ---- 3. matching ----------------------------------------------------------------------------------------------------
def feature_nn(Qd, Rd, chunk=512):
    """nn[i] = argmin_j sum_b (Qd_ib - Rd_jb)^2 in fp32, summed in b order, every operation rounded; ties: smaller j"""
    Qd, Rd = np.asarray(Qd, np.float32), np.asarray(Rd, np.float32)
    out = np.empty(len(Qd), np.int64)
    for s in range(0, len(Qd), chunk):
        q = Qd[s:s + chunk]
        d = np.zeros((len(q), len(Rd)), np.float32)
        for b in range(FPFH_DIM):
            t = q[:, b, None] - Rd[None, :, b]
            d = d + t * t
        out[s:s + chunk] = np.argmin(d, axis=1)
    return out


def correspondences(fe, fg, mutual=True):
    """(est index, gt index) pairs in est order"""
    e2g = feature_nn(fe, fg)
    if not mutual:
        return np.arange(len(fe)), e2g
    g2e = feature_nn(fg, fe)
    keep = g2e[e2g] == np.arange(len(fe))
    return np.flatnonzero(keep), e2g[keep]


# ---- 4. RANSAC ------------------------------------------------------------------------------------------------------
def draws(seed, nh, nc):
    """(nh, 3) correspondence indices min(floor(uniform53(seed, h, 16 + t) * nc), nc - 1)"""
    h = np.arange(nh, dtype=np.uint64)
    cols = [np.minimum(np.floor(perturb_ref.uniform53(seed, h, LANE_DRAW + t) * float(nc)), nc - 1) for t in range(3)]
    return np.stack(cols, 1).astype(np.int64)


def edge_ok(P, Q, ids, ratio):
    """distinct indices and min^2 >= ratio^2 max^2 of every edge's squared lengths"""
    ok = (ids[:, 0] != ids[:, 1]) & (ids[:, 0] != ids[:, 2]) & (ids[:, 1] != ids[:, 2])
    r2 = ratio * ratio
    for a, b in ((0, 1), (0, 2), (1, 2)):
        ds, dt = _sq3(P[ids[:, a]] - P[ids[:, b]]), _sq3(Q[ids[:, a]] - Q[ids[:, b]])
        ok &= np.minimum(ds, dt) >= r2 * np.maximum(ds, dt)
    return ok


def _sq3(d):
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def svd3(s):
    """svd3.cuh's one-sided Jacobi on (H, 9) row-major matrices: (U (H, 9) with its third column zero, w (H, 3), V (H, 9))"""
    a = np.array(s, np.float64).reshape(-1, 9).copy()
    H = len(a)
    V = np.tile(np.eye(3).reshape(9), (H, 1))
    active = np.ones(H, bool)
    for _ in range(60):
        off = np.zeros(H)
        for p, q in ((0, 1), (0, 2), (1, 2)):
            alpha, beta, gamma = np.zeros(H), np.zeros(H), np.zeros(H)
            for k in range(3):
                alpha = alpha + a[:, k * 3 + p] * a[:, k * 3 + p]
                beta = beta + a[:, k * 3 + q] * a[:, k * 3 + q]
                gamma = gamma + a[:, k * 3 + p] * a[:, k * 3 + q]
            m = active & (gamma != 0.0)
            with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
                rel = np.abs(gamma) / np.sqrt(alpha * beta)
                off = np.where(m & (off < rel), rel, off)
                zeta = (beta - alpha) / (2.0 * gamma)
                t = np.where(zeta >= 0, 1.0, -1.0) / (np.abs(zeta) + np.sqrt(1.0 + zeta * zeta))
                c = 1.0 / np.sqrt(1.0 + t * t)
                sn = c * t
            for k in range(3):
                ap, aq = a[:, k * 3 + p].copy(), a[:, k * 3 + q].copy()
                a[m, k * 3 + p] = (c * ap - sn * aq)[m]
                a[m, k * 3 + q] = (sn * ap + c * aq)[m]
                vp, vq = V[:, k * 3 + p].copy(), V[:, k * 3 + q].copy()
                V[m, k * 3 + p] = (c * vp - sn * vq)[m]
                V[m, k * 3 + q] = (sn * vp + c * vq)[m]
        active &= ~(off < 1e-15)
        if not active.any():
            break
    nw = np.stack([np.sqrt((a[:, j] * a[:, j] + a[:, 3 + j] * a[:, 3 + j]) + a[:, 6 + j] * a[:, 6 + j]) for j in range(3)], 1)
    order = np.argsort(-nw, axis=1, kind="stable")
    rows = np.arange(H)[:, None]
    w = nw[rows, order]
    U, Vs = np.zeros((H, 9)), np.zeros((H, 9))
    for j in range(3):
        for k in range(3):
            Vs[:, k * 3 + j] = V[np.arange(H), k * 3 + order[:, j]]
            if j < 2:
                with np.errstate(divide="ignore", invalid="ignore"):
                    U[:, k * 3 + j] = np.where(w[:, j] > 0, a[np.arange(H), k * 3 + order[:, j]] / w[:, j], 0.0)
    return U, w, Vs


def _det3(m):
    return (m[:, 0] * (m[:, 4] * m[:, 8] - m[:, 5] * m[:, 7]) - m[:, 1] * (m[:, 3] * m[:, 8] - m[:, 5] * m[:, 6])
            + m[:, 2] * (m[:, 3] * m[:, 7] - m[:, 4] * m[:, 6]))


def umeyama_from_sums(blk, c, with_sv=False):
    """svd3.cuh's umeyama_from_sums on (H, >= 16) blocks [count, sum p, sum q, sum q p^T] about c: (H, 4, 4), and with
    with_sv the singular values of sigma (H, 3)"""
    blk = np.atleast_2d(np.asarray(blk, np.float64))
    c = np.asarray(c, np.float64)
    n = blk[:, 0:1]
    pm, qm = blk[:, 1:4] / n, blk[:, 4:7] / n
    sigma = np.stack([blk[:, 7 + 3 * r + col] / n[:, 0] - qm[:, r] * pm[:, col] for r in range(3) for col in range(3)], 1)
    U, sv, Vs = svd3(sigma)
    U[:, 2] = U[:, 3] * U[:, 7] - U[:, 6] * U[:, 4]
    U[:, 5] = U[:, 6] * U[:, 1] - U[:, 0] * U[:, 7]
    U[:, 8] = U[:, 0] * U[:, 4] - U[:, 3] * U[:, 1]
    S = np.ones((len(blk), 3))
    S[_det3(U) * _det3(Vs) < 0, 2] = -1.0
    T = np.zeros((len(blk), 4, 4))
    T[:, 3, 3] = 1.0
    for r in range(3):
        for col in range(3):
            s = np.zeros(len(blk))
            for k in range(3):
                s = s + U[:, r * 3 + k] * S[:, k] * Vs[:, col * 3 + k]
            T[:, r, col] = s
    for r in range(3):
        rp = np.zeros(len(blk))
        for k in range(3):
            rp = rp + T[:, r, k] * (pm[:, k] + c[k])
        T[:, r, 3] = (qm[:, r] + c[r]) - rp
    return (T, sv) if with_sv else T


def three_point_sums(P, Q, ids, c):
    """the ME_ICP_BLOCK_P2P block of the three correspondences of every hypothesis, summed in t order about c"""
    H = len(ids)
    blk = np.zeros((H, 17))
    blk[:, 0] = 3.0
    for t in range(3):
        pc, qc = P[ids[:, t]] - c, Q[ids[:, t]] - c
        blk[:, 1:4] += pc
        blk[:, 4:7] += qc
        for r in range(3):
            for col in range(3):
                blk[:, 7 + 3 * r + col] += qc[:, r] * pc[:, col]
    return blk


def residual2(T, P, Q):
    """(H, m) |T p - q|^2 with the rows applied left to right, as the device rounds them"""
    T = T if T.ndim == 3 else T[None]
    out = []
    for r in range(3):
        x = ((T[:, r, 0, None] * P[None, :, 0] + T[:, r, 1, None] * P[None, :, 1]) + T[:, r, 2, None] * P[None, :, 2]) \
            + T[:, r, 3, None] - Q[None, :, r]
        out.append(x)
    return (out[0] * out[0] + out[1] * out[1]) + out[2] * out[2]


def inlier_counts(T, P, Q, d2max, chunk=256):
    return np.concatenate([(residual2(T[s:s + chunk], P, Q) < d2max).sum(1) for s in range(0, len(T), chunk)]) \
        if len(T) else np.zeros(0, np.int64)


def ransac(P, Q, c, seed, n_hypotheses, ratio, d2max):
    """dict(valid, counts, T (H, 4, 4), best, n_valid): every hypothesis; the winner has the most inliers, ties to the smallest h"""
    P, Q = np.asarray(P, np.float64), np.asarray(Q, np.float64)
    ids = draws(seed, n_hypotheses, len(P))
    valid = edge_ok(P, Q, ids, ratio)
    T = np.zeros((n_hypotheses, 4, 4))
    counts = np.full(n_hypotheses, -1, np.int64)
    vi = np.flatnonzero(valid)
    if len(vi):
        Tv, sv = umeyama_from_sums(three_point_sums(P, Q, ids[vi], c), c, with_sv=True)
        T[vi] = Tv
        valid[vi] = sv[:, 1] > RANK_EPS * sv[:, 0]
        vi = np.flatnonzero(valid)
        counts[vi] = inlier_counts(T[vi], P, Q, d2max)
    best = int(np.flatnonzero(counts == counts.max())[0]) if len(vi) else -1
    return dict(valid=valid, counts=counts, T=T, best=best, n_valid=int(valid.sum()), ids=ids)


# ---- 5. refinement --------------------------------------------------------------------------------------------------
def refine(P, Q, c, T_win, d2max):
    """(T, n_inliers, inlier_rmse): the rigid fit over the winner's inliers (the winner's T with fewer than 3), and its
    inliers among all correspondences"""
    P, Q = np.asarray(P, np.float64), np.asarray(Q, np.float64)
    m = residual2(T_win[None], P, Q)[0] < d2max
    T = T_win
    if m.sum() >= 3:
        pc, qc = P[m] - c, Q[m] - c
        blk = np.zeros(17)
        blk[0] = m.sum()
        blk[1:4], blk[4:7] = pc.sum(0), qc.sum(0)
        blk[7:16] = (qc[:, :, None] * pc[:, None, :]).sum(0).reshape(9)
        T = umeyama_from_sums(blk, c)[0]
    r2 = residual2(T[None], P, Q)[0]
    k = r2 < d2max
    return T, int(k.sum()), float(np.sqrt(r2[k].sum() / k.sum())) if k.any() else 0.0

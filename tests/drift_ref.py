"""numpy statement of the drift per region (me_drift*, drift.cu), bit for bit (not collected as a test module).

Regions: floor(x / s) per axis of the estimated cloud as handed in (IEEE division), listed ascending by (ix, iy, iz); a
region's points in caller order.  Each iteration:
  1. every point := T_r x^orig in transform_kernel's order (((T0 x + T1 y) + T2 z) + T3) / w, from the original coordinates;
  2. the nearest ground-truth point by (d2_kd, index), kept iff d2 < R^2 (exact_reg.kept_pairs);
  3. per region the 17 values of ME_ICP_BLOCK_P2P about c_r = (index + 0.5) s, in the fold's order: the region's points cut
     into chunks of CHUNK in caller order, lane l of a chunk adds the points l, l + 32, ... one rounded operation at a time,
     the 32 lanes are combined by the shuffle tree (lane l + o added to lane l for o = 16, 8, 4, 2, 1), and the chunks are
     added in chunk order starting from 0;
  4. the host update of drift_step: fitness, rmse, me_icp_step's convergence test, me_icp_update (the library's own host
     function) and T := update T with the 4 x 4 product summed from 0 in k order.
Adding 0.0 for a point that is not kept leaves every partial sum as it is (no partial sum is -0.0), so the statement adds
zeros where the kernel skips.
"""
import math

import numpy as np

from exact_ref import d2_kd
from exact_reg import kept_pairs

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import api, synth

CHUNK = 1024
NB = A.ME_ICP_BLOCK_P2P


def regions(est, s):
    """(index (R, 3) int64 ascending, rid (n,) int64) of the est points"""
    k = np.floor(np.asarray(est, np.float64) / float(s)).astype(np.int64)
    index, rid = np.unique(k, axis=0, return_inverse=True)
    return index, rid.reshape(-1)


def transform(orig, rid, T):
    """every point by the transform of its region, transform_kernel's rounding"""
    M = T[rid]
    x, y, z = orig[:, 0], orig[:, 1], orig[:, 2]
    o = [((M[:, r, 0] * x + M[:, r, 1] * y) + M[:, r, 2] * z) + M[:, r, 3] for r in range(4)]
    return np.stack([o[0] / o[3], o[1] / o[3], o[2] / o[3]], axis=1)


def nearest(src, tgt, R):
    """(nn index or -1, d2) per source point: exact_reg.kept_pairs, with the points whose nearest target is not in doubt
    (the second nearest is clearly farther) taken from one k-d tree query"""
    from scipy.spatial import cKDTree
    src, tgt = np.asarray(src, np.float64), np.asarray(tgt, np.float64)
    d, j = cKDTree(tgt).query(src, k=2)
    nn = j[:, 0].astype(np.int64)
    d2 = d2_kd(src, tgt[nn])
    doubt = ~(d[:, 1] - d[:, 0] > 1e-7 * d[:, 1] + 1e-12)
    keep = (d2 < R * R) & ~doubt
    out = np.where(keep, nn, -1)
    if doubt.any():
        sel = np.flatnonzero(doubt)
        si, ti, dd = kept_pairs(src[sel], tgt, R)
        out[sel[si]] = ti
        d2[sel[si]] = dd
    return out, d2


class Layout:
    """the fold's placement of every point: chunk, lane and step (the lane's k-th point), and the region of every chunk"""
    def __init__(self, rid, R):
        order = np.argsort(rid, kind="stable")                  # caller order inside a region
        counts = np.bincount(rid, minlength=R)
        start = np.concatenate([[0], np.cumsum(counts)])
        rank = np.arange(len(rid)) - start[rid[order]]          # position of the point inside its region
        nch = (counts + CHUNK - 1) // CHUNK
        self.chunk_off = np.concatenate([[0], np.cumsum(nch)])
        self.n_chunks = int(self.chunk_off[-1])
        self.order = order
        self.chunk = self.chunk_off[rid[order]] + rank // CHUNK
        self.lane = (rank % CHUNK) % 32
        self.step = (rank % CHUNK) // 32
        self.R = R


def fold(L, terms):
    """(R, F) block from per-point terms (n, F) in caller order, in the kernel's summation order"""
    t = np.asarray(terms, np.float64)[L.order]
    F = t.shape[1]
    acc = np.zeros((L.n_chunks, 32, F))
    for st in range(CHUNK // 32):
        m = L.step == st
        acc[L.chunk[m], L.lane[m]] = acc[L.chunk[m], L.lane[m]] + t[m]
    o = 16
    while o:
        acc = acc[:, :o] + acc[:, o:2 * o]
        o //= 2
    part = acc[:, 0]
    blk = np.zeros((L.R, F))
    per = np.diff(L.chunk_off)
    for k in range(int(per.max()) if L.R else 0):
        r = np.flatnonzero(per > k)
        blk[r] = blk[r] + part[L.chunk_off[r] + k]
    return blk


def block_terms(moved, gt, nn, d2, R, c_pt):
    """the 17 terms of every est point (zeros where the pair is not kept), about its region's centre c_pt (n, 3)"""
    kept = (nn >= 0) & (d2 < R * R)
    p = moved - c_pt
    q = np.where(kept[:, None], gt[np.maximum(nn, 0)], 0.0) - c_pt
    t = np.zeros((len(moved), NB))
    t[:, 0] = 1.0
    t[:, 1:4] = p
    t[:, 4:7] = q
    for r in range(3):
        for col in range(3):
            t[:, 7 + 3 * r + col] = q[:, r] * p[:, col]
    t[:, 16] = d2
    t[~kept] = 0.0
    return t


def mat4(upd, T):
    """drift_step's 4 x 4 product upd T, each entry summed from 0 in k order"""
    s = np.zeros_like(T)
    for k in range(4):
        s = s + upd[..., :, k, None] * T[..., None, k, :]
    return s


def drift(est, gt, s, R, max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6, compound=False, sweep=nearest):
    """the whole loop: (rows as api.drift_dict, the block of every iteration (list of (R, 17) arrays)).  compound=True moves the
    moved coordinates by each update instead of the originals by T (a deliberately wrong variant for the tests' teeth)."""
    est, gt = np.asarray(est, np.float64), np.asarray(gt, np.float64)
    s, R = float(s), float(R)
    index, rid = regions(est, s)
    nR = len(index)
    L = Layout(rid, nR)
    c = (index.astype(np.float64) + 0.5) * s
    cpt = c[rid]
    cen_terms = np.zeros((len(est), NB))
    cen_terms[:, 0] = 1.0
    cen_terms[:, 1:4] = est - cpt
    cb = fold(L, cen_terms)
    centroid = c + cb[:, 1:4] / cb[:, :1]
    n_est = np.bincount(rid, minlength=nR)
    T = np.tile(np.eye(4), (nR, 1, 1))
    status = np.full(nR, -1, np.int32)
    it = np.zeros(nR, np.int32)
    fit = np.zeros(nR); rmse = np.zeros(nR); ncorr = np.zeros(nR, np.int64)
    fit0 = np.zeros(nR); rmse0 = np.zeros(nR); ncorr0 = np.zeros(nR, np.int64)
    blocks = []
    moved = transform(est, rid, T)
    have_prev = False
    while True:
        nn, d2 = sweep(moved, gt, R)
        blk = fold(L, block_terms(moved, gt, nn, d2, R, cpt))
        blocks.append(blk)
        upd_all = np.tile(np.eye(4), (nR, 1, 1))
        running = False
        for r in np.flatnonzero(status < 0):
            b = blk[r]
            nc = int(round(b[0]))
            f = nc / float(n_est[r])
            e = math.sqrt(b[16] / nc) if nc > 0 else 0.0
            conv = False
            if have_prev:
                it[r] += 1
                conv = abs(fit[r] - f) < relative_fitness and abs(rmse[r] - e) < relative_rmse
            else:
                ncorr0[r], fit0[r], rmse0[r] = nc, f, e
            ncorr[r], fit[r], rmse[r] = nc, f, e
            if conv:
                status[r] = A.ME_DRIFT_CONVERGED
            elif it[r] >= max_iteration:
                status[r] = A.ME_DRIFT_ITERATION_LIMIT
            elif nc < 3:
                status[r] = A.ME_DRIFT_TOO_FEW
            else:
                upd_all[r] = api.icp_update(A.ME_ICP_POINT_TO_POINT, b, c[r])
                running = True
        run = np.flatnonzero(status < 0)
        T[run] = mat4(upd_all[run], T[run])
        have_prev = True
        if not running:
            break
        if compound:
            moved = transform(moved, rid, upd_all)
        else:
            moved = transform(est, rid, T)
    rows = dict(index=index, min=index * s, max=(index + 1) * s, n_est=n_est, n_corr_before=ncorr0, fitness_before=fit0,
                rmse_before=rmse0, n_corr=ncorr, fitness=fit, rmse=rmse, T=T, centroid=centroid, iterations=it, status=status)
    Tc = np.stack([((T[:, a, 0] * centroid[:, 0] + T[:, a, 1] * centroid[:, 1]) + T[:, a, 2] * centroid[:, 2]) + T[:, a, 3]
                   for a in range(3)], axis=1)
    rows["shift"] = Tc - centroid
    sh = rows["shift"]
    rows["shift_norm"] = np.sqrt((sh[:, 0] * sh[:, 0] + sh[:, 1] * sh[:, 1]) + sh[:, 2] * sh[:, 2])
    ax, ay, az = T[:, 2, 1] - T[:, 1, 2], T[:, 0, 2] - T[:, 2, 0], T[:, 1, 0] - T[:, 0, 1]
    rows["angle"] = np.arctan2(0.5 * np.sqrt((ax * ax + ay * ay) + az * az), (((T[:, 0, 0] + T[:, 1, 1]) + T[:, 2, 2]) - 1.0) / 2.0)
    return rows, blocks


def icp_whole(est, gt, R, max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6):
    """point-to-point ICP of the whole cloud as me_icp runs it (T_init = I): the moved cloud moved by every update, the sums
    about the centre of the ground truth's bounding box.  (T, fitness, rmse, n_corr, iterations, converged)"""
    est, gt = np.asarray(est, np.float64), np.asarray(gt, np.float64)
    c = 0.5 * (gt.min(0) + gt.max(0))
    T = np.eye(4)
    moved = est.copy()
    zero = np.zeros(len(est), np.int64)
    it, conv, have_prev, fit, e = 0, 0, False, 0.0, 0.0
    while True:
        nn, d2 = nearest(moved, gt, R)
        kept = (nn >= 0) & (d2 < R * R)
        t = block_terms(moved, gt, nn, d2, R, np.broadcast_to(c, moved.shape))
        b = t[kept].sum(0)
        nc = int(kept.sum())
        f2 = nc / float(len(est))
        e2 = math.sqrt(b[16] / nc) if nc > 0 else 0.0
        if have_prev:
            it += 1
            if abs(fit - f2) < relative_fitness and abs(e - e2) < relative_rmse:
                conv = 1
        fit, e, have_prev = f2, e2, True
        if conv or it >= max_iteration:
            return T, fit, e, nc, it, conv
        upd = api.icp_update(A.ME_ICP_POINT_TO_POINT, b, c)
        T = mat4(upd, T)
        moved = transform(moved, zero, upd[None])


# ---------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------
def rigid(angle_deg, axis, t):
    """4 x 4 rotation by angle_deg about the unit axis, then translation t"""
    a = np.radians(angle_deg)
    k = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    M = np.eye(4)
    M[:3, :3] = np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K
    M[:3, 3] = t
    return M


def apply(M, x, about=None):
    about = np.zeros(3) if about is None else np.asarray(about)
    return (x - about) @ M[:3, :3].T + about + M[:3, 3]


def indoor(n, rooms, seed, sigma=5e-4):
    """an indoor scene lifted into the regions of edge 8 (one room per region) and a rigid motion of about 1 cm and 0.05
    degrees per room about its centre; the moved points that left their room's region (floor and ceiling edges) are
    dropped.  Returns (est, gt, motions {region index: M})"""
    gt = synth.indoor_scene(n, seed, 0.0, rooms=rooms) + np.array([0.0, 0.0, 2.5])
    room = np.floor(gt / 8.0).astype(np.int64)
    rng = np.random.RandomState(seed)
    est = gt + sigma * rng.randn(*gt.shape)
    motions = {}
    for key in np.unique(room, axis=0):
        m = (room == key).all(1)
        M = rigid(0.05 * rng.uniform(0.5, 1.0), rng.randn(3), 0.006 * rng.uniform(-1, 1, 3))
        about = (key + 0.5) * 8.0
        est[m] = apply(M, est[m], about)
        Mabs = np.eye(4)
        Mabs[:3, :3] = M[:3, :3]
        Mabs[:3, 3] = M[:3, 3] + about - M[:3, :3] @ about
        motions[tuple(key)] = Mabs
    stay = (np.floor(est / 8.0).astype(np.int64) == room).all(1)
    assert stay.mean() > 0.99
    return np.ascontiguousarray(est[stay]), gt, motions


def angle_of(R):
    return np.degrees(np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1)))

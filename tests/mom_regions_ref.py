"""A numpy statement of the mutually orthogonal metric per region (me_mom_region*, DESIGN §3.17).

From a cloud's points, the MOM call's per-point v, family (0..2, -1 none) and planar flags, the region list and min_family:
per region floor(x / s) the cloud's points, its planar points, and per family of the whole map n_j, mean_j (sum v / n_j) and
median_j = numpy's quantile(v, 0.5, method="linear"); mom = (median_1 + median_2) + median_3 and the status.  The sums are
taken in the library's order: a segment's members ascending in v, chunks of 1024 members, lane l adding the chunk's members
l, l + 32, ..., a fixed xor shuffle tree, then the chunks added in order.  With that, the statement gives the library's bits.
"""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mom_ref as MR  # noqa: E402

CHUNK = 1024
NO_AXES = ("NO_PLANAR", "NO_SECOND_AXIS")


def region_keys(xyz, s):
    """floor(x / s) per axis, IEEE division (the library's key)"""
    return np.floor(np.asarray(xyz, np.float64).reshape(-1, 3) / np.float64(s)).astype(np.int64)


def region_list(est, gt, s):
    """the occupied regions of est ++ gt (est alone while gt is empty), ascending by (ix, iy, iz): (index (R, 3), the region
    of every est point, the region of every gt point)"""
    ke = region_keys(est, s)
    kg = region_keys(gt, s) if gt is not None and len(gt) else np.zeros((0, 3), np.int64)
    index, inv = np.unique(np.vstack([ke, kg]), axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    return index, inv[:len(ke)], inv[len(ke):]


def lerp_median(sorted_v, off, n):
    """numpy's linear quantile at 0.5 of the n values sorted_v[off:off + n] per segment (NaN where n = 0)"""
    out = np.full(len(n), np.nan)
    has = n > 0
    h = (n[has] - 1).astype(np.float64) * 0.5
    k = np.floor(h)
    g = h - k
    k = k.astype(np.int64)
    lo = sorted_v[off[has] + k]
    hi = sorted_v[off[has] + np.minimum(k + 1, n[has] - 1)]
    diff = hi - lo
    out[has] = np.where(g >= 0.5, hi - diff * (1.0 - g), lo + diff * g)
    return out


def segment_sums(sorted_v, off, n):
    """the library's fold of each segment's members in their sorted order (see the module docstring)"""
    S = len(n)
    nch = -(-n // CHUNK)
    chunk_off = np.concatenate([[0], np.cumsum(nch)])
    total = int(chunk_off[-1])
    sums = np.zeros(S)
    if total == 0:
        return sums
    seg = np.repeat(np.arange(S), n)
    p = np.arange(len(seg)) - off[seg]            # place inside the segment
    chunk = chunk_off[seg] + p // CHUNK
    q = p % CHUNK
    lane, rnd = q % 32, q // 32
    acc = np.zeros((total, 32))
    for t in range(CHUNK // 32):                  # lane l adds its members in order
        m = rnd == t
        acc[chunk[m], lane[m]] += sorted_v[m]
    part = MR._tree(acc)
    for c in range(int(nch.max())):               # the chunks of a segment in order
        m = nch > c
        sums[m] += part[chunk_off[:-1][m] + c]
    return sums


def statement(rid, R, v, family, planar, axes_status, min_family):
    """rid: region of every point (0..R-1); v, family, planar: the MOM call's per-point arrays; axes_status: the whole map's
    status before the family-size test ('OK', 'NO_PLANAR' or 'NO_SECOND_AXIS').  Returns a dict of arrays: n_points,
    n_planar (R,); n (R, 3) int; mean, median (R, 3); mom (R,); status (R,) names"""
    rid = np.asarray(rid, np.int64)
    v = np.asarray(v, np.float64)
    family = np.asarray(family, np.int64)
    planar = np.asarray(planar, bool)
    out = dict(n_points=np.bincount(rid, minlength=R).astype(np.int64),
               n_planar=np.bincount(rid[planar], minlength=R).astype(np.int64))
    if axes_status in NO_AXES:
        out.update(n=np.zeros((R, 3), np.int64), mean=np.full((R, 3), np.nan), median=np.full((R, 3), np.nan),
                   mom=np.full(R, np.nan), status=np.array([axes_status] * R, dtype=object))
        return out
    m = planar & (family >= 0)
    seg = rid[m] * 3 + family[m]
    vm = np.where(v[m] == 0.0, 0.0, v[m])        # -0 sorts and counts as +0
    order = np.lexsort((vm, seg))
    sv = vm[order]
    n = np.bincount(seg, minlength=3 * R).astype(np.int64)
    off = np.concatenate([[0], np.cumsum(n)[:-1]]).astype(np.int64)
    med = lerp_median(sv, off, n)
    sums = segment_sums(sv, off, n)
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = np.where(n > 0, sums / np.maximum(n, 1), np.nan)
    n, mean, med = n.reshape(R, 3), mean.reshape(R, 3), med.reshape(R, 3)
    small = (n < min_family).any(axis=1)
    mom = np.where(small, np.nan, (med[:, 0] + med[:, 1]) + med[:, 2])
    out.update(n=n, mean=mean, median=med, mom=mom,
               status=np.array(["SMALL_FAMILY" if x else "OK" for x in small], dtype=object))
    return out


def loop_statement(rid, R, v, family, planar, axes_status, min_family):
    """the rule region by region with np.quantile and np.mean: the check of statement() (means agree to rounding only)"""
    rows = []
    for r in range(R):
        inr = rid == r
        row = dict(n_points=int(inr.sum()), n_planar=int((inr & planar).sum()))
        if axes_status in NO_AXES:
            row.update(n=[0, 0, 0], mean=[math.nan] * 3, median=[math.nan] * 3, mom=math.nan, status=axes_status)
        else:
            ns, means, meds = [], [], []
            for j in range(3):
                x = v[inr & planar & (family == j)]
                ns.append(len(x))
                means.append(float(np.mean(x)) if len(x) else math.nan)
                meds.append(float(np.quantile(x, 0.5, method="linear")) if len(x) else math.nan)
            status = "SMALL_FAMILY" if min(ns) < min_family else "OK"
            row.update(n=ns, mean=means, median=meds, status=status,
                       mom=(meds[0] + meds[1]) + meds[2] if status == "OK" else math.nan)
        rows.append(row)
    return rows


def from_mom_points(xyz, est, gt, s, v, lambda2, family, rho, axes_status, min_family):
    """the statement for the MOM cloud xyz (est or gt, as listed) from me_get_mom_points' arrays"""
    index, rid_e, rid_g = region_list(est, gt, s)
    rid = rid_e if xyz is est else rid_g
    pl = MR.planar(v, lambda2, rho)
    out = statement(rid, len(index), v, family, pl, axes_status, min_family)
    out["index"] = index
    return out

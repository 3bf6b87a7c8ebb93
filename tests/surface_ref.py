"""numpy statement of the point-to-plane metrics (me_nn_surface*, DESIGN §3.14) from caller-order records.

fold() restates one direction's fold over the records me_get_nn returns; block() lays two folds out as the device block
(ME_SURFACE_BLOCK_SUM SUM values, then ME_SURFACE_BLOCK_MAX MAX values) that me_surface_finalize reads; finalize() restates
me_surface_finalize in me_nn_finalize's operation order.  Every e and c is formed with one numpy operation per step, so each
operation is rounded on its own as on the device."""
import numpy as np

from cloud_map_evaluation_b200 import _abi as A

NN = A.ME_NN_ACCUM_I64 + A.ME_NN_ACCUM_F64
MOM = 22                       # offset of rank_n in a direction's NN section


def sqnorm_eigen(v):
    v = np.asarray(v, np.float64)
    return v[:, 0] * v[:, 0] + (v[:, 1] * v[:, 1] + v[:, 2] * v[:, 2])


def usable(nrm):
    """(usable, squared norm): a normal is usable iff its squared norm is finite and > 0"""
    with np.errstate(invalid="ignore", over="ignore"):
        sq = sqnorm_eigen(nrm)
        return np.isfinite(sq) & (sq > 0.0), sq


def fold(query, ref, q_nrm, r_nrm, idx, d2, tau, R, cutoff_mode, want_full_cd):
    """one direction from the caller-order records (idx, d2) of the query cloud: counts, sums, maxima and the (n, mean, M2)
    of the kept e"""
    idx = np.asarray(idx)
    have = idx >= 0
    with np.errstate(invalid="ignore"):
        keep = have & ((d2 <= R) if cutoff_mode == A.ME_CUTOFF_SQDIST_LE_R else (d2 < R * R))
    qi = np.nonzero(have)[0]
    j = idx[qi].astype(np.int64)
    kept = keep[qi]
    ok_n, sn = usable(r_nrm[j])
    out = {"n_query": int(np.count_nonzero(idx != -2)),
           "n_no_normal": int(np.count_nonzero(kept & ~ok_n)),
           "n_no_normal_nn": int(np.count_nonzero(~ok_n)) if want_full_cd else 0}
    qi, j, kept, sn = qi[ok_n], j[ok_n], kept[ok_n], sn[ok_n]
    n = r_nrm[j]
    d = query[qi] - ref[j]
    dot = (d[:, 0] * n[:, 0] + d[:, 1] * n[:, 1]) + d[:, 2] * n[:, 2]
    len_n = np.sqrt(sn)
    e = np.abs(dot) / len_n
    out["sum_nn_dist"] = float(e.sum()) if want_full_cd else 0.0
    out["max_e_nn"] = float(e.max()) if want_full_cd and e.size else 0.0
    ek = e[kept]
    out["n_corr"] = int(ek.size)
    out["max_e"] = float(ek.max()) if ek.size else 0.0
    out["n_inlier"] = np.array([np.count_nonzero(ek <= t) for t in tau], np.int64)
    out["sum_d"] = np.array([ek[ek <= t].sum() for t in tau])
    out["sum_d2"] = np.array([(ek[ek <= t] * ek[ek <= t]).sum() for t in tau])
    out["mean_all"] = float(ek.mean()) if ek.size else 0.0
    out["m2_all"] = float(((ek - out["mean_all"]) ** 2).sum()) if ek.size else 0.0
    qk, nk, lk = qi[kept], n[kept], len_n[kept]
    ok_m, sm = usable(q_nrm[qk])
    m = q_nrm[qk][ok_m]
    nk, lk, sm = nk[ok_m], lk[ok_m], sm[ok_m]
    dmn = (m[:, 0] * nk[:, 0] + m[:, 1] * nk[:, 1]) + m[:, 2] * nk[:, 2]
    c = np.fmin(1.0, np.abs(dmn) / (np.sqrt(sm) * lk))        # fmin: a NaN ratio counts as 1, as on the device
    out["n_nc"] = int(c.size)
    out["sum_c"] = float(c.sum())
    out["e_kept"] = ek
    return out


def fold_both(est, gt, est_nrm, gt_nrm, records, params):
    """both directions; records = ((idx, d2) est->gt, (idx, d2) gt->est) in caller order; a direction the parameters did not
    evaluate is None"""
    dirs = params.directions or 3
    tau = list(params.tau)
    out = []
    for q, (query, ref, qn, rn) in enumerate(((est, gt, est_nrm, gt_nrm), (gt, est, gt_nrm, est_nrm))):
        if not dirs & (1 << q):
            out.append(None)
            continue
        idx, d2 = records[q]
        out.append(fold(query, ref, qn, rn, idx, d2, tau, params.icp_max_distance, params.cutoff_mode, params.want_full_cd))
    return out


def block(folds):
    """the device block of two folds (None: a direction not evaluated, all zero), this rank's moments in slot 0"""
    s = np.zeros(A.ME_SURFACE_BLOCK_SUM)
    mx = np.zeros(A.ME_SURFACE_BLOCK_MAX)
    for q, f in enumerate(folds):
        if f is None:
            continue
        b = s[q * NN:(q + 1) * NN]
        b[0], b[1], b[2:7] = f["n_query"], f["n_corr"], f["n_inlier"]
        b[9:14], b[14:19] = f["sum_d"], f["sum_d2"]
        n, m, m2 = float(f["n_corr"]), f["mean_all"], f["m2_all"]
        b[19], b[20], b[21] = n * m, m2 + n * m * m, f["sum_nn_dist"]
        b[MOM], b[MOM + A.ME_MAX_WORLD], b[MOM + 2 * A.ME_MAX_WORLD] = n, m, m2
        s[2 * NN + 4 * q:2 * NN + 4 * q + 4] = f["n_no_normal"], f["n_no_normal_nn"], f["n_nc"], f["sum_c"]
        mx[2 * q:2 * q + 2] = f["max_e"], f["max_e_nn"]
    return np.concatenate([s, mx])


def _merged_moments(b):
    """rank slots merged in slot order (Chan et al., as me_nn_finalize)"""
    n, m, m2 = 0.0, 0.0, 0.0
    for r in range(A.ME_MAX_WORLD):
        nb, mb, m2b = b[MOM + r], b[MOM + A.ME_MAX_WORLD + r], b[MOM + 2 * A.ME_MAX_WORLD + r]
        if nb == 0:
            continue
        tot = n + nb
        delta = mb - m
        m += delta * (nb / tot)
        m2 += m2b + delta * delta * (n * (nb / tot))
        n = tot
    return n, m, m2


def finalize(params, blk, n_est, n_gt):
    """me_surface_finalize in me_nn_finalize's operation order: surface_dict's layout"""
    blk = np.asarray(blk, np.float64)
    dirs = params.directions or 3
    out = {}
    with np.errstate(all="ignore"):
        for q, (name, n_src) in enumerate((("est_to_gt", n_est), ("gt_to_est", n_gt))):
            b = blk[q * NN:(q + 1) * NN]
            x = blk[2 * NN + 4 * q:2 * NN + 4 * q + 4]
            mx = blk[A.ME_SURFACE_BLOCK_SUM + 2 * q:A.ME_SURFACE_BLOCK_SUM + 2 * q + 2]
            D = {}
            if dirs & (1 << q):
                nc = b[1]
                n_all, m_all, m2_all = _merged_moments(b)
                moments = n_all == nc
                mean = b[9:14] / nc
                if moments:
                    dm = m_all - mean
                    ss = m2_all + nc * dm * dm
                else:
                    ss = b[20] - 2.0 * mean * b[19] + nc * mean * mean
                D.update(n_source=int(n_src), n_corr=int(b[1]), n_inlier=b[2:7].astype(np.int64), n_ub=0, mean=mean,
                         rmse=np.sqrt(b[14:19] / nc), fitness=b[2:7] * 1.0 / np.float64(int(n_src)), sigma=np.sqrt(ss / nc),
                         sum_nn_dist=b[21])
            else:
                D.update(n_source=0, n_corr=0, n_inlier=np.zeros(5, np.int64), n_ub=0, mean=np.zeros(5), rmse=np.zeros(5),
                         fitness=np.zeros(5), sigma=np.zeros(5), sum_nn_dist=0.0)
            D.update(n_no_normal=int(x[0]), n_no_normal_nn=int(x[1]), n_nc=int(x[2]),
                     normal_consistency=x[3] / x[2] if x[2] else np.nan, max_e=mx[0], max_e_nn=mx[1])
            out[name] = D
        e, g = out["est_to_gt"], out["gt_to_est"]
        out["cd"] = e["rmse"] + g["rmse"]
        out["f1"] = 2 * e["fitness"] * e["rmse"] / (e["fitness"] + e["rmse"])
        inter = e["n_inlier"]
        out["iou"] = inter.astype(np.float64) / (np.int64(n_est) + np.int64(n_gt) - inter).astype(np.float64)
        out["full_cd"] = (e["sum_nn_dist"] / np.float64(n_est) + g["sum_nn_dist"] / np.float64(n_gt)) if params.want_full_cd else 0.0
        out["normal_consistency"] = (e["normal_consistency"] + g["normal_consistency"]) / 2.0
    return out

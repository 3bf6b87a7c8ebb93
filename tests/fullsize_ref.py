"""Exact references applied at full size (C4: 50 M vs 20 M, C5: 200 M vs 200 M, S1: 100 M vs 100 M points), where the
CPU oracle would need hours: the definitions of tests/exact_ref.py, evaluated on every record where that is cheap and on
stratified samples where it is not.  CPU helpers for tests/test_gpu_fullsize_large.py; tests/test_fullsize_reference.py
checks them against exact_ref and brute force on small scenes, and that every check rejects a planted fault.

Tensors may live on any torch device: the whole-cloud work runs where the clouds are (the GPU test keeps 200 M-point
clouds in HBM and copies only crops to the host), and the same code runs on the CPU in the tests of these helpers.

* Windows with a margin guarantee.  The reference cloud is binned into cubic cells of edge m; a query's window is the
  3 x 3 x 3 block of cells around its own, and the crop is the union of the windows.  Inside the crop cKDTree proposes
  candidates, and d2_kd with ties to the smaller caller index decides, as exact_ref does.  A nearest neighbour is proven
  only when its distance is below the query's distance to its window's boundary (less a rounding slack); queries that fail
  go to a chunked brute force over the whole cloud.  Radius neighbourhoods use a window edge of r (1 + 1e-6), so the ball
  lies inside the block, and the strict d2_kd < r^2 test of exact_ref.mme_neighbours.
* Whole-cloud statistics.  kept_pairs and dir_stats of exact_ref restated on tensors; the exact sums of 10^8 doubles are
  formed with integer limbs summed by bincount in fp64 (every partial sum an integer below 2^53, so exact in any order),
  and d^2 exactly through Veltkamp's split.  The results equal exact_ref's bit for bit (test_fullsize_reference.py).
* Voxels.  Counts per key by torch.unique; the sampled voxels' points go to exact_ref.exact_moments / wasserstein2; SCS
  of the device's W table by shifted sums on a dense key grid, checked against exact_ref.scs_exact.
"""
import math
from fractions import Fraction

import mpmath as mp
import numpy as np
import torch

import exact_ref as X

FIRST_LAST = 1 << 16          # the first and the last 2^16 caller indices are always sampled
SLACK = 1e-12                 # relative rounding slack of a window boundary (keys are IEEE floor(x / m))


# ---------------------------------------------------------------------------------------------------------------
# exact arithmetic on tensors
# ---------------------------------------------------------------------------------------------------------------
def exact_sum_t(x):
    """the exact sum of an fp64 tensor, as a Fraction (exact_ref.exact_sum for 10^8 values): x = m 2^e with 53-bit m;
    the 18-bit limbs of |m| are summed per exponent with bincount in fp64, exact since every partial sum is an integer
    below 2^18 n < 2^53"""
    x = x.reshape(-1).to(torch.float64)
    x = x[x != 0]
    n = x.numel()
    if n == 0:
        return Fraction(0)
    assert n < (1 << 35)
    m, e = torch.frexp(x)
    mi = (m * 2.0 ** 53).to(torch.int64)
    e = e.to(torch.int64) - 53
    e0 = int(e.min())
    g = e - e0
    G = int(g.max()) + 1
    sgn, a = mi.sign(), mi.abs()
    tot = 0
    for sh in (0, 18, 36):
        limb = ((a >> sh) & ((1 << 18) - 1)) * sgn
        b = torch.bincount(g, weights=limb.to(torch.float64), minlength=G).cpu().tolist()
        tot += sum(int(v) << (i + sh) for i, v in enumerate(b) if v)
    return Fraction(tot) * Fraction(2) ** e0


def exact_sum_sq_t(d):
    """the exact sum of d^2 over an fp64 tensor (Veltkamp: d = hi + lo with 26-bit halves, so hi^2, 2 hi lo and lo^2 are
    exact doubles)"""
    d = d.reshape(-1).to(torch.float64)
    c = d * 134217729.0
    hi = c - (c - d)
    lo = d - hi
    return exact_sum_t(hi * hi) + exact_sum_t(2.0 * (hi * lo)) + exact_sum_t(lo * lo)


def d2_kd_t(q, p):
    """exact_ref.d2_kd on tensors: ((dx dx) + dy dy) + dz dz, one rounding per operation"""
    d = q - p
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def sqrt_rn(x):
    """the correctly rounded square root of an fp64 tensor (CUDA's sqrt is; torch's vectorised CPU sqrt is not always,
    so the CPU goes through numpy)"""
    return torch.sqrt(x) if x.is_cuda else torch.from_numpy(np.sqrt(x.numpy()))


def sqnorm_eigen_t(d):
    """exact_ref.sqnorm_eigen on tensors: x x + (y y + z z)"""
    return d[:, 0] * d[:, 0] + (d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])


# ---------------------------------------------------------------------------------------------------------------
# nearest neighbours: windows with a margin guarantee, brute force
# ---------------------------------------------------------------------------------------------------------------
def brute_nn_t(q, ref, q_block=32, r_chunk=1 << 21):
    """exact nearest neighbours of the rows of q (m, 3) in ref (n, 3), both tensors on one device: (index int64, d2) as
    numpy, d2_kd with ties to the smaller index"""
    best_d = torch.full((len(q),), float("inf"), dtype=torch.float64, device=q.device)
    best_i = torch.full((len(q),), -1, dtype=torch.int64, device=q.device)
    for a in range(0, len(q), q_block):
        qb = q[a:a + q_block, None, :]
        for b in range(0, len(ref), r_chunk):
            d2 = d2_kd_t(qb, ref[None, b:b + r_chunk, :])
            v, i = d2.min(dim=1)                         # the first minimum: the smaller index on a tie
            upd = v < best_d[a:a + q_block]
            best_d[a:a + q_block] = torch.where(upd, v, best_d[a:a + q_block])
            best_i[a:a + q_block] = torch.where(upd, i + b, best_i[a:a + q_block])
    return best_i.cpu().numpy(), best_d.cpu().numpy()


def _cell_keys(cells, lo, dims):
    c = cells - lo
    return (c[:, 0] * dims[1] + c[:, 1]) * dims[2] + c[:, 2]


def crop(ref, q, m):
    """the points of ref (tensor) in the 3 x 3 x 3 cells of edge m around each query of q (tensor): (points (k, 3) and
    their caller indices (k,), numpy, by increasing index)"""
    cr = torch.floor(div_rn(ref, m)).to(torch.int64)
    cq = torch.floor(div_rn(q, m)).to(torch.int64)
    off = torch.tensor([(i, j, k) for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1)], device=q.device)
    want = (cq[:, None, :] + off[None]).reshape(-1, 3)
    lo = torch.minimum(cr.min(0).values, want.min(0).values)
    dims = (torch.maximum(cr.max(0).values, want.max(0).values) - lo + 1).tolist()
    assert dims[0] * dims[1] * dims[2] < (1 << 62)
    sel = torch.isin(_cell_keys(cr, lo, dims), torch.unique(_cell_keys(want, lo, dims)))
    idx = torch.nonzero(sel).reshape(-1)
    return ref[idx].cpu().numpy(), idx.cpu().numpy()


def window_margin(q, m):
    """distance of each query (numpy (m, 3)) to the boundary of its 3 x 3 x 3 window, less the rounding slack"""
    c = np.floor(q / m)
    bd = np.minimum(q - (c - 1) * m, (c + 2) * m - q).min(1)
    return bd - SLACK * (np.abs(q).max(1) + m)


def window_nn(q, pts, idx, m, k=8):
    """exact NN of the queries q (numpy) inside a crop (pts, caller indices idx by increasing index) built with edge m:
    (index, d2, proven).  cKDTree proposes k candidates; when the k-th is not clearly farther than the best, every point
    within the best distance (plus a relative 1e-6) is examined.  proven = the NN is closer than the window boundary."""
    from scipy.spatial import cKDTree
    n = len(q)
    out_i = np.full(n, -1, np.int64)
    out_d = np.full(n, np.inf)
    if len(pts) == 0:
        return out_i, out_d, np.zeros(n, bool)
    tree = cKDTree(pts)
    k = min(k, len(pts))
    _, cand = tree.query(q, k=k)
    cand = cand.reshape(n, k)
    d2 = d2_kd_t(torch.from_numpy(q)[:, None, :], torch.from_numpy(pts[cand])).numpy()
    gi = idx[cand]
    key = np.argsort(gi, axis=1, kind="stable")
    d2s, gis = np.take_along_axis(d2, key, 1), np.take_along_axis(gi, key, 1)
    j = np.argmin(d2s, axis=1)                                       # first minimum over increasing caller index
    out_d = d2s[np.arange(n), j]
    out_i = gis[np.arange(n), j]
    unsure = (d2.max(1) <= out_d * (1 + 1e-6)) & (k < len(pts))
    for t in np.nonzero(unsure)[0]:
        c = np.asarray(tree.query_ball_point(q[t], math.sqrt(out_d[t]) * (1 + 1e-6) + 1e-300), dtype=np.int64)
        dd = X.d2_kd(q[t], pts[c])
        best = np.lexsort((idx[c], dd))[0]
        out_i[t], out_d[t] = idx[c][best], dd[best]
    proven = np.sqrt(out_d) * (1 + SLACK) < window_margin(q, m)
    return out_i, out_d, proven


def exact_nn_sample(q_cloud, ref, qi, d2_reported, m_min):
    """the exact NN (index, d2) of the queries q_cloud[qi] in ref (tensors on one device), and how many queries needed the
    brute force.  Queries are grouped by a window edge m = a power of two >= m_min just above their reported distance; a
    wrong report only sends a query to the brute force."""
    qi = np.asarray(qi, np.int64)
    q = q_cloud[torch.from_numpy(qi).to(q_cloud.device)]
    qh = q.cpu().numpy()
    rep = np.sqrt(np.nan_to_num(np.asarray(d2_reported, np.float64), nan=0.0, posinf=0.0)) * 1.01 + 1e-9
    ex = np.maximum(np.ceil(np.log2(np.maximum(rep, m_min))), math.log2(m_min)).astype(np.int64)
    out_i = np.full(len(qi), -1, np.int64)
    out_d = np.full(len(qi), np.inf)
    todo = np.zeros(len(qi), bool)
    for e in np.unique(ex):
        sel = np.nonzero(ex == e)[0]
        m = 2.0 ** int(e)
        pts, idx = crop(ref, q[torch.from_numpy(sel).to(q.device)], m)
        if len(pts) > 40_000_000:            # a window this large: the brute force is cheaper
            todo[sel] = True
            continue
        i, d, ok = window_nn(qh[sel], pts, idx, m)
        out_i[sel], out_d[sel], todo[sel] = i, d, ~ok
    t = np.nonzero(todo)[0]
    if len(t):
        out_i[t], out_d[t] = brute_nn_t(q[torch.from_numpy(t).to(q.device)], ref)
    return out_i, out_d, len(t)


def window_knn(q, pts, idx, m, k):
    """the exact k nearest neighbours of the queries q (numpy) inside a crop (pts, caller indices idx by increasing index)
    built with edge m, the query itself included when it lies in the crop: (caller indices (n, k) by (d2_kd, index), d2 of
    the k-th, proven).  cKDTree proposes k candidates; every point within the k-th distance (plus a relative 1e-6) is then
    ranked by d2_kd with ties to the smaller caller index.  proven = the k-th neighbour lies inside the window's boundary,
    so no point outside the crop can displace any of the k."""
    from scipy.spatial import cKDTree
    n = len(q)
    out = np.full((n, k), -1, np.int64)
    dk = np.full(n, np.inf)
    proven = np.zeros(n, bool)
    if len(pts) < k:
        return out, dk, proven
    tree = cKDTree(pts)
    dist, _ = tree.query(q, k=k)
    dist = dist.reshape(n, k)[:, -1]
    for t in range(n):
        c = np.asarray(tree.query_ball_point(q[t], dist[t] * (1 + 1e-6) + 1e-300), dtype=np.int64)
        dd = X.d2_kd(q[t], pts[c])
        order = np.lexsort((idx[c], dd))[:k]
        out[t], dk[t] = idx[c][order], dd[order[-1]]
    proven = np.sqrt(dk) * (1 + SLACK) < window_margin(q, m)
    return out, dk, proven


def brute_knn_t(q, ref, k, r_chunk=1 << 24):
    """exact k nearest neighbours of each row of q (tensor) in ref (tensor, same device) over the whole cloud: caller
    indices (numpy (m, k)) by (d2_kd, index).  The k-th smallest d2 is found by topk, then every point at or below it is
    ranked, so a tie at the k-th place goes to the smaller index."""
    out = np.empty((len(q), k), np.int64)
    for t in range(len(q)):
        d2 = torch.cat([d2_kd_t(q[t:t + 1], ref[b:b + r_chunk]) for b in range(0, len(ref), r_chunk)])
        kth = torch.topk(d2, k, largest=False).values.max()
        cand = torch.nonzero(d2 <= kth).reshape(-1)
        dd = d2[cand].cpu().numpy()
        ci = cand.cpu().numpy()
        out[t] = ci[np.lexsort((ci, dd))[:k]]
    return out


def exact_knn_sample(cloud, qi, k, m0, m_max):
    """the exact k nearest neighbours (query included) of the points cloud[qi] (tensor cloud): (caller indices (n, k), how
    many needed the brute force).  Windows start at edge m0 and double up to m_max for the queries not yet proven; the rest
    go to brute_knn_t."""
    qi = np.asarray(qi, np.int64)
    q = cloud[torch.from_numpy(qi).to(cloud.device)]
    qh = q.cpu().numpy()
    out = np.full((len(qi), k), -1, np.int64)
    todo = np.arange(len(qi))
    m = m0
    while len(todo) and m <= m_max:
        pts, idx = crop(cloud, q[torch.from_numpy(todo).to(q.device)], m)
        if len(pts) > 40_000_000:
            break
        nb, _, ok = window_knn(qh[todo], pts, idx, m, k)
        out[todo[ok]] = nb[ok]
        todo = todo[~ok]
        m *= 2
    if len(todo):
        out[todo] = brute_knn_t(q[torch.from_numpy(todo).to(q.device)], cloud, k)
    return out, len(todo)


def check_normals_sample(cloud, qi, nbs, normals):
    """each sampled normal (numpy (n, 3), rows of qi) against exact_reg.check_normal of its exact k-NN nbs (caller indices,
    query included): returns (checked, sign-checked, worst sin angle over its Davis-Kahan bound)"""
    import exact_reg as XR
    nbs = np.asarray(nbs, np.int64)
    qi = np.asarray(qi, np.int64)
    k = nbs.shape[1]
    sel = torch.from_numpy(np.concatenate([nbs, qi[:, None]], 1).reshape(-1)).to(cloud.device)
    local = cloud[sel].cpu().numpy().reshape(len(qi), k + 1, 3)     # the neighbours, then the query (the moments' origin)
    signed, worst = 0, 0.0
    for t, i in enumerate(qi):
        row = XR.normals_exact(local[t], [k], nbs=[np.arange(k)])[0]
        res = XR.check_normal(row, normals[t])
        assert res["ok"], (int(i), normals[t].tolist(), res["why"])
        signed += bool(res["sign_checked"])
        if row["cov"] is not None and 0 < res["sin_bound"] < math.inf:
            n = np.asarray(normals[t], np.float64)
            worst = max(worst, float(np.linalg.norm(np.cross(n, row["v0"]))) / float(np.linalg.norm(n)) / res["sin_bound"])
    return len(qi), signed, worst


def ball_neighbours(pts_cloud, qi, r):
    """exact_ref.mme_neighbours of the queries pts_cloud[qi] (tensor cloud): per query the caller indices of the points with
    d2_kd < r^2, the query itself removed once, and the neighbour coordinates (numpy)"""
    from scipy.spatial import cKDTree
    qi = np.asarray(qi, np.int64)
    q = pts_cloud[torch.from_numpy(qi).to(pts_cloud.device)]
    m = r * (1 + 1e-6)
    qh = q.cpu().numpy()
    assert np.all(window_margin(qh, m) > r * (1 + 1e-7))
    pts, idx = crop(pts_cloud, q, m)
    tree = cKDTree(pts)
    out = []
    for t, c in enumerate(tree.query_ball_point(qh, r * (1 + 1e-6) + 1e-300)):
        c = np.asarray(sorted(c), dtype=np.int64)
        c = c[X.d2_kd(qh[t], pts[c]) < r * r]
        self_pos = np.nonzero(idx[c] == qi[t])[0]
        assert len(self_pos) == 1
        c = np.delete(c, self_pos[0])
        out.append((idx[c], pts[c]))
    return qh, out


# ---------------------------------------------------------------------------------------------------------------
# stratified query samples
# ---------------------------------------------------------------------------------------------------------------
def strata(pts, d2, n_uniform, seed, h, per=256, n_top=1000, sparse_tile=None):
    """{stratum: caller indices (numpy)} over the cloud pts (tensor) with reported NN d2 (tensor or None):
    uniform, first / last 2^16, faces (the `per` points nearest each bounding-box face), corners (nearest each corner
    in L1), rows / layers (the lowest and highest occupied lattice rows (iy, iz) and z-layers of a lattice of edge h),
    top (the n_top largest reported d2) and, with sparse_tile, sparse (the points of the least populated tiles of that
    edge in x, y)"""
    n = len(pts)
    dev = pts.device
    rs = np.random.RandomState(seed)
    out = {"uniform": np.sort(rs.choice(n, min(n, n_uniform), replace=False)),
           "first": np.arange(min(n, FIRST_LAST)), "last": np.arange(max(0, n - FIRST_LAST), n)}
    k = min(per, n)
    lo, hi = pts.min(0).values, pts.max(0).values
    faces = []
    for a in range(3):
        faces.append(torch.topk(pts[:, a] - lo[a], k, largest=False).indices)
        faces.append(torch.topk(hi[a] - pts[:, a], k, largest=False).indices)
    out["faces"] = torch.unique(torch.cat(faces)).cpu().numpy()
    corners = []
    for c in range(8):
        corner = torch.stack([hi[a] if (c >> a) & 1 else lo[a] for a in range(3)])
        corners.append(torch.topk((pts - corner).abs().sum(1), min(32, n), largest=False).indices)
    out["corners"] = torch.unique(torch.cat(corners)).cpu().numpy()
    cell = torch.floor(div_rn(pts - lo, h)).to(torch.int64)
    iz = cell[:, 2]
    rows = []
    for z in (int(iz.min()), int(iz.max())):
        inz = torch.nonzero(iz == z).reshape(-1)
        rows.append(inz)
        iy = cell[inz, 1]
        for y in (int(iy.min()), int(iy.max())):
            rows.append(inz[iy == y])
    rows = torch.unique(torch.cat(rows)).cpu().numpy()
    out["rows"] = rows if len(rows) <= 8 * per else np.sort(rs.choice(rows, 8 * per, replace=False))
    if d2 is not None:
        out["top"] = torch.topk(d2, min(n_top, n)).indices.cpu().numpy()
    if sparse_tile is not None:
        t = torch.floor(div_rn(pts[:, :2] - lo[:2], sparse_tile)).to(torch.int64)
        key = t[:, 0] * (int(t[:, 1].max()) + 1) + t[:, 1]
        u, inv, cnt = torch.unique(key, return_inverse=True, return_counts=True)
        few = torch.argsort(cnt)[:64]
        sp = torch.nonzero(torch.isin(inv, few)).reshape(-1).cpu().numpy()
        out["sparse"] = sp if len(sp) <= 4 * per else np.sort(rs.choice(sp, 4 * per, replace=False))
    return {k2: np.unique(np.asarray(v, np.int64)) for k2, v in out.items()}


# ---------------------------------------------------------------------------------------------------------------
# whole-cloud NN statistics from the records
# ---------------------------------------------------------------------------------------------------------------
def check_records(query, ref, idx, d2):
    """every record of one direction: the index in range and d2 == d2_kd(q, ref[idx]) bit for bit (tensors; world 1 fills
    every record, so the -1 / NaN sentinel of another rank's range must not appear).  Returns the number of records."""
    n_ref = len(ref)
    bad_i = torch.nonzero((idx < 0) | (idx >= n_ref)).reshape(-1)
    assert bad_i.numel() == 0, f"{bad_i.numel()} indices out of range, first at queries {bad_i[:5].tolist()}"
    chunk = 1 << 25
    for a in range(0, len(query), chunk):
        i = idx[a:a + chunk].to(torch.int64)
        dd = d2_kd_t(query[a:a + chunk], ref[i])
        bad = torch.nonzero(dd != d2[a:a + chunk]).reshape(-1)
        assert bad.numel() == 0, (f"{bad.numel()} records whose d2 is not d2_kd(q, ref[idx]), first at queries "
                                  f"{(bad[:5] + a).tolist()}: {d2[a + bad[:5]].tolist()} vs {dd[bad[:5]].tolist()}")
    return len(query)


def check_sample(name, qi, idx, d2, ex_i, ex_d):
    """the records of the sampled queries qi (numpy) against their exact NN, bit for bit"""
    got_i, got_d = np.asarray(idx)[qi], np.asarray(d2)[qi]
    bad = np.nonzero((got_i != ex_i) | (got_d.view(np.int64) != np.asarray(ex_d, np.float64).view(np.int64)))[0]
    assert len(bad) == 0, (f"{name}: {len(bad)} of {len(qi)} sampled records differ from the exact NN, first "
                           f"{[(int(qi[b]), int(got_i[b]), float(got_d[b]), int(ex_i[b]), float(ex_d[b])) for b in bad[:5]]}")


def kept_pairs_t(query, ref, nn_idx, nn_d2, R, cutoff_mode, as_written=False):
    """exact_ref.kept_pairs on tensors: (sq, d, n_ub)"""
    keep = (nn_idx >= 0) & ((nn_d2 <= R) if cutoff_mode == 0 else (nn_d2 < R * R))
    qi = torch.nonzero(keep).reshape(-1)
    ri = nn_idx[qi].to(torch.int64)
    n_ub = 0
    if as_written:
        ok = (ri < len(query)) & (qi < len(ref))
        n_ub = int((~ok).sum())
        diff = query[ri[ok]] - ref[qi[ok]]
    else:
        diff = query[qi] - ref[ri]
    sq = sqnorm_eigen_t(diff)
    return sq, sqrt_rn(sq), n_ub


def dir_stats_t(sq, d, n_source, tau):
    """exact_ref.dir_stats on tensors, the same exact values"""
    nc = d.numel()
    s_all = exact_sum_t(d)
    q_all = exact_sum_sq_t(d)
    out = dict(n_corr=nc, n_inlier=[], mean=[], rmse=[], fitness=[], sigma=[], mean_all=(s_all / nc if nc else None))
    nan = float("nan")
    for t in tau:
        m = d <= t
        ni = int(m.sum())
        sk, qk = exact_sum_t(d[m]), exact_sum_t(sq[m])
        out["n_inlier"].append(ni)
        out["fitness"].append(X.to_float(Fraction(ni, int(n_source))))
        if nc == 0:
            out["mean"].append(nan); out["rmse"].append(nan); out["sigma"].append(nan)
            continue
        mean_k = sk / nc
        out["mean"].append(X.to_float(mean_k))
        out["rmse"].append(X.to_float(X._sqrt(qk / nc)))
        ss = q_all - 2 * mean_k * s_all + nc * mean_k * mean_k
        out["sigma"].append(X.to_float(X._sqrt(ss / nc)))
    return out


def check_accum(name, acc, ex, n_query, n_ub):
    """the integer counts of an me_nn_accum against the exact statistics"""
    got = [acc.n_query, acc.n_corr] + list(acc.n_inlier) + [acc.n_ub]
    want = [n_query, ex["n_corr"]] + list(ex["n_inlier"]) + [n_ub]
    assert got == want, (name, got, want)


def sweep_offsets(trace, r, maxabs):
    """the fp32 offset error E of the MME sweep that ran (None: fp64 offsets; 'unknown': a shared lattice whose edge the
    trace does not bound)"""
    if "ME_KBIT_MME_GENERIC" in trace:
        return None
    if "ME_KBIT_MME_SOLO" in trace:
        h, rings = 0.5 * r, 2
    else:
        rings = [k for k in (1, 2, 3) if any(f"MME_FLAT{k}_" in t or t.endswith(f"MME_ROWS{k}") for t in trace)]
        if not rings or rings[0] < 2:
            return "unknown"
        h, rings = r / (rings[0] - 1), rings[0]
    return X.mme_offset_error(h, rings, np.full((1, 3), maxabs))


class Meter:
    """device memory in use beyond the start (sampled after each stage) and wall time"""

    def __init__(self):
        import time
        torch.cuda.synchronize()
        free, total = torch.cuda.mem_get_info()
        self.base, self.peak, self.t0 = total - free, 0, time.time()

    def sample(self):
        torch.cuda.synchronize()
        free, total = torch.cuda.mem_get_info()
        self.peak = max(self.peak, total - free - self.base)


# ---------------------------------------------------------------------------------------------------------------
# mean map entropy on a sample
# ---------------------------------------------------------------------------------------------------------------
def mme_sample_exact(q, nbs, min_neighbors):
    """exact_ref.mme_point of each sampled query q[t] with neighbour coordinates nbs[t][1]"""
    res = []
    for t, (_, p) in enumerate(nbs):
        local = np.concatenate([q[t:t + 1], p])
        res.append(X.mme_point(local, 0, np.arange(1, len(local)), min_neighbors))
    return res


def mme_allowance(ex, E):
    """B64, plus B32(E) where B32(E) <= 2 tau (test_gpu_exact_mme.allowance); E = None: an fp64-offset sweep"""
    if not ex["valid"]:
        return 0.0
    b32 = X.mme_fp32_certificate(ex["cov"], ex["k"], E) if E is not None else 0.0
    return ex["b64"] + (b32 if b32 <= 2 * X.TAU_FP64 else 0.0)


def check_mme_sample(qi, ent, exs, E):
    """per sampled query: validity (ent != 0) exact where determined, |ent - e| <= allowance; returns (checked, worst
    error / bound, undetermined)"""
    worst, und = 0.0, 0
    for i, ex in zip(qi, exs):
        got = float(ent[i])
        if not ex["determined"]:
            und += 1
            continue
        assert (got != 0.0) == bool(ex["valid"]), (int(i), got, ex["k"], ex["valid"])
        if ex["valid"]:
            b = mme_allowance(ex, E)
            err = abs(got - ex["e"])
            assert err <= b, (int(i), got, ex["e"], err, b)
            worst = max(worst, err / b)
    return len(qi) - und, worst, und


# ---------------------------------------------------------------------------------------------------------------
# voxels
# ---------------------------------------------------------------------------------------------------------------
def div_rn(x, s):
    """x / s correctly rounded on any device.  torch divides a CUDA tensor by a Python number as a multiplication by its
    reciprocal, x (1 / s), which floors differently from x / s at some quotients next to an integer; a divisor held in a
    tensor on x's device takes the IEEE division"""
    return x / torch.tensor(s, dtype=torch.float64, device=x.device)


def voxel_key_t(pts, v):
    """exact_ref.voxel_keys on a tensor: (n, 3) int64 IEEE floor(x / v)"""
    return torch.floor(div_rn(pts, v)).to(torch.int64)


def pack_keys(k, lo, dims):
    return _cell_keys(k, lo, dims)


def voxel_counts(est, gt, v, min_points):
    """(packing (lo, dims), unique est keys, counts, unique gt keys, counts, packed keys of the pairs) — the voxel maps of
    calculateVMD and its pair filter (map_eval.cpp:270-284)"""
    ke, kg = voxel_key_t(est, v), voxel_key_t(gt, v)
    lo = torch.minimum(ke.min(0).values, kg.min(0).values)
    dims = (torch.maximum(ke.max(0).values, kg.max(0).values) - lo + 1).tolist()
    ue, ce = torch.unique(pack_keys(ke, lo, dims), return_counts=True)
    del ke
    ug, cg = torch.unique(pack_keys(kg, lo, dims), return_counts=True)
    pe, pg = ue[ce >= min_points], ug[cg >= min_points]
    pairs = pe[torch.isin(pe, pg)]
    return (lo, dims), ue, ce, ug, cg, pairs


def unpack_key(p, lo, dims):
    p = int(p)
    z = p % dims[2]
    y = (p // dims[2]) % dims[1]
    x = p // (dims[2] * dims[1])
    return (x + int(lo[0]), y + int(lo[1]), z + int(lo[2]))


def voxel_points(cloud, v, packing, keys):
    """{key tuple: (n, 3) numpy points} of the voxels `keys` (packed, tensor) of a tensor cloud"""
    lo, dims = packing
    pk = pack_keys(voxel_key_t(cloud, v), lo, dims)
    sel = torch.nonzero(torch.isin(pk, keys)).reshape(-1)      # increasing caller index: the summation order is irrelevant
    pts, k = cloud[sel].cpu().numpy(), pk[sel].cpu().numpy()
    out = {}
    for key in np.unique(k):
        out[unpack_key(key, lo, dims)] = pts[k == key]
    return out


def check_voxel_row(r, key, pe, pg, v):
    """one rows27 row against the exact Gaussians of its voxel's points pe, pg (numpy): counts exact, means, stored
    covariances and W^2 within exact_ref's bounds (test_exact_ref.check_voxel_rows)"""
    n_e, mu_e, m2_e = X.exact_moments(pe)
    n_g, mu_g, m2_g = X.exact_moments(pg)
    assert (int(r[10]), int(r[11])) == (n_g, n_e), (key, r[10], r[11], n_g, n_e)
    for mu_ex, got in ((mu_e, r[6:9]), (mu_g, r[18:21])):
        assert np.all(np.abs(got - np.array([float(x) for x in mu_ex])) <= X.mu_bound(got, v)), (key, got)
    st_e, st_g = X.stored_sigma(n_e, m2_e), X.stored_sigma(n_g, m2_g)
    tri = [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]
    for st, got, n in ((st_e, r[12:18], n_e), (st_g, r[21:27], n_g)):
        ex = np.array([float(st[a][b]) for a, b in tri])
        assert np.all(np.abs(got - ex) <= X.sigma_entry_bound(n, v)), (key, got, ex)
    w2, tr = X.wasserstein2(mu_g, st_g, n_g, mu_e, st_e, n_e)
    err, b = abs(r[9] ** 2 - float(w2)), X.w_bound(tr, r[6:9], r[18:21], v)
    assert err <= b, (key, r[9], float(mp.sqrt(w2)), err, b)
    return err / b if b > 0 else 0.0


def row_keys(rows, v):
    return np.floor(rows[:, 0:3] / v + 0.5).astype(np.int64)


def scs_grid(keys, w, radius=5, device="cpu"):
    """per key (rows order) the SCS term sqrt(var) / mean over the other keys of the table within the (2 radius + 1)^3 block,
    NaN where it has none, in fp64 by shifted sums on a dense grid (two passes: mean, then the centred squares)"""
    keys = torch.as_tensor(np.asarray(keys, np.int64), device=device)
    w = torch.as_tensor(np.asarray(w, np.float64), device=device)
    lo = keys.min(0).values
    c = keys - lo + radius
    dims = (c.max(0).values + radius + 1).tolist()
    W = torch.zeros(dims, dtype=torch.float64, device=device)
    P = torch.zeros(dims, dtype=torch.float64, device=device)
    W[c[:, 0], c[:, 1], c[:, 2]] = w
    P[c[:, 0], c[:, 1], c[:, 2]] = 1.0
    offs = [(a, b, g) for a in range(-radius, radius + 1) for b in range(-radius, radius + 1)
            for g in range(-radius, radius + 1) if (a, b, g) != (0, 0, 0)]
    cnt = torch.zeros(len(keys), dtype=torch.float64, device=device)
    s = torch.zeros_like(cnt)
    for a, b, g in offs:
        cnt += P[c[:, 0] + a, c[:, 1] + b, c[:, 2] + g]
        s += W[c[:, 0] + a, c[:, 1] + b, c[:, 2] + g]
    mean = s / cnt
    ss = torch.zeros_like(cnt)
    for a, b, g in offs:
        p = P[c[:, 0] + a, c[:, 1] + b, c[:, 2] + g]
        ss += p * (W[c[:, 0] + a, c[:, 1] + b, c[:, 2] + g] - mean) ** 2
    return (torch.sqrt(ss / cnt) / mean).cpu().numpy(), cnt.cpu().numpy()


def scs_key_exact(w_table, k, radius=5):
    """the SCS term of key k in mpmath (exact_ref.scs_exact's inner step), or None without neighbours"""
    nb = [w_table[(k[0] + dx, k[1] + dy, k[2] + dz)]
          for dx in range(-radius, radius + 1) for dy in range(-radius, radius + 1) for dz in range(-radius, radius + 1)
          if (dx, dy, dz) != (0, 0, 0) and (k[0] + dx, k[1] + dy, k[2] + dz) in w_table]
    if not nb:
        return None
    with mp.workdps(X.DPS):
        nb = [mp.mpf(x) for x in nb]
        mean = sum(nb) / len(nb)
        return mp.sqrt(sum((x - mean) ** 2 for x in nb) / len(nb)) / mean


# ---------------------------------------------------------------------------------------------------------------
# segmented exact sums: one exact sum per region
# ---------------------------------------------------------------------------------------------------------------
def seg_limbs_t(x, seg, n_seg):
    """exact_sum_t per segment: x (fp64 tensor) and seg (int64, 0 <= seg < n_seg) of the same length.  Returns (L, e0) with
    L (3, n_seg, G) fp64: per limb (bits 0-17, 18-35, 36-52 of |mantissa|, signed), segment and exponent g the bincount of
    the limbs, an integer below 2^18 n < 2^53 and so exact in any order.  Segment r's sum is
    sum_{s, g} L[s, r, g] 2^(18 s + g + e0) (seg_fraction), and its double-double is seg_sum_dd."""
    x = x.reshape(-1).to(torch.float64)
    seg = seg.reshape(-1)
    nz = x != 0
    x, seg = x[nz], seg[nz]
    if x.numel() == 0:
        return torch.zeros((3, n_seg, 1), dtype=torch.float64, device=x.device), 0
    assert x.numel() < (1 << 35)
    m, e = torch.frexp(x)
    mi = (m * 2.0 ** 53).to(torch.int64)
    e = e.to(torch.int64) - 53
    e0 = int(e.min())
    g = e - e0
    G = int(g.max()) + 1
    del m, e
    key = seg * G + g
    del g
    sgn, a = mi.sign(), mi.abs()
    L = torch.empty((3, n_seg * G), dtype=torch.float64, device=x.device)
    for s, sh in enumerate((0, 18, 36)):
        limb = ((a >> sh) & ((1 << 18) - 1)) * sgn
        L[s] = torch.bincount(key, weights=limb.to(torch.float64), minlength=n_seg * G)
    return L.reshape(3, n_seg, G), e0


def seg_fraction(L, e0, r):
    """the exact sum of segment r, as a Fraction"""
    rows = L[:, r, :].cpu().tolist()
    tot = 0
    for s, row in enumerate(rows):
        tot += sum(int(v) << (g + 18 * s) for g, v in enumerate(row) if v)
    return Fraction(tot) * Fraction(2) ** e0


def seg_sum_dd(L, e0):
    """per segment a double-double (hi, lo) of the exact sum: the terms L 2^w are exact doubles, added by increasing weight
    w with TwoSum, the rounding errors into lo.  |hi + lo - sum| <= (3 G)^2 u^2 sum |x|, far below any bound it meets."""
    _, n_seg, G = L.shape
    hi = torch.zeros(n_seg, dtype=torch.float64, device=L.device)
    lo = torch.zeros_like(hi)
    for w in sorted(set(g + 18 * s for s in range(3) for g in range(G))):
        for s in range(3):
            g = w - 18 * s
            if not 0 <= g < G:
                continue
            assert -1020 < w + e0 < 1020
            t = L[s, :, g] * math.ldexp(1.0, w + e0)
            tot = hi + t
            bp = tot - hi
            lo += (hi - (tot - bp)) + (t - bp)
            hi = tot
    return hi, lo


def seg_sums(x, seg, n_seg):
    """(exact sum as double-double, sum |x| (double-double's hi), limbs, e0) per segment"""
    L, e0 = seg_limbs_t(x, seg, n_seg)
    hi, lo = seg_sum_dd(L, e0)
    La, ea = seg_limbs_t(x.abs(), seg, n_seg)
    ab, _ = seg_sum_dd(La, ea)
    del La
    return hi, lo, ab, L, e0


def check_seg_sum(name, got, ref, count):
    """got (tensor, per segment) against the exact sums ref = seg_sums(...) within the bound of any summation order,
    (n_r - 1) u sum|x| (the double-double's own error and the rounding of this test are below 1e-12 of it, or 2^-100
    sum|x| where the bound is 0).  Returns the worst error as a fraction of the bound."""
    hi, lo, ab = ref[0], ref[1], ref[2]
    bound = (count.to(torch.float64) - 1).clamp(min=0) * X.U * ab
    err = ((got - hi) - lo).abs()
    tol = bound * (1 + 1e-12) + 2.0 ** -100 * ab
    bad = torch.nonzero(~(err <= tol)).reshape(-1)
    assert bad.numel() == 0, (f"{name}: {bad.numel()} segments beyond (n - 1) u sum|x|, first {bad[:5].tolist()}: got "
                              f"{got[bad[:5]].tolist()}, exact {hi[bad[:5]].tolist()}, bound {bound[bad[:5]].tolist()}")
    pos = bound > 0
    return float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0


# ---------------------------------------------------------------------------------------------------------------
# the region table (me_nn_regions, DESIGN §3.12) from all records
# ---------------------------------------------------------------------------------------------------------------
def region_keys_t(pts, s, recip=False):
    """(n, 3) int64 IEEE floor(x / s); recip: floor(x * (1 / s)), a deliberately wrong variant"""
    return torch.floor(pts * (1.0 / s) if recip else div_rn(pts, s)).to(torch.int64)


def division_is_rounded(x, s, n, seed):
    """n sampled coordinates of x (tensor) and the extremes: div_rn(x, s) on x's device equals the correctly rounded
    quotient (Fraction division rounds correctly).  Returns the number checked."""
    flat = x.reshape(-1)
    rs = np.random.RandomState(seed)
    pick = torch.from_numpy(rs.choice(flat.numel(), min(n, flat.numel()), replace=False)).to(x.device)
    v = torch.cat([flat[pick], flat.min().reshape(1), flat.max().reshape(1)])
    q = div_rn(v, s).cpu().tolist()
    for a, b in zip(v.cpu().tolist(), q):
        assert float(Fraction(a) / Fraction(s)) == b, (a, s, b)
    return len(q)


def region_list_t(est, gt, s, recip=False, chunk=1 << 25):
    """the occupied regions of est ++ gt at edge s: dict(lo, dims, keys (packed, ascending), index (R, 3), n_est, n_gt,
    seg_est, seg_gt (each point's region position)).  The keys are formed in chunks of points; the lowest and highest index
    per axis come from the bounding boxes (floor(x / s) is monotone in x)."""
    def key_of(pts):
        return region_keys_t(pts, s, recip)

    ends = torch.stack([key_of(torch.stack([c.min(0).values, c.max(0).values])) for c in (est, gt)]).reshape(-1, 3)
    lo = ends.min(0).values
    dims = (ends.max(0).values - lo + 1).tolist()
    assert dims[0] * dims[1] * dims[2] < (1 << 62)
    pe, pg = [torch.cat([_cell_keys(key_of(c[a:a + chunk]), lo, dims) for a in range(0, len(c), chunk)])
              for c in (est, gt)]
    keys = torch.unique(torch.cat([torch.unique(pe), torch.unique(pg)]))
    seg_e, seg_g = torch.searchsorted(keys, pe), torch.searchsorted(keys, pg)
    del pe, pg
    R = keys.numel()
    iz = keys % dims[2]
    iy = (keys // dims[2]) % dims[1]
    ix = keys // (dims[2] * dims[1])
    index = torch.stack([ix, iy, iz], 1) + lo
    return dict(lo=lo, dims=dims, keys=keys, index=index, n_est=torch.bincount(seg_e, minlength=R),
                n_gt=torch.bincount(seg_g, minlength=R), seg_est=seg_e, seg_gt=seg_g)


def region_pairs_t(query, ref, idx, d2, R, as_written=False):
    """the kept pairs of one direction with their query's caller index: (qi, sq, d); kept_pairs_t's rule"""
    keep = (idx >= 0) & (d2 <= R)
    qi = torch.nonzero(keep).reshape(-1)
    ri = idx[qi].to(torch.int64)
    if as_written:
        ok = (ri < len(query)) & (qi < len(ref))
        qi, ri = qi[ok], ri[ok]
        diff = query[ri] - ref[qi]
    else:
        diff = query[qi] - ref[ri]
    sq = sqnorm_eigen_t(diff)
    return qi, sq, sqrt_rn(sq)


def region_direction_t(seg, n_seg, idx, d2, qi, sq, d, tau, row=None, pick=None):
    """one direction of the table from all records: exact counts and maxima (bincount, scatter-amax of the same bits) and
    the exact sums per region (seg_sums) of d and sq per level and of sqrt(d2) over the queries with a neighbour.  With row
    (region_dict's direction) each sum is checked against it within the order bound (check_seg_sum; 'worst' is the largest
    error over its bound); the limbs are kept for the regions pick (tensor, default all) as (L, e0) for _ex_dir"""
    sg = seg[qi]
    out = dict(n_query=torch.bincount(seg, minlength=n_seg), n_corr=torch.bincount(sg, minlength=n_seg),
               n_inlier=[], sum_d=[], sum_d2=[], worst=0.0)
    zero = torch.zeros(n_seg, dtype=torch.float64, device=seg.device)
    out["max_d"] = zero.scatter_reduce(0, sg, d, "amax")

    def summed(name, x, s, cnt, k=None):
        ref = seg_sums(x, s, n_seg)
        if row is not None:
            got = row[name] if k is None else row[name][:, k]
            got = torch.from_numpy(np.ascontiguousarray(got)).to(x.device)
            out["worst"] = max(out["worst"], check_seg_sum(f"{name}[{k}]", got, ref, cnt))
        L, e0 = ref[3], ref[4]
        return (L if pick is None else L[:, pick, :].clone()), e0

    for k, t in enumerate(tau):
        m = d <= t
        out["n_inlier"].append(torch.bincount(sg[m], minlength=n_seg))
        out["sum_d"].append(summed("sum_d", d[m], sg[m], out["n_inlier"][k], k))
        out["sum_d2"].append(summed("sum_d2", sq[m], sg[m], out["n_inlier"][k], k))
    have = torch.nonzero(idx >= 0).reshape(-1)
    dn = sqrt_rn(d2[have])
    sh = seg[have]
    out["max_nn"] = zero.scatter_reduce(0, sh, dn, "amax")
    out["n_nn"] = torch.bincount(sh, minlength=n_seg)
    out["sum_nn"] = summed("sum_nn_dist", dn, sh, out["n_nn"])
    return out


def _ex_dir(D, r, pos, n_source, tau):
    """the exact mean / rmse / fitness / n_inlier (exact_ref.dir_stats's values) of region r, whose limbs sit at pos"""
    nc = int(D["n_corr"][r])
    out = dict(n_corr=nc, n_inlier=[], mean=[], rmse=[], fitness=[])
    for k in range(len(tau)):
        ni = int(D["n_inlier"][k][r])
        out["n_inlier"].append(ni)
        out["fitness"].append(X.to_float(Fraction(ni, n_source)) if n_source else float("nan"))
        if nc == 0:
            out["mean"].append(float("nan")); out["rmse"].append(float("nan"))
            continue
        sk = seg_fraction(*D["sum_d"][k], pos)
        qk = seg_fraction(*D["sum_d2"][k], pos)
        out["mean"].append(X.to_float(sk / nc))
        out["rmse"].append(X.to_float(X._sqrt(qk / nc)))
    return out


def _close(got, ex, bound):
    if math.isnan(ex):
        return math.isnan(got)
    return abs(got - ex) <= bound


def check_region_row(rows, i, E, G, tau, pos=None):
    """row i of region_dict against exact_ref's values and bounds from the exact region sums (region_direction_t of both
    directions, limbs of region i at pos): mean, rmse, fitness per direction, cd, f1, iou, and mean_nn = sum_nn / n_query"""
    pos = i if pos is None else pos
    n_e, n_g = int(rows["n_est"][i]), int(rows["n_gt"][i])
    ex_e, ex_g = _ex_dir(E, i, pos, n_e, tau), _ex_dir(G, i, pos, n_g, tau)
    for name, ex, D in (("est_to_gt", ex_e, E), ("gt_to_est", ex_g, G)):
        row = rows[name]
        for f in ("mean", "rmse", "fitness"):
            for k in range(len(tau)):
                got = float(row[f][i][k])
                assert _close(got, ex[f][k], X.rel_bound(ex[f][k])), (i, name, f, k, got, ex[f][k])
        nq = int(D["n_query"][i])
        mn = X.to_float(seg_fraction(*D["sum_nn"], pos) / nq) if nq else float("nan")
        got = float(row["mean_nn"][i])
        assert _close(got, mn, X.rel_bound(mn)), (i, name, "mean_nn", got, mn)
    if n_e and n_g:
        res = X.nn_result(ex_e, ex_g, n_e, n_g)
        for f in ("cd", "f1", "iou"):
            for k in range(len(tau)):
                got = float(rows[f][i][k])
                assert _close(got, res[f][k], X.rel_bound(res[f][k])), (i, f, k, got, res[f][k])


# ---------------------------------------------------------------------------------------------------------------
# point-to-plane metrics (me_nn_surface*, DESIGN §3.14) per pair
# ---------------------------------------------------------------------------------------------------------------
def surface_pairs_t(query, ref, q_nrm, r_nrm, idx, d2, R, chunk=1 << 25, wrong_norm=False):
    """per query, in caller order, one torch operation per kernel operation (every one rounds on its own, as the kernel's
    __d*_rn intrinsics): dict(have (a neighbour), kept, ok_n, ok_m (usable normals), e, c), e NaN without a usable n and c
    NaN without usable n and m.  wrong_norm: e divided by ||n||^2, a deliberately wrong variant"""
    n = len(query)
    dev = query.device
    out = dict(have=torch.zeros(n, dtype=torch.bool, device=dev), kept=torch.zeros(n, dtype=torch.bool, device=dev),
               ok_n=torch.zeros(n, dtype=torch.bool, device=dev), ok_m=torch.zeros(n, dtype=torch.bool, device=dev),
               e=torch.full((n,), float("nan"), dtype=torch.float64, device=dev),
               c=torch.full((n,), float("nan"), dtype=torch.float64, device=dev))
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        j = idx[a:b].to(torch.int64)
        have = j >= 0
        js = j.clamp(min=0)
        nv = r_nrm[js]
        sn = sqnorm_eigen_t(nv)
        ok_n = have & torch.isfinite(sn) & (sn > 0)
        dd = query[a:b] - ref[js]
        dot = (dd[:, 0] * nv[:, 0] + dd[:, 1] * nv[:, 1]) + dd[:, 2] * nv[:, 2]
        ln = sqrt_rn(sn)
        e = dot.abs() / (sn if wrong_norm else ln)
        m = q_nrm[a:b]
        sm = sqnorm_eigen_t(m)
        ok_m = torch.isfinite(sm) & (sm > 0)
        dmn = (m[:, 0] * nv[:, 0] + m[:, 1] * nv[:, 1]) + m[:, 2] * nv[:, 2]
        c = torch.fmin(torch.ones_like(dmn), dmn.abs() / (sqrt_rn(sm) * ln))
        out["have"][a:b] = have
        out["kept"][a:b] = have & (d2[a:b] <= R)
        out["ok_n"][a:b] = ok_n
        out["ok_m"][a:b] = ok_m
        out["e"][a:b] = torch.where(ok_n, e, torch.full_like(e, float("nan")))
        out["c"][a:b] = torch.where(ok_n & ok_m, c, torch.full_like(c, float("nan")))
    return out


def surface_direction_t(P, n_source, tau):
    """one direction's counts and maxima from surface_pairs_t, and exact_ref.dir_stats of the kept e (sq = e * e, rounded,
    as the kernel squares), plus the exact sums of e over every query (full CD) and of c"""
    sel = P["kept"] & P["ok_n"]
    ek = P["e"][sel]
    nn = P["have"] & P["ok_n"]
    nc_sel = sel & P["ok_m"]
    ex = dir_stats_t(ek * ek, ek, n_source, tau)
    ex.update(n_no_normal=int((P["kept"] & ~P["ok_n"]).sum()), n_no_normal_nn=int((P["have"] & ~P["ok_n"]).sum()),
              n_nc=int(nc_sel.sum()), max_e=float(ek.max()) if ek.numel() else 0.0,
              max_e_nn=float(P["e"][nn].max()) if bool(nn.any()) else 0.0,
              sum_nn=exact_sum_t(P["e"][nn]), n_nn=int(nn.sum()), sum_c=exact_sum_t(P["c"][nc_sel]))
    return ex


def check_surface_dir(name, got, ex, tau):
    """surface_dict's direction against surface_direction_t: counts and maxima exact, the statistics within exact_ref's
    bounds, sum_nn_dist within the order bound, the normal consistency within the relative bound"""
    want = [ex["n_corr"]] + list(ex["n_inlier"]) + [ex["n_no_normal"], ex["n_no_normal_nn"], ex["n_nc"]]
    have = [int(got["n_corr"])] + [int(x) for x in got["n_inlier"]] + [int(got["n_no_normal"]), int(got["n_no_normal_nn"]),
                                                                        int(got["n_nc"])]
    assert have == want, (name, have, want)
    assert (float(got["max_e"]), float(got["max_e_nn"])) == (ex["max_e"], ex["max_e_nn"]), (name, got["max_e"], ex["max_e"])
    for f in ("mean", "rmse", "fitness"):
        for k in range(len(tau)):
            assert _close(float(got[f][k]), ex[f][k], X.rel_bound(ex[f][k])), (name, f, k, got[f][k], ex[f][k])
    mean_all = float(ex["mean_all"]) if ex["mean_all"] is not None else 0.0
    for k in range(len(tau)):
        assert _close(float(got["sigma"][k]), ex["sigma"][k], X.sigma_bound(ex["sigma"][k], mean_all)), (name, k)
    s = float(ex["sum_nn"])
    assert abs(float(got["sum_nn_dist"]) - s) <= (ex["n_nn"] + 1) * X.U * abs(s), (name, got["sum_nn_dist"], s)
    nc = X.to_float(ex["sum_c"] / ex["n_nc"]) if ex["n_nc"] else float("nan")
    assert _close(float(got["normal_consistency"]), nc, X.rel_bound(nc)), (name, got["normal_consistency"], nc)
    return nc


def plane_beta(dd, nv):
    """beta per pair: a bound of |e - |d.n| / ||n|||, d the exact difference of the two points, for the kernel's e (numpy
    (k, 3) of the rounded d and n).  d rounds once, then three products, two sums, sqrt(||n||^2) and the division: to first
    order 4 u sum|d_i n_i| + 3.5 u e <= 7.5 u sum|d_i n_i| / ||n||, and 8 u with a relative 1e-10 covers the rest"""
    return 8.0 * X.U * (np.abs(dd) * np.abs(nv)).sum(1) / np.sqrt(X.sqnorm_eigen(nv)) * (1 + 1e-10)


def exact_plane(p, t, n, m=None):
    """e = |(p - t).n| / ||n|| and c = min(1, |m.n| / (||m|| ||n||)) of one pair in mpmath, p, t, n, m fp64 triples"""
    with mp.workdps(X.DPS):
        d = [Fraction(a) - Fraction(b) for a, b in zip(p, t)]
        fn = [Fraction(x) for x in n]
        dot = sum(a * b for a, b in zip(d, fn))
        nn = sum(x * x for x in fn)
        e = abs(X._mp(dot)) / mp.sqrt(X._mp(nn))
        if m is None:
            return float(e), None
        fm = [Fraction(x) for x in m]
        mn = sum(a * b for a, b in zip(fm, fn))
        mm = sum(x * x for x in fm)
        return float(e), float(min(mp.mpf(1), abs(X._mp(mn)) / (mp.sqrt(X._mp(mm)) * mp.sqrt(X._mp(nn)))))


def exact_inlier(p, t, n, tau):
    """e <= tau decided exactly: (d.n)^2 <= tau^2 ||n||^2 in rationals"""
    d = [Fraction(a) - Fraction(b) for a, b in zip(p, t)]
    fn = [Fraction(x) for x in n]
    dot = sum(a * b for a, b in zip(d, fn))
    return dot * dot <= Fraction(tau) ** 2 * sum(x * x for x in fn)


# ---------------------------------------------------------------------------------------------------------------
# local consistency (me_consistency*, DESIGN §3.15) from the per-point values
# ---------------------------------------------------------------------------------------------------------------
def consistency_regions_t(e, v, seg, n_seg):
    """per region of the per-point (entropy, plane variance) of get_consistency_points: exact n_query, n_valid (e != 0),
    n_pv (v finite) and max_pv (scatter-amax of the same bits), and the exact sums of e, v and sqrt(v) (seg_sums)"""
    valid, pv = e != 0, torch.isfinite(v)
    sv, vv = seg[pv], v[pv]
    zero = torch.zeros(n_seg, dtype=torch.float64, device=e.device)
    return dict(n_query=torch.bincount(seg, minlength=n_seg), n_valid=torch.bincount(seg[valid], minlength=n_seg),
                n_pv=torch.bincount(sv, minlength=n_seg), max_pv=zero.scatter_reduce(0, sv, vv, "amax"),
                sum_entropy=seg_sums(e[valid], seg[valid], n_seg)[:3], sum_pv=seg_sums(vv, sv, n_seg)[:3],
                sum_sqrt_pv=seg_sums(sqrt_rn(vv), sv, n_seg)[:3])


def consistency_sample_exact(q, nbs, exs, min_neighbors, divisor_k=False, largest=False):
    """per sampled query with MME's exact covariance (mme_sample_exact's cov, divisor k - 1): (lambda3 or NaN for k < m,
    consistency_ref.fp64_bound).  divisor_k (the covariance divided by k) and largest (the largest eigenvalue) are
    deliberately wrong variants"""
    import consistency_ref as CR
    out = []
    for t, ((_, p), ex) in enumerate(zip(nbs, exs)):
        k = len(p)
        if k < min_neighbors:
            out.append((float("nan"), 0.0))
            continue
        cov = ex["cov"]
        if divisor_k:
            cov = [[c * Fraction(k - 1, k) for c in row] for row in cov]
        with mp.workdps(CR.DPS):
            M = mp.matrix([[X._mp(c) for c in row] for row in cov])
            w = mp.eigsy(M, eigvals_only=True)
            lam = float((max if largest else min)(w[j] for j in range(3)))
        local = np.concatenate([q[t:t + 1], p])
        out.append((max(0.0, lam), CR.fp64_bound(local, 0, np.arange(1, k + 1), cov)))
    return out

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
    cr = torch.floor(ref / m).to(torch.int64)
    cq = torch.floor(q / m).to(torch.int64)
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
    cell = torch.floor((pts - lo) / h).to(torch.int64)
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
        t = torch.floor((pts[:, :2] - lo[:2]) / sparse_tile).to(torch.int64)
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
def voxel_key_t(pts, v):
    """exact_ref.voxel_keys on a tensor: (n, 3) int64 IEEE floor(x / v)"""
    return torch.floor(pts / v).to(torch.int64)


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

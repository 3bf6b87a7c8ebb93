"""tests/fullsize_ref.py on the CPU: its window searches against brute force, its tensor restatements against exact_ref
bit for bit, its stratified sampler stratum by stratum, and every check it offers test_gpu_fullsize_large.py against a
planted fault in otherwise exact records."""
import math
import os
import sys
from fractions import Fraction

import mpmath as mp
import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import exact_ref as X  # noqa: E402
import fullsize_ref as F  # noqa: E402
from test_exact_mme import tilted_plane  # noqa: E402


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def brute(q, ref):
    """exact NN by numpy: d2_kd, ties to the smaller index"""
    out_i, out_d = np.empty(len(q), np.int64), np.empty(len(q))
    for t in range(len(q)):
        d = X.d2_kd(q[t], ref)
        j = int(np.argmin(d))                  # the first minimum
        out_i[t], out_d[t] = j, d[j]
    return out_i, out_d


def box_scene(n_ref=20000, n_q=3000, seed=0):
    rs = np.random.RandomState(seed)
    ref = rs.uniform(-3.0, 5.0, (n_ref, 3))
    q = rs.uniform(-3.5, 5.5, (n_q, 3))
    return q, ref


# ---------------------------------------------------------------------------------------------------------------
# restatements against exact_ref
# ---------------------------------------------------------------------------------------------------------------
def test_exact_sums_equal_exact_ref():
    rs = np.random.RandomState(1)
    x = np.concatenate([rs.uniform(-1, 1, 5000) * 10.0 ** rs.randint(-30, 30, 5000), [0.0, -0.0, 5e-324, 1e300, -1e300],
                        np.full(1000, 0.1)])
    assert F.exact_sum_t(_t(x)) == X.exact_sum(x)
    d = np.abs(x[:5000])
    sq = sum(((X.to_ints(d[i:i + 1])[0][0] * X._pow2(X.to_ints(d[i:i + 1])[1])) ** 2 for i in range(len(d))), 0)
    assert F.exact_sum_sq_t(_t(d)) == sq
    assert F.exact_sum_t(_t(np.zeros(3))) == 0


@pytest.mark.parametrize("as_written", [False, True])
@pytest.mark.parametrize("mode", [0, 1])
def test_kept_pairs_and_dir_stats_equal_exact_ref(mode, as_written):
    q, ref = box_scene(4000, 3000, seed=2)
    i, d2 = brute(q, ref)
    tau = [1.0, 0.3, 0.2, 0.1, 0.05]
    R = 0.09
    sq, d, ub = X.kept_pairs(q, ref, i, d2, R, mode, as_written)
    sq_t, d_t, ub_t = F.kept_pairs_t(_t(q), _t(ref), _t(i), _t(d2), R, mode, as_written)
    np.testing.assert_array_equal(sq_t.numpy(), sq)
    np.testing.assert_array_equal(d_t.numpy(), d)
    assert ub_t == ub and (ub > 0) == as_written
    assert F.dir_stats_t(sq_t, d_t, len(q), tau) == X.dir_stats(sq, d, len(q), tau)


def test_d2_kd_equals_exact_ref():
    q, ref = box_scene(1000, 1000, seed=3)
    np.testing.assert_array_equal(F.d2_kd_t(_t(q), _t(ref)).numpy(), X.d2_kd(q, ref))


# ---------------------------------------------------------------------------------------------------------------
# windows
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("report", ["exact", "zero", "far"])
def test_window_search_equals_brute_force(report):
    """the windows follow the reported distances; a too small report only sends queries to the brute force"""
    q, ref = box_scene()
    bi, bd = brute(q, ref)
    rep = {"exact": bd, "zero": np.zeros_like(bd), "far": bd * 9.0}[report]
    i, d, n_brute = F.exact_nn_sample(_t(q), _t(ref), np.arange(len(q)), rep, 1 / 64)
    np.testing.assert_array_equal(i, bi)
    np.testing.assert_array_equal(d.view(np.int64), bd.view(np.int64))
    assert (n_brute > 100) == (report == "zero"), n_brute


def test_neighbour_just_outside_the_window_takes_the_fallback():
    """a query whose window (the 3 x 3 x 3 cells of edge 1 around its own) holds a point at distance 1.2, while the nearest
    point lies 1.1 away but outside the window: the window's answer is not proven and the brute force finds the nearest"""
    m = 1.0
    q = np.array([[0.05, 0.5, 0.5]])
    inside = np.array([[0.05, 0.5 + 1.2, 0.5]])                # in cell (0, 1, 0): inside the window, d = 1.2
    outside = np.array([[0.05 - 1.1, 0.5, 0.5]])               # in cell (-2, 0, 0): outside, d = 1.1
    ref = np.concatenate([inside, np.random.RandomState(4).uniform(10, 20, (50, 3)), outside])
    pts, idx = F.crop(_t(ref), _t(q), m)
    assert list(idx) == [0]
    wi, wd, proven = F.window_nn(q, pts, idx, m)
    assert wi[0] == 0 and not proven[0]
    i, d, n_brute = F.exact_nn_sample(_t(q), _t(ref), np.array([0]), np.array([0.5]), 1.0)
    assert n_brute == 1 and i[0] == len(ref) - 1 and d[0] == X.d2_kd(q[0], outside[0])


def test_ties_go_to_the_smaller_index():
    """a lattice with every query equidistant from 2, 4 or 8 points, in a shuffled caller order"""
    g = np.arange(-4, 5) * 0.25
    ref = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    ref = ref[np.random.RandomState(5).permutation(len(ref))]
    q = np.concatenate([ref[:40] + [0.125, 0, 0], ref[:40] + [0.125, 0.125, 0], ref[:40] + [0.125, 0.125, 0.125]])
    bi, bd = brute(q, ref)
    i, d, _ = F.exact_nn_sample(_t(q), _t(ref), np.arange(len(q)), bd, 1 / 64)
    np.testing.assert_array_equal(i, bi)
    np.testing.assert_array_equal(d, bd)
    assert (X.d2_kd(q[:, None, :], ref[None]) == bd[:, None]).sum(1).max() == 8


def test_ball_neighbours_equal_mme_neighbours():
    rs = np.random.RandomState(6)
    pts = np.concatenate([rs.uniform(0, 1.0, (3000, 3)), np.repeat(rs.uniform(0, 1.0, (5, 3)), 3, 0)])
    pts[-1] = pts[-2] + [0.125, 0, 0]                          # a pair exactly r apart: not neighbours
    r = 0.125
    nbs = X.mme_neighbours(pts, r)
    qi = np.concatenate([rs.choice(len(pts) - 20, 200, replace=False), np.arange(len(pts) - 20, len(pts))])
    qh, got = F.ball_neighbours(_t(pts), qi, r)
    np.testing.assert_array_equal(qh, pts[qi])
    for t, i in enumerate(qi):
        np.testing.assert_array_equal(got[t][0], nbs[i])
        np.testing.assert_array_equal(got[t][1], pts[nbs[i]])


# ---------------------------------------------------------------------------------------------------------------
# the sampler
# ---------------------------------------------------------------------------------------------------------------
def test_strata_contain_each_stratum():
    rs = np.random.RandomState(7)
    n = 3 * F.FIRST_LAST + 123
    pts = np.column_stack([rs.uniform(0, 400, n), rs.uniform(0, 300, n), rs.uniform(-5, 20, n)])
    pts[:1000, :2] = rs.uniform(0, 40, (1000, 2))               # a denser corner: the sparse tiles lie elsewhere
    d2 = rs.exponential(0.01, n)
    st = F.strata(_t(pts), _t(d2), 500, 8, 1.0, sparse_tile=10.0)
    assert len(st["uniform"]) == 500
    np.testing.assert_array_equal(st["first"], np.arange(F.FIRST_LAST))
    np.testing.assert_array_equal(st["last"], np.arange(n - F.FIRST_LAST, n))
    for a in range(3):
        assert int(np.argmin(pts[:, a])) in st["faces"] and int(np.argmax(pts[:, a])) in st["faces"]
    lo, hi = pts.min(0), pts.max(0)
    for c in range(8):
        corner = np.where([(c >> a) & 1 for a in range(3)], hi, lo)
        assert int(np.argmin(np.abs(pts - corner).sum(1))) in st["corners"]
    iz = np.floor((pts[:, 2] - lo[2]) / 1.0)
    assert set(np.nonzero(iz == iz.max())[0]) <= set(st["rows"]) or len(st["rows"]) == 8 * 256
    assert set(np.nonzero(iz == iz.min())[0]) & set(st["rows"])
    np.testing.assert_array_equal(np.sort(st["top"]), np.sort(np.argsort(-d2)[:1000]))
    t = np.floor((pts[:, :2] - lo[:2]) / 10.0).astype(np.int64)
    key = t[:, 0] * (t[:, 1].max() + 1) + t[:, 1]
    u, cnt = np.unique(key, return_counts=True)
    sparsest = np.nonzero(key == u[np.argmin(cnt)])[0]
    assert set(sparsest) <= set(st["sparse"]) or len(st["sparse"]) == 4 * 256
    assert np.mean(np.isin(st["sparse"], np.arange(1000))) < 0.01


# ---------------------------------------------------------------------------------------------------------------
# planted faults: each check rejects its fault in otherwise exact records
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def records():
    """exact records of 80 000 queries (more than 2^16) against 6 000 points"""
    q, ref = box_scene(6000, F.FIRST_LAST + 14464, seed=9)
    i, d, _ = F.exact_nn_sample(_t(q), _t(ref), np.arange(len(q)), np.zeros(len(q)), 1 / 4)
    return q, ref, i, d


def test_check_records_accepts_exact_records_and_rejects_a_one_ulp_d2(records):
    q, ref, i, d = records
    assert F.check_records(_t(q), _t(ref), _t(i), _t(d)) == len(q)
    bad = d.copy()
    bad[777] = np.nextafter(bad[777], np.inf)
    with pytest.raises(AssertionError, match="not d2_kd"):
        F.check_records(_t(q), _t(ref), _t(i), _t(bad))
    bad_i = i.copy()
    bad_i[5] = len(ref)
    with pytest.raises(AssertionError, match="out of range"):
        F.check_records(_t(q), _t(ref), _t(bad_i), _t(d))


def test_second_nearest_in_the_last_queries_is_caught_by_the_last_stratum(records):
    """the index of one query among the last 2^16 replaced by its second nearest, with that neighbour's d2: every record is
    self-consistent, the uniform stratum misses it and the sample check over all strata catches it"""
    q, ref, i, d = records
    st = F.strata(_t(q), _t(d), 200, 10, 1.0)
    t = next(x for x in range(len(q) - 3, 0, -1) if x not in set(st["uniform"]))
    assert t in st["last"]
    dd = X.d2_kd(q[t], ref)
    second = int(np.lexsort((np.arange(len(ref)), dd))[1])
    bi, bd = i.copy(), d.copy()
    bi[t], bd[t] = second, dd[second]
    F.check_records(_t(q), _t(ref), _t(bi), _t(bd))
    u = st["uniform"]
    F.check_sample("uniform", u, bi, bd, i[u], d[u])
    qi = np.unique(np.concatenate(list(st.values())))
    ex_i, ex_d, _ = F.exact_nn_sample(_t(q), _t(ref), qi, bd[qi], 1 / 4)
    with pytest.raises(AssertionError, match="differ from the exact NN"):
        F.check_sample("all strata", qi, bi, bd, ex_i, ex_d)


def test_inlier_count_off_by_one_is_rejected(records):
    from cloud_map_evaluation_b200 import _abi as A
    q, ref, i, d = records
    tau = [0.3, 0.2, 0.15, 0.1, 0.05]
    sq, dd, ub = F.kept_pairs_t(_t(q), _t(ref), _t(i), _t(d), 1.0, 0)
    ex = F.dir_stats_t(sq, dd, len(q), tau)
    acc = A.me_nn_accum()
    acc.n_query, acc.n_corr, acc.n_ub = len(q), ex["n_corr"], ub
    for k in range(5):
        acc.n_inlier[k] = ex["n_inlier"][k]
    F.check_accum("est_to_gt", acc, ex, len(q), ub)
    acc.n_inlier[2] += 1
    with pytest.raises(AssertionError):
        F.check_accum("est_to_gt", acc, ex, len(q), ub)


def _voxel_row(pe, pg, v):
    """the rows27 row an exact implementation writes for one voxel pair, and the W^2 bound"""
    n_e, mu_e, m2_e = X.exact_moments(pe)
    n_g, mu_g, m2_g = X.exact_moments(pg)
    st_e, st_g = X.stored_sigma(n_e, m2_e), X.stored_sigma(n_g, m2_g)
    w2, tr = X.wasserstein2(mu_g, st_g, n_g, mu_e, st_e, n_e)
    tri = [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]
    r = np.zeros(27)
    key = np.floor(pe[0] / v)
    r[0:3], r[3:6] = key * v, (key + 1) * v
    r[6:9], r[9], r[10], r[11] = [float(x) for x in mu_e], float(mp.sqrt(w2)), n_g, n_e
    r[12:18] = [float(st_e[a][b]) for a, b in tri]
    r[18:21] = [float(x) for x in mu_g]
    r[21:27] = [float(st_g[a][b]) for a, b in tri]
    return r, w2, X.w_bound(tr, r[6:9], r[18:21], v)


def test_voxel_checks_reject_a_count_and_a_w_beyond_the_bound():
    v = 3.0
    rs = np.random.RandomState(11)
    pe = (np.array([4, -2, 1]) + rs.uniform(0.1, 0.9, (300, 3)) * [1, 1, 0.01]) * v
    pg = (np.array([4, -2, 1]) + rs.uniform(0.1, 0.9, (250, 3)) * [1, 1, 0.02]) * v
    r, w2, b = _voxel_row(pe, pg, v)
    key = tuple(int(c) for c in np.floor(pe[0] / v))
    assert F.check_voxel_row(r, key, pe, pg, v) < 1
    bad = r.copy()
    bad[11] += 1
    with pytest.raises(AssertionError):
        F.check_voxel_row(bad, key, pe, pg, v)
    bad = r.copy()
    bad[10] -= 1
    with pytest.raises(AssertionError):
        F.check_voxel_row(bad, key, pe, pg, v)
    for f, ok in ((0.5, True), (1.5, False)):
        moved = r.copy()
        moved[9] = float(mp.sqrt(w2 + f * b))
        if ok:
            F.check_voxel_row(moved, key, pe, pg, v)
        else:
            with pytest.raises(AssertionError):
                F.check_voxel_row(moved, key, pe, pg, v)


def test_entropy_beyond_b64_plus_b32_is_rejected():
    """a tilted plane with 0.1 mm of noise 1.4 km out (B32 of fp32 offsets is well above B64 there): entropies moved by 0.9
    of B64 + B32(E) pass, by 1.1 of it fail; a rejected point reported valid fails"""
    pts = tilted_plane(1e-4, (1400.0, -900.0, 30.0), n=400, seed=12)
    r = 0.1
    qi = np.arange(0, 400, 7)
    qh, nbs = F.ball_neighbours(_t(pts), qi, r)
    exs = F.mme_sample_exact(qh, nbs, 10)
    ex_all = X.mme_exact(pts, r, 10)
    for t, i in enumerate(qi):
        assert exs[t]["valid"] == ex_all["valid"][i] and exs[t]["e"] == ex_all["e"][i]
    E = X.mme_offset_error(r / 2, 2, pts)
    allow = np.array([F.mme_allowance(ex, E) for ex in exs])
    valid = np.array([ex["valid"] and ex["determined"] for ex in exs])
    assert valid.sum() > 20 and np.all(allow[valid] > 10 * np.array([ex["b64"] for ex in exs])[valid])
    ent = np.zeros(len(pts))
    ent[qi] = [ex["e"] for ex in exs]
    F.check_mme_sample(qi, ent, exs, E)
    j = int(np.nonzero(valid)[0][0])
    for f, ok in ((0.9, True), (1.1, False)):
        moved = ent.copy()
        moved[qi[j]] += f * allow[j]
        if ok:
            F.check_mme_sample(qi, moved, exs, E)
        else:
            with pytest.raises(AssertionError):
                F.check_mme_sample(qi, moved, exs, E)
    inval = [t for t, ex in enumerate(exs) if not ex["valid"] and ex["determined"]]
    if inval:
        flipped = ent.copy()
        flipped[qi[inval[0]]] = -3.0
        with pytest.raises(AssertionError):
            F.check_mme_sample(qi, flipped, exs, E)


def test_scs_grid_equals_scs_exact():
    rs = np.random.RandomState(13)
    keys = np.unique(rs.randint(-6, 7, (400, 3)), axis=0)
    keys = np.concatenate([keys, [[40, 40, 40]]])             # an isolated key: no neighbours
    w = rs.uniform(0.01, 2.0, len(keys))
    table = {tuple(int(c) for c in k): x for k, x in zip(keys, w)}
    term, cnt = F.scs_grid(keys, w, 5)
    ex, count = X.scs_exact(table, 5)
    has = cnt > 0
    assert int(has.sum()) == count and not has[-1]
    assert abs(float(X.exact_sum(term[has]) / count) - float(ex)) <= 1e-13 * float(ex)
    for t in range(0, len(keys) - 1, 37):
        assert abs(term[t] - float(F.scs_key_exact(table, tuple(keys[t]), 5))) <= 1e-13 * term[t]
    assert F.scs_key_exact(table, (40, 40, 40), 5) is None and math.isnan(term[-1])


# ---------------------------------------------------------------------------------------------------------------
# segmented sums, the region table, point-to-plane pairs and local consistency
# ---------------------------------------------------------------------------------------------------------------
def test_segmented_sums_equal_exact_ref_per_segment():
    rs = np.random.RandomState(21)
    x = np.concatenate([rs.uniform(-1, 1, 6000) * 10.0 ** rs.randint(-20, 20, 6000), [0.0, 5e-200, -1e200, 1e200]])
    seg = rs.randint(0, 37, len(x))
    seg[-4:] = 36                                              # one segment whose sum cancels to 5e-200
    hi, lo, ab, L, e0 = F.seg_sums(_t(x), _t(seg), 37)
    for r in range(37):
        ex = X.exact_sum(x[seg == r])
        assert F.seg_fraction(L, e0, r) == ex
        assert hi[r].item() == float(ex) or abs(Fraction(hi[r].item()) + Fraction(lo[r].item()) - ex) <= \
            2.0 ** -100 * float(X.exact_sum(np.abs(x[seg == r])))
    got = torch.tensor([float(X.exact_sum(x[seg == r])) for r in range(37)], dtype=torch.float64)
    cnt = torch.bincount(_t(seg), minlength=37)
    assert F.check_seg_sum("exact", got, (hi, lo, ab), cnt) <= 1.0
    # a naive sum of each segment is within the order bound; one ulp beyond the bound is not
    naive = torch.tensor([float(np.sum(x[seg == r])) for r in range(37)], dtype=torch.float64)
    F.check_seg_sum("naive", naive, (hi, lo, ab), cnt)
    bad = got.clone()
    b = (cnt[5] - 1).item() * X.U * ab[5].item()
    bad[5] = float(X.exact_sum(x[seg == 5])) + 2 * b + 1e-300
    with pytest.raises(AssertionError):
        F.check_seg_sum("planted", bad, (hi, lo, ab), cnt)


def _region_scene(seed=22):
    """two clouds with coordinates on the region faces of s = 0.1: fl(k s), where x (1 / s) and x / s can floor apart"""
    rs = np.random.RandomState(seed)
    est = rs.uniform(-1.0, 2.0, (3000, 3))
    gt = rs.uniform(-1.0, 2.0, (2500, 3))
    face = np.arange(-10, 20) * 0.1
    est[:300, 0] = rs.choice(face, 300)
    gt[:300, 1] = rs.choice(face, 300)
    return est, gt, 0.1


def test_region_table_restatement_equals_a_loop_over_regions():
    """region_list_t and region_direction_t against per-region exact_ref.dir_stats, and check_region_row accepts rows built
    from those exact values; the reciprocal key moves points on the face scene, and a pair filed under its reference
    point's region changes n_corr"""
    est, gt, s = _region_scene()
    ie, de = brute(est, gt)
    tau = [0.3, 0.2, 0.1, 0.05, 0.02]
    Rc = 0.04
    L = F.region_list_t(_t(est), _t(gt), s)
    keys_e = X.voxel_keys(est, s)
    keys_g = X.voxel_keys(gt, s)
    occ = sorted(set(map(tuple, keys_e)) | set(map(tuple, keys_g)))
    np.testing.assert_array_equal(L["index"].numpy(), np.array(occ))
    n = len(occ)
    qi, sq, d = F.region_pairs_t(_t(est), _t(gt), _t(ie), _t(de), Rc)
    T = F.region_direction_t(L["seg_est"], n, _t(ie), _t(de), qi, sq, d, tau)
    sq_x, d_x, _ = X.kept_pairs(est, gt, ie, de, Rc, 0)
    kept = np.nonzero(de <= Rc)[0]
    pos = {k: i for i, k in enumerate(occ)}
    for r, key in enumerate(occ):
        mine = np.array([pos[tuple(keys_e[q])] == r for q in kept], bool)
        n_src = int((np.array([pos[tuple(k)] for k in keys_e]) == r).sum())
        ex = X.dir_stats(sq_x[mine], d_x[mine], max(n_src, 1), tau)
        assert int(T["n_corr"][r]) == ex["n_corr"]
        assert [int(T["n_inlier"][k][r]) for k in range(5)] == ex["n_inlier"]
        if n_src:
            got = F._ex_dir(T, r, r, n_src, tau)
            for f in ("mean", "rmse", "fitness"):
                np.testing.assert_array_equal(got[f], ex[f])
        for k in range(5):
            assert F.seg_fraction(*T["sum_d"][k], r) == X.exact_sum(d_x[mine][d_x[mine] <= tau[k]])
    W = F.region_list_t(_t(est), _t(gt), s, recip=True)
    assert int((W["keys"][W["seg_est"]] != L["keys"][L["seg_est"]]).sum()) > 0
    wrong = torch.bincount(L["seg_gt"][_t(ie)[qi]], minlength=n)
    assert not torch.equal(wrong, T["n_corr"])


def test_division_check_accepts_ieee_division():
    est, _, s = _region_scene()
    assert F.division_is_rounded(_t(est), s, 2000, 1) == 2002


def test_surface_pairs_equal_surface_ref():
    """e, c and the counts of surface_pairs_t equal surface_ref.fold bit for bit, with scaled, zero and NaN normals; e
    divided by ||n||^2 differs on non-unit normals"""
    import surface_ref as S
    rs = np.random.RandomState(23)
    est, gt = rs.uniform(0, 1, (2000, 3)), rs.uniform(0, 1, (1800, 3))
    ne, ng = rs.normal(size=(2000, 3)) * rs.uniform(0.5, 3, (2000, 1)), rs.normal(size=(1800, 3))
    ng[:20] = 0.0
    ng[20:25] = np.nan
    ne[:30] = 0.0
    ie, de = brute(est, gt)
    tau = [0.1, 0.05, 0.03, 0.02, 0.01]
    Rc = 0.003
    P = F.surface_pairs_t(_t(est), _t(gt), _t(ne), _t(ng), _t(ie), _t(de), Rc)
    ref = S.fold(est, gt, ne, ng, ie, de, tau, Rc, 0, 1)          # cut-off mode 0: d2 <= R
    ex = F.surface_direction_t(P, len(est), tau)
    assert (ex["n_corr"], ex["n_no_normal"], ex["n_no_normal_nn"], ex["n_nc"]) == \
        (ref["n_corr"], ref["n_no_normal"], ref["n_no_normal_nn"], ref["n_nc"])
    assert list(ex["n_inlier"]) == list(ref["n_inlier"])
    ek = P["e"][P["kept"] & P["ok_n"]].numpy()
    np.testing.assert_array_equal(ek, ref["e_kept"])
    assert ex["max_e"] == ref["max_e"] and ex["max_e_nn"] == ref["max_e_nn"]
    assert X.exact_sum(P["c"][P["kept"] & P["ok_n"] & P["ok_m"]].numpy()) == ex["sum_c"]
    Pw = F.surface_pairs_t(_t(est), _t(gt), _t(ne), _t(ng), _t(ie), _t(de), Rc, wrong_norm=True)
    assert not torch.equal(Pw["e"][Pw["kept"] & Pw["ok_n"]], P["e"][P["kept"] & P["ok_n"]])
    # against the definition: e within beta of mpmath
    sel = np.nonzero((P["have"] & P["ok_n"]).numpy())[0][:200]
    dd = est[sel] - gt[ie[sel]]
    beta = F.plane_beta(dd, ng[ie[sel]])
    for t, q in enumerate(sel):
        e_ex, c_ex = F.exact_plane(est[q], gt[ie[q]], ng[ie[q]], ne[q] if bool(P["ok_m"][q]) else None)
        assert abs(float(P["e"][q]) - e_ex) <= beta[t]
        assert F.exact_inlier(est[q], gt[ie[q]], ng[ie[q]], e_ex * (1 + 1e-9))
        assert not F.exact_inlier(est[q], gt[ie[q]], ng[ie[q]], e_ex * (1 - 1e-9))



def test_consistency_sample_equals_consistency_ref():
    """consistency_sample_exact's lambda3 and bound equal consistency_ref's on a sample of a tilted plane, and the
    covariance divided by k and the largest eigenvalue lie beyond the bound of the exact lambda3"""
    import consistency_ref as CR
    pts = tilted_plane(1e-3, np.zeros(3), 3000, 5)
    r = 0.12
    qi = np.arange(0, 3000, 97)
    qh, nbs = F.ball_neighbours(_t(pts), qi, r)
    exs = F.mme_sample_exact(qh, nbs, 10)
    got = F.consistency_sample_exact(qh, nbs, exs, 10)
    ref = CR.exact_points(pts, r, 10, qi)
    wk = F.consistency_sample_exact(qh, nbs, exs, 10, divisor_k=True)
    wm = F.consistency_sample_exact(qh, nbs, exs, 10, largest=True)
    bites = 0
    for t in range(len(qi)):
        if math.isnan(ref["lam"][t]):
            assert math.isnan(got[t][0])
            continue
        assert got[t][0] == ref["lam"][t] and got[t][1] == ref["bound"][t]
        bites += abs(wk[t][0] - got[t][0]) > got[t][1] and abs(wm[t][0] - got[t][0]) > got[t][1]
    assert bites > 0.9 * len(qi)


# ---------------------------------------------------------------------------------------------------------------
# the exact k nearest neighbours and the normal check
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m0", [1 / 64, 1 / 4])
def test_knn_windows_equal_brute_force(m0):
    """exact_knn_sample against exact_reg.knn_exact (k = 20, query included) on a box and on a shuffled lattice whose
    20th neighbour falls inside a tie group; a too small first window doubles, and a too small largest window takes the
    brute force"""
    import exact_reg as XR
    rs = np.random.RandomState(24)
    box = rs.uniform(0, 2.0, (6000, 3))
    g = np.arange(-5, 6) * 0.125
    lat = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    lat = lat[rs.permutation(len(lat))]
    for pts in (box, lat):
        qi = np.sort(rs.choice(len(pts), 300, replace=False))
        want = np.array(XR.knn_exact(pts, qi, 20))
        got, n_brute = F.exact_knn_sample(_t(pts), qi, 20, m0, 1.0)
        np.testing.assert_array_equal(got, want)
        got, n_brute = F.exact_knn_sample(_t(pts), qi, 20, 1 / 256, 1 / 128)
        np.testing.assert_array_equal(got, want)
        assert n_brute == len(qi)
    # a tie at the 20th place: the lattice's central queries have 6 + 12 + 8 neighbours within sqrt(3) spacings
    d = np.sort(X.d2_kd(lat[want[0][0]], lat))
    assert d[19] == d[20] or d[19] == d[18]


def test_knn_window_needs_the_kth_neighbour_inside():
    """the window (3 x 3 x 3 cells of edge 1, 1.5 from the query at its nearest face) holds a 21st neighbour at 1.598, but
    the true 21st lies 1.55 away outside it: not proven, and the fallback finds it"""
    import exact_reg as XR
    m = 1.0
    q = np.array([[0.5, 0.5, 0.5]])
    near = q + np.random.RandomState(25).uniform(-0.05, 0.05, (19, 3))
    inside = np.array([[0.5 + 1.13, 0.5 + 1.13, 0.5]])         # cell (1, 1, 0): in the window, d = 1.598
    outside = np.array([[0.5 + 1.55, 0.5, 0.5]])               # cell (2, 0, 0): outside it, d = 1.55
    ref = np.concatenate([q, near, inside, outside])
    pts, idx = F.crop(_t(ref), _t(q), m)
    assert list(idx) == list(range(21))
    nb, dk, proven = F.window_knn(q, pts, idx, m, 21)
    assert nb[0][-1] == 20 and not proven[0]
    got, n_brute = F.exact_knn_sample(_t(ref), [0], 21, 1.0, 1.0)
    assert n_brute == 1 and got[0][-1] == 21
    np.testing.assert_array_equal(got[0], XR.knn_exact(ref, [0], 21)[0])


def test_normal_check_accepts_fast_eigen_and_rejects_a_tilted_normal():
    """check_normals_sample on a 1 mm-noise tilted plane: FastEigen3x3's normal of the rounded covariance passes, the same
    normal tilted by 1e-3 rad does not"""
    import exact_reg as XR
    pts = tilted_plane(1e-3, np.zeros(3), 4000, 26)
    qi = np.arange(0, 4000, 40)
    nbs, _ = F.exact_knn_sample(_t(pts), qi, 20, 1 / 16, 1.0)
    rows = XR.normals_exact(pts, qi, nbs=list(nbs))
    good = np.array([r["stmt"] for r in rows])
    checked, signed, worst = F.check_normals_sample(_t(pts), qi, nbs, good)
    assert checked == len(qi) and signed > 0 and worst <= 1.0
    c, s_ = math.cos(1e-3), math.sin(1e-3)
    bad = good @ np.array([[c, -s_, 0], [s_, c, 0], [0, 0, 1]]).T
    with pytest.raises(AssertionError):
        F.check_normals_sample(_t(pts), qi, nbs, bad)

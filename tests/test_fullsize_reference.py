"""tests/fullsize_ref.py on the CPU: its window searches against brute force, its tensor restatements against exact_ref
bit for bit, its stratified sampler stratum by stratum, and every check it offers test_gpu_fullsize_large.py against a
planted fault in otherwise exact records."""
import math
import os
import sys

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

"""tests/exact_ref.py against plain-Python statements of the same definitions on tiny cases, and the oracle against
exact_ref on the scenes the GPU tests use (the bounds of exact_ref hold for an fp64 two-pass implementation, and fail for
the closed-form sigma the library used to compute)."""
import math
import os
import sys
from fractions import Fraction

import mpmath as mp
import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import exact_ref as X  # noqa: E402


@pytest.fixture(scope="module")
def O():
    from oracle import oracle as _O
    _O.build()
    return _O


def offset_scene(n_side=24, h=0.1, offset=(0.013, -0.021, 0.008), jitter=0.0, origin=0.0, seed=0):
    """ground truth on a cubic lattice of spacing h, est = gt + a constant offset (below h / 2 per axis) plus a jitter of
    `jitter` times |offset| per coordinate: every distance is |offset| up to the jitter and the rounding of the sums"""
    g = np.arange(n_side) * h
    gt = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) + origin
    off = np.asarray(offset)
    rng = np.random.RandomState(seed)
    est = gt + off + jitter * np.linalg.norm(off) * rng.uniform(-1, 1, gt.shape)
    return np.ascontiguousarray(est), np.ascontiguousarray(gt)


# ---------------------------------------------------------------------------------------------------------------
# exact_ref against plain statements
# ---------------------------------------------------------------------------------------------------------------
def test_dir_stats_against_plain_fractions():
    rng = np.random.RandomState(1)
    diff = rng.uniform(-0.2, 0.2, (37, 3))
    sq = diff[:, 0] * diff[:, 0] + (diff[:, 1] * diff[:, 1] + diff[:, 2] * diff[:, 2])
    d = np.sqrt(sq)
    tau = [0.3, 0.2, float(np.median(d)), 0.05, 0.0]
    got = X.dir_stats(sq, d, 50, tau)
    F = [Fraction(x) for x in d]
    for k, t in enumerate(tau):
        ins = [i for i in range(len(d)) if d[i] <= t]
        mean = sum((F[i] for i in ins), Fraction(0)) / len(d)
        ss = sum(((f - mean) ** 2 for f in F), Fraction(0)) / len(d)
        rm = sum((Fraction(sq[i]) for i in ins), Fraction(0)) / len(d)
        assert got["n_inlier"][k] == len(ins)
        assert got["mean"][k] == float(mean)
        assert got["fitness"][k] == len(ins) / 50
        assert got["sigma"][k] == float(mp.sqrt(mp.mpf(ss.numerator) / ss.denominator)) or \
            abs(got["sigma"][k] - math.sqrt(ss)) <= 2 * X.U * math.sqrt(ss)
        assert abs(got["rmse"][k] - math.sqrt(rm)) <= 2 * X.U * math.sqrt(rm)
    assert got["n_inlier"][4] == 0 and got["mean"][4] == 0.0 and got["sigma"][4] > 0
    empty = X.dir_stats(np.zeros(0), np.zeros(0), 10, tau)      # no kept pair: 0/0 -> NaN as the reference
    assert all(np.isnan(empty["mean"])) and all(np.isnan(empty["sigma"])) and empty["fitness"] == [0.0] * 5


def test_equal_distances_have_zero_sigma_exactly():
    d = np.full(1000, 0.0259)
    r = X.dir_stats(d * d, d, 1000, [1.0] * 5)
    assert r["sigma"] == [0.0] * 5 and r["mean"] == [0.0259] * 5


def test_voxel_moments_against_plain_fractions():
    rng = np.random.RandomState(2)
    pts = rng.uniform(-1500.3, -1497.6, (13, 3))
    n, mu, m2 = X.exact_moments(pts)
    P = [[Fraction(x) for x in p] for p in pts]
    mu_p = [sum(p[a] for p in P) / n for a in range(3)]
    assert n == 13 and mu == mu_p
    for a in range(3):
        for b in range(3):
            assert m2[a][b] == sum((p[a] - mu_p[a]) * (p[b] - mu_p[b]) for p in P)
    st = X.stored_sigma(n, m2)
    assert st[0][1] == m2[0][1] / 144 and X.stored_sigma(10, m2)[2][2] == m2[2][2]


def test_wasserstein_of_axis_aligned_gaussians_in_closed_form():
    """diagonal covariances: the Cholesky factors are square roots, so W^2 = |dmu|^2 + sum(a + b - 2 sqrt(a b)) with the
    eigenvalues clamped at 1e-6; n <= 1 gives the identity"""
    mu_g, mu_e = [1.0, 2.0, 3.0], [1.25, 2.0, 2.5]
    a, b = [4e-7, 2.0, 0.5], [3.0, 1e-9, 0.5]
    for n_g, n_e in ((2, 2), (11, 40), (1, 5)):
        sg = [[Fraction(a[i]) * (n_g - 1) if i == j else Fraction(0) for j in range(3)] for i in range(3)]
        se = [[Fraction(b[i]) * (n_e - 1) if i == j else Fraction(0) for j in range(3)] for i in range(3)]
        w2, tr = X.wasserstein2(mu_g, sg, n_g, mu_e, se, n_e)
        ca = [1.0] * 3 if n_g <= 1 else [max(x, X.CLAMP) for x in a]
        cb = [max(x, X.CLAMP) for x in b]
        with mp.workdps(40):
            exp = sum((mp.mpf(p) - q) ** 2 for p, q in zip(mu_g, mu_e)) + \
                sum(mp.mpf(p) + q - 2 * mp.sqrt(mp.mpf(p) * q) for p, q in zip(ca, cb))
            assert abs(w2 - exp) < mp.mpf(10) ** -35
            assert tr >= sum(mp.mpf(x) for x in ca + cb)


def test_wasserstein_of_a_gaussian_with_itself_is_not_zero():
    """the Cholesky-trace quirk: tr(chol(L S L^T)) is not tr(S) for a non-diagonal S, so W(G, G) > 0"""
    S = [[Fraction(2), Fraction(1), Fraction(0)], [Fraction(1), Fraction(2), Fraction(0)], [Fraction(0), Fraction(0), Fraction(1)]]
    w2, _ = X.wasserstein2([0, 0, 0], S, 2, [0, 0, 0], S, 2)
    assert w2 > mp.mpf("1e-3")


# ---------------------------------------------------------------------------------------------------------------
# the oracle against exact_ref
# ---------------------------------------------------------------------------------------------------------------
def _nn_case(O, est, gt, tau, R, mode, pairing):
    from cloud_map_evaluation_b200 import _abi as A
    p = A.make_nn_params(tau, R, cutoff_mode=mode, pairing=pairing)
    got = O.eval_nn(est, gt, p)
    ie, de = O.knn1(est, gt)
    ig, dg = O.knn1(gt, est)
    e = X.dir_stats(*X.kept_pairs(est, gt, ie, de, R, mode)[:2], len(est), tau)
    g = X.dir_stats(*X.kept_pairs(gt, est, ig, dg, R, mode, as_written=pairing == A.ME_PAIRING_AS_WRITTEN)[:2], len(gt), tau)
    res = X.nn_result(e, g, len(est), len(gt), np.sqrt(de), np.sqrt(dg))
    return got, e, g, res


def check_nn(got, e, g, res):
    """got: an me_nn_result (library or oracle) against the exact statistics; returns the worst sigma error / bound"""
    worst = 0.0
    for name, ex in (("est_to_gt", e), ("gt_to_est", g)):
        dr = getattr(got, name)
        assert list(dr.n_inlier) == ex["n_inlier"] and dr.n_corr == ex["n_corr"], name
        mean_all = float(ex["mean_all"]) if ex["mean_all"] is not None else 0.0
        for k in range(5):
            for f in ("mean", "rmse", "fitness"):
                x, xe = getattr(dr, f)[k], ex[f][k]
                if np.isnan(xe):
                    assert np.isnan(x), (name, f, k)
                else:
                    assert abs(x - xe) <= X.rel_bound(xe), (name, f, k, x, xe)
            s, se = dr.sigma[k], ex["sigma"][k]
            if np.isnan(se):
                assert np.isnan(s)
                continue
            err, bnd = abs(s - se), X.sigma_bound(se, mean_all)
            worst = max(worst, err / bnd)
            assert err <= bnd, (name, "sigma", k, s, se, err, bnd)
    for f in ("cd", "f1", "iou"):
        for k in range(5):
            x, xe = getattr(got, f)[k], res[f][k]
            assert (np.isnan(x) and np.isnan(xe)) or abs(x - xe) <= X.rel_bound(xe), (f, k, x, xe)
    assert abs(got.full_cd - res["full_cd"]) <= X.rel_bound(res["full_cd"])
    return worst


@pytest.mark.parametrize("jitter", [0.0, 1e-9, 1e-7, 1e-5, 1e-3])
@pytest.mark.parametrize("origin", [0.0, 1500.0])
def test_oracle_nn_statistics_against_exact(O, jitter, origin):
    from cloud_map_evaluation_b200 import _abi as A
    est, gt = offset_scene(n_side=16, jitter=jitter, origin=origin)
    d = np.sqrt(X.sqnorm_eigen(est - gt))
    # a threshold inside the cluster (mean_k != mean_all), one below it (n_inlier = 0), the rest above
    tau = [1.0, 0.1, float(np.median(d)), float(d.min()) * 0.999, 0.05]
    for mode, pairing in ((0, A.ME_PAIRING_AS_WRITTEN), (1, A.ME_PAIRING_GEOMETRIC)):
        got, e, g, res = _nn_case(O, est, gt, tau, 0.5, mode, pairing)
        assert e["n_inlier"][3] == 0 and e["n_corr"] == len(est)
        check_nn(got, e, g, res)


def test_oracle_nn_statistics_on_a_synthetic_scene(O):
    from cloud_map_evaluation_b200 import _abi as A, synth
    est, gt, cfg = synth.make_pair("C1", scale=0.05)
    for mode, pairing in ((0, A.ME_PAIRING_AS_WRITTEN), (1, A.ME_PAIRING_GEOMETRIC)):
        check_nn(*_nn_case(O, est, gt, cfg["tau"], 1.0, mode, pairing))


@pytest.mark.parametrize("jitter", [1e-9, 1e-7])
def test_the_sigma_bound_rejects_the_closed_form(jitter):
    """sum(d^2) - 2 mean sum(d) + n mean^2 on the offset scene: the cancellation the bound is there to catch"""
    est, gt = offset_scene(n_side=24, jitter=jitter, origin=1500.0)
    sq = X.sqnorm_eigen(est - gt)
    d = np.sqrt(sq)
    ex = X.dir_stats(sq, d, len(d), [1.0] * 5)
    n, mean = len(d), d.sum() / len(d)
    ss = (d * d).sum() - 2.0 * mean * d.sum() + n * mean * mean
    closed = math.sqrt(max(ss, 0.0) / n)
    assert abs(closed - ex["sigma"][0]) > X.sigma_bound(ex["sigma"][0], float(ex["mean_all"]))


def surface(n, extent, v, z0=0.0, seed=0, origin=(0.0, 0.0, 0.0)):
    """a wavy surface with 5 cm of noise across extent x extent metres"""
    rng = np.random.RandomState(seed)
    xy = rng.uniform(0, extent, (n, 2))
    z = z0 + 0.3 * np.sin(xy[:, 0] * 0.7) * np.cos(xy[:, 1] * 0.5) + rng.normal(0, 0.05, n)
    return np.ascontiguousarray(np.column_stack([xy, z]) + np.asarray(origin))


def _sym(t):
    s = np.empty(9)
    s[[0, 1, 2, 4, 5, 8]] = t
    s[3], s[6], s[7] = t[1], t[2], t[4]
    return s


def check_voxel_rows(rows, pairs, v, sample):
    """rows27 of calculateVMD (library or oracle) against the exact voxel Gaussians and W; returns (checked rows, rows with
    an eigenvalue above the clamp)"""
    keys = np.floor(rows[:, 0:3] / v + 0.5).astype(np.int64)
    assert len(rows) == len(pairs)
    above = 0
    for i in sample:
        key = tuple(int(c) for c in keys[i])
        n_e, mu_e, m2_e, n_g, mu_g, m2_g = pairs[key]
        r = rows[i]
        assert (int(r[10]), int(r[11])) == (n_g, n_e)
        for mu_ex, got in ((mu_e, r[6:9]), (mu_g, r[18:21])):
            assert np.all(np.abs(got - np.array([float(x) for x in mu_ex])) <= X.mu_bound(got, v)), (key, got)
        st_e, st_g = X.stored_sigma(n_e, m2_e), X.stored_sigma(n_g, m2_g)
        tri = [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]
        for st, got, n in ((st_e, r[12:18], n_e), (st_g, r[21:27], n_g)):
            ex = np.array([float(st[a][b]) for a, b in tri])
            assert np.all(np.abs(got - ex) <= X.sigma_entry_bound(n, v)), (key, got, ex)
        w2, tr = X.wasserstein2(mu_g, st_g, n_g, mu_e, st_e, n_e)
        assert abs(r[9] ** 2 - float(w2)) <= X.w_bound(tr, r[6:9], r[18:21], v), (key, r[9], float(mp.sqrt(w2)))
        if n_e <= 1:
            continue
        with mp.workdps(30):
            S = mp.matrix(3, 3)
            for a in range(3):
                for b in range(3):
                    S[a, b] = X._mp(st_e[a][b]) / (n_e - 1)
            above += max(mp.eigsy(S)[0]) > X.CLAMP
    return len(sample), above


@pytest.mark.parametrize("v", [2.0, 3.0])
def test_oracle_voxel_stage_against_exact(O, v):
    est = surface(60000, 24.0, v, seed=1)
    gt = surface(60000, 24.0, v, seed=2, origin=(0.01, -0.02, 0.03))
    got, rows = O.eval_awd(est, gt, v, 100, 5, want_rows=True)
    pairs, nve, nvg = X.voxel_pairs(est, gt, v, 100)
    assert (got.n_voxels_est, got.n_voxels_gt, got.n_pairs) == (nve, nvg, len(pairs))
    checked, above = check_voxel_rows(rows, pairs, v, range(0, len(rows), 3))
    assert above >= 0.3 * checked


def test_oracle_wasserstein_on_the_reference_fixture(golden_dir, O):
    """the reference's own voxel_errors.txt rows (3 m voxels): W from the stored values, exactly"""
    rows = np.load(os.path.join(golden_dir, "voxel_fixture.npz"))["rows"]
    for r in rows[::11]:
        sg, se = _sym(r[21:27]).reshape(3, 3), _sym(r[12:18]).reshape(3, 3)
        w2, tr = X.wasserstein2(r[18:21], sg.tolist(), int(r[10]), r[6:9], se.tolist(), int(r[11]))
        w = O.wasserstein(r[18:21], sg.ravel(), int(r[10]), r[6:9], se.ravel(), int(r[11]))
        assert abs(w * w - float(w2)) <= X.w_bound(tr, r[6:9], r[18:21], 3.0)

"""The numpy statement of global registration (tests/fpfh_ref.py) against plain-Python loops, hand-built pair features and
the properties the stages must have; the ctypes mirrors of its structs against the header.  No GPU."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fpfh_ref as R  # noqa: E402
import perturb_ref  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cloud(n, seed, side=1.0):
    rng = np.random.RandomState(seed)
    xyz = rng.rand(n, 3) * side
    nrm = rng.randn(n, 3)
    return xyz, nrm / np.linalg.norm(nrm, axis=1, keepdims=True)


def _rot(yaw, tilt_x, tilt_y):
    cz, sz, cx, sx, cy, sy = math.cos(yaw), math.sin(yaw), math.cos(tilt_x), math.sin(tilt_x), math.cos(tilt_y), math.sin(tilt_y)
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    return Rz @ Ry @ Rx


# ---- plain loops ----------------------------------------------------------------------------------------------------
def _loop_pair(p1, n1, p2, n2):
    dot = lambda a, b: a[0] * b[0] + (a[1] * b[1] + a[2] * b[2])  # noqa: E731
    cross = lambda a, b: [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]  # noqa: E731
    dp = [p2[k] - p1[k] for k in range(3)]
    ln = math.sqrt(dot(dp, dp))
    if ln == 0.0:
        return [0.0, 0.0, 0.0]
    a1, a2 = dot(n1, dp) / ln, dot(n2, dp) / ln
    m1, m2 = list(n1), list(n2)
    if math.acos(min(1.0, abs(a1))) > math.acos(min(1.0, abs(a2))):
        m1, m2, dp, f2 = list(n2), list(n1), [-x for x in dp], -a2
    else:
        f2 = a1
    v = cross(dp, m1)
    vn = math.sqrt(dot(v, v))
    if vn == 0.0:
        return [0.0, 0.0, 0.0]
    v = [x / vn for x in v]
    w = cross(m1, v)
    return [math.atan2(dot(w, m2), dot(m1, m2)), dot(v, m2), f2]


def _loop_features(xyz, nrm, radius, max_nn):
    n = len(xyz)
    nb = []
    for i in range(n):
        c = []
        for j in range(n):
            if j == i:
                continue
            d = [xyz[i][k] - xyz[j][k] for k in range(3)]
            d2 = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
            if d2 < radius * radius:
                c.append((d2, j))
        nb.append(sorted(c)[:max_nn])
    sp = [[0.0] * 33 for _ in range(n)]
    for i in range(n):
        for _, j in nb[i]:
            f = _loop_pair(xyz[i], nrm[i], xyz[j], nrm[j])
            scaled = [11 * (f[0] + math.pi) / (2.0 * math.pi), 11 * (f[1] + 1.0) * 0.5, 11 * (f[2] + 1.0) * 0.5]
            for g in range(3):
                sp[i][11 * g + min(10, max(0, math.floor(scaled[g])))] += 100.0 / len(nb[i])
    out = []
    for i in range(n):
        acc, s = [0.0] * 33, [0.0] * 3
        for d2, j in nb[i]:
            if d2 == 0.0:
                continue
            for b in range(33):
                acc[b] += sp[j][b] / d2
                s[b // 11] += sp[j][b] / d2
        s = [100.0 / x if x != 0.0 else 0.0 for x in s]
        out.append([acc[b] * s[b // 11] + sp[i][b] for b in range(33)])
    return nb, np.array(sp), np.array(out)


def test_statement_equals_plain_loops():
    xyz, nrm = _cloud(80, 1)
    nb_l, sp_l, f_l = _loop_features(xyz.tolist(), nrm.tolist(), 0.35, 12)
    f32, f64, flagged, nb = R.features(xyz, nrm, 0.35, 12)
    for i in range(len(xyz)):
        assert [j for _, j in nb_l[i]] == nb[i][0].tolist()
        assert [d for d, _ in nb_l[i]] == nb[i][1].tolist()
    sp, _ = R.spfh(xyz, nrm, nb)
    ok = ~flagged
    assert ok.sum() >= 75
    np.testing.assert_allclose(sp[ok], sp_l[ok], rtol=0, atol=1e-12)
    np.testing.assert_allclose(f64[ok], f_l[ok], rtol=0, atol=1e-10)
    assert (f32 == f64.astype(np.float32)).all()


def test_hand_built_pair_features():
    z, x, y = [0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]
    o, px = [0.0, 0.0, 0.0], [2.0, 0.0, 0.0]
    f = lambda p1, n1, p2, n2: R.pair_features(p1, n1, p2, n2)[0][0]  # noqa: E731
    np.testing.assert_array_equal(f(o, z, o, x), [0, 0, 0])                       # coincident points
    np.testing.assert_array_equal(f(o, x, px, y), [0, 0, 0])                      # dp x n1 = 0
    np.testing.assert_array_equal(f(o, z, px, x), [0, 0, 0])                      # after the swap, dp x n2 = 0
    np.testing.assert_allclose(f(o, z, px, z), [0, 0, 0], atol=1e-15)            # parallel normals across the line
    np.testing.assert_allclose(f(o, z, px, y), [0, -1, 0], atol=1e-15)           # perpendicular normals
    th = 0.3
    np.testing.assert_allclose(f(o, z, px, [0.0, -math.sin(th), math.cos(th)])[1], math.sin(th), atol=1e-15)
    # the frame sits on the point whose normal is closer to the line: swapping the pair gives the same features
    rng = np.random.RandomState(3)
    for _ in range(200):
        p1, p2 = rng.randn(3), rng.randn(3)
        n1, n2 = rng.randn(3), rng.randn(3)
        n1, n2 = n1 / np.linalg.norm(n1), n2 / np.linalg.norm(n2)
        a, b = f(p1, n1, p2, n2), f(p2, n2, p1, n1)
        np.testing.assert_allclose(a, b, atol=1e-12)
        np.testing.assert_allclose(a, _loop_pair(p1.tolist(), n1.tolist(), p2.tolist(), n2.tolist()), atol=1e-15)
    assert R.pair_bins(np.array([[0.0, -1.0, 1.0]])).tolist() == [[5, 11, 32]]
    assert R.bin_edge_flags(np.array([[-np.pi + 2 * np.pi / 11, 0.3, 0.3], [0.01, 0.3, 0.3]])).tolist() == [True, False]


def test_group_sums():
    xyz, nrm = _cloud(400, 2)
    nb = R.hybrid_neighbours(xyz, 0.3, 30)
    assert min(len(ix) for ix, _ in nb) > 0
    sp, _ = R.spfh(xyz, nrm, nb)
    _, f64, _ = R.fpfh(sp, nb)
    np.testing.assert_allclose(sp.reshape(-1, 3, 11).sum(2), 100.0, rtol=1e-12)
    np.testing.assert_allclose(f64.reshape(-1, 3, 11).sum(2), 200.0, rtol=1e-12)


def test_fpfh_is_invariant_under_a_rigid_motion():
    xyz, nrm = _cloud(500, 5, side=4.0)
    Rm = _rot(1.1, 0.07, -0.04)
    t = np.array([312.5, -87.25, 14.0])
    a32, a64, afl, _ = R.features(xyz, nrm, 0.9, 200)
    b32, b64, bfl, _ = R.features(xyz @ Rm.T + t, nrm @ Rm.T, 0.9, 200)
    ok = ~(afl | bfl)
    assert ok.sum() >= 490
    np.testing.assert_allclose(a64[ok], b64[ok], rtol=0, atol=1e-8)


def test_orientation_rule():
    xyz, nrm = _cloud(300, 6, side=10.0)
    xyz[:, 2] *= 0.01                                                          # a floor, normals of either sign
    nrm = np.c_[0.05 * nrm[:, :2], np.sign(nrm[:, 2])]
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    out, amb = R.orient_normals(xyz, nrm)
    assert not amb.any()
    assert (out[:, 2] >= 0).all() and (np.abs(out) == np.abs(nrm)).all()
    # the rule moves with a yaw of the map
    Rm = _rot(2.0, 0.0, 0.0)
    out2, _ = R.orient_normals(xyz @ Rm.T + [5.0, -3.0, 1.0], nrm @ Rm.T)
    np.testing.assert_allclose(out2, out @ Rm.T, atol=1e-15)


def test_matching_rounds_every_operation_and_breaks_ties_to_the_smaller_index():
    rng = np.random.RandomState(7)
    fe = (rng.rand(40, 33) * 50).astype(np.float32)
    fg = (rng.rand(50, 33) * 50).astype(np.float32)
    fg[17] = fg[3]                                                            # a tie
    fe[5] = fg[3]
    nn = R.feature_nn(fe, fg)
    for i in range(len(fe)):
        d = []
        for j in range(len(fg)):
            s = np.float32(0)
            for b in range(33):
                t = np.float32(fe[i, b] - fg[j, b])
                s = np.float32(s + np.float32(t * t))
            d.append(s)
        assert nn[i] == int(np.argmin(d))
    assert nn[5] == 3
    ie, ig = R.correspondences(fe, fg)
    g2e = R.feature_nn(fg, fe)
    assert all(g2e[j] == i and nn[i] == j for i, j in zip(ie, ig))
    ie2, ig2 = R.correspondences(fe, fg, mutual=False)
    assert ie2.tolist() == list(range(40)) and (ig2 == nn).all()


def test_draws_are_the_counter_hash_on_lanes_16_to_18():
    M = (1 << 64) - 1

    def mix(z):
        z = (z + 0x9E3779B97F4A7C15) & M
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        return z ^ (z >> 31)

    seed, nc = 987654321, 1234
    d = R.draws(seed, 300, nc)
    for h in range(300):
        for t in range(3):
            lane = 16 + t
            key = mix((seed + lane * 0xD1B54A32D192ED03) & M)
            u = (mix(key ^ ((h * 0x2545F4914F6CDD1D + lane) & M)) >> 11) * 2.0 ** -53
            assert d[h, t] == min(math.floor(u * nc), nc - 1)
    np.testing.assert_array_equal(d[:, 1], np.minimum(np.floor(perturb_ref.uniform53(seed, np.arange(300, dtype=np.uint64), 17) * nc), nc - 1))


def test_jacobi_svd_and_umeyama_restated():
    rng = np.random.RandomState(8)
    s = rng.randn(500, 9)
    s[:50, 6:] = 0.0                                                          # rank 2
    U, w, V = R.svd3(s)
    np.testing.assert_allclose(w, np.linalg.svd(s.reshape(-1, 3, 3), compute_uv=False), rtol=1e-12, atol=1e-14)
    # Umeyama of an exact rigid motion
    for k in range(20):
        Rm = _rot(*rng.uniform(-3, 3, 3))
        t = rng.uniform(-200, 200, 3)
        p = rng.randn(3, 3) * 5 + 1000.0
        q = p @ Rm.T + t
        c = np.array([1000.0, 1000.0, 1000.0])
        T = R.umeyama_from_sums(R.three_point_sums(p, q, np.array([[0, 1, 2]]), c), c)[0]
        np.testing.assert_allclose(T[:3, :3], Rm, atol=1e-11)
        np.testing.assert_allclose(T[:3, 3], t, atol=1e-8)


def test_ransac_recovers_exact_correspondences_among_half_outliers():
    rng = np.random.RandomState(9)
    n = 200
    P = rng.rand(n, 3) * 20.0 + [1500.0, -300.0, 20.0]
    Rm, t = _rot(2.3, 0.05, -0.03), np.array([-61.8, 53.1, 2.5])
    Q = P @ Rm.T + t
    out = rng.rand(n) < 0.5
    Q[out] = rng.rand(out.sum(), 3) * 20.0 + Q[~out].mean(0)
    c = 0.5 * (Q.min(0) + Q.max(0))
    res = R.ransac(P, Q, c, seed=11, n_hypotheses=3000, ratio=0.9, d2max=0.01)
    assert res["n_valid"] > 0 and res["counts"][res["best"]] >= (~out).sum()
    assert (res["counts"][res["best"]] > res["counts"][:res["best"]]).all()          # ties to the smallest h
    T, n_in, rmse = R.refine(P, Q, c, res["T"][res["best"]], 0.01)
    assert n_in == (~out).sum() and rmse < 1e-9
    np.testing.assert_allclose(T[:3, :3], Rm, atol=1e-9)
    np.testing.assert_allclose(T[:3, 3], t, atol=1e-9)


def test_struct_sizes_match_the_header(tmp_path):
    src = tmp_path / "sz.c"
    names = ["me_global_reg_params", "me_global_reg_result"]
    src.write_text('#include <stdio.h>\n#include "mapeval_b200.h"\nint main(){' +
                   "".join(f'printf("%zu\\n", sizeof({n}));' for n in names) + "return 0;}\n")
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    assert sizes == [C.sizeof(getattr(A, n)) for n in names]
    p = A.make_global_reg_params(0.5, seed=3, n_hypotheses=10)
    assert (p.feature_radius, p.feature_max_nn, p.max_correspondence_distance, p.n_hypotheses, p.seed) == (5.0, 128, 0.75, 10, 3)
    with pytest.raises(ValueError):
        A.make_global_reg_params(0.5, radius=1.0)

"""The numpy / scipy statements of tests/normals_ref.py — the reference of the GPU tests of normals carried through
VoxelDownSample and generalized ICP — against an independent plain-Python statement and against the oracle where the
oracle covers the same ground (down-sampled points, GetRotationFromE1ToX covariances, generalized ICP on k-NN normals)."""
import os
import sys

import numpy as np
import pytest

from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import normals_ref as ref  # noqa: E402


def _rot(rx, ry, rz):
    ca, sa, cb, sb, cg, sg = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    Ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    Rz = np.array([[cg, -sg, 0], [sg, cg, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def _scene(n, seed, noise):
    """a bumpy floor, a wall facing +y and a wall facing -x"""
    rs = np.random.RandomState(seed)
    m = n // 4
    x, y = rs.rand(n - 2 * m) * 6, rs.rand(n - 2 * m) * 6
    floor = np.stack([x, y, 0.15 * np.sin(1.3 * x) * np.cos(0.9 * y)], 1)
    u, v = rs.rand(m) * 6, rs.rand(m) * 2.5
    wall_y = np.stack([u, 6.0 + 0.1 * np.sin(u), v], 1)
    u, v = rs.rand(m) * 6, rs.rand(m) * 2.5
    wall_x = np.stack([0.05 * np.sin(u), u, v], 1)
    p = np.concatenate([floor, wall_y, wall_x]) + noise * rs.randn(n, 3)
    return p.astype(np.float32).astype(np.float64)


# ---- VoxelDownSample with normals -------------------------------------------------------------------------------------
def _py_downsample_normals(xyz, nrm, s):
    """one dict entry per voxel, points visited in input order (Python floats: IEEE fp64, no contraction)"""
    org = xyz.min(0) - s * 0.5
    keys = np.floor((xyz - org) / s).astype(np.int64)
    acc = {}
    for i in range(len(xyz)):
        a = acc.setdefault(tuple(keys[i]), [[0.0, 0.0, 0.0], 0, [0.0, 0.0, 0.0]])
        for k in range(3):
            a[0][k] += float(xyz[i, k])
        a[1] += 1
        if not np.isnan(nrm[i]).any():
            for k in range(3):
                a[2][k] += float(nrm[i, k])
    order = sorted(acc)
    pts = np.array([[acc[k][0][a] / acc[k][1] for a in range(3)] for k in order])
    nr = np.array([[acc[k][2][a] / acc[k][1] for a in range(3)] for k in order])
    return pts, nr


def _normals_fixture(seed=4):
    """scattered points with noisy unit normals plus voxels built for the corner cases of the averaging"""
    rs = np.random.RandomState(seed)
    s = 0.25
    xyz = rs.rand(3000, 3) * 5.0
    xyz = np.concatenate([xyz, xyz[:600] + 0.02 * rs.randn(600, 3)])          # voxels of several points
    nrm = rs.randn(len(xyz), 3)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    nrm[rs.rand(len(xyz)) < 0.05, rs.randint(0, 3)] = np.nan                   # a NaN component: skipped, still counted
    c = s * np.array([40.0, 41.0, 42.0])                                       # a voxel centre beyond the scattered points
    opp = c + 0.01 * rs.randn(4, 3)                                            # opposite normals: average ~ (0, 0, 0)
    opp_n = np.array([[0.3, 0.4, np.sqrt(0.75)]] * 2 + [[-0.3, -0.4, -np.sqrt(0.75)]] * 2)
    nan_p = c + [s, 0, 0] + 0.01 * rs.randn(3, 3)                              # all normals NaN: (0, 0, 0)
    nan_n = np.array([[np.nan, 0.0, 1.0], [0.0, np.nan, np.nan], [np.nan] * 3])
    one_p = (c + [0, s, 0])[None]                                              # a single point: its normal unchanged
    one_n = np.array([[0.1, -2.0, 0.7]])
    xyz = np.concatenate([xyz, opp, nan_p, one_p])
    nrm = np.concatenate([nrm, opp_n, nan_n, one_n])
    return xyz, nrm, s


def test_voxel_downsample_normals_reference():
    xyz, nrm, s = _normals_fixture()
    pts, nr = ref.voxel_downsample_normals(xyz, nrm, s)
    ep, en = _py_downsample_normals(xyz, nrm, s)
    np.testing.assert_array_equal(pts, ep)
    np.testing.assert_array_equal(nr, en)
    np.testing.assert_array_equal(pts, O.voxel_downsample(xyz, s))             # the oracle's points, same order
    assert len(pts) < len(xyz) and not np.isnan(nr).any()
    # the corner cases: opposite normals cancel, an all-NaN voxel gives zero, a single point keeps its (non-unit) normal
    row = {tuple(np.floor((p - (xyz.min(0) - s / 2)) / s).astype(int)): i for i, p in enumerate(pts)}
    assert np.abs(nr[row[(40, 41, 42)]]).max() < 1e-15
    np.testing.assert_array_equal(nr[row[(41, 41, 42)]], [0.0, 0.0, 0.0])
    np.testing.assert_array_equal(nr[row[(40, 42, 42)]], [0.1, -2.0, 0.7])


# ---- generalized ICP with given normals -------------------------------------------------------------------------------
def _py_cov(x, eps=1e-3):
    """GetRotationFromE1ToX(x) diag(eps, 1, 1) GetRotationFromE1ToX(x)^T, one vector at a time"""
    x = np.asarray(x, dtype=np.float64)
    R = np.eye(3)
    if not x[0] < -0.99:
        v = np.cross([1.0, 0.0, 0.0], x)
        K = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])
        R = np.eye(3) + K + K @ K / (1.0 + x[0])
    return R @ np.diag([eps, 1.0, 1.0]) @ R.T


def test_gicp_covariance_of_given_normals():
    rs = np.random.RandomState(5)
    cases = [rs.randn(3) * rs.uniform(0.3, 2.0) for _ in range(40)]           # non-unit normals as files may carry them
    cases += [np.array([-0.995, 0.1, 0.0]), np.array([-3.0, 0.2, 0.1]), np.zeros(3), np.array([0.0, 0.0, 0.5])]
    got = ref.gicp_covariances(np.array(cases))
    for x, g in zip(cases, got):
        for exp in (_py_cov(x), O.gicp_covariance(x)):
            np.testing.assert_allclose(g, exp, rtol=0, atol=1e-12 * max(1.0, np.abs(exp).max()))
    np.testing.assert_array_equal(got[-3], np.diag([1e-3, 1.0, 1.0]))          # n.x < -0.99 and zero: Rx = I
    np.testing.assert_array_equal(got[-2], np.diag([1e-3, 1.0, 1.0]))
    x = np.array([0.0, 0.6, 0.0])                                              # |x| != 1: not I + (eps - 1) x x^T
    assert np.abs(ref.gicp_covariances(x)[0] - (np.eye(3) + (1e-3 - 1) * np.outer(x, x))).max() > 0.1


def _pair():
    gt = _scene(9000, 11, 0.002)
    T_true = np.eye(4)
    T_true[:3, :3] = _rot(0.012, -0.008, 0.015)
    T_true[:3, 3] = [0.03, -0.02, 0.015]
    est = _scene(7000, 12, 0.006)
    est = ((est - T_true[:3, 3]) @ T_true[:3, :3]).astype(np.float32).astype(np.float64)
    return est, gt, T_true


def _file_like_normals(xyz, seed):
    """k-NN normals as a file might carry them: scaled away from unit length, the -x wall pointing to -e1 (n.x < -0.99:
    Rx = I), and a few zero normals"""
    rs = np.random.RandomState(seed)
    n = O.estimate_normals_knn(xyz, 20)
    flip = np.abs(n[:, 0]) > 0.995
    n[flip] *= -np.sign(n[flip, 0])[:, None]
    scale = rs.uniform(0.7, 1.3, len(n))
    scale[flip] = 1.0
    n *= scale[:, None]
    n[rs.rand(len(n)) < 0.01] = 0.0
    assert (n[:, 0] < -0.99).sum() > 100 and (np.abs(np.linalg.norm(n, axis=1) - 1) > 0.05).mean() > 0.5
    return n


def test_gicp_reference_on_knn_normals_is_the_oracle():
    """given the k-NN normals the oracle estimates itself, the reference is the oracle's generalized ICP"""
    est, gt, _ = _pair()
    T0 = np.eye(4)
    T0[:3, 3] = [0.004, 0.0, -0.003]
    To, fo, ro, nco, ito = O.icp_generalized(est, gt, 0.5, T0)
    T, f, r, nc, it = ref.icp_generalized(est, gt, O.estimate_normals_knn(est, 20), O.estimate_normals_knn(gt, 20), 0.5, T0)
    assert it == ito and nc == nco and 2 <= it <= 30
    np.testing.assert_allclose(T, To, rtol=0, atol=1e-9)
    np.testing.assert_allclose([f, r], [fo, ro], rtol=1e-9)


@pytest.mark.parametrize("which", ["gt", "both"])
def test_gicp_reference_with_given_normals_registers(which):
    est, gt, T_true = _pair()
    nt = _file_like_normals(gt, 1)
    ns = _file_like_normals(est, 2) if which == "both" else O.estimate_normals_knn(est, 20)
    T0 = np.eye(4)
    T0[:3, 3] = [0.004, 0.0, -0.003]
    T, fit, rmse, nc, it = ref.icp_generalized(est, gt, ns, nt, 0.5, T0)
    assert 2 <= it <= 30
    np.testing.assert_allclose(T[:3, 3], T_true[:3, 3], atol=5e-3)
    np.testing.assert_allclose(T[:3, :3], T_true[:3, :3], atol=2e-3)
    # the given normals are what the covariances are built from: the estimating path lands elsewhere
    assert np.abs(T - O.icp_generalized(est, gt, 0.5, T0)[0]).max() > 1e-7

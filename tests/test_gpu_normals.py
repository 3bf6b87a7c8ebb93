"""Normals a cloud carries, on the GPU, against the oracle: VoxelDownSample averages them (me_voxel_downsample),
point-to-plane ICP runs on the averaged normals of a down-sampled ground truth, and generalized ICP builds a cloud's
covariances from its own normals (InitializePointCloudForGeneralizedICP) instead of estimating them.  The reference for
the averaged normals and for generalized ICP on given normals is tests/normals_ref.py."""
import os
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import normals_ref as ref  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _rot(rx, ry, rz):
    ca, sa, cb, sb, cg, sg = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    Ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    Rz = np.array([[cg, -sg, 0], [sg, cg, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def _scene(n, seed, noise, origin=(0.0, 0.0, 0.0)):
    """bumpy floor + a wall facing +y + a wall facing -x"""
    rs = np.random.RandomState(seed)
    m = n // 4
    x, y = rs.rand(n - 2 * m) * 12, rs.rand(n - 2 * m) * 12
    floor = np.stack([x, y, 0.2 * np.sin(0.9 * x) * np.cos(0.7 * y)], 1)
    u, v = rs.rand(m) * 12, rs.rand(m) * 3
    wall_y = np.stack([u, 12.0 + 0.1 * np.sin(u), v], 1)
    u, v = rs.rand(m) * 12, rs.rand(m) * 3
    wall_x = np.stack([0.05 * np.sin(u), u, v], 1)
    p = np.concatenate([floor, wall_y, wall_x]) + noise * rs.randn(n, 3) + np.asarray(origin)
    return p.astype(np.float32).astype(np.float64)


def _pair(n_est=150_000, n_gt=200_000, origin=(0.0, 0.0, 0.0)):
    gt = _scene(n_gt, 21, 0.003, origin)
    T_true = np.eye(4)
    T_true[:3, :3] = _rot(0.01, -0.006, 0.012)
    T_true[:3, 3] = [0.04, -0.03, 0.02]
    est = _scene(n_est, 22, 0.008, origin)
    c = np.asarray(origin) + 6.0
    est = ((est - c - T_true[:3, 3]) @ T_true[:3, :3]) + c
    return est.astype(np.float32).astype(np.float64), gt


def _rotate_normals(nrm, T):
    """PointCloud::TransformNormals: (T00 nx + T01 ny) + T02 nz, every operation rounded on its own"""
    return np.stack([(T[r, 0] * nrm[:, 0] + T[r, 1] * nrm[:, 1]) + T[r, 2] * nrm[:, 2] for r in range(3)], 1)


def _by_point(pts):
    return np.lexsort((pts[:, 2], pts[:, 1], pts[:, 0]))


def _noisy_normals(n, seed):
    """random unit normals, some with a NaN component, some zero"""
    rs = np.random.RandomState(seed)
    nrm = rs.randn(n, 3)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    nrm[rs.rand(n) < 0.03, rs.randint(0, 3)] = np.nan
    nrm[rs.rand(n) < 0.01] = 0.0
    return nrm


def test_voxel_downsample_averages_normals(api, O):
    s = 0.1
    xyz = _scene(300_000, 3, 0.004, origin=(120.0, -40.0, 5.0))
    nrm = _noisy_normals(len(xyz), 4)
    org = xyz.min(0) - s / 2                                         # a voxel centre beyond the scene (the bounds stay)
    c = org + (np.floor((np.array([140.0, -20.0, 20.0]) - org) / s) + 0.5) * s
    extra = np.concatenate([c + 0.003 * np.arange(4)[:, None], c + [1.0, 0, 0] + 0.003 * np.arange(3)[:, None],
                            (c + [0, 1.0, 0])[None]])
    extra_n = np.array([[0.3, 0.4, np.sqrt(0.75)]] * 2 + [[-0.3, -0.4, -np.sqrt(0.75)]] * 2
                       + [[np.nan, 0.0, 1.0], [0.0, np.nan, np.nan], [np.nan] * 3] + [[0.1, -2.0, 0.7]])
    xyz, nrm = np.concatenate([xyz, extra]), np.concatenate([nrm, extra_n])
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(A.ME_CLOUD_EST, xyz)
        ctx.set_normals(A.ME_CLOUD_EST, nrm)
        nv = ctx.voxel_downsample(A.ME_CLOUD_EST, s)
        pts, nr = ctx.get_cloud(A.ME_CLOUD_EST), ctx.get_normals(A.ME_CLOUD_EST)
        T = np.eye(4)
        T[:3, :3] = _rot(0.3, -0.2, 1.1)
        T[:3, 3] = [5.0, -3.0, 2.0]
        ctx.transform(A.ME_CLOUD_EST, T)
        nr_moved = ctx.get_normals(A.ME_CLOUD_EST)
    with api.MapEvalB200() as ctx:                                  # the same cloud without normals: today's path
        ctx.set_cloud(A.ME_CLOUD_EST, xyz)
        ctx.voxel_downsample(A.ME_CLOUD_EST, s)
        pts_plain = ctx.get_cloud(A.ME_CLOUD_EST)
        with pytest.raises(api.MapEvalError, match="has no normals"):
            ctx.get_normals(A.ME_CLOUD_EST)
    assert nv == len(pts) == len(nr) and nv < len(xyz)
    np.testing.assert_array_equal(pts, pts_plain)
    opts, onr = ref.voxel_downsample_normals(xyz, nrm, s)
    g, o = _by_point(pts), _by_point(opts)
    np.testing.assert_array_equal(pts[g], opts[o])
    np.testing.assert_array_equal(nr[g], onr[o])
    assert not np.isnan(nr).any()
    corner = [np.argmin(np.abs(pts - p).sum(1)) for p in (c, c + [1.0, 0, 0], c + [0, 1.0, 0])]
    assert np.abs(nr[corner[0]]).max() < 1e-15                       # opposite normals cancel, not re-normalised
    np.testing.assert_array_equal(nr[corner[1]], [0.0, 0.0, 0.0])    # only NaN normals: (0, 0, 0)
    np.testing.assert_array_equal(nr[corner[2]], [0.1, -2.0, 0.7])   # a single point keeps its normal as given
    np.testing.assert_array_equal(nr_moved, _rotate_normals(nr, T))                 # me_transform rotates them


def test_point_to_plane_icp_on_averaged_normals(api, O):
    est, gt = _pair(100_000, 120_000)
    nrm = O.estimate_normals_knn(gt, 20)
    s = 0.1
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(A.ME_CLOUD_EST, est)
        ctx.set_cloud(A.ME_CLOUD_GT, gt)
        ctx.set_normals(A.ME_CLOUD_GT, nrm)
        ctx.voxel_downsample(A.ME_CLOUD_GT, s)
        dg, dn = ctx.get_cloud(A.ME_CLOUD_GT), ctx.get_normals(A.ME_CLOUD_GT)
        T, reg = ctx.performICPRegistration(0.5, method=A.ME_ICP_POINT_TO_PLANE)
        np.testing.assert_array_equal(ctx.get_normals(A.ME_CLOUD_GT), dn)
    odg, odn = ref.voxel_downsample_normals(gt, nrm, s)
    np.testing.assert_array_equal(dg, odg)                           # both emit the voxels in increasing (ix, iy, iz)
    np.testing.assert_array_equal(dn, odn)
    assert np.abs(np.linalg.norm(dn, axis=1) - 1).max() > 1e-3       # averaged: no longer unit length
    To, fit, rmse, nc, it = O.icp_point_to_plane(est, odg, odn, 0.5)
    assert reg.iterations == it and abs(reg.n_corr - nc) <= 2
    np.testing.assert_allclose(T, To, atol=1e-8)
    np.testing.assert_allclose([reg.fitness, reg.inlier_rmse], [fit, rmse], rtol=1e-6)


def _file_like_normals(O, xyz, seed):
    """k-NN normals as a file might carry them: scaled away from unit length, the -x wall pointing to -e1 (n.x < -0.99:
    GetRotationFromE1ToX falls back to I), and a few zero normals"""
    rs = np.random.RandomState(seed)
    n = O.estimate_normals_knn(xyz, 20)
    flip = np.abs(n[:, 0]) > 0.995
    n[flip] *= -np.sign(n[flip, 0])[:, None]
    scale = rs.uniform(0.7, 1.3, len(n))
    scale[flip] = 1.0
    n *= scale[:, None]
    n[rs.rand(len(n)) < 0.01] = 0.0
    assert (n[:, 0] < -0.99).sum() > 1000
    return n


@pytest.mark.parametrize("which", ["gt", "both"])
@pytest.mark.parametrize("origin", [(0.0, 0.0, 0.0), (1500.0, -800.0, 40.0)])
def test_generalized_icp_with_given_normals(api, O, origin, which):
    est, gt = _pair(origin=origin)
    nt = _file_like_normals(O, gt, 1)
    ns = _file_like_normals(O, est, 2) if which == "both" else None
    T0 = np.eye(4)
    T0[:3, 3] = [0.003, 0.0, -0.002]
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(A.ME_CLOUD_EST, est)
        ctx.set_cloud(A.ME_CLOUD_GT, gt)
        ctx.set_normals(A.ME_CLOUD_GT, nt)
        if ns is not None:
            ctx.set_normals(A.ME_CLOUD_EST, ns)
        T, reg = ctx.performICPRegistration(0.5, T0, method=A.ME_ICP_GENERALIZED)
        aligned = ctx.get_cloud(A.ME_CLOUD_EST)
        np.testing.assert_array_equal(ctx.get_normals(A.ME_CLOUD_GT), nt)          # the target's normals are untouched
        if ns is not None:                                                           # the source's move with the cloud
            np.testing.assert_array_equal(ctx.get_normals(A.ME_CLOUD_EST), _rotate_normals(ns, T))
        else:                                                                        # the k-NN estimate does not outlive the call
            with pytest.raises(api.MapEvalError, match="has no normals"):
                ctx.get_normals(A.ME_CLOUD_EST)
    To, fit, rmse, nc, it = ref.icp_generalized(est, gt, O.estimate_normals_knn(est, 20) if ns is None else ns, nt, 0.5, T0)
    far = origin[0] != 0.0
    assert abs(reg.iterations - it) <= (1 if far else 0) and 2 <= it <= 30
    assert abs(reg.n_corr - nc) <= 2
    moved, omoved = O.transform(est, T), O.transform(est, To)
    assert np.abs(moved - omoved).max() < (5e-6 if far else 1e-7)
    np.testing.assert_allclose(T[:3, :3], To[:3, :3], atol=1e-7 if far else 1e-8)
    np.testing.assert_allclose([reg.fitness, reg.inlier_rmse], [fit, rmse], rtol=1e-5 if far else 1e-6)
    np.testing.assert_allclose(aligned, moved, atol=1e-9)
    assert reg.inlier_rmse < 0.03

"""me_transform bit for bit against the statement of Open3D's PointCloud::Transform: every product and sum rounded on
its own (Eigen's 4×4 product, built without FMA), in the order

    p' = (((T00 x + T01 y) + T02 z) + T03) / w,   w = ((T30 x + T31 y) + T32 z) + T33
    n' = (T00 nx + T01 ny) + T02 nz              (the normals: no translation, no division)

at 1.5 km, for an exact 90° turn, a general rotation and a last row with w ≠ 1, and after registration, whose result is
the statement applied to the original estimate and its normals with the returned T.  numpy rounds every operation
separately, so the statement is numpy's plain expression."""
import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT


def _api():
    from cloud_map_evaluation_b200 import api
    return api


def transform_points(xyz, T):
    x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    o = [((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3] for r in range(4)]
    return np.stack([o[0] / o[3], o[1] / o[3], o[2] / o[3]], 1)


def transform_normals(nrm, T):
    x, y, z = nrm[:, 0], nrm[:, 1], nrm[:, 2]
    return np.stack([(T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z for r in range(3)], 1)


def _assert_bits(got, exp, what):
    assert got.shape == exp.shape
    bad = (np.ascontiguousarray(got).view(np.uint64) != np.ascontiguousarray(exp).view(np.uint64)).any(1)
    assert not bad.any(), f"{what}: {bad.sum()} of {len(bad)} rows differ, first at {np.flatnonzero(bad)[:5]}"


def _rot(rx, ry, rz):
    ca, sa, cb, sb, cg, sg = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    Ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    Rz = np.array([[cg, -sg, 0], [sg, cg, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def _matrix(kind):
    T = np.eye(4)
    if kind == "turn90":                                 # exact: every product and sum is exact, FMA or not
        T[:3, :3] = [[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]
        T[:3, 3] = [0.5, -0.25, 2.0]
    else:
        T[:3, :3] = _rot(0.3, -0.2, 1.1)
        T[:3, 3] = [5.0, -3.0, 2.0]
    if kind == "projective":
        T[3] = [1e-5, -2e-5, 3e-6, 1.25]
    return T


def _cloud(n=200_000, seed=0):
    rng = np.random.RandomState(seed)
    xyz = np.array([1500.0, -1500.0, 40.0]) + rng.uniform(-50.0, 50.0, (n, 3))
    nrm = rng.randn(n, 3)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    nrm[::97] *= 1.7                                     # not every normal is unit length
    return xyz, nrm


@pytest.mark.parametrize("kind", ["turn90", "general", "projective"])
def test_transform_matches_statement(kind):
    xyz, nrm = _cloud()
    T = _matrix(kind)
    with _api().MapEvalB200() as ctx:
        ctx.set_cloud(EST, xyz)
        ctx.set_normals(EST, nrm)
        ctx.transform(EST, T)
        pts, nr = ctx.get_cloud(EST), ctx.get_normals(EST)
    _assert_bits(pts, transform_points(xyz, T), "points")
    _assert_bits(nr, transform_normals(nrm, T), "normals")


def test_normals_after_registration():
    """performICPRegistration leaves est := Transform(original, T): the points and the normals handed in equal the
    statement applied to the originals with the returned T"""
    rng = np.random.RandomState(1)
    gt = np.array([1500.0, -1500.0, 40.0]) + np.concatenate([
        np.c_[rng.rand(60_000, 2) * 8.0, 0.02 * rng.randn(60_000)],
        np.c_[rng.rand(30_000) * 8.0, 8.0 + 0.02 * rng.randn(30_000), rng.rand(30_000) * 3.0],
        np.c_[0.02 * rng.randn(30_000), rng.rand(30_000) * 8.0, rng.rand(30_000) * 3.0]])
    T_true = np.eye(4)                                       # a small turn about the scene's centre and a shift
    T_true[:3, :3] = _rot(0.01, -0.008, 0.015)
    c = np.array([1504.0, -1496.0, 41.5])
    T_true[:3, 3] = c - T_true[:3, :3] @ c + [0.05, -0.04, 0.03]
    est = transform_points(gt[rng.permutation(len(gt))[:80_000]] + 0.003 * rng.randn(80_000, 3), T_true)
    nrm = rng.randn(len(est), 3)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    with _api().MapEvalB200() as ctx:
        ctx.set_cloud(EST, est)
        ctx.set_cloud(GT, gt)
        ctx.set_normals(EST, nrm)
        T, reg = ctx.performICPRegistration(0.5)
        pts, nr = ctx.get_cloud(EST), ctx.get_normals(EST)
    assert reg.iterations >= 2 and reg.fitness > 0.9
    assert np.abs(T[:3, :3] - np.eye(3)).max() > 1e-3        # a real turn: the rounding of the normals is visible
    _assert_bits(pts, transform_points(est, T), "points")
    _assert_bits(nr, transform_normals(nrm, T), "normals")

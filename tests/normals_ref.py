"""numpy / scipy statements of the two places where Open3D uses the normals a cloud carries, for the tests of that
feature (not collected as a test module):

* VoxelDownSample with normals (AccumulatedPoint::AddPoint / GetAverageNormal): per voxel the points and the normals are
  summed in INPUT order, a normal only when none of its components is NaN; both sums are divided by the count of all the
  voxel's points; the normal is not re-normalised.  Voxels come out in increasing (ix, iy, iz), the library's order.
* Generalized ICP on clouds with normals (InitializePointCloudForGeneralizedICP): C_i = Rx diag(eps, 1, 1) Rx^T with
  Rx = GetRotationFromE1ToX(n_i) = I + [v]x + [v]x^2 / (1 + c), v = e1 x n_i, c = n_i . e1, n_i as given (not normalised),
  Rx = I when c < -0.99; the registration loop of Open3D's RegistrationICP with the source covariances rotated along
  (R C R^T) and the normal equations sum A^T M^-1 A, sum A^T M^-1 d, M = Cs + Ct, A = [-skew(vs) | I].
"""
import numpy as np
from scipy.spatial import cKDTree

import downsample_ref


def voxel_downsample_normals(xyz, normals, s):
    """(points, normals) of VoxelDownSample(s); every sum is sequential in input order, hence bit-exact
    (tests/downsample_ref.py states it)."""
    pts, nrm, _ = downsample_ref.voxel_downsample(xyz, s, normals)
    return pts, nrm


def _skew(v):
    z = np.zeros(len(v))
    return np.stack([np.stack([z, -v[:, 2], v[:, 1]], 1), np.stack([v[:, 2], z, -v[:, 0]], 1),
                     np.stack([-v[:, 1], v[:, 0], z], 1)], 1)


def gicp_covariances(normals, eps=1e-3):
    """(N, 3, 3) Rx diag(eps, 1, 1) Rx^T of the normals as given"""
    x = np.atleast_2d(np.asarray(normals, dtype=np.float64))
    K = _skew(np.cross([1.0, 0.0, 0.0], x))
    c = x[:, 0]
    fallback = c < -0.99
    f = 1.0 / (1.0 + np.where(fallback, 0.0, c))
    Rx = np.eye(3)[None] + K + (K @ K) * f[:, None, None]
    Rx[fallback] = np.eye(3)
    return Rx @ np.diag([eps, 1.0, 1.0]) @ Rx.transpose(0, 2, 1)


def _rot(rx, ry, rz):
    ca, sa, cb, sb, cg, sg = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    Ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    Rz = np.array([[cg, -sg, 0], [sg, cg, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def icp_generalized(est, gt, est_normals, gt_normals, max_dist, T_init=None, max_iter=30, rel_fitness=1e-6, rel_rmse=1e-6):
    """RegistrationGeneralizedICP with the covariances built from the given normals.
    Returns (T 4x4, fitness, inlier_rmse, n_corr, iterations)."""
    est, gt = np.asarray(est, dtype=np.float64), np.asarray(gt, dtype=np.float64)
    tree = cKDTree(gt)
    T = np.eye(4) if T_init is None else np.array(T_init, dtype=np.float64)
    pcd = est @ T[:3, :3].T + T[:3, 3]
    Cs = T[:3, :3] @ gicp_covariances(est_normals) @ T[:3, :3].T
    Ct = gicp_covariances(gt_normals)

    def evaluate(p):
        d, j = tree.query(p, k=1, workers=-1)
        keep = d * d < max_dist * max_dist
        return keep, j, keep.mean(), (np.sqrt(np.mean(d[keep] ** 2)) if keep.any() else 0.0)
    keep, j, fit, rmse = evaluate(pcd)
    it = 0
    while it < max_iter:
        upd = np.eye(4)
        if keep.any():
            vs = pcd[keep]
            Minv = np.linalg.inv(Ct[j[keep]] + Cs[keep])
            A = np.concatenate([-_skew(vs), np.repeat(np.eye(3)[None], len(vs), 0)], 2)      # (m, 3, 6)
            BA = Minv @ A
            JTJ = np.einsum("mia,mib->ab", A, BA)
            JTr = np.einsum("mia,mi->a", BA, vs - gt[j[keep]])
            x = np.linalg.solve(JTJ, -JTr)
            upd[:3, :3] = _rot(x[0], x[1], x[2])
            upd[:3, 3] = x[3:]
        T = upd @ T
        pcd = pcd @ upd[:3, :3].T + upd[:3, 3]
        Cs = upd[:3, :3] @ Cs @ upd[:3, :3].T
        f0, r0 = fit, rmse
        keep, j, fit, rmse = evaluate(pcd)
        it += 1
        if abs(f0 - fit) < rel_fitness and abs(r0 - rmse) < rel_rmse:
            break
    return T, fit, rmse, int(keep.sum()), it

"""CPU side of the split registration: me_icp_update (the host algebra every rank runs on the reduced block) against numpy
statements of Umeyama and of the 6x6 normal equations, and a gloo replay of the sharded loop — numpy forms every rank's
partial sums over its query shard, gloo all-reduces them, me_icp_update iterates — against the oracle's ICP."""
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import _lib
from cloud_map_evaluation_b200 import dist as mdist

P2P, P2L, GICP = A.ME_ICP_POINT_TO_POINT, A.ME_ICP_POINT_TO_PLANE, A.ME_ICP_GENERALIZED
EPS = 1e-3


@pytest.fixture(scope="module")
def api():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _rot(rx, ry, rz):
    ca, sa, cb, sb, cg, sg = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    Ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    Rz = np.array([[cg, -sg, 0], [sg, cg, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def _p2p_block(p, q, c):
    """[count, sum p, sum q, sum q p^T (row-major), sum d2] about c"""
    pc, qc = p - c, q - c
    d2 = ((p - q) ** 2).sum(1)
    return np.concatenate([[len(p)], pc.sum(0), qc.sum(0), (qc.T @ pc).reshape(9), [d2.sum()]])


def _gicp_cov(n, R=None):
    """Rx diag(eps, 1, 1) Rx^T with Rx = GetRotationFromE1ToX(n) (n as given; Rx = I when n.x < -0.99), rotated by R"""
    x0, x1, x2 = n[:, 0], n[:, 1], n[:, 2]
    f = 1.0 / (1.0 + x0)
    Q = np.empty((len(n), 3, 3))
    Q[:, 0] = np.stack([1.0 - f * (x1 * x1 + x2 * x2), -x1, -x2], 1)
    Q[:, 1] = np.stack([x1, 1.0 - f * x1 * x1, -f * x1 * x2], 1)
    Q[:, 2] = np.stack([x2, -f * x1 * x2, 1.0 - f * x2 * x2], 1)
    Q[x0 < -0.99] = np.eye(3)
    if R is not None:
        Q = R @ Q
    return Q @ np.diag([EPS, 1.0, 1.0]) @ Q.transpose(0, 2, 1)


def _ne_block(vs, vt, nt, method, ns=None, R=None):
    """[count, J^T J upper triangle (row-major), J^T r, sum d2] of point-to-plane / generalized ICP"""
    d = vs - vt
    if method == P2L:
        J = np.concatenate([np.cross(vs, nt), nt], 1)
        r = (d * nt).sum(1)
        JTJ, JTr = J.T @ J, J.T @ r
    else:
        B = np.linalg.inv(_gicp_cov(ns, R) + _gicp_cov(nt))
        Am = np.zeros((len(vs), 3, 6))
        Am[:, 0, 1], Am[:, 0, 2], Am[:, 1, 0] = vs[:, 2], -vs[:, 1], -vs[:, 2]
        Am[:, 1, 2], Am[:, 2, 0], Am[:, 2, 1] = vs[:, 0], vs[:, 1], -vs[:, 0]
        Am[:, :, 3:] = np.eye(3)
        JTJ = np.einsum("nai,nab,nbj->ij", Am, B, Am)
        JTr = np.einsum("nai,nab,nb->i", Am, B, d)
    iu = np.triu_indices(6)
    return np.concatenate([[len(vs)], JTJ[iu], JTr, [(d ** 2).sum()]])


def _solve_update(blk):
    iu = np.triu_indices(6)
    JTJ = np.zeros((6, 6))
    JTJ[iu] = blk[1:22]
    JTJ = JTJ + JTJ.T - np.diag(np.diag(JTJ))
    x = np.linalg.solve(JTJ, -blk[22:28])
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = _rot(*x[:3]), x[3:]
    return T


def test_update_point_to_point_is_umeyama(api):
    rs = np.random.RandomState(0)
    c = np.array([120.0, -40.0, 3.0])
    p = c + rs.randn(5000, 3) * [8.0, 5.0, 1.5]
    Rt, tt = _rot(0.02, -0.01, 0.03), np.array([0.2, -0.1, 0.05])
    q = (p - c) @ Rt.T + c + tt + 0.01 * rs.randn(*p.shape)
    got = api.icp_update(P2P, _p2p_block(p, q, c), c)
    mp_, mq = p.mean(0), q.mean(0)
    U, _, Vt = np.linalg.svd((q - mq).T @ (p - mp_) / len(p))
    S = np.diag([1.0, 1.0, np.sign(np.linalg.det(U) * np.linalg.det(Vt))])
    Rn = U @ S @ Vt
    exp = np.eye(4)
    exp[:3, :3], exp[:3, 3] = Rn, mq - Rn @ mp_
    np.testing.assert_allclose(got, exp, rtol=0, atol=1e-12)


@pytest.mark.parametrize("method", [P2L, GICP])
def test_update_normal_equations(api, method):
    rs = np.random.RandomState(1 + method)
    vs = rs.randn(4000, 3) * [6.0, 6.0, 2.0]
    vt = vs + 0.02 * rs.randn(*vs.shape)
    nt = rs.randn(*vs.shape)
    nt /= np.linalg.norm(nt, axis=1, keepdims=True)
    ns = nt + 0.05 * rs.randn(*vs.shape)
    blk = _ne_block(vs, vt, nt, method, ns, _rot(0.01, 0.02, -0.01))
    np.testing.assert_allclose(api.icp_update(method, blk), _solve_update(blk), rtol=0, atol=1e-12)


def test_update_identity_without_correspondences_or_solution(api):
    assert (api.icp_update(P2P, np.zeros(A.ME_ICP_BLOCK_P2P), np.zeros(3)) == np.eye(4)).all()
    assert (api.icp_update(GICP, np.zeros(A.ME_ICP_BLOCK_NE)) == np.eye(4)).all()
    singular = np.zeros(A.ME_ICP_BLOCK_NE)
    singular[0], singular[22] = 10, 1.0             # count > 0, J^T J = 0: the solve fails
    assert (api.icp_update(P2L, singular) == np.eye(4)).all()
    with pytest.raises(ValueError):
        api.icp_update(P2P, np.zeros(A.ME_ICP_BLOCK_NE), np.zeros(3))


# ---------------------------------------------------------------------------------------------------------------
# gloo replay of the sharded loop
# ---------------------------------------------------------------------------------------------------------------
def _apply(T, x):
    return x @ T[:3, :3].T + T[:3, 3]


def _replay(rank, world, est, gt, method, nrm, R, T0, max_iter=30, rel=1e-6):
    """me_icp_begin .. me_icp_end with numpy partial sums over this rank's query shard and a gloo SUM all-reduce"""
    import torch
    from cloud_map_evaluation_b200 import api
    from oracle import oracle as O
    qb, qe = mdist.shard_range(len(est), rank, world)
    c = 0.5 * (gt.min(0) + gt.max(0))
    T, moved = T0.copy(), _apply(T0, est)

    def block():
        q = moved[qb:qe]
        idx, d2 = O.knn1(q, gt) if len(q) else (np.zeros(0, np.int64), np.zeros(0))
        keep = d2 < R * R
        if method == P2P:
            b = _p2p_block(q[keep], gt[idx[keep]], c) if keep.any() else np.zeros(A.ME_ICP_BLOCK_P2P)
        else:
            b = (_ne_block(q[keep], gt[idx[keep]], nrm[1][idx[keep]], method, nrm[0][qb:qe][keep], T[:3, :3])
                 if keep.any() else np.zeros(A.ME_ICP_BLOCK_NE))
        t = torch.tensor(b, dtype=torch.float64)
        dist.all_reduce(t)
        return t.numpy()

    blk, it, prev, conv = block(), 0, None, 0
    while True:
        n = blk[0]
        fit, rmse = n / len(est), (np.sqrt(blk[-1] / n) if n > 0 else 0.0)
        if prev is not None:
            it += 1
            if abs(prev[0] - fit) < rel and abs(prev[1] - rmse) < rel:
                conv = 1
                break
        if it >= max_iter:
            break
        upd = api.icp_update(method, blk, c)
        T = upd @ T
        moved = _apply(upd, moved)
        prev = (fit, rmse)
        blk = block()
    return T, fit, rmse, int(round(blk[0])), it, conv


def _worker(rank, world, port, out_dir, method):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle import oracle as O
        from test_gpu_icp import _pair
        est, gt = _pair(6000, 8000)
        T0 = np.eye(4)
        T0[:3, 3] = [0.003, 0.0, -0.002]
        R = 0.5
        nrm = (O.estimate_normals_knn(est, 20), O.estimate_normals_knn(gt, 20)) if method == GICP else None
        T, fit, rmse, nc, it, conv = _replay(rank, world, est, gt, method, nrm, R, T0)
        if method == P2P:
            To, fo, ro, nco, ito = O.icp_point_to_point(est, gt, R, T0)
        else:
            # the oracle's generalized ICP estimates the normals itself, as the reference does for clouds without them
            To, fo, ro, nco, ito = O.icp_generalized(est, gt, R, T0)
        assert it == ito and nc == nco, (it, ito, nc, nco)
        np.testing.assert_allclose(T, To, rtol=0, atol=1e-9)
        np.testing.assert_allclose([fit, rmse], [fo, ro], rtol=1e-9)
        assert 2 <= it <= 30
        open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("method", [P2P, GICP])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_icp_replay_gloo(api, world, method, tmp_path):
    from oracle import oracle as O
    O.build()
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_worker, args=(world, port, str(tmp_path), method), nprocs=world, join=True)
    assert all(os.path.exists(tmp_path / f"ok{r}") for r in range(world))

"""Registration kernels against exact arithmetic (tests/exact_reg.py): knn_normals_kernel on every point of small scenes
and a fixed sample of large ones (dense and sparse cell table, and the slices of world 2 and 3), the device ICP blocks of
icp_accum_kernel / icp_ne_accum_kernel for all three methods (one rank, and the sum of 2, 3 and 8 ranks), and a
point-to-point registration of a tilted near-planar pair end to end."""
import numpy as np
import pytest

import exact_reg as X
from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import dist as mdist

from test_exact_reg import FAR, RZ90, lattice, near_planar_pair, normal_scenes, rot

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
P2P, P2L, GICP = A.ME_ICP_POINT_TO_POINT, A.ME_ICP_POINT_TO_PLANE, A.ME_ICP_GENERALIZED
SPARSE = 1            # max_grid_cells: a budget of one cell forces the sparse cell table


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _view(ptr, n):
    """a torch view of n fp64 values of device memory owned by the library"""
    import torch
    return torch.as_tensor(mdist._DeviceBlock(ptr, n), device="cuda:0")


# ---------------------------------------------------------------------------------------------------------------
# k-NN normals
# ---------------------------------------------------------------------------------------------------------------
def _large_scenes():
    rs = np.random.RandomState(11)
    out = {}
    for noise in (1e-3, 1e-5, 1e-7):
        for far in (False, True):
            uv = rs.rand(40_000, 2) * 20.0
            p = np.stack([uv[:, 0], uv[:, 1], noise * rs.randn(40_000)], 1) @ rot(0.5, -0.2, 0.9).T
            out[f"big_plane_{noise:g}{'_far' if far else ''}"] = p + (FAR if far else 0.0)
    # isolated points tens of metres from a small cluster: the coarse phase, and c2 - c1 c1^T about a far query
    out["big_outliers"] = np.concatenate([rs.randn(30_000, 3) * [2.0, 2.0, 0.01], rs.rand(300, 3) * 80.0 - 40.0])
    out["big_cube_lattice"] = lattice(30, (0.25, 0.25, 0.25), seed=5)
    return out


SMALL = normal_scenes()
LARGE = _large_scenes()
SAMPLE = 2000
_ROWS = {}


def _rows(name):
    if name not in _ROWS:
        pts = SMALL[name] if name in SMALL else LARGE[name]
        q = None
        if name in LARGE:
            q = np.random.RandomState(0).choice(len(pts), SAMPLE, replace=False)
            if name == "big_outliers":
                q = np.union1d(q, np.arange(len(pts) - 300, len(pts)))
        _ROWS[name] = X.normals_exact(pts, q)
    return _ROWS[name]


def _device_normals(api, pts, max_grid_cells=0):
    with api.MapEvalB200(max_grid_cells=max_grid_cells) as c:
        c.set_cloud(EST, pts)
        c.set_cloud(GT, pts[:8])
        return c.estimate_normals(EST, 20)


def _check_all(name, rows, got):
    bad, signed = [], 0
    for row in rows:
        r = X.check_normal(row, got[row["q"]])
        signed += r["sign_checked"]
        if not r["ok"]:
            bad.append((row["q"], r["why"]))
    assert not bad, (name, len(bad), bad[:5])
    return signed


@pytest.mark.parametrize("table", ["dense", "sparse"])
@pytest.mark.parametrize("name", sorted(SMALL) + sorted(LARGE))
def test_normals_within_exact_bounds(api, name, table):
    pts = SMALL[name] if name in SMALL else LARGE[name]
    got = _device_normals(api, pts, SPARSE if table == "sparse" else 0)
    signed = _check_all(name, _rows(name), got)
    if "plane" in name or name == "strip":
        assert signed >= 0.9 * len(_rows(name))            # the sign is pinned nearly everywhere on a surface
    if name == "duplicates":
        assert (got[:30] == [0.0, 0.0, 1.0]).all()         # all 20 neighbours identical: the zero covariance


def test_normals_small_counts(api):
    """n < 3: the identity covariance gives (0, 0, 1); 3 <= n < 20: k = n, every point the same neighbourhood"""
    rs = np.random.RandomState(2)
    for n in (1, 2):
        assert (_device_normals(api, rs.rand(n, 3)) == [0.0, 0.0, 1.0]).all()
    for n in (3, 7, 19):
        pts = rs.rand(n, 3) @ np.diag([1.0, 0.7, 0.05])
        got = _device_normals(api, pts)
        _check_all(f"n{n}", X.normals_exact(pts), got)


@pytest.mark.parametrize("world", [2, 3])
def test_normal_slices_after_all_gather(api, world):
    """icp_normals_slice on `world` contexts, gathered: bit-identical to one estimate, and within the exact bounds"""
    import torch
    pts = LARGE["big_outliers"]
    ctxs = [api.MapEvalB200(rank=r, world=world) for r in range(world)]
    try:
        for c in ctxs:
            c.set_cloud(EST, pts)
            c.set_cloud(GT, pts[:100])
            c.icp_begin(0.5, None, method=GICP)
        sl = [c.icp_normals_slice(EST) for c in ctxs]
        s = sl[0][1]
        for c in ctxs:
            c.synchronize()
        views = [_view(p, world * s * 3) for p, _, _ in sl]
        full = torch.cat([views[r][r * s * 3:(r + 1) * s * 3] for r in range(world)])
        torch.cuda.synchronize()
        got = full[:3 * len(pts)].cpu().numpy().reshape(-1, 3)
    finally:
        for c in ctxs:
            c.close()
    assert got.tobytes() == _device_normals(api, pts).tobytes()
    _check_all(f"world{world}", _rows("big_outliers"), got)


# ---------------------------------------------------------------------------------------------------------------
# ICP blocks
# ---------------------------------------------------------------------------------------------------------------
R_MAX = 0.625          # R^2 = 0.390625 exactly: the pairs placed at offset (0.375, 0.5, 0) lie on it


def block_scene(far, T0, n=1500, seed=9):
    """(est, gt, est normals, gt normals): a bumpy tilted surface and its noisy copy, float32-quantised so that the
    moves of T0 (a signed permutation and a dyadic translation) are exact, est taken back by T0^-1 so that T0 moves it
    onto the surface; est normals not unit length, some of them near -e1; plus 8 pairs apart from the surface whose
    distance is exactly R_MAX (dropped) or just below it (kept)"""
    rs = np.random.RandomState(seed)
    uv = rs.rand(n, 2) * 8.0 - 4.0
    base = np.stack([uv[:, 0], uv[:, 1], 0.3 * np.sin(uv[:, 0]) * np.cos(0.5 * uv[:, 1])], 1) @ rot(0.3, -0.2, 0.5).T
    nt = rs.randn(n, 3) * 0.1 + [0.2, 0.3, 1.0]
    nt /= np.linalg.norm(nt, axis=1, keepdims=True)
    est = base + 0.01 * rs.randn(n, 3)
    ne = (nt + 0.05 * rs.randn(n, 3)) * (1 + 0.2 * rs.rand(n, 1))
    ne[::7] = [-0.995, 0.05, 0.08]
    on = np.array([[20.0, 20.0, 0.0], [20.0, 22.0, 0.0], [22.0, 20.0, 0.0], [22.0, 22.0, 0.0]])
    gt_on = np.concatenate([on, on + [0.0, 0.0, 2.0]])
    est_on = np.concatenate([on + [0.375, 0.5, 0.0], on + [0.375, 0.4375, 2.0]])      # d2 = R^2, d2 < R^2
    est = np.concatenate([est, est_on])
    gt = np.concatenate([base, gt_on])
    ne = np.concatenate([ne, np.tile([0.0, 0.0, 1.0], (8, 1))])
    nt = np.concatenate([nt, np.tile([0.0, 0.0, 1.0], (8, 1))])
    sh = FAR if far else 0.0
    f32 = lambda a: a.astype(np.float32).astype(np.float64)
    return (f32(est + sh) - T0[:3, 3]) @ T0[:3, :3], f32(gt + sh), ne, nt


_BLOCKS = {}
T_INITS = {"identity": np.eye(4), "rz90": np.block([[RZ90, np.array([[0.5], [-0.25], [0.0]])], [np.zeros((1, 3)), np.ones((1, 1))]])}


def _device_blocks(api, est, gt, ne, nt, method, T0, world):
    """icp_begin -> icp_block on `world` contexts: (per-rank blocks, the moved est cloud)"""
    ctxs = [api.MapEvalB200(rank=r, world=world) for r in range(world)]
    try:
        blocks = []
        for c in ctxs:
            c.set_cloud(EST, est)
            c.set_cloud(GT, gt)
            if method != P2P:
                c.set_normals(GT, nt)
            if method == GICP:
                c.set_normals(EST, ne)
            c.icp_begin(R_MAX, T0, method=method)
            ptr, n_sum = c.icp_block()
            c.synchronize()
            blocks.append(_view(ptr, n_sum).cpu().numpy().copy())
        moved = ctxs[0].get_cloud(EST)
    finally:
        for c in ctxs:
            c.close()
    return blocks, moved


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("t_init", sorted(T_INITS))
@pytest.mark.parametrize("far", [False, True], ids=["origin", "far"])
@pytest.mark.parametrize("method", [P2P, P2L, GICP], ids=["p2p", "p2l", "gicp"])
def test_block_within_exact_bound(api, method, far, t_init, world):
    if world > 1 and t_init != "identity":
        pytest.skip("ranks are checked at T_init = I")
    T0 = T_INITS[t_init]
    est, gt, ne, nt = block_scene(far, T0)
    blocks, moved = _device_blocks(api, est, gt, ne, nt, method, T0, world)
    # both initial transformations are exact on these points: the moved cloud is known exactly
    np.testing.assert_array_equal(moved, est @ T0[:3, :3].T + T0[:3, 3])
    key = (method, far, t_init)
    if key not in _BLOCKS:
        si, ti, d2 = X.kept_pairs(moved, gt, R_MAX)
        kept = set(si.tolist())
        assert not kept & set(range(len(est) - 8, len(est) - 4))          # d2 = R^2: dropped
        assert set(range(len(est) - 4, len(est))) <= kept                  # d2 < R^2: kept
        if method == P2P:
            _BLOCKS[key] = (len(si),) + X.p2p_block_exact(moved[si], gt[ti], d2, 0.5 * (gt.min(0) + gt.max(0)))
        else:
            _BLOCKS[key] = (len(si),) + X.ne_block_exact(moved[si], gt[ti], nt[ti], d2, method, ne[si], T0[:3, :3])
    m, blk, bound = _BLOCKS[key]
    exp = X.block_floats(blk)
    got = np.sum(blocks, 0)
    assert got[0] == m                                                      # the count is exact
    err = np.abs(got - exp)
    assert (err <= bound).all(), (np.flatnonzero(err > bound), (err / np.maximum(bound, 1e-300)).max())


# ---------------------------------------------------------------------------------------------------------------
# end to end: point-to-point on a tilted near-planar pair
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h", [0.1, 0.01])
def test_point_to_point_near_planar_end_to_end(api, h):
    from oracle import oracle as O
    p, q, c = near_planar_pair(h, n=20_000, seed=1)
    est, gt = p, q + 0.002 * np.random.RandomState(2).randn(*q.shape)      # a residual, so that rmse is not rounding
    T0 = np.eye(4)
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, est)
        ctx.set_cloud(GT, gt)
        T, reg = ctx.performICPRegistration(1.0, T0)
        aligned = ctx.get_cloud(EST)
        prm = A.make_nn_params([0.02, 0.05, 0.1, 0.2, 0.3], 1.0, cutoff_mode=A.ME_CUTOFF_DIST_LT_R,
                               pairing=A.ME_PAIRING_GEOMETRIC)
        nn = ctx.calculateMetricsWithInitialMatrix(prm)
    R = T[:3, :3]
    assert np.abs(R.T @ R - np.eye(3)).max() <= 1e-13 and abs(np.linalg.det(R) - 1) <= 1e-13
    To, fit, rmse, nc, it = O.icp_point_to_point(est, gt, 1.0, T0)
    assert (reg.n_corr, reg.iterations) == (nc, it)
    np.testing.assert_allclose(T, To, atol=1e-10)
    np.testing.assert_allclose([reg.fitness, reg.inlier_rmse], [fit, rmse], rtol=1e-9)
    onn = O.eval_nn(O.transform(est, To), gt, prm)
    assert list(nn.est_to_gt.n_inlier) == list(onn.est_to_gt.n_inlier)
    assert list(nn.gt_to_est.n_inlier) == list(onn.gt_to_est.n_inlier)
    np.testing.assert_allclose(aligned, O.transform(est, To), atol=1e-9)

"""Registration split at its collective (me_icp_begin / _normals_slice / _block / _step / _end) on 1 to 8 ranks.  One context
per rank on ONE device stands in for the ranks; the collectives of the job (the in-place all-gather of the k-NN normal
slices, the SUM all-reduce of the ICP block per iteration) are done here with torch on that device.  The sharded loop must
reproduce me_icp: equal iterations, convergence and correspondence counts, T to 1e-10, normals byte for byte."""
import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import dist as mdist

from test_gpu_icp import _pair

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
P2P, P2L, GICP = A.ME_ICP_POINT_TO_POINT, A.ME_ICP_POINT_TO_PLANE, A.ME_ICP_GENERALIZED
R = 0.5
T0 = np.eye(4)
T0[:3, 3] = [0.003, 0.0, -0.002]


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


@pytest.fixture(scope="module")
def scene():
    return _pair(100_000, 120_000)


@pytest.fixture(scope="module")
def normals(scene):
    from oracle import oracle as O
    est, gt = scene
    return O.estimate_normals_knn(est, 20), O.estimate_normals_knn(gt, 20)


def _view(ptr, n):
    import torch
    return torch.as_tensor(mdist._DeviceBlock(ptr, n), device="cuda:0")


def _setup(c, est, gt, nrm):
    c.set_cloud(EST, est)
    c.set_cloud(GT, gt)
    if nrm is not None:
        for which, n in zip((EST, GT), nrm):
            if n is not None:
                c.set_normals(which, n)


def _reference(api, est, gt, method, nrm=None, metric=None):
    """me_icp at world = 1 (and the metric pass after it)"""
    with api.MapEvalB200() as c:
        _setup(c, est, gt, nrm)
        T, reg = c.performICPRegistration(R, T0, method=method)
        out = dict(T=T, reg=reg, aligned=c.get_cloud(EST))
        if metric is not None:
            out["acc"] = c.eval_nn_accum(metric)
    return out


def _sharded(api, est, gt, method, world, nrm=None, metric=None, T_init=T0):
    """the split loop on `world` contexts; the collectives with torch"""
    import torch
    ctxs = [api.MapEvalB200(rank=r, world=world) for r in range(world)]
    out = {"gathered": {}}
    try:
        for c in ctxs:
            _setup(c, est, gt, nrm)
            c.icp_begin(R, T_init, method=method)
        for which, n in ((EST, len(est)), (GT, len(gt))):
            sl = [c.icp_normals_slice(which) for c in ctxs]
            assert len({(s, p) for _, s, p in sl}) == 1
            if not sl[0][2]:
                continue
            s = sl[0][1]
            assert s == -(-n // world)
            for c in ctxs:
                c.synchronize()
            views = [_view(p, world * s * 3) for p, _, _ in sl]
            full = torch.cat([views[r][r * s * 3:(r + 1) * s * 3] for r in range(world)])
            for v in views:
                v.copy_(full)
            torch.cuda.synchronize()
            out["gathered"][which] = [v[:3 * n].cpu().numpy().reshape(n, 3) for v in views]
        blocks = []
        for c in ctxs:
            ptr, n_sum = c.icp_block()
            assert n_sum == (A.ME_ICP_BLOCK_P2P if method == P2P else A.ME_ICP_BLOCK_NE)
            blocks.append(_view(ptr, n_sum))
        done, steps = False, 0
        while not done:
            for c in ctxs:
                c.synchronize()
            red = torch.stack(blocks).sum(0)
            for b in blocks:
                b.copy_(red)
            torch.cuda.synchronize()
            dn = {c.icp_step() for c in ctxs}
            assert len(dn) == 1
            done = dn.pop()
            steps += 1
            assert steps <= 40
        res = [c.icp_end() for c in ctxs]
        for T, _ in res[1:]:
            np.testing.assert_array_equal(T, res[0][0])            # every rank applied the same updates
        out["T"], out["reg"] = res[0]
        out["aligned"] = [c.get_cloud(EST) for c in ctxs]
        if metric is not None:
            blocks = []
            for c in ctxs:
                c.accum_reset()
                c.eval_nn_accum_device(metric)
                c.synchronize()
                ptr, n_sum, n_max = c.accum_block()
                blocks.append(_view(ptr, n_sum + n_max))
            red = torch.cat([torch.stack(blocks)[:, :n_sum].sum(0), torch.stack(blocks)[:, n_sum:].max(0).values])
            blocks[0].copy_(red)
            torch.cuda.synchronize()
            out["acc"] = ctxs[0].accum_fetch((False, False))[0]
    finally:
        for c in ctxs:
            c.close()
    return out


def _same(got, ref, tol=1e-10):
    g, r = got["reg"], ref["reg"]
    assert (g.iterations, g.converged, g.n_corr) == (r.iterations, r.converged, r.n_corr)
    np.testing.assert_allclose(got["T"], ref["T"], rtol=0, atol=tol)
    np.testing.assert_allclose([g.fitness, g.inlier_rmse], [r.fitness, r.inlier_rmse], rtol=1e-9)


VARIANTS = ["p2p", "p2l", "gicp_estimated", "gicp_given"]


def _case(variant, normals):
    n_est, n_gt = normals
    return {"p2p": (P2P, None), "p2l": (P2L, (None, n_gt)), "gicp_estimated": (GICP, None),
            "gicp_given": (GICP, (n_est, n_gt))}[variant]


@pytest.mark.parametrize("variant", VARIANTS)
def test_split_world1_matches_me_icp(api, scene, normals, variant):
    est, gt = scene
    method, nrm = _case(variant, normals)
    ref = _reference(api, est, gt, method, nrm)
    got = _sharded(api, est, gt, method, 1, nrm)
    _same(got, ref)
    assert got["gathered"] == {}                                     # world 1: nothing to gather
    np.testing.assert_allclose(got["aligned"][0], ref["aligned"], rtol=0, atol=1e-9)
    assert 2 <= ref["reg"].iterations <= 30


@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("variant", VARIANTS)
def test_sharded_matches_world1(api, scene, normals, variant, world):
    est, gt = scene
    method, nrm = _case(variant, normals)
    ref = _reference(api, est, gt, method, nrm)
    got = _sharded(api, est, gt, method, world, nrm)
    _same(got, ref)
    for a in got["aligned"]:
        np.testing.assert_allclose(a, ref["aligned"], rtol=0, atol=1e-9)


def test_sharded_far_from_the_origin(api):
    """1.5 km from the origin (the tolerances of test_gpu_icp.test_generalized_icp there): the 6x6 system is ill-conditioned,
    the fixed point is the same, the path to it may differ in the last digits"""
    est, gt = _pair(origin=(1500.0, -800.0, 40.0))
    ref = _reference(api, est, gt, GICP)
    got = _sharded(api, est, gt, GICP, 2)
    g, r = got["reg"], ref["reg"]
    assert abs(g.iterations - r.iterations) <= 1 and abs(g.n_corr - r.n_corr) <= 2
    np.testing.assert_allclose(got["T"][:3, :3], ref["T"][:3, :3], atol=1e-7)
    assert np.abs(got["aligned"][0] - ref["aligned"]).max() < 5e-6
    np.testing.assert_allclose([g.fitness, g.inlier_rmse], [r.fitness, r.inlier_rmse], rtol=1e-5)


def test_sharded_permuted_input(api, scene):
    """caller order is spatially random: the normal slices and the query ranges cut the cloud differently"""
    est, gt = scene
    rs = np.random.RandomState(3)
    pe, pg = rs.permutation(len(est)), rs.permutation(len(gt))
    ref = _reference(api, est, gt, GICP)
    got = _sharded(api, est[pe], gt[pg], GICP, 3)
    _same(got, ref, tol=1e-9)
    np.testing.assert_allclose(got["aligned"][1], ref["aligned"][pe], rtol=0, atol=1e-9)


@pytest.mark.parametrize("world", [2, 3, 8])
def test_gathered_normals_are_the_world1_normals(api, scene, world):
    est, gt = scene
    exp = {}
    with api.MapEvalB200() as c:
        _setup(c, est, gt, None)
        exp[EST] = c.estimate_normals(EST, 20)
        exp[GT] = c.estimate_normals(GT, 20)
    got = _sharded(api, est, gt, GICP, world)
    assert set(got["gathered"]) == {EST, GT}
    for which in (EST, GT):
        for r, g in enumerate(got["gathered"][which]):
            assert g.tobytes() == exp[which].tobytes(), (which, r)


def test_metric_pass_after_sharded_icp(api, scene):
    """after me_icp_end every rank holds the aligned cloud: the sharded metric pass counts the same inliers as the world = 1
    pass after me_icp"""
    est, gt = scene
    p = A.make_nn_params([0.02, 0.05, 0.1, 0.2, 0.3], R, cutoff_mode=A.ME_CUTOFF_DIST_LT_R, pairing=A.ME_PAIRING_GEOMETRIC,
                         directions=1)
    ref = _reference(api, est, gt, GICP, metric=p)
    got = _sharded(api, est, gt, GICP, 3, metric=p)
    e_ref, e_got = ref["acc"][0], got["acc"]
    assert list(e_got.n_inlier) == list(e_ref.n_inlier) and e_got.n_corr == e_ref.n_corr
    assert e_got.n_query == e_ref.n_query == len(est)


def test_call_order_errors(api, scene):
    est, gt = scene
    with api.MapEvalB200() as c:
        _setup(c, est, gt, None)
        with pytest.raises(api.MapEvalError, match="me_icp_step before me_icp_begin"):
            c.icp_step()
        with pytest.raises(api.MapEvalError, match="me_icp_end without me_icp_begin"):
            c.icp_end()
        with pytest.raises(api.MapEvalError, match="me_icp_block before me_icp_begin"):
            c.icp_block()
        # generalized ICP without normals: the first step (or block) before the normals were estimated
        c.icp_begin(R, T0, method=GICP)
        with pytest.raises(api.MapEvalError, match="still pending"):
            c.icp_step()
        # the failure closed the registration: the cloud is as handed in, and a new one can begin
        np.testing.assert_array_equal(c.get_cloud(EST), est)
        with pytest.raises(api.MapEvalError, match="before me_icp_begin"):
            c.icp_step()
        c.icp_begin(R, T0, method=P2P)
        with pytest.raises(api.MapEvalError, match="before the first me_icp_block"):
            c.icp_step()
        np.testing.assert_array_equal(c.get_cloud(EST), est)
        c.icp_begin(R, T0, method=GICP)
        c.icp_normals_slice(EST)
        with pytest.raises(api.MapEvalError, match="still pending"):
            c.icp_block()
        c.icp_begin(R, T0, method=P2P)
        c.icp_block()
        while not c.icp_step():
            pass
        T, reg = c.icp_end()
        assert reg.iterations >= 2
        with pytest.raises(api.MapEvalError, match="me_icp_end without me_icp_begin"):
            c.icp_end()


def test_slab_layout_is_refused(api, scene):
    """registration runs on the replicated layout: a context of a sharded job with ME_LAYOUT_SLAB requested refuses it, and
    takes it once the layout is switched back"""
    est, gt = scene
    with api.MapEvalB200(rank=0, world=2) as c:
        _setup(c, est, gt, None)
        c.set_layout(A.ME_LAYOUT_SLAB)
        with pytest.raises(api.MapEvalError, match="replicated layout"):
            c.icp_begin(R, T0, method=P2P)
        c.set_layout(A.ME_LAYOUT_REPLICATED)
        c.icp_begin(R, T0, method=P2P)
        with pytest.raises(api.MapEvalError, match="before the first me_icp_step"):
            c.icp_end()


@pytest.mark.parametrize("method", [P2P, P2L, GICP])
def test_no_correspondences_world3(api, method):
    """clouds 100 m apart with R = 0.5 (test_gpu_icp.test_no_correspondences at world 3): identity, one iteration, converged"""
    est, gt = _pair(20_000, 20_000)
    est = est + np.array([100.0, 0.0, 0.0])
    nrm = None
    if method == P2L:
        with api.MapEvalB200() as c:
            _setup(c, est, gt, None)
            nrm = (None, c.estimate_normals(GT, 20))
    got = _sharded(api, est, gt, method, 3, nrm, T_init=None)
    reg = got["reg"]
    assert (reg.n_corr, reg.iterations, reg.converged) == (0, 1, 1) and reg.fitness == 0.0
    np.testing.assert_array_equal(got["T"], np.eye(4))

"""Drift per region on the GPU (me_drift*): one point-to-point ICP per region of the estimated cloud.

- world 1, bit for bit against the numpy statement (drift_ref.py): the block of every iteration read through the split
  loop, and the rows' T, counts, fitness, rmse, iterations and status; at s = 0.1, on region faces, at negative coordinates,
  at max_iteration 0 and 1, with regions of fewer than 3 pairs and with regions that reach the limit;
- one region is me_icp point-to-point: the same iterations, status and n_corr; T, fitness and rmse to 1e-9;
- a known rigid motion per room of a 1 M-point indoor scene is recovered to 2 mm and 0.02 degrees;
- worlds 2, 3 and 8 on cuda:0: counts, iterations and status as world 1, T to 1e-9;
- the contract: determinism, the estimated cloud (points and normals) unchanged after the loop and after every refusal or
  failure, stale NN records, and every refusal."""
import numpy as np
import pytest

import drift_ref as D
from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import dist as mdist
from cloud_map_evaluation_b200 import synth

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
EXACT = ("n_est", "n_corr_before", "fitness_before", "rmse_before", "n_corr", "fitness", "rmse", "T", "iterations", "status",
         "index", "min", "max")
CLOSE = ("centroid", "shift", "shift_norm", "angle")


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    try:
        with _api.MapEvalB200(device=0):
            pass
    except _api.MapEvalError as e:
        pytest.skip(f"no sm_90 device: {e}")
    return _api


def _ctx(api, est, gt, **kw):
    c = api.MapEvalB200(**kw)
    c.set_cloud(EST, est)
    c.set_cloud(GT, gt)
    return c


def scene(n, seed, offset=(0.2, 0.3, 0.1), side=2.0, faces=0.0, s=None):
    """gt uniform in a box; est = gt moved by one small rigid motion per half of the box along x, plus noise.  faces: share
    of est coordinates put exactly on a region face k * s"""
    rng = np.random.RandomState(seed)
    gt = synth.uniform_box(n, side, seed) + np.asarray(offset)
    est = gt + 2e-3 * rng.randn(n, 3)
    half = est[:, 0] < gt[:, 0].mean()
    est[half] = D.apply(D.rigid(0.6, (0.2, 1, 0.4), (0.01, -0.004, 0.006)), est[half], est[half].mean(0))
    est[~half] = D.apply(D.rigid(0.4, (1, 0.1, 0.2), (-0.006, 0.008, 0.002)), est[~half], est[~half].mean(0))
    if faces:
        m = rng.rand(*est.shape) < faces
        est[m] = np.round(est[m] / s) * s
    return np.ascontiguousarray(est), gt


def loop(ctx, s, R, **kw):
    """the split loop at world 1: (rows, the block of every iteration)"""
    import torch
    n = ctx.drift_begin(s, R, **kw)
    blocks = []
    done = False
    while not done:
        ptr, n_sum = ctx.drift_block()
        assert n_sum == A.ME_ICP_BLOCK_P2P * n
        ctx.synchronize()
        blocks.append(torch.as_tensor(mdist._DeviceBlock(ptr, n_sum), device="cuda:0").cpu().numpy().reshape(n, -1).copy())
        done = ctx.drift_step()
    return ctx.drift_end(n), blocks


def check_rows(got, ref, exact=True):
    for k in EXACT:
        g, r = np.asarray(got[k]), np.asarray(ref[k])
        assert g.shape == r.shape, k
        if exact:
            assert g.tobytes() == r.astype(g.dtype).tobytes(), (k, np.flatnonzero((g != r).reshape(len(g), -1).any(1))[:5])
    for k in CLOSE:
        np.testing.assert_allclose(got[k], ref[k], rtol=0, atol=1e-12, err_msg=k)


CASES = [
    dict(n=30000, seed=1, s=0.5, R=0.05),
    dict(n=20000, seed=2, s=0.1, R=0.05),                                              # many regions, many too few
    dict(n=40000, seed=3, s=0.5, R=0.05, offset=(-1.3, -0.7, -2.1)),                   # negative coordinates
    dict(n=25000, seed=4, s=0.25, R=0.05, faces=0.05),                                 # points on region faces
    dict(n=20000, seed=5, s=0.5, R=0.05, max_iteration=0),
    dict(n=20000, seed=6, s=0.5, R=0.05, max_iteration=1),
    dict(n=30000, seed=7, s=0.5, R=0.05, max_iteration=4, relative_fitness=0.0, relative_rmse=0.0),   # every region at the limit
    dict(n=50000, seed=8, s=1.0, R=0.05),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"s{c['s']}-seed{c['seed']}")
def test_world_one_equals_the_statement_bit_for_bit(api, case):
    c = dict(case)
    n, seed, s, R = c.pop("n"), c.pop("seed"), c.pop("s"), c.pop("R")
    kw = {k: c.pop(k) for k in ("max_iteration", "relative_fitness", "relative_rmse") if k in c}
    est, gt = scene(n, seed, s=s, **c)
    with _ctx(api, est, gt) as ctx:
        got, blocks = loop(ctx, s, R, **kw)
        assert ctx.get_cloud(EST).tobytes() == est.tobytes()
    ref, ref_blocks = D.drift(est, gt, s, R, **kw)
    assert len(blocks) == len(ref_blocks)
    for i, (b, r) in enumerate(zip(blocks, ref_blocks)):
        assert b.tobytes() == r.tobytes(), f"block of iteration {i}"
    check_rows(got, ref)
    st = set(got["status"].tolist())
    if kw.get("max_iteration") == 0:
        assert st == {A.ME_DRIFT_ITERATION_LIMIT} and not got["iterations"].any()
    if s == 0.1:
        assert A.ME_DRIFT_TOO_FEW in st
    if kw.get("relative_fitness") == 0.0:
        assert A.ME_DRIFT_ITERATION_LIMIT in st


def test_one_region_is_me_icp_point_to_point(api):
    est, gt, cfg = synth.make_pair("C1", scale=0.3)
    est = D.apply(D.rigid(0.5, (0.3, 1, 0.2), (0.03, -0.02, 0.01)), est, est.mean(0))
    lift = 1.0 - np.minimum(est.min(0), gt.min(0))          # one region needs every coordinate >= 0
    est, gt = est + lift, gt + lift
    R = 0.5
    s = 4.0 * float(np.abs(np.concatenate([est, gt])).max()) + 1.0
    with _ctx(api, est, gt) as ctx:
        rows = ctx.region_drift(s, R)
    assert len(rows["n_est"]) == 1 and rows["n_est"][0] == len(est)
    with _ctx(api, est, gt) as ctx:
        T, res = ctx.performICPRegistration(R, method=A.ME_ICP_POINT_TO_POINT)
    assert rows["iterations"][0] == res.iterations and rows["n_corr"][0] == res.n_corr
    assert rows["status"][0] == (A.ME_DRIFT_CONVERGED if res.converged else A.ME_DRIFT_ITERATION_LIMIT)
    np.testing.assert_allclose(rows["T"][0], T, rtol=0, atol=1e-9)
    np.testing.assert_allclose([rows["fitness"][0], rows["rmse"][0]], [res.fitness, res.inlier_rmse], rtol=0, atol=1e-9)


def test_recovers_each_rooms_motion(api):
    est, gt, motions = D.indoor(1_000_000, 10, 21)
    with _ctx(api, est, gt) as ctx:
        rows = ctx.region_drift(8.0, 0.2)
    assert len(rows["n_est"]) == len(motions) == 100
    for r, key in enumerate(rows["index"]):
        M = motions[tuple(key)]
        Tinv = np.linalg.inv(rows["T"][r])
        assert np.abs(Tinv[:3, 3] - M[:3, 3]).max() < 2e-3, key
        assert D.angle_of(Tinv[:3, :3] @ M[:3, :3].T) < 0.02, key
        assert rows["rmse"][r] < rows["rmse_before"][r], key


def _sharded(api, est, gt, s, R, world):
    """`world` contexts on cuda:0, the blocks SUM-reduced with torch every iteration"""
    import torch
    ctxs = [_ctx(api, est, gt, rank=r, world=world) for r in range(world)]
    try:
        ns = [c.drift_begin(s, R) for c in ctxs]
        assert len(set(ns)) == 1
        done = [False] * world
        while not all(done):
            ts = []
            for c in ctxs:
                ptr, n_sum = c.drift_block()
                c.synchronize()
                ts.append(torch.as_tensor(mdist._DeviceBlock(ptr, n_sum), device="cuda:0"))
            total = torch.stack(ts).sum(0)
            for t in ts:
                t.copy_(total)
            torch.cuda.synchronize()
            done = [c.drift_step() for c in ctxs]
            assert len(set(done)) == 1
        res = [c.drift_end(ns[0]) for c in ctxs]
        for r in res[1:]:
            check_rows(r, res[0])
        return res[0]
    finally:
        for c in ctxs:
            c.close()


def test_sharded_equals_world_one(api):
    for n, seed, s in ((40000, 11, 0.5), (30000, 12, 0.25)):
        est, gt = scene(n, seed)
        with _ctx(api, est, gt) as ctx:
            ref = ctx.region_drift(s, 0.05)
        for world in (2, 3, 8):
            got = _sharded(api, est, gt, s, 0.05, world)
            for k in ("index", "n_est", "n_corr_before", "n_corr", "iterations", "status"):
                assert np.array_equal(got[k], ref[k]), (world, k)
            np.testing.assert_allclose(got["T"], ref["T"], rtol=0, atol=1e-9)


def _refused(api, fn, pattern):
    with pytest.raises(api.MapEvalError, match=pattern):
        fn()


def test_contract(api):
    est, gt = scene(30000, 31)
    nrm = np.random.RandomState(31).randn(len(est), 3)
    with _ctx(api, est, gt) as ctx:
        ctx.set_normals(EST, nrm)

        def intact():
            assert ctx.get_cloud(EST).tobytes() == est.tobytes()
            assert ctx.get_normals(EST).tobytes() == nrm.tobytes()

        a = ctx.region_drift(0.5, 0.05)
        intact()
        b = ctx.region_drift(0.5, 0.05)
        check_rows(a, b)
        for k in CLOSE:
            assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes()
        # the records of an NN evaluation are stale after the call
        ctx.calculateMetricsWithInitialMatrix(A.make_nn_params([0.1] * 5, 0.05))
        ctx.region_drift(0.5, 0.05)
        _refused(api, lambda: ctx.accuracy_curve([0.1, 0.2]), "no current NN records")
        # bad arguments
        for s, R, it in ((0.0, 0.05, 5), (np.inf, 0.05, 5), (np.nan, 0.05, 5), (-1.0, 0.05, 5), (0.5, 0.0, 5), (0.5, np.inf, 5),
                         (0.5, 0.05, -1)):
            _refused(api, lambda: ctx.drift_begin(s, R, max_iteration=it), "me_drift_begin")
            intact()
        # a begin refused for its arguments leaves an open loop running: the same rows as an undisturbed loop
        n = ctx.drift_begin(0.5, 0.05)
        _refused(api, lambda: ctx.drift_begin(-1.0, 0.05), "region_size must be finite")
        while not ctx.drift_step():
            pass
        check_rows(ctx.drift_end(n), a)
        intact()
        # the index range and the region count
        _refused(api, lambda: ctx.drift_begin(1e-7, 0.05), r"outside \|index\| < 2\^20")
        intact()
        # calls out of order
        _refused(api, lambda: ctx.drift_step(), "before me_drift_begin")
        _refused(api, lambda: ctx.drift_block(), "before me_drift_begin")
        _refused(api, lambda: ctx.drift_end(1), "before me_drift_begin")
        n = ctx.drift_begin(0.5, 0.05)
        _refused(api, lambda: ctx.drift_end(n), "before the loop is done")
        intact()
        n = ctx.drift_begin(0.5, 0.05)
        _refused(api, lambda: ctx.drift_begin(0.5, 0.05), "while a drift loop is open")
        intact()
        n = ctx.drift_begin(0.5, 0.05)
        _refused(api, lambda: ctx.icp_begin(0.05, method=A.ME_ICP_POINT_TO_POINT), "while a drift loop is open")
        ctx.drift_step()
        _refused(api, lambda: ctx.drift_begin(0.5, 0.05), "while a drift loop is open")
        intact()
        # a capacity below the region count fails and restores
        n = ctx.drift_begin(0.5, 0.05)
        while not ctx.drift_step():
            pass
        import ctypes as C
        rows = np.zeros(max(n, 1), [("x", "u1", C.sizeof(A.me_drift_row))])
        assert ctx._L.me_drift_end(ctx._ctx, rows.ctypes.data_as(C.POINTER(A.me_drift_row)), n - 1) == A.ME_ERR_INVALID
        intact()
        # the estimated cloud replaced mid-loop: the call fails and the cloud is restored
        n = ctx.drift_begin(0.5, 0.05)
        ctx.drift_step()
        other = est + 0.25                                   # other points of the same size: set into the same buffer
        ctx.set_cloud(EST, other)
        _refused(api, lambda: ctx.drift_step(), "a cloud changed during the drift loop")
        assert ctx.get_cloud(EST).tobytes() == est.tobytes()
        ctx.set_normals(EST, nrm)
        # a registration open refuses the drift loop
        ctx.icp_begin(0.05, method=A.ME_ICP_POINT_TO_POINT)
        _refused(api, lambda: ctx.drift_begin(0.5, 0.05), "while a registration is open")
        ctx.icp_block()
        while not ctx.icp_step():
            pass
        ctx.icp_end()
    # too many regions
    big = synth.uniform_box(2_500_000, 1.0, 41) + 0.5
    with _ctx(api, big, big[:1000]) as ctx:
        _refused(api, lambda: ctx.drift_begin(0.003, 0.05), "at most ME_REGION_MAX_REGIONS")
        assert ctx.get_cloud(EST).tobytes() == big.tobytes()
    # an empty ground truth, a borrowed estimated cloud, world > 1 with the slab layout
    import torch
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, est)
        _refused(api, lambda: ctx.drift_begin(0.5, 0.05), "both clouds must be set")
        t = torch.as_tensor(est, device="cuda:0")
        ctx.set_cloud(GT, gt)
        ctx.set_cloud_device(EST, t.data_ptr(), len(est), keepalive=t)
        _refused(api, lambda: ctx.drift_begin(0.5, 0.05), "library-owned estimated cloud")
    with _ctx(api, est, gt, rank=0, world=2) as ctx:
        ctx.set_layout(A.ME_LAYOUT_SLAB)
        _refused(api, lambda: ctx.drift_begin(0.5, 0.05), "replicated layout")
        _refused(api, lambda: ctx.region_drift(0.5, 0.05), "world == 1")

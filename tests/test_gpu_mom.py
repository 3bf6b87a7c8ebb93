"""The mutually orthogonal metric on the GPU (me_mom*, DESIGN §3.16).

- v per point equals me_get_consistency_points' bit for bit on the shared lattice at 1 and 2 rings, the solo lattice and a
  sparse cell table; lambda2 and the normal lie within the mpmath bounds of tests/mom_ref.py on sampled points;
- everything after the per-point values (histogram, axes, families, n_j, means, medians, the metric) equals the numpy
  statement from me_get_mom_points' arrays bit for bit;
- known answers: noisy rooms have family medians near sigma^2; a ghost copy of one wall lifts its family's median to the
  order of delta^2 / 4 while the whole-map MPV stays far below;
- worlds 2, 3 and 8 as contexts on one GPU, and a sparse table: counts, axes and families world 1's exactly, means and
  medians to 1e-12;
- the contract: determinism, refusals, staleness, MME's entropies and the consistency arrays untouched."""
import math
import os
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import dist as mdist

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import consistency_ref as CR  # noqa: E402
import mom_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
R0 = 0.3


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def _face(rng, n, origin, u, v, sigma):
    """n points uniform on the rectangle origin + s u + t v (s, t in [0, 1]) with Gaussian noise sigma along its normal"""
    u, v = np.asarray(u, float), np.asarray(v, float)
    nrm = np.cross(u, v)
    nrm /= np.linalg.norm(nrm)
    st = rng.random((n, 2))
    return origin + st[:, :1] * u + st[:, 1:] * v + rng.normal(0, sigma, (n, 1)) * nrm


def _room(seed, sigma=0.005, density=400.0, size=(6.0, 5.0, 3.0), rot=np.eye(3)):
    rng = np.random.default_rng(seed)
    X, Y, Z = size
    faces = [((0, 0, 0), (X, 0, 0), (0, Y, 0)), ((0, 0, Z), (X, 0, 0), (0, Y, 0)),
             ((0, 0, 0), (X, 0, 0), (0, 0, Z)), ((0, Y, 0), (X, 0, 0), (0, 0, Z)),
             ((0, 0, 0), (0, Y, 0), (0, 0, Z)), ((X, 0, 0), (0, Y, 0), (0, 0, Z))]
    pts = [_face(rng, int(density * np.linalg.norm(np.cross(u, v))), np.array(o, float), u, v, sigma) for o, u, v in faces]
    return np.vstack(pts) @ rot.T + np.array([3.0, -2.0, 0.5])


def _rot(yaw_deg, tilt_deg):
    y, t = math.radians(yaw_deg), math.radians(tilt_deg)
    Rz = np.array([[math.cos(y), -math.sin(y), 0], [math.sin(y), math.cos(y), 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, math.cos(t), -math.sin(t)], [0, math.sin(t), math.cos(t)]])
    return Rz @ Rx


def _check_statement(res, v, l2, n, fam, rho=0.5, angle=10.0, min_family=100):
    ref = R.statement(v, l2, n, rho, angle, min_family)
    assert res["status"] == ref["status"]
    assert res["n_planar"] == ref["n_planar"]
    assert np.array_equal(_bits(res["axis"]), _bits(ref["axis"]))
    assert np.array_equal(fam, ref["family"])
    assert np.array_equal(res["n"], ref["n"])
    assert np.array_equal(_bits(res["mean"]), _bits(ref["mean"]))
    assert np.array_equal(_bits(res["median"]), _bits(ref["median"]))
    assert _bits(res["mom"]) == _bits(ref["mom"])
    return ref


CASES = [   # id, context options, solo
    ("rings1", dict(nn_cell_size=0.3), 0),
    ("rings2", dict(nn_cell_size=0.15), 0),
    ("solo", dict(nn_cell_size=0.05), 1),
    ("sparse", dict(nn_cell_size=0.15, max_grid_cells=64), 0),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_v_equals_consistency_and_statement(api, case):
    _, kw, solo = case
    pts = _room(1)
    with api.MapEvalB200(**kw) as ctx:
        ctx.set_cloud(EST, pts)
        cons = ctx.local_consistency(EST, R0, 10)
        _, v_c = ctx.get_consistency_points(EST)
        res = ctx.mom(EST, R0, 10)
        v, l2, n, fam = ctx.get_mom_points(EST)
    assert res["solo"] == solo == cons["whole"]["solo"] and res["rings"] == cons["whole"]["rings"]
    assert np.array_equal(_bits(v), _bits(v_c))
    assert res["n_query"] == len(pts) and res["n_pv"] == cons["whole"]["n_pv"]
    assert res["status"] == "OK"
    ref = _check_statement(res, v, l2, n, fam)
    assert (ref["n"] >= 1000).all()


def test_lambda2_and_normal_within_the_exact_bounds(api):
    pts = _room(2, density=150.0)
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, pts)
        ctx.mom(EST, R0, 10)
        v, l2, n, fam = ctx.get_mom_points(EST)
    rng = np.random.default_rng(3)
    pl = np.flatnonzero(R.planar(v, l2, 0.5))
    ex = R.exact_points(pts, R0, rng.choice(pl, 60, replace=False))
    i = ex["i"]
    assert len(i) == 60
    assert np.all(np.abs(l2[i] - ex["l2"]) <= ex["eps"])
    dots = np.abs(np.sum(n[i] * ex["n"], axis=1))
    sin = np.sqrt(np.maximum(0.0, 1.0 - np.minimum(1.0, dots) ** 2))
    assert np.all(np.isfinite(ex["sin"])) and np.all(sin <= ex["sin"] + 2e-8)   # sqrt(1 - dot^2) resolves angles to ~1e-8
    assert np.allclose(np.linalg.norm(n[i], axis=1), 1.0, rtol=0, atol=4e-16)


@pytest.mark.parametrize("rot", [(0.0, 0.0), (27.0, 4.0)], ids=["aligned", "yawed"])
def test_noisy_rooms_median_near_sigma2(api, rot):
    sigma = 0.005
    pts = _room(4, sigma=sigma, rot=_rot(*rot))
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, pts)
        res = ctx.mom(EST, R0, 10)
        v, l2, n, fam = ctx.get_mom_points(EST)
    _check_statement(res, v, l2, n, fam)
    assert res["status"] == "OK"
    # against the exact eigenvalues: per family, the exact lambda3 of 101 sampled members (rational covariance, mpmath).  The
    # sampled v lie within their fp64 bounds of them, and the family's median lies between the sample's 31st and 71st order
    # statistics: for a sample of 101 the population median falls outside that range with probability
    # 2 P(Bin(101, 1/2) <= 30) < 1e-4 (the seeds are fixed, so the test is deterministic)
    rng = np.random.default_rng(11)
    for j in range(3):
        idx = rng.choice(np.flatnonzero(fam == j), 101, replace=False)
        ex = CR.exact_points(pts, R0, 10, idx=idx)
        assert np.all(np.abs(v[idx] - ex["lam"]) <= ex["bound"])
        lam = np.sort(ex["lam"])
        assert lam[30] <= res["median"][j] <= lam[70], (j, lam[30], res["median"][j], lam[70])
    # and sigma^2: the smallest eigenvalue of a sample covariance of ~100 points of a noisy plane is sigma^2 shrunk by the fit
    # (about (k - 3) / (k - 1)) and spread by the sampling
    assert np.all(res["median"] > sigma ** 2 / 1.5) and np.all(res["median"] < 1.5 * sigma ** 2), res["median"]
    truth = _rot(*rot)
    for j in range(3):
        assert max(abs(truth.T @ res["axis"][j])) > math.cos(math.radians(10.0))


def test_ghost_wall_lifts_its_family_while_mpv_stays_low(api):
    rng = np.random.default_rng(5)
    sigma, delta, dens = 0.004, 0.05, 300.0
    ground = _face(rng, int(dens * 900), np.array([0.0, 0.0, 0.0]), (30, 0, 0), (0, 30, 0), sigma)
    wall_x = _face(rng, int(dens * 30), np.array([10.0, 10.0, 0.3]), (0, 10, 0), (0, 0, 3), sigma)      # normal x
    ghost = _face(rng, int(dens * 30), np.array([10.0 + delta, 10.0, 0.3]), (0, 10, 0), (0, 0, 3), sigma)
    wall_y = _face(rng, int(dens * 30), np.array([12.0, 5.0, 0.3]), (10, 0, 0), (0, 0, 3), sigma)       # normal y
    pts = np.vstack([ground, wall_x, ghost, wall_y])
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, pts)
        res = ctx.mom(EST, R0, 10)
        cons = ctx.local_consistency(EST, R0, 10)
        ctx_v = ctx.get_consistency_points(EST)
    assert res["status"] == "OK"
    jx = int(np.argmax(np.abs(res["axis"][:, 0])))
    # two parallel sheets delta apart seen from a point between them: lambda3 = delta^2 / 4 + sigma^2 for equal shares; the
    # family median sits on the doubled wall (it holds most of the family)
    assert res["median"][jx] > delta ** 2 / 8
    assert res["mom"] > delta ** 2 / 8
    # the whole-map MPV from the measured per-population means: the ground (planar neighbourhoods) and everything else (the
    # walls, their ghost and the mixed neighbourhoods where the walls meet the ground, whose v can be far larger); the margin
    # between MPV and the ghosted family's median is measured on this scene, not proven in general
    _, vc = ctx_v
    near = np.zeros(len(pts), bool)
    near[len(ground):] = True
    near[:len(ground)] = ((np.abs(ground[:, 0] - 10.0) < 2 * R0) | (np.abs(ground[:, 1] - 5.0) < 2 * R0)) & \
        (ground[:, 0] > 9.0) & (ground[:, 0] < 22.5) & (ground[:, 1] > 4.5) & (ground[:, 1] < 20.5)
    ok = np.isfinite(vc)
    share = (near & ok).sum() / ok.sum()
    m_far, m_near = vc[~near & ok].mean(), vc[near & ok].mean()
    assert m_far < 2 * sigma ** 2                       # the open ground is a plane of noise sigma
    mpv = cons["whole"]["mpv"]
    assert mpv == pytest.approx((1 - share) * m_far + share * m_near, rel=1e-9)
    assert mpv < res["median"][jx] / 2, (mpv, share, m_far, m_near, res["median"][jx])


def _sharded(api, pts, world, **kw):
    import torch
    ctxs = [api.MapEvalB200(rank=r, world=world, **kw) for r in range(world)]
    try:
        for c in ctxs:
            c.set_cloud(EST, pts)
            c.mom_begin(EST, R0, 10)
        done = False
        passes = 0
        while not done:
            ts = []
            for c in ctxs:
                ptr, n = c.mom_block()
                assert n == A.ME_MOM_BLOCK
                c.synchronize()
                ts.append(torch.as_tensor(mdist._DeviceBlock(ptr, n), device="cuda:0"))
            total = torch.stack(ts).sum(0)
            for t in ts:
                t.copy_(total)
            torch.cuda.synchronize()
            dn = [c.mom_step() for c in ctxs]
            assert len(set(dn)) == 1
            done = dn[0]
            passes += 1
        res = [c.mom_end() for c in ctxs]
        pp = [c.get_mom_points(EST) for c in ctxs]
    finally:
        for c in ctxs:
            c.close()
    for r in res[1:]:
        for f in ("n", "n_planar", "n_query", "n_pv"):
            assert np.array_equal(r[f], res[0][f])
        for f in ("axis", "mean", "median", "mom"):
            assert np.array_equal(_bits(r[f]), _bits(res[0][f]))
    fam = np.max([p[3] for p in pp], axis=0)
    return res[0], fam, passes


def test_sharded_equals_world_one(api):
    pts = _room(6)
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, pts)
        ref = ctx.mom(EST, R0, 10)
        _, _, _, fam1 = ctx.get_mom_points(EST)
    assert ref["status"] == "OK"
    for world, kw in ((2, {}), (3, {}), (8, {}), (1, dict(max_grid_cells=64)), (3, dict(max_grid_cells=64))):
        got, fam, passes = _sharded(api, pts, world, **kw)
        assert passes == 9          # the histogram, the fold with digit 0, digits 1..7
        for f in ("n", "n_planar", "n_query", "n_pv"):
            assert np.array_equal(got[f], ref[f]), (world, f)
        assert np.array_equal(_bits(got["axis"]), _bits(ref["axis"]))
        assert np.array_equal(fam, fam1)
        np.testing.assert_allclose(got["mean"], ref["mean"], rtol=1e-12, atol=0)
        np.testing.assert_allclose(got["median"], ref["median"], rtol=1e-12, atol=0)


def test_c3_size(api):
    from cloud_map_evaluation_b200 import synth
    est, _, cfg = synth.make_pair("C3")
    r = cfg["nn_radius"]
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, est)
        cons = ctx.local_consistency(EST, r, 10)
        _, v_c = ctx.get_consistency_points(EST)
        res = ctx.mom(EST, r, 10)
        v, l2, n, fam = ctx.get_mom_points(EST)
    assert res["n_query"] == len(est) and res["n_pv"] == cons["whole"]["n_pv"]
    assert np.array_equal(_bits(v), _bits(v_c))
    _check_statement(res, v, l2, n, fam)


def _two_gpus():
    import torch
    return torch.cuda.device_count() >= 2


TWO_GPU_SCRIPT = r'''
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.getcwd())
sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
from cloud_map_evaluation_b200 import api, dist as mdist, _abi as A
from test_gpu_mom import _room
rank = int(os.environ["RANK"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl")
pts = _room(7)
with api.MapEvalB200(device=rank, rank=rank, world=2) as c:
    c.set_cloud(A.ME_CLOUD_EST, pts)
    res = mdist.mom_distributed(c, f"cuda:{rank}", A.ME_CLOUD_EST, 0.3, 10)
with api.MapEvalB200(device=rank) as c:
    c.set_cloud(A.ME_CLOUD_EST, pts)
    ref = c.mom(A.ME_CLOUD_EST, 0.3, 10)
assert (res["n"] == ref["n"]).all()
np.testing.assert_allclose(res["median"], ref["median"], rtol=1e-12)
dist.destroy_process_group()
'''


@pytest.mark.skipif(not _two_gpus(), reason="needs two GPUs")
def test_two_gpus_distributed(tmp_path):
    import subprocess
    script = tmp_path / "two_gpus.py"
    script.write_text(TWO_GPU_SCRIPT)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call([sys.executable, "-m", "torch.distributed.run", "--nproc_per_node=2", str(script)], cwd=root)


def test_contract(api):
    pts = _room(8, density=200.0)
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, pts)
        mme = ctx.computeMME(EST, R0, 10)
        e0 = ctx.get_entropies(EST)
        ctx.local_consistency(EST, R0, 10)
        ce, cv = ctx.get_consistency_points(EST)
        a = ctx.mom(EST, R0, 10)
        pa = ctx.get_mom_points(EST)
        b = ctx.mom(EST, R0, 10)
        pb = ctx.get_mom_points(EST)
        for f in ("axis", "mean", "median", "mom"):
            assert np.array_equal(_bits(a[f]), _bits(b[f]))
        for x, y in zip(pa, pb):
            assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
        # MME's entropies and the consistency arrays are untouched
        assert np.array_equal(_bits(ctx.get_entropies(EST)), _bits(e0))
        ce2, cv2 = ctx.get_consistency_points(EST)
        assert np.array_equal(_bits(ce2), _bits(ce)) and np.array_equal(_bits(cv2), _bits(cv))
        assert mme.n_valid > 0
        # refusals
        for kw in (dict(angle_deg=0.0), dict(angle_deg=31.0), dict(planarity=0.0), dict(planarity=1.5), dict(min_family=0)):
            with pytest.raises(api.MapEvalError):
                ctx.mom(EST, R0, 10, **kw)
        for r, m in ((0.0, 10), (float("inf"), 10), (R0, 2)):
            with pytest.raises(api.MapEvalError):
                ctx.mom(EST, r, m)
        with pytest.raises(api.MapEvalError):
            ctx.mom(GT, R0, 10)                      # empty cloud
        with pytest.raises(api.MapEvalError):
            ctx.mom_step()                           # nothing open
        # staleness: a cloud changed between begin and end voids the call and the points
        ctx.mom_begin(EST, R0, 10)
        ctx.set_cloud(EST, pts + 1.0)
        with pytest.raises(api.MapEvalError):
            ctx.mom_step()
        with pytest.raises(api.MapEvalError):
            ctx.get_mom_points(EST)
        # a small min_family passes where a large one is refused by the status
        c = ctx.mom(EST, R0, 10, min_family=10 ** 9)
        assert c["status"] == "SMALL_FAMILY" and math.isnan(c["mom"]) and np.isfinite(c["median"]).all()

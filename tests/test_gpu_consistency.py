"""Local map consistency on the GPU (me_consistency*): mean plane variance beside MME, whole map and per region.

- known answers: an exact grid plane (v == 0, no valid entropy), two parallel planes, a tilted noisy plane and a box against
  the exact covariance's smallest eigenvalue from mpmath, within the derived fp64 bound (tests/consistency_ref.py);
- the same neighbourhoods as MME: e per point equals me_get_entropies after me_eval_mme under ME_MME_WALK=1 bit for bit and
  n_valid equals the default me_eval_mme's, on the shared lattice at 1, 2, 3 and 5 rings, the solo lattice and a sparse cell
  table;
- the region table against a numpy restatement from the per-point arrays, its index list against region_errors', one region
  against the whole map, the rows summing to the whole;
- worlds 2, 3 and 8 as contexts on one GPU, and a sparse cell table: counts world 1's exactly, sums and maxima to 1e-12,
  the merged per-point arrays world 1's validity exactly and its values to rounding;
- the contract: determinism, refusals, staleness, MME's entropies and the kernel trace untouched;
- a ghost wall found by its regions' plane variance; one C3-size case against me_eval_mme."""
import math
import os
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import dist as mdist
from cloud_map_evaluation_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import consistency_ref as CR  # noqa: E402
import exact_ref as X  # noqa: E402

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
SUMS = ("sum_entropy", "sum_pv", "sum_sqrt_pv")
COUNTS = ("n_query", "n_valid", "n_pv")


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


class _env:
    def __init__(self, **kv):
        self.kv = kv

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kv}
        os.environ.update(self.kv)

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _room(n, seed, noise=0.002):
    return synth.indoor_scene(n, seed, noise, rooms=2).astype(np.float64)


def _grid_plane(nx, ny, step=0.125, z=0.0):
    return np.array([(x * step, y * step, z) for x in range(nx) for y in range(ny)], np.float64)


# ---- known answers ------------------------------------------------------------------------------------------------------
def test_exact_grid_plane(api):
    pts = _grid_plane(40, 30)
    r, m = 0.3, 3
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, pts)
        res = ctx.local_consistency(EST, r, m)
        e, v = ctx.get_consistency_points(EST)
    k = np.array([len(nb) for nb in X.mme_neighbours(pts, r)])
    ok = k >= m
    assert np.all(v[ok] == 0.0) and np.all(np.isnan(v[~ok]))
    assert np.all(e == 0.0)
    w = res["whole"]
    assert w["n_valid"] == 0 and w["n_pv"] == int(ok.sum()) and w["n_query"] == len(pts)
    assert w["mpv"] == 0.0 and w["mme"] == 0.0


def _check_exact(api, pts, r, m, sample=None, **kw):
    with api.MapEvalB200(**kw) as ctx:
        ctx.set_cloud(EST, pts)
        ctx.local_consistency(EST, r, m)
        _, v = ctx.get_consistency_points(EST)
    ex = CR.exact_points(pts, r, m, idx=sample)
    got = v[ex["i"]]
    bad = ex["k"] < m
    assert np.all(np.isnan(got[bad]))
    err = np.abs(got[~bad] - ex["lam"][~bad])
    assert np.all(err <= ex["bound"][~bad]), (err - ex["bound"][~bad]).max()
    return ex


def test_two_parallel_planes(api):
    delta = 0.01
    pts = np.vstack([_grid_plane(24, 24), _grid_plane(24, 24, z=delta)])
    ex = _check_exact(api, pts, 0.3, 5)
    assert np.nanmax(ex["lam"]) > 0.0


def test_tilted_noisy_plane_and_box(api):
    rng = np.random.default_rng(3)
    uv = rng.random((4000, 2)) * 2.0
    n = np.array([0.3, -0.2, 1.0]) / np.linalg.norm([0.3, -0.2, 1.0])
    a = np.cross(n, [1.0, 0.0, 0.0])
    a /= np.linalg.norm(a)
    b = np.cross(n, a)
    plane = uv[:, :1] * a + uv[:, 1:] * b + rng.normal(0, 0.003, (4000, 1)) * n + np.array([5.0, -3.0, 1.5])
    _check_exact(api, plane, 0.1, 10, sample=rng.choice(4000, 300, replace=False))
    box = rng.random((6000, 3))
    _check_exact(api, box, 0.1, 5, sample=rng.choice(6000, 300, replace=False))


# ---- the same neighbourhoods as MME -------------------------------------------------------------------------------------
R0 = 0.1
MME_CASES = [   # id, context options, environment, rings (None: not fixed), solo
    ("rings1", dict(nn_cell_size=0.1), {}, 1, 0),
    ("rings2", dict(nn_cell_size=0.05), {}, 2, 0),
    ("rings3", dict(nn_cell_size=0.034), {}, 3, 0),
    ("solo", dict(nn_cell_size=0.02), {}, 2, 1),
    ("sparse", dict(nn_cell_size=0.05, max_grid_cells=64), {}, None, 0),
    ("rings5", dict(nn_cell_size=0.02), {"ME_MME_SHARED_LATTICE": "1"}, None, 0),
]


@pytest.mark.parametrize("case", MME_CASES, ids=[c[0] for c in MME_CASES])
def test_same_neighbourhoods_as_mme(api, case):
    _, kw, env, rings, solo = case
    pts = _room(60_000, 5)
    with _env(**env), api.MapEvalB200(**kw) as ctx:
        ctx.set_cloud(EST, pts)
        mme_def = ctx.computeMME(EST, R0, 10)
        with _env(ME_MME_WALK="1"):
            mme_walk, e_walk = ctx.computeMME(EST, R0, 10, want_entropies=True)
        res = ctx.local_consistency(EST, R0, 10)
        e, v = ctx.get_consistency_points(EST)
    w = res["whole"]
    assert res["kernel"] == "WALK" and w["solo"] == solo
    if rings is not None:
        assert w["rings"] == rings
    elif env:
        assert w["rings"] > 3
    assert np.array_equal(_bits(e), _bits(e_walk))
    assert w["n_valid"] == mme_def.n_valid == mme_walk.n_valid
    assert w["mme"] == pytest.approx(mme_def.mme, abs=1e-3 + 1e-9)
    assert w["n_query"] == len(pts) and w["n_pv"] == int(np.isfinite(v).sum())


# ---- the region table ---------------------------------------------------------------------------------------------------
def _restate(pts, s, e, v):
    idx = np.floor(pts / s).astype(np.int64)
    keys, inv = np.unique(idx, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    R = len(keys)
    pv = np.isfinite(v)
    out = dict(index=keys, n_points=np.bincount(inv, minlength=R), n_query=np.bincount(inv, minlength=R),
               n_valid=np.bincount(inv[e != 0.0], minlength=R), n_pv=np.bincount(inv[pv], minlength=R),
               sum_entropy=np.bincount(inv, e, R), sum_pv=np.bincount(inv[pv], v[pv], R),
               sum_sqrt_pv=np.bincount(inv[pv], np.sqrt(v[pv]), R))
    mx = np.zeros(R)
    np.maximum.at(mx, inv[pv], v[pv])
    out["max_pv"] = np.where(out["n_pv"] > 0, mx, np.nan)
    return out


def test_region_table(api):
    est = _room(80_000, 7)
    gt = _room(80_000, 8, noise=0.0)
    p = A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], 1.0)
    for s in (0.5, 1.7):
        with api.MapEvalB200() as ctx:
            ctx.set_cloud(EST, est)
            ctx.set_cloud(GT, gt)
            ctx.calculateMetricsWithInitialMatrix(p)
            ref = ctx.region_errors(s)
            res = ctx.local_consistency(EST, R0, 10, region_size=s)
            e, v = ctx.get_consistency_points(EST)
            whole0 = ctx.local_consistency(EST, R0, 10)["whole"]
        assert np.array_equal(res["index"], ref["index"])           # the occupied list of est ++ gt
        np.testing.assert_array_equal(res["n_points"], ref["n_est"])
        rs = _restate(est, s, e, v)
        pos = {tuple(k): j for j, k in enumerate(res["index"])}
        at = np.array([pos[tuple(k)] for k in rs["index"]])
        keep = np.zeros(len(res["index"]), bool)
        keep[at] = True
        got = {f: res[f][at] for f in rs if f != "index"}
        for f in COUNTS + ("n_points",):
            np.testing.assert_array_equal(got[f], rs[f])
        assert np.all(res["n_points"][~keep] == 0)
        np.testing.assert_array_equal(_bits(got["max_pv"]), _bits(rs["max_pv"]))
        for f in SUMS:
            np.testing.assert_allclose(got[f], rs[f], rtol=1e-12, atol=0)
        w = res["whole"]
        for f in COUNTS:
            assert w[f] == res[f].sum() == whole0[f]
        for f in SUMS:
            assert w[f] == pytest.approx(whole0[f], rel=1e-12)
        assert _bits(w["max_pv"]) == _bits(whole0["max_pv"])
    # one region that holds the whole cloud reproduces the whole map
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, est - est.min(0) + 1.0)
        whole0 = ctx.local_consistency(EST, R0, 10)["whole"]
        one = ctx.local_consistency(EST, R0, 10, region_size=1000.0)
    assert len(one["index"]) == 1
    for f in COUNTS:
        assert one[f][0] == whole0[f] == one["whole"][f]
    for f in SUMS + ("max_pv",):
        assert one[f][0] == pytest.approx(whole0[f], rel=1e-12)


# ---- sharding -----------------------------------------------------------------------------------------------------------
def _sharded(api, pts, s, world, **kw):
    import torch
    ctxs = [api.MapEvalB200(rank=r, world=world, **kw) for r in range(world)]
    try:
        for c in ctxs:
            c.set_cloud(EST, pts)
        ns = [c.consistency_begin(EST, R0, 10, s) for c in ctxs]
        assert len(set(ns)) == 1
        sums, maxs = [], []
        for c in ctxs:
            ptr, n_sum, n_max = c.consistency_block()
            B = max(ns[0], 1)
            assert (n_sum, n_max) == (A.ME_CONSISTENCY_SUM_FIELDS * B, A.ME_CONSISTENCY_MAX_FIELDS * B)
            c.synchronize()
            t = torch.as_tensor(mdist._DeviceBlock(ptr, n_sum + n_max), device="cuda:0")
            sums.append(t[:n_sum])
            maxs.append(t[n_sum:])
        total, top = torch.stack(sums).sum(0), torch.stack(maxs).amax(0)
        for a, b in zip(sums, maxs):
            a.copy_(total)
            b.copy_(top)
        torch.cuda.synchronize()
        res = [c.consistency_end(ns[0]) for c in ctxs]
        pts_e, pts_v = zip(*[c.get_consistency_points(EST) for c in ctxs])
    finally:
        for c in ctxs:
            c.close()
    for r in res[1:]:
        for f in COUNTS + SUMS + ("max_pv",):
            assert np.array_equal(_bits(r[f]) if f in SUMS + ("max_pv",) else r[f],
                                  _bits(res[0][f]) if f in SUMS + ("max_pv",) else res[0][f])
    e = np.sum(pts_e, axis=0)
    vs = np.array(pts_v)
    v = np.where(np.isnan(vs).all(0), np.nan, np.nanmax(np.where(np.isnan(vs), -np.inf, vs), axis=0))
    return res[0], e, v


def _same(got, ref):
    for f in COUNTS + ("n_points", "index"):
        np.testing.assert_array_equal(got[f], ref[f])
    # a point's v depends on the order its context's layout gave the points of a cell (ranked with atomics), so maxima
    # agree to rounding
    np.testing.assert_allclose(got["max_pv"], ref["max_pv"], rtol=1e-12, atol=0)
    for f in SUMS:
        np.testing.assert_allclose(got[f], ref[f], rtol=1e-12, atol=0)
    for f in COUNTS:
        assert got["whole"][f] == ref["whole"][f]
    for f in SUMS:
        assert got["whole"][f] == pytest.approx(ref["whole"][f], rel=1e-12)


def test_sharded_equals_world_one(api):
    pts = _room(120_000, 9)
    for s in (0.0, 0.8):
        with api.MapEvalB200() as ctx:
            ctx.set_cloud(EST, pts)
            ref = ctx.local_consistency(EST, R0, 10, region_size=s)
            e1, v1 = ctx.get_consistency_points(EST)
        for world, kw in ((2, {}), (3, {}), (8, {}), (1, dict(max_grid_cells=64)), (3, dict(max_grid_cells=64))):
            got, e, v = _sharded(api, pts, s, world, **kw)
            _same(got, ref)
            # the points' own values: the same validity everywhere; the values to rounding, because every layout ranks the
            # points inside a cell with atomics (grid.cu), which orders the moments' fp64 sums differently
            assert np.array_equal(e != 0.0, e1 != 0.0) and np.array_equal(np.isnan(v), np.isnan(v1))
            np.testing.assert_allclose(e, e1, rtol=1e-12, atol=0)
            np.testing.assert_allclose(v, v1, rtol=1e-9, atol=1e-15)


def _two_gpus():
    import torch
    return torch.cuda.device_count() >= 2


TWO_GPU_SCRIPT = r'''
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.getcwd())
from cloud_map_evaluation_b200 import api, dist as mdist, synth, _abi as A
rank = int(os.environ["RANK"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl")
pts = synth.indoor_scene(100000, 4, 0.002, rooms=2).astype(np.float64)
with api.MapEvalB200(device=rank, rank=rank, world=2) as c:
    c.set_cloud(A.ME_CLOUD_EST, pts)
    res = mdist.consistency_distributed(c, f"cuda:{rank}", A.ME_CLOUD_EST, 0.1, 10, 0.8)
with api.MapEvalB200(device=rank) as c:
    c.set_cloud(A.ME_CLOUD_EST, pts)
    ref = c.local_consistency(A.ME_CLOUD_EST, 0.1, 10, 0.8)
for f in ("n_query", "n_valid", "n_pv"):
    assert (res[f] == ref[f]).all(), f
np.testing.assert_allclose(res["sum_pv"], ref["sum_pv"], rtol=1e-12)
dist.destroy_process_group()
'''


@pytest.mark.skipif(not _two_gpus(), reason="needs two GPUs")
def test_two_gpus_distributed(tmp_path):
    import subprocess
    script = tmp_path / "two_gpus.py"
    script.write_text(TWO_GPU_SCRIPT)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call([sys.executable, "-m", "torch.distributed.run", "--nproc_per_node=2", str(script)], cwd=root)


# ---- contract -----------------------------------------------------------------------------------------------------------
def test_contract(api):
    import torch
    pts = _room(50_000, 11)
    with api.MapEvalB200(nn_cell_size=0.05) as ctx:
        ctx.set_cloud(EST, pts)
        # determinism: two calls, the same block bits
        blocks = []
        for _ in range(2):
            n = ctx.consistency_begin(EST, R0, 10, 0.7)
            ptr, n_sum, n_max = ctx.consistency_block()
            ctx.synchronize()
            blocks.append(torch.as_tensor(mdist._DeviceBlock(ptr, n_sum + n_max), device="cuda:0").cpu().numpy().copy())
            ctx.consistency_end(n)
        assert np.array_equal(_bits(blocks[0]), _bits(blocks[1]))
        # MME's entropies and a later MME untouched; no trace bit set
        _, ent = ctx.computeMME(EST, R0, 10, want_entropies=True)
        ctx.kernel_trace(reset=True)
        for r in (R0, 0.3):           # 0.3 m lays the cloud out on a lattice of its own
            ctx.local_consistency(EST, r, 10)
            assert np.array_equal(_bits(ctx.get_entropies(EST)), _bits(ent))
        mask, _ = ctx.kernel_trace(reset=True, events=True)
        assert mask == set()
        _, ent2 = ctx.computeMME(EST, R0, 10, want_entropies=True)
        assert np.array_equal(_bits(ent2), _bits(ent))
        # refusals
        for args in ((EST, 0.0, 10, 0.0), (EST, math.inf, 10, 0.0), (EST, math.nan, 10, 0.0), (EST, R0, 2, 0.0),
                     (EST, R0, 10, -1.0), (EST, R0, 10, math.inf), (GT, R0, 10, 0.0), (EST, R0, 10, 1e-9)):
            with pytest.raises(api.MapEvalError, match="me_consistency"):
                ctx.local_consistency(*args)
        with pytest.raises(api.MapEvalError, match="without an open"):
            ctx.consistency_block()
        # staleness: a cloud change between begin and end, and of the per-point values
        ctx.local_consistency(EST, R0, 10)
        ctx.get_consistency_points(EST)
        n = ctx.consistency_begin(EST, R0, 10, 0.0)
        ctx.set_cloud(GT, pts[:100])
        with pytest.raises(api.MapEvalError, match="changed"):
            ctx.consistency_end(n)
        with pytest.raises(api.MapEvalError, match="changed"):
            ctx.get_consistency_points(EST)
        ctx.local_consistency(EST, R0, 10)
        ctx.transform(EST, np.eye(4))
        with pytest.raises(api.MapEvalError, match="changed"):
            ctx.get_consistency_points(EST)
        # an open registration or drift loop, the slab layout
        ctx.icp_begin(0.5, method=A.ME_ICP_POINT_TO_POINT)
        with pytest.raises(api.MapEvalError, match="registration"):
            ctx.local_consistency(EST, R0, 10)
        with pytest.raises(api.MapEvalError):      # closes the loop: no step ran
            ctx.icp_end()
        n = ctx.drift_begin(1.0, 0.5)
        with pytest.raises(api.MapEvalError, match="drift"):
            ctx.local_consistency(EST, R0, 10)
        while not ctx.drift_step():
            pass
        ctx.drift_end(n)
    with api.MapEvalB200(rank=0, world=2) as ctx:
        ctx.set_layout(A.ME_LAYOUT_SLAB)
        ctx.set_cloud(EST, pts)
        with pytest.raises(api.MapEvalError, match="me_set_layout"):
            ctx.consistency_begin(EST, R0, 10, 0.0)


# ---- a ghost wall -------------------------------------------------------------------------------------------------------
def test_ghost_wall(api):
    rng = np.random.default_rng(17)
    step = 0.02
    def wall(u0, u1, h, fix, axis):
        u = np.arange(u0, u1, step)
        z = np.arange(0.0, h, step)
        U, Z = np.meshgrid(u, z)
        P = np.zeros((U.size, 3))
        P[:, 1 - axis] = U.ravel()
        P[:, axis] = fix
        P[:, 2] = Z.ravel()
        return P
    # four walls that do not meet (a corner is thick at the scale of r as well), and the wall y = 0 again, 5 cm away
    room = [wall(0.5, 7.5, 2.5, 0.0, 0), wall(0.5, 7.5, 2.5, 8.0, 0), wall(0.5, 7.5, 2.5, 0.0, 1), wall(0.5, 7.5, 2.5, 8.0, 1)]
    ghost = wall(0.5, 7.5, 2.5, 0.05, 1)
    pts = np.vstack(room + [ghost]) + rng.normal(0, 0.002, (sum(len(w) for w in room) + len(ghost), 3))
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, pts)
        res = ctx.local_consistency(EST, R0, 10, region_size=1.0)
    mpv = res["mpv"]
    gidx = {tuple(k) for k in np.floor(ghost / 1.0).astype(np.int64)}
    ghosted = np.array([tuple(k) in gidx for k in res["index"]])
    med = np.nanmedian(mpv)
    assert ghosted.any()
    assert np.nanmin(mpv[ghosted]) >= 10 * med
    assert ghosted[int(np.nanargmax(mpv))]


# ---- C3 size ------------------------------------------------------------------------------------------------------------
def test_c3_size(api):
    est, _, cfg = synth.make_pair("C3")
    r = cfg["nn_radius"]
    with api.MapEvalB200(vmd_voxel_size=cfg["vmd_voxel_size"]) as ctx:
        ctx.set_cloud(EST, est)
        mme = ctx.computeMME(EST, r, 10)
        res = ctx.local_consistency(EST, r, 10)
    w = res["whole"]
    assert w["n_valid"] == mme.n_valid
    assert abs(w["mme"] - mme.mme) <= 1e-3 + 1e-9
    assert w["n_query"] == len(est) and w["n_pv"] >= w["n_valid"]

"""The mutually orthogonal metric per region on the GPU (me_mom_region*, DESIGN §3.17).

- rooms, tilted rooms and a ghost wall: n_points, n_planar, n, median, mom and status equal the numpy statement of
  tests/mom_regions_ref.py from me_get_mom_points' arrays bit for bit, means to 1e-12;
- a region larger than the map gives me_mom_end's n, medians and MOM bit for bit;
- the ghost wall's thickness lands on the wall family in the regions that hold the wall;
- worlds 2, 3 and 8 as contexts on one GPU, and a sparse table: every rank's rows the same bits, and world 1's counts,
  statuses and families exactly, means and medians to 1e-12;
- the rows align with local_consistency's at equal region size, for est with a gt loaded and for the gt cloud;
- the contract: the MOM result and points untouched, determinism, refusals; C3's estimate at 1 m."""
import math
import os
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import dist as mdist

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mom_regions_ref as MRR  # noqa: E402
from test_gpu_mom import _face, _room, _rot  # noqa: E402

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
R0 = 0.3


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def _ghost_scene(seed=5, sigma=0.004, delta=0.05, dens=300.0):
    """test_gpu_mom's ghost wall: a 30 m ground, a wall with normal x doubled delta away, a wall with normal y"""
    rng = np.random.default_rng(seed)
    ground = _face(rng, int(dens * 900), np.array([0.0, 0.0, 0.0]), (30, 0, 0), (0, 30, 0), sigma)
    wall_x = _face(rng, int(dens * 30), np.array([10.0, 10.0, 0.3]), (0, 10, 0), (0, 0, 3), sigma)
    ghost = _face(rng, int(dens * 30), np.array([10.0 + delta, 10.0, 0.3]), (0, 10, 0), (0, 0, 3), sigma)
    wall_y = _face(rng, int(dens * 30), np.array([12.0, 5.0, 0.3]), (10, 0, 0), (0, 0, 3), sigma)
    return np.vstack([ground, wall_x, ghost, wall_y]), len(ground), len(wall_x)


def _axes_status(res):
    return res["status"] if res["status"] in MRR.NO_AXES else "OK"


def _first_diff(a, b):
    bad = np.flatnonzero(np.asarray(a).reshape(len(a), -1).tolist() != np.asarray(b).reshape(len(b), -1).tolist()) \
        if len(a) == len(b) else []
    return f"{len(bad)} rows differ, first {bad[:3]}: {np.asarray(a)[bad[:3]]} vs {np.asarray(b)[bad[:3]]}" if len(bad) else ""


def _check(rows, ref, mean_rtol=1e-12):
    assert np.array_equal(rows["index"], ref["index"]), (len(rows["index"]), len(ref["index"]))
    for f in ("n_points", "n_planar", "n"):
        assert np.array_equal(rows[f], ref[f]), (f, _first_diff(rows[f], ref[f]))
    assert list(rows["status"]) == list(ref["status"]), _first_diff(rows["status"], ref["status"])
    assert np.array_equal(_bits(rows["median"]), _bits(ref["median"])), _first_diff(_bits(rows["median"]), _bits(ref["median"]))
    assert np.array_equal(_bits(rows["mom"]), _bits(ref["mom"])), _first_diff(_bits(rows["mom"]), _bits(ref["mom"]))
    has = ref["n"] > 0
    assert np.array_equal(np.isnan(rows["mean"]), ~has)
    np.testing.assert_allclose(rows["mean"][has], ref["mean"][has], rtol=mean_rtol, atol=0)


def _statement(pts, res, v, l2, fam, s, min_family=100, est=None, gt=None):
    est = pts if est is None else est
    return MRR.from_mom_points(pts, est, gt, s, v, l2, fam, 0.5, _axes_status(res), min_family)


SCENES = {
    "room": lambda: _room(1),
    "tilted": lambda: _room(4, rot=_rot(27.0, 4.0)),
    "ghost": lambda: _ghost_scene()[0],
}


@pytest.mark.parametrize("s", [1.0, 2.5])
@pytest.mark.parametrize("scene", sorted(SCENES))
def test_rows_equal_the_statement(api, scene, s):
    pts = SCENES[scene]()
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, pts)
        res = ctx.mom(EST, R0, 10)
        v, l2, _, fam = ctx.get_mom_points(EST)
        rows = ctx.mom_regions(s)
        rows_small = ctx.mom_regions(s, min_family=5)
    assert res["status"] == "OK"
    _check(rows, _statement(pts, res, v, l2, fam, s))
    _check(rows_small, _statement(pts, res, v, l2, fam, s, min_family=5))
    assert (rows["n"] >= 100).any() and (rows_small["status"] == "OK").sum() >= (rows["status"] == "OK").sum()


def test_one_region_larger_than_the_map_is_the_whole_map(api):
    pts = _room(2) + np.array([0.0, 10.0, 0.0])      # every coordinate positive: one region at s = 1000
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, pts)
        res = ctx.mom(EST, R0, 10)
        rows = ctx.mom_regions(1000.0)
    assert len(rows["index"]) == 1 and rows["n_points"][0] == len(pts) and rows["n_planar"][0] == res["n_planar"]
    assert np.array_equal(rows["n"][0], res["n"])
    assert np.array_equal(_bits(rows["median"][0]), _bits(res["median"]))
    assert _bits(rows["mom"][0]) == _bits(res["mom"]) and rows["status"][0] == res["status"]
    np.testing.assert_allclose(rows["mean"][0], res["mean"], rtol=1e-12)


def test_ghost_wall_lands_on_its_family_and_its_regions(api):
    delta = 0.05
    pts, n_ground, n_wall = _ghost_scene(delta=delta)
    s = 3.0
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, pts)
        res = ctx.mom(EST, R0, 10)
        rows = ctx.mom_regions(s)
    assert res["status"] == "OK"
    jx = int(np.argmax(np.abs(res["axis"][:, 0])))
    # the regions holding the doubled wall: those with at least 100 of the wall's or its ghost's points (at s = 3 m both
    # sheets, x = 10 and 10.05, lie inside the regions 9 <= x < 12)
    keys = MRR.region_keys(pts, s)
    doubled = keys[n_ground:n_ground + 2 * n_wall]
    held = {k for k in {tuple(x) for x in doubled} if (doubled == k).all(1).sum() >= 100}
    assert len(held) == 8 and all(k[0] == 3 for k in held)
    thr = delta ** 2 / 8
    hit = 0
    for r, idx in enumerate(map(tuple, rows["index"])):
        for j in range(3):
            if rows["n"][r, j] == 0:
                continue
            if idx in held and j == jx:
                assert rows["median"][r, j] > thr, (idx, j, rows["median"][r, j])
                hit += 1
            else:
                # every other (region, family), the ground family inside the wall's regions included; the margin is
                # measured on this scene, not proven in general
                assert rows["median"][r, j] < thr, (idx, j, rows["n"][r, j], rows["median"][r, j])
    assert hit == len(held)


def _sharded_rows(api, pts, world, s, **kw):
    import torch
    ctxs = [api.MapEvalB200(rank=r, world=world, **kw) for r in range(world)]
    try:
        for c in ctxs:
            c.set_cloud(EST, pts)
            c.mom_begin(EST, R0, 10)
        done = False
        while not done:
            ts = []
            for c in ctxs:
                ptr, n = c.mom_block()
                c.synchronize()
                ts.append(torch.as_tensor(mdist._DeviceBlock(ptr, n), device="cuda:0"))
            total = torch.stack(ts).sum(0)
            for t in ts:
                t.copy_(total)
            torch.cuda.synchronize()
            dn = [c.mom_step() for c in ctxs]
            done = dn[0]
        for c in ctxs:
            c.mom_end()
        nr = [c.mom_region_begin(s) for c in ctxs]
        assert len(set(nr)) == 1
        ts = []
        for c in ctxs:
            ptr, m = c.mom_region_block()
            assert m == 2 * len(pts)
            c.synchronize()
            ts.append(torch.as_tensor(mdist._DeviceBlock(ptr, m), device="cuda:0"))
        total = torch.stack(ts).sum(0)
        for t in ts:
            t.copy_(total)
        torch.cuda.synchronize()
        rows = [c.mom_region_end(nr[0]) for c in ctxs]
    finally:
        for c in ctxs:
            c.close()
    for r in rows[1:]:
        for f in ("index", "n_points", "n_planar", "n"):
            assert np.array_equal(r[f], rows[0][f])
        for f in ("mean", "median", "mom"):
            assert np.array_equal(_bits(r[f]), _bits(rows[0][f]))
        assert list(r["status"]) == list(rows[0]["status"])
    return rows[0]


def test_sharded_equals_world_one(api):
    pts = _room(6)
    s = 1.5
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, pts)
        ctx.mom(EST, R0, 10)
        ref = ctx.mom_regions(s)
    assert (ref["status"] == "OK").any()
    for world, kw in ((2, {}), (3, {}), (8, {}), (3, dict(max_grid_cells=64))):
        got = _sharded_rows(api, pts, world, s, **kw)
        for f in ("index", "n_points", "n_planar", "n"):
            assert np.array_equal(got[f], ref[f]), (world, f)
        assert list(got["status"]) == list(ref["status"])
        has = ref["n"] > 0
        np.testing.assert_allclose(got["median"][has], ref["median"][has], rtol=1e-12, atol=0)
        np.testing.assert_allclose(got["mean"][has], ref["mean"][has], rtol=1e-12, atol=0)


def test_rows_align_with_local_consistency_for_est_and_gt(api):
    est = _room(9)
    gt = _room(10) + np.array([6.5, 0.4, 0.0])            # beside est: regions of one cloud only on both sides
    s = 1.25
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, est)
        ctx.set_cloud(GT, gt)
        for which, pts in ((EST, est), (GT, gt)):
            res = ctx.mom(which, R0, 10)
            v, l2, _, fam = ctx.get_mom_points(which)
            rows = ctx.mom_regions(s)
            cons = ctx.local_consistency(which, R0, 10, region_size=s)
            assert np.array_equal(rows["index"], cons["index"]) and np.array_equal(rows["n_points"], cons["n_points"])
            assert (rows["n_points"] == 0).any()                 # the other cloud's regions are listed too
            _check(rows, _statement(pts, res, v, l2, fam, s, est=est, gt=gt))
            np.testing.assert_array_equal(rows["lo"], rows["index"] * s)


def test_contract(api):
    pts = _room(8, density=200.0)
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, pts)
        with pytest.raises(api.MapEvalError, match="finished MOM"):
            ctx.mom_regions(1.0, min_family=10)               # no MOM call yet
        with pytest.raises(api.MapEvalError):
            ctx.mom_regions(1.0)                              # min_family=None needs a MOM call
        res = ctx.mom(EST, R0, 10)
        pa = ctx.get_mom_points(EST)
        a = ctx.mom_regions(1.0)
        b = ctx.mom_regions(1.0, min_family=res["min_family"])
        pb = ctx.get_mom_points(EST)
        # the MOM points untouched, two calls the same bits
        for x, y in zip(pa, pb):
            assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
        for f in ("mean", "median", "mom"):
            assert np.array_equal(_bits(a[f]), _bits(b[f]))
        n = len(a["index"])
        assert n >= 2
        # refusals: arguments, list limits, order, capacity
        for s in (0.0, -1.0, float("inf"), float("nan")):
            with pytest.raises(api.MapEvalError, match="region_size"):
                ctx.mom_regions(s)
        with pytest.raises(api.MapEvalError, match="min_family"):
            ctx.mom_regions(1.0, min_family=0)
        with pytest.raises(api.MapEvalError, match="2\\^20"):
            ctx.mom_regions(1e-7)
        with pytest.raises(api.MapEvalError):
            ctx.mom_region_block()
        with pytest.raises(api.MapEvalError):
            ctx.mom_region_end(n)
        m = ctx.mom_region_begin(1.0)
        with pytest.raises(api.MapEvalError, match="capacity"):
            ctx.mom_region_end(m - 1)
        # a cloud changed between begin and end voids the call
        m = ctx.mom_region_begin(1.0)
        ctx.set_cloud(GT, pts[:100])
        with pytest.raises(api.MapEvalError, match="changed"):
            ctx.mom_region_end(m)
        # a cloud changed since the MOM call
        with pytest.raises(api.MapEvalError, match="changed"):
            ctx.mom_regions(1.0)
        ctx.mom(EST, R0, 10)
        ctx.transform(EST, np.eye(4))
        with pytest.raises(api.MapEvalError, match="changed"):
            ctx.mom_regions(1.0)
        # a MOM call begun but not finished
        ctx.mom_begin(EST, R0, 10)
        with pytest.raises(api.MapEvalError, match="finished MOM"):
            ctx.mom_regions(1.0)
        # an open registration or drift loop
        ctx.mom(EST, R0, 10)
        ctx.icp_begin(0.5, method=A.ME_ICP_POINT_TO_POINT)
        with pytest.raises(api.MapEvalError, match="registration"):
            ctx.mom_regions(1.0)
        with pytest.raises(api.MapEvalError):      # closes the loop: no step ran
            ctx.icp_end()
        nd = ctx.drift_begin(1.0, 0.5)
        with pytest.raises(api.MapEvalError, match="drift"):
            ctx.mom_regions(1.0)
        while not ctx.drift_step():
            pass
        ctx.drift_end(nd)
    with api.MapEvalB200(rank=0, world=2) as ctx:
        ctx.set_layout(A.ME_LAYOUT_SLAB)
        ctx.set_cloud(EST, pts)
        with pytest.raises(api.MapEvalError, match="me_set_layout"):
            ctx.mom_region_begin(1.0, min_family=10)


def test_no_axes_statuses_reach_every_row(api):
    # a single flat sheet: one family, so no second axis; a line of points: nothing planar
    rng = np.random.default_rng(12)
    sheet = _face(rng, 20000, np.zeros(3), (4, 0, 0), (0, 4, 0), 0.002)
    line = np.column_stack([np.linspace(0, 3, 3000), np.zeros(3000), np.zeros(3000)])
    for pts, status in ((sheet, "NO_SECOND_AXIS"), (line, "NO_PLANAR")):
        with api.MapEvalB200() as ctx:
            ctx.set_cloud(EST, pts)
            res = ctx.mom(EST, R0, 10)
            v, l2, _, fam = ctx.get_mom_points(EST)
            rows = ctx.mom_regions(1.0)
        assert res["status"] == status
        assert (rows["status"] == status).all() and (rows["n"] == 0).all() and np.isnan(rows["median"]).all()
        _check(rows, _statement(pts, res, v, l2, fam, 1.0))
        assert rows["n_planar"].sum() == res["n_planar"]


def test_c3_size(api):
    from cloud_map_evaluation_b200 import synth
    est, _, cfg = synth.make_pair("C3")
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, est)
        res = ctx.mom(EST, cfg["nn_radius"], 10)
        v, l2, _, fam = ctx.get_mom_points(EST)
        rows = ctx.mom_regions(1.0)
    assert len(rows["index"]) > 100
    _check(rows, _statement(est, res, v, l2, fam, 1.0))


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
    mdist.mom_distributed(c, f"cuda:{rank}", A.ME_CLOUD_EST, 0.3, 10)
    rows = mdist.mom_regions_distributed(c, f"cuda:{rank}", 1.0)
with api.MapEvalB200(device=rank) as c:
    c.set_cloud(A.ME_CLOUD_EST, pts)
    c.mom(A.ME_CLOUD_EST, 0.3, 10)
    ref = c.mom_regions(1.0)
assert (rows["n"] == ref["n"]).all() and list(rows["status"]) == list(ref["status"])
has = ref["n"] > 0
np.testing.assert_allclose(rows["median"][has], ref["median"][has], rtol=1e-12)
dist.destroy_process_group()
'''


@pytest.mark.skipif(not _two_gpus(), reason="needs two GPUs")
def test_two_gpus_distributed(tmp_path):
    import subprocess
    script = tmp_path / "two_gpus.py"
    script.write_text(TWO_GPU_SCRIPT)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call([sys.executable, "-m", "torch.distributed.run", "--nproc_per_node=2", str(script)], cwd=root)

"""The library's mean map entropy against the exact reference of tests/exact_ref.py, on every MME sweep, with no oracle.

Scenes: those of test_exact_mme.py — tilted planes with 1 mm .. 0.1 um of normal noise at the origin and 1.7 km out, exact
planes quantised to float32 at 10 and 100 m, an exact axis-aligned plane and line, a thin wire, duplicates, clusters
with k at min_neighbors - 1 .. + 1 and neighbours exactly on the radius, and a well-conditioned box.  Each runs through the
flat kernel at 1-3 rings (dense and sparse cell table), the rows kernel at the default (CAP, U) and at 16,4, the plane
kernel at 5 and 12 rings, the generic walk at 19 rings and under ME_MME_WALK, and the solo lattice; the trace shows which.

Per determined query |e - e_ex| <= B64 + (B32(E) if B32(E) <= 2 tau else 0): the fp32-offset kernels keep a query on the
fast path only while their own certificate is at most tau (kFp64FinishNats), and finish it in fp64 otherwise.  The
generic walk runs on fp64 offsets and must meet B64.  Aggregates: n_valid exact when every query is determined, the sum
and the extrema within the sum and the largest of the per-point bounds.  The fp64 finish must run on the planes of 10 um
and less and the float32-quantised planes, and must not run on the box and on small C4 and C5 scenes at their shipped
noise.  The device accumulators of 2, 3 and 8 ranks and the slab layout carry the same values (the slab layout skips on a
sparse cell table, ME_FORCE_SPARSE)."""
import os
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import dist as mdist

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import exact_ref as X  # noqa: E402
from test_exact_mme import A_DIR, B_DIR, FAR, N_DIR, SCENES, check_mme, exact  # noqa: E402

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
FORCED_SPARSE = bool(os.environ.get("ME_FORCE_SPARSE"))
HOOKS = ("ME_NN_KERNEL", "ME_NN_TILE", "ME_MME_KERNEL", "ME_MME_ROWS", "ME_MME_WALK", "ME_MME_SHARED_LATTICE")
FP64 = "ME_TEV_MME_FP64_FINISH"
MME_SWEEPS = {k for k in A.KERNEL_BITS if k.startswith("ME_KBIT_MME_")}
CELLS_PER_RADIUS = {1: 1.0, 2: 1.7, 3: 2.6, 5: 4.5, 12: 11.3, 19: 19.0}
SHARED = {"ME_MME_SHARED_LATTICE": "1"}

# selector -> (environment, cell table, rings, MME sweep bits, fp32 offsets)
SELECTORS = {
    **{f"flat-r{R}-{t}": (SHARED, t, R, {f"ME_KBIT_MME_FLAT{R}_{t.upper()}"}, True) for R in (1, 2, 3) for t in ("dense", "sparse")},
    "rows-r2": (dict(SHARED, ME_MME_KERNEL="rows"), "dense", 2, {"ME_KBIT_MME_ROWS2"}, True),
    "rows16x4-r3": (dict(SHARED, ME_MME_KERNEL="rows", ME_MME_ROWS="16,4"), "dense", 3, {"ME_KBIT_MME_ROWS3"}, True),
    "plane-r5": (SHARED, "dense", 5, {"ME_KBIT_MME_PLANE"}, True),
    "plane-r12": (SHARED, "dense", 12, {"ME_KBIT_MME_PLANE"}, True),
    "generic-r19": (SHARED, "dense", 19, {"ME_KBIT_MME_GENERIC"}, False),
    "walk-r2": (dict(SHARED, ME_MME_WALK="1"), "dense", 2, {"ME_KBIT_MME_GENERIC"}, False),
    "solo": ({}, "dense", 2, {"ME_KBIT_MME_SOLO", "ME_KBIT_MME_FLAT2_DENSE"}, True),
}
# scenes on which every fp32-offset sweep must hand queries to the fp64 finish, and scenes on which none may
NEEDS_FP64 = {f"plane_{s}_{w}" for s in ("10um", "1um", "0.1um") for w in ("0", "far")} | {"f32_10m", "f32_100m"}
NO_FP64 = {"box"}


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _env(monkeypatch, env):
    for k in HOOKS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _lattice(sel, r):
    """(nn_cell_size to ask for, cell edge and rings of the sweep)"""
    env, table, rings, _, _ = SELECTORS[sel]
    if sel == "solo":      # 4.5 shared cells per radius: the sweep lays the cloud out on a lattice of its own, h = r / 2
        return r / CELLS_PER_RADIUS[5], 0.5 * r, 2
    h = r / CELLS_PER_RADIUS[rings]
    return h, h, rings


def allowance(ex, pts, h, rings, fp32):
    """per-point bound of a sweep on the lattice (h, rings): B64, plus B32(E) where the exact certificate is within 2 tau"""
    if not fp32:
        return ex["b64"], None
    E = X.mme_offset_error(h, rings, pts)
    b32 = np.array([X.mme_fp32_certificate(c, k, E) if v else 0.0 for c, k, v in zip(ex["cov"], ex["k"], ex["valid"])])
    return ex["b64"] + np.where(b32 <= 2 * X.TAU_FP64, b32, 0.0), b32


CASES = [(s, v) for s in SCENES for v in SELECTORS]


@pytest.mark.parametrize("scene,sel", CASES, ids=[f"{s}-{v}" for s, v in CASES])
def test_mme_against_exact(api, monkeypatch, scene, sel):
    env, table, rings, bits, fp32 = SELECTORS[sel]
    if FORCED_SPARSE and table == "dense" and not sel.startswith("generic") and not sel.startswith("walk"):
        pytest.skip("ME_FORCE_SPARSE=1: this path needs a dense cell table")
    pts, r, k, ex = exact(scene)
    cell, h, rings = _lattice(sel, r)
    _env(monkeypatch, env)
    with api.MapEvalB200(nn_cell_size=cell, max_grid_cells=1 if table == "sparse" else 0) as ctx:
        ctx.set_cloud(EST, pts)
        ctx.set_cloud(GT, pts[:10])
        got, ent = ctx.computeMME(EST, r, k, want_entropies=True)
        trace, _ = ctx.kernel_trace(events=True)
    if not FORCED_SPARSE:
        assert trace & MME_SWEEPS == bits, sorted(trace)
    assert got.n_total == len(pts)
    allow, b32 = allowance(ex, pts, h, rings, fp32)
    worst = check_mme(ex, got.n_valid, got.mme, got.min_abs_entropy, got.max_abs_entropy, ent, allow)
    if fp32 and scene in NEEDS_FP64:
        assert FP64 in trace
    if scene in NO_FP64 or not fp32:
        assert FP64 not in trace
    print(f"{scene} {sel}: worst error / bound {worst:.3g}; fp64 finish {'ran' if FP64 in trace else 'did not run'}")


def test_fp64_finish_stays_off_on_shipped_scenes(api, monkeypatch):
    """a C4 window and a C5 room from synth at their shipped noise and radii stay on the fp32-offset sweeps"""
    from cloud_map_evaluation_b200 import synth
    _env(monkeypatch, {})
    for name, scale, window in (("C4", 0.004, None), ("C5", 0.05, 4.0)):
        est, _, cfg = synth.make_pair(name, scale=scale)
        if window:      # a room-sized window of the scene at its full point density
            lo = np.median(est, axis=0)
            est = np.ascontiguousarray(est[np.all(np.abs(est[:, :2] - lo[:2]) < window / 2, axis=1)])
        with api.MapEvalB200() as ctx:
            ctx.set_cloud(EST, est)
            ctx.set_cloud(GT, est[:10])
            got = ctx.computeMME(EST, cfg["nn_radius"], 10)
            trace, _ = ctx.kernel_trace(events=True)
        assert got.n_valid > 0.5 * len(est), name
        assert trace & MME_SWEEPS, name
        assert FP64 not in trace, name


# ---------------------------------------------------------------------------------------------------------------
# device accumulators of many ranks and the slab layout, on a thin plane
# ---------------------------------------------------------------------------------------------------------------
def _thin_scene():
    """a tilted plane with 1 um of normal noise, 0.3 x 16 m (long enough along y and z to be cut into slabs), 1.7 km out"""
    rng = np.random.RandomState(12)
    n = 9000
    uv = np.column_stack([rng.uniform(0, 0.3, n), rng.uniform(0, 16.0, n)])
    pts = uv[:, :1] * A_DIR + uv[:, 1:] * B_DIR + rng.normal(0, 1e-6, (n, 1)) * N_DIR + np.asarray(FAR)
    return np.ascontiguousarray(pts), 0.1, 10


_THIN = {}


def _thin_exact():
    if not _THIN:
        pts, r, k = _thin_scene()
        _THIN["v"] = (pts, r, k, X.mme_exact(pts, r, k))
    return _THIN["v"]


def _view(ptr, n):
    import torch
    return torch.as_tensor(mdist._DeviceBlock(ptr, n), device="cuda:0")


@pytest.mark.parametrize("world,slab", [(2, False), (3, False), (8, False), (2, True), (3, True)])
def test_thin_plane_through_the_device_accumulators(api, monkeypatch, world, slab):
    import torch
    _env(monkeypatch, {})
    pts, r, k, ex = _thin_exact()
    ctxs = [api.MapEvalB200(rank=q, world=world, vmd_voxel_size=0.5) for q in range(world)]
    try:
        trace = set()
        for c in ctxs:
            if slab:
                c.set_layout(A.ME_LAYOUT_SLAB)
            c.set_cloud(EST, pts)
            c.set_cloud(GT, pts[:100])
            c.accum_reset()
            c.eval_mme_accum_device(EST, r, k)
            c.synchronize()
            trace |= c.kernel_trace(events=True)[0]
        if slab and any(c.layout_active()["layout"] != A.ME_LAYOUT_SLAB for c in ctxs):
            assert FORCED_SPARSE, "the slab layout did not engage on a dense cell table"
            pytest.skip("ME_FORCE_SPARSE=1: no slab layout on a sparse cell table")
        blocks = []
        for c in ctxs:
            ptr, n_sum, n_max = c.accum_block()
            blocks.append(_view(ptr, n_sum + n_max))
        red = torch.stack(blocks)
        blocks[0][:n_sum].copy_(red[:, :n_sum].sum(0))
        blocks[0][n_sum:].copy_(red[:, n_sum:].max(0).values)
        torch.cuda.synchronize()
        _, _, (acc,) = ctxs[0].accum_fetch(want_mme=(True, False))
        got = ctxs[0].mme_finalize(acc, EST)
    finally:
        for c in ctxs:
            c.close()
    assert FP64 in trace
    assert acc.n_query == len(pts)
    und, s_b, ext_b = X.mme_aggregate_bounds(ex, ex["b64"])
    nv, s_ex, mn_ex, mx_ex = X.mme_summary(ex)
    assert und == 0 and acc.n_valid == nv, (acc.n_valid, nv, und)
    assert abs(acc.sum_entropy - s_ex) <= s_b, (acc.sum_entropy, s_ex, s_b)
    assert abs(got.min_abs_entropy - mn_ex) <= ext_b and abs(got.max_abs_entropy - mx_ex) <= ext_b

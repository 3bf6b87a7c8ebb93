"""Every sweep kernel of the library against the oracle, on the scenes where kernels go wrong, with the kernel that produced
each result read back from the context (me_kernel_trace).

The NN and MME sweeps pick their kernel from the lattice (dense or sparse cell table, cells along x), the cell occupancy,
the radius-to-cell ratio and the ME_* environment hooks.  Every case below names the ME_KBIT_* path it is written for and
asserts that the trace shows exactly that sweep, so a change of dispatch cannot quietly move a case off its kernel.  The
cases are generated per kernel bit: a bit of the enum without a case fails collection, and the last test checks that the
cases together reached every bit.  Scenes and their oracle results are built once per module and shared by all variants.

Under ME_FORCE_SPARSE=1 (every lattice on the sparse cell table) the cases whose kernel needs a dense table skip."""
import os

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import synth

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
FORCED_SPARSE = bool(os.environ.get("ME_FORCE_SPARSE"))
HOOKS = ("ME_NN_KERNEL", "ME_NN_TILE", "ME_MME_KERNEL", "ME_MME_ROWS", "ME_MME_WALK", "ME_MME_SHARED_LATTICE")
NN_SWEEPS = {"ME_KBIT_NN_ROWS_DENSE", "ME_KBIT_NN_ROWS_SPARSE", "ME_KBIT_NN_FLAT", "ME_KBIT_NN_TILE"}
MME_SWEEPS = {k for k in A.KERNEL_BITS if k.startswith("ME_KBIT_MME_")}
# paths that exist on a dense cell table only (the tile sweep and the slab layout need one)
DENSE_ONLY = {k for k in A.KERNEL_BITS if k.endswith("_DENSE")} | {"ME_KBIT_NN_TILE", "ME_KBIT_NN_BRUTE"}

RTOL = 1e-9          # NN sums: fp64 on both sides, only the summation order differs
RTOL_MME = 1e-7
RTOL_ENT = 1e-6
ENT_FLOOR = -25.0    # below this the neighbourhood covariance is singular to rounding: the entropy is a noise quantity

# --------------------------------------------------------------------------------------------------------------------
# the cases: (scene, selector) -> the trace bits it must show
# --------------------------------------------------------------------------------------------------------------------
# NN selectors: environment, cell table, sweep bit
NN_SELECTORS = {
    "rows-dense": ({}, "dense", "ME_KBIT_NN_ROWS_DENSE"),
    "rows-sparse": ({}, "sparse", "ME_KBIT_NN_ROWS_SPARSE"),
    "flat-dense": ({"ME_NN_KERNEL": "flat"}, "dense", "ME_KBIT_NN_FLAT"),
    "flat-sparse": ({"ME_NN_KERNEL": "flat"}, "sparse", "ME_KBIT_NN_FLAT"),
    "tile-dense": ({"ME_NN_TILE": "1"}, "dense", "ME_KBIT_NN_TILE"),
    # no tile sweep on a sparse table: run_direction falls back to the row walk
    "tile-sparse": ({"ME_NN_TILE": "1"}, "sparse", "ME_KBIT_NN_ROWS_SPARSE"),
    # no hook: the lattice alone decides (>= 2^24 cells along x -> tile sweep)
    "data-dense": ({}, "dense", "ME_KBIT_NN_TILE"),
}
# NN scenes: selectors, and the bits the scene's data must reach whatever the sweep
NN_SCENES = {
    "box": (("rows-dense", "rows-sparse", "flat-dense", "flat-sparse", "tile-dense", "tile-sparse"), set()),
    "ties_auto": (("rows-dense", "rows-sparse", "flat-dense", "flat-sparse", "tile-dense", "tile-sparse"), set()),
    "ties_h004": (("rows-dense", "rows-sparse", "flat-dense", "flat-sparse", "tile-dense", "tile-sparse"), set()),
    "clusters": (("rows-dense", "rows-sparse", "flat-dense", "flat-sparse", "tile-dense", "tile-sparse"),
                 {"ME_KBIT_NN_FAR", "ME_KBIT_NN_FAR_COARSE"}),
    "small_cutoff": (("rows-dense", "rows-sparse", "flat-dense", "flat-sparse", "tile-dense", "tile-sparse"), set()),
    "as_written_ub": (("rows-dense", "rows-sparse", "flat-dense", "flat-sparse", "tile-dense", "tile-sparse"), set()),
    "collinear": (("data-dense", "rows-sparse"), {"ME_KBIT_NN_FAR", "ME_KBIT_NN_FAR_COARSE"}),
}

# MME: rings on the shared lattice -> cells per radius (r / nn_cell_size)
CELLS_PER_RADIUS = {1: 1.0, 2: 1.7, 3: 2.6, 5: 4.5, 12: 11.3, 19: 19.0}
SHARED = {"ME_MME_SHARED_LATTICE": "1"}
ROWS_CFGS = ((12, 2), (8, 2), (16, 2), (12, 4), (16, 4))      # (12, 2) is what ME_MME_KERNEL=rows runs without ME_MME_ROWS


def _mme_selectors():
    """selector -> (environment, cell table, rings, exact set of MME trace bits, (CAP, U) of the rows kernel or None)"""
    sel = {}
    for R in (1, 2, 3):
        for table in ("dense", "sparse"):
            sel[f"flat-r{R}-{table}"] = (SHARED, table, R, {f"ME_KBIT_MME_FLAT{R}_{table.upper()}"}, None)
        for cap, u in ROWS_CFGS:
            env = dict(SHARED, ME_MME_KERNEL="rows")
            if (cap, u) != (12, 2):
                env["ME_MME_ROWS"] = f"{cap},{u}"
            sel[f"rows{cap}x{u}-r{R}"] = (env, "dense", R, {f"ME_KBIT_MME_ROWS{R}"}, (cap, u))
        sel[f"walk-r{R}"] = (dict(SHARED, ME_MME_WALK="1"), "dense", R, {"ME_KBIT_MME_GENERIC"}, None)
    for R in (5, 12):
        sel[f"plane-r{R}"] = (SHARED, "dense", R, {"ME_KBIT_MME_PLANE"}, None)
    sel["generic-r19"] = (SHARED, "dense", 19, {"ME_KBIT_MME_GENERIC"}, None)
    # default path: a radius of 4.5 cells lays the cloud out on a lattice of its own with h = r / 2 (2 rings)
    sel["solo"] = ({}, "dense", 5, {"ME_KBIT_MME_SOLO", "ME_KBIT_MME_FLAT2_DENSE"}, None)
    return sel


MME_SELECTORS = _mme_selectors()
MME_SCENES = {
    "box": tuple(MME_SELECTORS),
    "on_radius_origin": tuple(MME_SELECTORS),
    "on_radius_far": tuple(MME_SELECTORS),
    "near_flat": tuple(MME_SELECTORS),
    "thin_plane": ("flat-r2-dense", "flat-r3-sparse", "rows12x2-r1", "plane-r5", "solo"),
}
# data events (ME_TEV_*) a scene must raise on the sweeps it runs: on a 1 um plane the fp32 offsets cannot certify the
# entropies, so every fp32-offset sweep hands its queries to the fp64 finish
MME_SCENE_EVENTS = {"thin_plane": {"ME_TEV_MME_FP64_FINISH"}}
# the collinear cloud reaches the generic kernel through its lattice (>= 2^24 cells along x), without a hook
COLLINEAR_MME_BITS = {"ME_KBIT_MME_GENERIC"}
SCS_RADII = {5: "ME_KBIT_SCS_R5", 2: "ME_KBIT_SCS_RT_CACHED", 7: "ME_KBIT_SCS_RT_UNCACHED"}
SLAB_BITS = {"ME_KBIT_NN_BRUTE", "ME_KBIT_NN_ROWS_DENSE", "ME_KBIT_NN_FAR"}

NN_CASES = [(s, v, {NN_SELECTORS[v][2]} | extra) for s, (sels, extra) in NN_SCENES.items() for v in sels]
MME_CASES = [(s, v, MME_SELECTORS[v][3]) for s, sels in MME_SCENES.items() for v in sels] + \
            [("collinear", "data", COLLINEAR_MME_BITS)]
SCS_CASES = [(r, {b}) for r, b in SCS_RADII.items()]
ALL_CASE_BITS = {**{f"nn[{s}-{v}]": b for s, v, b in NN_CASES}, **{f"mme[{s}-{v}]": b for s, v, b in MME_CASES},
                 **{f"scs[{r}]": b for r, b in SCS_CASES}, "slab": SLAB_BITS}


def _check_coverage():
    """every kernel bit has at least one case (a bit without one fails collection), and no case names an unknown bit"""
    named = set().union(*ALL_CASE_BITS.values())
    unknown = named - set(A.KERNEL_BITS)
    missing = set(A.KERNEL_BITS) - named
    if unknown or missing:
        raise AssertionError(f"kernel bits without a (scene, selector) case: {sorted(missing)}; unknown bits: {sorted(unknown)}")


_check_coverage()

# what the cases of this module ran: case id -> the trace bits they recorded / the bits of the cases that skipped
_REACHED = {}
_SKIPPED = {}


def _enter(case_id, bits, dense_data=False):
    """skip a case whose kernel needs a dense table when every lattice is forced onto the sparse one"""
    if FORCED_SPARSE and (bits & DENSE_ONLY or dense_data):
        _SKIPPED[case_id] = bits
        pytest.skip("ME_FORCE_SPARSE=1: this path needs a dense cell table")
    _REACHED[case_id] = set()


def _env(monkeypatch, env):
    for k in HOOKS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


# --------------------------------------------------------------------------------------------------------------------
# scenes
# --------------------------------------------------------------------------------------------------------------------
def _f32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32).astype(np.float64))


def _ties(cell):
    """both clouds on a regular 4 cm lattice 512 m / -2 km from the origin; est on the cell centres (8-way ties) plus exact
    coincidences"""
    s = np.float32(0.04)
    g = np.arange(20, dtype=np.float32) * s
    a = np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3)
    off = np.array((512.5, -2048.25, 33.0), dtype=np.float32)
    gt = _f32(a + off)
    est = np.concatenate([_f32(a + off + np.float32(0.02)), gt[::7]])
    return est, gt, A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], 1.0, pairing=A.ME_PAIRING_GEOMETRIC), cell


COLLINEAR_CELL = 1e-6


def _collinear():
    """three 1 mm segments along x at 0, 9 and 18 m (spacing ~3e-7 m), y and z within 1e-7 m, and est points in the gaps.
    With 1 um cells the lattice has 1.8e7 >= 2^24 cells along x: more than the fp32 x index of the flat / rows sweeps
    holds, so the NN sweep takes the tile kernel and the MME sweep (3 rings) the generic one; the gap points leave the
    searched blocks and go through the far kernel's coarse phase (blocks of 2^17 cells along x, one row deep)."""
    rng = np.random.RandomState(21)

    def seg(n):
        x = np.concatenate([x0 + np.sort(rng.rand(n)) * 1e-3 for x0 in (0.0, 9.0, 18.0)])
        yz = 0.25 + rng.rand(len(x), 2) * 1e-7
        return np.column_stack([x, yz])

    gt = seg(3000)
    est = gt + np.column_stack([rng.randn(len(gt)) * 1e-7, np.zeros((len(gt), 2))])
    gap = np.column_stack([np.concatenate([rng.uniform(0.5, 8.5, 10), rng.uniform(9.5, 17.5, 10)]), np.full((20, 2), 0.25)])
    est = np.ascontiguousarray(np.concatenate([est, gap]))
    return est, np.ascontiguousarray(gt), A.make_nn_params([1e-6, 5e-7, 3e-7, 2e-7, 1e-7], 1e-10,
                                                           pairing=A.ME_PAIRING_GEOMETRIC), COLLINEAR_CELL


def _nn_scene(name):
    if name == "box":
        est, gt, cfg = synth.make_pair("C2", scale=0.1)
        return est, gt, A.make_nn_params(cfg["tau"], 1.0, pairing=A.ME_PAIRING_GEOMETRIC), 0.0
    if name == "ties_auto":
        return _ties(0.0)
    if name == "ties_h004":
        return _ties(0.04)      # cell faces through the lattice points
    if name == "clusters":
        # clustered ground truth (> 256 cells along x and y at 5 cm: the far kernel has a coarse grid), duplicated
        # reference points, exact coincidences, and outliers tens of metres from every cluster
        rng = np.random.RandomState(5)
        gt = np.concatenate([rng.randn(20000, 3) * 0.3 + c for c in ([0, 0, 0], [9, 1, -2], [-4, 12, 1])])
        gt = np.concatenate([gt, gt[:100]])
        lo, hi = np.array([-12.0, -10.0, -14.0]), np.array([18.0, 20.0, 14.0])
        est = np.concatenate([gt[::3] + rng.randn(len(gt[::3]), 3) * 0.01, lo + rng.rand(3000, 3) * (hi - lo), gt[:50]])
        return _f32(est), _f32(gt), A.make_nn_params([0.5, 0.3, 0.2, 0.1, 0.05], 1.0, pairing=A.ME_PAIRING_GEOMETRIC), 0.05
    if name in ("small_cutoff", "as_written_ub"):
        side = synth.box_side_for_density(60000)
        gt = synth.uniform_box(60000, side, 11)
        est = synth.uniform_box(83211, side, 12, noise_sigma=0.02)
        if name == "small_cutoff":      # sqrt(R) = 3 cm, as-written pairing with more est than gt points
            return est, gt, A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], 0.0009, pairing=A.ME_PAIRING_AS_WRITTEN), 0.0
        # roles swapped (n_est < n_gt): the reference's as-written lookups run out of range (n_ub > 0)
        return gt, est, A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], 1.0, pairing=A.ME_PAIRING_AS_WRITTEN), 0.0
    if name == "collinear":
        return _collinear()
    raise KeyError(name)


def _mme_scene(name):
    """(points, radius, min_neighbors, per-point rtol)"""
    if name == "box":
        est, _, cfg = synth.make_pair("C2", scale=0.1)
        return est, cfg["nn_radius"], 10, RTOL_ENT
    if name.startswith("on_radius"):
        # regular lattice with spacing r / 2 (fp32 coordinates, some points a hair off): thousands of pairs at, or one
        # rounding away from, d2 == r2 — every one must reach the exact fp64 test
        s = np.float32(0.05)
        g = np.arange(24, dtype=np.float32) * s
        pts = np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3)
        rng = np.random.RandomState(5)
        pts = pts + (rng.rand(*pts.shape) < 0.3) * rng.normal(0, 1e-7, pts.shape).astype(np.float32)
        origin = (0.0, 0.0, 0.0) if name == "on_radius_origin" else (-731.25, 1203.5, 88.125)
        return _f32(pts + np.array(origin, dtype=np.float32)), float(np.float64(np.float32(0.1))), 10, RTOL_ENT
    if name == "near_flat":
        # a tilted plane at 1 cm spacing with 0.2 mm noise 1.4 km out, k >= 5: lambda_1 / lambda_3 ~ 6e4 amplifies the
        # rounding of the accumulated offsets, which test_mme_on_nearly_flat_surfaces bounds at 2e-6 per point
        n = 160_000
        idx = np.arange(n, dtype=np.uint64)
        u = synth.uniform24(77, idx, 0).astype(np.float64) * 4.0
        v = synth.uniform24(77, idx, 1).astype(np.float64) * 4.0
        w = 2e-4 * synth.gaussian(77, idx, 8)
        a, b = np.array([0.8, 0.36, 0.48]), np.array([-0.6, 0.48, 0.64])
        pts = u[:, None] * a + v[:, None] * b + w[:, None] * np.cross(a, b) + np.array([731.25, -1204.5, 88.0])
        return _f32(pts), 0.1, 5, 2e-6
    if name == "thin_plane":
        # the near-flat plane with 1 um of normal noise
        n = 40_000
        idx = np.arange(n, dtype=np.uint64)
        u = synth.uniform24(78, idx, 0).astype(np.float64) * 2.0
        v = synth.uniform24(78, idx, 1).astype(np.float64) * 2.0
        w = 1e-6 * synth.gaussian(78, idx, 8)
        a, b = np.array([0.8, 0.36, 0.48]), np.array([-0.6, 0.48, 0.64])
        pts = u[:, None] * a + v[:, None] * b + w[:, None] * np.cross(a, b) + np.array([731.25, -1204.5, 88.0])
        return np.ascontiguousarray(pts), 0.1, 10, RTOL_ENT
    if name == "collinear":
        est = _collinear()[0]
        return est, 2.5e-6, 10, RTOL_ENT
    raise KeyError(name)


class _Scenes:
    """scenes and their oracle results, built on first use and shared by every variant of the module"""

    def __init__(self, O):
        self.O = O
        self.nn, self.mme, self.scs = {}, {}, {}

    def get_nn(self, name):
        if name not in self.nn:
            est, gt, p, cell = _nn_scene(name)
            exp, ie, ig = self.O.eval_nn(est, gt, p, want_indices=True)
            _, d2e = self.O.knn1(est, gt)
            _, d2g = self.O.knn1(gt, est)
            self.nn[name] = (est, gt, p, cell, exp, (ie, d2e), (ig, d2g))
        return self.nn[name]

    def get_mme(self, name):
        if name not in self.mme:
            pts, r, k, rtol = _mme_scene(name)
            exp, oent = self.O.eval_mme(pts, r, k, want_entropies=True)
            self.mme[name] = (pts, r, k, rtol, exp, oent)
        return self.mme[name]

    def get_scs(self):
        if not self.scs:
            est, gt, cfg = synth.make_pair("C2", scale=0.1)
            self.scs["scene"] = (est, gt, cfg["vmd_voxel_size"])
        return self.scs["scene"]


@pytest.fixture(scope="module")
def scenes():
    from oracle import oracle
    return _Scenes(oracle)


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _cmp_dir(got, exp):
    assert (got.n_source, got.n_corr, got.n_ub) == (exp.n_source, exp.n_corr, exp.n_ub)
    assert list(got.n_inlier) == list(exp.n_inlier)
    for k in ("mean", "rmse", "fitness", "sigma"):
        np.testing.assert_allclose(list(getattr(got, k)), list(getattr(exp, k)), rtol=RTOL, atol=1e-300, equal_nan=True,
                                   err_msg=k)
    np.testing.assert_allclose(got.sum_nn_dist, exp.sum_nn_dist, rtol=RTOL)


def _cmp_nn(got, exp):
    _cmp_dir(got.est_to_gt, exp.est_to_gt)
    _cmp_dir(got.gt_to_est, exp.gt_to_est)
    for k in ("cd", "f1", "iou"):
        np.testing.assert_allclose(list(getattr(got, k)), list(getattr(exp, k)), rtol=RTOL, equal_nan=True, err_msg=k)
    np.testing.assert_allclose(got.full_cd, exp.full_cd, rtol=RTOL)


# --------------------------------------------------------------------------------------------------------------------
# NN: indices and squared distances of both directions bit-identical, counts exact, sums to 1e-9
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene,sel,bits", NN_CASES, ids=[f"{s}-{v}" for s, v, _ in NN_CASES])
def test_nn_kernel(api, scenes, monkeypatch, scene, sel, bits):
    case = f"nn[{scene}-{sel}]"
    _enter(case, bits, dense_data=sel.startswith("data"))
    env, table, sweep = NN_SELECTORS[sel]
    est, gt, p, cell, exp, (ie, d2e), (ig, d2g) = scenes.get_nn(scene)
    _env(monkeypatch, env)
    with api.MapEvalB200(nn_cell_size=cell, max_grid_cells=1 if table == "sparse" else 0) as ctx:
        ctx.set_cloud(EST, est)
        ctx.set_cloud(GT, gt)
        e, g = ctx.eval_nn_accum(p)
        got = ctx.nn_finalize(p, e, g)
        nn_e, nn_g = ctx.get_nn(EST), ctx.get_nn(GT)
        trace, _ = ctx.kernel_trace()
    _REACHED[case] = trace
    assert trace & NN_SWEEPS == {sweep}, sorted(trace)
    assert bits <= trace, sorted(bits - trace)
    if scene == "clusters":
        assert e.n_far > 1000
    if scene == "as_written_ub":
        assert exp.gt_to_est.n_ub > 0
    _cmp_nn(got, exp)
    np.testing.assert_array_equal(nn_e[0], ie)
    np.testing.assert_array_equal(nn_e[1], d2e)
    np.testing.assert_array_equal(nn_g[0], ig)
    np.testing.assert_array_equal(nn_g[1], d2g)


# --------------------------------------------------------------------------------------------------------------------
# MME: n_valid, n_total and the non-zero pattern exact; entropies to 1e-6 where well conditioned; mme to 1e-7
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene,sel,bits", MME_CASES, ids=[f"{s}-{v}" for s, v, _ in MME_CASES])
def test_mme_kernel(api, scenes, monkeypatch, scene, sel, bits):
    case = f"mme[{scene}-{sel}]"
    _enter(case, bits, dense_data=scene == "collinear")
    pts, r, k, rtol, exp, oent = scenes.get_mme(scene)
    if scene == "collinear":
        env, table, cell, cfg = {}, "dense", COLLINEAR_CELL, None
    else:
        env, table, rings, _, cfg = MME_SELECTORS[sel]
        cell = r / CELLS_PER_RADIUS[rings]
    _env(monkeypatch, env)
    with api.MapEvalB200(nn_cell_size=cell, max_grid_cells=1 if table == "sparse" else 0) as ctx:
        ctx.set_cloud(EST, pts)
        ctx.set_cloud(GT, pts[:10])
        got, ent = ctx.computeMME(EST, r, k, want_entropies=True)
        trace, rows_cfg = ctx.kernel_trace(events=True)
    events = trace - set(A.KERNEL_BITS)
    trace = trace & set(A.KERNEL_BITS)
    _REACHED[case] = trace
    assert trace & MME_SWEEPS == bits, sorted(trace)
    assert MME_SCENE_EVENTS.get(scene, set()) <= events, sorted(events)
    assert rows_cfg == cfg
    assert (got.n_valid, got.n_total) == (exp.n_valid, exp.n_total)
    np.testing.assert_array_equal(ent != 0, oent != 0)
    ok = oent > ENT_FLOOR
    np.testing.assert_allclose(ent[ok], oent[ok], rtol=rtol, atol=0)
    if np.all(oent[oent != 0] > ENT_FLOOR):
        np.testing.assert_allclose(got.mme, exp.mme, rtol=RTOL_MME)
        np.testing.assert_allclose([got.min_abs_entropy, got.max_abs_entropy], [exp.min_abs_entropy, exp.max_abs_entropy],
                                   rtol=rtol)


# --------------------------------------------------------------------------------------------------------------------
# SCS: the compiled radius, and run-time radii with and without the per-lane cache
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("radius,bits", SCS_CASES, ids=[str(r) for r, _ in SCS_CASES])
def test_scs_kernel(api, scenes, monkeypatch, radius, bits):
    case = f"scs[{radius}]"
    _enter(case, bits)
    est, gt, v = scenes.get_scs()
    _env(monkeypatch, {})
    with api.MapEvalB200(vmd_voxel_size=v) as ctx:
        ctx.set_cloud(EST, est)
        ctx.set_cloud(GT, gt)
        got = ctx.calculateVMD(v, 40, radius)
        trace, _ = ctx.kernel_trace()
    _REACHED[case] = trace
    assert trace & {b for b in A.KERNEL_BITS if b.startswith("ME_KBIT_SCS_")} == bits
    exp = scenes.O.eval_awd(est, gt, v, 40, radius)
    assert (got.n_pairs, got.n_scs, got.n_active, got.n_old, got.n_new) == \
           (exp.n_pairs, exp.n_scs, exp.n_active, exp.n_old, exp.n_new)
    assert got.n_scs > 50
    np.testing.assert_allclose([got.awd, got.scs], [exp.awd, exp.scs], rtol=RTOL)


# --------------------------------------------------------------------------------------------------------------------
# slab layout: queries whose nearest neighbour lies on another rank's slab are finished over the whole cloud
# --------------------------------------------------------------------------------------------------------------------
def test_nn_slab_brute_finish(api, scenes, monkeypatch):
    """The ground truth covers the south half of the scene only: the nearest neighbour of most northern est points lies on
    the other rank's slab.  Two contexts stand in for the ranks; their per-point results together must be the oracle's,
    and their accumulators summed its statistics."""
    _enter("slab", SLAB_BITS)
    _env(monkeypatch, {})
    est, gt, cfg = synth.make_pair("C4", scale=0.004)
    gt = np.ascontiguousarray(gt[gt[:, 1] < 90.0])
    rs = np.random.RandomState(5)
    out = np.column_stack([rs.uniform(1, 199, 300), rs.uniform(1, 199, 300), rs.uniform(0.5, 6, 300)])
    est = np.ascontiguousarray(np.vstack([est, _f32(out)]))
    p = A.make_nn_params(cfg["tau"], 1.0, pairing=A.ME_PAIRING_GEOMETRIC)
    world = 2
    trace = set()
    tot_e, tot_g = A.me_nn_accum(), A.me_nn_accum()
    per_rank = []
    for r in range(world):
        with api.MapEvalB200(rank=r, world=world, vmd_voxel_size=cfg["vmd_voxel_size"], nn_cell_size=0.5) as ctx:
            ctx.set_layout(A.ME_LAYOUT_SLAB)
            ctx.set_cloud(EST, est)
            ctx.set_cloud(GT, gt)
            e, g = ctx.eval_nn_accum(p)
            assert ctx.layout_active()["layout"] == A.ME_LAYOUT_SLAB
            per_rank.append((ctx.get_nn(EST), ctx.get_nn(GT)))
            trace |= ctx.kernel_trace()[0]
            for tot, part in ((tot_e, e), (tot_g, g)):
                for name, _ in A.me_nn_accum._fields_:
                    v = getattr(part, name)
                    if hasattr(v, "__len__"):
                        for i in range(len(v)):
                            getattr(tot, name)[i] += v[i]
                    else:
                        setattr(tot, name, getattr(tot, name) + v)
            if r == world - 1:
                got = ctx.nn_finalize(p, tot_e, tot_g)
    _REACHED["slab"] = trace
    assert SLAB_BITS <= trace, sorted(SLAB_BITS - trace)
    assert tot_e.n_query == len(est) and tot_g.n_query == len(gt)
    _cmp_nn(got, scenes.O.eval_nn(est, gt, p))
    for d, (q, ref) in enumerate(((est, gt), (gt, est))):
        oi, od2 = scenes.O.knn1(q, ref)
        idx = np.stack([pr[d][0] for pr in per_rank])
        d2 = np.stack([pr[d][1] for pr in per_rank])
        evaluated = ~np.isnan(d2)
        assert np.all(evaluated.sum(0) == 1)            # every query evaluated by exactly one rank
        sel = evaluated.argmax(0)
        cols = np.arange(d2.shape[1])
        np.testing.assert_array_equal(d2[sel, cols], od2)
        np.testing.assert_array_equal(idx[sel, cols], oi)


# --------------------------------------------------------------------------------------------------------------------
def test_every_kernel_bit_was_reached():
    """The cases of this module together ran every path of the enum (under ME_FORCE_SPARSE=1: every path that exists on a
    sparse table)."""
    ran = set(_REACHED) | set(_SKIPPED)
    if ran != set(ALL_CASE_BITS):
        pytest.skip("needs every case of the module in the same session")
    assert not _SKIPPED or FORCED_SPARSE, sorted(_SKIPPED)
    reached = set().union(*_REACHED.values())
    skipped = set().union(*_SKIPPED.values()) if _SKIPPED else set()
    missing = set(A.KERNEL_BITS) - reached - skipped
    assert not missing, sorted(missing)
    if not FORCED_SPARSE:
        assert reached == set(A.KERNEL_BITS)

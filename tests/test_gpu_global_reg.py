"""me_global_registration on the device against the numpy statement tests/fpfh_ref.py, stage by stage with each stage's
input taken from the device (so that one stage's rounding cannot hide another's error), and the recovery of large
rigid motions of a furnished indoor scene."""
import math
import os
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fpfh_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
VOX = 0.5


def _api():
    from cloud_map_evaluation_b200 import api
    return api


def _rot(yaw, tilt_x=0.0, tilt_y=0.0):
    cz, sz, cx, sx, cy, sy = math.cos(yaw), math.sin(yaw), math.cos(tilt_x), math.sin(tilt_x), math.cos(tilt_y), math.sin(tilt_y)
    return np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) @ \
        np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])


def _motion(yaw_deg, tilt_deg, t):
    M = np.eye(4)
    M[:3, :3] = _rot(math.radians(yaw_deg), math.radians(tilt_deg), math.radians(-0.6 * tilt_deg))
    M[:3, 3] = t
    return M


def _apply(M, xyz):
    return np.ascontiguousarray(xyz @ M[:3, :3].T + M[:3, 3])


def _errors(T, T_true):
    dR = T[:3, :3] @ T_true[:3, :3].T
    ang = math.degrees(math.acos(max(-1.0, min(1.0, (np.trace(dR) - 1) / 2))))
    return ang, float(np.linalg.norm(T[:3, 3] - T_true[:3, 3]))


def _furnished_rooms(n, seed, noise):
    """indoor rooms (a 4 x 4 grid of identical 8 x 8 x 3 m rooms is symmetric under quarter turns) with 40 boxes placed
    at random, which make the pose unique"""
    rooms = synth.indoor_scene(int(n * 0.8), seed, noise, rooms=4)
    rng = np.random.RandomState(99)
    idx = np.arange(n - len(rooms), dtype=np.uint64)
    u = [synth.uniform24(seed + 7, idx, k).astype(np.float64) for k in range(4)]
    box = np.minimum((u[3] * 40).astype(np.int64), 39)
    centre = rng.uniform(1.0, 31.0, (40, 2))
    size = rng.uniform(0.4, 1.6, (40, 3))
    face = (u[2] * 6).astype(np.int64)
    loc = np.stack([u[0], u[1]], 1)
    p = np.zeros((len(idx), 3))
    for a in range(3):
        p[:, a] = np.where(face // 2 == a, (face % 2).astype(np.float64), 0.0)
    free = [[1, 2], [0, 2], [0, 1]]
    for a in range(3):
        for k, b in enumerate(free[a]):
            sel = face // 2 == a
            p[sel, b] = loc[sel, k]
    xyz = np.c_[centre[box, 0] - size[box, 0] / 2 + p[:, 0] * size[box, 0],
                centre[box, 1] - size[box, 1] / 2 + p[:, 1] * size[box, 1], p[:, 2] * size[box, 2]]
    if noise > 0:
        for a in range(3):
            xyz[:, a] += noise * synth.gaussian(seed + 7, idx, 8 + 2 * a)
    return np.ascontiguousarray(np.r_[rooms, xyz.astype(np.float32).astype(np.float64)])


def _site(n, seed, noise):
    """a 250 x 250 m piece of the site survey, moved to about 1.5 km from the origin"""
    xyz = synth.site_scene(n * 16, seed, noise)
    keep = (xyz[:, 0] > 650) & (xyz[:, 0] < 900) & (xyz[:, 1] > 600) & (xyz[:, 1] < 850)
    return np.ascontiguousarray(xyz[keep] + [700.0, 550.0, 0.0])


# (generator, feature voxel): the site piece holds ~4 points per m^2, so its features are taken at 1 m
SCENES = {
    "indoor": (lambda seed, noise: _furnished_rooms(400_000, seed, noise), 0.5),
    "outdoor": (lambda seed, noise: synth.outdoor_scene(600_000, seed, noise), 0.5),
    "site": (lambda seed, noise: _site(240_000, seed, noise), 1.0),
}


@pytest.fixture(scope="module", params=sorted(SCENES))
def scene(request):
    gen, vox = SCENES[request.param]
    gt = gen(synth.GT_SEED, 0.002)
    est = gen(synth.EST_SEED, 0.01)
    lo, hi = est.min(0), est.max(0)
    est = np.ascontiguousarray(est[est[:, 0] < lo[0] + 0.6 * (hi[0] - lo[0])])        # about 60 % of the ground truth
    return request.param, est, gt, vox


# ---- recovery ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("yaw", [0.0, 45.0, 90.0, 180.0, -131.7])
def test_recovery(scene, yaw):
    name, est0, gt, vox = scene
    M = _motion(yaw, 4.0 if yaw else 0.0, [63.0, -77.0, 4.5] if yaw else [0.0, 0.0, 0.0])
    est = _apply(M, est0)
    T_true = np.linalg.inv(M)
    with _api().MapEvalB200(device=0) as ctx:
        ctx.set_cloud(EST, est)
        ctx.set_cloud(GT, gt)
        r = ctx.global_registration(vox, seed=5)
        ang, dt = _errors(r["T"], T_true)
        assert ang <= 2.0 and dt <= 2 * vox, (name, yaw, ang, dt, r)
        T_icp, res = ctx.performICPRegistration(1.0, T_init=r["T"], method=A.ME_ICP_GENERALIZED)
        ang, dt = _errors(T_icp, T_true)
        assert ang <= 0.05 and dt <= 0.01, (name, yaw, ang, dt)
    if yaw:
        with _api().MapEvalB200(device=0) as ctx:                 # ICP alone from the identity misses
            ctx.set_cloud(EST, est)
            ctx.set_cloud(GT, gt)
            T_icp, _ = ctx.performICPRegistration(1.0, method=A.ME_ICP_GENERALIZED)
            ang, dt = _errors(T_icp, T_true)
            assert ang > 2.0 or dt > 1.0


# ---- stage by stage, small scene -------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["dense", "sparse"])
def staged(request):
    if request.param == "sparse":
        os.environ["ME_FORCE_SPARSE"] = "1"
    try:
        gt = synth.indoor_scene(120_000, synth.GT_SEED, 0.002, rooms=3)
        est = _apply(_motion(70.0, 3.0, [20.0, -35.0, 2.0]), synth.indoor_scene(90_000, synth.EST_SEED, 0.01, rooms=3))
        with _api().MapEvalB200(device=0) as ctx:
            ctx.set_cloud(EST, est)
            ctx.set_cloud(GT, gt)
            r = ctx.global_registration(VOX, seed=21, n_hypotheses=20000)
            r2 = ctx.global_registration(VOX, seed=21, n_hypotheses=20000)
            feats = [ctx.get_features(w) for w in (EST, GT)]
            corr = ctx.get_correspondences()
            # the reference inputs of stage 1: me_voxel_downsample and me_estimate_normals on the context's own slots
            ref = []
            for w, cloud in ((EST, est), (GT, gt)):
                with _api().MapEvalB200(device=0) as c2:
                    c2.set_cloud(w, cloud)
                    c2.voxel_downsample(w, VOX)
                    ref.append((c2.get_cloud(w), c2.estimate_normals(w, 30)))
        yield dict(r=r, r2=r2, feats=feats, ref=ref, corr=corr)
    finally:
        os.environ.pop("ME_FORCE_SPARSE", None)


def test_features_and_normals(staged):
    for (xyz, nrm, _), (rxyz, rnrm) in zip(staged["feats"], staged["ref"]):
        np.testing.assert_array_equal(xyz, rxyz)
        oriented, amb = R.orient_normals(rxyz, rnrm)
        assert amb.sum() == 0
        np.testing.assert_array_equal(nrm, oriented)


def test_fpfh(staged):
    for xyz, nrm, f in staged["feats"]:
        f32, f64, flagged, _ = R.features(xyz, nrm, 10 * VOX, 128)
        ok = ~flagged
        assert flagged.sum() <= 2, flagged.sum()
        err = np.abs(f[ok].astype(np.float64) - f64[ok])
        assert (err <= 0.5 * np.spacing(np.abs(f64[ok]).astype(np.float32)) + 1e-9).all()


def test_correspondences_ransac_and_refinement(staged):
    (xe, _, fe), (xg, _, fg) = staged["feats"]
    r = staged["r"]
    ie, ig = R.correspondences(fe, fg)
    assert r["n_correspondences"] == len(ie)
    np.testing.assert_array_equal(staged["corr"][0], ie)             # the pairs themselves, in est order
    np.testing.assert_array_equal(staged["corr"][1], ig)
    P, Q = xe[ie], xg[ig]
    c = 0.5 * (xg.min(0) + xg.max(0))
    res = R.ransac(P, Q, c, 21, 20000, 0.9, (1.5 * VOX) ** 2)
    assert r["n_valid_hypotheses"] == res["n_valid"]
    assert r["best_hypothesis"] == res["best"]
    T, n_in, rmse = R.refine(P, Q, c, res["T"][res["best"]], (1.5 * VOX) ** 2)
    assert r["n_inliers"] == n_in
    np.testing.assert_allclose(r["T"], T, rtol=0, atol=1e-12)
    np.testing.assert_allclose(r["inlier_rmse"], rmse, rtol=1e-12)
    # the same bits from a second call with the same seed
    np.testing.assert_array_equal(r["T"], staged["r2"]["T"])
    assert {k: v for k, v in r.items() if k not in ("T", "stage_ms")} == \
        {k: v for k, v in staged["r2"].items() if k not in ("T", "stage_ms")}


def _close(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], dict):
            _close(a[k], b[k])
        elif np.asarray(a[k]).dtype.kind in "iu":
            assert a[k] == b[k], k
        else:
            np.testing.assert_allclose(a[k], b[k], rtol=1e-12, atol=0, err_msg=k)


def test_the_context_clouds_are_left_alone():
    gt = synth.indoor_scene(100_000, synth.GT_SEED, 0.002, rooms=3)
    est = synth.indoor_scene(100_000, synth.EST_SEED, 0.01, rooms=3)
    p = A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], 1.0, pairing=A.ME_PAIRING_GEOMETRIC)

    def full_pass(ctx):
        nn = A.struct_to_dict(ctx.calculateMetricsWithInitialMatrix(p))
        idx, d2 = ctx.get_nn(EST)
        mme, ent = ctx.computeMME(EST, 0.3, 10, want_entropies=True)
        awd = A.struct_to_dict(ctx.calculateVMD(0.5, 20, 5))
        return nn, idx, d2, A.struct_to_dict(mme), ent, awd, ctx.get_cloud(EST), ctx.get_normals(GT)

    with _api().MapEvalB200(device=0, vmd_voxel_size=0.5) as ctx:
        ctx.set_cloud(EST, est)
        ctx.set_cloud(GT, gt)
        ctx.estimate_normals(GT, 20)
        before = full_pass(ctx)
        ctx.global_registration(VOX, seed=1, n_hypotheses=5000)
        after = full_pass(ctx)
    # per-point results, counts, clouds and normals bit for bit; the floating aggregates are sums the sweeps accumulate
    # with atomics, whose order (and with it the last bits) varies between any two passes
    for a, b in zip(before, after):
        if isinstance(a, dict):
            _close(a, b)
        else:
            np.testing.assert_array_equal(a, b)


def test_errors():
    api = _api()
    gt = synth.indoor_scene(50_000, synth.GT_SEED, 0.002, rooms=2)
    with api.MapEvalB200(device=0) as ctx:
        ctx.set_cloud(GT, gt)
        with pytest.raises(api.MapEvalError) as e:                # no estimate
            ctx.global_registration(VOX)
        assert e.value.code == A.ME_ERR_EMPTY
        with pytest.raises(api.MapEvalError) as e:                # nothing computed yet
            ctx.get_features(EST)
        assert e.value.code == A.ME_ERR_INVALID
        ctx.set_cloud(EST, gt[:2])
        with pytest.raises(api.MapEvalError) as e:                # two points: at most two correspondences
            ctx.global_registration(VOX)
        assert e.value.code == A.ME_ERR_INVALID and "correspondences" in str(e.value)
        moved = _apply(_motion(30.0, 0.0, [1.0, 2.0, 0.0]), gt)
        ctx.set_cloud(EST, moved)
        with pytest.raises(api.MapEvalError) as e:                # ratio 1: no two edges of a moved map agree exactly
            ctx.global_registration(VOX, n_hypotheses=10, edge_ratio=1.0)
        assert e.value.code == A.ME_ERR_INVALID and "no valid" in str(e.value)
        with pytest.raises(api.MapEvalError) as e:
            ctx.global_registration(VOX, edge_ratio=1.5)
        assert e.value.code == A.ME_ERR_INVALID
        with pytest.raises(api.MapEvalError) as e:
            ctx.global_registration(-1.0)
        assert e.value.code == A.ME_ERR_INVALID
        n = ctx.n[EST]
        np.testing.assert_array_equal(ctx.get_cloud(EST), moved)  # the failures left the clouds alone
        assert n == len(moved)

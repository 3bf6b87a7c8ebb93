"""me_voxel_downsample on the device against the numpy statement tests/downsample_ref.py, bit for bit: the points, the
normals and the number of voxels, at every key width the packed key can take (1 to 8 radix passes), at the per-axis
limit, on voxel faces to the ulp, on voxels whose sums change with the order of their members, at sizes around the
2048-key tiles of the sort and the scan and above 2^24 points, and on a borrowed cloud.  The same sizes run through
me_add_non_uniform_density, whose compaction shares the scan (tests/perturb_ref.py)."""
import os
import sys
import time

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import downsample_ref as ref  # noqa: E402
import perturb_ref  # noqa: E402

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
FAR = np.array([1500.0, -1500.0, 1500.0])


def _api():
    from cloud_map_evaluation_b200 import api
    return api


def _assert_bits(got, exp, what):
    assert got.shape == exp.shape, f"{what}: shape {got.shape} != {exp.shape}"
    bad = (np.ascontiguousarray(got).view(np.uint64) != np.ascontiguousarray(exp).view(np.uint64)).any(1)
    assert not bad.any(), f"{what}: {bad.sum()} of {len(bad)} rows differ, first at {np.flatnonzero(bad)[:5]}"


def _normals(n, seed, nan_share=0.05):
    rng = np.random.RandomState(seed)
    nrm = rng.randn(n, 3)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    nrm[rng.rand(n) < nan_share, rng.randint(0, 3)] = np.nan
    return nrm


def _check(xyz, s, nrm=None, what=""):
    """down-sample a library-owned copy and compare it with the statement; returns the statement's voxel counts"""
    with _api().MapEvalB200() as ctx:
        ctx.set_cloud(EST, xyz)
        if nrm is not None:
            ctx.set_normals(EST, nrm)
        n = ctx.voxel_downsample(EST, s)
        pts = ctx.get_cloud(EST)
        nr = ctx.get_normals(EST) if nrm is not None else None
    ep, en, cnt = ref.voxel_downsample(xyz, s, nrm)
    assert n == len(ep) == len(pts), what
    _assert_bits(pts, ep, f"{what} points")
    if nrm is not None:
        _assert_bits(nr, en, f"{what} normals")
    return cnt


def _check_density(xyz, region, seed=synth.EST_SEED, device_tensor=None):
    """me_add_non_uniform_density keeps exactly the statement's points, in input order (the compaction's scan)"""
    keep, xn, yn = perturb_ref.density_keep(xyz, 0.3, 0.8, region, seed)
    tiny = ((np.abs(xn) < 1e-9) & (xn != 0)) | ((np.abs(yn) < 1e-9) & (yn != 0))
    assert tiny.sum() == 0                   # where device and host sin could disagree in sign: none on these scenes
    with _api().MapEvalB200() as ctx:
        if device_tensor is None:
            ctx.set_cloud(GT, xyz)
        else:
            ctx.set_cloud_device(GT, device_tensor.data_ptr(), len(xyz), keepalive=device_tensor)
        ctx.copy_cloud(GT, EST)
        n = ctx.add_non_uniform_density(EST, 0.3, 0.8, region, seed)
        got = ctx.get_cloud(EST)
    assert n == keep.sum() > 0
    assert n < len(xyz) or len(xyz) < 100
    _assert_bits(got, xyz[keep], "kept points")


# ---- a. key widths: 1 to 8 radix passes ---------------------------------------------------------------------------------
# bits per axis; the packed key has their sum, the sort runs ceil(sum / 8) passes
KEY_CASES = [(2, 2, 2), (3, 3, 4), (6, 6, 6), (8, 8, 9), (11, 11, 11), (2, 21, 13), (14, 13, 14), (16, 17, 16),
             (21, 21, 21)]


def _key_cloud(bits, s=0.01, n=200_000, seed=0):
    """points in a box of 2^b − 3.8 voxels per axis (1.2 at b = 2), so that the library packs b bits for that axis; half
    uniform, half a second member or more jittered around a uniform point (voxels of several members all over the input)"""
    rng = np.random.RandomState(seed)
    ext = np.array([max(2.0 ** b - 3.8, 1.2) * s for b in bits])
    base = np.array([-1500.0, 250.0, 0.0])
    u = rng.rand(n // 2, 3) * ext
    v = np.clip(u[rng.randint(0, n // 2, n - n // 2)] + rng.uniform(-0.3 * s, 0.3 * s, (n - n // 2, 3)), 0.0, ext)
    pts = base + np.concatenate([u, v])[rng.permutation(n)]
    return np.concatenate([pts, [base, base + ext]])


def test_key_cases_cover_every_pass_count():
    seen = {}
    for bits in KEY_CASES:
        got = ref.key_bits(_key_cloud(bits), 0.01)
        assert got == list(bits)
        seen.setdefault(ref.radix_passes(bits), []).append(sum(bits))
    assert sorted(seen) == list(range(1, 9))
    assert min(min(v) for v in seen.values()) == 6 and max(max(v) for v in seen.values()) == 63
    assert {p % 2 for p in seen} == {0, 1}


@pytest.mark.parametrize("bits", KEY_CASES, ids=lambda b: f"{sum(b)}bit")
def test_key_widths(bits):
    xyz = _key_cloud(bits)
    cnt = _check(xyz, 0.01, _normals(len(xyz), sum(bits)), what=f"{bits}")
    assert (cnt > 1).sum() > (100 if sum(bits) > 6 else 7)


# ---- b. the per-axis limit ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_per_axis_limit(axis):
    """floor((max − org)/s) = 2^21 − 4 is the most the packed key holds per axis; one voxel more is refused with
    ME_ERR_RANGE and the refused call leaves the cloud and its normals as they were.  (Open3D accepts up to INT_MAX voxels
    per axis; this pins the library's narrower limit.)"""
    s = 0.01
    K = 2 ** 21 - 4
    rng = np.random.RandomState(axis)
    xyz = rng.rand(5000, 3) * 0.5
    xyz[0] = 0.0
    nrm = _normals(len(xyz), axis)
    ok = xyz.copy()
    ok[1, axis] = (K - 0.25) * s
    assert np.floor((ok[1, axis] + s * 0.5) / s) == K and ref.key_bits(ok, s)[axis] == 21
    _check(ok, s, nrm, what="at the limit")
    bad = xyz.copy()
    bad[1, axis] = (K + 0.75) * s
    assert np.floor((bad[1, axis] + s * 0.5) / s) == K + 1 and ref.key_bits(bad, s) is None
    api = _api()
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(EST, bad)
        ctx.set_normals(EST, nrm)
        with pytest.raises(api.MapEvalError) as e:
            ctx.voxel_downsample(EST, s)
        assert e.value.code == A.ME_ERR_RANGE
        _assert_bits(ctx.get_cloud(EST), bad, "refused cloud")
        _assert_bits(ctx.get_normals(EST), nrm, "refused normals")
        assert ctx.voxel_downsample(EST, 2 * s) > 0            # the context stays usable


# ---- c. voxel faces -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", [0.01, 0.1, 0.3])
@pytest.mark.parametrize("base", [0.0, 1500.0, -1500.0])
def test_voxel_faces(base, s):
    """points on org + k·s, one ulp either side, quotients that IEEE-round up to k, −0.0 at the origin"""
    xyz = ref.face_scene(base, s, n=40_000, seed=int(100 * s))
    _check(xyz, s, _normals(len(xyz), 9), what=f"faces {base} {s}")


# ---- d. stability -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["spread", "shuffled", "contiguous"])
def test_member_order(layout):
    """voxels of 3–50 members whose sums depend on the order of the members (tests/test_downsample_reference.py shows
    that a reversed order changes ≥ 30 % of them): the stable sort must keep the input order inside every voxel"""
    xyz, nrm = ref.order_scene(layout=layout)
    cnt = _check(xyz, 0.01, nrm, what=layout)
    assert (cnt >= 3).sum() == 6000


# ---- e. sizes around the tiles of the sort and the scan -----------------------------------------------------------------
SIZES = [1, 2, 31, 33, 2047, 2048, 2049, 32 * 2048, 32 * 2048 + 1, 33 * 2048 + 7]


def _sized_cloud(n, seed=1):
    """n points in a 20 cm box 1.5 km out: 8000 voxels of 1 cm, several members each at the larger sizes"""
    return FAR + np.random.RandomState(seed).rand(n, 3) * 0.2


@pytest.mark.parametrize("n", SIZES)
def test_sizes(n):
    xyz = _sized_cloud(n)
    _check(xyz, 0.01, _normals(n, n), what=f"n={n}")


@pytest.mark.parametrize("n", SIZES)
def test_density_compaction_sizes(n):
    _check_density(_sized_cloud(n), 0.037)


def test_every_point_its_own_voxel():
    s = 0.01
    g = np.arange(128)
    ijk = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    xyz = (FAR + ijk * s)[np.random.RandomState(2).permutation(len(ijk))]
    cnt = _check(xyz, s, _normals(len(xyz), 2), what="own voxels")
    assert len(cnt) == len(xyz) == 2 ** 21 and (cnt == 1).all()


def test_one_voxel_of_2_21_points():
    """one thread walks the whole voxel; the time of that walk is printed (DESIGN.md §3.5 records it)"""
    s = 0.01
    n = 2 ** 21
    xyz = FAR + np.random.RandomState(3).rand(n, 3) * (0.45 * s)
    nrm = _normals(n, 3)
    cnt = _check(xyz, s, nrm, what="one voxel")
    assert len(cnt) == 1 and cnt[0] == n
    import torch
    times = []
    with _api().MapEvalB200() as ctx:
        for _ in range(3):
            ctx.set_cloud(EST, xyz)
            ctx.set_normals(EST, nrm)
            ctx.synchronize()
            t0 = time.perf_counter()
            ctx.voxel_downsample(EST, s)                     # ends in a stream synchronise
            times.append(1e3 * (time.perf_counter() - t0))
    print(f"\none voxel of {n} points, with normals, on {torch.cuda.get_device_name(0)}: me_voxel_downsample "
          f"{', '.join(f'{t:.1f}' for t in times)} ms")


# ---- e/f/h. map-size clouds at 1 cm ---------------------------------------------------------------------------------------
def test_c3_estimate_at_1cm_with_nan_normals():
    """C3's estimated cloud (10 M points, box) at 1 cm, normals with NaN components; then its density compaction"""
    import torch
    from cloud_map_evaluation_b200 import synth_torch
    side = synth.box_side_for_density(synth.CONFIGS["C3"]["n_gt"])
    t = synth_torch.uniform_box(synth.CONFIGS["C3"]["n_est"], side, synth.EST_SEED, noise_sigma=synth.EST_NOISE_SIGMA,
                                device="cuda")
    xyz = t.cpu().numpy()
    del t
    torch.cuda.empty_cache()
    nrm = _normals(len(xyz), 10, nan_share=0.03)
    nrm[::1000] = np.nan
    cnt = _check(xyz, 0.01, nrm, what="C3 estimate")
    assert len(cnt) > 9_000_000 and cnt.max() > 1
    _check_density(xyz, 0.5113)


def test_above_2_24_points_generated_on_the_device():
    """20 M points of the outdoor scene made in HBM and borrowed by the context: the statement's result, and the
    caller's tensor untouched; then the density compaction of the same tensor"""
    from cloud_map_evaluation_b200 import synth_torch
    n = 20_000_000
    assert n > 2 ** 24
    t = synth_torch.outdoor_scene(n, synth.GT_SEED, synth.GT_SURFACE_NOISE_SIGMA, device="cuda")
    xyz = t.cpu().numpy()
    with _api().MapEvalB200() as ctx:
        ctx.set_cloud_device(EST, t.data_ptr(), n, keepalive=t)
        nv = ctx.voxel_downsample(EST, 0.01)
        pts = ctx.get_cloud(EST)
    _assert_bits(t.cpu().numpy(), xyz, "borrowed tensor")
    ep, _, cnt = ref.voxel_downsample(xyz, 0.01)
    assert nv == len(ep) and cnt.max() > 1
    _assert_bits(pts, ep, "20 M points")
    del pts, ep, cnt
    _check_density(xyz, 0.5113, device_tensor=t)


# ---- g. a borrowed cloud --------------------------------------------------------------------------------------------------
def test_borrowed_cloud():
    import torch
    xyz = _key_cloud((8, 8, 9), n=50_000)
    t = torch.from_numpy(xyz).cuda()
    keep = t.clone()
    with _api().MapEvalB200(stream=torch.cuda.current_stream().cuda_stream) as ctx:
        ctx.set_cloud_device(EST, t.data_ptr(), len(xyz), keepalive=t)
        n = ctx.voxel_downsample(EST, 0.01)
        pts = ctx.get_cloud(EST)
        torch.cuda.synchronize()
        assert torch.equal(t.view(torch.int64), keep.view(torch.int64))
        ctx.transform(EST, np.eye(4))                          # the result is the context's own cloud now
    ep, _, _ = ref.voxel_downsample(xyz, 0.01)
    assert n == len(ep)
    _assert_bits(pts, ep, "borrowed")

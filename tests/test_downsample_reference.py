"""The numpy statement of VoxelDownSample (tests/downsample_ref.py) against a plain Python loop and the oracle, and the
scenes of tests/test_gpu_downsample.py against the mistakes they are there to catch: an order-sensitive scene must change
when each voxel is summed in reverse, and a face scene must hold points that only IEEE division puts in their voxel."""
import os
import sys

import numpy as np
import pytest

from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import downsample_ref as ref  # noqa: E402


def _py_downsample(xyz, s, nrm=None):
    """one dict entry per voxel, points visited in input order (Python floats: IEEE fp64, no contraction)"""
    org = [min(float(p[a]) for p in xyz) - s * 0.5 for a in range(3)]
    acc = {}
    for i, p in enumerate(xyz):
        key = tuple(int(np.floor((float(p[a]) - org[a]) / s)) for a in range(3))
        e = acc.setdefault(key, [[0.0, 0.0, 0.0], 0, [0.0, 0.0, 0.0]])
        for a in range(3):
            e[0][a] += float(p[a])
        e[1] += 1
        if nrm is not None and not np.isnan(nrm[i]).any():
            for a in range(3):
                e[2][a] += float(nrm[i, a])
    keys = sorted(acc)
    pts = np.array([[acc[k][0][a] / acc[k][1] for a in range(3)] for k in keys])
    nr = np.array([[acc[k][2][a] / acc[k][1] for a in range(3)] for k in keys])
    return pts, nr, np.array([acc[k][1] for k in keys])


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint64),
                                                 np.ascontiguousarray(b).view(np.uint64))


def _small_clouds():
    rng = np.random.RandomState(7)
    one = np.array([[1.25, -3.5, 7.0]])
    dup = np.repeat(one, 5, 0)
    box = rng.rand(4000, 3) * 0.4 + [1500.0, -1500.0, 3.0]
    box = np.concatenate([box, box[:1500] + 0.002 * rng.randn(1500, 3)])
    faces = ref.face_scene(-1500.0, 0.1, n=3000, seed=1)
    spread, _ = ref.order_scene(n_vox=300, seed=2, layout="spread")
    return {"one": (one, 0.01), "dup": (dup, 0.01), "box": (box, 0.01), "faces": (faces, 0.1), "order": (spread, 0.01)}


@pytest.mark.parametrize("name", ["one", "dup", "box", "faces", "order"])
def test_statement_equals_python_loop_and_oracle(name):
    xyz, s = _small_clouds()[name]
    rng = np.random.RandomState(3)
    nrm = rng.randn(len(xyz), 3)
    nrm[rng.rand(len(xyz)) < 0.1, rng.randint(0, 3)] = np.nan
    pts, nr, cnt = ref.voxel_downsample(xyz, s, nrm)
    ep, en, ec = _py_downsample(xyz, s, nrm)
    assert _bits_equal(pts, ep) and _bits_equal(nr, en)
    np.testing.assert_array_equal(cnt, ec)
    assert _bits_equal(pts, O.voxel_downsample(xyz, s))                  # the oracle's points, same order
    plain, none, cnt2 = ref.voxel_downsample(xyz, s)
    assert none is None and _bits_equal(plain, pts)
    np.testing.assert_array_equal(cnt2, cnt)


def test_long_runs_use_the_same_sequential_chain(monkeypatch):
    """a voxel above LONG_RUN members goes through np.cumsum: the same bits as the rank-by-rank walk, −0.0 included"""
    rng = np.random.RandomState(5)
    xyz = np.concatenate([1500.0 + 0.004 * rng.rand(3000, 3), [[1500.0, 1500.0, 1500.1]] + 0.004 * rng.rand(50, 3)])
    xyz[:3000, 2] = -0.0                                    # an all −0.0 coordinate in the long voxel: +0.0 on the chain
    xyz[3000:, 2] = 0.004 * rng.rand(50)
    nrm = rng.randn(len(xyz), 3)
    nrm[::7, 1] = np.nan
    pts, nr, cnt = ref.voxel_downsample(xyz, 0.01, nrm)
    assert cnt.max() > ref.LONG_RUN
    monkeypatch.setattr(ref, "LONG_RUN", 10 ** 9)
    pts2, nr2, cnt2 = ref.voxel_downsample(xyz, 0.01, nrm)
    assert _bits_equal(pts, pts2) and _bits_equal(nr, nr2)
    ep, en, _ = _py_downsample(xyz, 0.01, nrm)
    assert _bits_equal(pts, ep) and _bits_equal(nr, en)
    assert np.signbit(pts[:, 2]).sum() == 0


@pytest.mark.parametrize("layout", ["spread", "shuffled", "contiguous"])
def test_order_scenes_are_order_sensitive(layout):
    """summing each voxel's members in reverse (the cloud fed back to front: same keys, same voxel order) changes a
    point or a normal in at least 30 % of the voxels; the spread layout keeps every voxel's members > 2048 places apart"""
    xyz, nrm = ref.order_scene(layout=layout)
    pts, nr, cnt = ref.voxel_downsample(xyz, 0.01, nrm)
    rp, rn, rc = ref.voxel_downsample(xyz[::-1], 0.01, nrm[::-1])
    np.testing.assert_array_equal(cnt, rc)
    multi = cnt > 1
    assert multi.sum() == 6000 and cnt[multi].min() >= 3 and cnt.max() <= 50
    changed = ((pts != rp).any(1) | (nr != rn).any(1))[multi]
    assert changed.mean() >= 0.3, changed.mean()
    assert (pts != rp).any(1)[multi].mean() >= 0.3
    if layout == "spread":
        k, _ = ref.voxel_keys(xyz, 0.01)
        packed = (k[:, 0] << 42) | (k[:, 1] << 21) | k[:, 2]
        order = np.argsort(packed, kind="stable")
        same = packed[order][1:] == packed[order][:-1]
        assert np.diff(order)[same].min() > 2048


@pytest.mark.parametrize("s", [0.01, 0.1, 0.3])
@pytest.mark.parametrize("base", [0.0, 1500.0, -1500.0])
def test_face_scenes_need_ieee_division(base, s):
    """the face scenes hold points below org + k·s in exact arithmetic whose quotient rounds up to k (checked with
    Fractions), and at 1 cm points that a multiplication by 1/s puts in another voxel than the division"""
    vals, up = ref.face_values(base, s)
    org = base - s * 0.5
    assert len(up) > 0
    xyz = ref.face_scene(base, s)
    assert xyz.min() == base and (xyz[0] == base).all()
    k, o = ref.voxel_keys(xyz, s)
    assert (o == org).all()
    hit = xyz[np.isin(xyz, up)]
    assert len(hit) > 100 and all(ref.rounds_up(x, org, s) for x in hit[:200])
    by_recip = np.floor((xyz - o) * (1.0 / s)).astype(np.int64)
    if s == 0.01:
        assert (by_recip != k).any(1).sum() > 100
    if base == 0.0:
        assert np.signbit(xyz[xyz == 0.0]).any() and (~np.signbit(xyz[xyz == 0.0])).any()
    pts, _, _ = ref.voxel_downsample(xyz, s)
    assert _bits_equal(pts, O.voxel_downsample(xyz, s))


def test_key_bits_follow_the_extent():
    """the library's formula: floor((max − org)/s) + 3 voxels per axis, 2^21 refused"""
    s = 0.01
    for b in range(2, 22):
        ext = max(2 ** b - 3.8, 1.2) * s
        assert ref.key_bits(np.array([[0.0, 0.0, 0.0], [ext, ext, ext]]), s) == [b, b, b]
    K = 2 ** 21 - 4
    x = (K - 0.25) * s
    assert np.floor((x + s * 0.5) / s) == K
    assert ref.key_bits(np.array([[0.0, 0.0, 0.0], [x, 0.0, 0.0]]), s) == [21, 2, 2]
    assert ref.key_bits(np.array([[0.0, 0.0, 0.0], [x + s, 0.0, 0.0]]), s) is None
    assert ref.radix_passes([2, 2, 2]) == 1 and ref.radix_passes([21, 21, 21]) == 8

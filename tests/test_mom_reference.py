"""The mutually orthogonal metric's rule (tests/mom_ref.py) on hand cases, without a GPU: rooms recover their axes, a
corridor without end walls has a small third family, the face-edge and corner bins, bin(-n) as bin(n)'s mirrored cell on
the opposite face, and the tie rules."""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mom_ref as R  # noqa: E402


HALF_CELL = math.degrees(math.atan(math.sqrt(2) / R.M)) + 1e-9


def _rot(yaw_deg, tilt_deg):
    y, t = math.radians(yaw_deg), math.radians(tilt_deg)
    Rz = np.array([[math.cos(y), -math.sin(y), 0], [math.sin(y), math.cos(y), 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, math.cos(t), -math.sin(t)], [0, math.sin(t), math.cos(t)]])
    return Rz @ Rx


def _normals(counts, rot=np.eye(3), jitter=0.0, seed=0):
    """planar normals: counts[a] points with normal +-e_a, rotated, each jittered by up to `jitter` radians"""
    rng = np.random.default_rng(seed)
    out = []
    for a, c in enumerate(counts):
        e = np.zeros(3)
        e[a] = 1.0
        n = np.tile(e, (c, 1)) * rng.choice([-1.0, 1.0], (c, 1)) + rng.normal(0, jitter, (c, 3))
        out.append(n / np.linalg.norm(n, axis=1, keepdims=True))
    n = np.vstack(out) @ rot.T
    return n


def _angle(a, b):
    return math.degrees(math.acos(min(1.0, abs(float(np.dot(a, b))))))


def test_axis_aligned_room_recovers_its_axes():
    n = _normals([3000, 2000, 5000], jitter=0.01)
    ax, st = R.axes(R.histogram(n), 10.0)
    assert st == "OK"
    # a1 is the lowest bin whose window holds the most normals: a tight cluster lies wholly inside it, so a1 is within the
    # angle of the cluster; a2 is within the angle of its cluster's projection
    assert _angle(ax[0], [0, 0, 1]) < 10.0           # the floor and ceiling family is the largest
    assert _angle(ax[1], [1, 0, 0]) < 10.0           # then the x walls
    assert _angle(ax[2], [0, 1, 0]) < 10.0
    fam = R.families(n, np.ones(len(n), bool), ax, 10.0)
    assert [(fam == j).sum() for j in range(3)] == [5000, 3000, 2000]
    np.testing.assert_allclose(ax @ ax.T, np.eye(3), atol=1e-12)


def test_yawed_tilted_room_recovers_its_axes():
    rot = _rot(27.0, 4.0)
    n = _normals([3000, 2000, 5000], rot=rot, jitter=0.01, seed=1)
    ax, st = R.axes(R.histogram(n), 10.0)
    assert st == "OK"
    assert _angle(ax[0], rot[:, 2]) < 10.0
    assert _angle(ax[1], rot[:, 0]) < 10.0
    assert _angle(ax[2], rot[:, 1]) < 10.0
    # a1 may sit up to the angle off the cluster's centre (the lowest bin of a plateau of equal scores), so the window can
    # cut the cluster's tail
    fam = R.families(n, np.ones(len(n), bool), ax, 10.0)
    got = [(fam == j).sum() for j in range(3)]
    assert got[0] >= 0.95 * 5000 and got[1] >= 0.95 * 3000 and got[2] >= 0.95 * 2000


def test_corridor_without_end_walls_has_a_small_third_family():
    n = _normals([4000, 0, 6000], jitter=0.01, seed=2)
    # a corridor along y: floor, ceiling and the two side walls; the end walls (normal y) are missing
    v = np.abs(np.random.default_rng(3).normal(0, 1e-4, len(n))) ** 2
    l2 = np.full(len(n), 1e-2)
    out = R.statement(v, l2, n, 0.5, 10.0, 100)
    assert out["n"][0] == 6000 and out["n"][1] == 4000 and out["n"][2] == 0
    assert out["status"] == "SMALL_FAMILY" and math.isnan(out["mom"])
    assert np.isnan(out["median"][2]) and np.isfinite(out["median"][:2]).all()


def test_no_planar_point_and_no_second_axis():
    ax, st = R.axes(np.zeros(R.BINS, np.int64), 10.0)
    assert st == "NO_PLANAR" and np.isnan(ax).all()
    ax, st = R.axes(R.histogram(_normals([0, 0, 100])), 10.0)
    assert st == "NO_SECOND_AXIS" and np.isfinite(ax[0]).all() and np.isnan(ax[1:]).all()


def test_face_edge_and_corner_bins():
    M = R.M
    # the face centre, its edges and its corners on the +z face (a = 2, b = x, c = y)
    assert R.bins([[0.0, 0.0, 1.0]])[0] == (4 * M + M // 2) * M + M // 2
    c = 1 / math.sqrt(3)
    assert R.bins([[c, c, c]])[0] == (0 * M + M - 1) * M + M - 1      # a tie of all three: axis 0, the last cell of both
    assert R.bins([[-c, -c, -c]])[0] == (1 * M + 0) * M + 0
    e = 1 / math.sqrt(2)
    assert R.bins([[e, 0.0, e]])[0] == (0 * M + M // 2) * M + M - 1   # a tie of x and z: axis 0, u = 0, w = 1
    assert R.bins([[0.0, -e, e]])[0] == (3 * M + M // 2) * M + M - 1  # a tie of y and z: axis 1, negative face


def test_antipode_is_the_mirrored_cell_on_the_opposite_face():
    rng = np.random.default_rng(4)
    n = rng.normal(size=(20000, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    M = R.M
    b, bn = R.bins(n), R.bins(-n)
    face, i, j = b // (M * M), (b // M) % M, b % M
    fn, inn, jn = bn // (M * M), (bn // M) % M, bn % M
    assert np.array_equal(fn, face ^ 1)
    # u -> -u: cell i -> M - 1 - i, except where (u + 1) M / 2 falls on a cell boundary
    assert np.array_equal(inn, M - 1 - i) and np.array_equal(jn, M - 1 - j)
    on = np.array([[1.0, 0.5, 0.0]]) / math.sqrt(1.25)       # u = 0.5: (u + 1) 8 = 12 exactly, a boundary
    b0, b1 = R.bins(on)[0], R.bins(-on)[0]
    assert (b0 // M) % M == 12 and (b1 // M) % M == 4        # the mirror of 12 would be 3
    h = R.histogram(n)
    assert h.sum() == 2 * len(n)


def test_tie_rules():
    # two equal peaks: a1 is the lowest bin of the highest score, which lies in the lower peak's window
    C = R.centres()
    lo, hi = int(np.argmax(C[:, 2])), int(np.argmax(C[:, 0]))      # near +z, near +x
    assert lo > hi
    h = np.zeros(R.BINS, np.int64)
    h[lo] = h[hi] = 5
    ax, st = R.axes(h, 10.0)
    assert st == "OK"
    assert _angle(ax[0], C[hi]) <= 10.0 and _angle(ax[1], C[lo]) <= 20.0
    # the family rule takes the lowest axis first
    fam = R.families(np.array([[0.0, 0.0, 1.0]]), np.array([True]), np.eye(3)[[2, 2, 0]], 10.0)
    assert fam[0] == 0


def test_fold_matches_plain_sums_to_rounding():
    rng = np.random.default_rng(5)
    v = rng.random(5000) * 1e-4
    fam = rng.integers(-1, 3, 5000).astype(np.int8)
    n, s = R.fold(v, fam)
    for j in range(3):
        assert n[j] == (fam == j).sum()
        assert s[j] == np.float64(s[j]) and abs(s[j] - v[fam == j].sum()) <= 1e-12 * s[j]

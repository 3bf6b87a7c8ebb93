"""The references of the exact k-NN walk (knn_walk.cuh) at every neighbour count it serves, on the CPU: lattice scenes whose
tie groups straddle the k-th slot, proof that the normal bounds of tests/exact_reg.py reject a wrong tie choice and a wrong
neighbour count there, the oracle's k-NN normals within those bounds at every k, and the FPFH statement of tests/fpfh_ref.py
against deliberately wrong neighbourhoods.  tests/test_gpu_knn_walk.py runs the device on the same scenes."""
import functools

import numpy as np
import pytest

import exact_reg as X
import fpfh_ref as R

from test_exact_reg import lattice, normal_scenes

# every k the GPU module runs: 1-3 (fewer than 3 neighbours: the identity covariance), the cubic shells' closures
# 7, 19, 27, 33, 57 with one past each, and the shared-memory boundary of knn_normals_kernel (k = 32: 48 KiB, 33: opt-in)
KS = [1, 2, 3, 4, 7, 8, 19, 20, 21, 27, 28, 32, 33, 34, 57, 58, 63, 64]
N_QUERIES = 40          # the central queries of a tie scene examined per k on the CPU
MIN_TIES = 16           # of them, at least this many have slot k and slot k + 1 at the same d2_kd where a cut is declared


def square_lattice(n, spacing, seed=0, origin=(0.0, 0.0, 0.0)):
    """an n x n lattice in the plane z = 0 with (dyadic) spacings (a, b), in a random caller order: shells of 4, 4, 4, 8, ...
    (a = b).  Every choice inside a shell leaves the normal at (0, 0, 1): the scene pins the cut, not the normal."""
    g = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2) * np.asarray(spacing, np.float64)
    g = np.c_[g, np.zeros(len(g))]
    return g[np.random.RandomState(seed).permutation(len(g))] + np.asarray(origin)


def stairs(nx, ny, spacing=0.25, tread=3, rise=2, seed=0, origin=(0.0, 0.0, 0.0)):
    """a staircase surface on the cubic lattice of the given (dyadic) spacing, in a random caller order: along x, `tread`
    columns at one height, then a column that carries the riser's rise - 1 points and the next tread's first point; ny rows
    along y.  Treads, risers and the edges between them give normals that vary inside a neighbourhood, and the lattice gives
    tie groups at every k."""
    prof, x, z = [], 0, 0
    while len(prof) < nx:
        for _ in range(tread - 1):
            prof.append((x, z))
            x += 1
        prof.append((x, z))
        x += 1
        for r in range(1, rise):
            prof.append((x, z + r))
        z += rise
    prof = np.array(prof[:nx], np.float64)
    p = np.array([(px, j, pz) for px, pz in prof for j in range(ny)], np.float64) * spacing
    return p[np.random.RandomState(seed).permutation(len(p))] + np.asarray(origin)


def tie_scenes():
    return {
        # spacings 1, 1.125, 1.25 (x 0.25): groups of 2, 4 and 8 (test_exact_reg.lattice)
        "aniso": lattice(8, (0.25, 0.28125, 0.3125), seed=3),
        # shells of 6, 12, 8, 6, 24, 24, closing at 7, 19, 27, 33, 57 and 81 with the query
        "cubic": lattice(9, (0.25, 0.25, 0.25), seed=4),
        "square": square_lattice(20, (0.25, 0.25), seed=5),
        "stairs": stairs(24, 16, seed=6),
    }


SCENES = tie_scenes()
DUP = normal_scenes()["duplicates"]     # 30 copies of one point: at k = 1 the tie falls on the query's own slot

# (scene, k) whose reference cut lies inside a tie group (slot k and k + 1 at the same distance); the other pairs cut on a
# shell boundary.  Every k is cut inside a tie somewhere.
TIE_CUT = {
    "aniso": {2, 4, 8, 20, 21, 28, 32, 33, 34, 58, 63, 64},
    "cubic": {2, 3, 4, 8, 20, 21, 28, 32, 34, 58, 63, 64},
    "square": {2, 3, 4, 7, 8, 19, 20, 27, 28, 32, 33, 34, 58, 63, 64},
    "stairs": {2, 3, 4, 7, 8, 19, 20, 21, 27, 28, 32, 33, 34, 57, 58, 63, 64},
}


def central(pts, m):
    """the m points nearest the centre of the bounding box (Chebyshev distance, ties to the smaller index)"""
    c = 0.5 * (pts.min(0) + pts.max(0))
    d = np.abs(pts - c).max(1)
    return np.lexsort((np.arange(len(pts)), d))[:m]


@functools.lru_cache(maxsize=None)
def _rows(name, k):
    pts = SCENES[name]
    return X.normals_exact(pts, central(pts, N_QUERIES), k=k)


def _tie_count(pts, queries, k):
    nb = X.knn_exact(pts, queries, k + 1)
    return sum(len(n) > k and X.d2_kd(pts[q], pts[n[k - 1]]) == X.d2_kd(pts[q], pts[n[k]]) for q, n in zip(queries, nb))


def _rejected(rows, nbs, pts):
    """how many rows reject the normal (the exactly rounded statement) of the neighbourhoods nbs"""
    wrong = X.normals_exact(pts, [r["q"] for r in rows], nbs=nbs)
    moved = sum(r["cov"] != w["cov"] for r, w in zip(rows, wrong))
    rej = sum(not X.check_normal(r, w["stmt"] if w["cov"] is not None else [0.0, 0.0, 1.0])["ok"] for r, w in zip(rows, wrong))
    return moved, rej


def test_every_k_has_a_tie_cut():
    for k in KS:
        assert k == 1 or any(k in ks for ks in TIE_CUT.values()), k


@pytest.mark.parametrize("k", KS)
def test_tie_cuts(k):
    """slot k and slot k + 1 tie on the declared scenes (k = 1: on the duplicates, where the query's copies tie with it)"""
    for name, pts in SCENES.items():
        t = _tie_count(pts, central(pts, N_QUERIES), k)
        if k in TIE_CUT[name]:
            assert t >= MIN_TIES, (name, k, t)
    if k == 1:
        assert _tie_count(DUP, np.arange(30), 1) == 30
        # the larger copies' nearest is the smallest copy, not themselves
        assert all(n[0] == min(np.flatnonzero((DUP == DUP[0]).all(1))) for n in X.knn_exact(DUP, np.arange(30), 1))


# the scene whose tie cut moves the normal at k beyond the bounds; at k <= 2 no choice can: fewer than 3 neighbours give
# the identity covariance and (0, 0, 1).  On the square lattice every choice keeps the plane, and on the anisotropic lattice
# at 32 - 34 the choices that change the covariance keep its smallest axis: neither is used for teeth.
TEETH = {k: "stairs" for k in KS if k >= 3}
TEETH.update({3: "cubic", 32: "cubic"})


@pytest.mark.parametrize("k", KS)
def test_wrong_tie_choice_is_rejected(k):
    if k <= 2:
        for name, pts in SCENES.items():
            rows = _rows(name, k)
            assert all(r["cov"] is None for r in rows)
        return
    name = TEETH[k]
    pts = SCENES[name]
    rows = _rows(name, k)
    moved, rej = _rejected(rows, X.knn_exact(pts, [r["q"] for r in rows], k, larger_index_on_tie=True), pts)
    assert moved > 0 and rej >= 1, (name, k, moved, rej)
    # symmetry: on the square lattice the covariance moves, the normal does not
    if k in TIE_CUT["square"]:
        rows = _rows("square", k)
        moved, rej = _rejected(rows, X.knn_exact(SCENES["square"], [r["q"] for r in rows], k, larger_index_on_tie=True),
                               SCENES["square"])
        assert rej == 0


def _variants(pts, queries, k):
    full = X.knn_exact(pts, queries, k + 1)
    return {
        "k-1": [n[:k - 1] for n in full],
        "k+1": full,
        "no query": [n[n != q][:k] for q, n in zip(queries, full)],
    }


@pytest.mark.parametrize("k", KS)
def test_wrong_neighbour_count_is_rejected(k):
    """k - 1 neighbours, k + 1 neighbours and the query left out are each rejected on some scene, wherever one side has at
    least 3 neighbours (below that both give (0, 0, 1))"""
    for var, size in (("k-1", k - 1), ("k+1", k + 1), ("no query", k)):
        if max(size, k) < 3:
            continue
        hit = []
        for name in ("stairs", "cubic", "aniso"):
            rows = _rows(name, k)
            nbs = _variants(SCENES[name], [r["q"] for r in rows], k)[var]
            hit.append(_rejected(rows, nbs, SCENES[name])[1])
            if hit[-1]:
                break
        assert hit[-1] >= 1, (var, k, hit)


# ---------------------------------------------------------------------------------------------------------------
# the oracle at every k
# ---------------------------------------------------------------------------------------------------------------
NORMAL_SCENES = normal_scenes()
N_ORACLE = 24           # queries per normal scene and k (every point of the tie scenes' central sample)


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle as O
    O.build()
    return O


@pytest.mark.parametrize("k", KS)
def test_oracle_normals_within_bounds_at_every_k(oracle, k):
    bad = []
    for name in SCENES:
        got = oracle.estimate_normals_knn(SCENES[name], k)
        for row in _rows(name, k):
            r = X.check_normal(row, got[row["q"]], raw=True)
            if not r["ok"]:
                bad.append((name, row["q"], r["why"]))
    for name, pts in sorted(NORMAL_SCENES.items()):
        q = np.random.RandomState(k).choice(len(pts), min(N_ORACLE, len(pts)), replace=False)
        got = oracle.estimate_normals_knn(pts, k)
        for row in X.normals_exact(pts, q, k=k):
            r = X.check_normal(row, got[row["q"]], raw=True)
            if not r["ok"]:
                bad.append((name, row["q"], r["why"]))
    assert not bad, (k, len(bad), bad[:5])


# ---------------------------------------------------------------------------------------------------------------
# FPFH: the neighbourhood statement's teeth, and FPFH on a sample
# ---------------------------------------------------------------------------------------------------------------
FEAT_V = 0.25           # the lattice spacing of the FPFH scenes = the voxel size (one point per voxel, at its centre)


def fpfh_stairs(nx=40, ny=32, seed=8, origin=(0.0, 0.0, 0.0)):
    """the FPFH staircase: treads of 3 and rises of 2 lattice steps; ny even, so that no row lies on the centroid's y and
    no orientation is ambiguous"""
    return stairs(nx, ny, FEAT_V, seed=seed, origin=origin)


def cpu_normals(xyz, k=30):
    """k-NN normals in plain fp64 (numpy), oriented like the feature clouds: a stand-in for the device's normals where only
    the neighbourhood statement is under test"""
    nb = X.knn_exact(xyz, np.arange(len(xyz)), k)
    out = np.empty_like(xyz)
    for i, n in enumerate(nb):
        w, v = np.linalg.eigh(np.cov(xyz[n].T, bias=True))
        out[i] = v[:, 0]
    return R.orient_normals(xyz, out)[0]


# (radius, max_nn) of the part-3 FPFH scenes on the staircase: the max_nn sweep at 7 spacings, and the radius exactly
# on the lattice distance 2 v (points on it are out) and the next double up (they are in)
FEAT_RADIUS = 7 * FEAT_V
FEAT_MAX_NN = [1, 2, 6, 7, 19, 20, 64, 127, 128]
ON_RADIUS = 2 * FEAT_V
FPFH_CASES = [(FEAT_RADIUS, m) for m in FEAT_MAX_NN] + [(ON_RADIUS, 128), (float(np.nextafter(ON_RADIUS, np.inf)), 128)]


def fpfh_tolerance(f64):
    """test_fpfh's tolerance of a device fp32 feature"""
    return 0.5 * np.spacing(np.abs(f64).astype(np.float32)) + 1e-9


@functools.lru_cache(maxsize=None)
def _fpfh_scene():
    xyz = fpfh_stairs()
    return xyz, cpu_normals(xyz)


def _breaks(xyz, nrm, radius, good, nb):
    """does the wrong neighbourhood nb change an unflagged fp32 feature beyond the tolerance?"""
    f32, f64, flagged, _ = good
    sp, fl = R.spfh(xyz, nrm, nb)
    w32, w64, wfl = R.fpfh(sp, nb, fl)
    ok = ~(flagged | wfl)
    return bool((np.abs(w32[ok].astype(np.float64) - f64[ok]) > fpfh_tolerance(f64[ok])).any())


@pytest.mark.parametrize("radius,max_nn", FPFH_CASES)
def test_fpfh_neighbourhood_teeth(radius, max_nn):
    xyz, nrm = _fpfh_scene()
    good = R.features(xyz, nrm, radius, max_nn)
    assert good[2].sum() <= 2
    wrong = {
        "larger index on a tie": R.hybrid_neighbours(xyz, radius, max_nn, larger_index_on_tie=True),
        "d2 <= r2": R.hybrid_neighbours(xyz, radius, max_nn, closed=True),
        "max_nn - 1": R.hybrid_neighbours(xyz, radius, max_nn - 1),
        "with the point itself": R.hybrid_neighbours(xyz, radius, max_nn, skip_self=False),
    }
    # the max_nn sweep cuts inside the radius, where the tie rule, the cap and the query itself decide; on the two radius
    # cases the cap does not bind (so neither the tie rule nor max_nn - 1 can change them) and the radius decides
    if radius == FEAT_RADIUS:
        names = ["larger index on a tie", "max_nn - 1", "with the point itself"]
    else:
        names = ["with the point itself"] + (["d2 <= r2"] if radius == ON_RADIUS else [])
    for name in names:
        assert _breaks(xyz, nrm, radius, good, wrong[name]), (name, radius, max_nn)


def test_fpfh_radius_edge_counts():
    xyz, _ = _fpfh_scene()
    on = [len(i) for i, _ in R.hybrid_neighbours(xyz, ON_RADIUS, 128)]
    up = [len(i) for i, _ in R.hybrid_neighbours(xyz, float(np.nextafter(ON_RADIUS, np.inf)), 128)]
    closed = [len(i) for i, _ in R.hybrid_neighbours(xyz, ON_RADIUS, 128, closed=True)]
    assert up == closed and sum(up) > sum(on)


def test_fpfh_sample_matches_features():
    xyz, nrm = _fpfh_scene()
    for radius, max_nn in ((FEAT_RADIUS, 20), (ON_RADIUS, 128)):
        f32, f64, flagged, _ = R.features(xyz, nrm, radius, max_nn)
        s = np.random.RandomState(1).choice(len(xyz), 150, replace=False)
        s32, s64, sfl = R.fpfh_sample(xyz, nrm, radius, max_nn, s)
        np.testing.assert_array_equal(s32, f32[s])
        np.testing.assert_array_equal(s64, f64[s])
        np.testing.assert_array_equal(sfl, flagged[s])

"""The mean map entropy of tests/exact_ref.py against plain-Python statements on tiny cases, the oracle and the library's
fp64 finish formula against it within B64, and a float32 emulation of the flat kernel's offset rebuild within B64 + B32(E)
— the certificate the fp32-offset kernels evaluate to decide which queries to finish in fp64.  The teeth show that the
bounds are tight enough to catch the fp32 offsets on thin surfaces, a divisor of k, a kept query and a neighbour counted
at exactly r.

The scenes (also run on the GPU by test_gpu_exact_mme.py): tilted planes with 1 mm .. 0.1 um of normal noise at the
origin and 1.7 km out, exact planes quantised to float32 at 10 and 100 m, an exact axis-aligned plane and line
(det = 0), a thin wire, duplicates, clusters with k at min_neighbors - 1 .. + 1 and neighbours exactly on the radius, and a
well-conditioned box.  The plane patches are 0.4 m across at r = 0.1 m, so many queries sit at a border or a corner."""
import math
import os
import sys
from fractions import Fraction

import mpmath as mp
import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import exact_ref as X  # noqa: E402

R_PLANE = 0.1
FAR = (1400.0, -900.0, 30.0)
A_DIR, B_DIR = np.array([0.8, 0.36, 0.48]), np.array([-0.6, 0.48, 0.64])
N_DIR = np.cross(A_DIR, B_DIR)
THIN = ("plane_10um_0", "plane_10um_far", "plane_1um_0", "plane_1um_far")


def _f32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32).astype(np.float64))


def tilted_plane(sigma, origin, n=300, seed=0):
    rng = np.random.RandomState(seed)
    uv = rng.uniform(0, 0.4, (n, 2))
    w = rng.normal(0, 1, n) * sigma
    return np.ascontiguousarray(uv[:, :1] * A_DIR + uv[:, 1:] * B_DIR + w[:, None] * N_DIR + np.asarray(origin))


def quantised_plane(dist, seed=3):
    """an exact tilted plane |x| = dist from the origin, stored as float32 (a PCD with TYPE F)"""
    return _f32(tilted_plane(0.0, np.array([0.6, -0.8, 0.0]) * dist, seed=seed))


def axis_plane(seed=4):
    rng = np.random.RandomState(seed)
    xy = rng.uniform(0, 0.4, (300, 2))
    return np.ascontiguousarray(np.column_stack([xy, np.full(300, 0.25)]))


def axis_line(seed=5):
    rng = np.random.RandomState(seed)
    return np.ascontiguousarray(np.column_stack([rng.uniform(0, 0.4, 120), np.full(120, 0.5), np.full(120, -0.75)]))


def wire(seed=6):
    """a 0.4 m wire along a tilted axis with 10 um of noise across it: two small eigenvalues"""
    rng = np.random.RandomState(seed)
    t = rng.uniform(0, 0.4, 150)
    return np.ascontiguousarray(t[:, None] * A_DIR + rng.normal(0, 1e-5, (150, 2)) @ np.stack([B_DIR, N_DIR]) +
                                np.asarray(FAR))


def box(n=1500, seed=7, dup=False):
    rng = np.random.RandomState(seed)
    p = rng.uniform(0, 0.5, (n, 3)) + np.array([3.0, -2.0, 1.0])
    if dup:     # a fifth of the points twice more, and one point ten times
        p = np.concatenate([p, p[::5], p[::5], np.repeat(p[:1], 10, 0)])
    return np.ascontiguousarray(p)


K_EDGE_R = 0.125      # exact in binary: the on-radius neighbours sit at d2 == r^2 exactly


def k_edges(seed=8):
    """clusters 1 m apart whose centre has m = 4, 5, 6, 9, 10, 11 neighbours strictly inside r, plus two exactly on it"""
    rng = np.random.RandomState(seed)
    out = []
    for j, m in enumerate((4, 5, 6, 9, 10, 11)):
        c = np.array([float(j), 0.5, -0.25])
        off = rng.uniform(-1, 1, (m, 3))
        off *= (rng.uniform(0.2, 0.45, m) * K_EDGE_R / np.linalg.norm(off, axis=1))[:, None]
        out += [c[None], c + off, c + np.array([[K_EDGE_R, 0, 0], [0, -K_EDGE_R, 0]])]
    return np.ascontiguousarray(np.concatenate(out))


def scene(name):
    """(points, radius, min_neighbors)"""
    sig = {"1mm": 1e-3, "0.1mm": 1e-4, "10um": 1e-5, "1um": 1e-6, "0.1um": 1e-7}
    if name.startswith("plane_"):
        _, s, where = name.split("_")
        return tilted_plane(sig[s], FAR if where == "far" else (0.0, 0.0, 0.0), seed=len(name)), R_PLANE, 10
    if name == "f32_10m":
        return quantised_plane(10.0), R_PLANE, 10
    if name == "f32_100m":
        return quantised_plane(100.0), R_PLANE, 10
    if name == "axis_plane":
        return axis_plane(), R_PLANE, 5
    if name == "axis_line":
        return axis_line(), R_PLANE, 5
    if name == "wire":
        return wire(), R_PLANE, 10
    if name == "k_edges_5":
        return k_edges(), K_EDGE_R, 5
    if name == "k_edges_10":
        return k_edges(), K_EDGE_R, 10
    if name == "duplicates":
        return box(600, dup=True), 0.1, 10
    if name == "box":
        return box(), 0.1, 10
    raise KeyError(name)


SCENES = [f"plane_{s}_{w}" for s in ("1mm", "0.1mm", "10um", "1um", "0.1um") for w in ("0", "far")] + \
         ["f32_10m", "f32_100m", "axis_plane", "axis_line", "wire", "k_edges_5", "k_edges_10", "duplicates", "box"]

_CACHE = {}


def exact(name, E=None):
    """the scene and its exact MME (cached per process)"""
    if name not in _CACHE:
        pts, r, k = scene(name)
        _CACHE[name] = (pts, r, k, X.mme_exact(pts, r, k))
    pts, r, k, ex = _CACHE[name]
    if E is not None:
        ex = dict(ex, b32=np.array([X.mme_fp32_certificate(c, kk, E) if v else 0.0
                                    for c, kk, v in zip(ex["cov"], ex["k"], ex["valid"])]))
    return pts, r, k, ex


def check_mme(ex, n_valid, mme, min_abs, max_abs, ent, allow):
    """per-point entropies `ent` and the aggregates of one evaluation against the exact values, with per-point bounds
    `allow`; returns the worst error / bound over the determined valid queries"""
    det, valid = ex["determined"], ex["valid"]
    np.testing.assert_array_equal((ent != 0)[det], valid[det])
    v = det & valid
    err = np.abs(ent - ex["e"])
    bad = np.nonzero(v & (err > allow))[0]
    assert len(bad) == 0, [(int(i), ent[i], ex["e"][i], err[i], allow[i]) for i in bad[:5]]
    und, s_b, ext_b = X.mme_aggregate_bounds(ex, allow)
    nv, s_ex, mn_ex, mx_ex = X.mme_summary(ex)
    assert abs(n_valid - nv) <= und, (n_valid, nv, und)
    if und == 0 and nv:
        assert abs(mme * n_valid - s_ex) <= s_b + abs(mme * n_valid) * 4 * X.U, (mme * n_valid, s_ex, s_b)
        assert abs(min_abs - mn_ex) <= ext_b and abs(max_abs - mx_ex) <= ext_b, (min_abs, mn_ex, max_abs, mx_ex, ext_b)
    return float((err[v] / allow[v]).max()) if v.any() else 0.0


# ---------------------------------------------------------------------------------------------------------------
# exact_ref against plain statements
# ---------------------------------------------------------------------------------------------------------------
def test_mme_point_against_a_hand_known_covariance():
    """the query at the origin and 10 neighbours with mean 0 and covariance diag(4, 16, 18) / 9 (k - 1 = 9); a point on the
    radius and one outside it are not neighbours"""
    nb = [(1, 0, 0), (-1, 0, 0), (1, 0, 0), (-1, 0, 0), (0, 2, 0), (0, -2, 0), (0, 2, 0), (0, -2, 0), (0, 0, 3), (0, 0, -3)]
    pts = np.array([(0.0, 0.0, 0.0)] + nb + [(5.0, 0, 0), (0, 0, 5.5)], dtype=np.float64)
    nbs = X.mme_neighbours(pts, 5.0)
    assert sorted(nbs[0].tolist()) == list(range(1, 11))
    p = X.mme_point(pts, 0, nbs[0], 10)
    assert p["k"] == 10 and p["valid"] and p["determined"]
    assert p["cov"] == [[Fraction(4, 9), 0, 0], [0, Fraction(16, 9), 0], [0, 0, Fraction(18, 9)]]
    with mp.workdps(40):
        assert p["e"] == float(0.5 * mp.log(2 * mp.pi * mp.e * mp.mpf(1152) / 729))
    assert not X.mme_point(pts, 0, nbs[0], 11)["valid"]


def test_mme_point_against_plain_fractions():
    """a random neighbourhood 1.4 km out: the exact centred covariance and entropy by plain Fractions"""
    rng = np.random.RandomState(3)
    pts = np.asarray(FAR) + rng.uniform(-0.05, 0.05, (40, 3))
    nbs = X.mme_neighbours(pts, 0.2)
    i, nb = 7, nbs[7]
    ref = [j for j in range(40) if j != i and X.d2_kd(pts[i], pts[j]) < 0.04]
    assert sorted(nb.tolist()) == ref
    P = [[Fraction(x) for x in pts[j]] for j in ref]
    k = len(P)
    mu = [sum(p[a] for p in P) / k for a in range(3)]
    cov = [[sum((p[a] - mu[a]) * (p[b] - mu[b]) for p in P) / (k - 1) for b in range(3)] for a in range(3)]
    got = X.mme_point(pts, i, nb, 5)
    assert got["cov"] == cov
    det = X._det3(cov)
    with mp.workdps(50):
        e = 0.5 * mp.log(2 * mp.pi * mp.e * mp.mpf(det.numerator) / det.denominator)
    assert got["e"] == float(e) and got["b64"] < 2e-12


def test_degenerate_neighbourhoods_are_determined_rejections():
    """an exact axis-aligned plane and line: det = 0 and ddet = 0, so every fp64 evaluation rejects every point"""
    for name in ("axis_plane", "axis_line"):
        _, _, _, ex = exact(name)
        big = ex["k"] >= 5
        assert big.sum() > 50
        assert np.all(ex["determined"]) and not ex["valid"].any(), name


def test_scenes_reach_their_edges():
    # k around both min_neighbors, decided by neighbours exactly on the radius
    pts, r, _, ex = exact("k_edges_5")
    centres = [int(i) for i in range(len(pts)) if np.all(pts[i] == np.round(pts[i] * 4) / 4)]
    assert sorted(ex["k"][centres].tolist()) == [4, 5, 6, 9, 10, 11]
    assert not ex["valid"][centres[0]] and ex["valid"][centres[1]]
    # borders and corners: the centroid of the neighbourhood far from the query
    pts, r, _, ex = exact("plane_1um_far")
    far_c = [np.linalg.norm(pts[nb].mean(0) - pts[i]) for i, nb in enumerate(ex["nbs"]) if len(nb)]
    assert max(far_c) > 0.4 * r
    # duplicates: coincident neighbours are kept
    _, _, _, ex = exact("duplicates")
    assert (ex["k"] >= 11).sum() > 10 and ex["valid"].sum() > 100


# ---------------------------------------------------------------------------------------------------------------
# the oracle and the library's fp64 formula within B64
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def O():
    from oracle import oracle as _O
    _O.build()
    return _O


@pytest.mark.parametrize("name", SCENES)
def test_oracle_mme_against_exact(O, name):
    pts, r, k, ex = exact(name)
    res, ent = O.eval_mme(pts, r, k, want_entropies=True)
    assert res.n_total == len(pts)
    check_mme(ex, res.n_valid, res.mme, res.min_abs_entropy, res.max_abs_entropy, ent, ex["b64"])
    if name in ("box", "plane_1mm_0", "k_edges_10"):
        assert np.all(ex["determined"])


@pytest.mark.parametrize("name", SCENES)
def test_fp64_moment_formula_against_exact(name):
    """finish_entropy's moments about the query, in fp64 from fp64 offsets: the fp64 finish of the fp32-offset sweeps and
    the generic walk"""
    pts, r, k, ex = exact(name)
    ent = np.array([X.finish_entropy_fp64(pts[nb] - pts[i], k) for i, nb in enumerate(ex["nbs"])])
    det, valid = ex["determined"], ex["valid"]
    np.testing.assert_array_equal((ent != 0)[det], valid[det])
    v = det & valid
    assert np.all(np.abs(ent - ex["e"])[v] <= ex["b64"][v])


def _emulate(name, h_cells=3):
    """the float32 offset rebuild on a lattice of edge r / h_cells (3 rings), finished in fp64, and E"""
    pts, r, k, _ = exact(name)
    h = r / h_cells
    E = X.mme_offset_error(h, h_cells, pts)
    _, _, _, ex = exact(name, E)
    ent = np.zeros(len(pts))
    own = np.full(len(pts), np.inf)
    for i, nb in enumerate(ex["nbs"]):
        if len(nb) < k:
            continue
        d = X.fp32_offsets(pts, i, nb, h, h_cells)
        ent[i] = X.finish_entropy_fp64(d, k)
        c = np.cov(d.T, ddof=1)
        own[i] = X.mme_fp32_certificate(c.tolist(), len(nb), E)
    return pts, r, k, ex, E, ent, own


@pytest.mark.parametrize("name", SCENES)
@pytest.mark.parametrize("h_cells", [3, 2])
def test_fp32_offset_emulation_within_the_certificate(name, h_cells):
    """every query the certificate covers (B32 finite) is within B64 + B32 of the exact entropy; and a query the kernel's
    own certificate keeps on the fast path (<= TAU_FP64) has an exact certificate within 2 TAU_FP64"""
    pts, r, k, ex, E, ent, own = _emulate(name, h_cells)
    v = ex["determined"] & ex["valid"] & np.isfinite(ex["b32"])
    err = np.abs(ent - ex["e"])
    allow = ex["b64"] + ex["b32"]
    assert np.all(err[v] <= allow[v]), float((err[v] / allow[v]).max())
    fast = ex["valid"] & (own <= X.TAU_FP64)
    assert np.all(ex["b32"][fast] <= 2 * X.TAU_FP64)
    if v.any():
        print(f"{name} h=r/{h_cells}: E={E:.2e} max err/B32 = {float((err[v] / ex['b32'][v]).max()):.3f}, "
              f"max err {float(err[v].max()):.2e}, fp64 finish of {int((ex['valid'] & ~(own <= X.TAU_FP64)).sum())} queries")


# ---------------------------------------------------------------------------------------------------------------
# teeth
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", THIN)
def test_fp32_offsets_break_b64_on_thin_planes(name):
    pts, r, k, ex, E, ent, own = _emulate(name)
    v = ex["determined"] & ex["valid"]
    err = np.abs(ent - ex["e"])
    assert np.any(err[v] > ex["b64"][v])
    assert np.any(own[v] > X.TAU_FP64)          # ... and the kernel's certificate sends those queries to the fp64 finish


def _variant_breaks(name, **kw):
    pts, r, k, ex = exact(name)
    nbs = X.mme_neighbours(pts, r, le=kw.pop("le", False))
    ints = X.to_ints(pts)
    for i, nb in enumerate(nbs):
        p = X.mme_point(pts, i, nb, k, ints, **kw)
        if not ex["determined"][i]:
            continue
        if p["valid"] != ex["valid"][i] or abs(p["e"] - ex["e"][i]) > ex["b64"][i]:
            return True
    return False


def test_dividing_by_k_breaks_the_bound():
    assert _variant_breaks("box", divisor="k")


def test_keeping_the_query_breaks_the_bound():
    assert _variant_breaks("plane_1mm_0", drop_query=False)


def test_counting_a_neighbour_at_exactly_r_breaks_the_bound():
    assert _variant_breaks("k_edges_5", le=True)
    assert _variant_breaks("k_edges_10", le=True)

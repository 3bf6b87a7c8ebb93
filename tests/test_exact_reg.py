"""Registration against exact arithmetic on the CPU (tests/exact_reg.py): the reference against plain statements on tiny
cases, the oracle's k-NN normals within the normal bounds, me_icp_update (pure host) against the exact updates on blocks
built exactly, and variants that are subtly wrong, each of which must break a bound."""
import math
import os
from fractions import Fraction

import numpy as np
import pytest

import exact_reg as X
from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import _lib

P2P, P2L, GICP = A.ME_ICP_POINT_TO_POINT, A.ME_ICP_POINT_TO_PLANE, A.ME_ICP_GENERALIZED
FAR = np.array([1500.0, -800.0, 40.0])


@pytest.fixture(scope="module")
def api():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    from cloud_map_evaluation_b200 import api as _api
    return _api


def rot(rx, ry, rz):
    ca, sa, cb, sb, cg, sg = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    Ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    Rz = np.array([[cg, -sg, 0], [sg, cg, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


RZ90 = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])      # exact in fp64


def near_planar_pair(h, tilt=True, n=2000, seed=0):
    """source spread 50 / 40 / h m (tilted by rot(0.7, -0.5, 1.1) or not) about c, target = source moved by a small known
    rotation and translation: (p, q, c)"""
    rs = np.random.RandomState(seed)
    p = rs.rand(n, 3) * [50.0, 40.0, h] - [25.0, 20.0, h / 2]
    if tilt:
        p = p @ rot(0.7, -0.5, 1.1).T
    c = np.array([3.0, -2.0, 1.0])
    p = p + c
    q = (p - c) @ rot(0.01, -0.02, 0.015).T + c + [0.1, -0.05, 0.02]
    return p, q, c


def lattice(n, spacing, seed=0, origin=(0.0, 0.0, 0.0)):
    """an n^3 lattice of the given (dyadic) spacings a <= b <= c with b^2 + c^2 < 3 a^2, in a random caller order: every
    interior point's 19 nearest are itself, the 6 faces and the 12 edges, and its 20th is one of the 8 corners, all at the
    same distance.  The tie rule fixes the covariance diag(a^2, b^2, c^2) / 2 + (19 / 400) e e^T (e the corner's offset),
    and with unequal spacings its normal is unique."""
    g = np.stack(np.meshgrid(*[np.arange(n)] * 3, indexing="ij"), -1).reshape(-1, 3) * np.asarray(spacing)
    return g[np.random.RandomState(seed).permutation(len(g))] + np.asarray(origin)


# ---------------------------------------------------------------------------------------------------------------
# sigma^T sigma: the SVD umeyama_from_sums took before, restated in numpy (teeth)
# ---------------------------------------------------------------------------------------------------------------
def _eig3_jacobi(a):
    a, v = [float(x) for x in a], [1.0, 0, 0, 0, 1.0, 0, 0, 0, 1.0]
    for _ in range(64):
        off, diag = a[1] ** 2 + a[2] ** 2 + a[5] ** 2, a[0] ** 2 + a[4] ** 2 + a[8] ** 2
        if off <= 1e-40 * diag or off == 0.0:
            break
        for p in range(2):
            for q in range(p + 1, 3):
                apq = a[p * 3 + q]
                if apq == 0.0:
                    continue
                th = (a[q * 3 + q] - a[p * 3 + p]) / (2.0 * apq)
                t = (1.0 if th >= 0 else -1.0) / (abs(th) + math.sqrt(th * th + 1.0))
                c = 1.0 / math.sqrt(t * t + 1.0)
                s = t * c
                for k in range(3):
                    x, y = a[k * 3 + p], a[k * 3 + q]
                    a[k * 3 + p], a[k * 3 + q] = c * x - s * y, s * x + c * y
                for k in range(3):
                    x, y = a[p * 3 + k], a[q * 3 + k]
                    a[p * 3 + k], a[q * 3 + k] = c * x - s * y, s * x + c * y
                for k in range(3):
                    x, y = v[k * 3 + p], v[k * 3 + q]
                    v[k * 3 + p], v[k * 3 + q] = c * x - s * y, s * x + c * y
    return [a[0], a[4], a[8]], np.array(v).reshape(3, 3)


def umeyama_sigma_t_sigma(blk, c):
    n = blk[0]
    pm, qm = blk[1:4] / n, blk[4:7] / n
    sig = blk[7:16].reshape(3, 3) / n - np.outer(qm, pm)
    w, V = _eig3_jacobi((sig.T @ sig).reshape(9))
    order = sorted(range(3), key=lambda j: -w[j])
    sv = np.sqrt(np.maximum([w[j] for j in order], 0.0))
    Vs = V[:, order]
    U = np.array([sig @ Vs[:, j] / sv[j] if sv[j] > 0 else np.zeros(3) for j in range(3)]).T
    if not sv[2] > 1e-8 * sv[0]:
        U[:, 2] = np.cross(U[:, 0], U[:, 1])
        if np.linalg.det(Vs) < 0:
            U[:, 2] = -U[:, 2]
    S = np.diag([1.0, 1.0, -1.0 if np.linalg.det(U) * np.linalg.det(Vs) < 0 else 1.0])
    T = np.eye(4)
    T[:3, :3] = U @ S @ Vs.T
    T[:3, 3] = (qm + c) - T[:3, :3] @ (pm + c)
    return T


def _p2p_case(h, tilt):
    p, q, c = near_planar_pair(h, tilt)
    blk, _ = X.p2p_block_exact(p, q, X.d2_kd(p, q), c)
    bf = X.block_floats(blk)
    T, bound, s = X.umeyama_exact(bf, c)
    return bf, c, T, bound, s


def _within(got, exp, bound):
    return bool((np.abs(got - exp)[:3] <= bound[:3]).all())


# ---------------------------------------------------------------------------------------------------------------
# the reference against plain statements
# ---------------------------------------------------------------------------------------------------------------
def test_blocks_match_plain_statements():
    # small integers: every fp64 operation of the plain statements is exact
    p = np.array([[1.0, 2.0, 3.0], [4.0, -1.0, 0.0], [2.0, 2.0, -2.0]])
    q = p + [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, -1.0]]
    c = np.array([1.0, 1.0, 1.0])
    blk, bound = X.p2p_block_exact(p, q, X.d2_kd(p, q), c)
    pc, qc = p - c, q - c
    exp = np.concatenate([[3], pc.sum(0), qc.sum(0), (qc.T @ pc).reshape(9), [3.0]])
    assert X.block_floats(blk).tolist() == exp.tolist() and bound[0] == 0.0
    nt = np.array([[0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
    blk, _ = X.ne_block_exact(p, q, nt, X.d2_kd(p, q), 1)
    J = np.concatenate([np.cross(p, nt), nt], 1)
    r = ((p - q) * nt).sum(1)
    iu = np.triu_indices(6)
    assert X.block_floats(blk).tolist() == np.concatenate([[3], (J.T @ J)[iu], J.T @ r, [3.0]]).tolist()
    # generalized ICP: the closed form Rx diag(eps, 1, 1) Rx^T of a unit normal is I + (eps - 1) n n^T
    n = np.array([0.6, 0.0, 0.8])
    C = np.array([[float(x) for x in row] for row in X.gicp_cov_exact(n)])
    np.testing.assert_allclose(C, np.eye(3) + (1e-3 - 1) * np.outer(n, n), rtol=0, atol=1e-15)
    assert X.gicp_cov_exact([-0.995, 0.0, 0.0998]) == X.gicp_cov_exact([-0.999, 0.01, 0.0])     # the quirk: both Rx = I
    # the update of an exact 90 degree rotation is that rotation
    q = p @ RZ90.T + [0.5, 0.25, -1.0]
    blk, _ = X.p2p_block_exact(p, q, X.d2_kd(p, q), c)
    T, bound, _ = X.umeyama_exact(X.block_floats(blk), c)
    assert np.abs(T[:3, :3] - RZ90).max() <= 1e-16 and np.abs(T[:3, 3] - [0.5, 0.25, -1.0]).max() <= 1e-15
    # the exact solve of a diagonal system and TransformVector6dToMatrix4d
    ne = np.zeros(A.ME_ICP_BLOCK_NE)
    ne[0] = 5
    ne[[1, 7, 12, 16, 19, 21]] = [2.0, 4.0, 8.0, 1.0, 1.0, 1.0]
    ne[22:28] = [-0.02, -0.04, 0.08, -1.0, 2.0, 0.5]
    T, _, x, kappa = X.ne_update_exact(ne)
    assert x.tolist() == [0.01, 0.01, -0.01, 1.0, -2.0, -0.5] and kappa == 8.0
    np.testing.assert_allclose(T[:3, :3], rot(0.01, 0.01, -0.01), rtol=0, atol=4e-16)


def test_knn_and_covariance_match_plain_statements():
    pts = lattice(4, (1.0, 1.125, 1.25), seed=1)
    q = int(np.flatnonzero((pts == [1.0, 1.125, 1.25]).all(1))[0])
    nb = X.knn_exact(pts, [q], 20)[0]
    d2 = X.d2_kd(pts[q], pts)
    brute = sorted(range(len(pts)), key=lambda j: (d2[j], j))[:20]
    assert nb.tolist() == brute and nb[0] == q
    corners = [j for j in range(len(pts)) if d2[j] == 1.0 + 1.265625 + 1.5625]
    assert len(corners) == 8 and nb[19] == min(corners)
    assert X.knn_exact(pts, [q], 20, larger_index_on_tie=True)[0][19] == max(corners)
    # cov = diag(a^2, b^2, c^2) / 2 + (19 / 400) e e^T, e the chosen corner's offset
    e = [Fraction(x) for x in pts[nb[19]] - pts[q]]
    exp = [[(Fraction([1, 81, 25][a], [1, 64, 16][a]) / 2 if a == b else 0) + Fraction(19, 400) * e[a] * e[b] for b in range(3)]
           for a in range(3)]
    assert X.covariance_exact(pts, nb) == exp


def test_fast_eigen_statement():
    rs = np.random.RandomState(4)
    for lam in ([1e-6, 1.0, 3.0], [1.0, 2.0, 50.0], [0.0, 1.0, 1.0], [1.0, 1.0, 9.0]):
        Q, _ = np.linalg.qr(rs.randn(3, 3))
        C = Q @ np.diag(lam) @ Q.T
        n = np.array(X.fast_eigen3x3(C.reshape(9)))
        assert abs(np.linalg.norm(n) - 1) < 1e-15
        assert n @ C @ n - lam[0] < 1e-13
    assert X.fast_eigen3x3(np.diag([2.0, 1.0, 3.0]).reshape(9)) == [0.0, 1.0, 0.0]
    assert X.fast_eigen3x3(np.zeros(9)) == [0.0, 0.0, 1.0]


# ---------------------------------------------------------------------------------------------------------------
# the oracle's k-NN normals
# ---------------------------------------------------------------------------------------------------------------
def normal_scenes():
    rs = np.random.RandomState(7)
    out = {}
    for noise in (1e-3, 1e-5, 1e-7):
        for far in (False, True):
            uv = rs.rand(400, 2) * 4.0
            p = np.stack([uv[:, 0], uv[:, 1], noise * rs.randn(400)], 1) @ rot(0.4, -0.3, 0.8).T
            out[f"plane_{noise:g}{'_far' if far else ''}"] = p + (FAR if far else 0.0)
    out["plane_f32"] = (np.stack([rs.rand(400) * 10, rs.rand(400) * 10, np.zeros(400)], 1) @ rot(0.3, 0.2, 0.1).T
                        + [10.0, 20.0, 5.0]).astype(np.float32).astype(np.float64)
    out["lattice"] = lattice(6, (0.5, 0.5625, 0.625), seed=2)
    out["strip"] = np.stack([rs.rand(300) * 10, rs.rand(300) * 0.6, 0.01 * rs.randn(300)], 1) @ rot(0.2, 0.5, -0.4).T
    out["blob"] = rs.randn(300, 3)
    out["line"] = np.outer(rs.rand(200) * 5, [0.48, 0.6, 0.64]) + 1e-4 * rs.randn(200, 3)
    out["duplicates"] = np.concatenate([np.repeat([[1.0, 2.0, 3.0]], 30, 0), rs.rand(60, 3)])
    out["small"] = rs.rand(12, 3)
    out["outliers"] = np.concatenate([rs.randn(200, 3) * 0.1, rs.rand(25, 3) * 60.0 - 30.0])
    return out


SCENES = normal_scenes()


@pytest.mark.parametrize("name", sorted(SCENES))
def test_oracle_normals_within_bounds(name):
    from oracle import oracle as O
    O.build()
    pts = SCENES[name]
    rows = X.normals_exact(pts)
    got = O.estimate_normals_knn(pts, 20)
    bad = []
    for row in rows:
        # the oracle forms the covariance from raw-coordinate cumulants, as Open3D does
        r = X.check_normal(row, got[row["q"]], raw=True)
        if not r["ok"]:
            bad.append((row["q"], r["why"]))
        # the numpy statement on the exactly rounded covariance meets the bounds of the kernel's formula
        if row["cov"] is not None:
            r = X.check_normal(row, row["stmt"])
            assert r["ok"], (name, row["q"], r["why"])
    assert not bad, (name, bad[:5])


def test_normals_check_has_teeth():
    """the 20th neighbour taken by the larger index on a tie gives normals the bounds reject"""
    pts = SCENES["lattice"]
    interior = [i for i in range(len(pts)) if (pts[i] > 0).all() and (pts[i] < pts.max(0)).all()]
    good = X.normals_exact(pts, interior)
    wrong = X.normals_exact(pts, interior, nbs=X.knn_exact(pts, interior, 20, larger_index_on_tie=True))
    # opposite corners give the same covariance: only the other choices change the normal
    moved = [g["cov"] != w["cov"] for g, w in zip(good, wrong)]
    rejected = [not X.check_normal(g, w["stmt"])["ok"] for g, w in zip(good, wrong)]
    assert rejected == moved and sum(moved) > len(interior) // 2


# ---------------------------------------------------------------------------------------------------------------
# me_icp_update against the exact updates
# ---------------------------------------------------------------------------------------------------------------
P2P_H = [1.5, 0.5, 0.1, 0.01, 1e-3, 1e-4, 5e-5, 0.0]        # s3 / s1 from ~1e-3 down to ~1e-12, and a planar cloud


@pytest.mark.parametrize("tilt", [True, False], ids=["tilted", "axis"])
@pytest.mark.parametrize("h", P2P_H)
def test_update_point_to_point_exact(api, h, tilt):
    bf, c, T, bound, s = _p2p_case(h, tilt)
    got = api.icp_update(P2P, bf, c)
    err = np.abs(got - T)
    assert _within(got, T, bound), (s[2] / s[0], err[:3].max(), bound[0, 0])
    R = got[:3, :3]
    assert np.abs(R.T @ R - np.eye(3)).max() <= 1e-13 and abs(np.linalg.det(R) - 1) <= 1e-13


def test_update_point_to_point_rank2(api):
    """an exactly rank-2 sigma (all points on the plane z = 1 and its image): the rotation is still unique"""
    rs = np.random.RandomState(5)
    p = np.stack([rs.rand(500) * 8.0 - 4.0, rs.rand(500) * 6.0 - 3.0, np.ones(500)], 1)
    q = p @ RZ90.T + [0.5, -0.25, 0.0]
    c = np.zeros(3)
    blk, _ = X.p2p_block_exact(p, q, X.d2_kd(p, q), c)
    bf = X.block_floats(blk)
    T, bound, s = X.umeyama_exact(bf, c)
    assert s[2] == 0.0
    assert _within(api.icp_update(P2P, bf, c), T, bound)
    np.testing.assert_allclose(T[:3, :3], RZ90, rtol=0, atol=1e-15)


@pytest.mark.parametrize("h", [1.0, 0.1, 0.01])
def test_sigma_t_sigma_route_breaks_the_bound(h):
    bf, c, T, bound, _ = _p2p_case(h, True)
    assert not _within(umeyama_sigma_t_sigma(bf, c), T, bound)


def ne_scene(method, far, R=None, n=300, seed=3):
    """(vs, vt, nt, ns, d2) of kept pairs near a tilted bumpy surface; source normals not unit length"""
    rs = np.random.RandomState(seed + method)
    uv = rs.rand(n, 2) * 8.0 - 4.0
    base = np.stack([uv[:, 0], uv[:, 1], 0.3 * np.sin(uv[:, 0]) * np.cos(0.5 * uv[:, 1])], 1)
    nt = np.stack([-0.3 * np.cos(uv[:, 0]) * np.cos(0.5 * uv[:, 1]), 0.15 * np.sin(uv[:, 0]) * np.sin(0.5 * uv[:, 1]),
                   np.ones(n)], 1)
    nt /= np.linalg.norm(nt, axis=1, keepdims=True)
    Rt = rot(0.3, -0.2, 0.5)
    vt = base @ Rt.T + (FAR if far else 0.0)
    nt = nt @ Rt.T
    vs = vt + 0.01 * rs.randn(n, 3)
    ns = (nt + 0.05 * rs.randn(n, 3)) * (1 + 0.1 * rs.rand(n, 1))
    return vs, vt, nt, ns, X.d2_kd(vs, vt)


@pytest.mark.parametrize("far", [False, True], ids=["origin", "far"])
@pytest.mark.parametrize("method", [P2L, GICP])
def test_update_normal_equations_exact(api, method, far):
    vs, vt, nt, ns, d2 = ne_scene(method, far)
    blk, _ = X.ne_block_exact(vs, vt, nt, d2, method, ns, rot(0.02, 0.01, -0.03))
    bf = X.block_floats(blk)
    T, bound, x, kappa = X.ne_update_exact(bf)
    got = api.icp_update(method, bf)
    assert _within(got, T, bound), (kappa, np.abs(got - T)[:3].max(), bound[0, 0])
    assert kappa > (1e6 if far else 1.0)


# ---------------------------------------------------------------------------------------------------------------
# generalized ICP block variants that must break the bound
# ---------------------------------------------------------------------------------------------------------------
def _shortcut(n, R):
    n = np.asarray(n, np.float64)
    return [[X._F(v) for v in row] for row in (0.5 * np.eye(3) + (X.EPS_GICP - 1) * np.outer(n, n))]


def _no_quirk(n, R):
    return X.gicp_cov_exact(n, R, quirk=False)


def _transposed(n, R):
    return X.gicp_cov_exact(n, None if R is None else np.asarray(R).T)


@pytest.mark.parametrize("variant", ["transposed_R", "shortcut", "no_quirk"])
def test_gicp_block_variants_break_the_bound(variant):
    vs, vt, nt, ns, d2 = ne_scene(GICP, False, n=120)
    if variant == "no_quirk":
        ns = ns.copy()
        ns[::3] = [-0.995, 0.0998, 0.0]                    # normals near -e1: Rx = I
    good, bound = X.ne_block_exact(vs, vt, nt, d2, GICP, ns, RZ90)
    cov = {"transposed_R": _transposed, "shortcut": _shortcut, "no_quirk": _no_quirk}[variant]
    bad, _ = X.ne_block_exact(vs, vt, nt, d2, GICP, ns, RZ90, cov=cov)
    assert (np.abs(X.block_floats(bad) - X.block_floats(good)) > bound).any()

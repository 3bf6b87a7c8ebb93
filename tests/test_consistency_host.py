"""Local consistency on the host (no GPU): me_consistency_finalize against the numpy statement of tests/consistency_ref.py
bit for bit, the struct mirrors against the header, the exports, and the reference statement against hand cases."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import consistency_ref as CR  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROW_FIELDS = ("n_points", "n_query", "n_valid", "n_pv", "sum_entropy", "sum_pv", "sum_sqrt_pv", "mme", "mpv", "mean_plane_std",
              "max_pv")
WHOLE_FIELDS = ("n_points", "n_query", "n_valid", "n_pv", "sum_entropy", "sum_pv", "sum_sqrt_pv", "mme", "mpv", "mean_plane_std",
                "max_pv")


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _bits(x):
    return np.asarray(x, np.float64).view(np.uint64)


def _block(rng, n, empty=(), no_pv=(), no_valid=()):
    B = max(n, 1)
    blk = np.zeros((CR.SUM_F + CR.MAX_F) * B)
    for r in range(B):
        nq = int(rng.integers(1, 5000))
        nv = int(rng.integers(0, nq + 1))
        npv = int(rng.integers(0, nq + 1))
        if r in empty:
            nq = nv = npv = 0
        if r in no_pv:
            npv = 0
        if r in no_valid:
            nv = 0
        pv = rng.random(npv) * 1e-4
        blk[r * CR.SUM_F:(r + 1) * CR.SUM_F] = [nq, nv, npv, rng.normal(-2.0, 1.0) * nv, pv.sum(), np.sqrt(pv).sum()]
        blk[CR.SUM_F * B + r] = pv.max() if npv else 0.0
    return blk


def _check(got, rows, whole):
    for f in ROW_FIELDS:
        want = np.array([r[f] for r in rows], dtype=got[f].dtype)
        assert np.array_equal(_bits(got[f]) if want.dtype == np.float64 else got[f],
                              _bits(want) if want.dtype == np.float64 else want), f
    if rows:
        assert np.array_equal(got["index"], np.array([r["index"] for r in rows]))
        assert np.array_equal(_bits(got["min"]), _bits(np.array([r["min"] for r in rows])))
        assert np.array_equal(_bits(got["max"]), _bits(np.array([r["max"] for r in rows])))
    for f in WHOLE_FIELDS:
        a, b = got["whole"][f], whole[f]
        if isinstance(b, float):
            assert _bits(a) == _bits(b), f
        else:
            assert a == b, f


@pytest.mark.parametrize("n", [0, 1, 7, 300])
def test_finalize_matches_numpy_bit_for_bit(api, n):
    rng = np.random.default_rng(n + 11)
    s = 0.0 if n == 0 else 0.37
    index = rng.integers(-50, 50, (n, 3))
    npts = rng.integers(1, 9000, n)
    kw = dict(empty={1, 4}, no_pv={2, 5}, no_valid={3}) if n > 5 else {}
    blk = _block(rng, n, **kw)
    got = api.consistency_finalize(s, index, npts, 123456, blk)
    rows, whole = CR.finalize(s, index, npts, 123456, blk)
    _check(got, rows, whole)
    assert got["whole"]["n_regions"] == n and got["whole"]["region_size"] == s


def test_finalize_empty_and_invalid_cases(api):
    blk = np.zeros(CR.SUM_F + CR.MAX_F)
    blk[:3] = [10, 0, 0]
    got = api.consistency_finalize(0.0, np.zeros((0, 3)), [], 10, blk)
    w = got["whole"]
    assert w["n_query"] == 10 and w["mme"] == 0.0
    assert math.isnan(w["mpv"]) and math.isnan(w["mean_plane_std"]) and math.isnan(w["max_pv"])
    # a perfect plane: no valid entropy, valid plane variances of 0
    blk[:3] = [10, 0, 10]
    w = api.consistency_finalize(0.0, np.zeros((0, 3)), [], 10, blk)["whole"]
    assert w["mme"] == 0.0 and w["mpv"] == 0.0 and w["max_pv"] == 0.0 and w["n_pv"] == 10


def test_finalize_refuses_bad_arguments(api):
    with pytest.raises(api.MapEvalError):
        api.consistency_finalize(-1.0, np.zeros((1, 3)), [1], 1, np.zeros(7))
    with pytest.raises(api.MapEvalError):       # s = 0 has no rows
        api.consistency_finalize(0.0, np.zeros((1, 3)), [1], 1, np.zeros(7))
    with pytest.raises(api.MapEvalError):       # s > 0 needs rows
        api.consistency_finalize(1.0, np.zeros((0, 3)), [], 1, np.zeros(7))
    with pytest.raises(ValueError):
        api.consistency_finalize(1.0, np.zeros((2, 3)), [1, 2], 1, np.zeros(7))


def test_struct_sizes_and_exports_match_the_header(tmp_path):
    names = ["me_consistency_row", "me_consistency_result"]
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "mapeval_b200.h"\nint main(void){' +
                   "".join(f'printf("%zu\\n", sizeof({n}));' for n in names) +
                   'printf("%d %d %d\\n", ME_CONSISTENCY_SUM_FIELDS, ME_CONSISTENCY_MAX_FIELDS, ME_CONSISTENCY_WALK);return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = subprocess.check_output([str(exe)]).decode().split("\n")
    assert [int(x) for x in out[:2]] == [C.sizeof(getattr(A, n)) for n in names]
    assert [int(x) for x in out[2].split()] == [A.ME_CONSISTENCY_SUM_FIELDS, A.ME_CONSISTENCY_MAX_FIELDS, A.ME_CONSISTENCY_WALK]
    from cloud_map_evaluation_b200 import _lib
    L = _lib.load()
    for s in ("me_consistency_begin", "me_consistency_block", "me_consistency_end", "me_consistency", "me_consistency_finalize",
              "me_get_consistency_points"):
        assert s in _lib.SYMBOLS
        getattr(L, s)


def test_reference_statement_hand_cases():
    # a square grid in the plane z = 0: the exact covariance has a zero row and column, lambda3 = 0 exactly
    g = np.array([(x * 0.125, y * 0.125, 0.0) for x in range(7) for y in range(7)])
    ex = CR.exact_points(g, 0.3, 3)
    ok = ex["k"] >= 3
    assert ok.any() and np.all(ex["lam"][ok] == 0.0)
    # two planes delta apart, a query with a neighbours on its plane at offset 0 and b on the other at offset delta:
    # the z variance is a b delta^2 / (k (k - 1)), and with the in-plane spread much larger it is the smallest eigenvalue
    delta = 0.01
    P = np.array([(x * 0.125, y * 0.125, z) for z in (0.0, delta) for x in range(9) for y in range(9)])
    i = 4 * 9 + 4
    nb = [j for j in range(len(P)) if j != i and ((P[j] - P[i]) ** 2).sum() < 0.3 ** 2]
    a = sum(1 for j in nb if P[j, 2] == 0.0)
    b = len(nb) - a
    k = len(nb)
    cov = CR.exact_cov(P, i, nb)
    assert float(cov[2][2]) == pytest.approx(a * b * delta ** 2 / (k * (k - 1)), rel=1e-12)
    lam = CR.smallest_eig(cov)
    assert lam == pytest.approx(float(cov[2][2]), rel=1e-9)
    assert CR.fp64_bound(P, i, np.array(nb), cov) < 1e-12
    # an isotropic cube corner set: all three eigenvalues equal
    c = np.array([(x, y, z) for x in (-1.0, 1.0) for y in (-1.0, 1.0) for z in (-1.0, 1.0)] + [(0.0, 0.0, 0.0)])
    cov = CR.exact_cov(c, 8, list(range(8)))
    assert CR.smallest_eig(cov) == pytest.approx(8.0 / 7.0, rel=1e-15)

"""CPU checks of the numpy statement of the drift per region (drift_ref.py) and of the C-ABI mirror of its rows: the
statement's fold order against a plain loop, one region against a whole-cloud point-to-point ICP, and the recovery of a
known rigid motion per room of an indoor scene."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import drift_ref as D
from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import _lib, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def lib():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return _lib.load()


def test_row_struct_matches_the_header(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mapeval_b200.h"\nint main(){printf("%zu %zu %zu\\n", '
                   'sizeof(me_drift_row), offsetof(me_drift_row, T), offsetof(me_drift_row, status));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    size, off_t, off_s = (int(x) for x in subprocess.check_output([str(exe)], text=True).split())
    assert size == C.sizeof(A.me_drift_row)
    assert off_t == A.me_drift_row.T.offset and off_s == A.me_drift_row.status.offset
    text = open(os.path.join(ROOT, "include", "mapeval_b200.h")).read()
    assert "ME_DRIFT_CONVERGED = 0, ME_DRIFT_ITERATION_LIMIT = 1, ME_DRIFT_TOO_FEW = 2" in text
    assert (A.ME_DRIFT_CONVERGED, A.ME_DRIFT_ITERATION_LIMIT, A.ME_DRIFT_TOO_FEW) == (0, 1, 2)


def test_fold_follows_the_documented_order():
    """the vectorised fold equals a plain loop over lanes, the shuffle tree and the chunks, bit for bit, and differs from a
    plain sum (the order is visible in the bits)"""
    rng = np.random.RandomState(3)
    n = 5000
    rid = rng.randint(0, 3, n)
    rid[:2600] = 1                                   # one region of three chunks
    t = rng.randn(n, 2) * np.exp(rng.randn(n, 2) * 4)
    L = D.Layout(rid, 3)
    got = D.fold(L, t)
    for r in range(3):
        pts = np.flatnonzero(rid == r)
        tot = np.zeros(2)
        for c0 in range(0, len(pts), D.CHUNK):
            ch = pts[c0:c0 + D.CHUNK]
            lanes = np.zeros((32, 2))
            for k, i in enumerate(ch):
                lanes[k % 32] = lanes[k % 32] + t[i]
            o = 16
            while o:
                lanes = lanes[:o] + lanes[o:2 * o]
                o //= 2
            tot = tot + lanes[0]
        assert got[r].tobytes() == tot.tobytes()
    assert any(got[r].tobytes() != t[rid == r].sum(0).tobytes() for r in range(3))


def _scene(n, seed, motion):
    gt = synth.uniform_box(n, 2.0, seed) + np.array([0.2, 1.3, 0.4])
    noise = 1e-3 * np.random.RandomState(seed).randn(n, 3)
    return D.apply(motion, gt + noise, about=gt.mean(0)), gt


def test_one_region_is_a_whole_cloud_point_to_point_icp():
    """with one region the loop is point-to-point ICP: the same iterations, pairs and convergence; T, fitness and rmse to
    1e-9 (the two differ in compounding and in the order of the sums)"""
    est, gt = _scene(6000, 11, D.rigid(0.8, (0.3, 0.2, 1.0), (0.01, -0.006, 0.004)))
    rows, blocks = D.drift(est, gt, 100.0, 0.1)
    assert len(rows["index"]) == 1
    T, fit, rmse, nc, it, conv = D.icp_whole(est, gt, 0.1)
    assert rows["iterations"][0] == it and rows["n_corr"][0] == nc
    assert rows["status"][0] == (A.ME_DRIFT_CONVERGED if conv else A.ME_DRIFT_ITERATION_LIMIT)
    np.testing.assert_allclose(rows["T"][0], T, rtol=0, atol=1e-9)
    np.testing.assert_allclose([rows["fitness"][0], rows["rmse"][0]], [fit, rmse], rtol=0, atol=1e-9)
    assert len(blocks) == it + 1
    assert rows["rmse"][0] < rows["rmse_before"][0]


def test_compounding_is_not_the_statement():
    """moving the moved points by each update (as whole-cloud ICP does) changes the bits of the result"""
    est, gt = _scene(4000, 12, D.rigid(1.0, (1, 0, 0.2), (0.02, 0.0, -0.01)))
    a, _ = D.drift(est, gt, 0.7, 0.15, max_iteration=6)
    b, _ = D.drift(est, gt, 0.7, 0.15, max_iteration=6, compound=True)
    assert a["T"].tobytes() != b["T"].tobytes()


def test_statement_recovers_each_rooms_motion():
    est, gt, motions = D.indoor(40000, 3, 5)
    rows, _ = D.drift(est, gt, 8.0, 0.2)
    assert len(rows["index"]) == len(motions) == 9
    for r, key in enumerate(rows["index"]):
        M = motions[tuple(key)]
        Tinv = np.linalg.inv(rows["T"][r])
        assert np.abs(Tinv[:3, 3] - M[:3, 3]).max() < 2e-3, key
        assert D.angle_of(Tinv[:3, :3] @ M[:3, :3].T) < 0.02, key
        assert rows["rmse"][r] < rows["rmse_before"][r]
        assert rows["status"][r] == A.ME_DRIFT_CONVERGED
        # the shift is the correction at the centroid: minus the motion's displacement there
        c = rows["centroid"][r]
        np.testing.assert_allclose(rows["shift"][r], -(M[:3, :3] @ c + M[:3, 3] - c), atol=2e-3)

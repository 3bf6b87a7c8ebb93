"""me_nn_curve_finalize (host only, no GPU): curve blocks built with numpy from the oracle's nearest neighbours against the
exact reference, against me_nn_finalize on five-level accumulators of the same pairs, and the rejection of bad levels."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import _lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import exact_ref as X  # noqa: E402

R = 1.0


@pytest.fixture(scope="module")
def api():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    from cloud_map_evaluation_b200 import api as _api
    return _api


@pytest.fixture(scope="module")
def pairs():
    """(sq, d) of the kept pairs of both directions (geometric pairing, d2 <= R), and the cloud sizes"""
    from oracle import oracle as O
    from cloud_map_evaluation_b200 import synth
    est, gt, _ = synth.make_pair("C1", scale=0.03)
    out = []
    for q, r in ((est, gt), (gt, est)):
        idx, d2 = O.knn1(q, r)
        sq, d, _ = X.kept_pairs(q, r, idx, d2, R, A.ME_CUTOFF_SQDIST_LE_R)
        out.append((sq, d))
    return out, len(est), len(gt)


def _accum(sq, d, n_query, tau5=None):
    a = A.me_nn_accum()
    a.n_query, a.n_corr = n_query, len(d)
    a.sum_d_all, a.sum_d2_all = d.sum(), sq.sum()
    a.rank_n[0], a.rank_mean[0] = len(d), d.mean()
    a.rank_m2[0] = ((d - d.mean()) ** 2).sum()
    for k, t in enumerate(tau5 or []):
        m = d <= t
        a.n_inlier[k], a.sum_d[k], a.sum_d2[k] = int(m.sum()), d[m].sum(), sq[m].sum()
    return a


def _block(dirs, levels):
    """the curve block of numpy: per direction count, sum d, sum sq of the bins 0..K, then n_ub (0)"""
    K = len(levels)
    parts = []
    for sq, d in dirs:
        b = np.searchsorted(levels, d, side="left")        # first k with d <= tau_k, K above every level
        parts += [np.bincount(b, minlength=K + 1).astype(float), np.bincount(b, d, minlength=K + 1),
                  np.bincount(b, sq, minlength=K + 1), [0.0]]
    return np.concatenate(parts)


def test_curve_finalize_against_exact(api, pairs):
    dirs, n_est, n_gt = pairs
    d_all = np.concatenate([dirs[0][1], dirs[1][1]])
    levels = np.unique(np.concatenate([np.linspace(0.0, 0.1, 40), np.quantile(d_all, [0.1, 0.5, 0.9]),
                                       np.nextafter(np.quantile(d_all, [0.5]), 0.0)]))
    p = A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], R, pairing=A.ME_PAIRING_GEOMETRIC)
    e, g = _accum(*dirs[0], n_est), _accum(*dirs[1], n_gt)
    cur = api.curve_finalize(p, e, g, _block(dirs, levels), levels, n_est, n_gt)
    for name, (sq, d), n in (("est_to_gt", dirs[0], n_est), ("gt_to_est", dirs[1], n_gt)):
        ex = X.dir_stats(sq, d, n, levels)
        assert list(cur[name]["n_inlier"]) == ex["n_inlier"]
        mean_all = float(ex["mean_all"])
        for k in range(len(levels)):
            for f in ("mean", "rmse", "fitness"):
                assert abs(cur[name][f][k] - ex[f][k]) <= X.rel_bound(ex[f][k]) + 1e-15 * len(d) * abs(ex[f][k]), (name, f, k)
            assert abs(cur[name]["sigma"][k] - ex["sigma"][k]) <= X.sigma_bound(ex["sigma"][k], mean_all) + \
                1e-15 * len(d) * mean_all, (name, k)


def test_curve_finalize_equals_nn_finalize_at_five_levels(api, pairs):
    dirs, n_est, n_gt = pairs
    tau5 = [0.01, 0.05, 0.08, 0.1, 0.2]
    p = A.make_nn_params(tau5, R, pairing=A.ME_PAIRING_GEOMETRIC)
    e, g = _accum(*dirs[0], n_est, tau5), _accum(*dirs[1], n_gt, tau5)
    L = _lib.load()
    ref = A.me_nn_result()
    assert L.me_nn_finalize(C.byref(p), C.byref(e), C.byref(g), n_est, n_gt, C.byref(ref)) == A.ME_OK
    cur = api.curve_finalize(p, e, g, _block(dirs, np.asarray(tau5)), tau5, n_est, n_gt)
    for name in ("est_to_gt", "gt_to_est"):
        r = getattr(ref, name)
        assert list(cur[name]["n_inlier"]) == list(r.n_inlier)
        for f in ("mean", "rmse", "fitness", "sigma"):
            np.testing.assert_allclose(cur[name][f], list(getattr(r, f)), rtol=1e-12, atol=0)
    for f in ("cd", "f1", "iou"):
        np.testing.assert_allclose(cur[f], list(getattr(ref, f)), rtol=1e-12, atol=0)
    np.testing.assert_array_equal(cur["tau"], tau5)


def test_curve_finalize_rejects_bad_levels_and_mismatched_blocks(api, pairs):
    dirs, n_est, n_gt = pairs
    p = A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], R, pairing=A.ME_PAIRING_GEOMETRIC)
    e, g = _accum(*dirs[0], n_est), _accum(*dirs[1], n_gt)
    L = _lib.load()
    rows = (A.me_curve_row * (A.ME_CURVE_MAX_LEVELS + 1))()
    dp = C.POINTER(C.c_double)
    for bad in ([0.1, float("nan")], [-1e-9, 0.1], [0.2, 0.1], [0.1, float("inf")], [0.0] * (A.ME_CURVE_MAX_LEVELS + 1)):
        t = np.asarray(bad, np.float64)
        blk = np.zeros(A.curve_block_len(len(t)))
        rc = L.me_nn_curve_finalize(C.byref(p), C.byref(e), C.byref(g), blk.ctypes.data_as(dp), t.ctypes.data_as(dp), len(t),
                                    n_est, n_gt, rows)
        assert rc == A.ME_ERR_INVALID, bad
    t = np.array([0.1])
    assert L.me_nn_curve_finalize(C.byref(p), C.byref(e), C.byref(g), np.zeros(4).ctypes.data_as(dp), t.ctypes.data_as(dp), 0,
                                  n_est, n_gt, rows) == A.ME_ERR_INVALID
    # a block whose counts do not add up to the accumulators' kept pairs comes from another evaluation
    levels = np.array([0.05, 0.1])
    with pytest.raises(api.MapEvalError):
        api.curve_finalize(p, e, g, np.zeros(A.curve_block_len(2)), levels, n_est, n_gt)
    api.curve_finalize(p, e, g, _block(dirs, levels), levels, n_est, n_gt)


def test_curve_row_mirror_matches_the_header(tmp_path):
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mapeval_b200.h"\n'
                   'int main(){printf("%zu %zu %zu %d\\n", sizeof(me_curve_row), offsetof(me_curve_row, gt_to_est), '
                   'sizeof(me_curve_dir), ME_CURVE_MAX_LEVELS);return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [C.sizeof(A.me_curve_row), A.me_curve_row.gt_to_est.offset, C.sizeof(A.me_curve_dir), A.ME_CURVE_MAX_LEVELS]

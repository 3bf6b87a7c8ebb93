"""me_surface_finalize (host only, no GPU): the point-to-plane result from a reduced block against the numpy statement of
tests/surface_ref.py bit for bit — on blocks folded from random records with zero, NaN and non-unit normals, with the moments
spread over several rank slots, with empty directions, with n_nc = 0 and with one direction — and the ctypes mirrors of
me_surface_dir / me_surface_result and the block lengths against the header, and the exports."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import _lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import surface_ref as S  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAU = [0.5, 0.3, 0.2, 0.1, 0.05]
SYMBOLS = ("me_nn_surface_begin", "me_nn_surface_normals_slice", "me_nn_surface_block", "me_nn_surface_end", "me_nn_surface",
           "me_surface_finalize")


@pytest.fixture(scope="module")
def api():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    from cloud_map_evaluation_b200 import api as _api
    return _api


def random_normals(rng, n):
    """unit, non-unit, zero, NaN and infinite normals"""
    v = rng.normal(size=(n, 3)) * rng.choice([1.0, 0.25, 3.0], (n, 1))
    v[rng.random(n) < 0.05] = 0.0
    v[rng.random(n) < 0.03, 1] = np.nan
    v[rng.random(n) < 0.01, 2] = np.inf
    return v


def random_records(rng, query, ref, R):
    """caller-order records: a random reference point for most queries (its d2 Eigen-ordered), none (-1) for the rest"""
    idx = rng.integers(0, len(ref), len(query)).astype(np.int32)
    idx[rng.random(len(query)) < 0.1] = -1
    d2 = np.full(len(query), np.inf)
    h = idx >= 0
    d2[h] = S.sqnorm_eigen(query[h] - ref[idx[h]])
    return idx, d2


def _bits_equal(got, want, path=""):
    for k, v in want.items():
        if isinstance(v, dict):
            _bits_equal(got[k], v, path + k + ".")
        elif np.asarray(v).dtype.kind == "f":
            np.testing.assert_array_equal(np.asarray(got[k], np.float64).view(np.uint64), np.asarray(v, np.float64).view(np.uint64),
                                          path + k)
        else:
            np.testing.assert_array_equal(got[k], v, path + k)


@pytest.mark.parametrize("seed,n_est,n_gt,mode,full,directions", [
    (0, 500, 700, A.ME_CUTOFF_SQDIST_LE_R, True, 0), (1, 2000, 1500, A.ME_CUTOFF_DIST_LT_R, True, 0),
    (2, 1000, 1000, A.ME_CUTOFF_SQDIST_LE_R, False, 0), (3, 800, 600, A.ME_CUTOFF_DIST_LT_R, True, 1)])
def test_finalize_matches_numpy_bit_for_bit(api, seed, n_est, n_gt, mode, full, directions):
    rng = np.random.default_rng(seed)
    est, gt = rng.uniform(-1, 1, (n_est, 3)), rng.uniform(-1, 1, (n_gt, 3))
    p = A.make_nn_params(TAU, 0.6, cutoff_mode=mode, pairing=A.ME_PAIRING_GEOMETRIC, want_full_cd=full, directions=directions)
    rec = (random_records(rng, est, gt, 0.6), random_records(rng, gt, est, 0.6))
    blk = S.block(S.fold_both(est, gt, random_normals(rng, n_est), random_normals(rng, n_gt), rec, p))
    _bits_equal(api.surface_finalize(p, blk, n_est, n_gt), S.finalize(p, blk, n_est, n_gt))


def test_moments_over_rank_slots(api):
    """three ranks' blocks SUM-reduced: the finalizer merges the slots in rank order"""
    rng = np.random.default_rng(7)
    est, gt = rng.uniform(-1, 1, (3000, 3)), rng.uniform(-1, 1, (2000, 3))
    p = A.make_nn_params(TAU, 0.6, pairing=A.ME_PAIRING_GEOMETRIC)
    ne, ng = random_normals(rng, len(est)), random_normals(rng, len(gt))
    (ie, de), (ig, dg) = random_records(rng, est, gt, 0.6), random_records(rng, gt, est, 0.6)
    total = np.zeros(A.ME_SURFACE_BLOCK_SUM + A.ME_SURFACE_BLOCK_MAX)
    for r, (a, b) in enumerate(((0, 1000), (1000, 2200), (2200, 3000))):
        ie_r = np.full_like(ie, -2)
        ie_r[a:b] = ie[a:b]
        ig_r = np.full_like(ig, -2)
        ig_r[a * 2 // 3:b * 2 // 3] = ig[a * 2 // 3:b * 2 // 3]
        blk = S.block(S.fold_both(est, gt, ne, ng, ((ie_r, de), (ig_r, dg)), p))
        for q in range(2):          # this rank's moments to slot r
            base = q * S.NN + S.MOM
            for k in range(3):
                v = blk[base + k * A.ME_MAX_WORLD]
                blk[base + k * A.ME_MAX_WORLD] = 0.0
                blk[base + k * A.ME_MAX_WORLD + r] = v
        s = A.ME_SURFACE_BLOCK_SUM
        total[:s] += blk[:s]
        total[s:] = np.maximum(total[s:], blk[s:])
    got = api.surface_finalize(p, total, len(est), len(gt))
    _bits_equal(got, S.finalize(p, total, len(est), len(gt)))
    whole = S.finalize(p, S.block(S.fold_both(est, gt, ne, ng, ((ie, de), (ig, dg)), p)), len(est), len(gt))
    for d in ("est_to_gt", "gt_to_est"):
        for f in ("n_corr", "n_inlier", "n_no_normal", "n_no_normal_nn", "n_nc", "max_e", "max_e_nn"):
            np.testing.assert_array_equal(got[d][f], whole[d][f], f)
        np.testing.assert_allclose(got[d]["sigma"], whole[d]["sigma"], rtol=1e-9)


def test_edge_cases(api):
    """an empty block: NaN means and normal consistency, zero maxima; pairs without usable query normals: n_nc = 0"""
    p = A.make_nn_params(TAU, 1.0, pairing=A.ME_PAIRING_GEOMETRIC)
    blk = np.zeros(A.ME_SURFACE_BLOCK_SUM + A.ME_SURFACE_BLOCK_MAX)
    r = api.surface_finalize(p, blk, 10, 20)
    _bits_equal(r, S.finalize(p, blk, 10, 20))
    for d in ("est_to_gt", "gt_to_est"):
        assert np.isnan(r[d]["normal_consistency"]) and r[d]["max_e"] == 0.0 and r[d]["n_nc"] == 0
        assert np.all(np.isnan(r[d]["mean"]))
    assert np.isnan(r["normal_consistency"])
    rng = np.random.default_rng(3)
    est, gt = rng.uniform(-1, 1, (400, 3)), rng.uniform(-1, 1, (300, 3))
    rec = (random_records(rng, est, gt, 1.0), random_records(rng, gt, est, 1.0))
    blk = S.block(S.fold_both(est, gt, np.zeros((400, 3)), rng.normal(size=(300, 3)), rec, p))
    r = api.surface_finalize(p, blk, 400, 300)
    _bits_equal(r, S.finalize(p, blk, 400, 300))
    assert r["est_to_gt"]["n_nc"] == 0 and np.isnan(r["est_to_gt"]["normal_consistency"])
    assert r["gt_to_est"]["n_corr"] == 0 and r["gt_to_est"]["n_no_normal"] > 0
    with pytest.raises(ValueError):
        api.surface_finalize(p, blk[:-1], 400, 300)


def test_struct_mirrors_match_the_header(tmp_path):
    fields = {"me_surface_dir": [f[0] for f in A.me_surface_dir._fields_],
              "me_surface_result": [f[0] for f in A.me_surface_result._fields_]}
    src = tmp_path / "sz.c"
    body = ""
    for name, fs in fields.items():
        body += f'printf("%zu\\n", sizeof({name}));'
        body += "".join(f'printf("%zu\\n", offsetof({name}, {f}));' for f in fs)
    body += 'printf("%d\\n%d\\n", ME_SURFACE_BLOCK_SUM, ME_SURFACE_BLOCK_MAX);'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mapeval_b200.h"\nint main(){' + body + "return 0;}\n")
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    want = []
    for name, fs in fields.items():
        st = getattr(A, name)
        want += [C.sizeof(st)] + [getattr(st, f).offset for f in fs]
    want += [A.ME_SURFACE_BLOCK_SUM, A.ME_SURFACE_BLOCK_MAX]
    assert got == want


def test_surface_symbols_are_exported():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    for s in SYMBOLS:
        assert f" T {s}\n" in out and s in _lib.SYMBOLS

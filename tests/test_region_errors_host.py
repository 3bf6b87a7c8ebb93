"""me_region_finalize (host only, no GPU): the per-region rows from a reduced block against a numpy restatement of
me_nn_finalize's per-level arithmetic (dir_level / pair_level, map_eval.cpp:1125-1131, 1245-1253) on random and edge-case
blocks, the rejection of bad arguments, and the ctypes mirrors of me_region_dir / me_region_row against the header."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F, M = A.ME_REGION_SUM_FIELDS, A.ME_REGION_MAX_FIELDS


@pytest.fixture(scope="module")
def api():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _block(rng, n, empty_every=0, no_pairs_every=0):
    """a reduced block of n regions with consistent counts: n_inlier[k] <= n_corr <= n_query <= the region's point count"""
    n_est = rng.integers(0, 2000, n)
    n_gt = rng.integers(0, 2000, n)
    if empty_every:
        n_est[::empty_every] = 0
        n_gt[1::empty_every] = 0
        n_est[n_est + n_gt == 0] = 1
    s = np.zeros((n, 2, F))
    mx = np.zeros((n, 2, M))
    for q, pts in enumerate((n_est, n_gt)):
        n_query = pts.copy()
        n_corr = (n_query * rng.random(n)).astype(np.int64)
        if no_pairs_every:
            n_corr[::no_pairs_every] = 0
        inl = np.sort((n_corr[:, None] * rng.random((n, 5))).astype(np.int64), axis=1)
        sum_d = inl * rng.random((n, 5)) * 0.1
        sum_d2 = inl * rng.random((n, 5)) * 0.01
        s[:, q, 0], s[:, q, 1], s[:, q, 2:7], s[:, q, 7:12], s[:, q, 12:17] = n_query, n_corr, inl, sum_d, sum_d2
        s[:, q, 17] = n_query * rng.random(n) * 0.2
        mx[:, q, 0] = np.where(n_corr > 0, rng.random(n), 0.0)
        mx[:, q, 1] = np.where(n_query > 0, rng.random(n) + 1.0, 0.0)
    return n_est, n_gt, np.concatenate([s.reshape(-1), mx.reshape(-1)])


def _restate(s_size, index, n_est, n_gt, blk):
    """numpy statement of me_region_finalize in me_nn_finalize's operation order"""
    n = len(n_est)
    s = blk[:2 * F * n].reshape(n, 2, F)
    mx = blk[2 * F * n:].reshape(n, 2, M)
    out = {"index": index, "min": index * s_size, "max": (index + 1) * s_size, "n_est": n_est, "n_gt": n_gt}
    with np.errstate(all="ignore"):
        for q, name in enumerate(("est_to_gt", "gt_to_est")):
            v = s[:, q]
            nc = v[:, 1:2]
            src = (n_est if q == 0 else n_gt).astype(np.float64)[:, None]
            out[name] = dict(n_query=v[:, 0].astype(np.int64), n_corr=v[:, 1].astype(np.int64), n_inlier=v[:, 2:7].astype(np.int64),
                             sum_d=v[:, 7:12], sum_d2=v[:, 12:17], sum_nn_dist=v[:, 17], max_d=mx[:, q, 0], max_nn=mx[:, q, 1],
                             mean=v[:, 7:12] / nc, rmse=np.sqrt(v[:, 12:17] / nc), fitness=v[:, 2:7] * 1.0 / src,
                             mean_nn=v[:, 17] / v[:, 0])
        e, g = out["est_to_gt"], out["gt_to_est"]
        out["cd"] = e["rmse"] + g["rmse"]
        out["f1"] = 2 * e["fitness"] * e["rmse"] / (e["fitness"] + e["rmse"])
        inter = e["n_inlier"]
        out["iou"] = inter.astype(np.float64) / (n_est[:, None] + n_gt[:, None] - inter).astype(np.float64)
    return out


def _same(got, want):
    for k, v in want.items():
        if isinstance(v, dict):
            _same(got[k], v)
        elif np.asarray(v).dtype.kind == "f":
            np.testing.assert_array_equal(np.asarray(got[k], np.float64).view(np.uint64), np.asarray(v, np.float64).view(np.uint64), k)
        else:
            np.testing.assert_array_equal(got[k], v, k)


@pytest.mark.parametrize("seed,n,empty_every,no_pairs_every", [(0, 1, 0, 0), (1, 37, 0, 0), (2, 1000, 3, 4), (3, 5000, 2, 2)])
def test_finalize_matches_numpy_bit_for_bit(api, seed, n, empty_every, no_pairs_every):
    rng = np.random.default_rng(seed)
    n_est, n_gt, blk = _block(rng, n, empty_every, no_pairs_every)
    index = np.sort(rng.integers(-(1 << 20) + 1, 1 << 20, (n, 3)), axis=0)
    s = [0.1, 3.0, 0.37][seed % 3]
    _same(api.region_finalize(s, index, n_est, n_gt, blk), _restate(s, index, n_est, n_gt, blk))


def test_edge_cases(api):
    """a region with no pairs gives NaN mean / rmse and zero fitness; a direction with no points gives NaN fitness too"""
    n_est, n_gt = np.array([5, 0, 3]), np.array([0, 4, 3])
    s = np.zeros((3, 2, F))
    s[0, 0, 0] = 5           # 5 est queries, no pair within reach
    s[1, 1, 0] = 4
    s[1, 1, 1] = 2           # 2 gt->est pairs, one within every level
    s[1, 1, 2:7] = 1
    s[1, 1, 7:12] = 0.25
    s[1, 1, 12:17] = 0.0625
    blk = np.concatenate([s.reshape(-1), np.zeros(3 * 2 * M)])
    r = api.region_finalize(1.0, np.zeros((3, 3), np.int64) + np.arange(3)[:, None], n_est, n_gt, blk)
    _same(r, _restate(1.0, np.zeros((3, 3), np.int64) + np.arange(3)[:, None], n_est, n_gt, blk))
    e, g = r["est_to_gt"], r["gt_to_est"]
    assert np.all(np.isnan(e["mean"][0])) and np.all(e["fitness"][0] == 0.0) and e["mean_nn"][0] == 0.0
    assert np.all(np.isnan(e["fitness"][1])) and np.isnan(e["mean_nn"][1])      # no est point in region 1
    assert np.all(g["mean"][1] == 0.125) and np.all(g["fitness"][1] == 0.25)
    assert np.all(np.isnan(r["cd"][1])) and np.all(r["iou"][2] == 0.0)


def test_bad_arguments_are_refused(api):
    blk = np.zeros(2 * (F + M))
    for s in (0.0, -1.0, np.nan, np.inf):
        with pytest.raises(api.MapEvalError):
            api.region_finalize(s, np.zeros((1, 3)), [1], [1], blk)
    with pytest.raises(ValueError):
        api.region_finalize(1.0, np.zeros((1, 3)), [1], [1], blk[:-1])
    assert api.region_finalize(1.0, np.zeros((0, 3)), [], [], [])["n_est"].shape == (0,)


def test_struct_mirrors_match_the_header(tmp_path):
    fields = {"me_region_dir": [f[0] for f in A.me_region_dir._fields_], "me_region_row": [f[0] for f in A.me_region_row._fields_]}
    src = tmp_path / "sz.c"
    body = ""
    for name, fs in fields.items():
        body += f'printf("%zu\\n", sizeof({name}));'
        body += "".join(f'printf("%zu\\n", offsetof({name}, {f}));' for f in fs)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mapeval_b200.h"\nint main(){' + body + "return 0;}\n")
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    want = []
    for name, fs in fields.items():
        st = getattr(A, name)
        want += [C.sizeof(st)] + [getattr(st, f).offset for f in fs]
    assert got == want
    text = open(os.path.join(ROOT, "include", "mapeval_b200.h")).read()
    assert f"#define ME_REGION_MAX_REGIONS (1 << 21)" in text and A.ME_REGION_MAX_REGIONS == 1 << 21
    assert f"#define ME_REGION_SUM_FIELDS {F}" in text and f"#define ME_REGION_MAX_FIELDS {M}" in text


def test_region_symbols_are_exported():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    for s in ("me_nn_region_begin", "me_nn_region_block", "me_nn_region_end", "me_nn_regions", "me_region_finalize"):
        assert f" T {s}\n" in out and s in _lib.SYMBOLS

"""me_quantile_finalize (host only, no GPU): the rank arithmetic and interpolation of the exact distance quantiles against
numpy's quantile(method="linear") bit for bit, the rejection of bad probabilities, and the ctypes mirror of the result."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def api():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _lo_hi(x, p):
    """(lo, hi) = (x_k, x_min(k+1, n-1)), k = floor((n - 1) p), of the sorted x"""
    n = x.size
    k = np.floor((n - 1) * p).astype(np.int64)
    return np.stack([x[k], x[np.minimum(k + 1, n - 1)]], axis=1)


def _check(api, x, p):
    xs = np.sort(x)
    got = api.quantile_finalize(xs.size, p, _lo_hi(xs, p))
    want = np.quantile(x, p, method="linear")
    np.testing.assert_array_equal(got.view(np.uint64), np.asarray(want, np.float64).view(np.uint64))


@pytest.mark.parametrize("n", [1, 2, 3, 17, 1000, 123457])
def test_finalize_matches_numpy_bit_for_bit(api, n):
    rng = np.random.default_rng(n)
    x = rng.exponential(0.05, n)
    p = np.concatenate([[0.0, 1.0, 0.5, 0.9, 0.95, 0.99], rng.random(58)])
    _check(api, x, p)


@pytest.mark.parametrize("n", [2, 3, 11, 1001])
def test_finalize_at_exact_multiples_of_the_spacing(api, n):
    """p = j / (n - 1) lands on an order statistic (g = 0 in exact arithmetic; in fp64 g may be a few ulp off either way)"""
    rng = np.random.default_rng(7 + n)
    x = rng.random(n) * 10.0
    for j0 in range(0, n, 64):
        p = np.arange(j0, min(n, j0 + 64)) / (n - 1)
        _check(api, x, p)


@pytest.mark.parametrize("seed", range(6))
def test_finalize_on_tie_heavy_arrays(api, seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(2, 5000))
    levels = rng.random(int(rng.integers(1, 6))) * 3.0
    x = levels[rng.integers(0, levels.size, n)]
    p = np.concatenate([[0.0, 1.0], rng.random(62)])
    _check(api, x, p)


def test_finalize_on_large_spread(api):
    """distances from 1e-9 m to 1e4 m: the interpolation's two branches far from each other"""
    rng = np.random.default_rng(3)
    x = 10.0 ** rng.uniform(-9, 4, 20000)
    p = np.linspace(0.0, 1.0, 64)
    _check(api, x, p)


@pytest.mark.parametrize("p", [[], [-0.1], [1.0000000000000002], [np.nan], [np.inf], [0.5] * 65])
def test_finalize_refuses_bad_probabilities(api, p):
    lo_hi = np.zeros((max(len(p), 1), 2))
    with pytest.raises(api.MapEvalError):
        api.quantile_finalize(10, np.array(p, np.float64), lo_hi[:len(p)] if p else lo_hi[:0])


def test_finalize_refuses_an_empty_population(api):
    with pytest.raises(api.MapEvalError):
        api.quantile_finalize(0, [0.5], [[0.0, 0.0]])


def test_finalize_accepts_the_limits(api):
    x = np.arange(65, dtype=np.float64)
    p = np.linspace(0.0, 1.0, A.ME_QUANTILE_MAX_PROBS)
    _check(api, x, p)


def test_quantile_struct_mirror_matches_the_header(tmp_path):
    names = ["me_quantile_dir", "me_quantile_result"]
    fields = {"me_quantile_dir": ["n", "min", "max", "rank", "lo", "hi", "value"],
              "me_quantile_result": ["population", "n_probs", "p", "est_to_gt", "gt_to_est", "hausdorff"]}
    body = "".join(f'printf("%zu\\n", sizeof({n}));' for n in names)
    body += "".join(f'printf("%zu\\n", offsetof({n}, {f}));' for n in names for f in fields[n])
    body += 'printf("%d %d %d\\n", ME_QUANTILE_MAX_PROBS, ME_DIST_KEPT, ME_DIST_NN);'
    src = tmp_path / "q.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mapeval_b200.h"\nint main(){' + body + "return 0;}\n")
    exe = tmp_path / "q"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = subprocess.check_output([str(exe)], text=True).split()
    want = [C.sizeof(getattr(A, n)) for n in names]
    want += [getattr(A, n).__dict__[f].offset for n in names for f in fields[n]]
    assert [int(v) for v in out[:len(want)]] == want
    assert [int(v) for v in out[len(want):]] == [A.ME_QUANTILE_MAX_PROBS, A.ME_DIST_KEPT, A.ME_DIST_NN]

"""me_mom_axes (host only) against the numpy statement bit for bit, its refusals, and the MOM structs and exports against
the header."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import _lib, api

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mom_ref as R  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _same(got, ref):
    a, s = got
    b, t = ref
    assert s == t
    assert np.array_equal(a.view(np.uint64)[np.isfinite(a)], b.view(np.uint64)[np.isfinite(b)])
    assert np.array_equal(np.isnan(a), np.isnan(b))


def _normals(rng, n):
    x = rng.normal(size=(n, 3))
    return x / np.linalg.norm(x, axis=1, keepdims=True)


@pytest.mark.parametrize("angle", [10.0, 1.5, 30.0])
def test_axes_bit_for_bit_structured(angle):
    rng = np.random.default_rng(1)
    rot = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    base = np.vstack([np.tile(e, (k, 1)) for e, k in zip(np.eye(3), (500, 300, 800))])
    n = (base + rng.normal(0, 0.02, base.shape)) @ rot.T
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    h = R.histogram(n)
    _same(api.mom_axes(h, angle), R.axes(h, angle))


def test_axes_bit_for_bit_random_and_degenerate():
    rng = np.random.default_rng(2)
    for seed in range(8):
        h = rng.integers(0, 50, R.BINS) * (rng.random(R.BINS) < 0.05)
        _same(api.mom_axes(h, 10.0), R.axes(h, 10.0))
        h = R.histogram(_normals(rng, 200 + 50 * seed))
        _same(api.mom_axes(h, 7.0), R.axes(h, 7.0))
    z = np.zeros(R.BINS, np.int64)
    _same(api.mom_axes(z, 10.0), R.axes(z, 10.0))
    one = z.copy()
    one[77] = 4
    _same(api.mom_axes(one, 10.0), R.axes(one, 10.0))


def test_axes_refusals():
    h = np.zeros(R.BINS, np.int64)
    for angle in (0.0, -1.0, 30.5, float("nan")):
        with pytest.raises(api.MapEvalError):
            api.mom_axes(h, angle)
    bad = h.copy()
    bad[3] = -1
    with pytest.raises(api.MapEvalError):
        api.mom_axes(bad, 10.0)
    L = _lib.load()
    axes = (C.c_double * 9)()
    st = C.c_int32(0)
    assert L.me_mom_axes(None, 16, 10.0, axes, C.byref(st)) == A.ME_ERR_INVALID
    assert L.me_mom_axes(h.ctypes.data_as(C.POINTER(C.c_int64)), 0, 10.0, axes, C.byref(st)) == A.ME_ERR_INVALID


def test_structs_and_exports_match_the_header(tmp_path):
    src = tmp_path / "sz.c"
    names = ["me_mom_params", "me_mom_result"]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mapeval_b200.h"\nint main(){' +
                   "".join(f'printf("%zu\\n", sizeof({n}));' for n in names) +
                   'printf("%zu %zu %zu %d %d %d\\n", offsetof(me_mom_result, axis), offsetof(me_mom_result, mom), '
                   'offsetof(me_mom_result, status), ME_MOM_BINS, ME_MOM_BLOCK, ME_MOM_SMALL_FAMILY);return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = subprocess.check_output([str(exe)], text=True).split()
    assert [int(x) for x in out[:2]] == [C.sizeof(A.me_mom_params), C.sizeof(A.me_mom_result)]
    assert [int(x) for x in out[2:]] == [A.me_mom_result.axis.offset, A.me_mom_result.mom.offset, A.me_mom_result.status.offset,
                                         A.ME_MOM_BINS, A.ME_MOM_BLOCK, A.ME_MOM_SMALL_FAMILY]
    text = open(os.path.join(ROOT, "include", "mapeval_b200.h")).read()
    declared = set(re.findall(r"^ME_API\s+[\w\s\*]+?\b(me_(?:mom|get_mom)[a-z_0-9]*)\s*\(", text, flags=re.M))
    assert declared == {s for s in _lib.SYMBOLS if "mom" in s}
    exported = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    for s in declared:
        assert re.search(rf" T {s}$", exported, flags=re.M), s

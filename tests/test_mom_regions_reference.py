"""The numpy statement of the per-region MOM (tests/mom_regions_ref.py) against a plain per-region loop, the ctypes row
against the header, and api.mom_region_dict on hand-made rows.  No GPU."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mom_regions_ref as MRR  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check(rid, R, v, fam, pl, axes_status, min_family):
    got = MRR.statement(rid, R, v, fam, pl, axes_status, min_family)
    ref = MRR.loop_statement(rid, R, v, fam, pl, axes_status, min_family)
    for r, row in enumerate(ref):
        assert got["n_points"][r] == row["n_points"] and got["n_planar"][r] == row["n_planar"]
        assert list(got["n"][r]) == row["n"]
        assert got["status"][r] == row["status"]
        for j in range(3):
            if row["n"][j]:
                assert got["median"][r, j] == row["median"][j]
                assert got["mean"][r, j] == pytest.approx(row["mean"][j], rel=1e-13)
            else:
                assert math.isnan(got["median"][r, j]) and math.isnan(got["mean"][r, j])
        if row["status"] == "OK":
            assert got["mom"][r] == row["mom"]
        else:
            assert math.isnan(got["mom"][r])
    return got


def test_statement_equals_the_loop_on_random_regions():
    rng = np.random.default_rng(1)
    n, R = 20000, 37
    rid = rng.integers(0, R, n)
    v = rng.gamma(2.0, 1e-5, n)
    v[rng.random(n) < 0.05] = 0.0                                    # exact planes
    v[rng.random(n) < 0.1] = 1e-5                                   # ties
    pl = rng.random(n) < 0.8
    fam = np.where(pl, rng.integers(-1, 3, n), -1)
    for min_family in (1, 50, 10 ** 6):
        _check(rid, R, v, fam, pl, "OK", min_family)


def test_ties_small_families_and_empty_families():
    # region 0: family 0 has one member, family 1 two, family 2 none; region 1: ties everywhere; region 2: nothing planar
    rid = np.array([0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 2, 2])
    v = np.array([3e-6, 1e-6, 2e-6, 9.0, 5e-6, 5e-6, 5e-6, 5e-6, 7e-6, 7e-6, 1.0, 2.0])
    fam = np.array([0, 1, 1, -1, 0, 0, 1, 1, 2, 2, -1, -1])
    pl = np.array([1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0], bool)
    got = _check(rid, 3, v, fam, pl, "OK", 1)
    assert list(got["n"][0]) == [1, 2, 0] and got["median"][0, 0] == 3e-6
    assert got["median"][0, 1] == np.quantile([1e-6, 2e-6], 0.5)
    assert got["status"][0] == "SMALL_FAMILY" and math.isnan(got["mom"][0])
    assert got["n_planar"][0] == 4 and got["n_planar"][2] == 0
    assert got["status"][1] == "OK" and got["mom"][1] == (5e-6 + 5e-6) + 7e-6
    assert got["status"][2] == "SMALL_FAMILY" and np.isnan(got["median"][2]).all()


@pytest.mark.parametrize("status", ["NO_PLANAR", "NO_SECOND_AXIS"])
def test_no_axes_statuses_carry_to_every_row(status):
    rng = np.random.default_rng(2)
    rid = rng.integers(0, 5, 300)
    pl = rng.random(300) < (0.0 if status == "NO_PLANAR" else 0.5)
    got = _check(rid, 5, rng.random(300), np.full(300, -1), pl, status, 1)
    assert (got["status"] == status).all() and (got["n"] == 0).all() and np.isnan(got["mom"]).all()
    assert got["n_planar"].sum() == pl.sum()


def test_sums_follow_the_library_fold():
    # one segment over several chunks: the fold of the sorted values, chunk by chunk, equals a hand-written fold
    rng = np.random.default_rng(3)
    v = np.sort(rng.random(2500))
    s = MRR.segment_sums(v, np.array([0]), np.array([2500]))[0]
    parts = []
    for c in range(0, 2500, 1024):
        x = v[c:c + 1024]
        lanes = np.zeros(32)
        for i, y in enumerate(x):
            lanes[i % 32] += y
        parts.append(MRR.MR._tree(lanes[None, :])[0])
    want = 0.0
    for p in parts:
        want += p
    assert s == want


def test_region_list_is_est_then_gt_ascending():
    est = np.array([[0.5, 0.5, 0.5], [-0.5, 0.0, 0.0], [2.5, 0.1, 0.1]])
    gt = np.array([[0.7, 0.2, 0.2], [5.0, 5.0, 5.0]])
    index, re, rg = MRR.region_list(est, gt, 1.0)
    assert index.tolist() == [[-1, 0, 0], [0, 0, 0], [2, 0, 0], [5, 5, 5]]
    assert re.tolist() == [1, 0, 2] and rg.tolist() == [1, 3]
    index, re, _ = MRR.region_list(est, np.zeros((0, 3)), 1.0)
    assert len(index) == 3


def test_row_struct_matches_the_header(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mapeval_b200.h"\nint main(){'
                   'printf("%zu %zu %zu\\n", sizeof(me_mom_region_row), offsetof(me_mom_region_row, mom), '
                   'offsetof(me_mom_region_row, status));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    size, off_mom, off_status = (int(x) for x in subprocess.check_output([str(exe)], text=True).split())
    assert size == C.sizeof(A.me_mom_region_row)
    assert off_mom == A.me_mom_region_row.mom.offset and off_status == A.me_mom_region_row.status.offset


def test_mom_region_dict_on_hand_made_rows():
    from cloud_map_evaluation_b200 import api
    rows = np.zeros(2, api._MOM_REGION_ROW_DT)
    rows[0]["index"] = (-1, 0, 2)
    rows[0]["n_points"], rows[0]["n_planar"] = 10, 7
    rows[0]["n"] = (3, 2, 1)
    rows[0]["mean"] = (1.0, 2.0, 3.0)
    rows[0]["median"] = (0.5, 1.5, 2.5)
    rows[0]["mom"] = 4.5
    rows[0]["status"] = A.ME_MOM_OK
    rows[1]["index"] = (4, 5, 6)
    rows[1]["mean"] = rows[1]["median"] = (math.nan,) * 3
    rows[1]["mom"] = math.nan
    rows[1]["status"] = A.ME_MOM_NO_SECOND_AXIS
    d = api.mom_region_dict(rows, 0.5)
    assert d["index"].shape == (2, 3) and d["n"].shape == (2, 3) and d["median"].shape == (2, 3)
    assert d["lo"].tolist() == [[-0.5, 0.0, 1.0], [2.0, 2.5, 3.0]]
    assert d["hi"].tolist() == [[0.0, 0.5, 1.5], [2.5, 3.0, 3.5]]
    assert d["n_points"].tolist() == [10, 0] and d["n_planar"].tolist() == [7, 0]
    assert d["n"][0].tolist() == [3, 2, 1] and d["median"][0].tolist() == [0.5, 1.5, 2.5] and d["mom"][0] == 4.5
    assert list(d["status"]) == ["OK", "NO_SECOND_AXIS"]
    assert set(d) == {"index", "lo", "hi", "n_points", "n_planar", "n", "mean", "median", "mom", "status"}
    empty = api.mom_region_dict(np.zeros(0, api._MOM_REGION_ROW_DT), 1.0)
    assert empty["index"].shape == (0, 3) and len(empty["status"]) == 0

"""The re-hosted `map_eval` with `mom_region_size`: the key in --dump-config; bad values and a missing evaluate_mom refused
when the configuration is loaded; map_mom_regions.txt's rows equal the Python API's on the same down-sampled clouds, with
and without a ground truth and under evaluate_without_gt, and align with map_consistency.txt at equal sizes; every other
output unchanged with the key on; two GPUs against one."""
import math
import subprocess

import numpy as np
import pytest

from test_host_driver_accuracy_curve import _stable, _write_pcd, exe  # noqa: F401  (module fixture)
from test_host_driver_mom import NO_GT, R0, _config, _run, maps  # noqa: F401  (module fixture)

COLS = (["cloud", "min_x", "min_y", "min_z", "max_x", "max_y", "max_z", "n_points", "n_planar"] +
        [f"{f}_{j}" for j in (1, 2, 3) for f in ("n", "mean", "median")] + ["mom", "status"])
S = 0.5


def _read(path):
    lines = path.read_text().splitlines()
    assert lines[0].startswith("# ") and lines[1].split() == COLS
    rows = []
    for line in lines[2:]:
        v = line.split()
        assert len(v) == len(COLS)
        rows.append({c: (x if c in ("cloud", "status") else int(x) if c.startswith("n") else float(x)) for c, x in zip(COLS, v)})
    return lines[0], rows


def test_dump_config_lists_the_key(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "evaluate_mom: true\nmom_region_size: 2.5\n"))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert "mom_region_size=2.5" in out.stdout.splitlines()
    cfg.write_text(_config(tmp_path, tmp_path, ""))
    assert "mom_region_size=0" in subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True).stdout.splitlines()


@pytest.mark.parametrize("extra", ["evaluate_mom: true\nmom_region_size: -1\n", "evaluate_mom: true\nmom_region_size: nan\n",
                                   "evaluate_mom: true\nmom_region_size: inf\n", "mom_region_size: 1.0\n",
                                   "evaluate_mom: false\nmom_region_size: 1.0\n"])
def test_bad_values_are_refused_at_load(exe, tmp_path, extra):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, extra))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)     # refused before anything runs
    assert out.returncode != 0 and "mom_region_size" in out.stderr
    if "evaluate_mom: true" not in extra:
        assert "evaluate_mom" in out.stderr.split("mom_region_size", 1)[1]


def test_zero_is_off(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "mom_region_size: 0\n"))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


def _api_rows(est, gt, which, n_est, n_gt=None):
    """the Python API on the driver's clouds: the files' fp32 coordinates, down-sampled as the driver does"""
    from cloud_map_evaluation_b200 import _abi as A
    from cloud_map_evaluation_b200 import api
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(A.ME_CLOUD_EST, est.astype(np.float32).astype(np.float64))
        assert ctx.voxel_downsample(A.ME_CLOUD_EST, 0.01) == n_est
        if gt is not None:
            ctx.set_cloud(A.ME_CLOUD_GT, gt.astype(np.float32).astype(np.float64))
            assert ctx.voxel_downsample(A.ME_CLOUD_GT, 0.01) == n_gt
        out = {}
        for w, name, m in ((A.ME_CLOUD_EST, "est", 10), (A.ME_CLOUD_GT, "gt", 5)):
            if w in which:
                ctx.mom(w, R0, m)
                out[name] = ctx.mom_regions(S)
                out[name + "_cons"] = ctx.local_consistency(w, R0, m, region_size=S)
    return out


def _compare(rows, ref, name):
    got = [r for r in rows if r["cloud"] == name]
    assert len(got) == len(ref["index"])
    for k, r in enumerate(got):
        for a, c in enumerate("xyz"):
            assert r[f"min_{c}"] == pytest.approx(ref["lo"][k, a], abs=1e-12)
            assert r[f"max_{c}"] == pytest.approx(ref["hi"][k, a], abs=1e-12)
        assert r["n_points"] == ref["n_points"][k]
        # a layout ranks the points of a cell with atomics, so per-point values agree to rounding; the counts are exact away
        # from the thresholds, which these maps keep clear of
        assert r["n_planar"] == ref["n_planar"][k]
        assert r["status"] == ref["status"][k]
        for j in range(3):
            assert r[f"n_{j + 1}"] == ref["n"][k, j]
            for f in ("mean", "median"):
                if ref["n"][k, j]:
                    assert r[f"{f}_{j + 1}"] == pytest.approx(ref[f][k, j], rel=1e-9, abs=1e-15)
                else:
                    assert math.isnan(r[f"{f}_{j + 1}"])
        if ref["status"][k] == "OK":
            assert r["mom"] == pytest.approx(ref["mom"][k], rel=1e-9)
        else:
            assert math.isnan(r["mom"])


def _consistency_rows(path, name):
    lines = path.read_text().splitlines()
    head = [i for i, l in enumerate(lines) if l.startswith("cloud min_x")]
    assert len(head) == 1
    return [l.split()[:8] for l in lines[head[0] + 1:] if l.split()[0] == name]


@pytest.mark.gpu
def test_without_gt_equals_the_python_api(exe, maps):
    d, est, _ = maps
    extra = NO_GT + f"consistency_region_size: {S}\nmom_region_size: {S}\n"
    out, res = _run(exe, d, "r_nogt", est, extra, with_gt=False)
    assert [l for l in out.stdout.splitlines() if l.startswith("INFO: MOM per region: est ")]
    names = sorted(p.name for p in res.iterdir())
    assert names == ["map_consistency.txt", "map_entropy.pcd", "map_mom.txt", "map_mom_regions.txt", "map_results.txt"]
    comment, rows = _read(res / "map_mom_regions.txt")
    assert "est as loaded" in comment and f"s = {S}" in comment and "min_family 100" in comment
    n_est = int([l for l in (res / "map_results.txt").read_text().splitlines()
                 if l.startswith("Estimated-Ground Truth point count: ")][0].split(":")[1].split("/")[0])
    ref = _api_rows(est, None, {0}, n_est)
    _compare(rows, ref["est"], "est")
    # the rows of map_consistency.txt at the same size, in the same order
    cons = _consistency_rows(res / "map_consistency.txt", "est")
    assert [c[1:8] for c in cons] == [[r[k] for k in COLS[1:8]] for r in
                                      [{c: x for c, x in zip(COLS, l.split())} for l in
                                       (res / "map_mom_regions.txt").read_text().splitlines()[2:]]]


def _run_gt(exe, d, name, est, extra):
    """a run with a ground truth, MME of both clouds (so MOM and local consistency run on the gt cloud too)"""
    est_dir = d / name / "est"
    est_dir.mkdir(parents=True)
    _write_pcd(str(est_dir / "map.pcd"), est)
    cfg = d / name / "config.yaml"
    cfg.write_text(_config(d, est_dir, extra, mme=True).replace("evaluate_gt_mme: false", "evaluate_gt_mme: true"))
    out = subprocess.run([exe, str(cfg)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    return out, est_dir / "map_results"


@pytest.mark.gpu
def test_with_gt_equals_the_python_api_and_changes_nothing_else(exe, maps):
    d, est, gt = maps
    base = f"evaluate_mom: true\nevaluate_consistency: true\nconsistency_region_size: {S}\n"
    out, on = _run_gt(exe, d, "r_on", est, base + f"mom_region_size: {S}\n")
    _, off = _run_gt(exe, d, "r_off", est, base)
    infos = [l for l in out.stdout.splitlines() if l.startswith("INFO: MOM per region: ")]
    assert len(infos) == 2 and "largest family median" in infos[0]
    comment, rows = _read(on / "map_mom_regions.txt")
    assert "ground truth's frame" in comment
    assert sorted({r["cloud"] for r in rows}) == ["est", "gt"]
    names = sorted(p.name for p in on.iterdir() if p.name != "map_mom_regions.txt")
    assert names == sorted(p.name for p in off.iterdir())
    for n in names:
        if n == "map_results.txt":
            assert _stable((on / n).read_text().splitlines()) == _stable((off / n).read_text().splitlines())
        elif n == "voxel_errors.txt":
            assert sorted((on / n).read_text().splitlines()) == sorted((off / n).read_text().splitlines())
        else:
            assert (on / n).read_bytes() == (off / n).read_bytes(), n
    for name in ("est", "gt"):
        cons = _consistency_rows(on / "map_consistency.txt", name)
        mine = [r for r in rows if r["cloud"] == name]
        assert len(cons) == len(mine)
        for c, r in zip(cons, mine):
            assert [float(x) for x in c[1:7]] == [r[k] for k in COLS[1:7]] and int(c[7]) == r["n_points"]
    # against the Python API on the same clouds (evaluate_using_initial with no initial matrix: est as loaded)
    count = [l for l in (on / "map_results.txt").read_text().splitlines() if l.startswith("Estimated-Ground Truth point count: ")]
    n_est, n_gt = (int(x) for x in count[0].split(":")[1].split("/"))
    ref = _api_rows(est, gt, {0, 1}, n_est, n_gt)
    _compare(rows, ref["est"], "est")
    _compare(rows, ref["gt"], "gt")


@pytest.mark.gpu
def test_two_gpus_match_one(exe, maps):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (NCCL cannot put two ranks of one communicator on one device)")
    d, est, _ = maps
    extra = NO_GT + f"mom_region_size: {S}\n"
    _, one = _run(exe, d, "rg1", est, extra, with_gt=False, args=("--gpus", "1"))
    _, two = _run(exe, d, "rg2", est, extra, with_gt=False, args=("--gpus", "2"))
    c1, a = _read(one / "map_mom_regions.txt")
    c2, b = _read(two / "map_mom_regions.txt")
    assert c1 == c2 and len(a) == len(b)
    for x, y in zip(a, b):
        for c, v in x.items():
            if c in ("cloud", "status") or c.startswith("n") or c.startswith("min") or c.startswith("max"):
                assert y[c] == v, c
            elif not math.isnan(v):
                assert y[c] == pytest.approx(v, rel=1e-9, abs=1e-15), c

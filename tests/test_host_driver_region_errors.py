"""The re-hosted `map_eval` with `region_size`: region_errors.txt next to map_results.txt on path A and on path B (generalized
ICP), its rows sorted and its point counts summing to the evaluated clouds, its path A values equal to the Python API's on
the same clouds; without the key no file and the same map_results.txt; the key in --dump-config; negative and non-finite
sizes refused when the configuration is loaded; two GPUs against one."""
import subprocess

import numpy as np
import pytest

from test_host_driver_accuracy_curve import CONFIG, _stable, _write_pcd, exe  # noqa: F401  (module fixture)

LEVELS = [0.2, 0.1, 0.08, 0.05, 0.01]
SIZE = 0.5
COLS = ["min_x", "min_y", "min_z", "max_x", "max_y", "max_z", "n_est", "n_gt"]
for _d in ("e2g", "g2e"):
    COLS += [f"{_d}_n_corr"] + [f"{_d}_{f}_{k}" for f in ("n_inlier", "mean", "rmse", "fitness") for k in range(1, 6)]
    COLS += [f"{_d}_max_d", f"{_d}_mean_nn"]
COLS += [f"{f}_{k}" for f in ("cd", "f1", "iou") for k in range(1, 6)]


@pytest.fixture(scope="module")
def maps(tmp_path_factory):
    from cloud_map_evaluation_b200 import synth
    d = tmp_path_factory.mktemp("region")
    est, gt, _ = synth.make_pair("C1", scale=0.3)
    _write_pcd(str(d / "gt.pcd"), gt)
    return d, est, gt


def _config(d, est_dir, initial, extra):
    text = CONFIG.format(levels=", ".join(repr(x) for x in LEVELS), est=str(est_dir), gt=str(d / "gt.pcd"), initial=initial,
                         extra=extra)
    return text.replace("downsample_size: 0.01", "downsample_size: 0.0")     # evaluate the clouds as loaded


def _run(exe, d, name, est, initial, extra="", args=()):
    est_dir = d / name / "est"
    est_dir.mkdir(parents=True)
    _write_pcd(str(est_dir / "map.pcd"), est)
    cfg = d / name / "config.yaml"
    cfg.write_text(_config(d, est_dir, initial, extra))
    out = subprocess.run([exe, str(cfg), *args], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    res = est_dir / "map_results"
    return out, (res / "map_results.txt").read_text().splitlines(), res / "region_errors.txt"


def _read(path):
    """{column: array} of region_errors.txt"""
    lines = path.read_text().splitlines()
    assert lines[0].split() == COLS
    rows = np.array([[float(x) for x in line.split()] for line in lines[1:]])
    assert rows.shape[1] == len(COLS)
    return {c: rows[:, i] for i, c in enumerate(COLS)}


def test_dump_config_lists_the_key(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "true", "region_size: 0.25\n"))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert "region_size=0.25" in out.stdout.splitlines()
    cfg.write_text(_config(tmp_path, tmp_path, "true", ""))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert "region_size=0" in out.stdout.splitlines()


@pytest.mark.parametrize("bad", ["-0.5", "nan", "inf", "-inf"])
def test_bad_sizes_are_refused_at_load(exe, tmp_path, bad):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "true", f"region_size: {bad}\n"))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)     # refused before anything runs
    assert out.returncode != 0 and "region_size" in out.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("initial", ["true", "false"])     # path A, path B (generalized ICP)
def test_region_file(exe, maps, initial):
    from cloud_map_evaluation_b200 import _abi as A
    from cloud_map_evaluation_b200 import api
    d, est, gt = maps
    out, lines, path = _run(exe, d, f"on_{initial}", est, initial, f"region_size: {SIZE}\n")
    assert sum(l.startswith("INFO: errors of ") and "region_errors.txt" in l for l in out.stdout.splitlines()) == 1
    t = _read(path)
    lo = np.stack([t["min_x"], t["min_y"], t["min_z"]], 1)
    idx = np.round(lo / SIZE).astype(np.int64)
    assert np.all(np.diff(idx[:, 0]) >= 0)
    assert sorted(map(tuple, idx)) == list(map(tuple, idx)) and len(set(map(tuple, idx))) == len(idx)
    assert t["n_est"].sum() == len(est) and t["n_gt"].sum() == len(gt)
    if initial == "true":      # path A: the same clouds through the Python API
        p = A.make_nn_params(LEVELS, 1.0)
        with api.MapEvalB200() as ctx:
            ctx.set_cloud(A.ME_CLOUD_EST, est.astype(np.float32).astype(np.float64))
            ctx.set_cloud(A.ME_CLOUD_GT, gt.astype(np.float32).astype(np.float64))
            ctx.transform(A.ME_CLOUD_EST, np.eye(4))
            ctx.calculateMetricsWithInitialMatrix(p)
            ref = ctx.region_errors(SIZE)
        np.testing.assert_array_equal(idx, ref["index"])
        for a, c in enumerate("xyz"):
            np.testing.assert_allclose(t[f"min_{c}"], ref["min"][:, a], rtol=0, atol=1e-15)
            np.testing.assert_allclose(t[f"max_{c}"], ref["max"][:, a], rtol=0, atol=1e-15)
        np.testing.assert_array_equal(t["n_est"], ref["n_est"])
        np.testing.assert_array_equal(t["n_gt"], ref["n_gt"])
        for dname, key in (("e2g", "est_to_gt"), ("g2e", "gt_to_est")):
            r = ref[key]
            np.testing.assert_array_equal(t[f"{dname}_n_corr"], r["n_corr"])
            for k in range(5):
                np.testing.assert_array_equal(t[f"{dname}_n_inlier_{k + 1}"], r["n_inlier"][:, k])
                for f in ("mean", "rmse", "fitness"):
                    np.testing.assert_allclose(t[f"{dname}_{f}_{k + 1}"], r[f][:, k], rtol=0, atol=1e-15)
            for f in ("max_d", "mean_nn"):
                np.testing.assert_allclose(t[f"{dname}_{f}"], r[f], rtol=0, atol=1e-15)
        for f in ("cd", "f1", "iou"):
            for k in range(5):
                np.testing.assert_allclose(t[f"{f}_{k + 1}"], ref[f][:, k], rtol=0, atol=1e-15)
    # without the key: no file, and the same results
    _, off, r_off = _run(exe, d, f"off_{initial}", est, initial)
    assert not r_off.exists()
    assert _stable(off) == _stable(lines)


@pytest.mark.gpu
def test_two_gpus_match_one(exe, maps):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (NCCL cannot put two ranks of one communicator on one device)")
    d, est, _ = maps
    key = f"region_size: {SIZE}\n"
    for initial in ("true", "false"):
        _, _, one = _run(exe, d, f"g1_{initial}", est, initial, key, ("--gpus", "1"))
        _, _, two = _run(exe, d, f"g2_{initial}", est, initial, key, ("--gpus", "2"))
        t1, t2 = _read(one), _read(two)
        for c in COLS:
            if initial == "true" and (c.startswith(("n_", "min_", "max_")) or "n_corr" in c or "n_inlier" in c or "max_d" in c):
                np.testing.assert_array_equal(t2[c], t1[c], c)       # counts, bounds and maxima do not depend on the world
            else:       # sums reduce in another order; on path B the ICP sums, and so T, may differ in the last bits too
                np.testing.assert_allclose(t2[c], t1[c], rtol=1e-9, atol=1e-12, err_msg=c)

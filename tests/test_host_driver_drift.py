"""The re-hosted `map_eval` with `drift_region_size`: region_drift.txt next to map_results.txt on path A and on path B
(generalized ICP), equal to the Python API's rows on the same clouds; one INFO line; without the key no file, the same
map_results.txt (but for the header timestamp and the timing lines) and the same voxel_errors.txt rows; the key in
--dump-config; negative and non-finite sizes refused when the configuration is loaded; two GPUs against one."""
import subprocess

import numpy as np
import pytest

from test_host_driver_accuracy_curve import CONFIG, _stable, _write_pcd, exe  # noqa: F401  (module fixture)

LEVELS = [0.2, 0.1, 0.08, 0.05, 0.01]
SIZE = 0.5
R = 1.0                   # icp_max_distance of CONFIG
INTS = ["n_est", "n_corr_before", "n_corr", "iterations", "status"]
COLS = (["min_x", "min_y", "min_z", "max_x", "max_y", "max_z", "n_est", "n_corr_before", "fitness_before", "rmse_before", "n_corr",
         "fitness", "rmse", "shift_x", "shift_y", "shift_z", "shift_norm", "angle_rad", "iterations", "status"]
        + [f"T{i}{j}" for i in range(3) for j in range(4)])


@pytest.fixture(scope="module")
def maps(tmp_path_factory):
    from cloud_map_evaluation_b200 import synth
    d = tmp_path_factory.mktemp("drift")
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
    return out, (res / "map_results.txt").read_text().splitlines(), res


def _read(path):
    """{column: array} of region_drift.txt; counts and codes written as integers"""
    lines = path.read_text().splitlines()
    assert lines[0].split() == COLS
    rows = [line.split() for line in lines[1:]]
    assert all(len(r) == len(COLS) for r in rows)
    out = {}
    for i, c in enumerate(COLS):
        if c in INTS:
            assert all("." not in r[i] for r in rows), c
            out[c] = np.array([int(r[i]) for r in rows], np.int64)
        else:
            assert all(len(r[i].split(".")[1]) == 15 for r in rows), c
            out[c] = np.array([float(r[i]) for r in rows])
    return out


def test_dump_config_lists_the_key(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "true", "drift_region_size: 0.25\n"))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert "drift_region_size=0.25" in out.stdout.splitlines()
    cfg.write_text(_config(tmp_path, tmp_path, "true", ""))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert "drift_region_size=0" in out.stdout.splitlines()


@pytest.mark.parametrize("bad", ["-0.5", "nan", "inf", "-inf"])
def test_bad_sizes_are_refused_at_load(exe, tmp_path, bad):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "true", f"drift_region_size: {bad}\n"))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)     # refused before anything runs
    assert out.returncode != 0 and "drift_region_size" in out.stderr


def _python_rows(est, gt, initial):
    """the same clouds through the Python API: path A evaluates the estimate as loaded (initial_matrix = I), path B after
    generalized ICP from I, as map_eval runs them"""
    from cloud_map_evaluation_b200 import _abi as A
    from cloud_map_evaluation_b200 import api
    with api.MapEvalB200() as ctx:
        ctx.set_cloud(A.ME_CLOUD_EST, est.astype(np.float32).astype(np.float64))
        ctx.set_cloud(A.ME_CLOUD_GT, gt.astype(np.float32).astype(np.float64))
        if initial == "true":
            ctx.transform(A.ME_CLOUD_EST, np.eye(4))
        else:
            ctx.performICPRegistration(R, method=A.ME_ICP_GENERALIZED)
        return ctx.region_drift(SIZE, R)


@pytest.mark.gpu
@pytest.mark.parametrize("initial", ["true", "false"])     # path A, path B (generalized ICP)
def test_drift_file(exe, maps, initial):
    d, est, gt = maps
    out, lines, res = _run(exe, d, f"on_{initial}", est, initial, f"drift_region_size: {SIZE}\n")
    info = [l for l in out.stdout.splitlines() if l.startswith("INFO: drift of ")]
    assert len(info) == 1 and "region_drift.txt" in info[0] and "converged" in info[0] and "largest shift" in info[0]
    t = _read(res / "region_drift.txt")
    ref = _python_rows(est, gt, initial)
    assert len(t["n_est"]) == len(ref["n_est"]) and t["n_est"].sum() == len(est)
    assert f"{len(ref['n_est'])} regions" in info[0]
    for k in ("min", "max"):
        for a, c in enumerate("xyz"):
            np.testing.assert_allclose(t[f"{k}_{c}"], ref[k][:, a], rtol=0, atol=1e-15, err_msg=k)
    np.testing.assert_array_equal(t["n_est"], ref["n_est"])
    if initial == "true":      # path A: the estimate as loaded, so every column is the Python API's
        for c in INTS:
            np.testing.assert_array_equal(t[c], ref[c], err_msg=c)
        pairs = [(f"shift_{c}", ref["shift"][:, a]) for a, c in enumerate("xyz")]
        pairs += [(k, ref[k]) for k in ("fitness_before", "rmse_before", "fitness", "rmse", "shift_norm")]
        pairs += [("angle_rad", ref["angle"])] + [(f"T{i}{j}", ref["T"][:, i, j]) for i in range(3) for j in range(4)]
        for c, v in pairs:
            np.testing.assert_allclose(t[c], v, rtol=0, atol=1e-15, err_msg=c)
        assert f"({int((ref['status'] == 0).sum())} converged)" in info[0]
    else:
        # path B: registration reduces its sums with floating-point atomics, so the registered estimate of two processes may
        # differ in the last bits, and a region whose rotation the points hardly constrain can end elsewhere.  The first sweep
        # (T = I) depends on the registered estimate alone.
        np.testing.assert_array_equal(t["n_corr_before"], ref["n_corr_before"])
        for c in ("fitness_before", "rmse_before"):
            np.testing.assert_allclose(t[c], ref[c], rtol=0, atol=1e-9, err_msg=c)
    # without the key: no file, the same results and the same voxel table (its rows come in the order the voxel pairs are
    # found, which varies from run to run, so they are compared as a set)
    _, off, r_off = _run(exe, d, f"off_{initial}", est, initial)
    assert not (r_off / "region_drift.txt").exists()
    assert _stable(off) == _stable(lines)
    v_off, v_on = (r_off / "voxel_errors.txt").read_text().splitlines(), (res / "voxel_errors.txt").read_text().splitlines()
    assert len(v_on) > 0 and sorted(v_off) == sorted(v_on)


@pytest.mark.gpu
def test_two_gpus_match_one(exe, maps):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (NCCL cannot put two ranks of one communicator on one device)")
    d, est, _ = maps
    key = f"drift_region_size: {SIZE}\n"
    for initial in ("true", "false"):
        _, _, one = _run(exe, d, f"g1_{initial}", est, initial, key, ("--gpus", "1"))
        _, _, two = _run(exe, d, f"g2_{initial}", est, initial, key, ("--gpus", "2"))
        t1, t2 = _read(one / "region_drift.txt"), _read(two / "region_drift.txt")
        for c in COLS:
            if c.startswith(("min_", "max_")) or (initial == "true" and c in INTS):
                np.testing.assert_array_equal(t2[c], t1[c], c)       # on path A counts and codes do not depend on the world
            elif initial == "true":       # the ranks' sums reduce in another order
                np.testing.assert_allclose(t2[c], t1[c], rtol=1e-9, atol=1e-9, err_msg=c)
            elif c.startswith("T"):       # on path B the registered estimate itself may differ in the last bits
                np.testing.assert_allclose(t2[c], t1[c], rtol=0, atol=1e-6, err_msg=c)

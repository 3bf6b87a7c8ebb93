"""The re-hosted `map_eval` with `distance_quantiles`: distance_quantiles.txt next to map_results.txt on path A and on path B
(generalized ICP), whose path A values equal the Python API's on the same clouds; without the key, or with it empty, no file
and the same map_results.txt; the key in --dump-config; bad values refused; two GPUs against one."""
import os
import subprocess

import numpy as np
import pytest

from test_host_driver_accuracy_curve import CONFIG, _stable, _write_pcd, exe  # noqa: F401  (module fixture)

PROBS = [0.5, 0.9, 0.95, 0.99]
LEVELS = [0.2, 0.1, 0.08, 0.05, 0.01]


@pytest.fixture(scope="module")
def maps(tmp_path_factory):
    from cloud_map_evaluation_b200 import synth
    d = tmp_path_factory.mktemp("quant")
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
    return out, (res / "map_results.txt").read_text().splitlines(), res / "distance_quantiles.txt"


def _read(path):
    """{(population, direction): (n, [(p, value, lo, hi)])}, {'hausdorff_est_to_gt', 'hausdorff_gt_to_est', 'hausdorff'}"""
    rows, tail = {}, {}
    lines = path.read_text().splitlines()
    assert lines[0].startswith("#") and lines[1].split() == ["population", "direction", "n", "p", "value", "lo", "hi"]
    for line in lines[2:]:
        f = line.split()
        if len(f) == 2:
            tail[f[0]] = float(f[1])
            continue
        n, vals = rows.setdefault((f[0], f[1]), (int(f[2]), []))
        vals.append(tuple(float(x) for x in f[3:]))
    return rows, tail


def test_dump_config_lists_the_key(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "true", "distance_quantiles: [0.5, 0.9, 0.95, 0.99]\n"))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert "distance_quantiles=0.5,0.90000000000000002,0.94999999999999996,0.98999999999999999" in out.stdout.splitlines()
    cfg.write_text(_config(tmp_path, tmp_path, "true", ""))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert "distance_quantiles=" in out.stdout.splitlines()


@pytest.mark.parametrize("bad", ["[0.5, 1.5]", "[-0.1]", "[" + ", ".join(["0.5"] * 65) + "]"])
def test_bad_probabilities_are_refused(exe, tmp_path, bad):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "true", f"distance_quantiles: {bad}\n"))
    out = subprocess.run([exe, str(cfg)], capture_output=True, text=True)
    assert out.returncode != 0 and "distance_quantiles" in out.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("initial", ["true", "false"])     # path A, path B (generalized ICP)
def test_quantile_file(exe, maps, initial):
    from cloud_map_evaluation_b200 import _abi as A
    from cloud_map_evaluation_b200 import api
    d, est, gt = maps
    keys = "distance_quantiles: [" + ", ".join(repr(x) for x in PROBS) + "]\n"
    out, lines, path = _run(exe, d, f"on_{initial}", est, initial, keys)
    assert sum(l.startswith("INFO: Hausdorff distance:") for l in out.stdout.splitlines()) == 1
    rows, tail = _read(path)
    assert set(rows) == {(p, q) for p in ("kept", "nn") for q in ("est_to_gt", "gt_to_est")}
    assert rows[("nn", "est_to_gt")][0] == len(est) and rows[("nn", "gt_to_est")][0] == len(gt)
    assert tail["hausdorff"] == max(tail["hausdorff_est_to_gt"], tail["hausdorff_gt_to_est"])
    for key, (n, vals) in rows.items():
        assert [v[0] for v in vals] == PROBS and n > 0, key
        assert all(lo <= v <= hi for _, v, lo, hi in vals) and np.all(np.diff([v[1] for v in vals]) >= 0), key
    if initial == "true":      # path A: the same clouds through the Python API
        p = A.make_nn_params(LEVELS, 1.0)
        with api.MapEvalB200() as ctx:
            ctx.set_cloud(A.ME_CLOUD_EST, est.astype(np.float32).astype(np.float64))
            ctx.set_cloud(A.ME_CLOUD_GT, gt.astype(np.float32).astype(np.float64))
            ctx.transform(A.ME_CLOUD_EST, np.eye(4))
            ctx.calculateMetricsWithInitialMatrix(p)
            ref = {pop: ctx.distance_quantiles(PROBS, pop) for pop in (A.ME_DIST_KEPT, A.ME_DIST_NN)}
        for (pop, q), (n, vals) in rows.items():
            r = ref[A.ME_DIST_KEPT if pop == "kept" else A.ME_DIST_NN][q]
            assert n == r["n"]
            np.testing.assert_allclose([v[1:] for v in vals], np.stack([r["value"], r["lo"], r["hi"]], 1), rtol=0, atol=1e-15)
        np.testing.assert_allclose(tail["hausdorff"], ref[A.ME_DIST_NN]["hausdorff"], rtol=0, atol=1e-15)
    # without the key, and with it empty: no file, and the same results
    _, off, q_off = _run(exe, d, f"off_{initial}", est, initial)
    _, empty, q_empty = _run(exe, d, f"empty_{initial}", est, initial, "distance_quantiles: []\n")
    assert not q_off.exists() and not q_empty.exists()
    assert _stable(off) == _stable(empty) == _stable(lines)


@pytest.mark.gpu
def test_two_gpus_match_one(exe, maps):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (NCCL cannot put two ranks of one communicator on one device)")
    d, est, _ = maps
    keys = "distance_quantiles: [" + ", ".join(repr(x) for x in PROBS) + "]\n"
    for initial in ("true", "false"):
        _, _, one = _run(exe, d, f"g1_{initial}", est, initial, keys, ("--gpus", "1"))
        _, _, two = _run(exe, d, f"g2_{initial}", est, initial, keys, ("--gpus", "2"))
        r1, t1 = _read(one)
        r2, t2 = _read(two)
        if initial == "true":
            assert r1 == r2 and t1 == t2        # exact selection over the same records
        else:                                   # ICP sums reduce in another order: T, and so the distances, may differ in the last bits
            for key in r1:
                assert r1[key][0] == r2[key][0]
                np.testing.assert_allclose(r2[key][1], r1[key][1], rtol=1e-9, atol=1e-12)

"""The re-hosted `map_eval` with `evaluate_mom: true` and `evaluate_without_gt: true`: the keys in --dump-config and bad
values refused when the configuration is loaded; a run with only map.pcd writes map_results.txt, map_entropy.pcd,
map_consistency.txt and map_mom.txt with the Python API's values on the same down-sampled cloud; every key that needs a
ground truth refused in that mode; a run with a ground truth and evaluate_mom writes map_mom.txt and leaves every other
output as the run without the key; two GPUs against one."""
import math
import subprocess

import numpy as np
import pytest

from test_host_driver_accuracy_curve import CONFIG, _stable, _write_pcd, exe  # noqa: F401  (module fixture)

LEVELS = [0.2, 0.1, 0.08, 0.05, 0.01]
NO_GT = "evaluate_without_gt: true\nevaluate_mme: true\nevaluate_consistency: true\nevaluate_mom: true\n"
COLS = (["cloud", "n_points", "n_query", "n_pv", "n_planar"] + [f"a{k}_{c}" for k in (1, 2, 3) for c in "xyz"] +
        [f"{f}_{j}" for j in (1, 2, 3) for f in ("n", "mean", "median")] + ["mom", "status"])
R0 = 0.1


def _config(d, est_dir, extra, with_gt=True, mme=False):
    text = CONFIG.format(levels=", ".join(repr(x) for x in LEVELS), est=str(est_dir), gt=str(d / "gt.pcd"), initial="true",
                         extra=extra)
    if not with_gt:
        text = "\n".join(l for l in text.splitlines() if not l.startswith("gt_map_path")) + "\n"
    if mme:
        text = text.replace("evaluate_mme: false", "evaluate_mme: true")
    return text


@pytest.fixture(scope="module")
def maps(tmp_path_factory):
    from cloud_map_evaluation_b200 import synth
    d = tmp_path_factory.mktemp("mom")
    est, gt, _ = synth.make_pair("C1", scale=0.3)
    _write_pcd(str(d / "gt.pcd"), gt)
    return d, est, gt


def _run(exe, d, name, est, extra, with_gt=True, mme=False, args=(), ok=True):
    est_dir = d / name / "est"
    est_dir.mkdir(parents=True)
    _write_pcd(str(est_dir / "map.pcd"), est)
    cfg = d / name / "config.yaml"
    cfg.write_text(_config(d, est_dir, extra, with_gt, mme))
    out = subprocess.run([exe, str(cfg), *args], capture_output=True, text=True)
    if ok:
        assert out.returncode == 0, out.stdout + out.stderr
    return out, est_dir / "map_results"


def _read(path):
    lines = path.read_text().splitlines()
    assert lines[0].startswith("# ") and lines[1].split() == COLS
    out = {}
    for line in lines[2:]:
        v = line.split()
        assert len(v) == len(COLS)
        out[v[0]] = {c: (x if c == "status" else int(x) if c.startswith("n") else float(x)) for c, x in zip(COLS[1:], v[1:])}
    return lines[0], out


def test_dump_config_lists_the_keys(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "evaluate_mom: true\nmom_angle_deg: 12.5\nmom_planarity: 0.25\nmom_min_family: 7\n"
                                               "evaluate_without_gt: true\n", with_gt=False))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.splitlines()
    for k in ("evaluate_mom=1", "mom_angle_deg=12.5", "mom_planarity=0.25", "mom_min_family=7", "evaluate_without_gt=1", "gt_map_path="):
        assert k in lines, k
    cfg.write_text(_config(tmp_path, tmp_path, ""))
    lines = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True).stdout.splitlines()
    for k in ("evaluate_mom=0", "mom_angle_deg=10", "mom_planarity=0.5", "mom_min_family=100", "evaluate_without_gt=0"):
        assert k in lines, k


@pytest.mark.parametrize("key,bad", [("mom_angle_deg", "0"), ("mom_angle_deg", "30.5"), ("mom_angle_deg", "nan"),
                                     ("mom_planarity", "0"), ("mom_planarity", "1.5"), ("mom_min_family", "0"),
                                     ("mom_min_family", "2.5")])
def test_bad_values_are_refused_at_load(exe, tmp_path, key, bad):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, f"evaluate_mom: true\n{key}: {bad}\n"))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)     # refused before anything runs
    assert out.returncode != 0 and key in out.stderr


def test_gt_map_path_is_still_required_with_a_ground_truth(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "evaluate_mom: true\n", with_gt=False))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert out.returncode != 0 and "gt_map_path" in out.stderr


@pytest.mark.parametrize("extra,key", [("evaluate_noised_gt: true\n", "evaluate_noised_gt"),
                                       ("global_registration: true\n", "global_registration"),
                                       ("accuracy_curve_steps: 4\n", "accuracy_curve_steps"),
                                       ("distance_quantiles: [0.5]\n", "distance_quantiles"),
                                       ("region_size: 1.0\n", "region_size"),
                                       ("drift_region_size: 1.0\n", "drift_region_size"),
                                       ("surface_metrics: true\n", "surface_metrics")])
def test_ground_truth_keys_are_refused_without_gt(exe, tmp_path, extra, key):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, NO_GT + extra, with_gt=False))
    out = subprocess.run([exe, str(cfg)], capture_output=True, text=True)
    assert out.returncode != 0 and key in out.stderr and "needs a ground truth" in out.stderr
    assert not (tmp_path / "map_results").exists()


def test_nothing_to_do_is_refused(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "evaluate_without_gt: true\n", with_gt=False))
    out = subprocess.run([exe, str(cfg)], capture_output=True, text=True)
    assert out.returncode != 0 and "nothing to do" in out.stderr


@pytest.mark.gpu
def test_without_gt_equals_the_python_api(exe, maps):
    from cloud_map_evaluation_b200 import _abi as A
    from cloud_map_evaluation_b200 import api
    d, est, _ = maps
    out, res = _run(exe, d, "nogt", est, NO_GT.replace("evaluate_mme: true\n", ""), with_gt=False, mme=True)
    assert any(l.startswith("INFO: evaluate_without_gt") for l in out.stdout.splitlines())
    assert [l for l in out.stdout.splitlines() if l.startswith("INFO: mutually orthogonal metric:")]
    names = sorted(p.name for p in res.iterdir())
    assert names == ["map_consistency.txt", "map_entropy.pcd", "map_mom.txt", "map_results.txt"]
    lines = (res / "map_results.txt").read_text().splitlines()
    count = [l for l in lines if l.startswith("Estimated-Ground Truth point count: ")]
    mme_line = [l for l in lines if l.startswith("MME: ")]
    assert len(count) == 1 and len(mme_line) == 1 and count[0].endswith(" / 0")
    n_est = int(count[0].split(":")[1].split("/")[0])
    with api.MapEvalB200() as ctx:        # the same cloud: the file's fp32 coordinates, down-sampled as the driver does
        ctx.set_cloud(A.ME_CLOUD_EST, est.astype(np.float32).astype(np.float64))
        assert ctx.voxel_downsample(A.ME_CLOUD_EST, 0.01) == n_est
        mme = ctx.computeMME(A.ME_CLOUD_EST, R0, 10)
        cons = ctx.local_consistency(A.ME_CLOUD_EST, R0, 10)
        mom = ctx.mom(A.ME_CLOUD_EST, R0, 10)
    assert abs(float(mme_line[0].split()[1]) - mme.mme) <= 5e-6 + 1e-12
    cl = (res / "map_consistency.txt").read_text().splitlines()
    assert "est as loaded" in cl[0]
    row = cl[2].split()
    assert row[0] == "est" and int(row[1]) == n_est and int(row[4]) == cons["whole"]["n_pv"]
    assert float(row[6]) == pytest.approx(cons["whole"]["mpv"], rel=1e-9)
    comment, got = _read(res / "map_mom.txt")
    assert "est as loaded" in comment and "angle_deg 10" in comment and sorted(got) == ["est"]
    g = got["est"]
    assert g["status"] == mom["status"] and g["n_points"] == n_est
    # a layout ranks the points of a cell with atomics, so per-point values agree to rounding; the counts are exact away from
    # the thresholds, which these maps keep clear of
    for j in range(3):
        assert g[f"n_{j + 1}"] == mom["n"][j]
        if mom["n"][j]:
            assert g[f"median_{j + 1}"] == pytest.approx(mom["median"][j], rel=1e-9, abs=1e-15)
    assert g["n_planar"] == mom["n_planar"] and g["n_pv"] == mom["n_pv"]
    np.testing.assert_allclose([g[f"a{k}_{c}"] for k in (1, 2, 3) for c in "xyz"], mom["axis"].reshape(-1), rtol=0, atol=1e-15)
    if mom["status"] == "OK":
        assert g["mom"] == pytest.approx(mom["mom"], rel=1e-9)
    else:
        assert math.isnan(g["mom"])


@pytest.mark.gpu
def test_with_gt_adds_only_map_mom(exe, maps):
    d, est, gt = maps
    _, on = _run(exe, d, "on", est, "evaluate_mom: true\n", mme=True)
    _, off = _run(exe, d, "off", est, "", mme=True)
    comment, got = _read(on / "map_mom.txt")
    assert "ground truth's frame" in comment and sorted(got) == ["est"]
    names = sorted(p.name for p in on.iterdir() if p.name != "map_mom.txt")
    assert names == sorted(p.name for p in off.iterdir())
    for n in names:
        if n == "map_results.txt":
            assert _stable((on / n).read_text().splitlines()) == _stable((off / n).read_text().splitlines())
        elif n == "voxel_errors.txt":
            assert sorted((on / n).read_text().splitlines()) == sorted((off / n).read_text().splitlines())
        else:
            assert (on / n).read_bytes() == (off / n).read_bytes(), n


@pytest.mark.gpu
def test_two_gpus_match_one(exe, maps):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (NCCL cannot put two ranks of one communicator on one device)")
    d, est, _ = maps
    _, one = _run(exe, d, "g1", est, NO_GT, with_gt=False, args=("--gpus", "1"))
    _, two = _run(exe, d, "g2", est, NO_GT, with_gt=False, args=("--gpus", "2"))
    c1, a = _read(one / "map_mom.txt")
    c2, b = _read(two / "map_mom.txt")
    assert c1 == c2
    for c, v in a["est"].items():
        if c == "status" or c.startswith("n"):
            assert b["est"][c] == v, c
        elif not math.isnan(v):
            assert b["est"][c] == pytest.approx(v, rel=1e-9, abs=1e-15), c

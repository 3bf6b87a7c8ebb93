"""`map_eval` with `evaluate_noised_gt: true` (config.yaml:55-59): the estimate file is not read; the estimate is a
degraded copy of the ground truth (deformation -> density -> noise -> outliers, seeded), evaluated by the unchanged
process().  Under save_immediate_result the degraded map is written as noise_gt_map.pcd (map_eval.cpp:502-507)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from test_host_driver import CONFIG, _dump, _write_pcd, exe  # noqa: F401  (module fixture)

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import perturb_ref as ref  # noqa: E402

SIM = """evaluate_noised_gt: true
noise_std_dev: {sigma}
simulation_seed: 777
"""


def _read_xyz_pcd(path):
    raw = open(path, "rb").read()
    head, data = raw.split(b"DATA binary\n", 1)
    lines = head.decode().splitlines()
    assert "FIELDS x y z" in lines and "TYPE F F F" in lines
    n = int([l for l in lines if l.startswith("POINTS")][0].split()[1])
    return np.frombuffer(data, dtype="<f4", count=3 * n).reshape(n, 3)


def _run(exe, d, gt, sim, gpus=1, initial="true"):  # noqa: F811
    est_dir = d / "est"
    est_dir.mkdir(parents=True, exist_ok=True)
    assert not (est_dir / "map.pcd").exists()
    if not (d / "gt.pcd").exists():
        _write_pcd(str(d / "gt.pcd"), gt, "binary")
    text = CONFIG.format(est=str(est_dir), gt=str(d / "gt.pcd"), gt_mme="true", initial=initial)
    text = text.replace("[1.0, 0.0, 0.0, 0.5]", "[1.0, 0.0, 0.0, 0.0]").replace("[0.0, 0.0, 1.0, -2]", "[0.0, 0.0, 1.0, 0.0]")
    (d / "config.yaml").write_text(text + sim)
    res_file = est_dir / "map_results" / "map_results.txt"
    if res_file.exists():
        res_file.unlink()
    out = subprocess.run([exe, str(d / "config.yaml"), "--gpus", str(gpus)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    res = res_file.read_text().splitlines()
    line = {l.split(":")[0]: l.split(":", 1)[1].split() for l in res if ":" in l and not l.startswith(("Ground", "Evaluation"))}
    return out, line, est_dir / "map_results"


@pytest.fixture(scope="module")
def gt():
    from cloud_map_evaluation_b200 import synth
    return synth.uniform_box(100_000, 2.0, synth.GT_SEED, origin=(0.123, 0.456, 0.0))


@pytest.mark.gpu
def test_noised_gt_writes_the_degraded_map(exe, tmp_path, gt):  # noqa: F811
    sim = SIM.format(sigma=0.01) + "outlier_ratio: 0.05\noutlier_range: 0.5\n"
    out, line, res = _run(exe, tmp_path, gt, sim)
    assert "INFO: evaluate_noised_gt: the estimated map is not read" in out.stdout
    assert "Gaussian noise (std_dev 0.01), then sparse outliers (ratio 0.05, range 0.5)" in out.stdout
    assert "initial_matrix is not the identity" not in out.stdout
    n_est = int(line["Estimated-Ground Truth point count"][0])
    assert n_est == len(gt) + len(gt) // 20 and int(line["Estimated-Ground Truth point count"][2]) == len(gt)
    pcd = _read_xyz_pcd(str(res / "noise_gt_map.pcd"))
    assert len(pcd) == n_est
    exp = ref.sparse_outliers(ref.gaussian_noise(gt, 0.01, 777), 0.05, 0.5, 777).astype(np.float32)
    np.testing.assert_allclose(pcd, exp, rtol=0, atol=np.spacing(np.float32(4.0)))
    comp = [float(x) for x in line["Comp"]]
    assert all(0 < c < 1 for c in comp)


@pytest.mark.gpu
def test_noised_gt_without_degradation_is_exact(exe, tmp_path, gt):  # noqa: F811
    """sigma = 0 and nothing else: the estimate is the ground truth, every point at distance 0 (path A)"""
    out, line, res = _run(exe, tmp_path, gt, SIM.format(sigma=0))
    assert "it is the ground truth unchanged" in out.stdout
    assert [float(x) for x in line["Comp"]] == [1.0] * 5
    assert [float(x) for x in line["RMSE/AC"]] == [0.0] * 5
    assert line["Estimated-Ground Truth point count"] == [str(len(gt)), "/", str(len(gt))]
    pcd = _read_xyz_pcd(str(res / "noise_gt_map.pcd"))
    np.testing.assert_array_equal(pcd, gt.astype(np.float32))


@pytest.mark.gpu
def test_noised_gt_path_b_with_every_operator(exe, tmp_path, gt):  # noqa: F811
    sim = SIM.format(sigma=0.005) + ("density_sparse_ratio: 0.4\ndensity_dense_ratio: 0.9\ndensity_region_size: 0.5\n"
                                     "outlier_ratio: 0.01\noutlier_range: 0.3\n"
                                     "deform_radius: 0.6\ndeform_strength: 0.05\ndeform_center: [1.0, 1.2, 0.9]\n")
    out, line, res = _run(exe, tmp_path, gt, sim, initial="false")
    assert "local deformation (radius 0.6, strength 0.05, centre 1 1.2 0.9), then non-uniform density" in out.stdout
    c = np.array([1.0, 1.2, 0.9])
    e = ref.local_deformation(gt, 0.6, 0.05, c)
    keep, _, _ = ref.density_keep(e, 0.4, 0.9, 0.5, 777)
    m = ref.outlier_count(keep.sum(), 0.01)
    assert int(line["Estimated-Ground Truth point count"][0]) == keep.sum() + m
    assert len(_read_xyz_pcd(str(res / "noise_gt_map.pcd"))) == keep.sum() + m
    assert "Aligned results" in line


def test_noised_gt_keys_in_dump_config(exe, tmp_path):  # noqa: F811
    cfg = tmp_path / "c.yaml"
    base = CONFIG.format(est=str(tmp_path / "est"), gt=str(tmp_path / "gt.pcd"), gt_mme="false", initial="true")
    cfg.write_text(base)
    _, kv = _dump(exe, str(cfg))
    assert kv["evaluate_noised_gt"] == "0" and float(kv["noise_std_dev"]) == 0.1 and kv["simulation_seed"] == "20250002"
    assert kv["density_set"] == "0" and float(kv["outlier_ratio"]) == 0 and float(kv["deform_radius"]) == 0
    cfg.write_text(base + "evaluate_noised_gt: true\nsimulation_seed: 18446744073709551615\ndensity_region_size: 2.5\n"
                   "density_sparse_ratio: 0.2\ndensity_dense_ratio: 0.7\noutlier_ratio: 0.1\noutlier_range: 3\n"
                   "deform_radius: 4\ndeform_strength: -0.5\ndeform_center: [1, -2, 3.5]\n")
    _, kv = _dump(exe, str(cfg))
    assert kv["evaluate_noised_gt"] == "1" and kv["simulation_seed"] == str(2 ** 64 - 1)
    assert kv["density_set"] == "1" and float(kv["density_region_size"]) == 2.5
    assert (float(kv["density_sparse_ratio"]), float(kv["density_dense_ratio"])) == (0.2, 0.7)
    assert (float(kv["outlier_ratio"]), float(kv["outlier_range"])) == (0.1, 3.0)
    assert (float(kv["deform_radius"]), float(kv["deform_strength"])) == (4.0, -0.5)
    assert [float(x) for x in kv["deform_center"].split(",")] == [1.0, -2.0, 3.5]


@pytest.mark.gpu
def test_noised_gt_two_gpus_matches_one(exe, tmp_path, gt):  # noqa: F811
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (NCCL cannot put two ranks of one communicator on one device)")
    sim = SIM.format(sigma=0.01) + "outlier_ratio: 0.02\noutlier_range: 0.5\ndensity_region_size: 0.5\n"
    outs = {}
    for n in (1, 2):
        _, outs[n], res = _run(exe, tmp_path / f"run{n}", gt, sim, gpus=n)
    assert outs[1]["Estimated-Ground Truth point count"] == outs[2]["Estimated-Ground Truth point count"]
    assert outs[1]["Comp"] == outs[2]["Comp"]
    for key in ("RMSE/AC", "MME", "VMD", "SCS"):
        np.testing.assert_allclose([float(x) for x in outs[2][key]], [float(x) for x in outs[1][key]], rtol=1e-12, atol=1e-12,
                                   err_msg=key)
    a = (tmp_path / "run1" / "est" / "map_results" / "noise_gt_map.pcd").read_bytes()
    assert a == (tmp_path / "run2" / "est" / "map_results" / "noise_gt_map.pcd").read_bytes()

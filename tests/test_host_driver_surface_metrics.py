"""The re-hosted `map_eval` with `surface_metrics: true`: surface_metrics.txt next to map_results.txt on path A and on path B
(generalized ICP), from a ground truth with normals in its file and from one without, its path A values equal to the Python
API's on the same clouds and normals; every other output unchanged by the key; both keys in --dump-config; bad
surface_normals_knn values refused when the configuration is loaded; two GPUs against one."""
import subprocess

import numpy as np
import pytest

from test_host_driver_accuracy_curve import CONFIG, _stable, _write_pcd, exe  # noqa: F401  (module fixture)
from test_host_driver_normals import _write_ply_normals

LEVELS = [0.2, 0.1, 0.08, 0.05, 0.01]
KEY = "surface_metrics: true\n"
DCOLS = ["direction", "n_corr", "n_no_normal"] + [f"{f}_{k}" for f in ("n_inlier", "mean", "rmse", "fitness", "sigma")
                                                  for k in range(1, 6)]
DCOLS += ["mean_nn", "max_e", "max_e_nn", "n_nc", "normal_consistency"]
PCOLS = [f"{f}_{k}" for f in ("cd", "f1", "iou") for k in range(1, 6)] + ["full_cd", "normal_consistency"]


@pytest.fixture(scope="module")
def maps(tmp_path_factory):
    from cloud_map_evaluation_b200 import synth
    d = tmp_path_factory.mktemp("surface")
    est, gt, _ = synth.make_pair("C1", scale=0.3)
    rng = np.random.default_rng(3)
    nrm = rng.normal(size=gt.shape) * rng.uniform(0.5, 2.0, (len(gt), 1))      # not unit length, as files may be
    _write_pcd(str(d / "gt.pcd"), gt)
    _write_ply_normals(str(d / "gt.ply"), gt, nrm)
    return d, est, gt, nrm


def _config(d, est_dir, gt_file, initial, extra):
    text = CONFIG.format(levels=", ".join(repr(x) for x in LEVELS), est=str(est_dir), gt=str(d / gt_file), initial=initial,
                         extra=extra)
    return text.replace("downsample_size: 0.01", "downsample_size: 0.0")     # evaluate the clouds as loaded


def _run(exe, d, name, est, gt_file, initial, extra="", args=()):
    est_dir = d / name / "est"
    est_dir.mkdir(parents=True)
    _write_pcd(str(est_dir / "map.pcd"), est)
    cfg = d / name / "config.yaml"
    cfg.write_text(_config(d, est_dir, gt_file, initial, extra))
    out = subprocess.run([exe, str(cfg), *args], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    return out, est_dir / "map_results"


def _read(path):
    """(comment line, {direction: {column: value}}, {column: value}) of surface_metrics.txt"""
    lines = path.read_text().splitlines()
    assert lines[0].startswith("# ") and lines[1].split() == DCOLS and lines[4].split() == PCOLS and len(lines) == 6
    rows = {}
    for line in lines[2:4]:
        v = line.split()
        assert len(v) == len(DCOLS)
        rows[v[0]] = {c: float(x) for c, x in zip(DCOLS[1:], v[1:])}
    pair = dict(zip(PCOLS, (float(x) for x in lines[5].split())))
    assert len(pair) == len(PCOLS)
    return lines[0], rows, pair


def test_dump_config_lists_the_keys(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "gt.pcd", "true", KEY + "surface_normals_knn: 12\n"))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert "surface_metrics=1" in out.stdout.splitlines() and "surface_normals_knn=12" in out.stdout.splitlines()
    cfg.write_text(_config(tmp_path, tmp_path, "gt.pcd", "true", ""))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert "surface_metrics=0" in out.stdout.splitlines() and "surface_normals_knn=20" in out.stdout.splitlines()


@pytest.mark.parametrize("bad", ["0", "65", "-3", "1000"])
def test_bad_knn_is_refused_at_load(exe, tmp_path, bad):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "gt.pcd", "true", KEY + f"surface_normals_knn: {bad}\n"))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)     # refused before anything runs
    assert out.returncode != 0 and "surface_normals_knn" in out.stderr


def _same_outputs(on, off, initial):
    """every file of the run with the key but surface_metrics.txt is the run without it: map_results.txt but for its header
    and timing lines; on path A voxel_errors.txt as a set of rows (they come in the order the voxel pairs are found, which
    varies from run to run) and every other file byte for byte (on path B the ICP sums use floating-point atomics, so the
    registered cloud may differ in its last bits between any two runs)"""
    names = sorted(p.name for p in on.iterdir() if p.name != "surface_metrics.txt")
    assert names == sorted(p.name for p in off.iterdir())
    for n in names:
        if n == "map_results.txt":
            assert _stable((on / n).read_text().splitlines()) == _stable((off / n).read_text().splitlines())
        elif initial != "true":
            continue
        elif n == "voxel_errors.txt":
            rows = (on / n).read_text().splitlines()
            assert len(rows) > 0 and sorted(rows) == sorted((off / n).read_text().splitlines())
        else:
            assert (on / n).read_bytes() == (off / n).read_bytes(), n


@pytest.mark.gpu
@pytest.mark.parametrize("initial", ["true", "false"])     # path A, path B (generalized ICP)
@pytest.mark.parametrize("gt_file", ["gt.ply", "gt.pcd"])  # gt normals from the file / k-NN normals
def test_surface_file(exe, maps, initial, gt_file):
    from cloud_map_evaluation_b200 import _abi as A
    from cloud_map_evaluation_b200 import api
    d, est, gt, nrm = maps
    name = f"{gt_file.split('.')[1]}_{initial}"
    out, res = _run(exe, d, f"on_{name}", est, gt_file, initial, KEY)
    info = [l for l in out.stdout.splitlines() if l.startswith("INFO: point-to-plane CD at level 1: ")]
    assert len(info) == 1 and "surface_metrics.txt" in info[0]
    comment, rows, pair = _read(res / "surface_metrics.txt")
    assert "est normals: k-NN (k = 20)" in comment
    assert ("gt normals: file" if gt_file == "gt.ply" else "gt normals: k-NN (k = 20)") in comment
    for dname, n in (("est_to_gt", len(est)), ("gt_to_est", len(gt))):
        r = rows[dname]
        assert 0 < r["n_corr"] <= n and r["n_no_normal"] == 0 and r["n_nc"] == r["n_corr"]
        assert 0.0 < r["normal_consistency"] <= 1.0
    if initial == "true":      # path A: the same clouds and normals through the Python API
        p = A.make_nn_params(LEVELS, 1.0)
        with api.MapEvalB200() as ctx:
            ctx.set_cloud(A.ME_CLOUD_EST, est.astype(np.float32).astype(np.float64))
            ctx.set_cloud(A.ME_CLOUD_GT, gt.astype(np.float32).astype(np.float64) if gt_file == "gt.pcd" else gt)
            if gt_file == "gt.ply":
                ctx.set_normals(A.ME_CLOUD_GT, nrm)
            ctx.transform(A.ME_CLOUD_EST, np.eye(4))
            ctx.calculateMetricsWithInitialMatrix(p)
            ref = ctx.surface_metrics(knn=20)
        for dname in ("est_to_gt", "gt_to_est"):
            r, w = rows[dname], ref[dname]
            for c in ("n_corr", "n_no_normal", "n_nc"):
                assert r[c] == w[c], c
            for k in range(5):
                assert r[f"n_inlier_{k + 1}"] == w["n_inlier"][k]
                for f, tol in (("mean", 1e-12), ("rmse", 1e-12), ("fitness", 1e-12), ("sigma", 1e-9)):
                    np.testing.assert_allclose(r[f"{f}_{k + 1}"], w[f][k], rtol=tol, atol=1e-15, err_msg=f)
            np.testing.assert_allclose(r["mean_nn"], w["sum_nn_dist"] / w["n_source"], rtol=1e-12, atol=1e-15)
            for c in ("max_e", "max_e_nn"):
                np.testing.assert_allclose(r[c], w[c], rtol=0, atol=1e-15)
            np.testing.assert_allclose(r["normal_consistency"], w["normal_consistency"], rtol=1e-12)
        for f in ("cd", "f1", "iou"):
            for k in range(5):
                np.testing.assert_allclose(pair[f"{f}_{k + 1}"], ref[f][k], rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(pair["full_cd"], ref["full_cd"], rtol=1e-12)
        np.testing.assert_allclose(pair["normal_consistency"], ref["normal_consistency"], rtol=1e-12)
    # without the key: no file, and every other output the same
    _, res_off = _run(exe, d, f"off_{name}", est, gt_file, initial)
    assert not (res_off / "surface_metrics.txt").exists()
    _same_outputs(res, res_off, initial)


@pytest.mark.gpu
def test_two_gpus_match_one(exe, maps):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (NCCL cannot put two ranks of one communicator on one device)")
    d, est, _, _ = maps
    for initial in ("true", "false"):
        _, one = _run(exe, d, f"g1_{initial}", est, "gt.pcd", initial, KEY, ("--gpus", "1"))
        _, two = _run(exe, d, f"g2_{initial}", est, "gt.pcd", initial, KEY, ("--gpus", "2"))
        c1, r1, p1 = _read(one / "surface_metrics.txt")
        c2, r2, p2 = _read(two / "surface_metrics.txt")
        assert c1 == c2
        for dname in r1:
            for c, v in r1[dname].items():
                if initial == "true" and (c.startswith(("n_", "max_e"))):
                    assert r2[dname][c] == v, c      # counts and maxima do not depend on the world
                else:        # sums reduce in another order; on path B the ICP sums, and so T, may differ in the last bits too
                    np.testing.assert_allclose(r2[dname][c], v, rtol=1e-9, atol=1e-12, err_msg=c)
        for c, v in p1.items():
            np.testing.assert_allclose(p2[c], v, rtol=1e-9, atol=1e-12, err_msg=c)

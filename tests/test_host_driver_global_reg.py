"""The re-hosted `map_eval` with `global_registration: true`: the estimate file holds a turned and moved map, the configuration
an identity initial_matrix.  The pose from me_global_registration replaces initial_matrix on path B (T_init of generalized
ICP) and on path A (the transform), and map_results.txt carries its lines only when the switch is on."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_global_reg import _apply, _errors, _furnished_rooms, _motion  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "cloud_map_evaluation_b200", "map_eval")

CONFIG = """registration_methods: 2
icp_max_distance: 1.0
accuracy_level: [0.2, 0.1, 0.08, 0.05, 0.01]
initial_matrix:
{matrix}
estimate_map_path: {est}
gt_map_path: "{gt}"
scene_name: global_reg_test
save_immediate_result: true
evaluate_mme: false
evaluate_gt_mme: false
nn_radius: 0.1
evaluate_using_initial: {initial}
vmd_voxel_size: 1.0
downsample_size: 0.05
enable_debug: false
{extra}"""

GR_KEYS = "global_registration: true\nglobal_registration_voxel_size: 0.5\nglobal_registration_seed: 7\n" \
          "global_registration_hypotheses: 50000\n"


@pytest.fixture(scope="module")
def exe():
    if not os.path.exists(EXE):
        import __graft_entry__ as g
        g.build()
    return EXE


def _write_pcd(path, xyz):
    n = len(xyz)
    hdr = (f"# .PCD v0.7\nVERSION 0.7\nFIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nCOUNT 1 1 1\nWIDTH {n}\nHEIGHT 1\n"
           f"VIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA binary\n")
    with open(path, "wb") as f:
        f.write(hdr.encode())
        f.write(xyz.astype(np.float32).tobytes())


def _matrix(T):
    return "\n".join("  - [" + ", ".join(repr(float(x)) for x in row) + "]" for row in T)


@pytest.fixture(scope="module")
def maps(tmp_path_factory):
    from cloud_map_evaluation_b200 import synth
    d = tmp_path_factory.mktemp("gr")
    gt = _furnished_rooms(300_000, synth.GT_SEED, 0.002)
    est = _furnished_rooms(300_000, synth.EST_SEED, 0.01)
    est = est[est[:, 0] < 0.6 * est[:, 0].max()]
    M = _motion(120.0, 3.0, [-61.8, 53.1, 2.5])
    _write_pcd(str(d / "gt.pcd"), gt)
    return d, np.ascontiguousarray(_apply(M, est)), np.linalg.inv(M)


def _run(exe, d, name, est, initial, T_init=np.eye(4), extra="", args=()):
    run = d / name
    est_dir = run / "est"
    est_dir.mkdir(parents=True)
    _write_pcd(str(est_dir / "map.pcd"), est)
    cfg = run / "config.yaml"
    cfg.write_text(CONFIG.format(matrix=_matrix(T_init), est=str(est_dir), gt=str(d / "gt.pcd"), initial=initial, extra=extra))
    out = subprocess.run([exe, str(cfg), *args], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = (est_dir / "map_results" / "map_results.txt").read_text().splitlines()
    return out, lines


def _matrix_after(lines, key):
    i0 = next(i for i, l in enumerate(lines) if l.startswith(key + ":"))
    return np.array([[float(x) for x in lines[i0].split(":", 1)[1].split()]] + [[float(x) for x in lines[i0 + k].split()] for k in (1, 2, 3)])


def _fields(lines):
    return {l.split(":")[0]: l.split(":", 1)[1].split() for l in lines
            if ":" in l and not l.startswith(("Ground", "Evaluation", "global_reg_test", "Estimated"))}


def test_dump_config_lists_the_keys(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(CONFIG.format(matrix=_matrix(np.eye(4)), est=str(tmp_path), gt=str(tmp_path / "gt.pcd"), initial="false", extra=GR_KEYS))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    for line in ("global_registration=1", "global_registration_voxel_size=0.5", "global_registration_seed=7",
                 "global_registration_hypotheses=50000"):
        assert line in out.stdout.splitlines(), line
    cfg.write_text(CONFIG.format(matrix=_matrix(np.eye(4)), est=str(tmp_path), gt=str(tmp_path / "gt.pcd"), initial="false", extra=""))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    for line in ("global_registration=0", "global_registration_voxel_size=0.5", "global_registration_seed=0",
                 "global_registration_hypotheses=100000"):
        assert line in out.stdout.splitlines(), line


@pytest.mark.gpu
def test_path_b_recovers_the_pose(exe, maps):
    d, est, T_true = maps
    out, lines = _run(exe, d, "b_gr", est, "false", extra=GR_KEYS)
    assert "replaces the initial_matrix" not in out.stdout          # identity initial_matrix: no warning
    Tg = _matrix_after(lines, "Global registration cloud")
    ang, dt = _errors(Tg, T_true)
    assert ang <= 2.0 and dt <= 1.0, (ang, dt)
    g = _fields(lines)["Global registration"]
    assert 0 < float(g[0]) <= 1 and int(g[1]) >= 3 and int(g[1]) <= int(g[2])
    Ta = _matrix_after(lines, "Aligned cloud")
    np.testing.assert_allclose(Ta, T_true, atol=1e-2)
    # the same run given the true matrix and no global registration
    _, ref = _run(exe, d, "b_true", est, "false", T_init=T_true)
    assert not any(l.startswith("Global registration") for l in ref)
    # ICP stops on relative criteria (1e-6 in fitness and rmse), so two starts a few cm apart end up to ~1 mm apart
    np.testing.assert_allclose(Ta, _matrix_after(ref, "Aligned cloud"), atol=2e-3)
    a, b = _fields(lines), _fields(ref)
    for key in ("RMSE/AC", "Aligned results"):
        np.testing.assert_allclose([float(x) for x in a[key]], [float(x) for x in b[key]], rtol=1e-2, atol=1e-5, err_msg=key)


@pytest.mark.gpu
def test_path_a_uses_the_pose(exe, maps):
    d, est, T_true = maps
    T_wrong = np.eye(4)
    T_wrong[:3, 3] = [1.0, 2.0, 0.0]
    out, lines = _run(exe, d, "a_gr", est, "true", T_init=T_wrong, extra=GR_KEYS)
    assert "replaces the initial_matrix" in out.stdout                # the configuration's matrix was not the identity
    Tg = _matrix_after(lines, "Global registration cloud")
    ang, dt = _errors(Tg, T_true)
    assert ang <= 2.0 and dt <= 1.0, (ang, dt)
    assert "Aligned cloud" not in _fields(lines)
    # path A evaluates at that pose: its accuracy is that of a run given the same matrix without global registration
    _, ref = _run(exe, d, "a_same", est, "true", T_init=np.round(Tg, 5))
    a, b = _fields(lines), _fields(ref)
    np.testing.assert_allclose([float(x) for x in a["RMSE/AC"]], [float(x) for x in b["RMSE/AC"]], rtol=1e-2)


@pytest.mark.gpu
def test_two_gpus_equal_one(exe, maps):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    d, est, _ = maps
    _, one = _run(exe, d, "g1", est, "false", extra=GR_KEYS, args=("--gpus", "1"))
    _, two = _run(exe, d, "g2", est, "false", extra=GR_KEYS, args=("--gpus", "2"))
    a, b = _fields(one), _fields(two)
    for key in ("Global registration cloud", "Global registration", "Aligned results"):
        assert a[key] == b[key], key

"""The re-hosted `map_eval` with `accuracy_curve_steps`: accuracy_curve.txt next to map_results.txt on path A and on path B
(generalized ICP), whose rows at the five accuracy_level grid values equal the RMSE/AC and Comp: lines; without the keys no
file and the same map_results.txt; both keys in --dump-config."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "cloud_map_evaluation_b200", "map_eval")

STEPS, MAX = 40, 0.2
PICK = (40, 20, 16, 10, 2)                    # accuracy_level = the grid values tau_k at these k
GRID = [(MAX * k) / STEPS for k in PICK]       # as the driver computes them, in double

CONFIG = """registration_methods: 2
icp_max_distance: 1.0
accuracy_level: [{levels}]
estimate_map_path: {est}
gt_map_path: "{gt}"
scene_name: curve_test
save_immediate_result: true
evaluate_mme: false
evaluate_gt_mme: false
nn_radius: 0.1
evaluate_using_initial: {initial}
vmd_voxel_size: 0.25
downsample_size: 0.01
enable_debug: false
{extra}"""


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


@pytest.fixture(scope="module")
def maps(tmp_path_factory):
    from cloud_map_evaluation_b200 import synth
    d = tmp_path_factory.mktemp("curve")
    est, gt, _ = synth.make_pair("C1", scale=0.3)
    _write_pcd(str(d / "gt.pcd"), gt)
    return d, est


def _config(d, est_dir, initial, extra):
    return CONFIG.format(levels=", ".join(repr(x) for x in GRID), est=str(est_dir), gt=str(d / "gt.pcd"), initial=initial,
                         extra=extra)


def _run(exe, d, name, est, initial, extra="", args=()):
    est_dir = d / name / "est"
    est_dir.mkdir(parents=True)
    _write_pcd(str(est_dir / "map.pcd"), est)
    cfg = d / name / "config.yaml"
    cfg.write_text(_config(d, est_dir, initial, extra))
    out = subprocess.run([exe, str(cfg), *args], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    res = est_dir / "map_results"
    return out, (res / "map_results.txt").read_text().splitlines(), res / "accuracy_curve.txt"


def _fields(lines):
    return {l.split(":")[0]: l.split(":", 1)[1].split() for l in lines if ":" in l}


def _stable(lines):
    """map_results.txt without the header (time stamp, paths) and the timing lines"""
    return [l for l in lines if "=====" not in l and "Time" not in l and not l.startswith(("Ground Truth", "Evaluation Map"))]


def test_dump_config_lists_the_keys(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "true", f"accuracy_curve_steps: {STEPS}\naccuracy_curve_max: 0.3\n"))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert "accuracy_curve_steps=40" in out.stdout.splitlines() and "accuracy_curve_max=0.29999999999999999" in out.stdout.splitlines()
    cfg.write_text(_config(tmp_path, tmp_path, "true", ""))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert "accuracy_curve_steps=0" in out.stdout.splitlines()
    assert "accuracy_curve_max=0.20000000000000001" in out.stdout.splitlines()      # the largest accuracy_level


def test_out_of_range_steps_are_refused(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "true", "accuracy_curve_steps: 1025\n"))
    out = subprocess.run([exe, str(cfg)], capture_output=True, text=True)
    assert out.returncode != 0 and "accuracy_curve_steps" in out.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("initial", ["true", "false"])     # path A, path B (generalized ICP)
def test_curve_file_matches_the_five_levels(exe, maps, initial):
    d, est = maps
    keys = f"accuracy_curve_steps: {STEPS}\n"
    out, lines, curve = _run(exe, d, f"on_{initial}", est, initial, keys)
    assert any(l.startswith("INFO: accuracy curve") and "accuracy_curve.txt" in l for l in out.stdout.splitlines())
    rows = curve.read_text().splitlines()
    assert rows[0].split()[0] == "tau" and len(rows) == STEPS + 1
    tab = np.array([[float(x) for x in r.split()] for r in rows[1:]])
    np.testing.assert_allclose(tab[:, 0], [(MAX * k) / STEPS for k in range(1, STEPS + 1)], rtol=0, atol=1e-15)
    assert np.all(np.diff(tab[:, 1]) >= 0) and np.all(np.diff(tab[:, 6]) >= 0)      # counts grow with tau
    f = _fields(lines)
    rmse = [float(x) for x in f["RMSE/AC"]]
    comp = [float(x) for x in f["Comp"]]
    for j, k in enumerate(PICK):
        np.testing.assert_allclose(tab[k - 1, 3], rmse[j], rtol=1e-12, atol=2e-15)     # e2g_rmse
        np.testing.assert_allclose(tab[k - 1, 4], comp[j], rtol=1e-12, atol=2e-15)     # e2g_fitness
    # without the keys: no file, and the same results as with accuracy_curve_steps: 0
    _, off, c_off = _run(exe, d, f"off_{initial}", est, initial)
    _, zero, c_zero = _run(exe, d, f"zero_{initial}", est, initial, "accuracy_curve_steps: 0\n")
    assert not c_off.exists() and not c_zero.exists()
    assert _stable(off) == _stable(zero)
    assert _stable(off) == _stable(lines)

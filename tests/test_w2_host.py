"""The re-hosted `map_eval` with `evaluate_w2`, without a GPU: both keys in --dump-config, bad values refused when the
configuration is loaded, and the key refused with evaluate_without_gt."""
import subprocess

import pytest

from test_host_driver_mom import NO_GT, _config
from test_host_driver_accuracy_curve import exe  # noqa: F401  (module fixture)


def _dump(exe, cfg):
    return subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)


def test_dump_config_lists_the_keys(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "evaluate_w2: true\nw2_min_points: 7\n"))
    out = _dump(exe, cfg)
    assert out.returncode == 0, out.stderr
    assert {"evaluate_w2=1", "w2_min_points=7"} <= set(out.stdout.splitlines())
    cfg.write_text(_config(tmp_path, tmp_path, ""))
    assert {"evaluate_w2=0", "w2_min_points=100"} <= set(_dump(exe, cfg).stdout.splitlines())


@pytest.mark.parametrize("bad", ["1", "0", "-5", "2.5", "nan"])
def test_bad_min_points_are_refused_at_load(exe, tmp_path, bad):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, f"evaluate_w2: true\nw2_min_points: {bad}\n"))
    out = _dump(exe, cfg)
    assert out.returncode != 0 and "w2_min_points" in out.stderr


def test_refused_without_gt(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, NO_GT + "evaluate_w2: true\n", with_gt=False))
    out = subprocess.run([exe, str(cfg)], capture_output=True, text=True)
    assert out.returncode != 0 and "evaluate_w2" in out.stderr and "needs a ground truth" in out.stderr
    assert not (tmp_path / "map_results").exists()

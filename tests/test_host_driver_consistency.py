"""The re-hosted `map_eval` with `evaluate_consistency: true`: map_consistency.txt next to map_results.txt on path A and on
path B, with and without evaluate_gt_mme, for the whole map and per region; at consistency_region_size = region_size its
region rows have region_errors.txt's bounds in its order; on path A with the identity initial_matrix the whole-map est MME
is within the fp32-path certificate (1e-3 nats) plus half a unit of the fifth decimal of map_results.txt's MME line; every
other output unchanged by the keys; both keys in --dump-config; bad region sizes refused when the configuration is loaded;
two GPUs against one."""
import math
import subprocess

import numpy as np
import pytest

from test_host_driver_accuracy_curve import CONFIG, _stable, _write_pcd, exe  # noqa: F401  (module fixture)

LEVELS = [0.2, 0.1, 0.08, 0.05, 0.01]
KEY = "evaluate_consistency: true\n"
STATS = ["n_query", "n_valid", "n_pv", "mme", "mpv", "mean_plane_std", "max_pv"]
WCOLS = ["cloud", "n_points"] + STATS
RCOLS = ["cloud", "min_x", "min_y", "min_z", "max_x", "max_y", "max_z", "n_points"] + STATS
S = 0.75


@pytest.fixture(scope="module")
def maps(tmp_path_factory):
    from cloud_map_evaluation_b200 import synth
    d = tmp_path_factory.mktemp("consistency")
    est, gt, _ = synth.make_pair("C1", scale=0.3)
    _write_pcd(str(d / "gt.pcd"), gt)
    return d, est, gt


def _config(d, est_dir, initial, extra, gt_mme=False):
    text = CONFIG.format(levels=", ".join(repr(x) for x in LEVELS), est=str(est_dir), gt=str(d / "gt.pcd"), initial=initial,
                         extra=extra)
    text = text.replace("downsample_size: 0.01", "downsample_size: 0.0").replace("evaluate_mme: false", "evaluate_mme: true")
    return text.replace("evaluate_gt_mme: false", f"evaluate_gt_mme: {'true' if gt_mme else 'false'}")


def _run(exe, d, name, est, initial, extra="", gt_mme=False, args=()):
    est_dir = d / name / "est"
    est_dir.mkdir(parents=True)
    _write_pcd(str(est_dir / "map.pcd"), est)
    cfg = d / name / "config.yaml"
    cfg.write_text(_config(d, est_dir, initial, extra, gt_mme))
    out = subprocess.run([exe, str(cfg), *args], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    return out, est_dir / "map_results"


def _read(path):
    """(comment line, {cloud: {column: value}}, [region rows as dicts])"""
    lines = path.read_text().splitlines()
    assert lines[0].startswith("# ") and lines[1].split() == WCOLS
    whole, rows, i = {}, [], 2
    while i < len(lines) and lines[i].split()[0] in ("est", "gt"):
        v = lines[i].split()
        assert len(v) == len(WCOLS)
        whole[v[0]] = {c: (int(x) if c.startswith("n_") else float(x)) for c, x in zip(WCOLS[1:], v[1:])}
        i += 1
    if i < len(lines):
        assert lines[i].split() == RCOLS
        for line in lines[i + 1:]:
            v = line.split()
            assert len(v) == len(RCOLS)
            row = {"cloud": v[0], "bounds": v[1:7]}
            row.update({c: (int(x) if c.startswith("n_") else float(x)) for c, x in zip(RCOLS[7:], v[7:])})
            rows.append(row)
    return lines[0], whole, rows


def test_dump_config_lists_the_keys(exe, tmp_path):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "true", KEY + "consistency_region_size: 0.5\n"))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.splitlines()
    assert "evaluate_consistency=1" in lines and "consistency_region_size=0.5" in lines
    cfg.write_text(_config(tmp_path, tmp_path, "true", ""))
    lines = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True).stdout.splitlines()
    assert "evaluate_consistency=0" in lines and "consistency_region_size=0" in lines


@pytest.mark.parametrize("bad", ["-0.5", "nan", "inf", "-inf"])
def test_bad_region_size_is_refused_at_load(exe, tmp_path, bad):
    cfg = tmp_path / "config.yaml"
    cfg.write_text(_config(tmp_path, tmp_path, "true", KEY + f"consistency_region_size: {bad}\n"))
    out = subprocess.run([exe, str(cfg), "--dump-config"], capture_output=True, text=True)     # refused before anything runs
    assert out.returncode != 0 and "consistency_region_size" in out.stderr


def _same_outputs(on, off, initial):
    """every file of the run with the keys but map_consistency.txt is the run without them: map_results.txt but for its
    header and timing lines; on path A voxel_errors.txt as a set of rows and every other file byte for byte (on path B the
    ICP sums use floating-point atomics, so the registered cloud may differ in its last bits between any two runs)"""
    names = sorted(p.name for p in on.iterdir() if p.name != "map_consistency.txt")
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
@pytest.mark.parametrize("initial", ["true", "false"])      # path A, path B (generalized ICP)
@pytest.mark.parametrize("gt_mme", [False, True])
@pytest.mark.parametrize("s", [0.0, S])
def test_consistency_file(exe, maps, initial, gt_mme, s):
    d, est, gt = maps
    name = f"{initial}_{int(gt_mme)}_{s}"
    extra = KEY + f"consistency_region_size: {s}\nregion_size: {S}\n"
    out, res = _run(exe, d, f"on_{name}", est, initial, extra, gt_mme)
    info = [l for l in out.stdout.splitlines() if l.startswith("INFO: local consistency:")]
    assert len(info) == 1 and "map_consistency.txt" in info[0] and "est MPV" in info[0] and ("gt MPV" in info[0]) == gt_mme
    comment, whole, rows = _read(res / "map_consistency.txt")
    assert "r = 0.10000000000000001" in comment and "est in the ground truth's frame" in comment
    assert ("gt 5" in comment) == gt_mme
    assert sorted(whole) == (["est", "gt"] if gt_mme else ["est"])
    for cloud, n in (("est", len(est)), ("gt", len(gt))):
        if cloud not in whole:
            continue
        w = whole[cloud]
        assert w["n_points"] == w["n_query"] == n and 0 < w["n_valid"] <= w["n_pv"] <= n
        assert w["mpv"] > 0 and w["max_pv"] >= w["mpv"] and math.isfinite(w["mme"])
    if s == 0.0:
        assert rows == []
    else:       # the rows of region_errors.txt, in its order, once per evaluated cloud
        reg = [l.split()[:6] for l in (res / "region_errors.txt").read_text().splitlines()[1:]]
        for cloud in whole:
            mine = [r for r in rows if r["cloud"] == cloud]
            assert [r["bounds"] for r in mine] == reg
            assert sum(r["n_points"] for r in mine) == whole[cloud]["n_points"]
            for c in ("n_query", "n_valid", "n_pv"):
                assert sum(r[c] for r in mine) == whole[cloud][c]
    if initial == "true":      # identity initial_matrix: the est cloud MME measured, within its certificate
        line = [l for l in (res / "map_results.txt").read_text().splitlines() if l.startswith("MME: ")][-1]
        assert abs(whole["est"]["mme"] - float(line.split()[1])) <= 1e-3 + 5e-6
    # without the keys: no file, and every other output the same
    _, res_off = _run(exe, d, f"off_{name}", est, initial, f"region_size: {S}\n", gt_mme)
    assert not (res_off / "map_consistency.txt").exists()
    _same_outputs(res, res_off, initial)


@pytest.mark.gpu
def test_two_gpus_match_one(exe, maps):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (NCCL cannot put two ranks of one communicator on one device)")
    d, est, _ = maps
    extra = KEY + f"consistency_region_size: {S}\n"
    for initial in ("true", "false"):
        _, one = _run(exe, d, f"g1_{initial}", est, initial, extra, True, ("--gpus", "1"))
        _, two = _run(exe, d, f"g2_{initial}", est, initial, extra, True, ("--gpus", "2"))
        c1, w1, r1 = _read(one / "map_consistency.txt")
        c2, w2, r2 = _read(two / "map_consistency.txt")
        assert c1 == c2 and len(r1) == len(r2)
        for a, b in [(w1[k], w2[k]) for k in w1] + list(zip(r1, r2)):
            for c, v in a.items():
                if c in ("cloud", "bounds") or (initial == "true" and c.startswith("n_")):
                    assert b[c] == v, c
                else:
                    np.testing.assert_allclose(b[c], v, rtol=1e-9, atol=1e-12, err_msg=c)

"""`map_eval --gpus 2` on path B (evaluate_using_initial: false, generalized ICP — what every shipped config runs): the
registration runs on both GPUs (each sweeps its query range and estimates its slice of the k-NN normals; NCCL all-gathers
the slices and all-reduces the ICP sums once per iteration).  The result lines must match the single-GPU run."""
import subprocess

import numpy as np
import pytest

from test_host_driver import CONFIG, _write_pcd, exe  # noqa: F401  (module fixture)


@pytest.mark.gpu
def test_map_eval_two_gpus_path_b_matches_one(exe, tmp_path):  # noqa: F811
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (NCCL cannot put two ranks of one communicator on one device)")
    from cloud_map_evaluation_b200 import synth
    est, gt, cfg = synth.make_pair("C2", scale=0.3)
    outs = {}
    for n in (1, 2):
        d = tmp_path / f"run{n}"
        est_dir = d / "est"
        est_dir.mkdir(parents=True)
        _write_pcd(str(est_dir / "map.pcd"), est, "binary")
        _write_pcd(str(d / "gt.pcd"), gt, "binary")
        text = CONFIG.format(est=str(est_dir), gt=str(d / "gt.pcd"), gt_mme="false", initial="false")
        text = text.replace("[1.0, 0.0, 0.0, 0.5]", "[1.0, 0.0, 0.0, 0.0]").replace("[0.0, 0.0, 1.0, -2]", "[0.0, 0.0, 1.0, 0.0]")
        text = text.replace("downsample_size: 0.0", "downsample_size: 0.02")
        (d / "config.yaml").write_text(text)
        out = subprocess.run([exe, str(d / "config.yaml"), "--gpus", str(n)], capture_output=True, text=True)
        assert out.returncode == 0, out.stdout + out.stderr
        assert "GPU 0 only" not in out.stdout
        res = (est_dir / "map_results" / "map_results.txt").read_text().splitlines()
        outs[n] = {l.split(":")[0]: l.split(":", 1)[1].split() for l in res if ":" in l and not l.startswith(("Ground", "Evaluation"))}
    for key in ("Aligned results", "Comp"):
        assert outs[1][key] == outs[2][key], key
    for key in ("RMSE/AC", "FULL CD", "VMD", "SCS"):
        np.testing.assert_allclose([float(x) for x in outs[2][key]], [float(x) for x in outs[1][key]], rtol=1e-9, atol=1e-9, err_msg=key)

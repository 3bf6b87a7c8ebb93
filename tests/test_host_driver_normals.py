"""The re-hosted `map_eval` on a ground-truth PLY that carries normals (nx ny nz): on path B the normals go through
VoxelDownSample with the points, point-to-plane ICP (registration_methods: 1) runs on the averaged normals, generalized
ICP (2) builds the ground truth's covariances from them; results against the oracle."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import normals_ref as ref  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "cloud_map_evaluation_b200", "map_eval")

CONFIG = """registration_methods: {method}
icp_max_distance: 1.0
accuracy_level: [0.2, 0.1, 0.08, 0.05, 0.01]
initial_matrix:
  - [1.0, 0.0, 0.0, 0.0]
  - [0.0, 1.0, 0.0, 0.0]
  - [0.0, 0.0, 1.0, 0.0]
  - [0.0, 0.0, 0.0, 1.0]
estimate_map_path: {est}
gt_map_path: "{gt}"
scene_name: normals_test
save_immediate_result: true
evaluate_mme: false
evaluate_gt_mme: false
nn_radius: 0.1
evaluate_using_initial: false
vmd_voxel_size: 0.25
downsample_size: {ds}
enable_debug: false
"""


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


def _write_ply_normals(path, xyz, nrm):
    n = len(xyz)
    hdr = (f"ply\nformat binary_little_endian 1.0\nelement vertex {n}\nproperty double x\nproperty double y\n"
           "property double z\nproperty double nx\nproperty double ny\nproperty double nz\nend_header\n")
    with open(path, "wb") as f:
        f.write(hdr.encode())
        f.write(np.ascontiguousarray(np.concatenate([xyz, nrm], 1), dtype="<f8").tobytes())


def _results(est_dir):
    res = (est_dir / "map_results" / "map_results.txt").read_text().splitlines()
    i0 = next(i for i, l in enumerate(res) if l.startswith("Aligned cloud:"))
    Tm = np.array([[float(x) for x in res[i0].split(":", 1)[1].split()]] + [[float(x) for x in res[i0 + k].split()] for k in (1, 2, 3)])
    line = {l.split(":")[0]: l.split(":", 1)[1].split() for l in res if ":" in l}
    return Tm, line


@pytest.mark.gpu
def test_map_eval_registration_with_file_normals(exe, tmp_path):
    from cloud_map_evaluation_b200 import _abi as A
    from cloud_map_evaluation_b200 import synth
    from oracle import oracle as O
    est, gt, _ = synth.make_pair("C2", scale=0.1)
    est = est.astype(np.float32).astype(np.float64)
    rs = np.random.RandomState(9)
    nrm = O.estimate_normals_knn(gt, 20) * rs.uniform(0.8, 1.2, (len(gt), 1))       # not unit length, as files may be
    nrm[rs.rand(len(gt)) < 0.02, 1] = np.nan                                         # skipped by the averaging
    est_dir = tmp_path / "est"
    est_dir.mkdir()
    _write_pcd(str(est_dir / "map.pcd"), est)
    _write_ply_normals(str(tmp_path / "gt.ply"), gt, nrm)
    s = 0.02
    de = O.voxel_downsample(est, s)
    dg, dn = ref.voxel_downsample_normals(gt, nrm, s)
    pb = A.make_nn_params([0.2, 0.1, 0.08, 0.05, 0.01], 1.0, cutoff_mode=A.ME_CUTOFF_DIST_LT_R, pairing=A.ME_PAIRING_GEOMETRIC)
    cfgp = tmp_path / "config.yaml"
    for method in (1, 2):
        cfgp.write_text(CONFIG.format(method=method, est=str(est_dir), gt=str(tmp_path / "gt.ply"), ds=s))
        out = subprocess.run([exe, str(cfgp)], capture_output=True, text=True)
        assert out.returncode == 0, out.stdout + out.stderr
        Tm, line = _results(est_dir)
        (est_dir / "map_results" / "map_results.txt").unlink()
        assert line["Estimated-Ground Truth point count"] == [str(len(de)), "/", str(len(dg))]
        if method == 1:          # point-to-plane on the down-sampled ground truth's averaged normals
            To, fit, rmse, nc, it = O.icp_point_to_plane(de, dg, dn, 1.0)
        else:                    # generalized ICP: ground-truth covariances from those normals, the map's estimated
            To, fit, rmse, nc, it = ref.icp_generalized(de, dg, O.estimate_normals_knn(de, 20), dn, 1.0)
        np.testing.assert_allclose(Tm, To, atol=6e-6)                                # printed with setprecision(5)
        assert int(line["Aligned results"][1]) == nc and abs(float(line["Aligned results"][0]) - fit) < 6e-6
        onb = O.eval_nn(O.transform(de, To), dg, pb)
        np.testing.assert_allclose([float(x) for x in line["RMSE/AC"]], list(onb.est_to_gt.rmse), rtol=1e-6, atol=1e-12)
    # the ground truth's normals matter: generalized ICP with estimated normals on both clouds lands elsewhere
    Te = O.icp_generalized(de, dg, 1.0)[0]
    assert np.abs(Te - To).max() > 1e-6
    # a ground truth without normals still cannot run point-to-plane ICP (Open3D raises), before any result is written
    _write_pcd(str(tmp_path / "gt.pcd"), gt)
    cfgp.write_text(CONFIG.format(method=1, est=str(est_dir), gt=str(tmp_path / "gt.pcd"), ds=s))
    out = subprocess.run([exe, str(cfgp)], capture_output=True, text=True)
    assert out.returncode != 0 and "requires pre-computed normal vectors" in out.stderr
    res = est_dir / "map_results" / "map_results.txt"
    assert not res.exists() or "Aligned cloud:" not in res.read_text()

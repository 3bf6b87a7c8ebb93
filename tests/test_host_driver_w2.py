"""The re-hosted `map_eval` with `evaluate_w2: true` on the GPU: map_w2.txt and voxel_w2.txt hold the Python API's values
on the same down-sampled clouds, and every other output is the one of the run without the key."""
import numpy as np
import pytest

from test_host_driver_accuracy_curve import _stable, exe  # noqa: F401  (module fixture)
from test_host_driver_mom import _run

pytestmark = pytest.mark.gpu

V = 0.25                   # vmd_voxel_size of the shared test configuration
HEAD = "aw2 mean_offset mean_shape scs n_pairs n_scs n_voxels_est n_voxels_gt".split()


@pytest.fixture(scope="module")
def maps(tmp_path_factory):
    from cloud_map_evaluation_b200 import synth
    from test_host_driver_accuracy_curve import _write_pcd
    d = tmp_path_factory.mktemp("w2")
    est, gt, _ = synth.make_pair("C1", scale=0.3)
    _write_pcd(str(d / "gt.pcd"), gt)
    return d, est, gt


def test_files_equal_the_python_api(exe, maps):
    from cloud_map_evaluation_b200 import _abi as A
    from cloud_map_evaluation_b200 import api
    d, est, gt = maps
    out, res = _run(exe, d, "on", est, "evaluate_w2: true\nw2_min_points: 10\n")
    assert [l for l in out.stdout.splitlines() if l.startswith("INFO: Gaussian 2-Wasserstein: AW2 ")]
    lines = (res / "map_w2.txt").read_text().splitlines()
    assert lines[0].startswith("# ") and "min_points 10" in lines[0] and lines[1].split() == HEAD and len(lines) == 3
    vals = dict(zip(HEAD, lines[2].split()))
    rl = (res / "voxel_w2.txt").read_text().splitlines()
    assert rl[0].startswith("# ") and len(rl[1].split()) == A.ME_W2_ROW_COLS
    rows = np.array([[float(x) for x in l.split()] for l in rl[2:]]).reshape(-1, A.ME_W2_ROW_COLS)
    with api.MapEvalB200(vmd_voxel_size=V) as ctx:     # the files' fp32 coordinates, down-sampled as the driver does
        ctx.set_cloud(A.ME_CLOUD_EST, est.astype(np.float32).astype(np.float64))
        ctx.set_cloud(A.ME_CLOUD_GT, gt.astype(np.float32).astype(np.float64))
        ctx.voxel_downsample(A.ME_CLOUD_EST, 0.01)
        ctx.voxel_downsample(A.ME_CLOUD_GT, 0.01)
        ref, ref_rows = ctx.voxel_w2(V, 10, 5, want_rows=True)
    assert ref.n_pairs > 20
    for k in ("n_pairs", "n_scs", "n_voxels_est", "n_voxels_gt"):
        assert int(vals[k]) == getattr(ref, k), k
    for k in ("aw2", "mean_offset", "mean_shape", "scs"):
        assert float(vals[k]) == pytest.approx(getattr(ref, k), rel=1e-9), k
    order = lambda r: r[np.lexsort(r[:, 2::-1].T)]        # noqa: E731
    a, b = order(rows), order(ref_rows)
    np.testing.assert_array_equal(a[:, 0:5], b[:, 0:5])
    np.testing.assert_allclose(a[:, 5:], b[:, 5:], rtol=1e-9, atol=1e-12)


def test_other_outputs_are_unchanged(exe, maps):
    d, est, _ = maps
    _, on = _run(exe, d, "on2", est, "evaluate_w2: true\n")
    _, off = _run(exe, d, "off", est, "")
    new = {"map_w2.txt", "voxel_w2.txt"}
    assert new <= {p.name for p in on.iterdir()}
    names = sorted(p.name for p in on.iterdir() if p.name not in new)
    assert names == sorted(p.name for p in off.iterdir())
    for n in names:
        if n == "map_results.txt":
            assert _stable((on / n).read_text().splitlines()) == _stable((off / n).read_text().splitlines())
        elif n in ("voxel_errors.txt", "voxel_wasserstein_cdf.txt"):
            assert sorted((on / n).read_text().splitlines()) == sorted((off / n).read_text().splitlines())
        else:
            assert (on / n).read_bytes() == (off / n).read_bytes(), n

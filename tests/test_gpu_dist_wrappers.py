"""The multi-GPU wrappers of dist.py at world 2 on one GPU.  Two gloo processes each hold library contexts of rank r, world 2
on cuda:0 and run the wrappers whose collectives are all-reduces: the accumulator block, the accuracy curve, the distance
quantiles, the region table, the point-to-plane metrics, drift, local consistency, MOM and its region rows, and ICP.  Every
rank's result must equal the world-1 call on the same clouds, to the tolerances of that metric's own sharded test (counts
exactly).  The clouds carry their normals (knn = 0) and ICP runs point-to-point, so no all-gather runs; gloo reduces the
device blocks through host memory."""
import os
import pickle
import socket

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import synth

import test_gpu_accuracy_curve as TA
import test_gpu_consistency as TC
import test_gpu_distance_quantiles as TQ
import test_gpu_drift as TD
import test_gpu_icp_sharded as TI
import test_gpu_mom as TM
import test_gpu_region_errors as TR
import test_gpu_surface_metrics as TS

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
LEVELS = np.linspace(0.0, 0.3, 64)
PROBS = np.array(TQ.FIXED_P)
REGION = 0.25
DRIFT = (0.5, 0.05)          # region size, max correspondence distance
CONS_REGION = 0.8
MOM_REGION = 1.5


def _nn_pair():
    est, gt, cfg = synth.make_pair("C1", scale=0.3)
    rng = np.random.default_rng(8)
    normals = (TS.random_normals(rng, len(est)), TS.random_normals(rng, len(gt)))
    p = A.make_nn_params(cfg["tau"], TR.R, cutoff_mode=A.ME_CUTOFF_DIST_LT_R, pairing=A.ME_PAIRING_GEOMETRIC)
    return est, gt, normals, p


def _ctx(api, kw, est, gt=None, normals=None):
    c = api.MapEvalB200(**kw)
    c.set_cloud(EST, est)
    if gt is not None:
        c.set_cloud(GT, gt)
    if normals is not None:
        c.set_normals(EST, normals[0])
        c.set_normals(GT, normals[1])
    return c


def _world_two(rank, port, out_dir):
    """one rank of the job: every result through dist.py, pickled to out_dir/rank<r>.pkl"""
    import torch
    import torch.distributed as dist

    from cloud_map_evaluation_b200 import api
    from cloud_map_evaluation_b200 import dist as mdist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=2)
    try:
        dev = torch.device("cuda", 0)
        torch.cuda.set_device(dev)
        # the contexts' kernels and torch's collectives on one stream, as bench.py runs them: allreduce_block does not
        # synchronise the host
        stream = torch.cuda.Stream(device=dev)
        torch.cuda.set_stream(stream)
        kw = dict(device=0, rank=rank, world=2, stream=stream.cuda_stream)
        out = {}
        est, gt, normals, p = _nn_pair()
        with _ctx(api, kw, est, gt, normals) as c:
            c.accum_reset()
            c.eval_nn_accum_device(p)
            mdist.allreduce_block(c, dev)
            e, g, _ = c.accum_fetch(want_mme=(False, False))
            out["nn"] = A.struct_to_dict(c.nn_finalize(p, e, g))
            out["curve"] = api.curve_finalize(p, e, g, mdist.allreduce_curve(c, LEVELS, dev), LEVELS, len(est), len(gt))
            out["quantiles"] = {pop: mdist.quantiles_distributed(c, dev, PROBS, pop) for pop in TQ.POPS}
            out["regions"] = mdist.regions_distributed(c, REGION, dev)
            out["surface"] = mdist.surface_distributed(c, dev, knn=0)
        with _ctx(api, kw, *TD.scene(40000, 11)) as c:
            out["drift"] = mdist.drift_distributed(c, dev, *DRIFT)
        with _ctx(api, kw, TC._room(120_000, 9)) as c:
            out["consistency"] = mdist.consistency_distributed(c, dev, EST, TC.R0, 10, CONS_REGION)
        with _ctx(api, kw, TM._room(6)) as c:
            out["mom"] = mdist.mom_distributed(c, dev, EST, TM.R0, 10)
            out["mom_regions"] = mdist.mom_regions_distributed(c, dev, MOM_REGION)
        with _ctx(api, kw, *TI._pair(100_000, 120_000)) as c:
            T, reg = mdist.icp_distributed(c, dev, TI.R, TI.T0, method=A.ME_ICP_POINT_TO_POINT)
            out["icp"] = dict(T=T, reg=A.struct_to_dict(reg))
        with open(os.path.join(out_dir, f"rank{rank}.pkl"), "wb") as f:
            pickle.dump(out, f)
    finally:
        dist.destroy_process_group()


@pytest.fixture(scope="module")
def world_two(tmp_path_factory):
    import torch.multiprocessing as mp
    out_dir = tmp_path_factory.mktemp("world_two")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_world_two, args=(port, str(out_dir)), nprocs=2, join=True)
    ranks = []
    for r in range(2):
        with open(out_dir / f"rank{r}.pkl", "rb") as f:
            ranks.append(pickle.load(f))
    return ranks


@pytest.fixture(scope="module")
def world_one():
    """the same calls at world 1"""
    from cloud_map_evaluation_b200 import api
    out = {}
    est, gt, normals, p = _nn_pair()
    with _ctx(api, {}, est, gt, normals) as c:
        out["nn"] = A.struct_to_dict(c.calculateMetricsWithInitialMatrix(p))
        out["curve"] = c.accuracy_curve(LEVELS)
        out["quantiles"] = {pop: c.distance_quantiles(PROBS, pop) for pop in TQ.POPS}
        out["regions"] = c.region_errors(REGION)
        out["surface"] = c.surface_metrics(0)
    with _ctx(api, {}, *TD.scene(40000, 11)) as c:
        out["drift"] = c.region_drift(*DRIFT)
    with _ctx(api, {}, TC._room(120_000, 9)) as c:
        out["consistency"] = c.local_consistency(EST, TC.R0, 10, CONS_REGION)
    with _ctx(api, {}, TM._room(6)) as c:
        out["mom"] = c.mom(EST, TM.R0, 10)
        out["mom_regions"] = c.mom_regions(MOM_REGION)
    with _ctx(api, {}, *TI._pair(100_000, 120_000)) as c:
        T, reg = c.performICPRegistration(TI.R, TI.T0, method=A.ME_ICP_POINT_TO_POINT)
        out["icp"] = dict(T=T, reg=A.struct_to_dict(reg))
    return out


@pytest.mark.parametrize("rank", [0, 1])
def test_accumulator_block_and_curve(world_two, world_one, rank):
    got, ref = world_two[rank]["nn"], world_one["nn"]
    for d in TA.DIRS:
        for f in ("n_corr", "n_inlier", "n_source"):
            assert got[d][f] == ref[d][f], (d, f)
        for f in TA.FIELDS:
            np.testing.assert_allclose(got[d][f], ref[d][f], rtol=1e-9, atol=0, err_msg=f"{d} {f}")
    for f in ("cd", "f1", "iou", "full_cd"):
        np.testing.assert_allclose(got[f], ref[f], rtol=1e-9, atol=0, err_msg=f)
    got, ref = world_two[rank]["curve"], world_one["curve"]
    for d in TA.DIRS:
        assert list(got[d]["n_inlier"]) == list(ref[d]["n_inlier"]), d
        for f in TA.FIELDS:
            TA._close(got[d][f], ref[d][f], 1e-11)
    for f in ("cd", "f1", "iou"):
        TA._close(got[f], ref[f], 1e-11)


@pytest.mark.parametrize("rank", [0, 1])
def test_quantiles(world_two, world_one, rank):
    for pop in TQ.POPS:
        TQ._same(world_two[rank]["quantiles"][pop], world_one["quantiles"][pop])


@pytest.mark.parametrize("rank", [0, 1])
def test_regions(world_two, world_one, rank):
    TR.check_table(world_two[rank]["regions"], world_one["regions"])


@pytest.mark.parametrize("rank", [0, 1])
def test_surface(world_two, world_one, rank):
    TS.check_result(world_two[rank]["surface"], world_one["surface"])


@pytest.mark.parametrize("rank", [0, 1])
def test_drift(world_two, world_one, rank):
    got, ref = world_two[rank]["drift"], world_one["drift"]
    for k in ("index", "n_est", "n_corr_before", "n_corr", "iterations", "status"):
        assert np.array_equal(got[k], ref[k]), k
    np.testing.assert_allclose(got["T"], ref["T"], rtol=0, atol=1e-9)


@pytest.mark.parametrize("rank", [0, 1])
def test_consistency(world_two, world_one, rank):
    got, ref = world_two[rank]["consistency"], world_one["consistency"]
    assert len(ref["index"]) > 1
    TC._same(got, ref)


@pytest.mark.parametrize("rank", [0, 1])
def test_mom_and_regions(world_two, world_one, rank):
    got, ref = world_two[rank]["mom"], world_one["mom"]
    assert ref["status"] == "OK" and got["status"] == ref["status"]
    for f in ("n", "n_planar", "n_query", "n_pv"):
        assert np.array_equal(got[f], ref[f]), f
    assert np.array_equal(TM._bits(got["axis"]), TM._bits(ref["axis"]))
    for f in ("mean", "median", "mom"):
        np.testing.assert_allclose(got[f], ref[f], rtol=1e-12, atol=0, err_msg=f)
    got, ref = world_two[rank]["mom_regions"], world_one["mom_regions"]
    assert (ref["status"] == "OK").any()
    for f in ("index", "n_points", "n_planar", "n"):
        assert np.array_equal(got[f], ref[f]), f
    assert list(got["status"]) == list(ref["status"])
    has = ref["n"] > 0
    for f in ("mean", "median"):
        np.testing.assert_allclose(got[f][has], ref[f][has], rtol=1e-12, atol=0, err_msg=f)


@pytest.mark.parametrize("rank", [0, 1])
def test_icp_point_to_point(world_two, world_one, rank):
    got, ref = world_two[rank]["icp"], world_one["icp"]
    g, r = got["reg"], ref["reg"]
    assert (g["iterations"], g["converged"], g["n_corr"]) == (r["iterations"], r["converged"], r["n_corr"])
    np.testing.assert_allclose(got["T"], ref["T"], rtol=0, atol=1e-10)
    np.testing.assert_allclose([g["fitness"], g["inlier_rmse"]], [r["fitness"], r["inlier_rmse"]], rtol=1e-9)

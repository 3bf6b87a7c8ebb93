"""N > 1 host logic on CPU: world_size-2 (and 3) gloo processes each own a shard of the queries, build the partial
accumulators for it, all-reduce them and finalise with the library's host-only me_nn_finalize / me_mme_finalize.  The
result must equal the unsharded oracle run (counts exactly)."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import _lib, synth
from cloud_map_evaluation_b200 import dist as mdist


def _partial_nn(query, ref, qb, qe, tau, R, slot=None):
    from oracle import oracle as O
    a = A.me_nn_accum()
    q = query[qb:qe]
    a.n_query = len(q)
    if len(q) == 0:
        return a
    idx, d2 = O.knn1(q, ref)
    keep = d2 <= R
    d = q[keep] - ref[idx[keep]]
    sq = d[:, 0] ** 2 + (d[:, 1] ** 2 + d[:, 2] ** 2)
    nd = np.sqrt(sq)
    a.n_corr = int(keep.sum())
    for k, t in enumerate(tau):
        m = nd <= t
        a.n_inlier[k], a.sum_d[k], a.sum_d2[k] = int(m.sum()), float(nd[m].sum()), float(sq[m].sum())
    a.sum_d_all, a.sum_d2_all, a.sum_nn_dist = float(nd.sum()), float(sq.sum()), float(np.sqrt(d2).sum())
    if slot is not None and len(nd):      # this rank's (n, mean, M2), the other slots stay 0: the SUM gathers them
        a.rank_n[slot], a.rank_mean[slot] = len(nd), float(nd.mean())
        a.rank_m2[slot] = float(((nd - nd.mean()) ** 2).sum())
    return a


def _allreduce(nn_e, nn_g, m):
    """the partial accumulators of every rank, reduced in place: SUM of each NN struct's int64 and fp64 fields and of the MME
    counts and entropy sum, MAX / MIN of the entropy extrema"""
    def field_sum(ctype, n, obj, offset=0):
        dist.all_reduce(torch.from_numpy(np.ctypeslib.as_array((ctype * n).from_buffer(obj, offset))))
    for a in (nn_e, nn_g):
        field_sum(C.c_int64, A.ME_NN_ACCUM_I64, a)
        field_sum(C.c_double, A.ME_NN_ACCUM_F64, a, 8 * A.ME_NN_ACCUM_I64)
    field_sum(C.c_int64, 2, m)
    t = torch.tensor([m.sum_entropy, m.min_entropy, m.max_entropy], dtype=torch.float64)
    for op, sl in ((dist.ReduceOp.SUM, t[0:1]), (dist.ReduceOp.MIN, t[1:2]), (dist.ReduceOp.MAX, t[2:3])):
        dist.all_reduce(sl, op=op)
    m.sum_entropy, m.min_entropy, m.max_entropy = t.tolist()


def _worker(rank, world, port, out_dir, moments=False):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle import oracle as O
        L = _lib.load()
        est, gt, cfg = synth.make_pair("C1", scale=0.08)
        tau = cfg["tau"]
        p = A.make_nn_params(tau, 1.0, pairing=A.ME_PAIRING_GEOMETRIC)
        eb, ee = mdist.shard_range(len(est), rank, world)
        gb, ge = mdist.shard_range(len(gt), rank, world)
        slot = rank if moments else None
        nn_e = _partial_nn(est, gt, eb, ee, tau, 1.0, slot)
        nn_g = _partial_nn(gt, est, gb, ge, tau, 1.0, slot)
        # MME partial: entropies of this rank's points from the oracle's per-point output
        _, ent = O.eval_mme(est, 0.1, 10, want_entropies=True)
        mine = ent[eb:ee]
        m = A.me_mme_accum()
        nz = mine[mine != 0]
        m.n_query, m.n_valid, m.sum_entropy = len(mine), int((mine != 0).sum()), float(mine.sum())
        m.min_entropy, m.max_entropy = (float(nz.min()), float(nz.max())) if len(nz) else (np.inf, -np.inf)
        _allreduce(nn_e, nn_g, m)
        res = A.me_nn_result()
        assert L.me_nn_finalize(C.byref(p), C.byref(nn_e), C.byref(nn_g), len(est), len(gt), C.byref(res)) == 0
        mres = A.me_mme_result()
        assert L.me_mme_finalize(C.byref(m), len(est), C.byref(mres)) == 0
        if rank == 0:
            exp = O.eval_nn(est, gt, p)
            emme = O.eval_mme(est, 0.1, 10)
            assert nn_e.n_query == len(est) and nn_g.n_query == len(gt)
            if moments:
                assert sum(nn_e.rank_n) == nn_e.n_corr and sum(nn_g.rank_n) == nn_g.n_corr
            for d in ("est_to_gt", "gt_to_est"):
                g, e = getattr(res, d), getattr(exp, d)
                assert list(g.n_inlier) == list(e.n_inlier) and g.n_corr == e.n_corr
                for k in ("mean", "rmse", "fitness", "sigma"):
                    np.testing.assert_allclose(list(getattr(g, k)), list(getattr(e, k)), rtol=1e-9)
            np.testing.assert_allclose(res.full_cd, exp.full_cd, rtol=1e-12)
            assert mres.n_valid == emme.n_valid
            np.testing.assert_allclose([mres.mme, mres.min_abs_entropy, mres.max_abs_entropy],
                                       [emme.mme, emme.min_abs_entropy, emme.max_abs_entropy], rtol=1e-12)
            open(os.path.join(out_dir, "ok"), "w").write("ok")
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_partials_finalize_to_the_unsharded_result_gloo(world, tmp_path):
    """partial accumulators of each rank's shard, summed over the ranks: me_nn_finalize / me_mme_finalize give the
    unsharded result"""
    assert mdist.shard_range(10, 0, 3) == (0, 3) and mdist.shard_range(10, 2, 3) == (6, 10)
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    from oracle import oracle as O
    O.build()
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    assert os.path.exists(tmp_path / "ok")



@pytest.mark.parametrize("world", [2, 3])
def test_sharded_moment_slots_merge_in_finalize_gloo(world, tmp_path):
    """the per-rank (n, mean, M2) slots through the same SUM over the ranks: me_nn_finalize merges them into sigma"""
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    from oracle import oracle as O
    O.build()
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_worker, args=(world, port, str(tmp_path), True), nprocs=world, join=True)
    assert os.path.exists(tmp_path / "ok")


# ---------------------------------------------------------------------------------------------------------------
# Slab layout on CPU: the decomposition the voxel stage uses across ranks (DESIGN §4) — every voxel layer has one owner
# (me_plan_slab_cut), an owner computes the Gaussians / W of its layers from the points that fall into them, the W table is
# MAX-all-reduced (-1 = no pair) so that SCS sees the neighbours' voxels, and eight counters / sums are SUM-all-reduced.
# Here the per-rank compute is the oracle (CPU) and the collectives are gloo; the reduced result must equal calculateVMD
# on the whole clouds.
# ---------------------------------------------------------------------------------------------------------------
def _plan_on_cpu(est, v, m, world):
    """plane histograms of the estimated cloud along y and z (cells of v / m), as plan_slabs reduces them on the device"""
    L = _lib.load()
    k_lo = np.floor(est.min(0) / v).astype(np.int64)
    nvox = np.floor(est.max(0) / v).astype(np.int64) - k_lo + 1
    cell = np.floor((est - k_lo * v) / (v / m)).astype(np.int64)
    cell = np.minimum(np.maximum(cell, 0), nvox * m - 1)
    py = np.bincount(cell[:, 1], minlength=int(nvox[1] * m)).astype(np.uint64)
    pz = np.bincount(cell[:, 2], minlength=int(nvox[2] * m)).astype(np.uint64)
    axis, share = C.c_int32(0), C.c_double(0)
    b = (C.c_int32 * (world + 1))()
    u64 = C.POINTER(C.c_uint64)
    assert L.me_plan_slab_cut(py.ctypes.data_as(u64), len(py), pz.ctypes.data_as(u64), len(pz), m, world, 4, C.byref(axis), b,
                              C.byref(share)) == 0
    return axis.value, [int(k_lo[axis.value]) + x for x in b], k_lo, nvox


def _slab_worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle import oracle as O
        est, gt, cfg = synth.make_pair("C2", scale=0.2)
        v, radius, min_points = cfg["vmd_voxel_size"], 5, 20
        axis, kb, k_lo, nvox = _plan_on_cpu(est, v, 4, world)
        assert axis in (1, 2)
        lo = kb[rank] if rank > 0 else -(1 << 40)
        hi = kb[rank + 1] if rank < world - 1 else (1 << 40)
        own = lambda c: c[(np.floor(c[:, axis] / v) >= lo) & (np.floor(c[:, axis] / v) < hi)]      # noqa: E731
        e_own, g_own = own(est), own(gt)
        # W table over the estimated cloud's voxels, -1 = no pair (the all-reducible encoding)
        w_tab = torch.full(tuple(int(x) for x in nvox), -1.0, dtype=torch.float64)
        part = np.zeros(8)
        keys = np.zeros((0, 3), np.int64)
        if len(e_own) and len(g_own):
            r, rows = O.eval_awd(e_own, g_own, v, min_points, radius, want_rows=True)
            keys = np.rint(rows[:, 0:3] / v).astype(np.int64) - k_lo
            w_tab[keys[:, 0], keys[:, 1], keys[:, 2]] = torch.from_numpy(rows[:, 9].copy())
            part[:] = [r.n_pairs, 0, r.n_voxels_est, r.n_voxels_gt, r.n_active, r.n_new, rows[:, 9].sum(), 0.0]
        elif len(e_own):
            part[2] = part[5] = len(O.voxel_map(e_own, v)[0])
        elif len(g_own):
            part[3] = len(O.voxel_map(g_own, v)[0])
        dist.all_reduce(w_tab, op=dist.ReduceOp.MAX)
        # SCS over this rank's pairs on the merged table (map_eval.cpp:351-387)
        w = w_tab.numpy()
        pad = np.full(tuple(s + 2 * radius for s in w.shape), -1.0)
        pad[radius:-radius, radius:-radius, radius:-radius] = w
        for k in keys:
            nb = pad[k[0]:k[0] + 2 * radius + 1, k[1]:k[1] + 2 * radius + 1, k[2]:k[2] + 2 * radius + 1].copy()
            nb[radius, radius, radius] = -1.0
            nb = nb[nb >= 0]
            if len(nb):
                part[1] += 1
                part[7] += np.sqrt(((nb - nb.mean()) ** 2).mean()) / nb.mean()
        blk = torch.from_numpy(part)
        dist.all_reduce(blk)
        if rank == 0:
            exp = O.eval_awd(est, gt, v, min_points, radius)
            got = blk.numpy()
            assert [int(got[0]), int(got[1]), int(got[2]), int(got[3]), int(got[4]), int(got[5])] == \
                [exp.n_pairs, exp.n_scs, exp.n_voxels_est, exp.n_voxels_gt, exp.n_active, exp.n_new]
            assert int(got[3]) - int(got[4]) == exp.n_old
            assert exp.n_pairs > 100 and exp.n_scs > 100
            np.testing.assert_allclose([got[6] / got[0], got[7] / got[1]], [exp.awd, exp.scs], rtol=1e-12)
            open(os.path.join(out_dir, "ok"), "w").write("ok")
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_slab_voxel_stage_decomposition_gloo(world, tmp_path):
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    from oracle import oracle as O
    O.build()
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_slab_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    assert os.path.exists(tmp_path / "ok")

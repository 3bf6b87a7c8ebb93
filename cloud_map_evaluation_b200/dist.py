"""Multi-GPU plumbing: one process per GPU; the evaluated cloud's query ranges sharded by rank with both lattices laid out whole
(replicated layout), or every rank laying out and evaluating only its voxel layers (slab layout, MapEvalB200.set_layout); ONE
all-reduce of the sum-reducible accumulators (plus a MAX pair for the entropy extrema; on a slab layout a MAX all-reduce of
the voxel stage's W table).

The reference is single-process (SURVEY.md §5); this is the H100-native equivalent of its TBB/OpenMP reductions
(map_eval.cpp:1411,1420,1704-1708).  torch.distributed is used for the collectives only: backend "nccl" on GPUs
(NVLink / NVSwitch), "gloo" in the CPU tests.
"""
from . import _abi as A

_NN_I = A.ME_NN_ACCUM_I64
_NN_F = A.ME_NN_ACCUM_F64


def pack(nn_e, nn_g, mme_list):
    """Flatten the accumulators into (int64 list, fp64 list, min list, max list)."""
    ints, flts, mins, maxs = [], [], [], []
    for a in (nn_e, nn_g):
        ints += [a.n_query, a.n_corr] + list(a.n_inlier) + [a.n_ub, a.n_far]
        flts += list(a.sum_d) + list(a.sum_d2) + [a.sum_d_all, a.sum_d2_all, a.sum_nn_dist] + list(a.rank_n) + list(a.rank_mean) + list(a.rank_m2)
    for m in mme_list:
        ints += [m.n_query, m.n_valid]
        flts += [m.sum_entropy]
        mins.append(m.min_entropy)
        maxs.append(m.max_entropy)
    return ints, flts, mins, maxs


def unpack(ints, flts, mins, maxs, nn_e, nn_g, mme_list):
    ii = fi = 0
    for a in (nn_e, nn_g):
        a.n_query, a.n_corr = int(ints[ii]), int(ints[ii + 1])
        for k in range(5):
            a.n_inlier[k] = int(ints[ii + 2 + k])
        a.n_ub, a.n_far = int(ints[ii + 7]), int(ints[ii + 8])
        ii += _NN_I
        for k in range(5):
            a.sum_d[k] = float(flts[fi + k])
            a.sum_d2[k] = float(flts[fi + 5 + k])
        a.sum_d_all, a.sum_d2_all, a.sum_nn_dist = float(flts[fi + 10]), float(flts[fi + 11]), float(flts[fi + 12])
        W = A.ME_MAX_WORLD
        for r in range(W):
            a.rank_n[r] = float(flts[fi + 13 + r])
            a.rank_mean[r] = float(flts[fi + 13 + W + r])
            a.rank_m2[r] = float(flts[fi + 13 + 2 * W + r])
        fi += _NN_F
    for j, m in enumerate(mme_list):
        m.n_query, m.n_valid = int(ints[ii]), int(ints[ii + 1])
        ii += 2
        m.sum_entropy = float(flts[fi])
        fi += 1
        m.min_entropy, m.max_entropy = float(mins[j]), float(maxs[j])


def allreduce_accumulators(nn_e, nn_g, mme_list, device=None, group=None):
    """In-place all-reduce of the partial accumulators of every rank: ONE SUM all-reduce over the whole block (the
    integer counts ride along as fp64 — they stay below 2^53, so their sum is exact and order-independent: the reduced
    inlier counts are bit-exact for any world size; fp64 sums differ from the 1-GPU run by rounding only), plus one MAX
    all-reduce over [max entropy, -min entropy] when MME was evaluated (map_eval.cpp:697-701)."""
    import torch
    import torch.distributed as dist
    ints, flts, mins, maxs = pack(nn_e, nn_g, mme_list)
    assert all(abs(v) < 2 ** 53 for v in ints)
    t = torch.tensor([float(v) for v in ints] + flts, dtype=torch.float64, device=device)
    dist.all_reduce(t, group=group)
    out = t.cpu().tolist()
    ri, rf = [int(round(v)) for v in out[:len(ints)]], out[len(ints):]
    rmin, rmax = [], []
    if mins:
        tx = torch.tensor(list(maxs) + [-v for v in mins], dtype=torch.float64, device=device)
        dist.all_reduce(tx, op=dist.ReduceOp.MAX, group=group)
        ox = tx.cpu().tolist()
        rmax, rmin = ox[:len(maxs)], [-v for v in ox[len(maxs):]]
    unpack(ri, rf, rmin, rmax, nn_e, nn_g, mme_list)


def shard_range(n, rank, world):
    """The contiguous range a rank owns — the same rule as libmapeval_b200 (common.cuh shard_range)."""
    return n * rank // world, n * (rank + 1) // world


class _DeviceBlock:
    """zero-copy view of a raw device pointer for torch.as_tensor (CUDA array interface)"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (int(ptr), False), "version": 2}


def allreduce_block(ctx, device, group=None):
    """All-reduce the context's device-resident accumulator block in place: ONE SUM all-reduce over the sum-reducible
    values (counts ride as fp64, exact) and one MAX all-reduce over the entropy extrema — NCCL over NVLink / NVSwitch, no
    host round trip; the caller fetches the block afterwards (MapEvalB200.accum_fetch)."""
    import torch
    import torch.distributed as dist
    ptr, n_sum, n_max = ctx.accum_block()
    t = torch.as_tensor(_DeviceBlock(ptr, n_sum + n_max), device=device)
    dist.all_reduce(t[:n_sum], group=group)
    dist.all_reduce(t[n_sum:], op=dist.ReduceOp.MAX, group=group)


def allreduce_curve(ctx, tau, device, group=None):
    """The accuracy curve block of every rank at the levels tau (MapEvalB200.curve_accum_device), SUM-all-reduced in place
    on the device (counts ride as fp64, exact), returned as a host numpy array for api.curve_finalize, which every rank
    then runs with its reduced NN accumulators."""
    import torch
    import torch.distributed as dist
    ptr, n = ctx.curve_accum_device(tau)
    ctx.synchronize()
    t = torch.as_tensor(_DeviceBlock(ptr, n), device=device)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, group=group)
    return t.cpu().numpy().copy()


def quantiles_distributed(ctx, device, p, population=A.ME_DIST_KEPT, group=None):
    """Exact distance quantiles of the last NN evaluation over every rank of the job (MapEvalB200.distance_quantiles for
    world > 1): the selection loop with ONE in-place SUM all-reduce of the pass's integer counts (as fp64, exact) per pass.
    Every rank reads the same reduced counts, so every rank returns the same result."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    ctx.quantile_begin(p, population)
    done = False
    while not done:
        if world > 1:
            ptr, n = ctx.quantile_block()
            ctx.synchronize()
            dist.all_reduce(torch.as_tensor(_DeviceBlock(ptr, n), device=device), group=group)
            torch.cuda.current_stream(device).synchronize()
        done = ctx.quantile_step()
    return ctx.quantile_end()


def icp_distributed(ctx, device, max_correspondence_distance, T_init=None, max_iteration=30, relative_fitness=1e-6,
                    relative_rmse=1e-6, method=A.ME_ICP_GENERALIZED, group=None):
    """performICPRegistration on every rank of the job (map_eval.cpp:1366-1394): the clouds are replicated, every rank
    sweeps its query range and estimates its slice of the missing k-NN normals.  One in-place all-gather per estimated
    cloud, then ONE SUM all-reduce of the 17 / 29-value block per iteration; every rank applies the same update to the same
    reduced doubles, so T is identical everywhere.  Returns (T 4x4, me_icp_result) like performICPRegistration; the
    estimated cloud held by ctx is the original transformed by T."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    assert (rank, world) == (ctx.rank, ctx.world), "the context's shard must be this process's rank in the group"

    def _torch_waits_for_ctx():
        ctx.synchronize()

    def _ctx_waits_for_torch():
        torch.cuda.current_stream(device).synchronize()

    ctx.icp_begin(max_correspondence_distance, T_init, max_iteration, relative_fitness, relative_rmse, method)
    for which in (A.ME_CLOUD_EST, A.ME_CLOUD_GT):
        ptr, s, pending = ctx.icp_normals_slice(which)
        if pending:
            _torch_waits_for_ctx()
            buf = torch.as_tensor(_DeviceBlock(ptr, world * s * 3), device=device)
            dist.all_gather_into_tensor(buf, buf[rank * s * 3:(rank + 1) * s * 3], group=group)
            _ctx_waits_for_torch()
    done = False
    ptr, n_sum = ctx.icp_block()
    blk = torch.as_tensor(_DeviceBlock(ptr, n_sum), device=device)
    while not done:
        if world > 1:
            _torch_waits_for_ctx()
            dist.all_reduce(blk, group=group)
            _ctx_waits_for_torch()
        done = ctx.icp_step()
    return ctx.icp_end()


def allreduce_voxel_w(ctx, device, group=None):
    """Slab layout, between MapEvalB200.voxel_begin and voxel_finish_accum_device: MAX-all-reduce of the W table over the
    estimated cloud's voxels in place (-1 = no pair; every voxel has one owner), so that the SCS sweep of every rank sees
    the W of the neighbouring ranks' voxels."""
    import torch
    import torch.distributed as dist
    ptr, n = ctx.voxel_w_table()
    if n > 0:
        dist.all_reduce(torch.as_tensor(_DeviceBlock(ptr, n), device=device), op=dist.ReduceOp.MAX, group=group)

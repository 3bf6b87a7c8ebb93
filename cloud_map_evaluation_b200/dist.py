"""Multi-GPU plumbing: one process per GPU; the evaluated cloud's query ranges sharded by rank with both lattices laid out whole
(replicated layout), or every rank laying out and evaluating only its voxel layers (slab layout, MapEvalB200.set_layout); ONE
in-place all-reduce of the device accumulator block's sum-reducible values (plus a MAX all-reduce of its entropy extrema;
on a slab layout a MAX all-reduce of the voxel stage's W table).  allreduce_block is the one way to reduce accumulators:
the *_accum_device sweeps fill the block, accum_fetch decodes it.

The reference is single-process (SURVEY.md §5); this is the H100-native equivalent of its TBB/OpenMP reductions
(map_eval.cpp:1411,1420,1704-1708).  torch.distributed is used for the collectives only: backend "nccl" on GPUs
(NVLink / NVSwitch), "gloo" in the CPU tests.
"""
from . import _abi as A


def shard_range(n, rank, world):
    """The contiguous range a rank owns — the same rule as libmapeval_b200 (common.cuh shard_range)."""
    return n * rank // world, n * (rank + 1) // world


class _DeviceBlock:
    """zero-copy view of a raw device pointer for torch.as_tensor (CUDA array interface)"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (int(ptr), False), "version": 2}


def _world(group):
    """(rank, world) of this process in the group; (0, 1) without torch.distributed"""
    import torch.distributed as dist
    if not dist.is_initialized():
        return 0, 1
    return dist.get_rank(group), dist.get_world_size(group)


def _reduce(ctx, ptr, n_sum, n_max, device, group=None, sync=True):
    """All-reduce a device block the context owns, in place: SUM over its first n_sum values (counts ride as fp64, exact),
    MAX over the next n_max; on one rank there is nothing to reduce.  sync: the collectives wait for the context's stream
    and torch's stream is synchronised after them; without it the caller orders both on one stream.  Returns the block as
    a tensor (None when it is empty)."""
    import torch
    import torch.distributed as dist
    if n_sum + n_max == 0:
        return None
    t = torch.as_tensor(_DeviceBlock(ptr, n_sum + n_max), device=device)
    if _world(group)[1] == 1:
        return t
    if sync:
        ctx.synchronize()
    if n_sum > 0:
        dist.all_reduce(t[:n_sum], group=group)
    if n_max > 0:
        dist.all_reduce(t[n_sum:], op=dist.ReduceOp.MAX, group=group)
    if sync:
        torch.cuda.current_stream(device).synchronize()
    return t


def _gather_normals(ctx, slice_fn, device, group=None):
    """The all-gather of the working normals: for each cloud whose slices are pending (this rank filled rows
    [rank * slice, (rank + 1) * slice) of the world * slice * 3 fp64 buffer), ONE in-place all-gather"""
    import torch
    import torch.distributed as dist
    rank, world = _world(group)
    for which in (A.ME_CLOUD_EST, A.ME_CLOUD_GT):
        ptr, s, pending = slice_fn(which)
        if pending:
            ctx.synchronize()
            buf = torch.as_tensor(_DeviceBlock(ptr, world * s * 3), device=device)
            dist.all_gather_into_tensor(buf, buf[rank * s * 3:(rank + 1) * s * 3], group=group)
            torch.cuda.current_stream(device).synchronize()


def allreduce_block(ctx, device, group=None):
    """All-reduce the context's device-resident accumulator block in place: ONE SUM all-reduce over the sum-reducible
    values (counts ride as fp64, exact) and one MAX all-reduce over the entropy extrema — NCCL over NVLink / NVSwitch, no
    host round trip (order the context's and torch's work on one stream); the caller fetches the block afterwards
    (MapEvalB200.accum_fetch)."""
    _reduce(ctx, *ctx.accum_block(), device, group, sync=False)


def allreduce_curve(ctx, tau, device, group=None):
    """The accuracy curve block of every rank at the levels tau (MapEvalB200.curve_accum_device), SUM-all-reduced in place
    on the device (counts ride as fp64, exact), returned as a host numpy array for api.curve_finalize, which every rank
    then runs with its reduced NN accumulators."""
    ptr, n = ctx.curve_accum_device(tau)
    ctx.synchronize()
    return _reduce(ctx, ptr, n, 0, device, group, sync=False).cpu().numpy().copy()


def regions_distributed(ctx, region_size, device, group=None):
    """AC / COM / CD / F1 / IoU per region over every rank of the job (MapEvalB200.region_errors for world > 1): every rank
    lists the same occupied regions and folds its own records, then ONE in-place SUM all-reduce of the block's sums (counts
    ride as fp64, exact) and ONE MAX all-reduce of its maxima.  Every rank returns the same table."""
    n = ctx.region_begin(region_size)
    _reduce(ctx, *ctx.region_block(), device, group)
    return ctx.region_end(n)


def surface_distributed(ctx, device, knn=0, group=None):
    """Point-to-plane metrics and normal consistency over every rank of the job (MapEvalB200.surface_metrics for world > 1):
    every rank estimates its caller-index slice of a cloud's missing working normals, ONE in-place all-gather per such cloud,
    then every rank folds its own records, ONE in-place SUM all-reduce of the block's sums (counts ride as fp64, exact) and
    ONE MAX all-reduce of its maxima.  Every rank returns the same result."""
    ctx.surface_begin(knn)
    _gather_normals(ctx, ctx.surface_normals_slice, device, group)
    _reduce(ctx, *ctx.surface_block(), device, group)
    return ctx.surface_end()


def consistency_distributed(ctx, device, which, radius, min_neighbors=10, region_size=0.0, group=None):
    """Local map consistency over every rank of the job (MapEvalB200.local_consistency for world > 1): every rank sweeps its
    query range of the replicated cloud and folds it by region, then ONE in-place SUM all-reduce of the block's sums (counts
    ride as fp64, exact) and ONE MAX all-reduce of its maxima.  Every rank returns the same result."""
    n = ctx.consistency_begin(which, radius, min_neighbors, region_size)
    _reduce(ctx, *ctx.consistency_block(), device, group)
    return ctx.consistency_end(n)


def mom_distributed(ctx, device, which, radius, min_neighbors=10, angle_deg=10.0, planarity=0.5, min_family=100, group=None):
    """The mutually orthogonal metric over every rank of the job (MapEvalB200.mom for world > 1): every rank sweeps its
    query range of the replicated cloud, then ONE in-place SUM all-reduce per pass: the direction histogram, the family
    fold with the medians' first digit, then the selection's later digits (counts ride as fp64, exact).  Every rank
    returns the same result."""
    ctx.mom_begin(which, radius, min_neighbors, angle_deg, planarity, min_family)
    done = False
    while not done:
        _reduce(ctx, *ctx.mom_block(), 0, device, group)
        done = ctx.mom_step()
    return ctx.mom_end()


def mom_regions_distributed(ctx, device, region_size, min_family=None, group=None):
    """The last finished MOM call per region over every rank of the job (MapEvalB200.mom_regions for world > 1): every rank
    writes the points it swept into the block [v | code], ONE in-place SUM all-reduce gathers them exactly (x + 0 = x), and
    every rank runs the same segmented selection on the same bits, so every rank returns the same rows."""
    n = ctx.mom_region_begin(region_size, min_family)
    _reduce(ctx, *ctx.mom_region_block(), 0, device, group)
    return ctx.mom_region_end(n)


def quantiles_distributed(ctx, device, p, population=A.ME_DIST_KEPT, group=None):
    """Exact distance quantiles of the last NN evaluation over every rank of the job (MapEvalB200.distance_quantiles for
    world > 1): the selection loop with ONE in-place SUM all-reduce of the pass's integer counts (as fp64, exact) per pass.
    Every rank reads the same reduced counts, so every rank returns the same result."""
    ctx.quantile_begin(p, population)
    done = False
    while not done:
        _reduce(ctx, *ctx.quantile_block(), 0, device, group)
        done = ctx.quantile_step()
    return ctx.quantile_end()


def icp_distributed(ctx, device, max_correspondence_distance, T_init=None, max_iteration=30, relative_fitness=1e-6,
                    relative_rmse=1e-6, method=A.ME_ICP_GENERALIZED, group=None):
    """performICPRegistration on every rank of the job (map_eval.cpp:1366-1394): the clouds are replicated, every rank
    sweeps its query range and estimates its slice of the missing k-NN normals.  One in-place all-gather per estimated
    cloud, then ONE SUM all-reduce of the 17 / 29-value block per iteration; every rank applies the same update to the same
    reduced doubles, so T is identical everywhere.  Returns (T 4x4, me_icp_result) like performICPRegistration; the
    estimated cloud held by ctx is the original transformed by T."""
    assert _world(group) == (ctx.rank, ctx.world), "the context's shard must be this process's rank in the group"
    ctx.icp_begin(max_correspondence_distance, T_init, max_iteration, relative_fitness, relative_rmse, method)
    _gather_normals(ctx, ctx.icp_normals_slice, device, group)
    ptr, n_sum = ctx.icp_block()
    done = False
    while not done:
        _reduce(ctx, ptr, n_sum, 0, device, group)
        done = ctx.icp_step()
    return ctx.icp_end()


def drift_distributed(ctx, device, region_size, max_correspondence_distance, max_iteration=30, relative_fitness=1e-6,
                      relative_rmse=1e-6, group=None):
    """The drift per region on every rank of the job (MapEvalB200.region_drift for world > 1): the clouds are replicated,
    every rank lists the same regions and folds the pairs of its query range, then ONE in-place SUM all-reduce of the
    17-value block per region per iteration; every rank applies the same updates to the same reduced doubles, so every rank
    returns the same rows."""
    n = ctx.drift_begin(region_size, max_correspondence_distance, max_iteration, relative_fitness, relative_rmse)
    ptr, n_sum = ctx.drift_block()
    done = False
    while not done:
        _reduce(ctx, ptr, n_sum, 0, device, group)
        done = ctx.drift_step()
    return ctx.drift_end(n)


def allreduce_voxel_w(ctx, device, group=None):
    """Slab layout, between MapEvalB200.voxel_begin and voxel_finish_accum_device: MAX-all-reduce of the W table over the
    estimated cloud's voxels in place (-1 = no pair; every voxel has one owner), so that the SCS sweep of every rank sees
    the W of the neighbouring ranks' voxels."""
    ptr, n = ctx.voxel_w_table()
    _reduce(ctx, ptr, 0, n, device, group, sync=False)


def w2_distributed(ctx, device, voxel_size, min_points=100, scs_radius=5, group=None):
    """The Gaussian 2-Wasserstein stage over every rank of the job (MapEvalB200.voxel_w2 for world > 1).  On a replicated
    layout every rank computes the whole stage, with no collective.  On a slab layout every rank computes the voxels it
    owns, then ONE in-place MAX all-reduce of the W2 table (-1 = no pair; every voxel has one owner), the SCS sweep over
    its pairs, and ONE in-place SUM all-reduce of the stage's block (counts ride as fp64, exact).  Every rank returns the
    same result."""
    ctx.w2_begin(voxel_size, min_points)
    if ctx.layout_active()["layout"] != A.ME_LAYOUT_SLAB:
        ctx.w2_finish_accum_device(scs_radius)
        return ctx.w2_fetch()
    ptr, n = ctx.w2_w_table()
    _reduce(ctx, ptr, 0, n, device, group)
    ctx.w2_finish_accum_device(scs_radius)
    _reduce(ctx, *ctx.w2_block(), 0, device, group)
    return ctx.w2_fetch()

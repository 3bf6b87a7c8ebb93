// mom_region.cu — the mutually orthogonal metric per region (me_mom_region_*, DESIGN §3.17): the last finished MOM call's
// family medians, counts and means split by the region floor(x / s), without a new sweep.
//
// Begin, on every rank:
//   list_regions + region_ids (region.cu)  the occupied list (est ++ gt, or est alone) and the region of every point of the cloud
//   mom_region_fill_kernel                 the block [v | code] of this rank's points (zeros elsewhere): one SUM all-reduce
//                                          gathers every rank's points exactly (x + 0 = x)
// End, the same work on every rank from the reduced block:
//   mom_region_keys_kernel                 per family member the pair (v bits, segment rid * 3 + j), compacted in any order;
//                                          integer counts per segment and planar points per region (warp-aggregated atomics)
//   radix_sort_pairs (sort.cu)             stable by v (63 bits: v >= +0 orders like its bit pattern)
//   mom_region_segkey_kernel               (segment, position) of every sorted pair
//   radix_sort_pairs                       stable by segment (< 3 * 2^21, at most 23 bits): each segment's members contiguous,
//                                          ascending in v
//   exclusive_scan_inplace                 the segments' offsets from their counts
//   mom_region_select_kernel               per segment the median's two order statistics and their lerp (quantile_rank /
//                                          quantile_lerp, the host's definition), and its chunks of kRegionChunk members
//   mom_region_fold_kernel                 one warp per chunk: lane l adds the chunk's members l, l + 32, ...; a fixed shuffle tree
//   mom_region_merge_kernel                one thread per segment adds its chunks in chunk order
// The members' order inside a segment is their v order, so the selected values and the sums do not depend on the order in
// which the compaction placed equal keys: every rank, and every call on the same block, gives the same bits.  No
// floating-point atomics.  Compiled with -fmad=false, so the lerp rounds as numpy's does.
#include "common.cuh"
#include "radix.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace me {

static constexpr int kThreads = 256;
static constexpr int kCodeNoFamily = 4;    // a planar point without a family
enum : uint8_t { kPlanar = 4 };            // mom.cu's flag byte: 4 planar, family + 1 in bits 3..4

__global__ void __launch_bounds__(kThreads) mom_region_fill_kernel(long long n, const double *__restrict__ v,
                                                                   const uint8_t *__restrict__ flag, double *__restrict__ blk) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint8_t f = __ldg(flag + i);
    const int code = (f & kPlanar) ? ((f >> 3) ? (f >> 3) : kCodeNoFamily) : 0;
    blk[i] = code ? __ldg(v + i) : 0.0;
    blk[n + i] = (double)code;
  }
}

struct RegionCounts {
  uint32_t *seg;       // members per segment (3 R, then 0 for the scan)
  uint32_t *planar;    // planar points per region (R)
  uint32_t *members;   // the compaction's counter
};

// one thread per point of the reduced block; the whole warp calls the warp-aggregated steps
__global__ void __launch_bounds__(kThreads) mom_region_keys_kernel(long long n, const double *__restrict__ blk,
                                                                   const uint32_t *__restrict__ rid, RegionCounts C,
                                                                   unsigned long long *__restrict__ keys, uint32_t *__restrict__ vals) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long base = (long long)blockIdx.x * kThreads; base < n; base += stride) {   // warp-uniform bound
    const long long i = base + threadIdx.x;
    const int code = i < n ? (int)__ldg(blk + n + i) : 0;
    const int r = code ? (int)__ldg(rid + i) : -1;
    const int seg = code >= 1 && code <= 3 ? r * 3 + code - 1 : -1;
    const unsigned int members = __ballot_sync(0xffffffffu, seg >= 0);
    uint32_t first = 0;
    if (members && lane == __ffs(members) - 1) first = atomicAdd(C.members, (uint32_t)__popc(members));
    first = __shfl_sync(0xffffffffu, first, members ? __ffs(members) - 1 : 0);
    if (seg >= 0) {
      const uint32_t at = first + __popc(members & ((1u << lane) - 1u));
      keys[at] = quant_key(__ldg(blk + i));
      vals[at] = (uint32_t)seg;
    }
    const unsigned int same_seg = __match_any_sync(0xffffffffu, seg);
    if (seg >= 0 && lane == __ffs(same_seg) - 1) atomicAdd(C.seg + seg, (uint32_t)__popc(same_seg));
    const unsigned int same_region = __match_any_sync(0xffffffffu, r);
    if (r >= 0 && lane == __ffs(same_region) - 1) atomicAdd(C.planar + r, (uint32_t)__popc(same_region));
  }
}

__global__ void __launch_bounds__(kThreads) mom_region_segkey_kernel(long long m, const uint32_t *__restrict__ seg,
                                                                     unsigned long long *__restrict__ key, uint32_t *__restrict__ pos) {
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < m; p += (long long)gridDim.x * blockDim.x) {
    key[p] = __ldg(seg + p);
    pos[p] = (uint32_t)p;
  }
}

// the v of the member at segment-sorted position q: the v-sorted key at the position the second sort carried along
__device__ __forceinline__ double member_v(const unsigned long long *__restrict__ vkeys, const uint32_t *__restrict__ perm, long long q) {
  return __longlong_as_double((long long)__ldg(vkeys + __ldg(perm + q)));
}

// segment s < S: off[s] .. off[s + 1] its members; median[s] (NaN when empty); chunks[s] (chunks[S] = 0 for the scan)
__global__ void __launch_bounds__(kThreads) mom_region_select_kernel(long long S, const uint32_t *__restrict__ off,
                                                                     const unsigned long long *__restrict__ vkeys,
                                                                     const uint32_t *__restrict__ perm, double *__restrict__ median,
                                                                     uint32_t *__restrict__ chunks) {
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s <= S; s += (long long)gridDim.x * blockDim.x) {
    if (s == S) { chunks[S] = 0; continue; }
    const long long o = __ldg(off + s), n = (long long)__ldg(off + s + 1) - o;
    double med = NAN;
    if (n > 0) {
      long long k;
      double g;
      quantile_rank(n, 0.5, &k, &g);
      med = quantile_lerp(member_v(vkeys, perm, o + k), member_v(vkeys, perm, o + min(k + 1, n - 1)), g);
    }
    median[s] = med;
    chunks[s] = (uint32_t)((n + kRegionChunk - 1) / kRegionChunk);
  }
}

__global__ void __launch_bounds__(kThreads) mom_region_fold_kernel(long long S, long long n_chunks, const uint32_t *__restrict__ off,
                                                                   const uint32_t *__restrict__ chunk_off,
                                                                   const unsigned long long *__restrict__ vkeys,
                                                                   const uint32_t *__restrict__ perm, double *__restrict__ part) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (kThreads / 32);
  for (long long c = blockIdx.x * (long long)(kThreads / 32) + (threadIdx.x >> 5); c < n_chunks; c += warps) {
    long long lo = 0, hi = S;          // the segment of chunk c: chunk_off[lo] <= c < chunk_off[lo + 1]
    while (hi - lo > 1) {
      const long long mid = (lo + hi) >> 1;
      if ((long long)__ldg(chunk_off + mid) <= c) lo = mid; else hi = mid;
    }
    const long long j0 = (long long)__ldg(off + lo) + (c - (long long)__ldg(chunk_off + lo)) * kRegionChunk;
    const long long j1 = min((long long)__ldg(off + lo + 1), j0 + kRegionChunk);
    double sum = 0.0;
    for (long long j = j0 + lane; j < j1; j += 32) sum += member_v(vkeys, perm, j);
    sum = warp_sum(sum);
    if (lane == 0) part[c] = sum;
  }
}

__global__ void __launch_bounds__(kThreads) mom_region_merge_kernel(long long S, const uint32_t *__restrict__ chunk_off,
                                                                    const double *__restrict__ part, double *__restrict__ sum) {
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < S; s += (long long)gridDim.x * blockDim.x) {
    double v = 0.0;
    for (long long c = chunk_off[s]; c < (long long)chunk_off[s + 1]; ++c) v += part[c];
    sum[s] = v;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host driver
// ---------------------------------------------------------------------------------------------------------------
void mom_region_free(me_ctx *ctx) {
  MomRegionRun &G = ctx->mom_region;
  if (G.d_blk) { cudaFree(G.d_blk); G.d_blk = nullptr; G.cap_blk = 0; }
  if (G.d_rid) { cudaFree(G.d_rid); G.d_rid = nullptr; G.cap_rid = 0; }
  if (G.d_keys) { cudaFree(G.d_keys); G.d_keys = nullptr; G.cap_keys = 0; }
  if (G.d_vals) { cudaFree(G.d_vals); G.d_vals = nullptr; G.cap_vals = 0; }
  if (G.d_cnt) { cudaFree(G.d_cnt); G.d_cnt = nullptr; G.cap_cnt = 0; }
  if (G.d_out) { cudaFree(G.d_out); G.d_out = nullptr; G.cap_out = 0; }
  if (G.d_part) { cudaFree(G.d_part); G.d_part = nullptr; G.cap_part = 0; }
  G.open = false;
}

static int grid_of(const me_ctx *ctx, long long n) {
  return (int)std::max<long long>(1, std::min<long long>((n + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16));
}

int mom_region_begin(me_ctx *ctx, double s, long long min_family, int64_t *n_regions) {
  MomRegionRun &G = ctx->mom_region;
  G.open = false;
  *n_regions = 0;
  if (ctx->icp.open) return fail(ctx, ME_ERR_INVALID, "me_mom_region_begin while a registration is open (me_icp_end first)");
  if (ctx->drift.open) return fail(ctx, ME_ERR_INVALID, "me_mom_region_begin while a drift loop is open (me_drift_end first)");
  if (ctx->slab_request && ctx->world > 1)
    return fail(ctx, ME_ERR_INVALID, "me_mom_region_begin needs the replicated layout; the slab layout is requested (me_set_layout "
                                     "ME_LAYOUT_REPLICATED first)");
  const MomRun &M = ctx->mom;
  if (!M.ended) return fail(ctx, ME_ERR_INVALID, "me_mom_region_begin without a finished MOM call (me_mom_end first)");
  if (M.gen != ctx->cloud_gen || !M.pts_valid[M.which] || M.pts_gen[M.which] != ctx->cloud_gen)
    return fail(ctx, ME_ERR_INVALID, "me_mom_region_begin: the clouds changed after the MOM call's me_mom_begin (run the MOM "
                                     "call again)");
  const int which = M.which;
  const long long n = ctx->cloud[which].n;
  RegionList RL;
  ME_TRY(list_regions(ctx, "me_mom_region_begin", s, ctx->cloud[ME_CLOUD_GT].n > 0, &RL));
  ME_TRY(ensure(ctx, (void **)&G.d_rid, &G.cap_rid, n, sizeof(uint32_t)));
  ME_TRY(ensure(ctx, (void **)&G.d_blk, &G.cap_blk, 2 * n, sizeof(double)));
  ME_TRY(region_ids(ctx, RL, which, G.d_rid));
  mom_region_fill_kernel<<<grid_of(ctx, n), kThreads, 0, ctx->stream>>>(n, M.d_v[which], M.d_flag[which], G.d_blk);
  ME_LAUNCH_CHECK(ctx);
  G.which = which;
  G.status = M.status;
  G.min_family = min_family;
  G.s = s;
  G.R = RL.R;
  G.n = n;
  G.index = std::move(RL.index);
  G.n_points = which == ME_CLOUD_EST ? std::move(RL.n_est) : std::move(RL.n_gt);
  G.gen = ctx->cloud_gen;
  G.open = true;
  *n_regions = G.R;
  return ME_OK;
}

static int mom_region_ready(me_ctx *ctx, const char *who) {
  MomRegionRun &G = ctx->mom_region;
  if (!G.open) return fail(ctx, ME_ERR_INVALID, std::string(who) + " without an open MOM region call (me_mom_region_begin first)");
  if (G.gen != ctx->cloud_gen) {
    G.open = false;
    return fail(ctx, ME_ERR_INVALID, std::string(who) + ": the clouds changed after me_mom_region_begin; the call is void "
                                     "(run the MOM call and me_mom_region_begin again)");
  }
  return ME_OK;
}

int mom_region_block(me_ctx *ctx, double **device_block, int64_t *n) {
  ME_TRY(mom_region_ready(ctx, "me_mom_region_block"));
  *device_block = ctx->mom_region.d_blk;
  *n = 2 * ctx->mom_region.n;
  return ME_OK;
}

// the segmented selection over the reduced block: per segment rid * 3 + j its median and sum of v into d_out, its member count
// and the planar points per region into d_cnt
static int mom_region_select(me_ctx *ctx) {
  MomRegionRun &G = ctx->mom_region;
  const long long n = G.n, R = G.R, S = 3 * R;
  ME_TRY(ensure(ctx, (void **)&G.d_keys, &G.cap_keys, 3 * std::max<long long>(n, 1), sizeof(unsigned long long)));
  ME_TRY(ensure(ctx, (void **)&G.d_vals, &G.cap_vals, 2 * std::max<long long>(n, 1), sizeof(uint32_t)));
  ME_TRY(ensure(ctx, (void **)&G.d_cnt, &G.cap_cnt, 2 * (S + 1) + R + 1, sizeof(uint32_t)));
  ME_TRY(ensure(ctx, (void **)&G.d_out, &G.cap_out, 2 * S, sizeof(double)));
  uint32_t *seg_off = G.d_cnt, *planar = seg_off + S + 1, *chunk_off = planar + R, *members = chunk_off + S + 1;
  ME_CUDA(ctx, cudaMemsetAsync(G.d_cnt, 0, (size_t)(2 * (S + 1) + R + 1) * sizeof(uint32_t), ctx->stream));
  unsigned long long *k0 = G.d_keys, *k1 = G.d_keys + n, *k2 = G.d_keys + 2 * n;
  uint32_t *v0 = G.d_vals, *v1 = G.d_vals + n;
  mom_region_keys_kernel<<<grid_of(ctx, n), kThreads, 0, ctx->stream>>>(n, G.d_blk, G.d_rid, RegionCounts{seg_off, planar, members}, k0, v0);
  ME_LAUNCH_CHECK(ctx);
  uint32_t *h = (uint32_t *)ctx->h_pinned;
  ME_CUDA(ctx, cudaMemcpyAsync(h, members, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const long long m = h[0];
  ME_TRY(exclusive_scan_inplace(ctx, seg_off, S + 1));
  // by v, then stably by segment
  unsigned long long *kv = nullptr;
  uint32_t *seg_sorted = nullptr;
  ME_TRY(radix_sort_pairs(ctx, k0, v0, k1, v1, m, 63, &kv, &seg_sorted));
  unsigned long long *ks = kv == k0 ? k1 : k0;            // the buffer the first sort left free
  uint32_t *pos = seg_sorted == v0 ? v1 : v0;
  if (m > 0) {
    mom_region_segkey_kernel<<<grid_of(ctx, m), kThreads, 0, ctx->stream>>>(m, seg_sorted, ks, pos);
    ME_LAUNCH_CHECK(ctx);
  }
  int seg_bits = 0;
  while ((1ll << seg_bits) < S) ++seg_bits;
  unsigned long long *unused = nullptr;
  uint32_t *perm = nullptr;
  ME_TRY(radix_sort_pairs(ctx, ks, pos, k2, seg_sorted, m, seg_bits, &unused, &perm));
  double *median = G.d_out, *sum = G.d_out + S;
  mom_region_select_kernel<<<grid_of(ctx, S + 1), kThreads, 0, ctx->stream>>>(S, seg_off, kv, perm, median, chunk_off);
  ME_LAUNCH_CHECK(ctx);
  ME_TRY(exclusive_scan_inplace(ctx, chunk_off, S + 1));
  ME_CUDA(ctx, cudaMemcpyAsync(h, chunk_off + S, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const long long n_chunks = h[0];
  ME_TRY(ensure(ctx, (void **)&G.d_part, &G.cap_part, std::max<long long>(n_chunks, 1), sizeof(double)));
  if (n_chunks > 0) {
    const int fblocks = (int)std::min<long long>((n_chunks + kThreads / 32 - 1) / (kThreads / 32), (long long)ctx->sm_count * 32);
    mom_region_fold_kernel<<<fblocks, kThreads, 0, ctx->stream>>>(S, n_chunks, seg_off, chunk_off, kv, perm, G.d_part);
    ME_LAUNCH_CHECK(ctx);
  }
  mom_region_merge_kernel<<<grid_of(ctx, S), kThreads, 0, ctx->stream>>>(S, chunk_off, G.d_part, sum);
  ME_LAUNCH_CHECK(ctx);
  return ME_OK;
}

int mom_region_end(me_ctx *ctx, me_mom_region_row *rows, int64_t capacity) {
  ME_TRY(mom_region_ready(ctx, "me_mom_region_end"));
  MomRegionRun &G = ctx->mom_region;
  if (capacity < G.R)
    return fail(ctx, ME_ERR_INVALID, "me_mom_region_end: capacity " + std::to_string(capacity) + " < " + std::to_string(G.R) + " regions");
  if (G.R > 0 && !rows) return fail(ctx, ME_ERR_INVALID, "me_mom_region_end: null rows");
  G.open = false;
  const long long R = G.R, S = 3 * R;
  ME_TRY(mom_region_select(ctx));
  std::vector<uint32_t> cnt((size_t)(S + 1 + R));      // the segments' offsets, then the planar counts
  std::vector<double> out((size_t)2 * S);
  ME_CUDA(ctx, cudaMemcpyAsync(cnt.data(), G.d_cnt, cnt.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaMemcpyAsync(out.data(), G.d_out, out.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const bool axes = G.status == ME_MOM_OK;
  for (long long r = 0; r < R; ++r) {
    me_mom_region_row &x = rows[r];
    std::memset(&x, 0, sizeof(x));
    for (int a = 0; a < 3; ++a) x.index[a] = G.index[3 * r + a];
    x.n_points = G.n_points[r];
    x.n_planar = cnt[S + 1 + r];
    int status = axes ? ME_MOM_OK : G.status;
    for (int j = 0; j < 3; ++j) {
      const long long s = 3 * r + j, n = axes ? (long long)cnt[s + 1] - cnt[s] : 0;
      x.n[j] = n;
      x.mean[j] = n > 0 ? out[S + s] / (double)n : NAN;
      x.median[j] = n > 0 ? out[s] : NAN;
      if (axes && n < G.min_family) status = ME_MOM_SMALL_FAMILY;
    }
    x.status = status;
    x.mom = status == ME_MOM_OK ? (x.median[0] + x.median[1]) + x.median[2] : NAN;
  }
  return ME_OK;
}

}  // namespace me

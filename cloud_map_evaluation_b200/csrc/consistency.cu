// consistency.cu — local map consistency without a ground truth (me_consistency_*, DESIGN §3.15): per point, MME's radius
// neighbourhood, its entropy and its plane variance (the smallest eigenvalue of the neighbourhood covariance), folded per
// region floor(x / s).
//
//   consistency_walk_kernel         walk_global per query (mme_kernel's walk: fp64 offsets of the records, rows by dz, then
//                                   dy, x-runs ascending), so the moments, and with them e, equal MME's generic walk's bit for
//                                   bit.  MME's fp32-screened run-table walk with a record load per screened candidate was
//                                   measured slower than this walk on every scene of tools/consistency_time.py (DESIGN §3.15)
// Both write e, v and a flag byte per point in caller order.  The fold follows the region table (region.cu):
//   consistency_fold_kernel         one warp per chunk of kRegionChunk caller-order points of a region; lane l takes the
//                                   chunk's points l, l + 32, ...; a fixed shuffle tree; lane 0 writes the chunk's values
//   consistency_merge_kernel        one warp per region: lane l adds the region's chunks l, l + 32, ... in order, then a fixed
//                                   shuffle tree
// No floating-point atomics: two calls give the same bits as long as the cloud is not laid out again in between (a new
// layout can order the points of a cell differently: grid.cu ranks them with atomics).
#include "common.cuh"
#include "plane.cuh"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

namespace me {

static constexpr int kThreads = 256;
static constexpr int kWalkThreads = 128;
static constexpr int kSumF = ME_CONSISTENCY_SUM_FIELDS, kMaxF = ME_CONSISTENCY_MAX_FIELDS;
static constexpr int kPart = kSumF + kMaxF;
enum : uint8_t { kEvaluated = 1, kEntropyValid = 2, kPvValid = 4 };

struct PointOut {            // caller order
  double *e, *v;
  uint8_t *flag;
};

// entropy and plane variance of one query from its moments (plane_eig, shared with the mutually orthogonal metric's sweep)
__device__ __forceinline__ void finish_point(const Moments &m, int min_neighbors, long long o, const PointOut &O) {
  PlaneEig P;
  plane_eig(m, min_neighbors, P);
  uint8_t flag = kEvaluated;
  if (P.e_valid) flag |= kEntropyValid;
  if (isfinite(P.v)) flag |= kPvValid;
  O.e[o] = P.e;
  O.v[o] = P.v;
  O.flag[o] = flag;
}

// the generic walk: walk_global per query, one thread per query in cell-sorted order
__global__ void __launch_bounds__(kWalkThreads)
consistency_walk_kernel(const P4 *__restrict__ S, long long q_begin, long long q_end, CellIndex I, Lattice L, double r2,
                        float rc2, int rings, int min_neighbors, PointOut O) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = q_begin + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < q_end; i += stride) {
    const P4 q = load_p4(S + i);
    Moments m;
    m.init();
    walk_global(q, S, I, L, r2, rc2, rings, m);
    finish_point(m, min_neighbors, orig_of(q.idx), O);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// fold by region
// ---------------------------------------------------------------------------------------------------------------
struct ConsFoldSrc {
  const uint32_t *val;         // caller ids sorted by region (est ++ gt); nullptr: one region, the whole cloud in caller order
  const uint32_t *seg, *est_end;
  const uint32_t *chunk_off;   // this cloud's scanned chunk counts, R + 1
  long long R, n_chunks, n;
  uint32_t id0;                // caller id of the cloud's point 0 in val (0 or n_est)
  int q;                       // 0: est, 1: gt
  const double *e, *v;
  const uint8_t *flag;
};

__global__ void __launch_bounds__(kThreads) consistency_fold_kernel(ConsFoldSrc F, double *__restrict__ part) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (kThreads / 32);
  for (long long c = blockIdx.x * (long long)(kThreads / 32) + (threadIdx.x >> 5); c < F.n_chunks; c += warps) {
    long long j0, j1;
    if (F.val) {
      long long lo = 0, hi = F.R;          // the region of chunk c: chunk_off[lo] <= c < chunk_off[lo + 1]
      while (hi - lo > 1) {
        const long long mid = (lo + hi) >> 1;
        if ((long long)__ldg(F.chunk_off + mid) <= c) lo = mid; else hi = mid;
      }
      const long long seg0 = __ldg(F.seg + lo), ee = __ldg(F.est_end + lo);
      const long long ne_r = ee ? ee - seg0 : 0;
      const long long a = F.q == 0 ? seg0 : seg0 + ne_r, b = F.q == 0 ? seg0 + ne_r : (long long)__ldg(F.seg + lo + 1);
      j0 = a + (c - (long long)__ldg(F.chunk_off + lo)) * kRegionChunk;
      j1 = min(b, j0 + kRegionChunk);
    } else {
      j0 = c * kRegionChunk;
      j1 = min(F.n, j0 + kRegionChunk);
    }
    unsigned int n_query = 0, n_valid = 0, n_pv = 0;
    double sum_e = 0.0, sum_v = 0.0, sum_sv = 0.0, max_v = 0.0;
    for (long long j = j0 + lane; j < j1; j += 32) {
      const long long i = F.val ? (long long)(__ldg(F.val + j) - F.id0) : j;
      const uint8_t f = __ldg(F.flag + i);
      if (!(f & kEvaluated)) continue;
      ++n_query;
      if (f & kEntropyValid) { ++n_valid; sum_e += __ldg(F.e + i); }
      if (f & kPvValid) {
        const double v = __ldg(F.v + i);
        ++n_pv;
        sum_v += v;
        sum_sv += __dsqrt_rn(v);
        max_v = fmax(max_v, v);
      }
    }
    double o[kPart] = {(double)n_query, (double)n_valid, (double)n_pv, sum_e, sum_v, sum_sv, max_v};
#pragma unroll
    for (int f = 0; f < kSumF; ++f) o[f] = warp_sum(o[f]);
#pragma unroll
    for (int f = kSumF; f < kPart; ++f) o[f] = warp_max(o[f]);
    if (lane == 0) {
#pragma unroll
      for (int f = 0; f < kPart; ++f) part[c * kPart + f] = o[f];
    }
  }
}

// region r, one warp: lane l adds the region's chunks l, l + 32, ... in order, then a fixed shuffle tree; lane 0 writes
// blk[r * kSumF ..] and the maxima to blk[kSumF * R + r * kMaxF ..].  chunk_off == nullptr: one region of n_chunks chunks.
__global__ void __launch_bounds__(kThreads) consistency_merge_kernel(const double *__restrict__ part, const uint32_t *__restrict__ chunk_off,
                                                                     long long R, long long n_chunks, double *__restrict__ blk) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (kThreads / 32);
  for (long long r = blockIdx.x * (long long)(kThreads / 32) + (threadIdx.x >> 5); r < R; r += warps) {
    double v[kPart];
#pragma unroll
    for (int f = 0; f < kPart; ++f) v[f] = 0.0;
    const long long c0 = chunk_off ? (long long)chunk_off[r] : 0, c1 = chunk_off ? (long long)chunk_off[r + 1] : n_chunks;
    for (long long c = c0 + lane; c < c1; c += 32) {
#pragma unroll
      for (int f = 0; f < kSumF; ++f) v[f] += part[c * kPart + f];
#pragma unroll
      for (int f = kSumF; f < kPart; ++f) v[f] = fmax(v[f], part[c * kPart + f]);
    }
#pragma unroll
    for (int f = 0; f < kSumF; ++f) v[f] = warp_sum(v[f]);
#pragma unroll
    for (int f = kSumF; f < kPart; ++f) v[f] = warp_max(v[f]);
    if (lane == 0) {
#pragma unroll
      for (int f = 0; f < kSumF; ++f) blk[r * kSumF + f] = v[f];
#pragma unroll
      for (int f = 0; f < kMaxF; ++f) blk[kSumF * R + r * kMaxF + f] = v[kSumF + f];
    }
  }
}

__global__ void __launch_bounds__(kThreads) consistency_init_kernel(long long n, double *__restrict__ e, double *__restrict__ v,
                                                                    uint8_t *__restrict__ flag) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    e[i] = 0.0;
    v[i] = NAN;
    flag[i] = 0;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host driver
// ---------------------------------------------------------------------------------------------------------------
void consistency_free(me_ctx *ctx) {
  ConsistencyRun &K = ctx->consistency;
  if (K.d_blk) { cudaFree(K.d_blk); K.d_blk = nullptr; K.cap_blk = 0; }
  if (K.d_part) { cudaFree(K.d_part); K.d_part = nullptr; K.cap_part = 0; }
  for (int w = 0; w < 2; ++w) {
    if (K.d_e[w]) { cudaFree(K.d_e[w]); K.d_e[w] = nullptr; K.cap_e[w] = 0; }
    if (K.d_v[w]) { cudaFree(K.d_v[w]); K.d_v[w] = nullptr; K.cap_v[w] = 0; }
    if (K.d_flag[w]) { cudaFree(K.d_flag[w]); K.d_flag[w] = nullptr; K.cap_flag[w] = 0; }
    K.pts_valid[w] = false;
  }
  K.open = false;
}

// the lattice of a radius sweep of cloud `which` (MME's: the shared one, or the cloud's own with h = r / 2), this rank's
// query range, and run_mme's ring count and row slack (the same rows and candidates as mme_kernel); shared with mom.cu
int radius_sweep_layout(me_ctx *ctx, int which, double radius, const char *who, RadiusSweep *out) {
  Cloud &c = ctx->cloud[which];
  bool solo = false;
  ME_TRY(radius_lattice(ctx, which, radius, &solo));
  const double solo_h = solo ? 0.5 * radius : 0.0;
  // MME's entropies of a lattice the build below replaces would be void: keep them in caller order (me_get_entropies)
  if (c.entropy_valid && !c.entropy_caller_valid && !(c.grid_valid && c.grid_solo == solo && (!solo || c.solo_h == solo_h))) {
    ME_TRY(ensure(ctx, (void **)&c.d_entropy_caller, &c.cap_entropy_caller, c.n, sizeof(double)));
    const int blocks = (int)std::min<long long>((c.n + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
    unsort_f64_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.d_sorted, c.ns, c.d_entropy, c.d_entropy_caller);
    ME_LAUNCH_CHECK(ctx);
    c.entropy_caller_valid = true;
  }
  ME_TRY(build_grid(ctx, which, solo_h));
  ME_TRY(query_shard(ctx, which, &out->qb, &out->qe));
  const double rings_f = std::max(1.0, std::ceil(radius / c.lat.h - 1e-9));
  if (rings_f > 1.0e6) return fail(ctx, ME_ERR_RANGE, std::string(who) + ": radius spans too many lattice cells");
  out->rings = (int)rings_f;
  const double rc = radius / c.lat.h;
  out->rc2 = (float)(rc * rc * (1.0 + 1e-5) + 1e-4);
  return ME_OK;
}

// the sweep of this rank's query range into the per-point arrays of cloud `which`
static int consistency_sweep(me_ctx *ctx, int which, double radius, int min_neighbors) {
  ConsistencyRun &K = ctx->consistency;
  Cloud &c = ctx->cloud[which];
  K.pts_valid[which] = false;
  RadiusSweep RS;
  ME_TRY(radius_sweep_layout(ctx, which, radius, "me_consistency_begin", &RS));
  const long long qb = RS.qb, qe = RS.qe;
  const int rings = RS.rings;
  const float rc2 = RS.rc2;
  ME_TRY(ensure(ctx, (void **)&K.d_e[which], &K.cap_e[which], c.n, sizeof(double)));
  ME_TRY(ensure(ctx, (void **)&K.d_v[which], &K.cap_v[which], c.n, sizeof(double)));
  ME_TRY(ensure(ctx, (void **)&K.d_flag[which], &K.cap_flag[which], c.n, sizeof(uint8_t)));
  const PointOut O{K.d_e[which], K.d_v[which], K.d_flag[which]};
  {
    const int blocks = (int)std::min<long long>((c.n + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
    consistency_init_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.n, O.e, O.v, O.flag);
    ME_LAUNCH_CHECK(ctx);
  }
  K.rings = rings;
  K.solo = c.grid_solo ? 1 : 0;
  K.kernel = ME_CONSISTENCY_WALK;
  if (qe > qb) {
    const int blocks = (int)std::min<long long>((qe - qb + kWalkThreads - 1) / kWalkThreads, (long long)ctx->sm_count * 64);
    consistency_walk_kernel<<<blocks, kWalkThreads, 0, ctx->stream>>>(c.d_sorted, qb, qe, index_of(c), c.lat, radius * radius, rc2,
                                                                     rings, min_neighbors, O);
    ME_LAUNCH_CHECK(ctx);
  }
  K.pts_valid[which] = true;
  K.pts_gen[which] = ctx->cloud_gen;
  return ME_OK;
}

int consistency_begin(me_ctx *ctx, int which, double radius, int min_neighbors, double s, int64_t *n_regions) {
  ConsistencyRun &K = ctx->consistency;
  K.open = false;
  *n_regions = 0;
  const Cloud &c = ctx->cloud[which];
  if (c.n <= 0) return fail(ctx, ME_ERR_EMPTY, "me_consistency_begin: the cloud is empty");
  if (ctx->icp.open) return fail(ctx, ME_ERR_INVALID, "me_consistency_begin while a registration is open (me_icp_end first)");
  if (ctx->drift.open) return fail(ctx, ME_ERR_INVALID, "me_consistency_begin while a drift loop is open (me_drift_end first)");
  if (ctx->slab_request && ctx->world > 1)
    return fail(ctx, ME_ERR_INVALID, "me_consistency_begin needs the replicated layout; the slab layout is requested (me_set_layout "
                                     "ME_LAYOUT_REPLICATED first)");
  ME_TRY(consistency_sweep(ctx, which, radius, min_neighbors));

  // the occupied list (s > 0) or one region, the whole cloud in caller order (s = 0)
  RegionList RL;
  long long R = 1, n_chunks = (c.n + kRegionChunk - 1) / kRegionChunk;
  ConsFoldSrc F{};
  F.n = c.n; F.q = which;
  F.e = K.d_e[which]; F.v = K.d_v[which]; F.flag = K.d_flag[which];
  if (s > 0.0) {
    const bool with_gt = ctx->cloud[ME_CLOUD_GT].n > 0;
    ME_TRY(list_regions(ctx, "me_consistency_begin", s, with_gt, &RL));
    R = RL.R;
    n_chunks = RL.n_chunks[which];
    F.val = RL.val; F.seg = RL.seg; F.est_end = RL.est_end; F.chunk_off = RL.chunks + which * (R + 1);
    F.id0 = which == ME_CLOUD_EST ? 0u : (uint32_t)ctx->cloud[ME_CLOUD_EST].n;
  }
  F.R = R; F.n_chunks = n_chunks;
  ME_TRY(ensure(ctx, (void **)&K.d_blk, &K.cap_blk, (long long)kPart * R, sizeof(double)));
  ME_TRY(ensure(ctx, (void **)&K.d_part, &K.cap_part, (long long)kPart * std::max<long long>(1, n_chunks), sizeof(double)));
  if (n_chunks > 0) {
    const int fblocks = (int)std::min<long long>((n_chunks + kThreads / 32 - 1) / (kThreads / 32), (long long)ctx->sm_count * 32);
    consistency_fold_kernel<<<fblocks, kThreads, 0, ctx->stream>>>(F, K.d_part);
    ME_LAUNCH_CHECK(ctx);
  }
  const int rblocks = (int)std::min<long long>((R + kThreads / 32 - 1) / (kThreads / 32), (long long)ctx->sm_count * 32);
  consistency_merge_kernel<<<rblocks, kThreads, 0, ctx->stream>>>(K.d_part, F.chunk_off, R, n_chunks, K.d_blk);
  ME_LAUNCH_CHECK(ctx);

  K.which = which;
  K.radius = radius;
  K.min_neighbors = min_neighbors;
  K.s = s;
  K.R = s > 0.0 ? R : 0;
  if (s > 0.0) {
    K.index = std::move(RL.index);
    K.n_points = which == ME_CLOUD_EST ? std::move(RL.n_est) : std::move(RL.n_gt);
  } else {
    K.index.clear();
    K.n_points.clear();
  }
  K.gen = ctx->cloud_gen;
  K.open = true;
  *n_regions = K.R;
  return ME_OK;
}

static int consistency_ready(me_ctx *ctx, const char *who) {
  ConsistencyRun &K = ctx->consistency;
  if (!K.open) return fail(ctx, ME_ERR_INVALID, std::string(who) + " without an open consistency call (me_consistency_begin first)");
  if (K.gen != ctx->cloud_gen) {
    K.open = false;
    return fail(ctx, ME_ERR_INVALID, std::string(who) + ": the clouds changed after me_consistency_begin; the call is void "
                                     "(run me_consistency_begin again)");
  }
  return ME_OK;
}

int consistency_block(me_ctx *ctx, double **device_block, int32_t *n_sum, int32_t *n_max) {
  ME_TRY(consistency_ready(ctx, "me_consistency_block"));
  const ConsistencyRun &K = ctx->consistency;
  const long long R = std::max<long long>(K.R, 1);
  *device_block = K.d_blk;
  *n_sum = (int32_t)(kSumF * R);
  *n_max = (int32_t)(kMaxF * R);
  return ME_OK;
}

int consistency_end(me_ctx *ctx, me_consistency_row *rows, int64_t capacity, me_consistency_result *whole) {
  ME_TRY(consistency_ready(ctx, "me_consistency_end"));
  ConsistencyRun &K = ctx->consistency;
  if (capacity < K.R)
    return fail(ctx, ME_ERR_INVALID, "me_consistency_end: capacity " + std::to_string(capacity) + " < " + std::to_string(K.R) + " regions");
  if (K.R > 0 && !rows) return fail(ctx, ME_ERR_INVALID, "me_consistency_end: null rows");
  K.open = false;
  std::vector<double> h((size_t)kPart * std::max<long long>(K.R, 1));
  ME_CUDA(ctx, cudaMemcpyAsync(h.data(), K.d_blk, h.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (me_consistency_finalize(K.R, K.s, K.index.data(), K.n_points.data(), ctx->cloud[K.which].n, h.data(), rows, whole) != ME_OK)
    return fail(ctx, ME_ERR_INVALID, "me_consistency_finalize failed");
  whole->radius = K.radius;
  whole->min_neighbors = K.min_neighbors;
  whole->kernel = K.kernel;
  whole->rings = K.rings;
  whole->solo = K.solo;
  return ME_OK;
}

int consistency_points(me_ctx *ctx, int which, double *entropy, double *plane_variance) {
  const ConsistencyRun &K = ctx->consistency;
  if (!K.pts_valid[which])
    return fail(ctx, ME_ERR_INVALID, "me_get_consistency_points before me_consistency_begin on this cloud");
  if (K.pts_gen[which] != ctx->cloud_gen)
    return fail(ctx, ME_ERR_INVALID, "me_get_consistency_points: the clouds changed after me_consistency_begin (run it again)");
  const long long n = ctx->cloud[which].n;
  if (entropy) ME_CUDA(ctx, cudaMemcpyAsync(entropy, K.d_e[which], (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  if (plane_variance)
    ME_CUDA(ctx, cudaMemcpyAsync(plane_variance, K.d_v[which], (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return ME_OK;
}

}  // namespace me

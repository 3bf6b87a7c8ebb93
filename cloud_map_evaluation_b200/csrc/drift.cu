// drift.cu — one rigid point-to-point ICP per region of the estimated cloud (me_drift_*), all regions in one pass over the
// cloud per iteration (DESIGN §3.13).  A region's transform separates drift (the region is shifted or turned as a whole) from
// damage (what remains after it).
//
// Begin:
//   list_regions (region.cu, est only)  the occupied regions floor(x / s) in caller order
//   region_ids (region.cu)             rid[i] = the region of caller index i
//   drift_fold_kernel<true> + merge     per region count and sum (x - c_r) of the original points: the centroids
// Per iteration:
//   drift_transform_kernel              x_i := T_{rid[i]} x_i^orig, transform_kernel's rounding, from the original coordinates
//   run_nn                              the est->gt sweep of registration (icp_sweep's parameters), this rank's queries
//   record_positions (region.cu)        caller index -> record position in the new layout
//   drift_fold_kernel<false>            one warp per chunk of kRegionChunk points of a region in caller order: lane l walks the
//                                       chunk's points l, l + 32, ..., keeps nn >= 0 and d2 < R^2, and adds the 17 values of
//                                       ME_ICP_BLOCK_P2P about c_r, every product and sum rounded on its own (no FMA); then a
//                                       fixed shuffle tree; lane 0 writes the chunk's values
//   drift_merge_kernel                  one thread per region adds its chunks in chunk order into the block
// The summation order depends only on the occupied list and on the records this rank holds: two calls give the same bits.
// No floating-point atomics.  The host reads the reduced block and runs the per-region update (icp_update_host).
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace me {

static constexpr int kThreads = 256;
static constexpr int kB = ME_ICP_BLOCK_P2P;         // values per region

// transform_kernel's operation order: o_r = (((T_r0 x + T_r1 y) + T_r2 z) + T_r3), x' = o_0 / o_3, ..., with T of the point's
// region
__global__ void __launch_bounds__(kThreads) drift_transform_kernel(const double *__restrict__ orig, const uint32_t *__restrict__ rid,
                                                                   const double *__restrict__ Ttab, long long n,
                                                                   double *__restrict__ xyz) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double x = __ldg(orig + 3 * i), y = __ldg(orig + 3 * i + 1), z = __ldg(orig + 3 * i + 2);
    const double *T = Ttab + 16ll * __ldg(rid + i);
    double o[4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
      o[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(__ldg(T + r * 4), x), __dmul_rn(__ldg(T + r * 4 + 1), y)),
                                 __dmul_rn(__ldg(T + r * 4 + 2), z)), __ldg(T + r * 4 + 3));
    xyz[3 * i] = __ddiv_rn(o[0], o[3]);
    xyz[3 * i + 1] = __ddiv_rn(o[1], o[3]);
    xyz[3 * i + 2] = __ddiv_rn(o[2], o[3]);
  }
}

struct DriftSrc {
  const uint32_t *val, *seg, *chunk_off;   // caller ids by region; R + 1 first positions; R + 1 scanned chunk counts
  const uint32_t *pos_of;                  // caller index -> record position (kCentroid: unused)
  const double *xyz;                       // est points, caller order (kCentroid: the original ones)
  const double *c;                         // 3 per region
  long long R, n_chunks;
  // !kCentroid: the records of the sweep
  const int32_t *nn_idx;
  const double *nn_d2, *gt;
  long long nb, ne;                        // the sorted range this rank swept
  double r2;
};

// kCentroid: every point counts, v = [count, sum (x - c) (3), 0 ...]; else the kept pairs' ME_ICP_BLOCK_P2P values
template <bool kCentroid>
__global__ void __launch_bounds__(kThreads) drift_fold_kernel(DriftSrc F, double *__restrict__ part) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (kThreads / 32);
  for (long long ch = blockIdx.x * (long long)(kThreads / 32) + (threadIdx.x >> 5); ch < F.n_chunks; ch += warps) {
    long long lo = 0, hi = F.R;          // the region of chunk ch: chunk_off[lo] <= ch < chunk_off[lo + 1]
    while (hi - lo > 1) {
      const long long mid = (lo + hi) >> 1;
      if ((long long)__ldg(F.chunk_off + mid) <= ch) lo = mid; else hi = mid;
    }
    const long long j0 = (long long)__ldg(F.seg + lo) + (ch - (long long)__ldg(F.chunk_off + lo)) * kRegionChunk;
    const long long j1 = min((long long)__ldg(F.seg + lo + 1), j0 + kRegionChunk);
    const double cx = __ldg(F.c + 3 * lo), cy = __ldg(F.c + 3 * lo + 1), cz = __ldg(F.c + 3 * lo + 2);
    double v[kB];
#pragma unroll
    for (int f = 0; f < kB; ++f) v[f] = 0.0;
    for (long long j = j0 + lane; j < j1; j += 32) {
      const uint32_t i = __ldg(F.val + j);
      const double px = __dsub_rn(__ldg(F.xyz + 3ll * i), cx), py = __dsub_rn(__ldg(F.xyz + 3ll * i + 1), cy),
                   pz = __dsub_rn(__ldg(F.xyz + 3ll * i + 2), cz);
      if (kCentroid) {
        v[0] = __dadd_rn(v[0], 1.0);
        v[1] = __dadd_rn(v[1], px); v[2] = __dadd_rn(v[2], py); v[3] = __dadd_rn(v[3], pz);
        continue;
      }
      const uint32_t k = __ldg(F.pos_of + i);
      if (k == 0xffffffffu || k < F.nb || k >= F.ne) continue;
      const int32_t nn = __ldg(F.nn_idx + k);
      if (nn < 0) continue;
      const double d2 = __ldg(F.nn_d2 + k);
      if (!(d2 < F.r2)) continue;                    // SearchHybrid keeps d2 < R^2
      const double qx = __dsub_rn(__ldg(F.gt + 3ll * nn), cx), qy = __dsub_rn(__ldg(F.gt + 3ll * nn + 1), cy),
                   qz = __dsub_rn(__ldg(F.gt + 3ll * nn + 2), cz);
      const double p[3] = {px, py, pz}, q[3] = {qx, qy, qz};
      v[0] = __dadd_rn(v[0], 1.0);
#pragma unroll
      for (int a = 0; a < 3; ++a) { v[1 + a] = __dadd_rn(v[1 + a], p[a]); v[4 + a] = __dadd_rn(v[4 + a], q[a]); }
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int col = 0; col < 3; ++col) v[7 + 3 * r + col] = __dadd_rn(v[7 + 3 * r + col], __dmul_rn(q[r], p[col]));
      v[16] = __dadd_rn(v[16], d2);
    }
#pragma unroll
    for (int f = 0; f < kB; ++f) v[f] = warp_sum(v[f]);
    if (lane == 0) {
#pragma unroll
      for (int f = 0; f < kB; ++f) part[ch * kB + f] = v[f];
    }
  }
}

// region r: its chunks added in chunk order, starting from 0 -> blk[r * kB ..]
__global__ void __launch_bounds__(kThreads) drift_merge_kernel(const double *__restrict__ part, const uint32_t *__restrict__ chunk_off,
                                                               long long R, double *__restrict__ blk) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < R; r += (long long)gridDim.x * blockDim.x) {
    double v[kB];
#pragma unroll
    for (int f = 0; f < kB; ++f) v[f] = 0.0;
    for (long long c = chunk_off[r]; c < (long long)chunk_off[r + 1]; ++c)
#pragma unroll
      for (int f = 0; f < kB; ++f) v[f] = __dadd_rn(v[f], part[c * kB + f]);
#pragma unroll
    for (int f = 0; f < kB; ++f) blk[r * kB + f] = v[f];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host driver
// ---------------------------------------------------------------------------------------------------------------
static void free_dev(void *p) { if (p) cudaFree(p); }

// every failure of an open loop closes it: the estimated cloud comes back as it was at me_drift_begin
void drift_close(me_ctx *ctx, bool restore) {
  DriftRun &D = ctx->drift;
  if (!D.open && !D.orig) return;
  Cloud &E = ctx->cloud[ME_CLOUD_EST];
  if (D.open) {
    if (restore && D.orig && E.d_xyz == D.xyz && E.n == D.n_est) {
      wait_upload(ctx, ME_CLOUD_EST);      // a cloud set during the loop into the same buffer lands before the restore
      cudaMemcpyAsync(E.d_xyz, D.orig, (size_t)E.n * 3 * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream);
    }
    invalidate_cloud(E);
  }
  cudaStreamSynchronize(ctx->stream);
  for (void *p : {(void *)D.orig, (void *)D.d_rid, (void *)D.d_val, (void *)D.d_pos_of, (void *)D.d_seg, (void *)D.d_chunk_off,
                  (void *)D.d_T, (void *)D.d_c, (void *)D.d_blk, (void *)D.d_part})
    free_dev(p);
  D = DriftRun();
}
static int drift_fail(me_ctx *ctx, int rc) {
  drift_close(ctx, true);
  return rc;
}

// step 1 to 3 of an iteration at the transforms D.T: move, sweep, fold into D.d_blk
static int drift_iterate(me_ctx *ctx) {
  DriftRun &D = ctx->drift;
  Cloud &E = ctx->cloud[ME_CLOUD_EST], &G = ctx->cloud[ME_CLOUD_GT];
  ME_CUDA(ctx, cudaMemcpyAsync(D.d_T, D.T.data(), (size_t)16 * D.R * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  const int blocks = (int)std::min<long long>((D.n_est + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
  drift_transform_kernel<<<blocks, kThreads, 0, ctx->stream>>>(D.orig, D.d_rid, D.d_T, D.n_est, E.d_xyz);
  ME_LAUNCH_CHECK(ctx);
  invalidate_cloud(E);
  me_nn_params p;      // icp_sweep's sweep
  std::memset(&p, 0, sizeof(p));
  p.icp_max_distance = D.max_dist;
  p.cutoff_mode = ME_CUTOFF_DIST_LT_R;
  p.pairing = ME_PAIRING_GEOMETRIC;
  p.want_full_cd = 0;
  p.directions = 1;
  ME_TRY(run_nn(ctx, &p, false));
  ME_TRY(record_positions(ctx, ME_CLOUD_EST, D.d_pos_of));
  DriftSrc F;
  F.val = D.d_val; F.seg = D.d_seg; F.chunk_off = D.d_chunk_off; F.pos_of = D.d_pos_of; F.xyz = E.d_xyz; F.c = D.d_c;
  F.R = D.R; F.n_chunks = D.n_chunks;
  F.nn_idx = E.d_nn_idx; F.nn_d2 = E.d_nn_d2; F.gt = G.d_xyz; F.nb = E.nn_b; F.ne = E.nn_e;
  F.r2 = D.max_dist * D.max_dist;
  const int fblocks = (int)std::min<long long>((D.n_chunks + kThreads / 32 - 1) / (kThreads / 32), (long long)ctx->sm_count * 32);
  drift_fold_kernel<false><<<fblocks, kThreads, 0, ctx->stream>>>(F, D.d_part);
  ME_LAUNCH_CHECK(ctx);
  const int rblocks = (int)std::min<long long>((D.R + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
  drift_merge_kernel<<<rblocks, kThreads, 0, ctx->stream>>>(D.d_part, D.d_chunk_off, D.R, D.d_blk);
  ME_LAUNCH_CHECK(ctx);
  return ME_OK;
}

int drift_begin(me_ctx *ctx, double s, double max_dist, int max_iter, double rel_fitness, double rel_rmse, int64_t *n_regions) {
  *n_regions = 0;
  if (ctx->drift.open) return drift_fail(ctx, fail(ctx, ME_ERR_INVALID, "me_drift_begin while a drift loop is open (me_drift_end first)"));
  if (ctx->icp.open) return fail(ctx, ME_ERR_INVALID, "me_drift_begin while a registration is open (me_icp_end first)");
  Cloud &E = ctx->cloud[ME_CLOUD_EST], &G = ctx->cloud[ME_CLOUD_GT];
  if (E.n <= 0 || G.n <= 0) return fail(ctx, ME_ERR_EMPTY, "me_drift_begin: both clouds must be set");
  if (!E.owned) return fail(ctx, ME_ERR_INVALID, "me_drift needs a library-owned estimated cloud (use me_set_cloud)");
  if (ctx->world > 1 && ctx->slab_request)
    return fail(ctx, ME_ERR_INVALID, "the drift loop needs the replicated layout: me_set_layout(ME_LAYOUT_REPLICATED) before "
                                     "me_drift_begin, ME_LAYOUT_SLAB again afterwards");
  ME_TRY(wait_upload(ctx, ME_CLOUD_EST));
  RegionList RL;
  ME_TRY(list_regions(ctx, "me_drift_begin", s, false, &RL));
  DriftRun &D = ctx->drift;
  const long long n = E.n, R = RL.R;
  D.xyz = E.d_xyz; D.n_est = n; D.R = R; D.n_chunks = RL.n_chunks[0];
  D.s = s; D.max_dist = max_dist; D.max_iter = max_iter; D.rel_fitness = rel_fitness; D.rel_rmse = rel_rmse;
  long long cap = 0;
  int rc = ensure(ctx, (void **)&D.orig, &cap, 3 * n, sizeof(double));
  if (rc == ME_OK) rc = ensure(ctx, (void **)&D.d_rid, &cap, n, sizeof(uint32_t));
  if (rc == ME_OK) rc = ensure(ctx, (void **)&D.d_val, &cap, n, sizeof(uint32_t));
  if (rc == ME_OK) rc = ensure(ctx, (void **)&D.d_pos_of, &cap, n, sizeof(uint32_t));
  if (rc == ME_OK) rc = ensure(ctx, (void **)&D.d_seg, &cap, R + 1, sizeof(uint32_t));
  if (rc == ME_OK) rc = ensure(ctx, (void **)&D.d_chunk_off, &cap, R + 1, sizeof(uint32_t));
  if (rc == ME_OK) rc = ensure(ctx, (void **)&D.d_T, &cap, 16 * R, sizeof(double));
  if (rc == ME_OK) rc = ensure(ctx, (void **)&D.d_c, &cap, 3 * R, sizeof(double));
  if (rc == ME_OK) rc = ensure(ctx, (void **)&D.d_blk, &cap, kB * R, sizeof(double));
  if (rc == ME_OK) rc = ensure(ctx, (void **)&D.d_part, &cap, kB * std::max<long long>(1, D.n_chunks), sizeof(double));
  if (rc != ME_OK) { drift_close(ctx, false); return rc; }
  D.open = true;
  D.gen = ctx->cloud_gen;
  // the list lives in d_work, which the sweeps reuse: keep what the loop needs
  rc = region_ids(ctx, RL, ME_CLOUD_EST, D.d_rid);
  if (rc != ME_OK) return drift_fail(ctx, rc);
  if (cudaMemcpyAsync(D.d_val, RL.val, (size_t)n * 4, cudaMemcpyDeviceToDevice, ctx->stream) != cudaSuccess ||
      cudaMemcpyAsync(D.d_seg, RL.seg, (size_t)(R + 1) * 4, cudaMemcpyDeviceToDevice, ctx->stream) != cudaSuccess ||
      cudaMemcpyAsync(D.d_chunk_off, RL.chunks, (size_t)(R + 1) * 4, cudaMemcpyDeviceToDevice, ctx->stream) != cudaSuccess ||
      cudaMemcpyAsync(D.orig, E.d_xyz, (size_t)n * 3 * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream) != cudaSuccess)
    return drift_fail(ctx, fail(ctx, ME_ERR_CUDA, "me_drift_begin: device copies failed"));
  D.index = std::move(RL.index);
  D.n_est_r = std::move(RL.n_est);
  D.c.resize((size_t)3 * R);
  for (long long r = 0; r < 3 * R; ++r) D.c[r] = ((double)D.index[r] + 0.5) * s;
  D.T.assign((size_t)16 * R, 0.0);
  for (long long r = 0; r < R; ++r) D.T[16 * r] = D.T[16 * r + 5] = D.T[16 * r + 10] = D.T[16 * r + 15] = 1.0;
  D.fitness.assign(R, 0.0); D.rmse.assign(R, 0.0); D.fitness0.assign(R, 0.0); D.rmse0.assign(R, 0.0);
  D.n_corr.assign(R, 0); D.n_corr0.assign(R, 0); D.it.assign(R, 0); D.status.assign(R, -1);
  D.h_blk.resize((size_t)kB * R);
  if (cudaMemcpyAsync(D.d_c, D.c.data(), (size_t)3 * R * sizeof(double), cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess)
    return drift_fail(ctx, fail(ctx, ME_ERR_CUDA, "me_drift_begin: upload of the region centres failed"));
  // the centroids: the same fold over every original point (d_xyz is whole on every rank)
  DriftSrc F{};
  F.val = D.d_val; F.seg = D.d_seg; F.chunk_off = D.d_chunk_off; F.xyz = D.orig; F.c = D.d_c; F.R = R; F.n_chunks = D.n_chunks;
  const int fblocks = (int)std::min<long long>((D.n_chunks + kThreads / 32 - 1) / (kThreads / 32), (long long)ctx->sm_count * 32);
  const int rblocks = (int)std::min<long long>((R + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
  drift_fold_kernel<true><<<fblocks, kThreads, 0, ctx->stream>>>(F, D.d_part);
  drift_merge_kernel<<<rblocks, kThreads, 0, ctx->stream>>>(D.d_part, D.d_chunk_off, R, D.d_blk);
  ctx->launches += 2;
  if (cudaGetLastError() != cudaSuccess ||
      cudaMemcpyAsync(D.h_blk.data(), D.d_blk, D.h_blk.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
      cudaStreamSynchronize(ctx->stream) != cudaSuccess)
    return drift_fail(ctx, fail(ctx, ME_ERR_CUDA, "me_drift_begin: the centroid fold failed"));
  D.centroid.resize((size_t)3 * R);
  for (long long r = 0; r < R; ++r)
    for (int a = 0; a < 3; ++a) D.centroid[3 * r + a] = D.c[3 * r + a] + D.h_blk[kB * r + 1 + a] / D.h_blk[kB * r];
  rc = drift_iterate(ctx);
  if (rc != ME_OK) return drift_fail(ctx, rc);
  *n_regions = R;
  return ME_OK;
}

static int drift_ready(me_ctx *ctx, const char *call) {
  DriftRun &D = ctx->drift;
  if (!D.open) return fail(ctx, ME_ERR_INVALID, std::string(call) + " before me_drift_begin");
  const Cloud &E = ctx->cloud[ME_CLOUD_EST];
  if (D.gen != ctx->cloud_gen || E.d_xyz != D.xyz || E.n != D.n_est)
    return drift_fail(ctx, fail(ctx, ME_ERR_INVALID, std::string(call) + ": a cloud changed during the drift loop; the loop is "
                                                     "closed and the estimated cloud restored"));
  return ME_OK;
}

int drift_block(me_ctx *ctx, double **device_block, int32_t *n_sum) {
  ME_TRY(drift_ready(ctx, "me_drift_block"));
  *device_block = ctx->drift.d_blk;
  *n_sum = (int32_t)(kB * ctx->drift.R);
  return ME_OK;
}

int drift_step(me_ctx *ctx, int32_t *done) {
  *done = 0;
  ME_TRY(drift_ready(ctx, "me_drift_step"));
  DriftRun &D = ctx->drift;
  if (std::none_of(D.status.begin(), D.status.end(), [](int32_t s) { return s < 0; })) { *done = 1; return ME_OK; }
  if (cudaMemcpyAsync(D.h_blk.data(), D.d_blk, D.h_blk.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
      cudaStreamSynchronize(ctx->stream) != cudaSuccess)
    return drift_fail(ctx, fail(ctx, ME_ERR_CUDA, "reading the drift block failed"));
  bool running = false;
  for (long long r = 0; r < D.R; ++r) {
    if (D.status[r] >= 0) continue;
    const double *blk = D.h_blk.data() + kB * r;
    const long long nc = (long long)std::llround(blk[0]);
    const double fitness = (double)nc / (double)D.n_est_r[r];
    const double rmse = nc > 0 ? std::sqrt(blk[kB - 1] / (double)nc) : 0.0;
    bool converged = false;
    if (D.have_prev) {      // the block of an update: ICPConvergenceCriteria, as me_icp_step
      ++D.it[r];
      converged = std::fabs(D.fitness[r] - fitness) < D.rel_fitness && std::fabs(D.rmse[r] - rmse) < D.rel_rmse;
    } else {
      D.n_corr0[r] = nc; D.fitness0[r] = fitness; D.rmse0[r] = rmse;
    }
    D.n_corr[r] = nc; D.fitness[r] = fitness; D.rmse[r] = rmse;
    if (converged) { D.status[r] = ME_DRIFT_CONVERGED; continue; }
    if (D.it[r] >= D.max_iter) { D.status[r] = ME_DRIFT_ITERATION_LIMIT; continue; }
    if (nc < 3) { D.status[r] = ME_DRIFT_TOO_FEW; continue; }
    double upd[16], Tn[16], *T = D.T.data() + 16 * r;
    icp_update_host(ME_ICP_POINT_TO_POINT, blk, D.c.data() + 3 * r, upd);
    for (int i = 0; i < 4; ++i)
      for (int col = 0; col < 4; ++col) { double s = 0; for (int k = 0; k < 4; ++k) s += upd[i * 4 + k] * T[k * 4 + col]; Tn[i * 4 + col] = s; }
    std::memcpy(T, Tn, sizeof(Tn));
    running = true;
  }
  D.have_prev = true;
  if (!running) { *done = 1; return ME_OK; }
  const int rc = drift_iterate(ctx);
  if (rc != ME_OK) return drift_fail(ctx, rc);
  return ME_OK;
}

int drift_end(me_ctx *ctx, me_drift_row *rows, int64_t capacity) {
  ME_TRY(drift_ready(ctx, "me_drift_end"));
  DriftRun &D = ctx->drift;
  if (std::any_of(D.status.begin(), D.status.end(), [](int32_t s) { return s < 0; }))
    return drift_fail(ctx, fail(ctx, ME_ERR_INVALID, "me_drift_end before the loop is done (me_drift_step until *done = 1)"));
  if (capacity < D.R)
    return drift_fail(ctx, fail(ctx, ME_ERR_INVALID, "me_drift_end: capacity " + std::to_string(capacity) + " < " +
                                                     std::to_string(D.R) + " regions"));
  for (long long r = 0; r < D.R; ++r) {
    me_drift_row &W = rows[r];
    std::memset(&W, 0, sizeof(W));
    const double *T = D.T.data() + 16 * r, *c = D.centroid.data() + 3 * r;
    for (int a = 0; a < 3; ++a) {
      W.index[a] = D.index[3 * r + a];
      W.min[a] = (double)W.index[a] * D.s;
      W.max[a] = (double)(W.index[a] + 1) * D.s;
      W.centroid[a] = c[a];
      W.shift[a] = (((T[a * 4] * c[0] + T[a * 4 + 1] * c[1]) + T[a * 4 + 2] * c[2]) + T[a * 4 + 3]) - c[a];
    }
    W.shift_norm = std::sqrt((W.shift[0] * W.shift[0] + W.shift[1] * W.shift[1]) + W.shift[2] * W.shift[2]);
    const double ax = T[9] - T[6], ay = T[2] - T[8], az = T[4] - T[1];      // R32 - R23, R13 - R31, R21 - R12
    W.angle = std::atan2(0.5 * std::sqrt((ax * ax + ay * ay) + az * az), (((T[0] + T[5]) + T[10]) - 1.0) / 2.0);
    W.n_est = D.n_est_r[r];
    W.n_corr_before = D.n_corr0[r]; W.fitness_before = D.fitness0[r]; W.rmse_before = D.rmse0[r];
    W.n_corr = D.n_corr[r]; W.fitness = D.fitness[r]; W.rmse = D.rmse[r];
    std::memcpy(W.T, T, sizeof(W.T));
    W.iterations = D.it[r];
    W.status = D.status[r];
  }
  drift_close(ctx, true);
  return ME_OK;
}

}  // namespace me

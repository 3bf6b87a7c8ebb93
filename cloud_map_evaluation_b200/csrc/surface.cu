// surface.cu — point-to-plane AC / COM / CD / F1 / IoU and normal consistency (me_nn_surface_*): the records of the last NN
// sweep measured against the tangent plane of each neighbour, without a new sweep (DESIGN §3.14).
//
//   surface_fold_kernel   block b owns the fixed contiguous slice b of a direction's records; thread t walks its records
//                         t, t + 256, ... and sums in that order; every warp reduces with a fixed shuffle tree (the (n, mean,
//                         M2) of e with chan_merge) and lane 0 writes the warp's values
//   surface_merge_kernel  one block: the warps' values added (and their moments merged) in warp order, block after block,
//                         into the direction's section of the block
// The summation order depends only on the record range and the grid: two calls give the same bits.  No floating-point
// atomics.  Working k-NN normals come from estimate_normals (icp.cu) into the cloud's normal buffer, as generalized ICP does.
#include "common.cuh"
#include "records.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace me {

static constexpr int kThreads = 256;
static constexpr int kWarps = kThreads / 32;
// per warp: the SUM fields n_query n_corr n_inlier[5] sum_e[5] sum_e2[5] sum_nn n_no_normal n_no_normal_nn n_nc sum_c, the MAX
// fields max_e max_e_nn, then the (n, mean, M2) of the kept e
static constexpr int kSumF = 22, kMaxF = 2;
static constexpr int kPart = kSumF + kMaxF + 3;
static constexpr int kExtra = 2 * kBlkNN;                      // offset of the per-direction extras in the block
static constexpr int kMaxOff = ME_SURFACE_BLOCK_SUM;            // offset of the MAX part
static_assert(kExtra + 8 == ME_SURFACE_BLOCK_SUM, "block layout");

struct SurfSrc {
  long long b, e;              // the records walked (record_src's range)
  long long nb, ne;            // the queries the five-level pass counts in n_query
  const P4 *Q;                 // the query cloud, cell-sorted: the caller index of record i
  const int32_t *nn_idx;
  const double *nn_d2;
  const double *q_xyz, *r_xyz; // caller order
  const double *q_nrm, *r_nrm; // caller order
};

// normal j of nrm, and whether it is usable: its squared norm finite and > 0
__device__ __forceinline__ bool load_normal(const double *__restrict__ nrm, long long j, double &x, double &y, double &z, double &sq) {
  x = __ldg(nrm + 3 * j); y = __ldg(nrm + 3 * j + 1); z = __ldg(nrm + 3 * j + 2);
  sq = sqnorm_eigen(x, y, z);
  return sq > 0.0 && sq < INFINITY;
}

__global__ void __launch_bounds__(kThreads) surface_fold_kernel(SurfSrc S, NNConst C, long long per_block, double *__restrict__ part) {
  unsigned int n_query = 0, n_corr = 0, n_inl[5] = {0, 0, 0, 0, 0}, n_no = 0, n_no_nn = 0, n_nc = 0;
  double sum_e[5] = {0, 0, 0, 0, 0}, sum_e2[5] = {0, 0, 0, 0, 0}, sum_nn = 0.0, sum_c = 0.0, max_e = 0.0, max_e_nn = 0.0;
  double shift = 0.0, s1 = 0.0, s2 = 0.0;      // the kept e as sums of (e - shift), shift = the thread's first kept e
  const long long b0 = S.b + blockIdx.x * per_block, b1 = min(S.e, b0 + per_block);
  for (long long i = b0 + threadIdx.x; i < b1; i += kThreads) {
    const int32_t j = __ldg(S.nn_idx + i);
    n_query += (i >= S.nb && i < S.ne && j != -2);
    if (j < 0) continue;
    const bool kept = keep_pair(__ldg(S.nn_d2 + i), C);
    if (!kept && !C.want_full_cd) continue;
    double nx, ny, nz, sn;
    if (!load_normal(S.r_nrm, j, nx, ny, nz, sn)) {
      n_no += kept;
      n_no_nn += C.want_full_cd;
      continue;
    }
    const long long o = orig_of(__double_as_longlong(__ldg(reinterpret_cast<const double *>(S.Q + i) + 3)));
    const double dx = __dsub_rn(__ldg(S.q_xyz + 3 * o), __ldg(S.r_xyz + 3ll * j));
    const double dy = __dsub_rn(__ldg(S.q_xyz + 3 * o + 1), __ldg(S.r_xyz + 3ll * j + 1));
    const double dz = __dsub_rn(__ldg(S.q_xyz + 3 * o + 2), __ldg(S.r_xyz + 3ll * j + 2));
    const double dot = __dadd_rn(__dadd_rn(__dmul_rn(dx, nx), __dmul_rn(dy, ny)), __dmul_rn(dz, nz));
    const double len_n = __dsqrt_rn(sn);
    const double e = __ddiv_rn(fabs(dot), len_n);
    if (C.want_full_cd) { sum_nn += e; max_e_nn = fmax(max_e_nn, e); }
    if (!kept) continue;
    if (n_corr++ == 0) shift = e;
    const double t = e - shift;
    s1 += t;
    s2 += t * t;
    max_e = fmax(max_e, e);
    const double ee = __dmul_rn(e, e);
#pragma unroll
    for (int k = 0; k < 5; ++k)
      if (e <= C.tau[k]) { ++n_inl[k]; sum_e[k] += e; sum_e2[k] += ee; }
    double mx, my, mz, sm;
    if (load_normal(S.q_nrm, o, mx, my, mz, sm)) {
      const double dmn = __dadd_rn(__dadd_rn(__dmul_rn(mx, nx), __dmul_rn(my, ny)), __dmul_rn(mz, nz));
      ++n_nc;
      sum_c += fmin(1.0, __ddiv_rn(fabs(dmn), __dmul_rn(__dsqrt_rn(sm), len_n)));
    }
  }
  double v[kPart];
  v[0] = (double)n_query;
  v[1] = (double)n_corr;
#pragma unroll
  for (int k = 0; k < 5; ++k) { v[2 + k] = (double)n_inl[k]; v[7 + k] = sum_e[k]; v[12 + k] = sum_e2[k]; }
  v[17] = sum_nn;
  v[18] = (double)n_no;
  v[19] = (double)n_no_nn;
  v[20] = (double)n_nc;
  v[21] = sum_c;
  v[22] = max_e;
  v[23] = max_e_nn;
#pragma unroll
  for (int f = 0; f < kSumF; ++f) v[f] = warp_sum(v[f]);
#pragma unroll
  for (int f = kSumF; f < kSumF + kMaxF; ++f) v[f] = warp_max(v[f]);
  double mn = (double)n_corr, mm = 0.0, m2 = 0.0;
  if (n_corr) { mm = shift + s1 / mn; m2 = fmax(0.0, s2 - s1 * (s1 / mn)); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double nb = __shfl_xor_sync(0xffffffffu, mn, o), mb = __shfl_xor_sync(0xffffffffu, mm, o),
                 m2b = __shfl_xor_sync(0xffffffffu, m2, o);
    chan_merge(mn, mm, m2, nb, mb, m2b);
  }
  v[24] = mn; v[25] = mm; v[26] = m2;
  if ((threadIdx.x & 31) == 0) {
    double *out = part + ((long long)blockIdx.x * kWarps + (threadIdx.x >> 5)) * kPart;
#pragma unroll
    for (int f = 0; f < kPart; ++f) out[f] = v[f];
  }
}

// one block of 32 threads: field f of direction q summed (or maxed) over the n_warps partials in order by thread f, the moments
// merged in order by thread kSumF + kMaxF; written where the NN section of the accumulator block keeps them (pack_nn_kernel)
__global__ void surface_merge_kernel(const double *__restrict__ part, long long n_warps, int q, int rank, double *__restrict__ blk) {
  const int f = threadIdx.x;
  double *nn = blk + q * kBlkNN;
  if (f < kSumF) {
    double s = 0.0;
    for (long long w = 0; w < n_warps; ++w) s += part[w * kPart + f];
    const int at = f < 7 ? f : (f < 17 ? f + 2 : (f == 17 ? 21 : -1));     // n_query n_corr n_inlier | sum_d sum_d2 | sum_nn
    if (at >= 0) nn[at] = s;
    else blk[kExtra + 4 * q + (f - 18)] = s;
  } else if (f < kSumF + kMaxF) {
    double m = 0.0;
    for (long long w = 0; w < n_warps; ++w) m = fmax(m, part[w * kPart + f]);
    blk[kMaxOff + 2 * q + (f - kSumF)] = m;
  } else if (f == kSumF + kMaxF) {
    double n = 0, m = 0, m2 = 0;
    for (long long w = 0; w < n_warps; ++w) chan_merge(n, m, m2, part[w * kPart + f], part[w * kPart + f + 1], part[w * kPart + f + 2]);
    nn[19] = n * m;
    nn[20] = m2 + n * m * m;
    nn[kBlkMoments + rank] = n;
    nn[kBlkMoments + ME_MAX_WORLD + rank] = m;
    nn[kBlkMoments + 2 * ME_MAX_WORLD + rank] = m2;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host driver
// ---------------------------------------------------------------------------------------------------------------
void nn_surface_free(me_ctx *ctx) {
  SurfaceRun &S = ctx->surface;
  if (S.d_blk) { cudaFree(S.d_blk); S.d_blk = nullptr; }
  if (S.d_part) { cudaFree(S.d_part); S.d_part = nullptr; S.cap_part = 0; }
  S.open = false;
}

static const char *cloud_name(int w) { return w == ME_CLOUD_EST ? "estimated" : "ground-truth"; }

int nn_surface_begin(me_ctx *ctx, int knn) {
  SurfaceRun &S = ctx->surface;
  S.open = false;
  S.done = false;
  if (ctx->icp.open) return fail(ctx, ME_ERR_INVALID, "me_nn_surface_begin while a registration is open (me_icp_end first)");
  if (ctx->drift.open) return fail(ctx, ME_ERR_INVALID, "me_nn_surface_begin while a drift loop is open (me_drift_end first)");
  ME_TRY(nn_records_fresh(ctx, "me_nn_surface*"));
  for (int w = 0; w < 2; ++w) {
    const Cloud &c = ctx->cloud[w];
    S.had_normals[w] = c.normal_valid;
    S.pending[w] = !c.normal_valid;
    if (c.normal_valid) continue;
    if (knn == 0)
      return fail(ctx, ME_ERR_INVALID, std::string("me_nn_surface_begin: the ") + cloud_name(w) + " cloud has no normals; set them "
                                       "(me_set_normals), estimate them (me_estimate_normals) or pass knn in 1..64");
    // the NN records pin the lattice the sweep laid the cloud out on; a slab holds only part of the cloud
    if (c.slab)
      return fail(ctx, ME_ERR_INVALID, std::string("me_nn_surface_begin: working k-NN normals of the ") + cloud_name(w) +
                                       " cloud need the replicated layout (ME_LAYOUT_REPLICATED); or give the cloud its normals");
  }
  if (!S.d_blk) ME_CUDA(ctx, cudaMalloc((void **)&S.d_blk, (ME_SURFACE_BLOCK_SUM + ME_SURFACE_BLOCK_MAX) * sizeof(double)));
  S.knn = knn;
  S.gen = ctx->cloud_gen;
  S.open = true;
  return ME_OK;
}

static int surface_ready(me_ctx *ctx, const char *who) {
  SurfaceRun &S = ctx->surface;
  if (!S.open) return fail(ctx, ME_ERR_INVALID, std::string(who) + " without an open surface call (me_nn_surface_begin first)");
  if (S.gen != ctx->cloud_gen) {
    S.open = false;
    return fail(ctx, ME_ERR_INVALID, std::string(who) + ": the clouds changed after me_nn_surface_begin; the call is void "
                                     "(run me_eval_nn* and me_nn_surface_begin again)");
  }
  return ME_OK;
}

int nn_surface_normals_slice(me_ctx *ctx, int which, double **d_normals, int64_t *slice_points, int32_t *pending) {
  SurfaceRun &S = ctx->surface;
  *d_normals = nullptr; *slice_points = 0; *pending = 0;
  ME_TRY(surface_ready(ctx, "me_nn_surface_normals_slice"));
  if (S.done) { S.open = false; return fail(ctx, ME_ERR_INVALID, "me_nn_surface_normals_slice after me_nn_surface_block"); }
  if (!S.pending[which]) return ME_OK;
  Cloud &c = ctx->cloud[which];
  // Rank r: caller indices [r s, (r + 1) s), s = ceil(N / world), into the buffer padded to world * s.  The records being
  // fresh, the cloud's lattice is valid and not a solo one, so estimate_normals' build_grid lays nothing out again.
  const long long s = (c.n + ctx->world - 1) / ctx->world, lo = (long long)ctx->rank * s;
  int rc = ctx->world == 1 ? estimate_normals(ctx, which, S.knn) : estimate_normals(ctx, which, S.knn, lo, lo + s, s * ctx->world);
  c.normal_valid = false;            // a working copy: the cloud still has no normals
  if (rc == ME_OK) rc = nn_records_fresh(ctx, "me_nn_surface_normals_slice");
  if (rc != ME_OK) { S.open = false; return rc; }
  S.pending[which] = false;
  *d_normals = c.d_normal; *slice_points = s; *pending = ctx->world > 1 ? 1 : 0;
  return ME_OK;
}

static int surface_fold(me_ctx *ctx) {
  SurfaceRun &S = ctx->surface;
  const me_nn_params *p = &ctx->curve_p;
  const int dirs = p->directions ? p->directions : 3;
  ME_CUDA(ctx, cudaMemsetAsync(S.d_blk, 0, (ME_SURFACE_BLOCK_SUM + ME_SURFACE_BLOCK_MAX) * sizeof(double), ctx->stream));
  const int max_blocks = ctx->sm_count * 4;
  ME_TRY(ensure(ctx, (void **)&S.d_part, &S.cap_part, (long long)max_blocks * kWarps * kPart, sizeof(double)));
  for (int q = 0; q < 2; ++q) {
    if (!(dirs & (1 << q))) continue;
    const Cloud &Qc = ctx->cloud[q], &Rc = ctx->cloud[1 - q];
    const CurveSrc R = record_src(ctx, q);
    if (R.e <= R.b) continue;
    NNConst C{};
    for (int k = 0; k < 5; ++k) C.tau[k] = p->tau[k];
    set_cutoff(C, p);
    C.want_full_cd = p->want_full_cd ? 1 : 0;
    SurfSrc F;
    F.b = R.b; F.e = R.e; F.nb = Qc.nn_b; F.ne = Qc.nn_e;
    F.Q = Qc.d_sorted; F.nn_idx = Qc.d_nn_idx; F.nn_d2 = Qc.d_nn_d2;
    F.q_xyz = Qc.d_xyz; F.r_xyz = Rc.d_xyz; F.q_nrm = Qc.d_normal; F.r_nrm = Rc.d_normal;
    const int n_blocks = (int)std::min<long long>((R.e - R.b + kThreads - 1) / kThreads, max_blocks);
    const long long per_block = (R.e - R.b + n_blocks - 1) / n_blocks;
    surface_fold_kernel<<<n_blocks, kThreads, 0, ctx->stream>>>(F, C, per_block, S.d_part);
    ME_LAUNCH_CHECK(ctx);
    surface_merge_kernel<<<1, 32, 0, ctx->stream>>>(S.d_part, (long long)n_blocks * kWarps, q, ctx->rank, S.d_blk);
    ME_LAUNCH_CHECK(ctx);
  }
  return ME_OK;
}

int nn_surface_block(me_ctx *ctx, double **device_block, int32_t *n_sum, int32_t *n_max) {
  ME_TRY(surface_ready(ctx, "me_nn_surface_block"));
  SurfaceRun &S = ctx->surface;
  if (S.pending[0] || S.pending[1]) {
    S.open = false;
    return fail(ctx, ME_ERR_INVALID, "me_nn_surface_block: working normals are still pending (me_nn_surface_normals_slice for both "
                                     "clouds, all-gathered, first)");
  }
  if (!S.done) {
    const int rc = surface_fold(ctx);
    if (rc != ME_OK) { S.open = false; return rc; }
    S.done = true;
  }
  *device_block = S.d_blk;
  *n_sum = ME_SURFACE_BLOCK_SUM;
  *n_max = ME_SURFACE_BLOCK_MAX;
  return ME_OK;
}

int nn_surface_end(me_ctx *ctx, me_surface_result *out) {
  ME_TRY(surface_ready(ctx, "me_nn_surface_end"));
  SurfaceRun &S = ctx->surface;
  S.open = false;
  if (!S.done) return fail(ctx, ME_ERR_INVALID, "me_nn_surface_end before me_nn_surface_block");
  double h[ME_SURFACE_BLOCK_SUM + ME_SURFACE_BLOCK_MAX];
  ME_CUDA(ctx, cudaMemcpyAsync(h, S.d_blk, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (me_surface_finalize(&ctx->curve_p, h, ctx->cloud[ME_CLOUD_EST].n, ctx->cloud[ME_CLOUD_GT].n, out) != ME_OK)
    return fail(ctx, ME_ERR_INVALID, "me_surface_finalize failed");
  return ME_OK;
}

}  // namespace me

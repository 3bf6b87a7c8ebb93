// icp.cu — the three registration methods of MapEval::performICPRegistration (map_eval.cpp:1366-1394) on top of the
// 1-NN sweep (SURVEY.md §8f N2): registration_methods 0 = point-to-point, 1 = point-to-plane, 2 = generalized ICP (what
// every shipped config uses).
//
// Replaces (reference) open3d::pipelines::registration::RegistrationICP / RegistrationGeneralizedICP(source = est,
// target = gt, icp_max_distance, initial_matrix, estimation, ICPConvergenceCriteria()) [ext, Open3D 0.15-0.17]:
//   pcd = est transformed by init;  result = correspondences(pcd)          (SearchHybrid(p, R, 1): NN kept iff d2 < R^2)
//   loop (max_iteration 30): update = estimation.ComputeTransformation(corr); T = update T; pcd.Transform(update);
//                            backup = result; result = correspondences(pcd);
//                            stop when |d fitness| < 1e-6 and |d inlier_rmse| < 1e-6
//   fitness = |corr| / |est|, inlier_rmse = sqrt(sum d2 / |corr|) (point-to-point quantities for every estimation)
// and afterwards map_3d_ = map_3d_->Transform(trans) on the ORIGINAL cloud (:1392).
//   point-to-point:  Eigen::umeyama without scaling — icp_accum_kernel reduces count, sum p, sum q, sum q p^T, sum d2
//                    (17 doubles); the 3x3 algebra runs on the host.
//   point-to-plane:  r = (vs - vt) . nt, J = [vs x nt, nt]; needs target normals (me_set_normals / me_estimate_normals).
//   generalized:     InitializePointCloudForGeneralizedICP, per cloud: the cloud's normals when it has them (me_set_normals,
//                    me_estimate_normals, averaged by me_voxel_downsample), else EstimateNormals(KNN 20) into a working
//                    buffer (knn_normals_kernel: exact k-NN by ring expansion over the lattice, covariance, Eberly's robust
//                    3x3 eigenvector = Open3D's FastEigen3x3); covariance_i = Rx diag(1e-3, 1, 1) Rx^T with
//                    Rx = GetRotationFromE1ToX(n_i), n_i as given (not normalised; Rx = I when n.x < -0.99, sic), built per
//                    correspondence from the 3 doubles of the normal (gicp_cov); PointCloud::Transform's R C R^T of the
//                    source is R_T C(n_i) R_T^T with R_T the rotation block of the accumulated transformation (T_init
//                    included): the source normals themselves stay as handed in during the loop.
//                    ComputeTransformation: M = Cs + Ct, J = M^-1/2 [-skew(vs) | I], r = M^-1/2 d, i.e. the 6x6 normal
//                    equations sum A^T M^-1 A, sum A^T M^-1 d, reduced on the device (icp_ne_accum_kernel, 28 doubles);
//                    the 6x6 solve and TransformVector6dToMatrix4d run on the host.
// Per iteration: the est lattice is laid out again (the cloud moved), the flat NN sweep finds the correspondences, one
// reduction kernel, one transform.
//
// The loop is split at its only collective (me_icp_begin / _normals_slice / _block / _step / _end): a rank sweeps the query
// range of the cell-sorted moved cloud that query_shard gives it, and its reduction kernel leaves the partial sums as a
// block of fp64 (the count rides as fp64, exact below 2^53) in device memory.  The caller SUM-all-reduces the block in
// place; every rank then runs the same host algebra on the same doubles, so T stays identical on all ranks.  me_icp is the
// same sequence at world = 1 without the collective.  The k-NN normals of generalized ICP shard by caller index: rank r
// estimates [r s, (r + 1) s), s = ceil(N / world), visiting those points in cell-sorted order through a compacted list,
// and the caller all-gathers the slices in place.
#include "common.cuh"
#include "knn_walk.cuh"
#include "svd3.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace me {

static constexpr int kThreads = 256;

// the fp64 block of one sweep: [0] count, then the sums (ME_ICP_BLOCK_P2P / ME_ICP_BLOCK_NE values in all)
static double *icp_block_dev(me_ctx *ctx) { return (double *)((char *)ctx->d_scratch + 2048); }
static double *icp_block_host(me_ctx *ctx) { return (double *)((char *)ctx->h_pinned + 2048); }
static int icp_block_len(int method) { return method == ME_ICP_POINT_TO_POINT ? ME_ICP_BLOCK_P2P : ME_ICP_BLOCK_NE; }

// sums about `c` (a point near the clouds: keeps the magnitudes, and with them the cancellation in sigma, small) over the
// queries [qb, qe) of the cell-sorted cloud; acc = [count, sum p (3), sum q (3), sum q p^T (9, row-major), sum d2]
__global__ void __launch_bounds__(kThreads)
icp_accum_kernel(const P4 *__restrict__ Q, long long qb, long long qe, const int32_t *__restrict__ nn_idx, const double *__restrict__ nn_d2,
                 const double *__restrict__ gt_xyz, double r2, double cx, double cy, double cz, double *__restrict__ acc) {
  double v[17];
#pragma unroll
  for (int k = 0; k < 17; ++k) v[k] = 0.0;
  unsigned long long cnt = 0;
  for (long long i = qb + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < qe; i += (long long)gridDim.x * blockDim.x) {
    const int32_t j = __ldg(nn_idx + i);
    if (j < 0) continue;
    const double d2 = __ldg(nn_d2 + i);
    if (!(d2 < r2)) continue;                              // SearchHybrid: lower_bound(..., radius^2) keeps d2 < R^2
    const P4 p = load_p4(Q + i);
    const double px = p.x - cx, py = p.y - cy, pz = p.z - cz;
    const double qx = __ldg(gt_xyz + 3ll * j) - cx, qy = __ldg(gt_xyz + 3ll * j + 1) - cy, qz = __ldg(gt_xyz + 3ll * j + 2) - cz;
    cnt++;
    v[0] += px; v[1] += py; v[2] += pz; v[3] += qx; v[4] += qy; v[5] += qz;
    v[6] += qx * px; v[7] += qx * py; v[8] += qx * pz;
    v[9] += qy * px; v[10] += qy * py; v[11] += qy * pz;
    v[12] += qz * px; v[13] += qz * py; v[14] += qz * pz;
    v[15] += d2;
  }
  __shared__ double sh[kThreads / 32][17];
  __shared__ unsigned long long shc[kThreads / 32];
#pragma unroll
  for (int k = 0; k < 16; ++k) v[k] = warp_sum(v[k]);
  cnt = (unsigned long long)warp_sum_ll((long long)cnt);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 16; ++k) sh[warp][k] = v[k];
    shc[warp] = cnt;
  }
  __syncthreads();
  if (threadIdx.x < 16) {
    double s = 0;
    for (int w = 0; w < kThreads / 32; ++w) s += sh[w][threadIdx.x];
    if (s != 0.0) atomicAdd(acc + 1 + threadIdx.x, s);
  } else if (threadIdx.x == 32) {
    unsigned long long s = 0;
    for (int w = 0; w < kThreads / 32; ++w) s += shc[w];
    if (s) atomicAdd(acc, (double)s);                      // block counts < 2^53: the fp64 sum is exact
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Open3D FastEigen3x3 (Eberly, "A Robust Eigensolver for 3x3 Symmetric Matrices"): unit eigenvector of the smallest
// eigenvalue of a symmetric 3x3 (row-major, 9 entries); the zero vector for the zero matrix
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cross3d(const double a[3], const double b[3], double o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ double dot3d(const double a[3], const double b[3]) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

__device__ void eberly_evec0(const double A[9], double eval0, double out[3]) {
  const double row0[3] = {A[0] - eval0, A[1], A[2]}, row1[3] = {A[1], A[4] - eval0, A[5]}, row2[3] = {A[2], A[5], A[8] - eval0};
  double r01[3], r02[3], r12[3];
  cross3d(row0, row1, r01); cross3d(row0, row2, r02); cross3d(row1, row2, r12);
  const double d0 = dot3d(r01, r01), d1 = dot3d(r02, r02), d2 = dot3d(r12, r12);
  double dmax = d0; int imax = 0;
  if (d1 > dmax) { dmax = d1; imax = 1; }
  if (d2 > dmax) imax = 2;
  const double s = sqrt(imax == 0 ? d0 : (imax == 1 ? d1 : d2));
#pragma unroll
  for (int k = 0; k < 3; ++k) out[k] = (imax == 0 ? r01[k] : (imax == 1 ? r02[k] : r12[k])) / s;
}
__device__ void eberly_evec1(const double A[9], const double e0[3], double eval1, double out[3]) {
  double U[3], V[3];
  if (fabs(e0[0]) > fabs(e0[1])) {
    const double inv = 1.0 / sqrt(e0[0] * e0[0] + e0[2] * e0[2]);
    U[0] = -e0[2] * inv; U[1] = 0; U[2] = e0[0] * inv;
  } else {
    const double inv = 1.0 / sqrt(e0[1] * e0[1] + e0[2] * e0[2]);
    U[0] = 0; U[1] = e0[2] * inv; U[2] = -e0[1] * inv;
  }
  cross3d(e0, U, V);
  const double AU[3] = {A[0] * U[0] + A[1] * U[1] + A[2] * U[2], A[1] * U[0] + A[4] * U[1] + A[5] * U[2], A[2] * U[0] + A[5] * U[1] + A[8] * U[2]};
  const double AV[3] = {A[0] * V[0] + A[1] * V[1] + A[2] * V[2], A[1] * V[0] + A[4] * V[1] + A[5] * V[2], A[2] * V[0] + A[5] * V[1] + A[8] * V[2]};
  double m00 = dot3d(U, AU) - eval1, m01 = dot3d(U, AV), m11 = dot3d(V, AV) - eval1;
  const double a00 = fabs(m00), a01 = fabs(m01), a11 = fabs(m11);
  if (a00 >= a11) {
    if (fmax(a00, a01) > 0) {
      if (a00 >= a01) { m01 /= m00; m00 = 1 / sqrt(1 + m01 * m01); m01 *= m00; }
      else { m00 /= m01; m01 = 1 / sqrt(1 + m00 * m00); m00 *= m01; }
#pragma unroll
      for (int k = 0; k < 3; ++k) out[k] = m01 * U[k] - m00 * V[k];
    } else {
#pragma unroll
      for (int k = 0; k < 3; ++k) out[k] = U[k];
    }
  } else {
    if (fmax(a11, a01) > 0) {
      if (a11 >= a01) { m01 /= m11; m11 = 1 / sqrt(1 + m01 * m01); m01 *= m11; }
      else { m11 /= m01; m01 = 1 / sqrt(1 + m11 * m11); m11 *= m01; }
#pragma unroll
      for (int k = 0; k < 3; ++k) out[k] = m11 * U[k] - m01 * V[k];
    } else {
#pragma unroll
      for (int k = 0; k < 3; ++k) out[k] = U[k];
    }
  }
}
__device__ void fast_eigen3x3_normal(const double cov[9], double nrm[3]) {
  double max_coeff = cov[0];
#pragma unroll
  for (int k = 1; k < 9; ++k) max_coeff = fmax(max_coeff, cov[k]);
  nrm[0] = nrm[1] = nrm[2] = 0.0;
  if (max_coeff == 0) return;
  double A[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) A[k] = cov[k] / max_coeff;
  const double norm = A[1] * A[1] + A[2] * A[2] + A[5] * A[5];
  if (norm > 0) {
    const double q = (A[0] + A[4] + A[8]) / 3;
    const double b00 = A[0] - q, b11 = A[4] - q, b22 = A[8] - q;
    const double p = sqrt((b00 * b00 + b11 * b11 + b22 * b22 + norm * 2) / 6);
    const double c00 = b11 * b22 - A[5] * A[5], c01 = A[1] * b22 - A[5] * A[2], c02 = A[1] * A[5] - b11 * A[2];
    const double det = (b00 * c00 - A[1] * c01 + A[2] * c02) / (p * p * p);
    const double half_det = fmin(fmax(det * 0.5, -1.0), 1.0);
    const double angle = acos(half_det) / 3.0;
    const double two_thirds_pi = 2.09439510239319549;
    const double beta2 = cos(angle) * 2, beta0 = cos(angle + two_thirds_pi) * 2, beta1 = -(beta0 + beta2);
    const double ev0 = q + p * beta0, ev1 = q + p * beta1, ev2 = q + p * beta2;
    double ea[3], eb[3];
    if (half_det >= 0) {
      eberly_evec0(A, ev2, ea);                                   // ea = evec2
      if (ev2 < ev0 && ev2 < ev1) { nrm[0] = ea[0]; nrm[1] = ea[1]; nrm[2] = ea[2]; return; }
      eberly_evec1(A, ea, ev1, eb);                               // eb = evec1
      if (ev1 < ev0 && ev1 < ev2) { nrm[0] = eb[0]; nrm[1] = eb[1]; nrm[2] = eb[2]; return; }
      cross3d(eb, ea, nrm);                                       // evec0 = evec1 x evec2
    } else {
      eberly_evec0(A, ev0, ea);                                   // ea = evec0
      if (ev0 < ev1 && ev0 < ev2) { nrm[0] = ea[0]; nrm[1] = ea[1]; nrm[2] = ea[2]; return; }
      eberly_evec1(A, ea, ev1, eb);                               // eb = evec1
      if (ev1 < ev0 && ev1 < ev2) { nrm[0] = eb[0]; nrm[1] = eb[1]; nrm[2] = eb[2]; return; }
      cross3d(ea, eb, nrm);                                       // evec2 = evec0 x evec1
    }
  } else {
    if (cov[0] < cov[4] && cov[0] < cov[8]) nrm[0] = 1;
    else if (cov[4] < cov[0] && cov[4] < cov[8]) nrm[1] = 1;
    else nrm[2] = 1;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// PointCloud::EstimateNormals(KDTreeSearchParamKNN(k)) [ext]: per point the k nearest neighbours (the point itself
// included), their covariance, the eigenvector of its smallest eigenvalue.  One thread per point; the k best (d2,
// position) pairs sit sorted in shared memory ([slot][thread]), found by knn_walk (knn_walk.cuh).  Ties go to the
// smaller caller index.
// The queries are the n points of the cell-sorted cloud, or (list != nullptr) the sorted positions list[0 .. n): the
// neighbours, and with them the arithmetic of every normal, do not depend on which points are queried together.
// ---------------------------------------------------------------------------------------------------------------
static constexpr int kKnnThreads = 128;

__global__ void __launch_bounds__(kKnnThreads)
knn_normals_kernel(const P4 *__restrict__ S, long long n, const uint32_t *__restrict__ list, CellIndex I, Lattice L,
                   CoarseGrid CG, int k, double slack, double *__restrict__ normals, unsigned int *trace) {
  extern __shared__ __align__(16) unsigned char knn_smem[];
  double *dk = reinterpret_cast<double *>(knn_smem) + threadIdx.x;                                     // dk[t * kKnnThreads]
  uint32_t *ik = reinterpret_cast<uint32_t *>(knn_smem + (size_t)k * kKnnThreads * sizeof(double)) + threadIdx.x;
  for (long long i = blockIdx.x * (long long)kKnnThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kKnnThreads) {
    const P4 q = load_p4(S + (list ? (long long)__ldg(list + i) : i));
    const int cnt = knn_walk<kKnnThreads>(S, I, L, CG, q, k, slack, INFINITY, false, dk, ik, trace);
    // utility::ComputeCovariance over the neighbours (cumulants about the query point instead of the origin: same
    // covariance, without the cancellation of raw coordinates); fewer than 3 neighbours -> identity
    double cov[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    if (cnt >= 3) {
      double c1[3] = {0, 0, 0}, c2[6] = {0, 0, 0, 0, 0, 0};
      for (int t = 0; t < cnt; ++t) {
        const P4 p = load_p4(S + ik[t * kKnnThreads]);
        const double dx = p.x - q.x, dy = p.y - q.y, dz = p.z - q.z;
        c1[0] += dx; c1[1] += dy; c1[2] += dz;
        c2[0] += dx * dx; c2[1] += dx * dy; c2[2] += dx * dz; c2[3] += dy * dy; c2[4] += dy * dz; c2[5] += dz * dz;
      }
      const double inv = 1.0 / (double)cnt;
#pragma unroll
      for (int a = 0; a < 3; ++a) c1[a] *= inv;
#pragma unroll
      for (int a = 0; a < 6; ++a) c2[a] *= inv;
      cov[0] = c2[0] - c1[0] * c1[0]; cov[4] = c2[3] - c1[1] * c1[1]; cov[8] = c2[5] - c1[2] * c1[2];
      cov[1] = cov[3] = c2[1] - c1[0] * c1[1]; cov[2] = cov[6] = c2[2] - c1[0] * c1[2]; cov[5] = cov[7] = c2[4] - c1[1] * c1[2];
    }
    double nr[3];
    fast_eigen3x3_normal(cov, nr);
    if (sqrt(nr[0] * nr[0] + nr[1] * nr[1] + nr[2] * nr[2]) == 0.0) { nr[0] = 0; nr[1] = 0; nr[2] = 1; }
    const long long o = orig_of(q.idx);
    normals[3 * o] = nr[0]; normals[3 * o + 1] = nr[1]; normals[3 * o + 2] = nr[2];
  }
}

// the sorted positions whose caller index lies in [lo, hi), in sorted order: flag (n + 1 entries, the last 0) -> exclusive
// scan -> compaction
__global__ void __launch_bounds__(kThreads) slice_flag_kernel(const P4 *__restrict__ S, long long n, long long lo, long long hi,
                                                              uint32_t *__restrict__ flag) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i <= n; i += (long long)gridDim.x * blockDim.x) {
    bool in = false;
    if (i < n) {
      const long long o = orig_of(__double_as_longlong(__ldg(reinterpret_cast<const double *>(S + i) + 3)));
      in = o >= lo && o < hi;
    }
    flag[i] = in ? 1u : 0u;
  }
}
__global__ void __launch_bounds__(kThreads) slice_compact_kernel(const uint32_t *__restrict__ pos, long long n,
                                                                 uint32_t *__restrict__ list) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t p = __ldg(pos + i);
    if (__ldg(pos + i + 1) != p) list[p] = (uint32_t)i;
  }
}

// the normals of the points with caller index in [lo, hi) (hi < 0: all of them) into c.d_normal, which holds at least
// `cap_points` normals (the padded buffer of a sharded estimate)
int estimate_normals(me_ctx *ctx, int which, int knn, long long lo, long long hi, long long cap_points) {
  Cloud &c = ctx->cloud[which];
  if (c.n <= 0) return fail(ctx, ME_ERR_EMPTY, "cloud is empty");
  if (knn < 1 || knn > 64) return fail(ctx, ME_ERR_INVALID, "knn must be in 1..64");
  ME_TRY(build_grid(ctx, which, c.grid_valid && c.grid_solo ? c.solo_h : 0.0));
  if (c.slab) return fail(ctx, ME_ERR_INVALID, "me_estimate_normals needs the replicated layout (ME_LAYOUT_REPLICATED)");
  ME_TRY(ensure(ctx, (void **)&c.d_normal, &c.cap_normal, 3 * std::max(c.n, cap_points), sizeof(double)));
  const bool sliced = hi >= 0;
  lo = sliced ? std::min(std::max(lo, 0ll), c.n) : 0;
  hi = sliced ? std::min(std::max(hi, lo), c.n) : c.n;
  const long long nq = hi - lo;
  uint32_t *list = nullptr;
  if (sliced && nq < c.n) {
    ME_TRY(ensure_work(ctx, (size_t)(c.n + 1 + nq) * sizeof(uint32_t)));
    uint32_t *pos = (uint32_t *)ctx->d_work;
    list = pos + c.n + 1;
    const int fb = (int)std::min<long long>((c.n + kThreads) / kThreads, (long long)ctx->sm_count * 16);
    slice_flag_kernel<<<fb, kThreads, 0, ctx->stream>>>(c.d_sorted, c.n, lo, hi, pos);
    ME_LAUNCH_CHECK(ctx);
    ME_TRY(exclusive_scan_inplace(ctx, pos, c.n + 1));
    slice_compact_kernel<<<fb, kThreads, 0, ctx->stream>>>(pos, c.n, list);
    ME_LAUNCH_CHECK(ctx);
  }
  if (nq > 0) {
    const int k = (int)std::min<long long>(knn, c.n);
    const size_t smem = (size_t)k * kKnnThreads * (sizeof(double) + sizeof(uint32_t));
    if (smem > 48 * 1024)
      ME_CUDA(ctx, cudaFuncSetAttribute(knn_normals_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    double maxabs = 0;
    for (int a = 0; a < 3; ++a) maxabs = std::max(maxabs, std::max(std::fabs(c.bbox_min[a]), std::fabs(c.bbox_max[a])));
    const double slack = 1e-9 * c.lat.h + 4e-14 * maxabs;
    const int blocks = (int)std::min<long long>((nq + kKnnThreads - 1) / kKnnThreads, (long long)ctx->sm_count * 32);
    knn_normals_kernel<<<blocks, kKnnThreads, smem, ctx->stream>>>(c.d_sorted, nq, list, index_of(c), c.lat, coarse_of(c), k,
                                                                   slack, c.d_normal, ctx->d_trace);
    ME_LAUNCH_CHECK(ctx);
  }
  c.normal_valid = true;
  return ME_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// normal equations of point-to-plane (method 1) and generalized ICP (method 2) over the kept correspondences of the
// queries [qb, qe): acc = [count, v] with v[0..20] the upper triangle of JTJ (row-major), v[21..26] JTr, v[27] sum d2
// ---------------------------------------------------------------------------------------------------------------
struct Mat9 { double r[9]; };

// GetRotationFromE1ToX(x) diag(eps, 1, 1) GetRotationFromE1ToX(x)^T with x as given (Open3D does not normalise it):
// Rx = I + [v]x + [v]x^2 / (1 + c), v = e1 x x = (0, -x2, x1), c = x0, written out; Rx = I when c < -0.99.  When R is
// given, the covariance is rotated: (R Rx) diag(eps, 1, 1) (R Rx)^T.  C: upper triangle xx xy xz yy yz zz.
__device__ __forceinline__ void gicp_cov(const double x[3], double eps, const double *R, double C[6]) {
  double Q[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0};
  if (!(x[0] < -0.99)) {
    const double f = 1.0 / (1.0 + x[0]), fxy = f * x[1] * x[2];
    Q[0] = 1.0 - f * (x[1] * x[1] + x[2] * x[2]); Q[1] = -x[1];                 Q[2] = -x[2];
    Q[3] = x[1];                                  Q[4] = 1.0 - f * x[1] * x[1]; Q[5] = -fxy;
    Q[6] = x[2];                                  Q[7] = -fxy;                  Q[8] = 1.0 - f * x[2] * x[2];
  }
  if (R) {
    double P[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int col = 0; col < 3; ++col) P[r * 3 + col] = R[r * 3] * Q[col] + R[r * 3 + 1] * Q[3 + col] + R[r * 3 + 2] * Q[6 + col];
#pragma unroll
    for (int k = 0; k < 9; ++k) Q[k] = P[k];
  }
  int t = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = a; b < 3; ++b) C[t++] = eps * Q[a * 3] * Q[b * 3] + Q[a * 3 + 1] * Q[b * 3 + 1] + Q[a * 3 + 2] * Q[b * 3 + 2];
}

__global__ void __launch_bounds__(kThreads)
icp_ne_accum_kernel(const P4 *__restrict__ Q, long long qb, long long qe, const int32_t *__restrict__ nn_idx,
                    const double *__restrict__ nn_d2, const double *__restrict__ gt_xyz, const double *__restrict__ gt_nrm,
                    const double *__restrict__ est_nrm, Mat9 Rs, double r2, double eps, int method, double *__restrict__ acc) {
  double v[28];
#pragma unroll
  for (int k = 0; k < 28; ++k) v[k] = 0.0;
  unsigned long long cnt = 0;
  for (long long i = qb + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < qe; i += (long long)gridDim.x * blockDim.x) {
    const int32_t j = __ldg(nn_idx + i);
    if (j < 0) continue;
    const double d2 = __ldg(nn_d2 + i);
    if (!(d2 < r2)) continue;                              // SearchHybrid keeps d2 < R^2
    const P4 p = load_p4(Q + i);
    const double vs[3] = {p.x, p.y, p.z};
    const double d[3] = {p.x - __ldg(gt_xyz + 3ll * j), p.y - __ldg(gt_xyz + 3ll * j + 1), p.z - __ldg(gt_xyz + 3ll * j + 2)};
    const double nt[3] = {__ldg(gt_nrm + 3ll * j), __ldg(gt_nrm + 3ll * j + 1), __ldg(gt_nrm + 3ll * j + 2)};
    cnt++;
    v[27] += d2;
    if (method == ME_ICP_POINT_TO_PLANE) {
      double J[6];
      cross3d(vs, nt, J);
      J[3] = nt[0]; J[4] = nt[1]; J[5] = nt[2];
      const double r = dot3d(d, nt);
      int t = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a) {
#pragma unroll
        for (int b = a; b < 6; ++b) v[t++] += J[a] * J[b];
        v[21 + a] += J[a] * r;
      }
    } else {
      const long long o = orig_of(p.idx);
      const double ns[3] = {__ldg(est_nrm + 3 * o), __ldg(est_nrm + 3 * o + 1), __ldg(est_nrm + 3 * o + 2)};
      // M = Cs + Ct with Cs = Rs C(ns) Rs^T; B = M^-1 (symmetric, by cofactors)
      double cs[6], ct[6];
      gicp_cov(ns, eps, Rs.r, cs);
      gicp_cov(nt, eps, nullptr, ct);
      const double m00 = cs[0] + ct[0], m01 = cs[1] + ct[1], m02 = cs[2] + ct[2];
      const double m11 = cs[3] + ct[3], m12 = cs[4] + ct[4], m22 = cs[5] + ct[5];
      const double c00 = m11 * m22 - m12 * m12, c01 = m02 * m12 - m01 * m22, c02 = m01 * m12 - m02 * m11;
      const double c11 = m00 * m22 - m02 * m02, c12 = m01 * m02 - m00 * m12, c22 = m00 * m11 - m01 * m01;
      const double idet = 1.0 / (m00 * c00 + m01 * c01 + m02 * c02);
      const double B[9] = {c00 * idet, c01 * idet, c02 * idet, c01 * idet, c11 * idet, c12 * idet, c02 * idet, c12 * idet, c22 * idet};
      // A = [-skew(vs) | I] (3 x 6), BA = B A, JTJ = A^T B A, JTr = A^T B d
      const double A[18] = {0.0, vs[2], -vs[1], 1.0, 0.0, 0.0, -vs[2], 0.0, vs[0], 0.0, 1.0, 0.0, vs[1], -vs[0], 0.0, 0.0, 0.0, 1.0};
      double BA[18], g[3];
#pragma unroll
      for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int col = 0; col < 6; ++col) BA[r * 6 + col] = B[r * 3] * A[col] + B[r * 3 + 1] * A[6 + col] + B[r * 3 + 2] * A[12 + col];
        g[r] = B[r * 3] * d[0] + B[r * 3 + 1] * d[1] + B[r * 3 + 2] * d[2];
      }
      int t = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a) {
#pragma unroll
        for (int b = a; b < 6; ++b) v[t++] += A[a] * BA[b] + A[6 + a] * BA[6 + b] + A[12 + a] * BA[12 + b];
        v[21 + a] += A[a] * g[0] + A[6 + a] * g[1] + A[12 + a] * g[2];
      }
    }
  }
  __shared__ double sh[kThreads / 32][28];
  __shared__ unsigned long long shc[kThreads / 32];
#pragma unroll
  for (int k = 0; k < 28; ++k) v[k] = warp_sum(v[k]);
  cnt = (unsigned long long)warp_sum_ll((long long)cnt);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 28; ++k) sh[warp][k] = v[k];
    shc[warp] = cnt;
  }
  __syncthreads();
  if (threadIdx.x < 28) {
    double s = 0;
    for (int w2 = 0; w2 < kThreads / 32; ++w2) s += sh[w2][threadIdx.x];
    if (s != 0.0) atomicAdd(acc + 1 + threadIdx.x, s);
  } else if (threadIdx.x == 32) {
    unsigned long long s = 0;
    for (int w2 = 0; w2 < kThreads / 32; ++w2) s += shc[w2];
    if (s) atomicAdd(acc, (double)s);
  }
}

// symmetric 6x6 solve (Open3D: JTJ.ldlt().solve(-JTr)); Gaussian elimination with partial pivoting
static bool solve6_host(const double A_in[36], const double b_in[6], double x[6]) {
  double A[36], b[6];
  std::memcpy(A, A_in, sizeof(A)); std::memcpy(b, b_in, sizeof(b));
  for (int c = 0; c < 6; ++c) {
    int piv = c;
    for (int r = c + 1; r < 6; ++r) if (std::fabs(A[r * 6 + c]) > std::fabs(A[piv * 6 + c])) piv = r;
    if (A[piv * 6 + c] == 0.0) return false;
    if (piv != c) { for (int k = 0; k < 6; ++k) std::swap(A[c * 6 + k], A[piv * 6 + k]); std::swap(b[c], b[piv]); }
    for (int r = c + 1; r < 6; ++r) {
      const double f = A[r * 6 + c] / A[c * 6 + c];
      for (int k = c; k < 6; ++k) A[r * 6 + k] -= f * A[c * 6 + k];
      b[r] -= f * b[c];
    }
  }
  for (int r = 5; r >= 0; --r) {
    double s = b[r];
    for (int k = r + 1; k < 6; ++k) s -= A[r * 6 + k] * x[k];
    x[r] = s / A[r * 6 + r];
  }
  for (int k = 0; k < 6; ++k) if (!std::isfinite(x[k])) return false;
  return true;
}
// utility::TransformVector6dToMatrix4d: Rz(x2) Ry(x1) Rx(x0), translation x[3..5]
static void vec6_to_mat4_host(const double x[6], double T[16]) {
  const double ca = std::cos(x[0]), sa = std::sin(x[0]), cb = std::cos(x[1]), sb = std::sin(x[1]), cg = std::cos(x[2]), sg = std::sin(x[2]);
  const double Rx[9] = {1, 0, 0, 0, ca, -sa, 0, sa, ca}, Ry[9] = {cb, 0, sb, 0, 1, 0, -sb, 0, cb}, Rz[9] = {cg, -sg, 0, sg, cg, 0, 0, 0, 1};
  double t[9], R[9];
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) t[r * 3 + c] = Rz[r * 3] * Ry[c] + Rz[r * 3 + 1] * Ry[3 + c] + Rz[r * 3 + 2] * Ry[6 + c];
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) R[r * 3 + c] = t[r * 3] * Rx[c] + t[r * 3 + 1] * Rx[3 + c] + t[r * 3 + 2] * Rx[6 + c];
  for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) T[r * 4 + c] = R[r * 3 + c]; T[r * 4 + 3] = x[3 + r]; }
  T[12] = T[13] = T[14] = 0; T[15] = 1;
}

// the update of one iteration from a reduced block: Umeyama (point-to-point, sums about c) or the 6x6 solve +
// TransformVector6dToMatrix4d; the identity when there are no correspondences or the solve fails (Open3D)
void icp_update_host(int method, const double *blk, const double c[3], double upd[16]) {
  static const double I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  std::memcpy(upd, I, sizeof(I));
  if (!(blk[0] > 0)) return;
  if (method == ME_ICP_POINT_TO_POINT) { umeyama_from_sums(blk, c, upd); return; }
  const double *v = blk + 1;
  double JTJ[36], nb[6], x[6];
  int t = 0;
  for (int a = 0; a < 6; ++a)
    for (int b = a; b < 6; ++b) { JTJ[a * 6 + b] = v[t]; JTJ[b * 6 + a] = v[t]; ++t; }
  for (int a = 0; a < 6; ++a) nb[a] = -v[21 + a];
  if (solve6_host(JTJ, nb, x)) vec6_to_mat4_host(x, upd);
}

// every failure of an open registration closes it: the estimated cloud (and its normals) come back as they were handed in
void icp_close(me_ctx *ctx, bool restore) {
  IcpRun &S = ctx->icp;
  if (!S.open) return;
  Cloud &E = ctx->cloud[ME_CLOUD_EST], &G = ctx->cloud[ME_CLOUD_GT];
  if (restore && S.orig && E.d_xyz == S.xyz && E.n == S.n_est)
    cudaMemcpyAsync(E.d_xyz, S.orig, (size_t)E.n * 3 * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream);
  invalidate_cloud(E);
  E.normal_valid = S.had_normals[ME_CLOUD_EST];      // the working normals of generalized ICP do not outlive the call
  G.normal_valid = S.had_normals[ME_CLOUD_GT];
  cudaStreamSynchronize(ctx->stream);
  if (S.orig) cudaFree(S.orig);
  S = IcpRun();
}
static int icp_fail(me_ctx *ctx, int rc) {
  icp_close(ctx, true);
  return rc;
}

int icp_begin(me_ctx *ctx, int method, double max_dist, int max_iter, double rel_fitness, double rel_rmse, const double T_init[16]) {
  if (ctx->icp.open) return icp_fail(ctx, fail(ctx, ME_ERR_INVALID, "me_icp_begin while a registration is open (me_icp_end first)"));
  Cloud &E = ctx->cloud[ME_CLOUD_EST], &G = ctx->cloud[ME_CLOUD_GT];
  if (E.n <= 0 || G.n <= 0) return fail(ctx, ME_ERR_EMPTY, "both clouds must be set (map_eval.cpp:32-35)");
  if (method != ME_ICP_POINT_TO_POINT && method != ME_ICP_POINT_TO_PLANE && method != ME_ICP_GENERALIZED)
    return fail(ctx, ME_ERR_INVALID, "Invalid registration type specified (map_eval.cpp:1387)");
  if (!E.owned) return fail(ctx, ME_ERR_INVALID, "me_icp needs a library-owned estimated cloud (use me_set_cloud)");
  if (!(max_dist > 0) || max_iter < 0) return fail(ctx, ME_ERR_INVALID, "bad ICP parameters");
  if (method == ME_ICP_POINT_TO_PLANE && !G.normal_valid)
    return fail(ctx, ME_ERR_INVALID, "TransformationEstimationPointToPlane requires pre-computed normal vectors for the target "
                                     "PointCloud (me_set_normals / me_estimate_normals on the ground-truth cloud)");
  if (ctx->world > 1 && ctx->slab_request)
    return fail(ctx, ME_ERR_INVALID, "registration needs the replicated layout: me_set_layout(ME_LAYOUT_REPLICATED) before "
                                     "me_icp_begin, ME_LAYOUT_SLAB again afterwards");
  ME_TRY(wait_upload(ctx, ME_CLOUD_EST));
  IcpRun &S = ctx->icp;
  S = IcpRun();
  // the original cloud: RegistrationICP iterates on a copy, the caller's cloud is transformed once at the end (:1392)
  ME_TRY(ensure(ctx, (void **)&S.orig, &S.cap_orig, 3 * E.n, sizeof(double)));
  S.open = true;
  S.xyz = E.d_xyz; S.n_est = E.n;
  S.method = method; S.max_iter = max_iter; S.max_dist = max_dist; S.rel_fitness = rel_fitness; S.rel_rmse = rel_rmse;
  std::memcpy(S.T, T_init, sizeof(S.T));
  for (int w = 0; w < 2; ++w) {
    S.had_normals[w] = ctx->cloud[w].normal_valid;
    // InitializePointCloudForGeneralizedICP per cloud: the cloud's own normals, else EstimateNormals(KNN 20)
    S.normals_pending[w] = method == ME_ICP_GENERALIZED && !S.had_normals[w];
  }
  if (cudaMemcpyAsync(S.orig, E.d_xyz, (size_t)E.n * 3 * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream) != cudaSuccess)
    return icp_fail(ctx, fail(ctx, ME_ERR_CUDA, "copy of the estimated cloud failed"));
  return ME_OK;
}

int icp_normals_slice(me_ctx *ctx, int which, double **d_normals, int64_t *slice_points, int32_t *pending) {
  IcpRun &S = ctx->icp;
  *d_normals = nullptr; *slice_points = 0; *pending = 0;
  if (!S.open) return fail(ctx, ME_ERR_INVALID, "me_icp_normals_slice before me_icp_begin");
  if (S.swept) return icp_fail(ctx, fail(ctx, ME_ERR_INVALID, "me_icp_normals_slice after the first me_icp_block"));
  if (!S.normals_pending[which]) return ME_OK;      // the cloud's own normals, or a method without source covariances
  Cloud &c = ctx->cloud[which];
  // estimated before the initial transform, as Open3D does; into the cloud's normal buffer as a working copy that stays
  // invalid afterwards.  Rank r: caller indices [r s, (r + 1) s), s = ceil(N / world), the buffer padded to world * s.
  const long long s = (c.n + ctx->world - 1) / ctx->world, lo = (long long)ctx->rank * s;
  int rc = build_both(ctx);
  if (rc == ME_OK) rc = ctx->world == 1 ? estimate_normals(ctx, which, 20) : estimate_normals(ctx, which, 20, lo, lo + s, s * ctx->world);
  c.normal_valid = false;
  if (rc != ME_OK) return icp_fail(ctx, rc);
  S.normals_pending[which] = false;
  *d_normals = c.d_normal; *slice_points = s; *pending = ctx->world > 1 ? 1 : 0;
  return ME_OK;
}

// one correspondence sweep of the moved cloud and this rank's partial sums into the block
static int icp_sweep(me_ctx *ctx) {
  IcpRun &S = ctx->icp;
  Cloud &E = ctx->cloud[ME_CLOUD_EST], &G = ctx->cloud[ME_CLOUD_GT];
  me_nn_params p;
  std::memset(&p, 0, sizeof(p));
  p.icp_max_distance = S.max_dist;
  p.cutoff_mode = ME_CUTOFF_DIST_LT_R;
  p.pairing = ME_PAIRING_GEOMETRIC;
  p.want_full_cd = 0;
  p.directions = 1;
  ME_TRY(run_nn(ctx, &p, false));      // lays the moved cloud out again, then sweeps this rank's queries
  const long long qb = E.nn_b, qe = E.nn_e;
  const int blocks = (int)std::max(1ll, std::min<long long>((qe - qb + kThreads - 1) / kThreads, (long long)ctx->sm_count * 8));
  double *blk = icp_block_dev(ctx);
  ME_CUDA(ctx, cudaMemsetAsync(blk, 0, ME_ICP_BLOCK_NE * sizeof(double), ctx->stream));
  const double r2 = S.max_dist * S.max_dist;
  if (S.method == ME_ICP_POINT_TO_POINT) {
    for (int a = 0; a < 3; ++a) S.c[a] = 0.5 * (G.bbox_min[a] + G.bbox_max[a]);
    icp_accum_kernel<<<blocks, kThreads, 0, ctx->stream>>>(E.d_sorted, qb, qe, E.d_nn_idx, E.d_nn_d2, G.d_xyz, r2, S.c[0], S.c[1],
                                                          S.c[2], blk);
  } else {
    Mat9 R;      // rotation block of the accumulated transformation: the source covariances are R C(n) R^T
    for (int r = 0; r < 3; ++r)
      for (int col = 0; col < 3; ++col) R.r[r * 3 + col] = S.T[r * 4 + col];
    const double eps = 1e-3;      // TransformationEstimationForGeneralizedICP() default epsilon
    icp_ne_accum_kernel<<<blocks, kThreads, 0, ctx->stream>>>(E.d_sorted, qb, qe, E.d_nn_idx, E.d_nn_d2, G.d_xyz, G.d_normal,
                                                             E.d_normal, R, r2, eps, S.method, blk);
  }
  ME_LAUNCH_CHECK(ctx);
  return ME_OK;
}

static int icp_ready(me_ctx *ctx, const char *call) {
  IcpRun &S = ctx->icp;
  if (!S.open) return fail(ctx, ME_ERR_INVALID, std::string(call) + " before me_icp_begin");
  const Cloud &E = ctx->cloud[ME_CLOUD_EST];
  if (E.d_xyz != S.xyz || E.n != S.n_est)
    return icp_fail(ctx, fail(ctx, ME_ERR_INVALID, std::string(call) + ": the estimated cloud was replaced during the registration"));
  if (S.normals_pending[0] || S.normals_pending[1])
    return icp_fail(ctx, fail(ctx, ME_ERR_INVALID, std::string(call) + ": the k-NN normals of generalized ICP are still pending "
                                                   "(me_icp_normals_slice for both clouds, all-gathered, first)"));
  return ME_OK;
}

int icp_block(me_ctx *ctx, double **d_block, int32_t *n_sum) {
  ME_TRY(icp_ready(ctx, "me_icp_block"));
  IcpRun &S = ctx->icp;
  if (!S.swept) {      // the initial sweep: pcd = est transformed by init, result = correspondences(pcd)
    Cloud &E = ctx->cloud[ME_CLOUD_EST];
    E.normal_valid = false;      // the estimated cloud's normals stay as handed in while the copy moves
    int rc = transform_cloud(ctx, ME_CLOUD_EST, S.T);
    if (rc == ME_OK) rc = icp_sweep(ctx);
    if (rc != ME_OK) return icp_fail(ctx, rc);
    S.swept = true;
  }
  *d_block = icp_block_dev(ctx);
  *n_sum = icp_block_len(S.method);
  return ME_OK;
}

int icp_step(me_ctx *ctx, int32_t *done) {
  *done = 0;
  ME_TRY(icp_ready(ctx, "me_icp_step"));
  IcpRun &S = ctx->icp;
  if (!S.swept) return icp_fail(ctx, fail(ctx, ME_ERR_INVALID, "me_icp_step before the first me_icp_block"));
  if (S.done) { *done = 1; return ME_OK; }
  const int nb = icp_block_len(S.method);
  double *h = icp_block_host(ctx);
  if (cudaMemcpyAsync(h, icp_block_dev(ctx), nb * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
      cudaStreamSynchronize(ctx->stream) != cudaSuccess)
    return icp_fail(ctx, fail(ctx, ME_ERR_CUDA, "reading the ICP block failed"));
  double blk[ME_ICP_BLOCK_NE];
  std::memcpy(blk, h, nb * sizeof(double));
  const double n_est = (double)ctx->cloud[ME_CLOUD_EST].n;
  S.n_corr = (long long)std::llround(blk[0]);
  const double fitness = (double)S.n_corr / n_est;
  const double rmse = S.n_corr > 0 ? std::sqrt(blk[nb - 1] / (double)S.n_corr) : 0.0;
  if (S.have_prev) {      // the block of an update: ICPConvergenceCriteria
    ++S.it;
    if (std::fabs(S.fitness - fitness) < S.rel_fitness && std::fabs(S.rmse - rmse) < S.rel_rmse) S.converged = 1;
  }
  S.fitness = fitness; S.rmse = rmse; S.have_prev = true;
  if (S.converged || S.it >= S.max_iter) { S.done = true; *done = 1; return ME_OK; }
  double upd[16], Tn[16];
  icp_update_host(S.method, blk, S.c, upd);
  for (int r = 0; r < 4; ++r)
    for (int col = 0; col < 4; ++col) { double s = 0; for (int k = 0; k < 4; ++k) s += upd[r * 4 + k] * S.T[k * 4 + col]; Tn[r * 4 + col] = s; }
  std::memcpy(S.T, Tn, sizeof(Tn));
  int rc = transform_cloud(ctx, ME_CLOUD_EST, upd);
  if (rc == ME_OK) rc = icp_sweep(ctx);
  if (rc != ME_OK) return icp_fail(ctx, rc);
  return ME_OK;
}

int icp_end(me_ctx *ctx, me_icp_result *out) {
  std::memset(out, 0, sizeof(*out));
  IcpRun &S = ctx->icp;
  if (!S.open) return fail(ctx, ME_ERR_INVALID, "me_icp_end without me_icp_begin");
  if (!S.have_prev) return icp_fail(ctx, fail(ctx, ME_ERR_INVALID, "me_icp_end before the first me_icp_step"));
  // est := Transform(original, T) (map_eval.cpp:1392), normals handed in included
  double T[16];
  std::memcpy(T, S.T, sizeof(T));
  out->fitness = S.fitness; out->inlier_rmse = S.rmse; out->n_corr = (int64_t)S.n_corr;
  out->iterations = S.it; out->converged = S.converged;
  std::memcpy(out->transformation, T, sizeof(T));
  icp_close(ctx, true);
  int rc = transform_cloud(ctx, ME_CLOUD_EST, T);
  if (rc == ME_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess) rc = fail(ctx, ME_ERR_CUDA, "synchronize after ICP failed");
  if (rc != ME_OK) std::memset(out, 0, sizeof(*out));
  return rc;
}

int run_icp(me_ctx *ctx, int method, double max_dist, int max_iter, double rel_fitness, double rel_rmse, const double T_init[16],
            me_icp_result *out) {
  std::memset(out, 0, sizeof(*out));
  if (ctx->world != 1) return fail(ctx, ME_ERR_INVALID, "me_icp needs world == 1 (the update needs all correspondences; "
                                                        "use me_icp_begin .. me_icp_end with an all-reduce per iteration)");
  // the split loop without its collectives: at world = 1 the normals need no gather and the block no reduction
  ME_TRY(icp_begin(ctx, method, max_dist, max_iter, rel_fitness, rel_rmse, T_init));
  double *d = nullptr;
  int64_t s = 0;
  int32_t pending = 0, n_sum = 0, done = 0;
  ME_TRY(icp_normals_slice(ctx, ME_CLOUD_EST, &d, &s, &pending));
  ME_TRY(icp_normals_slice(ctx, ME_CLOUD_GT, &d, &s, &pending));
  ME_TRY(icp_block(ctx, &d, &n_sum));
  while (!done) ME_TRY(icp_step(ctx, &done));
  return icp_end(ctx, out);
}

}  // namespace me

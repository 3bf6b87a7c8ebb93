// globalreg.cu — coarse global registration (me_global_registration): the initial pose est -> gt from the maps alone, for
// users who would otherwise align the two maps by hand and copy the matrix into the configuration's initial_matrix.
//
// Stages, all on the device, on two private feature clouds (me_ctx::cloud[kFeatureSlot + which]) so that the context's
// clouds, normals, lattices and per-point results stay as they were:
//   1. copy + me_voxel_downsample at voxel_size; exact k-NN normals (estimate_normals, knn_normals_kernel) on a solo lattice
//      of cell edge feature_radius / 2; orient_kernel flips n where n . (v - p) < 0, v = centroid + (0, 0, 10 * bbox diagonal).
//      FastEigen3x3 leaves a sign that is a function of the covariance entries and does not turn with the map, and mixed
//      signs inside a neighbourhood ruin the descriptor; the viewpoint gives floors and terrain +z and walls a side set by
//      the map's own centroid, both of which move with a yaw of the map.
//   2. fpfh_spfh_kernel / fpfh_kernel, one thread per point: the neighbourhood is knn_walk with a radius bound (<= max_nn
//      nearest other points with d^2 < r^2, ties to the smaller index); Open3D's ComputePairFeatures, 11 bins per group over
//      f0 in [-pi, pi], f1, f2 in [-1, 1] (clamped), increments 100 / k; FPFH = SPFH + the neighbours' SPFH weighted by
//      1 / d^2, normalised to 100 per group.  fp64 throughout, stored as fp32.  The swap of ComputePairFeatures,
//      acos|a1| > acos|a2|, is evaluated as |a1| < |a2| (acos is decreasing): no acos rounding decides it.
//   3. feature_nn_kernel: exact fp32 nearest neighbour in descriptor space, both directions; squared distances summed in
//      dimension order with __fsub_rn / __fmul_rn / __fadd_rn, ties to the smaller index (numpy rounds the same operations).
//      Mutual filter, then flag / scan / compact into the correspondence list (est order).
//   4. ransac_kernel, one warp per hypothesis h: correspondences min(floor(uniform53(seed, h, 16 + t) * n), n - 1), t < 3
//      (rng.cuh); rejected when two coincide, an edge fails min^2 >= ratio^2 max^2, or the three are (nearly) collinear
//      (w1 <= 1e-6 w0 of their cross-covariance); otherwise the rigid fit of the three
//      (umeyama_from_sums, svd3.cuh, every lane the same arithmetic) and the inliers |R p + t - q|^2 < d^2 counted by the
//      lanes.  One packed atomicMax picks the most inliers, ties to the smallest h.  No early exit.
//   5. refinement: the winner's inliers flagged, scanned and compacted; their point-to-point sums reduced by ONE block in a
//      fixed order (bit-reproducible), umeyama_from_sums on the host; n_inliers and inlier_rmse under that T, likewise.
// This file is compiled without fused multiply-adds (Makefile): every operation rounds on its own, so the hypotheses, their
// inlier counts and the winner equal a numpy statement of the same operations (tests/fpfh_ref.py).
#include "common.cuh"
#include "knn_walk.cuh"
#include "rng.cuh"
#include "svd3.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace me {

static constexpr int kThreads = 256;
static constexpr int kFeat = 33;                 // FPFH dimensions: 3 groups of 11 bins
static constexpr int kFpfhThreads = 64;          // threads per block of the FPFH kernels (neighbour slots in shared memory)
static constexpr int kMaxFeatureNN = 128;
static constexpr int kNnThreads = 128;           // feature_nn_kernel: queries per block = descriptors per shared tile
static constexpr double kPi = 3.141592653589793;
static constexpr int kLaneDraw = 16;             // RANSAC draws: lanes 16, 17, 18 (rng.cuh)
static constexpr double kRankEps = 1e-6;         // a hypothesis' second singular value must exceed this share of the first

// ---- stage 1: centroid and orientation ----------------------------------------------------------------------------
// one block, fixed order: the sum of every thread's strided points, then a fixed tree (the result does not depend on timing)
__global__ void __launch_bounds__(kThreads) centroid_kernel(const double *__restrict__ xyz, long long n, double *__restrict__ out) {
  __shared__ double sh[3][kThreads];
  double s[3] = {0.0, 0.0, 0.0};
  for (long long i = threadIdx.x; i < n; i += kThreads)
    for (int a = 0; a < 3; ++a) s[a] += xyz[3 * i + a];
  for (int a = 0; a < 3; ++a) sh[a][threadIdx.x] = s[a];
  __syncthreads();
  for (int w = kThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w)
      for (int a = 0; a < 3; ++a) sh[a][threadIdx.x] += sh[a][threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x < 3) out[threadIdx.x] = sh[threadIdx.x][0] / (double)n;
}

// flip n where n . (v - p) < 0, v = centroid + (0, 0, lift)
__global__ void __launch_bounds__(kThreads) orient_kernel(const double *__restrict__ xyz, double *__restrict__ nrm, long long n,
                                                          const double *__restrict__ centroid, double lift) {
  const double vx = centroid[0], vy = centroid[1], vz = centroid[2] + lift;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double nx = nrm[3 * i], ny = nrm[3 * i + 1], nz = nrm[3 * i + 2];
    const double d = nx * (vx - xyz[3 * i]) + ny * (vy - xyz[3 * i + 1]) + nz * (vz - xyz[3 * i + 2]);
    if (d < 0.0) { nrm[3 * i] = -nx; nrm[3 * i + 1] = -ny; nrm[3 * i + 2] = -nz; }
  }
}

// ---- stage 2: FPFH ------------------------------------------------------------------------------------------------
// Open3D ComputePairFeatures: (f0, f1, f2) = (atan2(w . n2, n1 . n2), v . n2, n1 . d / |d|) in the Darboux frame of the
// pair, the frame on the point whose normal makes the smaller angle with the line; zeros when the points coincide or n1
// is parallel to the line.  Norms and dots in Eigen's order for three components: x*x + (y*y + z*z).
__device__ __forceinline__ double dot3e(const double a[3], const double b[3]) { return a[0] * b[0] + (a[1] * b[1] + a[2] * b[2]); }
__device__ __forceinline__ void pair_features(const double p1[3], const double n1[3], const double p2[3], const double n2[3],
                                              double f[3]) {
  f[0] = f[1] = f[2] = 0.0;
  double dp[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  const double len = sqrt(dot3e(dp, dp));
  if (len == 0.0) return;
  const double a1 = dot3e(n1, dp) / len, a2 = dot3e(n2, dp) / len;
  const double *m1 = n1, *m2 = n2;
  double f2;
  if (fabs(a1) < fabs(a2)) {       // acos(|a1|) > acos(|a2|)
    m1 = n2; m2 = n1;
    dp[0] = -dp[0]; dp[1] = -dp[1]; dp[2] = -dp[2];
    f2 = -a2;
  } else {
    f2 = a1;
  }
  double v[3] = {dp[1] * m1[2] - dp[2] * m1[1], dp[2] * m1[0] - dp[0] * m1[2], dp[0] * m1[1] - dp[1] * m1[0]};
  const double vn = sqrt(dot3e(v, v));
  if (vn == 0.0) return;
  v[0] /= vn; v[1] /= vn; v[2] /= vn;
  const double w[3] = {m1[1] * v[2] - m1[2] * v[1], m1[2] * v[0] - m1[0] * v[2], m1[0] * v[1] - m1[1] * v[0]};
  f[1] = dot3e(v, m2);
  f[0] = atan2(dot3e(w, m2), dot3e(m1, m2));
  f[2] = f2;
}
__device__ __forceinline__ int bin_of(double t) {      // floor, clamped to the 11 bins
  const int h = (int)floor(t);
  return h < 0 ? 0 : (h > 10 ? 10 : h);
}
__device__ __forceinline__ void pair_bins(const double f[3], int b[3]) {
  b[0] = bin_of(11.0 * (f[0] + kPi) / (2.0 * kPi));
  b[1] = 11 + bin_of(11.0 * (f[1] + 1.0) * 0.5);
  b[2] = 22 + bin_of(11.0 * (f[2] + 1.0) * 0.5);
}

struct FeatGeom {
  const P4 *S; CellIndex I; Lattice L; CoarseGrid CG;
  const double *nrm;      // caller order
  int k; double slack, r2;
  unsigned int *trace;    // me_kernel_trace's device word (ME_TEV_KNN_COARSE)
};

// the neighbourhood of sorted point s into this thread's slots; returns its size
__device__ __forceinline__ int feature_neighbours(const FeatGeom &G, long long s, P4 &q, double *dk, uint32_t *ik) {
  q = load_p4(G.S + s);
  return knn_walk<kFpfhThreads>(G.S, G.I, G.L, G.CG, q, G.k, G.slack, G.r2, true, dk, ik, G.trace);
}

__global__ void __launch_bounds__(kFpfhThreads) fpfh_spfh_kernel(FeatGeom G, long long n, double *__restrict__ spfh) {
  extern __shared__ __align__(16) unsigned char fpfh_smem[];
  double *dk = reinterpret_cast<double *>(fpfh_smem) + threadIdx.x;
  uint32_t *ik = reinterpret_cast<uint32_t *>(fpfh_smem + (size_t)G.k * kFpfhThreads * sizeof(double)) + threadIdx.x;
  for (long long s = blockIdx.x * (long long)kFpfhThreads + threadIdx.x; s < n; s += (long long)gridDim.x * kFpfhThreads) {
    P4 q;
    const int cnt = feature_neighbours(G, s, q, dk, ik);
    const long long o = orig_of(q.idx);
    double h[kFeat];
#pragma unroll
    for (int b = 0; b < kFeat; ++b) h[b] = 0.0;
    if (cnt > 0) {
      const double inc = 100.0 / (double)cnt;
      const double p1[3] = {q.x, q.y, q.z}, n1[3] = {G.nrm[3 * o], G.nrm[3 * o + 1], G.nrm[3 * o + 2]};
      for (int t = 0; t < cnt; ++t) {
        const P4 p = load_p4(G.S + ik[t * kFpfhThreads]);
        const long long j = orig_of(p.idx);
        const double p2[3] = {p.x, p.y, p.z}, n2[3] = {G.nrm[3 * j], G.nrm[3 * j + 1], G.nrm[3 * j + 2]};
        double f[3];
        int bb[3];
        pair_features(p1, n1, p2, n2, f);
        pair_bins(f, bb);
        h[bb[0]] += inc; h[bb[1]] += inc; h[bb[2]] += inc;
      }
    }
#pragma unroll
    for (int b = 0; b < kFeat; ++b) spfh[kFeat * o + b] = h[b];
  }
}

__global__ void __launch_bounds__(kFpfhThreads) fpfh_kernel(FeatGeom G, long long n, const double *__restrict__ spfh,
                                                            float *__restrict__ fpfh) {
  extern __shared__ __align__(16) unsigned char fpfh_smem[];
  double *dk = reinterpret_cast<double *>(fpfh_smem) + threadIdx.x;
  uint32_t *ik = reinterpret_cast<uint32_t *>(fpfh_smem + (size_t)G.k * kFpfhThreads * sizeof(double)) + threadIdx.x;
  for (long long s = blockIdx.x * (long long)kFpfhThreads + threadIdx.x; s < n; s += (long long)gridDim.x * kFpfhThreads) {
    P4 q;
    const int cnt = feature_neighbours(G, s, q, dk, ik);
    const long long o = orig_of(q.idx);
    double h[kFeat], sum[3] = {0.0, 0.0, 0.0};
#pragma unroll
    for (int b = 0; b < kFeat; ++b) h[b] = 0.0;
    for (int t = 0; t < cnt; ++t) {
      const double d2 = dk[t * kFpfhThreads];
      if (d2 == 0.0) continue;
      const long long j = orig_of(load_p4(G.S + ik[t * kFpfhThreads]).idx);
#pragma unroll
      for (int b = 0; b < kFeat; ++b) {
        const double val = __ldg(spfh + kFeat * j + b) / d2;
        sum[b / 11] += val;
        h[b] += val;
      }
    }
#pragma unroll
    for (int g = 0; g < 3; ++g) sum[g] = sum[g] != 0.0 ? 100.0 / sum[g] : 0.0;
#pragma unroll
    for (int b = 0; b < kFeat; ++b) fpfh[kFeat * o + b] = (float)(h[b] * sum[b / 11] + __ldg(spfh + kFeat * o + b));
  }
}

// ---- stage 3: matching --------------------------------------------------------------------------------------------
// nn[i] = argmin_j |Qd_i - Rd_j|^2, one thread per query, its descriptor in registers; the reference descriptors stream
// through shared memory one tile of kNnThreads at a time (every thread reads the same word: a broadcast)
__global__ void __launch_bounds__(kNnThreads) feature_nn_kernel(const float *__restrict__ Qd, long long nq, const float *__restrict__ Rd,
                                                                long long nr, int32_t *__restrict__ nn) {
  __shared__ float tile[kNnThreads * kFeat];
  const long long i = blockIdx.x * (long long)kNnThreads + threadIdx.x;
  float qv[kFeat];
#pragma unroll
  for (int b = 0; b < kFeat; ++b) qv[b] = i < nq ? __ldg(Qd + kFeat * i + b) : 0.0f;
  float best = INFINITY;
  long long bi = -1;
  for (long long t0 = 0; t0 < nr; t0 += kNnThreads) {
    const int m = (int)min((long long)kNnThreads, nr - t0);
    __syncthreads();
    for (int e = threadIdx.x; e < m * kFeat; e += kNnThreads) tile[e] = __ldg(Rd + kFeat * t0 + e);
    __syncthreads();
    for (int j = 0; j < m; ++j) {
      float d = 0.0f;
#pragma unroll
      for (int b = 0; b < kFeat; ++b) {
        const float t = __fsub_rn(qv[b], tile[j * kFeat + b]);
        d = __fadd_rn(d, __fmul_rn(t, t));
      }
      if (d < best) { best = d; bi = t0 + j; }
    }
  }
  if (i < nq) nn[i] = (int32_t)bi;
}

// flag[i] = est point i keeps its pair (its nearest gt descriptor, whose nearest est descriptor is i when mutual); flag[n] = 0
__global__ void __launch_bounds__(kThreads) corr_flag_kernel(const int32_t *__restrict__ e2g, const int32_t *__restrict__ g2e, long long n,
                                                             int mutual, uint32_t *__restrict__ flag) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i <= n; i += (long long)gridDim.x * blockDim.x) {
    if (i == n) { flag[n] = 0u; continue; }
    const int32_t j = e2g[i];
    flag[i] = (j >= 0 && (!mutual || g2e[j] == (int32_t)i)) ? 1u : 0u;
  }
}
// correspondence k = (est i, gt e2g[i]) for the flagged i, in est order: indices and both points
__global__ void __launch_bounds__(kThreads) corr_compact_kernel(const uint32_t *__restrict__ pos, const int32_t *__restrict__ e2g, long long n,
                                                                const double *__restrict__ exyz, const double *__restrict__ gxyz,
                                                                int32_t *__restrict__ ce, int32_t *__restrict__ cg, double *__restrict__ P,
                                                                double *__restrict__ Q) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t k = pos[i];
    if (pos[i + 1] == k) continue;
    const int32_t j = e2g[i];
    ce[k] = (int32_t)i; cg[k] = j;
#pragma unroll
    for (int a = 0; a < 3; ++a) { P[3ll * k + a] = exyz[3 * i + a]; Q[3ll * k + a] = gxyz[3ll * j + a]; }
  }
}

// ---- stage 4: RANSAC ----------------------------------------------------------------------------------------------
struct RansacArgs {
  const double *P, *Q;          // correspondences: est point, gt point
  long long nc, nh;
  unsigned long long key[3];    // lane keys of lanes 16, 17, 18
  double ratio2, d2max;
  double c[3];                  // the sums of a fit are taken about c (centre of the gt feature cloud's bounding box)
};

__device__ __forceinline__ long long draw_corr(const RansacArgs &A, long long h, int t) {
  const double b = floor(uniform53(A.key[t], h, kLaneDraw + t) * (double)A.nc);
  return b < (double)(A.nc - 1) ? (long long)b : A.nc - 1;
}
__device__ __forceinline__ double sqdist3(const double *a, const double *b) {
  const double dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
  return dx * dx + dy * dy + dz * dz;
}
// hypothesis h: false when rejected, else its rigid fit T (row-major 4x4)
__device__ bool hypothesis(const RansacArgs &A, long long h, double T[16]) {
  long long id[3];
  for (int t = 0; t < 3; ++t) id[t] = draw_corr(A, h, t);
  if (id[0] == id[1] || id[0] == id[2] || id[1] == id[2]) return false;
  for (int a = 0; a < 2; ++a)
    for (int b = a + 1; b < 3; ++b) {      // CorrespondenceCheckerBasedOnEdgeLength on squared lengths
      const double ds = sqdist3(A.P + 3 * id[a], A.P + 3 * id[b]), dt = sqdist3(A.Q + 3 * id[a], A.Q + 3 * id[b]);
      const double lo = ds < dt ? ds : dt, hi = ds < dt ? dt : ds;
      if (!(lo >= A.ratio2 * hi)) return false;
    }
  double blk[ME_ICP_BLOCK_P2P];
  for (int k = 0; k < ME_ICP_BLOCK_P2P; ++k) blk[k] = 0.0;
  blk[0] = 3.0;
  for (int t = 0; t < 3; ++t) {
    const double *p = A.P + 3 * id[t], *q = A.Q + 3 * id[t];
    const double pc[3] = {p[0] - A.c[0], p[1] - A.c[1], p[2] - A.c[2]}, qc[3] = {q[0] - A.c[0], q[1] - A.c[1], q[2] - A.c[2]};
    for (int a = 0; a < 3; ++a) { blk[1 + a] += pc[a]; blk[4 + a] += qc[a]; }
    for (int r = 0; r < 3; ++r)
      for (int col = 0; col < 3; ++col) blk[7 + 3 * r + col] += qc[r] * pc[col];
  }
  double sv[3];
  umeyama_from_sums(blk, A.c, T, sv);
  return sv[1] > kRankEps * sv[0];      // (nearly) collinear triples have no unique rotation
}
// |T p - q|^2, the rows of T applied left to right
__device__ __forceinline__ double residual2(const double T[16], const double *p, const double *q) {
  const double x = T[0] * p[0] + T[1] * p[1] + T[2] * p[2] + T[3] - q[0];
  const double y = T[4] * p[0] + T[5] * p[1] + T[6] * p[2] + T[7] - q[1];
  const double z = T[8] * p[0] + T[9] * p[1] + T[10] * p[2] + T[11] - q[2];
  return x * x + y * y + z * z;
}

// best = max over valid h of ((inliers + 1) << 32) | (2^32 - 1 - h): the most inliers, then the smallest h
__global__ void __launch_bounds__(kThreads) ransac_kernel(RansacArgs A, unsigned long long *__restrict__ best,
                                                          unsigned long long *__restrict__ n_valid) {
  const int lane = threadIdx.x & 31;
  const long long w0 = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, ws = ((long long)gridDim.x * blockDim.x) >> 5;
  unsigned long long valid = 0;
  for (long long h = w0; h < A.nh; h += ws) {
    double T[16];
    if (!hypothesis(A, h, T)) continue;      // the same decision on every lane
    long long cnt = 0;
    for (long long k = lane; k < A.nc; k += 32) cnt += residual2(T, A.P + 3 * k, A.Q + 3 * k) < A.d2max ? 1 : 0;
    cnt = warp_sum_ll(cnt);
    if (lane == 0) atomicMax(best, ((unsigned long long)(cnt + 1) << 32) | (0xffffffffull - (unsigned long long)h));
    ++valid;
  }
  if (lane == 0 && valid) atomicAdd(n_valid, valid);
}

// ---- stage 5: refinement ------------------------------------------------------------------------------------------
// the winner's fit (the same function the warps ran) and its inlier flags; flag[nc] = 0
__global__ void __launch_bounds__(kThreads) winner_flag_kernel(RansacArgs A, long long h, double *__restrict__ Tw, uint32_t *__restrict__ flag) {
  double T[16];
  hypothesis(A, h, T);
  if (blockIdx.x == 0 && threadIdx.x < 16) Tw[threadIdx.x] = T[threadIdx.x];
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k <= A.nc; k += (long long)gridDim.x * blockDim.x)
    flag[k] = k < A.nc && residual2(T, A.P + 3 * k, A.Q + 3 * k) < A.d2max ? 1u : 0u;
}
__global__ void __launch_bounds__(kThreads) inlier_compact_kernel(const uint32_t *__restrict__ pos, long long n, uint32_t *__restrict__ list) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x)
    if (pos[k + 1] != pos[k]) list[pos[k]] = (uint32_t)k;
}

// one block, fixed order.  mode 0: point-to-point sums about c over the listed correspondences into out[0..16]
// (ME_ICP_BLOCK_P2P layout); mode 1: out[0] = inliers of T among all correspondences, out[1] = sum of their |T p - q|^2
static constexpr int kSumVals = ME_ICP_BLOCK_P2P;
struct Mat16Arg { double t[16]; };
__global__ void __launch_bounds__(kThreads) ordered_sums_kernel(const double *__restrict__ P, const double *__restrict__ Q,
                                                                const uint32_t *__restrict__ list, long long n, int mode, Mat16Arg T,
                                                                double cx, double cy, double cz, double d2max, double *__restrict__ out) {
  __shared__ double sh[kSumVals][kThreads];
  double v[kSumVals];
  for (int k = 0; k < kSumVals; ++k) v[k] = 0.0;
  for (long long i = threadIdx.x; i < n; i += kThreads) {
    if (mode == 0) {
      const long long k = list[i];
      const double pc[3] = {P[3 * k] - cx, P[3 * k + 1] - cy, P[3 * k + 2] - cz};
      const double qc[3] = {Q[3 * k] - cx, Q[3 * k + 1] - cy, Q[3 * k + 2] - cz};
      v[0] += 1.0;
      for (int a = 0; a < 3; ++a) { v[1 + a] += pc[a]; v[4 + a] += qc[a]; }
      for (int r = 0; r < 3; ++r)
        for (int col = 0; col < 3; ++col) v[7 + 3 * r + col] += qc[r] * pc[col];
    } else {
      const double d2 = residual2(T.t, P + 3 * i, Q + 3 * i);
      if (d2 < d2max) { v[0] += 1.0; v[1] += d2; }
    }
  }
  for (int k = 0; k < kSumVals; ++k) sh[k][threadIdx.x] = v[k];
  __syncthreads();
  for (int w = kThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w)
      for (int k = 0; k < kSumVals; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x < kSumVals) out[threadIdx.x] = sh[threadIdx.x][0];
}

// ---- host ---------------------------------------------------------------------------------------------------------
static int grid_blocks(const me_ctx *ctx, long long n, int threads = kThreads) {
  return (int)std::max(1ll, std::min<long long>((n + threads - 1) / threads, (long long)ctx->sm_count * 16));
}
static double slack_of(const Cloud &c) {
  double maxabs = 0;
  for (int a = 0; a < 3; ++a) maxabs = std::max(maxabs, std::max(std::fabs(c.bbox_min[a]), std::fabs(c.bbox_max[a])));
  return 1e-9 * c.lat.h + 4e-14 * maxabs;
}

// stage 1 and 2 for one cloud: feature cloud, oriented normals, FPFH into ctx->d_fpfh[which]
// stage times of a call: event pairs [begin, end) summed per stage (me_global_reg_result.stage_ms)
struct RegTimer {
  cudaStream_t s;
  static constexpr int kMax = 16;      // intervals per call: 3 per cloud, then matching, RANSAC, refinement
  cudaEvent_t ev[2 * kMax] = {};
  int stage_of[kMax] = {};
  int n = 0;
  explicit RegTimer(cudaStream_t st) : s(st) {}
  ~RegTimer() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }
  void begin(int stage) {
    if (n >= kMax) return;
    if (!ev[2 * n]) { cudaEventCreate(&ev[2 * n]); cudaEventCreate(&ev[2 * n + 1]); }
    stage_of[n] = stage;
    cudaEventRecord(ev[2 * n], s);
  }
  void end() { if (n < kMax) cudaEventRecord(ev[2 * n + 1], s), ++n; }
  void read(double ms[6]) {      // after a synchronisation of the stream
    for (int k = 0; k < 6; ++k) ms[k] = 0.0;
    for (int i = 0; i < n; ++i) {
      float t = 0.f;
      if (cudaEventElapsedTime(&t, ev[2 * i], ev[2 * i + 1]) == cudaSuccess) ms[stage_of[i]] += t;
      else cudaGetLastError();
    }
  }
};

static int features_of(me_ctx *ctx, int which, const me_global_reg_params *p, RegTimer &tm) {
  const int slot = kFeatureSlot + which;
  Cloud &c = ctx->cloud[slot];
  tm.begin(0);
  ME_TRY(copy_cloud(ctx, which, slot, false));      // the feature cloud's normals are its own k-NN normals
  int64_t nf = 0;
  ME_TRY(voxel_downsample(ctx, slot, p->voxel_size, &nf));
  tm.end();
  tm.begin(1);
  ME_TRY(build_grid(ctx, slot, 0.5 * p->feature_radius));
  ME_TRY(estimate_normals(ctx, slot, p->normal_knn));
  // orientation: viewpoint above the centroid by ten bounding-box diagonals
  double diag2 = 0;
  for (int a = 0; a < 3; ++a) diag2 += (c.bbox_max[a] - c.bbox_min[a]) * (c.bbox_max[a] - c.bbox_min[a]);
  double *d_cen = (double *)((char *)ctx->d_scratch + 3072);
  centroid_kernel<<<1, kThreads, 0, ctx->stream>>>(c.d_xyz, c.n, d_cen);
  ME_LAUNCH_CHECK(ctx);
  orient_kernel<<<grid_blocks(ctx, c.n), kThreads, 0, ctx->stream>>>(c.d_xyz, c.d_normal, c.n, d_cen, 10.0 * std::sqrt(diag2));
  ME_LAUNCH_CHECK(ctx);
  tm.end();
  // FPFH
  tm.begin(2);
  FeatGeom G;
  G.S = c.d_sorted; G.I = index_of(c); G.L = c.lat; G.CG = coarse_of(c); G.nrm = c.d_normal;
  G.k = p->feature_max_nn; G.slack = slack_of(c); G.r2 = p->feature_radius * p->feature_radius;
  G.trace = ctx->d_trace;
  ME_TRY(ensure_work(ctx, (size_t)c.n * kFeat * sizeof(double)));
  double *spfh = (double *)ctx->d_work;
  ME_TRY(ensure(ctx, (void **)&ctx->d_fpfh[which], &ctx->cap_fpfh[which], c.n * kFeat, sizeof(float)));
  const size_t smem = (size_t)G.k * kFpfhThreads * (sizeof(double) + sizeof(uint32_t));
  ME_CUDA(ctx, cudaFuncSetAttribute(fpfh_spfh_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ME_CUDA(ctx, cudaFuncSetAttribute(fpfh_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int fb = (int)std::min<long long>((c.n + kFpfhThreads - 1) / kFpfhThreads, (long long)ctx->sm_count * 32);
  fpfh_spfh_kernel<<<fb, kFpfhThreads, smem, ctx->stream>>>(G, c.n, spfh);
  ME_LAUNCH_CHECK(ctx);
  fpfh_kernel<<<fb, kFpfhThreads, smem, ctx->stream>>>(G, c.n, spfh, ctx->d_fpfh[which]);
  ME_LAUNCH_CHECK(ctx);
  tm.end();
  return ME_OK;
}

static int reg_fail(me_ctx *ctx, const std::string &msg) { return fail(ctx, ME_ERR_INVALID, "me_global_registration: " + msg); }

int global_registration(me_ctx *ctx, const me_global_reg_params *p, me_global_reg_result *out) {
  std::memset(out, 0, sizeof(*out));
  if (!(std::isfinite(p->voxel_size) && p->voxel_size > 0)) return reg_fail(ctx, "voxel_size must be finite and > 0");
  if (p->normal_knn < 3 || p->normal_knn > 64) return reg_fail(ctx, "normal_knn must be in 3..64");
  if (!(std::isfinite(p->feature_radius) && p->feature_radius > 0)) return reg_fail(ctx, "feature_radius must be finite and > 0");
  if (p->feature_max_nn < 1 || p->feature_max_nn > kMaxFeatureNN) return reg_fail(ctx, "feature_max_nn must be in 1..128");
  if (!(std::isfinite(p->max_correspondence_distance) && p->max_correspondence_distance > 0))
    return reg_fail(ctx, "max_correspondence_distance must be finite and > 0");
  if (!(p->edge_ratio >= 0 && p->edge_ratio <= 1)) return reg_fail(ctx, "edge_ratio must be in [0, 1]");
  if (p->n_hypotheses < 1 || p->n_hypotheses > 0xffffffffll) return reg_fail(ctx, "n_hypotheses must be in 1..2^32-1");
  if (ctx->cloud[ME_CLOUD_EST].n <= 0 || ctx->cloud[ME_CLOUD_GT].n <= 0)
    return fail(ctx, ME_ERR_EMPTY, "me_global_registration: both clouds must be set");
  ctx->features_valid = false;
  ctx->n_corr = 0;
  RegTimer tm(ctx->stream);
  ME_TRY(features_of(ctx, ME_CLOUD_EST, p, tm));
  ME_TRY(features_of(ctx, ME_CLOUD_GT, p, tm));
  ctx->features_valid = true;
  const Cloud &E = ctx->cloud[kFeatureSlot + ME_CLOUD_EST], &G = ctx->cloud[kFeatureSlot + ME_CLOUD_GT];
  const long long ne = E.n, ng = G.n;
  out->n_est_features = ne; out->n_gt_features = ng;

  // stage 3: work = e2g | g2e | pos (ne + 1) | ce | cg | P | Q | flag (ne + 1) | list (ne)
  auto align = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t o_g2e = align((size_t)ne * 4), o_pos = o_g2e + align((size_t)ng * 4), o_ce = o_pos + align((size_t)(ne + 1) * 4),
               o_cg = o_ce + align((size_t)ne * 4), o_P = o_cg + align((size_t)ne * 4), o_Q = o_P + align((size_t)ne * 24),
               o_flag = o_Q + align((size_t)ne * 24), o_list = o_flag + align((size_t)(ne + 1) * 4), total = o_list + align((size_t)ne * 4);
  ME_TRY(ensure_work(ctx, total));
  char *base = (char *)ctx->d_work;
  int32_t *e2g = (int32_t *)base, *g2e = (int32_t *)(base + o_g2e), *ce = (int32_t *)(base + o_ce), *cg = (int32_t *)(base + o_cg);
  uint32_t *pos = (uint32_t *)(base + o_pos), *flag = (uint32_t *)(base + o_flag), *list = (uint32_t *)(base + o_list);
  double *P = (double *)(base + o_P), *Q = (double *)(base + o_Q);
  tm.begin(3);
  feature_nn_kernel<<<(unsigned)((ne + kNnThreads - 1) / kNnThreads), kNnThreads, 0, ctx->stream>>>(ctx->d_fpfh[0], ne, ctx->d_fpfh[1], ng, e2g);
  ME_LAUNCH_CHECK(ctx);
  feature_nn_kernel<<<(unsigned)((ng + kNnThreads - 1) / kNnThreads), kNnThreads, 0, ctx->stream>>>(ctx->d_fpfh[1], ng, ctx->d_fpfh[0], ne, g2e);
  ME_LAUNCH_CHECK(ctx);
  corr_flag_kernel<<<grid_blocks(ctx, ne + 1), kThreads, 0, ctx->stream>>>(e2g, g2e, ne, p->mutual_filter ? 1 : 0, pos);
  ME_LAUNCH_CHECK(ctx);
  ME_TRY(exclusive_scan_inplace(ctx, pos, ne + 1));
  corr_compact_kernel<<<grid_blocks(ctx, ne), kThreads, 0, ctx->stream>>>(pos, e2g, ne, E.d_xyz, G.d_xyz, ce, cg, P, Q);
  ME_LAUNCH_CHECK(ctx);
  tm.end();
  uint32_t *h32 = (uint32_t *)ctx->h_pinned;
  ME_CUDA(ctx, cudaMemcpyAsync(h32, pos + ne, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const long long nc = (long long)h32[0];
  out->n_correspondences = nc;
  // kept for me_get_correspondences
  ME_TRY(ensure(ctx, (void **)&ctx->d_corr, &ctx->cap_corr, 2 * std::max(nc, 1ll), sizeof(int32_t)));
  ME_CUDA(ctx, cudaMemcpyAsync(ctx->d_corr, ce, (size_t)nc * sizeof(int32_t), cudaMemcpyDeviceToDevice, ctx->stream));
  ME_CUDA(ctx, cudaMemcpyAsync(ctx->d_corr + nc, cg, (size_t)nc * sizeof(int32_t), cudaMemcpyDeviceToDevice, ctx->stream));
  ctx->n_corr = nc;
  if (nc < 3) return reg_fail(ctx, "fewer than 3 feature correspondences (" + std::to_string(nc) + ")");

  // stage 4
  RansacArgs A;
  A.P = P; A.Q = Q; A.nc = nc; A.nh = p->n_hypotheses;
  for (int t = 0; t < 3; ++t) A.key[t] = lane_key(p->seed, kLaneDraw + t);
  A.ratio2 = p->edge_ratio * p->edge_ratio;
  A.d2max = p->max_correspondence_distance * p->max_correspondence_distance;
  for (int a = 0; a < 3; ++a) A.c[a] = 0.5 * (G.bbox_min[a] + G.bbox_max[a]);
  unsigned long long *d_best = (unsigned long long *)((char *)ctx->d_scratch + 3072);
  ME_CUDA(ctx, cudaMemsetAsync(d_best, 0, 2 * sizeof(unsigned long long), ctx->stream));
  const int rb = (int)std::min<long long>((A.nh * 32 + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
  tm.begin(4);
  ransac_kernel<<<rb, kThreads, 0, ctx->stream>>>(A, d_best, d_best + 1);
  ME_LAUNCH_CHECK(ctx);
  tm.end();
  unsigned long long *h64 = (unsigned long long *)ctx->h_pinned;
  ME_CUDA(ctx, cudaMemcpyAsync(h64, d_best, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const unsigned long long best = h64[0];
  out->n_valid_hypotheses = (int64_t)h64[1];
  if (out->n_valid_hypotheses == 0)
    return reg_fail(ctx, "no valid RANSAC hypothesis (every draw repeated a correspondence, failed the edge-length check or was "
                         "collinear)");
  const long long hw = (long long)(0xffffffffull - (best & 0xffffffffull));
  out->best_hypothesis = hw;

  // stage 5
  double *d_sums = (double *)((char *)ctx->d_scratch + 3072);
  double *d_T = d_sums + 32;
  tm.begin(5);
  winner_flag_kernel<<<grid_blocks(ctx, nc + 1), kThreads, 0, ctx->stream>>>(A, hw, d_T, flag);
  ME_LAUNCH_CHECK(ctx);
  ME_TRY(exclusive_scan_inplace(ctx, flag, nc + 1));
  inlier_compact_kernel<<<grid_blocks(ctx, nc), kThreads, 0, ctx->stream>>>(flag, nc, list);
  ME_LAUNCH_CHECK(ctx);
  double *h = (double *)ctx->h_pinned;
  ME_CUDA(ctx, cudaMemcpyAsync(h32, flag + nc, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaMemcpyAsync(h + 32, d_T, 16 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const long long n_win = (long long)h32[0];
  double T[16];
  std::memcpy(T, h + 32, sizeof(T));
  Mat16Arg M;
  std::memcpy(M.t, T, sizeof(T));
  if (n_win >= 3) {      // the rigid fit over the winner's inliers; with fewer the hypothesis' own fit stays
    ordered_sums_kernel<<<1, kThreads, 0, ctx->stream>>>(P, Q, list, n_win, 0, M, A.c[0], A.c[1], A.c[2], 0.0, d_sums);
    ME_LAUNCH_CHECK(ctx);
    ME_CUDA(ctx, cudaMemcpyAsync(h, d_sums, kSumVals * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    double blk[kSumVals];
    std::memcpy(blk, h, sizeof(blk));
    umeyama_from_sums(blk, A.c, T);
  }
  std::memcpy(M.t, T, sizeof(T));
  ordered_sums_kernel<<<1, kThreads, 0, ctx->stream>>>(P, Q, nullptr, nc, 1, M, 0.0, 0.0, 0.0, A.d2max, d_sums);
  ME_LAUNCH_CHECK(ctx);
  ME_CUDA(ctx, cudaMemcpyAsync(h, d_sums, 2 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  std::memcpy(out->T, T, sizeof(T));
  out->n_inliers = (int64_t)std::llround(h[0]);
  out->inlier_rmse = out->n_inliers > 0 ? std::sqrt(h[1] / (double)out->n_inliers) : 0.0;
  tm.end();
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  tm.read(out->stage_ms);
  return ME_OK;
}

int get_correspondences(me_ctx *ctx, int32_t *est_idx, int32_t *gt_idx, int64_t capacity, int64_t *n) {
  if (n) *n = ctx->n_corr;
  if (!est_idx && !gt_idx) return ME_OK;
  if (capacity < ctx->n_corr) return fail(ctx, ME_ERR_INVALID, "me_get_correspondences: host buffers too small");
  if (ctx->n_corr > 0) {
    if (est_idx) ME_CUDA(ctx, cudaMemcpyAsync(est_idx, ctx->d_corr, (size_t)ctx->n_corr * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    if (gt_idx) ME_CUDA(ctx, cudaMemcpyAsync(gt_idx, ctx->d_corr + ctx->n_corr, (size_t)ctx->n_corr * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return ME_OK;
}

int get_features(me_ctx *ctx, int which, double *xyz, double *normals, float *fpfh33, int64_t capacity, int64_t *n) {
  if (!ctx->features_valid) return fail(ctx, ME_ERR_INVALID, "me_get_features: no me_global_registration has computed features");
  const Cloud &c = ctx->cloud[kFeatureSlot + which];
  if (n) *n = c.n;
  if (!xyz && !normals && !fpfh33) return ME_OK;
  if (capacity < c.n) return fail(ctx, ME_ERR_INVALID, "me_get_features: host buffers too small");
  if (xyz) ME_CUDA(ctx, cudaMemcpyAsync(xyz, c.d_xyz, (size_t)c.n * 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  if (normals) ME_CUDA(ctx, cudaMemcpyAsync(normals, c.d_normal, (size_t)c.n * 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  if (fpfh33) ME_CUDA(ctx, cudaMemcpyAsync(fpfh33, ctx->d_fpfh[which], (size_t)c.n * kFeat * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return ME_OK;
}

}  // namespace me

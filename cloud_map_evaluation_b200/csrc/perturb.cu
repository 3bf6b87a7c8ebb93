// perturb.cu — degraded copies of the ground truth: the simulation operators of the reference (MapEval::addGaussianNoise,
// addNonUniformDensity, addSparseOutliers, addLocalDeformation, map_eval.cpp:1745-1829) on a cloud held by the context.
//
// The reference draws from std::random_device, so no run of it can be repeated.  Here every draw is the counter-based hash
// of synth.py — splitmix64 of (seed, index, lane) — so a degraded map is a pure function of (cloud, parameters, seed): the
// same on every GPU of a job without communication, and its integer structure (kept points, outlier bases) equal bit for bit
// to the numpy statement in tests/perturb_ref.py.  Lanes (disjoint, so one seed serves all four operators and the RANSAC
// draws of global registration; the helpers live in rng.cuh):
//   noise          gaussian(seed, i, 2a), a = x, y, z        lanes 0-5
//   density        uniform24(seed, i, 6)                     lane 6
//   outliers       uniform53(seed, j, 7) for the base,       lane 7
//                  gaussian(seed, j, 8 + 2a) for the offset  lanes 8-13
//   (globalreg.cu) uniform53(seed, h, 16 + t), t = 0, 1, 2   lanes 16-18: the three correspondences of hypothesis h
// uniform24 = (h >> 40) * 2^-24 in fp32 (synth.uniform24), uniform53 = (h >> 11) * 2^-53, gaussian = Box-Muller in fp64 with
// u1 = max(u24, 2^-25) (synth.gaussian).  The final multiply-adds are rounded separately (__dmul_rn / __dadd_rn), as numpy
// and the reference round them; only the device's log / cos / sin differ from the host's libm, by an ulp or two.
//
// After every operator the cloud's lattice, plan and per-point results are stale (invalidate_cloud), as after me_transform.
// Borrowed clouds (me_set_cloud_device) are refused: the operators never write caller memory.
#include "common.cuh"
#include "rng.cuh"
#include <algorithm>
#include <cmath>

namespace me {

static constexpr int kThreads = 256;
static constexpr double kPi = 3.141592653589793;          // M_PI
static constexpr double kTwoPi = 6.283185307179586;       // 2.0 * np.pi, rounded once as numpy forms it

struct LaneKeys { unsigned long long k[14]; };
static LaneKeys lane_keys(uint64_t seed) {
  LaneKeys L;
  for (int l = 0; l < 14; ++l) L.k[l] = lane_key(seed, l);
  return L;
}

// synth.gaussian: sqrt(-2 log u1) * cos(2 pi u2) from lanes (lane, lane + 1)
__device__ __forceinline__ double gaussian(const LaneKeys &L, long long idx, int lane) {
  const double u1 = fmax(uniform24(L.k[lane], idx, lane), 0x1p-25);
  const double u2 = uniform24(L.k[lane + 1], idx, lane + 1);
  return __dmul_rn(sqrt(__dmul_rn(-2.0, log(u1))), cos(__dmul_rn(kTwoPi, u2)));
}

// blocks of a grid-stride launch over n items: a multiple of the SM count, at most 16 blocks per SM
static int stream_blocks(const me_ctx *ctx, long long n) {
  const long long want = (n + kThreads - 1) / kThreads;
  const long long per_sm = std::min<long long>(16, std::max<long long>(1, (want + ctx->sm_count - 1) / ctx->sm_count));
  return (int)(per_sm * ctx->sm_count);
}

// ---- kernels --------------------------------------------------------------------------------------------------------

// addGaussianNoise (:1745-1755): p_a += sigma * N(0, 1), in place
__global__ void __launch_bounds__(kThreads) noise_kernel(double *__restrict__ xyz, long long n, double sigma, LaneKeys L) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
#pragma unroll
    for (int a = 0; a < 3; ++a) xyz[3 * i + a] = __dadd_rn(xyz[3 * i + a], __dmul_rn(sigma, gaussian(L, i, 2 * a)));
  }
}

// addNonUniformDensity (:1757-1784): flag[i] = keep; flag[n] = 0, so that the exclusive scan leaves the kept count there
__global__ void __launch_bounds__(kThreads) density_flag_kernel(const double *__restrict__ xyz, long long n, double sparse_ratio,
                                                                double dense_ratio, double region_size, unsigned long long key,
                                                                uint32_t *__restrict__ flag) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i <= n; i += (long long)gridDim.x * blockDim.x) {
    if (i == n) { flag[n] = 0u; continue; }
    // sin(point(0) / region_size * M_PI): the division first, then the product
    const double xn = sin(__dmul_rn(__ddiv_rn(__ldg(xyz + 3 * i), region_size), kPi));
    const double yn = sin(__dmul_rn(__ddiv_rn(__ldg(xyz + 3 * i + 1), region_size), kPi));
    const double threshold = __dmul_rn(xn, yn) > 0.0 ? sparse_ratio : dense_ratio;   // NaN signs (region_size 0): dense
    flag[i] = uniform24(key, i, 6) < threshold ? 1u : 0u;
  }
}

// stable compaction: the point i with pos[i + 1] != pos[i] goes to pos[i] (its normal with it)
template <bool kNormals>
__global__ void __launch_bounds__(kThreads) compact_kernel(const double *__restrict__ xyz, const double *__restrict__ nrm,
                                                           const uint32_t *__restrict__ pos, long long n, double *__restrict__ out,
                                                           double *__restrict__ out_nrm) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t p = pos[i];
    if (pos[i + 1] == p) continue;
#pragma unroll
    for (int a = 0; a < 3; ++a) out[3ll * p + a] = __ldg(xyz + 3 * i + a);
    if (kNormals) {
#pragma unroll
      for (int a = 0; a < 3; ++a) out_nrm[3ll * p + a] = __ldg(nrm + 3 * i + a);
    }
  }
}

// addSparseOutliers (:1786-1806): outlier j = p[base] + range * N(0, 1) per axis, written after the n originals
__global__ void __launch_bounds__(kThreads) outlier_kernel(double *__restrict__ xyz, long long n, long long m, double range,
                                                           LaneKeys L) {
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < m; j += (long long)gridDim.x * blockDim.x) {
    const double b = floor(__dmul_rn(uniform53(L.k[7], j, 7), (double)n));
    const long long base = b < (double)(n - 1) ? (long long)b : n - 1;
#pragma unroll
    for (int a = 0; a < 3; ++a)
      xyz[3 * (n + j) + a] = __dadd_rn(xyz[3 * base + a], __dmul_rn(range, gaussian(L, j, 8 + 2 * a)));
  }
}

// addLocalDeformation (:1808-1829): inside the radius (strict), p += ((p - c) / |p - c| * strength) * w,
// w = 0.5 (1 + cos(pi d / r)); |.| = sqrt of Eigen's squaredNorm, and normalize() leaves a zero vector as it is
__global__ void __launch_bounds__(kThreads) deform_kernel(double *__restrict__ xyz, long long n, double radius, double strength,
                                                          double cx, double cy, double cz) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    const double dx = __dsub_rn(x, cx), dy = __dsub_rn(y, cy), dz = __dsub_rn(z, cz);
    const double d = sqrt(sqnorm_eigen(dx, dy, dz));
    if (!(d < radius)) continue;
    const double w = __dmul_rn(0.5, __dadd_rn(1.0, cos(__ddiv_rn(__dmul_rn(kPi, d), radius))));
    if (!(d > 0.0)) continue;                         // direction (0, 0, 0): the point stays
    xyz[3 * i] = __dadd_rn(x, __dmul_rn(__dmul_rn(__ddiv_rn(dx, d), strength), w));
    xyz[3 * i + 1] = __dadd_rn(y, __dmul_rn(__dmul_rn(__ddiv_rn(dy, d), strength), w));
    xyz[3 * i + 2] = __dadd_rn(z, __dmul_rn(__dmul_rn(__ddiv_rn(dz, d), strength), w));
  }
}

// ---- entry points ---------------------------------------------------------------------------------------------------

static int owned_cloud(me_ctx *ctx, int which, const char *what) {
  if (!ctx->cloud[which].owned)
    return fail(ctx, ME_ERR_INVALID, std::string(what) + " needs a library-owned cloud (me_set_cloud or me_copy_cloud)");
  return wait_upload(ctx, which);
}

int copy_cloud(me_ctx *ctx, int src, int dst, bool with_normals) {
  Cloud &s = ctx->cloud[src], &d = ctx->cloud[dst];
  ME_TRY(wait_upload(ctx, src));
  ME_TRY(wait_upload(ctx, dst));
  if (!d.owned) { d.d_xyz = nullptr; d.cap_xyz = 0; }
  ME_TRY(ensure(ctx, (void **)&d.d_xyz, &d.cap_xyz, 3 * s.n, sizeof(double)));
  d.owned = true;
  if (s.n > 0) ME_CUDA(ctx, cudaMemcpyAsync(d.d_xyz, s.d_xyz, (size_t)s.n * 3 * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
  d.n = s.n;
  invalidate_cloud(d);
  d.normal_valid = false;
  if (with_normals && s.normal_valid && s.n > 0) {
    ME_TRY(ensure(ctx, (void **)&d.d_normal, &d.cap_normal, 3 * s.n, sizeof(double)));
    ME_CUDA(ctx, cudaMemcpyAsync(d.d_normal, s.d_normal, (size_t)s.n * 3 * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    d.normal_valid = true;
  }
  return ME_OK;
}

int add_gaussian_noise(me_ctx *ctx, int which, double std_dev, uint64_t seed) {
  ME_TRY(owned_cloud(ctx, which, "me_add_gaussian_noise"));
  Cloud &c = ctx->cloud[which];
  if (std_dev == 0.0 || c.n == 0) return ME_OK;      // the cloud is unchanged, and so is everything computed from it
  noise_kernel<<<stream_blocks(ctx, c.n), kThreads, 0, ctx->stream>>>(c.d_xyz, c.n, std_dev, lane_keys(seed));
  ME_LAUNCH_CHECK(ctx);
  invalidate_cloud(c);
  return ME_OK;
}

int add_non_uniform_density(me_ctx *ctx, int which, double sparse_ratio, double dense_ratio, double region_size, uint64_t seed,
                            int64_t *n_out) {
  if (n_out) *n_out = ctx->cloud[which].n;
  ME_TRY(owned_cloud(ctx, which, "me_add_non_uniform_density"));
  Cloud &c = ctx->cloud[which];
  const long long n = c.n;
  if (n == 0) return ME_OK;
  ME_TRY(ensure_work(ctx, (size_t)(n + 1) * sizeof(uint32_t)));
  uint32_t *pos = (uint32_t *)ctx->d_work;
  const int blocks = stream_blocks(ctx, n + 1);
  density_flag_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.d_xyz, n, sparse_ratio, dense_ratio, region_size, lane_key(seed, 6), pos);
  ME_LAUNCH_CHECK(ctx);
  ME_TRY(exclusive_scan_inplace(ctx, pos, n + 1));
  uint32_t *h = (uint32_t *)ctx->h_pinned;
  ME_CUDA(ctx, cudaMemcpyAsync(h, pos + n, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const long long kept = (long long)h[0];
  double *out = nullptr, *out_nrm = nullptr;
  long long cap_out = 0, cap_nrm = 0;
  ME_TRY(ensure(ctx, (void **)&out, &cap_out, 3 * kept, sizeof(double)));
  if (c.normal_valid) {
    if (ensure(ctx, (void **)&out_nrm, &cap_nrm, 3 * kept, sizeof(double)) != ME_OK) { cudaFree(out); return ME_ERR_NOMEM; }
    compact_kernel<true><<<blocks, kThreads, 0, ctx->stream>>>(c.d_xyz, c.d_normal, pos, n, out, out_nrm);
  } else {
    compact_kernel<false><<<blocks, kThreads, 0, ctx->stream>>>(c.d_xyz, nullptr, pos, n, out, nullptr);
  }
  ME_LAUNCH_CHECK(ctx);
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // the old buffers may be released now
  cudaFree(c.d_xyz);
  c.d_xyz = out; c.cap_xyz = cap_out; c.n = kept;
  if (c.normal_valid) {                               // the normals follow their points
    cudaFree(c.d_normal);
    c.d_normal = out_nrm; c.cap_normal = cap_nrm;
  }
  invalidate_cloud(c);
  if (n_out) *n_out = kept;
  return ME_OK;
}

int add_sparse_outliers(me_ctx *ctx, int which, double outlier_ratio, double outlier_range, uint64_t seed, int64_t *n_out) {
  if (n_out) *n_out = ctx->cloud[which].n;
  ME_TRY(owned_cloud(ctx, which, "me_add_sparse_outliers"));
  Cloud &c = ctx->cloud[which];
  const long long n = c.n;
  // static_cast<int>(points_.size() * outlier_ratio): a count at or above 2^31 does not fit the reference's int
  const double want = (double)n * outlier_ratio;
  if (!(want < 2147483648.0)) return fail(ctx, ME_ERR_RANGE, "me_add_sparse_outliers: N * outlier_ratio >= 2^31");
  const long long m = want > 0.0 ? (long long)want : 0;
  if (n + m >= 0x7fffffffll) return fail(ctx, ME_ERR_RANGE, "me_add_sparse_outliers: more than 2^31-1 points per cloud");
  if (m == 0) return ME_OK;
  if (c.cap_xyz < 3 * (n + m)) {                      // grow: the originals move to a buffer with room for the outliers
    double *out = nullptr;
    long long cap_out = 0;
    ME_TRY(ensure(ctx, (void **)&out, &cap_out, 3 * (n + m), sizeof(double)));
    ME_CUDA(ctx, cudaMemcpyAsync(out, c.d_xyz, (size_t)n * 3 * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    cudaFree(c.d_xyz);
    c.d_xyz = out; c.cap_xyz = cap_out;
  }
  outlier_kernel<<<stream_blocks(ctx, m), kThreads, 0, ctx->stream>>>(c.d_xyz, n, m, outlier_range, lane_keys(seed));
  ME_LAUNCH_CHECK(ctx);
  c.n = n + m;
  invalidate_cloud(c);
  c.normal_valid = false;       // Open3D: normals_ and points_ differ in size, HasNormals() is false
  if (n_out) *n_out = c.n;
  return ME_OK;
}

int add_local_deformation(me_ctx *ctx, int which, double radius, double strength, const double center[3]) {
  ME_TRY(owned_cloud(ctx, which, "me_add_local_deformation"));
  Cloud &c = ctx->cloud[which];
  if (c.n == 0 || !(radius > 0.0)) return ME_OK;      // d < radius <= 0 holds for no point
  deform_kernel<<<stream_blocks(ctx, c.n), kThreads, 0, ctx->stream>>>(c.d_xyz, c.n, radius, strength, center[0], center[1], center[2]);
  ME_LAUNCH_CHECK(ctx);
  invalidate_cloud(c);
  return ME_OK;
}

}  // namespace me

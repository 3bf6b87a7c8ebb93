// voxel.cu — voxel Gaussians, voxel-pair Wasserstein distance (AWD / "VMD") and spatial consistency score (SCS).
//
// Replaces (reference):
//   voxel_calculator.cpp:21-56    VoxelCalculator::buildVoxelMap   (sequential Welford into an unordered_map)
//   voxel_calculator.cpp:97-113   computeVoxelEntropy              (second division by n-1)
//   voxel_calculator.cpp:142-172  updateVoxelMap(const VoxelMap&)  (active / old / new labelling)
//   voxel_calculator.cpp:115-140  computeWassersteinDistanceGaussian (third division, eigen-clamp, Cholesky trace)
//   voxel_calculator.cpp:7-19     getNeighborIndices
//   map_eval.cpp:240-390          MapEval::calculateVMD            (pair filter >= 100 points, mean, SCS)
//
// The lattice cells are sub-cells of the reference's voxels floor(x / v) (see Lattice in common.cuh), so a voxel is
// m x m contiguous x-runs of the cell-sorted cloud: one warp reduces one voxel with no hashing and no atomics, and
// est/gt voxels pair up by index arithmetic.  Moments are taken about the voxel centre in fp64
// (mu = c + S1/n, M2 = S2 - S1 S1^T / n), which equals the Welford result to rounding.
#include "common.cuh"
#include "eig3.cuh"
#include "svd3.cuh"
#include <algorithm>
#include <cstring>
#include <cstdlib>
#include <vector>
#include <climits>

namespace me {

static constexpr int kThreads = 256;

// ---- per-voxel moments -----------------------------------------------------------------------------------------
// out: cnt[nvoxels] (int32), mom[nvoxels * 9] = S1(3), S2(xx,xy,xz,yy,yz,zz) about the voxel centre
// One HALF-warp per voxel (a voxel is m x m x-runs; with m = 4 that is 16 runs — one per lane of the half-warp).
// sparse lattices: the voxel grid of a site-scale scene is mostly empty, and probing the m x m rows of an empty voxel costs
// hash lookups — count the points per voxel from the sorted cloud first, the moments kernel then skips empty voxels
__global__ void __launch_bounds__(kThreads)
voxel_precount_kernel(const P4 *__restrict__ S, const float4 *__restrict__ rel, long long n, CellIndex I, Lattice L,
                      int32_t *__restrict__ cnt) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int ix, iy, iz;
    cell_from_tag(I, __double_as_longlong(__ldg(reinterpret_cast<const double *>(S + i) + 3)), (int)__ldg(rel + i).w, ix, iy, iz);
    atomicAdd(cnt + ((long long)(iz / L.m) * L.nvox[1] + iy / L.m) * L.nvox[0] + ix / L.m, 1);
  }
}

__global__ void __launch_bounds__(kThreads)
voxel_moments_kernel(const P4 *__restrict__ S, CellIndex I, Lattice L, int precounted, Owned vown,
                     int32_t *__restrict__ cnt, double *__restrict__ mom, unsigned long long *__restrict__ n_occupied) {
  const int sub = threadIdx.x & 15;
  const long long group = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 4;
  const long long ngroups = ((long long)gridDim.x * blockDim.x) >> 4;
  const int m = L.m;
  unsigned long long occ = 0;
  // both half-warps of a warp iterate the same number of times (the shuffles below are full-warp)
  const long long iters = (L.nvoxels + ngroups - 1) / ngroups;
  for (long long it = 0; it < iters; ++it) {
    const long long vox = group + it * ngroups;
    const bool live = vox < L.nvoxels;
    double s[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    int n = 0;
    const int vx = (int)(vox % L.nvox[0]);
    const int vy = (int)((vox / L.nvox[0]) % L.nvox[1]);
    const int vz = (int)(vox / ((long long)L.nvox[0] * L.nvox[1]));
    // slab layout: a voxel layer has one owner; the voxels of other ranks stay empty here (their W arrives by all-reduce)
    if (live && owns(vown, vy, vz) && !(precounted && cnt[vox] == 0)) {
      const double cx = ((double)(L.k_lo[0] + vx) + 0.5) * L.v, cy = ((double)(L.k_lo[1] + vy) + 0.5) * L.v,
                   cz = ((double)(L.k_lo[2] + vz) + 0.5) * L.v;
      for (int t = sub; t < m * m; t += 16) {
        const long long z = (long long)vz * m + t / m, y = (long long)vy * m + t % m;
        uint32_t b, e;
        cell_range(I, (int)z, (int)y, vx * m, vx * m + m - 1, b, e);
        for (uint32_t j = b; j < e; ++j) {
          const P4 p = load_p4(S + j);
          const double dx = p.x - cx, dy = p.y - cy, dz = p.z - cz;
          n++;
          s[0] += dx; s[1] += dy; s[2] += dz;
          s[3] += dx * dx; s[4] += dx * dy; s[5] += dx * dz; s[6] += dy * dy; s[7] += dy * dz; s[8] += dz * dz;
        }
      }
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
#pragma unroll
    for (int k = 0; k < 9; ++k)
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
    if (live && sub == 0) {
      cnt[vox] = n;
      if (n > 0) {
        occ++;
#pragma unroll
        for (int k = 0; k < 9; ++k) mom[vox * 9 + k] = s[k];
      }
    }
  }
  if (sub == 0 && occ) atomicAdd(n_occupied, occ);
}

// ---- 3x3 algebra (fp64) ---------------------------------------------------------------------------------------
// Eigen LLT (unblocked, lower, in place); stops at the first non-positive pivot leaving the rest untouched
__device__ void llt3_inplace(double *m) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    double x = m[k * 3 + k];
    for (int j = 0; j < k; ++j) x -= m[k * 3 + j] * m[k * 3 + j];
    if (x <= 0.0) return;
    x = sqrt(x);
    m[k * 3 + k] = x;
    for (int i = k + 1; i < 3; ++i) {
      double s = m[i * 3 + k];
      for (int j = 0; j < k; ++j) s -= m[i * 3 + j] * m[k * 3 + j];
      m[i * 3 + k] = s / x;
    }
  }
}

// voxel_calculator.cpp:118-125: sigma / (n - 1), symmetrise, clamp eigenvalues at 1e-6
__device__ void clamp_cov(const double *stored, int n, double *out) {
#pragma unroll
  for (int i = 0; i < 9; ++i) out[i] = (i % 4 == 0) ? 1.0 : 0.0;
  if (n > 1) {
    double s[9], sym[9], w[3], v[9];
    const double nm1 = (double)(n - 1);
#pragma unroll
    for (int i = 0; i < 9; ++i) s[i] = stored[i] / nm1;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) sym[r * 3 + c] = (s[r * 3 + c] + s[c * 3 + r]) / 2;
    eig3_jacobi(sym, w, v);
#pragma unroll
    for (int k = 0; k < 3; ++k) w[k] = fmax(w[k], 1e-6);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        double acc = 0;
#pragma unroll
        for (int k = 0; k < 3; ++k) acc += v[r * 3 + k] * w[k] * v[c * 3 + k];
        out[r * 3 + c] = acc;
      }
  }
}

// voxel_calculator.cpp:115-140, arguments in the reference's call order (voxel1 = gt, voxel2 = est; map_eval.cpp:284)
__device__ double wasserstein(const double *mu1, const double *sig1, int n1, const double *mu2, const double *sig2, int n2) {
  double s1[9], s2[9], l1[9], tmp[9], a[9];
  clamp_cov(sig1, n1, s1);
  clamp_cov(sig2, n2, s2);
  const double dm0 = mu1[0] - mu2[0], dm1 = mu1[1] - mu2[1], dm2 = mu1[2] - mu2[2];
  const double tr_sum = (s1[0] + s2[0]) + (s1[4] + s2[4]) + (s1[8] + s2[8]);
#pragma unroll
  for (int i = 0; i < 9; ++i) l1[i] = s1[i];
  llt3_inplace(l1);
  l1[1] = l1[2] = l1[5] = 0.0;                       // matrixL(): lower triangular view
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      double s = 0;
#pragma unroll
      for (int k = 0; k < 3; ++k) s += l1[i * 3 + k] * s2[k * 3 + j];
      tmp[i * 3 + j] = s;
    }
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      double s = 0;
#pragma unroll
      for (int k = 0; k < 3; ++k) s += tmp[i * 3 + k] * l1[j * 3 + k];   // * L1^T
      a[i * 3 + j] = s;
    }
  llt3_inplace(a);
  const double tr_sqrt = a[0] + a[4] + a[8];
  const double dist = (dm0 * dm0 + dm1 * dm1 + dm2 * dm2) + tr_sum - 2 * tr_sqrt;
  return sqrt(fmax(0.0, dist));
}

// mu and the sigma the reference has stored after buildVoxelMap: M2 for n <= 10 (voxel_calculator.cpp:47),
// (M2 / (n-1)) / (n-1) otherwise (:48 then :102)
__device__ void stored_gaussian(const double *mom, int n, double cx, double cy, double cz, double *mu, double *sig) {
  const double nd = (double)n;
  mu[0] = cx + mom[0] / nd; mu[1] = cy + mom[1] / nd; mu[2] = cz + mom[2] / nd;
  double m2[6];
  m2[0] = mom[3] - mom[0] * mom[0] / nd; m2[1] = mom[4] - mom[0] * mom[1] / nd; m2[2] = mom[5] - mom[0] * mom[2] / nd;
  m2[3] = mom[6] - mom[1] * mom[1] / nd; m2[4] = mom[7] - mom[1] * mom[2] / nd; m2[5] = mom[8] - mom[2] * mom[2] / nd;
  if (n > 10) {
    const double nm1 = (double)(n - 1);
#pragma unroll
    for (int k = 0; k < 6; ++k) m2[k] = (m2[k] / nm1) / nm1;
  }
  sig[0] = m2[0]; sig[1] = m2[1]; sig[2] = m2[2];
  sig[3] = m2[1]; sig[4] = m2[3]; sig[5] = m2[4];
  sig[6] = m2[2]; sig[7] = m2[4]; sig[8] = m2[5];
}

struct AwdAcc {
  unsigned long long n_pairs, n_active, n_new, n_scs;
  double sum_w, sum_scs;
};

// ---- pairing + Wasserstein: one thread per est voxel -----------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
awd_kernel(Lattice Le, Lattice Lg, const int32_t *__restrict__ cnt_e, const double *__restrict__ mom_e,
           const int32_t *__restrict__ cnt_g, const double *__restrict__ mom_g, int min_points, double missing,
           double *__restrict__ w_out, uint32_t *__restrict__ pair_list, double *__restrict__ rows27,
           AwdAcc *__restrict__ acc) {
  unsigned long long l_active = 0, l_new = 0;
  for (long long vox = blockIdx.x * (long long)blockDim.x + threadIdx.x; vox < Le.nvoxels;
       vox += (long long)gridDim.x * blockDim.x) {
    double w = missing;      // NaN, or -1 when the table is MAX-all-reduced across ranks (slab layout)
    const int ne = cnt_e[vox];
    if (ne > 0) {
      const int vx = (int)(vox % Le.nvox[0]);
      const int vy = (int)((vox / Le.nvox[0]) % Le.nvox[1]);
      const int vz = (int)(vox / ((long long)Le.nvox[0] * Le.nvox[1]));
      const long long kx = (long long)Le.k_lo[0] + vx, ky = (long long)Le.k_lo[1] + vy, kz = (long long)Le.k_lo[2] + vz;
      const long long gx = kx - Lg.k_lo[0], gy = ky - Lg.k_lo[1], gz = kz - Lg.k_lo[2];
      int ng = 0;
      long long gvox = -1;
      if (gx >= 0 && gx < Lg.nvox[0] && gy >= 0 && gy < Lg.nvox[1] && gz >= 0 && gz < Lg.nvox[2]) {
        gvox = (gz * Lg.nvox[1] + gy) * (long long)Lg.nvox[0] + gx;
        ng = cnt_g[gvox];
      }
      if (ng > 0) l_active++; else l_new++;
      if (ng > 0 && ne >= min_points && ng >= min_points) {       // map_eval.cpp:274-281
        const double cx = ((double)kx + 0.5) * Le.v, cy = ((double)ky + 0.5) * Le.v, cz = ((double)kz + 0.5) * Le.v;
        double mu_e[3], sig_e[9], mu_g[3], sig_g[9];
        stored_gaussian(mom_e + vox * 9, ne, cx, cy, cz, mu_e, sig_e);
        stored_gaussian(mom_g + gvox * 9, ng, cx, cy, cz, mu_g, sig_g);
        w = wasserstein(mu_g, sig_g, ng, mu_e, sig_e, ne);         // (gt_voxel, est_voxel) map_eval.cpp:284
        const unsigned long long slot = atomicAdd(&acc->n_pairs, 1ull);
        pair_list[slot] = (uint32_t)vox;
        atomicAdd(&acc->sum_w, w);
        if (rows27) {                                              // map_eval.cpp:288-302
          double *r = rows27 + slot * 27;
          r[0] = (double)kx * Le.v; r[1] = (double)ky * Le.v; r[2] = (double)kz * Le.v;
          r[3] = ((double)kx + 1.0) * Le.v; r[4] = ((double)ky + 1.0) * Le.v; r[5] = ((double)kz + 1.0) * Le.v;
          r[6] = mu_e[0]; r[7] = mu_e[1]; r[8] = mu_e[2];
          r[9] = w; r[10] = (double)ng; r[11] = (double)ne;
          r[12] = sig_e[0]; r[13] = sig_e[1]; r[14] = sig_e[2]; r[15] = sig_e[4]; r[16] = sig_e[5]; r[17] = sig_e[8];
          r[18] = mu_g[0]; r[19] = mu_g[1]; r[20] = mu_g[2];
          r[21] = sig_g[0]; r[22] = sig_g[1]; r[23] = sig_g[2]; r[24] = sig_g[4]; r[25] = sig_g[5]; r[26] = sig_g[8];
        }
      }
    }
    w_out[vox] = w;
  }
  l_active = (unsigned long long)warp_sum_ll((long long)l_active);
  l_new = (unsigned long long)warp_sum_ll((long long)l_new);
  if ((threadIdx.x & 31) == 0) {
    if (l_active) atomicAdd(&acc->n_active, l_active);
    if (l_new) atomicAdd(&acc->n_new, l_new);
  }
}

// ---- SCS: one warp per paired voxel, lanes over the (2R+1)^3 - 1 neighbour offsets (map_eval.cpp:351-387) -------
static constexpr int kScsMaxPerLane = 48;      // neighbour values a lane keeps in registers (radius <= 5: 1331 / 32 = 42)

// me_kernel_trace: which scs_kernel path a radius takes
static void trace_scs(me_ctx *ctx, int radius) {
  const int side = 2 * radius + 1;
  trace_kernel(ctx, radius == 5 ? ME_KBIT_SCS_R5
                    : ((side * side * side + 31) / 32 <= kScsMaxPerLane ? ME_KBIT_SCS_RT_CACHED : ME_KBIT_SCS_RT_UNCACHED));
}

template <int RADIUS>      // RADIUS > 0: compile-time neighbourhood (the reference hard-codes 5, map_eval.cpp:353); 0: run time
__global__ void __launch_bounds__(kThreads)
scs_kernel(Lattice Le, const double *__restrict__ w_vox, const uint32_t *__restrict__ pair_list, int radius_rt,
           AwdAcc *__restrict__ acc) {
  const int radius = RADIUS > 0 ? RADIUS : radius_rt;
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const unsigned long long npairs = acc->n_pairs;
  const int side = 2 * radius + 1, total = side * side * side;
  double l_scs = 0.0;
  unsigned long long l_cnt = 0;
  for (long long pi = warp; pi < (long long)npairs; pi += nwarps) {
    const long long vox = pair_list[pi];
    const int vx = (int)(vox % Le.nvox[0]);
    const int vy = (int)((vox / Le.nvox[0]) % Le.nvox[1]);
    const int vz = (int)(vox / ((long long)Le.nvox[0] * Le.nvox[1]));
    // the lane's share of the (2R+1)^3 - 1 neighbour values is fetched once (all loads in flight together) and kept for
    // both passes of the reference's mean / population-variance computation (map_eval.cpp:364-381)
    constexpr int kMaxPerLane = kScsMaxPerLane;
    double wv[kMaxPerLane];
    const int per_lane = (total + 31) / 32;
    const bool cached = per_lane <= kMaxPerLane;
    double sum = 0.0;
    int n = 0;
    auto fetch = [&](int t) -> double {
      if (t >= total) return NAN;
      const int dx = t / (side * side) - radius, dy = (t / side) % side - radius, dz = t % side - radius;
      if (dx == 0 && dy == 0 && dz == 0) return NAN;
      const int x = vx + dx, y = vy + dy, z = vz + dz;
      if (x < 0 || x >= Le.nvox[0] || y < 0 || y >= Le.nvox[1] || z < 0 || z >= Le.nvox[2]) return NAN;
      const double w = __ldg(w_vox + ((long long)z * Le.nvox[1] + y) * Le.nvox[0] + x);
      return w < 0.0 ? NAN : w;      // -1: no pair in that voxel (the all-reducible encoding)
    };
    if (cached) {
#pragma unroll
      for (int k = 0; k < kMaxPerLane; ++k) wv[k] = k < per_lane ? fetch(lane + 32 * k) : NAN;
#pragma unroll
      for (int k = 0; k < kMaxPerLane; ++k) if (!isnan(wv[k])) { sum += wv[k]; n++; }
    } else {
      for (int t = lane; t < total; t += 32) { const double w = fetch(t); if (!isnan(w)) { sum += w; n++; } }
    }
    sum = warp_sum(sum);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
    if (n == 0) continue;
    const double mean = sum / (double)n;
    double ss = 0.0;
    if (cached) {
#pragma unroll
      for (int k = 0; k < kMaxPerLane; ++k) if (!isnan(wv[k])) ss += (wv[k] - mean) * (wv[k] - mean);
    } else {
      for (int t = lane; t < total; t += 32) { const double w = fetch(t); if (!isnan(w)) ss += (w - mean) * (w - mean); }
    }
    ss = warp_sum(ss);
    if (lane == 0) {
      const double var = ss / (double)n;
      l_scs += sqrt(var) / mean;
      l_cnt++;
    }
  }
  if (lane == 0 && l_cnt) { atomicAdd(&acc->sum_scs, l_scs); atomicAdd(&acc->n_scs, l_cnt); }
}

__global__ void zero_awd_acc_kernel(AwdAcc *a, unsigned long long *occ2) {
  a->n_pairs = a->n_active = a->n_new = a->n_scs = 0;
  a->sum_w = a->sum_scs = 0.0;
  occ2[0] = occ2[1] = 0;
}

// ---------------------------------------------------------------------------------------------------------------
// The stage in two halves.  voxel_begin: lattices, per-voxel moments, pairing + Wasserstein distances (the W table over the
// estimated cloud's voxels stays in the work buffer).  voxel_scs: the SCS sweep over the paired voxels of this rank.  On a
// slab layout every rank computes the voxel layers it owns and the caller MAX-all-reduces the W table between the halves
// (SCS reads the 11^3 neighbourhood of a voxel, map_eval.cpp:353); all eight counters / sums are then SUM-reducible.
// ---------------------------------------------------------------------------------------------------------------
static Owned voxel_owned(const Cloud &c) {
  Owned o;
  o.axis = c.slab ? c.sl_axis : 0;
  o.lo = c.so_lo / std::max(1, c.lat.m); o.hi = c.so_hi / std::max(1, c.lat.m);      // slab planes are whole voxel layers
  return o;
}

// The part of the stage both voxel metrics (AWD and W2) share: lattices aligned with the voxel size and the work layout
// cnt_e | cnt_g | mom_e | mom_g | w_vox | pair_list | rows (row_cols fp64 per pair when want_rows).  Both stages keep their
// tables in this one work buffer, so laying it out closes whichever of them was open.
struct VoxelTables {
  Lattice Le, Lg;
  bool slab;
  int32_t *cnt_e, *cnt_g;
  double *mom_e, *mom_g, *w_vox, *rows;
  uint32_t *pair_list;
  size_t o_w, o_pairs;
};

static int voxel_layout(me_ctx *ctx, double voxel_size, int min_points, int row_cols, bool want_rows, VoxelTables &t) {
  ctx->vox_open = false;
  ctx->w2_open = false;
  if (!(voxel_size > 0)) return fail(ctx, ME_ERR_INVALID, "vmd_voxel_size must be > 0");
  if (ctx->cloud[0].n <= 0 || ctx->cloud[1].n <= 0) return fail(ctx, ME_ERR_EMPTY, "both clouds must be set");
  // the lattices must be aligned with this voxel size; rebuild them if they are not
  for (int w = 0; w < 2; ++w) {
    Cloud &c = ctx->cloud[w];
    if (c.grid_valid && c.lat.v != voxel_size) c.grid_valid = false;
  }
  ctx->voxel_hint = voxel_size;
  ME_TRY(build_both(ctx));
  Cloud &E = ctx->cloud[ME_CLOUD_EST], &G = ctx->cloud[ME_CLOUD_GT];
  const Lattice Le = E.lat, Lg = G.lat;
  if (Le.nvoxels < 0 || Lg.nvoxels < 0 || Le.nvoxels >= 0x7fffffffll || Lg.nvoxels >= 0x7fffffffll)
    return fail(ctx, ME_ERR_RANGE, "vmd_voxel_size is too small for the extent of the clouds: the voxel tables are dense (2^31 voxels at most)");
  const bool slab = E.slab || G.slab;
  if (slab && want_rows)
    return fail(ctx, ME_ERR_INVALID, "the per-voxel rows are not available on a slab layout (every rank holds its own voxels only)");

  auto align = [](size_t x) { return (x + 255) & ~(size_t)255; };
  size_t o_cnt_e = 0;
  size_t o_cnt_g = o_cnt_e + align((size_t)Le.nvoxels * sizeof(int32_t));
  size_t o_mom_e = o_cnt_g + align((size_t)Lg.nvoxels * sizeof(int32_t));
  size_t o_mom_g = o_mom_e + align((size_t)Le.nvoxels * 9 * sizeof(double));
  size_t o_w = o_mom_g + align((size_t)Lg.nvoxels * 9 * sizeof(double));
  size_t o_pairs = o_w + align((size_t)Le.nvoxels * sizeof(double));
  size_t o_rows = o_pairs + align((size_t)Le.nvoxels * sizeof(uint32_t));
  // a voxel pair needs >= min_points points in each cloud, which bounds the number of rows
  long long max_pairs = std::min<long long>(Le.nvoxels, std::min(E.n, G.n) / std::max(1, min_points) + 1);
  size_t total = o_rows + (want_rows ? align((size_t)max_pairs * row_cols * sizeof(double)) : 0);
  ME_TRY(ensure_work(ctx, total));
  char *base = (char *)ctx->d_work;
  t.Le = Le; t.Lg = Lg; t.slab = slab;
  t.cnt_e = (int32_t *)(base + o_cnt_e); t.cnt_g = (int32_t *)(base + o_cnt_g);
  t.mom_e = (double *)(base + o_mom_e); t.mom_g = (double *)(base + o_mom_g);
  t.w_vox = (double *)(base + o_w);
  t.pair_list = (uint32_t *)(base + o_pairs);
  t.rows = want_rows ? (double *)(base + o_rows) : nullptr;
  t.o_w = o_w; t.o_pairs = o_pairs;
  return ME_OK;
}

// the per-voxel moments of both clouds into the tables; occ[0], occ[1]: the occupied voxels of est and gt (zeroed by the caller)
static int voxel_moments(me_ctx *ctx, const VoxelTables &t, unsigned long long *occ) {
  Cloud &E = ctx->cloud[ME_CLOUD_EST], &G = ctx->cloud[ME_CLOUD_GT];
  const Lattice &Le = t.Le, &Lg = t.Lg;
  StageTimer timer(ctx, 6);
  int blocks_e = (int)std::min<long long>((Le.nvoxels * 16 + kThreads - 1) / kThreads, (long long)ctx->sm_count * 8);
  const int pb_e = (int)std::min<long long>((E.n + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
  const int pb_g = (int)std::min<long long>((G.n + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
  if (Le.sparse) {
    ME_CUDA(ctx, cudaMemsetAsync(t.cnt_e, 0, (size_t)Le.nvoxels * sizeof(int32_t), ctx->stream));
    voxel_precount_kernel<<<pb_e, kThreads, 0, ctx->stream>>>(E.d_sorted, E.d_rel, E.ns, index_of(E), Le, t.cnt_e);
    ME_LAUNCH_CHECK(ctx);
  }
  if (Lg.sparse) {
    ME_CUDA(ctx, cudaMemsetAsync(t.cnt_g, 0, (size_t)Lg.nvoxels * sizeof(int32_t), ctx->stream));
    voxel_precount_kernel<<<pb_g, kThreads, 0, ctx->stream>>>(G.d_sorted, G.d_rel, G.ns, index_of(G), Lg, t.cnt_g);
    ME_LAUNCH_CHECK(ctx);
  }
  voxel_moments_kernel<<<std::max(1, blocks_e), kThreads, 0, ctx->stream>>>(E.d_sorted, index_of(E), Le, Le.sparse, voxel_owned(E), t.cnt_e, t.mom_e, occ);
  ME_LAUNCH_CHECK(ctx);
  int blocks_g = (int)std::min<long long>((Lg.nvoxels * 16 + kThreads - 1) / kThreads, (long long)ctx->sm_count * 8);
  voxel_moments_kernel<<<std::max(1, blocks_g), kThreads, 0, ctx->stream>>>(G.d_sorted, index_of(G), Lg, Lg.sparse, voxel_owned(G), t.cnt_g, t.mom_g, occ + 1);
  ME_LAUNCH_CHECK(ctx);
  return ME_OK;
}

static int voxel_begin_impl(me_ctx *ctx, double voxel_size, int min_points, bool want_rows, double **d_rows_out) {
  VoxelTables t;
  ME_TRY(voxel_layout(ctx, voxel_size, min_points, 27, want_rows, t));
  if (d_rows_out) *d_rows_out = t.rows;
  AwdAcc *acc = (AwdAcc *)ctx->d_scratch;
  unsigned long long *occ = (unsigned long long *)((char *)ctx->d_scratch + 256);
  zero_awd_acc_kernel<<<1, 1, 0, ctx->stream>>>(acc, occ);
  ME_LAUNCH_CHECK(ctx);
  ME_TRY(voxel_moments(ctx, t, occ));
  {
    StageTimer timer(ctx, 7);
    const Lattice Le = t.Le;
    int blocks = (int)std::min<long long>((Le.nvoxels + kThreads - 1) / kThreads, (long long)ctx->sm_count * 8);
    awd_kernel<<<std::max(1, blocks), kThreads, 0, ctx->stream>>>(t.Le, t.Lg, t.cnt_e, t.mom_e, t.cnt_g, t.mom_g, min_points,
                                                                 t.slab ? -1.0 : (double)NAN, t.w_vox, t.pair_list, t.rows, acc);
    ME_LAUNCH_CHECK(ctx);
  }
  ctx->vox_open = true;
  ctx->vox_nvox = t.Le.nvoxels;
  ctx->vox_o_w = t.o_w;
  ctx->vox_o_pairs = t.o_pairs;
  return ME_OK;
}

static int voxel_scs_impl(me_ctx *ctx, int scs_radius) {
  if (!ctx->vox_open) return fail(ctx, ME_ERR_INVALID, "me_voxel_finish before me_voxel_begin");
  if (scs_radius < 0 || scs_radius > 64) return fail(ctx, ME_ERR_INVALID, "scs_radius out of range");
  ctx->vox_open = false;
  const Lattice Le = ctx->cloud[ME_CLOUD_EST].lat;
  const double *w_vox = (const double *)((char *)ctx->d_work + ctx->vox_o_w);
  const uint32_t *pair_list = (const uint32_t *)((char *)ctx->d_work + ctx->vox_o_pairs);
  AwdAcc *acc = (AwdAcc *)ctx->d_scratch;
  StageTimer timer(ctx, 8);
  if (scs_radius == 5) scs_kernel<5><<<ctx->sm_count * 4, kThreads, 0, ctx->stream>>>(Le, w_vox, pair_list, scs_radius, acc);
  else scs_kernel<0><<<ctx->sm_count * 4, kThreads, 0, ctx->stream>>>(Le, w_vox, pair_list, scs_radius, acc);
  ME_LAUNCH_CHECK(ctx);
  trace_scs(ctx, scs_radius);
  return ME_OK;
}

int voxel_begin(me_ctx *ctx, double voxel_size, int min_points) { return voxel_begin_impl(ctx, voxel_size, min_points, false, nullptr); }

int voxel_w_table(me_ctx *ctx, double **d_w, int64_t *n) {
  if (!ctx->vox_open) return fail(ctx, ME_ERR_INVALID, "me_voxel_w_table before me_voxel_begin");
  *d_w = (double *)((char *)ctx->d_work + ctx->vox_o_w);
  *n = (int64_t)ctx->vox_nvox;
  return ME_OK;
}

// the eight SUM-reducible values of the stage -> the context's accumulator block
__global__ void pack_awd_kernel(const AwdAcc *__restrict__ a, const unsigned long long *__restrict__ occ, double *__restrict__ blk) {
  if (threadIdx.x != 0) return;
  blk[0] = (double)a->n_pairs; blk[1] = (double)a->n_scs; blk[2] = (double)occ[0]; blk[3] = (double)occ[1];
  blk[4] = (double)a->n_active; blk[5] = (double)a->n_new; blk[6] = a->sum_w; blk[7] = a->sum_scs;
}

int voxel_finish_block(me_ctx *ctx, int scs_radius) {
  ME_TRY(voxel_scs_impl(ctx, scs_radius));
  pack_awd_kernel<<<1, 32, 0, ctx->stream>>>((const AwdAcc *)ctx->d_scratch, (const unsigned long long *)((char *)ctx->d_scratch + 256),
                                            ctx->d_block + kBlkAwd);
  ME_LAUNCH_CHECK(ctx);
  return ME_OK;
}

void awd_result(const double v[8], me_awd_result *out) {
  auto i64 = [](double x) { return (int64_t)std::llround(x); };
  std::memset(out, 0, sizeof(*out));
  out->n_pairs = i64(v[0]); out->n_scs = i64(v[1]);
  out->n_voxels_est = i64(v[2]); out->n_voxels_gt = i64(v[3]);
  out->n_active = i64(v[4]); out->n_new = i64(v[5]);
  out->n_old = out->n_voxels_gt - out->n_active;
  out->awd = v[6] / (double)out->n_pairs;        // 0/0 -> NaN as map_eval.cpp:324
  out->scs = v[7] / (double)out->n_scs;          // map_eval.cpp:387
}

int run_awd(me_ctx *ctx, double voxel_size, int min_points, int scs_radius, me_awd_result *out, int64_t *n_rows,
            double **rows27) {
  std::memset(out, 0, sizeof(*out));
  if (n_rows) *n_rows = 0;
  if (rows27) *rows27 = nullptr;
  if (scs_radius < 0 || scs_radius > 64) return fail(ctx, ME_ERR_INVALID, "scs_radius out of range");
  double *d_rows = nullptr;
  ME_TRY(voxel_begin_impl(ctx, voxel_size, min_points, rows27 != nullptr, &d_rows));
  if (ctx->cloud[ME_CLOUD_EST].slab || ctx->cloud[ME_CLOUD_GT].slab) {
    ctx->vox_open = false;
    return fail(ctx, ME_ERR_INVALID, "slab layout: run the voxel stage as me_voxel_begin / all-reduce of me_voxel_w_table / "
                                     "me_voxel_finish_accum_device");
  }
  ME_TRY(voxel_scs_impl(ctx, scs_radius));
  struct Host { AwdAcc a; char pad[256 - sizeof(AwdAcc)]; unsigned long long occ[2]; };
  Host *h = (Host *)ctx->h_pinned;
  ME_CUDA(ctx, cudaMemcpyAsync(h, ctx->d_scratch, sizeof(Host), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  // the values pack_awd_kernel would write (counts exact in fp64 below 2^53); no launch on this single-GPU path
  const double v[8] = {(double)h->a.n_pairs, (double)h->a.n_scs, (double)h->occ[0], (double)h->occ[1],
                       (double)h->a.n_active, (double)h->a.n_new, h->a.sum_w, h->a.sum_scs};
  awd_result(v, out);
  if (n_rows) *n_rows = out->n_pairs;
  if (rows27) {
    size_t bytes = (size_t)std::max<int64_t>(out->n_pairs, 1) * 27 * sizeof(double);
    double *hr = (double *)std::malloc(bytes);
    if (!hr) return fail(ctx, ME_ERR_NOMEM, "malloc(rows27) failed");
    if (out->n_pairs > 0) {
      ME_CUDA(ctx, cudaMemcpyAsync(hr, d_rows, (size_t)out->n_pairs * 27 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
      ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    *rows27 = hr;
  }
  return ME_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// The voxel-pair stage on GIVEN voxel Gaussians: rows in the 27-column layout of voxel_errors.txt (map_eval.cpp:292-302).
// Recomputes W with the device implementation of computeWassersteinDistanceGaussian and AWD / SCS over those voxels with
// the production scs_kernel.  Lets the tests pin the kernels directly to the reference's shipped sample output.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
awd_rows_kernel(const double *__restrict__ rows, long long n, const long long *__restrict__ vox_of_row,
                double *__restrict__ w_rows, double *__restrict__ w_vox, uint32_t *__restrict__ pair_list,
                AwdAcc *__restrict__ acc) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double *r = rows + i * 27;
    double mu_e[3] = {r[6], r[7], r[8]}, mu_g[3] = {r[18], r[19], r[20]}, sig_e[9], sig_g[9];
    sig_e[0] = r[12]; sig_e[1] = r[13]; sig_e[2] = r[14]; sig_e[3] = r[13]; sig_e[4] = r[15]; sig_e[5] = r[16];
    sig_e[6] = r[14]; sig_e[7] = r[16]; sig_e[8] = r[17];
    sig_g[0] = r[21]; sig_g[1] = r[22]; sig_g[2] = r[23]; sig_g[3] = r[22]; sig_g[4] = r[24]; sig_g[5] = r[25];
    sig_g[6] = r[23]; sig_g[7] = r[25]; sig_g[8] = r[26];
    const double w = wasserstein(mu_g, sig_g, (int)r[10], mu_e, sig_e, (int)r[11]);    // (gt, est), map_eval.cpp:284
    w_rows[i] = w;
    w_vox[vox_of_row[i]] = w;
    pair_list[i] = (uint32_t)vox_of_row[i];
    atomicAdd(&acc->sum_w, w);
    if (i == 0) acc->n_pairs = (unsigned long long)n;
  }
}
__global__ void fill_nan_kernel(double *p, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = NAN;
}

int run_awd_rows(me_ctx *ctx, const double *rows27, int64_t n_rows, double voxel_size, int scs_radius, double *w_out,
                 me_awd_result *out) {
  std::memset(out, 0, sizeof(*out));
  if (n_rows <= 0 || !rows27 || !(voxel_size > 0)) return fail(ctx, ME_ERR_INVALID, "bad arguments");
  if (scs_radius < 0 || scs_radius > 64) return fail(ctx, ME_ERR_INVALID, "scs_radius out of range");
  ctx->w2_open = false;      // the W2 stage's tables share the work buffer
  // voxel keys = vmin / v (columns 0-2), dense index inside their bounding box
  std::vector<long long> key(3 * (size_t)n_rows), vox((size_t)n_rows);
  long long lo[3] = {LLONG_MAX, LLONG_MAX, LLONG_MAX}, hi[3] = {LLONG_MIN, LLONG_MIN, LLONG_MIN};
  for (int64_t i = 0; i < n_rows; ++i)
    for (int a = 0; a < 3; ++a) {
      const long long k = llround(rows27[i * 27 + a] / voxel_size);
      key[3 * i + a] = k; lo[a] = std::min(lo[a], k); hi[a] = std::max(hi[a], k);
    }
  Lattice L;
  std::memset(&L, 0, sizeof(L));
  long long nvox = 1;
  for (int a = 0; a < 3; ++a) {
    if (hi[a] - lo[a] + 1 > 4096) return fail(ctx, ME_ERR_RANGE, "voxel keys span too large a box");
    L.nvox[a] = (int)(hi[a] - lo[a] + 1); nvox *= L.nvox[a];
  }
  L.nvoxels = nvox; L.v = voxel_size;
  for (int64_t i = 0; i < n_rows; ++i)
    vox[i] = ((key[3 * i + 2] - lo[2]) * L.nvox[1] + (key[3 * i + 1] - lo[1])) * L.nvox[0] + (key[3 * i] - lo[0]);
  auto align = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t o_rows = 0, o_vox = o_rows + align((size_t)n_rows * 27 * 8), o_w = o_vox + align((size_t)n_rows * 8),
               o_wv = o_w + align((size_t)n_rows * 8), o_pl = o_wv + align((size_t)nvox * 8), total = o_pl + align((size_t)n_rows * 4);
  ME_TRY(ensure_work(ctx, total));
  char *base = (char *)ctx->d_work;
  double *d_rows = (double *)(base + o_rows), *d_w = (double *)(base + o_w), *d_wv = (double *)(base + o_wv);
  long long *d_vox = (long long *)(base + o_vox);
  uint32_t *d_pl = (uint32_t *)(base + o_pl);
  AwdAcc *acc = (AwdAcc *)ctx->d_scratch;
  unsigned long long *occ = (unsigned long long *)((char *)ctx->d_scratch + 256);
  ME_CUDA(ctx, cudaMemcpyAsync(d_rows, rows27, (size_t)n_rows * 27 * 8, cudaMemcpyHostToDevice, ctx->stream));
  ME_CUDA(ctx, cudaMemcpyAsync(d_vox, vox.data(), (size_t)n_rows * 8, cudaMemcpyHostToDevice, ctx->stream));
  zero_awd_acc_kernel<<<1, 1, 0, ctx->stream>>>(acc, occ);
  ME_LAUNCH_CHECK(ctx);
  fill_nan_kernel<<<ctx->sm_count * 4, kThreads, 0, ctx->stream>>>(d_wv, nvox);
  ME_LAUNCH_CHECK(ctx);
  awd_rows_kernel<<<std::max(1, (int)std::min<long long>((n_rows + kThreads - 1) / kThreads, ctx->sm_count * 8)), kThreads, 0, ctx->stream>>>(
      d_rows, n_rows, d_vox, d_w, d_wv, d_pl, acc);
  ME_LAUNCH_CHECK(ctx);
  if (scs_radius == 5) scs_kernel<5><<<ctx->sm_count * 4, kThreads, 0, ctx->stream>>>(L, d_wv, d_pl, scs_radius, acc);
  else scs_kernel<0><<<ctx->sm_count * 4, kThreads, 0, ctx->stream>>>(L, d_wv, d_pl, scs_radius, acc);
  ME_LAUNCH_CHECK(ctx);
  trace_scs(ctx, scs_radius);
  AwdAcc *h = (AwdAcc *)ctx->h_pinned;
  ME_CUDA(ctx, cudaMemcpyAsync(h, acc, sizeof(AwdAcc), cudaMemcpyDeviceToHost, ctx->stream));
  if (w_out) ME_CUDA(ctx, cudaMemcpyAsync(w_out, d_w, (size_t)n_rows * 8, cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  out->n_pairs = n_rows;
  out->n_scs = (int64_t)h->n_scs;
  out->awd = h->sum_w / (double)n_rows;
  out->scs = h->sum_scs / (double)h->n_scs;
  return ME_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// The Gaussian 2-Wasserstein distance per voxel pair (DESIGN §3.18): mu, Sigma = M2 / (n - 1), offset o = |mu_est - mu_gt|,
// shape b = Bures(Sigma_gt, Sigma_est), W2 = sqrt(o^2 + b^2).  b^2 = tr Sigma_gt + tr Sigma_est - 2 tr((A Sigma_est A)^1/2)
// (A = Sigma_gt^1/2, B = Sigma_est^1/2) subtracts nearly equal numbers; it is also min over orthogonal U of |A - B U|_F^2,
// reached at U = P Q^T for the SVD B A = P S Q^T, and that residual is a sum of squares in which nothing cancels.
// ---------------------------------------------------------------------------------------------------------------
struct W2Acc {            // scs_kernel reads and updates the AwdAcc in front (n_active / n_new stay 0)
  AwdAcc a;
  double sum_offset, sum_shape;
};
struct W2Dev {            // me_ctx::d_w2
  W2Acc acc;
  unsigned long long occ[2];
  double blk[ME_W2_BLOCK];
};

// Sigma^1/2 of a symmetric 3x3 (row-major), eigenvalues clamped at 0
__device__ void sqrt_psd(const double *sig, double *r) {
  double w[3], v[9];
  eig3_jacobi(sig, w, v);
#pragma unroll
  for (int k = 0; k < 3; ++k) w[k] = sqrt(fmax(w[k], 0.0));
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) r[i * 3 + j] = v[i * 3] * w[0] * v[j * 3] + v[i * 3 + 1] * w[1] * v[j * 3 + 1] + v[i * 3 + 2] * w[2] * v[j * 3 + 2];
}

// offset and shape terms of (mu_g, Sigma_g) against (mu_e, Sigma_e); symmetric in the two up to rounding
__device__ void w2_terms(const double *mu_g, const double *sig_g, const double *mu_e, const double *sig_e, double &o, double &b) {
  const double d0 = mu_e[0] - mu_g[0], d1 = mu_e[1] - mu_g[1], d2 = mu_e[2] - mu_g[2];
  o = sqrt(d0 * d0 + d1 * d1 + d2 * d2);
  double A[9], B[9], M[9], P[9], s[3], Q[9], R[9];
  sqrt_psd(sig_g, A);
  sqrt_psd(sig_e, B);
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) M[i * 3 + j] = B[i * 3] * A[j] + B[i * 3 + 1] * A[3 + j] + B[i * 3 + 2] * A[6 + j];
  svd3(M, P, s, Q);
  if (!(s[0] > 0.0)) {
    // B A = 0: tr(A B U) = 0 for every U, so U = I reaches the minimum
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
  } else {
    if (!(s[1] > 0.0)) {
      // rank 1: svd3 leaves P's second column 0; any unit vector orthogonal to the first serves (s_2 = s_3 = 0)
      const double ax = fabs(P[0]), ay = fabs(P[3]), az = fabs(P[6]);
      const int k = (ax <= ay && ax <= az) ? 0 : (ay <= az ? 1 : 2);
      double e[3] = {0.0, 0.0, 0.0};
      e[k] = 1.0;
      const double pk = P[k * 3];
      double n2 = 0.0;
#pragma unroll
      for (int i = 0; i < 3; ++i) { P[i * 3 + 1] = e[i] - pk * P[i * 3]; n2 += P[i * 3 + 1] * P[i * 3 + 1]; }
      const double inv = 1.0 / sqrt(n2);
#pragma unroll
      for (int i = 0; i < 3; ++i) P[i * 3 + 1] *= inv;
    }
    // the third column: orthogonal to the first two, with the sign for which P S Q^T = B A, i.e. p3 . (B A q3) >= 0 (when
    // s_3 = 0 both signs give the same residual)
    P[2] = P[3] * P[7] - P[6] * P[4]; P[5] = P[6] * P[1] - P[0] * P[7]; P[8] = P[0] * P[4] - P[3] * P[1];
    double dot = 0.0;
#pragma unroll
    for (int i = 0; i < 3; ++i) dot += P[i * 3 + 2] * (M[i * 3] * Q[2] + M[i * 3 + 1] * Q[5] + M[i * 3 + 2] * Q[8]);
    if (dot < 0.0) { P[2] = -P[2]; P[5] = -P[5]; P[8] = -P[8]; }
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) R[i * 3 + j] = P[i * 3] * Q[j * 3] + P[i * 3 + 1] * Q[j * 3 + 1] + P[i * 3 + 2] * Q[j * 3 + 2];
  }
  double ss = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double r = A[i * 3 + j] - (B[i * 3] * R[j] + B[i * 3 + 1] * R[3 + j] + B[i * 3 + 2] * R[6 + j]);
      ss += r * r;
    }
  b = sqrt(ss);
}

// mu and the unbiased covariance M2 / (n - 1) (xx xy xz yy yz zz) of a voxel from its moments about the centre c
__device__ void unbiased_gaussian(const double *mom, int n, double cx, double cy, double cz, double *mu, double *sig6) {
  const double nd = (double)n, nm1 = (double)(n - 1);
  mu[0] = cx + mom[0] / nd; mu[1] = cy + mom[1] / nd; mu[2] = cz + mom[2] / nd;
  sig6[0] = (mom[3] - mom[0] * mom[0] / nd) / nm1; sig6[1] = (mom[4] - mom[0] * mom[1] / nd) / nm1;
  sig6[2] = (mom[5] - mom[0] * mom[2] / nd) / nm1; sig6[3] = (mom[6] - mom[1] * mom[1] / nd) / nm1;
  sig6[4] = (mom[7] - mom[1] * mom[2] / nd) / nm1; sig6[5] = (mom[8] - mom[2] * mom[2] / nd) / nm1;
}

__device__ inline void sym9(const double *t, double *s) {
  s[0] = t[0]; s[1] = t[1]; s[2] = t[2]; s[3] = t[1]; s[4] = t[3]; s[5] = t[4]; s[6] = t[2]; s[7] = t[4]; s[8] = t[5];
}

// one pair's terms into the accumulators and, when asked, its row (ME_W2_ROW_COLS columns)
__device__ double w2_pair(const double *mu_e, const double *sig6_e, const double *mu_g, const double *sig6_g, W2Acc *acc,
                          double *row) {
  double se[9], sg[9], o, b;
  sym9(sig6_e, se);
  sym9(sig6_g, sg);
  w2_terms(mu_g, sg, mu_e, se, o, b);
  const double w = sqrt(o * o + b * b);
  atomicAdd(&acc->a.sum_w, w);
  atomicAdd(&acc->sum_offset, o);
  atomicAdd(&acc->sum_shape, b);
  if (row) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { row[5 + k] = mu_e[k]; row[8 + k] = mu_g[k]; }
#pragma unroll
    for (int k = 0; k < 6; ++k) { row[11 + k] = sig6_e[k]; row[17 + k] = sig6_g[k]; }
    row[23] = o; row[24] = b; row[25] = w;
  }
  return w;
}

// pairing as awd_kernel: one thread per est voxel
__global__ void __launch_bounds__(kThreads)
w2_kernel(Lattice Le, Lattice Lg, const int32_t *__restrict__ cnt_e, const double *__restrict__ mom_e,
          const int32_t *__restrict__ cnt_g, const double *__restrict__ mom_g, int min_points, double missing,
          double *__restrict__ w_out, uint32_t *__restrict__ pair_list, double *__restrict__ rows, W2Acc *__restrict__ acc) {
  for (long long vox = blockIdx.x * (long long)blockDim.x + threadIdx.x; vox < Le.nvoxels;
       vox += (long long)gridDim.x * blockDim.x) {
    double w = missing;      // NaN, or -1 when the table is MAX-all-reduced across ranks (slab layout)
    const int ne = cnt_e[vox];
    if (ne >= min_points) {
      const int vx = (int)(vox % Le.nvox[0]);
      const int vy = (int)((vox / Le.nvox[0]) % Le.nvox[1]);
      const int vz = (int)(vox / ((long long)Le.nvox[0] * Le.nvox[1]));
      const long long kx = (long long)Le.k_lo[0] + vx, ky = (long long)Le.k_lo[1] + vy, kz = (long long)Le.k_lo[2] + vz;
      const long long gx = kx - Lg.k_lo[0], gy = ky - Lg.k_lo[1], gz = kz - Lg.k_lo[2];
      int ng = 0;
      long long gvox = -1;
      if (gx >= 0 && gx < Lg.nvox[0] && gy >= 0 && gy < Lg.nvox[1] && gz >= 0 && gz < Lg.nvox[2]) {
        gvox = (gz * Lg.nvox[1] + gy) * (long long)Lg.nvox[0] + gx;
        ng = cnt_g[gvox];
      }
      if (ng >= min_points) {
        const double cx = ((double)kx + 0.5) * Le.v, cy = ((double)ky + 0.5) * Le.v, cz = ((double)kz + 0.5) * Le.v;
        double mu_e[3], sig_e[6], mu_g[3], sig_g[6];
        unbiased_gaussian(mom_e + vox * 9, ne, cx, cy, cz, mu_e, sig_e);
        unbiased_gaussian(mom_g + gvox * 9, ng, cx, cy, cz, mu_g, sig_g);
        const unsigned long long slot = atomicAdd(&acc->a.n_pairs, 1ull);
        pair_list[slot] = (uint32_t)vox;
        double *r = rows ? rows + slot * ME_W2_ROW_COLS : nullptr;
        if (r) {
          r[0] = (double)kx * Le.v; r[1] = (double)ky * Le.v; r[2] = (double)kz * Le.v;
          r[3] = (double)ng; r[4] = (double)ne;
        }
        w = w2_pair(mu_e, sig_e, mu_g, sig_g, acc, r);
      }
    }
    w_out[vox] = w;
  }
}

// the eight SUM-reducible values of the stage -> its block
__global__ void pack_w2_kernel(W2Dev *d) {
  if (threadIdx.x != 0) return;
  const W2Acc &a = d->acc;
  double *blk = d->blk;
  blk[0] = (double)a.a.n_pairs; blk[1] = (double)a.a.n_scs; blk[2] = (double)d->occ[0]; blk[3] = (double)d->occ[1];
  blk[4] = a.a.sum_w; blk[5] = a.a.sum_scs; blk[6] = a.sum_offset; blk[7] = a.sum_shape;
}

static int w2_state(me_ctx *ctx, W2Dev **d) {
  if (!ctx->d_w2) {
    const cudaError_t e = cudaMalloc(&ctx->d_w2, sizeof(W2Dev));
    if (e != cudaSuccess) {
      ctx->d_w2 = nullptr;
      cudaGetLastError();
      return fail(ctx, ME_ERR_NOMEM, std::string("cudaMalloc of the W2 accumulators: ") + cudaGetErrorString(e));
    }
  }
  *d = (W2Dev *)ctx->d_w2;
  ME_CUDA(ctx, cudaMemsetAsync(*d, 0, sizeof(W2Dev), ctx->stream));
  return ME_OK;
}

static int w2_begin_impl(me_ctx *ctx, double voxel_size, int min_points, bool want_rows, double **d_rows_out) {
  ctx->w2_finished = false;
  if (min_points < 2) return fail(ctx, ME_ERR_INVALID, "W2: min_points must be >= 2 (the unbiased covariance divides by n - 1)");
  VoxelTables t;
  ME_TRY(voxel_layout(ctx, voxel_size, min_points, ME_W2_ROW_COLS, want_rows, t));
  if (d_rows_out) *d_rows_out = t.rows;
  W2Dev *d = nullptr;
  ME_TRY(w2_state(ctx, &d));
  ME_TRY(voxel_moments(ctx, t, d->occ));
  int blocks = (int)std::min<long long>((t.Le.nvoxels + kThreads - 1) / kThreads, (long long)ctx->sm_count * 8);
  w2_kernel<<<std::max(1, blocks), kThreads, 0, ctx->stream>>>(t.Le, t.Lg, t.cnt_e, t.mom_e, t.cnt_g, t.mom_g, min_points,
                                                              t.slab ? -1.0 : (double)NAN, t.w_vox, t.pair_list, t.rows, &d->acc);
  ME_LAUNCH_CHECK(ctx);
  ctx->w2_open = true;
  ctx->vox_nvox = t.Le.nvoxels;
  ctx->vox_o_w = t.o_w;
  ctx->vox_o_pairs = t.o_pairs;
  return ME_OK;
}

static int launch_scs(me_ctx *ctx, const Lattice &L, const double *w_vox, const uint32_t *pair_list, int scs_radius, AwdAcc *acc) {
  if (scs_radius == 5) scs_kernel<5><<<ctx->sm_count * 4, kThreads, 0, ctx->stream>>>(L, w_vox, pair_list, scs_radius, acc);
  else scs_kernel<0><<<ctx->sm_count * 4, kThreads, 0, ctx->stream>>>(L, w_vox, pair_list, scs_radius, acc);
  ME_LAUNCH_CHECK(ctx);
  trace_scs(ctx, scs_radius);
  return ME_OK;
}

int w2_begin(me_ctx *ctx, double voxel_size, int min_points) { return w2_begin_impl(ctx, voxel_size, min_points, false, nullptr); }

int w2_w_table(me_ctx *ctx, double **d_w, int64_t *n) {
  if (!ctx->w2_open) return fail(ctx, ME_ERR_INVALID, "me_w2_w_table before me_w2_begin");
  *d_w = (double *)((char *)ctx->d_work + ctx->vox_o_w);
  *n = (int64_t)ctx->vox_nvox;
  return ME_OK;
}

int w2_finish_block(me_ctx *ctx, int scs_radius) {
  if (!ctx->w2_open) return fail(ctx, ME_ERR_INVALID, "me_w2_finish_accum_device before me_w2_begin");
  if (scs_radius < 0 || scs_radius > 64) return fail(ctx, ME_ERR_INVALID, "scs_radius out of range");
  ctx->w2_open = false;
  W2Dev *d = (W2Dev *)ctx->d_w2;
  ME_TRY(launch_scs(ctx, ctx->cloud[ME_CLOUD_EST].lat, (const double *)((char *)ctx->d_work + ctx->vox_o_w),
                    (const uint32_t *)((char *)ctx->d_work + ctx->vox_o_pairs), scs_radius, &d->acc.a));
  pack_w2_kernel<<<1, 32, 0, ctx->stream>>>(d);
  ME_LAUNCH_CHECK(ctx);
  ctx->w2_finished = true;
  return ME_OK;
}

int w2_block(me_ctx *ctx, double **d_block, int32_t *n) {
  if (!ctx->w2_finished) return fail(ctx, ME_ERR_INVALID, "me_w2_block before me_w2_finish_accum_device");
  *d_block = ((W2Dev *)ctx->d_w2)->blk;
  *n = ME_W2_BLOCK;
  return ME_OK;
}

static void w2_result(const double v[ME_W2_BLOCK], me_w2_result *out) {
  auto i64 = [](double x) { return (int64_t)std::llround(x); };
  std::memset(out, 0, sizeof(*out));
  out->n_pairs = i64(v[0]); out->n_scs = i64(v[1]);
  out->n_voxels_est = i64(v[2]); out->n_voxels_gt = i64(v[3]);
  out->aw2 = v[4] / (double)out->n_pairs;           // 0/0 -> NaN
  out->scs = v[5] / (double)out->n_scs;
  out->mean_offset = v[6] / (double)out->n_pairs;
  out->mean_shape = v[7] / (double)out->n_pairs;
}

int w2_fetch(me_ctx *ctx, me_w2_result *out) {
  std::memset(out, 0, sizeof(*out));
  if (!ctx->w2_finished) return fail(ctx, ME_ERR_INVALID, "me_w2_fetch before me_w2_finish_accum_device");
  double *h = (double *)ctx->h_pinned;
  ME_CUDA(ctx, cudaMemcpyAsync(h, ((W2Dev *)ctx->d_w2)->blk, ME_W2_BLOCK * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  w2_result(h, out);
  return ME_OK;
}

int run_w2(me_ctx *ctx, double voxel_size, int min_points, int scs_radius, me_w2_result *out, int64_t *n_rows, double **rows) {
  std::memset(out, 0, sizeof(*out));
  if (n_rows) *n_rows = 0;
  if (rows) *rows = nullptr;
  if (scs_radius < 0 || scs_radius > 64) return fail(ctx, ME_ERR_INVALID, "scs_radius out of range");
  double *d_rows = nullptr;
  ME_TRY(w2_begin_impl(ctx, voxel_size, min_points, rows != nullptr, &d_rows));
  if (ctx->cloud[ME_CLOUD_EST].slab || ctx->cloud[ME_CLOUD_GT].slab) {
    ctx->w2_open = false;
    return fail(ctx, ME_ERR_INVALID, "slab layout: run the W2 stage as me_w2_begin / all-reduce of me_w2_w_table / "
                                     "me_w2_finish_accum_device / all-reduce of me_w2_block / me_w2_fetch");
  }
  ME_TRY(w2_finish_block(ctx, scs_radius));
  ME_TRY(w2_fetch(ctx, out));
  if (n_rows) *n_rows = out->n_pairs;
  if (rows) {
    const size_t row_bytes = ME_W2_ROW_COLS * sizeof(double);
    double *hr = (double *)std::malloc((size_t)std::max<int64_t>(out->n_pairs, 1) * row_bytes);
    if (!hr) return fail(ctx, ME_ERR_NOMEM, "malloc(W2 rows) failed");
    if (out->n_pairs > 0) {
      const cudaError_t e = cudaMemcpyAsync(hr, d_rows, (size_t)out->n_pairs * row_bytes, cudaMemcpyDeviceToHost, ctx->stream);
      if (e != cudaSuccess || cudaStreamSynchronize(ctx->stream) != cudaSuccess) {
        std::free(hr);
        return fail(ctx, ME_ERR_CUDA, std::string("copying the W2 rows: ") + cudaGetErrorString(cudaGetLastError()));
      }
    }
    *rows = hr;
  }
  return ME_OK;
}

// W2 and SCS on GIVEN Gaussians (ME_W2_ROW_COLS rows): the counterpart of awd_rows_kernel
__global__ void __launch_bounds__(kThreads)
w2_rows_kernel(const double *__restrict__ rows, long long n, const long long *__restrict__ vox_of_row, double *__restrict__ w_rows,
               double *__restrict__ w_vox, uint32_t *__restrict__ pair_list, W2Acc *__restrict__ acc) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double *r = rows + i * ME_W2_ROW_COLS;
    double se[9], sg[9], o, b;
    sym9(r + 11, se);
    sym9(r + 17, sg);
    w2_terms(r + 8, sg, r + 5, se, o, b);
    const double w = sqrt(o * o + b * b);
    w_rows[3 * i] = o; w_rows[3 * i + 1] = b; w_rows[3 * i + 2] = w;
    w_vox[vox_of_row[i]] = w;
    pair_list[i] = (uint32_t)vox_of_row[i];
    atomicAdd(&acc->a.sum_w, w);
    atomicAdd(&acc->sum_offset, o);
    atomicAdd(&acc->sum_shape, b);
    if (i == 0) acc->a.n_pairs = (unsigned long long)n;
  }
}

int run_w2_rows(me_ctx *ctx, const double *rows, int64_t n_rows, double voxel_size, int scs_radius, double *w_out,
                me_w2_result *out) {
  std::memset(out, 0, sizeof(*out));
  if (n_rows <= 0 || !rows || !(voxel_size > 0)) return fail(ctx, ME_ERR_INVALID, "bad arguments");
  if (scs_radius < 0 || scs_radius > 64) return fail(ctx, ME_ERR_INVALID, "scs_radius out of range");
  ctx->vox_open = false;      // the work buffer is reused below
  ctx->w2_open = false;
  ctx->w2_finished = false;
  std::vector<long long> key(3 * (size_t)n_rows), vox((size_t)n_rows);
  long long lo[3] = {LLONG_MAX, LLONG_MAX, LLONG_MAX}, hi[3] = {LLONG_MIN, LLONG_MIN, LLONG_MIN};
  for (int64_t i = 0; i < n_rows; ++i)
    for (int a = 0; a < 3; ++a) {
      const long long k = llround(rows[i * ME_W2_ROW_COLS + a] / voxel_size);
      key[3 * i + a] = k; lo[a] = std::min(lo[a], k); hi[a] = std::max(hi[a], k);
    }
  Lattice L;
  std::memset(&L, 0, sizeof(L));
  long long nvox = 1;
  for (int a = 0; a < 3; ++a) {
    if (hi[a] - lo[a] + 1 > 4096) return fail(ctx, ME_ERR_RANGE, "voxel keys span too large a box");
    L.nvox[a] = (int)(hi[a] - lo[a] + 1); nvox *= L.nvox[a];
  }
  L.nvoxels = nvox; L.v = voxel_size;
  for (int64_t i = 0; i < n_rows; ++i)
    vox[i] = ((key[3 * i + 2] - lo[2]) * L.nvox[1] + (key[3 * i + 1] - lo[1])) * L.nvox[0] + (key[3 * i] - lo[0]);
  auto align = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t o_rows = 0, o_vox = o_rows + align((size_t)n_rows * ME_W2_ROW_COLS * 8), o_w = o_vox + align((size_t)n_rows * 8),
               o_wv = o_w + align((size_t)n_rows * 3 * 8), o_pl = o_wv + align((size_t)nvox * 8), total = o_pl + align((size_t)n_rows * 4);
  ME_TRY(ensure_work(ctx, total));
  char *base = (char *)ctx->d_work;
  double *d_rows = (double *)(base + o_rows), *d_w = (double *)(base + o_w), *d_wv = (double *)(base + o_wv);
  long long *d_vox = (long long *)(base + o_vox);
  uint32_t *d_pl = (uint32_t *)(base + o_pl);
  W2Dev *d = nullptr;
  ME_TRY(w2_state(ctx, &d));
  ME_CUDA(ctx, cudaMemcpyAsync(d_rows, rows, (size_t)n_rows * ME_W2_ROW_COLS * 8, cudaMemcpyHostToDevice, ctx->stream));
  ME_CUDA(ctx, cudaMemcpyAsync(d_vox, vox.data(), (size_t)n_rows * 8, cudaMemcpyHostToDevice, ctx->stream));
  fill_nan_kernel<<<ctx->sm_count * 4, kThreads, 0, ctx->stream>>>(d_wv, nvox);
  ME_LAUNCH_CHECK(ctx);
  w2_rows_kernel<<<std::max(1, (int)std::min<long long>((n_rows + kThreads - 1) / kThreads, ctx->sm_count * 8)), kThreads, 0, ctx->stream>>>(
      d_rows, n_rows, d_vox, d_w, d_wv, d_pl, &d->acc);
  ME_LAUNCH_CHECK(ctx);
  ME_TRY(launch_scs(ctx, L, d_wv, d_pl, scs_radius, &d->acc.a));
  pack_w2_kernel<<<1, 32, 0, ctx->stream>>>(d);
  ME_LAUNCH_CHECK(ctx);
  ctx->w2_finished = true;
  if (w_out) ME_CUDA(ctx, cudaMemcpyAsync(w_out, d_w, (size_t)n_rows * 3 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  return w2_fetch(ctx, out);
}

}  // namespace me

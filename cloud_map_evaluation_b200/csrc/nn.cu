// nn.cu — exact 1-NN sweeps and the inlier statistics built on them.
//
// Replaces (reference, map_eval/src/map_eval.cpp):
//   :1213-1236  two serial KDTreeFlann::SearchKNN(p, 1) loops of calculateMetricsWithInitialMatrix
//   :1069-1145  getDiffRegResultWithCorrespondence (five-threshold accumulators; == :990-1067, :828-897)
//   :1398-1431  computeChamferDistance (sum of sqrt(d2) over ALL points, unbounded NN)
//
// One thread per query, queries walked in their own cell-sorted order so that a warp's 32 queries sit in the same
// few lattice rows and its candidate loads hit the same L1 lines.  Per query the 3x3x3 cell block of the reference
// lattice is 9 contiguous x-runs (3 x-adjacent cells are adjacent in the CSR layout).  Candidates are screened in fp32
// on the cell-relative copies; the winner — and every candidate inside the fp32 error bound of the winner — is evaluated
// in fp64 with exactly the reference's operation order (no FMA contraction), so the arg-min, the cut-off test and every
// inlier comparison are bit-identical to the CPU path.  A query whose best distance does not beat the distance to the
// faces of its searched block is finished by a warp-per-query ring-expansion kernel (rare: ~0.05 % of queries on
// volume-filling clouds).  The sweeps only record (index, nanoflann-order d2, Eigen-order squared norm) per query;
// nn_stats_kernel folds those arrays into the accumulators.
//   nn_flat_kernel   default: per-thread run table in shared memory + flattened candidate walk
//   nn_tile_kernel   lattices the flat kernel cannot index (>= 2^24 cells along x or points per run): one CTA per
//                    4x4x4-cell query tile, 6x6x6-cell region staged with TMA bulk copies.  ME_NN_TILE (env) forces it.
#include "common.cuh"
#include "records.cuh"
#include "tile.cuh"
#include "flat.cuh"
#include "radix.cuh"
#include <algorithm>
#include <cstdlib>
#include <cstring>

namespace me {

static constexpr int kThreads = 256;

// distance (in cells) from lattice coordinate (uy, uz) to the nearest plane of the reference lattice that is NOT laid out on
// this rank: beyond it the cloud is unknown, not empty
__device__ __forceinline__ double cover_dist_cells(const NNConst &C, double uy, double uz) {
  if (C.cov_axis == 0) return INFINITY;
  const double ua = C.cov_axis == 1 ? uy : uz;
  return fmin(C.cov_lo > 0 ? ua - (double)C.cov_lo : INFINITY, C.cov_hi < C.cov_dim ? (double)C.cov_hi - ua : INFINITY);
}

// device accumulator block of one direction: 8 x int64, 11 fp64 summed with atomics, then what merge_moments_kernel
// derives from the blocks' (n, mean, M2) of the kept d: their mean and M2, and sum(d), sum(d^2) (= n mean, M2 + n mean^2)
struct AccBlock {
  unsigned long long n_corr, n_inl[5], n_ub, n_far;
  double sum_d[5], sum_d2[5], sum_nn;
  double mean_all, m2_all, sum_d_all, sum_d2_all;
};

struct LocalAcc {
  unsigned int n_corr, n_inl[5], n_ub;
  double sum_d[5], sum_d2[5], sum_nn;
  // this thread's kept d as sums of (d - shift) and (d - shift)^2, shift = its first kept d: the sums then cancel by at
  // most a factor n_corr + 1 when they are turned into (mean, M2), since n (mean - shift)^2 <= n M2
  double shift, s1, s2;
  __device__ void clear() {
    n_corr = 0; n_ub = 0; sum_nn = 0; shift = 0; s1 = 0; s2 = 0;
#pragma unroll
    for (int k = 0; k < 5; ++k) { n_inl[k] = 0; sum_d[k] = 0; sum_d2[k] = 0; }
  }
  __device__ __forceinline__ void pair(double nd, double) {
    if (n_corr++ == 0) shift = nd;
    const double t = nd - shift;
    s1 += t;
    s2 += t * t;
  }
  __device__ __forceinline__ void inlier(int k, double nd, double sq) { sum_d[k] += nd; sum_d2[k] += sq; n_inl[k]++; }
  __device__ __forceinline__ void nn_dist(double d) { sum_nn += d; }
  __device__ __forceinline__ void ub() { n_ub++; }
};

// (n, mean, M2) of the whole block from every thread's (n, mean, M2), valid in thread 0; every thread of the block calls it
__device__ void block_moments(double &n, double &m, double &m2) {
  __shared__ double sh[kThreads / 32][3];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double nb = __shfl_xor_sync(0xffffffffu, n, o), mb = __shfl_xor_sync(0xffffffffu, m, o),
                 m2b = __shfl_xor_sync(0xffffffffu, m2, o);
    chan_merge(n, m, m2, nb, mb, m2b);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { sh[warp][0] = n; sh[warp][1] = m; sh[warp][2] = m2; }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) chan_merge(n, m, m2, sh[w][0], sh[w][1], sh[w][2]);
}

// the sums and counts go to g with atomics; the block's (n, mean, M2) of the kept d to mom[3 * blockIdx.x ..] (nullable:
// the kernel keeps no pairs), which merge_moments_kernel folds in block order
__device__ void flush_acc(LocalAcc &a, AccBlock *g, double *mom) {
  __shared__ double sh_d[kThreads / 32][11];
  __shared__ unsigned long long sh_i[kThreads / 32][7];
  double mn = (double)a.n_corr, mm = 0, m2 = 0;
  if (a.n_corr) { mm = a.shift + a.s1 / mn; m2 = fmax(0.0, a.s2 - a.s1 * (a.s1 / mn)); }
  block_moments(mn, mm, m2);
  if (mom && threadIdx.x == 0) { mom[3 * blockIdx.x] = mn; mom[3 * blockIdx.x + 1] = mm; mom[3 * blockIdx.x + 2] = m2; }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double dv[11];
  long long iv[7];
#pragma unroll
  for (int k = 0; k < 5; ++k) { dv[k] = a.sum_d[k]; dv[5 + k] = a.sum_d2[k]; iv[1 + k] = a.n_inl[k]; }
  dv[10] = a.sum_nn;
  iv[0] = a.n_corr; iv[6] = a.n_ub;
#pragma unroll
  for (int k = 0; k < 11; ++k) dv[k] = warp_sum(dv[k]);
#pragma unroll
  for (int k = 0; k < 7; ++k) iv[k] = warp_sum_ll(iv[k]);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 11; ++k) sh_d[warp][k] = dv[k];
#pragma unroll
    for (int k = 0; k < 7; ++k) sh_i[warp][k] = (unsigned long long)iv[k];
  }
  __syncthreads();
  const int nwarps = blockDim.x >> 5;
  if (threadIdx.x < 11) {
    double s = 0;
    for (int w = 0; w < nwarps; ++w) s += sh_d[w][threadIdx.x];
    double *dst = &g->sum_d[0];
    if (s != 0.0) atomicAdd(dst + threadIdx.x, s);
  } else if (threadIdx.x >= 32 && threadIdx.x < 39) {
    int k = threadIdx.x - 32;
    unsigned long long s = 0;
    for (int w = 0; w < nwarps; ++w) s += sh_i[w][k];
    unsigned long long *dst = &g->n_corr;   // n_corr, n_inl[5], n_ub are contiguous
    if (s) atomicAdd(dst + k, s);
  }
}

// face distance of the searched block [ic - r, ic + r] (cells) around continuous coordinate u, in cells;
// faces beyond the lattice are at infinity (nothing lives there)
__device__ __forceinline__ double face_dist_cells(double u, long long ic, int r, int dim) {
  double lo = (ic - r <= 0) ? INFINITY : u - (double)(ic - r);
  double hi = (ic + r + 1 >= dim) ? INFINITY : (double)(ic + r + 1) - u;
  return fmin(lo, hi);
}

// ---------------------------------------------------------------------------------------------------------------
// shared pieces of the sweep
// ---------------------------------------------------------------------------------------------------------------
struct Best {
  double d2; int idx; double dx, dy, dz;
  __device__ __forceinline__ void init() { d2 = INFINITY; idx = 0x7fffffff; dx = dy = dz = 0; }
  // exact fp64 evaluation in the reference's operation order; ties go to the smaller caller index
  __device__ __forceinline__ bool offer(const P4 &q, double px, double py, double pz, int pidx) {
    const double ddx = __dsub_rn(q.x, px), ddy = __dsub_rn(q.y, py), ddz = __dsub_rn(q.z, pz);
    const double v = __dadd_rn(__dadd_rn(__dmul_rn(ddx, ddx), __dmul_rn(ddy, ddy)), __dmul_rn(ddz, ddz));
    if (v < d2 || (v == d2 && pidx < idx)) { d2 = v; idx = pidx; dx = ddx; dy = ddy; dz = ddz; return true; }
    return false;
  }
};

// 3x3x3 block around reference cell (ix,iy,iz), straight from global memory (fallback path)
__device__ __forceinline__ void search_block_global(const P4 &q, long long ix, long long iy, long long iz,
                                                    const P4 *__restrict__ R, const uint32_t *__restrict__ cell_off,
                                                    const Lattice &L, Best &b) {
  const int x0 = (int)max(ix - 1, 0ll), x1 = (int)min(ix + 1, (long long)L.dims[0] - 1);
  if (x0 > x1) return;
  for (int dz = -1; dz <= 1; ++dz) {
    const long long z = iz + dz;
    if (z < 0 || z >= L.dims[2]) continue;
    for (int dy = -1; dy <= 1; ++dy) {
      const long long y = iy + dy;
      if (y < 0 || y >= L.dims[1]) continue;
      const long long row = (z * L.dims[1] + y) * (long long)L.dims[0];
      const uint32_t s = __ldg(cell_off + row + x0), e = __ldg(cell_off + row + x1 + 1);
      for (uint32_t j = s; j < e; ++j) {
        const P4 p = load_p4(R + j);
        b.offer(q, p.x, p.y, p.z, orig_of(p.idx));
      }
    }
  }
}

// after the 3x3x3 block: is the best provably the global nearest neighbour?  If so record it (index, nanoflann-order d2 for
// the cut-off, Eigen-order squared norm for the statistics; nn_stats_kernel folds them into the accumulators), otherwise
// hand the query to the ring-expansion kernel.  AW: ME_PAIRING_AS_WRITTEN gt->est (C.accumulate == 0), compiled apart so
// that the other sweeps keep their code (and AW's drops the winner's offsets, which only the Eigen-order norm reads).
template <bool AW>
__device__ __forceinline__ void finish_query(const P4 &q, uint32_t i, long long ix, long long iy, long long iz,
                                             const Lattice &L, const NNConst &C, const Best &b,
                                             int32_t *__restrict__ nn_idx, double *__restrict__ nn_d2,
                                             double *__restrict__ nn_sq, uint32_t *__restrict__ far_list,
                                             unsigned int *__restrict__ far_count, double ux, double uy, double uz,
                                             double slack_h) {
  const double gcov = cover_dist_cells(C, uy, uz);
  const double g = fmin(fmin(fmin(face_dist_cells(ux, ix, 1, L.dims[0]), face_dist_cells(uy, iy, 1, L.dims[1])),
                             face_dist_cells(uz, iz, 1, L.dims[2])), gcov) * L.h;
  const double slack = slack_h * L.h + 1e-14 * (fabs(q.x) + fabs(q.y) + fabs(q.z) + C.ref_maxabs);
  const double ge = g - slack;
  const double ge2 = ge > 0 ? ge * ge : 0.0;
  bool resolved = b.d2 < ge2;
  bool beyond = false;
  if (!resolved && ge2 > C.max_d2) { resolved = true; beyond = b.d2 > C.max_d2; }   // nothing farther matters
  if (!resolved) {
    nn_idx[i] = b.d2 < INFINITY ? b.idx : -1;
    nn_d2[i] = b.d2;
    far_list[atomicAdd(far_count, 1u)] = i;
    return;
  }
  if (beyond || !(b.d2 < INFINITY)) { nn_idx[i] = -1; nn_d2[i] = INFINITY; return; }
  nn_idx[i] = b.idx;
  nn_d2[i] = b.d2;
  if (!AW) nn_sq[i] = sqnorm_eigen(b.dx, b.dy, b.dz);
  // as-written: the swapped pair's squared norm (two random gathers, issued here inside the latency-bound sweep) for
  // pair_as_written_kernel to fold; pairs past the cut-off are never read
  else if (keep_pair(b.d2, C))
    nn_sq[i] = as_written_sq(b.idx, orig_of(q.idx), C.aw_gt_xyz, C.aw_n_gt, C.aw_est_xyz, C.aw_n_est);
}

// clamp a (possibly far outside) lattice coordinate to one cell beyond the lattice
__device__ __forceinline__ long long clamp_cell(long long i, int dim) { return i < -1 ? -1 : (i > dim ? dim : i); }

// ---------------------------------------------------------------------------------------------------------------
// tile sweep.  One CTA = one query tile (4x4x4 cells of the shared cell grid).  The 6x6x6 reference cells around it
// are 36 contiguous x-runs of the cell-sorted reference cloud; each run is brought into shared memory with one TMA
// bulk copy (raw 32-byte records), then re-expressed as fp32 offsets from the tile centre (error < 2e-7 h).  Every
// thread owns one query of the tile and walks its own 3x3x3 window inside the staged region: candidates are screened
// with fp32 arithmetic, and every candidate that could still be the nearest neighbour given the fp32 error bound is
// re-evaluated in fp64 from the raw record with the reference's exact operation order.
// ---------------------------------------------------------------------------------------------------------------
static constexpr int kRegW = kTileEdge + 2;            // 6 cells per region row
static constexpr int kRegRows = kRegW * kRegW;         // 36 rows
static constexpr int kNNCap = 640;                     // staged candidates per tile (48 B each)
static constexpr int kSegs = kTileEdge * kTileEdge;    // 16 query row segments per tile

template <bool AW>
__global__ void __launch_bounds__(kTileThreads)
nn_tile_kernel(const P4 *__restrict__ Q, const uint32_t *__restrict__ q_off, Lattice Lq,
               const uint32_t *__restrict__ tiles, long long t_begin, long long t_end, const P4 *__restrict__ R,
               const uint32_t *__restrict__ r_off, Lattice Lr, NNConst C, int32_t *__restrict__ nn_idx,
               double *__restrict__ nn_d2, double *__restrict__ nn_sq, uint32_t *__restrict__ far_list,
               unsigned int *__restrict__ far_count) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  P4 *raw = reinterpret_cast<P4 *>(smem_raw);
  float4 *rel = reinterpret_cast<float4 *>(smem_raw + (size_t)kNNCap * sizeof(P4));
  __shared__ uint32_t row_g0[kRegRows];                // global start of each region row
  __shared__ uint32_t row_pref[kRegRows + 1];          // staged prefix
  __shared__ uint16_t cell_rel[kRegRows][kRegW + 1];   // staged offset of each cell boundary inside its row
  __shared__ uint32_t seg_g0[kSegs], seg_pref[kSegs + 1];
  __shared__ uint32_t run_tab[9 * kTileThreads];       // per-thread window runs, [run][thread]
  __shared__ __align__(8) uint64_t mbar;

  const int tid = threadIdx.x;
  // the two lattices share (v, m): reference cell = query cell + integer shift
  const long long shx = (long long)(Lq.k_lo[0] - Lr.k_lo[0]) * Lq.m, shy = (long long)(Lq.k_lo[1] - Lr.k_lo[1]) * Lq.m,
                  shz = (long long)(Lq.k_lo[2] - Lr.k_lo[2]) * Lq.m;
  // fp32 screening error: |offset| <= 3.5 h per axis -> representation error <= 2^-24 * 3.5 h per operand; eta bounds
  // the error of the difference VECTOR with a generous factor
  const float eta = (float)(7.0 * 3.5 * Lq.h * 5.9604645e-8);
  if (tid == 0) mbar_init(&mbar, 1);
  uint32_t phase = 0;

  for (long long t = t_begin + blockIdx.x; t < t_end; t += gridDim.x) {
    const uint32_t tile = tiles[t];
    const int bx = (int)(tile % Lq.nb[0]), by = (int)((tile / Lq.nb[0]) % Lq.nb[1]), bz = (int)(tile / ((uint32_t)Lq.nb[0] * Lq.nb[1]));
    const long long r0x = (long long)bx * kTileEdge + shx - 1, r0y = (long long)by * kTileEdge + shy - 1,
                    r0z = (long long)bz * kTileEdge + shz - 1;   // region origin in reference cells (may be outside)
    uint32_t my_cnt = 0;
    if (tid < kRegRows) {
      const long long y = r0y + tid % kRegW, z = r0z + tid / kRegW;
      uint32_t g0 = 0;
      const long long xa = max(r0x, 0ll), xb = min(r0x + kRegW - 1, (long long)Lr.dims[0] - 1);
      if (y >= 0 && y < Lr.dims[1] && z >= 0 && z < Lr.dims[2] && xa <= xb) {
        const long long row = (z * Lr.dims[1] + y) * (long long)Lr.dims[0];
        g0 = __ldg(r_off + row + xa);
#pragma unroll
        for (int c = 0; c <= kRegW; ++c) {
          long long x = r0x + c;
          x = x < xa ? xa : (x > xb + 1 ? xb + 1 : x);
          cell_rel[tid][c] = (uint16_t)min(__ldg(r_off + row + x) - g0, 0xffffu);
        }
        my_cnt = __ldg(r_off + row + xb + 1) - g0;
      } else {
#pragma unroll
        for (int c = 0; c <= kRegW; ++c) cell_rel[tid][c] = 0;
      }
      row_g0[tid] = g0;
    } else if (tid >= 64 && tid < 64 + kSegs) {
      const int s = tid - 64;
      const int y = by * kTileEdge + s % kTileEdge, z = bz * kTileEdge + s / kTileEdge;
      uint32_t g0 = 0, n = 0;
      if (y < Lq.dims[1] && z < Lq.dims[2]) {
        const long long row = ((long long)z * Lq.dims[1] + y) * Lq.dims[0];
        const int xa = bx * kTileEdge, xb = min(xa + kTileEdge, Lq.dims[0]);
        g0 = __ldg(q_off + row + xa);
        n = __ldg(q_off + row + xb) - g0;
      }
      seg_g0[s] = g0;
      my_cnt = n;
    }
    // warp-level exclusive scans: warps 0-1 hold the 36 region rows, warp 2 the 16 query segments
    {
      const int lane = tid & 31, warp = tid >> 5;
      uint32_t inc = my_cnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
      if (warp == 0) { row_pref[tid + 1] = inc; if (lane == 0) row_pref[0] = 0; }
      __syncthreads();
      if (warp == 1 && tid < kRegRows) row_pref[tid + 1] = inc + row_pref[32];
      if (warp == 2) { if (lane < kSegs) seg_pref[lane + 1] = inc; if (lane == 0) seg_pref[0] = 0; }
      __syncthreads();
    }
    const uint32_t nc = row_pref[kRegRows], nq = seg_pref[kSegs];
    const bool staged = nc <= (uint32_t)kNNCap;
    // tile centre (absolute coordinates) — origin of the fp32 offsets
    const double ocx = ((double)Lq.k_lo[0] * Lq.v) + ((double)bx * kTileEdge + 0.5 * kTileEdge) * Lq.h;
    const double ocy = ((double)Lq.k_lo[1] * Lq.v) + ((double)by * kTileEdge + 0.5 * kTileEdge) * Lq.h;
    const double ocz = ((double)Lq.k_lo[2] * Lq.v) + ((double)bz * kTileEdge + 0.5 * kTileEdge) * Lq.h;
    if (staged && nc > 0) {
      if (tid == 0) mbar_expect_tx(&mbar, nc * (uint32_t)sizeof(P4));
      if (tid < kRegRows && my_cnt > 0)
        tma_bulk_g2s(raw + row_pref[tid], R + row_g0[tid], my_cnt * (uint32_t)sizeof(P4), &mbar);
      mbar_wait(&mbar, phase);
      phase ^= 1u;
      for (uint32_t i = tid; i < nc; i += kTileThreads) {
        const P4 p = raw[i];
        rel[i] = make_float4((float)(p.x - ocx), (float)(p.y - ocy), (float)(p.z - ocz), 0.f);
      }
      __syncthreads();
    }

    for (uint32_t qb = 0; qb < nq; qb += kTileThreads) {
      const uint32_t qi = qb + tid;
      if (qi >= nq) break;
      int seg = 0;
#pragma unroll
      for (int s = 1; s < kSegs; ++s) seg += (qi >= seg_pref[s]) ? 1 : 0;
      const uint32_t pos = seg_g0[seg] + (qi - seg_pref[seg]);
      const P4 q = load_p4(Q + pos);
      const int qcx = (int)(cell_of(q.idx) % (uint32_t)Lq.dims[0]);
      const int lx = qcx - bx * kTileEdge + 1, ly = seg % kTileEdge + 1, lz = seg / kTileEdge + 1;   // region-local cell
      Best b;
      b.init();
      if (staged) {
        const float qx = (float)(q.x - ocx), qy = (float)(q.y - ocy), qz = (float)(q.z - ocz);
        // per-thread run table: the (up to 9) non-empty window runs of this query, packed start | end << 16
        int nrun = 0;
#pragma unroll
        for (int r = 0; r < 9; ++r) {
          const int rr = (lz + r / 3 - 1) * kRegW + (ly + r % 3 - 1);
          const uint32_t base = row_pref[rr];
          const uint32_t so = base + cell_rel[rr][lx - 1], eo = base + cell_rel[rr][lx + 2];
          if (eo > so) { run_tab[nrun * kTileThreads + tid] = so | (eo << 16); ++nrun; }
        }
        // pass 1, fp32 only: smallest and second smallest screened distance, the runs walked as ONE flattened loop
        // so that the lanes of a warp stay in step
        float b1 = INFINITY, b2 = INFINITY;
        uint32_t j1 = 0, j = 0, e = 0;
        int r = 0;
        for (;;) {
          if (j >= e) {
            if (r >= nrun) break;
            const uint32_t pk = run_tab[r * kTileThreads + tid];
            ++r;
            j = pk & 0xffffu; e = pk >> 16;
          }
          const float4 c = rel[j];
          const float ddx = c.x - qx, ddy = c.y - qy, ddz = c.z - qz;
          const float d32 = fmaf(ddz, ddz, fmaf(ddy, ddy, ddx * ddx));
          const bool lt = d32 < b1;
          b2 = fminf(b2, lt ? b1 : d32);
          j1 = lt ? j : j1;
          b1 = fminf(b1, d32);
          ++j;
        }
        if (b1 < INFINITY) {
          // every candidate whose true distance is <= that of j1 has d32 <= b1 + 2 E(b1); 1.5x for fp32 rounding
          const float lim = (b1 + 3.0f * (2.f * sqrtf(b1) * eta + eta * eta + 1e-6f * b1)) * 1.0000005f + 1e-30f;
          if (b2 > lim) {
            const P4 p = raw[j1];
            b.offer(q, p.x, p.y, p.z, orig_of(p.idx));
          } else {
            // near-tie (or duplicate points): settle it in fp64 with the reference's operation order
            for (int rr9 = 0; rr9 < nrun; ++rr9) {
              const uint32_t pk = run_tab[rr9 * kTileThreads + tid];
              for (uint32_t jj = pk & 0xffffu; jj < (pk >> 16); ++jj) {
                const float4 c = rel[jj];
                const float ddx = c.x - qx, ddy = c.y - qy, ddz = c.z - qz;
                if (fmaf(ddz, ddz, fmaf(ddy, ddy, ddx * ddx)) <= lim) {
                  const P4 p = raw[jj];
                  b.offer(q, p.x, p.y, p.z, orig_of(p.idx));
                }
              }
            }
          }
        }
      } else {
        search_block_global(q, r0x + lx, r0y + ly, r0z + lz, R, r_off, Lr, b);
      }
      // the searched block is centred on the query's own (unclamped) reference cell; the far kernel restarts from ring 0
      finish_query<AW>(q, pos, r0x + lx, r0y + ly, r0z + lz, Lr, C, b, nn_idx, nn_d2, nn_sq, far_list, far_count,
                   cell_coord_cont(q.x, Lr, 0), cell_coord_cont(q.y, Lr, 1), cell_coord_cont(q.z, Lr, 2), 1e-9);
    }
    __syncthreads();   // shared tables and the staged region are re-used by the next tile
  }
}

// ---------------------------------------------------------------------------------------------------------------
// flat sweep.  One thread per query, queries in cell-sorted order (a warp = ~20 x-adjacent cells of one lattice row,
// so its lanes walk the same 9 rows of the reference lattice and their loads hit the same L1 lines).  The 3x3x3 block
// is 9 x-runs of the reference cloud; their bounds go to a per-thread run table in shared memory and the candidates
// are walked as ONE flattened loop (lanes stay in step).  Candidates are screened in fp32 on the cell-relative copies
// of both clouds (16 B/point; the offset between two points is rebuilt as (ix_c - ix_q) h + (rel_c - rel_q), error
// ~1e-6 h whatever the world extent): the loop keeps the smallest and second smallest screened distance.  If the
// runner-up is outside the fp32 error bound of the winner, only the winner is evaluated in fp64 (reference operation
// order); otherwise every candidate inside the bound is, and ties go to the smaller caller index.
// ---------------------------------------------------------------------------------------------------------------
struct FlatGeom {
  int qdimx, qdimy;            // query lattice (to decode the query's cell)
  Owned own;                   // slab layout: the planes of the query lattice whose points this rank evaluates
  int q_sparse;                // the query cloud's tag holds the row id (sparse table) instead of the cell id
  int rdimx, rdimy, rdimz;     // reference lattice
  long long shx, shy, shz;     // reference cell = query cell + shift (the lattices share v and m)
  float h;                     // cell edge
  float eta;                   // bound on the error of the fp32 offset VECTOR
  double inv_h;
};

template <bool E16, int U2, bool AW>      // U2: 0 plain walk, 1 two candidates (two loads in flight) per iteration
// 8 CTAs/SM: faster on C3 than 10 or 12 (spills + less L1; chosen on B200, not re-measured on H100)
__global__ void __launch_bounds__(kFlatThreads, 8)
nn_flat_kernel(const P4 *__restrict__ Q, const float4 *__restrict__ qrel, long long q_begin, long long q_end,
               const P4 *__restrict__ R, const float4 *__restrict__ rrel, CellIndex Ir,
               Lattice Lr, FlatGeom G, NNConst C, int32_t *__restrict__ nn_idx, double *__restrict__ nn_d2,
               double *__restrict__ nn_sq, uint32_t *__restrict__ far_list, unsigned int *__restrict__ far_count) {
  __shared__ __align__(16) unsigned char tab_smem[9 * kFlatThreads * RunTab<E16>::kEntryBytes];
  RunTab<E16> T(tab_smem);
  const int tid = threadIdx.x;
  const float h = G.h;
  const long long stride = (long long)gridDim.x * kFlatThreads;
  for (long long i = q_begin + blockIdx.x * (long long)kFlatThreads + tid; i < q_end; i += stride) {
    const float4 qr = __ldg(qrel + i);
    const P4 q = load_p4(Q + i);      // needed after the walk only; issued here so its latency hides behind the walk
    const uint32_t cq = cell_of(q.idx);
    const uint32_t cyz = G.q_sparse ? cq : cq / (uint32_t)G.qdimx;      // row id z * dimy + y of the query's own lattice
    if (!owns(G.own, (int)(cyz % (uint32_t)G.qdimy), (int)(cyz / (uint32_t)G.qdimy))) continue;      // a halo point
    // the query's cell in reference-lattice coordinates (may lie outside the reference lattice)
    const long long cx = (long long)(int)qr.w + G.shx, cy = (long long)(cyz % (uint32_t)G.qdimy) + G.shy,
                    cz = (long long)(cyz / (uint32_t)G.qdimy) + G.shz;
    const long long xa = max(cx - 1, 0ll), xb = min(cx + 1, (long long)G.rdimx - 1);
    int nrun = 0;
#pragma unroll
    for (int dz = -1; dz <= 1; ++dz) {
      const long long z = cz + dz;
      const float czv = (float)dz * h - qr.z;
#pragma unroll
      for (int dy = -1; dy <= 1; ++dy) {
        const long long y = cy + dy;
        uint32_t s = 0, e = 0;
        if (z >= 0 && z < G.rdimz && y >= 0 && y < G.rdimy && xa <= xb) cell_range(Ir, (int)z, (int)y, (int)xa, (int)xb, s, e);
        if (e > s) { T.put(nrun, tid, s, e, dy + 1, dz + 1, (float)dy * h - qr.y, czv); ++nrun; }
      }
    }
    // pass 1, fp32 only: smallest and second smallest screened distance
    const float tq = (float)cx;
    float b1 = INFINITY, b2 = INFINITY;
    uint32_t j1 = 0;
    auto screen = [&](const float4 &c, float cyf, float czf) {
      const float ddx = fmaf(c.w - tq, h, c.x - qr.x), ddy = c.y + cyf, ddz = c.z + czf;
      return fmaf(ddz, ddz, fmaf(ddy, ddy, ddx * ddx));
    };
    auto offer32 = [&](float d32, uint32_t j) {
      const bool lt = d32 < b1;
      b2 = fminf(b2, lt ? b1 : d32);
      j1 = lt ? j : j1;
      b1 = fminf(b1, d32);
    };
    RunWalk w;
    w.start(nrun);
    if (U2 == 1) {
      for (;;) {
        uint32_t j0, jn;
        float y0, z0, y1, z1;
        if (!w.next(T, tid, h, qr.y, qr.z, 1, j0, y0, z0)) break;
        const bool v1 = w.next(T, tid, h, qr.y, qr.z, 1, jn, y1, z1);
        const float4 c0 = __ldg(rrel + j0);
        const float4 c1 = __ldg(rrel + (v1 ? jn : j0));
        offer32(screen(c0, y0, z0), j0);
        if (v1) offer32(screen(c1, y1, z1), jn);
      }
    } else {
      uint32_t j0;
      float y0, z0;
      while (w.next(T, tid, h, qr.y, qr.z, 1, j0, y0, z0)) offer32(screen(__ldg(rrel + j0), y0, z0), j0);
    }
    Best b;
    b.init();
    if (b1 < INFINITY) {
      // every candidate whose true distance is <= that of j1 has d32 <= b1 + 2 E(b1), E(d2) = 2 sqrt(d2) eta + eta^2 + fp32 rounding
      const float lim = (b1 + 3.0f * (2.f * sqrtf(b1) * G.eta + G.eta * G.eta + 1e-6f * b1)) * 1.0000005f + 1e-30f;
      if (b2 > lim) {
        const P4 p = load_p4(R + j1);
        b.offer(q, p.x, p.y, p.z, orig_of(p.idx));
      } else {
        // near-tie (or duplicate points): settle it in fp64 with the reference's operation order
        w.start(nrun);
        uint32_t jj;
        float y0, z0;
        while (w.next(T, tid, h, qr.y, qr.z, 1, jj, y0, z0)) {
          if (screen(__ldg(rrel + jj), y0, z0) <= lim) {
            const P4 p = load_p4(R + jj);
            b.offer(q, p.x, p.y, p.z, orig_of(p.idx));
          }
        }
      }
    }
    // position inside the own cell from the cell-relative copy (error ~1e-7 cells, covered by the face-test slack)
    finish_query<AW>(q, (uint32_t)i, cx, cy, cz, Lr, C, b, nn_idx, nn_d2, nn_sq, far_list, far_count,
                 (double)cx + (double)qr.x * G.inv_h, (double)cy + (double)qr.y * G.inv_h,
                 (double)cz + (double)qr.z * G.inv_h, 2e-6);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// rows sweep: the same decomposition and the same exactness rules as the flat sweep, with WARP-UNIFORM control flow — the
// nine lattice rows of the 3x3x3 block are walked one after the other by all 32 lanes together, and inside a row every
// lane scans its own three-cell run for max-over-lanes(len) steps (REDUX.MAX).  At any time the lanes of a warp read one
// row of the reference cloud: a window of a few consecutive 128-byte lines instead of up to nine rows at once, no run
// table in shared memory, no per-lane refill branches.  The near-tie pass re-walks the rows the same way.
// ---------------------------------------------------------------------------------------------------------------
// U candidates loaded per inner iteration (all issued before the first test); SP: sparse reference table; AW: finish_query
template <int U, int SP, bool AW>
__global__ void __launch_bounds__(kFlatThreads, (U <= 2 ? 8 : (U <= 4 ? 6 : 4)))
nn_rows_kernel(const P4 *__restrict__ Q, const float4 *__restrict__ qrel, long long q_begin, long long q_end,
               const P4 *__restrict__ R, const float4 *__restrict__ rrel, CellIndex Ir,
               Lattice Lr, FlatGeom G, NNConst C, int32_t *__restrict__ nn_idx, double *__restrict__ nn_d2,
               double *__restrict__ nn_sq, uint32_t *__restrict__ far_list, unsigned int *__restrict__ far_count) {
  const unsigned FULL = 0xffffffffu;
  const float h = G.h;
  const long long stride = (long long)gridDim.x * kFlatThreads;
  for (long long base = q_begin + blockIdx.x * (long long)kFlatThreads; base < q_end; base += stride) {
    const long long i = base + threadIdx.x;
    const long long il = i < q_end ? i : q_end - 1;
    const float4 qr = __ldg(qrel + il);
    const uint32_t cq = cell_of(__double_as_longlong(__ldg(reinterpret_cast<const double *>(Q + il) + 3)));
    const uint32_t cyz = G.q_sparse ? cq : cq / (uint32_t)G.qdimx;
    const bool live = i < q_end && owns(G.own, (int)(cyz % (uint32_t)G.qdimy), (int)(cyz / (uint32_t)G.qdimy));
    // the query's cell in reference-lattice coordinates (may lie outside the reference lattice)
    const long long cx = (long long)(int)qr.w + G.shx, cy = (long long)(cyz % (uint32_t)G.qdimy) + G.shy,
                    cz = (long long)(cyz / (uint32_t)G.qdimy) + G.shz;
    const long long xa = max(cx - 1, 0ll), xb = min(cx + 1, (long long)G.rdimx - 1);
    const float tq = (float)cx;
    float b1 = INFINITY, b2 = INFINITY;
    uint32_t j1 = 0;
    uint32_t rs[9];
    int rl[9];
#pragma unroll
    for (int row = 0; row < 9; ++row) {
      const int dz = row / 3 - 1, dy = row % 3 - 1;
      const long long z = cz + dz, y = cy + dy;
      uint32_t s = 0, e = 0;
      if (live && z >= 0 && z < G.rdimz && y >= 0 && y < G.rdimy && xa <= xb) cell_range<SP>(Ir, (int)z, (int)y, (int)xa, (int)xb, s, e);
      rs[row] = s; rl[row] = (int)(e - s);
    }
#pragma unroll
    for (int row = 0; row < 9; ++row) {
      const int dz = row / 3 - 1, dy = row % 3 - 1;
      const float cyf = (float)dy * h - qr.y, czf = (float)dz * h - qr.z;
      const int len = rl[row];
      const int maxlen = __reduce_max_sync(FULL, len);
      const float4 *p = rrel + rs[row];
      float4 c[U];
#pragma unroll
      for (int u = 0; u < U; ++u) c[u] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
      for (int k0 = 0; k0 < maxlen; k0 += U) {
#pragma unroll
        for (int u = 0; u < U; ++u)
          if (k0 + u < len) c[u] = __ldg(p + k0 + u);
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const float ddx = fmaf(c[u].w - tq, h, c[u].x - qr.x), ddy = c[u].y + cyf, ddz = c[u].z + czf;
          const float d32 = (k0 + u < len) ? fmaf(ddz, ddz, fmaf(ddy, ddy, ddx * ddx)) : INFINITY;
          const bool lt = d32 < b1;
          b2 = fminf(b2, lt ? b1 : d32);
          j1 = lt ? rs[row] + (uint32_t)(k0 + u) : j1;
          b1 = fminf(b1, d32);
        }
      }
    }
    if (!live) continue;
    const P4 q = load_p4(Q + i);
    Best b;
    b.init();
    if (b1 < INFINITY) {
      // every candidate whose true distance is <= that of j1 has d32 <= b1 + 2 E(b1), E(d2) = 2 sqrt(d2) eta + eta^2 + fp32 rounding
      const float lim = (b1 + 3.0f * (2.f * sqrtf(b1) * G.eta + G.eta * G.eta + 1e-6f * b1)) * 1.0000005f + 1e-30f;
      if (b2 > lim) {
        const P4 pw = load_p4(R + j1);
        b.offer(q, pw.x, pw.y, pw.z, orig_of(pw.idx));
      } else {
        // near-tie (or duplicate points): settle it in fp64 with the reference's operation order
#pragma unroll
        for (int row = 0; row < 9; ++row) {
          const int dz = row / 3 - 1, dy = row % 3 - 1;
          const float cyf = (float)dy * h - qr.y, czf = (float)dz * h - qr.z;
#pragma unroll 1
          for (int k = 0; k < rl[row]; ++k) {
            const uint32_t jj = rs[row] + (uint32_t)k;
            const float4 cc = __ldg(rrel + jj);
            const float ddx = fmaf(cc.w - tq, h, cc.x - qr.x), ddy = cc.y + cyf, ddz = cc.z + czf;
            if (fmaf(ddz, ddz, fmaf(ddy, ddy, ddx * ddx)) <= lim) {
              const P4 pw = load_p4(R + jj);
              b.offer(q, pw.x, pw.y, pw.z, orig_of(pw.idx));
            }
          }
        }
      }
    }
    finish_query<AW>(q, (uint32_t)i, cx, cy, cz, Lr, C, b, nn_idx, nn_d2, nn_sq, far_list, far_count,
                 (double)cx + (double)qr.x * G.inv_h, (double)cy + (double)qr.y * G.inv_h,
                 (double)cz + (double)qr.z * G.inv_h, 2e-6);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// far queries: one warp per query, Chebyshev rings r = 0, 1, 2, ... until the best beats the block faces
// ---------------------------------------------------------------------------------------------------------------
// distance (in cells) from continuous coordinate u to the faces of the cell block [a, b] on one axis; faces at or beyond the
// lattice border are at infinity (nothing lives there)
__device__ __forceinline__ double block_face_cells(double u, long long a, long long b, int dim) {
  const double lo = (a <= 0) ? INFINITY : u - (double)a;
  const double hi = (b + 1 >= dim) ? INFINITY : (double)(b + 1) - u;
  return fmin(lo, hi);
}

__global__ void __launch_bounds__(kThreads)
nn_far_kernel(const P4 *__restrict__ Q, const P4 *__restrict__ R, CellIndex I, Lattice L, CoarseGrid CG,
              NNConst C, int32_t *__restrict__ nn_idx, double *__restrict__ nn_d2,
              const uint32_t *__restrict__ far_list, const unsigned int *__restrict__ far_count,
              uint32_t *__restrict__ unres_list, unsigned int *__restrict__ unres_count, AccBlock *__restrict__ acc,
              unsigned int *__restrict__ trace) {
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const unsigned int nfar = *far_count;
  if (blockIdx.x == 0 && threadIdx.x == 0 && nfar > 0) atomicOr(trace, 1u << ME_KBIT_NN_FAR);
  // with a coarse grid the cell-by-cell rings stop after kFineRings and blocks of f^3 cells take over
  const int fine_rings = CG.cnt ? 4 : 0x7fffffff;
  for (long long w = warp; w < nfar; w += nwarps) {
    const long long i = far_list[w];
    const P4 q = load_p4(Q + i);
    const long long ix = clamp_cell(cell_coord(q.x, L, 0), L.dims[0]), iy = clamp_cell(cell_coord(q.y, L, 1), L.dims[1]),
                    iz = clamp_cell(cell_coord(q.z, L, 2), L.dims[2]);
    const double ux = cell_coord_cont(q.x, L, 0), uy = cell_coord_cont(q.y, L, 1), uz = cell_coord_cont(q.z, L, 2);
    const double slack = 1e-9 * L.h + 1e-14 * (fabs(q.x) + fabs(q.y) + fabs(q.z) + C.ref_maxabs);
    double best = nn_d2[i];
    int bidx = nn_idx[i] >= 0 ? nn_idx[i] : 0x7fffffff;
    bool beyond = false, done = false, unresolved = false;
    const double gcov = cover_dist_cells(C, uy, uz);
    auto warp_argmin = [&]() {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(FULL, best, o);
        const int oi = __shfl_xor_sync(FULL, bidx, o);
        if (ob < best || (ob == best && oi < bidx)) { best = ob; bidx = oi; }
      }
    };
    // after a searched block whose faces are g cells away: resolved?  (sets done / beyond)
    auto settle = [&](double g_block) {
      const double g = fmin(g_block, gcov) * L.h;
      const double ge = g - slack;
      const double ge2 = ge > 0 ? ge * ge : 0.0;
      if (best < ge2) { done = true; return; }
      if (ge2 > C.max_d2) { beyond = best > C.max_d2; done = true; return; }
      if (g == INFINITY) { done = true; return; }      // the block covers the whole lattice
      // the searched block has grown past the planes of this rank and the best still does not beat them: the answer may
      // lie on another rank's planes — finished by brute force over the whole cloud (nn_brute_kernel)
      if (g_block >= gcov) { unresolved = true; done = true; }
    };
    for (int r = 0; r <= fine_rings && !done; ++r) {
      const int side = 2 * r + 1;
      // rows of the shell: every (dy,dz) in [-r,r]^2; border rows scan the full x range, inner rows two end cells
      for (int t = lane; t < side * side; t += 32) {
        const int dz = t / side - r, dy = t % side - r;
        const long long z = iz + dz, y = iy + dy;
        if (z < 0 || z >= L.dims[2] || y < 0 || y >= L.dims[1]) continue;
        const bool border = (dz == -r || dz == r || dy == -r || dy == r);
        for (int part = 0; part < 2; ++part) {
          long long xa, xb;
          if (border) { if (part) break; xa = ix - r; xb = ix + r; }
          else { xa = xb = part ? ix + r : ix - r; }
          xa = max(xa, 0ll); xb = min(xb, (long long)L.dims[0] - 1);
          if (xa > xb) continue;
          uint32_t s, e;
          cell_range(I, (int)z, (int)y, (int)xa, (int)xb, s, e);
          for (uint32_t j = s; j < e; ++j) {
            const P4 p = load_p4(R + j);
            const double d2 = d2_kd(q.x, q.y, q.z, p.x, p.y, p.z);
            const int pi = orig_of(p.idx);
            if (d2 < best || (d2 == best && pi < bidx)) { best = d2; bidx = pi; }
          }
        }
      }
      warp_argmin();
      settle(fmin(fmin(block_face_cells(ux, ix - r, ix + r, L.dims[0]), block_face_cells(uy, iy - r, iy + r, L.dims[1])),
                  block_face_cells(uz, iz - r, iz + r, L.dims[2])));
    }
    if (!done) {
      // coarse phase: Chebyshev rings of blocks of f^3 cells around the query's block; empty blocks cost one count load,
      // occupied blocks that can still hold a closer point are scanned by the whole warp (lanes over the block's f^2 rows)
      const int f = CG.f;
      if (lane == 0) atomicOr(trace, 1u << ME_KBIT_NN_FAR_COARSE);
      const long long cqx = min(max(ix, 0ll), (long long)L.dims[0] - 1) / f, cqy = min(max(iy, 0ll), (long long)L.dims[1] - 1) / f,
                      cqz = min(max(iz, 0ll), (long long)L.dims[2] - 1) / f;
      for (int rc = 0; !done; ++rc) {
        const int side = 2 * rc + 1;
        for (int t0 = 0; t0 < side * side; t0 += 32) {
          const int t = t0 + lane;
          const bool tv = t < side * side;
          const int dz = tv ? t / side - rc : 0, dy = tv ? t % side - rc : 0;
          const long long bz = cqz + dz, by = cqy + dy;
          const bool row_ok = tv && bz >= 0 && bz < CG.cd[2] && by >= 0 && by < CG.cd[1];
          const bool border = (dz == -rc || dz == rc || dy == -rc || dy == rc);
          for (int dxi = 0; dxi < side; ++dxi) {
            const long long bx = cqx + dxi - rc;
            bool occ = row_ok && (border || dxi == 0 || dxi == side - 1) && bx >= 0 && bx < CG.cd[0];
            if (occ) occ = __ldg(CG.cnt + (bz * CG.cd[1] + by) * (long long)CG.cd[0] + bx) != 0;
            if (occ) {      // can the block hold a point closer than the best so far?
              const double ex = fmax(0.0, fmax((double)(bx * f) - ux, ux - (double)((bx + 1) * f)));
              const double ey = fmax(0.0, fmax((double)(by * f) - uy, uy - (double)((by + 1) * f)));
              const double ez = fmax(0.0, fmax((double)(bz * f) - uz, uz - (double)((bz + 1) * f)));
              const double lb = sqrt(ex * ex + ey * ey + ez * ez) * L.h - slack;
              occ = !(lb > 0 && lb * lb > best);
            }
            unsigned mask = __ballot_sync(FULL, occ);
            while (mask) {
              const int src = __ffs(mask) - 1;
              mask &= mask - 1;
              const long long sbx = __shfl_sync(FULL, bx, src), sby = __shfl_sync(FULL, by, src), sbz = __shfl_sync(FULL, bz, src);
              const int xa = (int)(sbx * f), xb = (int)min(sbx * f + f - 1, (long long)L.dims[0] - 1);
              // the block's rows inside the lattice only: on a lattice long along x (f = 2^17 for 1.8e7 cells) the f^2 rows
              // of a full block would overflow an int, and nearly all of them lie outside a thin lattice
              const long long ny = min((long long)f, (long long)L.dims[1] - sby * f), nz = min((long long)f, (long long)L.dims[2] - sbz * f);
              for (long long row = lane; row < ny * nz; row += 32) {
                const long long z = sbz * f + row / ny, y = sby * f + row % ny;
                uint32_t s, e;
                cell_range(I, (int)z, (int)y, xa, xb, s, e);
                for (uint32_t j = s; j < e; ++j) {
                  const P4 p = load_p4(R + j);
                  const double d2 = d2_kd(q.x, q.y, q.z, p.x, p.y, p.z);
                  const int pi = orig_of(p.idx);
                  if (d2 < best || (d2 == best && pi < bidx)) { best = d2; bidx = pi; }
                }
              }
              warp_argmin();
            }
          }
        }
        settle(fmin(fmin(block_face_cells(ux, (cqx - rc) * f, (cqx + rc) * f + f - 1, L.dims[0]),
                         block_face_cells(uy, (cqy - rc) * f, (cqy + rc) * f + f - 1, L.dims[1])),
                    block_face_cells(uz, (cqz - rc) * f, (cqz + rc) * f + f - 1, L.dims[2])));
      }
    }
    if (lane == 0) {
      atomicAdd(&acc->n_far, 1ull);
      if (unresolved) unres_list[atomicAdd(unres_count, 1u)] = (uint32_t)i;
      else if (beyond || !(best < INFINITY)) { nn_idx[i] = -1; nn_d2[i] = INFINITY; }
      else {
        nn_idx[i] = bidx;
        nn_d2[i] = best;      // the Eigen-order squared norm follows in nn_far_sq_kernel (needs the winner's coordinates)
      }
    }
  }
}

// slab mode, queries whose search left the planes of this rank: exact nearest neighbour over the WHOLE reference cloud (caller
// order, resident on every rank) — one warp per query, lanes stride over the points.  Rare by construction (the halo is
// several cells wide); correct for any count.
__global__ void __launch_bounds__(kThreads)
nn_brute_kernel(const P4 *__restrict__ Q, const double *__restrict__ ref_xyz, long long n_ref, NNConst C,
                int32_t *__restrict__ nn_idx, double *__restrict__ nn_d2, const uint32_t *__restrict__ unres_list,
                const unsigned int *__restrict__ unres_count, unsigned int *__restrict__ trace) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const unsigned int nu = *unres_count;
  if (blockIdx.x == 0 && threadIdx.x == 0 && nu > 0) atomicOr(trace, 1u << ME_KBIT_NN_BRUTE);
  for (long long w = warp; w < nu; w += nwarps) {
    const long long i = unres_list[w];
    const P4 q = load_p4(Q + i);
    double best = INFINITY;
    int bidx = 0x7fffffff;
    for (long long j = lane; j < n_ref; j += 32) {
      const double d2 = d2_kd(q.x, q.y, q.z, __ldg(ref_xyz + 3 * j), __ldg(ref_xyz + 3 * j + 1), __ldg(ref_xyz + 3 * j + 2));
      if (d2 < best) { best = d2; bidx = (int)j; }      // j increases: the first (smallest) index of a tie is kept
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
      if (ob < best || (ob == best && oi < bidx)) { best = ob; bidx = oi; }
    }
    if (lane == 0) {
      if (!(best < INFINITY) || best > C.max_d2) { nn_idx[i] = -1; nn_d2[i] = INFINITY; }
      else { nn_idx[i] = bidx; nn_d2[i] = best; }
    }
  }
}

// far queries: Eigen-order squared norm of (query - winner); the winner's coordinates come from the caller-order array.
// ME_PAIRING_AS_WRITTEN gt->est (C.accumulate == 0): the as-written pair's, as finish_query gives it to the swept queries
__global__ void __launch_bounds__(kThreads)
nn_far_sq_kernel(const P4 *__restrict__ Q, const double *__restrict__ ref_xyz, const int32_t *__restrict__ nn_idx,
                 const double *__restrict__ nn_d2, NNConst C, double *__restrict__ nn_sq, const uint32_t *__restrict__ far_list,
                 const unsigned int *__restrict__ far_count) {
  const unsigned int nfar = *far_count;
  for (long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x; w < nfar; w += (long long)gridDim.x * blockDim.x) {
    const long long i = far_list[w];
    const int32_t j = nn_idx[i];
    if (j < 0) continue;
    const P4 q = load_p4(Q + i);
    if (!C.accumulate) {
      if (keep_pair(nn_d2[i], C)) nn_sq[i] = as_written_sq(j, orig_of(q.idx), C.aw_gt_xyz, C.aw_n_gt, C.aw_est_xyz, C.aw_n_est);
      continue;
    }
    const double px = __ldg(ref_xyz + 3ll * j), py = __ldg(ref_xyz + 3ll * j + 1), pz = __ldg(ref_xyz + 3ll * j + 2);
    nn_sq[i] = sqnorm_eigen(__dsub_rn(q.x, px), __dsub_rn(q.y, py), __dsub_rn(q.z, pz));
  }
}

// streaming pass over the per-query results of a sweep: the five-threshold accumulators (map_eval.cpp:1095-1123) and the
// full-Chamfer sum (:1416).  Entries < 0 are queries without a neighbour within reach (-1) or owned by another rank (-2).
__global__ void __launch_bounds__(kThreads, 4)      // 4 blocks per SM, as before the moments: the grid is 8 per SM
nn_stats_kernel(long long i_begin, long long i_end, const int32_t *__restrict__ nn_idx, const double *__restrict__ nn_d2,
                const double *__restrict__ nn_sq, NNConst C, AccBlock *__restrict__ acc, double *__restrict__ mom) {
  LocalAcc a;
  a.clear();
  for (long long i = i_begin + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < i_end;
       i += (long long)gridDim.x * blockDim.x) {
    if (__ldg(nn_idx + i) < 0) continue;
    const double d2 = __ldg(nn_d2 + i);
    if (C.want_full_cd) a.nn_dist(__dsqrt_rn(d2));
    if (C.accumulate && keep_pair(d2, C)) accum_sq(__ldg(nn_sq + i), C, a);
  }
  flush_acc(a, acc, mom);
}

// ME_PAIRING_AS_WRITTEN gt->est (as_written_pair, records.cuh), a streaming fold of the records: the sweep and
// nn_far_sq_kernel left the squared norm of every kept as-written pair in nn_sq (kAwOutOfRangeSq: out of range).  Walks
// every gt point; points this rank did not evaluate carry the marker -2.
__global__ void __launch_bounds__(kThreads, 4)      // as nn_stats_kernel
pair_as_written_kernel(long long n, const int32_t *__restrict__ nn_idx, const double *__restrict__ nn_d2,
                       const double *__restrict__ nn_sq, NNConst C, AccBlock *__restrict__ acc, double *__restrict__ mom) {
  LocalAcc a;
  a.clear();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (__ldg(nn_idx + i) < 0 || !keep_pair(__ldg(nn_d2 + i), C)) continue;
    const double sq = __ldg(nn_sq + i);
    if (sq < 0) a.ub();
    else accum_sq(sq, C, a);
  }
  flush_acc(a, acc, mom);
}

// ---------------------------------------------------------------------------------------------------------------
// Accuracy curve (me_nn_curve_accum_device): the records of the last sweep folded into K + 1 distance bins.  A kept
// pair goes to bin b = the first level k with d <= tau_k (K when it exceeds every level); it counts for every level
// k >= b, so the host forms each level's sums as prefix sums over the bins.  Per bin: count, sum d, sum sq.
// Deterministic: block j owns the fixed contiguous slice j of the records; per tile every warp sorts its 32 pairs by
// bin (bitonic, keys unique by lane) and sums each bin's segment with a fixed shuffle tree; warp 0 adds the segment
// totals of the 8 warps in warp order into the block's bins in shared memory.  nn_curve_merge_kernel sums the blocks'
// bins in block order.  No floating-point atomics anywhere.
// ---------------------------------------------------------------------------------------------------------------
static constexpr int kCurveThreads = 256;
static constexpr int kCurveWarps = kCurveThreads / 32;

// first k in [0, K) with d <= tau[k], K if none (tau non-decreasing)
__device__ __forceinline__ int curve_bin(const double *tau, int K, double d) {
  int lo = 0, hi = K;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (d <= tau[mid]) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// per block: part[blockIdx.x * stride ..] = cnt[K + 1], sum_d[K + 1], sum_sq[K + 1], n_ub  (stride = 3 (K + 1) + 1)
__global__ void __launch_bounds__(kCurveThreads, 4)
nn_curve_kernel(CurveSrc S, NNConst C, const double *__restrict__ tau, int K, long long per_block, double *__restrict__ part) {
  extern __shared__ double curve_sm[];
  double *s_tau = curve_sm, *s_cnt = curve_sm + K, *s_sd = s_cnt + (K + 1), *s_sq = s_sd + (K + 1);
  __shared__ int seg_bin[2][kCurveThreads], seg_n[2][kCurveThreads];
  __shared__ double seg_d[2][kCurveThreads], seg_q[2][kCurveThreads];
  __shared__ unsigned long long s_ub;
  const int lane = threadIdx.x & 31;
  for (int t = threadIdx.x; t < K; t += kCurveThreads) s_tau[t] = tau[t];
  for (int t = threadIdx.x; t < 3 * (K + 1); t += kCurveThreads) s_cnt[t] = 0.0;
  if (threadIdx.x == 0) s_ub = 0;
  __syncthreads();
  const long long b0 = S.b + blockIdx.x * per_block, b1 = min(S.e, b0 + per_block);
  unsigned int ub = 0;
  int buf = 0;
  for (long long base = b0; base < b1; base += kCurveThreads) {
    const long long i = base + threadIdx.x;
    int bin = K + 1;                 // no kept pair: sorts last, never folded
    double d = 0.0, sq = 0.0;
    if (i < b1 && kept_record(S, C, i, sq, ub)) { d = pair_dist(sq); bin = curve_bin(s_tau, K, d); }
    // sort the warp's (bin, lane) keys ascending, then fetch the values in that order
    unsigned int key = ((unsigned int)bin << 5) | (unsigned int)lane;
#pragma unroll
    for (int k = 2; k <= 32; k <<= 1)
#pragma unroll
      for (int j = k >> 1; j > 0; j >>= 1) {
        const unsigned int o = __shfl_xor_sync(0xffffffffu, key, j);
        const bool up = (lane & k) == 0 || k == 32, lower = (lane & j) == 0;
        key = (lower == up) ? min(key, o) : max(key, o);
      }
    const int src = (int)(key & 31u), kb = (int)(key >> 5);
    d = __shfl_sync(0xffffffffu, d, src);
    sq = __shfl_sync(0xffffffffu, sq, src);
    const int prev = __shfl_up_sync(0xffffffffu, kb, 1);
    const unsigned int heads = __ballot_sync(0xffffffffu, lane == 0 || prev != kb);
    const int head = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));     // first lane of this lane's segment
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {      // inclusive scan within the segment, a fixed tree
      const double du = __shfl_up_sync(0xffffffffu, d, o), qu = __shfl_up_sync(0xffffffffu, sq, o);
      if (lane - o >= head) { d += du; sq += qu; }
    }
    const bool tail = lane == 31 || ((heads >> (lane + 1)) & 1u);
    seg_bin[buf][threadIdx.x] = (tail && kb <= K) ? kb : -1;
    seg_n[buf][threadIdx.x] = lane - head + 1;
    seg_d[buf][threadIdx.x] = d;
    seg_q[buf][threadIdx.x] = sq;
    __syncthreads();
    if (threadIdx.x < 32) {      // the bins of one warp's tails are distinct: one pass per warp, in warp order
      for (int w = 0; w < kCurveWarps; ++w) {
        const int s = w * 32 + lane, bb = seg_bin[buf][s];
        if (bb >= 0) { s_cnt[bb] += (double)seg_n[buf][s]; s_sd[bb] += seg_d[buf][s]; s_sq[bb] += seg_q[buf][s]; }
        __syncwarp();
      }
    }
    buf ^= 1;      // the other buffer: warp 0 folds this one while the others fill the next
  }
  if (ub) atomicAdd(&s_ub, (unsigned long long)ub);
  __syncthreads();
  const int stride = 3 * (K + 1) + 1;
  double *out = part + (long long)blockIdx.x * stride;
  for (int t = threadIdx.x; t < 3 * (K + 1); t += kCurveThreads) out[t] = s_cnt[t];
  if (threadIdx.x == 0) out[3 * (K + 1)] = (double)s_ub;
}

// blk[t] = sum over the blocks, in block order, of part[. * stride + t]
__global__ void nn_curve_merge_kernel(const double *__restrict__ part, int n_blocks, int stride, double *__restrict__ blk) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= stride) return;
  double s = 0.0;
  for (int b = 0; b < n_blocks; ++b) s += part[(long long)b * stride + t];
  blk[t] = s;
}

// ---------------------------------------------------------------------------------------------------------------
// Exact distance quantiles (me_nn_quantile_*): radix selection over the records (radix.cuh).  Pass 0 turns every record of
// a direction into a 64-bit key — the bit pattern of its d, or kQuantOut outside the population — and histograms the top
// 8-bit digit; the later passes are nn_quantile_hist_kernel's.
// ---------------------------------------------------------------------------------------------------------------
// d of record i of the population, false when the record is not in it
__device__ __forceinline__ bool quant_record(const CurveSrc &S, const NNConst &C, int nn_pop, long long i, double &d) {
  if (nn_pop) {            // the terms of nn_stats_kernel's full-CD sum
    if (__ldg(S.nn_idx + i) < 0) return false;
    d = __dsqrt_rn(__ldg(S.nn_d2 + i));
    return true;
  }
  double sq;
  unsigned int ub = 0;
  if (!kept_record(S, C, i, sq, ub)) return false;
  d = pair_dist(sq);
  return true;
}

// pass 0: keys[i - S.b] for every record of [S.b, S.e), and the histogram of the top digit into hist[0 .. 255]
__global__ void __launch_bounds__(kQuantThreads)
nn_quantile_keys_kernel(CurveSrc S, NNConst C, int nn_pop, unsigned long long *__restrict__ keys, unsigned long long *__restrict__ hist) {
  __shared__ unsigned int s_hist[kQuantBins];
  for (int t = threadIdx.x; t < kQuantBins; t += kQuantThreads) s_hist[t] = 0;
  __syncthreads();
  const long long stride = (long long)gridDim.x * kQuantThreads;
  for (long long base = S.b + (long long)blockIdx.x * kQuantThreads; base < S.e; base += stride) {   // warp-uniform bound
    const long long i = base + threadIdx.x;
    int bin = -1;
    if (i < S.e) {
      double d;
      unsigned long long key = kQuantOut;
      if (quant_record(S, C, nn_pop, i, d)) {
        key = quant_key(d);
        bin = (int)(key >> 56);
      }
      keys[i - S.b] = key;
    }
    quant_count(s_hist, bin);
  }
  quant_flush(s_hist, kQuantBins, hist);
}

__global__ void quant_to_block_kernel(const unsigned long long *__restrict__ hist, int n, double *__restrict__ blk) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) blk[t] = (double)hist[t];
}

__global__ void fill_i32_kernel(int32_t *p, long long n, int32_t v) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void fill_nn_kernel(int32_t *idx, double *d2, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    idx[i] = -1; d2[i] = NAN;
  }
}
__global__ void unsort_nn_kernel(const P4 *__restrict__ Q, long long n, const int32_t *__restrict__ sidx,
                                 const double *__restrict__ sd2, int32_t *__restrict__ oidx, double *__restrict__ od2) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int32_t v = sidx[i];
    if (v == -2) continue;    // not evaluated by this rank
    const long long o = orig_of(__double_as_longlong(__ldg(reinterpret_cast<const double *>(Q + i) + 3)));
    oidx[o] = v; od2[o] = sd2[i];
  }
}
__global__ void count_marked_kernel(const int32_t *__restrict__ idx, long long n, unsigned long long *out) {
  unsigned long long c = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) c += idx[i] != -2;
  c = (unsigned long long)warp_sum_ll((long long)c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}

// the per-block (n, mean, M2) of a stats pass, merged in block order into acc (one block)
__global__ void __launch_bounds__(kThreads) merge_moments_kernel(const double *__restrict__ mom, int n_slots, AccBlock *__restrict__ acc) {
  double n = 0, m = 0, m2 = 0;
  for (int s = threadIdx.x; s < n_slots; s += blockDim.x) chan_merge(n, m, m2, mom[3 * s], mom[3 * s + 1], mom[3 * s + 2]);
  block_moments(n, m, m2);
  if (threadIdx.x == 0) { acc->mean_all = m; acc->m2_all = m2; acc->sum_d_all = n * m; acc->sum_d2_all = m2 + n * m * m; }
}

// accumulator block of one direction -> the context's fp64 block (me_eval_nn_accum*): no host round trip.  The
// moments go to this rank's slot; the other ranks' slots are zeroed, so that the SUM all-reduce gathers them.
__global__ void pack_nn_kernel(const AccBlock *__restrict__ a, const unsigned long long *__restrict__ n_eval, long long n_query,
                               int rank, double *__restrict__ blk) {
  for (int r = threadIdx.x; r < ME_MAX_WORLD; r += blockDim.x) {
    const bool mine = r == rank;
    blk[kBlkMoments + r] = mine ? (double)a->n_corr : 0.0;
    blk[kBlkMoments + ME_MAX_WORLD + r] = mine ? a->mean_all : 0.0;
    blk[kBlkMoments + 2 * ME_MAX_WORLD + r] = mine ? a->m2_all : 0.0;
  }
  if (threadIdx.x != 0) return;
  blk[0] = (double)(n_eval ? (long long)*n_eval : n_query);
  blk[1] = (double)a->n_corr;
  for (int k = 0; k < 5; ++k) blk[2 + k] = (double)a->n_inl[k];
  blk[7] = (double)a->n_ub; blk[8] = (double)a->n_far;
  for (int k = 0; k < 5; ++k) { blk[9 + k] = a->sum_d[k]; blk[14 + k] = a->sum_d2[k]; }
  blk[19] = a->sum_d_all; blk[20] = a->sum_d2_all; blk[21] = a->sum_nn;
}

// ---------------------------------------------------------------------------------------------------------------
// host driver
// ---------------------------------------------------------------------------------------------------------------
void set_cutoff(NNConst &C, const me_nn_params *p) {
  C.cutoff_mode = p->cutoff_mode;
  C.cutoff = p->cutoff_mode == ME_CUTOFF_SQDIST_LE_R ? p->icp_max_distance : p->icp_max_distance * p->icp_max_distance;
}

static int run_direction(me_ctx *ctx, int qwhich, const me_nn_params *p, int stage, bool pack) {
  Cloud &Qc = ctx->cloud[qwhich];
  Cloud &Rc = ctx->cloud[1 - qwhich];
  StageTimer timer(ctx, stage);

  NNConst C;
  for (int k = 0; k < 5; ++k) C.tau[k] = p->tau[k];
  set_cutoff(C, p);
  const bool as_written = (qwhich == ME_CLOUD_GT && p->pairing == ME_PAIRING_AS_WRITTEN);
  C.accumulate = as_written ? 0 : 1;
  C.want_full_cd = p->want_full_cd ? 1 : 0;
  C.max_d2 = p->want_full_cd ? INFINITY : C.cutoff;
  C.cov_axis = Rc.slab ? Rc.sl_axis : 0;
  C.cov_lo = Rc.sc_lo; C.cov_hi = Rc.sc_hi;
  C.cov_dim = Rc.slab ? Rc.lat.dims[Rc.sl_axis] : 0;
  C.ref_maxabs = 0;
  for (int a = 0; a < 3; ++a) C.ref_maxabs = std::max(C.ref_maxabs, std::max(std::fabs(Rc.bbox_min[a]), std::fabs(Rc.bbox_max[a])));
  C.aw_gt_xyz = Qc.d_xyz; C.aw_n_gt = Qc.n;      // read only when as_written (Qc is the gt cloud then)
  C.aw_est_xyz = Rc.d_xyz; C.aw_n_est = Rc.n;

  // the flat kernel packs run lengths into 24 bits and x indices into an fp32 mantissa; otherwise the tile kernel runs
  const bool any_sparse = Qc.lat.sparse || Rc.lat.sparse;
  const bool use_tile = !any_sparse && (getenv("ME_NN_TILE") != nullptr || Qc.lat.dims[0] >= (1 << 24) || Rc.lat.dims[0] >= (1 << 24) ||
                                        3 * Rc.max_cell_count >= (1 << 24));
  if (any_sparse && 3 * Rc.max_cell_count >= (1 << 24))
    return fail(ctx, ME_ERR_RANGE, "more than 2^24 / 3 points in one lattice cell of a sparse lattice");
  if (use_tile && (Qc.slab || Rc.slab))
    return fail(ctx, ME_ERR_RANGE, "the tile sweep cannot run on a slab layout (use ME_LAYOUT_REPLICATED for this data)");
  long long qb, qe, tb = 0, te = 0;
  ME_TRY(query_shard(ctx, qwhich, &qb, &qe));  // flat sweep: contiguous, cell-aligned range of the cell-sorted query order
  if (use_tile) {                              // (before the work buffer is carved up: the tile build scans in it)
    ME_TRY(build_tiles(ctx, qwhich));
    shard_range(ctx, Qc.n_tiles, &tb, &te);    // tile sweep: the (ordered) list of query tiles is sharded across ranks
  }

  ME_TRY(ensure(ctx, (void **)&Qc.d_nn_idx, &Qc.cap_nn, Qc.n, sizeof(int32_t)));
  ME_TRY(ensure(ctx, (void **)&Qc.d_nn_d2, &Qc.cap_nn_d2, Qc.n, sizeof(double)));
  ME_TRY(ensure(ctx, (void **)&Qc.d_nn_sq, &Qc.cap_nn_sq, Qc.n, sizeof(double)));
  // work buffer: far list and unresolved list (n uint32 each) after a 256-byte header holding the counters, then the
  // per-block moments of the stats pass (3 fp64 per block, at most sm_count * 16 blocks)
  const int max_mom_slots = ctx->sm_count * 16;
  ME_TRY(ensure_work(ctx, 256 + 2 * (size_t)Qc.n * sizeof(uint32_t) + 3 * sizeof(double) * (size_t)max_mom_slots));
  unsigned int *far_count = (unsigned int *)ctx->d_work;
  unsigned long long *n_eval = (unsigned long long *)((char *)ctx->d_work + 64);
  unsigned int *unres_count = (unsigned int *)((char *)ctx->d_work + 128);
  uint32_t *far_list = (uint32_t *)((char *)ctx->d_work + 256);
  uint32_t *unres_list = far_list + Qc.n;
  double *mom = (double *)(unres_list + Qc.n);
  AccBlock *acc = (AccBlock *)ctx->d_scratch;
  ME_CUDA(ctx, cudaMemsetAsync(acc, 0, sizeof(AccBlock), ctx->stream));
  ME_CUDA(ctx, cudaMemsetAsync(ctx->d_work, 0, 256, ctx->stream));
  const int fill_blocks = (int)std::min<long long>((Qc.n + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
  const bool sharded = ctx->world > 1;
  if (sharded) {   // mark the queries other ranks own
    fill_i32_kernel<<<fill_blocks, kThreads, 0, ctx->stream>>>(Qc.d_nn_idx, Qc.n, -2);
    ME_LAUNCH_CHECK(ctx);
  }
  // the sweeps, compiled for the as-written pairing apart (finish_query)
  auto *const tile_kernel = as_written ? nn_tile_kernel<true> : nn_tile_kernel<false>;
  auto *const flat_kernel = as_written ? nn_flat_kernel<true, 0, true> : nn_flat_kernel<true, 0, false>;
  auto *const rows_sparse = as_written ? nn_rows_kernel<4, 1, true> : nn_rows_kernel<4, 1, false>;
  auto *const rows_dense = as_written ? nn_rows_kernel<4, 0, true> : nn_rows_kernel<4, 0, false>;
  const size_t dyn_smem = (size_t)kNNCap * (sizeof(P4) + sizeof(float4));
  if (use_tile)      // per launch: function attributes are per device
    ME_CUDA(ctx, cudaFuncSetAttribute(tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_smem));
  if (use_tile ? te > tb : qe > qb) {
    if (use_tile) {
      // persistent CTAs: each walks tiles tb + blockIdx.x, + gridDim.x, ... and flushes its accumulators once
      const unsigned grid = (unsigned)std::min<long long>(te - tb, (long long)ctx->sm_count * 16);
      tile_kernel<<<grid, kTileThreads, dyn_smem, ctx->stream>>>(
          Qc.d_sorted, Qc.d_cell_off, Qc.lat, Qc.d_tiles, tb, te, Rc.d_sorted, Rc.d_cell_off, Rc.lat, C, Qc.d_nn_idx,
          Qc.d_nn_d2, Qc.d_nn_sq, far_list, far_count);
      trace_kernel(ctx, ME_KBIT_NN_TILE);
    } else {
      FlatGeom G;
      G.qdimx = Qc.lat.dims[0]; G.qdimy = Qc.lat.dims[1];
      G.q_sparse = Qc.lat.sparse;
      G.own = owned_of(Qc);
      G.rdimx = Rc.lat.dims[0]; G.rdimy = Rc.lat.dims[1]; G.rdimz = Rc.lat.dims[2];
      G.shx = (long long)(Qc.lat.k_lo[0] - Rc.lat.k_lo[0]) * Qc.lat.m;
      G.shy = (long long)(Qc.lat.k_lo[1] - Rc.lat.k_lo[1]) * Qc.lat.m;
      G.shz = (long long)(Qc.lat.k_lo[2] - Rc.lat.k_lo[2]) * Qc.lat.m;
      G.h = (float)Qc.lat.h;
      G.inv_h = 1.0 / Qc.lat.h;
      double maxabs = C.ref_maxabs;
      for (int a = 0; a < 3; ++a) maxabs = std::max(maxabs, std::max(std::fabs(Qc.bbox_min[a]), std::fabs(Qc.bbox_max[a])));
      // per-axis offset error <= 1e-6 h + fp64 rounding of the cell origins (see mme.cu); vector norm <= sqrt(3) times that
      G.eta = (float)(1.7320508 * (1e-6 * Qc.lat.h + 4e-15 * maxabs));
      const unsigned grid = (unsigned)std::min<long long>((qe - qb + kFlatThreads - 1) / kFlatThreads, (long long)ctx->sm_count * 32);
      // default: the warp-synchronous row walk, 4 candidates per iteration (C3 on one H100: 1.6 / 2.3 ms per direction
      // against 1.7 / 2.4 ms for the run-table walk, which stays behind ME_NN_KERNEL=flat)
      const char *kv = getenv("ME_NN_KERNEL");
      if (kv && !strcmp(kv, "flat")) {
        flat_kernel<<<grid, kFlatThreads, 0, ctx->stream>>>(Qc.d_sorted, Qc.d_rel, qb, qe, Rc.d_sorted, Rc.d_rel, index_of(Rc),
                                                            Rc.lat, G, C, Qc.d_nn_idx, Qc.d_nn_d2, Qc.d_nn_sq, far_list, far_count);
        trace_kernel(ctx, ME_KBIT_NN_FLAT);
      } else if (Rc.lat.sparse) {
        rows_sparse<<<grid, kFlatThreads, 0, ctx->stream>>>(Qc.d_sorted, Qc.d_rel, qb, qe, Rc.d_sorted, Rc.d_rel, index_of(Rc),
                                                            Rc.lat, G, C, Qc.d_nn_idx, Qc.d_nn_d2, Qc.d_nn_sq, far_list, far_count);
        trace_kernel(ctx, ME_KBIT_NN_ROWS_SPARSE);
      } else {
        rows_dense<<<grid, kFlatThreads, 0, ctx->stream>>>(Qc.d_sorted, Qc.d_rel, qb, qe, Rc.d_sorted, Rc.d_rel, index_of(Rc),
                                                           Rc.lat, G, C, Qc.d_nn_idx, Qc.d_nn_d2, Qc.d_nn_sq, far_list, far_count);
        trace_kernel(ctx, ME_KBIT_NN_ROWS_DENSE);
      }
    }
    ME_LAUNCH_CHECK(ctx);
    nn_far_kernel<<<ctx->sm_count * 4, kThreads, 0, ctx->stream>>>(Qc.d_sorted, Rc.d_sorted, index_of(Rc), Rc.lat, coarse_of(Rc), C,
                                                                  Qc.d_nn_idx, Qc.d_nn_d2, far_list, far_count, unres_list, unres_count, acc,
                                                                  ctx->d_trace);
    ME_LAUNCH_CHECK(ctx);
    if (Rc.slab) {
      nn_brute_kernel<<<ctx->sm_count * 4, kThreads, 0, ctx->stream>>>(Qc.d_sorted, Rc.d_xyz, Rc.n, C, Qc.d_nn_idx, Qc.d_nn_d2,
                                                                      unres_list, unres_count, ctx->d_trace);
      ME_LAUNCH_CHECK(ctx);
    }
    nn_far_sq_kernel<<<ctx->sm_count, kThreads, 0, ctx->stream>>>(Qc.d_sorted, Rc.d_xyz, Qc.d_nn_idx, Qc.d_nn_d2, C, Qc.d_nn_sq,
                                                                  far_list, far_count);
    ME_LAUNCH_CHECK(ctx);
    int mom_slots = 0;     // blocks of the kernel that kept the pairs
    if (C.accumulate || C.want_full_cd) {
      const long long sb = use_tile ? 0 : qb, se = use_tile ? Qc.n : qe;
      const int sblocks = std::max(1, (int)std::min<long long>((se - sb + kThreads - 1) / kThreads, (long long)ctx->sm_count * 8));
      nn_stats_kernel<<<sblocks, kThreads, 0, ctx->stream>>>(sb, se, Qc.d_nn_idx, Qc.d_nn_d2, Qc.d_nn_sq, C, acc,
                                                             C.accumulate ? mom : nullptr);
      ME_LAUNCH_CHECK(ctx);
      if (C.accumulate) mom_slots = sblocks;
    }
    if (as_written) {
      pair_as_written_kernel<<<fill_blocks, kThreads, 0, ctx->stream>>>(Qc.ns, Qc.d_nn_idx, Qc.d_nn_d2, Qc.d_nn_sq, C, acc, mom);
      ME_LAUNCH_CHECK(ctx);
      mom_slots = fill_blocks;
    }
    if (mom_slots) {
      merge_moments_kernel<<<1, kThreads, 0, ctx->stream>>>(mom, mom_slots, acc);
      ME_LAUNCH_CHECK(ctx);
    }
  }
  Qc.nn_b = use_tile ? 0 : qb;
  Qc.nn_e = use_tile ? Qc.n : qe;
  if (pack) {      // the accumulators stay on the device (all-reduced there, fetched once per pass)
    if (sharded && use_tile) {
      count_marked_kernel<<<fill_blocks, kThreads, 0, ctx->stream>>>(Qc.d_nn_idx, Qc.n, n_eval);
      ME_LAUNCH_CHECK(ctx);
    }
    pack_nn_kernel<<<1, 32, 0, ctx->stream>>>(acc, (sharded && use_tile) ? n_eval : nullptr, Qc.slab ? Qc.n_owned : (sharded ? qe - qb : Qc.n),
                                              ctx->rank, ctx->d_block + (qwhich == ME_CLOUD_EST ? 0 : kBlkNN));
    ME_LAUNCH_CHECK(ctx);
  }
  Qc.nn_valid = true;
  return ME_OK;
}

int build_both(me_ctx *ctx) {
  // a later build may re-plan the shared lattice and invalidate the earlier one: iterate to a fixed point
  for (int it = 0; it < 3; ++it) {
    ME_TRY(build_grid(ctx, ME_CLOUD_EST));
    ME_TRY(build_grid(ctx, ME_CLOUD_GT));
    if (ctx->cloud[0].grid_valid && ctx->cloud[1].grid_valid) return ME_OK;
  }
  return fail(ctx, ME_ERR_RANGE, "could not lay both clouds out on a common lattice");
}

int run_nn(me_ctx *ctx, const me_nn_params *p, bool pack) {
  if (ctx->cloud[0].n <= 0 || ctx->cloud[1].n <= 0)
    return fail(ctx, ME_ERR_EMPTY, "both clouds must be set (map_eval.cpp:32-35)");
  ME_TRY(build_both(ctx));
  const int dirs = p->directions ? p->directions : 3;
  if (dirs & 1) ME_TRY(run_direction(ctx, ME_CLOUD_EST, p, 2, pack));
  if (dirs & 2) ME_TRY(run_direction(ctx, ME_CLOUD_GT, p, 3, pack));
  return ME_OK;
}

// the records of the last me_eval_nn* still describe the clouds: no call has changed them since, and every direction that
// call evaluated holds its records.  `who` names the caller in the message.
int nn_records_fresh(me_ctx *ctx, const char *who) {
  const me_nn_params *p = &ctx->curve_p;
  const int dirs = p->directions ? p->directions : 3;
  bool fresh = ctx->curve_valid && ctx->curve_gen == ctx->cloud_gen;
  for (int q = 0; q < 2; ++q) fresh = fresh && (!(dirs & (1 << q)) || ctx->cloud[q].nn_valid);
  if (!fresh)
    return fail(ctx, ME_ERR_INVALID, std::string(who) + ": no current NN records; run me_eval_nn* after the last change of the clouds "
                                     "(me_set_cloud*, me_transform, me_voxel_downsample, me_copy_cloud, me_add_*, ICP, a new layout)");
  return ME_OK;
}

// the records of direction q (query cloud q) over the ranges nn_stats_kernel / pair_as_written_kernel walk
CurveSrc record_src(const me_ctx *ctx, int q) {
  const me_nn_params *p = &ctx->curve_p;
  const Cloud &Qc = ctx->cloud[q], &Rc = ctx->cloud[1 - q];
  CurveSrc S;
  S.as_written = q == ME_CLOUD_GT && p->pairing == ME_PAIRING_AS_WRITTEN;
  S.b = S.as_written ? 0 : Qc.nn_b;
  S.e = S.as_written ? Qc.ns : Qc.nn_e;
  S.nn_idx = Qc.d_nn_idx; S.nn_d2 = Qc.d_nn_d2; S.nn_sq = Qc.d_nn_sq;
  S.Qgt = Qc.d_sorted; S.gt_xyz = Qc.d_xyz; S.n_gt = Qc.n; S.est_xyz = Rc.d_xyz; S.n_est = Rc.n;
  return S;
}

int nn_curve(me_ctx *ctx, const double *tau, int K, double **device_block, int32_t *n) {
  const me_nn_params *p = &ctx->curve_p;
  const int dirs = p->directions ? p->directions : 3;
  ME_TRY(nn_records_fresh(ctx, "me_nn_curve*"));
  const int stride = 3 * (K + 1) + 1;
  ME_TRY(ensure(ctx, (void **)&ctx->d_curve, &ctx->cap_curve, 2 * stride + K, sizeof(double)));
  double *blk = ctx->d_curve, *d_tau = ctx->d_curve + 2 * stride;
  const int max_blocks = ctx->sm_count * 4;
  ME_TRY(ensure_work(ctx, (size_t)max_blocks * stride * sizeof(double)));
  ME_CUDA(ctx, cudaMemcpyAsync(d_tau, tau, (size_t)K * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  ME_CUDA(ctx, cudaMemsetAsync(blk, 0, 2 * (size_t)stride * sizeof(double), ctx->stream));
  const size_t smem = (size_t)(K + 3 * (K + 1)) * sizeof(double);
  for (int q = 0; q < 2; ++q) {
    if (!(dirs & (1 << q))) continue;
    NNConst C{};
    set_cutoff(C, p);
    const CurveSrc S = record_src(ctx, q);
    if (S.e <= S.b) continue;
    const int n_blocks = (int)std::min<long long>((S.e - S.b + kCurveThreads - 1) / kCurveThreads, max_blocks);
    const long long per_block = (S.e - S.b + n_blocks - 1) / n_blocks;
    nn_curve_kernel<<<n_blocks, kCurveThreads, smem, ctx->stream>>>(S, C, d_tau, K, per_block, (double *)ctx->d_work);
    ME_LAUNCH_CHECK(ctx);
    nn_curve_merge_kernel<<<(stride + 255) / 256, 256, 0, ctx->stream>>>((const double *)ctx->d_work, n_blocks, stride,
                                                                        blk + q * stride);
    ME_LAUNCH_CHECK(ctx);
  }
  *device_block = blk;
  *n = 2 * stride;
  return ME_OK;
}

// ---- exact distance quantiles: the loop state is QuantRun (common.cuh), the same on every rank -------------------------------
void nn_quantile_free(me_ctx *ctx) {
  QuantRun &R = ctx->quant;
  for (int q = 0; q < 2; ++q)
    if (R.d_keys[q]) { cudaFree(R.d_keys[q]); R.d_keys[q] = nullptr; R.cap_keys[q] = 0; }
  if (R.d_hist) { cudaFree(R.d_hist); R.d_hist = nullptr; R.d_blk = nullptr; R.d_pfx = nullptr; }
  R.open = false;
}

// launch pass R.sel.pass of every direction: pass 0 writes the keys, the later ones read them under the slots' prefixes
static int quant_launch(me_ctx *ctx) {
  QuantRun &R = ctx->quant;
  ME_CUDA(ctx, cudaMemsetAsync(R.d_hist, 0, (size_t)kQuantBlock * sizeof(unsigned long long), ctx->stream));
  if (R.sel.pass > 0)
    ME_CUDA(ctx, cudaMemcpyAsync(R.d_pfx, R.sel.slot_pfx, sizeof(R.sel.slot_pfx), cudaMemcpyHostToDevice, ctx->stream));
  for (int q = 0; q < 2; ++q) {
    const long long n = R.ke[q] - R.kb[q];
    if (n <= 0 || R.sel.n_slots[q] == 0) continue;
    unsigned long long *hist = R.d_hist + (size_t)q * kQuantSlots * kQuantBins;
    if (R.sel.pass == 0) {
      NNConst C{};
      set_cutoff(C, &ctx->curve_p);
      CurveSrc S = record_src(ctx, q);
      S.b = R.kb[q]; S.e = R.ke[q];
      const int grid = (int)std::min<long long>((n + kQuantThreads - 1) / kQuantThreads, (long long)ctx->sm_count * 4);
      nn_quantile_keys_kernel<<<grid, kQuantThreads, 0, ctx->stream>>>(S, C, R.population == ME_DIST_NN, R.d_keys[q], hist);
      ME_LAUNCH_CHECK(ctx);
    } else {
      ME_TRY(quant_hist_launch(ctx, R.d_keys[q], n, R.sel.pass, R.d_pfx + q * kQuantSlots, R.sel.n_slots[q], hist));
    }
  }
  quant_to_block_kernel<<<(kQuantBlock + 255) / 256, 256, 0, ctx->stream>>>(R.d_hist, kQuantBlock, R.d_blk);
  ME_LAUNCH_CHECK(ctx);
  return ME_OK;
}

int nn_quantile_begin(me_ctx *ctx, int population, const double *p, int K) {
  QuantRun &R = ctx->quant;
  R.open = false;
  ME_TRY(nn_records_fresh(ctx, "me_nn_quantile*"));
  if (population == ME_DIST_NN && !ctx->curve_p.want_full_cd)
    return fail(ctx, ME_ERR_INVALID, "me_nn_quantile*: ME_DIST_NN needs every query's nearest neighbour; the last me_eval_nn* "
                                     "ran with want_full_cd = 0, so queries beyond the cut-off were never resolved");
  R.population = population;
  R.K = K;
  for (int k = 0; k < K; ++k) R.p[k] = p[k];
  R.dirs = ctx->curve_p.directions ? ctx->curve_p.directions : 3;
  R.gen = ctx->cloud_gen;
  R.done = false;
  R.sel.pass = 0;
  if (!R.d_hist) {      // the integer histogram, its fp64 block and the slot prefixes in one allocation
    const size_t bytes = (size_t)kQuantBlock * (sizeof(unsigned long long) + sizeof(double)) + sizeof(R.sel.slot_pfx);
    ME_CUDA(ctx, cudaMalloc((void **)&R.d_hist, bytes));
    R.d_blk = (double *)(R.d_hist + kQuantBlock);
    R.d_pfx = (unsigned long long *)(R.d_blk + kQuantBlock);
  }
  for (int q = 0; q < 2; ++q) {
    R.sel.set_targets(q, 0, R.p, R.K);
    R.kb[q] = R.ke[q] = 0;
    if (!(R.dirs & (1 << q))) continue;
    const CurveSrc S = record_src(ctx, q);
    const Cloud &Qc = ctx->cloud[q];
    R.kb[q] = population == ME_DIST_NN ? Qc.nn_b : S.b;      // ME_DIST_NN: the range of the full-CD sum
    R.ke[q] = std::max(R.kb[q], population == ME_DIST_NN ? Qc.nn_e : S.e);
    ME_TRY(ensure(ctx, (void **)&R.d_keys[q], &R.cap_keys[q], R.ke[q] - R.kb[q], sizeof(unsigned long long)));
    R.sel.n_slots[q] = 1;      // pass 0: the empty prefix
    R.sel.slot_pfx[q][0] = 0;
  }
  ME_TRY(quant_launch(ctx));
  R.open = true;
  return ME_OK;
}

static int quant_ready(me_ctx *ctx, const char *who) {
  QuantRun &R = ctx->quant;
  if (!R.open) return fail(ctx, ME_ERR_INVALID, std::string(who) + " without an open selection (me_nn_quantile_begin first)");
  if (R.gen != ctx->cloud_gen) {
    R.open = false;
    return fail(ctx, ME_ERR_INVALID, std::string(who) + ": the clouds changed after me_nn_quantile_begin; the selection is void "
                                     "(run me_eval_nn* and me_nn_quantile_begin again)");
  }
  return ME_OK;
}

int nn_quantile_block(me_ctx *ctx, double **device_block, int32_t *n) {
  ME_TRY(quant_ready(ctx, "me_nn_quantile_block"));
  *device_block = ctx->quant.d_blk;
  *n = kQuantBlock;
  return ME_OK;
}

int nn_quantile_step(me_ctx *ctx, int32_t *done) {
  ME_TRY(quant_ready(ctx, "me_nn_quantile_step"));
  QuantRun &R = ctx->quant;
  auto &T = R.sel;
  if (R.done) { *done = 1; return ME_OK; }
  // the reduced block of pass T.pass: only the rows of the slots in use are read
  R.h_blk.resize(kQuantBlock);
  for (int q = 0; q < 2; ++q)
    if (T.n_slots[q])
      ME_CUDA(ctx, cudaMemcpyAsync(R.h_blk.data() + (size_t)q * kQuantSlots * kQuantBins, R.d_blk + (size_t)q * kQuantSlots * kQuantBins,
                                   (size_t)T.n_slots[q] * kQuantBins * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int q = 0; q < 2; ++q) {
    if (!T.n_slots[q]) continue;
    const double *rows = R.h_blk.data() + (size_t)q * kQuantSlots * kQuantBins;
    if (T.pass == 0) {      // the population size, then the target ranks: k and k + 1 per probability, 0 and n - 1
      double n = 0;
      for (int b = 0; b < kQuantBins; ++b) n += rows[b];
      T.set_targets(q, (long long)n, R.p, R.K);
    }
    if (!T.take_digits(q, rows)) {
      R.open = false;
      return fail(ctx, ME_ERR_INVALID, "me_nn_quantile_step: the block does not hold a rank the selection needs (a block not "
                                       "SUM-reduced over all ranks, or of another selection)");
    }
  }
  if (T.pass == kQuantPasses - 1) {
    R.done = true;
    *done = 1;
    return ME_OK;
  }
  T.next_pass();
  ME_TRY(quant_launch(ctx));
  *done = 0;
  return ME_OK;
}

int nn_quantile_end(me_ctx *ctx, me_quantile_result *out) {
  ME_TRY(quant_ready(ctx, "me_nn_quantile_end"));
  QuantRun &R = ctx->quant;
  if (!R.done) return fail(ctx, ME_ERR_INVALID, "me_nn_quantile_end before the last me_nn_quantile_step (*done = 1)");
  R.open = false;
  std::memset(out, 0, sizeof(*out));
  out->population = R.population;
  out->n_probs = R.K;
  for (int k = 0; k < R.K; ++k) out->p[k] = R.p[k];
  for (int q = 0; q < 2; ++q) {
    me_quantile_dir &D = q == 0 ? out->est_to_gt : out->gt_to_est;
    D.n = R.sel.n[q];
    auto x = [&](long long r) { return R.sel.value(q, r); };      // the order statistic of rank r, one of the targets
    D.min = D.n > 0 ? x(0) : NAN;
    D.max = D.n > 0 ? x(D.n - 1) : NAN;
    for (int k = 0; k < R.K; ++k) {
      if (D.n == 0) { D.lo[k] = D.hi[k] = D.value[k] = NAN; continue; }
      long long kk;
      double g;
      quantile_rank(D.n, R.p[k], &kk, &g);
      D.rank[k] = kk;
      D.lo[k] = x(kk);
      D.hi[k] = x(std::min<long long>(kk + 1, D.n - 1));
      D.value[k] = quantile_lerp(D.lo[k], D.hi[k], g);
    }
  }
  const bool both = R.population == ME_DIST_NN && R.dirs == 3 && out->est_to_gt.n > 0 && out->gt_to_est.n > 0;
  out->hausdorff = both ? std::max(out->est_to_gt.max, out->gt_to_est.max) : NAN;
  return ME_OK;
}

int unsort_nn(me_ctx *ctx, int which_query, int32_t *h_idx, double *h_d2) {
  Cloud &Qc = ctx->cloud[which_query];
  if (!Qc.nn_valid) return fail(ctx, ME_ERR_INVALID, "me_get_nn before me_eval_nn");
  size_t bytes = (size_t)Qc.n * (sizeof(int32_t) + sizeof(double)) + 256;
  ME_TRY(ensure_work(ctx, bytes));
  double *od2 = (double *)ctx->d_work;
  int32_t *oidx = (int32_t *)((char *)ctx->d_work + (size_t)Qc.n * sizeof(double));
  int blocks = (int)std::min<long long>((Qc.n + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
  fill_nn_kernel<<<blocks, kThreads, 0, ctx->stream>>>(oidx, od2, Qc.n);
  ME_LAUNCH_CHECK(ctx);
  unsort_nn_kernel<<<blocks, kThreads, 0, ctx->stream>>>(Qc.d_sorted, Qc.ns, Qc.d_nn_idx, Qc.d_nn_d2, oidx, od2);
  ME_LAUNCH_CHECK(ctx);
  if (h_idx) ME_CUDA(ctx, cudaMemcpyAsync(h_idx, oidx, (size_t)Qc.n * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  if (h_d2) ME_CUDA(ctx, cudaMemcpyAsync(h_d2, od2, (size_t)Qc.n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return ME_OK;
}

}  // namespace me

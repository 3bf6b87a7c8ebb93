// mme.cu — mean map entropy: per-point radius neighbourhood -> 3x3 covariance -> 0.5 ln(2 pi e det).
//
// Replaces (reference, map_eval/src/map_eval.cpp):
//   :1608-1737  ComputeMeanMapEntropyUsingNormalTBB   (k >= 10, default for the estimated map)
//   :1538-1606  ComputeMeanMapEntropyUsingNormal      (k >= 10, OpenMP variant)
//   :1438-1535  ComputeMeanMapEntropy                 (k >=  5, serial, ground truth)
//   :1433-1436  ComputeEntropy, and the min/max side effect of ColorPointCloudByMME (:697-701)
//
// The reference materialises every neighbour list (KDTreeFlann::SearchRadius -> Eigen::MatrixXd(3,k)); here no list
// exists.  Accepted points are folded into nine fp64 moments taken about the query point itself (sum d, sum d d^T):
// the query is its own nearest neighbour at d = 0 and contributes nothing, which is exactly the reference's
// "erase the first hit" (:1672-1673), and cov = (S2 - S1 S1^T / k) / (k - 1) equals the reference's centred product.
//
// Kernels, all one thread per query with the queries in cell-sorted order (a warp = x-neighbours of one lattice row):
//   mme_flat_kernel<R>  (R = ceil(r/h) <= 3, the dominant kernel of the pass): per-thread run table in shared memory,
//                       flattened candidate walk, fp32 screening on the cell-relative copy, exact fp64 decision inside
//                       the fp32 error band (the neighbour COUNT is bit-exact), fp64 moment accumulation.
//   mme_plane_kernel    (4..15 rings): the same walk with a run table of one dz plane at a time.
//   mme_kernel          (> 15 rings): nested row walk with fp64 tests on the 32-byte records.
//   mme_fp64_finish_kernel: the queries the fp32-offset kernels could not certify (thin surfaces), walked again as mme_kernel.
// run_mme picks the lattice per radius: when the radius spans more than 3 cells of the shared lattice the cloud is laid
// out on a lattice of its own with h = r/2 for this sweep.  Variants that were measured slower and dropped: shared-memory
// tile + TMA staging, 16-byte table entries, software prefetch, plane tables at R = 2.
// Test hooks (environment): ME_MME_WALK forces mme_kernel, ME_MME_SHARED_LATTICE keeps the shared lattice.
#include "common.cuh"
#include "flat.cuh"
#include "mme_walk.cuh"
#include <algorithm>
#include <cstdlib>
#include <cstring>

namespace me {

static constexpr int kThreads = 128;
// trace events sit above the sweep bits, in the 32-bit device word
static_assert((int)ME_KBIT_COUNT <= (int)ME_TEV_MME_FP64_FINISH && (int)ME_TEV_MME_FP64_FINISH < 32, "trace event bit");
// an fp32-offset kernel finishes a query in fp64 when its certificate of the offsets' effect on the entropy exceeds this
// (nats); below it the certified error is at most this (a float32 emulation of the offsets stays 13-330 times below the
// certificate, tests/test_exact_mme.py)
static constexpr double kFp64FinishNats = 1e-3;

struct MmeAcc {
  unsigned long long n_valid, n_query;
  double sum;
  unsigned long long min_enc, max_enc;   // ordered encodings of the extrema over entropies != 0
  unsigned long long n_fp64;             // queries an fp32-offset kernel left to mme_fp64_finish_kernel
};

__global__ void mme_init_kernel(MmeAcc *a) {
  a->n_valid = 0; a->n_query = 0; a->sum = 0.0; a->n_fp64 = 0;
  a->min_enc = enc_ordered(INFINITY); a->max_enc = enc_ordered(-INFINITY);
}

struct ThreadStats {
  double sum, mn, mx;
  unsigned int valid, queries;
  __device__ __forceinline__ void init() { sum = 0.0; mn = INFINITY; mx = -INFINITY; valid = 0; queries = 0; }
};

struct MmeConst {
  float h, inv_h;            // cell edge and its inverse
  float rc2;                 // (r/h)^2 with slack: row / cell pruning is conservative, the point test decides
  float r2_lo, r2_hi;        // fp32 screening band around r^2
  double r2;                 // exact r^2
  int min_neighbors;
  int dimx, dimy, dimz;
  Owned own;                 // slab layout: the planes whose points this rank evaluates (the halo points are neighbours only)
  double E2;                 // square of the bound E of the fp32 offsets' error per axis
  double s2_max;             // fp64 finish when s^2 exceeds this (the s at which 0.5 |ln(1 - rho')| = kFp64FinishNats)
  uint32_t *fp64_list;       // sorted indices of the queries left to the fp64 finish (count: MmeAcc::n_fp64)
};

// map_eval.cpp:1675-1697 for one query.
// CERT (the fp32-offset kernels): the moments were accumulated from offsets that carry an error of up to C.E per axis.
// To first order that moves ln det by at most rho = 2 sqrt(3) s + 3 s^2, s = E sqrt(k / (k - 1) * tr adj(C) / det) (rotation
// invariant: on a surface of normal noise sigma it grows like E / sigma); rho' = rho + 3 rho^2 bounds the quadratic terms.
// rho' grows with s, so the test is s^2 <= s2_max, cleared of the square root and the division.  A query whose
// certificate exceeds kFp64FinishNats — thin surfaces, det <= 0 — is not finished here: its sorted index goes to
// C.fp64_list, and mme_fp64_finish_kernel evaluates it again from fp64 offsets (tests/exact_ref.py states the bounds).
template <bool CERT = false>
__device__ __forceinline__ double finish_entropy(const Moments &m, int min_neighbors, ThreadStats &t,
                                                 const MmeConst *C = nullptr, long long i = 0, MmeAcc *acc = nullptr) {
  t.queries++;
  if (m.cnt == 0) return 0.0;
  const long long k = (long long)m.cnt - 1;                 // erase(begin()): the query itself (:1672-1673)
  if (k < (long long)min_neighbors) return 0.0;
  const double kd = (double)k, inv = 1.0 / (double)(k - 1);
  double c[9];
  c[0] = (m.sxx - m.s1x * m.s1x / kd) * inv;
  c[1] = (m.sxy - m.s1x * m.s1y / kd) * inv;
  c[2] = (m.sxz - m.s1x * m.s1z / kd) * inv;
  c[4] = (m.syy - m.s1y * m.s1y / kd) * inv;
  c[5] = (m.syz - m.s1y * m.s1z / kd) * inv;
  c[8] = (m.szz - m.s1z * m.s1z / kd) * inv;
  c[3] = c[1]; c[6] = c[2]; c[7] = c[5];
  const double det = det3(c);
  if (CERT) {
    const double adj = (c[0] * c[4] - c[1] * c[1]) + (c[0] * c[8] - c[2] * c[2]) + (c[4] * c[8] - c[5] * c[5]);
    // s^2 = E^2 k / (k - 1) adj / det <= s2_max, with det > 0; NaN fails the test and is listed too
    if (!(det > 0.0 && C->E2 * kd * adj <= C->s2_max * (kd - 1.0) * det)) {
      C->fp64_list[atomicAdd(&acc->n_fp64, 1ull)] = (uint32_t)i;
      return 0.0;
    }
  }
  const double e = 0.5 * log(2 * M_PI * M_E * det);         // map_eval.cpp:1434 / :1656
  if (isnan(e) || isinf(e)) return 0.0;
  t.sum += e; t.valid++;
  if (e != 0.0) { t.mn = fmin(t.mn, e); t.mx = fmax(t.mx, e); }
  return e;
}

__device__ void flush_stats(ThreadStats &t, MmeAcc *acc) {
  __shared__ double sh_sum[32], sh_min[32], sh_max[32];
  __shared__ unsigned long long sh_cnt[32], sh_q[32];
  t.sum = warp_sum(t.sum); t.mn = warp_min(t.mn); t.mx = warp_max(t.mx);
  const long long tv = warp_sum_ll((long long)t.valid), tq = warp_sum_ll((long long)t.queries);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  if (lane == 0) { sh_sum[warp] = t.sum; sh_min[warp] = t.mn; sh_max[warp] = t.mx; sh_cnt[warp] = (unsigned long long)tv; sh_q[warp] = (unsigned long long)tq; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0, mn = INFINITY, mx = -INFINITY;
    unsigned long long c = 0, q = 0;
    for (int w = 0; w < nwarps; ++w) { s += sh_sum[w]; mn = fmin(mn, sh_min[w]); mx = fmax(mx, sh_max[w]); c += sh_cnt[w]; q += sh_q[w]; }
    if (c) { atomicAdd(&acc->n_valid, c); atomicAdd(&acc->sum, s); }
    if (q) atomicAdd(&acc->n_query, q);
    if (mn <= mx) { atomicMin(&acc->min_enc, enc_ordered(mn)); atomicMax(&acc->max_enc, enc_ordered(mx)); }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// one thread per query, queries in cell-sorted order: the 32 queries of a warp are neighbours along x in one lattice
// row, so they walk the same (2k+1)^2 rows and their candidate loads hit the same L1 lines (measured: handing the
// queries out tile by tile instead costs 20 %)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
mme_kernel(const P4 *__restrict__ S, long long q_begin, long long q_end, CellIndex I,
           Lattice L, double r2, float rc2, int rings, int min_neighbors, Owned own, double *__restrict__ entropy_sorted,
           MmeAcc *__restrict__ acc) {
  ThreadStats ts;
  ts.init();
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = q_begin + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < q_end; i += stride) {
    const P4 q = load_p4(S + i);
    if (own.axis) {      // slab layout (dense table): halo points are neighbours only
      int cx, cy, cz;
      cell_from_tag(I, q.idx, 0, cx, cy, cz);
      if (!owns(own, cy, cz)) continue;
    }
    Moments m;
    m.init();
    walk_global(q, S, I, L, r2, rc2, rings, m);
    entropy_sorted[i] = finish_entropy(m, min_neighbors, ts);
  }
  flush_stats(ts, acc);
}

// the queries an fp32-offset kernel listed (finish_entropy<true>): walked again with fp64 offsets (the differences of the
// records, as mme_kernel), finished and folded into the accumulators.  The count is read on the device, so the launch
// needs no host round trip; with an empty list it returns at once.  The listing kernel has counted the queries.
__global__ void __launch_bounds__(kThreads)
mme_fp64_finish_kernel(const P4 *__restrict__ S, const uint32_t *__restrict__ list, CellIndex I, Lattice L, double r2,
                       float rc2, int rings, int min_neighbors, double *__restrict__ entropy_sorted, MmeAcc *__restrict__ acc,
                       unsigned int *trace) {
  const unsigned long long n = *(volatile unsigned long long *)&acc->n_fp64;
  if (n == 0) return;
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicOr(trace, 1u << ME_TEV_MME_FP64_FINISH);
  ThreadStats ts;
  ts.init();
  for (unsigned long long t = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; t < n;
       t += (unsigned long long)gridDim.x * blockDim.x) {
    const uint32_t i = list[t];
    Moments m;
    m.init();
    walk_global(load_p4(S + i), S, I, L, r2, rc2, rings, m);
    entropy_sorted[i] = finish_entropy(m, min_neighbors, ts);
  }
  ts.queries = 0;
  flush_stats(ts, acc);
}

// ---------------------------------------------------------------------------------------------------------------
// flat kernel (rings <= 3): the dominant kernel of the pass.
//
// One thread per query, queries in cell-sorted order.  Per query the (2R+1)^2 lattice rows of the neighbourhood are
// pruned against the sphere with a handful of fp32 compares (no sqrt: the x-extent of a row is found by comparing the
// row's remaining squared radius against the 2R per-query squared gaps to the neighbouring cell faces), and the
// surviving x-runs are written to a per-thread run table in shared memory ([row][thread], conflict-free).  The
// candidates are then walked as ONE flattened loop, so that the 32 lanes of a warp — neighbours along x, hence with
// near-identical run tables — stay in step whatever the occupancy of the individual rows.
//
// Candidates are screened in fp32 on the cell-relative copy of the cloud (Cloud::d_rel, 16 B/point): the offset
// between two points is rebuilt as (ix_c - ix_q) h + (rel_c - rel_q), whose error is ~1e-6 h independent of the world
// extent.  A candidate whose fp32 d^2 falls inside the error band around r^2 is decided exactly, in fp64, from the
// raw records with the reference's operation order (nanoflann: d2 < r2, strict), so the neighbour COUNT — and with it
// the k >= min_neighbors validity test — is bit-exact.  Accepted offsets are accumulated in fp64.
// ---------------------------------------------------------------------------------------------------------------

template <int R, bool E16, int U2, int SP>      // U2: 0 plain walk, 1 two candidates (two loads in flight) per iteration; SP: sparse cell table
// 8 CTAs/SM at R <= 2 (64 registers, a few spilled words) beat the unbounded register count on C3 (chosen on B200, not
// re-measured on H100, which has the same register file and shared memory per SM); at R = 3 the 49-row
// table bounds it at 4
__global__ void __launch_bounds__(kFlatThreads, (R <= 2 ? 8 : 4))
mme_flat_kernel(const P4 *__restrict__ S, const float4 *__restrict__ rel, long long q_begin, long long q_end,
                CellIndex I, MmeConst C, double *__restrict__ entropy_sorted,
                MmeAcc *__restrict__ acc) {
  extern __shared__ __align__(16) unsigned char flat_smem[];
  RunTab<E16> T(flat_smem);
  const int tid = threadIdx.x;
  const float h = C.h, r2_lo = C.r2_lo, r2_hi = C.r2_hi;
  ThreadStats ts;
  ts.init();
  const long long stride = (long long)gridDim.x * kFlatThreads;
  for (long long i = q_begin + blockIdx.x * (long long)kFlatThreads + tid; i < q_end; i += stride) {
    const float4 qr = __ldg(rel + i);
    const uint32_t cq = cell_of(__double_as_longlong(__ldg(reinterpret_cast<const double *>(S + i) + 3)));
    const int ix = (int)qr.w;
    const uint32_t cyz = SP ? cq : cq / (uint32_t)C.dimx;
    const int iy = (int)(cyz % (uint32_t)C.dimy), iz = (int)(cyz / (uint32_t)C.dimy);
    if (!owns(C.own, iy, iz)) continue;
    const float ux = qr.x * C.inv_h, uy = qr.y * C.inv_h, uz = qr.z * C.inv_h;
    float gl[R], gr[R];      // squared gaps to the d-th cell on the left / right along x (increasing in d)
#pragma unroll
    for (int d = 1; d <= R; ++d) { gl[d - 1] = gap2(-d, ux); gr[d - 1] = gap2(d, ux); }
    int nrun = 0;
#pragma unroll
    for (int dz = -R; dz <= R; ++dz) {
      const int z = iz + dz;
      const float remz = C.rc2 - gap2(dz, uz);
      const float czv = (float)dz * h - qr.z;
#pragma unroll
      for (int dy = -R; dy <= R; ++dy) {
        const int y = iy + dy;
        const float rem = remz - gap2(dy, uy);
        int da = 0, db = 0;
#pragma unroll
        for (int d = 0; d < R; ++d) { da -= (gl[d] <= rem) ? 1 : 0; db += (gr[d] <= rem) ? 1 : 0; }
        const int xa = max(ix + da, 0), xb = min(ix + db, C.dimx - 1);
        uint32_t s = 0, e = 0;
        if ((unsigned)z < (unsigned)C.dimz && (unsigned)y < (unsigned)C.dimy && rem >= 0.f) cell_range<SP>(I, z, y, xa, xb, s, e);
        if (e > s) { T.put(nrun, tid, s, e, dy + R, dz + R, (float)dy * h - qr.y, czv); ++nrun; }
      }
    }
    Moments m;
    m.init();
    // one candidate: fp32 screen on the cell-relative offsets, exact fp64 decision inside the error band (rare)
    auto process = [&](const float4 &c, float cy, float cz, uint32_t j) {
      const float dx = fmaf(c.w - qr.w, h, c.x - qr.x), dy = c.y + cy, dz = c.z + cz;
      const float d2 = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
      if (d2 < r2_hi) {
        bool in = true;
        if (d2 > r2_lo) {
          const P4 q = load_p4(S + i), p = load_p4(S + j);
          in = d2_kd(q.x, q.y, q.z, p.x, p.y, p.z) < C.r2;      // nanoflann RadiusResultSet: strict <
        }
        if (in) m.add((double)dx, (double)dy, (double)dz);
      }
    };
    RunWalk w;
    w.start(nrun);
    if (U2 == 1) {
      for (;;) {
        uint32_t j0, j1;
        float y0, z0, y1, z1;
        if (!w.next(T, tid, h, qr.y, qr.z, R, j0, y0, z0)) break;
        const bool v1 = w.next(T, tid, h, qr.y, qr.z, R, j1, y1, z1);
        const float4 c0 = __ldg(rel + j0);
        const float4 c1 = __ldg(rel + (v1 ? j1 : j0));
        process(c0, y0, z0, j0);
        if (v1) process(c1, y1, z1, j1);
      }
    } else {
      uint32_t j0;
      float y0, z0;
      while (w.next(T, tid, h, qr.y, qr.z, R, j0, y0, z0)) process(__ldg(rel + j0), y0, z0, j0);
    }
    entropy_sorted[i] = finish_entropy<true>(m, C.min_neighbors, ts, &C, i, acc);
  }
  flush_stats(ts, acc);
}

// ---------------------------------------------------------------------------------------------------------------
// rows kernel (rings <= 3): warp-synchronous row walk with deferred fp64 accumulation.
//
// Same decomposition as the flat kernel (one thread per query, queries in cell-sorted order, the (2R+1)^2 lattice rows
// pruned against the sphere), but the control flow is WARP-UNIFORM: the rows are enumerated by a compile-time loop that
// all 32 lanes run together, and inside a row every lane walks its own x-run for max-over-lanes(len) steps
// (REDUX.MAX).  No run table, no per-lane refill branches: at any time the 32 lanes read the same row of the reference
// cloud, i.e. a window of a few consecutive 128-byte lines (the flat walk has its lanes in up to 27 different rows at
// once).  The price is lanes idling while the longest run of the row finishes (~50 % of the slots on C3).
//
// The fp64 work is taken off the walk: a candidate that passes the fp32 screen (d2 < r2_hi) is only APPENDED — one
// predicated STS.128 of (dx, dy, dz, index) to a per-thread ring in shared memory ([slot][thread], conflict-free).
// When some lane's ring is nearly full the warp drains all rings together: a dense loop in which ~3 of 4 lanes hold an
// entry, where the exact fp64 decision inside the error band (rare) and the 12 fp64 moment updates run.  In the flat
// kernel those 16 fp64-pipe instructions were issued at every step for the ~40 % of lanes that accept.
// ---------------------------------------------------------------------------------------------------------------
static constexpr int kRowsThreads = 128;

// shared-memory ring accessed through 32-bit shared addresses held in one register (the compiler otherwise rebuilds the
// generic pointer from %tid at every store)
__device__ __forceinline__ void ring_put(uint32_t addr, float a, float b, float c, uint32_t d, bool p) {
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %5, 0;\n\t@q st.shared.v4.b32 [%0], {%1, %2, %3, %4};\n\t}\n"
               ::"r"(addr), "r"(__float_as_uint(a)), "r"(__float_as_uint(b)), "r"(__float_as_uint(c)), "r"(d), "r"((uint32_t)p));
}
__device__ __forceinline__ uint4 ring_get(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];\n" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ float sqrt_approx(float x) {
  float y;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int R, int CAP, int U>      // CAP ring slots per thread, U candidates per inner iteration
__global__ void __launch_bounds__(kRowsThreads, (R <= 2 ? 6 : 5))
mme_rows_kernel(const P4 *__restrict__ S, const float4 *__restrict__ rel, long long q_begin, long long q_end,
                CellIndex I, MmeConst C, double *__restrict__ entropy_sorted,
                MmeAcc *__restrict__ acc) {
  constexpr int NS = 2 * R + 1;
  constexpr uint32_t kSlot = kRowsThreads * sizeof(uint4);      // bytes between two slots of one thread
  extern __shared__ __align__(16) unsigned char rows_smem[];
  // slot t of this thread: ring0 + t * kSlot
  uint32_t ring0 = (uint32_t)__cvta_generic_to_shared(rows_smem) + threadIdx.x * (uint32_t)sizeof(uint4);
  asm volatile("" : "+r"(ring0));      // opaque: keep it in a register
  // per-thread squared gaps (in cells) to the lattice rows dy / planes dz away: gyz[dy + R][thread], gyz[NS + dz + R][thread]
  float *gyz = reinterpret_cast<float *>(rows_smem + (size_t)CAP * kSlot) + threadIdx.x;
  const unsigned FULL = 0xffffffffu;
  const float h = C.h, r2_lo = C.r2_lo, r2_hi = C.r2_hi;
  ThreadStats ts;
  ts.init();
  const long long stride = (long long)gridDim.x * kRowsThreads;
  for (long long base = q_begin + blockIdx.x * (long long)kRowsThreads; base < q_end; base += stride) {
    const long long i = base + threadIdx.x;
    const long long il = i < q_end ? i : q_end - 1;
    const float4 qr = __ldg(rel + il);
    const uint32_t cq = cell_of(__double_as_longlong(__ldg(reinterpret_cast<const double *>(S + il) + 3)));
    const int ix = (int)qr.w;
    const uint32_t cyz = I.sparse ? cq : cq / (uint32_t)C.dimx;
    const int iy = (int)(cyz % (uint32_t)C.dimy), izq = (int)(cyz / (uint32_t)C.dimy);
    const bool live = i < q_end && owns(C.own, iy, izq);      // dead lanes run along with empty runs (warp collectives need them)
    const int iz = live ? izq : -1000000;
    const float ux = qr.x * C.inv_h;
    {
      const float uy = qr.y * C.inv_h, uz = qr.z * C.inv_h;
#pragma unroll
      for (int d = -R; d <= R; ++d) { gyz[(d + R) * kRowsThreads] = gap2(d, uy); gyz[(NS + d + R) * kRowsThreads] = gap2(d, uz); }
    }

    Moments m;
    m.init();
    uint32_t wp = ring0;                               // next free slot of this thread's ring
    // drain the rings of the whole warp: exact decision inside the fp32 error band, then the fp64 moments
    auto drain = [&]() {
      const uint32_t mx = __reduce_max_sync(FULL, wp - ring0);
#pragma unroll 1
      for (uint32_t t = 0; t < mx; t += kSlot) {
        if (ring0 + t < wp) {
          const uint4 v = ring_get(ring0 + t);
          const float dx = __uint_as_float(v.x), dy = __uint_as_float(v.y), dz = __uint_as_float(v.z);
          const float d2 = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
          bool in = true;
          if (d2 > r2_lo) {
            const P4 q = load_p4(S + i), p = load_p4(S + v.w);
            in = d2_kd(q.x, q.y, q.z, p.x, p.y, p.z) < C.r2;      // nanoflann RadiusResultSet: strict <
          }
          if (in) m.add((double)dx, (double)dy, (double)dz);
        }
      }
      wp = ring0;
    };

    // the (2R+1)^2 rows, one after the other for the whole warp (a runtime loop: one copy of the walk in the instruction
    // cache instead of 25)
    int dy = -R, dz = -R;
#pragma unroll 1
    for (int row_i = 0; row_i < NS * NS; ++row_i) {
      const int z = iz + dz, y = iy + dy;
      const float rem = C.rc2 - gyz[(NS + dz + R) * kRowsThreads] - gyz[(dy + R) * kRowsThreads];
      uint32_t s = 0, e = 0;
      if ((unsigned)z < (unsigned)C.dimz && (unsigned)y < (unsigned)C.dimy && rem >= 0.f) {
        // cells d steps to the left have gap ux + d - 1, to the right d - ux: keep those with gap <= sqrt(rem) (+ slack)
        const float xw = sqrt_approx(rem) + 1e-3f;
        const int da = min(R, (int)(xw - ux + 1.f)), db = min(R, (int)(xw + ux));
        const int xa = max(ix - da, 0), xb = min(ix + db, C.dimx - 1);
        cell_range(I, z, y, xa, xb, s, e);
      }
      const int len = (int)(e - s);
      const int maxlen = __reduce_max_sync(FULL, len);
      const float cyv = (float)dy * h - qr.y, czv = (float)dz * h - qr.z;
      const float4 *p = rel + s;
      uint32_t j = s;
      float4 c[U];
#pragma unroll
      for (int u = 0; u < U; ++u) c[u] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
      for (int k0 = 0; k0 < maxlen; k0 += U, p += U, j += U) {
        if (__any_sync(FULL, wp > ring0 + (uint32_t)(CAP - U) * kSlot)) drain();
#pragma unroll
        for (int u = 0; u < U; ++u)
          if (k0 + u < len) c[u] = __ldg(p + u);       // lanes past their run keep a stale candidate; `take` masks it
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const float dx = fmaf(c[u].w - qr.w, h, c[u].x - qr.x), dyf = c[u].y + cyv, dzf = c[u].z + czv;
          const float d2 = fmaf(dzf, dzf, fmaf(dyf, dyf, dx * dx));
          const bool take = (k0 + u < len) && (d2 < r2_hi);
          ring_put(wp, dx, dyf, dzf, j + (uint32_t)u, take);
          wp += take ? kSlot : 0u;
        }
      }
      if (++dy > R) { dy = -R; ++dz; }
    }
    drain();
    const double ent = finish_entropy<true>(m, C.min_neighbors, ts, &C, i, acc);      // dead lanes have no moments
    if (live) entropy_sorted[i] = ent;
    else ts.queries--;       // finish_entropy counted the dead lane
  }
  flush_stats(ts, acc);
}

template <int R, int CAP, int U>
static int launch_rows_v(me_ctx *ctx, Cloud &c, long long qb, long long qe, const MmeConst &C, MmeAcc *acc) {
  const size_t smem = (size_t)CAP * kRowsThreads * sizeof(uint4) + (size_t)2 * (2 * R + 1) * kRowsThreads * sizeof(float);
  if (smem > 48 * 1024)
    ME_CUDA(ctx, cudaFuncSetAttribute(mme_rows_kernel<R, CAP, U>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int blocks = (int)std::min<long long>((qe - qb + kRowsThreads - 1) / kRowsThreads, (long long)ctx->sm_count * 192);
  mme_rows_kernel<R, CAP, U><<<blocks, kRowsThreads, smem, ctx->stream>>>(c.d_sorted, c.d_rel, qb, qe, index_of(c), C, c.d_entropy, acc);
  ME_LAUNCH_CHECK(ctx);
  trace_kernel(ctx, ME_KBIT_MME_ROWS1 + R - 1);
  ctx->mme_rows_cfg = (CAP << 8) | U;
  return ME_OK;
}

template <int R>
static int launch_rows(me_ctx *ctx, Cloud &c, long long qb, long long qe, const MmeConst &C, MmeAcc *acc) {
  const char *v = getenv("ME_MME_ROWS");      // tuning hook: ring capacity / candidates per iteration
  if (v && !strcmp(v, "8,2")) return launch_rows_v<R, 8, 2>(ctx, c, qb, qe, C, acc);
  if (v && !strcmp(v, "16,2")) return launch_rows_v<R, 16, 2>(ctx, c, qb, qe, C, acc);
  if (v && !strcmp(v, "12,4")) return launch_rows_v<R, 12, 4>(ctx, c, qb, qe, C, acc);
  if (v && !strcmp(v, "16,4")) return launch_rows_v<R, 16, 4>(ctx, c, qb, qe, C, acc);
  return launch_rows_v<R, 12, 2>(ctx, c, qb, qe, C, acc);
}

// ---------------------------------------------------------------------------------------------------------------
// plane kernel (3 < rings <= kMaxPlaneRings): the same fp32-screened walk for radii spanning many cells (e.g. r = 1.0 m
// on a ~0.15 m lattice).  The run table holds the 2R+1 rows of ONE dz plane at a time (a full (2R+1)^2 table would not
// fit), the candidates of a plane are walked flattened, lanes re-synchronise at the plane boundaries — cheap here,
// because with many cells per radius every row run holds many candidates.
// ---------------------------------------------------------------------------------------------------------------
static constexpr int kMaxPlaneRings = 15;

__global__ void __launch_bounds__(kFlatThreads)
mme_plane_kernel(const P4 *__restrict__ S, const float4 *__restrict__ rel, long long q_begin, long long q_end,
                 CellIndex I, MmeConst C, int R, double *__restrict__ entropy_sorted,
                 MmeAcc *__restrict__ acc) {
  extern __shared__ __align__(16) unsigned char flat_smem[];
  uint2 *tab = reinterpret_cast<uint2 *>(flat_smem);      // [slot][thread] {begin, len << 8 | dy + R}
  const int tid = threadIdx.x;
  const float h = C.h, r2_lo = C.r2_lo, r2_hi = C.r2_hi;
  ThreadStats ts;
  ts.init();
  const long long stride = (long long)gridDim.x * kFlatThreads;
  for (long long i = q_begin + blockIdx.x * (long long)kFlatThreads + tid; i < q_end; i += stride) {
    const float4 qr = __ldg(rel + i);
    const uint32_t cq = cell_of(__double_as_longlong(__ldg(reinterpret_cast<const double *>(S + i) + 3)));
    const int ix = (int)qr.w;
    const uint32_t cyz = I.sparse ? cq : cq / (uint32_t)C.dimx;
    const int iy = (int)(cyz % (uint32_t)C.dimy), iz = (int)(cyz / (uint32_t)C.dimy);
    if (!owns(C.own, iy, iz)) continue;
    const float ux = qr.x * C.inv_h, uy = qr.y * C.inv_h, uz = qr.z * C.inv_h;
    Moments m;
    m.init();
    for (int dz = -R; dz <= R; ++dz) {
      const int z = iz + dz;
      const float remz = C.rc2 - gap2(dz, uz);
      const float cz = (float)dz * h - qr.z;
      int nrun = 0;
      if ((unsigned)z < (unsigned)C.dimz && remz >= 0.f) {
        for (int dy = -R; dy <= R; ++dy) {
          const int y = iy + dy;
          const float rem = remz - gap2(dy, uy);
          if ((unsigned)y >= (unsigned)C.dimy || rem < 0.f) continue;
          // cells d steps to the left have gap ux + d - 1, to the right d - ux: keep those with gap <= sqrt(rem) (+ slack)
          const float xw = sqrtf(rem) + 1e-3f;
          const int da = -min(R, max(0, (int)floorf(xw - ux + 1.f))), db = min(R, max(0, (int)floorf(xw + ux)));
          const int xa = max(ix + da, 0), xb = min(ix + db, C.dimx - 1);
          uint32_t s, e;
          cell_range(I, z, y, xa, xb, s, e);
          if (e > s) { tab[nrun * kFlatThreads + tid] = make_uint2(s, ((e - s) << 8) | (uint32_t)(dy + R)); ++nrun; }
        }
      }
      uint32_t j = 0, e = 0;
      int r = 0;
      float cy = 0.f;
      auto next = [&](uint32_t &idx, float &ocy) -> bool {
        if (j >= e) {
          if (r >= nrun) return false;
          const uint2 t = tab[r * kFlatThreads + tid];
          ++r;
          j = t.x; e = t.x + (t.y >> 8);
          cy = fmaf((float)((int)(t.y & 255u) - R), h, -qr.y);
        }
        idx = j++; ocy = cy;
        return true;
      };
      auto process = [&](const float4 &c, float cyv, uint32_t jj) {
        const float dx = fmaf(c.w - qr.w, h, c.x - qr.x), dy = c.y + cyv, dzf = c.z + cz;
        const float d2 = fmaf(dzf, dzf, fmaf(dy, dy, dx * dx));
        if (d2 < r2_hi) {
          bool in = true;
          if (d2 > r2_lo) {
            const P4 q = load_p4(S + i), p = load_p4(S + jj);
            in = d2_kd(q.x, q.y, q.z, p.x, p.y, p.z) < C.r2;      // nanoflann RadiusResultSet: strict <
          }
          if (in) m.add((double)dx, (double)dy, (double)dzf);
        }
      };
      for (;;) {
        uint32_t j0, j1;
        float y0, y1;
        if (!next(j0, y0)) break;
        const bool v1 = next(j1, y1);
        const float4 c0 = __ldg(rel + j0);
        const float4 c1 = __ldg(rel + (v1 ? j1 : j0));
        process(c0, y0, j0);
        if (v1) process(c1, y1, j1);
      }
    }
    entropy_sorted[i] = finish_entropy<true>(m, C.min_neighbors, ts, &C, i, acc);
  }
  flush_stats(ts, acc);
}

static int launch_plane(me_ctx *ctx, Cloud &c, long long qb, long long qe, const MmeConst &C, int rings, MmeAcc *acc) {
  const size_t smem = (size_t)(2 * rings + 1) * kFlatThreads * sizeof(uint2);
  const int blocks = (int)std::min<long long>((qe - qb + kFlatThreads - 1) / kFlatThreads, (long long)ctx->sm_count * 64);
  mme_plane_kernel<<<blocks, kFlatThreads, smem, ctx->stream>>>(c.d_sorted, c.d_rel, qb, qe, index_of(c), C, rings, c.d_entropy, acc);
  ME_LAUNCH_CHECK(ctx);
  trace_kernel(ctx, ME_KBIT_MME_PLANE);
  return ME_OK;
}

template <int R>
static int launch_flat(me_ctx *ctx, Cloud &c, long long qb, long long qe, const MmeConst &C, MmeAcc *acc) {
  // 8-byte table entries + two candidates per iteration: the fastest combination on C3 (chosen on B200, not re-measured
  // on H100)
  constexpr bool E16 = false;
  constexpr int U2 = 1;
  constexpr int NROW = (2 * R + 1) * (2 * R + 1);
  const size_t smem = (size_t)NROW * kFlatThreads * RunTab<E16>::kEntryBytes;
  // per launch (function attributes are per device; a process may drive several devices through several contexts)
  if (smem > 48 * 1024) {
    ME_CUDA(ctx, cudaFuncSetAttribute(mme_flat_kernel<R, E16, U2, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ME_CUDA(ctx, cudaFuncSetAttribute(mme_flat_kernel<R, E16, U2, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  // fine-grained grid (~2 queries per thread): 256 CTAs/SM beat 64 and 1024 on C3 (chosen on B200, not re-measured on H100)
  const int blocks = (int)std::min<long long>((qe - qb + kFlatThreads - 1) / kFlatThreads, (long long)ctx->sm_count * 256);
  if (c.lat.sparse)
    mme_flat_kernel<R, E16, U2, 1><<<blocks, kFlatThreads, smem, ctx->stream>>>(c.d_sorted, c.d_rel, qb, qe, index_of(c), C, c.d_entropy, acc);
  else
    mme_flat_kernel<R, E16, U2, 0><<<blocks, kFlatThreads, smem, ctx->stream>>>(c.d_sorted, c.d_rel, qb, qe, index_of(c), C, c.d_entropy, acc);
  ME_LAUNCH_CHECK(ctx);
  trace_kernel(ctx, (c.lat.sparse ? ME_KBIT_MME_FLAT1_SPARSE : ME_KBIT_MME_FLAT1_DENSE) + R - 1);
  return ME_OK;
}

// MME accumulators -> the context's fp64 block (me_eval_mme_accum*)
__global__ void pack_mme_kernel(const MmeAcc *__restrict__ a, double *__restrict__ sum3, double *__restrict__ max2) {
  if (threadIdx.x != 0) return;
  sum3[0] = (double)a->n_query; sum3[1] = (double)a->n_valid; sum3[2] = a->sum;
  max2[0] = dec_ordered(a->max_enc);
  max2[1] = -dec_ordered(a->min_enc);
}

__global__ void unsort_f64_kernel(const P4 *__restrict__ S, long long n, const double *__restrict__ src,
                                  double *__restrict__ dst) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long o = orig_of(__double_as_longlong(__ldg(reinterpret_cast<const double *>(S + i) + 3)));
    dst[o] = src[i];
  }
}

// The lattice of a radius sweep (MME, local consistency) of cloud `which`: *solo = lay the cloud out on a lattice of its own
// with h = r/2, else on the shared lattice.  The caller lays it out: build_grid(ctx, which, *solo ? 0.5 * radius : 0.0).
// On a remembered plan the box is not measured ahead of the build: the decision is taken on the remembered box and the
// build checks it; if the box was another, the decision is taken again on the measured one.
int radius_lattice(me_ctx *ctx, int which, double radius, bool *solo) {
  Cloud &c = ctx->cloud[which];
  ME_TRY(wait_upload(ctx, which));
  const bool remembered = speculate_bbox(ctx, which);
  if (!remembered) ME_TRY(compute_bbox(ctx, which));
  *solo = false;
  if (!getenv("ME_MME_SHARED_LATTICE")) {
    const double h_now = (c.grid_valid && !c.grid_solo) ? c.lat.h : (ctx->nn_cell_size > 0 ? ctx->nn_cell_size : density_edge(c));
    *solo = radius / h_now > 3.0 + 1e-9;
    if (!*solo && !(c.grid_valid && !c.grid_solo)) {      // the estimate may be refined downwards by the build
      ME_TRY(build_grid(ctx, which));
      // a wrong remembered box: the decision the measured box gives (the shared lattice it was laid out on is then
      // replaced by the solo build, as after any MME sweep on a solo lattice)
      if (remembered && c.bbox_missed && radius / (ctx->nn_cell_size > 0 ? ctx->nn_cell_size : density_edge(c)) > 3.0 + 1e-9) *solo = true;
      else *solo = radius / c.lat.h > 3.0 + 1e-9;
    }
  }
  if (c.bbox_spec) {      // decided without a build that checks the box: measure it and decide again
    c.bbox_valid = false;
    ME_TRY(compute_bbox(ctx, which));
    return radius_lattice(ctx, which, radius, solo);
  }
  return ME_OK;
}

int run_mme(me_ctx *ctx, int which, double radius, int min_neighbors) {
  Cloud &c = ctx->cloud[which];
  if (c.n <= 0) return fail(ctx, ME_ERR_EMPTY, "cloud is empty");
  if (!(radius > 0)) return fail(ctx, ME_ERR_INVALID, "nn_radius must be > 0");
  // Lattice for this radius.  The shared lattice is tuned for the 1-NN sweeps (~2 points per occupied cell); when the
  // radius spans more than 3 of its cells (dense surfaces: 1 cm spacing, r = 0.1 m -> 7 cells; or r = 1.0 m), most of
  // the (2R+1)^2 rows of a neighbourhood are empty and enumerating them dominates.  The cloud is then laid out on a
  // lattice of its own with h = r/2 (rings = 2) for this sweep; the next NN / voxel stage lays it out again.
  bool solo = false;
  ME_TRY(radius_lattice(ctx, which, radius, &solo));
  ME_TRY(build_grid(ctx, which, solo ? 0.5 * radius : 0.0));
  if (c.grid_solo) trace_kernel(ctx, ME_KBIT_MME_SOLO);
  StageTimer timer(ctx, which == ME_CLOUD_EST ? 4 : 5);
  long long qb, qe;
  ME_TRY(query_shard(ctx, which, &qb, &qe));     // contiguous, cell-aligned range of the cell-sorted order
  ME_TRY(ensure(ctx, (void **)&c.d_entropy, &c.cap_entropy, c.n, sizeof(double)));
  MmeAcc *acc = (MmeAcc *)ctx->d_scratch;
  mme_init_kernel<<<1, 1, 0, ctx->stream>>>(acc);
  ME_LAUNCH_CHECK(ctx);
  if (ctx->world > 1) ME_CUDA(ctx, cudaMemsetAsync(c.d_entropy, 0, (size_t)c.n * sizeof(double), ctx->stream));
  // a neighbour sits at most ceil(r/h) cells away; the -1e-9 keeps r = k*h (exactly) at k rings
  const double rings_f = std::max(1.0, std::ceil(radius / c.lat.h - 1e-9));
  if (rings_f > 1.0e6) return fail(ctx, ME_ERR_RANGE, "nn_radius spans too many lattice cells");
  const int rings = (int)rings_f;
  if (c.slab && rings > ctx->slab_halo)      // only with ME_MME_SHARED_LATTICE: the shared lattice keeps radius <= 3 cells
    return fail(ctx, ME_ERR_RANGE, "nn_radius spans more lattice cells than the halo of the slab layout");
  const double rc = radius / c.lat.h;
  const float rc2 = (float)(rc * rc * (1.0 + 1e-5) + 1e-4);   // row pruning is conservative; the point test decides
  if (qe > qb) {
    // the flat kernel packs run lengths into 24 bits and x indices into an fp32 mantissa
    const bool flat = rings <= kMaxPlaneRings && c.lat.dims[0] < (1 << 24) &&
                      (2 * rings + 1) * c.max_cell_count < (1 << 24) && !getenv("ME_MME_WALK");
    if (flat) {
      MmeConst C;
      C.h = (float)c.lat.h; C.inv_h = (float)(1.0 / c.lat.h);
      C.rc2 = rc2;
      C.r2 = radius * radius;
      // fp32 screening error: |offset error| <= E per axis (plus the fp64 rounding of the cell origins), so
      // |d2_fp32 - d2| <= 2 sqrt(3) E d + 3 E^2 + 4 * 2^-24 d2; the band is several times that at d = r
      double maxabs = 0;
      for (int a = 0; a < 3; ++a) maxabs = std::max(maxabs, std::max(std::fabs(c.bbox_min[a]), std::fabs(c.bbox_max[a])));
      // per axis: two fp32 representations (2 x 3e-8 h), their difference (3e-8 h), fl32(h) times up to R+1 cells and the
      // FMA rounding (3e-8 h (2R + 3)) -> 3e-8 h (2R + 6); taken with a 3.3x margin
      const double E = 1e-7 * (2.0 * rings + 6.0) * c.lat.h + 4e-15 * maxabs;
      const double band = 8.0 * radius * E + 12.0 * E * E + 1e-6 * C.r2;
      C.r2_lo = (float)((C.r2 - band) * (1.0 - 1e-7));
      C.r2_hi = (float)((C.r2 + band) * (1.0 + 1e-7));
      C.min_neighbors = min_neighbors;
      C.dimx = c.lat.dims[0]; C.dimy = c.lat.dims[1]; C.dimz = c.lat.dims[2];
      C.own = owned_of(c);
      C.E2 = E * E;
      {      // rho' = rho + 3 rho^2 at 0.5 |ln(1 - rho')| = tau, then rho = 2 sqrt(3) s + 3 s^2 solved for s
        const double rho_p = -std::expm1(-2.0 * kFp64FinishNats);
        const double rho = (std::sqrt(1.0 + 12.0 * rho_p) - 1.0) / 6.0;
        const double s = (std::sqrt(12.0 + 12.0 * rho) - 2.0 * std::sqrt(3.0)) / 6.0;
        C.s2_max = s * s;
      }
      ME_TRY(ensure(ctx, (void **)&c.d_fp64_list, &c.cap_fp64_list, qe - qb, sizeof(uint32_t)));
      C.fp64_list = c.d_fp64_list;
      // default: the run-table walk; ME_MME_KERNEL=rows selects the warp-synchronous row walk with deferred accumulation
      // (6.2 ms against 5.3 ms for C3's sweep on one H100: half of its issue slots idle while the longest run of a row
      // finishes)
      const char *kv = getenv("ME_MME_KERNEL");
      const bool use_flat = !(kv && !strcmp(kv, "rows"));
      if (rings <= 3 && !use_flat) {
        if (rings == 1) ME_TRY(launch_rows<1>(ctx, c, qb, qe, C, acc));
        else if (rings == 2) ME_TRY(launch_rows<2>(ctx, c, qb, qe, C, acc));
        else ME_TRY(launch_rows<3>(ctx, c, qb, qe, C, acc));
      }
      else if (rings == 1) ME_TRY(launch_flat<1>(ctx, c, qb, qe, C, acc));
      else if (rings == 2) ME_TRY(launch_flat<2>(ctx, c, qb, qe, C, acc));
      else if (rings == 3) ME_TRY(launch_flat<3>(ctx, c, qb, qe, C, acc));
      else ME_TRY(launch_plane(ctx, c, qb, qe, C, rings, acc));
      // the listed queries (thin surfaces: certificate above kFp64FinishNats) again with fp64 offsets
      mme_fp64_finish_kernel<<<ctx->sm_count * 4, kThreads, 0, ctx->stream>>>(c.d_sorted, c.d_fp64_list, index_of(c), c.lat,
                                                                             radius * radius, rc2, rings, min_neighbors,
                                                                             c.d_entropy, acc, ctx->d_trace);
      ME_LAUNCH_CHECK(ctx);
      if (getenv("ME_DEBUG_MME")) {
        unsigned long long nf = 0;
        ME_CUDA(ctx, cudaMemcpyAsync(&nf, &acc->n_fp64, sizeof(nf), cudaMemcpyDeviceToHost, ctx->stream));
        ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        fprintf(stderr, "[mapeval] mme: rank %d cloud %d: %llu of %lld queries finished in fp64\n", ctx->rank, which, nf, qe - qb);
      }
    } else {
      const int blocks = (int)std::min<long long>((qe - qb + kThreads - 1) / kThreads, (long long)ctx->sm_count * 64);
      mme_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.d_sorted, qb, qe, index_of(c), c.lat, radius * radius, rc2, rings,
                                                      min_neighbors, owned_of(c), c.d_entropy, acc);
      ME_LAUNCH_CHECK(ctx);
      trace_kernel(ctx, ME_KBIT_MME_GENERIC);
    }
  }
  pack_mme_kernel<<<1, 32, 0, ctx->stream>>>(acc, ctx->d_block + kBlkMmeSum + 3 * which, ctx->d_block + kBlkMax + 2 * which);
  ME_LAUNCH_CHECK(ctx);
  c.entropy_valid = true;
  c.entropy_caller_valid = false;
  if (c.grid_solo) {      // the solo lattice (and with it the sorted order of d_entropy) does not survive the next build
    ME_TRY(ensure(ctx, (void **)&c.d_entropy_caller, &c.cap_entropy_caller, c.n, sizeof(double)));
    const int blocks = (int)std::min<long long>((c.n + 255) / 256, (long long)ctx->sm_count * 16);
    unsort_f64_kernel<<<blocks, 256, 0, ctx->stream>>>(c.d_sorted, c.ns, c.d_entropy, c.d_entropy_caller);
    ME_LAUNCH_CHECK(ctx);
    c.entropy_caller_valid = true;
  }
  return ME_OK;
}

int unsort_entropy(me_ctx *ctx, int which, double *h_entropy) {
  Cloud &c = ctx->cloud[which];
  if (c.entropy_caller_valid) {
    ME_CUDA(ctx, cudaMemcpyAsync(h_entropy, c.d_entropy_caller, (size_t)c.n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return ME_OK;
  }
  if (!c.entropy_valid) return fail(ctx, ME_ERR_INVALID, "me_get_entropies before me_eval_mme");
  ME_TRY(ensure_work(ctx, (size_t)c.n * sizeof(double)));
  double *dst = (double *)ctx->d_work;
  int blocks = (int)std::min<long long>((c.n + 255) / 256, (long long)ctx->sm_count * 16);
  ME_CUDA(ctx, cudaMemsetAsync(dst, 0, (size_t)c.n * sizeof(double), ctx->stream));      // slab mode: only this rank's points are written
  unsort_f64_kernel<<<blocks, 256, 0, ctx->stream>>>(c.d_sorted, c.ns, c.d_entropy, dst);
  ME_LAUNCH_CHECK(ctx);
  ME_CUDA(ctx, cudaMemcpyAsync(h_entropy, dst, (size_t)c.n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return ME_OK;
}

}  // namespace me

// mom.cu — the mutually orthogonal metric without a ground truth (me_mom_*, DESIGN §3.16): per point MME's radius
// neighbourhood, its plane variance v, middle eigenvalue and unit normal; the planar points' normals histogrammed on a cube
// map; three orthogonal axes picked from the reduced histogram on the host (me_mom_axes); per axis the family of planar
// points whose normal lies within the angle, its count, sum of v and exact median of v.
//
//   mom_sweep_kernel   walk_global per query as consistency_walk_kernel, finished by plane_eig (plane.cuh), so v equals
//                      me_get_consistency_points' bit for bit; writes v, lambda2, n and a flag byte in caller order and
//                      histograms bin(n), bin(-n) and three counts into a shared uint32 table, merged with integer atomics
//   mom_fold_kernel    one warp per chunk of kRegionChunk caller-order points: the family of every planar point (into its
//                      flag byte), the chunk's count and sum of v per family through a fixed shuffle tree
//   mom_merge_kernel   one warp: lane l adds the chunks l, l + 32, ... in order, then a fixed shuffle tree
//   mom_keys_kernel    the v keys of this rank's family members, family by family, and the histogram of their top digit
// The later digits are the distance quantiles' passes (radix.cuh, RadixSel): one SUM all-reduce per pass.  No floating-point
// atomics: two calls give the same bits as long as the cloud is not laid out again in between.
#include "common.cuh"
#include "plane.cuh"
#include "radix.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace me {

static constexpr int kThreads = 256;
static constexpr int kWalkThreads = 128;
static constexpr int kM = ME_MOM_CELLS_PER_EDGE, kBins = ME_MOM_BINS;
static constexpr int kCntQuery = kBins, kCntPv = kBins + 1, kCntPlanar = kBins + 2, kSweepBins = kBins + 3;
static constexpr int kFold = 6;                                    // n_j, then sum v_j
static constexpr int kSelBins = 3 * kMomSlots * kQuantBins;        // [family][slot][digit], after the fold in the block
static_assert(kFold + kSelBins == ME_MOM_BLOCK && kSweepBins <= ME_MOM_BLOCK, "ME_MOM_BLOCK layout");
enum : uint8_t { kEvaluated = 1, kPvValid = 2, kPlanar = 4 };      // family j + 1 in bits 3..4

struct MomOut {              // caller order
  double *v, *l2, *n;
  uint8_t *flag;
};

// the cube-map bin of a unit vector (DESIGN §3.16): face axis a = argmax |n_a| (lowest on a tie), sign s, the other two
// components over |n_a| cut into M cells each
__device__ __forceinline__ int mom_bin(double x, double y, double z) {
  const double ax = fabs(x), ay = fabs(y), az = fabs(z);
  int a = 0;
  double m = ax;
  if (ay > m) { a = 1; m = ay; }
  if (az > m) { a = 2; m = az; }
  const double na = a == 0 ? x : (a == 1 ? y : z);
  const double nb = a == 0 ? y : x, nc = a == 2 ? y : z;
  const double u = __ddiv_rn(nb, m), w = __ddiv_rn(nc, m);
  const int i = min(kM - 1, (int)floor(__dmul_rn(__dadd_rn(u, 1.0), 0.5 * kM)));
  const int j = min(kM - 1, (int)floor(__dmul_rn(__dadd_rn(w, 1.0), 0.5 * kM)));
  return ((2 * a + (na < 0.0 ? 1 : 0)) * kM + i) * kM + j;
}

__global__ void __launch_bounds__(kWalkThreads)
mom_sweep_kernel(const P4 *__restrict__ S, long long q_begin, long long q_end, CellIndex I, Lattice L, double r2, float rc2,
                 int rings, int min_neighbors, double planarity, MomOut O, unsigned long long *__restrict__ hist) {
  __shared__ unsigned int s_hist[kSweepBins];
  for (int t = threadIdx.x; t < kSweepBins; t += kWalkThreads) s_hist[t] = 0;
  __syncthreads();
  const long long stride = (long long)gridDim.x * kWalkThreads;
  for (long long base = q_begin + (long long)blockIdx.x * kWalkThreads; base < q_end; base += stride) {   // warp-uniform bound
    const long long i = base + threadIdx.x;
    int c_q = -1, c_pv = -1, c_pl = -1, b_pos = -1, b_neg = -1;
    if (i < q_end) {
      const P4 q = load_p4(S + i);
      Moments m;
      m.init();
      walk_global(q, S, I, L, r2, rc2, rings, m);
      PlaneEig P;
      plane_eig(m, min_neighbors, P);
      const long long o = orig_of(q.idx);
      double l2 = NAN, nx = NAN, ny = NAN, nz = NAN;
      uint8_t flag = kEvaluated;
      c_q = kCntQuery;
      if (P.ok) {
        // selects rather than indexing by P.lo keep the arrays in registers
        const double w1 = P.lo == 0 ? P.w[1] : P.w[0], w2 = P.lo == 2 ? P.w[1] : P.w[2];   // the other two, ascending axis
        l2 = w1 <= w2 ? w1 : w2;
        nx = P.lo == 0 ? P.vec[0] : (P.lo == 1 ? P.vec[1] : P.vec[2]);
        ny = P.lo == 0 ? P.vec[3] : (P.lo == 1 ? P.vec[4] : P.vec[5]);
        nz = P.lo == 0 ? P.vec[6] : (P.lo == 1 ? P.vec[7] : P.vec[8]);
        const double nrm = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(nx, nx), __dmul_rn(ny, ny)), __dmul_rn(nz, nz)));
        nx = __ddiv_rn(nx, nrm); ny = __ddiv_rn(ny, nrm); nz = __ddiv_rn(nz, nrm);
        const double ax = fabs(nx), ay = fabs(ny), az = fabs(nz);
        const double big = ay > ax ? (az > ay ? nz : ny) : (az > ax ? nz : nx);
        if (big < 0.0) { nx = -nx; ny = -ny; nz = -nz; }
        if (isfinite(P.v)) {
          flag |= kPvValid;
          c_pv = kCntPv;
          if (l2 > 0.0 && P.v <= __dmul_rn(planarity, l2)) {
            flag |= kPlanar;
            c_pl = kCntPlanar;
            b_pos = mom_bin(nx, ny, nz);
            b_neg = mom_bin(-nx, -ny, -nz);
          }
        }
      }
      O.v[o] = P.v;
      O.l2[o] = l2;
      O.n[3 * o] = nx; O.n[3 * o + 1] = ny; O.n[3 * o + 2] = nz;
      O.flag[o] = flag;
    }
    quant_count(s_hist, c_q);
    quant_count(s_hist, c_pv);
    quant_count(s_hist, c_pl);
    quant_count(s_hist, b_pos);
    quant_count(s_hist, b_neg);
  }
  quant_flush(s_hist, kSweepBins, hist);
}

__global__ void __launch_bounds__(kThreads) mom_init_kernel(long long n, MomOut O) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    O.v[i] = NAN;
    O.l2[i] = NAN;
    O.n[3 * i] = NAN; O.n[3 * i + 1] = NAN; O.n[3 * i + 2] = NAN;
    O.flag[i] = 0;
  }
}

struct MomAxes {
  double a[9];
  double cos_a;
};

// family of a planar normal: the first axis j with |n . a_j| >= cos(angle), the dot product as ((x x') + y y') + z z'; -1 none
__device__ __forceinline__ int mom_family(const MomAxes &A, double x, double y, double z) {
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const double d = __dadd_rn(__dadd_rn(__dmul_rn(x, A.a[3 * j]), __dmul_rn(y, A.a[3 * j + 1])), __dmul_rn(z, A.a[3 * j + 2]));
    if (fabs(d) >= A.cos_a) return j;
  }
  return -1;
}

__global__ void __launch_bounds__(kThreads)
mom_fold_kernel(long long n, const double *__restrict__ v, const double *__restrict__ nrm, uint8_t *__restrict__ flag, MomAxes A,
                double *__restrict__ part) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (kThreads / 32);
  const long long n_chunks = (n + kRegionChunk - 1) / kRegionChunk;
  for (long long c = blockIdx.x * (long long)(kThreads / 32) + (threadIdx.x >> 5); c < n_chunks; c += warps) {
    const long long j0 = c * kRegionChunk, j1 = min(n, j0 + kRegionChunk);
    double o[kFold] = {0, 0, 0, 0, 0, 0};
    for (long long i = j0 + lane; i < j1; i += 32) {
      uint8_t f = flag[i] & 7;
      if (f & kPlanar) {
        const int j = mom_family(A, __ldg(nrm + 3 * i), __ldg(nrm + 3 * i + 1), __ldg(nrm + 3 * i + 2));
        if (j >= 0) {
          f |= (uint8_t)((j + 1) << 3);
          const double vi = __ldg(v + i);
#pragma unroll
          for (int k = 0; k < 3; ++k)
            if (k == j) { o[k] += 1.0; o[3 + k] += vi; }
        }
      }
      flag[i] = f;
    }
#pragma unroll
    for (int k = 0; k < kFold; ++k) o[k] = warp_sum(o[k]);
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < kFold; ++k) part[c * kFold + k] = o[k];
    }
  }
}

// one warp: lane l adds the chunks l, l + 32, ... in order, then a fixed shuffle tree
__global__ void mom_merge_kernel(const double *__restrict__ part, long long n_chunks, double *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  double s[kFold] = {0, 0, 0, 0, 0, 0};
  for (long long c = lane; c < n_chunks; c += 32)
#pragma unroll
    for (int k = 0; k < kFold; ++k) s[k] += part[c * kFold + k];
#pragma unroll
  for (int k = 0; k < kFold; ++k) s[k] = warp_sum(s[k]);
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < kFold; ++k) out[k] = s[k];
}

struct KeyDst {
  unsigned long long *keys;
  long long off[3];            // first position of family j in keys
  unsigned long long *ctr;     // 3 counters, zeroed
};

// the key of every family member at off[j] + (its place among family j's members, in atomic order — the selection counts
// keys, so their order does not matter), and the histogram of the top digit into hist[j * kMomSlots * 256 + digit]
__global__ void __launch_bounds__(kQuantThreads)
mom_keys_kernel(long long n, const double *__restrict__ v, const uint8_t *__restrict__ flag, KeyDst D, unsigned long long *__restrict__ hist) {
  __shared__ unsigned int s_hist[kSelBins];
  for (int t = threadIdx.x; t < kSelBins; t += kQuantThreads) s_hist[t] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * kQuantThreads;
  for (long long base = (long long)blockIdx.x * kQuantThreads; base < n; base += stride) {   // warp-uniform bound
    const long long i = base + threadIdx.x;
    const int j = i < n ? (int)(__ldg(flag + i) >> 3) - 1 : -1;
    unsigned long long key = 0;
    if (j >= 0) key = quant_key(__ldg(v + i));
    const unsigned int peers = __match_any_sync(0xffffffffu, j);
    const int leader = __ffs(peers) - 1;
    unsigned long long first = 0;
    if (j >= 0 && lane == leader) first = atomicAdd(D.ctr + j, (unsigned long long)__popc(peers));
    first = __shfl_sync(0xffffffffu, first, leader);
    const long long off = j == 0 ? D.off[0] : (j == 1 ? D.off[1] : D.off[2]);
    if (j >= 0) D.keys[off + (long long)first + __popc(peers & ((1u << lane) - 1u))] = key;
    quant_count(s_hist, j >= 0 ? j * kMomSlots * kQuantBins + (int)(key >> 56) : -1);
  }
  quant_flush(s_hist, kSelBins, hist);
}

__global__ void mom_to_block_kernel(const unsigned long long *__restrict__ hist, int n, double *__restrict__ blk) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) blk[t] = (double)hist[t];
}

// ---------------------------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------------------------
void mom_free(me_ctx *ctx) {
  MomRun &R = ctx->mom;
  if (R.d_hist) { cudaFree(R.d_hist); R.d_hist = nullptr; R.d_blk = nullptr; R.d_pfx = nullptr; R.d_ctr = nullptr; R.d_fold = nullptr; }
  if (R.d_part) { cudaFree(R.d_part); R.d_part = nullptr; R.cap_part = 0; }
  if (R.d_keys) { cudaFree(R.d_keys); R.d_keys = nullptr; R.cap_keys = 0; }
  for (int w = 0; w < 2; ++w) {
    if (R.d_v[w]) { cudaFree(R.d_v[w]); R.d_v[w] = nullptr; R.cap_v[w] = 0; }
    if (R.d_l2[w]) { cudaFree(R.d_l2[w]); R.d_l2[w] = nullptr; R.cap_l2[w] = 0; }
    if (R.d_n[w]) { cudaFree(R.d_n[w]); R.d_n[w] = nullptr; R.cap_n[w] = 0; }
    if (R.d_flag[w]) { cudaFree(R.d_flag[w]); R.d_flag[w] = nullptr; R.cap_flag[w] = 0; }
    R.pts_valid[w] = false;
  }
  R.open = false;
}

// the centre of bin b of the cube map: the face point, normalised
static void bin_centre(int b, int M, double c[3]) {
  const int j = b % M, i = (b / M) % M, face = b / (M * M), a = face / 2;
  const int ob = a == 0 ? 1 : 0, oc = a == 2 ? 1 : 2;
  double p[3];
  p[a] = (face & 1) ? -1.0 : 1.0;
  p[ob] = -1.0 + (double)(2 * i + 1) / (double)M;
  p[oc] = -1.0 + (double)(2 * j + 1) / (double)M;
  const double nrm = std::sqrt((p[0] * p[0] + p[1] * p[1]) + p[2] * p[2]);
  for (int k = 0; k < 3; ++k) c[k] = p[k] / nrm;
}
static double dot3(const double *x, const double *y) { return (x[0] * y[0] + x[1] * y[1]) + x[2] * y[2]; }

}  // namespace me

using namespace me;

int me_mom_axes(const int64_t *hist, int32_t M, double angle_deg, double *axes, int32_t *status) {
  if (!hist || !axes || !status || M < 1 || M > 1024 || !(angle_deg > 0.0 && angle_deg <= 30.0)) return ME_ERR_INVALID;
  const int B = 6 * M * M;
  for (int b = 0; b < B; ++b)
    if (hist[b] < 0) return ME_ERR_INVALID;
  for (int k = 0; k < 9; ++k) axes[k] = NAN;
  const double rad = angle_deg * M_PI / 180.0, cos_a = std::cos(rad), sin_a = std::sin(rad);
  std::vector<double> C((size_t)B * 3);
  for (int b = 0; b < B; ++b) bin_centre(b, M, &C[(size_t)3 * b]);
  std::vector<int64_t> S(B, 0);
  int64_t total = 0;
  for (int b = 0; b < B; ++b) {
    total += hist[b];
    int64_t s = 0;
    for (int b2 = 0; b2 < B; ++b2)
      if (hist[b2] && dot3(&C[(size_t)3 * b], &C[(size_t)3 * b2]) >= cos_a) s += hist[b2];
    S[b] = s;
  }
  if (total == 0) { *status = ME_MOM_NO_PLANAR; return ME_OK; }
  int b1 = 0;
  for (int b = 1; b < B; ++b)
    if (S[b] > S[b1]) b1 = b;
  const double *a1 = &C[(size_t)3 * b1];
  int b2 = -1;
  for (int b = 0; b < B; ++b)
    if (S[b] > 0 && std::fabs(dot3(&C[(size_t)3 * b], a1)) <= sin_a && (b2 < 0 || S[b] > S[b2])) b2 = b;
  for (int k = 0; k < 3; ++k) axes[k] = a1[k];
  if (b2 < 0) { *status = ME_MOM_NO_SECOND_AXIS; return ME_OK; }
  const double *c2 = &C[(size_t)3 * b2];
  const double t = dot3(c2, a1);
  double d[3];
  for (int k = 0; k < 3; ++k) d[k] = c2[k] - t * a1[k];
  const double nrm = std::sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]);
  double *a2 = axes + 3, *a3 = axes + 6;
  for (int k = 0; k < 3; ++k) a2[k] = d[k] / nrm;
  a3[0] = a1[1] * a2[2] - a1[2] * a2[1];
  a3[1] = a1[2] * a2[0] - a1[0] * a2[2];
  a3[2] = a1[0] * a2[1] - a1[1] * a2[0];
  *status = ME_MOM_OK;
  return ME_OK;
}

namespace me {

static int mom_to_block(me_ctx *ctx, int n) {
  MomRun &R = ctx->mom;
  mom_to_block_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(R.d_hist, n, R.d_blk);
  ME_LAUNCH_CHECK(ctx);
  return ME_OK;
}

int mom_begin(me_ctx *ctx, int which, double radius, int min_neighbors, const me_mom_params *p) {
  MomRun &R = ctx->mom;
  R.open = false;
  R.ended = false;
  Cloud &c = ctx->cloud[which];
  if (c.n <= 0) return fail(ctx, ME_ERR_EMPTY, "me_mom_begin: the cloud is empty");
  if (ctx->icp.open) return fail(ctx, ME_ERR_INVALID, "me_mom_begin while a registration is open (me_icp_end first)");
  if (ctx->drift.open) return fail(ctx, ME_ERR_INVALID, "me_mom_begin while a drift loop is open (me_drift_end first)");
  if (ctx->slab_request && ctx->world > 1)
    return fail(ctx, ME_ERR_INVALID, "me_mom_begin needs the replicated layout; the slab layout is requested (me_set_layout "
                                     "ME_LAYOUT_REPLICATED first)");
  R.pts_valid[which] = false;
  if (!R.d_hist) {      // the integer counts, the block, the slot prefixes, the key counters and this rank's fold in one allocation
    const size_t bytes = (size_t)ME_MOM_BLOCK * (sizeof(unsigned long long) + sizeof(double)) + sizeof(R.sel.slot_pfx) +
                         3 * sizeof(unsigned long long) + kFold * sizeof(double);
    ME_CUDA(ctx, cudaMalloc((void **)&R.d_hist, bytes));
    R.d_blk = (double *)(R.d_hist + ME_MOM_BLOCK);
    R.d_pfx = (unsigned long long *)(R.d_blk + ME_MOM_BLOCK);
    R.d_ctr = R.d_pfx + 3 * kMomSlots;
    R.d_fold = (double *)(R.d_ctr + 3);
  }
  RadiusSweep RS;
  ME_TRY(radius_sweep_layout(ctx, which, radius, "me_mom_begin", &RS));
  ME_TRY(ensure(ctx, (void **)&R.d_v[which], &R.cap_v[which], c.n, sizeof(double)));
  ME_TRY(ensure(ctx, (void **)&R.d_l2[which], &R.cap_l2[which], c.n, sizeof(double)));
  ME_TRY(ensure(ctx, (void **)&R.d_n[which], &R.cap_n[which], 3 * c.n, sizeof(double)));
  ME_TRY(ensure(ctx, (void **)&R.d_flag[which], &R.cap_flag[which], c.n, sizeof(uint8_t)));
  const MomOut O{R.d_v[which], R.d_l2[which], R.d_n[which], R.d_flag[which]};
  {
    const int blocks = (int)std::min<long long>((c.n + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
    mom_init_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.n, O);
    ME_LAUNCH_CHECK(ctx);
  }
  ME_CUDA(ctx, cudaMemsetAsync(R.d_hist, 0, (size_t)ME_MOM_BLOCK * sizeof(unsigned long long), ctx->stream));
  if (RS.qe > RS.qb) {
    const int blocks = (int)std::min<long long>((RS.qe - RS.qb + kWalkThreads - 1) / kWalkThreads, (long long)ctx->sm_count * 64);
    mom_sweep_kernel<<<blocks, kWalkThreads, 0, ctx->stream>>>(c.d_sorted, RS.qb, RS.qe, index_of(c), c.lat, radius * radius, RS.rc2,
                                                               RS.rings, min_neighbors, p->planarity, O, R.d_hist);
    ME_LAUNCH_CHECK(ctx);
  }
  ME_TRY(mom_to_block(ctx, ME_MOM_BLOCK));
  R.which = which;
  R.radius = radius;
  R.min_neighbors = min_neighbors;
  R.angle_deg = p->angle_deg;
  R.planarity = p->planarity;
  R.min_family = p->min_family;
  R.cos_a = std::cos(p->angle_deg * M_PI / 180.0);
  R.rings = RS.rings;
  R.solo = c.grid_solo ? 1 : 0;
  R.kb = RS.qb;
  R.ke = RS.qe;
  R.stage = 0;
  R.done = false;
  R.status = ME_MOM_OK;
  R.n_query = R.n_pv = R.n_planar = 0;
  for (int j = 0; j < 3; ++j) { R.n_fam[j] = 0; R.sum_v[j] = 0.0; R.sel.set_targets(j, 0, nullptr, 0); }
  R.sel.pass = 0;
  for (int k = 0; k < 9; ++k) R.axes[k] = NAN;
  R.pts_valid[which] = true;
  R.pts_gen[which] = ctx->cloud_gen;
  R.gen = ctx->cloud_gen;
  R.open = true;
  return ME_OK;
}

static int mom_ready(me_ctx *ctx, const char *who) {
  MomRun &R = ctx->mom;
  if (!R.open) return fail(ctx, ME_ERR_INVALID, std::string(who) + " without an open MOM call (me_mom_begin first)");
  if (R.gen != ctx->cloud_gen) {
    R.open = false;
    return fail(ctx, ME_ERR_INVALID, std::string(who) + ": the clouds changed after me_mom_begin; the call is void "
                                     "(run me_mom_begin again)");
  }
  return ME_OK;
}

int mom_block(me_ctx *ctx, double **device_block, int32_t *n) {
  ME_TRY(mom_ready(ctx, "me_mom_block"));
  *device_block = ctx->mom.d_blk;
  *n = ME_MOM_BLOCK;
  return ME_OK;
}

// the selection pass R.sel.pass >= 1 of every family with a slot
static int mom_select_launch(me_ctx *ctx) {
  MomRun &R = ctx->mom;
  ME_CUDA(ctx, cudaMemsetAsync(R.d_hist, 0, (size_t)ME_MOM_BLOCK * sizeof(unsigned long long), ctx->stream));
  ME_CUDA(ctx, cudaMemcpyAsync(R.d_pfx, R.sel.slot_pfx, sizeof(R.sel.slot_pfx), cudaMemcpyHostToDevice, ctx->stream));
  long long off = 0;
  for (int j = 0; j < 3; ++j) {
    const long long nk = R.keys_local[j];
    if (nk > 0 && R.sel.n_slots[j] > 0)
      ME_TRY(quant_hist_launch(ctx, R.d_keys + off, nk, R.sel.pass, R.d_pfx + j * kMomSlots, R.sel.n_slots[j],
                               R.d_hist + kFold + (size_t)j * kMomSlots * kQuantBins));
    off += nk;
  }
  return mom_to_block(ctx, ME_MOM_BLOCK);
}

// stage 0 -> 1: the axes from the reduced histogram, the families and their fold, the keys and their top digit
static int mom_families(me_ctx *ctx, const double *blk, int32_t *done) {
  MomRun &R = ctx->mom;
  const Cloud &c = ctx->cloud[R.which];
  R.n_query = (long long)blk[kCntQuery];
  R.n_pv = (long long)blk[kCntPv];
  R.n_planar = (long long)blk[kCntPlanar];
  std::vector<int64_t> h(kBins);
  for (int b = 0; b < kBins; ++b) h[b] = (int64_t)blk[b];
  int32_t st = 0;
  if (me_mom_axes(h.data(), kM, R.angle_deg, R.axes, &st) != ME_OK) return fail(ctx, ME_ERR_INVALID, "me_mom_step: me_mom_axes failed");
  R.status = st;
  if (st != ME_MOM_OK) { R.done = true; *done = 1; return ME_OK; }
  MomAxes A;
  for (int k = 0; k < 9; ++k) A.a[k] = R.axes[k];
  A.cos_a = R.cos_a;
  const long long n_chunks = (c.n + kRegionChunk - 1) / kRegionChunk;
  ME_TRY(ensure(ctx, (void **)&R.d_part, &R.cap_part, kFold * std::max<long long>(1, n_chunks), sizeof(double)));
  const int fblocks = (int)std::min<long long>((n_chunks + kThreads / 32 - 1) / (kThreads / 32), (long long)ctx->sm_count * 32);
  mom_fold_kernel<<<fblocks, kThreads, 0, ctx->stream>>>(c.n, R.d_v[R.which], R.d_n[R.which], R.d_flag[R.which], A, R.d_part);
  ME_LAUNCH_CHECK(ctx);
  mom_merge_kernel<<<1, 32, 0, ctx->stream>>>(R.d_part, n_chunks, R.d_fold);
  ME_LAUNCH_CHECK(ctx);
  double fold[kFold];
  ME_CUDA(ctx, cudaMemcpyAsync(fold, R.d_fold, sizeof(fold), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  KeyDst D;
  long long total = 0;
  for (int j = 0; j < 3; ++j) {
    R.keys_local[j] = (long long)fold[j];
    D.off[j] = total;
    total += R.keys_local[j];
  }
  ME_TRY(ensure(ctx, (void **)&R.d_keys, &R.cap_keys, std::max<long long>(1, total), sizeof(unsigned long long)));
  D.keys = R.d_keys;
  D.ctr = R.d_ctr;
  ME_CUDA(ctx, cudaMemsetAsync(R.d_ctr, 0, 3 * sizeof(unsigned long long), ctx->stream));
  ME_CUDA(ctx, cudaMemsetAsync(R.d_hist, 0, (size_t)ME_MOM_BLOCK * sizeof(unsigned long long), ctx->stream));
  if (total > 0) {
    const int grid = (int)std::min<long long>((c.n + kQuantThreads - 1) / kQuantThreads, (long long)ctx->sm_count * 4);
    mom_keys_kernel<<<grid, kQuantThreads, 0, ctx->stream>>>(c.n, R.d_v[R.which], R.d_flag[R.which], D, R.d_hist + kFold);
    ME_LAUNCH_CHECK(ctx);
  }
  ME_TRY(mom_to_block(ctx, ME_MOM_BLOCK));
  ME_CUDA(ctx, cudaMemcpyAsync(R.d_blk, R.d_fold, sizeof(fold), cudaMemcpyDeviceToDevice, ctx->stream));
  R.stage = 1;
  *done = 0;
  return ME_OK;
}

int mom_step(me_ctx *ctx, int32_t *done) {
  ME_TRY(mom_ready(ctx, "me_mom_step"));
  MomRun &R = ctx->mom;
  if (R.done) { *done = 1; return ME_OK; }
  R.h_blk.resize(ME_MOM_BLOCK);
  ME_CUDA(ctx, cudaMemcpyAsync(R.h_blk.data(), R.d_blk, (size_t)ME_MOM_BLOCK * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const double *blk = R.h_blk.data();
  if (R.stage == 0) return mom_families(ctx, blk, done);
  if (R.stage == 1) {      // the reduced fold: the family sizes and sums, then the median's target ranks
    const double half = 0.5;
    for (int j = 0; j < 3; ++j) {
      R.n_fam[j] = (long long)blk[j];
      R.sum_v[j] = blk[3 + j];
      R.sel.set_targets(j, R.n_fam[j], &half, 1);
    }
    R.sel.pass = 0;
  }
  for (int j = 0; j < 3; ++j)
    if (R.sel.n_slots[j] && !R.sel.take_digits(j, blk + kFold + (size_t)j * kMomSlots * kQuantBins)) {
      R.open = false;
      return fail(ctx, ME_ERR_INVALID, "me_mom_step: the block does not hold a rank the selection needs (a block not SUM-reduced "
                                       "over all ranks, or of another call)");
    }
  if (R.sel.pass == kQuantPasses - 1 || (!R.sel.n_slots[0] && !R.sel.n_slots[1] && !R.sel.n_slots[2])) {
    R.done = true;
    *done = 1;
    return ME_OK;
  }
  R.sel.next_pass();
  ++R.stage;
  ME_TRY(mom_select_launch(ctx));
  *done = 0;
  return ME_OK;
}

int mom_end(me_ctx *ctx, me_mom_result *out) {
  ME_TRY(mom_ready(ctx, "me_mom_end"));
  MomRun &R = ctx->mom;
  if (!R.done) return fail(ctx, ME_ERR_INVALID, "me_mom_end before the last me_mom_step (*done = 1)");
  R.open = false;
  std::memset(out, 0, sizeof(*out));
  out->radius = R.radius;
  out->angle_deg = R.angle_deg;
  out->planarity = R.planarity;
  out->min_family = R.min_family;
  out->min_neighbors = R.min_neighbors;
  out->kernel = ME_CONSISTENCY_WALK;
  out->rings = R.rings;
  out->solo = R.solo;
  out->n_points = ctx->cloud[R.which].n;
  out->n_query = R.n_query;
  out->n_pv = R.n_pv;
  out->n_planar = R.n_planar;
  for (int k = 0; k < 9; ++k) out->axis[k] = R.axes[k];
  int status = R.status;
  for (int j = 0; j < 3; ++j) {
    const long long n = status == ME_MOM_OK ? R.n_fam[j] : 0;
    out->n[j] = n;
    out->mean[j] = n > 0 ? R.sum_v[j] / (double)n : NAN;
    if (n > 0) {
      long long kk;
      double g;
      quantile_rank(n, 0.5, &kk, &g);
      out->median[j] = quantile_lerp(R.sel.value(j, kk), R.sel.value(j, std::min<long long>(kk + 1, n - 1)), g);
    } else {
      out->median[j] = NAN;
    }
  }
  if (status == ME_MOM_OK)
    for (int j = 0; j < 3; ++j)
      if (out->n[j] < R.min_family) status = ME_MOM_SMALL_FAMILY;
  out->status = status;
  out->mom = status == ME_MOM_OK ? (out->median[0] + out->median[1]) + out->median[2] : NAN;
  R.ended = true;
  return ME_OK;
}

int mom_points(me_ctx *ctx, int which, double *v, double *lambda2, double *normal, int8_t *family) {
  const MomRun &R = ctx->mom;
  if (!R.pts_valid[which]) return fail(ctx, ME_ERR_INVALID, "me_get_mom_points before me_mom_begin on this cloud");
  if (R.pts_gen[which] != ctx->cloud_gen)
    return fail(ctx, ME_ERR_INVALID, "me_get_mom_points: the clouds changed after me_mom_begin (run it again)");
  const long long n = ctx->cloud[which].n;
  std::vector<uint8_t> flag;
  if (v) ME_CUDA(ctx, cudaMemcpyAsync(v, R.d_v[which], (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  if (lambda2) ME_CUDA(ctx, cudaMemcpyAsync(lambda2, R.d_l2[which], (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  if (normal) ME_CUDA(ctx, cudaMemcpyAsync(normal, R.d_n[which], (size_t)n * 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  if (family) {
    flag.resize((size_t)n);
    ME_CUDA(ctx, cudaMemcpyAsync(flag.data(), R.d_flag[which], (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  }
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (family)
    for (long long i = 0; i < n; ++i) family[i] = (int8_t)((flag[i] >> 3) - 1);
  return ME_OK;
}

}  // namespace me

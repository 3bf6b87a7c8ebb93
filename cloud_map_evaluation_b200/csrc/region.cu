// region.cu — AC / COM / CD / F1 / IoU per region (me_nn_region_*): the records of the last NN sweep split by the region
// floor(x / s) of their query point, without a new sweep (DESIGN §3.12).
//
// Occupied list, from the whole clouds in caller order (d_xyz is whole on every rank in both layouts), so that it is the
// same on every rank:
//   region_key_kernel    one packed key per point of est ++ gt; per axis the index minus the lowest index of the two
//                        bounding boxes, in as many bits as the extent needs
//   radix_sort_pairs     (sort.cu) STABLE: a region's est points precede its gt points, each in caller order
//   region_head_kernel   + exclusive_scan_inplace: the region of every sorted point and the region count
//   region_list_kernel   first sorted position, est/gt split and key of every region
//   region_count_kernel  n_est / n_gt per region, and the chunks of kRegionChunk query points per region and direction
//   region_rid_kernel    (region_ids) the region of every caller index of one cloud: the drift loop, the MOM breakdown
// Record fold, per evaluated direction, over this rank's records:
//   record_pos_kernel    caller index -> position of its record in the cell-sorted cloud (~0u: not laid out here)
//   region_fold_kernel   one warp per chunk: lane l walks the chunk's points l, l + 32, ..., keeps the pairs with
//                        kept_record / accum_sq (records.cuh), then a fixed shuffle tree; lane 0 writes the chunk's values
//   region_merge_kernel  one thread per region adds its chunks in chunk order into the block
// The summation order depends only on the occupied list and on the records this rank holds: two calls give the same bits.
// No floating-point atomics.
#include "common.cuh"
#include "records.cuh"
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstring>

namespace me {

static constexpr int kThreads = 256;
static constexpr double kAxisLimit = 1048576.0;                            // |index| < 2^20 per axis
static constexpr int kSumF = ME_REGION_SUM_FIELDS, kMaxF = ME_REGION_MAX_FIELDS;
static constexpr int kPart = kSumF + kMaxF;                                // values per chunk: the SUM fields, then the MAX fields

struct RegionGeom {
  double s;
  long long lo[3];     // lowest index per axis
  int bits[3];         // key bits per axis
};

__global__ void __launch_bounds__(kThreads) region_key_kernel(const double *__restrict__ est, long long n_est,
                                                              const double *__restrict__ gt, long long n, RegionGeom g,
                                                              unsigned long long *__restrict__ key, uint32_t *__restrict__ val) {
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < n; j += (long long)gridDim.x * blockDim.x) {
    const double *p = j < n_est ? est + 3 * j : gt + 3 * (j - n_est);
    unsigned long long k = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const long long r = (long long)floor(__ddiv_rn(__ldg(p + a), g.s)) - g.lo[a];
      k = (k << g.bits[a]) | (unsigned long long)r;
    }
    key[j] = k;
    val[j] = (uint32_t)j;
  }
}

// head[i] = 1 where a new region starts in the sorted key sequence (head[n] = 0: after the scan it holds the region count)
__global__ void __launch_bounds__(kThreads) region_head_kernel(const unsigned long long *__restrict__ key, long long n,
                                                               uint32_t *__restrict__ head) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i <= n; i += (long long)gridDim.x * blockDim.x)
    head[i] = (i < n && (i == 0 || key[i] != key[i - 1])) ? 1u : 0u;
}

// pos = the scanned heads: sorted point i lies in region pos[i + 1] - 1 and starts it when pos[i + 1] != pos[i].
// seg[r] = first sorted position of region r (seg[R] = n), est_end[r] = one past its last est point (0: none; zero-filled),
// rkey[r] = its key
__global__ void __launch_bounds__(kThreads) region_list_kernel(const unsigned long long *__restrict__ key, const uint32_t *__restrict__ val,
                                                               const uint32_t *__restrict__ pos, long long n, long long n_est,
                                                               uint32_t *__restrict__ seg, uint32_t *__restrict__ est_end,
                                                               unsigned long long *__restrict__ rkey) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t r = pos[i + 1] - 1;
    if (pos[i + 1] != pos[i]) { seg[r] = (uint32_t)i; rkey[r] = key[i]; }
    const bool last = i + 1 == n || pos[i + 2] != pos[i + 1];
    if (val[i] < n_est && (last || val[i + 1] >= n_est)) est_end[r] = (uint32_t)(i + 1);
    if (i == n - 1) seg[r + 1] = (uint32_t)n;
  }
}

// rid[val[j] - id0] = the region of sorted point j, for the caller ids [id0, id0 + n_c) of one cloud (the other cloud's ids
// wrap to >= n_c)
__global__ void __launch_bounds__(kThreads) region_rid_kernel(const uint32_t *__restrict__ val, const uint32_t *__restrict__ pos,
                                                              long long n, uint32_t id0, uint32_t n_c, uint32_t *__restrict__ rid) {
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < n; j += (long long)gridDim.x * blockDim.x) {
    const uint32_t i = __ldg(val + j) - id0;
    if (i < n_c) rid[i] = __ldg(pos + j + 1) - 1;
  }
}

// cnt[r] / cnt[R + r] = n_est / n_gt of region r; chunks[q * (R + 1) + r] = its chunks of direction q (0 at r = R, so that
// the exclusive scan leaves the total there)
__global__ void __launch_bounds__(kThreads) region_count_kernel(const uint32_t *__restrict__ seg, const uint32_t *__restrict__ est_end,
                                                                long long R, uint32_t *__restrict__ cnt, uint32_t *__restrict__ chunks) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r <= R; r += (long long)gridDim.x * blockDim.x) {
    if (r == R) { chunks[R] = 0; chunks[2 * R + 1] = 0; continue; }
    const uint32_t ne = est_end[r] ? est_end[r] - seg[r] : 0u, ng = seg[r + 1] - seg[r] - ne;
    cnt[r] = ne;
    cnt[R + r] = ng;
    chunks[r] = (ne + kRegionChunk - 1) / kRegionChunk;
    chunks[R + 1 + r] = (ng + kRegionChunk - 1) / kRegionChunk;
  }
}

__global__ void __launch_bounds__(kThreads) record_pos_kernel(const P4 *__restrict__ Q, long long ns, uint32_t *__restrict__ pos_of) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < ns; i += (long long)gridDim.x * blockDim.x)
    pos_of[orig_of(__double_as_longlong(__ldg(reinterpret_cast<const double *>(Q + i) + 3)))] = (uint32_t)i;
}

// accum_sq's accumulator for one lane: the kept pairs, the five levels as nn_stats_kernel forms them, the largest d
struct RegionAcc {
  unsigned int n_corr, n_inl[5];
  double sum_d[5], sum_d2[5], max_d;
  __device__ void clear() {
    n_corr = 0; max_d = 0.0;
#pragma unroll
    for (int k = 0; k < 5; ++k) { n_inl[k] = 0; sum_d[k] = 0.0; sum_d2[k] = 0.0; }
  }
  __device__ __forceinline__ void pair(double nd, double) { ++n_corr; max_d = fmax(max_d, nd); }
  __device__ __forceinline__ void inlier(int k, double nd, double sq) { sum_d[k] += nd; sum_d2[k] += sq; n_inl[k]++; }
};

struct FoldSrc {
  const uint32_t *val;         // sorted caller ids, est ++ gt
  const uint32_t *seg, *est_end;
  const uint32_t *chunk_off;   // this direction's scanned chunk counts, R + 1
  const uint32_t *pos_of;      // the query cloud's caller index -> record position
  long long R, n_chunks;
  uint32_t id0;                // caller id of the query cloud's point 0 (0 or n_est)
  int q;
  long long nb, ne;            // the range of the evaluated queries (n_query, the NN distances)
};

__global__ void __launch_bounds__(kThreads) region_fold_kernel(FoldSrc F, CurveSrc S, NNConst C, double *__restrict__ part) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (kThreads / 32);
  for (long long c = blockIdx.x * (long long)(kThreads / 32) + (threadIdx.x >> 5); c < F.n_chunks; c += warps) {
    long long lo = 0, hi = F.R;          // the region of chunk c: chunk_off[lo] <= c < chunk_off[lo + 1]
    while (hi - lo > 1) {
      const long long mid = (lo + hi) >> 1;
      if ((long long)__ldg(F.chunk_off + mid) <= c) lo = mid; else hi = mid;
    }
    const long long seg0 = __ldg(F.seg + lo), ee = __ldg(F.est_end + lo);
    const long long ne_r = ee ? ee - seg0 : 0;
    const long long a = F.q == 0 ? seg0 : seg0 + ne_r, b = F.q == 0 ? seg0 + ne_r : (long long)__ldg(F.seg + lo + 1);
    const long long j0 = a + (c - (long long)__ldg(F.chunk_off + lo)) * kRegionChunk, j1 = min(b, j0 + kRegionChunk);
    unsigned int n_query = 0, ub = 0;
    double sum_nn = 0.0, max_nn = 0.0;
    RegionAcc A;
    A.clear();
    for (long long j = j0 + lane; j < j1; j += 32) {
      const uint32_t i = __ldg(F.pos_of + (__ldg(F.val + j) - F.id0));
      if (i == 0xffffffffu) continue;
      if (i >= F.nb && i < F.ne) {       // the queries nn_stats_kernel counts and the terms of its full-CD sum
        const int32_t nn = __ldg(S.nn_idx + i);
        n_query += nn != -2;
        if (nn >= 0 && C.want_full_cd) {
          const double dn = __dsqrt_rn(__ldg(S.nn_d2 + i));
          sum_nn += dn;
          max_nn = fmax(max_nn, dn);
        }
      }
      double sq;
      if (i >= S.b && i < S.e && kept_record(S, C, i, sq, ub)) accum_sq(sq, C, A);
    }
    double v[kPart];
    v[0] = (double)n_query;
    v[1] = (double)A.n_corr;
#pragma unroll
    for (int k = 0; k < 5; ++k) { v[2 + k] = (double)A.n_inl[k]; v[7 + k] = A.sum_d[k]; v[12 + k] = A.sum_d2[k]; }
    v[17] = sum_nn;
    v[18] = A.max_d;
    v[19] = max_nn;
#pragma unroll
    for (int f = 0; f < kSumF; ++f) v[f] = warp_sum(v[f]);
#pragma unroll
    for (int f = kSumF; f < kPart; ++f) v[f] = warp_max(v[f]);
    if (lane == 0) {
#pragma unroll
      for (int f = 0; f < kPart; ++f) part[c * kPart + f] = v[f];
    }
  }
}

// region r of direction q: its chunks added in chunk order -> blk[(r * 2 + q) * kSumF ..], the maxima -> the MAX part
__global__ void __launch_bounds__(kThreads) region_merge_kernel(const double *__restrict__ part, const uint32_t *__restrict__ chunk_off,
                                                                long long R, int q, double *__restrict__ blk) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < R; r += (long long)gridDim.x * blockDim.x) {
    double v[kPart];
#pragma unroll
    for (int f = 0; f < kPart; ++f) v[f] = 0.0;
    for (long long c = chunk_off[r]; c < (long long)chunk_off[r + 1]; ++c) {
#pragma unroll
      for (int f = 0; f < kSumF; ++f) v[f] += part[c * kPart + f];
#pragma unroll
      for (int f = kSumF; f < kPart; ++f) v[f] = fmax(v[f], part[c * kPart + f]);
    }
#pragma unroll
    for (int f = 0; f < kSumF; ++f) blk[(r * 2 + q) * kSumF + f] = v[f];
#pragma unroll
    for (int f = 0; f < kMaxF; ++f) blk[2 * kSumF * R + (r * 2 + q) * kMaxF + f] = v[kSumF + f];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host driver
// ---------------------------------------------------------------------------------------------------------------
void nn_region_free(me_ctx *ctx) {
  RegionRun &G = ctx->region;
  if (G.d_blk) { cudaFree(G.d_blk); G.d_blk = nullptr; G.cap_blk = 0; }
  if (G.d_part) { cudaFree(G.d_part); G.d_part = nullptr; G.cap_part = 0; }
  G.open = false;
}

// every point with a coordinate in [mn, mx] along one axis has |floor(x / s)| < 2^20 (x / s is monotone in x)
static bool axis_fits(double mn, double mx, double s) {
  return std::fabs(std::floor(mn / s)) < kAxisLimit && std::fabs(std::floor(mx / s)) < kAxisLimit;
}
// the smallest s for which axis_fits holds
static double smallest_fit(double mn, double mx) {
  double s = std::max(std::max(mx, 0.0) / kAxisLimit, std::max(-mn, 0.0) / (kAxisLimit - 1.0));
  if (!(s > 0.0)) s = DBL_MIN;
  for (int it = 0; it < 64 && !axis_fits(mn, mx, s); ++it) s = std::nextafter(s, INFINITY);
  for (int it = 0; it < 64 && axis_fits(mn, mx, std::nextafter(s, 0.0)); ++it) s = std::nextafter(s, 0.0);
  return s;
}

static std::string num(double x) {
  char b[64];
  std::snprintf(b, sizeof(b), "%.17g", x);
  return b;
}

// The occupied list of est ++ gt (with_gt = false: of est alone), in d_work.  The size checks and their messages are the
// same for every caller; `who` names the call in them.
int list_regions(me_ctx *ctx, const char *who, double s, bool with_gt, RegionList *L) {
  const Cloud &E = ctx->cloud[ME_CLOUD_EST], &T = ctx->cloud[ME_CLOUD_GT];
  ME_TRY(compute_bbox(ctx, ME_CLOUD_EST));
  if (with_gt) ME_TRY(compute_bbox(ctx, ME_CLOUD_GT));
  RegionGeom g;
  g.s = s;
  double mn[3], mx[3];
  for (int a = 0; a < 3; ++a) {
    mn[a] = with_gt ? std::min(E.bbox_min[a], T.bbox_min[a]) : E.bbox_min[a];
    mx[a] = with_gt ? std::max(E.bbox_max[a], T.bbox_max[a]) : E.bbox_max[a];
  }
  for (int a = 0; a < 3; ++a) {
    if (axis_fits(mn[a], mx[a], s)) continue;
    double s_fit = 0.0;      // the smallest size that fits along every axis
    for (int b = 0; b < 3; ++b) s_fit = std::max(s_fit, smallest_fit(mn[b], mx[b]));
    return fail(ctx, ME_ERR_INVALID, std::string(who) + ": region_size " + num(s) + " puts region indices along " +
                                         "xyz"[a] + " outside |index| < 2^20 (" + num(std::floor(mn[a] / s)) + " .. " +
                                         num(std::floor(mx[a] / s)) + "); the smallest region_size that fits is " + num(s_fit));
  }
  int key_bits = 0;
  for (int a = 0; a < 3; ++a) {
    g.lo[a] = (long long)std::floor(mn[a] / s);
    const long long span = (long long)std::floor(mx[a] / s) - g.lo[a] + 1;
    int b = 0;
    while ((1ll << b) < span) ++b;
    g.bits[a] = b;
    key_bits += b;
  }
  const long long n_est = E.n, n_gt = with_gt ? T.n : 0, n = n_est + n_gt;
  if (n >= 0xffffffffll) return fail(ctx, ME_ERR_RANGE, std::string(who) + ": more than 2^32 - 1 points in the two clouds");
  const long long r_cap = std::min<long long>(n, ME_REGION_MAX_REGIONS);
  auto align = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t o_key0 = 0, o_key1 = o_key0 + align((size_t)n * 8), o_val0 = o_key1 + align((size_t)n * 8),
               o_val1 = o_val0 + align((size_t)n * 4), o_pos = o_val1 + align((size_t)n * 4),
               o_pos_of = o_pos + align((size_t)(n + 1) * 4), o_seg = o_pos_of + align((size_t)std::max(n_est, n_gt) * 4),
               o_ee = o_seg + align((size_t)(r_cap + 1) * 4), o_rkey = o_ee + align((size_t)r_cap * 4),
               o_cnt = o_rkey + align((size_t)r_cap * 8), o_chunks = o_cnt + align((size_t)2 * r_cap * 4),
               total = o_chunks + align((size_t)2 * (r_cap + 1) * 4);
  ME_TRY(ensure_work(ctx, total));
  char *base = (char *)ctx->d_work;
  unsigned long long *key0 = (unsigned long long *)(base + o_key0), *key1 = (unsigned long long *)(base + o_key1);
  uint32_t *val0 = (uint32_t *)(base + o_val0), *val1 = (uint32_t *)(base + o_val1), *pos = (uint32_t *)(base + o_pos);
  uint32_t *seg = (uint32_t *)(base + o_seg), *est_end = (uint32_t *)(base + o_ee);
  unsigned long long *rkey = (unsigned long long *)(base + o_rkey);
  uint32_t *cnt = (uint32_t *)(base + o_cnt), *chunks = (uint32_t *)(base + o_chunks);
  const int blocks = (int)std::min<long long>((n + kThreads) / kThreads, (long long)ctx->sm_count * 16);

  region_key_kernel<<<blocks, kThreads, 0, ctx->stream>>>(E.d_xyz, n_est, T.d_xyz, n, g, key0, val0);
  ME_LAUNCH_CHECK(ctx);
  unsigned long long *ks = nullptr;
  uint32_t *vs = nullptr;
  ME_TRY(radix_sort_pairs(ctx, key0, val0, key1, val1, n, key_bits, &ks, &vs));      // stable
  region_head_kernel<<<blocks, kThreads, 0, ctx->stream>>>(ks, n, pos);
  ME_LAUNCH_CHECK(ctx);
  ME_TRY(exclusive_scan_inplace(ctx, pos, n + 1));
  uint32_t *h = (uint32_t *)ctx->h_pinned;
  ME_CUDA(ctx, cudaMemcpyAsync(h, pos + n, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const long long R = (long long)h[0];
  if (R > ME_REGION_MAX_REGIONS)
    return fail(ctx, ME_ERR_INVALID, std::string(who) + ": " + std::to_string(R) + " occupied regions at region_size " + num(s) +
                                         ", at most ME_REGION_MAX_REGIONS = 2^21; choose a larger region_size");
  ME_CUDA(ctx, cudaMemsetAsync(est_end, 0, (size_t)R * 4, ctx->stream));
  region_list_kernel<<<blocks, kThreads, 0, ctx->stream>>>(ks, vs, pos, n, n_est, seg, est_end, rkey);
  ME_LAUNCH_CHECK(ctx);
  const int rblocks = (int)std::min<long long>((R + kThreads) / kThreads, (long long)ctx->sm_count * 16);
  region_count_kernel<<<rblocks, kThreads, 0, ctx->stream>>>(seg, est_end, R, cnt, chunks);
  ME_LAUNCH_CHECK(ctx);
  ME_TRY(exclusive_scan_inplace(ctx, chunks, R + 1));
  ME_TRY(exclusive_scan_inplace(ctx, chunks + R + 1, R + 1));
  std::vector<unsigned long long> hkey((size_t)R);
  std::vector<uint32_t> hcnt((size_t)2 * R);
  ME_CUDA(ctx, cudaMemcpyAsync(hkey.data(), rkey, (size_t)R * 8, cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaMemcpyAsync(hcnt.data(), cnt, (size_t)2 * R * 4, cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaMemcpyAsync(&L->n_chunks[0], chunks + R, 4, cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaMemcpyAsync(&L->n_chunks[1], chunks + 2 * R + 1, 4, cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  L->R = R;
  L->n = n;
  L->val = vs; L->pos = pos; L->pos_of = (uint32_t *)(base + o_pos_of); L->seg = seg; L->est_end = est_end; L->chunks = chunks;
  L->index.resize((size_t)3 * R);
  L->n_est.resize((size_t)R);
  L->n_gt.resize((size_t)R);
  for (long long r = 0; r < R; ++r) {
    unsigned long long k = hkey[r];
    for (int a = 2; a >= 0; --a) {
      L->index[3 * r + a] = g.lo[a] + (long long)(g.bits[a] ? k & ((1ull << g.bits[a]) - 1) : 0ull);
      k = g.bits[a] ? k >> g.bits[a] : k;
    }
    L->n_est[r] = hcnt[r];
    L->n_gt[r] = hcnt[R + r];
  }
  return ME_OK;
}

int region_ids(me_ctx *ctx, const RegionList &L, int which, uint32_t *rid) {
  const uint32_t id0 = which == ME_CLOUD_EST ? 0u : (uint32_t)ctx->cloud[ME_CLOUD_EST].n;
  const int blocks = (int)std::min<long long>((L.n + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
  region_rid_kernel<<<std::max(blocks, 1), kThreads, 0, ctx->stream>>>(L.val, L.pos, L.n, id0, (uint32_t)ctx->cloud[which].n, rid);
  ME_LAUNCH_CHECK(ctx);
  return ME_OK;
}

// pos_of[caller index] = position of the point's record in the cloud's cell-sorted layout (~0u: not laid out here)
int record_positions(me_ctx *ctx, int which, uint32_t *pos_of) {
  const Cloud &Qc = ctx->cloud[which];
  ME_CUDA(ctx, cudaMemsetAsync(pos_of, 0xff, (size_t)Qc.n * 4, ctx->stream));
  const int qblocks = (int)std::min<long long>((Qc.ns + kThreads - 1) / kThreads + 1, (long long)ctx->sm_count * 16);
  record_pos_kernel<<<qblocks, kThreads, 0, ctx->stream>>>(Qc.d_sorted, Qc.ns, pos_of);
  ME_LAUNCH_CHECK(ctx);
  return ME_OK;
}

int nn_region_begin(me_ctx *ctx, double s, int64_t *n_regions) {
  RegionRun &G = ctx->region;
  G.open = false;
  *n_regions = 0;
  ME_TRY(nn_records_fresh(ctx, "me_nn_region*"));
  RegionList RL;
  ME_TRY(list_regions(ctx, "me_nn_region_begin", s, true, &RL));
  const long long R = RL.R, n_est = ctx->cloud[ME_CLOUD_EST].n;
  const uint32_t *n_chunks = RL.n_chunks;
  uint32_t *vs = RL.val, *pos_of = RL.pos_of, *seg = RL.seg, *est_end = RL.est_end, *chunks = RL.chunks;
  const int rblocks = (int)std::min<long long>((R + kThreads) / kThreads, (long long)ctx->sm_count * 16);

  // the block: zero for a direction the last me_eval_nn* did not evaluate
  const long long n_blk = (long long)(2 * kSumF + 2 * kMaxF) * R;
  ME_TRY(ensure(ctx, (void **)&G.d_blk, &G.cap_blk, n_blk, sizeof(double)));
  ME_CUDA(ctx, cudaMemsetAsync(G.d_blk, 0, (size_t)n_blk * sizeof(double), ctx->stream));
  G.s = s;
  G.n = R;
  G.index = std::move(RL.index);
  G.n_est = std::move(RL.n_est);
  G.n_gt = std::move(RL.n_gt);

  // the record fold, per evaluated direction
  const me_nn_params *p = &ctx->curve_p;
  const int dirs = p->directions ? p->directions : 3;
  ME_TRY(ensure(ctx, (void **)&G.d_part, &G.cap_part, (long long)kPart * std::max<long long>(1, std::max(n_chunks[0], n_chunks[1])),
                sizeof(double)));
  for (int q = 0; q < 2; ++q) {
    if (!(dirs & (1 << q)) || n_chunks[q] == 0) continue;
    const Cloud &Qc = ctx->cloud[q];
    ME_TRY(record_positions(ctx, q, pos_of));
    NNConst C{};
    for (int k = 0; k < 5; ++k) C.tau[k] = p->tau[k];
    set_cutoff(C, p);
    C.want_full_cd = p->want_full_cd ? 1 : 0;
    FoldSrc F;
    F.val = vs; F.seg = seg; F.est_end = est_end; F.chunk_off = chunks + q * (R + 1); F.pos_of = pos_of;
    F.R = R; F.n_chunks = n_chunks[q]; F.id0 = q == 0 ? 0u : (uint32_t)n_est; F.q = q;
    F.nb = Qc.nn_b; F.ne = Qc.nn_e;
    const int fblocks = (int)std::min<long long>((n_chunks[q] + kThreads / 32 - 1) / (kThreads / 32), (long long)ctx->sm_count * 32);
    region_fold_kernel<<<fblocks, kThreads, 0, ctx->stream>>>(F, record_src(ctx, q), C, G.d_part);
    ME_LAUNCH_CHECK(ctx);
    region_merge_kernel<<<rblocks, kThreads, 0, ctx->stream>>>(G.d_part, F.chunk_off, R, q, G.d_blk);
    ME_LAUNCH_CHECK(ctx);
  }
  G.gen = ctx->cloud_gen;
  G.open = true;
  *n_regions = R;
  return ME_OK;
}

static int region_ready(me_ctx *ctx, const char *who) {
  RegionRun &G = ctx->region;
  if (!G.open) return fail(ctx, ME_ERR_INVALID, std::string(who) + " without an open region table (me_nn_region_begin first)");
  if (G.gen != ctx->cloud_gen) {
    G.open = false;
    return fail(ctx, ME_ERR_INVALID, std::string(who) + ": the clouds changed after me_nn_region_begin; the table is void "
                                     "(run me_eval_nn* and me_nn_region_begin again)");
  }
  return ME_OK;
}

int nn_region_block(me_ctx *ctx, double **device_block, int32_t *n_sum, int32_t *n_max) {
  ME_TRY(region_ready(ctx, "me_nn_region_block"));
  const RegionRun &G = ctx->region;
  *device_block = G.d_blk;
  *n_sum = (int32_t)(2 * kSumF * G.n);
  *n_max = (int32_t)(2 * kMaxF * G.n);
  return ME_OK;
}

int nn_region_end(me_ctx *ctx, me_region_row *rows, int64_t capacity) {
  ME_TRY(region_ready(ctx, "me_nn_region_end"));
  RegionRun &G = ctx->region;
  if (capacity < G.n)
    return fail(ctx, ME_ERR_INVALID, "me_nn_region_end: capacity " + std::to_string(capacity) + " < " + std::to_string(G.n) + " regions");
  G.open = false;
  std::vector<double> h((size_t)(2 * kSumF + 2 * kMaxF) * G.n);
  ME_CUDA(ctx, cudaMemcpyAsync(h.data(), G.d_blk, h.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (me_region_finalize(G.n, G.s, G.index.data(), G.n_est.data(), G.n_gt.data(), h.data(), rows) != ME_OK)
    return fail(ctx, ME_ERR_INVALID, "me_region_finalize failed");
  return ME_OK;
}

}  // namespace me

// grid.cu — lays a cloud out once into a dense, voxel-aligned, cell-sorted lattice in HBM.
//
//   bbox reduce -> lattice choice (host) -> cell histogram -> in-place exclusive scan -> scatter (counting sort)
//
// The layout replaces the reference's per-call KD-tree builds (open3d::geometry::KDTreeFlann::SetGeometry,
// map_eval.cpp:1213-1214,1226-1227,1401-1402,1448-1449,1550-1551,1618-1619) and its std::unordered_map voxel
// hashing (voxel_calculator.cpp:21-56).  All kernels here are HBM-streaming integer/byte work: coalesced loads,
// grids sized in multiples of the SM count, no tensor cores.
#include <cstdio>
#include "common.cuh"
#include <algorithm>
#include <climits>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace me {

static constexpr int kThreads = 256;

// ---------------------------------------------------------------------------------------------------------------
// bbox: min/max per axis + count of non-finite coordinates
// scratch layout (uint64): [0..2] min xyz (ordered encoding), [3..5] max xyz, [6] non-finite count
// ---------------------------------------------------------------------------------------------------------------
__global__ void bbox_init_kernel(unsigned long long *s) {
  int t = threadIdx.x;
  if (t < 3) s[t] = 0xffffffffffffffffull;
  else if (t < 6) s[t] = 0ull;
  else if (t == 6) s[t] = 0ull;
}

__global__ void __launch_bounds__(kThreads) bbox_kernel(const double *__restrict__ xyz, long long n, int lead,
                                                        unsigned long long *__restrict__ s) {
  double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  unsigned long long bad = 0;
  // the coordinates as 16-byte pairs (after `lead` = 0 or 1 leading scalars that make the rest 16-byte aligned):
  // thread t of a pass reads pair t = coordinates lead + 2t, lead + 2t + 1; the stride of a pass is a multiple of 3
  // pairs, so a thread always sees the same two axes
  const long long ncoord = 3 * n - lead, npairs = ncoord / 2;
  const long long stride = ((long long)gridDim.x * blockDim.x / 3) * 3;
  const long long t0 = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const int a0 = (int)((lead + 2 * t0) % 3), a1 = (a0 + 1) % 3;
  double lo0 = INFINITY, hi0 = -INFINITY, lo1 = INFINITY, hi1 = -INFINITY;
  if (t0 < stride) {
    const double2 *pairs = reinterpret_cast<const double2 *>(xyz + lead);
    for (long long t = t0; t < npairs; t += stride) {
      const double2 v = __ldg(pairs + t);
      if (isfinite(v.x)) { lo0 = fmin(lo0, v.x); hi0 = fmax(hi0, v.x); } else bad++;
      if (isfinite(v.y)) { lo1 = fmin(lo1, v.y); hi1 = fmax(hi1, v.y); } else bad++;
    }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (a0 == k) { mn[k] = fmin(mn[k], lo0); mx[k] = fmax(mx[k], hi0); }
    if (a1 == k) { mn[k] = fmin(mn[k], lo1); mx[k] = fmax(mx[k], hi1); }
  }
  if (t0 == 0) {      // the scalars the pairs do not cover: the leading one (x of point 0) and, if odd, the last one
    for (int e = 0; e < 2; ++e) {
      const long long ci = e == 0 ? 0 : lead + 2 * npairs;
      if ((e == 0 && lead == 0) || ci >= 3 * n) continue;
      const double v = __ldg(xyz + ci);
      const int k = (int)(ci % 3);
      if (isfinite(v)) {
#pragma unroll
        for (int kk = 0; kk < 3; ++kk) if (kk == k) { mn[kk] = fmin(mn[kk], v); mx[kk] = fmax(mx[kk], v); }
      } else bad++;
    }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) { mn[k] = warp_min(mn[k]); mx[k] = warp_max(mx[k]); }
  bad = (unsigned long long)warp_sum_ll((long long)bad);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (mn[k] <= mx[k]) {
        atomicMin(s + k, enc_ordered(mn[k]));
        atomicMax(s + 3 + k, enc_ordered(mx[k]));
      }
    }
    if (bad) atomicAdd(s + 6, bad);
  }
}

// kernels on the compute stream must not read a cloud before its H2D copy (on the copy stream) has landed
int wait_upload(me_ctx *ctx, int which) {
  Cloud &c = ctx->cloud[which];
  if (c.upload_pending) {
    ME_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, c.upload_done, 0));
    c.upload_pending = false;
  }
  return ME_OK;
}

int compute_bbox(me_ctx *ctx, int which) {
  Cloud &c = ctx->cloud[which];
  if (c.bbox_valid) return ME_OK;
  if (c.n <= 0) return fail(ctx, ME_ERR_EMPTY, "cloud is empty");
  ME_TRY(wait_upload(ctx, which));
  unsigned long long *s = (unsigned long long *)ctx->d_scratch;
  bbox_init_kernel<<<1, 32, 0, ctx->stream>>>(s);
  ME_LAUNCH_CHECK(ctx);
  int blocks = (int)std::min<long long>((3 * c.n / 2 + kThreads - 1) / kThreads + 1, (long long)ctx->sm_count * 16);
  const int lead = (int)(((uintptr_t)c.d_xyz >> 3) & 1);     // 8- but not 16-byte aligned device buffers
  bbox_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.d_xyz, c.n, lead, s);
  ME_LAUNCH_CHECK(ctx);
  unsigned long long *h = (unsigned long long *)ctx->h_pinned;
  ME_CUDA(ctx, cudaMemcpyAsync(h, s, 7 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (h[6] != 0)
    return fail(ctx, ME_ERR_RANGE, "cloud holds non-finite coordinates (the reference drops them at load, map_eval.cpp:6)");
  for (int k = 0; k < 3; ++k) { c.bbox_min[k] = dec_ordered(h[k]); c.bbox_max[k] = dec_ordered(h[3 + k]); }
  c.bbox_valid = true;
  c.bbox_spec = false;
  return ME_OK;
}

static bool slab_wanted(const me_ctx *ctx);

// A cloud handed over again (repeated passes over the same maps) most likely has the box of its last shared dense build:
// take that box, unmeasured, so that the build plans without a round trip to the host; the build's histogram measures
// the box on the way and build_grid checks it at its one synchronise.  Not for slab layouts (their builds synchronise
// more than once) or when the plan is not remembered.
int speculate_bbox(me_ctx *ctx, int which) {
  Cloud &c = ctx->cloud[which];
  if (c.bbox_valid || !c.last_box_valid || c.last_box_n != c.n || slab_wanted(ctx) || getenv("ME_NO_PLAN_CACHE")) return 0;
  c.bbox_missed = false;
  for (int k = 0; k < 3; ++k) { c.bbox_min[k] = c.last_bmin[k]; c.bbox_max[k] = c.last_bmax[k]; }
  c.bbox_valid = true;
  c.bbox_spec = true;
  return 1;
}

// ---------------------------------------------------------------------------------------------------------------
// dense build: cell histogram -> exclusive scan -> scatter -> fp32 screening copy.  Both point passes read the
// caller-order fp64 cloud through shared memory, one tile of kThreads points at a time: the block loads the tile's
// 3 * kThreads coordinates with consecutive 16-byte loads (8-byte loads if the cloud is only 8-byte aligned), so every
// load instruction is fully used, and each thread then takes its point from shared memory.  The histogram keeps the
// value its atomic returned, the point's rank in its cell; the scatter recomputes the cell from the coordinates and
// writes the point to off[cell] + rank with plain loads of the scanned table.  (The atomics in the histogram meet a
// count table that lives in L2; taking the slots with atomics in the scatter instead, against 320 MB of random record
// writes, made the scatter 1.2x slower on C3.)
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void stage_tile(const double *__restrict__ xyz, long long n, bool aligned16, long long p0,
                                           double *__restrict__ s) {
  const long long nd = 3 * (n - p0 < kThreads ? n - p0 : kThreads);      // coordinates in this tile
  const double *src = xyz + 3 * p0;
  if (aligned16 && nd == 3 * kThreads) {       // a tile starts 16-byte aligned: 3 * kThreads * 8 B is a multiple of 16
    const double2 *q = reinterpret_cast<const double2 *>(src);
    double2 *d = reinterpret_cast<double2 *>(s);
    for (int k = threadIdx.x; k < 3 * kThreads / 2; k += kThreads) d[k] = __ldg(q + k);
  } else {
    for (int k = threadIdx.x; k < nd; k += kThreads) s[k] = __ldg(src + k);
  }
}

// lattice cell of a point; points define the lattice, so the coordinates are in range by construction: clamp against
// surprises
__device__ __forceinline__ void point_cell(double x, double y, double z, const Lattice &L, int &ix, int &iy, int &iz) {
  long long cx = cell_coord(x, L, 0), cy = cell_coord(y, L, 1), cz = cell_coord(z, L, 2);
  ix = (int)(cx < 0 ? 0 : (cx >= L.dims[0] ? L.dims[0] - 1 : cx));
  iy = (int)(cy < 0 ? 0 : (cy >= L.dims[1] ? L.dims[1] - 1 : cy));
  iz = (int)(cz < 0 ? 0 : (cz >= L.dims[2] ? L.dims[2] - 1 : cz));
}

// BOX: the lattice was planned on a remembered box (speculate_bbox); the histogram also reduces the box of the points it
// stages into box[0..6] (bbox_kernel's layout and encoding: the same box, bit for bit).  Points outside the lattice are
// clamped to its faces by point_cell, so a wrong guess costs a rebuild, never a write out of bounds.
template <bool BOX>
__device__ __forceinline__ void cell_count(const double *__restrict__ xyz, long long n, const Lattice &L,
                                           uint32_t *__restrict__ count, uint32_t *__restrict__ rank,
                                           unsigned long long *__restrict__ box) {
  __shared__ __align__(16) double s[3 * kThreads];
  const bool aligned16 = ((uintptr_t)xyz & 15) == 0;
  double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  unsigned long long bad = 0;
  for (long long p0 = (long long)blockIdx.x * kThreads; p0 < n; p0 += (long long)gridDim.x * kThreads) {
    __syncthreads();
    stage_tile(xyz, n, aligned16, p0, s);
    __syncthreads();
    if (p0 + threadIdx.x < n) {
      const double x = s[3 * threadIdx.x], y = s[3 * threadIdx.x + 1], z = s[3 * threadIdx.x + 2];
      if (BOX) {
        const double v[3] = {x, y, z};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          if (isfinite(v[k])) { mn[k] = fmin(mn[k], v[k]); mx[k] = fmax(mx[k], v[k]); } else bad++;
        }
      }
      int ix, iy, iz;
      point_cell(x, y, z, L, ix, iy, iz);
      rank[p0 + threadIdx.x] = atomicAdd(count + ((long long)iz * L.dims[1] + iy) * (long long)L.dims[0] + ix, 1u);
    }
  }
  if (BOX) {      // warps -> the block's box in shared memory -> one set of global atomics per block
    __shared__ unsigned long long sbox[7];
    if (threadIdx.x < 7) sbox[threadIdx.x] = threadIdx.x < 3 ? 0xffffffffffffffffull : 0ull;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 3; ++k) { mn[k] = warp_min(mn[k]); mx[k] = warp_max(mx[k]); }
    bad = (unsigned long long)warp_sum_ll((long long)bad);
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        if (mn[k] <= mx[k]) {
          atomicMin(sbox + k, enc_ordered(mn[k]));
          atomicMax(sbox + 3 + k, enc_ordered(mx[k]));
        }
      }
      if (bad) atomicAdd(sbox + 6, bad);
    }
    __syncthreads();
    if (threadIdx.x < 3) atomicMin(box + threadIdx.x, sbox[threadIdx.x]);
    else if (threadIdx.x < 6) atomicMax(box + threadIdx.x, sbox[threadIdx.x]);
    else if (threadIdx.x == 6 && sbox[6]) atomicAdd(box + 6, sbox[6]);
  }
}

__global__ void __launch_bounds__(kThreads) cell_count_kernel(const double *__restrict__ xyz, long long n, Lattice L,
                                                              uint32_t *__restrict__ count, uint32_t *__restrict__ rank) {
  cell_count<false>(xyz, n, L, count, rank, nullptr);
}

// 5 blocks per SM, as cell_count_kernel gets (47 registers): the running box would otherwise take it to 63 and 4 blocks
__global__ void __launch_bounds__(kThreads, 5) cell_count_box_kernel(const double *__restrict__ xyz, long long n, Lattice L,
                                                                     uint32_t *__restrict__ count, uint32_t *__restrict__ rank,
                                                                     unsigned long long *__restrict__ box) {
  cell_count<true>(xyz, n, L, count, rank, box);
}

// ---------------------------------------------------------------------------------------------------------------
// in-place exclusive scan, single pass (decoupled look-back): every block scans its tile of kScanTile values, publishes
// the tile's sum, and takes its offset from the published sums / inclusive prefixes of the tiles before it.  Blocks start
// in blockIdx order, so a tile only ever waits on tiles that are running or done.  Optionally it also reduces the
// statistics of the values: stats[0] += number of non-zero values, stats[1] = max(stats[1], largest value).
// ---------------------------------------------------------------------------------------------------------------
static constexpr int kScanItems = 8;                       // per thread
static constexpr int kScanTile = kThreads * kScanItems;    // 2048 values per block
// tile status word: flag in the high 32 bits (0: nothing yet, 1: tile sum, 2: inclusive prefix), the value in the low 32
static constexpr unsigned long long kTileSum = 1ull << 32, kTilePrefix = 2ull << 32;

__global__ void __launch_bounds__(kThreads) scan_kernel(uint32_t *__restrict__ a, long long n,
                                                        unsigned long long *__restrict__ status,
                                                        unsigned long long *__restrict__ stats) {
  __shared__ uint32_t s[kScanTile + kScanTile / 32];      // padded: conflict-free in both the striped and blocked order
  __shared__ uint32_t ws[kThreads / 32];
  __shared__ uint32_t tile_off;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long tile = blockIdx.x, base = tile * kScanTile;
  // coalesced loads (a need not be 16-byte aligned), then every thread takes kScanItems consecutive values
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const int j = k * kThreads + threadIdx.x;
    s[j + (j >> 5)] = base + j < n ? a[base + j] : 0u;
  }
  __syncthreads();
  uint32_t v[kScanItems], sum = 0, occ = 0, mx = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const int j = threadIdx.x * kScanItems + k;
    v[k] = s[j + (j >> 5)];
    sum += v[k]; occ += v[k] != 0u; mx = max(mx, v[k]);
  }
  uint32_t inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
  if (lane == 31) ws[warp] = inc;
  if (stats) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { occ += __shfl_xor_sync(0xffffffffu, occ, o); mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
    if (lane == 0 && (occ || mx)) { atomicAdd(stats, (unsigned long long)occ); atomicMax(stats + 1, (unsigned long long)mx); }
  }
  __syncthreads();
  if (warp == 0) {
    uint32_t w = lane < kThreads / 32 ? ws[lane] : 0u, winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= o) winc += t; }
    if (lane < kThreads / 32) ws[lane] = winc - w;                       // exclusive prefix of the warp sums
    const uint32_t total = __shfl_sync(0xffffffffu, winc, 31);
    volatile unsigned long long *st = status;
    uint32_t off = 0;
    if (tile == 0) {
      if (lane == 0) st[0] = kTilePrefix | total;
    } else {
      if (lane == 0) st[tile] = kTileSum | total;
      // look back over windows of 32 predecessors (lane l: tile - 1 - l) until one holds an inclusive prefix
      for (long long w0 = tile - 1;; w0 -= 32) {
        const long long t = w0 - lane;
        unsigned long long x;
        do {
          x = kTilePrefix;      // before tile 0: an inclusive prefix of 0
          if (t >= 0) x = st[t];
        } while (__any_sync(0xffffffffu, (x >> 32) == 0ull));
        const unsigned pre = __ballot_sync(0xffffffffu, (x >> 32) == 2ull);
        const int stop = pre ? __ffs(pre) - 1 : 32;                    // nearest predecessor with its inclusive prefix
        uint32_t part = lane <= stop ? (uint32_t)x : 0u;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
        off += part;
        if (pre) break;
      }
      if (lane == 0) st[tile] = kTilePrefix | (off + total);
    }
    if (lane == 0) tile_off = off;
  }
  __syncthreads();
  uint32_t run = tile_off + ws[warp] + inc - sum;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const int j = threadIdx.x * kScanItems + k;
    s[j + (j >> 5)] = run;
    run += v[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const int j = k * kThreads + threadIdx.x;
    if (base + j < n) a[base + j] = s[j + (j >> 5)];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// scatter: point i of cell c goes to slot off[c] + rank[i]; off[] is the CSR offset array of the scan and stays as it is
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) scatter_kernel(const double *__restrict__ xyz, long long n, Lattice L,
                                                           const uint32_t *__restrict__ off, const uint32_t *__restrict__ rank,
                                                           P4 *__restrict__ sorted, int axis, int c_lo, int c_hi) {
  __shared__ __align__(16) double s[3 * kThreads];
  const bool aligned16 = ((uintptr_t)xyz & 15) == 0;
  for (long long p0 = (long long)blockIdx.x * kThreads; p0 < n; p0 += (long long)gridDim.x * kThreads) {
    __syncthreads();
    stage_tile(xyz, n, aligned16, p0, s);
    __syncthreads();
    const long long i = p0 + threadIdx.x;
    if (i >= n) continue;
    const double x = s[3 * threadIdx.x], y = s[3 * threadIdx.x + 1], z = s[3 * threadIdx.x + 2];
    int ix, iy, iz;
    point_cell(x, y, z, L, ix, iy, iz);
    if (axis) {      // slab layout: points outside this rank's planes are not laid out
      const int a = axis == 2 ? iz : iy;
      if (a < c_lo || a >= c_hi) continue;
    }
    const uint32_t c = (uint32_t)(((long long)iz * L.dims[1] + iy) * (long long)L.dims[0] + ix);
    const uint32_t slot = __ldg(off + c) + __ldg(rank + i);
    double2 *o = reinterpret_cast<double2 *>(sorted + slot);
    o[0] = make_double2(x, y);
    o[1] = make_double2(z, __longlong_as_double((long long)(((unsigned long long)c << 32) | (unsigned long long)i)));
  }
}

// fp32 screening copy of the sorted cloud (streaming pass, coalesced both ways): offset of every point from the origin
// of its own cell (|offset| < ~h, so the fp32 rounding error is ~3e-8 h whatever the world extent) and the cell's x
// index.  The sweeps rebuild the offset between two points as (ix_a - ix_b) * h + (rel_a - rel_b).  A pass of its own:
// written from the scatter, as a random 16-byte write next to each record, it made the scatter 2.3x slower on C3, far
// more than this pass costs.
__global__ void __launch_bounds__(kThreads) rel_kernel(const P4 *__restrict__ sorted, long long n, Lattice L,
                                                       float4 *__restrict__ rel) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const P4 p = load_p4(sorted + i);
    const uint32_t c = cell_of(p.idx);
    const uint32_t ix = c % (uint32_t)L.dims[0];
    const uint32_t cyz = c / (uint32_t)L.dims[0];
    const uint32_t iy = cyz % (uint32_t)L.dims[1], iz = cyz / (uint32_t)L.dims[1];
    rel[i] = make_float4((float)cell_rel(p.x, ix, L, 0), (float)cell_rel(p.y, iy, L, 1), (float)cell_rel(p.z, iz, L, 2), (float)ix);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// query tiles (tile sweep only, built on demand): every kTileEdge^3 block of cells that holds at least one point, in
// increasing tile id (flag -> exclusive scan -> compaction: the same list on every rank, so that ranks can shard it)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) tile_flag_kernel(const uint32_t *__restrict__ off, Lattice L,
                                                             uint32_t *__restrict__ flag) {
  const long long nt = (long long)L.nb[0] * L.nb[1] * L.nb[2];
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t <= nt; t += (long long)gridDim.x * blockDim.x) {
    uint32_t tot = 0;
    if (t < nt) {
      const int bx = (int)(t % L.nb[0]), by = (int)((t / L.nb[0]) % L.nb[1]), bz = (int)(t / ((long long)L.nb[0] * L.nb[1]));
      const int xa = bx * kTileEdge, xb = min(xa + kTileEdge, L.dims[0]);
      for (int dz = 0; dz < kTileEdge; ++dz) {
        const int z = bz * kTileEdge + dz;
        if (z >= L.dims[2]) break;
        for (int dy = 0; dy < kTileEdge; ++dy) {
          const int y = by * kTileEdge + dy;
          if (y >= L.dims[1]) break;
          const long long row = ((long long)z * L.dims[1] + y) * L.dims[0];
          tot += __ldg(off + row + xb) - __ldg(off + row + xa);
        }
      }
    }
    flag[t] = tot ? 1u : 0u;      // flag[nt] = 0: after the exclusive scan it holds the number of tiles
  }
}
__global__ void __launch_bounds__(kThreads) tile_compact_kernel(const uint32_t *__restrict__ pos, long long nt,
                                                                uint32_t *__restrict__ tiles) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < nt; t += (long long)gridDim.x * blockDim.x) {
    const uint32_t p = __ldg(pos + t);
    if (__ldg(pos + t + 1) != p) tiles[p] = (uint32_t)t;
  }
}


int build_tiles(me_ctx *ctx, int which) {
  Cloud &c = ctx->cloud[which];
  if (c.tiles_valid) return ME_OK;
  const Lattice &L = c.lat;
  if (L.sparse) return fail(ctx, ME_ERR_RANGE, "the tile sweep needs a dense cell table");
  const long long nt = (long long)L.nb[0] * L.nb[1] * L.nb[2];
  ME_TRY(ensure(ctx, (void **)&c.d_tiles, &c.cap_tiles, std::min<long long>(nt, c.n), sizeof(uint32_t)));
  ME_TRY(ensure(ctx, (void **)&c.d_tile_pos, &c.cap_tile_pos, nt + 1, sizeof(uint32_t)));
  const int blocks = (int)std::min<long long>((nt + kThreads) / kThreads, (long long)ctx->sm_count * 16);
  tile_flag_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.d_cell_off, L, c.d_tile_pos);
  ME_LAUNCH_CHECK(ctx);
  ME_TRY(exclusive_scan_inplace(ctx, c.d_tile_pos, nt + 1));
  tile_compact_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.d_tile_pos, nt, c.d_tiles);
  ME_LAUNCH_CHECK(ctx);
  uint32_t *h_nt = (uint32_t *)((unsigned long long *)ctx->h_pinned + 8);
  ME_CUDA(ctx, cudaMemcpyAsync(h_nt, c.d_tile_pos + nt, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  c.n_tiles = (long long)*h_nt;
  c.tiles_valid = true;
  return ME_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// query range of this rank: [n r / W, n (r+1) / W) of the cell-sorted order, snapped DOWN to cell boundaries.  The order
// of the points inside a cell is not reproducible between ranks (the scatter takes its slots with atomics), the cell
// boundaries are: with cell-aligned shards every point is evaluated by exactly one rank.
// ---------------------------------------------------------------------------------------------------------------
__global__ void shard_bounds_kernel(const P4 *__restrict__ sorted, const float4 *__restrict__ rel, CellIndex I, long long n,
                                    int rank, int world, unsigned long long *__restrict__ out) {
  const int k = threadIdx.x;      // 0: begin, 1: end
  if (k > 1) return;
  const int r = rank + k;
  long long b = n * r / world;
  if (r >= world) b = n;
  else if (b > 0) {               // first point of the cell that holds point b
    int ix, iy, iz;
    cell_from_tag(I, __double_as_longlong(__ldg(reinterpret_cast<const double *>(sorted + b) + 3)), (int)__ldg(rel + b).w, ix, iy, iz);
    uint32_t s, e;
    cell_range(I, iz, iy, ix, ix, s, e);
    b = s;
  }
  out[k] = (unsigned long long)b;
}

int query_shard(me_ctx *ctx, int which, long long *b, long long *e) {
  Cloud &c = ctx->cloud[which];
  if (ctx->world == 1) { *b = 0; *e = c.n; return ME_OK; }
  if (c.slab) { *b = 0; *e = c.ns; return ME_OK; }      // slab layout: the sweeps walk what is laid out here and skip the halo (Owned)
  if (!(c.shard_valid && c.shard_rank == ctx->rank && c.shard_world == ctx->world)) {
    unsigned long long *d = (unsigned long long *)ctx->d_scratch + 12, *h = (unsigned long long *)ctx->h_pinned + 12;
    shard_bounds_kernel<<<1, 32, 0, ctx->stream>>>(c.d_sorted, c.d_rel, index_of(c), c.n, ctx->rank, ctx->world, d);
    ME_LAUNCH_CHECK(ctx);
    ME_CUDA(ctx, cudaMemcpyAsync(h, d, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    c.shard_b = (long long)h[0]; c.shard_e = (long long)h[1];
    c.shard_rank = ctx->rank; c.shard_world = ctx->world; c.shard_valid = true;
  }
  *b = c.shard_b; *e = c.shard_e;
  return ME_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// host: lattice choice
// ---------------------------------------------------------------------------------------------------------------
// sparse cell tables are used when the dense table would exceed the budget (test hook: ME_NO_SPARSE keeps the round-1
// behaviour of coarsening the cells instead)
static bool sparse_allowed() { return getenv("ME_NO_SPARSE") == nullptr; }

static bool make_lattice(const Cloud &c, double v, int m, long long budget, Lattice *out, bool allow_sparse) {
  Lattice L;
  L.v = v; L.m = m; L.h = v / m; L.m_over_v = m / v;
  L.sparse = 0; L.nsegx = 0;
  double nc = 1.0, nv = 1.0;
  for (int a = 0; a < 3; ++a) {
    double klo = std::floor(c.bbox_min[a] / v), khi = std::floor(c.bbox_max[a] / v);
    if (!(klo > -2.0e9 && khi < 2.0e9)) return false;   // the reference casts to int (voxel_calculator.cpp:242)
    L.k_lo[a] = (int)klo;
    double nvx = khi - klo + 1.0;
    if (nvx * m > 2.0e9) return false;
    L.nvox[a] = (int)nvx;
    L.dims[a] = L.nvox[a] * m;
    L.nb[a] = (L.dims[a] + kTileEdge - 1) / kTileEdge;
    nc *= (double)L.dims[a];
    nv *= nvx;
  }
  L.nvoxels = nv < 9.0e18 ? (long long)nv : -1;         // the voxel stage checks its own (dense) table budget
  if (nc <= (double)budget && nc < 4294967295.0) {
    L.ncells = (long long)nc;
    *out = L;
    return true;
  }
  if (!allow_sparse) return false;
  // sparse table: x indices live in an fp32 mantissa, row ids (z * dimy + y) in the 32-bit half of the point tag
  if (L.dims[0] >= (1 << 24) || L.dims[1] >= (1 << 24) || L.dims[2] >= (1 << 24)) return false;
  if ((double)L.dims[1] * (double)L.dims[2] >= 4294967295.0) return false;
  L.sparse = 1;
  L.nsegx = (L.dims[0] + kSegCells - 1) / kSegCells;
  L.ncells = 0;
  *out = L;
  return true;
}

static int histogram(me_ctx *ctx, Cloud &c, const Lattice &L) {
  ME_TRY(ensure(ctx, (void **)&c.d_cell_off, &c.cap_cells, L.ncells + 1, sizeof(uint32_t)));
  // counts live at off[0..ncells-1] and off[ncells] stays 0, so the exclusive scan of all ncells + 1 entries turns off[]
  // into the CSR offset array; the in-cell rank of every point goes to ctx->d_rank
  ME_CUDA(ctx, cudaMemsetAsync(c.d_cell_off, 0, (size_t)(L.ncells + 1) * sizeof(uint32_t), ctx->stream));
  ME_TRY(ensure(ctx, (void **)&ctx->d_rank, &ctx->cap_rank, c.n, sizeof(uint32_t)));
  int blocks = (int)std::min<long long>((c.n + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
  if (c.bbox_spec) {      // the box is measured here (scratch [0..6]) and read back with the cell statistics
    unsigned long long *box = (unsigned long long *)ctx->d_scratch;
    bbox_init_kernel<<<1, 32, 0, ctx->stream>>>(box);
    ME_LAUNCH_CHECK(ctx);
    cell_count_box_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.d_xyz, c.n, L, c.d_cell_off, ctx->d_rank, box);
  } else {
    cell_count_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.d_xyz, c.n, L, c.d_cell_off, ctx->d_rank);
  }
  ME_LAUNCH_CHECK(ctx);
  return ME_OK;
}

// exclusive scan of the cell counts, in place, with their statistics on the way: pinned slots [9] occupied cells, [10]
// points in the fullest cell (bounds the run lengths of the sweeps), valid once the stream is synchronized.  On a remembered
// box the measured box (slots [0..6], see histogram) comes back in the same copy.
static int scan_cells(me_ctx *ctx, Cloud &c, const Lattice &L) {
  unsigned long long *d = (unsigned long long *)ctx->d_scratch + 9;
  ME_CUDA(ctx, cudaMemsetAsync(d, 0, 2 * sizeof(unsigned long long), ctx->stream));
  ME_TRY(exclusive_scan_inplace(ctx, c.d_cell_off, L.ncells + 1, d));
  const int first = c.bbox_spec ? 0 : 9;
  ME_CUDA(ctx, cudaMemcpyAsync((unsigned long long *)ctx->h_pinned + first, (unsigned long long *)ctx->d_scratch + first,
                               (11 - first) * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
  return ME_OK;
}

// h the cloud would like on its own: ~2 points per cell for a volume-filling cloud
double density_edge(const Cloud &c) {
  double ext[3], vol = 1.0, ext_max = 0.0;
  for (int a = 0; a < 3; ++a) { ext[a] = c.bbox_max[a] - c.bbox_min[a]; ext_max = std::max(ext_max, ext[a]); }
  if (ext_max <= 0.0) ext_max = 1.0;
  for (int a = 0; a < 3; ++a) vol *= std::max(ext[a], 1e-3 * ext_max);
  return std::cbrt(2.0 * vol / (double)c.n);
}

// (v, m) for a target cell edge, fitting `c` (and `other`, if its bbox is known) into the budget
static constexpr int kMaxCellsPerVoxelEdge = 512;

static bool pick_spec(const Cloud &c, const Cloud *other, double v_req, double h_target, long long budget, double *v,
                      int *m, Lattice *out, bool allow_sparse) {
  Lattice tmp;
  if (v_req > 0) {
    // cells per voxel edge: at most kMaxCellsPerVoxelEdge — the voxel stage walks the m x m lattice rows of every voxel, and
    // degenerate data (duplicates, collinear points) would otherwise drive the cell edge towards zero once the sparse table
    // lifts the budget
    int mm = (int)std::max(1.0, std::floor(v_req / h_target + 0.5));
    mm = std::min(mm, kMaxCellsPerVoxelEdge);
    for (; mm >= 1; --mm) {
      if (make_lattice(c, v_req, mm, budget, out, allow_sparse) && (!other || make_lattice(*other, v_req, mm, budget, &tmp, allow_sparse))) {
        *v = v_req; *m = mm;
        return true;
      }
      if (mm > 64) mm = (int)(mm * 0.8);   // far over budget: shrink geometrically
    }
    return false;
  }
  double h = h_target;
  for (int t = 0; t < 96; ++t, h *= 1.26)
    if (make_lattice(c, h, 1, budget, out, allow_sparse) && (!other || make_lattice(*other, h, 1, budget, &tmp, allow_sparse))) {
      *v = h; *m = 1;
      return true;
    }
  return false;
}

// one planning step: the dense table at the wanted edge if it fits the budget; if the budget forces cells noticeably coarser
// than wanted (or nothing fits), a sparse table at the wanted edge instead
static bool choose_lattice(const Cloud &c, const Cloud *other, double v_req, double h_target, long long budget, bool sp,
                           double *v, int *m, Lattice *cand) {
  bool ok = pick_spec(c, other, v_req, h_target, budget, v, m, cand, false);
  if (sp && (!ok || cand->h > 1.25 * h_target)) {
    Lattice cs;
    double vs; int ms;
    if (pick_spec(c, other, v_req, h_target, budget, &vs, &ms, &cs, true)) { *cand = cs; *v = vs; *m = ms; ok = true; }
  }
  return ok;
}

static long long auto_budget(long long n_max) { return std::min<long long>(1ll << 31, std::max<long long>(1ll << 28, 16 * n_max)); }

// the planning step as a pure host function (me_plan_lattice): bounding boxes and sizes in, lattice out
bool plan_lattice_host(const double bmin[3], const double bmax[3], long long n, const double *obmin, const double *obmax,
                       long long other_n, double v_req, double h_target, long long budget, bool allow_sparse, Lattice *out) {
  Cloud c, o;
  c.n = n; o.n = other_n;
  for (int a = 0; a < 3; ++a) {
    c.bbox_min[a] = bmin[a]; c.bbox_max[a] = bmax[a];
    o.bbox_min[a] = obmin ? obmin[a] : 0.0; o.bbox_max[a] = obmax ? obmax[a] : 0.0;
  }
  c.bbox_valid = true; o.bbox_valid = obmin && obmax;
  if (budget <= 0) budget = auto_budget(std::max(n, o.bbox_valid ? other_n : 0));
  if (!(h_target > 0)) h_target = density_edge(c);
  double v; int m;
  return choose_lattice(c, o.bbox_valid ? &o : nullptr, v_req, h_target, budget, allow_sparse, &v, &m, out);
}

// in-place exclusive scan of n uint32, one pass (scan_kernel; the tile status words live in a small buffer of their own,
// so callers may keep data in the work buffer across the scan).  stats: see scan_kernel; the caller clears them.
int exclusive_scan_inplace(me_ctx *ctx, uint32_t *a, long long n, unsigned long long *stats) {
  const long long ntiles = (n + kScanTile - 1) / kScanTile;
  ME_TRY(ensure(ctx, (void **)&ctx->d_scan_tmp, &ctx->cap_scan_tmp, ntiles, sizeof(unsigned long long)));
  ME_CUDA(ctx, cudaMemsetAsync(ctx->d_scan_tmp, 0, (size_t)ntiles * sizeof(unsigned long long), ctx->stream));
  scan_kernel<<<(unsigned)ntiles, kThreads, 0, ctx->stream>>>(a, n, ctx->d_scan_tmp, stats);
  ME_LAUNCH_CHECK(ctx);
  return ME_OK;
}

// Budget of the dense cell table (4 B per cell).  Automatic: 2^28 cells, growing with the clouds up to 2^31 (16 cells per
// point: a 200 M-point surface scan at 1 cm spacing keeps ~4 points per occupied cell instead of ~18; the table then
// takes 8.6 GB of the 80 GB, and clearing and scanning it is a small part of a build next to the sweeps at that size).
static long long grid_budget(const me_ctx *ctx) {
  if (getenv("ME_FORCE_SPARSE")) return 1;      // test hook: every lattice gets a sparse cell table
  if (ctx->max_grid_cells > 0) return ctx->max_grid_cells;
  return auto_budget(std::max(ctx->cloud[0].n, ctx->cloud[1].n));
}

// ---------------------------------------------------------------------------------------------------------------
// sparse lattice build: points sorted by their 64-bit cell key (row * 32 nsegx + ix) with the library's radix sort, the
// occupied row segments found as runs of the sorted keys, their 32-cell count blocks laid out in the same order (a CSR
// table over occupied segments only) and entered into a hash table (segment key -> rank)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) sparse_key_kernel(const double *__restrict__ xyz, long long n, Lattice L,
                                                              unsigned long long *__restrict__ key, uint32_t *__restrict__ val) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double x = __ldg(xyz + 3 * i), y = __ldg(xyz + 3 * i + 1), z = __ldg(xyz + 3 * i + 2);
    long long ix = cell_coord(x, L, 0), iy = cell_coord(y, L, 1), iz = cell_coord(z, L, 2);
    ix = ix < 0 ? 0 : (ix >= L.dims[0] ? L.dims[0] - 1 : ix);
    iy = iy < 0 ? 0 : (iy >= L.dims[1] ? L.dims[1] - 1 : iy);
    iz = iz < 0 ? 0 : (iz >= L.dims[2] ? L.dims[2] - 1 : iz);
    const unsigned long long row = (unsigned long long)iz * (unsigned long long)L.dims[1] + (unsigned long long)iy;
    key[i] = row * (unsigned long long)(L.nsegx * kSegCells) + (unsigned long long)ix;
    val[i] = (uint32_t)i;
  }
}
// head[i] = 1 where a new segment (key >> 5) starts in the sorted key sequence; head[n] = 0 (after the scan: segment count)
__global__ void __launch_bounds__(kThreads) sparse_head_kernel(const unsigned long long *__restrict__ key, long long n,
                                                               uint32_t *__restrict__ head) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i <= n; i += (long long)gridDim.x * blockDim.x)
    head[i] = (i < n && (i == 0 || (key[i] >> 5) != (key[i - 1] >> 5))) ? 1u : 0u;
}
// per point: count into its cell of the compact table; per segment head: hash insert (segment key -> rank).
// rank_excl = exclusive scan of the head flags: the segment of point i has rank rank_excl[i + 1] - 1.
__global__ void __launch_bounds__(kThreads) sparse_count_kernel(const unsigned long long *__restrict__ key, const uint32_t *__restrict__ rank_excl,
                                                                long long n, uint32_t *__restrict__ count,
                                                                unsigned long long *__restrict__ hkey, uint32_t *__restrict__ hval,
                                                                uint32_t hmask) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = key[i];
    const uint32_t r = rank_excl[i + 1] - 1u;
    atomicAdd(count + ((unsigned long long)r << 5) + (k & 31ull), 1u);
    if (i == 0 || (key[i - 1] >> 5) != (k >> 5)) {      // the first point of a segment enters it into the hash table
      const unsigned long long sk = k >> 5;
      uint32_t h = seg_hash(sk) & hmask;
      for (;;) {
        const unsigned long long old = atomicCAS(hkey + h, ~0ull, sk);
        if (old == ~0ull || old == sk) { hval[h] = r; break; }
        h = (h + 1) & hmask;
      }
    }
  }
}
// the sorted records and their fp32 screening copies, written in sorted order (gather from the caller-order array)
__global__ void __launch_bounds__(kThreads) sparse_gather_kernel(const double *__restrict__ xyz, const unsigned long long *__restrict__ key,
                                                                 const uint32_t *__restrict__ val, long long n, Lattice L,
                                                                 P4 *__restrict__ sorted, float4 *__restrict__ rel) {
  const unsigned long long rowlen = (unsigned long long)(L.nsegx * kSegCells);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = key[i];
    const uint32_t o = val[i];
    const unsigned long long row = k / rowlen;
    const uint32_t ix = (uint32_t)(k - row * rowlen);
    const uint32_t iy = (uint32_t)(row % (unsigned long long)L.dims[1]), iz = (uint32_t)(row / (unsigned long long)L.dims[1]);
    const double x = __ldg(xyz + 3ll * o), y = __ldg(xyz + 3ll * o + 1), z = __ldg(xyz + 3ll * o + 2);
    double2 *out = reinterpret_cast<double2 *>(sorted + i);
    out[0] = make_double2(x, y);
    out[1] = make_double2(z, __longlong_as_double((long long)((row << 32) | (unsigned long long)o)));      // tag: row id | caller index
    rel[i] = make_float4((float)cell_rel(x, ix, L, 0), (float)cell_rel(y, iy, L, 1), (float)cell_rel(z, iz, L, 2), (float)ix);
  }
}
__global__ void fill_u64_kernel(unsigned long long *p, long long n, unsigned long long v) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = v;
}

// lays `c` out on the sparse lattice L; *occupied = cells that hold at least one point
static int build_sparse(me_ctx *ctx, Cloud &c, const Lattice &L, long long *occupied) {
  const long long n = c.n;
  auto align = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t o_key0 = 0, o_key1 = o_key0 + align((size_t)n * 8), o_val0 = o_key1 + align((size_t)n * 8),
               o_val1 = o_val0 + align((size_t)n * 4), o_rank = o_val1 + align((size_t)n * 4), total = o_rank + align((size_t)(n + 1) * 4);
  ME_TRY(ensure_work(ctx, total));
  char *base = (char *)ctx->d_work;
  unsigned long long *key0 = (unsigned long long *)(base + o_key0), *key1 = (unsigned long long *)(base + o_key1);
  uint32_t *val0 = (uint32_t *)(base + o_val0), *val1 = (uint32_t *)(base + o_val1), *rank = (uint32_t *)(base + o_rank);
  const int blocks = (int)std::min<long long>((n + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
  sparse_key_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.d_xyz, n, L, key0, val0);
  ME_LAUNCH_CHECK(ctx);
  int key_bits = 1;
  const double kmax = (double)L.dims[1] * (double)L.dims[2] * (double)(L.nsegx * kSegCells);
  while (key_bits < 63 && std::ldexp(1.0, key_bits) < kmax) ++key_bits;
  unsigned long long *keys = nullptr;
  uint32_t *vals = nullptr;
  ME_TRY(radix_sort_pairs(ctx, key0, val0, key1, val1, n, key_bits, &keys, &vals));      // stable: points of a cell keep the caller's order
  sparse_head_kernel<<<blocks, kThreads, 0, ctx->stream>>>(keys, n, rank);
  ME_LAUNCH_CHECK(ctx);
  ME_TRY(exclusive_scan_inplace(ctx, rank, n + 1));
  uint32_t *h_nseg = (uint32_t *)((unsigned long long *)ctx->h_pinned + 8);
  ME_CUDA(ctx, cudaMemcpyAsync(h_nseg, rank + n, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const long long nseg = (long long)*h_nseg;
  if (nseg * kSegCells >= 0xffffffffll) return fail(ctx, ME_ERR_RANGE, "sparse lattice: more than 2^27 occupied row segments");
  long long slots = 1;
  while (slots < 2 * nseg) slots <<= 1;
  ME_TRY(ensure(ctx, (void **)&c.d_cell_off, &c.cap_cells, nseg * kSegCells + 1, sizeof(uint32_t)));
  if (!(c.d_hkey && c.cap_hash >= slots)) {
    if (c.d_hkey) cudaFree(c.d_hkey);
    if (c.d_hval) cudaFree(c.d_hval);
    c.d_hkey = nullptr; c.d_hval = nullptr; c.cap_hash = 0;
    long long cap = 0;
    ME_TRY(ensure(ctx, (void **)&c.d_hkey, &cap, slots, sizeof(unsigned long long)));
    cap = 0;
    ME_TRY(ensure(ctx, (void **)&c.d_hval, &cap, slots, sizeof(uint32_t)));
    c.cap_hash = slots;
  }
  c.hmask = (uint32_t)(slots - 1);
  c.n_seg = nseg;
  ME_CUDA(ctx, cudaMemsetAsync(c.d_cell_off, 0, (size_t)(nseg * kSegCells + 1) * sizeof(uint32_t), ctx->stream));
  fill_u64_kernel<<<(int)std::min<long long>((slots + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16), kThreads, 0, ctx->stream>>>(c.d_hkey, slots, ~0ull);
  ME_LAUNCH_CHECK(ctx);
  // count of compact cell k at off[k]; the exclusive scan over the ncomp + 1 entries (the last one zero) makes it a CSR array
  sparse_count_kernel<<<blocks, kThreads, 0, ctx->stream>>>(keys, rank, n, c.d_cell_off, c.d_hkey, c.d_hval, c.hmask);
  ME_LAUNCH_CHECK(ctx);
  unsigned long long *d_nt = (unsigned long long *)ctx->d_scratch + 8;
  ME_CUDA(ctx, cudaMemsetAsync(d_nt, 0, 3 * sizeof(unsigned long long), ctx->stream));
  ME_TRY(exclusive_scan_inplace(ctx, c.d_cell_off, nseg * kSegCells + 1, d_nt + 1));      // [9] occupied cells, [10] fullest cell
  unsigned long long *h_nt = (unsigned long long *)ctx->h_pinned + 8;
  ME_CUDA(ctx, cudaMemcpyAsync(h_nt, d_nt, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
  ME_TRY(ensure(ctx, (void **)&c.d_sorted, &c.cap_sorted, n, sizeof(P4)));
  ME_TRY(ensure(ctx, (void **)&c.d_rel, &c.cap_rel, n, sizeof(float4)));
  sparse_gather_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.d_xyz, keys, vals, n, L, c.d_sorted, c.d_rel);
  ME_LAUNCH_CHECK(ctx);
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  *occupied = (long long)h_nt[1];
  c.max_cell_count = (long long)h_nt[2];
  return ME_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// coarse occupancy grid: point counts of blocks of f^3 lattice cells (f a power of two, at most 256 blocks per axis).
// The ring expansion of the far-query kernel costs O(r^3) cell lookups in empty space; on fine lattices over large extents
// (est maps that reach beyond the ground truth, outliers) it walks coarse blocks instead and descends only into occupied
// ones.  Built for lattices with more than 256 cells along some axis.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) coarse_count_kernel(const P4 *__restrict__ sorted, const float4 *__restrict__ rel, long long n,
                                                                CellIndex I, int shift, int cdx, int cdy, uint32_t *__restrict__ cnt) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int ix, iy, iz;
    cell_from_tag(I, __double_as_longlong(__ldg(reinterpret_cast<const double *>(sorted + i) + 3)), (int)__ldg(rel + i).w, ix, iy, iz);
    atomicAdd(cnt + ((long long)(iz >> shift) * cdy + (iy >> shift)) * cdx + (ix >> shift), 1u);
  }
}

static int build_coarse(me_ctx *ctx, Cloud &c) {
  const Lattice &L = c.lat;
  c.coarse_f = 0;
  const int dmax = std::max(L.dims[0], std::max(L.dims[1], L.dims[2]));
  if (dmax <= 256) return ME_OK;
  int shift = 2;
  while (((dmax + (1 << shift) - 1) >> shift) > 256) ++shift;
  const int f = 1 << shift;
  long long ncoarse = 1;
  for (int a = 0; a < 3; ++a) { c.coarse_dims[a] = (L.dims[a] + f - 1) >> shift; ncoarse *= c.coarse_dims[a]; }
  ME_TRY(ensure(ctx, (void **)&c.d_coarse, &c.cap_coarse, ncoarse, sizeof(uint32_t)));
  ME_CUDA(ctx, cudaMemsetAsync(c.d_coarse, 0, (size_t)ncoarse * sizeof(uint32_t), ctx->stream));
  const int blocks = (int)std::min<long long>((c.ns + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
  coarse_count_kernel<<<std::max(1, blocks), kThreads, 0, ctx->stream>>>(c.d_sorted, c.d_rel, c.ns, index_of(c), shift, c.coarse_dims[0],
                                                          c.coarse_dims[1], c.d_coarse);
  ME_LAUNCH_CHECK(ctx);
  c.coarse_f = f;
  return ME_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// slab layout (me_set_layout, world > 1, dense lattices).  The query ranges of the sweeps are sharded anyway; laying out BOTH
// WHOLE clouds on every rank is what bounds strong scaling (the builds dominated a pass on 8 B200s; not re-measured on
// H100).  In slab layout
// a rank lays out only the lattice planes of the voxel layers it owns along one lattice axis (y or z, whichever balances —
// terrestrial scans are flat in z), plus slab_halo cells on either side, of both clouds: the histogram still covers the whole
// cloud (a streaming pass), the counts outside the slab are cleared, and the expensive random-write scatter touches about
// 1/W of the points.  The layers are balanced on the layer histogram of the cloud laid out first and are expressed in WORLD
// voxel indices, so the slabs of the two clouds coincide and every voxel has one owner.  The sweeps walk the laid-out points
// and skip the halo ones (Owned); searches that would leave the halo are finished by brute force over the caller-order
// cloud (nn.cu).
// ---------------------------------------------------------------------------------------------------------------
// out[p] = points in lattice plane p along `axis` (1: y, 2: z)
__global__ void __launch_bounds__(kThreads) plane_count_kernel(const uint32_t *__restrict__ count, int dimx, int dimy, int dimz,
                                                               int axis, unsigned long long *__restrict__ out) {
  __shared__ unsigned long long ws[kThreads / 32];
  const int np = axis == 2 ? dimz : dimy;
  for (int p = blockIdx.x; p < np; p += gridDim.x) {
    unsigned long long s = 0;
    if (axis == 2) {
      const long long pl = (long long)dimx * dimy;
      const uint32_t *q = count + (long long)p * pl;
      for (long long i = threadIdx.x; i < pl; i += kThreads) s += __ldg(q + i);
    } else {
      for (int z = 0; z < dimz; ++z) {
        const uint32_t *q = count + ((long long)z * dimy + p) * dimx;
        for (int i = threadIdx.x; i < dimx; i += kThreads) s += __ldg(q + i);
      }
    }
    s = (unsigned long long)warp_sum_ll((long long)s);
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) { unsigned long long t = 0; for (int w = 0; w < kThreads / 32; ++w) t += ws[w]; out[p] = t; }
    __syncthreads();
  }
}

// clear the counts of the cells outside the covered planes; out[0] += points in the owned planes
__global__ void __launch_bounds__(kThreads) slab_mask_kernel(uint32_t *__restrict__ count, long long ncells, int dimx, int dimy,
                                                             int axis, int c_lo, int c_hi, int o_lo, int o_hi,
                                                             unsigned long long *__restrict__ out) {
  unsigned long long own = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < ncells; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / dimx;
    const int a = axis == 2 ? (int)(row / dimy) : (int)(row % dimy);
    if (a < c_lo || a >= c_hi) count[i] = 0u;
    else if (a >= o_lo && a < o_hi) own += __ldg(count + i);
  }
  own = (unsigned long long)warp_sum_ll((long long)own);
  if ((threadIdx.x & 31) == 0 && own) atomicAdd(out, own);
}

static bool slab_wanted(const me_ctx *ctx) { return ctx->slab_request && ctx->world > 1 && getenv("ME_NO_SLAB") == nullptr; }

// The cut itself — pure host arithmetic on the per-plane point counts along y and z (also behind me_plan_slab_cut for the CPU
// tests).  The voxel layers of an axis (m planes each) are cut into `world` contiguous groups of about equal point count;
// the axis whose busiest rank lays out (owned layers + halo planes) the smallest share of the cloud wins.  *axis = 0 if
// neither axis has 2 * world layers.  bounds[0..world]: first owned layer of every rank (bounds[world] = number of layers).
void slab_cut(const unsigned long long *planes_y, int n_planes_y, const unsigned long long *planes_z, int n_planes_z, int m,
              int world, int halo, int *axis_out, int *bounds, double *share_out) {
  const int W = world, H = halo;
  double best_share = 2.0;
  std::vector<int> best_b;
  int best_axis = 0;
  for (int axis = 1; axis <= 2; ++axis) {
    const unsigned long long *hp = axis == 2 ? planes_z : planes_y;
    const int nl = (axis == 2 ? n_planes_z : n_planes_y) / std::max(1, m);
    if (nl < 2 * W) continue;                            // too few voxel layers to cut
    std::vector<unsigned long long> cum((size_t)nl * m + 1, 0);      // per plane
    for (int p = 0; p < nl * m; ++p) cum[p + 1] = cum[p] + hp[p];
    const unsigned long long total = cum[(size_t)nl * m];
    if (total == 0) continue;
    std::vector<int> b((size_t)W + 1, 0);
    b[W] = nl;
    for (int r = 1; r < W; ++r) {
      const unsigned long long want = total / (unsigned long long)W * (unsigned long long)r;
      int lo = b[r - 1] + 1, hi = nl - (W - r);
      int l = lo;
      while (l < hi && cum[(size_t)l * m] < want) ++l;      // first layer boundary at or past the target
      if (l > lo && want - cum[(size_t)(l - 1) * m] < cum[(size_t)l * m] - want) --l;
      b[r] = l;
    }
    // the share of the cloud the busiest rank lays out (owned layers + halo)
    unsigned long long worst = 0;
    for (int r = 0; r < W; ++r) {
      const int p0 = std::max(0, b[r] * m - H), p1 = std::min(nl * m, b[r + 1] * m + H);
      worst = std::max(worst, cum[p1] - cum[p0]);
    }
    const double share = (double)worst / (double)total;
    if (share < best_share) { best_share = share; best_b = b; best_axis = axis; }
  }
  *axis_out = best_axis;
  *share_out = best_share;
  if (best_axis) for (int r = 0; r <= W; ++r) bounds[r] = best_b[r];
}

// plan the owned voxel layers of every rank from the layer histograms of cloud c (histogram in c.d_cell_off); the same
// arithmetic on the same (replicated) cloud on every rank gives the same plan
static int plan_slabs(me_ctx *ctx, Cloud &c, const Lattice &L) {
  ctx->slab_planned = true;
  ctx->slab_on = false;
  const int W = ctx->world, H = ctx->slab_halo;
  const int np = L.dims[1] + L.dims[2];
  ME_TRY(ensure_work(ctx, (size_t)np * sizeof(unsigned long long)));
  unsigned long long *d_pl = (unsigned long long *)ctx->d_work;
  plane_count_kernel<<<std::min(L.dims[1], ctx->sm_count * 8), kThreads, 0, ctx->stream>>>(c.d_cell_off, L.dims[0], L.dims[1], L.dims[2], 1, d_pl);
  ME_LAUNCH_CHECK(ctx);
  plane_count_kernel<<<std::min(L.dims[2], ctx->sm_count * 8), kThreads, 0, ctx->stream>>>(c.d_cell_off, L.dims[0], L.dims[1], L.dims[2], 2, d_pl + L.dims[1]);
  ME_LAUNCH_CHECK(ctx);
  std::vector<unsigned long long> h((size_t)np);
  ME_CUDA(ctx, cudaMemcpyAsync(h.data(), d_pl, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  int best_axis = 0;
  double best_share = 2.0;
  std::vector<int> best_b((size_t)W + 1, 0);
  slab_cut(h.data(), L.dims[1], h.data() + L.dims[1], L.dims[2], L.m, W, H, &best_axis, best_b.data(), &best_share);
  if (getenv("ME_DEBUG_SLAB"))
    fprintf(stderr, "[mapeval] slab plan: rank %d/%d lattice %d x %d x %d (m = %d), axis %d, busiest share %.3f\n", ctx->rank, W,
            L.dims[0], L.dims[1], L.dims[2], L.m, best_axis, best_share);
  // worth it only if the busiest rank lays out clearly less than the whole cloud
  if (best_axis == 0 || best_share > kSlabMaxShare) return ME_OK;
  const int r = ctx->rank;
  ctx->slab_axis = best_axis;
  ctx->slab_k0 = r == 0 ? LLONG_MIN / 4 : (long long)L.k_lo[best_axis] + best_b[r];
  ctx->slab_k1 = r == W - 1 ? LLONG_MAX / 4 : (long long)L.k_lo[best_axis] + best_b[r + 1];
  ctx->slab_on = true;
  return ME_OK;
}

// owned / covered lattice planes of cloud c on lattice L for the planned layers
static void slab_planes(const me_ctx *ctx, const Lattice &L, Cloud &c) {
  const int ax = ctx->slab_axis, dim = L.dims[ax];
  auto plane = [&](long long k) -> int {
    if (k <= LLONG_MIN / 8) return 0;
    if (k >= LLONG_MAX / 8) return dim;
    const long long z = (k - (long long)L.k_lo[ax]) * L.m;
    return (int)std::min<long long>(std::max<long long>(z, 0), dim);
  };
  c.sl_axis = ax;
  c.so_lo = plane(ctx->slab_k0); c.so_hi = plane(ctx->slab_k1);
  if (c.so_lo >= c.so_hi) { c.sc_lo = c.sc_hi = c.so_hi = c.so_lo; return; }      // nothing of this cloud here
  c.sc_lo = std::max(0, c.so_lo - ctx->slab_halo);
  c.sc_hi = std::min(dim, c.so_hi + ctx->slab_halo);
}

// solo_h > 0: lay the cloud out on a lattice of its own with cells of (about) that edge — used by the MME sweep when the
// search radius spans many cells of the shared lattice (mme.cu).  A solo lattice is not voxel-aligned and not shared with
// the other cloud; the next ordinary build_grid() replaces it.
int build_grid(me_ctx *ctx, int which, double solo_h) {
  Cloud &c = ctx->cloud[which];
  Cloud &o = ctx->cloud[which ^ 1];      // the partner cloud: est <-> gt (feature clouds are only ever laid out solo)
  if (c.n <= 0) return fail(ctx, ME_ERR_EMPTY, "cloud is empty");
  if (c.n >= 0x7fffffffll) return fail(ctx, ME_ERR_RANGE, "more than 2^31-1 points per cloud (the reference indexes with int)");
  const bool solo = solo_h > 0;
  if (c.grid_valid && c.grid_solo == solo && (!solo || c.solo_h == solo_h)) return ME_OK;
  ME_TRY(wait_upload(ctx, which));
  StageTimer timer(ctx, which >= kFeatureSlot ? -1 : (which == ME_CLOUD_EST ? 0 : 1));
  if (!solo) speculate_bbox(ctx, which);
  else if (c.bbox_spec) c.bbox_valid = false;      // a solo lattice is planned on the measured box
  ME_TRY(compute_bbox(ctx, which));
  // what a build on a remembered box changes before the box is checked: restored when it turns out wrong
  struct {
    bool o_grid, o_nn, o_entropy, slab_planned;
    double spec_v; int spec_m;
    PlanCache pc;
  } const before = {o.grid_valid, o.nn_valid, o.entropy_valid, ctx->slab_planned, ctx->spec_v, ctx->spec_m,
                    ctx->plan_cache[which]};
  // the remembered box is wrong (bad_box) or the plan on it needs a sparse table (built on the measured box only): undo,
  // take the measured box and build again
  auto restart = [&](const unsigned long long *bad_box) -> int {
    o.grid_valid = before.o_grid; o.nn_valid = before.o_nn; o.entropy_valid = before.o_entropy;
    ctx->slab_planned = before.slab_planned; ctx->spec_v = before.spec_v; ctx->spec_m = before.spec_m;
    ctx->plan_cache[which] = before.pc;
    c.bbox_valid = false; c.bbox_spec = false;
    if (!bad_box) ME_TRY(compute_bbox(ctx, which));
    else {
      if (bad_box[6] != 0)
        return fail(ctx, ME_ERR_RANGE, "cloud holds non-finite coordinates (the reference drops them at load, map_eval.cpp:6)");
      for (int k = 0; k < 3; ++k) { c.bbox_min[k] = dec_ordered(bad_box[k]); c.bbox_max[k] = dec_ordered(bad_box[3 + k]); }
      c.bbox_valid = true;
      c.bbox_missed = true;
      trace_kernel(ctx, ME_TEV_BOX_MISSED);
    }
    return build_grid(ctx, which, solo_h);
  };
  const long long budget = grid_budget(ctx);
  const double v_req = ctx->voxel_hint;
  const bool sp = sparse_allowed();

  // Both clouds share one lattice spec (v, m) so that their cells coincide.  The spec is re-planned whenever no
  // valid grid depends on it (i.e. at the first build of a pass); a later build re-uses it.
  // A cloud whose dense cell table would exceed the budget at the wanted cell edge gets a SPARSE table at that edge
  // (occupied row segments only) instead of coarser cells.
  Lattice L;
  bool built = false;      // the sparse build lays the cloud out while planning
  bool scanned = false;    // the dense table already holds the scan of the histogram (planning measured the occupancy)
  long long occupied = 0;
  if (solo) {
    double v; int m;
    if (!pick_spec(c, nullptr, 0.0, solo_h, budget, &v, &m, &L, sp))
      return fail(ctx, ME_ERR_RANGE, "cannot fit the cloud into the lattice");
    if (L.sparse) { ME_TRY(build_sparse(ctx, c, L, &occupied)); built = true; }
    else ME_TRY(histogram(ctx, c, L));
  } else if (o.grid_valid && !o.grid_solo && ctx->spec_m > 0 && (v_req <= 0 || ctx->spec_v == v_req) &&
             make_lattice(c, ctx->spec_v, ctx->spec_m, budget, &L, sp)) {
    if (L.sparse && c.bbox_spec) return restart(nullptr);
    if (L.sparse) { ME_TRY(build_sparse(ctx, c, L, &occupied)); built = true; }
    else ME_TRY(histogram(ctx, c, L));
  } else {
    if (o.grid_valid && !o.grid_solo) {   // the other grid's spec cannot host this cloud: both are laid out again
      o.grid_valid = false; o.nn_valid = false; o.entropy_valid = false;
    }
    ctx->slab_planned = false;              // the slabs are planned again with the spec
    const Cloud *other = (o.n > 0 && o.bbox_valid) ? &o : nullptr;
    double h_target = ctx->nn_cell_size > 0 ? ctx->nn_cell_size : density_edge(c);
    // the same constellation was planned before (repeated passes over the same maps): one iteration at the remembered edge
    PlanCache &pc = ctx->plan_cache[which];
    bool hit = pc.valid && !getenv("ME_NO_PLAN_CACHE") && pc.n == c.n && pc.other_n == (other ? other->n : -1) && pc.v_req == v_req &&
               pc.nn_cell == ctx->nn_cell_size && pc.budget == budget && pc.sp == sp && pc.slab_request == ctx->slab_request &&
               pc.rank == ctx->rank && pc.world == ctx->world;
    for (int a = 0; a < 3 && hit; ++a) {
      hit = pc.bmin[a] == c.bbox_min[a] && pc.bmax[a] == c.bbox_max[a];
      if (hit && other) hit = pc.obmin[a] == other->bbox_min[a] && pc.obmax[a] == other->bbox_max[a];
    }
    if (hit) h_target = pc.h_target;
    bool have = false;
    double h_used = h_target;
    for (int iter = 0; iter < 4; ++iter) {
      Lattice cand;
      double v; int m;
      const bool ok = choose_lattice(c, other, v_req, h_target, budget, sp, &v, &m, &cand);
      if (!ok) {
        if (have) break;      // the refined edge does not fit: keep the lattice of the previous iteration
        if (c.bbox_spec) return restart(nullptr);
        return fail(ctx, ME_ERR_RANGE, v_req > 0 ? "voxel size too small for the lattice (dense budget and sparse limits exceeded)"
                                                 : "cannot fit the cloud into the lattice");
      }
      if (have && cand.sparse == L.sparse && cand.m == L.m && cand.v == L.v && cand.dims[0] == L.dims[0]) break;   // refinement changed nothing
      L = cand; have = true;
      h_used = h_target;
      ctx->spec_v = v; ctx->spec_m = m;
      if (L.sparse && c.bbox_spec) return restart(nullptr);
      if (L.sparse) { ME_TRY(build_sparse(ctx, c, L, &occupied)); built = true; }
      else { built = false; scanned = false; ME_TRY(histogram(ctx, c, L)); }
      if (ctx->nn_cell_size > 0) break;   // caller fixed the cell size
      if (hit && L.sparse == pc.lat.sparse && L.m == pc.lat.m && L.v == pc.lat.v && L.dims[0] == pc.lat.dims[0] &&
          L.dims[1] == pc.lat.dims[1] && L.dims[2] == pc.lat.dims[2])
        break;                            // the remembered lattice: no need to measure the occupancy again
      hit = false;
      if (!L.sparse) {
        ME_TRY(scan_cells(ctx, c, L));
        ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        scanned = true;
        occupied = (long long)((unsigned long long *)ctx->h_pinned)[9];
      }
      const double mean_occ = (double)c.n / (double)std::max<long long>(1, occupied);
      if (mean_occ <= 4.0 || iter == 3) break;
      // surface-like data: occupancy of occupied cells scales ~h^2; aim at ~2 points per occupied cell
      const double h_new = std::max(L.h * std::sqrt(2.0 / mean_occ), L.h * 0.25);
      if (h_new >= 0.9 * L.h) break;
      h_target = h_new;
    }
    if (hit && pc.slab_planned) {          // the slabs of this constellation
      ctx->slab_planned = true; ctx->slab_on = pc.slab_on; ctx->slab_axis = pc.slab_axis;
      ctx->slab_k0 = pc.slab_k0; ctx->slab_k1 = pc.slab_k1;
    }
    pc.valid = true;
    pc.n = c.n; pc.other_n = other ? other->n : -1;
    for (int a = 0; a < 3; ++a) {
      pc.bmin[a] = c.bbox_min[a]; pc.bmax[a] = c.bbox_max[a];
      pc.obmin[a] = other ? other->bbox_min[a] : 0.0; pc.obmax[a] = other ? other->bbox_max[a] : 0.0;
    }
    pc.v_req = v_req; pc.nn_cell = ctx->nn_cell_size; pc.budget = budget; pc.sp = sp; pc.slab_request = ctx->slab_request;
    pc.rank = ctx->rank; pc.world = ctx->world;
    pc.h_target = h_used; pc.lat = L;
    pc.slab_planned = false;               // filled in below, once the slabs are planned on this lattice
  }
  c.grid_solo = solo;
  c.solo_h = solo ? solo_h : 0.0;
  c.lat = L;

  c.slab = false;
  c.ns = c.n;
  c.n_owned = c.n;
  if (!built && !solo && slab_wanted(ctx)) {
    if (scanned) { ME_TRY(histogram(ctx, c, L)); scanned = false; }      // the slab cut and mask work on the counts
    if (!ctx->slab_planned) ME_TRY(plan_slabs(ctx, c, L));
    {
      PlanCache &pc = ctx->plan_cache[which];
      if (pc.valid && !pc.slab_planned && pc.lat.dims[0] == L.dims[0] && pc.lat.dims[1] == L.dims[1] && pc.lat.dims[2] == L.dims[2] &&
          pc.lat.m == L.m && pc.lat.v == L.v) {
        pc.slab_planned = true; pc.slab_on = ctx->slab_on; pc.slab_axis = ctx->slab_axis;
        pc.slab_k0 = ctx->slab_k0; pc.slab_k1 = ctx->slab_k1;
      }
    }
    if (ctx->slab_on) {
      slab_planes(ctx, L, c);
      unsigned long long *d_own = (unsigned long long *)ctx->d_scratch + 11;
      ME_CUDA(ctx, cudaMemsetAsync(d_own, 0, sizeof(unsigned long long), ctx->stream));
      const int mb = (int)std::min<long long>((L.ncells + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
      slab_mask_kernel<<<mb, kThreads, 0, ctx->stream>>>(c.d_cell_off, L.ncells, L.dims[0], L.dims[1], c.sl_axis, c.sc_lo, c.sc_hi,
                                                        c.so_lo, c.so_hi, d_own);
      ME_LAUNCH_CHECK(ctx);
      c.slab = true;
    }
  } else if (built && !solo && slab_wanted(ctx)) {
    // a sparse lattice is laid out whole: the pass falls back to replicated lattices (the other cloud is laid out again)
    if (getenv("ME_DEBUG_SLAB")) fprintf(stderr, "[mapeval] slab plan: rank %d sparse cell table, replicated layout\n", ctx->rank);
    ctx->slab_planned = true;
    if (ctx->slab_on) {
      ctx->slab_on = false;
      if (o.slab && o.grid_valid) { o.grid_valid = false; o.nn_valid = false; o.entropy_valid = false; }
    }
  }
  if (!built) {
    if (!scanned) ME_TRY(scan_cells(ctx, c, L));
    ME_TRY(ensure(ctx, (void **)&c.d_sorted, &c.cap_sorted, c.n, sizeof(P4)));
    ME_TRY(ensure(ctx, (void **)&c.d_rel, &c.cap_rel, c.n, sizeof(float4)));
    int blocks = (int)std::min<long long>((c.n + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
    scatter_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.d_xyz, c.n, L, c.d_cell_off, ctx->d_rank, c.d_sorted,
                                                        c.slab ? c.sl_axis : 0, c.sc_lo, c.sc_hi);
    ME_LAUNCH_CHECK(ctx);
    if (c.slab) {
      // the last entry of the CSR array = the points laid out here
      uint32_t *h_sl = (uint32_t *)((unsigned long long *)ctx->h_pinned + 16);
      unsigned long long *h_own = (unsigned long long *)ctx->h_pinned + 11;
      ME_CUDA(ctx, cudaMemcpyAsync(h_sl, c.d_cell_off + L.ncells, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
      ME_CUDA(ctx, cudaMemcpyAsync(h_own, (unsigned long long *)ctx->d_scratch + 11, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
      ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
      c.ns = (long long)h_sl[0];
      c.n_owned = (long long)*h_own;
    }
    {
      const int rb = (int)std::min<long long>((c.ns + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
      rel_kernel<<<std::max(1, rb), kThreads, 0, ctx->stream>>>(c.d_sorted, c.ns, L, c.d_rel);
      ME_LAUNCH_CHECK(ctx);
    }
    ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    c.max_cell_count = (long long)((unsigned long long *)ctx->h_pinned)[10];
    if (c.bbox_spec) {      // the box the histogram measured (scan_cells brought it back with the statistics)
      const unsigned long long *h = (const unsigned long long *)ctx->h_pinned;
      bool same = h[6] == 0;
      for (int k = 0; k < 3; ++k) same = same && h[k] == enc_ordered(c.bbox_min[k]) && h[3 + k] == enc_ordered(c.bbox_max[k]);
      if (!same) return restart(h);
      c.bbox_spec = false;
      trace_kernel(ctx, ME_TEV_BOX_REMEMBERED);
    }
    if (!solo && !c.slab) {      // the box a later build of this cloud may start from
      c.last_box_valid = true;
      c.last_box_n = c.n;
      for (int k = 0; k < 3; ++k) { c.last_bmin[k] = c.bbox_min[k]; c.last_bmax[k] = c.bbox_max[k]; }
    }
  }
  ME_TRY(build_coarse(ctx, c));
  c.tiles_valid = false;
  c.shard_valid = false;
  c.grid_valid = true;
  c.nn_valid = false;
  c.entropy_valid = false;
  return ME_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Open3D PointCloud::Transform (map_eval.cpp:1206): p' = (T [p,1]).head<3>() / w, in place on the caller-order array
// ---------------------------------------------------------------------------------------------------------------
struct Mat16 { double t[16]; };
__global__ void __launch_bounds__(kThreads) transform_kernel(double *__restrict__ xyz, long long n, Mat16 T) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2], o[4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
      o[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T.t[r * 4], x), __dmul_rn(T.t[r * 4 + 1], y)),
                                 __dmul_rn(T.t[r * 4 + 2], z)), T.t[r * 4 + 3]);
    xyz[3 * i] = __ddiv_rn(o[0], o[3]);
    xyz[3 * i + 1] = __ddiv_rn(o[1], o[3]);
    xyz[3 * i + 2] = __ddiv_rn(o[2], o[3]);
  }
}

// PointCloud::TransformNormals: n' = T.block<3,3>(0,0) n, every product and sum rounded like Eigen's product in a build
// without FMA, in the order of transform_kernel: (T0 x + T1 y) + T2 z.  The plain expression would be contracted to FMAs.
__global__ void __launch_bounds__(kThreads) rotate_normals_kernel(double *__restrict__ nrm, long long n, Mat16 T) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double x = nrm[3 * i], y = nrm[3 * i + 1], z = nrm[3 * i + 2];
#pragma unroll
    for (int r = 0; r < 3; ++r)
      nrm[3 * i + r] = __dadd_rn(__dadd_rn(__dmul_rn(T.t[r * 4], x), __dmul_rn(T.t[r * 4 + 1], y)), __dmul_rn(T.t[r * 4 + 2], z));
  }
}

int transform_cloud(me_ctx *ctx, int which, const double T[16]) {
  Cloud &c = ctx->cloud[which];
  if (c.n <= 0) return fail(ctx, ME_ERR_EMPTY, "cloud is empty");
  if (!c.owned) return fail(ctx, ME_ERR_INVALID, "me_transform needs a library-owned cloud (use me_set_cloud)");
  ME_TRY(wait_upload(ctx, which));
  Mat16 M;
  std::memcpy(M.t, T, sizeof(M.t));
  int blocks = (int)std::min<long long>((c.n + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
  transform_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.d_xyz, c.n, M);
  ME_LAUNCH_CHECK(ctx);
  if (c.normal_valid) {      // Open3D's PointCloud::Transform moves the normals along
    rotate_normals_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.d_normal, c.n, M);
    ME_LAUNCH_CHECK(ctx);
  }
  invalidate_cloud(c);
  return ME_OK;
}

}  // namespace me

// common.cuh — context, lattice and device helpers shared by the kernels of libmapeval_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>
#include "../../include/mapeval_b200.h"

namespace me {

// One point of a cell-sorted cloud: absolute fp64 coordinates (the reference's storage type,
// std::vector<Eigen::Vector3d>) + a tag: low 32 bits = index the point had in the caller's array, high 32 bits =
// lattice cell of the point.  32 B, so a point is two aligned 16-byte loads (and a valid TMA bulk-copy unit).
struct __align__(32) P4 {
  double x, y, z;
  long long idx;
};
__host__ __device__ __forceinline__ int orig_of(long long tag) { return (int)(tag & 0xffffffffll); }
__host__ __device__ __forceinline__ unsigned int cell_of(long long tag) { return (unsigned int)((unsigned long long)tag >> 32); }

static constexpr int kTileEdge = 4;   // query tiles are kTileEdge^3 cells
static constexpr int kFeatureSlot = 2;   // me_ctx::cloud[kFeatureSlot + which]: feature cloud of global registration

// Dense lattice of a cloud.  Cells are cubes of edge h = v / m whose boundaries coincide with the voxel
// boundaries floor(x / v) of the reference (voxel_calculator.cpp:241-245): every cell belongs to exactly one
// voxel, so the voxel stage needs no hashing and no atomics.  Without a voxel size v := h, m := 1.
struct Lattice {
  double v;          // voxel edge
  double h;          // cell edge = v / m
  double m_over_v;   // m / v
  int m;             // cells per voxel edge
  int k_lo[3];       // lowest voxel index per axis (floor(min / v))
  int nvox[3];       // voxels per axis
  int dims[3];       // cells per axis = nvox * m
  int nb[3];         // tiles (kTileEdge^3 cells) per axis
  long long ncells;  // dense table only
  long long nvoxels;
  int sparse;        // 1: the cell table holds occupied row segments only (CellIndex below)
  int nsegx;         // sparse: segments of kSegCells cells per lattice row = ceil(dims[0] / kSegCells)
};

// Cell table of a lattice = CSR offsets into the cell-sorted cloud, cells in (z, y, x) order, so that x-adjacent cells are
// adjacent in the cloud and the run of cells [xa, xb] of one lattice row is one contiguous range of points.
//   dense : off[c] for every cell c (ncells + 1 entries) — scenes whose bounding box fits the cell budget
//   sparse: every lattice row is cut into segments of 32 cells along x; only OCCUPIED segments are stored, still in
//           (z, y, x) order — off[rank * 32 + (x & 31)] — and an open-addressing hash table maps the segment key
//           (row * nsegx + x / 32) to its rank.  Site-scale surface scans keep ~2 points per occupied cell whatever
//           the extent; the point order, and with it every run-walking kernel, is the same as in the dense case.
static constexpr int kSegCells = 32;
struct CellIndex {
  const uint32_t *off;
  const unsigned long long *hkey;   // sparse: hash slots, ~0 = empty (linear probing)
  const uint32_t *hval;             // rank of the segment
  uint32_t hmask;                   // slots - 1
  int nsegx;
  int sparse;
  int dimx, dimy, dimz;
};

struct Cloud {
  long long n = 0;
  long long ns = 0;             // points in the sorted arrays: n, or the points of this rank's slab (+ halo) in slab mode
  // slab layout: only the lattice planes [sc_lo, sc_hi) along lattice axis sl_axis (1: y, 2: z) are laid out here, and this
  // rank owns the queries of the planes [so_lo, so_hi) — n_owned points; the sweeps skip the halo points
  bool slab = false;
  int sl_axis = 0, so_lo = 0, so_hi = 0, sc_lo = 0, sc_hi = 0;
  long long n_owned = 0;
  double *d_xyz = nullptr;      // caller order, fp64 AoS
  bool owned = false;
  long long cap_xyz = 0;
  bool grid_valid = false;
  bool grid_solo = false;       // the lattice is this cloud's own (MME with a large radius), not the shared voxel-aligned one
  double solo_h = 0.0;
  double bbox_min[3], bbox_max[3];
  bool bbox_valid = false;
  // bbox_spec: bbox_min/max hold the box of the last shared dense build (last_box), not yet measured; the next build
  // measures the box on the way (cell_count_kernel) and lays the cloud out again if it differs (bbox_missed).  last_box is
  // kept across me_set_cloud* and dropped when the library moves the points (invalidate_cloud)
  bool bbox_spec = false, bbox_missed = false;
  bool last_box_valid = false;
  long long last_box_n = 0;
  double last_bmin[3], last_bmax[3];
  Lattice lat;
  P4 *d_sorted = nullptr;       // cell-sorted points
  long long cap_sorted = 0;
  float4 *d_rel = nullptr;      // cell-sorted fp32 screening copy: xyz relative to the point's own cell origin, w = (float)ix
  long long cap_rel = 0;
  uint32_t *d_cell_off = nullptr;   // dense: ncells + 1 CSR offsets into d_sorted: cell c = [off[c], off[c+1]); sparse: nseg * 32 + 1
  long long cap_cells = 0;
  uint32_t *d_coarse = nullptr;     // point counts of coarse cells (coarse_f^3 lattice cells each): lets far queries skip empty space
  long long cap_coarse = 0;
  int coarse_f = 0;                 // 0: no coarse grid (small lattices)
  int coarse_dims[3] = {0, 0, 0};
  unsigned long long *d_hkey = nullptr;   // sparse lattice: segment hash table (CellIndex)
  uint32_t *d_hval = nullptr;
  long long cap_hash = 0;
  uint32_t hmask = 0;
  long long n_seg = 0;
  uint32_t *d_tiles = nullptr;      // non-empty query tiles (tile id = (bz*nb[1]+by)*nb[0]+bx)
  long long cap_tiles = 0;
  long long n_tiles = 0;
  bool tiles_valid = false;
  uint32_t *d_tile_pos = nullptr;   // tile-list build scratch (flags -> positions)
  long long cap_tile_pos = 0;
  long long shard_b = 0, shard_e = 0;   // this rank's cell-aligned query range (query_shard)
  int shard_rank = -1, shard_world = 0;
  bool shard_valid = false;
  long long nn_b = 0, nn_e = 0;         // sorted range of the queries the last NN sweep may have filled (others: -2)
  long long max_cell_count = 0;     // points in the fullest cell
  cudaEvent_t upload_done = nullptr;  // recorded on the copy stream after me_set_cloud's H2D
  bool upload_pending = false;
  // per-query results, SORTED order of this cloud (unsorted on demand)
  int32_t *d_nn_idx = nullptr;      // nearest neighbour in the other cloud (caller index there)
  double *d_nn_d2 = nullptr;        // squared distance as nanoflann accumulates it (cut-off tests, full Chamfer)
  double *d_nn_sq = nullptr;        // squared norm as Eigen accumulates it (inlier statistics)
  long long cap_nn = 0, cap_nn_d2 = 0, cap_nn_sq = 0;
  bool nn_valid = false;
  double *d_entropy = nullptr;      // sorted order of the lattice the MME sweep ran on
  long long cap_entropy = 0;
  bool entropy_valid = false;
  double *d_entropy_caller = nullptr;   // caller order, kept when the sweep ran on a solo lattice (which the next build replaces)
  long long cap_entropy_caller = 0;
  bool entropy_caller_valid = false;
  uint32_t *d_fp64_list = nullptr;      // MME: sorted indices of the queries left to the fp64 finish
  long long cap_fp64_list = 0;
  double *d_normal = nullptr;           // caller order, 3 fp64 per point: normals (me_set_normals / me_estimate_normals, averaged
  long long cap_normal = 0;             // by me_voxel_downsample); the working k-NN normals of generalized ICP when !normal_valid
  bool normal_valid = false;
};

// Lattice planning is data dependent (the cell edge is refined on the measured occupancy; the slabs are cut on the layer
// histogram) and costs extra histogram passes and host round trips.  The outcome for one (cloud, other cloud, settings)
// constellation is remembered: evaluating a cloud pair of the same sizes and bounding boxes again — repeated passes over the
// same maps — re-uses it.  The plan only steers performance; results do not depend on it.
struct PlanCache {
  bool valid = false;
  // key
  long long n = 0, other_n = -1;
  double bmin[3], bmax[3], obmin[3], obmax[3];
  double v_req = 0, nn_cell = 0;
  long long budget = 0;
  bool sp = false, slab_request = false;
  int rank = 0, world = 1;
  // value
  double h_target = 0;
  Lattice lat;
  bool slab_planned = false, slab_on = false;
  int slab_axis = 0;
  long long slab_k0 = 0, slab_k1 = 0;
};

// an open registration (me_icp_begin .. me_icp_end, icp.cu): the loop state, identical on every rank
struct IcpRun {
  bool open = false;
  int method = 0, max_iter = 0;
  double max_dist = 0, rel_fitness = 0, rel_rmse = 0;
  double T[16];                       // accumulated transformation (T_init included)
  double c[3] = {0, 0, 0};            // point-to-point: the point the sums are taken about (centre of the gt bounding box)
  double *orig = nullptr;             // the estimated cloud as handed in
  long long cap_orig = 0;
  const double *xyz = nullptr;        // the estimated cloud's buffer and size at me_icp_begin
  long long n_est = 0;
  bool had_normals[2] = {false, false};       // the clouds' own normals
  bool normals_pending[2] = {false, false};   // generalized ICP: k-NN normals not estimated yet (me_icp_normals_slice)
  bool swept = false;                 // the initial sweep ran (first me_icp_block)
  bool have_prev = false, done = false;
  double fitness = 0, rmse = 0;       // of the last block me_icp_step read
  long long n_corr = 0;
  int it = 0, converged = 0;
};

// numpy's method="linear" position of probability p among n sorted values: h = (n - 1) p, k = floor(h), g = h - k.  Also
// called on the device (mom_region.cu): a device caller is compiled with -fmad=false, so that it rounds every operation as the
// host does.
__host__ __device__ inline void quantile_rank(long long n, double p, long long *k, double *g) {
  const double h = (double)(n - 1) * p;
  const double f = std::floor(h);
  *k = (long long)f;
  *g = h - f;
}
// numpy's _lerp in its operation order: lo + (hi - lo) g below g = 0.5, hi - (hi - lo) (1 - g) from there
__host__ __device__ inline double quantile_lerp(double lo, double hi, double g) {
  const double diff = hi - lo;
  return g >= 0.5 ? hi - diff * (1.0 - g) : lo + diff * g;
}

// exact order statistics by radix selection over 64-bit keys (the bit patterns of finite doubles >= 0), the same loop on
// every rank: pass j histograms digit j (8 bits, most significant first) of the keys under each slot's prefix; the host
// reads the reduced counts and fixes digit j of every target rank.  Slot s of a population is one distinct prefix (the key
// bits the passes so far fixed) that some target rank still lies under.  P populations are selected side by side: the two
// directions of me_nn_quantile* (nn.cu), the three plane families of me_mom* (mom.cu).
static constexpr int kQuantSlots = 2 * ME_QUANTILE_MAX_PROBS + 2;   // ranks k and k + 1 per probability, then 0 and n - 1
static constexpr int kQuantBins = 256;                               // 8-bit digits
static constexpr int kQuantPasses = 8;                               // 64-bit keys
static constexpr int kQuantBlock = 2 * kQuantSlots * kQuantBins;     // fp64 counts per pass: [direction][slot][digit]
template <int P, int Slots>
struct RadixSel {
  int pass = 0;                        // the digit the next reduced histogram holds
  long long n[P] = {};                 // population sizes
  int n_targets[P] = {};
  long long rank[P][Slots];            // target ranks in the sorted population
  long long resid[P][Slots];           // rank of the target among the keys under its prefix
  unsigned long long key[P][Slots];    // the prefix of the target: the digits fixed so far, lower bits zero
  int n_slots[P] = {};
  unsigned long long slot_pfx[P][Slots];   // distinct prefixes of the running pass, ascending

  // population q of nq keys (before pass 0): the target ranks k and k + 1 of numpy's linear quantile per probability p[0..K-1],
  // then 0 and nq - 1; one slot, the empty prefix.  nq = 0: no targets, no slot
  void set_targets(int q, long long nq, const double *p, int K) {
    n[q] = nq;
    n_targets[q] = 0;
    n_slots[q] = 0;
    if (nq <= 0) return;
    int t = 0;
    for (int k = 0; k < K; ++k) {
      long long kk;
      double g;
      quantile_rank(nq, p[k], &kk, &g);
      rank[q][t++] = kk;
      rank[q][t++] = kk + 1 < nq - 1 ? kk + 1 : nq - 1;
    }
    rank[q][t++] = 0;
    rank[q][t++] = nq - 1;
    n_targets[q] = t;
    for (int i = 0; i < t; ++i) { resid[q][i] = rank[q][i]; key[q][i] = 0; }
    n_slots[q] = 1;
    slot_pfx[q][0] = 0;
  }
  // digit `pass` of every target of population q from its reduced counts rows[slot * kQuantBins + digit]; false when a
  // target's rank does not lie under the rows (a block not SUM-reduced over all ranks, or of another selection)
  bool take_digits(int q, const double *rows) {
    const int shift = 56 - 8 * pass;
    for (int i = 0; i < n_targets[q]; ++i) {
      const unsigned long long top = pass == 0 ? 0 : key[q][i] >> (shift + 8);
      int s = 0;                       // first slot with prefix >= top
      while (s < n_slots[q] && slot_pfx[q][s] < top) ++s;
      if (s >= n_slots[q]) return false;
      const double *row = rows + (size_t)s * kQuantBins;
      long long below = 0;
      int d = 0;
      for (; d < kQuantBins; ++d) {
        const long long c = (long long)row[d];
        if (resid[q][i] < below + c) break;
        below += c;
      }
      if (d == kQuantBins) return false;
      resid[q][i] -= below;
      key[q][i] |= (unsigned long long)d << shift;
    }
    return true;
  }
  // after the digits of every population: the distinct prefixes of the next pass, ascending
  void next_pass() {
    ++pass;
    for (int q = 0; q < P; ++q) {
      if (!n_slots[q]) continue;
      unsigned long long *s = slot_pfx[q];
      for (int i = 0; i < n_targets[q]; ++i) s[i] = key[q][i] >> (64 - 8 * pass);
      std::sort(s, s + n_targets[q]);
      n_slots[q] = (int)(std::unique(s, s + n_targets[q]) - s);
    }
  }
  // the order statistic of rank r of population q once every pass ran, one of the targets (NaN otherwise)
  double value(int q, long long r) const {
    for (int i = 0; i < n_targets[q]; ++i)
      if (rank[q][i] == r) {
        double v;
        std::memcpy(&v, &key[q][i], sizeof(v));
        return v;
      }
    return (double)NAN;
  }
};

// exact distance quantiles (me_nn_quantile_begin .. me_nn_quantile_end, nn.cu): radix selection over the NN records of
// both directions
struct QuantRun {
  bool open = false, done = false;
  unsigned long long gen = 0;          // cloud_gen at me_nn_quantile_begin
  int population = 0, K = 0, dirs = 0;
  double p[ME_QUANTILE_MAX_PROBS];
  RadixSel<2, kQuantSlots> sel;        // the targets of both directions; sel.pass: the digit the running pass histograms
  long long kb[2] = {0, 0}, ke[2] = {0, 0};      // the record range the keys cover
  unsigned long long *d_keys[2] = {nullptr, nullptr};
  long long cap_keys[2] = {0, 0};
  unsigned long long *d_hist = nullptr;          // integer histogram of the running pass, kQuantBlock counts
  double *d_blk = nullptr;                       // the same as fp64: the SUM-reducible block
  unsigned long long *d_pfx = nullptr;           // slot_pfx on the device
  std::vector<double> h_blk;
};

// the mutually orthogonal metric (me_mom_begin .. me_mom_end, mom.cu): the per-point values of the last call per cloud, the
// loop state (the same on every rank) and the block, ME_MOM_BLOCK fp64 values in every pass
static constexpr int kMomSlots = 4;     // ranks k and k + 1 of the median, then 0 and n - 1
struct MomRun {
  bool open = false, done = false;
  unsigned long long gen = 0;          // cloud_gen at me_mom_begin
  int which = 0, min_neighbors = 0, rings = 0, solo = 0;
  double radius = 0.0, angle_deg = 0.0, planarity = 0.0, cos_a = 0.0;
  long long min_family = 0;
  int stage = 0;                       // what the block holds: 0 the direction histogram, 1 the fold and digit 0, 2.. digit stage - 1
  bool ended = false;                  // me_mom_end filled the result of this call (the per-region breakdown reads it)
  long long n_query = 0, n_pv = 0, n_planar = 0;
  int status = 0;
  double axes[9];
  long long n_fam[3] = {0, 0, 0};
  double sum_v[3] = {0, 0, 0};
  RadixSel<3, kMomSlots> sel;
  long long keys_local[3] = {0, 0, 0};    // this rank's members per family: its keys, family by family, in d_keys
  long long kb = 0, ke = 0;            // this rank's sorted query range
  unsigned long long *d_hist = nullptr;   // ME_MOM_BLOCK integer counts, then the block as fp64, the slot prefixes, 3 counters
  double *d_blk = nullptr;
  unsigned long long *d_pfx = nullptr, *d_ctr = nullptr;
  double *d_fold = nullptr;            // this rank's fold: n_j, sum_v_j
  double *d_part = nullptr;            // the fold's per-chunk values
  long long cap_part = 0;
  unsigned long long *d_keys = nullptr;   // v of this rank's family members, family by family
  long long cap_keys = 0;
  std::vector<double> h_blk;
  // per cloud, caller order: v, lambda2, the unit normal and a flag byte (1 evaluated, 2 v valid, 4 planar, family + 1 in bits 3..4)
  double *d_v[2] = {nullptr, nullptr}, *d_l2[2] = {nullptr, nullptr}, *d_n[2] = {nullptr, nullptr};
  uint8_t *d_flag[2] = {nullptr, nullptr};
  long long cap_v[2] = {0, 0}, cap_l2[2] = {0, 0}, cap_n[2] = {0, 0}, cap_flag[2] = {0, 0};
  bool pts_valid[2] = {false, false};
  unsigned long long pts_gen[2] = {0, 0};
};

// the per-region breakdown of the last finished MOM call (me_mom_region_begin .. me_mom_region_end, mom_region.cu): the
// occupied list, the [v | code] block (2 n fp64, the same length on every rank) and the scratch of the segmented selection
struct MomRegionRun {
  bool open = false;
  unsigned long long gen = 0;          // cloud_gen at me_mom_region_begin
  int which = 0, status = 0;           // the MOM call's cloud and its whole-map status (before the family-size test)
  long long min_family = 0;
  double s = 0.0;
  long long R = 0, n = 0;              // listed regions; points of the cloud
  std::vector<int64_t> index, n_points;   // 3 per region; per region
  double *d_blk = nullptr;             // v of every planar point, then its code (0, family + 1, 4 planar without a family)
  long long cap_blk = 0;
  uint32_t *d_rid = nullptr;           // caller index -> region
  long long cap_rid = 0;
  unsigned long long *d_keys = nullptr;   // 3 n: the two buffers of the sort by v, then one of the sort by segment
  long long cap_keys = 0;
  uint32_t *d_vals = nullptr;          // 2 n
  long long cap_vals = 0;
  uint32_t *d_cnt = nullptr;           // segment counts (3 R + 1), planar counts (R), chunk counts (3 R + 1), the member counter
  long long cap_cnt = 0;
  double *d_out = nullptr;             // per segment: the median, then the sum of v
  long long cap_out = 0;
  double *d_part = nullptr;            // the fold's per-chunk sums
  long long cap_part = 0;
};

// the per-region table (me_nn_region_begin .. me_nn_region_end, region.cu): the occupied list and the block, the same
// length on every rank
struct RegionRun {
  bool open = false;
  unsigned long long gen = 0;          // cloud_gen at me_nn_region_begin
  double s = 0.0;
  long long n = 0;                     // occupied regions
  std::vector<int64_t> index, n_est, n_gt;   // 3 per region; per region
  double *d_blk = nullptr;             // SUM part (ME_REGION_SUM_FIELDS x 2 per region), then MAX part (ME_REGION_MAX_FIELDS x 2)
  long long cap_blk = 0;
  double *d_part = nullptr;            // the fold's per-chunk values
  long long cap_part = 0;
};

// the occupied regions floor(x / s) of est ++ gt, or of est alone (list_regions, region.cu).  The device arrays live in
// d_work until its next user: val = caller ids sorted by region (stable: caller order inside a region, est before gt),
// pos = the scanned heads (sorted point j lies in region pos[j + 1] - 1), seg[r] / est_end[r] = first sorted position and one
// past the last est point of region r (seg[R] = n), chunks = the scanned chunk counts per direction ((R + 1) each), pos_of =
// scratch for record_positions (max(n_est, n_gt) entries)
static constexpr int kRegionChunk = 1024;      // points per warp of the region folds (region.cu, drift.cu): the unit of `chunks`
struct RegionList {
  long long R = 0, n = 0;
  uint32_t *val = nullptr, *pos = nullptr, *pos_of = nullptr, *seg = nullptr, *est_end = nullptr, *chunks = nullptr;
  uint32_t n_chunks[2] = {0, 0};
  std::vector<int64_t> index, n_est, n_gt;   // 3 per region; per region
};

// an open drift loop (me_drift_begin .. me_drift_end, drift.cu): one point-to-point ICP per region of the estimated cloud,
// the same state on every rank
struct DriftRun {
  bool open = false;
  unsigned long long gen = 0;          // cloud_gen at me_drift_begin
  double s = 0, max_dist = 0, rel_fitness = 0, rel_rmse = 0;
  int max_iter = 0;
  long long R = 0, n_chunks = 0;
  const double *xyz = nullptr;         // the estimated cloud's buffer and size at me_drift_begin
  long long n_est = 0;
  double *orig = nullptr;              // the estimated cloud as handed in
  uint32_t *d_rid = nullptr;           // caller index -> region
  uint32_t *d_val = nullptr;           // caller ids sorted by region, caller order inside a region
  uint32_t *d_pos_of = nullptr;        // caller index -> record position after the last re-layout
  uint32_t *d_seg = nullptr;           // R + 1 first positions in d_val
  uint32_t *d_chunk_off = nullptr;     // R + 1 scanned chunk counts
  double *d_T = nullptr;               // 16 per region, row-major
  double *d_c = nullptr;               // 3 per region: the centre the sums are taken about
  double *d_blk = nullptr;             // ME_ICP_BLOCK_P2P per region
  double *d_part = nullptr;            // the fold's per-chunk values
  bool have_prev = false;
  std::vector<int64_t> index, n_est_r;
  std::vector<double> c, T, centroid, fitness, rmse, fitness0, rmse0;
  std::vector<int64_t> n_corr, n_corr0;
  std::vector<int32_t> it, status;     // status < 0: running
  std::vector<double> h_blk;
};

// point-to-plane metrics (me_nn_surface_begin .. me_nn_surface_end, surface.cu): one fold of the NN records, the same calls
// on every rank
struct SurfaceRun {
  bool open = false, done = false;     // done: the block holds this rank's fold
  unsigned long long gen = 0;          // cloud_gen at me_nn_surface_begin
  int knn = 0;
  bool had_normals[2] = {false, false};       // the clouds' own normals
  bool pending[2] = {false, false};           // working k-NN normals not estimated yet (me_nn_surface_normals_slice)
  double *d_blk = nullptr;             // ME_SURFACE_BLOCK_SUM SUM values, then ME_SURFACE_BLOCK_MAX MAX values
  double *d_part = nullptr;            // the fold's per-warp values
  long long cap_part = 0;
};

// local map consistency (me_consistency_begin .. me_consistency_end, consistency.cu): the per-point values of the last call
// per cloud, and the block of the open call, the same length on every rank
struct ConsistencyRun {
  bool open = false;
  unsigned long long gen = 0;          // cloud_gen at me_consistency_begin
  int which = 0, min_neighbors = 0, kernel = 0, rings = 0, solo = 0;
  double radius = 0.0, s = 0.0;
  long long R = 0;                     // listed regions (0 at s = 0: the block holds one, the whole map)
  std::vector<int64_t> index, n_points;   // 3 per region; per region
  double *d_blk = nullptr;             // ME_CONSISTENCY_SUM_FIELDS per region, then ME_CONSISTENCY_MAX_FIELDS per region
  long long cap_blk = 0;
  double *d_part = nullptr;            // the fold's per-chunk values
  long long cap_part = 0;
  // per cloud, caller order: entropy, plane variance and flags (1 evaluated here, 2 entropy valid, 4 plane variance valid)
  double *d_e[2] = {nullptr, nullptr}, *d_v[2] = {nullptr, nullptr};
  uint8_t *d_flag[2] = {nullptr, nullptr};
  long long cap_e[2] = {0, 0}, cap_v[2] = {0, 0}, cap_flag[2] = {0, 0};
  bool pts_valid[2] = {false, false};
  unsigned long long pts_gen[2] = {0, 0};   // cloud_gen when they were computed
};

}  // namespace me

struct me_ctx {
  int device = 0;
  int rank = 0, world = 1;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  double nn_cell_size = 0.0;
  long long max_grid_cells = 0;     // budget of the dense cell table; 0 = automatic (grid_budget)
  double voxel_hint = 0.0;          // lattice alignment requested by the voxel stage
  // slab layout (me_set_layout, world > 1, dense lattices): every rank lays out only the voxel layers it owns (+ a halo of
  // slab_halo cells) of both clouds instead of the whole clouds; planned from the layer histogram of the cloud that is laid
  // out first after the lattice spec was (re)planned — identical on every rank, the clouds being replicated
  bool slab_request = false, slab_planned = false, slab_on = false;
  int slab_axis = 0;                       // 1: y, 2: z
  long long slab_k0 = 0, slab_k1 = 0;      // owned world voxel layers [k0, k1) along slab_axis (LLONG_MIN/4, LLONG_MAX/4 at the ends)
  int slab_halo = 4;                       // cells; covers the 3 rings of an MME sweep on the shared lattice
  me::PlanCache plan_cache[2];
  // voxel stage split in two (me_voxel_begin / me_voxel_finish_accum_device): state kept between the halves
  bool vox_open = false;
  long long vox_nvox = 0;
  size_t vox_o_w = 0, vox_o_pairs = 0;
  // the W2 stage (me_w2_begin .. me_w2_fetch) keeps its tables in the same work buffer, so at most one of the two is open
  bool w2_open = false, w2_finished = false;
  void *d_w2 = nullptr;             // its accumulators and block (voxel.cu W2Dev), allocated on first use
  // lattice spec shared by both clouds, so that their cells coincide (same v, m; integer index offsets)
  double spec_v = 0.0;
  int spec_m = 0;
  cudaStream_t copy_stream = nullptr;   // H2D uploads run here and overlap kernels that do not need them yet
  cudaEvent_t compute_mark = nullptr;
  // [ME_CLOUD_EST], [ME_CLOUD_GT]: the clouds of the public calls; [kFeatureSlot + which]: the private feature clouds of global
  // registration (globalreg.cu), which no public `which` reaches
  me::Cloud cloud[4];
  float *d_fpfh[2] = {nullptr, nullptr};     // FPFH of the feature clouds, 33 per point
  long long cap_fpfh[2] = {0, 0};
  int32_t *d_corr = nullptr;                 // the last call's correspondences: est indices, then gt indices
  long long cap_corr = 0, n_corr = 0;
  bool features_valid = false;
  // small device scratch for reductions / accumulators
  void *d_scratch = nullptr;
  size_t scratch_bytes = 0;
  void *h_pinned = nullptr;         // pinned host mirror of the scratch
  void *stage = nullptr;            // pinned bounce buffers + streams of the pageable-memory upload path (api.cu)
  double *d_block = nullptr;        // device-resident accumulator block of the me_eval_*_accum* calls (kBlk* layout below)
  // large device scratch (scan partials, far list, voxel tables)
  void *d_work = nullptr;
  size_t work_bytes = 0;
  unsigned long long *d_scan_tmp = nullptr;   // tile status words of exclusive_scan_inplace
  long long cap_scan_tmp = 0;
  uint32_t *d_rank = nullptr;       // dense build: in-cell rank of every point of the cloud being laid out (caller order)
  long long cap_rank = 0;
  uint32_t *d_rs_hist = nullptr;    // radix sort: digit histograms of every tile
  long long cap_rs_hist = 0;
  cudaEvent_t ev[2 * ME_N_STAGE_TIMES];
  bool ev_used[ME_N_STAGE_TIMES];
  int sm_count = 132;
  long long launches = 0;
  // me_kernel_trace: sweep paths chosen on the host (1 << ME_KBIT_*), the last mme_rows_kernel configuration, and a device
  // word the far / brute kernels OR their bits into when a query reaches them
  unsigned long long kernel_mask = 0;
  int mme_rows_cfg = 0;
  unsigned int *d_trace = nullptr;
  me::IcpRun icp;
  // accuracy curve (me_nn_curve*): the records of the last me_eval_nn* serve it while no call has since moved, replaced or
  // re-swept a cloud — every such call bumps cloud_gen
  unsigned long long cloud_gen = 0;
  bool curve_valid = false;            // the last me_eval_nn* succeeded
  unsigned long long curve_gen = 0;    // cloud_gen at that call
  me_nn_params curve_p{};              // its parameters
  double *d_curve = nullptr;           // the curve block (both directions), then the levels
  long long cap_curve = 0;
  me::QuantRun quant;                  // distance quantiles (me_nn_quantile*), from the same records
  me::RegionRun region;                // the per-region table (me_nn_region*), from the same records
  me::DriftRun drift;                  // the per-region drift loop (me_drift*)
  me::SurfaceRun surface;              // point-to-plane metrics (me_nn_surface*), from the NN records
  me::ConsistencyRun consistency;      // local map consistency (me_consistency*): MPV and MME per region
  me::MomRun mom;                      // the mutually orthogonal metric (me_mom*)
  me::MomRegionRun mom_region;         // its per-region breakdown (me_mom_region*)
  std::string err;
};

namespace me {

int fail(me_ctx *ctx, int code, const std::string &msg);
int ensure(me_ctx *ctx, void **ptr, long long *cap, long long need, size_t elem);
int ensure_work(me_ctx *ctx, size_t bytes);

#define ME_CUDA(ctx, call)                                                                         \
  do {                                                                                             \
    cudaError_t e__ = (call);                                                                      \
    if (e__ != cudaSuccess)                                                                        \
      return me::fail((ctx), ME_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e__));    \
  } while (0)

#define ME_TRY(expr)                \
  do {                              \
    int rc__ = (expr);              \
    if (rc__ != ME_OK) return rc__; \
  } while (0)

#define ME_LAUNCH_CHECK(ctx)                                                                       \
  do {                                                                                             \
    (ctx)->launches++;                                                                             \
    cudaError_t e__ = cudaGetLastError();                                                          \
    if (e__ != cudaSuccess)                                                                        \
      return me::fail((ctx), ME_ERR_CUDA, std::string("kernel launch: ") + cudaGetErrorString(e__)); \
  } while (0)

// me_kernel_trace: the sweep path `bit` (ME_KBIT_*) was launched
inline void trace_kernel(me_ctx *ctx, int bit) { ctx->kernel_mask |= 1ull << bit; }

// contiguous range r of W over n items (tile lists; the point ranges of the sweeps come from query_shard, which snaps
// them to cell boundaries)
inline void shard_range(const me_ctx *ctx, long long n, long long *b, long long *e) {
  *b = n * ctx->rank / ctx->world;
  *e = n * (ctx->rank + 1) / ctx->world;
}

struct StageTimer {
  me_ctx *ctx; int stage;
  // s < 0: not timed (the lattices of the feature clouds of global registration)
  StageTimer(me_ctx *c, int s) : ctx(c), stage(s) { if (s >= 0) cudaEventRecord(c->ev[2 * s], c->stream); }
  ~StageTimer() { if (stage >= 0) { cudaEventRecord(ctx->ev[2 * stage + 1], ctx->stream); ctx->ev_used[stage] = true; } }
};

// the queries a sweep evaluates: all of [q_begin, q_end), or in slab layout those whose cell lies in the owned planes
struct Owned {
  int axis;      // 0: everything, 1: y, 2: z
  int lo, hi;
};
__host__ __device__ inline bool owns(const Owned &o, int iy, int iz) {
  if (o.axis == 0) return true;
  const int a = o.axis == 1 ? iy : iz;
  return a >= o.lo && a < o.hi;
}
inline Owned owned_of(const Cloud &c) {
  Owned o;
  o.axis = c.slab ? c.sl_axis : 0; o.lo = c.so_lo; o.hi = c.so_hi;
  return o;
}

// coarse occupancy grid of a lattice (grid.cu build_coarse): cnt[(cz * cd[1] + cy) * cd[0] + cx] points in the block of f^3 cells
struct CoarseGrid {
  const uint32_t *cnt;      // nullptr: none
  int f;
  int cd[3];
};
inline CoarseGrid coarse_of(const Cloud &c) {
  CoarseGrid g;
  g.cnt = c.coarse_f > 0 ? c.d_coarse : nullptr;
  g.f = c.coarse_f;
  for (int a = 0; a < 3; ++a) g.cd[a] = c.coarse_dims[a];
  return g;
}

inline CellIndex index_of(const Cloud &c) {
  CellIndex I;
  I.off = c.d_cell_off; I.hkey = c.d_hkey; I.hval = c.d_hval; I.hmask = c.hmask;
  I.nsegx = c.lat.nsegx; I.sparse = c.lat.sparse;
  I.dimx = c.lat.dims[0]; I.dimy = c.lat.dims[1]; I.dimz = c.lat.dims[2];
  return I;
}

// stage entry points (implemented in grid.cu / nn.cu / mme.cu / voxel.cu)
int wait_upload(me_ctx *ctx, int which);
int compute_bbox(me_ctx *ctx, int which);
int speculate_bbox(me_ctx *ctx, int which);
int build_grid(me_ctx *ctx, int which, double solo_h = 0.0);
double density_edge(const Cloud &c);
int build_both(me_ctx *ctx);
int build_tiles(me_ctx *ctx, int which);
int query_shard(me_ctx *ctx, int which, long long *b, long long *e);
int exclusive_scan_inplace(me_ctx *ctx, uint32_t *a, long long n, unsigned long long *stats = nullptr);
int voxel_downsample(me_ctx *ctx, int which, double voxel_size, int64_t *n_out);
int radix_sort_pairs(me_ctx *ctx, unsigned long long *keys, uint32_t *vals, unsigned long long *keys_tmp, uint32_t *vals_tmp,
                     long long n, int key_bits, unsigned long long **keys_sorted, uint32_t **vals_sorted);
// pack: the accumulators of every evaluated direction into its section of d_block; false: the per-query results only
// (d_nn_idx / d_nn_d2, registration)
int run_nn(me_ctx *ctx, const me_nn_params *p, bool pack);
int unsort_nn(me_ctx *ctx, int which_query, int32_t *h_idx, double *h_d2);
// the curve block of the last me_eval_nn* at the K levels tau (host memory, checked by the caller) — me_nn_curve_accum_device
int nn_curve(me_ctx *ctx, const double *tau, int K, double **device_block, int32_t *n);
// exact distance quantiles of the last me_eval_nn*'s records (arguments checked by the caller) — me_nn_quantile_*
int nn_quantile_begin(me_ctx *ctx, int population, const double *p, int K);
int nn_quantile_block(me_ctx *ctx, double **device_block, int32_t *n);
int nn_quantile_step(me_ctx *ctx, int32_t *done);
int nn_quantile_end(me_ctx *ctx, me_quantile_result *out);
void nn_quantile_free(me_ctx *ctx);
// the per-region table of the last me_eval_nn*'s records (region_size checked by the caller) — me_nn_region_* (region.cu)
int nn_region_begin(me_ctx *ctx, double s, int64_t *n_regions);
int nn_region_block(me_ctx *ctx, double **device_block, int32_t *n_sum, int32_t *n_max);
int nn_region_end(me_ctx *ctx, me_region_row *rows, int64_t capacity);
void nn_region_free(me_ctx *ctx);
int list_regions(me_ctx *ctx, const char *who, double s, bool with_gt, RegionList *L);
// rid[i] = the region of point i of cloud `which` in the list L (which must be listed)
int region_ids(me_ctx *ctx, const RegionList &L, int which, uint32_t *rid);
int record_positions(me_ctx *ctx, int which, uint32_t *pos_of);
// one point-to-point ICP per region of the estimated cloud (arguments checked by the caller) — me_drift_* (drift.cu)
int drift_begin(me_ctx *ctx, double s, double max_dist, int max_iter, double rel_fitness, double rel_rmse, int64_t *n_regions);
int drift_block(me_ctx *ctx, double **device_block, int32_t *n_sum);
int drift_step(me_ctx *ctx, int32_t *done);
int drift_end(me_ctx *ctx, me_drift_row *rows, int64_t capacity);
void drift_close(me_ctx *ctx, bool restore);
// point-to-plane metrics of the last me_eval_nn*'s records (knn checked by the caller) — me_nn_surface_* (surface.cu)
int nn_surface_begin(me_ctx *ctx, int knn);
int nn_surface_normals_slice(me_ctx *ctx, int which, double **d_normals, int64_t *slice_points, int32_t *pending);
int nn_surface_block(me_ctx *ctx, double **device_block, int32_t *n_sum, int32_t *n_max);
int nn_surface_end(me_ctx *ctx, me_surface_result *out);
void nn_surface_free(me_ctx *ctx);
// the accumulators go to the cloud's MME section of d_block
int run_mme(me_ctx *ctx, int which, double radius, int min_neighbors);
// dst[caller index] = src[sorted position] over the n points of a cell-sorted cloud (mme.cu)
__global__ void unsort_f64_kernel(const P4 *__restrict__ S, long long n, const double *__restrict__ src, double *__restrict__ dst);
// the lattice of the radius sweeps (MME and local consistency; mme.cu)
int radius_lattice(me_ctx *ctx, int which, double radius, bool *solo);
// local map consistency (me_consistency_*, consistency.cu; arguments checked by the caller)
int consistency_begin(me_ctx *ctx, int which, double radius, int min_neighbors, double s, int64_t *n_regions);
int consistency_block(me_ctx *ctx, double **device_block, int32_t *n_sum, int32_t *n_max);
int consistency_end(me_ctx *ctx, me_consistency_row *rows, int64_t capacity, me_consistency_result *whole);
int consistency_points(me_ctx *ctx, int which, double *entropy, double *plane_variance);
void consistency_free(me_ctx *ctx);
struct RadiusSweep {
  long long qb, qe;      // this rank's sorted query range
  int rings;
  float rc2;
};
int radius_sweep_layout(me_ctx *ctx, int which, double radius, const char *who, RadiusSweep *out);
// the mutually orthogonal metric (me_mom_*, mom.cu; arguments checked by the caller)
int mom_begin(me_ctx *ctx, int which, double radius, int min_neighbors, const me_mom_params *p);
int mom_block(me_ctx *ctx, double **device_block, int32_t *n);
int mom_step(me_ctx *ctx, int32_t *done);
int mom_end(me_ctx *ctx, me_mom_result *out);
int mom_points(me_ctx *ctx, int which, double *v, double *lambda2, double *normal, int8_t *family);
void mom_free(me_ctx *ctx);
// its per-region breakdown (me_mom_region_*, mom_region.cu; arguments checked by the caller)
int mom_region_begin(me_ctx *ctx, double s, long long min_family, int64_t *n_regions);
int mom_region_block(me_ctx *ctx, double **device_block, int64_t *n);
int mom_region_end(me_ctx *ctx, me_mom_region_row *rows, int64_t capacity);
void mom_region_free(me_ctx *ctx);

// layout of me_ctx::d_block (fp64): the SUM-reducible part first, then the MAX-reducible part.  Counts ride as fp64 (exact
// below 2^53, so their sums are exact and order-independent).
// per direction: n_query n_corr n_inlier[5] n_ub n_far | sum_d[5] sum_d2[5] sum_d_all sum_d2_all sum_nn |
// rank_n[W] rank_mean[W] rank_m2[W]
// (me_nn_accum; a rank fills only its own moment slot, so the SUM all-reduce gathers the slots)
static constexpr int kBlkNN = ME_NN_ACCUM_I64 + ME_NN_ACCUM_F64;
static constexpr int kBlkMoments = 22;               // offset of rank_n within a direction
static constexpr int kBlkMmeSum = 2 * kBlkNN;        // per cloud: n_query n_valid sum_entropy
static constexpr int kBlkAwd = kBlkMmeSum + 6;       // voxel stage: n_pairs n_scs n_voxels_est n_voxels_gt n_active n_new sum_w sum_scs
static constexpr int kBlkSumCount = kBlkAwd + 8;     // = 442 SUM values
static constexpr int kBlkMax = kBlkSumCount;         // per cloud: max_entropy, -min_entropy
static constexpr int kBlkMaxCount = 4;
static constexpr int kBlkTotal = kBlkSumCount + kBlkMaxCount;
int unsort_entropy(me_ctx *ctx, int which, double *h_entropy);
int run_awd(me_ctx *ctx, double voxel_size, int min_points, int scs_radius, me_awd_result *out, int64_t *n_rows,
            double **rows27);
// the voxel stage's eight values in the order of the block's AWD section -> the result (map_eval.cpp:324,387)
void awd_result(const double v[8], me_awd_result *out);
bool plan_lattice_host(const double bmin[3], const double bmax[3], long long n, const double *obmin, const double *obmax,
                       long long other_n, double v_req, double h_target, long long budget, bool allow_sparse, Lattice *out);
static constexpr double kSlabMaxShare = 0.75;      // a slab cut whose busiest rank lays out more than this share is not worth it
void slab_cut(const unsigned long long *planes_y, int n_planes_y, const unsigned long long *planes_z, int n_planes_z, int m,
              int world, int halo, int *axis_out, int *bounds, double *share_out);
int voxel_begin(me_ctx *ctx, double voxel_size, int min_points);
int voxel_w_table(me_ctx *ctx, double **d_w, int64_t *n);
int voxel_finish_block(me_ctx *ctx, int scs_radius);
// the Gaussian 2-Wasserstein stage (voxel.cu; ME_W2_BLOCK values in me_ctx::d_w2)
int run_w2(me_ctx *ctx, double voxel_size, int min_points, int scs_radius, me_w2_result *out, int64_t *n_rows, double **rows);
int run_w2_rows(me_ctx *ctx, const double *rows, int64_t n_rows, double voxel_size, int scs_radius, double *w_out,
                me_w2_result *out);
int w2_begin(me_ctx *ctx, double voxel_size, int min_points);
int w2_w_table(me_ctx *ctx, double **d_w, int64_t *n);
int w2_finish_block(me_ctx *ctx, int scs_radius);
int w2_block(me_ctx *ctx, double **d_block, int32_t *n);
int w2_fetch(me_ctx *ctx, me_w2_result *out);
int transform_cloud(me_ctx *ctx, int which, const double T[16]);
int run_icp(me_ctx *ctx, int method, double max_dist, int max_iter, double rel_fitness, double rel_rmse, const double T_init[16],
            me_icp_result *out);
int icp_begin(me_ctx *ctx, int method, double max_dist, int max_iter, double rel_fitness, double rel_rmse, const double T_init[16]);
int icp_normals_slice(me_ctx *ctx, int which, double **d_normals, int64_t *slice_points, int32_t *pending);
int icp_block(me_ctx *ctx, double **d_block, int32_t *n_sum);
int icp_step(me_ctx *ctx, int32_t *done);
int icp_end(me_ctx *ctx, me_icp_result *out);
void icp_close(me_ctx *ctx, bool restore);
void icp_update_host(int method, const double *blk, const double c[3], double upd[16]);
int estimate_normals(me_ctx *ctx, int which, int knn, long long lo = 0, long long hi = -1, long long cap_points = 0);
void invalidate_cloud(Cloud &c);      // the cloud's coordinates changed: bbox, lattice, NN and entropy results are stale
int run_awd_rows(me_ctx *ctx, const double *rows27, int64_t n_rows, double voxel_size, int scs_radius, double *w_out,
                 me_awd_result *out);
// degraded copies of a cloud (perturb.cu)
int copy_cloud(me_ctx *ctx, int src, int dst, bool with_normals = true);
int add_gaussian_noise(me_ctx *ctx, int which, double std_dev, uint64_t seed);
int add_non_uniform_density(me_ctx *ctx, int which, double sparse_ratio, double dense_ratio, double region_size, uint64_t seed,
                            int64_t *n_out);
int add_sparse_outliers(me_ctx *ctx, int which, double outlier_ratio, double outlier_range, uint64_t seed, int64_t *n_out);
int add_local_deformation(me_ctx *ctx, int which, double radius, double strength, const double center[3]);
// coarse global registration (globalreg.cu)
int global_registration(me_ctx *ctx, const me_global_reg_params *p, me_global_reg_result *out);
int get_features(me_ctx *ctx, int which, double *xyz, double *normals, float *fpfh33, int64_t capacity, int64_t *n);
int get_correspondences(me_ctx *ctx, int32_t *est_idx, int32_t *gt_idx, int64_t capacity, int64_t *n);

// ------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------

// squared distance exactly as nanoflann's L2_Adaptor accumulates it: ((dx*dx) + dy*dy) + dz*dz, no contraction
__device__ __forceinline__ double d2_kd(double ax, double ay, double az, double bx, double by, double bz) {
  double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by), dz = __dsub_rn(az, bz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}
// Eigen fixed-size squaredNorm: x*x + (y*y + z*z)
__device__ __forceinline__ double sqnorm_eigen(double dx, double dy, double dz) {
  return __dadd_rn(__dmul_rn(dx, dx), __dadd_rn(__dmul_rn(dy, dy), __dmul_rn(dz, dz)));
}

// lattice coordinate of one axis: voxel index floor(x / v) (IEEE division, as the reference) and the cell inside it
__device__ __forceinline__ long long cell_coord(double x, const Lattice &L, int axis) {
  double kf = floor(__ddiv_rn(x, L.v));
  double fx = __dsub_rn(x, __dmul_rn(kf, L.v));
  int s = (int)floor(fx * L.m_over_v);
  s = s < 0 ? 0 : (s >= L.m ? L.m - 1 : s);
  // clamp far-away queries before the integer conversion can overflow
  double kk = kf - (double)L.k_lo[axis];
  if (kk < -4.0e9) kk = -4.0e9;
  if (kk > 4.0e9) kk = 4.0e9;
  return (long long)kk * L.m + s;
}
// continuous cell coordinate (for face distances)
__device__ __forceinline__ double cell_coord_cont(double x, const Lattice &L, int axis) {
  return (x - (double)L.k_lo[axis] * L.v) / L.h;
}

// offset of coordinate x from the origin of lattice cell `ic` on `axis` (fp64; the caller rounds it to fp32).
// Origin = (k_lo + ic / m) * v + (ic % m) * h, the same products cell_coord() forms, so |offset| < ~h.
__device__ __forceinline__ double cell_rel(double x, uint32_t ic, const Lattice &L, int axis) {
  const uint32_t kv = ic / (uint32_t)L.m, s = ic - kv * (uint32_t)L.m;
  const double fx = __dsub_rn(x, __dmul_rn((double)(L.k_lo[axis] + (int)kv), L.v));
  return fx - (double)s * L.h;
}

__device__ __forceinline__ P4 load_p4(const P4 *p) {
  const double2 *q = reinterpret_cast<const double2 *>(p);
  double2 a = __ldg(q), b = __ldg(q + 1);
  P4 r;
  r.x = a.x; r.y = a.y; r.z = b.x; r.idx = __double_as_longlong(b.y);
  return r;
}

// ---- cell table access -------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t seg_hash(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 29;
  return (uint32_t)k;
}
__device__ __forceinline__ bool seg_find(const CellIndex &I, unsigned long long key, uint32_t &rank) {
  uint32_t h = seg_hash(key) & I.hmask;
  for (;;) {
    const unsigned long long k = __ldg(I.hkey + h);
    if (k == key) { rank = __ldg(I.hval + h); return true; }
    if (k == ~0ull) return false;
    h = (h + 1) & I.hmask;
  }
}
// points of the cells [xa, xb] of lattice row (y, z): [s, e) of the sorted cloud; the caller keeps 0 <= xa <= xb < dimx
// and the row inside the lattice
// SP: -1 = decide at run time (I.sparse), 0 / 1 = compile-time dense / sparse (the hot sweeps are instantiated for both, so
// the dense path carries no trace of the hash lookup)
template <int SP = -1>
__device__ __forceinline__ void cell_range(const CellIndex &I, int z, int y, int xa, int xb, uint32_t &s, uint32_t &e) {
  if (SP == 0 || (SP < 0 && !I.sparse)) {
    const uint32_t row = ((uint32_t)z * (uint32_t)I.dimy + (uint32_t)y) * (uint32_t)I.dimx;
    s = __ldg(I.off + row + (uint32_t)xa);
    e = __ldg(I.off + row + (uint32_t)xb + 1);
    return;
  }
  const unsigned long long rowkey = ((unsigned long long)z * (unsigned long long)I.dimy + (unsigned long long)y) * (unsigned long long)I.nsegx;
  const int ga = xa >> 5, gb = xb >> 5;
  s = 0; e = 0;
  bool have = false;
  for (int g = ga; g <= gb; ++g) {
    uint32_t r;
    if (!seg_find(I, rowkey + (unsigned long long)g, r)) continue;
    const uint32_t base = r << 5;
    if (!have) { s = __ldg(I.off + base + (g == ga ? (uint32_t)(xa & 31) : 0u)); have = true; }
    e = __ldg(I.off + base + (g == gb ? (uint32_t)(xb & 31) + 1u : 32u));
  }
}
// lattice cell of a point of the sorted cloud from its tag (dense: the cell id; sparse: the row id z * dimy + y, the x
// index comes from the cell-relative copy or from the coordinate)
__device__ __forceinline__ void cell_from_tag(const CellIndex &I, long long tag, int ix_if_sparse, int &ix, int &iy, int &iz) {
  const uint32_t t = cell_of(tag);
  if (I.sparse) { ix = ix_if_sparse; iy = (int)(t % (uint32_t)I.dimy); iz = (int)(t / (uint32_t)I.dimy); }
  else {
    ix = (int)(t % (uint32_t)I.dimx);
    const uint32_t cyz = t / (uint32_t)I.dimx;
    iy = (int)(cyz % (uint32_t)I.dimy); iz = (int)(cyz / (uint32_t)I.dimy);
  }
}

// order-preserving map double -> uint64 (for atomicMin/atomicMax on doubles)
__device__ __host__ __forceinline__ unsigned long long enc_ordered(double d) {
#ifdef __CUDA_ARCH__
  unsigned long long u = (unsigned long long)__double_as_longlong(d);
#else
  unsigned long long u; memcpy(&u, &d, 8);
#endif
  return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __host__ __forceinline__ double dec_ordered(unsigned long long u) {
  u = (u & 0x8000000000000000ull) ? (u & 0x7fffffffffffffffull) : ~u;
#ifdef __CUDA_ARCH__
  return __longlong_as_double((long long)u);
#else
  double d; memcpy(&d, &u, 8); return d;
#endif
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// Chan, Golub & LeVeque's pairwise update: (na, ma, m2a) <- the count, mean and sum of squared deviations of the union of
// two sets given those of each.  No cancellation: m2 only ever adds non-negative terms.
__host__ __device__ __forceinline__ void chan_merge(double &na, double &ma, double &m2a, double nb, double mb, double m2b) {
  if (nb == 0) return;
  const double n = na + nb, delta = mb - ma;
  ma += delta * (nb / n);
  m2a += m2b + delta * delta * (na * (nb / n));
  na = n;
}
__device__ __forceinline__ long long warp_sum_ll(long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Eigen 3x3 determinant (cofactor expansion, bruteforce_det3_helper); m row-major
__device__ __forceinline__ double det3(const double *m) {
  double a = m[0] * (m[4] * m[8] - m[5] * m[7]);
  double b = m[1] * (m[3] * m[8] - m[5] * m[6]);
  double c = m[2] * (m[3] * m[7] - m[4] * m[6]);
  return a - b + c;
}

}  // namespace me

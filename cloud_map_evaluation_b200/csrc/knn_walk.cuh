// knn_walk.cuh — the exact k-nearest-neighbour walk over a cell-sorted cloud, shared by the k-NN normals (icp.cu) and the
// FPFH neighbourhoods of global registration (globalreg.cu).
#pragma once
#include "common.cuh"

namespace me {

// The k best (d2, sorted position) pairs of query q among the points of S, kept sorted in the caller's per-thread slots
// dk[t * STRIDE], ik[t * STRIDE] (t < k); returns how many were found.  Ties go to the smaller caller index.  Only points
// with d2 < r2 are candidates (r2 = INFINITY: none is excluded), and with skip_self the point with q's caller index is not
// one.  The lattice is searched shell by shell (Chebyshev rings) until the k-th distance beats the distance to the border
// of the searched block, or that border lies beyond the radius; points far from everything go on to blocks of f^3 cells
// of the coarse occupancy grid, where empty blocks cost one load.  A query that goes on to those blocks sets
// ME_TEV_KNN_COARSE in me_kernel_trace's device word *trace (nullable): one lane per warp of the queries that enter the phase
// together, and none once the word carries the bit.  (A flag carried to the end of the kernel and voted there costs the
// FPFH kernels registers: fpfh_kernel's spills grew from 280 to 516 bytes.)
template <int STRIDE>
__device__ __forceinline__ int knn_walk(const P4 *__restrict__ S, const CellIndex &I, const Lattice &L, const CoarseGrid &CG,
                                        const P4 &q, int k, double slack, double r2, bool skip_self, double *dk, uint32_t *ik,
                                        unsigned int *trace) {
  int cix, ciy, ciz;
  long long xs = I.sparse ? cell_coord(q.x, L, 0) : 0;
  xs = xs < 0 ? 0 : (xs >= L.dims[0] ? L.dims[0] - 1 : xs);
  cell_from_tag(I, q.idx, (int)xs, cix, ciy, ciz);
  const long long ix = cix, iy = ciy, iz = ciz;
  const int self = orig_of(q.idx);
  int cnt = 0;
  double kth = INFINITY;
  // one candidate: keep the k best (d2, position) pairs sorted; ties go to the smaller caller index
  auto offer = [&](uint32_t j) {
    const P4 p = load_p4(S + j);
    const double d2 = d2_kd(q.x, q.y, q.z, p.x, p.y, p.z);
    if (!(d2 < r2)) return;
    if (skip_self && orig_of(p.idx) == self) return;
    if (cnt == k) {
      if (d2 > kth) return;
      if (d2 == kth && orig_of(p.idx) > orig_of(__double_as_longlong(__ldg(reinterpret_cast<const double *>(S + ik[(k - 1) * STRIDE]) + 3)))) return;
    }
    int pos = cnt < k ? cnt++ : k - 1;
    while (pos > 0) {
      const double dp = dk[(pos - 1) * STRIDE];
      if (dp < d2) break;
      if (dp == d2 && orig_of(__double_as_longlong(__ldg(reinterpret_cast<const double *>(S + ik[(pos - 1) * STRIDE]) + 3))) < orig_of(p.idx)) break;
      dk[pos * STRIDE] = dp; ik[pos * STRIDE] = ik[(pos - 1) * STRIDE];
      --pos;
    }
    dk[pos * STRIDE] = d2; ik[pos * STRIDE] = j;
    if (cnt == k) kth = dk[(k - 1) * STRIDE];
  };
  // everything closer than g has been seen: the walk is over once the k-th best is closer, or the radius is
  auto done = [&](double g) { return g > 0 && ((cnt == k && kth < g * g) || r2 <= g * g); };
  bool resolved = false;
  const int fine_rings = CG.cnt ? 8 : 0x7fffffff;      // isolated points: blocks of f^3 cells take over (empty space is skipped)
  for (int r = 0; r <= fine_rings; ++r) {
    for (int dz = -r; dz <= r; ++dz) {
      const long long z = iz + dz;
      if (z < 0 || z >= L.dims[2]) continue;
      for (int dy = -r; dy <= r; ++dy) {
        const long long y = iy + dy;
        if (y < 0 || y >= L.dims[1]) continue;
        const bool border = (dz == -r || dz == r || dy == -r || dy == r);
        for (int part = 0; part < 2; ++part) {
          long long xa, xb;
          if (border) { if (part) break; xa = ix - r; xb = ix + r; }
          else { xa = xb = part ? ix + r : ix - r; }
          xa = max(xa, 0ll); xb = min(xb, (long long)L.dims[0] - 1);
          if (xa > xb) continue;
          uint32_t s, e;
          cell_range(I, (int)z, (int)y, (int)xa, (int)xb, s, e);
          for (uint32_t j = s; j < e; ++j) offer(j);
        }
      }
    }
    // everything closer than the border of the searched block [i - r, i + r]^3 has been seen
    if (done((double)r * L.h - slack)) { resolved = true; break; }
    if (ix - r <= 0 && ix + r >= L.dims[0] - 1 && iy - r <= 0 && iy + r >= L.dims[1] - 1 && iz - r <= 0 && iz + r >= L.dims[2] - 1) { resolved = true; break; }
  }
  if (!resolved) {
    if (trace) {
      const unsigned int m = __activemask();
      if ((threadIdx.x & 31) == __ffs(m) - 1 && !((*(volatile unsigned int *)trace >> ME_TEV_KNN_COARSE) & 1u))
        atomicOr(trace, 1u << ME_TEV_KNN_COARSE);
    }
    // coarse phase, from scratch (the blocks cover the cells of the fine phase again): Chebyshev rings of blocks, empty
    // blocks cost one count load, blocks that cannot hold a candidate closer than the k-th best (or the radius) are skipped
    const int f = CG.f;
    const long long cqx = ix / f, cqy = iy / f, cqz = iz / f;
    const double ux = cell_coord_cont(q.x, L, 0), uy = cell_coord_cont(q.y, L, 1), uz = cell_coord_cont(q.z, L, 2);
    cnt = 0; kth = INFINITY;
    for (int rc = 0;; ++rc) {
      for (int dz = -rc; dz <= rc; ++dz) {
        const long long bz = cqz + dz;
        if (bz < 0 || bz >= CG.cd[2]) continue;
        for (int dy = -rc; dy <= rc; ++dy) {
          const long long by = cqy + dy;
          if (by < 0 || by >= CG.cd[1]) continue;
          const bool border = (dz == -rc || dz == rc || dy == -rc || dy == rc);
          for (int dx = -rc; dx <= rc; dx += (border || rc == 0) ? 1 : 2 * rc) {
            const long long bx = cqx + dx;
            if (bx < 0 || bx >= CG.cd[0]) continue;
            if (__ldg(CG.cnt + (bz * CG.cd[1] + by) * (long long)CG.cd[0] + bx) == 0) continue;
            if (cnt == k || r2 < INFINITY) {
              const double ex = fmax(0.0, fmax((double)(bx * f) - ux, ux - (double)((bx + 1) * f)));
              const double ey = fmax(0.0, fmax((double)(by * f) - uy, uy - (double)((by + 1) * f)));
              const double ez = fmax(0.0, fmax((double)(bz * f) - uz, uz - (double)((bz + 1) * f)));
              const double lb = sqrt(ex * ex + ey * ey + ez * ez) * L.h - slack;
              if (lb > 0 && ((cnt == k && lb * lb > kth) || lb * lb >= r2)) continue;
            }
            const int xa = (int)(bx * f), xb = (int)min(bx * f + f - 1, (long long)L.dims[0] - 1);
            for (int row = 0; row < f * f; ++row) {
              const long long z = bz * f + row / f, y = by * f + row % f;
              if (z >= L.dims[2] || y >= L.dims[1]) continue;
              uint32_t s, e;
              cell_range(I, (int)z, (int)y, xa, xb, s, e);
              for (uint32_t j = s; j < e; ++j) offer(j);
            }
          }
        }
      }
      // the point lies inside its own block: everything closer than rc blocks has been seen
      if (done((double)rc * (double)f * L.h - slack)) break;
      if (cqx - rc <= 0 && cqx + rc >= CG.cd[0] - 1 && cqy - rc <= 0 && cqy + rc >= CG.cd[1] - 1 && cqz - rc <= 0 && cqz + rc >= CG.cd[2] - 1) break;
    }
  }
  return cnt;
}

static_assert((int)ME_KBIT_COUNT <= (int)ME_TEV_KNN_COARSE && (int)ME_TEV_KNN_COARSE < 32, "trace event bit");

}  // namespace me

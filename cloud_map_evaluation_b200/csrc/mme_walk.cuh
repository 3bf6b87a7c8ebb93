// mme_walk.cuh — the fp64 moments of a radius neighbourhood and the generic walk that accumulates them, shared by the MME
// sweeps (mme.cu) and the local consistency sweeps (consistency.cu), so that both accept the same points in the same order.
#pragma once
#include "common.cuh"

namespace me {

// the nine fp64 moments of the accepted offsets d = q - p about the query q (sum d, sum d d^T) and their count
struct Moments {
  double s1x, s1y, s1z, sxx, sxy, sxz, syy, syz, szz;
  unsigned int cnt;
  __device__ __forceinline__ void init() { s1x = s1y = s1z = sxx = sxy = sxz = syy = syz = szz = 0.0; cnt = 0; }
  __device__ __forceinline__ void add(double dx, double dy, double dz) {
    cnt++;
    s1x += dx; s1y += dy; s1z += dz;
    sxx += dx * dx; sxy += dx * dy; sxz += dx * dz;
    syy += dy * dy; syz += dy * dz; szz += dz * dz;
  }
};

// the radius walk of one query over the cell-sorted cloud
__device__ __forceinline__ void walk_global(const P4 &q, const P4 *__restrict__ S, const CellIndex &I,
                                            const Lattice &L, double r2, float rc2, int rings, Moments &m) {
  // the query's own cell comes with its record (high half of the tag; the x index of a sparse lattice from the coordinate)
  int cix, ciy, ciz;
  long long xs = I.sparse ? cell_coord(q.x, L, 0) : 0;
  xs = xs < 0 ? 0 : (xs >= L.dims[0] ? L.dims[0] - 1 : xs);
  cell_from_tag(I, q.idx, (int)xs, cix, ciy, ciz);
  const long long ix = cix, iy = ciy, iz = ciz;
  const float ux = (float)(cell_coord_cont(q.x, L, 0) - (double)ix), uy = (float)(cell_coord_cont(q.y, L, 1) - (double)iy),
              uz = (float)(cell_coord_cont(q.z, L, 2) - (double)iz);   // position inside the own cell, [0,1)
  for (int dz = -rings; dz <= rings; ++dz) {
    const long long z = iz + dz;
    if (z < 0 || z >= L.dims[2]) continue;
    const float mz = dz == 0 ? 0.f : (dz > 0 ? (float)dz - uz : uz - (float)(dz + 1));
    const float remz = rc2 - (mz > 0.f ? mz * mz : 0.f);
    if (remz < 0.f) continue;
    for (int dy = -rings; dy <= rings; ++dy) {
      const long long y = iy + dy;
      if (y < 0 || y >= L.dims[1]) continue;
      const float my = dy == 0 ? 0.f : (dy > 0 ? (float)dy - uy : uy - (float)(dy + 1));
      const float rem = remz - (my > 0.f ? my * my : 0.f);
      if (rem < 0.f) continue;
      const float xw = sqrtf(rem) + 1e-4f;
      const int da = max((int)floorf(ux - xw), -rings), db = min((int)floorf(ux + xw), rings);
      const long long xa = max(ix + da, 0ll), xb = min(ix + db, (long long)L.dims[0] - 1);
      if (xa > xb) continue;
      uint32_t s, e;
      cell_range(I, (int)z, (int)y, (int)xa, (int)xb, s, e);
      for (uint32_t j = s; j < e; ++j) {
        const P4 p = load_p4(S + j);
        const double dx = __dsub_rn(q.x, p.x), dy2 = __dsub_rn(q.y, p.y), dz2 = __dsub_rn(q.z, p.z);
        const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy2, dy2)), __dmul_rn(dz2, dz2));
        if (d2 < r2) m.add(dx, dy2, dz2);                     // nanoflann RadiusResultSet: strict <
      }
    }
  }
}

// squared gap (in cells) between a point at u in [0,1) of its cell and the cell d steps away on the same axis
__device__ __forceinline__ float gap2(int d, float u) {
  const float g = d == 0 ? 0.f : (d > 0 ? (float)d - u : u - (float)(d + 1));
  return g > 0.f ? g * g : 0.f;
}

}  // namespace me

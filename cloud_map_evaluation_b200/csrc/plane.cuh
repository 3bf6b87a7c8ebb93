// plane.cuh — the finish of one radius query: the neighbourhood covariance from MME's moments, its entropy and its
// eigen-decomposition, shared by the local consistency sweep (consistency.cu) and the mutually orthogonal metric's sweep
// (mom.cu), so that both give the same plane variance v bit for bit.
#pragma once
#include "eig3.cuh"
#include "mme_walk.cuh"

namespace me {

struct PlaneEig {
  bool ok;              // k >= min_neighbors (k = accepted points - 1, the query itself)
  bool e_valid;         // ok and the entropy is finite
  double e;             // 0.5 ln(2 pi e det C); meaningful when e_valid
  double v;             // max(0, smallest eigenvalue); NaN when !ok or an eigenvalue is NaN
  int lo;               // the eigenvector column of the smallest eigenvalue (lowest index on ties)
  double w[3], vec[9];  // eig3_jacobi's eigenvalues and eigenvectors (columns, row-major); meaningful when ok
};

// the covariance and the entropy are finish_entropy's (mme.cu) expressions, so e equals MME's bit for bit on the same moments
__device__ __forceinline__ void plane_eig(const Moments &m, int min_neighbors, PlaneEig &P) {
  P.ok = false;
  P.e_valid = false;
  P.e = 0.0;
  P.v = NAN;
  P.lo = 0;
  const long long k = (long long)m.cnt - 1;
  if (!(m.cnt > 0 && k >= (long long)min_neighbors)) return;
  P.ok = true;
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
  const double ent = 0.5 * log(2 * M_PI * M_E * det);
  if (!(isnan(ent) || isinf(ent))) { P.e = ent; P.e_valid = true; }
  eig3_jacobi(c, P.w, P.vec);
  // no indexing by lo: a run-time index would put w in local memory
  int lo = 0;
  double l = P.w[0];
  if (P.w[1] < l) { lo = 1; l = P.w[1]; }
  if (P.w[2] < l) { lo = 2; l = P.w[2]; }
  P.lo = lo;
  if (isnan(P.w[0]) || isnan(P.w[1]) || isnan(P.w[2])) l = NAN;
  P.v = l < 0.0 ? 0.0 : l;                                  // NaN stays NaN
}

}  // namespace me

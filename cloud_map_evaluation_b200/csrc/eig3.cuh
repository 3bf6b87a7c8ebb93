// eig3.cuh — cyclic Jacobi eigen-decomposition of a symmetric 3x3 fp64 matrix, shared by the voxel Gaussians (voxel.cu) and
// the plane variance of the local consistency sweeps (consistency.cu).
#pragma once
#include "common.cuh"

namespace me {

// a_in row-major and symmetric; w = the eigenvalues (unordered), v = the eigenvectors as columns, row-major
static __device__ void eig3_jacobi(const double *a_in, double *w, double *v) {
  double a[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) { a[i] = a_in[i]; v[i] = (i % 4 == 0) ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < 64; ++sweep) {
    const double off = a[1] * a[1] + a[2] * a[2] + a[5] * a[5];
    const double diag = a[0] * a[0] + a[4] * a[4] + a[8] * a[8];
    if (off <= 1e-34 * diag || off == 0.0) break;
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
      for (int q = p + 1; q < 3; ++q) {
        const double apq = a[p * 3 + q];
        if (apq == 0.0) continue;
        const double app = a[p * 3 + p], aqq = a[q * 3 + q];
        const double theta = (aqq - app) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double akp = a[k * 3 + p], akq = a[k * 3 + q];
          a[k * 3 + p] = c * akp - s * akq;
          a[k * 3 + q] = s * akp + c * akq;
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double apk = a[p * 3 + k], aqk = a[q * 3 + k];
          a[p * 3 + k] = c * apk - s * aqk;
          a[q * 3 + k] = s * apk + c * aqk;
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double vkp = v[k * 3 + p], vkq = v[k * 3 + q];
          v[k * 3 + p] = c * vkp - s * vkq;
          v[k * 3 + q] = s * vkp + c * vkq;
        }
      }
  }
  w[0] = a[0]; w[1] = a[4]; w[2] = a[8];
}

}  // namespace me

// svd3.cuh — the 3x3 algebra of the point-to-point fit, on the host (ICP's update, icp.cu) and on the device (the RANSAC
// hypotheses of global registration, globalreg.cu).  One implementation for both: a hypothesis and an ICP update from the
// same sums give the same rotation.
#pragma once
#include <math.h>

namespace me {

// SVD of a 3x3 by one-sided Jacobi (Hestenes): plane rotations V orthogonalise the columns of a = sigma V, so
// sigma = U diag(w) V^T with U's columns a_j / w_j.  It works on sigma itself: the eigen-problem of sigma^T sigma would
// square the condition number, and with it the error of the small singular values (a tilted near-planar cloud made R
// a shear of a few per cent).  Singular values descending (ties keep column order); only U's first two columns are formed.
__host__ __device__ inline void svd3(const double s_in[9], double U[9], double w[3], double V[9]) {
  double a[9];
  for (int i = 0; i < 9; ++i) { a[i] = s_in[i]; V[i] = (i % 4 == 0) ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < 60; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        double alpha = 0, beta = 0, gamma = 0;
        for (int k = 0; k < 3; ++k) { alpha += a[k * 3 + p] * a[k * 3 + p]; beta += a[k * 3 + q] * a[k * 3 + q]; gamma += a[k * 3 + p] * a[k * 3 + q]; }
        if (gamma == 0.0) continue;
        const double rel = fabs(gamma) / sqrt(alpha * beta);
        off = off < rel ? rel : off;
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
        for (int k = 0; k < 3; ++k) {
          const double ap = a[k * 3 + p], aq = a[k * 3 + q];
          a[k * 3 + p] = c * ap - s * aq; a[k * 3 + q] = s * ap + c * aq;
          const double vp = V[k * 3 + p], vq = V[k * 3 + q];
          V[k * 3 + p] = c * vp - s * vq; V[k * 3 + q] = s * vp + c * vq;
        }
      }
    if (off < 1e-15) break;
  }
  double nw[3];
  for (int j = 0; j < 3; ++j) nw[j] = sqrt(a[j] * a[j] + a[3 + j] * a[3 + j] + a[6 + j] * a[6 + j]);
  int ord[3] = {0, 1, 2};
  for (int i = 1; i < 3; ++i)            // insertion sort, descending, stable
    for (int j = i; j > 0 && nw[ord[j]] > nw[ord[j - 1]]; --j) { const int t = ord[j]; ord[j] = ord[j - 1]; ord[j - 1] = t; }
  double Vs[9];
  for (int j = 0; j < 3; ++j) {
    w[j] = nw[ord[j]];
    for (int k = 0; k < 3; ++k) { Vs[k * 3 + j] = V[k * 3 + ord[j]]; U[k * 3 + j] = j < 2 && w[j] > 0 ? a[k * 3 + ord[j]] / w[j] : 0.0; }
  }
  for (int i = 0; i < 9; ++i) V[i] = Vs[i];
}

__host__ __device__ inline double det3_rm(const double *m) {
  return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}

// Eigen::umeyama without scaling from point-to-point sums taken about c (blk = [count, sum p (3), sum q (3),
// sum q p^T (9, row-major), ...]): R = U S V^T of sigma = (1/n) sum (q - qm)(p - pm)^T; upd = row-major 4x4
// sv (nullable): the singular values of sigma, descending
__host__ __device__ inline void umeyama_from_sums(const double *blk, const double c[3], double upd[16], double *sv_out = nullptr) {
  const double n = blk[0];
  const double *sp = blk + 1, *sq = blk + 4, *sqp = blk + 7;
  double pm[3], qm[3], sigma[9];
  for (int k = 0; k < 3; ++k) { pm[k] = sp[k] / n; qm[k] = sq[k] / n; }
  for (int r = 0; r < 3; ++r)
    for (int col = 0; col < 3; ++col) sigma[r * 3 + col] = sqp[r * 3 + col] / n - qm[r] * pm[col];
  double U[9], sv[3], Vs[9];
  svd3(sigma, U, sv, Vs);
  if (sv_out) for (int k = 0; k < 3; ++k) sv_out[k] = sv[k];
  // U's third column is always the cross product of the first two: a_3 / w_3 carries an error of u w_1 / w_3 (and is
  // undefined at rank 2), while R = U S V^T only needs the orientation of U, which the cross product fixes (det U = +1).
  // Eigen's rule S_3 = -1 when det(U) det(V) < 0 then makes R a rotation; in exact arithmetic this is umeyama's R.
  U[2] = U[3] * U[7] - U[6] * U[4]; U[5] = U[6] * U[1] - U[0] * U[7]; U[8] = U[0] * U[4] - U[3] * U[1];
  double S[3] = {1, 1, 1};
  if (det3_rm(U) * det3_rm(Vs) < 0) S[2] = -1;
  for (int i = 0; i < 16; ++i) upd[i] = 0.0;
  upd[15] = 1.0;
  for (int r = 0; r < 3; ++r)
    for (int col = 0; col < 3; ++col) { double s = 0; for (int k = 0; k < 3; ++k) s += U[r * 3 + k] * S[k] * Vs[col * 3 + k]; upd[r * 4 + col] = s; }
  // t = dst_mean - R src_mean, means back in absolute coordinates
  for (int r = 0; r < 3; ++r) {
    double rp = 0;
    for (int k = 0; k < 3; ++k) rp += upd[r * 4 + k] * (pm[k] + c[k]);
    upd[r * 4 + 3] = (qm[r] + c[r]) - rp;
  }
}

}  // namespace me

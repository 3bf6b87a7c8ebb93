// records.cuh — the per-query records of the last NN sweep and the rules that turn them into statistics, shared by the
// five-level pass, the accuracy curve and the distance quantiles (nn.cu) and the per-region table (region.cu), so that every
// consumer keeps the same pairs over the same ranges with the same distance.
#pragma once
#include "common.cuh"

namespace me {

struct NNConst {
  double tau[5];
  double cutoff;        // R (mode 0) or R*R (mode 1)
  int cutoff_mode;
  int accumulate;       // accumulate pair statistics in the sweep (0 for ME_PAIRING_AS_WRITTEN gt->est)
  int want_full_cd;
  double max_d2;        // nothing beyond this squared distance matters (inf when full CD is wanted)
  double ref_maxabs;    // max |coordinate| of the reference cloud (slack of the face test)
  // ME_PAIRING_AS_WRITTEN gt->est (accumulate == 0): the caller-order clouds the sweep reads the as-written pair from
  const double *aw_gt_xyz, *aw_est_xyz;
  long long aw_n_gt, aw_n_est;
  // slab layout: only the planes [cov_lo, cov_hi) of the reference lattice along axis cov_axis (1: y, 2: z; 0: everything)
  // are laid out on this rank
  int cov_axis, cov_lo, cov_hi, cov_dim;
};

__device__ __forceinline__ bool keep_pair(double d2, const NNConst &c) {
  return c.cutoff_mode == ME_CUTOFF_SQDIST_LE_R ? (d2 <= c.cutoff) : (d2 < c.cutoff);
}

// the distance d of a kept pair, map_eval.cpp:1095: sqrt of Eigen's squaredNorm
__device__ __forceinline__ double pair_dist(double sq) { return __dsqrt_rn(sq); }

// map_eval.cpp:1095-1123 for one kept pair (source - target)
// sq = Eigen's squaredNorm of (source - target), x*x + (y*y + z*z)
template <class Acc>
__device__ __forceinline__ void accum_sq(double sq, const NNConst &c, Acc &a) {
  double nd = pair_dist(sq);
  a.pair(nd, sq);
#pragma unroll
  for (int k = 0; k < 5; ++k)
    if (nd <= c.tau[k]) a.inlier(k, nd, sq);
}

// ---------------------------------------------------------------------------------------------------------------
// ME_PAIRING_AS_WRITTEN: map_eval.cpp:1233 stores (nn_est, i_gt); :1241 passes (source = gt, target = est), so
// :1093-1094 reads gt[nn_est] and est[i_gt].  Reproduced verbatim; out-of-range (UB in the reference) is counted.
// Walks every gt point; points this rank did not evaluate carry the marker -2.
// ---------------------------------------------------------------------------------------------------------------
enum { kAwNone = 0, kAwOutOfRange = 1, kAwPair = 2 };
// the nn_sq record of an out-of-range pair (a squared norm is never negative)
static constexpr double kAwOutOfRangeSq = -1.0;

// Eigen's squaredNorm of gt[s] - est[t] for source index s = nn_est into gt and target index t = i_gt into est, or
// kAwOutOfRangeSq when either index is past its cloud
__device__ __forceinline__ double as_written_sq(long long s, long long t, const double *__restrict__ gt_xyz, long long n_gt,
                                                const double *__restrict__ est_xyz, long long n_est) {
  if (s >= n_gt || t >= n_est) return kAwOutOfRangeSq;
  const double dx = __dsub_rn(__ldg(gt_xyz + 3 * s), __ldg(est_xyz + 3 * t));
  const double dy = __dsub_rn(__ldg(gt_xyz + 3 * s + 1), __ldg(est_xyz + 3 * t + 1));
  const double dz = __dsub_rn(__ldg(gt_xyz + 3 * s + 2), __ldg(est_xyz + 3 * t + 2));
  return sqnorm_eigen(dx, dy, dz);
}

// gt query i (sorted order): kAwNone (no kept pair), kAwOutOfRange (counted in n_ub) or kAwPair with sq = Eigen's
// squaredNorm of gt[nn_est] - est[i_gt]
__device__ __forceinline__ int as_written_pair(const P4 *__restrict__ Qgt, long long i, const int32_t *__restrict__ nn_idx,
                                               const double *__restrict__ nn_d2, const double *__restrict__ gt_xyz, long long n_gt,
                                               const double *__restrict__ est_xyz, long long n_est, const NNConst &C, double &sq) {
  const int32_t nn_est = nn_idx[i];
  if (nn_est < 0) return kAwNone;
  if (!keep_pair(nn_d2[i], C)) return kAwNone;
  const long long i_gt = orig_of(__double_as_longlong(__ldg(reinterpret_cast<const double *>(Qgt + i) + 3)));
  sq = as_written_sq(nn_est, i_gt, gt_xyz, n_gt, est_xyz, n_est);
  return sq < 0 ? kAwOutOfRange : kAwPair;
}

struct CurveSrc {           // the per-query records of one direction
  long long b, e;           // sorted range the sweep filled (entries < 0 in it: no neighbour / another rank's query)
  const int32_t *nn_idx;
  const double *nn_d2, *nn_sq;
  int as_written;           // ME_PAIRING_AS_WRITTEN gt->est: the distance comes from the swapped indices
  const P4 *Qgt;
  const double *gt_xyz, *est_xyz;
  long long n_gt, n_est;
};

// the kept-pair rule of the five-level pass on record i of S (me_nn_curve*, me_nn_quantile* and me_nn_region* share it): true
// with sq = the pair's squared norm, whose pair_dist is d; an out-of-range ME_PAIRING_AS_WRITTEN pair adds one to ub and is
// not kept
__device__ __forceinline__ bool kept_record(const CurveSrc &S, const NNConst &C, long long i, double &sq, unsigned int &ub) {
  if (S.as_written) {
    const int r = as_written_pair(S.Qgt, i, S.nn_idx, S.nn_d2, S.gt_xyz, S.n_gt, S.est_xyz, S.n_est, C, sq);
    ub += r == kAwOutOfRange;
    return r == kAwPair;
  }
  if (__ldg(S.nn_idx + i) >= 0 && keep_pair(__ldg(S.nn_d2 + i), C)) {
    sq = __ldg(S.nn_sq + i);
    return true;
  }
  return false;
}

// host side (nn.cu)
void set_cutoff(NNConst &C, const me_nn_params *p);
// the records of the last me_eval_nn* still describe the clouds; `who` names the caller in the message
int nn_records_fresh(me_ctx *ctx, const char *who);
// the records of direction q (query cloud q) over the ranges nn_stats_kernel / pair_as_written_kernel walk
CurveSrc record_src(const me_ctx *ctx, int q);

}  // namespace me

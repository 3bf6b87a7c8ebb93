/*
 * mapeval_b200.h — C-ABI of libmapeval_b200.so
 *
 * H100-native (sm_90a) replacement for the metric hot path of MapEval
 * (JokerJohn/Cloud_Map_Evaluation).  The reference has no FFI of its own: the
 * path sits behind C++ member functions of `class MapEval` that talk through
 * member state (map_eval/src/map_eval.h:121-362).  Each entry point below names
 * the reference member function(s) it replaces (paths relative to the reference
 * root, `map_eval/src/`).  Plain C: pointers, sizes, PODs.  No C++/torch types.
 *
 * Conventions
 *   - every function returns ME_OK (0) or a negative me_status; after an error
 *     me_last_error(ctx) holds a message (the reference's convention is the
 *     0 / -1 return of MapEval::process(), map_eval.cpp:16,28,34,101).
 *   - clouds are N x 3 fp64, array-of-structs — the layout of Open3D's
 *     `std::vector<Eigen::Vector3d> points_` that the reference reads.
 *   - one me_ctx = one GPU = one caller thread at a time.  Multi-GPU = one
 *     context per process/GPU with {rank, world} set; the *_accum_device entry
 *     points leave this rank's partial accumulators in the context's device
 *     block, the caller all-reduces it in place (NCCL), fetches it once
 *     (me_accum_fetch) and calls the host-side *_finalize.
 *   - there is NO CPU fallback in this library: without a usable CUDA device
 *     me_create fails with ME_ERR_NO_DEVICE.
 */
#ifndef MAPEVAL_B200_H_
#define MAPEVAL_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ME_ABI_VERSION 2

#if defined(__GNUC__)
#define ME_API __attribute__((visibility("default")))
#else
#define ME_API
#endif

typedef enum {
  ME_OK = 0,
  ME_ERR_INVALID = -1,     /* bad argument / call order                       */
  ME_ERR_NO_DEVICE = -2,   /* no CUDA device / wrong architecture             */
  ME_ERR_CUDA = -3,        /* a CUDA runtime call failed (see me_last_error)  */
  ME_ERR_NOMEM = -4,       /* device or host allocation failed                */
  ME_ERR_EMPTY = -5,       /* a required cloud is empty (map_eval.cpp:32-35)  */
  ME_ERR_RANGE = -6        /* coordinates / voxel indices outside what the grids can index */
} me_status;

enum { ME_CLOUD_EST = 0, ME_CLOUD_GT = 1 };

/* kept-pair cut-off of the 1-NN sweep */
enum {
  ME_CUTOFF_SQDIST_LE_R = 0,  /* keep iff d2 <= icp_max_distance  (path A as written, map_eval.cpp:1219,1232) */
  ME_CUTOFF_DIST_LT_R = 1     /* keep iff d2 <  icp_max_distance^2 (Open3D EvaluateRegistration, map_eval.cpp:1168) */
};

/* how the gt->est pairs are looked up by the accumulator pass */
enum {
  ME_PAIRING_AS_WRITTEN = 0,  /* map_eval.cpp:1233 stores (nn_est, i_gt) but :1241 passes (source=gt,target=est),
                                 so :1093-1094 reads gt[nn_est] and est[i_gt]; reproduced verbatim.  Pairs whose
                                 swapped indices fall outside the clouds (undefined behaviour in the reference)
                                 are dropped and counted in n_ub. */
  ME_PAIRING_GEOMETRIC = 1    /* distance between the gt point and its nearest est point */
};

typedef struct me_ctx me_ctx;

typedef struct {
  int32_t abi_version;     /* must be ME_ABI_VERSION                                       */
  int32_t device;          /* CUDA device ordinal                                          */
  int32_t rank, world;     /* this context evaluates queries [rank*N/world,(rank+1)*N/world) */
  void   *stream;          /* cudaStream_t to launch on; NULL = library-owned stream       */
  double  nn_cell_size;    /* edge of the lattice cells in metres; <= 0 = auto         */
  int64_t max_grid_cells;  /* budget for the dense cell table; <= 0 = automatic (2^28 .. 2^31 with the cloud sizes) */
  double  vmd_voxel_size;  /* voxel edge the lattices should align to (the config's vmd_voxel_size);
                              <= 0 = unknown: me_eval_awd then re-lays the clouds out once     */
} me_options;

/* ---- a1/a2/a4: AC / COM / CD inlier statistics and full Chamfer ------------------------------- */

typedef struct {
  double  tau[5];            /* accuracy_level / trunc_dist_ (map_eval.h:85)               */
  double  icp_max_distance;  /* R (map_eval.h:69)                                          */
  int32_t cutoff_mode;       /* ME_CUTOFF_*                                                */
  int32_t pairing;           /* ME_PAIRING_* (gt->est direction only)                      */
  int32_t want_full_cd;      /* also accumulate sum sqrt(d2) over ALL queries (map_eval.cpp:1398-1431) */
  int32_t directions;        /* bit0: est->gt, bit1: gt->est; 0 = both                     */
} me_nn_params;

/* Largest world size of a sharded pass (me_create / me_set_shard refuse more): every rank owns one slot of the per-rank
 * moments below, so that the single SUM all-reduce of the accumulators gathers them. */
#define ME_MAX_WORLD 64

/* sum-reducible partial accumulators of one direction (int64 block first, then fp64 block).  sigma needs the spread of d
 * over ALL kept pairs; sum(d) and sum(d^2) lose u (mean / spread)^2 of it to cancellation, so every rank also reports the
 * count, mean and sum of squared deviations (M2) of its kept d in its own slot [rank], zeros elsewhere, and
 * me_nn_finalize merges the slots (Chan et al.).  Accumulators whose slots do not account for all n_corr pairs (filled by
 * a caller that sets the sums only) are finalised from sum_d_all / sum_d2_all instead. */
#define ME_NN_ACCUM_I64 9
#define ME_NN_ACCUM_F64 (13 + 3 * ME_MAX_WORLD)
typedef struct {
  int64_t n_query;           /* queries evaluated by this rank                             */
  int64_t n_corr;            /* kept pairs |C|                                             */
  int64_t n_inlier[5];       /* pairs with d <= tau_k (number_vec, map_eval.cpp:1099-1123) */
  int64_t n_ub;              /* ME_PAIRING_AS_WRITTEN: dropped out-of-range pairs          */
  int64_t n_far;             /* queries resolved by the far (ring-expansion) kernel        */
  double  sum_d[5];          /* sum of d   over pairs with d <= tau_k (mean_vec)           */
  double  sum_d2[5];         /* sum of d^2 over pairs with d <= tau_k (rmse_vec)           */
  double  sum_d_all;         /* sum of d   over all kept pairs                             */
  double  sum_d2_all;        /* sum of d^2 over all kept pairs                             */
  double  sum_nn_dist;       /* sum of sqrt(d2_nn) over ALL queries (full CD)              */
  double  rank_n[ME_MAX_WORLD];     /* kept pairs of rank r (= n_corr of that rank)        */
  double  rank_mean[ME_MAX_WORLD];  /* mean of d over them                                 */
  double  rank_m2[ME_MAX_WORLD];    /* sum of (d - rank_mean)^2 over them                  */
} me_nn_accum;

typedef struct {             /* == est_gt_results / gt_est_results (map_eval.cpp:1140-1144) */
  int64_t n_source, n_corr;
  int64_t n_inlier[5];
  int64_t n_ub;
  double  mean[5], rmse[5], fitness[5], sigma[5];
  double  sum_nn_dist;
} me_dir_result;

typedef struct {
  me_dir_result est_to_gt, gt_to_est;
  double cd[5], f1[5], iou[5];   /* map_eval.cpp:1245-1253 */
  double full_cd;                /* map_eval.cpp:1429      */
} me_nn_result;

/* ---- a5-a9: mean map entropy -------------------------------------------------------------------- */

typedef struct {
  int64_t n_query, n_valid;
  double  sum_entropy;
  double  min_entropy, max_entropy;  /* over entropies != 0 (map_eval.cpp:697-701); +inf / -inf if none */
} me_mme_accum;

typedef struct {
  double  mme;                       /* sum/n_valid, 0 if none (map_eval.cpp:1720-1724) */
  int64_t n_valid, n_total;
  double  min_abs_entropy, max_abs_entropy;  /* |max|, |min| (map_eval.cpp:700-701); NaN if no non-zero entropy */
} me_mme_result;

/* ---- a10-a16: voxel Gaussians, AWD ("VMD"), SCS ------------------------------------------------ */

typedef struct {
  double  awd, scs;                  /* vmd (map_eval.cpp:324-325), scs_overall (:387); NaN when the reference divides 0/0 */
  int64_t n_pairs, n_scs;            /* |wasserstein_distances|, scs_count */
  int64_t n_voxels_est, n_voxels_gt; /* voxel_map_.size() after buildVoxelMap (voxel_calculator.cpp:55) */
  int64_t n_active, n_old, n_new;    /* voxel_calculator.cpp:170 */
} me_awd_result;

/* ---- N2: registration (registration_methods: 0 point-to-point, 1 point-to-plane, 2 generalized ICP) --------- */
#define ME_ICP_POINT_TO_POINT 0     /* map_eval.cpp:1370-1374 */
#define ME_ICP_POINT_TO_PLANE 1     /* :1375-1379 */
#define ME_ICP_GENERALIZED    2     /* :1380-1385, the value every shipped config uses */

typedef struct {             /* == open3d RegistrationResult (map_eval.cpp:1367-1394) */
  double  transformation[16];        /* row-major 4x4: registration_result.transformation_ -> trans            */
  double  fitness, inlier_rmse;      /* fitness_ (|corr| / |est|), inlier_rmse_                                  */
  int64_t n_corr;                    /* correspondence_set_.size()                                               */
  int32_t iterations, converged;     /* updates applied; 1 if the relative criteria stopped the loop             */
} me_icp_result;

/* one planning step of the cell lattice (me_plan_lattice) */
typedef struct {
  double  v, h;            /* voxel edge; cell edge h = v / m                                  */
  int32_t m;               /* cells per voxel edge                                             */
  int32_t sparse;          /* 1: occupied 32-cell row segments + hash; 0: dense table          */
  int32_t nvox[3];         /* voxels per axis                                                  */
  int32_t dims[3];         /* cells per axis = nvox * m                                        */
  int64_t ncells;          /* dense table: cells (4 B each); sparse: 0                         */
} me_lattice_plan;

/* ---- lifecycle ---------------------------------------------------------------------------------- */

ME_API int  me_abi_version(void);
ME_API int  me_create(const me_options *opt, me_ctx **out);
ME_API void me_destroy(me_ctx *ctx);
ME_API const char *me_last_error(const me_ctx *ctx);      /* ctx may be NULL: last error of me_create on this thread */
ME_API int  me_set_stream(me_ctx *ctx, void *cuda_stream);
ME_API int  me_set_shard(me_ctx *ctx, int32_t rank, int32_t world);
/* How a context of a multi-GPU job (world > 1) lays the clouds out.  ME_LAYOUT_REPLICATED (default): both whole clouds on
 * every rank, the query ranges of the sweeps sharded.  ME_LAYOUT_SLAB: every rank lays out only the voxel layers it owns
 * along y or z (whichever balances), plus a halo of four lattice cells, of BOTH clouds, and evaluates the points of its
 * layers — the lattice builds and the voxel stage shard with the sweeps.  The clouds themselves stay replicated (caller
 * order, set with me_set_cloud*): searches that leave the halo are finished exactly over the whole cloud.  The partial
 * accumulators are reduced as before (me_accum_block); the voxel stage runs as me_voxel_begin / all-reduce(MAX) of
 * me_voxel_w_table / me_voxel_finish_accum_device.  A scene that cannot be cut (sparse cell table, fewer than 2 x world voxel
 * layers, one rank holding > 75 %) silently stays replicated — me_layout_active tells.  me_eval_awd, the tile sweep and
 * per-point outputs of other ranks' points are not available on an active slab layout. */
#define ME_LAYOUT_REPLICATED 0
#define ME_LAYOUT_SLAB 1
ME_API int  me_set_layout(me_ctx *ctx, int32_t layout);
/* after the lattices were built (any sweep): *layout = the layout in force, *axis = 1 (y) / 2 (z) / 0, n_laid_out[2] = the
 * points of (est, gt) this rank laid out, n_owned[2] = the points it evaluates.  Any pointer may be NULL. */
ME_API int  me_layout_active(me_ctx *ctx, int32_t *layout, int32_t *axis, int64_t n_laid_out[2], int64_t n_owned[2]);
/* The planner of the slab layout as a pure host function (no context, no device): given the number of points in every
 * lattice plane along y and along z (cells_per_voxel planes per voxel layer), cut the voxel layers of one axis into `world`
 * contiguous groups of about equal point count.  *axis = 1 (y) / 2 (z), or 0 when the scene cannot be cut (fewer than
 * 2 x world layers on both axes, or the busiest rank — owned layers + halo_cells planes either side — would lay out more than
 * 75 % of the points); layer_bounds[0..world] = first owned layer of every rank; *busiest_share = that rank's share.  This
 * is the arithmetic every rank runs on the (replicated) cloud's histogram, which is why the ranks agree without talking. */
/* One planning step of the cell lattice as a pure host function (no context, no device): the lattice a cloud of n points
 * with this bounding box gets for a wanted cell edge (<= 0: ~2 points per cell of the box volume), aligned with voxel_size
 * (<= 0: free), fitting `other` (nullable bounding box of the second cloud) under the same spec, within max_grid_cells
 * (<= 0: the automatic budget, 2^28 .. 2^31 growing with the clouds).  Dense if the dense table at that edge fits; sparse
 * when the budget would force cells > 1.25x coarser (allow_sparse).  ME_ERR_RANGE if nothing fits.  The library runs this
 * step 1-3 times per cloud pair, refining the edge on the measured occupancy in between (DESIGN §2). */
ME_API int  me_plan_lattice(const double bbox_min[3], const double bbox_max[3], int64_t n, const double *other_bbox_min,
                            const double *other_bbox_max, int64_t other_n, double voxel_size, double cell_edge_target,
                            int64_t max_grid_cells, int32_t allow_sparse, me_lattice_plan *out);
ME_API int  me_plan_slab_cut(const uint64_t *plane_counts_y, int32_t n_planes_y, const uint64_t *plane_counts_z,
                             int32_t n_planes_z, int32_t cells_per_voxel, int32_t world, int32_t halo_cells, int32_t *axis,
                             int32_t *layer_bounds, double *busiest_share);
ME_API int  me_synchronize(me_ctx *ctx);

/* replaces: io::ReadPointCloud* results held in map_3d_/gt_3d_ (map_eval.cpp:10-21) — the clouds the path reads.
 * me_set_cloud copies host memory (async on the stream; pinned memory makes it truly async);
 * me_set_cloud_device borrows an fp64 N x 3 device buffer that must outlive the context's use of it. */
ME_API int  me_set_cloud(me_ctx *ctx, int which, const double *xyz_host, int64_t n);
ME_API int  me_set_cloud_device(me_ctx *ctx, int which, const double *xyz_device, int64_t n);
/* replaces: map_3d_->Transform(initial_matrix) (map_eval.cpp:1206); T is a row-major 4x4 */
ME_API int  me_transform(me_ctx *ctx, int which, const double T[16]);
/* replaces: map_3d_ = map_3d_->VoxelDownSample(param_.downsample_size) and the same for gt_3d_ (map_eval.cpp:38-39;
 * open3d::geometry::PointCloud::VoxelDownSample: voxel index floor((p - (min_bound - s/2)) / s), output = mean of the
 * voxel's points accumulated in input order).  The cloud held by the context is replaced by its down-sampled version;
 * *n_out (nullable) receives the new point count.  The output points are bit-identical to the CPU path as a set; they
 * are ordered by increasing voxel index (Open3D: std::unordered_map iteration order, implementation-defined).  A cloud
 * that holds normals keeps them: per voxel the sum, in input order, of the normals without a NaN component, divided by
 * the voxel's point count and not re-normalised (Open3D AccumulatedPoint::GetAverageNormal), in the output order. */
ME_API int  me_voxel_downsample(me_ctx *ctx, int which, double voxel_size, int64_t *n_out);
/* the cloud currently held by the context (after me_transform / me_voxel_downsample), caller order, N x 3 fp64.
 * xyz_host == NULL: size query only (*n).  capacity_points < N is an error. */
ME_API int  me_get_cloud(me_ctx *ctx, int which, double *xyz_host, int64_t capacity_points, int64_t *n);

/* ---- simulated degradation of a map (evaluate_noised_gt: map_eval.h:79,87, config.yaml:55-59) ---------------------------
 * The operators of MapEval::addGaussianNoise / addNonUniformDensity / addSparseOutliers / addLocalDeformation
 * (map_eval.cpp:1745-1829, map_eval.h:296-310) on a cloud held by the context, applied in the order the caller calls them,
 * on library-owned buffers.  Borrowed clouds (me_set_cloud_device) are refused with ME_ERR_INVALID: the operators never
 * write caller memory.  Afterwards the cloud's lattice and per-point results are stale, as after me_transform.
 * The reference draws from std::random_device; here every draw is the counter-based hash of synth.py — splitmix64 of
 * (seed, index, lane) — so a degraded cloud is a pure function of (cloud, parameters, seed), identical on every GPU of a
 * job, and its kept points, counts and outlier bases equal a numpy statement bit for bit.  The lanes of the four operators
 * are disjoint (noise 0-5, density 6, outliers 7-13), so one seed serves them all. */
/* dst := src, points and normals (when src holds them), into library-owned memory; src != dst.  This is how a borrowed
 * ground truth becomes an owned estimate. */
ME_API int  me_copy_cloud(me_ctx *ctx, int src, int dst);
/* addGaussianNoise (:1745-1755): p_a += std_dev * gaussian(seed, i, 2a), a = x, y, z (Box-Muller, u1 = max(u24, 2^-25)),
 * in place.  std_dev finite and >= 0; 0 leaves the cloud unchanged.  Normals are untouched (the reference moves points_). */
ME_API int  me_add_gaussian_noise(me_ctx *ctx, int which, double std_dev, uint64_t seed);
/* addNonUniformDensity (:1757-1784): xn = sin(x / region_size * pi), yn = sin(y / region_size * pi); threshold =
 * sparse_ratio if xn * yn > 0, else dense_ratio; the point is kept iff uniform24(seed, i, 6) < threshold.  Stable: the kept
 * points keep their order, and normals go with their points.  region_size = 0 gives NaN signs: every point takes
 * dense_ratio, as in the reference.  *n_out (nullable) = the new point count. */
ME_API int  me_add_non_uniform_density(me_ctx *ctx, int which, double sparse_ratio, double dense_ratio, double region_size,
                                       uint64_t seed, int64_t *n_out);
/* addSparseOutliers (:1786-1806): m = (int)(N * outlier_ratio) outliers (none for a negative ratio) appended after the N
 * points in j order: base = min(floor(uniform53(seed, j, 7) * N), N - 1), uniform53 = (h >> 11) * 2^-53, and
 * o_a = p_base,a + outlier_range * gaussian(seed, j, 8 + 2a).  outlier_range finite and >= 0.  ME_ERR_RANGE when
 * N * outlier_ratio >= 2^31 or N + m >= 2^31 - 1.  The cloud loses its normals (Open3D: HasNormals() is false once
 * normals_ and points_ differ in size), so generalized ICP estimates them.  *n_out (nullable) = N + m. */
ME_API int  me_add_sparse_outliers(me_ctx *ctx, int which, double outlier_ratio, double outlier_range, uint64_t seed,
                                   int64_t *n_out);
/* addLocalDeformation (:1808-1829): d = sqrt of Eigen's squaredNorm of p - c; where d < radius (strict),
 * w = 0.5 (1 + cos(pi d / radius)) and p += ((p - c) / d * strength) * w, every operation rounded on its own (no FMA); the
 * point at the centre stays (Eigen's normalize() leaves a zero vector).  No draws.  radius <= 0 moves nothing.  Normals are
 * untouched. */
ME_API int  me_add_local_deformation(me_ctx *ctx, int which, double radius, double strength, const double center[3]);
/* replaces: MapEval::performICPRegistration case 0 (map_eval.cpp:1366-1394): open3d RegistrationICP(est, gt,
 * icp_max_distance, initial_matrix, TransformationEstimationPointToPoint(), ICPConvergenceCriteria{relative_fitness,
 * relative_rmse, max_iteration} = {1e-6, 1e-6, 30}).  On return the estimated cloud held by the context is the original
 * cloud transformed once by the result (map_3d_->Transform(trans), :1392), ready for me_eval_nn with
 * ME_CUTOFF_DIST_LT_R / ME_PAIRING_GEOMETRIC / want_full_cd (calculateMetrics, :1147-1202).  world must be 1. */
ME_API int  me_icp_point_to_point(me_ctx *ctx, double max_correspondence_distance, int32_t max_iteration,
                           double relative_fitness, double relative_rmse, const double T_init[16], me_icp_result *out);
/* replaces: MapEval::performICPRegistration (map_eval.cpp:1366-1394), all three cases; method = param_.evaluation_method_
 * (ME_ICP_*).  ME_ICP_POINT_TO_PLANE = RegistrationICP with TransformationEstimationPointToPlane: the ground-truth cloud
 * needs normals (me_set_normals, e.g. from a PCD that carries them, or me_estimate_normals) — without them the call fails
 * like Open3D does.  ME_ICP_GENERALIZED = RegistrationGeneralizedICP with TransformationEstimationForGeneralizedICP()
 * (epsilon 1e-3): per-point covariances Rx diag(eps, 1, 1) Rx^T, Rx = GetRotationFromE1ToX(normal) of the normal as held
 * (not normalised), as InitializePointCloudForGeneralizedICP builds them — from the cloud's own normals when it has them
 * (me_set_normals, me_estimate_normals, averaged by me_voxel_downsample), else from EstimateNormals(KNN 20) computed
 * inside, which do not outlive the call (the cloud still has no normals afterwards).  Same post-condition as
 * me_icp_point_to_point; normals the estimated cloud held are rotated by the result, the ground truth's are unchanged. */
ME_API int  me_icp(me_ctx *ctx, int32_t method, double max_correspondence_distance, int32_t max_iteration,
                   double relative_fitness, double relative_rmse, const double T_init[16], me_icp_result *out);
/* Registration on every rank of a multi-GPU job: me_icp split at its collective (me_icp is this sequence at world = 1).
 * Both clouds are replicated; every rank runs the same calls with the same arguments:
 *   me_icp_begin                        checks as me_icp, keeps a copy of the estimated cloud
 *   me_icp_normals_slice(EST), (GT)     generalized ICP, cloud without normals: this rank's k-NN normals (KNN 20) of the
 *                                       caller indices [rank s, (rank + 1) s), s = *slice_points = ceil(N / world), into
 *                                       *device_normals, a buffer of world * s * 3 doubles (caller order).  *pending = 1:
 *                                       the caller all-gathers it in place (ncclAllGather, sendbuff = *device_normals +
 *                                       rank * s * 3, s * 3 doubles).  *pending = 0 and NULL: nothing to gather (the cloud's
 *                                       own normals are used, another method, or world = 1).  The gathered normals are
 *                                       bit-identical to me_estimate_normals at world = 1.
 *   me_icp_block                        the first call moves the cloud by T_init and sweeps; every call hands out the DEVICE
 *                                       address of the fp64 block of this rank's partial sums (*n_sum values: count first,
 *                                       exact below 2^53).  The caller SUM-all-reduces it in place.
 *   me_icp_step(&done)                  reads the reduced block: convergence test, update, move, sweep -> the next block
 *                                       (same address); *done = 1: nothing left to reduce
 *   me_icp_end                          est := Transform(original, T) with the result, as me_icp leaves it
 * The device work of a call is queued on the context's stream: the caller orders its collective after it (me_synchronize,
 * or a collective on that stream).  Out of order calls (step / block / end before begin, a block or step with normals still
 * pending, a step before the first block) fail with ME_ERR_INVALID; any failure while a registration is open closes it
 * and leaves the estimated cloud as it was handed in.  A context of world > 1 with ME_LAYOUT_SLAB requested refuses
 * me_icp_begin: the sweeps of the registration run on the replicated layout (set it for the registration, back afterwards). */
#define ME_ICP_BLOCK_P2P 17   /* count, sum p (3), sum q (3), sum q p^T (9, row-major), sum d2; p, q about the centre */
#define ME_ICP_BLOCK_NE 29    /* count, J^T J upper triangle (21, row-major), J^T r (6), sum d2 */
ME_API int  me_icp_begin(me_ctx *ctx, int32_t method, double max_correspondence_distance, int32_t max_iteration,
                         double relative_fitness, double relative_rmse, const double T_init[16]);
ME_API int  me_icp_normals_slice(me_ctx *ctx, int which, double **device_normals, int64_t *slice_points, int32_t *pending);
ME_API int  me_icp_block(me_ctx *ctx, double **device_block, int32_t *n_sum);
ME_API int  me_icp_step(me_ctx *ctx, int32_t *done);
ME_API int  me_icp_end(me_ctx *ctx, me_icp_result *out);
/* The update of one iteration from a reduced block as a pure host function (no context, no device): Eigen::umeyama
 * without scaling (point-to-point; the sums are taken about `center`, the centre of the ground truth's bounding box), or
 * the 6x6 normal equations solved with partial pivoting + TransformVector6dToMatrix4d (point-to-plane, generalized ICP;
 * center may be NULL).  The identity when the count is 0 or the solve fails (Open3D).  update: row-major 4x4. */
ME_API int  me_icp_update(int32_t method, const double *block, const double center[3], double update[16]);
/* normals of a cloud held by the context, caller order, N x 3 fp64 (open3d PointCloud::normals_): upload / estimate as
 * PointCloud::EstimateNormals(KDTreeSearchParamKNN(knn)) does (k nearest neighbours incl. the point, covariance, the
 * eigenvector of the smallest eigenvalue; sign as Open3D's FastEigen3x3 leaves it) / read back.  me_transform rotates them. */
ME_API int  me_set_normals(me_ctx *ctx, int which, const double *normals_host, int64_t n);
ME_API int  me_estimate_normals(me_ctx *ctx, int which, int32_t knn);
ME_API int  me_get_normals(me_ctx *ctx, int which, double *normals_host);
/* builds (or rebuilds) the cell-sorted grid of one cloud; the eval calls build lazily if needed */
ME_API int  me_build_grid(me_ctx *ctx, int which);

/* ---- coarse global registration: the initial pose est -> gt without a hand-made initial_matrix ---------------------------
 * FPFH descriptors, mutual nearest-neighbour matching in descriptor space and RANSAC over the correspondences, all on the
 * device (Open3D's registration_ransac_based_on_feature_matching in spirit; the reference never calls it, its users align the
 * maps by hand).  The call works on two private feature clouds: the context's est and gt clouds, their normals, lattices and
 * per-point results are left as they were.  Pipeline:
 *   1. feature clouds: each cloud copied and down-sampled at voxel_size (me_voxel_downsample), exact k-NN normals
 *      (normal_knn, me_estimate_normals) oriented towards centroid + (0, 0, 10 * bbox diagonal) of that feature cloud;
 *   2. FPFH (33 fp32 per point): neighbourhood = the <= feature_max_nn nearest other points with d^2 < feature_radius^2
 *      (ties to the smaller index); pair features, 11 bins per group, SPFH + the neighbours' SPFH weighted by 1 / d^2;
 *   3. exact fp32 nearest neighbour in descriptor space (fixed dimension order, no contraction, ties to the smaller index)
 *      est -> gt and gt -> est; mutual_filter != 0 keeps the pairs that are each other's nearest;
 *   4. n_hypotheses RANSAC hypotheses h: three correspondences min(floor(uniform53(seed, h, 16 + t) * n), n - 1),
 *      rejected when two coincide, an edge fails min^2 >= edge_ratio^2 max^2 or the three are (nearly) collinear (the
 *      second singular value of their cross-covariance <= 1e-6 times the first), otherwise the rigid fit of the three and
 *      the count of correspondences with |R p + t - q|^2 < max_correspondence_distance^2.  The most inliers win, ties to
 *      the smallest h; every hypothesis is evaluated, so T is a pure function of (clouds, params, seed);
 *   5. refinement: the rigid fit over the winner's inliers; n_inliers and inlier_rmse under it.
 * Errors: ME_ERR_EMPTY for an empty cloud, ME_ERR_INVALID for bad parameters, fewer than 3 correspondences or no valid
 * hypothesis (the message says which). */
typedef struct {
  double  voxel_size;                  /* feature cloud: me_voxel_downsample at this size                              */
  int32_t normal_knn;                  /* 30                                                                            */
  double  feature_radius;              /* 10 * voxel_size (5 * voxel_size does not separate smooth terrain)            */
  int32_t feature_max_nn;              /* 128 (the largest): at most this many neighbours within the radius            */
  int32_t mutual_filter;               /* 1                                                                             */
  double  max_correspondence_distance; /* 1.5 * voxel_size: inlier test                                                 */
  double  edge_ratio;                  /* 0.9                                                                           */
  int64_t n_hypotheses;                /* 100000 (< 2^32)                                                               */
  uint64_t seed;
} me_global_reg_params;
typedef struct {
  double  T[16];                       /* row-major, est -> gt, like me_icp's transformation                           */
  int64_t n_est_features, n_gt_features, n_correspondences, n_valid_hypotheses;
  int64_t best_hypothesis, n_inliers;  /* the winner; inliers of the correspondences under the refined T              */
  double  inlier_rmse;                 /* sqrt(mean |T p - q|^2) over them                                             */
  double  stage_ms[6];                 /* CUDA-event times: copy + down-sample, normals, FPFH (both clouds), matching,
                                          RANSAC, refinement                                                           */
} me_global_reg_result;
ME_API int me_global_registration(me_ctx *ctx, const me_global_reg_params *p, me_global_reg_result *out);
/* the feature cloud of the last me_global_registration (which = ME_CLOUD_EST / ME_CLOUD_GT): points, oriented normals and
 * FPFH descriptors (33 fp32 per point), in the order of the down-sampled cloud.  Any of the three arrays may be NULL;
 * xyz == normals == fpfh33 == NULL: size query (*n).  capacity < n is an error. */
ME_API int me_get_features(me_ctx *ctx, int which, double *xyz, double *normals, float *fpfh33, int64_t capacity, int64_t *n);
/* the correspondences of the last me_global_registration that reached matching: (est feature index, gt feature index) in
 * est order.  est_idx == gt_idx == NULL: size query (*n).  capacity < n is an error. */
ME_API int me_get_correspondences(me_ctx *ctx, int32_t *est_idx, int32_t *gt_idx, int64_t capacity, int64_t *n);

/* replaces: MapEval::calculateMetricsWithInitialMatrix (map_eval.cpp:1204-1260), getDiffRegResultWithCorrespondence
 * (:1069-1145), the metric half of calculateMetrics (:1147-1202) and computeChamferDistance (:1398-1431).
 * me_eval_nn_accum: this rank's accumulators of the requested directions (the others zeroed), through the accumulator
 * block: it overwrites the block's NN sections of those directions, the sections me_eval_nn_accum_device writes. */
ME_API int  me_eval_nn_accum(me_ctx *ctx, const me_nn_params *p, me_nn_accum *est_to_gt, me_nn_accum *gt_to_est);
ME_API int  me_nn_finalize(const me_nn_params *p, const me_nn_accum *est_to_gt, const me_nn_accum *gt_to_est,
                    int64_t n_est, int64_t n_gt, me_nn_result *out);      /* host only, no device work */
ME_API int  me_eval_nn(me_ctx *ctx, const me_nn_params *p, me_nn_result *out);   /* accum + finalize, world must be 1 */
/* per-query nearest neighbour of the last me_eval_nn*, original point order of the QUERY cloud;
 * which_query = ME_CLOUD_EST -> est->gt sweep.  Only this rank's query range is filled (others -1 / NaN). */
ME_API int  me_get_nn(me_ctx *ctx, int which_query, int32_t *nn_index, double *nn_sqdist);

/* ---- accuracy curve: AC / COM / CD / F1 / IoU at any number of thresholds ------------------------------------------------
 * The five-level statistics of me_eval_nn* at K levels tau[0..K-1] (1 <= K <= ME_CURVE_MAX_LEVELS, finite, >= 0,
 * non-decreasing; anything else is ME_ERR_INVALID), from the per-query records of the LAST me_eval_nn* call: the same kept
 * pairs, the same distance d (ME_PAIRING_AS_WRITTEN: from the swapped indices, out-of-range pairs counted), d <= tau_k as
 * the reference compares.  No new sweep.  The records go stale with any me_set_cloud*, me_transform, me_voxel_downsample,
 * me_copy_cloud, me_add_*, ICP call or layout change after that call; the curve then fails with ME_ERR_INVALID.
 * me_nn_curve_accum_device: this rank's SUM-reducible block, on the device, *n = 2 (3 (K + 1) + 1) fp64 values: per direction
 * (est->gt, then gt->est) the count, sum d and sum d^2 (Eigen's squaredNorm) of the pairs of every bin b = 0..K (bin b: the
 * first level with d <= tau_b; bin K: above every level), then n_ub.  Directions the last call did not evaluate are zero.
 * Deterministic: two calls on the same device, world and layout give the same bits.  The caller all-reduces the block in
 * place (ncclAllReduce / torch.distributed after me_synchronize), copies it to the host and calls me_nn_curve_finalize with
 * the reduced accumulators of that me_eval_nn* call (host only; the formulas of me_nn_finalize per level, sigma from the
 * rank moments).  me_nn_curve: both steps, world must be 1. */
#define ME_CURVE_MAX_LEVELS 1024
typedef struct {
  int64_t n_inlier;                 /* pairs with d <= tau                                          */
  double  mean, rmse, fitness, sigma;
} me_curve_dir;
typedef struct {
  double  tau;
  me_curve_dir est_to_gt, gt_to_est;
  double  cd, f1, iou;              /* map_eval.cpp:1245-1253 at this level                          */
} me_curve_row;
ME_API int  me_nn_curve_accum_device(me_ctx *ctx, const double *tau, int32_t n_tau, double **device_block, int32_t *n);
ME_API int  me_nn_curve_finalize(const me_nn_params *p, const me_nn_accum *est_to_gt, const me_nn_accum *gt_to_est,
                                 const double *host_block, const double *tau, int32_t n_tau, int64_t n_est, int64_t n_gt,
                                 me_curve_row *rows);   /* host only, no device work */
ME_API int  me_nn_curve(me_ctx *ctx, const double *tau, int32_t n_tau, me_curve_row *rows);

/* ---- exact distance quantiles and the Hausdorff distance ------------------------------------------------------------------
 * From the per-query records of the LAST me_eval_nn* call (stale as for me_nn_curve*), per direction one population of fp64
 * distances:
 *   ME_DIST_KEPT  the kept pairs and their d, exactly as the five-level statistics and me_nn_curve* keep them (both cut-off
 *                 modes; ME_PAIRING_AS_WRITTEN gt->est: d from the swapped indices, out-of-range pairs left out).  n = n_corr.
 *   ME_DIST_NN    every evaluated query's nearest-neighbour distance sqrt(d2), the terms of sum_nn_dist (full CD).  Needs
 *                 want_full_cd = 1 in that call (else ME_ERR_INVALID).  n = n_query.
 * For probabilities p[0..K-1] (1 <= K <= ME_QUANTILE_MAX_PROBS, each finite and in [0, 1]; anything else is ME_ERR_INVALID) and
 * the sorted population x_0 <= .. <= x_{n-1}: h = (double)(n - 1) p, k = floor(h), g = h - k, lo = x_k, hi = x_{min(k+1, n-1)}
 * (both exact), value = lo + (hi - lo) g if g < 0.5 else hi - (hi - lo) (1 - g) — numpy's quantile(method="linear").  An empty
 * population, or a direction the call did not evaluate, has n = 0 and NaN values.  Exact and deterministic for any world:
 * only integer counts cross ranks.
 * The loop (as me_icp_begin .. me_icp_end): me_nn_quantile_begin checks the arguments and the records and runs pass 0;
 * me_nn_quantile_block hands out the running pass's SUM-reducible block (*n fp64 counts, the same length on every rank and
 * in every pass), which the caller all-reduces in place (after me_synchronize); me_nn_quantile_step reads the reduced block
 * and runs the next pass (*done = 1 after the last one); me_nn_quantile_end fills the result.  A call that changes the clouds
 * between begin and end makes step and end fail.  me_nn_quantiles: the whole loop, world must be 1.
 * me_quantile_finalize (host only): value[k] from n, p[k] and lo_hi[2k] = lo, lo_hi[2k + 1] = hi, by the rule above. */
#define ME_QUANTILE_MAX_PROBS 64
enum { ME_DIST_KEPT = 0, ME_DIST_NN = 1 };
typedef struct {
  int64_t n;                                    /* population size                                           */
  double  min, max;                             /* x_0, x_{n-1}; max is the one-sided Hausdorff distance (ME_DIST_NN) */
  int64_t rank[ME_QUANTILE_MAX_PROBS];          /* k = floor((n - 1) p)                                      */
  double  lo[ME_QUANTILE_MAX_PROBS], hi[ME_QUANTILE_MAX_PROBS], value[ME_QUANTILE_MAX_PROBS];
} me_quantile_dir;
typedef struct {
  int32_t population, n_probs;
  double  p[ME_QUANTILE_MAX_PROBS];
  me_quantile_dir est_to_gt, gt_to_est;
  double  hausdorff;                            /* ME_DIST_NN, both directions: max of the two maxima; else NaN */
} me_quantile_result;
ME_API int  me_nn_quantile_begin(me_ctx *ctx, int32_t population, const double *p, int32_t n_probs);
ME_API int  me_nn_quantile_block(me_ctx *ctx, double **device_block, int32_t *n);
ME_API int  me_nn_quantile_step(me_ctx *ctx, int32_t *done);
ME_API int  me_nn_quantile_end(me_ctx *ctx, me_quantile_result *out);
ME_API int  me_nn_quantiles(me_ctx *ctx, int32_t population, const double *p, int32_t n_probs, me_quantile_result *out);
ME_API int  me_quantile_finalize(int64_t n, const double *p, int32_t n_probs, const double *lo_hi, double *values);  /* host only */

/* ---- AC / COM / CD / F1 / IoU per region ----------------------------------------------------------------------------------
 * From the per-query records of the LAST me_eval_nn* call (stale as for me_nn_curve*), the five-level statistics split by the
 * region of the query point.  For region edge s (finite, > 0) a point's region is (ix, iy, iz) = floor(x / s) per axis (IEEE
 * division, as the voxel index of the AWD stage), taken from the clouds as they are now; every index must satisfy
 * |index| < 2^20 (else ME_ERR_INVALID, naming the axis and the smallest s that fits).  The occupied regions — those holding a
 * point of either whole cloud — are listed ascending by (ix, iy, iz), at most ME_REGION_MAX_REGIONS (else ME_ERR_INVALID);
 * the list and n_est / n_gt per region are the same on every rank.  A record counts in the region of its query point and is
 * kept exactly as the five-level pass keeps it (cut-off modes, ME_PAIRING_AS_WRITTEN gt->est distances).
 * Device block: n_sum = ME_REGION_SUM_FIELDS * 2 * n_regions SUM-reducible values, [region][direction][field] with the fields
 *   n_query n_corr n_inlier[5] sum_d[5] sum_d2[5] sum_nn_dist   (counts as fp64; sum_nn_dist only after want_full_cd = 1)
 * then n_max = ME_REGION_MAX_FIELDS * 2 * n_regions MAX-reducible values, [region][direction][max_d, max_nn] (0 when the set is
 * empty; max_nn only after want_full_cd = 1).  The same length on every rank.  No floating-point atomics: two calls on the
 * same device, world and layout give the same bits; counts and maxima are the same for any world and layout.
 * The loop: me_nn_region_begin lists the regions and folds this rank's records into the block; me_nn_region_block hands the
 * block out (all-reduce the SUM part with SUM and the MAX part with MAX, in place, after me_synchronize); me_nn_region_end
 * reads the reduced block and fills rows[0 .. n_regions - 1] (capacity >= n_regions).  A call that changes the clouds between
 * begin and end makes block and end fail.  me_nn_regions: the whole loop at world 1, rows allocated by the library (me_free).
 * me_region_finalize (host only): rows from a reduced host block (SUM part, then MAX part), the region indices (3 per region)
 * and the counts — mean / rmse / fitness per direction and level as me_nn_finalize forms them with n_source = the region's
 * point count of the query cloud, cd / f1 / iou with the region's n_est / n_gt, mean_nn = sum_nn_dist / n_query.  There is no
 * sigma per region (DESIGN §3.12). */
#define ME_REGION_MAX_REGIONS (1 << 21)
#define ME_REGION_SUM_FIELDS 18
#define ME_REGION_MAX_FIELDS 2
typedef struct {
  int64_t n_query, n_corr, n_inlier[5];
  double  sum_d[5], sum_d2[5], sum_nn_dist;
  double  max_d, max_nn;                        /* largest kept d, largest sqrt(d2); 0 for an empty set */
  double  mean[5], rmse[5], fitness[5];
  double  mean_nn;                              /* sum_nn_dist / n_query */
} me_region_dir;
typedef struct {
  int64_t index[3];                             /* (ix, iy, iz) */
  double  min[3], max[3];                       /* index * s, (index + 1) * s */
  int64_t n_est, n_gt;                          /* points of each whole cloud in the region */
  me_region_dir est_to_gt, gt_to_est;
  double  cd[5], f1[5], iou[5];
} me_region_row;
ME_API int  me_nn_region_begin(me_ctx *ctx, double region_size, int64_t *n_regions);
ME_API int  me_nn_region_block(me_ctx *ctx, double **device_block, int32_t *n_sum, int32_t *n_max);
ME_API int  me_nn_region_end(me_ctx *ctx, me_region_row *rows, int64_t capacity);
ME_API int  me_nn_regions(me_ctx *ctx, double region_size, me_region_row **rows, int64_t *n_regions);
ME_API int  me_region_finalize(int64_t n_regions, double region_size, const int64_t *index, const int64_t *n_est,
                               const int64_t *n_gt, const double *host_block, me_region_row *rows);   /* host only */

/* ---- point-to-plane metrics and normal consistency ---------------------------------------------------------------------
 * From the per-query records of the LAST me_eval_nn* call (stale as for me_nn_curve*), with that call's tau, cut-off mode and
 * want_full_cd: the five-level statistics with the point-to-point distance d replaced by the distance of the query point to
 * the tangent plane of its nearest neighbour, and the agreement of the two normals of every pair.  No reference counterpart.
 * Direction q (query cloud q, reference cloud 1 - q) walks its records with GEOMETRIC pairing always: under
 * ME_PAIRING_AS_WRITTEN the gt->est pair is a pair of swapped indices, whose tangent plane means nothing, so n_corr of the
 * gt->est table equals me_eval_nn's only under geometric pairing.  For a record with neighbour j >= 0: p = query point,
 * t = reference point j (caller order), n = reference normal j, m = the query's own normal.  A normal is usable iff its
 * squared norm (x*x + (y*y + z*z)) is finite and > 0.  With d = p - t, every operation rounded on its own (no FMA):
 *   e = |(dx nx + dy ny) + dz nz| / sqrt(|n|^2),   c = min(1, |(mx nx + my ny) + mz nz| / (sqrt(|m|^2) sqrt(|n|^2))).
 * (the min is fmin: a NaN ratio counts as 1).
 * A kept pair (the five-level pass's cut-off on the record's d2) with usable n counts in n_corr and its e goes where the
 * five-level pass puts d (n_inlier / sum_d / sum_d2 per level with e <= tau_k, the rank's moment slot); with unusable n it
 * counts in n_no_normal and nowhere else.  A kept pair with usable n and m adds 1 to n_nc and c to sum_c.  After
 * want_full_cd = 1 every query with j >= 0 and usable n adds e to sum_nn_dist and to max_e_nn (unusable n: n_no_normal_nn).
 * max_e is the largest kept e; n_query is the five-level pass's; n_ub and n_far are 0.
 * Device block: ME_SURFACE_BLOCK_SUM SUM-reducible values — the two directions laid out as the NN section of the accumulator
 * block (ME_NN_ACCUM_I64 + ME_NN_ACCUM_F64 each, me_nn_accum's fields as fp64), then per direction n_no_normal,
 * n_no_normal_nn, n_nc, sum_c — and ME_SURFACE_BLOCK_MAX MAX-reducible values, per direction max_e, max_e_nn.  No
 * floating-point atomics: two calls on one device, world and layout give the same bits; counts and maxima are the same for
 * any world and layout.
 * Normals (knn): 0 — both clouds must hold normals (me_set_normals / me_estimate_normals, a file's, averaged by
 * me_voxel_downsample); 1..64 — a cloud without normals gets exact k-NN normals (me_estimate_normals' rule) as a working
 * copy: the cloud still has no normals afterwards, after a failure too.  A working estimate needs the replicated layout.
 * The loop: me_nn_surface_begin checks; me_nn_surface_normals_slice per cloud estimates this rank's caller-index slice of a
 * working normal set into the buffer it returns (*pending = 1: all-gather slice_points * 3 fp64 per rank in place after
 * me_synchronize; 0: nothing to do); me_nn_surface_block folds the records into the block on its first call (SUM-reduce the
 * first n_sum values and MAX-reduce the next n_max in place); me_nn_surface_end reads the reduced block.  The records are
 * only read.  Refused: knn outside 0..64, stale records, missing normals with knn = 0, a working estimate on ME_LAYOUT_SLAB,
 * begin while a registration or drift loop is open, calls out of order, and a cloud changed between begin and end.
 * me_nn_surface: the whole loop at world 1.  me_surface_finalize (host only): the result from a reduced host block;
 * plane is me_nn_finalize of the NN-laid-out part. */
#define ME_SURFACE_BLOCK_SUM (2 * (ME_NN_ACCUM_I64 + ME_NN_ACCUM_F64) + 8)
#define ME_SURFACE_BLOCK_MAX 4
typedef struct {
  int64_t n_no_normal;                          /* kept pairs without a usable reference normal */
  int64_t n_no_normal_nn;                       /* full-CD queries without a usable reference normal */
  int64_t n_nc;                                 /* kept pairs with both normals usable */
  double  normal_consistency;                   /* sum_c / n_nc; NaN when n_nc = 0 */
  double  max_e, max_e_nn;                      /* largest kept e, largest full-CD e; 0 for an empty set */
} me_surface_dir;
typedef struct {
  me_nn_result   plane;                         /* the five-level table of e; full_cd from the e of every query */
  me_surface_dir est_to_gt, gt_to_est;
  double         normal_consistency;            /* mean of the two directions'; NaN if either is NaN */
} me_surface_result;
ME_API int  me_nn_surface_begin(me_ctx *ctx, int32_t knn);
ME_API int  me_nn_surface_normals_slice(me_ctx *ctx, int which, double **device_normals, int64_t *slice_points, int32_t *pending);
ME_API int  me_nn_surface_block(me_ctx *ctx, double **device_block, int32_t *n_sum, int32_t *n_max);
ME_API int  me_nn_surface_end(me_ctx *ctx, me_surface_result *out);
ME_API int  me_nn_surface(me_ctx *ctx, int32_t knn, me_surface_result *out);
ME_API int  me_surface_finalize(const me_nn_params *p, const double *host_block, int64_t n_est, int64_t n_gt,
                                me_surface_result *out);   /* host only */

/* ---- drift per region: every region of the estimated cloud aligned to the ground truth on its own --------------------------
 * Separates a region that is shifted or turned as a whole (drift) from one that is noisy or smeared (damage): a rigid
 * point-to-point ICP per region, all of them in one pass over the cloud per iteration.
 * Regions: an est point's region is floor(x / s) per axis (IEEE division), the rule of me_nn_region_begin, taken from the
 * estimated cloud as it is at me_drift_begin; only regions holding est points are listed, ascending by (ix, iy, iz), with
 * the limits and messages of me_nn_region_begin (|index| < 2^20, at most ME_REGION_MAX_REGIONS).  Membership is fixed at
 * begin.  Region r has a transform T_r, I at first.  Each iteration:
 *   1. every est point i := T_{r(i)} x_i (original coordinates, me_transform's rounding: never compounded on moved points);
 *   2. one est->gt sweep as registration runs it (ME_CUTOFF_DIST_LT_R, geometric pairing, est->gt only);
 *   3. per region the ME_ICP_BLOCK_P2P sums of its kept pairs (nn >= 0, d2 < R^2), about the region centre
 *      c_r = ((ix + 0.5) s, (iy + 0.5) s, (iz + 0.5) s);
 *   4. every region not done: fitness = n_corr / n_est, rmse = sqrt(sum d2 / n_corr) (0 without pairs), me_icp_step's
 *      convergence test, then update = me_icp_update(ME_ICP_POINT_TO_POINT, block_r, c_r) and T_r := update T_r.
 * A region is done when it converged (ME_DRIFT_CONVERGED), made max_iteration updates (ME_DRIFT_ITERATION_LIMIT), or an update
 * was due with fewer than 3 pairs (ME_DRIFT_TOO_FEW, T_r kept).  The loop ends when every region is done.
 * Device block: n_sum = ME_ICP_BLOCK_P2P * n_regions SUM-reducible values, [region][count, sum p (3), sum q (3), sum q p^T (9),
 * sum d2].  Folded in caller order per region with a fixed shuffle tree and every product and sum rounded on its own; no
 * floating-point atomics, so two calls give the same bits.
 * The loop (as me_icp_begin .. me_icp_end; every rank the same calls): me_drift_begin checks, lists the regions, keeps a copy
 * of the estimated cloud and runs the first sweep; me_drift_block hands out the block (SUM-all-reduce it in place after
 * me_synchronize); me_drift_step reads the reduced block, updates, moves and sweeps (*done = 1: nothing left to reduce);
 * me_drift_end fills rows[0 .. n_regions - 1] (capacity >= n_regions).  After me_drift_end, and after any failure while the
 * loop is open, the estimated cloud's points and normals are as they were at begin; the NN records are stale.  Refused: s or R
 * not finite and > 0, max_iteration < 0, an empty cloud, a borrowed estimated cloud, world > 1 with ME_LAYOUT_SLAB requested,
 * begin while a registration or drift loop is open (and me_icp_begin while a drift loop is open), calls out of order, and a
 * cloud changed during the loop (the next loop call fails and closes the loop; an estimated cloud set into the same buffer is
 * overwritten by the one held at begin).  Arguments are checked before anything else, so a begin refused for them leaves an
 * open loop running.  me_drift: the whole loop at world 1, rows allocated by the library (me_free). */
enum { ME_DRIFT_CONVERGED = 0, ME_DRIFT_ITERATION_LIMIT = 1, ME_DRIFT_TOO_FEW = 2 };
typedef struct {
  int64_t index[3];                             /* (ix, iy, iz) */
  double  min[3], max[3];                       /* index * s, (index + 1) * s */
  int64_t n_est;                                /* est points in the region */
  int64_t n_corr_before;                        /* the first sweep, T_r = I */
  double  fitness_before, rmse_before;
  int64_t n_corr;                               /* the sweep at the final T_r */
  double  fitness, rmse;
  double  T[16];                                /* row-major: moves the region onto the ground truth */
  double  centroid[3];                          /* mean of the region's original est points */
  double  shift[3], shift_norm;                 /* T_r centroid - centroid, and its length */
  double  angle;                                /* rotation angle of T_r in radians */
  int32_t iterations, status;                   /* updates applied; ME_DRIFT_* */
} me_drift_row;
ME_API int  me_drift_begin(me_ctx *ctx, double region_size, double max_correspondence_distance, int32_t max_iteration,
                           double relative_fitness, double relative_rmse, int64_t *n_regions);
ME_API int  me_drift_block(me_ctx *ctx, double **device_block, int32_t *n_sum);
ME_API int  me_drift_step(me_ctx *ctx, int32_t *done);
ME_API int  me_drift_end(me_ctx *ctx, me_drift_row *rows, int64_t capacity);
ME_API int  me_drift(me_ctx *ctx, double region_size, double max_correspondence_distance, int32_t max_iteration,
                     double relative_fitness, double relative_rmse, me_drift_row **rows, int64_t *n_regions);

/* ---- local map consistency without a ground truth: mean plane variance beside MME ----------------------------------------
 * For cloud `which` as it is now, radius r (finite, > 0) and min_neighbors m (>= 3), per point q: MME's neighbourhood (the
 * points p of the same cloud with d2 < r^2, nanoflann's d2 and strict test, q included; k = accepted - 1) and MME's moments,
 * taken about q from the fp64 offsets q - p of the raw coordinates in the order of MME's fp64 walk (rows by dz, then dy,
 * ascending; x-runs ascending in the cell-sorted order).  C = (S2 - S1 S1^T / k) / (k - 1) as MME forms it.
 *   entropy e = 0.5 ln(2 pi e det C) as MME: valid when k >= m and e is finite (n_valid, sum_entropy); invalid points store 0.
 *   plane variance v = max(0, smallest eigenvalue of C) (cyclic Jacobi, fp64): valid when k >= m and v is finite (n_pv,
 *   sum_pv, sum_sqrt_pv, max_pv); a point with k < m stores NaN.  A perfect plane has v = 0 (valid) and no entropy.
 * Whole map: mme = sum_entropy / n_valid (0 when n_valid = 0, as me_mme_finalize), mpv = sum_pv / n_pv and mean_plane_std =
 * sum_sqrt_pv / n_pv (NaN when n_pv = 0), max_pv (NaN when n_pv = 0).
 * Regions, for region_size s > 0: a point's region is floor(x / s) per axis, the occupied list of me_nn_region_begin over est ++
 * gt (est alone while the gt cloud is empty), with its limits and messages; one row per listed region, n_points = the region's
 * points of this cloud.  s = 0: no rows.  The whole-map result is the rows' sums added in list order (s > 0).
 * Device block: ME_CONSISTENCY_SUM_FIELDS SUM-reducible values per region [n_query n_valid n_pv sum_entropy sum_pv sum_sqrt_pv]
 * (counts as fp64), then ME_CONSISTENCY_MAX_FIELDS MAX-reducible values per region [max_pv] (0 for an empty set); at s = 0 the
 * block holds one region, the whole map.  The same length on every rank.  Folded in caller order per region (chunks of 1024
 * points, a fixed shuffle tree, chunks added in order); no floating-point atomics, so two calls on one device, world and
 * lattice give the same bits while the cloud is not laid out again in between (a new layout may order the points of a cell
 * differently), and counts are the same for any world.
 * The sweep lays the cloud out as me_eval_mme does (the shared lattice, or a lattice of its own with h = r / 2 when r spans
 * more than 3 shared cells), which can make that cloud's NN records stale; it leaves MME's results (me_get_entropies) and
 * the kernel trace alone.  *kernel / rings / solo of the result say which sweep ran (me_consistency_kernel).
 * The loop (every rank the same calls): me_consistency_begin checks, sweeps this rank's query range and folds it; *n_regions =
 * the rows me_consistency_end will fill (0 at s = 0).  me_consistency_block hands out the block (SUM-reduce the first n_sum
 * values and MAX-reduce the next n_max in place, after me_synchronize); me_consistency_end reads the reduced block and fills
 * rows[0 .. n_regions - 1] (capacity >= n_regions; rows may be NULL when n_regions = 0) and *whole.  Refused: r not finite
 * and > 0, m < 3, s negative or not finite, an empty cloud, an open registration or drift loop, world > 1 with ME_LAYOUT_SLAB
 * requested, the region list's limits, calls out of order, and a cloud changed between begin and end.
 * me_consistency: the whole loop at world 1, rows allocated by the library (me_free; NULL at s = 0).
 * me_consistency_finalize (host only): rows and the whole-map result from a reduced host block, the region indices (3 per
 * region), the per-region point counts and the cloud size (radius, min_neighbors, kernel, rings and solo are left 0).
 * me_get_consistency_points: the last call's e and v of cloud `which`, caller order (either pointer may be NULL); points
 * another rank evaluated hold 0 and NaN.  Valid until the cloud changes. */
#define ME_CONSISTENCY_SUM_FIELDS 6
#define ME_CONSISTENCY_MAX_FIELDS 1
enum me_consistency_kernel {
  ME_CONSISTENCY_WALK = 0           /* consistency_walk_kernel: MME's fp64 generic walk (mme_kernel's order)   */
};
typedef struct {
  int64_t index[3];                             /* (ix, iy, iz) */
  double  min[3], max[3];                       /* index * s, (index + 1) * s */
  int64_t n_points;                             /* points of the cloud in the region */
  int64_t n_query, n_valid, n_pv;               /* evaluated points; valid entropies; valid plane variances */
  double  sum_entropy, sum_pv, sum_sqrt_pv;
  double  mme, mpv, mean_plane_std, max_pv;
} me_consistency_row;
typedef struct {
  double  radius, region_size;
  int32_t min_neighbors, kernel, rings, solo;   /* kernel: me_consistency_kernel; solo: the cloud's own lattice (h = r / 2) */
  int64_t n_regions;
  int64_t n_points, n_query, n_valid, n_pv;
  double  sum_entropy, sum_pv, sum_sqrt_pv;
  double  mme, mpv, mean_plane_std, max_pv;
} me_consistency_result;
ME_API int  me_consistency_begin(me_ctx *ctx, int which, double radius, int32_t min_neighbors, double region_size,
                                 int64_t *n_regions);
ME_API int  me_consistency_block(me_ctx *ctx, double **device_block, int32_t *n_sum, int32_t *n_max);
ME_API int  me_consistency_end(me_ctx *ctx, me_consistency_row *rows, int64_t capacity, me_consistency_result *whole);
ME_API int  me_consistency(me_ctx *ctx, int which, double radius, int32_t min_neighbors, double region_size,
                           me_consistency_row **rows, int64_t *n_regions, me_consistency_result *whole);
ME_API int  me_consistency_finalize(int64_t n_regions, double region_size, const int64_t *index, const int64_t *n_points,
                                    int64_t n_total, const double *host_block, me_consistency_row *rows,
                                    me_consistency_result *whole);   /* host only */
ME_API int  me_get_consistency_points(me_ctx *ctx, int which, double *entropy, double *plane_variance);

/* ---- the mutually orthogonal metric (MOM) without a ground truth: plane thickness on three orthogonal plane families ------
 * After Kornilova & Ferrer (ECMR 2021), by this project's own rule (DESIGN §3.16).  For cloud `which` as it is now, radius r
 * and min_neighbors m as me_consistency_begin, and the parameters p (angle_deg in (0, 30], planarity in (0, 1], min_family >=
 * 1), per point: me_consistency's neighbourhood, covariance and v (the same bits), lambda2 = the middle eigenvalue, and the
 * unit normal n = the eigenvector of v's eigenvalue, normalised in fp64, its largest component positive (the lowest axis on a
 * tie).  Planar: k >= m, v finite, lambda2 > 0 and v <= planarity * lambda2.  Every planar point adds 1 to the cube-map bins
 * of n and of -n (6 ME_MOM_CELLS_PER_EDGE^2 bins; DESIGN §3.16); me_mom_axes picks a1, a2, a3 from the reduced histogram.
 * Family j: the planar points with |n . a_j| >= cos(angle) (the lowest j first).  Per family: n_j, mean_j = sum v / n_j and
 * median_j = numpy's quantile(v, 0.5, method="linear"), exact.  mom = median_1 + median_2 + median_3, NaN unless status is
 * ME_MOM_OK (any n_j < min_family: ME_MOM_SMALL_FAMILY; the per-family fields are still filled).  Without axes
 * (ME_MOM_NO_PLANAR, ME_MOM_NO_SECOND_AXIS) no family is formed: n_j = 0, mean_j and median_j are NaN, every point's family
 * is -1, and axis holds a1 (ME_MOM_NO_SECOND_AXIS) or NaN.
 * The loop (every rank the same calls): me_mom_begin checks, sweeps this rank's query range and histograms it;
 * me_mom_block hands out the running pass's block (*n = ME_MOM_BLOCK fp64 values, every rank and pass), which the caller
 * SUM-reduces in place (after me_synchronize); me_mom_step reads the reduced block and runs the next pass (*done = 1 after
 * the last); me_mom_end fills the result.  Refused as me_consistency_begin (r, m, an empty cloud, an open registration or
 * drift loop, world > 1 with ME_LAYOUT_SLAB requested, calls out of order, a cloud changed between begin and end), and
 * angle_deg, planarity or min_family out of range.  The sweep lays the cloud out as me_consistency_begin does.
 * me_mom: the whole loop at world 1.  me_mom_axes (host only): the axes (9 values, a1 a2 a3, NaN when not found) and the
 * status (ME_MOM_OK, ME_MOM_NO_PLANAR, ME_MOM_NO_SECOND_AXIS) from an integer histogram of 6 M^2 bins.
 * me_get_mom_points: the last call's v, lambda2, normal (3 per point) and family (0..2, -1 none) of cloud `which`, caller
 * order (any pointer may be NULL); points another rank evaluated hold NaN and -1.  Valid until the cloud changes. */
#define ME_MOM_CELLS_PER_EDGE 16
#define ME_MOM_BINS (6 * ME_MOM_CELLS_PER_EDGE * ME_MOM_CELLS_PER_EDGE)
#define ME_MOM_BLOCK (6 + 3 * 4 * 256)
enum me_mom_status {
  ME_MOM_OK = 0,
  ME_MOM_NO_PLANAR = 1,             /* no planar point                                  */
  ME_MOM_NO_SECOND_AXIS = 2,        /* no populated bin within angle_deg of a1's plane   */
  ME_MOM_SMALL_FAMILY = 3           /* a family has fewer than min_family points         */
};
typedef struct {
  double  angle_deg;                            /* (0, 30]; 10 by default */
  double  planarity;                            /* (0, 1];  0.5 by default */
  int64_t min_family;                           /* >= 1;    100 by default */
} me_mom_params;
typedef struct {
  double  radius, angle_deg, planarity;
  int64_t min_family;
  int32_t min_neighbors, kernel, rings, solo;   /* as me_consistency_result */
  int64_t n_points, n_query, n_pv, n_planar;
  double  axis[9];                              /* a1, a2, a3 */
  int64_t n[3];
  double  mean[3], median[3];
  double  mom;
  int32_t status, reserved;
} me_mom_result;
ME_API int  me_mom_begin(me_ctx *ctx, int which, double radius, int32_t min_neighbors, const me_mom_params *p);
ME_API int  me_mom_block(me_ctx *ctx, double **device_block, int32_t *n);
ME_API int  me_mom_step(me_ctx *ctx, int32_t *done);
ME_API int  me_mom_end(me_ctx *ctx, me_mom_result *out);
ME_API int  me_mom(me_ctx *ctx, int which, double radius, int32_t min_neighbors, const me_mom_params *p, me_mom_result *out);
ME_API int  me_mom_axes(const int64_t *hist, int32_t cells_per_edge, double angle_deg, double *axes, int32_t *status);  /* host only */
ME_API int  me_get_mom_points(me_ctx *ctx, int which, double *v, double *lambda2, double *normal, int8_t *family);

/* ---- the mutually orthogonal metric per region: where a plane family is thick ---------------------------------------------
 * A breakdown of the last finished MOM call (me_mom_end) by region, without a new sweep (DESIGN §3.17): that call's cloud,
 * axes, families and per-point v, valid while no cloud changed since its me_mom_begin.  A point's region is floor(x / s) per
 * axis, the occupied list of me_consistency_begin (est ++ gt, est alone while the gt cloud is empty) with its limits and
 * messages; at equal s the rows are the rows of me_consistency_end, in the same order.  Per region: n_points (the cloud's
 * points), n_planar (its planar points, with a family or not), and per family j of the whole map: n_j, mean_j = sum v / n_j
 * and median_j = numpy's quantile(v, 0.5, method="linear") of the members in the region, exact (NaN where n_j = 0);
 * mom = (median_1 + median_2) + median_3.  status: the whole-map status when it is ME_MOM_NO_PLANAR or ME_MOM_NO_SECOND_AXIS
 * (then n_j = 0 and NaN values); else ME_MOM_SMALL_FAMILY when some n_j < min_family (mom NaN, the per-family fields filled);
 * else ME_MOM_OK.  The axes are the whole map's: a region whose surfaces do not lie along them has empty families.
 * The loop (every rank the same calls): me_mom_region_begin checks and writes this rank's points into the block, *n_regions =
 * the rows me_mom_region_end will fill; me_mom_region_block hands out the block (*n = 2 n_points fp64 values [v | code], code
 * 0 for a point not planar or not swept by this rank, family + 1, or 4 for a planar point without a family; the same length
 * on every rank), which the caller SUM-reduces in place (after me_synchronize); me_mom_region_end sorts the members of the
 * reduced block by (region, family, v) and fills rows[0 .. n_regions - 1] (capacity >= n_regions).  Every rank computes the
 * same bits from the reduced block.  Refused: no finished me_mom_end, a cloud changed since that call's me_mom_begin, s not
 * finite or <= 0, min_family < 1, the region list's limits, an open registration or drift loop, world > 1 with ME_LAYOUT_SLAB
 * requested, calls out of order, and a cloud changed between begin and end.  The MOM call's result and me_get_mom_points are
 * left as they were.  me_mom_regions: the whole loop at world 1, rows allocated by the library (me_free). */
typedef struct {
  int64_t index[3];                             /* (ix, iy, iz) */
  int64_t n_points, n_planar;
  int64_t n[3];
  double  mean[3], median[3];
  double  mom;
  int32_t status, reserved;                     /* status: me_mom_status */
} me_mom_region_row;
ME_API int  me_mom_region_begin(me_ctx *ctx, double region_size, int64_t min_family, int64_t *n_regions);
ME_API int  me_mom_region_block(me_ctx *ctx, double **device_block, int64_t *n);
ME_API int  me_mom_region_end(me_ctx *ctx, me_mom_region_row *rows, int64_t capacity);
ME_API int  me_mom_regions(me_ctx *ctx, double region_size, int64_t min_family, me_mom_region_row **rows, int64_t *n_regions);

/* replaces: ComputeMeanMapEntropyUsingNormalTBB / ...UsingNormal (min_neighbors 10, map_eval.cpp:1608-1737, 1538-1606),
 * ComputeMeanMapEntropy (min_neighbors 5, :1438-1535), ComputeEntropy (:1433-1436) and the min/max side effect of
 * ColorPointCloudByMME (:697-701).  entropies_host (nullable) receives N fp64, zeros where invalid.
 * me_eval_mme_accum goes through the accumulator block: it overwrites the MME section of cloud `which`, the section
 * me_eval_mme_accum_device writes for that cloud. */
ME_API int  me_eval_mme_accum(me_ctx *ctx, int which, double radius, int32_t min_neighbors, me_mme_accum *out);
ME_API int  me_mme_finalize(const me_mme_accum *acc, int64_t n_total, me_mme_result *out);   /* host only */
ME_API int  me_eval_mme(me_ctx *ctx, int which, double radius, int32_t min_neighbors, me_mme_result *out,
                 double *entropies_host);
ME_API int  me_get_entropies(me_ctx *ctx, int which, double *entropies_host);

/* Device-resident accumulators, for multi-GPU passes without host round trips: me_accum_reset clears the context's
 * accumulator block; the *_device calls run the same sweeps as me_eval_nn_accum / me_eval_mme_accum but leave the partial
 * accumulators in that block (fp64; counts ride as fp64, exact below 2^53) — each call writes only its own sections (NN: those of
 * the evaluated directions; MME: the cloud's), as do me_eval_nn_accum / me_eval_mme_accum, so a section survives calls that
 * write other sections; me_accum_block hands out its DEVICE address:
 * the first *n_sum values are SUM-reducible, the following *n_max values MAX-reducible (entropy maximum and negated
 * minimum per cloud) — the caller all-reduces them in place (ncclAllReduce / torch.distributed on the context's stream);
 * me_accum_fetch copies the block back ONCE and fills the accumulator structs (any of them may be NULL), ready for
 * me_nn_finalize / me_mme_finalize.  Replaces the reductions of map_eval.cpp:1411,1420,1704-1708 across GPUs. */
ME_API int  me_accum_reset(me_ctx *ctx);
ME_API int  me_eval_nn_accum_device(me_ctx *ctx, const me_nn_params *p);
ME_API int  me_eval_mme_accum_device(me_ctx *ctx, int which, double radius, int32_t min_neighbors);
ME_API int  me_accum_block(me_ctx *ctx, double **device_block, int32_t *n_sum, int32_t *n_max);
ME_API int  me_accum_fetch(me_ctx *ctx, me_nn_accum *est_to_gt, me_nn_accum *gt_to_est, me_mme_accum *mme_est,
                           me_mme_accum *mme_gt);
/* The voxel stage (calculateVMD, map_eval.cpp:240-390) in two halves, for either layout.  me_voxel_begin: lattices,
 * per-voxel Gaussians, pairing and Wasserstein distances of the voxels this rank owns (all of them on a replicated layout).
 * me_voxel_w_table: DEVICE address and length of the W table over the estimated cloud's voxels (-1 = no pair) — on an
 * active slab layout the caller MAX-all-reduces it in place, so that every rank sees the W of its neighbours' voxels (SCS
 * reads 11^3 voxels around each pair, map_eval.cpp:353).  me_voxel_finish_accum_device: the SCS sweep over this rank's
 * pairs; leaves the stage's eight SUM-reducible values in the accumulator block.  me_accum_fetch_awd: after the block's
 * all-reduce, AWD / SCS / the voxel counts (map_eval.cpp:324-325,387) from the block. */
ME_API int  me_voxel_begin(me_ctx *ctx, double voxel_size, int32_t min_points);
ME_API int  me_voxel_w_table(me_ctx *ctx, double **device_w, int64_t *n);
ME_API int  me_voxel_finish_accum_device(me_ctx *ctx, int32_t scs_radius);
ME_API int  me_accum_fetch_awd(me_ctx *ctx, me_awd_result *out);

/* replaces: MapEval::calculateVMD (map_eval.cpp:240-390) with VoxelCalculator::buildVoxelMap / computeVoxelEntropy /
 * updateVoxelMap / computeWassersteinDistanceGaussian / getNeighborIndices (voxel_calculator.cpp:7-56,97-172,241-245).
 * rows27 (nullable): library-allocated n_rows x 27 table = the columns of voxel_errors.txt (map_eval.cpp:292-302),
 * release with me_free.  Replicated layout only: every rank computes the whole voxel stage (me_voxel_* shards it). */
ME_API int  me_eval_awd(me_ctx *ctx, double voxel_size, int32_t min_points, int32_t scs_radius, me_awd_result *out,
                 int64_t *n_rows, double **rows27);
/* The voxel-pair half of calculateVMD on GIVEN voxel Gaussians: rows27 = n_rows x 27 in the column layout of
 * voxel_errors.txt (map_eval.cpp:292-302: vmin[3] vmax[3] mu_est[3] W n_gt n_est sigma_est[6] mu_gt[3] sigma_gt[6]).
 * Recomputes W per row (w_out, nullable) with the device implementation of computeWassersteinDistanceGaussian
 * (voxel_calculator.cpp:115-140) and AWD / SCS over those voxels (map_eval.cpp:324-325, 351-387).  This is how the
 * tests pin the kernels to the sample output the reference ships (map_eval/scripts/voxel_errors.txt). */
ME_API int  me_awd_from_rows(me_ctx *ctx, const double *rows27, int64_t n_rows, double voxel_size, int32_t scs_radius,
                      double *w_out, me_awd_result *out);
ME_API void me_free(void *p);

/* ---- the Gaussian 2-Wasserstein distance per voxel (no reference counterpart; DESIGN §3.18) -----------------------------
 * Voxels floor(x / v) as for AWD; a voxel is paired when it is occupied in both clouds with >= min_points (>= 2) points in
 * each.  Per pair: mu = the mean of the voxel's points, Sigma = M2 / (n - 1) (unbiased, no clamp), offset o = |mu_est -
 * mu_gt|, shape b = Bures(Sigma_gt, Sigma_est) with b^2 = tr Sigma_gt + tr Sigma_est - 2 tr((Sigma_gt^1/2 Sigma_est
 * Sigma_gt^1/2)^1/2), W2 = sqrt(o^2 + b^2), symmetric in the two clouds.  b is taken as the residual |A - B P Q^T|_F of the
 * square roots A = Sigma_gt^1/2, B = Sigma_est^1/2 and the SVD B A = P S Q^T, in which nothing cancels: on an exact copy of
 * the ground truth it is at the rounding of the moments, where the trace formula leaves ~sqrt(u tr Sigma).  SCS is the
 * AWD stage's rule over W2.  Everything runs in fp64. */
#define ME_W2_ROW_COLS 26     /* vmin[3] n_gt n_est mu_est[3] mu_gt[3] sigma_est[6] sigma_gt[6] offset shape w2;
                                 sigma as xx xy xz yy yz zz */
#define ME_W2_BLOCK 8         /* the SUM-reducible block: n_pairs n_scs n_voxels_est n_voxels_gt sum_w2 sum_scs
                                 sum_offset sum_shape */
typedef struct {
  double  aw2;                       /* mean of W2 over the pairs (NaN without pairs)                                  */
  double  mean_offset, mean_shape;   /* means of o and b over the pairs                                                */
  double  scs;                       /* SCS over W2: population std / mean of the paired neighbours' W2, mean over the
                                        voxels that have any (NaN if none)                                             */
  int64_t n_pairs, n_scs;
  int64_t n_voxels_est, n_voxels_gt; /* occupied voxels of each cloud                                                  */
} me_w2_result;
/* One call on a replicated layout.  rows (nullable): library-allocated n_rows x ME_W2_ROW_COLS, one row per pair, release
 * with me_free.  min_points < 2 or voxel_size <= 0: ME_ERR_INVALID; more than 2^31 voxels: ME_ERR_RANGE. */
ME_API int  me_eval_w2(me_ctx *ctx, double voxel_size, int32_t min_points, int32_t scs_radius, me_w2_result *out,
                       int64_t *n_rows, double **rows);
/* W2 and SCS on GIVEN Gaussians: rows = n_rows x ME_W2_ROW_COLS (vmin, mu and sigma are read; n, offset, shape and w2 are
 * not).  w_out (nullable): n_rows x 3 = offset, shape, w2 per row.  The counterpart of me_awd_from_rows. */
ME_API int  me_w2_from_rows(me_ctx *ctx, const double *rows, int64_t n_rows, double voxel_size, int32_t scs_radius,
                            double *w_out, me_w2_result *out);
/* The stage in halves, for either layout (the pattern of me_voxel_begin): me_w2_begin computes the Gaussians and W2 of the
 * voxels this rank owns; me_w2_w_table hands out the DEVICE W2 table over the estimated cloud's voxels (no pair: NaN, or
 * -1 on an active slab layout, where the caller MAX-all-reduces it in place); me_w2_finish_accum_device runs SCS over this rank's
 * pairs and fills the stage's block; me_w2_block hands it out (*n = ME_W2_BLOCK fp64 values, SUM-reduce them all);
 * me_w2_fetch decodes it.  The stage shares the voxel stage's work buffer: a me_voxel_begin closes an open W2 stage and
 * the other way round. */
ME_API int  me_w2_begin(me_ctx *ctx, double voxel_size, int32_t min_points);
ME_API int  me_w2_w_table(me_ctx *ctx, double **device_w, int64_t *n);
ME_API int  me_w2_finish_accum_device(me_ctx *ctx, int32_t scs_radius);
ME_API int  me_w2_block(me_ctx *ctx, double **device_block, int32_t *n);
ME_API int  me_w2_fetch(me_ctx *ctx, me_w2_result *out);

/* timing of the last call of each stage in milliseconds (CUDA events on the context's stream):
 * [0] grid est [1] grid gt [2] nn est->gt [3] nn gt->est [4] mme est [5] mme gt [6] voxel moments [7] awd [8] scs */
#define ME_N_STAGE_TIMES 9
ME_API int  me_get_stage_times(me_ctx *ctx, double ms[ME_N_STAGE_TIMES]);
/* kernels launched by this context since creation (bench.py's gpu_launches) */
ME_API int64_t me_launch_count(const me_ctx *ctx);

/* Which sweep kernels a context has run: bit (1 << ME_KBIT_x) of the trace mask is set once the path ran.  The kernel
 * choice depends on the lattice, the cell occupancy, the radius-to-cell ratio and the ME_* environment hooks; the trace
 * lets a caller (tests, A/B tools) check which one produced a result.  NN_FAR, NN_FAR_COARSE and NN_BRUTE are set only when
 * at least one query reached that path (recorded on the device); every other bit when its kernel was launched. */
enum me_kernel_bit {
  ME_KBIT_NN_ROWS_DENSE = 0,       /* nn_rows_kernel, dense reference table (default)                      */
  ME_KBIT_NN_ROWS_SPARSE = 1,      /* nn_rows_kernel, sparse reference table                               */
  ME_KBIT_NN_FLAT = 2,             /* nn_flat_kernel, run-table walk (ME_NN_KERNEL=flat)                   */
  ME_KBIT_NN_TILE = 3,             /* nn_tile_kernel (>= 2^24 cells along x, crowded cells, ME_NN_TILE)    */
  ME_KBIT_NN_FAR = 4,              /* nn_far_kernel resolved queries with cell rings                       */
  ME_KBIT_NN_FAR_COARSE = 5,       /* ... and some went on to its coarse-block phase                       */
  ME_KBIT_NN_BRUTE = 6,            /* nn_brute_kernel finished queries that left this rank's slab          */
  ME_KBIT_MME_FLAT1_DENSE = 7,     /* mme_flat_kernel at 1 / 2 / 3 rings, dense table                      */
  ME_KBIT_MME_FLAT2_DENSE = 8,
  ME_KBIT_MME_FLAT3_DENSE = 9,
  ME_KBIT_MME_FLAT1_SPARSE = 10,   /* mme_flat_kernel at 1 / 2 / 3 rings, sparse table                     */
  ME_KBIT_MME_FLAT2_SPARSE = 11,
  ME_KBIT_MME_FLAT3_SPARSE = 12,
  ME_KBIT_MME_ROWS1 = 13,          /* mme_rows_kernel at 1 / 2 / 3 rings (ME_MME_KERNEL=rows)              */
  ME_KBIT_MME_ROWS2 = 14,
  ME_KBIT_MME_ROWS3 = 15,
  ME_KBIT_MME_PLANE = 16,          /* mme_plane_kernel, 4 .. 15 rings                                      */
  ME_KBIT_MME_GENERIC = 17,        /* mme_kernel, the fp64 row walk                                        */
  ME_KBIT_MME_SOLO = 18,           /* the MME sweep laid the cloud out on a lattice of its own (h = r / 2) */
  ME_KBIT_SCS_R5 = 19,             /* scs_kernel with the compiled radius 5                                */
  ME_KBIT_SCS_RT_CACHED = 20,      /* scs_kernel, run-time radius, neighbour values cached per lane        */
  ME_KBIT_SCS_RT_UNCACHED = 21,    /* scs_kernel, run-time radius too large for the per-lane cache         */
  ME_KBIT_COUNT = 22
};
/* Data events of the same mask, above the sweep bits.  They record what the data made a sweep or a lattice build do rather
 * than which sweep ran, so they are not part of enum me_kernel_bit; a sweep's events are set on the device only when a
 * query reaches the path. */
enum me_trace_event {
  ME_TEV_BOX_REMEMBERED = 28,      /* a lattice build planned on the remembered box of its cloud, and the box held     */
  ME_TEV_BOX_MISSED = 29,          /* ... and the box it measured was another: the cloud was laid out again            */
  ME_TEV_KNN_COARSE = 30,          /* a k-NN walk query left the fine rings for the coarse blocks (normals, FPFH)      */
  ME_TEV_MME_FP64_FINISH = 31      /* an fp32-offset MME sweep left queries to mme_fp64_finish_kernel (thin surfaces)  */
};
/* *mask (nullable) = the trace since creation or the last reset; *mme_rows_cfg (nullable) = (CAP << 8) | U of the last
 * mme_rows_kernel<R, CAP, U> launched (ring slots, candidates per iteration), 0 if none.  reset != 0 clears both.
 * Synchronises the context's stream. */
ME_API int me_kernel_trace(me_ctx *ctx, uint64_t *mask, int32_t *mme_rows_cfg, int32_t reset);

#ifdef __cplusplus
}
#endif
#endif /* MAPEVAL_B200_H_ */

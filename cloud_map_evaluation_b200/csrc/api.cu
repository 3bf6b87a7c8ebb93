// api.cu — the C-ABI of libmapeval_b200.so (include/mapeval_b200.h): context lifecycle, cloud upload, host-side
// finalisation of the sum-reducible accumulators.  No CPU fallback exists: every evaluation runs the sm_90a kernels.
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <new>
#include <thread>
#include <vector>

static thread_local std::string g_create_error;

namespace me {

int fail(me_ctx *ctx, int code, const std::string &msg) {
  if (ctx) ctx->err = msg; else g_create_error = msg;
  return code;
}

int ensure(me_ctx *ctx, void **ptr, long long *cap, long long need, size_t elem) {
  if (*ptr && *cap >= need) return ME_OK;
  if (*ptr) { cudaFree(*ptr); *ptr = nullptr; *cap = 0; }
  long long want = std::max<long long>(need, 1);
  cudaError_t e = cudaMalloc(ptr, (size_t)want * elem);
  if (e != cudaSuccess) {
    *ptr = nullptr;
    cudaGetLastError();
    return fail(ctx, ME_ERR_NOMEM, std::string("cudaMalloc of ") + std::to_string((size_t)want * elem) + " bytes: " + cudaGetErrorString(e));
  }
  *cap = want;
  return ME_OK;
}

int ensure_work(me_ctx *ctx, size_t bytes) {
  if (ctx->d_work && ctx->work_bytes >= bytes) return ME_OK;
  if (ctx->d_work) { cudaStreamSynchronize(ctx->stream); cudaFree(ctx->d_work); ctx->d_work = nullptr; ctx->work_bytes = 0; }
  size_t want = std::max<size_t>(bytes, 1 << 20);
  cudaError_t e = cudaMalloc(&ctx->d_work, want);
  if (e != cudaSuccess) {
    ctx->d_work = nullptr;
    cudaGetLastError();
    return fail(ctx, ME_ERR_NOMEM, std::string("cudaMalloc(work) of ") + std::to_string(want) + " bytes: " + cudaGetErrorString(e));
  }
  ctx->work_bytes = want;
  return ME_OK;
}

static void forget_results(Cloud &c) {
  c.grid_valid = false; c.bbox_valid = false; c.nn_valid = false; c.entropy_valid = false; c.entropy_caller_valid = false;
}
// the library moved the points (transform, ICP, drift, degradation, copy): the box of the last build is no guess for them
void invalidate_cloud(Cloud &c) {
  forget_results(c);
  c.last_box_valid = false;
}
// a cloud handed over (me_set_cloud*): its normals go as well; the box of the last build stays the guess of the next one,
// which repeated passes over the same maps hand over every time
static void invalidate(Cloud &c) {
  forget_results(c);
  c.normal_valid = false;
}

static void free_cloud(Cloud &c) {
  if (c.owned && c.d_xyz) cudaFree(c.d_xyz);
  if (c.d_sorted) cudaFree(c.d_sorted);
  if (c.d_rel) cudaFree(c.d_rel);
  if (c.d_cell_off) cudaFree(c.d_cell_off);
  if (c.d_coarse) cudaFree(c.d_coarse);
  if (c.d_hkey) cudaFree(c.d_hkey);
  if (c.d_hval) cudaFree(c.d_hval);
  if (c.d_nn_idx) cudaFree(c.d_nn_idx);
  if (c.d_nn_d2) cudaFree(c.d_nn_d2);
  if (c.d_nn_sq) cudaFree(c.d_nn_sq);
  if (c.d_entropy) cudaFree(c.d_entropy);
  if (c.d_entropy_caller) cudaFree(c.d_entropy_caller);
  if (c.d_fp64_list) cudaFree(c.d_fp64_list);
  if (c.d_normal) cudaFree(c.d_normal);
  if (c.d_tiles) cudaFree(c.d_tiles);
  if (c.d_tile_pos) cudaFree(c.d_tile_pos);
  if (c.upload_done) cudaEventDestroy(c.upload_done);
  c = Cloud();
}

}  // namespace me

using namespace me;

static constexpr size_t kScratchBytes = 8192;   // h_pinned: up to 4 KB of per-stage scratch, then the accumulator block

// ---- upload from PAGEABLE host memory ------------------------------------------------------------------------------
// cudaMemcpyAsync from pageable memory goes through the driver's single staging buffer, which for the 480 MB of the
// 10 M vs 10 M pair takes longer than the whole metric pass.  A std::vector / numpy caller cannot be asked to pin its
// clouds, so the library stages them itself: kStageThreads host threads copy interleaved chunks into pinned bounce
// buffers (two per thread) and push each chunk with its own async H2D copy; the cloud's upload event is recorded once
// all chunks are queued.  Like the driver's path, the call returns when the caller's buffer has been read.
static constexpr int kStageThreads = 8;
static constexpr size_t kStageChunk = 8u << 20;

struct StagePool {
  void *pinned[kStageThreads][2] = {};
  cudaStream_t stream[kStageThreads] = {};
  cudaEvent_t done[kStageThreads][2] = {};
  bool ok = false;
};

static StagePool *stage_pool(me_ctx *ctx) {
  if (ctx->stage) return (StagePool *)ctx->stage;
  StagePool *p = new (std::nothrow) StagePool();
  if (!p) return nullptr;
  bool ok = true;
  for (int t = 0; ok && t < kStageThreads; ++t) {
    ok = cudaStreamCreateWithFlags(&p->stream[t], cudaStreamNonBlocking) == cudaSuccess;
    for (int b = 0; ok && b < 2; ++b)
      ok = cudaMallocHost(&p->pinned[t][b], kStageChunk) == cudaSuccess &&
           cudaEventCreateWithFlags(&p->done[t][b], cudaEventDisableTiming) == cudaSuccess;
  }
  p->ok = ok;
  ctx->stage = p;
  if (!ok) cudaGetLastError();
  return p;
}

static void stage_pool_free(me_ctx *ctx) {
  StagePool *p = (StagePool *)ctx->stage;
  if (!p) return;
  for (int t = 0; t < kStageThreads; ++t) {
    if (p->stream[t]) { cudaStreamSynchronize(p->stream[t]); cudaStreamDestroy(p->stream[t]); }
    for (int b = 0; b < 2; ++b) {
      if (p->pinned[t][b]) cudaFreeHost(p->pinned[t][b]);
      if (p->done[t][b]) cudaEventDestroy(p->done[t][b]);
    }
  }
  delete p;
  ctx->stage = nullptr;
}

// true if the staged upload ran (the copy stream then waits for every chunk); false = use the plain cudaMemcpyAsync
static bool staged_upload(me_ctx *ctx, void *dst, const void *src, size_t bytes) {
  if (bytes < 4 * kStageChunk || getenv("ME_NO_STAGED_UPLOAD")) return false;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, src) != cudaSuccess) { cudaGetLastError(); return false; }
  if (at.type != cudaMemoryTypeUnregistered) return false;      // pinned / managed / device memory: the direct copy is async
  StagePool *p = stage_pool(ctx);
  if (!p || !p->ok) return false;
  const size_t nchunks = (bytes + kStageChunk - 1) / kStageChunk;
  const int dev = ctx->device;
  std::vector<int> rc(kStageThreads, 0);
  std::vector<std::thread> th;
  for (int t = 0; t < kStageThreads; ++t)
    th.emplace_back([=, &rc] {
      if (cudaSetDevice(dev) != cudaSuccess) { rc[t] = 1; return; }
      int use = 0;
      for (size_t c = (size_t)t; c < nchunks; c += kStageThreads, ++use) {
        const int b = use & 1;
        const size_t off = c * kStageChunk, len = std::min(kStageChunk, bytes - off);
        // the bounce buffer is free once the copy that last used it has run (also one queued by an earlier call; an event
        // never recorded counts as complete)
        if (cudaEventSynchronize(p->done[t][b]) != cudaSuccess) { rc[t] = 1; return; }
        std::memcpy(p->pinned[t][b], (const char *)src + off, len);
        if (cudaMemcpyAsync((char *)dst + off, p->pinned[t][b], len, cudaMemcpyHostToDevice, p->stream[t]) != cudaSuccess ||
            cudaEventRecord(p->done[t][b], p->stream[t]) != cudaSuccess) { rc[t] = 1; return; }
      }
    });
  for (auto &x : th) x.join();
  for (int t = 0; t < kStageThreads; ++t) if (rc[t]) { cudaGetLastError(); return false; }
  // the copy stream (whose event the consumers wait on) waits for the last chunk of every staging stream
  for (int t = 0; t < kStageThreads; ++t)
    for (int b = 0; b < 2; ++b)
      if (cudaStreamWaitEvent(ctx->copy_stream, p->done[t][b], 0) != cudaSuccess) { cudaGetLastError(); return false; }
  return true;
}

#define ME_ENTER(ctx)                                                                    \
  if (!(ctx)) return ME_ERR_INVALID;                                                     \
  do {                                                                                   \
    cudaError_t e__ = cudaSetDevice((ctx)->device);                                      \
    if (e__ != cudaSuccess) return me::fail((ctx), ME_ERR_CUDA, cudaGetErrorString(e__)); \
  } while (0)

extern "C" {

int me_abi_version(void) { return ME_ABI_VERSION; }

int me_create(const me_options *opt, me_ctx **out) {
  if (!out) return ME_ERR_INVALID;
  *out = nullptr;
  if (!opt || opt->abi_version != ME_ABI_VERSION) return fail(nullptr, ME_ERR_INVALID, "me_options.abi_version mismatch");
  if (opt->world < 1 || opt->rank < 0 || opt->rank >= opt->world) return fail(nullptr, ME_ERR_INVALID, "bad rank/world");
  if (opt->world > ME_MAX_WORLD)
    return fail(nullptr, ME_ERR_INVALID, "world " + std::to_string(opt->world) + " > ME_MAX_WORLD = " + std::to_string(ME_MAX_WORLD));
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev <= 0) {
    cudaGetLastError();
    return fail(nullptr, ME_ERR_NO_DEVICE, std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0") +
                                               " (libmapeval_b200 has no CPU path)");
  }
  if (opt->device < 0 || opt->device >= ndev) return fail(nullptr, ME_ERR_NO_DEVICE, "device ordinal out of range");
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, opt->device) != cudaSuccess) return fail(nullptr, ME_ERR_CUDA, "cudaGetDeviceProperties failed");
  if (prop.major != 9 || prop.minor != 0)      // sm_90a code runs on compute capability 9.0 only
    return fail(nullptr, ME_ERR_NO_DEVICE, std::string("device '") + prop.name + "' is sm_" + std::to_string(prop.major) +
                                               std::to_string(prop.minor) + "; this library carries sm_90a code only");
  if (cudaSetDevice(opt->device) != cudaSuccess) return fail(nullptr, ME_ERR_CUDA, "cudaSetDevice failed");
  me_ctx *ctx = new (std::nothrow) me_ctx();
  if (!ctx) return fail(nullptr, ME_ERR_NOMEM, "out of host memory");
  ctx->device = opt->device;
  ctx->rank = opt->rank; ctx->world = opt->world;
  ctx->sm_count = prop.multiProcessorCount;
  ctx->nn_cell_size = opt->nn_cell_size > 0 ? opt->nn_cell_size : 0.0;
  ctx->max_grid_cells = opt->max_grid_cells > 0 ? std::min<long long>(opt->max_grid_cells, 0xfffffff0ll) : 0;   // 0 = automatic
  ctx->voxel_hint = opt->vmd_voxel_size > 0 ? opt->vmd_voxel_size : 0.0;
  if (opt->stream) { ctx->stream = (cudaStream_t)opt->stream; ctx->own_stream = false; }
  else {
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return fail(nullptr, ME_ERR_CUDA, "cudaStreamCreate failed"); }
    ctx->own_stream = true;
  }
  bool ok = cudaMalloc(&ctx->d_scratch, kScratchBytes) == cudaSuccess && cudaMallocHost(&ctx->h_pinned, kScratchBytes) == cudaSuccess;
  ok = ok && cudaMalloc((void **)&ctx->d_block, kBlkTotal * sizeof(double)) == cudaSuccess;
  ok = ok && cudaMalloc((void **)&ctx->d_trace, sizeof(unsigned int)) == cudaSuccess &&
       cudaMemsetAsync(ctx->d_trace, 0, sizeof(unsigned int), ctx->stream) == cudaSuccess;
  ok = ok && cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&ctx->compute_mark, cudaEventDisableTiming) == cudaSuccess;
  for (int w = 0; ok && w < 2; ++w) ok = cudaEventCreateWithFlags(&ctx->cloud[w].upload_done, cudaEventDisableTiming) == cudaSuccess;
  for (int i = 0; ok && i < 2 * ME_N_STAGE_TIMES; ++i) ok = cudaEventCreate(&ctx->ev[i]) == cudaSuccess;
  for (int i = 0; i < ME_N_STAGE_TIMES; ++i) ctx->ev_used[i] = false;
  if (!ok) { me_destroy(ctx); return fail(nullptr, ME_ERR_NOMEM, "context allocation failed"); }
  ctx->scratch_bytes = kScratchBytes;
  *out = ctx;
  return ME_OK;
}

void me_destroy(me_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  icp_close(ctx, false);
  nn_quantile_free(ctx);
  nn_region_free(ctx);
  nn_surface_free(ctx);
  consistency_free(ctx);
  mom_free(ctx);
  mom_region_free(ctx);
  drift_close(ctx, false);
  if (ctx->copy_stream) { cudaStreamSynchronize(ctx->copy_stream); cudaStreamDestroy(ctx->copy_stream); }
  if (ctx->compute_mark) cudaEventDestroy(ctx->compute_mark);
  for (Cloud &c : ctx->cloud) free_cloud(c);
  for (float *f : ctx->d_fpfh) if (f) cudaFree(f);
  if (ctx->d_corr) cudaFree(ctx->d_corr);
  stage_pool_free(ctx);
  if (ctx->d_scratch) cudaFree(ctx->d_scratch);
  if (ctx->d_block) cudaFree(ctx->d_block);
  if (ctx->d_w2) cudaFree(ctx->d_w2);
  if (ctx->d_trace) cudaFree(ctx->d_trace);
  if (ctx->h_pinned) cudaFreeHost(ctx->h_pinned);
  if (ctx->d_work) cudaFree(ctx->d_work);
  if (ctx->d_scan_tmp) cudaFree(ctx->d_scan_tmp);
  if (ctx->d_rank) cudaFree(ctx->d_rank);
  if (ctx->d_rs_hist) cudaFree(ctx->d_rs_hist);
  for (int i = 0; i < 2 * ME_N_STAGE_TIMES; ++i) if (ctx->ev[i]) cudaEventDestroy(ctx->ev[i]);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

const char *me_last_error(const me_ctx *ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int me_set_stream(me_ctx *ctx, void *cuda_stream) {
  ME_ENTER(ctx);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->own_stream) { cudaStreamDestroy(ctx->stream); ctx->own_stream = false; }
  if (cuda_stream) ctx->stream = (cudaStream_t)cuda_stream;
  else {
    ME_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    ctx->own_stream = true;
  }
  return ME_OK;
}

int me_set_shard(me_ctx *ctx, int32_t rank, int32_t world) {
  ME_ENTER(ctx);
  if (world < 1 || rank < 0 || rank >= world) return fail(ctx, ME_ERR_INVALID, "bad rank/world");
  if (world > ME_MAX_WORLD)
    return fail(ctx, ME_ERR_INVALID, "world " + std::to_string(world) + " > ME_MAX_WORLD = " + std::to_string(ME_MAX_WORLD));
  ctx->rank = rank; ctx->world = world;
  ctx->slab_planned = false; ctx->slab_on = false; ctx->vox_open = false;
  ctx->cloud[0].grid_valid = ctx->cloud[1].grid_valid = false;      // slab lattices belong to one (rank, world)
  ctx->cloud[0].nn_valid = ctx->cloud[1].nn_valid = false;
  ctx->cloud[0].entropy_valid = ctx->cloud[1].entropy_valid = false;
  ctx->cloud[0].entropy_caller_valid = ctx->cloud[1].entropy_caller_valid = false;
  ctx->cloud[0].shard_valid = ctx->cloud[1].shard_valid = false;
  return ME_OK;
}

int me_set_layout(me_ctx *ctx, int32_t layout) {
  ME_ENTER(ctx);
  if (layout != ME_LAYOUT_REPLICATED && layout != ME_LAYOUT_SLAB) return fail(ctx, ME_ERR_INVALID, "bad layout");
  const bool want = layout == ME_LAYOUT_SLAB;
  if (want == ctx->slab_request) return ME_OK;
  ctx->slab_request = want;
  ctx->slab_planned = false; ctx->slab_on = false; ctx->vox_open = false;
  for (int w = 0; w < 2; ++w) {      // the lattices are laid out again under the new layout
    ctx->cloud[w].grid_valid = false; ctx->cloud[w].nn_valid = false; ctx->cloud[w].entropy_valid = false;
    ctx->cloud[w].shard_valid = false;
  }
  return ME_OK;
}

int me_plan_lattice(const double bbox_min[3], const double bbox_max[3], int64_t n, const double *other_bbox_min,
                    const double *other_bbox_max, int64_t other_n, double voxel_size, double cell_edge_target,
                    int64_t max_grid_cells, int32_t allow_sparse, me_lattice_plan *out) {
  if (!bbox_min || !bbox_max || !out || n < 1) return ME_ERR_INVALID;
  for (int a = 0; a < 3; ++a)
    if (!(bbox_min[a] <= bbox_max[a])) return ME_ERR_INVALID;
  me::Lattice L;
  if (!me::plan_lattice_host(bbox_min, bbox_max, n, other_bbox_min, other_bbox_max, other_n, voxel_size, cell_edge_target,
                             max_grid_cells, allow_sparse != 0, &L))
    return ME_ERR_RANGE;
  out->v = L.v; out->h = L.h; out->m = L.m; out->sparse = L.sparse;
  for (int a = 0; a < 3; ++a) { out->nvox[a] = L.nvox[a]; out->dims[a] = L.dims[a]; }
  out->ncells = L.sparse ? 0 : L.ncells;
  return ME_OK;
}

int me_plan_slab_cut(const uint64_t *plane_counts_y, int32_t n_planes_y, const uint64_t *plane_counts_z, int32_t n_planes_z,
                     int32_t cells_per_voxel, int32_t world, int32_t halo_cells, int32_t *axis, int32_t *layer_bounds,
                     double *busiest_share) {
  if (!plane_counts_y || !plane_counts_z || !axis || !layer_bounds || !busiest_share) return ME_ERR_INVALID;
  if (n_planes_y < 0 || n_planes_z < 0 || cells_per_voxel < 1 || world < 1 || halo_cells < 0) return ME_ERR_INVALID;
  static_assert(sizeof(uint64_t) == sizeof(unsigned long long), "plane counts are 64-bit");
  int ax = 0;
  double share = 2.0;
  std::vector<int> b((size_t)world + 1, 0);
  me::slab_cut((const unsigned long long *)plane_counts_y, n_planes_y, (const unsigned long long *)plane_counts_z, n_planes_z,
               cells_per_voxel, world, halo_cells, &ax, b.data(), &share);
  if (ax && share > me::kSlabMaxShare) ax = 0;
  *axis = ax;
  *busiest_share = share;
  for (int r = 0; r <= world; ++r) layer_bounds[r] = ax ? b[r] : 0;
  return ME_OK;
}

int me_layout_active(me_ctx *ctx, int32_t *layout, int32_t *axis, int64_t n_laid_out[2], int64_t n_owned[2]) {
  ME_ENTER(ctx);
  const bool slab = (ctx->cloud[0].grid_valid && ctx->cloud[0].slab) || (ctx->cloud[1].grid_valid && ctx->cloud[1].slab);
  if (layout) *layout = slab ? ME_LAYOUT_SLAB : ME_LAYOUT_REPLICATED;
  if (axis) *axis = slab ? ctx->slab_axis : 0;
  for (int w = 0; w < 2; ++w) {
    const Cloud &c = ctx->cloud[w];
    if (n_laid_out) n_laid_out[w] = c.grid_valid ? c.ns : 0;
    if (n_owned) n_owned[w] = c.grid_valid ? c.n_owned : 0;
  }
  return ME_OK;
}

int me_synchronize(me_ctx *ctx) {
  ME_ENTER(ctx);
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return ME_OK;
}

int me_set_cloud(me_ctx *ctx, int which, const double *xyz_host, int64_t n) {
  ME_ENTER(ctx);
  ctx->cloud_gen++;      // stales the NN records (me_nn_curve*)
  if (which != ME_CLOUD_EST && which != ME_CLOUD_GT) return fail(ctx, ME_ERR_INVALID, "which must be ME_CLOUD_EST or ME_CLOUD_GT");
  if (n < 0 || (n > 0 && !xyz_host)) return fail(ctx, ME_ERR_INVALID, "bad cloud pointer/size");
  if (n >= 0x7fffffffll) return fail(ctx, ME_ERR_RANGE, "more than 2^31-1 points per cloud (the reference indexes with int)");
  Cloud &c = ctx->cloud[which];
  if (!c.owned) { c.d_xyz = nullptr; c.cap_xyz = 0; }
  ME_TRY(ensure(ctx, (void **)&c.d_xyz, &c.cap_xyz, 3 * n, sizeof(double)));
  c.owned = true;
  c.n = n;
  invalidate(c);
  if (n > 0) {
    // the copy runs on its own stream: it may overlap kernels that work on the other cloud, but must not overtake
    // kernels already queued that still read this buffer
    ME_CUDA(ctx, cudaEventRecord(ctx->compute_mark, ctx->stream));
    ME_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->compute_mark, 0));
    // the staging streams must not overtake kernels that still read this buffer either
    bool staged = false;
    {
      StagePool *sp = (StagePool *)ctx->stage;
      if (sp && sp->ok)
        for (int t = 0; t < kStageThreads; ++t) cudaStreamWaitEvent(sp->stream[t], ctx->compute_mark, 0);
      staged = staged_upload(ctx, c.d_xyz, xyz_host, (size_t)n * 3 * sizeof(double));
    }
    if (!staged)
      ME_CUDA(ctx, cudaMemcpyAsync(c.d_xyz, xyz_host, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, ctx->copy_stream));
    ME_CUDA(ctx, cudaEventRecord(c.upload_done, ctx->copy_stream));
    c.upload_pending = true;
  }
  return ME_OK;
}

int me_set_cloud_device(me_ctx *ctx, int which, const double *xyz_device, int64_t n) {
  ME_ENTER(ctx);
  ctx->cloud_gen++;      // stales the NN records (me_nn_curve*)
  if (which != ME_CLOUD_EST && which != ME_CLOUD_GT) return fail(ctx, ME_ERR_INVALID, "which must be ME_CLOUD_EST or ME_CLOUD_GT");
  if (n < 0 || (n > 0 && !xyz_device)) return fail(ctx, ME_ERR_INVALID, "bad cloud pointer/size");
  if (n >= 0x7fffffffll) return fail(ctx, ME_ERR_RANGE, "more than 2^31-1 points per cloud");
  Cloud &c = ctx->cloud[which];
  if (c.owned && c.d_xyz) { cudaStreamSynchronize(ctx->stream); cudaFree(c.d_xyz); }
  c.d_xyz = const_cast<double *>(xyz_device);
  c.cap_xyz = 0;
  c.owned = false;
  c.upload_pending = false;
  c.n = n;
  invalidate(c);
  return ME_OK;
}

int me_transform(me_ctx *ctx, int which, const double T[16]) {
  ME_ENTER(ctx);
  ctx->cloud_gen++;      // stales the NN records (me_nn_curve*)
  if ((which != ME_CLOUD_EST && which != ME_CLOUD_GT) || !T) return fail(ctx, ME_ERR_INVALID, "bad arguments");
  return transform_cloud(ctx, which, T);
}

int me_voxel_downsample(me_ctx *ctx, int which, double voxel_size, int64_t *n_out) {
  ME_ENTER(ctx);
  ctx->cloud_gen++;      // stales the NN records (me_nn_curve*)
  if (which != ME_CLOUD_EST && which != ME_CLOUD_GT) return fail(ctx, ME_ERR_INVALID, "bad cloud id");
  return voxel_downsample(ctx, which, voxel_size, n_out);
}

static bool cloud_id(int which) { return which == ME_CLOUD_EST || which == ME_CLOUD_GT; }

int me_copy_cloud(me_ctx *ctx, int src, int dst) {
  ME_ENTER(ctx);
  ctx->cloud_gen++;      // stales the NN records (me_nn_curve*)
  if (!cloud_id(src) || !cloud_id(dst) || src == dst) return fail(ctx, ME_ERR_INVALID, "me_copy_cloud: src and dst must be the two clouds");
  return copy_cloud(ctx, src, dst);
}

int me_add_gaussian_noise(me_ctx *ctx, int which, double std_dev, uint64_t seed) {
  ME_ENTER(ctx);
  ctx->cloud_gen++;      // stales the NN records (me_nn_curve*)
  if (!cloud_id(which)) return fail(ctx, ME_ERR_INVALID, "bad cloud id");
  if (!(std::isfinite(std_dev) && std_dev >= 0.0)) return fail(ctx, ME_ERR_INVALID, "me_add_gaussian_noise: std_dev must be finite and >= 0");
  return add_gaussian_noise(ctx, which, std_dev, seed);
}

int me_add_non_uniform_density(me_ctx *ctx, int which, double sparse_ratio, double dense_ratio, double region_size, uint64_t seed,
                               int64_t *n_out) {
  ME_ENTER(ctx);
  ctx->cloud_gen++;      // stales the NN records (me_nn_curve*)
  if (!cloud_id(which)) return fail(ctx, ME_ERR_INVALID, "bad cloud id");
  return add_non_uniform_density(ctx, which, sparse_ratio, dense_ratio, region_size, seed, n_out);
}

int me_add_sparse_outliers(me_ctx *ctx, int which, double outlier_ratio, double outlier_range, uint64_t seed, int64_t *n_out) {
  ME_ENTER(ctx);
  ctx->cloud_gen++;      // stales the NN records (me_nn_curve*)
  if (!cloud_id(which)) return fail(ctx, ME_ERR_INVALID, "bad cloud id");
  if (!(std::isfinite(outlier_range) && outlier_range >= 0.0))
    return fail(ctx, ME_ERR_INVALID, "me_add_sparse_outliers: outlier_range must be finite and >= 0");
  return add_sparse_outliers(ctx, which, outlier_ratio, outlier_range, seed, n_out);
}

int me_add_local_deformation(me_ctx *ctx, int which, double radius, double strength, const double center[3]) {
  ME_ENTER(ctx);
  ctx->cloud_gen++;      // stales the NN records (me_nn_curve*)
  if (!cloud_id(which) || !center) return fail(ctx, ME_ERR_INVALID, "bad arguments");
  return add_local_deformation(ctx, which, radius, strength, center);
}

int me_get_cloud(me_ctx *ctx, int which, double *xyz_host, int64_t capacity_points, int64_t *n) {
  ME_ENTER(ctx);
  if (which != ME_CLOUD_EST && which != ME_CLOUD_GT) return fail(ctx, ME_ERR_INVALID, "bad cloud id");
  Cloud &c = ctx->cloud[which];
  if (n) *n = c.n;
  if (!xyz_host) return ME_OK;                       // size query
  if (capacity_points < c.n) return fail(ctx, ME_ERR_INVALID, "me_get_cloud: host buffer too small");
  ME_TRY(wait_upload(ctx, which));
  if (c.n > 0) {
    ME_CUDA(ctx, cudaMemcpyAsync(xyz_host, c.d_xyz, (size_t)c.n * 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return ME_OK;
}

// a registration cannot start while a drift loop moves the estimated cloud; refused before the call stales anything, so the
// drift loop stays open
static bool drift_blocks_icp(me_ctx *ctx) {
  if (!ctx->drift.open) return false;
  fail(ctx, ME_ERR_INVALID, "me_icp_begin while a drift loop is open (me_drift_end first)");
  return true;
}

int me_icp_point_to_point(me_ctx *ctx, double max_correspondence_distance, int32_t max_iteration, double relative_fitness,
                          double relative_rmse, const double T_init[16], me_icp_result *out) {
  ME_ENTER(ctx);
  if (drift_blocks_icp(ctx)) return ME_ERR_INVALID;
  ctx->cloud_gen++;      // stales the NN records (me_nn_curve*)
  if (!T_init || !out) return fail(ctx, ME_ERR_INVALID, "null argument");
  return run_icp(ctx, ME_ICP_POINT_TO_POINT, max_correspondence_distance, max_iteration, relative_fitness, relative_rmse, T_init, out);
}

int me_icp(me_ctx *ctx, int32_t method, double max_correspondence_distance, int32_t max_iteration, double relative_fitness,
           double relative_rmse, const double T_init[16], me_icp_result *out) {
  ME_ENTER(ctx);
  if (drift_blocks_icp(ctx)) return ME_ERR_INVALID;
  ctx->cloud_gen++;      // stales the NN records (me_nn_curve*)
  if (!T_init || !out) return fail(ctx, ME_ERR_INVALID, "null argument");
  return run_icp(ctx, method, max_correspondence_distance, max_iteration, relative_fitness, relative_rmse, T_init, out);
}

int me_icp_begin(me_ctx *ctx, int32_t method, double max_correspondence_distance, int32_t max_iteration, double relative_fitness,
                 double relative_rmse, const double T_init[16]) {
  ME_ENTER(ctx);
  if (drift_blocks_icp(ctx)) return ME_ERR_INVALID;
  ctx->cloud_gen++;      // stales the NN records (me_nn_curve*)
  if (!T_init) return fail(ctx, ME_ERR_INVALID, "null argument");
  return icp_begin(ctx, method, max_correspondence_distance, max_iteration, relative_fitness, relative_rmse, T_init);
}

int me_icp_normals_slice(me_ctx *ctx, int which, double **device_normals, int64_t *slice_points, int32_t *pending) {
  ME_ENTER(ctx);
  if (which != ME_CLOUD_EST && which != ME_CLOUD_GT) return fail(ctx, ME_ERR_INVALID, "bad cloud id");
  if (!device_normals || !slice_points || !pending) return fail(ctx, ME_ERR_INVALID, "null argument");
  return icp_normals_slice(ctx, which, device_normals, slice_points, pending);
}

int me_icp_block(me_ctx *ctx, double **device_block, int32_t *n_sum) {
  ME_ENTER(ctx);
  if (!device_block || !n_sum) return fail(ctx, ME_ERR_INVALID, "null argument");
  return icp_block(ctx, device_block, n_sum);
}

int me_icp_step(me_ctx *ctx, int32_t *done) {
  ME_ENTER(ctx);
  if (!done) return fail(ctx, ME_ERR_INVALID, "null argument");
  return icp_step(ctx, done);
}

int me_icp_end(me_ctx *ctx, me_icp_result *out) {
  ME_ENTER(ctx);
  if (!out) return fail(ctx, ME_ERR_INVALID, "null argument");
  return icp_end(ctx, out);
}

int me_icp_update(int32_t method, const double *block, const double center[3], double update[16]) {
  if (!block || !update) return ME_ERR_INVALID;
  if (method != ME_ICP_POINT_TO_POINT && method != ME_ICP_POINT_TO_PLANE && method != ME_ICP_GENERALIZED) return ME_ERR_INVALID;
  if (method == ME_ICP_POINT_TO_POINT && !center) return ME_ERR_INVALID;
  icp_update_host(method, block, center, update);
  return ME_OK;
}

int me_global_registration(me_ctx *ctx, const me_global_reg_params *p, me_global_reg_result *out) {
  ME_ENTER(ctx);
  if (!p || !out) return fail(ctx, ME_ERR_INVALID, "null argument");
  return global_registration(ctx, p, out);
}

int me_get_features(me_ctx *ctx, int which, double *xyz, double *normals, float *fpfh33, int64_t capacity, int64_t *n) {
  ME_ENTER(ctx);
  if (!cloud_id(which)) return fail(ctx, ME_ERR_INVALID, "bad cloud id");
  return get_features(ctx, which, xyz, normals, fpfh33, capacity, n);
}

int me_get_correspondences(me_ctx *ctx, int32_t *est_idx, int32_t *gt_idx, int64_t capacity, int64_t *n) {
  ME_ENTER(ctx);
  return get_correspondences(ctx, est_idx, gt_idx, capacity, n);
}

int me_set_normals(me_ctx *ctx, int which, const double *normals_host, int64_t n) {
  ME_ENTER(ctx);
  if (which != ME_CLOUD_EST && which != ME_CLOUD_GT) return fail(ctx, ME_ERR_INVALID, "bad cloud id");
  Cloud &c = ctx->cloud[which];
  if (!normals_host || n != c.n || n <= 0) return fail(ctx, ME_ERR_INVALID, "me_set_normals: one normal per point of the cloud held by the context");
  ME_TRY(ensure(ctx, (void **)&c.d_normal, &c.cap_normal, 3 * c.n, sizeof(double)));
  ME_CUDA(ctx, cudaMemcpyAsync(c.d_normal, normals_host, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  c.normal_valid = true;
  return ME_OK;
}

int me_estimate_normals(me_ctx *ctx, int which, int32_t knn) {
  ME_ENTER(ctx);
  if (which != ME_CLOUD_EST && which != ME_CLOUD_GT) return fail(ctx, ME_ERR_INVALID, "bad cloud id");
  return estimate_normals(ctx, which, knn);
}

int me_get_normals(me_ctx *ctx, int which, double *normals_host) {
  ME_ENTER(ctx);
  if ((which != ME_CLOUD_EST && which != ME_CLOUD_GT) || !normals_host) return fail(ctx, ME_ERR_INVALID, "bad arguments");
  Cloud &c = ctx->cloud[which];
  if (!c.normal_valid) return fail(ctx, ME_ERR_INVALID, "me_get_normals: the cloud has no normals");
  ME_CUDA(ctx, cudaMemcpyAsync(normals_host, c.d_normal, (size_t)c.n * 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return ME_OK;
}

int me_build_grid(me_ctx *ctx, int which) {
  ME_ENTER(ctx);
  if (which != ME_CLOUD_EST && which != ME_CLOUD_GT) return fail(ctx, ME_ERR_INVALID, "bad cloud id");
  ctx->cloud[which].grid_valid = false;
  return build_grid(ctx, which);
}

}  // extern "C"

// ---- accumulators: sweep -> d_block -> (all-reduce on the device by the caller) -> one fetch per pass ------------------------
// The block is the only encoding of the accumulators: me_eval_*_accum decode their sections right after the sweep.

// the arguments of me_eval_nn_accum* that the sweep reads
static int check_nn_params(me_ctx *ctx, const me_nn_params *p) {
  if (!p) return fail(ctx, ME_ERR_INVALID, "null params");
  if (p->cutoff_mode != ME_CUTOFF_SQDIST_LE_R && p->cutoff_mode != ME_CUTOFF_DIST_LT_R) return fail(ctx, ME_ERR_INVALID, "bad cutoff_mode");
  if (p->pairing != ME_PAIRING_AS_WRITTEN && p->pairing != ME_PAIRING_GEOMETRIC) return fail(ctx, ME_ERR_INVALID, "bad pairing");
  return ME_OK;
}

// the NN sweeps of the requested directions into their sections of the block; on success the records serve me_nn_curve* and
// me_nn_quantile* until the clouds change
static int eval_nn_block(me_ctx *ctx, const me_nn_params *p) {
  ctx->curve_valid = false;
  ME_TRY(run_nn(ctx, p, true));
  ctx->curve_valid = true;
  ctx->curve_gen = ctx->cloud_gen;
  ctx->curve_p = *p;
  return ME_OK;
}

// the block, copied to the pinned host scratch once the stream has finished with it
static int fetch_block(me_ctx *ctx, const double **h_out) {
  static_assert(4096 + kBlkTotal * sizeof(double) <= kScratchBytes, "the accumulator block fits the pinned scratch");
  double *h = (double *)((char *)ctx->h_pinned + 4096);
  ME_CUDA(ctx, cudaMemcpyAsync(h, ctx->d_block, kBlkTotal * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  *h_out = h;
  return ME_OK;
}

// the block's NN and MME sections (host copy) -> the accumulator structs; a NULL struct is skipped.  Counts come back
// through fp64 exactly (below 2^53), the entropy minimum through an exact negation.
static void decode_block(const double *h, me_nn_accum *est_to_gt, me_nn_accum *gt_to_est, me_mme_accum *mme_est, me_mme_accum *mme_gt) {
  auto i64 = [](double v) { return (int64_t)std::llround(v); };
  me_nn_accum *dirs[2] = {est_to_gt, gt_to_est};
  for (int d = 0; d < 2; ++d) {
    me_nn_accum *a = dirs[d];
    if (!a) continue;
    const double *b = h + d * kBlkNN;
    a->n_query = i64(b[0]); a->n_corr = i64(b[1]);
    for (int k = 0; k < 5; ++k) a->n_inlier[k] = i64(b[2 + k]);
    a->n_ub = i64(b[7]); a->n_far = i64(b[8]);
    for (int k = 0; k < 5; ++k) { a->sum_d[k] = b[9 + k]; a->sum_d2[k] = b[14 + k]; }
    a->sum_d_all = b[19]; a->sum_d2_all = b[20]; a->sum_nn_dist = b[21];
    for (int r = 0; r < ME_MAX_WORLD; ++r) {
      a->rank_n[r] = b[kBlkMoments + r]; a->rank_mean[r] = b[kBlkMoments + ME_MAX_WORLD + r];
      a->rank_m2[r] = b[kBlkMoments + 2 * ME_MAX_WORLD + r];
    }
  }
  me_mme_accum *mm[2] = {mme_est, mme_gt};
  for (int w = 0; w < 2; ++w) {
    me_mme_accum *m = mm[w];
    if (!m) continue;
    const double *b = h + kBlkMmeSum + 3 * w, *x = h + kBlkMax + 2 * w;
    m->n_query = i64(b[0]); m->n_valid = i64(b[1]); m->sum_entropy = b[2];
    m->max_entropy = x[0]; m->min_entropy = -x[1];
  }
}

// the tail of a one-shot call that hands the caller library-allocated rows (me_free): max(n, min_rows) rows (NULL when that
// is 0), filled by end(rows) and freed when it fails.  close() leaves the context as a failed call must when the allocation
// fails.
template <class Row, class End, class Close>
static int one_shot_rows(me_ctx *ctx, int64_t n, int64_t min_rows, const char *nomem, End end, Close close, Row **rows,
                         int64_t *n_regions) {
  Row *r = nullptr;
  const int64_t cap = std::max(n, min_rows);
  if (cap > 0 && !(r = (Row *)std::malloc((size_t)cap * sizeof(Row)))) {
    close();
    return fail(ctx, ME_ERR_NOMEM, nomem);
  }
  const int rc = end(r);
  if (rc != ME_OK) {
    std::free(r);
    return rc;
  }
  *rows = r;
  *n_regions = n;
  return ME_OK;
}

extern "C" {

__global__ void block_init_kernel(double *blk) {
  for (int t = threadIdx.x; t < me::kBlkTotal; t += blockDim.x) blk[t] = t < me::kBlkSumCount ? 0.0 : -INFINITY;
}

int me_eval_nn_accum(me_ctx *ctx, const me_nn_params *p, me_nn_accum *est_to_gt, me_nn_accum *gt_to_est) {
  ME_ENTER(ctx);
  ME_TRY(check_nn_params(ctx, p));
  const int dirs = p->directions ? p->directions : 3;
  if (((dirs & 1) && !est_to_gt) || ((dirs & 2) && !gt_to_est)) return fail(ctx, ME_ERR_INVALID, "null accumulator for a requested direction");
  if (est_to_gt) std::memset(est_to_gt, 0, sizeof(*est_to_gt));      // a direction not requested stays zero
  if (gt_to_est) std::memset(gt_to_est, 0, sizeof(*gt_to_est));
  ME_TRY(eval_nn_block(ctx, p));
  const double *h = nullptr;
  ME_TRY(fetch_block(ctx, &h));
  decode_block(h, (dirs & 1) ? est_to_gt : nullptr, (dirs & 2) ? gt_to_est : nullptr, nullptr, nullptr);
  return ME_OK;
}

int me_accum_reset(me_ctx *ctx) {
  ME_ENTER(ctx);
  block_init_kernel<<<1, 256, 0, ctx->stream>>>(ctx->d_block);
  ME_LAUNCH_CHECK(ctx);
  return ME_OK;
}

int me_eval_nn_accum_device(me_ctx *ctx, const me_nn_params *p) {
  ME_ENTER(ctx);
  ME_TRY(check_nn_params(ctx, p));
  return eval_nn_block(ctx, p);
}

int me_eval_mme_accum_device(me_ctx *ctx, int which, double radius, int32_t min_neighbors) {
  ME_ENTER(ctx);
  if (which != ME_CLOUD_EST && which != ME_CLOUD_GT) return fail(ctx, ME_ERR_INVALID, "bad arguments");
  return run_mme(ctx, which, radius, min_neighbors);
}

int me_accum_block(me_ctx *ctx, double **device_block, int32_t *n_sum, int32_t *n_max) {
  ME_ENTER(ctx);
  if (device_block) *device_block = ctx->d_block;
  if (n_sum) *n_sum = kBlkSumCount;
  if (n_max) *n_max = kBlkMaxCount;
  return ME_OK;
}

int me_voxel_begin(me_ctx *ctx, double voxel_size, int32_t min_points) {
  ME_ENTER(ctx);
  return voxel_begin(ctx, voxel_size, min_points);
}

int me_voxel_w_table(me_ctx *ctx, double **device_w, int64_t *n) {
  ME_ENTER(ctx);
  if (!device_w || !n) return fail(ctx, ME_ERR_INVALID, "null argument");
  return voxel_w_table(ctx, device_w, n);
}

int me_voxel_finish_accum_device(me_ctx *ctx, int32_t scs_radius) {
  ME_ENTER(ctx);
  return voxel_finish_block(ctx, scs_radius);
}

int me_accum_fetch_awd(me_ctx *ctx, me_awd_result *out) {
  ME_ENTER(ctx);
  if (!out) return fail(ctx, ME_ERR_INVALID, "null result");
  const double *h = nullptr;
  ME_TRY(fetch_block(ctx, &h));
  awd_result(h + kBlkAwd, out);
  return ME_OK;
}

int me_accum_fetch(me_ctx *ctx, me_nn_accum *est_to_gt, me_nn_accum *gt_to_est, me_mme_accum *mme_est, me_mme_accum *mme_gt) {
  ME_ENTER(ctx);
  const double *h = nullptr;
  ME_TRY(fetch_block(ctx, &h));
  decode_block(h, est_to_gt, gt_to_est, mme_est, mme_gt);
  return ME_OK;
}

// the per-level arithmetic of me_nn_finalize, shared with me_nn_curve_finalize so that a level both compute is one expression
struct DirMoments {           // one direction's accumulator, reduced over the ranks
  const me_nn_accum *a;
  double nc;                  // |C|
  bool moments;
  double mean_all, m2_all;    // moments of d over all kept pairs, ranks merged in order
};
static DirMoments dir_moments(const me_nn_accum *a) {
  DirMoments M;
  M.a = a;
  M.nc = (double)a->n_corr;
  double n_all = 0;
  M.mean_all = 0; M.m2_all = 0;
  for (int s = 0; s < ME_MAX_WORLD; ++s) chan_merge(n_all, M.mean_all, M.m2_all, a->rank_n[s], a->rank_mean[s], a->rank_m2[s]);
  // every sweep of the library fills the moments; an accumulator built from the sums only (its slots do not account for
  // its pairs) has nothing better than the closed form, which cancels when the spread of d is small against its mean
  M.moments = n_all == M.nc;
  return M;
}
// one level (n_inlier pairs with d <= tau, their sum d and sum d^2) -> mean, rmse, fitness, sigma
static void dir_level(const DirMoments &M, int64_t n_inlier, double sum_d, double sum_d2, int64_t n_source, double *mean_out,
                      double *rmse_out, double *fitness_out, double *sigma_out) {
  const double nc = M.nc;
  const int target_num = (int)n_source;                       // map_eval.cpp:1128
  const double mean = sum_d / nc;                              // :1125
  *mean_out = mean;
  *rmse_out = std::sqrt(sum_d2 / nc);                          // :1126,1131
  *fitness_out = (double)n_inlier * 1.0 / target_num;          // :1130
  // :1132-1138, the sum over ALL kept pairs of (d - mean_k)^2 = M2 + n (mean_all - mean_k)^2: both terms are >= 0, so
  // nothing cancels however small the spread of d is against its mean
  double ss;
  if (M.moments) {
    const double dm = M.mean_all - mean;
    ss = M.m2_all + nc * dm * dm;
  } else {
    ss = M.a->sum_d2_all - 2.0 * mean * M.a->sum_d_all + nc * mean * mean;
    if (ss < 0 && ss > -1e-9 * M.a->sum_d2_all) ss = 0;
  }
  *sigma_out = std::sqrt(ss / nc);
}
// map_eval.cpp:1245-1253 at one level
static void pair_level(double e2g_fitness, double e2g_rmse, int64_t e2g_n_inlier, double g2e_rmse, int64_t n_est, int64_t n_gt,
                       double *cd, double *f1, double *iou) {
  *cd = e2g_rmse + g2e_rmse;
  const double overlap = e2g_fitness, rmse = e2g_rmse;
  *f1 = 2 * overlap * rmse / (overlap + rmse);
  const int num_intersection = (int)e2g_n_inlier;
  const int num_union = (int)(n_est + n_gt - num_intersection);
  *iou = (double)num_intersection / num_union;
}

static void finalize_dir(const me_nn_accum *a, int64_t n_source, me_dir_result *r) {
  std::memset(r, 0, sizeof(*r));
  r->n_source = n_source;
  r->n_corr = a->n_corr;
  r->n_ub = a->n_ub;
  r->sum_nn_dist = a->sum_nn_dist;
  const DirMoments M = dir_moments(a);
  for (int k = 0; k < 5; ++k) {
    r->n_inlier[k] = a->n_inlier[k];
    dir_level(M, a->n_inlier[k], a->sum_d[k], a->sum_d2[k], n_source, &r->mean[k], &r->rmse[k], &r->fitness[k], &r->sigma[k]);
  }
}

int me_nn_finalize(const me_nn_params *p, const me_nn_accum *est_to_gt, const me_nn_accum *gt_to_est, int64_t n_est,
                   int64_t n_gt, me_nn_result *out) {
  if (!p || !out) return ME_ERR_INVALID;
  std::memset(out, 0, sizeof(*out));
  me_nn_accum zero;
  std::memset(&zero, 0, sizeof(zero));
  const int dirs = p->directions ? p->directions : 3;
  if (dirs & 1) finalize_dir(est_to_gt ? est_to_gt : &zero, n_est, &out->est_to_gt);
  if (dirs & 2) finalize_dir(gt_to_est ? gt_to_est : &zero, n_gt, &out->gt_to_est);
  for (int k = 0; k < 5; ++k)
    pair_level(out->est_to_gt.fitness[k], out->est_to_gt.rmse[k], out->est_to_gt.n_inlier[k], out->gt_to_est.rmse[k], n_est, n_gt,
               &out->cd[k], &out->f1[k], &out->iou[k]);
  out->full_cd = p->want_full_cd ? (out->est_to_gt.sum_nn_dist / (double)n_est + out->gt_to_est.sum_nn_dist / (double)n_gt) : 0.0;
  return ME_OK;
}

// 1 <= K <= ME_CURVE_MAX_LEVELS, every level finite and >= 0, non-decreasing
static bool curve_levels_ok(const double *tau, int32_t K) {
  if (!tau || K < 1 || K > ME_CURVE_MAX_LEVELS) return false;
  for (int k = 0; k < K; ++k)
    if (!(std::isfinite(tau[k]) && tau[k] >= 0.0) || (k && tau[k] < tau[k - 1])) return false;
  return true;
}

int me_nn_curve_finalize(const me_nn_params *p, const me_nn_accum *est_to_gt, const me_nn_accum *gt_to_est,
                         const double *host_block, const double *tau, int32_t n_tau, int64_t n_est, int64_t n_gt,
                         me_curve_row *rows) {
  if (!p || !host_block || !rows || !curve_levels_ok(tau, n_tau)) return ME_ERR_INVALID;
  const int K = n_tau, stride = 3 * (K + 1) + 1;
  std::memset(rows, 0, (size_t)K * sizeof(me_curve_row));
  me_nn_accum zero;
  std::memset(&zero, 0, sizeof(zero));
  const int dirs = p->directions ? p->directions : 3;
  const me_nn_accum *acc[2] = {est_to_gt ? est_to_gt : &zero, gt_to_est ? gt_to_est : &zero};
  const int64_t n_src[2] = {n_est, n_gt};
  for (int q = 0; q < 2; ++q) {
    if (!(dirs & (1 << q))) continue;
    const double *cnt = host_block + q * stride, *sd = cnt + (K + 1), *sq = sd + (K + 1);
    double all = 0;
    for (int b = 0; b <= K; ++b) all += cnt[b];
    if (all != (double)acc[q]->n_corr) return ME_ERR_INVALID;      // the block and the accumulators of different evaluations
    const DirMoments M = dir_moments(acc[q]);
    double c = 0, s1 = 0, s2 = 0;       // prefix sums over the bins: the pairs with d <= tau_k
    for (int k = 0; k < K; ++k) {
      c += cnt[k]; s1 += sd[k]; s2 += sq[k];
      me_curve_dir *r = q == 0 ? &rows[k].est_to_gt : &rows[k].gt_to_est;
      r->n_inlier = (int64_t)std::llround(c);
      dir_level(M, r->n_inlier, s1, s2, n_src[q], &r->mean, &r->rmse, &r->fitness, &r->sigma);
    }
  }
  for (int k = 0; k < K; ++k) {
    me_curve_row &r = rows[k];
    r.tau = tau[k];
    pair_level(r.est_to_gt.fitness, r.est_to_gt.rmse, r.est_to_gt.n_inlier, r.gt_to_est.rmse, n_est, n_gt, &r.cd, &r.f1, &r.iou);
  }
  return ME_OK;
}

int me_nn_curve_accum_device(me_ctx *ctx, const double *tau, int32_t n_tau, double **device_block, int32_t *n) {
  ME_ENTER(ctx);
  if (!device_block || !n) return fail(ctx, ME_ERR_INVALID, "null argument");
  if (!curve_levels_ok(tau, n_tau))
    return fail(ctx, ME_ERR_INVALID, "me_nn_curve*: 1 <= n_tau <= ME_CURVE_MAX_LEVELS levels, finite, >= 0 and non-decreasing");
  return nn_curve(ctx, tau, n_tau, device_block, n);
}

int me_nn_curve(me_ctx *ctx, const double *tau, int32_t n_tau, me_curve_row *rows) {
  ME_ENTER(ctx);
  if (!rows) return fail(ctx, ME_ERR_INVALID, "null argument");
  if (ctx->world != 1) return fail(ctx, ME_ERR_INVALID, "me_nn_curve needs world == 1; use me_nn_curve_accum_device + all-reduce + me_nn_curve_finalize");
  double *d_blk = nullptr;
  int32_t n = 0;
  ME_TRY(me_nn_curve_accum_device(ctx, tau, n_tau, &d_blk, &n));
  me_nn_accum acc[2];
  ME_TRY(me_accum_fetch(ctx, &acc[0], &acc[1], nullptr, nullptr));
  std::vector<double> h((size_t)n);
  ME_CUDA(ctx, cudaMemcpyAsync(h.data(), d_blk, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (me_nn_curve_finalize(&ctx->curve_p, &acc[0], &acc[1], h.data(), tau, n_tau, ctx->cloud[0].n, ctx->cloud[1].n, rows) != ME_OK)
    return fail(ctx, ME_ERR_INVALID, "me_nn_curve_finalize: the curve block does not match the accumulators");
  return ME_OK;
}

// 1 <= K <= ME_QUANTILE_MAX_PROBS, every probability finite and in [0, 1]
static bool quantile_probs_ok(const double *p, int32_t K) {
  if (!p || K < 1 || K > ME_QUANTILE_MAX_PROBS) return false;
  for (int k = 0; k < K; ++k)
    if (!(std::isfinite(p[k]) && p[k] >= 0.0 && p[k] <= 1.0)) return false;
  return true;
}

int me_quantile_finalize(int64_t n, const double *p, int32_t n_probs, const double *lo_hi, double *values) {
  if (n < 1 || !lo_hi || !values || !quantile_probs_ok(p, n_probs)) return ME_ERR_INVALID;
  for (int k = 0; k < n_probs; ++k) {
    long long kk;
    double g;
    me::quantile_rank(n, p[k], &kk, &g);
    values[k] = me::quantile_lerp(lo_hi[2 * k], lo_hi[2 * k + 1], g);
  }
  return ME_OK;
}

int me_nn_quantile_begin(me_ctx *ctx, int32_t population, const double *p, int32_t n_probs) {
  ME_ENTER(ctx);
  if (population != ME_DIST_KEPT && population != ME_DIST_NN) return fail(ctx, ME_ERR_INVALID, "population must be ME_DIST_KEPT or ME_DIST_NN");
  if (!quantile_probs_ok(p, n_probs))
    return fail(ctx, ME_ERR_INVALID, "me_nn_quantile*: 1 <= n_probs <= ME_QUANTILE_MAX_PROBS probabilities, each finite and in [0, 1]");
  return nn_quantile_begin(ctx, population, p, n_probs);
}

int me_nn_quantile_block(me_ctx *ctx, double **device_block, int32_t *n) {
  ME_ENTER(ctx);
  if (!device_block || !n) return fail(ctx, ME_ERR_INVALID, "null argument");
  return nn_quantile_block(ctx, device_block, n);
}

int me_nn_quantile_step(me_ctx *ctx, int32_t *done) {
  ME_ENTER(ctx);
  if (!done) return fail(ctx, ME_ERR_INVALID, "null argument");
  return nn_quantile_step(ctx, done);
}

int me_nn_quantile_end(me_ctx *ctx, me_quantile_result *out) {
  ME_ENTER(ctx);
  if (!out) return fail(ctx, ME_ERR_INVALID, "null argument");
  return nn_quantile_end(ctx, out);
}

int me_nn_quantiles(me_ctx *ctx, int32_t population, const double *p, int32_t n_probs, me_quantile_result *out) {
  ME_ENTER(ctx);
  if (!out) return fail(ctx, ME_ERR_INVALID, "null argument");
  if (ctx->world != 1)
    return fail(ctx, ME_ERR_INVALID, "me_nn_quantiles needs world == 1; use me_nn_quantile_begin / _block + all-reduce / _step / _end");
  ME_TRY(me_nn_quantile_begin(ctx, population, p, n_probs));
  int32_t done = 0;
  while (!done) ME_TRY(me_nn_quantile_step(ctx, &done));
  return me_nn_quantile_end(ctx, out);
}

int me_region_finalize(int64_t n_regions, double region_size, const int64_t *index, const int64_t *n_est, const int64_t *n_gt,
                       const double *host_block, me_region_row *rows) {
  if (n_regions < 0 || !(std::isfinite(region_size) && region_size > 0.0)) return ME_ERR_INVALID;
  if (n_regions > 0 && (!index || !n_est || !n_gt || !host_block || !rows)) return ME_ERR_INVALID;
  const int F = ME_REGION_SUM_FIELDS;
  const double *mx = host_block + (size_t)2 * F * n_regions;
  me_nn_accum none;
  std::memset(&none, 0, sizeof(none));
  for (int64_t r = 0; r < n_regions; ++r) {
    me_region_row &R = rows[r];
    std::memset(&R, 0, sizeof(R));
    for (int a = 0; a < 3; ++a) {
      R.index[a] = index[3 * r + a];
      R.min[a] = (double)R.index[a] * region_size;
      R.max[a] = (double)(R.index[a] + 1) * region_size;
    }
    R.n_est = n_est[r];
    R.n_gt = n_gt[r];
    for (int q = 0; q < 2; ++q) {
      const double *v = host_block + ((size_t)r * 2 + q) * F;
      me_region_dir &D = q == 0 ? R.est_to_gt : R.gt_to_est;
      D.n_query = (int64_t)v[0];
      D.n_corr = (int64_t)v[1];
      for (int k = 0; k < 5; ++k) { D.n_inlier[k] = (int64_t)v[2 + k]; D.sum_d[k] = v[7 + k]; D.sum_d2[k] = v[12 + k]; }
      D.sum_nn_dist = v[17];
      D.max_d = mx[((size_t)r * 2 + q) * ME_REGION_MAX_FIELDS];
      D.max_nn = mx[((size_t)r * 2 + q) * ME_REGION_MAX_FIELDS + 1];
      // no sigma per region (DESIGN §3.12): dir_level's sigma output is dropped, so the moments it would read do not matter
      const DirMoments M{&none, (double)D.n_corr, true, 0.0, 0.0};
      double sigma;
      for (int k = 0; k < 5; ++k)
        dir_level(M, D.n_inlier[k], D.sum_d[k], D.sum_d2[k], q == 0 ? R.n_est : R.n_gt, &D.mean[k], &D.rmse[k], &D.fitness[k], &sigma);
      D.mean_nn = D.sum_nn_dist / (double)D.n_query;
    }
    for (int k = 0; k < 5; ++k)
      pair_level(R.est_to_gt.fitness[k], R.est_to_gt.rmse[k], R.est_to_gt.n_inlier[k], R.gt_to_est.rmse[k], R.n_est, R.n_gt, &R.cd[k],
                 &R.f1[k], &R.iou[k]);
  }
  return ME_OK;
}

int me_nn_region_begin(me_ctx *ctx, double region_size, int64_t *n_regions) {
  ME_ENTER(ctx);
  if (!n_regions) return fail(ctx, ME_ERR_INVALID, "null argument");
  if (!(std::isfinite(region_size) && region_size > 0.0)) return fail(ctx, ME_ERR_INVALID, "me_nn_region*: region_size must be finite and > 0");
  return nn_region_begin(ctx, region_size, n_regions);
}

int me_nn_region_block(me_ctx *ctx, double **device_block, int32_t *n_sum, int32_t *n_max) {
  ME_ENTER(ctx);
  if (!device_block || !n_sum || !n_max) return fail(ctx, ME_ERR_INVALID, "null argument");
  return nn_region_block(ctx, device_block, n_sum, n_max);
}

int me_nn_region_end(me_ctx *ctx, me_region_row *rows, int64_t capacity) {
  ME_ENTER(ctx);
  if (!rows) return fail(ctx, ME_ERR_INVALID, "null argument");
  return nn_region_end(ctx, rows, capacity);
}

int me_nn_regions(me_ctx *ctx, double region_size, me_region_row **rows, int64_t *n_regions) {
  ME_ENTER(ctx);
  if (!rows || !n_regions) return fail(ctx, ME_ERR_INVALID, "null argument");
  *rows = nullptr;
  *n_regions = 0;
  if (ctx->world != 1)
    return fail(ctx, ME_ERR_INVALID, "me_nn_regions needs world == 1; use me_nn_region_begin / _block + all-reduce / _end");
  int64_t n = 0;
  ME_TRY(me_nn_region_begin(ctx, region_size, &n));
  return one_shot_rows(ctx, n, 1, "me_nn_regions: host allocation of the rows failed",
                       [&](me_region_row *r) { return me_nn_region_end(ctx, r, n); }, [] {}, rows, n_regions);
}

int me_surface_finalize(const me_nn_params *p, const double *host_block, int64_t n_est, int64_t n_gt, me_surface_result *out) {
  if (!p || !host_block || !out) return ME_ERR_INVALID;
  std::memset(out, 0, sizeof(*out));
  me_nn_accum a, b;
  std::memset(&a, 0, sizeof(a));
  std::memset(&b, 0, sizeof(b));
  decode_block(host_block, &a, &b, nullptr, nullptr);      // the NN-laid-out part: the five-level table of e
  ME_TRY(me_nn_finalize(p, &a, &b, n_est, n_gt, &out->plane));
  const double *x = host_block + 2 * kBlkNN, *mx = host_block + ME_SURFACE_BLOCK_SUM;
  for (int q = 0; q < 2; ++q) {
    me_surface_dir &D = q == 0 ? out->est_to_gt : out->gt_to_est;
    D.n_no_normal = (int64_t)std::llround(x[4 * q]);
    D.n_no_normal_nn = (int64_t)std::llround(x[4 * q + 1]);
    D.n_nc = (int64_t)std::llround(x[4 * q + 2]);
    D.normal_consistency = D.n_nc ? x[4 * q + 3] / x[4 * q + 2] : NAN;
    D.max_e = mx[2 * q];
    D.max_e_nn = mx[2 * q + 1];
  }
  out->normal_consistency = (out->est_to_gt.normal_consistency + out->gt_to_est.normal_consistency) / 2.0;
  return ME_OK;
}

int me_nn_surface_begin(me_ctx *ctx, int32_t knn) {
  ME_ENTER(ctx);
  if (knn < 0 || knn > 64) return fail(ctx, ME_ERR_INVALID, "me_nn_surface*: knn must be 0 (the clouds' own normals) or in 1..64");
  return nn_surface_begin(ctx, knn);
}

int me_nn_surface_normals_slice(me_ctx *ctx, int which, double **device_normals, int64_t *slice_points, int32_t *pending) {
  ME_ENTER(ctx);
  if (!cloud_id(which)) return fail(ctx, ME_ERR_INVALID, "bad cloud id");
  if (!device_normals || !slice_points || !pending) return fail(ctx, ME_ERR_INVALID, "null argument");
  return nn_surface_normals_slice(ctx, which, device_normals, slice_points, pending);
}

int me_nn_surface_block(me_ctx *ctx, double **device_block, int32_t *n_sum, int32_t *n_max) {
  ME_ENTER(ctx);
  if (!device_block || !n_sum || !n_max) return fail(ctx, ME_ERR_INVALID, "null argument");
  return nn_surface_block(ctx, device_block, n_sum, n_max);
}

int me_nn_surface_end(me_ctx *ctx, me_surface_result *out) {
  ME_ENTER(ctx);
  if (!out) return fail(ctx, ME_ERR_INVALID, "null argument");
  return nn_surface_end(ctx, out);
}

int me_nn_surface(me_ctx *ctx, int32_t knn, me_surface_result *out) {
  ME_ENTER(ctx);
  if (!out) return fail(ctx, ME_ERR_INVALID, "null argument");
  if (ctx->world != 1)
    return fail(ctx, ME_ERR_INVALID, "me_nn_surface needs world == 1; use me_nn_surface_begin / _normals_slice / _block + all-reduce / _end");
  ME_TRY(me_nn_surface_begin(ctx, knn));
  double *d = nullptr;
  int64_t s = 0;
  int32_t pending = 0, n_sum = 0, n_max = 0;
  ME_TRY(me_nn_surface_normals_slice(ctx, ME_CLOUD_EST, &d, &s, &pending));
  ME_TRY(me_nn_surface_normals_slice(ctx, ME_CLOUD_GT, &d, &s, &pending));
  ME_TRY(me_nn_surface_block(ctx, &d, &n_sum, &n_max));
  return me_nn_surface_end(ctx, out);
}

// the means of one region (or of the whole map) from its counts and sums: me_consistency_finalize
static void consistency_means(int64_t n_valid, int64_t n_pv, double sum_e, double sum_v, double sum_sv, double max_v, double *mme,
                              double *mpv, double *mean_std, double *max_pv) {
  *mme = n_valid > 0 ? sum_e / (double)n_valid : 0.0;      // as me_mme_finalize
  *mpv = n_pv > 0 ? sum_v / (double)n_pv : NAN;
  *mean_std = n_pv > 0 ? sum_sv / (double)n_pv : NAN;
  *max_pv = n_pv > 0 ? max_v : NAN;
}

int me_consistency_finalize(int64_t n_regions, double region_size, const int64_t *index, const int64_t *n_points, int64_t n_total,
                            const double *host_block, me_consistency_row *rows, me_consistency_result *whole) {
  if (!host_block || !whole || n_regions < 0 || n_total < 0 || !(std::isfinite(region_size) && region_size >= 0.0)) return ME_ERR_INVALID;
  if ((region_size == 0.0) != (n_regions == 0)) return ME_ERR_INVALID;
  if (n_regions > 0 && (!index || !n_points || !rows)) return ME_ERR_INVALID;
  const int S = ME_CONSISTENCY_SUM_FIELDS;
  const int64_t B = std::max<int64_t>(n_regions, 1);      // s = 0: the block holds one region, the whole map
  const double *mx = host_block + (size_t)S * B;
  me_consistency_result &W = *whole;
  std::memset(&W, 0, sizeof(W));
  W.region_size = region_size;
  W.n_regions = n_regions;
  W.n_points = n_total;
  double max_v = 0.0;
  for (int64_t r = 0; r < B; ++r) {      // the whole map: the regions' sums in list order
    const double *v = host_block + (size_t)r * S;
    const int64_t nq = (int64_t)v[0], nv = (int64_t)v[1], np = (int64_t)v[2];
    W.n_query += nq; W.n_valid += nv; W.n_pv += np;
    W.sum_entropy += v[3]; W.sum_pv += v[4]; W.sum_sqrt_pv += v[5];
    max_v = std::fmax(max_v, mx[r * ME_CONSISTENCY_MAX_FIELDS]);
    if (n_regions == 0) continue;
    me_consistency_row &R = rows[r];
    std::memset(&R, 0, sizeof(R));
    for (int a = 0; a < 3; ++a) {
      R.index[a] = index[3 * r + a];
      R.min[a] = (double)R.index[a] * region_size;
      R.max[a] = (double)(R.index[a] + 1) * region_size;
    }
    R.n_points = n_points[r];
    R.n_query = nq; R.n_valid = nv; R.n_pv = np;
    R.sum_entropy = v[3]; R.sum_pv = v[4]; R.sum_sqrt_pv = v[5];
    consistency_means(nv, np, v[3], v[4], v[5], mx[r * ME_CONSISTENCY_MAX_FIELDS], &R.mme, &R.mpv, &R.mean_plane_std, &R.max_pv);
  }
  consistency_means(W.n_valid, W.n_pv, W.sum_entropy, W.sum_pv, W.sum_sqrt_pv, max_v, &W.mme, &W.mpv, &W.mean_plane_std, &W.max_pv);
  return ME_OK;
}

int me_consistency_begin(me_ctx *ctx, int which, double radius, int32_t min_neighbors, double region_size, int64_t *n_regions) {
  ME_ENTER(ctx);
  if (!n_regions) return fail(ctx, ME_ERR_INVALID, "null argument");
  *n_regions = 0;
  ctx->consistency.open = false;
  if (!cloud_id(which)) return fail(ctx, ME_ERR_INVALID, "me_consistency_begin: which must be ME_CLOUD_EST or ME_CLOUD_GT");
  if (!(std::isfinite(radius) && radius > 0.0)) return fail(ctx, ME_ERR_INVALID, "me_consistency_begin: radius must be finite and > 0");
  if (min_neighbors < 3) return fail(ctx, ME_ERR_INVALID, "me_consistency_begin: min_neighbors must be >= 3");
  if (!(std::isfinite(region_size) && region_size >= 0.0))
    return fail(ctx, ME_ERR_INVALID, "me_consistency_begin: region_size must be finite and >= 0 (0: the whole map only)");
  return consistency_begin(ctx, which, radius, min_neighbors, region_size, n_regions);
}

int me_consistency_block(me_ctx *ctx, double **device_block, int32_t *n_sum, int32_t *n_max) {
  ME_ENTER(ctx);
  if (!device_block || !n_sum || !n_max) return fail(ctx, ME_ERR_INVALID, "null argument");
  return consistency_block(ctx, device_block, n_sum, n_max);
}

int me_consistency_end(me_ctx *ctx, me_consistency_row *rows, int64_t capacity, me_consistency_result *whole) {
  ME_ENTER(ctx);
  if (!whole) return fail(ctx, ME_ERR_INVALID, "null argument");
  return consistency_end(ctx, rows, capacity, whole);
}

int me_consistency(me_ctx *ctx, int which, double radius, int32_t min_neighbors, double region_size, me_consistency_row **rows,
                   int64_t *n_regions, me_consistency_result *whole) {
  ME_ENTER(ctx);
  if (!rows || !n_regions || !whole) return fail(ctx, ME_ERR_INVALID, "null argument");
  *rows = nullptr;
  *n_regions = 0;
  if (ctx->world != 1)
    return fail(ctx, ME_ERR_INVALID, "me_consistency needs world == 1; use me_consistency_begin / _block + all-reduce / _end");
  int64_t n = 0;
  ME_TRY(me_consistency_begin(ctx, which, radius, min_neighbors, region_size, &n));
  return one_shot_rows(ctx, n, 0, "me_consistency: host allocation of the rows failed",
                       [&](me_consistency_row *r) { return me_consistency_end(ctx, r, n, whole); },
                       [&] { ctx->consistency.open = false; }, rows, n_regions);
}

int me_get_consistency_points(me_ctx *ctx, int which, double *entropy, double *plane_variance) {
  ME_ENTER(ctx);
  if (!cloud_id(which)) return fail(ctx, ME_ERR_INVALID, "bad cloud id");
  return consistency_points(ctx, which, entropy, plane_variance);
}

static int mom_params_ok(me_ctx *ctx, const me_mom_params *p) {
  if (!p) return fail(ctx, ME_ERR_INVALID, "null argument");
  if (!(p->angle_deg > 0.0 && p->angle_deg <= 30.0)) return fail(ctx, ME_ERR_INVALID, "me_mom_begin: angle_deg must be in (0, 30]");
  if (!(p->planarity > 0.0 && p->planarity <= 1.0)) return fail(ctx, ME_ERR_INVALID, "me_mom_begin: planarity must be in (0, 1]");
  if (p->min_family < 1) return fail(ctx, ME_ERR_INVALID, "me_mom_begin: min_family must be >= 1");
  return ME_OK;
}

int me_mom_begin(me_ctx *ctx, int which, double radius, int32_t min_neighbors, const me_mom_params *p) {
  ME_ENTER(ctx);
  ctx->mom.open = false;
  if (!cloud_id(which)) return fail(ctx, ME_ERR_INVALID, "me_mom_begin: which must be ME_CLOUD_EST or ME_CLOUD_GT");
  if (!(std::isfinite(radius) && radius > 0.0)) return fail(ctx, ME_ERR_INVALID, "me_mom_begin: radius must be finite and > 0");
  if (min_neighbors < 3) return fail(ctx, ME_ERR_INVALID, "me_mom_begin: min_neighbors must be >= 3");
  ME_TRY(mom_params_ok(ctx, p));
  return mom_begin(ctx, which, radius, min_neighbors, p);
}

int me_mom_block(me_ctx *ctx, double **device_block, int32_t *n) {
  ME_ENTER(ctx);
  if (!device_block || !n) return fail(ctx, ME_ERR_INVALID, "null argument");
  return mom_block(ctx, device_block, n);
}

int me_mom_step(me_ctx *ctx, int32_t *done) {
  ME_ENTER(ctx);
  if (!done) return fail(ctx, ME_ERR_INVALID, "null argument");
  return mom_step(ctx, done);
}

int me_mom_end(me_ctx *ctx, me_mom_result *out) {
  ME_ENTER(ctx);
  if (!out) return fail(ctx, ME_ERR_INVALID, "null argument");
  return mom_end(ctx, out);
}

int me_mom(me_ctx *ctx, int which, double radius, int32_t min_neighbors, const me_mom_params *p, me_mom_result *out) {
  ME_ENTER(ctx);
  if (!out) return fail(ctx, ME_ERR_INVALID, "null argument");
  if (ctx->world != 1) return fail(ctx, ME_ERR_INVALID, "me_mom needs world == 1; use me_mom_begin / _block + all-reduce / _step / _end");
  ME_TRY(me_mom_begin(ctx, which, radius, min_neighbors, p));
  int32_t done = 0;
  while (!done) ME_TRY(me_mom_step(ctx, &done));
  return me_mom_end(ctx, out);
}

int me_get_mom_points(me_ctx *ctx, int which, double *v, double *lambda2, double *normal, int8_t *family) {
  ME_ENTER(ctx);
  if (!cloud_id(which)) return fail(ctx, ME_ERR_INVALID, "bad cloud id");
  return mom_points(ctx, which, v, lambda2, normal, family);
}

int me_mom_region_begin(me_ctx *ctx, double region_size, int64_t min_family, int64_t *n_regions) {
  ME_ENTER(ctx);
  if (!n_regions) return fail(ctx, ME_ERR_INVALID, "null argument");
  *n_regions = 0;
  ctx->mom_region.open = false;
  if (!(std::isfinite(region_size) && region_size > 0.0))
    return fail(ctx, ME_ERR_INVALID, "me_mom_region_begin: region_size must be finite and > 0");
  if (min_family < 1) return fail(ctx, ME_ERR_INVALID, "me_mom_region_begin: min_family must be >= 1");
  return mom_region_begin(ctx, region_size, min_family, n_regions);
}

int me_mom_region_block(me_ctx *ctx, double **device_block, int64_t *n) {
  ME_ENTER(ctx);
  if (!device_block || !n) return fail(ctx, ME_ERR_INVALID, "null argument");
  return mom_region_block(ctx, device_block, n);
}

int me_mom_region_end(me_ctx *ctx, me_mom_region_row *rows, int64_t capacity) {
  ME_ENTER(ctx);
  return mom_region_end(ctx, rows, capacity);
}

int me_mom_regions(me_ctx *ctx, double region_size, int64_t min_family, me_mom_region_row **rows, int64_t *n_regions) {
  ME_ENTER(ctx);
  if (!rows || !n_regions) return fail(ctx, ME_ERR_INVALID, "null argument");
  *rows = nullptr;
  *n_regions = 0;
  if (ctx->world != 1)
    return fail(ctx, ME_ERR_INVALID, "me_mom_regions needs world == 1; use me_mom_region_begin / _block + all-reduce / _end");
  int64_t n = 0;
  ME_TRY(me_mom_region_begin(ctx, region_size, min_family, &n));
  return one_shot_rows(ctx, n, 1, "me_mom_regions: host allocation of the rows failed",
                       [&](me_mom_region_row *r) { return me_mom_region_end(ctx, r, n); },
                       [&] { ctx->mom_region.open = false; }, rows, n_regions);
}

int me_drift_begin(me_ctx *ctx, double region_size, double max_correspondence_distance, int32_t max_iteration,
                   double relative_fitness, double relative_rmse, int64_t *n_regions) {
  ME_ENTER(ctx);
  // bad arguments are refused before anything is staled: an open drift loop stays open
  if (!n_regions) return fail(ctx, ME_ERR_INVALID, "null argument");
  *n_regions = 0;
  if (!(std::isfinite(region_size) && region_size > 0.0)) return fail(ctx, ME_ERR_INVALID, "me_drift_begin: region_size must be finite and > 0");
  if (!(std::isfinite(max_correspondence_distance) && max_correspondence_distance > 0.0))
    return fail(ctx, ME_ERR_INVALID, "me_drift_begin: max_correspondence_distance must be finite and > 0");
  if (max_iteration < 0) return fail(ctx, ME_ERR_INVALID, "me_drift_begin: max_iteration must be >= 0");
  ctx->cloud_gen++;      // stales the NN records (me_nn_curve*)
  return drift_begin(ctx, region_size, max_correspondence_distance, max_iteration, relative_fitness, relative_rmse, n_regions);
}

int me_drift_block(me_ctx *ctx, double **device_block, int32_t *n_sum) {
  ME_ENTER(ctx);
  if (!device_block || !n_sum) return fail(ctx, ME_ERR_INVALID, "null argument");
  return drift_block(ctx, device_block, n_sum);
}

int me_drift_step(me_ctx *ctx, int32_t *done) {
  ME_ENTER(ctx);
  if (!done) return fail(ctx, ME_ERR_INVALID, "null argument");
  return drift_step(ctx, done);
}

int me_drift_end(me_ctx *ctx, me_drift_row *rows, int64_t capacity) {
  ME_ENTER(ctx);
  if (!rows) return fail(ctx, ME_ERR_INVALID, "null argument");
  const int rc = drift_end(ctx, rows, capacity);
  ctx->cloud_gen++;      // the estimated cloud is back as it was: records of the moved cloud are stale
  return rc;
}

int me_drift(me_ctx *ctx, double region_size, double max_correspondence_distance, int32_t max_iteration, double relative_fitness,
             double relative_rmse, me_drift_row **rows, int64_t *n_regions) {
  ME_ENTER(ctx);
  if (!rows || !n_regions) return fail(ctx, ME_ERR_INVALID, "null argument");
  *rows = nullptr;
  *n_regions = 0;
  if (ctx->world != 1)
    return fail(ctx, ME_ERR_INVALID, "me_drift needs world == 1; use me_drift_begin / _block + all-reduce / _step / _end");
  int64_t n = 0;
  ME_TRY(me_drift_begin(ctx, region_size, max_correspondence_distance, max_iteration, relative_fitness, relative_rmse, &n));
  int32_t done = 0;
  while (!done) ME_TRY(me_drift_step(ctx, &done));
  return one_shot_rows(ctx, n, 1, "me_drift: host allocation of the rows failed",
                       [&](me_drift_row *r) { return me_drift_end(ctx, r, n); },
                       [&] { drift_close(ctx, true); ctx->cloud_gen++; }, rows, n_regions);
}

int me_eval_nn(me_ctx *ctx, const me_nn_params *p, me_nn_result *out) {
  ME_ENTER(ctx);
  if (!p || !out) return fail(ctx, ME_ERR_INVALID, "null argument");
  if (ctx->world != 1) return fail(ctx, ME_ERR_INVALID, "me_eval_nn needs world == 1; use me_eval_nn_accum + all-reduce + me_nn_finalize");
  me_nn_accum a, b;
  ME_TRY(me_eval_nn_accum(ctx, p, &a, &b));
  return me_nn_finalize(p, &a, &b, ctx->cloud[0].n, ctx->cloud[1].n, out);
}

int me_get_nn(me_ctx *ctx, int which_query, int32_t *nn_index, double *nn_sqdist) {
  ME_ENTER(ctx);
  if (which_query != ME_CLOUD_EST && which_query != ME_CLOUD_GT) return fail(ctx, ME_ERR_INVALID, "bad cloud id");
  return unsort_nn(ctx, which_query, nn_index, nn_sqdist);
}

int me_eval_mme_accum(me_ctx *ctx, int which, double radius, int32_t min_neighbors, me_mme_accum *out) {
  ME_ENTER(ctx);
  if ((which != ME_CLOUD_EST && which != ME_CLOUD_GT) || !out) return fail(ctx, ME_ERR_INVALID, "bad arguments");
  ME_TRY(run_mme(ctx, which, radius, min_neighbors));
  const double *h = nullptr;
  ME_TRY(fetch_block(ctx, &h));
  decode_block(h, nullptr, nullptr, which == ME_CLOUD_EST ? out : nullptr, which == ME_CLOUD_GT ? out : nullptr);
  return ME_OK;
}

int me_mme_finalize(const me_mme_accum *acc, int64_t n_total, me_mme_result *out) {
  if (!acc || !out) return ME_ERR_INVALID;
  out->n_total = n_total;
  out->n_valid = acc->n_valid;
  out->mme = acc->n_valid > 0 ? acc->sum_entropy / (double)acc->n_valid : 0.0;   // map_eval.cpp:1720-1724
  if (acc->min_entropy <= acc->max_entropy) {                                     // :700-701
    out->max_abs_entropy = std::fabs(acc->min_entropy);
    out->min_abs_entropy = std::fabs(acc->max_entropy);
  } else {
    out->max_abs_entropy = out->min_abs_entropy = std::numeric_limits<double>::quiet_NaN();
  }
  return ME_OK;
}

int me_get_entropies(me_ctx *ctx, int which, double *entropies_host) {
  ME_ENTER(ctx);
  if ((which != ME_CLOUD_EST && which != ME_CLOUD_GT) || !entropies_host) return fail(ctx, ME_ERR_INVALID, "bad arguments");
  return unsort_entropy(ctx, which, entropies_host);
}

int me_eval_mme(me_ctx *ctx, int which, double radius, int32_t min_neighbors, me_mme_result *out, double *entropies_host) {
  ME_ENTER(ctx);
  if (!out) return fail(ctx, ME_ERR_INVALID, "null result");
  if (ctx->world != 1) return fail(ctx, ME_ERR_INVALID, "me_eval_mme needs world == 1; use me_eval_mme_accum + all-reduce + me_mme_finalize");
  me_mme_accum acc;
  ME_TRY(me_eval_mme_accum(ctx, which, radius, min_neighbors, &acc));
  ME_TRY(me_mme_finalize(&acc, ctx->cloud[which].n, out));
  if (entropies_host) ME_TRY(unsort_entropy(ctx, which, entropies_host));
  return ME_OK;
}

int me_eval_awd(me_ctx *ctx, double voxel_size, int32_t min_points, int32_t scs_radius, me_awd_result *out,
                int64_t *n_rows, double **rows27) {
  ME_ENTER(ctx);
  if (!out) return fail(ctx, ME_ERR_INVALID, "null result");
  return run_awd(ctx, voxel_size, min_points, scs_radius, out, n_rows, rows27);
}

int me_eval_w2(me_ctx *ctx, double voxel_size, int32_t min_points, int32_t scs_radius, me_w2_result *out, int64_t *n_rows,
               double **rows) {
  ME_ENTER(ctx);
  if (!out) return fail(ctx, ME_ERR_INVALID, "null result");
  return run_w2(ctx, voxel_size, min_points, scs_radius, out, n_rows, rows);
}

int me_w2_from_rows(me_ctx *ctx, const double *rows, int64_t n_rows, double voxel_size, int32_t scs_radius, double *w_out,
                    me_w2_result *out) {
  ME_ENTER(ctx);
  if (!out) return fail(ctx, ME_ERR_INVALID, "null result");
  return run_w2_rows(ctx, rows, n_rows, voxel_size, scs_radius, w_out, out);
}

int me_w2_begin(me_ctx *ctx, double voxel_size, int32_t min_points) {
  ME_ENTER(ctx);
  return w2_begin(ctx, voxel_size, min_points);
}

int me_w2_w_table(me_ctx *ctx, double **device_w, int64_t *n) {
  ME_ENTER(ctx);
  if (!device_w || !n) return fail(ctx, ME_ERR_INVALID, "null argument");
  return w2_w_table(ctx, device_w, n);
}

int me_w2_finish_accum_device(me_ctx *ctx, int32_t scs_radius) {
  ME_ENTER(ctx);
  return w2_finish_block(ctx, scs_radius);
}

int me_w2_block(me_ctx *ctx, double **device_block, int32_t *n) {
  ME_ENTER(ctx);
  if (!device_block || !n) return fail(ctx, ME_ERR_INVALID, "null argument");
  return w2_block(ctx, device_block, n);
}

int me_w2_fetch(me_ctx *ctx, me_w2_result *out) {
  ME_ENTER(ctx);
  if (!out) return fail(ctx, ME_ERR_INVALID, "null result");
  return w2_fetch(ctx, out);
}

int me_awd_from_rows(me_ctx *ctx, const double *rows27, int64_t n_rows, double voxel_size, int32_t scs_radius, double *w_out,
                     me_awd_result *out) {
  ME_ENTER(ctx);
  if (!out) return fail(ctx, ME_ERR_INVALID, "null result");
  return run_awd_rows(ctx, rows27, n_rows, voxel_size, scs_radius, w_out, out);
}

void me_free(void *p) { std::free(p); }

int me_get_stage_times(me_ctx *ctx, double ms[ME_N_STAGE_TIMES]) {
  ME_ENTER(ctx);
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int s = 0; s < ME_N_STAGE_TIMES; ++s) {
    ms[s] = 0.0;
    if (!ctx->ev_used[s]) continue;
    float t = 0.f;
    if (cudaEventElapsedTime(&t, ctx->ev[2 * s], ctx->ev[2 * s + 1]) == cudaSuccess) ms[s] = t;
    else cudaGetLastError();
  }
  return ME_OK;
}

int64_t me_launch_count(const me_ctx *ctx) { return ctx ? ctx->launches : 0; }

int me_kernel_trace(me_ctx *ctx, uint64_t *mask, int32_t *mme_rows_cfg, int32_t reset) {
  ME_ENTER(ctx);
  unsigned int dev = 0;      // the bits the far / brute kernels set
  ME_CUDA(ctx, cudaMemcpyAsync(&dev, ctx->d_trace, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (mask) *mask = (uint64_t)(ctx->kernel_mask | dev);
  if (mme_rows_cfg) *mme_rows_cfg = ctx->mme_rows_cfg;
  if (reset) {
    ctx->kernel_mask = 0;
    ctx->mme_rows_cfg = 0;
    ME_CUDA(ctx, cudaMemsetAsync(ctx->d_trace, 0, sizeof(unsigned int), ctx->stream));
  }
  return ME_OK;
}

}  // extern "C"

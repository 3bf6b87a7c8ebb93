// downsample.cu — voxel down-sampling of a cloud held by the context (SURVEY.md §8f N1: the step right before the path).
//
// Replaces (reference): map_3d_ = map_3d_->VoxelDownSample(param_.downsample_size); gt_3d_ likewise (map_eval.cpp:38-39),
// i.e. open3d::geometry::PointCloud::VoxelDownSample [ext, Open3D 0.15-0.17 PointCloud.cpp]:
//   voxel_min_bound = GetMinBound() - 0.5 * voxel_size
//   voxel index     = int(floor((p - voxel_min_bound) / voxel_size))   per axis, fp64, IEEE division
//   output point    = (sum of the voxel's points, accumulated in INPUT order) / double(count)
//   output normal   = (sum of the voxel's normals without a NaN component, INPUT order) / double(count), not re-normalised;
//                     only when the cloud holds normals (me_set_normals / me_estimate_normals), otherwise there are none
// Open3D emits the voxels in std::unordered_map iteration order (implementation-defined); here they come out in
// increasing (ix, iy, iz).  The SET of output points (and of point-normal pairs) is bit-identical to the CPU path: the
// 64-bit voxel keys are sorted with a STABLE radix sort (points of a voxel stay in input order) and each voxel is summed
// sequentially by one thread.
//
// The sort is the library's own LSD radix sort (sort.cu); key building, run detection and the ordered sums follow.
#include "common.cuh"
#include <algorithm>

namespace me {

static constexpr int kThreads = 256;
static constexpr int kAxisBits = 21;      // voxel indices per axis < 2^21 (1 cm voxels: 20 km)

struct VdsGeom { double org[3]; double s; int bits[3]; };      // bits per axis of the packed key (from the extent)

__global__ void __launch_bounds__(kThreads) vds_key_kernel(const double *__restrict__ xyz, long long n, VdsGeom g,
                                                           unsigned long long *__restrict__ key,
                                                           uint32_t *__restrict__ val, unsigned int *__restrict__ bad) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    unsigned long long k = 0;
    bool ok = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double r = floor(__ddiv_rn(__dsub_rn(__ldg(xyz + 3 * i + a), g.org[a]), g.s));
      ok = ok && r >= 0.0 && r < (double)(1ll << g.bits[a]);
      k = (k << g.bits[a]) | (unsigned long long)(ok ? (long long)r : 0ll);
    }
    if (!ok) atomicAdd(bad, 1u);
    key[i] = k;
    val[i] = (uint32_t)i;
  }
}

// head[i] = 1 where a new voxel starts in the sorted key sequence (head[n] = 0: after the scan it holds the voxel count)
__global__ void __launch_bounds__(kThreads) vds_head_kernel(const unsigned long long *__restrict__ key, long long n,
                                                            uint32_t *__restrict__ head) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i <= n; i += (long long)gridDim.x * blockDim.x)
    head[i] = (i < n && (i == 0 || key[i] != key[i - 1])) ? 1u : 0u;
}

// one thread per voxel start: sequential sum in input order (the sort is stable), then the division by the count.
// kNormals: AccumulatedPoint's normal sum in the same walk — a normal is added only when none of its components is NaN,
// the division is by the count of ALL the voxel's points, and the result is not re-normalised (GetAverageNormal)
template <bool kNormals>
__global__ void __launch_bounds__(kThreads) vds_mean_kernel(const double *__restrict__ xyz, const unsigned long long *__restrict__ key,
                                                            const uint32_t *__restrict__ val, const uint32_t *__restrict__ pos,
                                                            long long n, double *__restrict__ out, const double *__restrict__ nrm,
                                                            double *__restrict__ out_nrm) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t p = pos[i];
    if (pos[i + 1] == p) continue;                    // not the first point of its voxel
    const unsigned long long k = key[i];
    double sx = 0.0, sy = 0.0, sz = 0.0, nx = 0.0, ny = 0.0, nz = 0.0;
    long long cnt = 0;
    for (long long j = i; j < n && key[j] == k; ++j) {
      const long long o = val[j];
      sx = __dadd_rn(sx, __ldg(xyz + 3 * o)); sy = __dadd_rn(sy, __ldg(xyz + 3 * o + 1)); sz = __dadd_rn(sz, __ldg(xyz + 3 * o + 2));
      if (kNormals) {
        const double a = __ldg(nrm + 3 * o), b = __ldg(nrm + 3 * o + 1), c = __ldg(nrm + 3 * o + 2);
        if (!isnan(a) && !isnan(b) && !isnan(c)) { nx = __dadd_rn(nx, a); ny = __dadd_rn(ny, b); nz = __dadd_rn(nz, c); }
      }
      ++cnt;
    }
    const double c = (double)cnt;
    out[3ll * p] = __ddiv_rn(sx, c); out[3ll * p + 1] = __ddiv_rn(sy, c); out[3ll * p + 2] = __ddiv_rn(sz, c);
    if (kNormals) { out_nrm[3ll * p] = __ddiv_rn(nx, c); out_nrm[3ll * p + 1] = __ddiv_rn(ny, c); out_nrm[3ll * p + 2] = __ddiv_rn(nz, c); }
  }
}

int voxel_downsample(me_ctx *ctx, int which, double voxel_size, int64_t *n_out) {
  Cloud &c = ctx->cloud[which];
  if (n_out) *n_out = 0;
  if (c.n <= 0) return fail(ctx, ME_ERR_EMPTY, "cloud is empty");
  if (!(voxel_size > 0.0)) return fail(ctx, ME_ERR_INVALID, "voxel_size must be > 0 (Open3D: voxel_size <= 0 is an error)");
  ME_TRY(wait_upload(ctx, which));
  ME_TRY(compute_bbox(ctx, which));                   // also rejects non-finite coordinates
  const long long n = c.n;
  VdsGeom g;
  g.s = voxel_size;
  int key_bits = 0;
  for (int a = 0; a < 3; ++a) {
    g.org[a] = c.bbox_min[a] - voxel_size * 0.5;      // voxel_min_bound
    // voxels along this axis (+2 of slack for the rounding of the division): only as many key bits as the extent needs,
    // so that the radix sort runs 4-5 passes instead of 8
    const double nv_axis = std::floor((c.bbox_max[a] - g.org[a]) / voxel_size) + 3.0;
    if (!(nv_axis < (double)(1 << kAxisBits)))
      return fail(ctx, ME_ERR_RANGE, "voxel_size is too small for the extent of the cloud (more than 2^21 voxels per axis)");
    int b = 1;
    while ((1ll << b) < (long long)nv_axis) ++b;
    g.bits[a] = b;
    key_bits += b;
  }

  auto align = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t o_key0 = 256, o_key1 = o_key0 + align((size_t)n * 8), o_val0 = o_key1 + align((size_t)n * 8),
               o_val1 = o_val0 + align((size_t)n * 4), o_pos = o_val1 + align((size_t)n * 4),
               total = o_pos + align((size_t)(n + 1) * 4);
  ME_TRY(ensure_work(ctx, total));
  char *base = (char *)ctx->d_work;
  unsigned int *d_bad = (unsigned int *)base;
  unsigned long long *key0 = (unsigned long long *)(base + o_key0), *key1 = (unsigned long long *)(base + o_key1);
  uint32_t *val0 = (uint32_t *)(base + o_val0), *val1 = (uint32_t *)(base + o_val1), *pos = (uint32_t *)(base + o_pos);
  ME_CUDA(ctx, cudaMemsetAsync(d_bad, 0, 256, ctx->stream));
  const int blocks = (int)std::min<long long>((n + kThreads - 1) / kThreads, (long long)ctx->sm_count * 16);
  vds_key_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.d_xyz, n, g, key0, val0, d_bad);
  ME_LAUNCH_CHECK(ctx);
  unsigned long long *key1s = nullptr;
  uint32_t *val1s = nullptr;
  ME_TRY(radix_sort_pairs(ctx, key0, val0, key1, val1, n, key_bits, &key1s, &val1s));      // stable
  key1 = key1s; val1 = val1s;
  vds_head_kernel<<<blocks, kThreads, 0, ctx->stream>>>(key1, n, pos);
  ME_LAUNCH_CHECK(ctx);
  ME_TRY(exclusive_scan_inplace(ctx, pos, n + 1));
  unsigned int *h = (unsigned int *)ctx->h_pinned;
  ME_CUDA(ctx, cudaMemcpyAsync(h, d_bad, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaMemcpyAsync(h + 1, pos + n, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (h[0] != 0) return fail(ctx, ME_ERR_RANGE, "voxel_size is too small for the extent of the cloud (more than 2^21 voxels per axis)");
  const long long nv = (long long)h[1];
  double *out = nullptr, *out_nrm = nullptr;
  long long cap_out = 0, cap_nrm = 0;
  ME_TRY(ensure(ctx, (void **)&out, &cap_out, 3 * nv, sizeof(double)));
  if (c.normal_valid) {
    if (ensure(ctx, (void **)&out_nrm, &cap_nrm, 3 * nv, sizeof(double)) != ME_OK) { cudaFree(out); return ME_ERR_NOMEM; }
    vds_mean_kernel<true><<<blocks, kThreads, 0, ctx->stream>>>(c.d_xyz, key1, val1, pos, n, out, c.d_normal, out_nrm);
  } else {
    vds_mean_kernel<false><<<blocks, kThreads, 0, ctx->stream>>>(c.d_xyz, key1, val1, pos, n, out, nullptr, nullptr);
  }
  ME_LAUNCH_CHECK(ctx);
  ME_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // the old buffers may be released (or handed back) now
  if (c.owned && c.d_xyz) cudaFree(c.d_xyz);
  c.d_xyz = out; c.cap_xyz = cap_out; c.owned = true; c.n = nv;
  if (c.normal_valid) {                               // the normals follow the points: averaged, in the output order
    cudaFree(c.d_normal);
    c.d_normal = out_nrm; c.cap_normal = cap_nrm;
  }
  invalidate_cloud(c);
  if (n_out) *n_out = nv;
  return ME_OK;
}

}  // namespace me

// gpu_group.hpp — the multi-GPU side of the re-hosted MapEval driver: one me_ctx per GPU in ONE process, the sweeps'
// query ranges sharded by rank, both lattices replicated, and the sum-reducible accumulators combined with ONE NCCL
// all-reduce over NVLink / NVSwitch (plus a MAX all-reduce for the entropy extrema).
//
// The reference is single-process with TBB / OpenMP reductions (map_eval.cpp:1411,1420,1704-1708); this is their
// H100-native counterpart.  The C-ABI stays free of NCCL: the library returns per-rank partial accumulators
// (me_eval_nn_accum / me_eval_mme_accum) and finalises reduced ones on the host (me_nn_finalize / me_mme_finalize).
#pragma once
#include <cuda_runtime_api.h>
#include <nccl.h>

#include <cmath>
#include <cstring>
#include <functional>
#include <string>
#include <thread>
#include <vector>

#include "../../include/mapeval_b200.h"

class GpuGroup {
 public:
  GpuGroup() = default;
  GpuGroup(const GpuGroup &) = delete;
  GpuGroup &operator=(const GpuGroup &) = delete;
  ~GpuGroup() { destroy(); }

  int size() const { return (int)ctx_.size(); }
  me_ctx *ctx(int r) const { return ctx_[r]; }
  const std::string &error() const { return err_; }

  // contexts on devices first_device .. first_device + n - 1, rank r of world n each
  bool create(int n, int first_device, double vmd_voxel_size) {
    destroy();
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || first_device < 0 || first_device + n > ndev) {
      err_ = "n_gpus = " + std::to_string(n) + " from device " + std::to_string(first_device) + ", but " + std::to_string(ndev) +
             " CUDA device(s) are visible";
      return false;
    }
    for (int r = 0; r < n; ++r) {
      me_options opt{};
      opt.abi_version = ME_ABI_VERSION;
      opt.device = first_device + r;
      opt.rank = r;
      opt.world = n;
      opt.vmd_voxel_size = vmd_voxel_size;
      me_ctx *c = nullptr;
      if (me_create(&opt, &c) != ME_OK) { err_ = me_last_error(nullptr); destroy(); return false; }
      ctx_.push_back(c);
      dev_.push_back(first_device + r);
    }
    if (n > 1) {
      comm_.resize(n);
      if (ncclCommInitAll(comm_.data(), n, dev_.data()) != ncclSuccess) { comm_.clear(); err_ = "ncclCommInitAll failed"; destroy(); return false; }
      stream_.resize(n, nullptr);
      buf_.resize(n, nullptr);
      for (int r = 0; r < n; ++r) {
        cudaSetDevice(dev_[r]);
        if (cudaStreamCreateWithFlags(&stream_[r], cudaStreamNonBlocking) != cudaSuccess ||
            cudaMalloc((void **)&buf_[r], kMaxValues * sizeof(double)) != cudaSuccess) {
          err_ = "allocating the all-reduce buffers failed"; destroy(); return false;
        }
      }
    }
    return true;
  }

  // f(rank, ctx) on one host thread per GPU (the C-ABI calls block until their GPU is done); returns the first failure
  int for_each(const std::function<int(int, me_ctx *)> &f) {
    const int n = size();
    std::vector<int> rc(n, ME_OK);
    if (n == 1) rc[0] = f(0, ctx_[0]);
    else {
      std::vector<std::thread> th;
      for (int r = 0; r < n; ++r) th.emplace_back([&, r] { rc[r] = f(r, ctx_[r]); });
      for (auto &t : th) t.join();
    }
    for (int r = 0; r < n; ++r)
      if (rc[r] != ME_OK) { err_ = std::string("rank ") + std::to_string(r) + ": " + me_last_error(ctx_[r]); return rc[r]; }
    return ME_OK;
  }

  // in-place all-reduce of per-rank value vectors (all of the same length <= kMaxValues); every rank ends with the result
  bool allreduce(std::vector<std::vector<double>> &v, ncclRedOp_t op) {
    const int n = size();
    if (n == 1) return true;
    const size_t len = v[0].size();
    if (len == 0) return true;
    if (len > (size_t)kMaxValues) { err_ = "all-reduce block too large"; return false; }
    for (int r = 0; r < n; ++r) {
      cudaSetDevice(dev_[r]);
      if (cudaMemcpyAsync(buf_[r], v[r].data(), len * sizeof(double), cudaMemcpyHostToDevice, stream_[r]) != cudaSuccess) { err_ = "H2D failed"; return false; }
    }
    ncclGroupStart();
    for (int r = 0; r < n; ++r) ncclAllReduce(buf_[r], buf_[r], len, ncclDouble, op, comm_[r], stream_[r]);
    if (ncclGroupEnd() != ncclSuccess) { err_ = "ncclAllReduce failed"; return false; }
    for (int r = 0; r < n; ++r) {
      cudaSetDevice(dev_[r]);
      if (cudaMemcpyAsync(v[r].data(), buf_[r], len * sizeof(double), cudaMemcpyDeviceToHost, stream_[r]) != cudaSuccess ||
          cudaStreamSynchronize(stream_[r]) != cudaSuccess) { err_ = "D2H failed"; return false; }
    }
    return true;
  }

  // collectives on buffers the contexts own (the ICP block, the normal slices), in place on the devices.  The caller has
  // waited for the contexts' streams (me_synchronize); on return the result is complete on every device.
  bool allreduce_device(const std::vector<double *> &ptr, size_t len, ncclRedOp_t op) {
    const int n = size();
    if (n == 1 || len == 0) return true;
    ncclGroupStart();
    for (int r = 0; r < n; ++r) ncclAllReduce(ptr[r], ptr[r], len, ncclDouble, op, comm_[r], stream_[r]);
    if (ncclGroupEnd() != ncclSuccess) { err_ = "ncclAllReduce failed"; return false; }
    return sync_streams();
  }
  // rank r contributes ptr[r] + r * per_rank (per_rank doubles); every ptr[r] holds all n slices afterwards
  bool allgather_device(const std::vector<double *> &ptr, size_t per_rank) {
    const int n = size();
    if (n == 1 || per_rank == 0) return true;
    ncclGroupStart();
    for (int r = 0; r < n; ++r) ncclAllGather(ptr[r] + (size_t)r * per_rank, ptr[r], per_rank, ncclDouble, comm_[r], stream_[r]);
    if (ncclGroupEnd() != ncclSuccess) { err_ = "ncclAllGather failed"; return false; }
    return sync_streams();
  }

  // the accuracy curve blocks the contexts hold (me_nn_curve_accum_device, after me_synchronize): ONE grouped SUM all-reduce
  // in place, then rank 0's reduced block into `host` (its size = the block's length)
  bool reduce_curve(const std::vector<double *> &ptr, std::vector<double> &host) {
    if (!allreduce_device(ptr, host.size(), ncclSum)) return false;
    if (cudaSetDevice(dev_[0]) != cudaSuccess ||
        cudaMemcpy(host.data(), ptr[0], host.size() * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess) {
      err_ = "copying the accuracy curve block back failed";
      return false;
    }
    return true;
  }

  // sum-reduce the NN accumulators of all ranks (counts ride along as fp64: exact below 2^53, order-independent)
  bool reduce_nn(std::vector<me_nn_accum> &e2g, std::vector<me_nn_accum> &g2e) {
    const int n = size();
    std::vector<std::vector<double>> v(n);
    for (int r = 0; r < n; ++r) { pack(e2g[r], v[r]); pack(g2e[r], v[r]); }
    if (!allreduce(v, ncclSum)) return false;
    for (int r = 0; r < n; ++r) { size_t k = 0; unpack(v[r], k, e2g[r]); unpack(v[r], k, g2e[r]); }
    return true;
  }
  bool reduce_mme(std::vector<me_mme_accum> &m) {
    const int n = size();
    std::vector<std::vector<double>> s(n), x(n);
    for (int r = 0; r < n; ++r) {
      s[r] = {(double)m[r].n_query, (double)m[r].n_valid, m[r].sum_entropy};
      x[r] = {m[r].max_entropy, -m[r].min_entropy};
    }
    if (!allreduce(s, ncclSum) || !allreduce(x, ncclMax)) return false;
    for (int r = 0; r < n; ++r) {
      m[r].n_query = (int64_t)std::llround(s[r][0]); m[r].n_valid = (int64_t)std::llround(s[r][1]); m[r].sum_entropy = s[r][2];
      m[r].max_entropy = x[r][0]; m[r].min_entropy = -x[r][1];
    }
    return true;
  }

  void destroy() {
    for (size_t r = 0; r < buf_.size(); ++r) if (buf_[r]) { cudaSetDevice(dev_[r]); cudaFree(buf_[r]); }
    for (size_t r = 0; r < stream_.size(); ++r) if (stream_[r]) { cudaSetDevice(dev_[r]); cudaStreamDestroy(stream_[r]); }
    for (auto &c : comm_) ncclCommDestroy(c);
    for (auto *c : ctx_) me_destroy(c);
    buf_.clear(); stream_.clear(); comm_.clear(); ctx_.clear(); dev_.clear();
  }

 private:
  bool sync_streams() {
    for (int r = 0; r < size(); ++r) {
      cudaSetDevice(dev_[r]);
      if (cudaStreamSynchronize(stream_[r]) != cudaSuccess) { err_ = "collective failed on its stream"; return false; }
    }
    return true;
  }
  static constexpr int kMaxValues = 2 * (ME_NN_ACCUM_I64 + ME_NN_ACCUM_F64);
  static void pack(const me_nn_accum &a, std::vector<double> &v) {
    v.push_back((double)a.n_query); v.push_back((double)a.n_corr);
    for (int k = 0; k < 5; ++k) v.push_back((double)a.n_inlier[k]);
    v.push_back((double)a.n_ub); v.push_back((double)a.n_far);
    for (int k = 0; k < 5; ++k) v.push_back(a.sum_d[k]);
    for (int k = 0; k < 5; ++k) v.push_back(a.sum_d2[k]);
    v.push_back(a.sum_d_all); v.push_back(a.sum_d2_all); v.push_back(a.sum_nn_dist);
    v.insert(v.end(), a.rank_n, a.rank_n + ME_MAX_WORLD);
    v.insert(v.end(), a.rank_mean, a.rank_mean + ME_MAX_WORLD);
    v.insert(v.end(), a.rank_m2, a.rank_m2 + ME_MAX_WORLD);
  }
  static void unpack(const std::vector<double> &v, size_t &k, me_nn_accum &a) {
    auto i64 = [&](void) { return (int64_t)std::llround(v[k++]); };
    a.n_query = i64(); a.n_corr = i64();
    for (int j = 0; j < 5; ++j) a.n_inlier[j] = i64();
    a.n_ub = i64(); a.n_far = i64();
    for (int j = 0; j < 5; ++j) a.sum_d[j] = v[k++];
    for (int j = 0; j < 5; ++j) a.sum_d2[j] = v[k++];
    a.sum_d_all = v[k++]; a.sum_d2_all = v[k++]; a.sum_nn_dist = v[k++];
    for (int j = 0; j < ME_MAX_WORLD; ++j) a.rank_n[j] = v[k++];
    for (int j = 0; j < ME_MAX_WORLD; ++j) a.rank_mean[j] = v[k++];
    for (int j = 0; j < ME_MAX_WORLD; ++j) a.rank_m2[j] = v[k++];
  }

  std::vector<me_ctx *> ctx_;
  std::vector<int> dev_;
  std::vector<ncclComm_t> comm_;
  std::vector<cudaStream_t> stream_;
  std::vector<double *> buf_;
  std::string err_;
};

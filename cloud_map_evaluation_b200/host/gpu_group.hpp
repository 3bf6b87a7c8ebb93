// gpu_group.hpp — the multi-GPU side of the re-hosted MapEval driver: one me_ctx per GPU in ONE process, the sweeps'
// query ranges sharded by rank, both lattices replicated, and every reduction done in place on the devices with grouped
// NCCL collectives over NVLink / NVSwitch: the accumulator block of each metric stage (ONE SUM all-reduce, plus a MAX
// all-reduce for the entropy extrema), the accuracy curve block, the distance quantile counts and the ICP block.
//
// The reference is single-process with TBB / OpenMP reductions (map_eval.cpp:1411,1420,1704-1708); this is their
// H100-native counterpart.  The C-ABI stays free of NCCL: the library leaves per-rank partial accumulators in device
// blocks (me_eval_*_accum_device, me_accum_block), and finalises reduced ones on the host (me_nn_finalize / me_mme_finalize).
#pragma once
#include <cuda_runtime_api.h>
#include <nccl.h>

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
      for (int r = 0; r < n; ++r) {
        cudaSetDevice(dev_[r]);
        if (cudaStreamCreateWithFlags(&stream_[r], cudaStreamNonBlocking) != cudaSuccess) {
          err_ = "creating the collective streams failed"; destroy(); return false;
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

  // fn(ctx, &x) on every GPU and rank 0's x into *out: the done flag of a loop's step or the result of its end, which every
  // rank computes from the same reduced blocks
  template <class T> int each(int (*fn)(me_ctx *, T *), T *out) {
    return for_each([&](int r, me_ctx *c) {
      T x{};
      const int rc = fn(c, &x);
      if (r == 0) *out = x;
      return rc;
    });
  }

  // one reduction of a block the contexts own: f(rank, ctx, &ptr, &n_sum, &n_max) fills it on every GPU (n_max stays 0 for a
  // block without a MAX part; N is the count type of the block's C call), me_synchronize, then ONE grouped SUM all-reduce of
  // its first n_sum values and a MAX all-reduce of the next n_max, in place.  On return the block is reduced on every device.
  template <class N = int32_t, class F> bool reduce_block(const F &f) {
    const int n = size();
    std::vector<double *> ptr(n, nullptr), ptr_max(n, nullptr);
    std::vector<N> n_sum(n, 0), n_max(n, 0);
    if (for_each([&](int r, me_ctx *c) {
          const int rc = f(r, c, &ptr[r], &n_sum[r], &n_max[r]);
          if (rc != ME_OK) return rc;
          ptr_max[r] = ptr[r] + n_sum[r];
          return me_synchronize(c);
        }) != ME_OK)
      return false;
    return allreduce_device(ptr, (size_t)n_sum[0], ncclSum) && allreduce_device(ptr_max, (size_t)n_max[0], ncclMax);
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

  // the accuracy curve at the K levels tau (me_nn_curve_accum_device on every GPU): ONE grouped SUM all-reduce of the blocks,
  // then rank 0's reduced block into `host`
  bool reduce_curve(const double *tau, int32_t K, std::vector<double> &host) {
    double *blk0 = nullptr;
    if (!reduce_block([&](int r, me_ctx *c, double **ptr, int32_t *n, int32_t *) {
          const int rc = me_nn_curve_accum_device(c, tau, K, ptr, n);
          if (r == 0 && rc == ME_OK) {
            blk0 = *ptr;
            host.resize((size_t)*n);
          }
          return rc;
        }))
      return false;
    if (cudaSetDevice(dev_[0]) != cudaSuccess ||
        cudaMemcpy(host.data(), blk0, host.size() * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess) {
      err_ = "copying the accuracy curve block back failed";
      return false;
    }
    return true;
  }

  // one metric stage over every GPU: on each, me_accum_reset and the stage's *_device sweep(s) `sweep`, then the accumulator
  // block reduced (reduce_block) and rank 0's reduced block into the structs (any may be NULL).  The reset keeps values of
  // earlier stages out of the sums.
  bool reduce_accum(const std::function<int(me_ctx *)> &sweep, me_nn_accum *e2g, me_nn_accum *g2e, me_mme_accum *mme_est,
                    me_mme_accum *mme_gt) {
    if (!reduce_block([&](int, me_ctx *c, double **ptr, int32_t *n_sum, int32_t *n_max) {
          int rc = me_accum_reset(c);
          if (rc == ME_OK) rc = sweep(c);
          return rc != ME_OK ? rc : me_accum_block(c, ptr, n_sum, n_max);
        }))
      return false;
    if (me_accum_fetch(ctx_[0], e2g, g2e, mme_est, mme_gt) != ME_OK) { err_ = me_last_error(ctx_[0]); return false; }
    return true;
  }

  void destroy() {
    for (size_t r = 0; r < stream_.size(); ++r) if (stream_[r]) { cudaSetDevice(dev_[r]); cudaStreamDestroy(stream_[r]); }
    for (auto &c : comm_) ncclCommDestroy(c);
    for (auto *c : ctx_) me_destroy(c);
    stream_.clear(); comm_.clear(); ctx_.clear(); dev_.clear();
  }

 private:
  // collectives on buffers the contexts own, in place on the devices.  The caller has waited for the contexts' streams
  // (me_synchronize); on return the result is complete on every device.
  bool allreduce_device(const std::vector<double *> &ptr, size_t len, ncclRedOp_t op) {
    const int n = size();
    if (n == 1 || len == 0) return true;
    ncclGroupStart();
    for (int r = 0; r < n; ++r) ncclAllReduce(ptr[r], ptr[r], len, ncclDouble, op, comm_[r], stream_[r]);
    if (ncclGroupEnd() != ncclSuccess) { err_ = "ncclAllReduce failed"; return false; }
    return sync_streams();
  }
  bool sync_streams() {
    for (int r = 0; r < size(); ++r) {
      cudaSetDevice(dev_[r]);
      if (cudaStreamSynchronize(stream_[r]) != cudaSuccess) { err_ = "collective failed on its stream"; return false; }
    }
    return true;
  }
  std::vector<me_ctx *> ctx_;
  std::vector<int> dev_;
  std::vector<ncclComm_t> comm_;
  std::vector<cudaStream_t> stream_;
  std::string err_;
};

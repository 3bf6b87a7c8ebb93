// radix.cuh — the device side of the exact radix selection (RadixSel, common.cuh), shared by the distance quantiles (nn.cu)
// and the per-family medians of the mutually orthogonal metric (mom.cu).  A key is the bit pattern of a finite double >= 0,
// which sorts as an unsigned integer, or kQuantOut outside the population.  Pass j histograms digit j of the keys under
// each slot's prefix (the top 8j bits some target rank still lies under).  Prefixes of one length are disjoint, so a key
// falls under at most one slot, found by binary search over the ascending prefixes.  Counts only: per block a shared
// integer histogram (warp-aggregated), merged into the global one with integer atomics — the result does not depend on
// the order of the additions.
#pragma once
#include "common.cuh"

namespace me {

static constexpr int kQuantThreads = 512;
static constexpr unsigned long long kQuantOut = ~0ull;     // not in the population (no finite d >= 0 has the sign bit)

// the key of a finite d >= 0; -0 sorts with +0
__device__ __forceinline__ unsigned long long quant_key(double d) {
  return (unsigned long long)__double_as_longlong(d == 0.0 ? 0.0 : d);
}

// one count into s_hist[bin] (bin < 0: none), the lanes of a warp with the same bin added by one atomic; the whole warp calls
__device__ __forceinline__ void quant_count(unsigned int *s_hist, int bin) {
  const unsigned int peers = __match_any_sync(0xffffffffu, bin);
  if (bin >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(s_hist + bin, (unsigned int)__popc(peers));
}

// the block's histogram of nbins bins, added into hist
__device__ __forceinline__ void quant_flush(const unsigned int *s_hist, int nbins, unsigned long long *__restrict__ hist) {
  __syncthreads();
  for (int t = threadIdx.x; t < nbins; t += blockDim.x)
    if (s_hist[t]) atomicAdd(hist + t, (unsigned long long)s_hist[t]);
}

// pass j >= 1 (shift = 56 - 8j): per key under the prefix of slot s (pfx[s] = its top 8j bits, ascending), one count into
// hist[s * 256 + digit j]
static __global__ void __launch_bounds__(kQuantThreads)
nn_quantile_hist_kernel(const unsigned long long *__restrict__ keys, long long n, int shift, const unsigned long long *__restrict__ pfx,
                        int n_slots, unsigned long long *__restrict__ hist) {
  extern __shared__ unsigned int s_hist_dyn[];        // n_slots * 256
  __shared__ unsigned long long s_pfx[kQuantSlots];
  for (int t = threadIdx.x; t < n_slots * kQuantBins; t += kQuantThreads) s_hist_dyn[t] = 0;
  for (int t = threadIdx.x; t < n_slots; t += kQuantThreads) s_pfx[t] = pfx[t];
  __syncthreads();
  const long long stride = (long long)gridDim.x * kQuantThreads;
  for (long long base = (long long)blockIdx.x * kQuantThreads; base < n; base += stride) {
    const long long i = base + threadIdx.x;
    int bin = -1;
    if (i < n) {
      const unsigned long long key = __ldg(keys + i);
      if (key != kQuantOut) {
        const unsigned long long top = key >> (shift + 8);
        int lo = 0, hi = n_slots;          // first slot with prefix >= top
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (s_pfx[mid] < top) lo = mid + 1; else hi = mid;
        }
        if (lo < n_slots && s_pfx[lo] == top) bin = lo * kQuantBins + (int)((key >> shift) & 0xffu);
      }
    }
    quant_count(s_hist_dyn, bin);
  }
  quant_flush(s_hist_dyn, n_slots * kQuantBins, hist);
}

// pass `pass` >= 1 of one population: the n keys, its n_slots prefixes on the device; counts added into hist[slot * 256 + digit]
static inline int quant_hist_launch(me_ctx *ctx, const unsigned long long *keys, long long n, int pass, const unsigned long long *d_pfx,
                                    int n_slots, unsigned long long *hist) {
  const size_t smem = (size_t)n_slots * kQuantBins * sizeof(unsigned int);
  ME_CUDA(ctx, cudaFuncSetAttribute(nn_quantile_hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)(kQuantSlots * kQuantBins * sizeof(unsigned int))));
  int per_sm = 0;
  ME_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, nn_quantile_hist_kernel, kQuantThreads, smem));
  const int grid = (int)std::min<long long>((n + kQuantThreads - 1) / kQuantThreads, (long long)ctx->sm_count * std::max(per_sm, 1));
  nn_quantile_hist_kernel<<<grid, kQuantThreads, smem, ctx->stream>>>(keys, n, 56 - 8 * pass, d_pfx, n_slots, hist);
  ME_LAUNCH_CHECK(ctx);
  return ME_OK;
}

}  // namespace me

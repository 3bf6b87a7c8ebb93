// rng.cuh — the counter-based hash of synth.py: splitmix64 of (seed, index, lane).  Every draw of the library is a pure
// function of those three, so a result that depends on draws is the same on every GPU and equals a numpy statement.
// Lanes in use (one seed may serve all of them):
//   perturb.cu      noise 0-5, density 6, outlier base 7, outlier offsets 8-13
//   globalreg.cu    RANSAC correspondence draws 16, 17, 18
#pragma once
#include <stdint.h>

namespace me {

__host__ __device__ __forceinline__ unsigned long long mix64(unsigned long long z) {     // synth._mix
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// the per-lane key synth.uniform24 derives from the seed (computed once on the host)
static inline unsigned long long lane_key(uint64_t seed, int lane) { return mix64(seed + (unsigned long long)lane * 0xD1B54A32D192ED03ull); }

__device__ __forceinline__ unsigned long long draw(unsigned long long key, long long idx, int lane) {
  return mix64(key ^ ((unsigned long long)idx * 0x2545F4914F6CDD1Dull + (unsigned long long)lane));
}
// synth.uniform24: (h >> 40) * 2^-24 in fp32
__device__ __forceinline__ double uniform24(unsigned long long key, long long idx, int lane) {
  return (double)((float)(draw(key, idx, lane) >> 40) * (1.0f / 16777216.0f));
}
// (h >> 11) * 2^-53 in fp64
__device__ __forceinline__ double uniform53(unsigned long long key, long long idx, int lane) {
  return (double)(draw(key, idx, lane) >> 11) * 0x1p-53;
}

}  // namespace me

// Counter-based random numbers of the device priors (stroke, Omniglot): a draw is a hash of (seed, tag, counters), so a
// batch is a pure function of its seed and the order in which threads draw does not matter.
#pragma once
#include <stdint.h>

namespace pfn {

__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7FEB352Du;
  x ^= x >> 15; x *= 0x846CA68Bu;
  x ^= x >> 16;
  return x;
}
__device__ __forceinline__ uint32_t hash5(uint32_t seed, uint32_t tag, uint32_t a, uint32_t b, uint32_t c) {
  uint32_t h = mix32(seed ^ (tag * 0x9E3779B1u));
  h = mix32(h ^ (a * 0x85EBCA77u));
  h = mix32(h ^ (b * 0xC2B2AE3Du));
  return mix32(h ^ (c * 0x27D4EB2Fu));
}
// U{lo..hi}, both ends included (random.randint)
__device__ __forceinline__ int uniform_int(uint32_t h, int lo, int hi) {
  return lo + static_cast<int>((static_cast<uint64_t>(h) * static_cast<uint32_t>(hi - lo + 1)) >> 32);
}
// U[0, 1) with 53 random bits (random.random)
__device__ __forceinline__ double uniform_double(uint32_t hi, uint32_t lo) {
  return (static_cast<double>(hi >> 5) * 67108864.0 + static_cast<double>(lo >> 6)) * (1.0 / 9007199254740992.0);
}

}  // namespace pfn

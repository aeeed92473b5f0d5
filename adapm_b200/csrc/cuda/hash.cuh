// Counter-based random numbers of the device kernels: a 64-bit finaliser (MurmurHash3's fmix64) applied to a key that
// names the draw, so a draw depends only on what it is for, never on the thread or launch that makes it.
#pragma once
#include <cstdint>

namespace adapm {
namespace cudaops {

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdULL;
  x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL;
  x ^= x >> 33;
  return x;
}

}  // namespace cudaops
}  // namespace adapm

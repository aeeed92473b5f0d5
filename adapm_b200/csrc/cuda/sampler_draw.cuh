// One draw of the device key sampler from a 64-bit hash: shared by the sampler kernel (ops_sampler.cu) and the kernels
// that draw their own negatives inline (ops_doc2vec.cu), so both draw the same key from the same hash.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "ops.h"

namespace adapm {
namespace cudaops {

// kind: 0 = alias table, 1 = uniform over [first, first+n), 2 = log-uniform over [first, first+n); lg = ln(n + 1)
// (log-uniform only). The rules are replayed bit for bit by ops.sample_keys_reference.
static __device__ __forceinline__ Key draw_key(int kind, const float* __restrict__ prob,
                                               const int32_t* __restrict__ alias, int64_t n, double lg, Key first,
                                               Key stride, uint64_t h) {
  uint32_t hi = (uint32_t)(h >> 32), lo = (uint32_t)h;
  if (kind == 0) {
    int64_t i = (int64_t)(((uint64_t)hi * (uint64_t)n) >> 32);
    float u = (float)lo * 2.3283064365386963e-10f;
    int64_t j = (u < __ldg(prob + i)) ? i : (int64_t)__ldg(alias + i);
    return first + j * stride;
  }
  if (kind == 1) return first + (Key)(((uint64_t)hi * (uint64_t)n) >> 32) * stride;
  // log-uniform: floor(exp(u * ln(n + 1))) - 1   (reference bindings.cc:72-76), u = hi / 2^32. In double: float32 u
  // and the fast intrinsics err by about 1e-6 relative, which moves whole keys once n reaches 10^5 to 10^6.
  double u = (double)hi * 0x1p-32;
  int64_t j = (int64_t)exp(u * lg) - 1;
  j = j < 0 ? 0 : (j >= n ? n - 1 : j);
  return first + j * stride;
}

}  // namespace cudaops
}  // namespace adapm

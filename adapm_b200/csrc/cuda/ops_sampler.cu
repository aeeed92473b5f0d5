// Negative / key sampling on the device (SURVEY K11 + K13): alias-table (unigram^0.75 or any
// weights), uniform and log-uniform draws with a counter-based generator, and the "local"
// scheme's rejection against the residency map (reference sampling.h:426-446: redraw until the
// key is resident on this node; never communicates; does not preserve the distribution).
#include <cuda_runtime.h>

#include <cmath>

#include "hash.cuh"
#include "ops.h"
#include "pm_kernels.cuh"
#include "sampler_draw.cuh"

namespace adapm {
namespace cudaops {

namespace {

// Residency probe with plain (L2-cached) loads: a momentarily stale answer only costs one more
// draw or one remote access, so no acquire/system-scope ordering is needed here.
__device__ __forceinline__ bool resident_weak(const Ctx& c, Key k) {
  int32_t s = __ldcg(slot_of(c, c.rank) + k);
  if (s < 0) return false;
  uint32_t st = meta_state(__ldcg(meta_of(c, c.rank) + s));
  return st == S_OWNED || st == S_REPLICA || st == S_INCOMING_REPLICA;
}

__global__ void sample_kernel(const __grid_constant__ Ctx c, int kind, const float* __restrict__ prob,
                              const int32_t* __restrict__ alias, int64_t n_table, double lg, Key first, Key stride,
                              Key* __restrict__ out, int64_t n, uint64_t seed, int local_only, int max_tries,
                              unsigned long long* __restrict__ stats) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned checks = 0, misses = 0;
  if (i < n) {
    Key k = 0;
    int t = 0;
    for (;;) {
      uint64_t h = mix64(seed ^ ((uint64_t)i * 0x9E3779B97F4A7C15ULL + (uint64_t)t * 0xD1B54A32D192ED03ULL));
      k = draw_key(kind, prob, alias, n_table, lg, first, stride, h);
      if (!local_only) break;
      ++checks;
      if (resident_weak(c, k)) break;
      if (++t >= max_tries) { ++misses; break; }  // give up: the row will be fetched over NVLink
    }
    out[i] = k;
  }
  if (stats) {  // one atomic per warp, not per thread (same-address atomics serialise in L2)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      checks += __shfl_xor_sync(0xffffffffu, checks, o);
      misses += __shfl_xor_sync(0xffffffffu, misses, o);
    }
    if ((threadIdx.x & 31) == 0) {
      if (checks) atomicAdd(stats + 0, (unsigned long long)checks);
      if (misses) atomicAdd(stats + 1, (unsigned long long)misses);
    }
  }
}

}  // namespace

void sample_keys(CudaBackend& be, cudaStream_t stream, int kind, const float* prob, const int32_t* alias,
                 int64_t n_table, Key first, Key stride, Key* out, int64_t n, uint64_t seed, bool local_only,
                 int max_tries, unsigned long long* stats) {
  // the bucket is (hi * n_table) >> 32 in 64 bits, and an alias index is an int32
  ADAPM_CHECK(n_table >= 1 && n_table < (kind == 0 ? ((int64_t)1 << 31) : ((int64_t)1 << 32)),
              "sample_keys: " << n_table << " keys, need 1 <= keys < " << (kind == 0 ? "2^31" : "2^32"));
  if (n == 0) return;
  be.track_stream(stream);
  int blocks = (int)((n + 255) / 256);
  sample_kernel<<<blocks, 256, 0, stream>>>(be.ctx(), kind, prob, alias, n_table, std::log((double)(n_table + 1)),
                                            first, stride, out, n, seed, local_only ? 1 : 0, max_tries, stats);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

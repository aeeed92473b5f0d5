// WarpGroup: the device-side "group of lanes" for protocol.h (one 32-wide warp per key/slot).
#pragma once
#include <sstream>

#include "../adapm/log.h"
#include "../adapm/protocol.h"

namespace adapm {

struct WarpGroup {
  __device__ __forceinline__ int lane() const { return (int)(threadIdx.x & 31u); }
  __device__ __forceinline__ int size() const { return 32; }
  __device__ __forceinline__ bool any(bool p) const { return __any_sync(0xffffffffu, p); }
  __device__ __forceinline__ void sync() const { __syncwarp(); }
  __device__ __forceinline__ uint32_t bcast(uint32_t v) const { return __shfl_sync(0xffffffffu, v, 0); }
  __device__ __forceinline__ int32_t bcast(int32_t v) const { return __shfl_sync(0xffffffffu, v, 0); }
  __device__ __forceinline__ uint64_t bcast(uint64_t v) const {
    return (uint64_t)__shfl_sync(0xffffffffu, (unsigned long long)v, 0);
  }
  __device__ __forceinline__ uint32_t bcast_from(uint32_t v, int src) const { return __shfl_sync(0xffffffffu, v, src); }
  __device__ __forceinline__ double sum(double v) const {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
  }
};

// LaneGroup: one thread on its own (the per-row gather threads of the GEMM kernels).
struct LaneGroup {
  __device__ __forceinline__ int lane() const { return 0; }
  __device__ __forceinline__ int size() const { return 1; }
  __device__ __forceinline__ bool any(bool p) const { return p; }
  __device__ __forceinline__ void sync() const {}
  __device__ __forceinline__ uint32_t bcast(uint32_t v) const { return v; }
  __device__ __forceinline__ int32_t bcast(int32_t v) const { return v; }
  __device__ __forceinline__ uint64_t bcast(uint64_t v) const { return v; }
  __device__ __forceinline__ uint32_t bcast_from(uint32_t v, int) const { return v; }
  __device__ __forceinline__ double sum(double v) const { return v; }
};

#define ADAPM_CUDA_CHECK(expr)                                                                 \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) {                                                                    \
      std::ostringstream _os;                                                                   \
      _os << "[adapm] CUDA error " << cudaGetErrorName(_e) << " (" << cudaGetErrorString(_e)    \
          << ") at " << __FILE__ << ":" << __LINE__ << ": " #expr;                              \
      throw ::adapm::Error(_os.str());                                                          \
    }                                                                                           \
  } while (0)

// Raises Kernel's dynamic shared memory limit to `bytes` on the first call in the process (a function-local static,
// initialised once and thread-safely); a failure throws here instead of surfacing as a later launch error.
template <auto Kernel>
inline void set_max_dynamic_smem(int bytes) {
  static const bool done = [bytes] {
    ADAPM_CUDA_CHECK(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    return true;
  }();
  (void)done;
}

}  // namespace adapm

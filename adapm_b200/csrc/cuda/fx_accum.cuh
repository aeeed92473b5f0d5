// Deterministic accumulation of the fused training steps on one GPU (ComplEx, RESCAL, MF). The SGNS step groups its
// contributions by key instead (ops_sgns_tma.cu) and shares only FxScratch's key map, id list, counters and loss word.
//
// A deterministic step adds its updates as 64-bit fixed-point integers into an accumulator region per key touched by
// the step instead of into the store rows, so every call reads only start-of-step values and the sums do not depend on
// the order in which warps add them; fx::apply then adds each region's sum to the key's store row (one writer per row)
// and clears the region. The three passes of a step:
//   fx::begin    sizes the scratch by the step and gives every key of the step a region of its own row length
//                (index kernel: offset = atomicAdd on a running total, in units of the step's shortest row);
//   the step     fx::add / fx::add4 into the regions (fx::region finds a key's region);
//   fx::apply    one warp per region: row += sum / scale, region = 0; the step's loss is reduced in a fixed order.
// Which region a key gets may vary from run to run; what is summed into it does not.
//
// Rows are [value half (h) | AdaGrad half (h)]. Within each half of a region, element e sits at fx::pos(e, h): for
// h % 4 == 0 element 4j + c sits at c * h/4 + j, so that one warp-wide atomic over the lanes' float4 index j covers
// contiguous memory; other h are stored in element order. fx::elem is the inverse; both sides use these two.
#pragma once
#include <cuda_runtime.h>

#include "cuda_backend.h"

namespace adapm {
namespace fx {

__host__ __device__ __forceinline__ int pos(int e, int h) { return (h & 3) ? e : (e & 3) * (h >> 2) + (e >> 2); }
__host__ __device__ __forceinline__ int elem(int i, int h) {
  if (h & 3) return i;
  const int n = h >> 2;
  return 4 * (i % n) + i / n;
}

__device__ __forceinline__ void add(long long* a, float v, float scale) {
  atomicAdd(reinterpret_cast<unsigned long long*>(a), (unsigned long long)__float2ll_rn(v * scale));
}
// element e of a half of length h
__device__ __forceinline__ void add1(long long* half, int e, int h, float v, float scale) { add(half + pos(e, h), v, scale); }
// elements 4j .. 4j+3 of a half of nvec float4 (h % 4 == 0)
__device__ __forceinline__ void add4(long long* half, int j, int nvec, float4 v, float scale) {
  add(half + j, v.x, scale);
  add(half + nvec + j, v.y, scale);
  add(half + 2 * nvec + j, v.z, scale);
  add(half + 3 * nvec + j, v.w, scale);
}
// the accumulator region of `key` (unit = the step's unit row length in values)
__device__ __forceinline__ long long* region(long long* acc, const int* cidx, Key key, int unit) {
  return acc + (size_t)__ldg(cidx + key) * unit;
}

// One group of update sources of a step: n keys whose rows are `units` x the step's unit row length.
struct Source {
  const Key* keys;
  long n;
  int units;
};

// Sizes the backend's scratch for a step over `src` (at most 4 sources; unit = row length in values of a 1-unit key)
// and launches the index kernel on `stream`. n_calls > 0 also provides a per-call loss buffer (fx::apply reduces it).
CudaBackend::FxScratch& begin(CudaBackend& be, cudaStream_t stream, const Source* src, int n_src, int unit,
                              long n_calls = 0);
// Adds every region to its store row and clears it. Values are divided by scale_val, AdaGrad sums by scale_ada. The
// loss: fx_loss_scale > 0 moves the fixed-point sum in FxScratch::loss (divided by the scale) into loss_out; otherwise
// the n_calls per-call losses of FxScratch::call_loss are summed in a fixed order (float64) into loss_out.
void apply(CudaBackend& be, cudaStream_t stream, int unit, float scale_val, float scale_ada, float fx_loss_scale,
           long n_calls, float* loss_out);

}  // namespace fx
}  // namespace adapm

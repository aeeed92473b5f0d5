// Device helpers of the warp-per-triple KGE steps (ops_transe.cu, ops_rotate.cu) and the BPR step of matrix
// factorisation (ops_bpr.cu): float4 arithmetic, row loads into a lane's float4 registers and the three-mode AdaGrad push
// (in place, onto a staged copy, into a fixed-point region).
#pragma once
#include <cuda_runtime.h>

#include "fx_accum.cuh"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {
namespace kge {

__device__ __forceinline__ float4 f4(float v) { return make_float4(v, v, v, v); }
__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 sub4(float4 a, float4 b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
__device__ __forceinline__ float4 mul4(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float dot4(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
__device__ __forceinline__ float4 ld4(const float* p, int j) { return *reinterpret_cast<const float4*>(p + 4 * j); }
__device__ __forceinline__ void st4(float* p, int j, float4 v) { *reinterpret_cast<float4*>(p + 4 * j) = v; }

// float4 lane, lane + 32, ... of a row (zeros past nv float4)
template <int VPL>
__device__ __forceinline__ void load_row(const float* row, int nv, int lane, float4 (&v)[VPL]) {
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int j = lane + 32 * i;
    v[i] = j < nv ? dev::ld_row4(row + 4 * j) : f4(0.f);
  }
}

// AdaGrad push of gradient g onto float4 j of a row [emb (d) | acc (d)]: in place (REDs), onto a staged copy (the
// generic path pushes it afterwards) or into the key's fixed-point region (values scaled by fx_val, AdaGrad increments
// clamped to fx_ada_max and scaled by fx_ada).
template <bool FX>
__device__ __forceinline__ void push4(float* row, int d, int j, float4 g, bool staged, long long* region, int nv,
                                      float eta, float fx_val, float fx_ada, float fx_ada_max) {
  const float4 a = dev::ld_row4(row + d + 4 * j);
  const float4 ua = make_float4(g.x * g.x, g.y * g.y, g.z * g.z, g.w * g.w);
  const float4 ue = make_float4(g.x != 0.f ? -eta * g.x * rsqrtf(a.x + ua.x) : 0.f,
                                g.y != 0.f ? -eta * g.y * rsqrtf(a.y + ua.y) : 0.f,
                                g.z != 0.f ? -eta * g.z * rsqrtf(a.z + ua.z) : 0.f,
                                g.w != 0.f ? -eta * g.w * rsqrtf(a.w + ua.w) : 0.f);
  if (FX) {
    fx::add4(region, j, nv, ue, fx_val);
    fx::add4(region + d, j, nv,
             make_float4(fminf(ua.x, fx_ada_max), fminf(ua.y, fx_ada_max), fminf(ua.z, fx_ada_max),
                         fminf(ua.w, fx_ada_max)),
             fx_ada);
  } else if (staged) {
    *reinterpret_cast<float4*>(row + 4 * j) = ue;
    *reinterpret_cast<float4*>(row + d + 4 * j) = ua;
  } else {
    dev::red_row4(row + 4 * j, ue);
    dev::red_row4(row + d + 4 * j, ua);
  }
}

}  // namespace kge
}  // namespace cudaops
}  // namespace adapm

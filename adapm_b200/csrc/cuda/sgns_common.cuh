// Shared pieces of the two word2vec SGNS step kernels (ops_sgns.cu: register-resident rows, ops_sgns_tma.cu: TMA ring).
#pragma once
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {
namespace sgns {

constexpr float kMaxExp = 6.0f;   // MAX_EXP of the reference (apps/word2vec.cc): gradients saturate outside [-6, 6]

// ---- slow path (key in a transitional protocol state: INCOMING, FINALIZING, ...). Rare, so it is
// kept out of line and works through shared memory with the generic protocol functions.
//   stage: 2*d floats scratch; e0s: center embedding (d); g0s: center gradient accumulator (d)
// SKIP_SATURATED = false: the gradient saturates at |f| > 6 (negative sampling). true: a target with |f| >= 6 gets no
// update and adds nothing to g0s (word2vec.c's hierarchical softmax); its loss is counted either way.
template <bool SKIP_SATURATED = false>
static __device__ __noinline__ float slow_target(const Ctx& c, Key tkey, float label, float alpha, int d, float* stage,
                                          const float* e0s, float* g0s, bool* applied) {
  WarpGroup g;
  const int lane = threadIdx.x & 31;
  *applied = false;
  if (!pull_key<float>(c, g, tkey, stage, false, nullptr)) return 0.f;
  __syncwarp();
  float f = 0.f;
  for (int j = lane; j < d; j += 32) f += e0s[j] * stage[j];
  f = dev::warp_sum(f);
  float gs;
  if (SKIP_SATURATED) {
    if (fabsf(f) >= kMaxExp) return __logf(1.f + __expf(-fminf(fmaxf(label > 0.5f ? f : -f, -kMaxExp), kMaxExp)));
    gs = label - 1.f / (1.f + __expf(-f));
  } else if (f > kMaxExp) gs = label - 1.f;
  else if (f < -kMaxExp) gs = label;
  else gs = label - 1.f / (1.f + __expf(-f));
  for (int j = lane; j < d; j += 32) {
    float e1 = stage[j], a1 = stage[d + j];
    g0s[j] += gs * e1;
    float gr = gs * e0s[j];
    float ua = gr * gr;
    stage[j] = alpha * gr * rsqrtf(a1 + ua);
    stage[d + j] = ua;
  }
  __syncwarp();
  *applied = push_key<float>(c, g, tkey, stage, nullptr);
  __syncwarp();
  float z = label > 0.5f ? f : -f;
  z = fminf(fmaxf(z, -kMaxExp), kMaxExp);
  return __logf(1.f + __expf(-z));
}

}  // namespace sgns
}  // namespace cudaops
}  // namespace adapm

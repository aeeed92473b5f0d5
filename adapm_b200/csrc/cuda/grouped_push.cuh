// Pieces of the grouped, one-push-per-key AdaGrad update over rows [values (E) | AdaGrad accumulator (E)] that the
// embedding-bag backward (ops_embbag.cu) and the FFM step (ops_ffm.cu) share: statistics, the slow path of keys in a
// transitional state, and the push of one key's summed gradient by a group of lanes.
#pragma once
#include <cuda_runtime.h>

#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {
namespace grouped {

// stats: [0] local rows, [1] peer rows, [2] rows that took the slow path, [3] rows updated, [4] rows that could not be
// resolved (read as zeros / update dropped). The frequent ones are counted per lane and added once per warp; the rare
// ones (slow path) go straight to `stats`, so that they hold no register across the kernel.
struct Counts {
  unsigned local = 0, remote = 0, upd = 0;
};

__device__ __forceinline__ void count_rare(unsigned long long* stats, bool resolved) {
  if (!stats) return;
  atomicAdd(stats + 2, 1ull);
  if (!resolved) atomicAdd(stats + 4, 1ull);
}

__device__ __forceinline__ void flush_counts(Counts n, unsigned long long* stats) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    n.local += __shfl_xor_sync(0xffffffffu, n.local, o); n.remote += __shfl_xor_sync(0xffffffffu, n.remote, o);
    n.upd += __shfl_xor_sync(0xffffffffu, n.upd, o);
  }
  if ((threadIdx.x & 31) == 0 && stats) {
    if (n.local) atomicAdd(stats + 0, (unsigned long long)n.local);
    if (n.remote) atomicAdd(stats + 1, (unsigned long long)n.remote);
    if (n.upd) atomicAdd(stats + 3, (unsigned long long)n.upd);
  }
}

// Keys in a transitional state (a relocation in flight): dev::gather_locate / dev::gather_reread, and locate_push, with
// a one-lane group, inlined. (Out-of-line calls would make these kernels save their accumulators around every call
// site: local-memory spills.)
__device__ __forceinline__ dev::GatherRow locate_row(const Ctx& c, Key key) {
  LaneGroup g;
  const PullLoc<float> l = locate_pull<float>(c, g, key, false);
  dev::GatherRow r;
  r.row = l.kind == LOC_FAIL ? nullptr : l.row;
  r.base = l.kind == LOC_SUM3 ? l.base : nullptr;
  r.row2 = l.row2; r.meta_ptr = l.meta_ptr; r.meta_val = l.meta_val; r.local = l.local;
  return r;
}

__device__ __forceinline__ bool reread_row(const Ctx& c, Key key, dev::GatherRow& r) {
  if (!r.base) return false;
  mem::fence();
  if (mem::ld_acquire(r.meta_ptr) == r.meta_val) return false;
  r = locate_row(c, key);
  return true;
}

__device__ __forceinline__ dev::Target push_locate(const Ctx& c, Key key) {
  LaneGroup g;
  const PushLoc<float> l = locate_push<float>(c, g, key);
  dev::Target t;
  t.row = l.row; t.version = l.version; t.flag = l.flag;
  return t;
}

// dev::resolve_fast, counting into `n` (through locals: a counter whose address escapes ends up in local memory)
__device__ __forceinline__ dev::Target resolve(const Ctx& c, Key key, Counts& n) {
  unsigned nl = 0, nr = 0;
  const dev::Target t = dev::resolve_fast(c, key, class_of_key(c, key), &nl, &nr);
  n.local += nl; n.remote += nr;
  return t;
}

__device__ __forceinline__ unsigned long long shfl_ptr(unsigned mask, const void* p, int src, int width) {
  return __shfl_sync(mask, (unsigned long long)p, src, width);
}

// one element: update -lr g / sqrt(acc + g^2) (0 where g == 0, not 0/0 at acc = 0) and accumulator increment g^2.
// rsqrtf, as the other fused AdaGrad kernels: the IEEE division and square root have out-of-line slow paths, and
// their call sites would make the kernel save its accumulators to local memory.
__device__ __forceinline__ void adagrad(float g, float acc, float lr, float& upd, float& sq) {
  sq = g * g;
  upd = g == 0.f ? 0.f : -lr * g * rsqrtf(acc + sq);
}

// The update of one key by one group of G lanes (lane `sub` owns float4 j = sub + G * v): resolve the row (the group's
// lane 0), read the accumulator, push [-lr G / sqrt(acc + G^2) | G^2]. `mask`: the group's lanes.
template <int VPL>
__device__ __forceinline__ void push_update(const Ctx& c, Key key, const float4 (&g)[VPL], int E, int sub, int G,
                                            unsigned mask, float lr, Counts& n,
                                            unsigned long long* stats) {
  const int E4 = E >> 2;
  dev::Target t;
  t.row = nullptr; t.version = nullptr; t.flag = nullptr;
  if (sub == 0) t = resolve(c, key, n);
  dev::GatherRow src = {nullptr, nullptr, nullptr, nullptr, 0u, false};
  src.row = (const float*)__shfl_sync(mask, (unsigned long long)t.row, 0, G);
  float* dst = const_cast<float*>(src.row);
  if (!src.row) {                        // transitional slot: locate the push target and the accumulator's source
    if (sub == 0) {
      t = push_locate(c, key);
      src = locate_row(c, key);
      count_rare(stats, t.row && src.row);
      if (t.row && src.row) { if (src.local) ++n.local; else ++n.remote; }
    }
    dst = (float*)shfl_ptr(mask, t.row, 0, G);
    src.row = (const float*)shfl_ptr(mask, src.row, 0, G);
    src.base = (const float*)shfl_ptr(mask, src.base, 0, G);
    src.row2 = (const float*)shfl_ptr(mask, src.row2, 0, G);
    src.meta_ptr = (const uint32_t*)shfl_ptr(mask, src.meta_ptr, 0, G);
    src.meta_val = __shfl_sync(mask, src.meta_val, 0, G);
    if (!dst || !src.row) return;
  }
  float4 a[VPL];
  do {
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int j = sub + G * v;
      a[v] = j < E4 ? dev::ld_gather4(src, E + 4 * j) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  } while (reread_row(c, key, src));
#pragma unroll
  for (int v = 0; v < VPL; ++v) {
    const int j = sub + G * v;
    if (j < E4) {
      float4 u, q;
      adagrad(g[v].x, a[v].x, lr, u.x, q.x); adagrad(g[v].y, a[v].y, lr, u.y, q.y);
      adagrad(g[v].z, a[v].z, lr, u.z, q.z); adagrad(g[v].w, a[v].w, lr, u.w, q.w);
      dev::red_row4(dst + 4 * j, u);
      dev::red_row4(dst + E + 4 * j, q);
    }
  }
  if (sub == 0) { dev::mark_pushed(t); ++n.upd; }
}

__device__ __forceinline__ unsigned group_mask(int lane, int log_g) {
  const int G = 1 << log_g;
  return G == 32 ? 0xffffffffu : ((1u << G) - 1u) << (lane & ~(G - 1));
}

// ---- host side
inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

// the significant bits of a key, for the radix sort
inline int key_bits(int64_t num_keys) {
  int b = 1;
  while (b < 63 && ((int64_t)1 << b) < num_keys) ++b;
  return b;
}

// lanes per group (log2, the smallest power of two >= E / 4, at most 32) and float4 per lane
inline void lane_shape(int E, int* log_g, int* vpl) {
  const int E4 = E / 4;
  int lg = 0;
  while ((1 << lg) < E4 && lg < 5) ++lg;
  *log_g = lg;
  *vpl = (E4 + 31) / 32;
}

}  // namespace grouped
}  // namespace cudaops
}  // namespace adapm

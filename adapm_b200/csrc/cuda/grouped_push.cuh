// The grouped, one-push-per-key AdaGrad update over rows [values (E) | AdaGrad accumulator (E)] that the
// embedding-bag backward (ops_embbag.cu) and the FFM step (ops_ffm.cu) share. Given the step's keys and, for every
// position, what the occurrence there adds to its key's gradient (the op's source, below), for every distinct key k
//   G_k = sum of the occurrences of k in position order (in fp32), then whatever the source applies to the sum,
//   push [-lr G / sqrt(acc + G^2) | G^2] to the owner's row (an element with G == 0 gets 0, not 0/0),
// in three launches (sort_and_push):
//   1. sort:   cub radix sort of (key, position) over the significant key bits; stable, so every key's occurrences
//              stay in position order
//   2. tile:   the sorted occurrences are cut into tiles of kTile; one lane group per tile sums each key's run in fp32
//              in position order. A run that lies inside the tile is pushed right away; a run that crosses a tile
//              boundary leaves one partial sum per tile it touches (tile_pass)
//   3. finish: one warp per run that crosses a boundary adds its partials in tile order and pushes (finish_pass).
// Every distinct key gets one push with one fixed sum: on one GPU two runs of the same step give bit-identical rows.
//
// A source (a struct passed by value to the op's kernels) provides
//   Item load(int pos)                                   what a lane reads for the occurrence at position `pos`
//   Item share(Item, unsigned mask, int src, int G)      lane `src`'s item, to every lane of the group
//   const float4* row(Item, int E)                       the occurrence's E values, read with __ldg
//   void add(float4& acc, float4 x, Item)                the occurrence's 4 values x added to the sum
//   template <int VPL> void before_push(float4 (&acc)[VPL])   applied to a key's sum before it is pushed
#pragma once
#include <cuda_runtime.h>

#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {
namespace grouped {

constexpr int kThreads = 256;  // threads per CTA of the tile and finish passes
constexpr int kTile = 32;      // sorted occurrences per lane group in the tile pass

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

// 2. one group of G = 2^log_g lanes per tile of kTile sorted occurrences (sk: keys, spos: their positions).
// part[t][0]: the partial of the run that was open at the tile's start (it began in an earlier tile); part[t][1]: the
// partial of a run that begins in the tile and crosses its end.
template <int VPL, class Src>
__device__ __forceinline__ void tile_pass(const Ctx& c, const Key* sk, const int* spos, const Src& src, int nnz, int E,
                                          int log_g, float lr, float* part, unsigned long long* stats) {
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int G = 1 << log_g;
  const int sub = lane & (G - 1);
  const unsigned mask = group_mask(lane, log_g);
  const int E4 = E >> 2;
  const int n_tiles = (nnz + kTile - 1) / kTile;
  const int groups_per_warp = 32 >> log_g;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  Counts n;
  for (int wt = warp * groups_per_warp; wt < n_tiles; wt += nwarps * groups_per_warp) {
    const int t = wt + (lane >> log_g);
    if (t >= n_tiles) continue;          // (group-uniform; the shuffles below only involve the group)
    const int lo = t * kTile, hi = min(nnz, lo + kTile);
    Key cur = sk[lo];
    bool open_before = lo > 0 && sk[lo - 1] == cur;
    float4 acc[VPL];
#pragma unroll
    for (int v = 0; v < VPL; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int p0 = lo; p0 <= hi; p0 += G) {
      // lane `sub` loads occurrence p0 + sub; position hi is the end of the last run
      Key kk = -1;
      typename Src::Item it{};
      if (p0 + sub < hi) { kk = sk[p0 + sub]; it = src.load(spos[p0 + sub]); }
      const int cnt = min(G, hi + 1 - p0);
      for (int u = 0; u < cnt; ++u) {
        const Key k = (Key)__shfl_sync(mask, (long long)kk, u, G);
        const typename Src::Item iu = src.share(it, mask, u, G);
        if (k != cur) {                  // the run of `cur` ends here (k == -1: at the tile's end)
          const bool crosses = k == -1 && hi < nnz && sk[hi] == cur;
          if (open_before || crosses) {
            float* dst = part + ((size_t)t * 2 + (open_before ? 0 : 1)) * E;
#pragma unroll
            for (int v = 0; v < VPL; ++v) {
              const int j = sub + G * v;
              if (j < E4) reinterpret_cast<float4*>(dst)[j] = acc[v];
            }
          } else {
            src.template before_push<VPL>(acc);
            push_update<VPL>(c, cur, acc, E, sub, G, mask, lr, n, stats);
          }
          if (k == -1) break;
          cur = k;
          open_before = false;
#pragma unroll
          for (int v = 0; v < VPL; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        const float4* x = src.row(iu, E);
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int j = sub + G * v;
          if (j < E4) src.add(acc[v], __ldg(x + j), iu);
        }
      }
    }
  }
  __syncwarp();
  flush_counts(n, stats);
  dev::cta_exit(c);
}

// 3. one warp per tile boundary q = i * kTile: if a run crosses q and does not cross q - kTile, the warp owns it: its
// partials part[i - 1][1], part[i][0], part[i + 1][0], ... are added in tile order, and the key is pushed.
template <int VPL, class Src>
__device__ __forceinline__ void finish_pass(const Ctx& c, const Key* sk, int nnz, int E, float lr, const float* part,
                                            unsigned long long* stats, const Src& src) {
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int E4 = E >> 2;
  const int n_tiles = (nnz + kTile - 1) / kTile;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  Counts n;
  for (int i = 1 + warp; i < n_tiles; i += nwarps) {
    const int q = i * kTile;
    const Key k = sk[q];
    if (sk[q - 1] != k || (q - kTile - 1 >= 0 && sk[q - kTile - 1] == k)) continue;   // (warp-uniform)
    float4 acc[VPL];
    const float* p0 = part + ((size_t)(i - 1) * 2 + 1) * E;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int j = lane + 32 * v;
      acc[v] = j < E4 ? reinterpret_cast<const float4*>(p0)[j] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int t = i;; ++t) {
      const float* pt = part + (size_t)t * 2 * E;
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int j = lane + 32 * v;
        if (j < E4) {
          const float4 x = reinterpret_cast<const float4*>(pt)[j];
          acc[v].x += x.x; acc[v].y += x.y; acc[v].z += x.z; acc[v].w += x.w;
        }
      }
      const int e = (t + 1) * kTile;
      if (e >= nnz || sk[e] != k) break;
    }
    src.template before_push<VPL>(acc);
    push_update<VPL>(c, k, acc, E, lane, 32, 0xffffffffu, lr, n, stats);
  }
  flush_counts(n, stats);
  dev::cta_exit(c);
}

// ---- host side
inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

// the significant bits of a key, for the radix sort
inline int key_bits(int64_t num_keys) {
  int b = 1;
  while (b < 63 && ((int64_t)1 << b) < num_keys) ++b;
  return b;
}

// Slices of 256-byte aligned arrays cut from a workspace in order; base null: only the size is counted.
struct Carve {
  char* base;
  size_t off = 0;
  template <class T>
  T* take(size_t n) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += align_up(n * sizeof(T));
    return p;
  }
};

// The arrays of the sort and the passes: sorted keys | positions (in, out) | tile partials [n_tiles][2][E] | sort
// scratch. An op carves its own arrays after them.
struct PushWorkspace {
  Key* sk; int* pos_in; int* pos_out; float* part; void* sort_tmp; size_t sort_bytes;
};
PushWorkspace carve_push(Carve& a, int64_t nnz, int E);

// the stable radix sort of (keys, w.pos_in) into (w.sk, w.pos_out) over the significant bits of the store's keys
void sort_pairs(CudaBackend& be, cudaStream_t stream, const Key* keys, const PushWorkspace& w, int nnz);

// The backward after the op has written each occurrence's position to w.pos_in: the sort, then Tile (a tile_pass) and
// Finish (a finish_pass) over src, on the instantiation for E's lane shape (log_g from lane_shape). Three launches,
// the sort counted as one (cub runs one or more kernels, depending on nnz and the bits).
template <auto Tile, auto Finish, class Src>
void sort_and_push(CudaBackend& be, cudaStream_t stream, const Key* keys, const PushWorkspace& w, const Src& src,
                   int nnz, int E, int log_g, float lr, unsigned long long* stats) {
  sort_pairs(be, stream, keys, w, nnz);
  ADAPM_COUNT_LAUNCH();
  const int n_tiles = (nnz + kTile - 1) / kTile;
  const int tiles_per_block = (kThreads / 32) << (5 - log_g);
  const int tile_blocks = std::max(1, std::min((n_tiles + tiles_per_block - 1) / tiles_per_block, be.num_sms() * 16));
  const int fin_blocks = std::max(1, std::min((n_tiles + kThreads / 32 - 1) / (kThreads / 32), be.num_sms() * 8));
  Tile<<<tile_blocks, kThreads, 0, stream>>>(be.ctx(), w.sk, w.pos_out, src, nnz, E, log_g, lr, w.part, stats);
  ADAPM_COUNT_LAUNCH();
  Finish<<<fin_blocks, kThreads, 0, stream>>>(be.ctx(), w.sk, nnz, E, lr, w.part, stats, src);
  ADAPM_COUNT_LAUNCH();
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

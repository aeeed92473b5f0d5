// Multi-hot embedding bags on the parameter store for sm_90a: pooled gather (forward) and grouped AdaGrad push
// (backward) over rows [embedding (E) | AdaGrad accumulator (E)], read and updated in local HBM / NVLink peers.
//
// Inputs are CSR bags: keys[nnz], offsets[nbags + 1] (offsets[0] = 0, offsets[nbags] = nnz), optional weights[nnz].
//
// Forward (one launch): out[b] = sum_{i in bag b} w_i * row(keys[i])[0:E], divided by the bag length for mean; an empty
// bag gives zeros. Each bag is summed in fp32 in key order by one group of G = 2^ceil(log2(E/4)) lanes (capped at 32;
// a lane owns float4 j = sub + G * v), so the result does not depend on the grid.
//
// Backward (four launches): for every distinct key k
//   G_k = grad_scale * sum_{occurrences i of k} c_i * grad_out[bag(i)],   c_i = w_i (sum) | 1 / len (mean) | 1
//   push [-lr * G / sqrt(acc + G^2) | G^2] to the owner's row (an element with G == 0 gets 0, not 0/0)
//   1. prep:   position i -> (bag(i), c_i)
//   2.-4.      the sort, tile and finish passes of grouped_push.cuh, which the FFM step shares, over BagSource.
// Every distinct key gets one push with one fixed sum: on one GPU two runs of the same step give bit-identical rows.
#include <cuda_runtime.h>

#include "grouped_push.cuh"
#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {

namespace {

using namespace grouped;

// ------------------------------------------------------------------------------------------------ forward
// One group of G lanes per bag. The group resolves G keys at a time (lane `sub` resolves key base + sub) and then adds
// the G rows in key order; the loop bounds are warp-uniform (the longest bag of the warp), so the group shuffles are
// executed by the whole warp.
template <int VPL>
__global__ void __launch_bounds__(kThreads, 2)
embbag_fwd_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ keys, const int64_t* __restrict__ offsets,
                  const float* __restrict__ weights, int nbags, int E, int log_g, bool mean, float* __restrict__ out,
                  unsigned long long* __restrict__ stats) {
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int G = 1 << log_g;
  const int sub = lane & (G - 1);
  const int E4 = E >> 2;
  const int bags_per_warp = 32 >> log_g;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  Counts n;
  for (int wb = warp * bags_per_warp; wb < nbags; wb += nwarps * bags_per_warp) {
    const int b = wb + (lane >> log_g);
    int64_t start = 0;
    int len = 0;
    if (b < nbags) { start = offsets[b]; len = (int)(offsets[b + 1] - start); }
    const int maxlen = __reduce_max_sync(0xffffffffu, (unsigned)len);
    float4 acc[VPL];
#pragma unroll
    for (int v = 0; v < VPL; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int base = 0; base < maxlen; base += G) {
      // lane `sub` resolves key base + sub of its bag
      const float* rp = nullptr;
      int slow = 0;
      float w = 1.f;
      if (base + sub < len) {
        const Key key = keys[start + base + sub];
        if (weights) w = weights[start + base + sub];
        rp = resolve(c, key, n).row;
        if (!rp) {                              // transitional slot (relocation in flight)
          const dev::GatherRow r = locate_row(c, key);
          count_rare(stats, r.row != nullptr);
          if (r.row && r.local) ++n.local; else if (r.row) ++n.remote;
          slow = 1;
        }
      }
      const int cnt = min(G, maxlen - base);
      for (int t = 0; t < cnt; ++t) {
        const float* p = (const float*)shfl_ptr(0xffffffffu, rp, t, G);
        const int sl = __shfl_sync(0xffffffffu, slow, t, G);
        const float wt = __shfl_sync(0xffffffffu, w, t, G);
        if (base + t >= len) continue;
        float4 x[VPL];
        if (!sl) {
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            const int j = sub + G * v;
            x[v] = j < E4 ? dev::ld_row4(p + 4 * j) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
        } else {                                // every lane of the group locates the row itself (rare)
          const Key key = keys[start + base + t];
          dev::GatherRow r = locate_row(c, key);
          do {
#pragma unroll
            for (int v = 0; v < VPL; ++v) {
              const int j = sub + G * v;
              x[v] = (r.row && j < E4) ? dev::ld_gather4(r, 4 * j) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
          } while (reread_row(c, key, r));
        }
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          if (weights) {
            acc[v].x = fmaf(wt, x[v].x, acc[v].x); acc[v].y = fmaf(wt, x[v].y, acc[v].y);
            acc[v].z = fmaf(wt, x[v].z, acc[v].z); acc[v].w = fmaf(wt, x[v].w, acc[v].w);
          } else {
            acc[v].x += x[v].x; acc[v].y += x[v].y; acc[v].z += x[v].z; acc[v].w += x[v].w;
          }
        }
      }
    }
    if (b < nbags) {
      const float inv = mean && len > 0 ? __frcp_rn((float)len) : 1.f;
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int j = sub + G * v;
        if (j < E4) {
          float4 o = acc[v];
          if (mean) { o.x *= inv; o.y *= inv; o.z *= inv; o.w *= inv; }
          reinterpret_cast<float4*>(out + (size_t)b * E)[j] = o;
        }
      }
    }
  }
  flush_counts(n, stats);
  dev::cta_exit(c);
}

// ------------------------------------------------------------------------------------------------ backward
// 1. position i -> its bag and its coefficient c_i
__global__ void __launch_bounds__(kThreads, 2)
embbag_prep_kernel(const int64_t* __restrict__ offsets, const float* __restrict__ weights, int nbags, int nnz, bool mean,
                   int* __restrict__ pos, int* __restrict__ bag_of, float* __restrict__ coef) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nnz; i += gridDim.x * blockDim.x) {
    int lo = 0, hi = nbags;            // the last bag b with offsets[b] <= i (empty bags before it are skipped)
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (offsets[mid] <= i) lo = mid; else hi = mid;
    }
    pos[i] = i;
    bag_of[i] = lo;
    coef[i] = weights ? weights[i] : mean ? __frcp_rn((float)(offsets[lo + 1] - offsets[lo])) : 1.f;
  }
}

// 3. and 4.: the passes of grouped_push.cuh over BagSource, which adds c_i * grad_out[bag(i)] (fmaf) for the
// occurrence at position i and scales each key's sum by grad_scale before the push.
struct BagSource {
  const int* bag_of;
  const float* coef;
  const float* grad;
  float grad_scale;
  struct Item { int bag; float coef; };
  // __ldg: a struct member is not a __restrict__ parameter, so the compiler would not use the read-only path itself
  __device__ __forceinline__ Item load(int pos) const { return {__ldg(bag_of + pos), __ldg(coef + pos)}; }
  __device__ __forceinline__ Item share(const Item& it, unsigned mask, int src, int G) const {
    return {__shfl_sync(mask, it.bag, src, G), __shfl_sync(mask, it.coef, src, G)};
  }
  __device__ __forceinline__ const float4* row(const Item& it, int E) const {
    return reinterpret_cast<const float4*>(grad + (size_t)it.bag * E);
  }
  __device__ __forceinline__ void add(float4& a, const float4& x, const Item& it) const {
    a.x = fmaf(it.coef, x.x, a.x); a.y = fmaf(it.coef, x.y, a.y);
    a.z = fmaf(it.coef, x.z, a.z); a.w = fmaf(it.coef, x.w, a.w);
  }
  template <int VPL>
  __device__ __forceinline__ void before_push(float4 (&acc)[VPL]) const {
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      acc[v].x *= grad_scale; acc[v].y *= grad_scale; acc[v].z *= grad_scale; acc[v].w *= grad_scale;
    }
  }
};

template <int VPL>
__global__ void __launch_bounds__(kThreads, 2)
embbag_grad_tile_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ sk, const int* __restrict__ spos,
                        const BagSource src, int nnz, int E, int log_g, float lr,
                        float* __restrict__ part, unsigned long long* __restrict__ stats) {
  tile_pass<VPL>(c, sk, spos, src, nnz, E, log_g, lr, part, stats);
}

template <int VPL>
__global__ void __launch_bounds__(kThreads, 2)
embbag_grad_finish_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ sk, int nnz, int E, float lr,
                          const float* __restrict__ part, unsigned long long* __restrict__ stats,
                          const BagSource src) {
  finish_pass<VPL>(c, sk, nnz, E, lr, part, stats, src);
}

// ------------------------------------------------------------------------------------------------ host side
// workspace layout: the sort's and the passes' arrays (grouped::carve_push) | bag of position | coefficient
struct Workspace {
  PushWorkspace g; int* bag_of; float* coef; size_t total;
};

Workspace carve(void* base, int64_t nnz, int E) {
  Carve a{static_cast<char*>(base)};
  Workspace w{};
  w.g = carve_push(a, nnz, E);
  w.bag_of = a.take<int>(nnz);
  w.coef = a.take<float>(nnz);
  w.total = a.off;
  return w;
}

void check_shape(const CudaBackend& be, int64_t nnz, int E) {
  const Ctx& c = be.ctx();
  ADAPM_CHECK(c.L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  ADAPM_CHECK(E % 4 == 0 && E >= 4 && E <= kEmbBagMaxDim, "embedding_bag: dim must be a multiple of 4 in [4, 512]");
  ADAPM_CHECK(c.L.num_classes == 1 && !c.L.per_key_len && c.L.cls[0].len == (uint32_t)(2 * E),
              "embedding_bag: every row must be [embedding (dim) | AdaGrad (dim)]");
  ADAPM_CHECK(nnz >= 0 && nnz < ((int64_t)1 << 31), "embedding_bag: nnz must be < 2^31");
}

}  // namespace

size_t embedding_bag_workspace_bytes(int64_t nnz, int E) {
  return carve(nullptr, nnz, E).total;
}

void embedding_bag_forward(CudaBackend& be, cudaStream_t stream, const Key* keys, const int64_t* offsets,
                           const float* weights, int64_t nnz, int nbags, int E, bool mean, float* out,
                           unsigned long long* stats) {
  check_shape(be, nnz, E);
  if (nbags == 0) return;
  be.track_stream(stream);
  int log_g, vpl;
  lane_shape(E, &log_g, &vpl);
  const int bags_per_block = (kThreads / 32) << (5 - log_g);
  const int blocks = std::max(1, std::min((nbags + bags_per_block - 1) / bags_per_block, be.num_sms() * 16));
  const Ctx& c = be.ctx();
  switch (vpl) {
#define ADAPM_EMBBAG_FWD(V) \
  case V: embbag_fwd_kernel<V><<<blocks, kThreads, 0, stream>>>(c, keys, offsets, weights, nbags, E, log_g, mean, out, stats); break
    ADAPM_EMBBAG_FWD(1); ADAPM_EMBBAG_FWD(2); ADAPM_EMBBAG_FWD(3); ADAPM_EMBBAG_FWD(4);
#undef ADAPM_EMBBAG_FWD
    default: ADAPM_CHECK(false, "embedding_bag: bad dim " << E);
  }
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

void embedding_bag_backward(CudaBackend& be, cudaStream_t stream, const Key* keys, const int64_t* offsets,
                            const float* weights, int64_t nnz, int nbags, int E, bool mean, const float* grad_out,
                            float lr, float grad_scale, void* workspace, size_t workspace_bytes,
                            unsigned long long* stats) {
  check_shape(be, nnz, E);
  if (nnz == 0 || nbags == 0) return;
  be.track_stream(stream);
  Workspace w = carve(workspace, nnz, E);
  ADAPM_CHECK(workspace && workspace_bytes >= w.total, "embedding_bag: workspace too small");
  int log_g, vpl;
  lane_shape(E, &log_g, &vpl);
  const int n = (int)nnz;
  const int grid_n = be.num_sms() * 8;
  auto blocks_for = [&](long items) { return (int)std::max<long>(1, std::min<long>((items + kThreads - 1) / kThreads, grid_n)); };

  embbag_prep_kernel<<<blocks_for(n), kThreads, 0, stream>>>(offsets, weights, nbags, n, mean, w.g.pos_in, w.bag_of,
                                                             w.coef);
  ADAPM_COUNT_LAUNCH();
  const BagSource src{w.bag_of, w.coef, grad_out, grad_scale};
  switch (vpl) {
#define ADAPM_EMBBAG_BWD(V)                                                                                           \
  case V:                                                                                                             \
    sort_and_push<embbag_grad_tile_kernel<V>, embbag_grad_finish_kernel<V>>(be, stream, keys, w.g, src, n, E, log_g, \
                                                                            lr, stats);                               \
    break
    ADAPM_EMBBAG_BWD(1); ADAPM_EMBBAG_BWD(2); ADAPM_EMBBAG_BWD(3); ADAPM_EMBBAG_BWD(4);
#undef ADAPM_EMBBAG_BWD
    default: ADAPM_CHECK(false, "embedding_bag: bad dim " << E);
  }
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

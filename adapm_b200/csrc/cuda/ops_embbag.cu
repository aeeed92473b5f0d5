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
//   2. sort:   cub radix sort of (key, position) over the significant key bits; stable, so every key's occurrences
//              stay in position order
//   3. tile:   the sorted occurrences are cut into tiles of kTile; one lane group per tile sums each key's run in fp32
//              in position order. A run that lies inside the tile is pushed right away; a run that crosses a tile
//              boundary leaves one partial sum per tile it touches
//   4. finish: one warp per run that crosses a boundary adds its partials in tile order and pushes.
// Every distinct key gets one push with one fixed sum: on one GPU two runs of the same step give bit-identical rows.
#include <cuda_runtime.h>

#include <cub/cub.cuh>

#include "grouped_push.cuh"
#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {

namespace {

constexpr int kThreads = 256;
constexpr int kTile = 32;     // sorted occurrences per lane group in the tile pass

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

// 3. one group per tile of kTile sorted occurrences. part[t][0]: the partial of the run that was open at the tile's
// start (it began in an earlier tile); part[t][1]: the partial of a run that begins in the tile and crosses its end.
template <int VPL>
__global__ void __launch_bounds__(kThreads, 2)
embbag_grad_tile_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ sk, const int* __restrict__ spos,
                        const int* __restrict__ bag_of, const float* __restrict__ coef, const float* __restrict__ grad,
                        int nnz, int E, int log_g, float lr, float grad_scale, float* __restrict__ part,
                        unsigned long long* __restrict__ stats) {
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
      int bb = 0;
      float cc = 0.f;
      if (p0 + sub < hi) {
        kk = sk[p0 + sub];
        const int ps = spos[p0 + sub];
        bb = bag_of[ps];
        cc = coef[ps];
      }
      const int cnt = min(G, hi + 1 - p0);
      for (int u = 0; u < cnt; ++u) {
        const Key k = (Key)__shfl_sync(mask, (long long)kk, u, G);
        const int bu = __shfl_sync(mask, bb, u, G);
        const float cu = __shfl_sync(mask, cc, u, G);
        if (k != cur) {                  // the run of `cur` ends here (k == -1: at the tile's end)
          const bool crosses = k == -1 && hi < nnz && sk[hi] == cur;
          if (open_before || crosses) {
            float* pp = part + ((size_t)t * 2 + (open_before ? 0 : 1)) * E;
#pragma unroll
            for (int v = 0; v < VPL; ++v) {
              const int j = sub + G * v;
              if (j < E4) reinterpret_cast<float4*>(pp)[j] = acc[v];
            }
          } else {
#pragma unroll
            for (int v = 0; v < VPL; ++v) {
              acc[v].x *= grad_scale; acc[v].y *= grad_scale; acc[v].z *= grad_scale; acc[v].w *= grad_scale;
            }
            push_update<VPL>(c, cur, acc, E, sub, G, mask, lr, n, stats);
          }
          if (k == -1) break;
          cur = k;
          open_before = false;
#pragma unroll
          for (int v = 0; v < VPL; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        const float* gr = grad + (size_t)bu * E;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int j = sub + G * v;
          if (j < E4) {
            const float4 x = __ldg(reinterpret_cast<const float4*>(gr) + j);
            acc[v].x = fmaf(cu, x.x, acc[v].x); acc[v].y = fmaf(cu, x.y, acc[v].y);
            acc[v].z = fmaf(cu, x.z, acc[v].z); acc[v].w = fmaf(cu, x.w, acc[v].w);
          }
        }
      }
    }
  }
  __syncwarp();
  flush_counts(n, stats);
  dev::cta_exit(c);
}

// 4. one warp per tile boundary q = i * kTile: if a run crosses q and does not cross q - kTile, the warp owns it: its
// partials part[i - 1][1], part[i][0], part[i + 1][0], ... are added in tile order, and the key is pushed.
template <int VPL>
__global__ void __launch_bounds__(kThreads, 2)
embbag_grad_finish_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ sk, int nnz, int E, float lr,
                          float grad_scale, const float* __restrict__ part, unsigned long long* __restrict__ stats) {
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
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      acc[v].x *= grad_scale; acc[v].y *= grad_scale; acc[v].z *= grad_scale; acc[v].w *= grad_scale;
    }
    push_update<VPL>(c, k, acc, E, lane, 32, 0xffffffffu, lr, n, stats);
  }
  flush_counts(n, stats);
  dev::cta_exit(c);
}

// ------------------------------------------------------------------------------------------------ host side
// workspace layout: sorted keys | positions (in, out) | bag of position | coefficient | tile partials | sort scratch
struct Workspace {
  Key* sk; int* pos_in; int* pos_out; int* bag_of; float* coef; float* part; void* sort_tmp; size_t sort_bytes;
  size_t total;
};

Workspace carve(void* base, int64_t nnz, int E) {
  Workspace w{};
  size_t sort_bytes = 0;
  ADAPM_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const unsigned long long*)nullptr,
                                                   (unsigned long long*)nullptr, (const int*)nullptr, (int*)nullptr,
                                                   (int)nnz, 0, 64));
  const size_t n_tiles = (size_t)(nnz + kTile - 1) / kTile;
  char* p = static_cast<char*>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) { char* q = p ? p + off : nullptr; off += align_up(bytes); return q; };
  w.sk = reinterpret_cast<Key*>(take((size_t)nnz * sizeof(Key)));
  w.pos_in = reinterpret_cast<int*>(take((size_t)nnz * sizeof(int)));
  w.pos_out = reinterpret_cast<int*>(take((size_t)nnz * sizeof(int)));
  w.bag_of = reinterpret_cast<int*>(take((size_t)nnz * sizeof(int)));
  w.coef = reinterpret_cast<float*>(take((size_t)nnz * sizeof(float)));
  w.part = reinterpret_cast<float*>(take(n_tiles * 2 * E * sizeof(float)));
  w.sort_tmp = take(sort_bytes);
  w.sort_bytes = sort_bytes;
  w.total = off;
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

size_t embedding_bag_workspace_bytes(int64_t nnz, int64_t nbags, int E) {
  (void)nbags;
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
  const Ctx& c = be.ctx();
  Workspace w = carve(workspace, nnz, E);
  ADAPM_CHECK(workspace && workspace_bytes >= w.total, "embedding_bag: workspace too small");
  int log_g, vpl;
  lane_shape(E, &log_g, &vpl);
  const int n = (int)nnz;
  const int grid_n = be.num_sms() * 8;
  auto blocks_for = [&](long items) { return (int)std::max<long>(1, std::min<long>((items + kThreads - 1) / kThreads, grid_n)); };

  embbag_prep_kernel<<<blocks_for(n), kThreads, 0, stream>>>(offsets, weights, nbags, n, mean, w.pos_in, w.bag_of, w.coef);
  ADAPM_COUNT_LAUNCH();
  size_t sort_bytes = w.sort_bytes;
  ADAPM_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(w.sort_tmp, sort_bytes, reinterpret_cast<const unsigned long long*>(keys),
                                                   reinterpret_cast<unsigned long long*>(w.sk), w.pos_in, w.pos_out, n, 0,
                                                   key_bits(c.L.num_keys), stream));
  ADAPM_COUNT_LAUNCH();   // (the sort counts as one launch; cub runs one or more kernels, depending on nnz and the bits)
  const int n_tiles = (n + kTile - 1) / kTile;
  const int tiles_per_block = (kThreads / 32) << (5 - log_g);
  const int tile_blocks = std::max(1, std::min((n_tiles + tiles_per_block - 1) / tiles_per_block, be.num_sms() * 16));
  const int fin_blocks = std::max(1, std::min((n_tiles + kThreads / 32 - 1) / (kThreads / 32), grid_n));
  switch (vpl) {
#define ADAPM_EMBBAG_BWD(V)                                                                                             \
  case V:                                                                                                               \
    embbag_grad_tile_kernel<V><<<tile_blocks, kThreads, 0, stream>>>(c, w.sk, w.pos_out, w.bag_of, w.coef, grad_out, n, \
                                                                     E, log_g, lr, grad_scale, w.part, stats);          \
    ADAPM_COUNT_LAUNCH();                                                                                               \
    embbag_grad_finish_kernel<V><<<fin_blocks, kThreads, 0, stream>>>(c, w.sk, n, E, lr, grad_scale, w.part, stats);    \
    ADAPM_COUNT_LAUNCH();                                                                                               \
    break
    ADAPM_EMBBAG_BWD(1); ADAPM_EMBBAG_BWD(2); ADAPM_EMBBAG_BWD(3); ADAPM_EMBBAG_BWD(4);
#undef ADAPM_EMBBAG_BWD
    default: ADAPM_CHECK(false, "embedding_bag: bad dim " << E);
  }
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

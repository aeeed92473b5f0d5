// Random walks on a CSR graph for node2vec / DeepWalk, and their expansion into skip-gram pairs, for sm_90a.
//
// Walks (node2vec_walk_kernel, one thread per walk). Node v's out-neighbours are nbrs[off[v] .. off[v + 1]), sorted; a
// weighted graph also has cumw there, the inclusive prefix sums of its integer (quantised) edge weights. Position 0 of
// a walk is its start; a node without out-edges ends the walk and the rest of its row is -1.
//   first order  unweighted: neighbour floor(h32 deg / 2^32); weighted: r = floor(h T / 2^64) (T = the node's total
//                weight) and the first neighbour whose cumulative weight exceeds r.
//   second order rejection sampling (KnightKing): a candidate x from v's first-order distribution is accepted when a
//                24-bit uniform is below the threshold of alpha(t, x) / alpha_max, with alpha = 1 / p (x = t), 1 (x in
//                N(t), a binary search of t's sorted list) or 1 / q. The three thresholds come from the host; a uniform
//                below the smaller of the last two accepts without the search. No per-edge table is built, and a trial
//                succeeds with probability >= min alpha / alpha_max.
// Every number is a counter hash: walk base b = mix64(mix64(s0 ^ start) ^ walk number), s0 = mix64(mix64(seed) ^
// epoch); the draw of step k, trial j is h = mix64(b ^ (k << 32 | j)), h32 = h >> 32, and the acceptance uniform is
// mix64(h) >> 40. A walk is therefore a function of (seed, epoch, start, walk number, graph, p, q) alone.
//
// Pairs (three passes: count -> cub inclusive scan -> write). Position i of walk row r draws its window shrink
// b = floor(h32 window / 2^32) from h = mix64(mix64(seed) ^ (r << 32 | i)); with radius window - b it makes the pairs
// (2 walk[j], 2 walk[i] + 1) for every valid j != i within the radius, ascending j, rows in order, then positions.
#include <cuda_runtime.h>

#include <cub/cub.cuh>

#include "group.cuh"
#include "hash.cuh"
#include "ops.h"

namespace adapm {
namespace cudaops {

namespace {

constexpr int kWalkThreads = 128;
constexpr int kPairThreads = 256;

struct WalkArgs {
  const int64_t* off;
  const int32_t* nbrs;
  const int64_t* cumw;        // null: unweighted
  const int64_t* starts;
  const int64_t* walk_nos;
  int64_t n_walks;
  int L;
  uint64_t s0;
  uint32_t thr_return, thr_in, thr_out;
  int64_t* out;
};

// index of the first-order pick among v's out-edges [lo, hi), hi > lo
template <bool WEIGHTED>
__device__ __forceinline__ int64_t first_order(const WalkArgs& a, int64_t lo, int64_t hi, uint64_t h) {
  if (!WEIGHTED) return lo + (int64_t)(((h >> 32) * (uint64_t)(hi - lo)) >> 32);
  const uint64_t r = __umul64hi(h, (uint64_t)__ldg(a.cumw + hi - 1));
  --hi;                                         // the first e in [lo, hi] with cumw[e] > r; cumw[hi] = T > r
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if ((uint64_t)__ldg(a.cumw + mid) > r) hi = mid; else lo = mid + 1;
  }
  return lo;
}

__device__ __forceinline__ bool has_edge(const WalkArgs& a, int64_t t, int32_t x) {
  int64_t lo = __ldg(a.off + t), hi = __ldg(a.off + t + 1);
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    const int32_t y = __ldg(a.nbrs + mid);
    if (y == x) return true;
    if (y < x) lo = mid + 1; else hi = mid;
  }
  return false;
}

template <bool WEIGHTED, bool SECOND_ORDER>
__global__ void __launch_bounds__(kWalkThreads, 8) node2vec_walk_kernel(const __grid_constant__ WalkArgs a) {
  const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= a.n_walks) return;
  int64_t* row = a.out + w * a.L;
  int64_t v = __ldg(a.starts + w), t = -1;
  const uint64_t base = mix64(mix64(a.s0 ^ (uint64_t)v) ^ (uint64_t)__ldg(a.walk_nos + w));
  const uint32_t thr_min = min(a.thr_in, a.thr_out);
  row[0] = v;
  int k = 1;
  for (; k < a.L; ++k) {
    const int64_t lo = __ldg(a.off + v), hi = __ldg(a.off + v + 1);
    if (hi == lo) break;
    int32_t x;
    for (uint32_t j = 0;; ++j) {
      const uint64_t h = mix64(base ^ ((uint64_t)k << 32 | j));
      x = __ldg(a.nbrs + first_order<WEIGHTED>(a, lo, hi, h));
      if (!SECOND_ORDER || t < 0) break;
      const uint32_t u = (uint32_t)(mix64(h) >> 40);
      if (x == t) {
        if (u < a.thr_return) break;
      } else if (u < thr_min || u < (has_edge(a, t, x) ? a.thr_in : a.thr_out)) {
        break;
      }
    }
    row[k] = x;
    t = v;
    v = x;
  }
  for (; k < a.L; ++k) row[k] = -1;
}

// the window shrink b in [0, window) of position i of row r
__device__ __forceinline__ int shrink(uint64_t s, int64_t r, int i, int window) {
  const uint64_t h = mix64(s ^ ((uint64_t)r << 32 | (uint32_t)i));
  return (int)(((h >> 32) * (uint64_t)window) >> 32);
}

__global__ void __launch_bounds__(kPairThreads)
walk_pair_count_kernel(const int64_t* __restrict__ walks, int64_t n_items, int L, int window, uint64_t s,
                       int64_t* __restrict__ counts) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_items) return;
  const int64_t r = p / L;
  const int i = (int)(p - r * L);
  const int64_t* row = walks + r * L;
  int64_t c = 0;
  if (__ldg(row + i) >= 0) {
    const int rad = window - shrink(s, r, i, window);
    c = i - max(0, i - rad);                      // positions before i are valid
    for (int j = i + 1; j < min(L, i + rad + 1) && __ldg(row + j) >= 0; ++j) ++c;
  }
  counts[p] = c;
}

__global__ void __launch_bounds__(kPairThreads)
walk_pair_write_kernel(const int64_t* __restrict__ walks, int64_t n_items, int L, int window, uint64_t s,
                       const int64_t* __restrict__ ends, int64_t n_pairs, Key* __restrict__ out) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_items) return;
  const int64_t r = p / L;
  const int i = (int)(p - r * L);
  const int64_t* row = walks + r * L;
  const int64_t ctr = __ldg(row + i);
  if (ctr < 0) return;
  int64_t o = p == 0 ? 0 : __ldg(ends + p - 1);
  const int rad = window - shrink(s, r, i, window);
  const Key target = 2 * ctr + 1;
  for (int j = max(0, i - rad); j < min(L, i + rad + 1); ++j) {
    if (j == i) continue;
    const int64_t c = __ldg(row + j);
    if (c < 0) break;
    out[o] = 2 * c;
    out[n_pairs + o] = target;
    ++o;
  }
}

int blocks_for(int64_t n, int threads) { return (int)((n + threads - 1) / threads); }

}  // namespace

void node2vec_walks(cudaStream_t stream, const int64_t* offsets, const int32_t* nbrs, const int64_t* cumw,
                    const int64_t* starts, const int64_t* walk_nos, int64_t n_walks, int L, uint64_t seed,
                    uint64_t epoch, uint32_t thr_return, uint32_t thr_in, uint32_t thr_out, bool second_order,
                    int64_t* out) {
  ADAPM_CHECK(L >= 2, "walk length must be at least 2, got " << L);
  ADAPM_CHECK(n_walks < ((int64_t)1 << 31) * kWalkThreads, "too many walks in one call: " << n_walks);
  if (n_walks == 0) return;
  WalkArgs a{offsets, nbrs, cumw, starts, walk_nos, n_walks, L, mix64(mix64(seed) ^ epoch), thr_return, thr_in,
             thr_out, out};
  const int blocks = blocks_for(n_walks, kWalkThreads);
  if (cumw) {
    if (second_order) node2vec_walk_kernel<true, true><<<blocks, kWalkThreads, 0, stream>>>(a);
    else node2vec_walk_kernel<true, false><<<blocks, kWalkThreads, 0, stream>>>(a);
  } else {
    if (second_order) node2vec_walk_kernel<false, true><<<blocks, kWalkThreads, 0, stream>>>(a);
    else node2vec_walk_kernel<false, false><<<blocks, kWalkThreads, 0, stream>>>(a);
  }
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

size_t walk_pair_scan_bytes(int64_t n_items) {
  size_t bytes = 0;
  ADAPM_CUDA_CHECK(cub::DeviceScan::InclusiveSum(nullptr, bytes, (const int64_t*)nullptr, (int64_t*)nullptr,
                                                 (int)n_items));
  return bytes;
}

void walk_pair_ends(cudaStream_t stream, const int64_t* walks, int64_t n_walks, int L, int window, uint64_t seed,
                    int64_t* counts, int64_t* ends, void* temp, size_t temp_bytes) {
  const int64_t n_items = n_walks * L;
  ADAPM_CHECK(window >= 1, "window must be at least 1, got " << window);
  ADAPM_CHECK(n_items < ((int64_t)1 << 31), "too many walk positions in one call: " << n_items);
  if (n_items == 0) return;
  walk_pair_count_kernel<<<blocks_for(n_items, kPairThreads), kPairThreads, 0, stream>>>(walks, n_items, L, window,
                                                                                          mix64(seed), counts);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
  size_t bytes = temp_bytes;
  ADAPM_CUDA_CHECK(cub::DeviceScan::InclusiveSum(temp, bytes, counts, ends, (int)n_items, stream));
  ADAPM_COUNT_LAUNCH();
}

void walk_pairs_write(cudaStream_t stream, const int64_t* walks, int64_t n_walks, int L, int window, uint64_t seed,
                      const int64_t* ends, int64_t n_pairs, Key* out) {
  const int64_t n_items = n_walks * L;
  if (n_items == 0 || n_pairs == 0) return;
  walk_pair_write_kernel<<<blocks_for(n_items, kPairThreads), kPairThreads, 0, stream>>>(walks, n_items, L, window,
                                                                                          mix64(seed), ends, n_pairs,
                                                                                          out);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

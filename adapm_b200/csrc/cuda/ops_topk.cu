// Top-k retrieval on the tensor cores (sm_90a): for every query row i, the k columns j with the largest
//     score(i, j) = <q_i, e_j>  (bf16 operands, fp32 wgmma accumulation)  [* col_scale[j]]
// without an [M, N] score matrix. Two tile kernels share the TOPK epilogue:
//   gemm_nt_topk_kernel       E is a dense bf16 matrix; Q and E tiles arrive by TMA (as in gemm_nt_wgmma_kernel)
//   gather_gemm_topk_kernel   row j of E is the parameter-store row keys[j], gathered through the directory from local
//                             HBM, replicas or NVLink peers (as in gather_gemm_kernel); Q arrives by TMA
// The k-block order and the wgmma sequence of a tile are those of the existing kernels, so every score is bit-identical
// to gemm_nt_bf16 / gather_gemm (when gemm_nt_bf16 does not split K).
//
// Order: score descending, ties to the smaller column - a total order, so the result does not depend on how the
// columns are split over CTAs. NaN scores are never selected; rows with fewer than k eligible columns are padded with
// (-inf, -1). Optional exclusions: a CSR list of columns per row (sorted ascending).
//
// Grid: (M tiles) x (S N-slices). CTA (m, s) accumulates the N tiles s, s + S, ... of its M tile: the producer runs its
// ring straight across the tile boundaries. The CTAs that read the same N tiles have consecutive ids, so they run at
// the same time and share the B rows in L2. Each CTA keeps a running top-k list per query row in shared memory, with
// the row's current k-th entry (the threshold) next to it. After a tile, the four lanes that hold a row compare their
// 32 scores against the threshold; only the survivors are checked against the row's exclusions (binary search, all
// lanes at once) and inserted - one lane of each row at a time. At the end each CTA writes its list, sorted, to a workspace [M, S, k]
// and topk_merge_kernel (one warp per row) merges the S lists with the same total order.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>

#include "ops.h"
#include "pm_kernels.cuh"
#include "wgmma_utils.cuh"

namespace adapm {
namespace cudaops {

namespace {

using namespace tc;

constexpr int TK_STAGES = 4;          // 128 KiB ring + 66 KiB of lists (a 6-stage ring would leave no room)
constexpr int LSTRIDE = kTopkMax + 1; // padded list row: the 8 rows that a lane group scans sit in distinct banks
constexpr uint32_t NO_COL = 0xFFFFFFFFu;  // padding entry (-inf, NO_COL): loses to every eligible column
constexpr int kMaxSlices = 2048;
constexpr int kMergeWarps = 4;

struct TopkSmem {
  Ring<TK_STAGES> ring;
  float list_v[BM][LSTRIDE];
  uint32_t list_c[BM][LSTRIDE];
  float thr_v[BM];                    // the row's worst list entry = the score a new column has to beat
  uint32_t thr_c[BM];
  int worst[BM];                      // its position in the list
};

struct TopkArgs {
  int M, N, K, k, S;
  const float* col_scale;             // [N] or null
  const int64_t* ex_off;              // [M + 1] or null
  const int64_t* ex_cols;             // [nnz], ascending per row
  float* part_v;                      // [M, S, k]
  int* part_c;
};

// (v, c) comes before (tv, tc): higher score, or the same score and a smaller column. False for a NaN v.
__device__ __forceinline__ bool beats(float v, uint32_t c, float tv, uint32_t tc) {
  return v > tv || (v == tv && c < tc);
}

// the 16 rows of a consumer warp start with k padding entries each
__device__ __forceinline__ void init_lists(TopkSmem& sm, int rbase, int k, int lane) {
  for (int i = lane; i < 16 * k; i += 32) {
    sm.list_v[rbase + i / k][i % k] = -INFINITY;
    sm.list_c[rbase + i / k][i % k] = NO_COL;
  }
  if (lane < 16) { sm.thr_v[rbase + lane] = -INFINITY; sm.thr_c[rbase + lane] = NO_COL; sm.worst[rbase + lane] = 0; }
  __syncwarp();
}

__device__ __forceinline__ bool excluded(const TopkArgs& a, int row, uint32_t col) {
  if (!a.ex_off) return false;
  int64_t lo = a.ex_off[row];
  const int64_t end = a.ex_off[row + 1];
  int64_t hi = end;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a.ex_cols[mid] < (int64_t)col) lo = mid + 1; else hi = mid;
  }
  return lo < end && a.ex_cols[lo] == (int64_t)col;
}

// (v, col) replaces the worst entry of list r if it still beats it; then the new worst is found.
__device__ __forceinline__ void list_insert(TopkSmem& sm, const TopkArgs& a, int r, float v, uint32_t col) {
  if (!beats(v, col, sm.thr_v[r], sm.thr_c[r])) return;   // the threshold may have risen since the screen
  float* lv = sm.list_v[r];
  uint32_t* lc = sm.list_c[r];
  const int w0 = sm.worst[r];
  lv[w0] = v; lc[w0] = col;
  float wv = lv[0];
  uint32_t wc = lc[0];
  int w = 0;
  for (int i = 1; i < a.k; ++i) {
    const float x = lv[i];
    const uint32_t xc = lc[i];
    if (beats(wv, wc, x, xc)) { wv = x; wc = xc; w = i; }
  }
  sm.worst[r] = w; sm.thr_v[r] = wv; sm.thr_c[r] = wc;
}

// TOPK epilogue of one tile. Accumulator fragment as in store_fragment: d[4j + 2h + e] = D[row(h)][col0 + 8j + 2(lane%4) + e].
__device__ __forceinline__ void topk_tile(TopkSmem& sm, const TopkArgs& a, float (&d)[64], int rbase, int tile_m, int col0,
                                          int lane) {
  const int q = lane & 3;
  uint32_t mask[2];
  float tv[2];
  uint32_t tcol[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = rbase + (lane >> 2) + 8 * h;
    tv[h] = sm.thr_v[r]; tcol[h] = sm.thr_c[r]; mask[h] = 0u;
  }
#pragma unroll
  for (int j = 0; j < 16; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int col = col0 + 8 * j + 2 * q + e;
      if (col < a.N) {
        const float cs = a.col_scale ? __ldg(a.col_scale + col) : 1.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float v = d[4 * j + 2 * h + e];
          if (a.col_scale) v *= cs;
          d[4 * j + 2 * h + e] = v;
          if (beats(v, (uint32_t)col, tv[h], tcol[h])) mask[h] |= 1u << (2 * j + e);
        }
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int grow = tile_m * BM + rbase + (lane >> 2) + 8 * h;
    if (grow >= a.M) { mask[h] = 0u; continue; }   // padding rows of the last M tile
    // exclusion checks of the survivors: in all lanes at once, before the serialised insertion
    for (uint32_t m = a.ex_off ? mask[h] : 0u; m; m &= m - 1u) {
      const int b = __ffs(m) - 1;
      if (excluded(a, grow, (uint32_t)(col0 + 8 * (b >> 1) + 2 * q + (b & 1)))) mask[h] &= ~(1u << b);
    }
  }
  // survivors go in one lane of each row at a time (the 8 lanes of a group own 8 different rows)
  for (int qq = 0; qq < 4; ++qq) {
    if (q == qq) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = rbase + (lane >> 2) + 8 * h;
        while (mask[h]) {
          const int b = __ffs(mask[h]) - 1;
          mask[h] &= mask[h] - 1u;
          float v = 0.f;
#pragma unroll
          for (int t = 0; t < 32; ++t)
            if (t == b) v = d[4 * (t >> 1) + 2 * h + (t & 1)];   // static register indices: no local memory
          list_insert(sm, a, r, v, (uint32_t)(col0 + 8 * (b >> 1) + 2 * q + (b & 1)));
        }
      }
    }
    __syncwarp();
  }
}

// the warp's lists -> part[row, s, 0..k), sorted by the total order (rank = number of entries that come first)
__device__ __forceinline__ void write_partial(TopkSmem& sm, const TopkArgs& a, int rbase, int tile_m, int s, int lane) {
  for (int rr = 0; rr < 16; ++rr) {
    const int r = rbase + rr;
    const int grow = tile_m * BM + r;
    if (grow >= a.M) break;
    const float* lv = sm.list_v[r];
    const uint32_t* lc = sm.list_c[r];
    for (int i = lane; i < a.k; i += 32) {
      const float v = lv[i];
      const uint32_t c = lc[i];
      int rank = 0;
      for (int j = 0; j < a.k; ++j) {
        const float x = lv[j];
        const uint32_t xc = lc[j];
        rank += (beats(x, xc, v, c) || (x == v && xc == c && j < i)) ? 1 : 0;   // padding entries are all equal
      }
      const size_t o = ((size_t)grow * a.S + s) * a.k + rank;
      a.part_v[o] = v;
      a.part_c[o] = (int)c;   // NO_COL -> -1
    }
  }
}

// Consumer warps of both top-k kernels: the N tiles slice, slice + S, ... of M tile tile_m, accumulated tile after tile
// from the ring and screened into the running lists, which then go to the workspace.
__device__ __forceinline__ void topk_consume(TopkSmem& sm, const TopkArgs& a, int tile_m, int slice, int num_kb) {
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = (warp >> 2) - 1;
  const int rbase = frag_row0(warp);
  init_lists(sm, rbase, a.k, lane);
  uint32_t it = 0;
  float d[64];
  for (int tn = slice; tn < (a.N + BN - 1) / BN; tn += a.S) {
    consume<KIND_BF16>(sm.ring, num_kb, it, true, wg, lane, d);
    topk_tile(sm, a, d, rbase, tile_m, tn * BN, lane);
  }
  write_partial(sm, a, rbase, tile_m, slice, lane);
}

__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_nt_topk_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                    const __grid_constant__ TopkArgs a) {
  TopkSmem& sm = smem_as<TopkSmem>();
  const int tile_m = blockIdx.x, slice = blockIdx.y;
  const int n_tiles = (a.N + BN - 1) / BN;
  const int num_kb = (a.K + BK<KIND_BF16> - 1) / BK<KIND_BF16>;

  if (threadIdx.x == 0) {
    sm.ring.init(1);
    prefetch_tensormap(&tmap_a);
    prefetch_tensormap(&tmap_b);
  }
  __syncthreads();

  if (threadIdx.x >= 128) {
    topk_consume(sm, a, tile_m, slice, num_kb);
  } else if (threadIdx.x == 0) {
    // TMA producer: the ring runs across the tiles of the slice
    uint32_t it = 0;
    for (int tn = slice; tn < n_tiles; tn += a.S)
      produce_tma<KIND_BF16>(sm.ring, tmap_a, tmap_b, tile_m * BM, tn * BN, 0, num_kb, it);
  }
}

__global__ void __launch_bounds__(kGemmThreads, 1)
gather_gemm_topk_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ Ctx c,
                        const Key* __restrict__ keys, const __grid_constant__ TopkArgs a,
                        unsigned long long* __restrict__ stats) {
  TopkSmem& sm = smem_as<TopkSmem>();
  const int tile_m = blockIdx.x, slice = blockIdx.y;
  const int n_tiles = (a.N + BN - 1) / BN;
  const int num_kb = (a.K + BK<KIND_BF16> - 1) / BK<KIND_BF16>;
  // The gather warps read store rows through the directory: this CTA counts in the grace epoch for all its tiles, so a
  // sync round that relocates rows waits for it (the host bounds the tiles per CTA through S).
  dev::cta_enter(c);

  if (threadIdx.x == 0) {
    sm.ring.init(5);   // full: the TMA of the Q tile + one arrival per gather warp
    prefetch_tensormap(&tmap_q);
  }
  __syncthreads();

  if (threadIdx.x >= 128) {
    topk_consume(sm, a, tile_m, slice, num_kb);
  } else {
    // gatherers: store rows -> swizzled smem, tile after tile; thread 0 also TMAs Q
    GatherStats st;
    uint32_t it = 0;
    for (int tn = slice; tn < n_tiles; tn += a.S)
      produce_gather(sm.ring, tmap_q, c, keys, tn * BN, a.N, a.K, tile_m * BM, num_kb, it, st);
    st.flush(stats);
  }
  dev::cta_exit(c);
}

// One warp per row: k-way merge of the row's S sorted lists; a lane owns the list heads of slices lane, lane + 32, ...
__global__ void __launch_bounds__(kMergeWarps * 32)
topk_merge_kernel(const float* __restrict__ part_v, const int* __restrict__ part_c, int M, int S, int k,
                  float* __restrict__ out_v, int64_t* __restrict__ out_i) {
  extern __shared__ int merge_heads[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * kMergeWarps + w;
  if (row >= M) return;   // (warp-uniform; no block-wide barrier follows)
  int* head = merge_heads + w * S;
  for (int s = lane; s < S; s += 32) head[s] = 0;
  __syncwarp();
  const float* pv = part_v + (size_t)row * S * k;
  const int* pc = part_c + (size_t)row * S * k;
  for (int r = 0; r < k; ++r) {
    float bv = -INFINITY;
    uint32_t bc = NO_COL;
    int bs = -1;
    for (int s = lane; s < S; s += 32) {
      const int h = head[s];
      if (h >= k) continue;
      const int cc = pc[s * k + h];
      if (cc < 0) continue;                // the rest of this list is padding
      const float v = pv[s * k + h];
      if (beats(v, (uint32_t)cc, bv, bc)) { bv = v; bc = (uint32_t)cc; bs = s; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const uint32_t oc = __shfl_xor_sync(0xffffffffu, bc, o);
      const int os = __shfl_xor_sync(0xffffffffu, bs, o);
      if (beats(ov, oc, bv, bc)) { bv = ov; bc = oc; bs = os; }
    }
    if (lane == 0) {
      out_v[(size_t)row * k + r] = bs >= 0 ? bv : -INFINITY;
      out_i[(size_t)row * k + r] = bs >= 0 ? (int64_t)bc : -1;
    }
    if (bs >= 0 && lane == (bs & 31)) head[bs] += 1;
    __syncwarp();
  }
}

TopkArgs make_args(int M, int N, int K, int k, int S, const float* col_scale, const int64_t* ex_off, const int64_t* ex_cols,
                   float* part_v, int* part_c) {
  ADAPM_CHECK(k >= 1 && k <= kTopkMax, "topk: k must be in [1, " << kTopkMax << "]");
  ADAPM_CHECK(S >= 1 && S <= kMaxSlices, "topk: bad slice count " << S);
  ADAPM_CHECK(K > 0, "topk: empty K extent");
  TopkArgs a;
  a.M = M; a.N = N; a.K = K; a.k = k; a.S = S;
  a.col_scale = col_scale; a.ex_off = ex_off; a.ex_cols = ex_cols; a.part_v = part_v; a.part_c = part_c;
  return a;
}

void launch_merge(cudaStream_t stream, const TopkArgs& a, float* out_v, int64_t* out_i) {
  const size_t smem = (size_t)kMergeWarps * a.S * sizeof(int);   // list heads: at most 32 KiB
  topk_merge_kernel<<<(a.M + kMergeWarps - 1) / kMergeWarps, kMergeWarps * 32, smem, stream>>>(a.part_v, a.part_c, a.M, a.S,
                                                                                             a.k, out_v, out_i);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace

int topk_num_slices(int M, int N, int max_tiles_per_cta) {
  const int m_tiles = (M + BM - 1) / BM, n_tiles = (N + BN - 1) / BN;
  if (m_tiles == 0 || n_tiles == 0) return 1;
  int S = (2 * num_sms() + m_tiles - 1) / m_tiles;   // about two waves of one CTA per SM
  if (max_tiles_per_cta > 0) S = std::max(S, (n_tiles + max_tiles_per_cta - 1) / max_tiles_per_cta);
  return std::max(1, std::min({S, n_tiles, kMaxSlices}));
}

void gemm_nt_topk(cudaStream_t stream, const void* A, const void* B, int M, int N, int K, int k, int S,
                  const float* col_scale, const int64_t* ex_off, const int64_t* ex_cols, float* part_v, int* part_c,
                  float* out_v, int64_t* out_i) {
  if (M == 0) return;
  const TopkArgs a = make_args(M, N, K, k, S, col_scale, ex_off, ex_cols, part_v, part_c);
  ADAPM_CHECK(N > 0, "gemm_nt_topk: no columns");
  const CUtensorMap ma = make_map("gemm_nt_topk", A, M, K, BM, KIND_BF16);
  const CUtensorMap mb = make_map("gemm_nt_topk", B, N, K, BN, KIND_BF16);
  launch<gemm_nt_topk_kernel, TopkSmem>(dim3((M + BM - 1) / BM, S), stream, ma, mb, a);
  launch_merge(stream, a, out_v, out_i);
}

void topk_merge(cudaStream_t stream, const float* part_v, const int* part_c, int M, int S, int k, float* out_v,
                int64_t* out_i) {
  if (M == 0) return;
  const TopkArgs a = make_args(M, 1, 1, k, S, nullptr, nullptr, nullptr, const_cast<float*>(part_v), const_cast<int*>(part_c));
  launch_merge(stream, a, out_v, out_i);
}

void gather_gemm_topk(CudaBackend& be, cudaStream_t stream, const void* Q, const Key* keys, int M, int N, int K, int ldq,
                      int k, int S, const float* col_scale, const int64_t* ex_off, const int64_t* ex_cols, float* part_v,
                      int* part_c, float* out_v, int64_t* out_i, unsigned long long* stats) {
  if (M == 0) return;
  const TopkArgs a = make_args(M, N, K, k, S, col_scale, ex_off, ex_cols, part_v, part_c);
  ADAPM_CHECK(N > 0, "gather_gemm_topk: no keys");
  ADAPM_CHECK(K % 4 == 0, "gather_gemm_topk: the embedding length must be a multiple of 4");
  ADAPM_CHECK(ldq >= K, "gather_gemm_topk: Q's row pitch must be at least K");
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  be.track_stream(stream);
  const CUtensorMap mq = make_map("gather_gemm_topk", Q, M, ldq, BM, KIND_BF16);
  launch<gather_gemm_topk_kernel, TopkSmem>(dim3((M + BM - 1) / BM, S), stream, mq, be.ctx(), keys, a, stats);
  launch_merge(stream, a, out_v, out_i);
}

}  // namespace cudaops
}  // namespace adapm

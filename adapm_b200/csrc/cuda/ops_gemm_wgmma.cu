// Hand-written Hopper tensor-core GEMM for sm_90a:
//     C[M, N] (fp32) = A[M, K] (bf16 or e4m3, K-major) x B[N, K]^T (same type, K-major)
// used for the 1-vs-all scoring of the KGE filtered-ranking evaluation (SURVEY K12: q(s,r) x E^T)
// and for the dense layers of the CTR DeepFM model. Two epilogues:
//   STORE       write the fp32 scores
//   RANK_COUNT  do not materialise the scores at all: per row count the candidates whose score
//               beats the row's true score (reference kge.cc:716-774 loops over all entities per
//               triple) and atomically accumulate the count -> the [B x ne] score matrix never
//               touches HBM.
//
// Structure (one 128 x 128 output tile per CTA, 384 threads, see wgmma_utils.cuh):
//   warpgroup 0      TMA producer   one thread issues cp.async.bulk.tensor.2d (128B-swizzled 128x64 bf16 boxes)
//                                   into a 6-stage shared-memory ring guarded by full / empty mbarriers
//   warpgroups 1-2   consumers      wgmma.mma_async m64n128 (A/B from shared-memory descriptors, D in registers),
//                                   then the epilogue straight from the accumulator fragment
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>

#include "ops.h"
#include "wgmma_utils.cuh"

namespace adapm {
namespace cudaops {

namespace {

using namespace tc;

enum Epilogue : int { EPI_STORE = 0, EPI_RANK_COUNT = 1 };

template <int EPI, int KIND>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_nt_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, int M,
                     int N, int K, float* __restrict__ C, int ldc, float alpha, const float* __restrict__ true_score,
                     const int* __restrict__ true_col, int* __restrict__ rank_out) {
  const int tile_n = blockIdx.x, tile_m = blockIdx.y;
  // split-K (gridDim.z > 1, EPI_STORE only): this CTA accumulates its split's k-blocks and ADDS its partial tile to C,
  // which the host zeroed - for problems with few output tiles and a long K extent
  const KRange kr = k_split((K + BK<KIND> - 1) / BK<KIND>);
  float d[64];
  if (!tma_tile<KIND>(tmap_a, tmap_b, tile_m * BM, tile_n * BN, kr.kb0, kr.num_kb, d)) return;
  // consumers: the epilogue straight from the accumulator fragment
  const int lane = threadIdx.x & 31;
  const int row0 = tile_m * BM + frag_row0(threadIdx.x >> 5);
  const int col0 = tile_n * BN;
  if (EPI == EPI_STORE) store_fragment(d, alpha, C, ldc, row0, col0, M, N, lane, gridDim.z > 1);
  else rank_count_fragment(d, true_score, true_col, rank_out, row0, col0, M, N, lane);
}

template <int EPI, int KIND>
void launch_gemm(cudaStream_t stream, const void* A, const void* B, int M, int N, int K, float* C, int ldc, float alpha,
                 const float* true_score, const int* true_col, int* rank_out) {
  const CUtensorMap ma = make_map("gemm_nt", A, M, K, BM, KIND);
  const CUtensorMap mb = make_map("gemm_nt", B, N, K, BN, KIND);
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
  // split-K: few output tiles and a long K extent (e.g. the G^T E0 gradient GEMM of the shared-negative SGNS step:
  // 1024 x 304 x 32768 = 24 tiles) - spread the k-blocks of a tile over gridDim.z CTAs that add their partial tiles
  // into the zeroed C.
  if (EPI == EPI_STORE) {
    const int total_kb = (K + BK<KIND> - 1) / BK<KIND>;
    const long tiles = (long)grid.x * grid.y;
    int splits = 1;
    if (tiles * 2 <= num_sms() && total_kb >= 32) splits = (int)std::min<long>(num_sms() / tiles, total_kb / 8);
    splits = std::max(1, std::min(splits, std::min(total_kb, 64)));
    if (splits > 1) {
      const int kb_per = (total_kb + splits - 1) / splits;
      splits = (total_kb + kb_per - 1) / kb_per;          // no empty split
      ADAPM_CUDA_CHECK(cudaMemset2DAsync(C, (size_t)ldc * sizeof(float), 0, (size_t)N * sizeof(float), (size_t)M, stream));
      grid.z = (unsigned)splits;
    }
  }
  launch<gemm_nt_wgmma_kernel<EPI, KIND>, Ring<STAGES>>(grid, stream, ma, mb, M, N, K, C, ldc, alpha, true_score, true_col,
                                                        rank_out);
}

}  // namespace

void gemm_nt_bf16(cudaStream_t stream, const void* A, const void* B, int M, int N, int K, float* C, int ldc) {
  if (M == 0 || N == 0) return;
  launch_gemm<EPI_STORE, KIND_BF16>(stream, A, B, M, N, K, C, ldc, 1.f, nullptr, nullptr, nullptr);
}

// fp8 (e4m3) operands, fp32 accumulation, C = alpha * A B^T  (alpha = product of the per-tensor scales)
void gemm_nt_e4m3(cudaStream_t stream, const void* A, const void* B, int M, int N, int K, float* C, int ldc, float alpha) {
  if (M == 0 || N == 0) return;
  launch_gemm<EPI_STORE, KIND_E4M3>(stream, A, B, M, N, K, C, ldc, alpha, nullptr, nullptr, nullptr);
}

void gemm_nt_bf16_rank_count(cudaStream_t stream, const void* A, const void* B, int M, int N, int K,
                             const float* true_score, const int* true_col, int* rank_out) {
  if (M == 0 || N == 0) return;
  launch_gemm<EPI_RANK_COUNT, KIND_BF16>(stream, A, B, M, N, K, nullptr, 0, 1.f, true_score, true_col, rank_out);
}

}  // namespace cudaops
}  // namespace adapm

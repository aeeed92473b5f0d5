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
#include <cstdlib>

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
  constexpr int BK = KIND == KIND_BF16 ? 64 : 128;   // elements per 128-byte K-block row
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  SmemLayout& sm = *reinterpret_cast<SmemLayout*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tile_n = blockIdx.x, tile_m = blockIdx.y;
  // split-K (gridDim.z > 1, EPI_STORE only): this CTA accumulates k-blocks [kb0, kb0 + num_kb) and ADDS its partial tile
  // to C, which the host zeroed - for problems with few output tiles and a long K extent
  const int total_kb = (K + BK - 1) / BK;
  const int kb_per = (total_kb + (int)gridDim.z - 1) / (int)gridDim.z;
  const int kb0 = (int)blockIdx.z * kb_per;
  const int num_kb = min(kb_per, total_kb - kb0);
  if (num_kb <= 0) return;          // (uniform for the CTA)

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&sm.full_bar[s], 1); mbar_init(&sm.empty_bar[s], kConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_b) : "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % STAGES;
        const uint32_t ph = (uint32_t)(kb / STAGES) & 1u;
        mbar_wait(&sm.empty_bar[s], ph ^ 1u);  // first pass over the ring passes immediately
        mbar_expect_tx(&sm.full_bar[s], A_BYTES + B_BYTES);
        tma_load_2d(sm.a[s], &tmap_a, &sm.full_bar[s], (kb0 + kb) * BK, tile_m * BM);
        tma_load_2d(sm.b[s], &tmap_b, &sm.full_bar[s], (kb0 + kb) * BK, tile_n * BN);
      }
    }
  } else {
    // ===================== consumers: wgmma -> registers -> C / counts =====================
    const int wg = (warp >> 2) - 1;
    float d[64];
    consume_ring<KIND>(sm, num_kb, wg, lane, d);
    const int row0 = tile_m * BM + wg * 64 + (warp & 3) * 16;
    const int col0 = tile_n * BN;
    if (EPI == EPI_STORE) store_fragment(d, alpha, C, ldc, row0, col0, M, N, lane, gridDim.z > 1);
    else rank_count_fragment(d, true_score, true_col, rank_out, row0, col0, M, N, lane);
  }
}

template <int EPI, int KIND>
void launch(cudaStream_t stream, const void* A, const void* B, int M, int N, int K, float* C, int ldc, float alpha,
            const float* true_score, const int* true_col, int* rank_out) {
  ADAPM_CHECK((K * (KIND == KIND_BF16 ? 2 : 1)) % 16 == 0, "gemm_nt: the K extent must be a multiple of 16 bytes (TMA row pitch)");
  ADAPM_CHECK((((uintptr_t)A) & 15u) == 0 && (((uintptr_t)B) & 15u) == 0, "gemm_nt: operands must be 16-byte aligned");
  CUtensorMap ma = make_map(A, M, K, BM, KIND);
  CUtensorMap mb = make_map(B, N, K, BN, KIND);
  const size_t smem = sizeof(SmemLayout) + 1024;
  static bool attr_set = false;
  static int num_sms = 0;
  if (!attr_set) {
    ADAPM_CUDA_CHECK(cudaFuncSetAttribute(gemm_nt_wgmma_kernel<EPI, KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int dev = 0;
    ADAPM_CUDA_CHECK(cudaGetDevice(&dev));
    ADAPM_CUDA_CHECK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    attr_set = true;
  }
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
  // split-K: few output tiles and a long K extent (e.g. the G^T E0 gradient GEMM of the shared-negative SGNS step:
  // 1024 x 304 x 32768 = 24 tiles) - spread the k-blocks of a tile over gridDim.z CTAs that add their partial tiles
  // into the zeroed C. ADAPM_GEMM_SPLITK=<n> forces n splits (1 = off).
  if (EPI == EPI_STORE) {
    static const int split_env = [] { const char* e = getenv("ADAPM_GEMM_SPLITK"); return e ? atoi(e) : 0; }();
    const int BKh = KIND == KIND_BF16 ? 64 : 128;
    const int total_kb = (K + BKh - 1) / BKh;
    const long tiles = (long)grid.x * grid.y;
    int splits = 1;
    if (split_env > 0) splits = split_env;
    else if (tiles * 2 <= num_sms && total_kb >= 32) splits = (int)std::min<long>(num_sms / tiles, total_kb / 8);
    splits = std::max(1, std::min(splits, std::min(total_kb, 64)));
    if (splits > 1) {
      const int kb_per = (total_kb + splits - 1) / splits;
      splits = (total_kb + kb_per - 1) / kb_per;          // no empty split
      ADAPM_CUDA_CHECK(cudaMemset2DAsync(C, (size_t)ldc * sizeof(float), 0, (size_t)N * sizeof(float), (size_t)M, stream));
      grid.z = (unsigned)splits;
    }
  }
  gemm_nt_wgmma_kernel<EPI, KIND><<<grid, kGemmThreads, smem, stream>>>(ma, mb, M, N, K, C, ldc, alpha, true_score,
                                                                        true_col, rank_out);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace

void gemm_nt_bf16(cudaStream_t stream, const void* A, const void* B, int M, int N, int K, float* C, int ldc) {
  if (M == 0 || N == 0) return;
  launch<EPI_STORE, KIND_BF16>(stream, A, B, M, N, K, C, ldc, 1.f, nullptr, nullptr, nullptr);
}

// fp8 (e4m3) operands, fp32 accumulation, C = alpha * A B^T  (alpha = product of the per-tensor scales)
void gemm_nt_e4m3(cudaStream_t stream, const void* A, const void* B, int M, int N, int K, float* C, int ldc, float alpha) {
  if (M == 0 || N == 0) return;
  launch<EPI_STORE, KIND_E4M3>(stream, A, B, M, N, K, C, ldc, alpha, nullptr, nullptr, nullptr);
}

void gemm_nt_bf16_rank_count(cudaStream_t stream, const void* A, const void* B, int M, int N, int K,
                             const float* true_score, const int* true_col, int* rank_out) {
  if (M == 0 || N == 0) return;
  launch<EPI_RANK_COUNT, KIND_BF16>(stream, A, B, M, N, K, nullptr, 0, 1.f, true_score, true_col, rank_out);
}

}  // namespace cudaops
}  // namespace adapm

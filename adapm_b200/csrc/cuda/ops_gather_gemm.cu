// Fused parameter gather + tensor-core GEMM (sm_90a): the "Intent-prefetch all-gather (+) consumer GEMM"
// hot path of the north star. Scores C[M, N] = Q[M, K] x E[keys[0..N), 0..K)^T where the rows of E are
// NOT a dense matrix: they live in the parameter store, spread over the HBM of all GPUs. Producer warps
// resolve each key through the replicated directory, read the fp32 embedding rows straight from the local
// slab / local replica / a peer GPU over NVLink (16-byte loads on peer-mapped pointers), convert to bf16
// and write them into the 128-byte-swizzled K-major shared-memory layout that wgmma consumes - in the
// same kernel as the wgmma tiles, overlapped with them through an mbarrier ring. The query tile arrives
// through TMA. Epilogues: STORE (fp32 scores) or RANK_COUNT (filtered-ranking evaluation of the KGE models:
// the [M x N] score matrix and the gathered entity matrix never exist in HBM).
//
// Warpgroup roles (384 threads): 0 row gatherers (thread 0 also issues the TMA of Q) | 1-2 wgmma consumers + epilogue.
#include <cuda_runtime.h>

#include "ops.h"
#include "pm_kernels.cuh"
#include "wgmma_utils.cuh"

namespace adapm {
namespace cudaops {

namespace {

using namespace tc;

enum GEpilogue : int { G_STORE = 0, G_RANK_COUNT = 1 };

template <int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gather_gemm_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ Ctx c,
                   const Key* __restrict__ keys, int M, int N, int K, float* __restrict__ C, int ldc,
                   const float* __restrict__ true_score, const int* __restrict__ true_col, int* __restrict__ rank_out,
                   unsigned long long* __restrict__ stats) {
  Ring<STAGES>& r = smem_as<Ring<STAGES>>();
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tile_n = blockIdx.x, tile_m = blockIdx.y;
  const int num_kb = (K + BK<KIND_BF16> - 1) / BK<KIND_BF16>;
  dev::cta_enter(c);   // the gather warps read store rows through the directory: count this CTA in the grace epoch

  if (threadIdx.x == 0) {
    r.init(5);   // full: the TMA of the Q tile + one arrival per gather warp
    prefetch_tensormap(&tmap_q);
  }
  __syncthreads();

  uint32_t it = 0;
  if (warp < 4) {
    GatherStats st;
    produce_gather(r, tmap_q, c, keys, tile_n * BN, N, K, tile_m * BM, num_kb, it, st);
    st.flush(stats);
  } else {
    // ===================== consumers: wgmma -> registers -> C / counts =====================
    const int wg = (warp >> 2) - 1;
    float d[64];
    consume<KIND_BF16>(r, num_kb, it, false, wg, lane, d);
    const int row0 = tile_m * BM + frag_row0(warp);
    const int col0 = tile_n * BN;
    if (EPI == G_STORE) store_fragment(d, 1.f, C, ldc, row0, col0, M, N, lane, false);
    else rank_count_fragment(d, true_score, true_col, rank_out, row0, col0, M, N, lane);
  }
  dev::cta_exit(c);
}

template <int EPI>
void launch_gather(CudaBackend& be, cudaStream_t stream, const void* Q, const Key* keys, int M, int N, int K, int ldq, float* C,
                   int ldc, const float* true_score, const int* true_col, int* rank_out, unsigned long long* stats) {
  ADAPM_CHECK(K % 4 == 0, "gather_gemm: the embedding length must be a multiple of 4");
  ADAPM_CHECK(ldq >= K, "gather_gemm: Q's row pitch must be at least K");
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  be.track_stream(stream);
  const CUtensorMap mq = make_map("gather_gemm", Q, M, ldq, BM, KIND_BF16);
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
  launch<gather_gemm_kernel<EPI>, Ring<STAGES>>(grid, stream, mq, be.ctx(), keys, M, N, K, C, ldc, true_score, true_col,
                                               rank_out, stats);
}

}  // namespace

void gather_gemm(CudaBackend& be, cudaStream_t stream, const void* Q, const Key* keys, int M, int N, int K, int ldq, float* C,
                 int ldc, unsigned long long* stats) {
  if (M == 0 || N == 0) return;
  launch_gather<G_STORE>(be, stream, Q, keys, M, N, K, ldq, C, ldc, nullptr, nullptr, nullptr, stats);
}

void gather_gemm_rank_count(CudaBackend& be, cudaStream_t stream, const void* Q, const Key* keys, int M, int N, int K, int ldq,
                            const float* true_score, const int* true_col, int* rank_out, unsigned long long* stats) {
  if (M == 0 || N == 0) return;
  launch_gather<G_RANK_COUNT>(be, stream, Q, keys, M, N, K, ldq, nullptr, 0, true_score, true_col, rank_out, stats);
}

}  // namespace cudaops
}  // namespace adapm

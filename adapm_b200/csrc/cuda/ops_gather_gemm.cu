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

constexpr int BK_ELEMS = 64;  // bf16 elements per 128-byte K-block row

enum GEpilogue : int { G_STORE = 0, G_RANK_COUNT = 1 };

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

template <int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gather_gemm_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ Ctx c,
                   const Key* __restrict__ keys, int M, int N, int K, float* __restrict__ C, int ldc,
                   const float* __restrict__ true_score, const int* __restrict__ true_col, int* __restrict__ rank_out,
                   unsigned long long* __restrict__ stats) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  SmemLayout& sm = *reinterpret_cast<SmemLayout*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tile_n = blockIdx.x, tile_m = blockIdx.y;
  const int num_kb = (K + BK_ELEMS - 1) / BK_ELEMS;
  dev::cta_enter(c);   // the gather warps read store rows through the directory: count this CTA in the grace epoch

  if (threadIdx.x == 0) {
    // full: 1 arrival (TMA expect_tx for the Q tile) + 4 arrivals (one per gather warp)
    for (int s = 0; s < STAGES; ++s) { mbar_init(&sm.full_bar[s], 5); mbar_init(&sm.empty_bar[s], kConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_q) : "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== gatherers: store rows (local HBM / NVLink peers) -> swizzled smem; thread 0 also TMAs Q ==
    const int t = threadIdx.x;                // tile row handled by this thread (0..127)
    const int n = tile_n * BN + t;
    const float* row = nullptr;
    unsigned nl = 0, nr = 0;
    if (n < N) {
      const Key key = keys[n];
      const int cls = class_of_key(c, key);
      for (int attempt = 0; attempt < 4096 && !row; ++attempt) {
        dev::Target tg = dev::resolve_fast(c, key, cls, &nl, &nr);
        row = tg.row;
        if (!row) __nanosleep(256);            // transitional slot (relocation in flight): retry
      }
    }
    for (int kb = 0; kb < num_kb; ++kb) {
      const int s = kb % STAGES;
      const uint32_t ph = (uint32_t)(kb / STAGES) & 1u;
      mbar_wait(&sm.empty_bar[s], ph ^ 1u);
      if (t == 0) {
        mbar_expect_tx(&sm.full_bar[s], A_BYTES);
        tma_load_2d(sm.a[s], &tmap_q, &sm.full_bar[s], kb * BK_ELEMS, tile_m * BM);
      }
      unsigned char* dst_row = sm.b[s] + (size_t)t * ROW_BYTES;
      const int k0 = kb * BK_ELEMS;
      // 64 floats of this row -> 8 chunks of 8 bf16; chunk c goes to position c ^ (t & 7)  (128B swizzle)
      float4 v[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int k = k0 + 4 * j;
        v[j] = (row && k < K) ? dev::ld_row4(row + k) : make_float4(0.f, 0.f, 0.f, 0.f);  // K % 4 == 0
      }
#pragma unroll
      for (int ch = 0; ch < 8; ++ch) {
        uint4 o;
        o.x = pack_bf16(v[2 * ch].x, v[2 * ch].y);
        o.y = pack_bf16(v[2 * ch].z, v[2 * ch].w);
        o.z = pack_bf16(v[2 * ch + 1].x, v[2 * ch + 1].y);
        o.w = pack_bf16(v[2 * ch + 1].z, v[2 * ch + 1].w);
        *reinterpret_cast<uint4*>(dst_row + ((ch ^ (t & 7)) << 4)) = o;
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> visible to the tensor core
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.full_bar[s]);
    }
    if (stats) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) { nl += __shfl_xor_sync(0xffffffffu, nl, o); nr += __shfl_xor_sync(0xffffffffu, nr, o); }
      if (lane == 0) {
        if (nl) atomicAdd(stats + 0, (unsigned long long)nl);
        if (nr) atomicAdd(stats + 1, (unsigned long long)nr);
      }
    }
  } else {
    // ===================== consumers: wgmma -> registers -> C / counts =====================
    const int wg = (warp >> 2) - 1;
    float d[64];
    consume_ring<KIND_BF16>(sm, num_kb, wg, lane, d);
    const int row0 = tile_m * BM + wg * 64 + (warp & 3) * 16;
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
  ADAPM_CHECK(ldq % 8 == 0 && ldq >= K, "gather_gemm: Q must be bf16 with a row pitch that is a multiple of 8 elements");
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  be.track_stream(stream);
  CUtensorMap mq = make_map(Q, M, ldq, BM, KIND_BF16);
  const size_t smem = sizeof(SmemLayout) + 1024;
  static bool attr_set = false;
  if (!attr_set) {
    ADAPM_CUDA_CHECK(cudaFuncSetAttribute(gather_gemm_kernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set = true;
  }
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
  gather_gemm_kernel<EPI><<<grid, kGemmThreads, smem, stream>>>(mq, be.ctx(), keys, M, N, K, C, ldc, true_score, true_col,
                                                                  rank_out, stats);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
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

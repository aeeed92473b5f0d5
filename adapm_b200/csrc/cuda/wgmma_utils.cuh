// wgmma / TMA / mbarrier building blocks shared by the Hopper tensor-core kernels
// (ops_gemm_wgmma.cu, ops_gather_gemm.cu). Raw PTX only - no CUTLASS.
//
// Tile: 128 x 128 output per CTA, three warpgroups (384 threads). Warpgroup 0 fills the shared-memory ring (TMA or,
// in the fused gather kernel, row gatherers); warpgroups 1 and 2 are the consumers, each owning 64 rows of the tile
// with a wgmma.m64n128 accumulator in registers (64 fp32 per thread).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "group.cuh"
#include "../adapm/log.h"

namespace adapm {
namespace cudaops {
namespace tc {

constexpr int BM = 128, BN = 128;
constexpr int ROW_BYTES = 128;                // one K-block row = 128 B = one swizzle-128B row
constexpr int MMA_K_BYTES = 32;               // one wgmma consumes 32 B of K per row (16 bf16 / 32 fp8)
constexpr int STAGES = 6;
constexpr int A_BYTES = BM * ROW_BYTES;       // 16 KiB
constexpr int B_BYTES = BN * ROW_BYTES;       // 16 KiB
enum Kind : int { KIND_BF16 = 0, KIND_E4M3 = 1 };
constexpr int kGemmThreads = 384;             // producer warpgroup + 2 consumer warpgroups
constexpr int kConsumerWarps = 8;             // one empty-barrier arrival per consumer warp

struct SmemLayout {
  alignas(1024) unsigned char a[STAGES][A_BYTES];
  alignas(1024) unsigned char b[STAGES][B_BYTES];
  alignas(8) unsigned long long full_bar[STAGES];
  alignas(8) unsigned long long empty_bar[STAGES];
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, unsigned long long* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}

// wgmma shared-memory matrix descriptor (sm_90): K-major operand, 128-byte swizzle, 8-row groups 1024 B apart.
// Advancing the start address by 32 B selects the next K slice inside the swizzled 128-byte row.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);        // start address            bits [0,14)
  d |= (uint64_t)1 << 16;                              // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;                    // stride byte offset       bits [32,46)
  d |= (uint64_t)1 << 62;                              // layout type: SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x 128] (fp32, registers) += A[64 x K-slice] * B[128 x K-slice]^T, both operands from shared memory
template <int KIND>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  if constexpr (KIND == KIND_BF16) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
        "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(1));
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
        "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(1));
  }
}

// Consumer warpgroup `wg` (0 or 1): accumulate its 64 rows of the tile over k-blocks [0, num_kb) of the ring.
// A stage is released (one arrival per consumer warp) once the wgmmas that read it have retired; wait_group<1> keeps
// the MMAs of one k-block in flight while the next k-block is issued.
template <int KIND>
__device__ __forceinline__ void consume_ring(SmemLayout& sm, int num_kb, int wg, int lane, float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = 0.f;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % STAGES;
    mbar_wait(&sm.full_bar[s], (uint32_t)(kb / STAGES) & 1u);
    const uint32_t a_addr = smem_u32(sm.a[s]) + (uint32_t)(wg * 64 * ROW_BYTES);
    const uint32_t b_addr = smem_u32(sm.b[s]);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < ROW_BYTES / MMA_K_BYTES; ++k)
      wgmma_m64n128<KIND>(d, wgmma_desc(a_addr + k * MMA_K_BYTES), wgmma_desc(b_addr + k * MMA_K_BYTES));
    wgmma_commit();
    wgmma_wait<1>();
    if (kb > 0 && lane == 0) mbar_arrive(&sm.empty_bar[(kb - 1) % STAGES]);
  }
  wgmma_wait<0>();
}

// Accumulator fragment of wgmma m64nN (fp32): thread (warp w of the warpgroup, lane l) holds, for j in [0, N/8),
// d[4j + 2h + e] = D[16 w + l / 4 + 8 h][8 j + 2 (l % 4) + e]   (h, e in {0, 1}).
// STORE epilogue: alpha * D -> C (or added to C when `add`, the split-K case; the host zeroed C).
__device__ __forceinline__ void store_fragment(const float (&d)[64], float alpha, float* C, int ldc, int row0, int col0,
                                               int M, int N, int lane, bool add) {
  const bool vec2 = !add && (ldc & 1) == 0 && (reinterpret_cast<uintptr_t>(C) & 7u) == 0;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + (lane >> 2) + 8 * h;
    if (row >= M) continue;
    float* crow = C + (size_t)row * ldc;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int col = col0 + 8 * j + 2 * (lane & 3);
      const float v0 = alpha * d[4 * j + 2 * h], v1 = alpha * d[4 * j + 2 * h + 1];
      if (add) {
        if (col < N) atomicAdd(crow + col, v0);
        if (col + 1 < N) atomicAdd(crow + col + 1, v1);
      } else if (vec2 && col + 1 < N) {
        *reinterpret_cast<float2*>(crow + col) = make_float2(v0, v1);
      } else {
        if (col < N) crow[col] = v0;
        if (col + 1 < N) crow[col + 1] = v1;
      }
    }
  }
}

// RANK_COUNT epilogue: per row, count the columns (other than the row's true column) whose score beats the row's true
// score, and add the count to rank_out[row]. The four lanes that share a row combine their counts first.
__device__ __forceinline__ void rank_count_fragment(const float (&d)[64], const float* __restrict__ true_score,
                                                    const int* __restrict__ true_col, int* __restrict__ rank_out, int row0,
                                                    int col0, int M, int N, int lane) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + (lane >> 2) + 8 * h;
    float ts = 0.f;
    int tcol = -1, cnt = 0;
    if (row < M) { ts = true_score[row]; tcol = true_col[row]; }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = col0 + 8 * j + 2 * (lane & 3) + e;
        cnt += (col < N && col != tcol && d[4 * j + 2 * h + e] > ts) ? 1 : 0;
      }
    }
    cnt += __shfl_xor_sync(0xffffffffu, cnt, 1);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, 2);
    if ((lane & 3) == 0 && row < M && cnt) atomicAdd(rank_out + row, cnt);
  }
}


// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    ADAPM_CHECK(e == cudaSuccess && qres == cudaDriverEntryPointSuccess && p, "cuTensorMapEncodeTiled is not available");
    return (EncodeTiledFn)p;
  }();
  return fn;
}

// row-major [rows, cols] matrix of 2-byte (bf16) or 1-byte (e4m3) elements,
// box = [box_rows, 128 bytes of K], 128-byte swizzle
inline CUtensorMap make_map(const void* base, int64_t rows, int64_t cols, int box_rows, int kind) {
  CUtensorMap m;
  const int esz = kind == KIND_BF16 ? 2 : 1;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * esz};
  cuuint32_t box[2] = {(cuuint32_t)(ROW_BYTES / esz), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = encode_fn()(&m, kind == KIND_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2,
                           const_cast<void*>(base), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  ADAPM_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with code " << (int)r);
  return m;
}


}  // namespace tc
}  // namespace cudaops
}  // namespace adapm

// The tile pipeline of the Hopper tensor-core kernels (ops_gemm_wgmma.cu, ops_kge_1vsall.cu, ops_gather_gemm.cu,
// ops_topk.cu): shared-memory ring, producers, consumer, epilogues and launch. Raw PTX only - no CUTLASS.
//
// Tile: 128 x 128 output per CTA, three warpgroups (384 threads). Warpgroup 0 fills the shared-memory ring (one TMA
// thread, or four warps of row gatherers); warpgroups 1 and 2 are the consumers, each owning 64 rows of the tile with a
// wgmma.m64n128 accumulator in registers (64 fp32 per thread).
//
// Ring protocol. A stage holds one 128-byte k-block of the A and the B tile. Its full barrier completes when the stage
// is loaded (1 arrival, the TMA expect_tx; 5 when the four gather warps arrive too), its empty barrier when all 8
// consumer warps have released it. Producer and consumers count k-blocks with one running counter `it` over all tiles
// of the CTA: stage it % S, parity (it / S) & 1; the producer waits for the opposite parity on the empty barrier, so
// its first pass over the ring does not wait.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "cuda_backend.h"
#include "group.cuh"
#include "mbarrier.cuh"
#include "pm_kernels.cuh"
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
template <int KIND>
constexpr int BK = KIND == KIND_BF16 ? 64 : 128;   // elements per 128-byte K-block row
constexpr int kGemmThreads = 384;             // producer warpgroup + 2 consumer warpgroups
constexpr int kConsumerWarps = 8;             // one empty-barrier arrival per consumer warp

template <int S>
struct Ring {
  alignas(1024) unsigned char a[S][A_BYTES];
  alignas(1024) unsigned char b[S][B_BYTES];
  alignas(8) unsigned long long full_bar[S];
  alignas(8) unsigned long long empty_bar[S];

  __device__ __forceinline__ static int stage(uint32_t it) { return (int)(it % S); }
  __device__ __forceinline__ static uint32_t parity(uint32_t it) { return (it / S) & 1u; }

  // thread 0, before the CTA's first barrier: full barriers complete on `full_arrivals` arrivals, empty ones on one
  // arrival per consumer warp
  __device__ __forceinline__ void init(uint32_t full_arrivals) {
    for (int s = 0; s < S; ++s) { mbar_init(&full_bar[s], full_arrivals); mbar_init(&empty_bar[s], kConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
};

// The kernel's dynamic shared memory as a T at its first 1024-byte boundary (the 128-byte swizzle of TMA and wgmma
// wants 1024-byte aligned stages); launch() asks for sizeof(T) + 1024 bytes.
template <class T>
__device__ __forceinline__ T& smem_as() {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  return *reinterpret_cast<T*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
}

__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
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

// TMA producer (one thread): k-blocks [kb0, kb0 + num_kb) of the A tile at row a_row and the B tile at row b_row into
// the ring, continuing the running counter `it`.
template <int KIND, int S>
__device__ __forceinline__ void produce_tma(Ring<S>& r, const CUtensorMap& tmap_a, const CUtensorMap& tmap_b, int a_row,
                                            int b_row, int kb0, int num_kb, uint32_t& it) {
  for (int kb = kb0; kb < kb0 + num_kb; ++kb, ++it) {
    const int s = Ring<S>::stage(it);
    mbar_wait(&r.empty_bar[s], Ring<S>::parity(it) ^ 1u);
    mbar_expect_tx(&r.full_bar[s], A_BYTES + B_BYTES);
    tma_load_2d(r.a[s], &tmap_a, &r.full_bar[s], kb * BK<KIND>, a_row);
    tma_load_2d(r.b[s], &tmap_b, &r.full_bar[s], kb * BK<KIND>, b_row);
  }
}

// Consumer warpgroup `wg` (0 or 1): accumulate its 64 rows of one tile over the next num_kb (>= 1) k-blocks of the ring,
// continuing the running counter `it`. A stage is released (one arrival per consumer warp) once the wgmmas that read it
// have retired: wait_group<1> keeps the MMAs of one k-block in flight while the next k-block is issued. The tile's last
// stage is released after wait_group<0> when more tiles follow on the ring; a kernel of one tile per CTA skips that
// arrival, which nobody waits for and which cost the rank-count GEMM about 5 % at 16384 x 14951 x 512 (H100 80GB HBM3,
// 700 W).
template <int KIND, int S>
__device__ __forceinline__ void consume(Ring<S>& r, int num_kb, uint32_t& it, bool more_tiles, int wg, int lane,
                                        float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = 0.f;
  for (int kb = 0; kb < num_kb; ++kb, ++it) {
    const int s = Ring<S>::stage(it);
    mbar_wait(&r.full_bar[s], Ring<S>::parity(it));
    const uint32_t a_addr = smem_u32(r.a[s]) + (uint32_t)(wg * 64 * ROW_BYTES);
    const uint32_t b_addr = smem_u32(r.b[s]);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < ROW_BYTES / MMA_K_BYTES; ++k)
      wgmma_m64n128<KIND>(d, wgmma_desc(a_addr + k * MMA_K_BYTES), wgmma_desc(b_addr + k * MMA_K_BYTES));
    wgmma_commit();
    wgmma_wait<1>();
    if (kb > 0 && lane == 0) mbar_arrive(&r.empty_bar[Ring<S>::stage(it - 1)]);
  }
  wgmma_wait<0>();
  if (more_tiles && lane == 0) mbar_arrive(&r.empty_bar[Ring<S>::stage(it - 1)]);
}

// First of the 16 tile rows whose accumulator fragment consumer warp `warp` (4 .. 11) holds.
__device__ __forceinline__ int frag_row0(int warp) { return ((warp >> 2) - 1) * 64 + (warp & 3) * 16; }

// Split-K over gridDim.z: split blockIdx.z takes k-blocks [kb0, kb0 + num_kb) of total_kb (num_kb <= 0: none).
struct KRange { int kb0, num_kb; };
__device__ __forceinline__ KRange k_split(int total_kb) {
  const int kb_per = (total_kb + (int)gridDim.z - 1) / (int)gridDim.z;
  const int kb0 = (int)blockIdx.z * kb_per;
  return {kb0, min(kb_per, total_kb - kb0)};
}

// One output tile of A B^T on a STAGES-deep ring: the TMA producer loads k-blocks [kb0, kb0 + num_kb) of the A rows from
// a_row and the B rows from b_row, the consumer warpgroups accumulate them. Returns true in the consumer threads, with
// their fragment in d (rows from frag_row0); false in all threads when num_kb <= 0.
template <int KIND>
__device__ __forceinline__ bool tma_tile(const CUtensorMap& tmap_a, const CUtensorMap& tmap_b, int a_row, int b_row,
                                         int kb0, int num_kb, float (&d)[64]) {
  if (num_kb <= 0) return false;   // (uniform for the CTA)
  Ring<STAGES>& r = smem_as<Ring<STAGES>>();
  if (threadIdx.x == 0) {
    r.init(1);
    prefetch_tensormap(&tmap_a);
    prefetch_tensormap(&tmap_b);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5;
  uint32_t it = 0;
  if (warp >= 4) {
    consume<KIND>(r, num_kb, it, false, (warp >> 2) - 1, threadIdx.x & 31, d);
    return true;
  }
  if (threadIdx.x == 0) produce_tma<KIND>(r, tmap_a, tmap_b, a_row, b_row, kb0, num_kb, it);
  return false;
}

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// Gather thread t: k-block [k0, k0 + 64) of its store row -> bf16 -> row t of the swizzled K-major B tile (zeros past K
// or for a null row; K % 4 == 0).
__device__ __forceinline__ void stage_row_bf16(unsigned char* tile, const Ctx& c, Key key, dev::GatherRow& row, int t,
                                               int k0, int K) {
  unsigned char* dst_row = tile + (size_t)t * ROW_BYTES;
  float4 v[16];
  do {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int k = k0 + 4 * j;
      v[j] = (row.row && k < K) ? dev::ld_gather4(row, k) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  } while (dev::gather_reread(c, key, row));
  // 8 chunks of 8 bf16; chunk c goes to position c ^ (t & 7)  (128-byte swizzle)
#pragma unroll
  for (int ch = 0; ch < 8; ++ch) {
    uint4 o;
    o.x = pack_bf16(v[2 * ch].x, v[2 * ch].y);
    o.y = pack_bf16(v[2 * ch].z, v[2 * ch].w);
    o.z = pack_bf16(v[2 * ch + 1].x, v[2 * ch + 1].y);
    o.w = pack_bf16(v[2 * ch + 1].z, v[2 * ch + 1].w);
    *reinterpret_cast<uint4*>(dst_row + ((ch ^ (t & 7)) << 4)) = o;
  }
}

// Row counts of a gather thread: stats[0..2] += (local rows, peer rows, unresolved rows staged as zeros), summed over
// the warp. (dev::flush_stats takes its slow-path count as warp-uniform; the unresolved count here is per thread.)
struct GatherStats {
  unsigned local = 0, remote = 0, unresolved = 0;
  __device__ __forceinline__ void flush(unsigned long long* stats) {
    if (!stats) return;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      local += __shfl_xor_sync(0xffffffffu, local, o); remote += __shfl_xor_sync(0xffffffffu, remote, o);
      unresolved += __shfl_xor_sync(0xffffffffu, unresolved, o);
    }
    if ((threadIdx.x & 31) == 0) {
      if (local) atomicAdd(stats + 0, (unsigned long long)local);
      if (remote) atomicAdd(stats + 1, (unsigned long long)remote);
      if (unresolved) atomicAdd(stats + 2, (unsigned long long)unresolved);
    }
  }
};

// Gather producer, warps 0-3: thread t stages row t of the B tile, the store row of keys[n0 + t] (local HBM, replica or
// NVLink peer; zeros past N), over the next num_kb k-blocks of the ring, continuing the running counter `it`; thread 0
// also loads the Q tile at row q_row by TMA. A full barrier takes the TMA and one arrival per gather warp (init 5).
template <int S>
__device__ __forceinline__ void produce_gather(Ring<S>& r, const CUtensorMap& tmap_q, const Ctx& c, const Key* keys,
                                               int n0, int N, int K, int q_row, int num_kb, uint32_t& it,
                                               GatherStats& st) {
  const int t = threadIdx.x;
  const int n = n0 + t;
  const Key key = n < N ? keys[n] : 0;
  dev::GatherRow row = {nullptr, nullptr, nullptr, nullptr, 0u, false};
  if (n < N) {
    row.row = dev::resolve_fast(c, key, class_of_key(c, key), &st.local, &st.remote).row;
    if (!row.row) {                          // transitional slot (relocation in flight)
      row = dev::gather_locate(c, key);
      if (!row.row) ++st.unresolved; else if (row.local) ++st.local; else ++st.remote;
    }
  }
  for (int kb = 0; kb < num_kb; ++kb, ++it) {
    const int s = Ring<S>::stage(it);
    mbar_wait(&r.empty_bar[s], Ring<S>::parity(it) ^ 1u);
    if (t == 0) {
      mbar_expect_tx(&r.full_bar[s], A_BYTES);
      tma_load_2d(r.a[s], &tmap_q, &r.full_bar[s], kb * BK<KIND_BF16>, q_row);
    }
    stage_row_bf16(r.b[s], c, key, row, t, kb * BK<KIND_BF16>, K);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> visible to the tensor core
    __syncwarp();
    if ((t & 31) == 0) mbar_arrive(&r.full_bar[s]);
  }
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

// row-major [rows, cols] matrix of 2-byte (bf16) or 1-byte (e4m3) elements, rows `pitch` elements apart (0: cols),
// box = [box_rows, 128 bytes of K], 128-byte swizzle. `op` names the caller in the error for an operand that TMA cannot
// read: its base must be 16-byte aligned and its row pitch a multiple of 16 bytes. Columns past cols read as zeros.
inline CUtensorMap make_map(const char* op, const void* base, int64_t rows, int64_t cols, int box_rows, int kind,
                            int64_t pitch = 0) {
  CUtensorMap m;
  const int esz = kind == KIND_BF16 ? 2 : 1;
  if (pitch == 0) pitch = cols;
  ADAPM_CHECK((reinterpret_cast<uintptr_t>(base) & 15u) == 0 && (pitch * esz) % 16 == 0 && pitch >= cols,
              op << ": tensor-core operands must be 16-byte aligned, with rows a multiple of 16 bytes long");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)pitch * esz};
  cuuint32_t box[2] = {(cuuint32_t)(ROW_BYTES / esz), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = encode_fn()(&m, kind == KIND_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2,
                           const_cast<void*>(base), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  ADAPM_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with code " << (int)r);
  return m;
}

// SM count of the device current at the first call, read once per process
inline int num_sms() {
  static const int n = [] {
    int dev = 0, v = 0;
    ADAPM_CUDA_CHECK(cudaGetDevice(&dev));
    ADAPM_CUDA_CHECK(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev));
    return v;
  }();
  return n;
}

// Launches a tile kernel whose shared memory is a Smem (smem_as): 384-thread CTAs, the kernel's dynamic shared memory
// limit raised once per process, the launch counted and checked.
template <auto Kernel, class Smem, class... Args>
void launch(dim3 grid, cudaStream_t stream, const Args&... args) {
  const size_t smem = sizeof(Smem) + 1024;
  set_max_dynamic_smem<Kernel>((int)smem);
  Kernel<<<grid, kGemmThreads, smem, stream>>>(args...);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace tc
}  // namespace cudaops
}  // namespace adapm

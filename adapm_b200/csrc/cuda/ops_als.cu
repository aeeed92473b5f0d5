// Alternating least squares (ALS) for matrix factorisation on sm_90a: one CTA per target row gathers the target's
// other-side rows from the store (local HBM, replicas, NVLink peers, keys in flight), accumulates its normal equations
// in fp32 and solves them by Cholesky in registers and shared memory.
//
// Rule (target t with entries e = (other key o_e, a_e, b_e); h_e the factor half of row o_e; rows [factors (rank) |
// AdaGrad (rank)]):
//   A_t = G + lam I + sum_e a_e h_e h_e^T,  r_t = sum_e b_e h_e,  w_t <- A_t^{-1} r_t
// pushed as [w_new - w_old | 0] (the AdaGrad half is left as it is). A half-step writes only target rows and reads only
// other-side rows, so the values a CTA reads do not change while it runs, and every sum is taken in a fixed order: the
// result of a target does not depend on the CTA that solves it, on the order of the targets or on where the rows live.
//
// Layout of the work: 256 threads; the lower triangle of A (padded to KP x KP, KP in {32, 64, 128}) is a 16 x 16 grid
// of TM x TM register tiles (TM = KP / 16), of which the 136 lower ones (diagonal tiles included) belong to threads
// 0..135. Entries are staged kChunk rows at a time in shared memory; per entry, a tile thread adds a_e h_i h_j to its
// TM^2 accumulators (entry order). The accumulators stay in registers through the factorisation: right-looking
// Cholesky, one column per step (the owners of column j publish it, every tile thread subtracts l_j l_j^T from its
// tile), with r carried along as the forward substitution; L goes column by column to shared memory for the back
// substitution (one warp, fixed-order dot products). A pivot <= 0 (or NaN) leaves the target unchanged: it is not
// counted as solved.
//
// The Gram kernel sums h h^T over a key range with the same staging and tiles: one partial per kGramRows keys, then
// the partials are added in index order, so G is bit-identical from call to call and on every rank.
#include <cuda_runtime.h>

#include <algorithm>

#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {

namespace {

constexpr int kThreads = 256;
constexpr int kChunk = 32;            // other-side rows staged per pass (one resolving thread each: warp 0)
constexpr int kTiles = 16 * 17 / 2;   // lower register tiles of the 16 x 16 grid
constexpr int kGramRows = 1024;       // keys per partial of the Gram kernel (fixed: it sets the summation order)

template <int KP>
struct Smem {
  static constexpr int TM = KP / 16;
  // [KP * KP] staged rows (kChunk x KP) during the gather, L column-major (row j = column j of L) afterwards; then
  // the slow path's staged target row
  static constexpr size_t kMat = (size_t)KP * KP;
  static constexpr size_t bytes() {
    return kMat * sizeof(float) + 5 * KP * sizeof(float) + 2 * kChunk * sizeof(float) + kChunk * sizeof(dev::GatherRow);
  }
};

struct SmemPtrs {
  float* mat;
  float *colv, *rv, *yv, *xv, *diag;
  float *sa, *sb;
  dev::GatherRow* gr;
};

template <int KP>
__device__ __forceinline__ SmemPtrs smem_ptrs(unsigned char* base) {
  SmemPtrs p;
  float* f = reinterpret_cast<float*>(base);
  p.mat = f; f += Smem<KP>::kMat;
  p.colv = f; f += KP;
  p.rv = f; f += KP;
  p.yv = f; f += KP;
  p.xv = f; f += KP;
  p.diag = f; f += KP;
  p.sa = f; f += kChunk;
  p.sb = f; f += kChunk;
  p.gr = reinterpret_cast<dev::GatherRow*>(f);
  return p;
}

// lower tile t (< kTiles) -> (block row bi, block column bj), bi >= bj
__device__ __forceinline__ void tile_of(int t, int& bi, int& bj) {
  bi = 0;
  while ((bi + 1) * (bi + 2) / 2 <= t) ++bi;
  bj = t - bi * (bi + 1) / 2;
}

template <int TM>
__device__ __forceinline__ void lds(const float* p, float (&v)[TM]) {
  if constexpr (TM % 4 == 0) {
#pragma unroll
    for (int i = 0; i < TM / 4; ++i) {
      const float4 q = reinterpret_cast<const float4*>(p)[i];
      v[4 * i] = q.x; v[4 * i + 1] = q.y; v[4 * i + 2] = q.z; v[4 * i + 3] = q.w;
    }
  } else {
#pragma unroll
    for (int i = 0; i < TM / 2; ++i) {
      const float2 q = reinterpret_cast<const float2*>(p)[i];
      v[2 * i] = q.x; v[2 * i + 1] = q.y;
    }
  }
}

struct Counts {
  unsigned local, remote, slow;
  bool unresolved;
};

// Stages the factor halves of keys[0 .. cnt) (cnt <= kChunk) into mat[kChunk][KP], zero-padded past rank and past
// cnt. Thread e < cnt resolves key e: resolve_fast, else gather_locate (three-way read of a key in flight). Ends with
// the stage visible to the CTA.
template <int KP>
__device__ __forceinline__ void stage_chunk(const Ctx& c, const Key* keys, int cnt, int rank, const SmemPtrs& s,
                                            Counts& n) {
  const int tid = threadIdx.x;
  if (tid < cnt) {
    const Key key = keys[tid];
    dev::GatherRow row = {nullptr, nullptr, nullptr, nullptr, 0u, false};
    row.row = dev::resolve_fast(c, key, class_of_key(c, key), &n.local, &n.remote).row;
    if (!row.row) {
      row = dev::gather_locate(c, key);
      ++n.slow;
      if (!row.row) n.unresolved = true;
    }
    s.gr[tid] = row;
  }
  __syncthreads();
  constexpr int nv = KP / 4;
  for (int idx = tid; idx < kChunk * nv; idx += kThreads) {
    const int e = idx / nv, j = idx % nv;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (e < cnt && 4 * j < rank) {
      dev::GatherRow row = s.gr[e];
      if (row.row) {
        do {
          v = dev::ld_gather4(row, 4 * j);
        } while (dev::gather_reread(c, keys[e], row));
      }
    }
    reinterpret_cast<float4*>(s.mat + (size_t)e * KP)[j] = v;
  }
  __syncthreads();
}

// acc += sum over the staged entries e of sa[e] h_e[rows] h_e[cols]^T (tile threads), racc += sb[e] h_e[ri] (RHS)
template <int KP, bool RHS>
__device__ __forceinline__ void accumulate(const SmemPtrs& s, int bi, int bj, bool tile, int ri,
                                           float (&acc)[KP / 16][KP / 16], float& racc) {
  constexpr int TM = KP / 16;
  if (tile) {
#pragma unroll 4
    for (int e = 0; e < kChunk; ++e) {
      float u[TM], v[TM];
      lds<TM>(s.mat + (size_t)e * KP + bi * TM, u);
      lds<TM>(s.mat + (size_t)e * KP + bj * TM, v);
      const float ae = s.sa[e];
#pragma unroll
      for (int ii = 0; ii < TM; ++ii) {
        const float w = ae * u[ii];
#pragma unroll
        for (int jj = 0; jj < TM; ++jj) acc[ii][jj] = fmaf(w, v[jj], acc[ii][jj]);
      }
    }
  }
  if (RHS && ri >= 0) {
    for (int e = 0; e < kChunk; ++e) racc = fmaf(s.sb[e], s.mat[(size_t)e * KP + ri], racc);
  }
}

struct SolveArgs {
  const Key* targets;
  const int64_t* offsets;
  const Key* others;
  const float* a;
  const float* b;
  const float* gram;     // [rank, rank] or null
  int rank;
  float lam;
};

template <int KP>
__global__ void __launch_bounds__(kThreads, 2)
als_solve_kernel(const __grid_constant__ Ctx c, const __grid_constant__ SolveArgs A, unsigned long long* __restrict__ stats) {
  constexpr int TM = KP / 16;
  extern __shared__ __align__(16) unsigned char als_smem[];
  const SmemPtrs s = smem_ptrs<KP>(als_smem);
  __shared__ int s_bad;
  __shared__ dev::Target s_tg;
  // the CTA reads rows through the directory until its push: it counts in the sync round's grace period meanwhile
  dev::cta_enter(c);
  const int tid = threadIdx.x, lane = tid & 31, rank = A.rank;
  const bool tile = tid < kTiles;
  int bi = 0, bj = 0;
  if (tile) tile_of(tid, bi, bj);
  const int ri = tid >= kThreads - KP && tid - (kThreads - KP) < rank ? tid - (kThreads - KP) : -1;
  const int64_t e0 = A.offsets[blockIdx.x], e1 = A.offsets[blockIdx.x + 1];
  float acc[TM][TM];
#pragma unroll
  for (int ii = 0; ii < TM; ++ii)
#pragma unroll
    for (int jj = 0; jj < TM; ++jj) acc[ii][jj] = 0.f;
  float racc = 0.f;
  Counts n = {0u, 0u, 0u, false};
  if (tid == 0) s_bad = 0;

  // ---- A = sum_e a_e h_e h_e^T, r = sum_e b_e h_e, kChunk entries at a time in entry order
  for (int64_t base = e0; base < e1; base += kChunk) {
    const int cnt = e1 - base < kChunk ? (int)(e1 - base) : kChunk;
    if (tid < kChunk) {
      s.sa[tid] = tid < cnt ? A.a[base + tid] : 0.f;
      s.sb[tid] = tid < cnt ? A.b[base + tid] : 0.f;
    }
    stage_chunk<KP>(c, A.others + base, cnt, rank, s, n);
    accumulate<KP, true>(s, bi, bj, tile, ri, acc, racc);
    __syncthreads();
  }
  if (n.unresolved) s_bad = 1;

  // ---- + G + lam I (lower triangle), r to shared memory
  if (tile) {
#pragma unroll
    for (int ii = 0; ii < TM; ++ii)
#pragma unroll
      for (int jj = 0; jj < TM; ++jj) {
        const int i = bi * TM + ii, l = bj * TM + jj;
        if (i < rank && l <= i) {
          if (A.gram) acc[ii][jj] += A.gram[(size_t)i * rank + l];
          if (i == l) acc[ii][jj] += A.lam;
        }
      }
  }
  if (tid < KP) s.rv[tid] = 0.f;
  __syncthreads();
  if (ri >= 0) s.rv[ri] = racc;

  // ---- Cholesky A = L L^T with the forward substitution L y = r, one column per step
  bool failed = false;
  for (int j = 0; j < rank; ++j) {
    // the owners of column j publish it (rows >= j of their tiles)
    if (tile && bj == j / TM) {
      const int jm = j % TM;
#pragma unroll
      for (int jj = 0; jj < TM; ++jj)
        if (jj == jm) {
#pragma unroll
          for (int ii = 0; ii < TM; ++ii) s.colv[bi * TM + ii] = acc[ii][jj];
        }
    }
    __syncthreads();
    const float piv = s.colv[j];
    if (!(piv > 0.f)) { failed = true; break; }   // uniform: every thread read the same pivot
    const float d = sqrtf(piv);
    if (tid < KP) s.mat[(size_t)j * KP + tid] = tid < j || tid >= rank ? 0.f : (tid == j ? d : s.colv[tid] / d);
    if (tid == j) { s.diag[j] = d; s.yv[j] = s.rv[j] / d; }
    __syncthreads();
    const float* Lj = s.mat + (size_t)j * KP;
    if (tile) {
      float u[TM], v[TM];
      lds<TM>(Lj + bi * TM, u);
      lds<TM>(Lj + bj * TM, v);
#pragma unroll
      for (int ii = 0; ii < TM; ++ii)
#pragma unroll
        for (int jj = 0; jj < TM; ++jj) acc[ii][jj] = fmaf(-u[ii], v[jj], acc[ii][jj]);
    }
    if (tid > j && tid < rank) s.rv[tid] = fmaf(-Lj[tid], s.yv[j], s.rv[tid]);
  }
  __syncthreads();

  // ---- back substitution L^T x = y (warp 0), then the push [x - w_old | 0]
  if (tid < 32 && !failed && !s_bad) {
    for (int j = rank - 1; j >= 0; --j) {
      float t = 0.f;
      for (int i = j + 1 + lane; i < rank; i += 32) t = fmaf(s.mat[(size_t)j * KP + i], s.xv[i], t);
      t = dev::warp_sum(t);
      const float xj = (s.yv[j] - t) / s.diag[j];
      if (lane == 0) s.xv[j] = xj;
      __syncwarp();
    }
    if (lane == 0) {
      unsigned dl = 0, dr = 0;
      const Key key = A.targets[blockIdx.x];
      s_tg = dev::resolve_fast(c, key, class_of_key(c, key), &dl, &dr);
    }
    __syncwarp();
  }
  __syncthreads();
  bool pushed = false;
  if (!failed && !s_bad) {
    float* row = s_tg.row;
    if (row) {
      for (int j = tid; j < rank / 4; j += kThreads) {
        const float4 w = dev::ld_row4(row + 4 * j);
        dev::red_row4(row + 4 * j, make_float4(s.xv[4 * j] - w.x, s.xv[4 * j + 1] - w.y, s.xv[4 * j + 2] - w.z,
                                               s.xv[4 * j + 3] - w.w));
      }
      __syncthreads();
      if (tid == 0) dev::mark_pushed(s_tg);
      pushed = true;
    } else if (tid < 32) {
      // a target in a transitional protocol state: stage it through the generic Pull / Push (shared memory)
      const Key key = A.targets[blockIdx.x];
      float* st = s.mat;
      if (lane == 0) ++n.slow;
      if (dev::slow_pull(c, key, st)) {
        for (int i = lane; i < 2 * rank; i += 32) st[i] = i < rank ? s.xv[i] - st[i] : 0.f;
        pushed = dev::slow_push(c, key, st);
      }
    }
  }

  // ---- stats: the resolving threads are warp 0
  if (tid < 32) {
    unsigned sl = n.local, sr = n.remote, ss = n.slow;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sl += __shfl_xor_sync(0xffffffffu, sl, o);
      sr += __shfl_xor_sync(0xffffffffu, sr, o);
      ss += __shfl_xor_sync(0xffffffffu, ss, o);
    }
    if (lane == 0 && stats) {
      if (sl) atomicAdd(stats + 0, (unsigned long long)sl);
      if (sr) atomicAdd(stats + 1, (unsigned long long)sr);
      if (ss) atomicAdd(stats + 2, (unsigned long long)ss);
      if (pushed) atomicAdd(stats + 3, 1ull);
    }
  }
  dev::cta_exit(c);
}

// partial Gram matrix of keys [blockIdx.x * kGramRows, ...): lower tiles of sum h h^T into part[blockIdx.x][KP][KP]
template <int KP>
__global__ void __launch_bounds__(kThreads, 2)
als_gram_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ keys, int64_t n, int rank, float* __restrict__ part) {
  constexpr int TM = KP / 16;
  extern __shared__ __align__(16) unsigned char als_smem[];
  const SmemPtrs s = smem_ptrs<KP>(als_smem);
  dev::cta_enter(c);
  const int tid = threadIdx.x;
  const bool tile = tid < kTiles;
  int bi = 0, bj = 0;
  if (tile) tile_of(tid, bi, bj);
  float acc[TM][TM];
#pragma unroll
  for (int ii = 0; ii < TM; ++ii)
#pragma unroll
    for (int jj = 0; jj < TM; ++jj) acc[ii][jj] = 0.f;
  float racc = 0.f;
  Counts cn = {0u, 0u, 0u, false};
  const int64_t e0 = (int64_t)blockIdx.x * kGramRows, e1 = n < e0 + kGramRows ? n : e0 + kGramRows;
  for (int64_t base = e0; base < e1; base += kChunk) {
    const int cnt = e1 - base < kChunk ? (int)(e1 - base) : kChunk;
    if (tid < kChunk) s.sa[tid] = tid < cnt ? 1.f : 0.f;
    stage_chunk<KP>(c, keys + base, cnt, rank, s, cn);
    accumulate<KP, false>(s, bi, bj, tile, -1, acc, racc);
    __syncthreads();
  }
  if (tile) {
    float* out = part + (size_t)blockIdx.x * KP * KP;
#pragma unroll
    for (int ii = 0; ii < TM; ++ii)
#pragma unroll
      for (int jj = 0; jj < TM; ++jj) out[(size_t)(bi * TM + ii) * KP + bj * TM + jj] = acc[ii][jj];
  }
  dev::cta_exit(c);
}

// G[i][j] = sum over the partials p in index order of part[p][max(i, j)][min(i, j)]: symmetric by construction
__global__ void als_gram_reduce_kernel(const float* __restrict__ part, int nparts, int KP, int rank, float* __restrict__ G) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rank * rank) return;
  const int i = idx / rank, j = idx % rank;
  const size_t off = (size_t)max(i, j) * KP + min(i, j);
  float t = 0.f;
  for (int p = 0; p < nparts; ++p) t += part[(size_t)p * KP * KP + off];
  G[idx] = t;
}

template <int KP>
void launch_solve(cudaStream_t stream, int n, const Ctx& c, const SolveArgs& A, unsigned long long* stats) {
  set_max_dynamic_smem<als_solve_kernel<KP>>((int)Smem<KP>::bytes());
  als_solve_kernel<KP><<<n, kThreads, Smem<KP>::bytes(), stream>>>(c, A, stats);
}

template <int KP>
void launch_gram(cudaStream_t stream, int blocks, const Ctx& c, const Key* keys, int64_t n, int rank, float* part) {
  set_max_dynamic_smem<als_gram_kernel<KP>>((int)Smem<KP>::bytes());
  als_gram_kernel<KP><<<blocks, kThreads, Smem<KP>::bytes(), stream>>>(c, keys, n, rank, part);
}

int padded_rank(int rank) { return rank <= 32 ? 32 : rank <= 64 ? 64 : 128; }

void check_rank(int rank, const char* op) {
  ADAPM_CHECK(rank % 4 == 0 && rank >= 4 && rank <= kAlsMaxRank,
              op << ": rank must be a multiple of 4 in [4, " << kAlsMaxRank << "]");
}

}  // namespace

void als_solve(CudaBackend& be, cudaStream_t stream, const Key* targets, const int64_t* offsets, const Key* others,
               const float* a, const float* b, int n, int rank, float lam, const float* gram,
               unsigned long long* stats) {
  if (n == 0) return;
  check_rank(rank, "als_solve");
  ADAPM_CHECK(lam > 0.f, "als_solve: lam must be > 0");
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  be.track_stream(stream);
  const Ctx& c = be.ctx();
  SolveArgs A;
  A.targets = targets; A.offsets = offsets; A.others = others; A.a = a; A.b = b; A.gram = gram; A.rank = rank;
  A.lam = lam;
  switch (padded_rank(rank)) {
    case 32: launch_solve<32>(stream, n, c, A, stats); break;
    case 64: launch_solve<64>(stream, n, c, A, stats); break;
    default: launch_solve<128>(stream, n, c, A, stats); break;
  }
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

void als_gram(CudaBackend& be, cudaStream_t stream, const Key* keys, int64_t n, int rank, float* G) {
  check_rank(rank, "als_gram");
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  be.track_stream(stream);
  const Ctx& c = be.ctx();
  const int KP = padded_rank(rank);
  const int blocks = (int)((n + kGramRows - 1) / kGramRows);
  float* part = nullptr;
  if (blocks > 0) {
    part = static_cast<float*>(be.step_buffer(CudaBackend::kStepBuffers - 1, (size_t)blocks * KP * KP * sizeof(float)));
    switch (KP) {
      case 32: launch_gram<32>(stream, blocks, c, keys, n, rank, part); break;
      case 64: launch_gram<64>(stream, blocks, c, keys, n, rank, part); break;
      default: launch_gram<128>(stream, blocks, c, keys, n, rank, part); break;
    }
    ADAPM_COUNT_LAUNCH();
    ADAPM_CUDA_CHECK(cudaGetLastError());
  }
  als_gram_reduce_kernel<<<(rank * rank + 255) / 256, 256, 0, stream>>>(part, blocks, KP, rank, G);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

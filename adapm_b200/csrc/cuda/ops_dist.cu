// Distance ranking and top-k against parameter-store rows on the CUDA cores (sm_90a), for translational models (TransE,
// RotatE):
//     D(i, j) = |q_i - e_j|_p,  p = 1 or 2,  e_j = first `dim` values of store row keys[j]  [/ max(|e_j|_2, 1e-12)]
//     D(i, j) = sum_k sqrt((q_2k - e_2k)^2 + (q_2k+1 - e_2k+1)^2)  (p = kDistComplex: complex moduli of interleaved
//               (re, im) rows, never normalised)
// without an [M, N] distance matrix. L1 has no tensor-core form, and the L2 expansion |q|^2 - 2 q.e + |e|^2 loses too
// much in bf16 to count ranks, so the distances are fp32 sums on the CUDA cores.
//
// Every distance is summed by one thread over k = 0 .. dim-1 (pairs k = 0 .. dim/2-1) in order with explicitly rounded
// operations, and every row
// norm by four threads in a fixed pattern, so D(i, j) is bit-identical whichever CTA (or the true-distance kernel)
// computes it.
//
// Grid: (M tiles of 64 queries) x (S column slices); CTA (m, s) runs the 64-column tiles s, s + S, ... Four threads per
// tile row gather the candidate rows through the directory (resolve_fast, else gather_locate with the three-way read for
// keys in flight), as the gather GEMM kernels do; the CTA counts in the sync round's grace epoch for all its tiles, and
// the host bounds the tiles per CTA on several ranks. Rows that cannot be resolved are read as zeros and counted in
// stats[2].
//   dist_rank_kernel   raw[i] += #{j != true_col[i] : D(i, j) < Dt[i]}, filt[i] the same without the row's exclusions;
//                      Dt[i] = D(i, true_col[i]) from dist_true_kernel (the same distance function)
//   dist_topk_kernel   running per-row lists of (-D, column), ties to the smaller column, NaN never selected; sorted
//                      partial lists [M, S, k] that topk_merge (ops_topk.cu) merges
#include <cuda_runtime.h>

#include <algorithm>

#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {

namespace {

constexpr int DB = 64;                 // queries and candidates per tile
constexpr int DKC = 32;                // floats of a row per chunk
constexpr int kDistThreads = 256;      // 16 x 16 threads, 4 x 4 distances each
constexpr int DLSTRIDE = kTopkMax + 1;
constexpr uint32_t NO_COL = 0xFFFFFFFFu;
constexpr int kMaxSlices = 2048;
constexpr float kNormEps = 1e-12f;

struct DistArgs {
  const float* q;                      // [M, dim]
  const Key* keys;                     // [N]
  int M, N, dim, p, k, S;
  bool normalize;
  const int64_t* ex_off;               // [M + 1] or null
  const int64_t* ex_cols;
  const int64_t* true_col;             // rank count: [M]
  const float* dtrue;                  // [M]
  int64_t* raw;                        // [M]
  int64_t* filt;
  float* part_v;                       // top-k: [M, S, k]
  int* part_c;
};

struct DistSmem {
  float qs[DKC][DB];
  float es[DKC][DB];
};
struct TopkLists {
  float v[DB][DLSTRIDE];
  uint32_t c[DB][DLSTRIDE];
  float thr_v[DB];
  uint32_t thr_c[DB];
  int worst[DB];
};

// the row of `key` for a gather thread; nl / nr / nu count local, peer and unresolved rows
__device__ __forceinline__ dev::GatherRow gather_row(const Ctx& c, Key key, unsigned& nl, unsigned& nr, unsigned& nu) {
  dev::GatherRow row = {nullptr, nullptr, nullptr, nullptr, 0u, false};
  row.row = dev::resolve_fast(c, key, class_of_key(c, key), &nl, &nr).row;
  if (!row.row) {
    row = dev::gather_locate(c, key);
    if (!row.row) ++nu; else if (row.local) ++nl; else ++nr;
  }
  return row;
}

// 1 / max(|row[0, dim)|_2, eps) by the four threads g = 0..3 of a group of consecutive lanes: thread g sums the squares
// of float4 g, g + 4, ... in order, then a fixed butterfly over the group (the same value in all four)
__device__ __forceinline__ float group_inv_norm(const Ctx& c, Key key, dev::GatherRow& row, int dim, int g) {
  float s;
  do {
    s = 0.f;
    if (row.row)
      for (int f = g; 4 * f < dim; f += 4) {
        const float4 v = dev::ld_gather4(row, 4 * f);
        s = __fadd_rn(s, __fadd_rn(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)),
                                   __fadd_rn(__fmul_rn(v.z, v.z), __fmul_rn(v.w, v.w))));
      }
  } while (dev::gather_reread(c, key, row));
  s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 1));
  s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 2));
  return __frcp_rn(fmaxf(__fsqrt_rn(s), kNormEps));
}

// one term of a distance sum
template <int P>
__device__ __forceinline__ float dterm(float acc, float q, float e) {
  const float df = __fsub_rn(q, e);
  return P == 1 ? __fadd_rn(acc, fabsf(df)) : __fmaf_rn(df, df, acc);
}
template <int P>
__device__ __forceinline__ float dfinish(float acc) { return P == 2 ? __fsqrt_rn(acc) : acc; }
// one term of a complex-modulus sum: acc + |(q0 - e0) + i (q1 - e1)|
__device__ __forceinline__ float cterm(float acc, float q0, float e0, float q1, float e1) {
  const float d0 = __fsub_rn(q0, e0), d1 = __fsub_rn(q1, e1);
  return __fadd_rn(acc, __fsqrt_rn(__fmaf_rn(d0, d0, __fmul_rn(d1, d1))));
}

__device__ __forceinline__ bool beats(float v, uint32_t c, float tv, uint32_t tc) {
  return v > tv || (v == tv && c < tc);
}

__device__ __forceinline__ bool excluded(const DistArgs& a, int row, int64_t col) {
  if (!a.ex_off) return false;
  int64_t lo = a.ex_off[row];
  const int64_t end = a.ex_off[row + 1];
  int64_t hi = end;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a.ex_cols[mid] < col) lo = mid + 1; else hi = mid;
  }
  return lo < end && a.ex_cols[lo] == col;
}

// The 64 x 64 distances of column tile tn: d[a][b] = D(m0 + 4 ty + a, tn * 64 + 4 tx + b). Gather threads: tile row
// r = tid / 4, part g = tid % 4 (float4 2g and 2g + 1 of each chunk).
template <int P>
__device__ __forceinline__ void dist_tile(DistSmem& sm, const Ctx& c, const DistArgs& a, int m0, int tn, float (&d)[4][4],
                                          unsigned& nl, unsigned& nr, unsigned& nu) {
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15, r = tid >> 2, g = tid & 3;
  const int n = tn * DB + r;
  const Key key = n < a.N ? a.keys[n] : 0;
  unsigned dl = 0, dr = 0, du = 0;
  dev::GatherRow row = {nullptr, nullptr, nullptr, nullptr, 0u, false};
  if (n < a.N) row = gather_row(c, key, dl, dr, du);
  if (g == 0) { nl += dl; nr += dr; nu += du; }
  const float inv = a.normalize ? group_inv_norm(c, key, row, a.dim, g) : 1.f;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) d[i][j] = 0.f;
  for (int k0 = 0; k0 < a.dim; k0 += DKC) {
    __syncthreads();   // the previous chunk's readers are done
    // queries: 64 rows x 8 float4 of the chunk, two per thread
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int idx = tid + h * kDistThreads, qr = idx >> 3, f = idx & 7, kk = k0 + 4 * f;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m0 + qr < a.M && kk < a.dim) v = __ldg(reinterpret_cast<const float4*>(a.q + (size_t)(m0 + qr) * a.dim + kk));
      sm.qs[4 * f][qr] = v.x; sm.qs[4 * f + 1][qr] = v.y; sm.qs[4 * f + 2][qr] = v.z; sm.qs[4 * f + 3][qr] = v.w;
    }
    float4 v0, v1;
    do {
      const int kk0 = k0 + 8 * g, kk1 = kk0 + 4;
      v0 = (row.row && kk0 < a.dim) ? dev::ld_gather4(row, kk0) : make_float4(0.f, 0.f, 0.f, 0.f);
      v1 = (row.row && kk1 < a.dim) ? dev::ld_gather4(row, kk1) : make_float4(0.f, 0.f, 0.f, 0.f);
    } while (dev::gather_reread(c, key, row));
    if (a.normalize) {
      v0 = make_float4(__fmul_rn(v0.x, inv), __fmul_rn(v0.y, inv), __fmul_rn(v0.z, inv), __fmul_rn(v0.w, inv));
      v1 = make_float4(__fmul_rn(v1.x, inv), __fmul_rn(v1.y, inv), __fmul_rn(v1.z, inv), __fmul_rn(v1.w, inv));
    }
    sm.es[8 * g][r] = v0.x; sm.es[8 * g + 1][r] = v0.y; sm.es[8 * g + 2][r] = v0.z; sm.es[8 * g + 3][r] = v0.w;
    sm.es[8 * g + 4][r] = v1.x; sm.es[8 * g + 5][r] = v1.y; sm.es[8 * g + 6][r] = v1.z; sm.es[8 * g + 7][r] = v1.w;
    __syncthreads();
    const int kn = min(DKC, a.dim - k0);
    if (P == kDistComplex) {
      for (int kk = 0; kk < kn; kk += 2) {
        const float4 q0 = *reinterpret_cast<const float4*>(&sm.qs[kk][4 * ty]);
        const float4 e0 = *reinterpret_cast<const float4*>(&sm.es[kk][4 * tx]);
        const float4 q1 = *reinterpret_cast<const float4*>(&sm.qs[kk + 1][4 * ty]);
        const float4 e1 = *reinterpret_cast<const float4*>(&sm.es[kk + 1][4 * tx]);
        const float qa[4] = {q0.x, q0.y, q0.z, q0.w}, ea[4] = {e0.x, e0.y, e0.z, e0.w};
        const float qb[4] = {q1.x, q1.y, q1.z, q1.w}, eb[4] = {e1.x, e1.y, e1.z, e1.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) d[i][j] = cterm(d[i][j], qa[i], ea[j], qb[i], eb[j]);
      }
      continue;
    }
    for (int kk = 0; kk < kn; ++kk) {
      const float4 qv = *reinterpret_cast<const float4*>(&sm.qs[kk][4 * ty]);
      const float4 ev = *reinterpret_cast<const float4*>(&sm.es[kk][4 * tx]);
      const float qa[4] = {qv.x, qv.y, qv.z, qv.w}, ea[4] = {ev.x, ev.y, ev.z, ev.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) d[i][j] = dterm<P>(d[i][j], qa[i], ea[j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) d[i][j] = dfinish<P>(d[i][j]);
}

__device__ __forceinline__ void flush_stats(unsigned long long* stats, unsigned nl, unsigned nr, unsigned nu) {
  if (!stats) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    nl += __shfl_xor_sync(0xffffffffu, nl, o); nr += __shfl_xor_sync(0xffffffffu, nr, o);
    nu += __shfl_xor_sync(0xffffffffu, nu, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (nl) atomicAdd(stats + 0, (unsigned long long)nl);
    if (nr) atomicAdd(stats + 1, (unsigned long long)nr);
    if (nu) atomicAdd(stats + 2, (unsigned long long)nu);
  }
}

// Dt[i] = D(i, true_col[i]) with the distance function of the tiles: four threads per query, thread 0 of the group sums
template <int P>
__device__ __forceinline__ void dist_true_run(const Ctx& c, const DistArgs& a, float* __restrict__ dtrue,
                                              unsigned long long* __restrict__ stats) {
  dev::cta_enter(c);
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 2, g = threadIdx.x & 3;
  unsigned nl = 0, nr = 0, nu = 0;
  const bool in = i < a.M;
  const Key key = in ? a.keys[a.true_col[i]] : 0;
  dev::GatherRow row = {nullptr, nullptr, nullptr, nullptr, 0u, false};
  if (in) row = gather_row(c, key, nl, nr, nu);
  const float inv = a.normalize ? group_inv_norm(c, key, row, a.dim, g) : 1.f;
  if (in && g == 0) {
    float acc;
    do {
      acc = 0.f;
      for (int k = 0; k < a.dim; k += 4) {
        float4 v = row.row ? dev::ld_gather4(row, k) : make_float4(0.f, 0.f, 0.f, 0.f);
        if (a.normalize)
          v = make_float4(__fmul_rn(v.x, inv), __fmul_rn(v.y, inv), __fmul_rn(v.z, inv), __fmul_rn(v.w, inv));
        const float4 qv = __ldg(reinterpret_cast<const float4*>(a.q + (size_t)i * a.dim + k));
        if (P == kDistComplex) {
          acc = cterm(acc, qv.x, v.x, qv.y, v.y); acc = cterm(acc, qv.z, v.z, qv.w, v.w);
        } else {
          acc = dterm<P>(acc, qv.x, v.x); acc = dterm<P>(acc, qv.y, v.y);
          acc = dterm<P>(acc, qv.z, v.z); acc = dterm<P>(acc, qv.w, v.w);
        }
      }
    } while (dev::gather_reread(c, key, row));
    dtrue[i] = dfinish<P>(acc);
  }
  flush_stats(stats, 0u, 0u, g == 0 ? nu : 0u);   // (the true rows are not counted as gathered rows)
  dev::cta_exit(c);
}

template <int P>
__device__ __forceinline__ void dist_rank_run(const Ctx& c, const DistArgs& a, unsigned long long* __restrict__ stats) {
  __shared__ __align__(16) DistSmem sm;
  dev::cta_enter(c);
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int m0 = blockIdx.x * DB, n_tiles = (a.N + DB - 1) / DB;
  unsigned nl = 0, nr = 0, nu = 0;
  int64_t tcol[4];
  float dt[4];
  unsigned raw[4] = {0u, 0u, 0u, 0u}, filt[4] = {0u, 0u, 0u, 0u};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = m0 + 4 * ty + i;
    tcol[i] = row < a.M ? a.true_col[row] : -1;
    dt[i] = row < a.M ? a.dtrue[row] : __int_as_float(0x7fc00000);   // NaN: counts nothing
  }
  for (int tn = blockIdx.y; tn < n_tiles; tn += a.S) {
    float d[4][4];
    dist_tile<P>(sm, c, a, m0, tn, d, nl, nr, nu);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int64_t col = (int64_t)tn * DB + 4 * tx + j;
        if (col < a.N && col != tcol[i] && d[i][j] < dt[i]) {
          ++raw[i];
          if (!excluded(a, m0 + 4 * ty + i, col)) ++filt[i];
        }
      }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int o = 1; o < 16; o <<= 1) {
      raw[i] += __shfl_xor_sync(0xffffffffu, raw[i], o);
      filt[i] += __shfl_xor_sync(0xffffffffu, filt[i], o);
    }
    const int row = m0 + 4 * ty + i;
    if (tx == 0 && row < a.M) {
      if (raw[i]) atomicAdd(reinterpret_cast<unsigned long long*>(a.raw + row), (unsigned long long)raw[i]);
      if (filt[i]) atomicAdd(reinterpret_cast<unsigned long long*>(a.filt + row), (unsigned long long)filt[i]);
    }
  }
  flush_stats(stats, nl, nr, nu);
  dev::cta_exit(c);
}

// (v, col) replaces the worst entry of list r if it still beats it; then the new worst is found
__device__ __forceinline__ void list_insert(TopkLists& L, int k, int r, float v, uint32_t col) {
  if (!beats(v, col, L.thr_v[r], L.thr_c[r])) return;
  const int w0 = L.worst[r];
  L.v[r][w0] = v; L.c[r][w0] = col;
  float wv = L.v[r][0];
  uint32_t wc = L.c[r][0];
  int w = 0;
  for (int i = 1; i < k; ++i) {
    const float x = L.v[r][i];
    const uint32_t xc = L.c[r][i];
    if (beats(wv, wc, x, xc)) { wv = x; wc = xc; w = i; }
  }
  L.worst[r] = w; L.thr_v[r] = wv; L.thr_c[r] = wc;
}

template <int P>
__device__ __forceinline__ void dist_topk_run(const Ctx& c, const DistArgs& a, unsigned long long* __restrict__ stats) {
  extern __shared__ __align__(16) unsigned char dist_smem[];
  DistSmem& sm = *reinterpret_cast<DistSmem*>(dist_smem);
  TopkLists& L = *reinterpret_cast<TopkLists*>(dist_smem + sizeof(DistSmem));
  dev::cta_enter(c);
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int m0 = blockIdx.x * DB, n_tiles = (a.N + DB - 1) / DB;
  for (int i = tid; i < DB * a.k; i += kDistThreads) { L.v[i / a.k][i % a.k] = -INFINITY; L.c[i / a.k][i % a.k] = NO_COL; }
  if (tid < DB) { L.thr_v[tid] = -INFINITY; L.thr_c[tid] = NO_COL; L.worst[tid] = 0; }
  unsigned nl = 0, nr = 0, nu = 0;
  for (int tn = blockIdx.y; tn < n_tiles; tn += a.S) {
    float d[4][4];
    dist_tile<P>(sm, c, a, m0, tn, d, nl, nr, nu);   // (its barriers also order the list initialisation)
    // screen against the row thresholds, then the exclusions; survivors go in one thread of a row at a time
    unsigned mask = 0u;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = 4 * ty + i;
      const float tv = L.thr_v[r];
      const uint32_t tc = L.thr_c[r];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = tn * DB + 4 * tx + j;
        d[i][j] = -d[i][j];
        if (col < a.N && m0 + r < a.M && beats(d[i][j], (uint32_t)col, tv, tc) && !excluded(a, m0 + r, col))
          mask |= 1u << (4 * i + j);
      }
    }
    for (int qq = 0; qq < 16; ++qq) {
      if (tx == qq) {
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (mask >> (4 * i + j) & 1u) list_insert(L, a.k, 4 * ty + i, d[i][j], (uint32_t)(tn * DB + 4 * tx + j));
      }
      __syncwarp();
    }
  }
  __syncthreads();
  // the lists -> part[row, s, 0..k), sorted (rank = number of entries that come first); one warp per 8 rows
  const int warp = tid >> 5, lane = tid & 31;
  for (int r = warp * 8; r < warp * 8 + 8; ++r) {
    const int grow = m0 + r;
    if (grow >= a.M) break;
    for (int i = lane; i < a.k; i += 32) {
      const float v = L.v[r][i];
      const uint32_t cc = L.c[r][i];
      int rank = 0;
      for (int j = 0; j < a.k; ++j) {
        const float x = L.v[r][j];
        const uint32_t xc = L.c[r][j];
        rank += (beats(x, xc, v, cc) || (x == v && xc == cc && j < i)) ? 1 : 0;   // padding entries are all equal
      }
      const size_t o = ((size_t)grow * a.S + blockIdx.y) * a.k + rank;
      a.part_v[o] = v;
      a.part_c[o] = (int)cc;   // NO_COL -> -1
    }
  }
  flush_stats(stats, nl, nr, nu);
  dev::cta_exit(c);
}

// The kernels: L1 / L2 (P = 1, 2) and the complex metric (cdist_*)
template <int P>
__global__ void __launch_bounds__(128)
dist_true_kernel(const __grid_constant__ Ctx c, const __grid_constant__ DistArgs a, float* __restrict__ dtrue,
                 unsigned long long* __restrict__ stats) {
  dist_true_run<P>(c, a, dtrue, stats);
}
template <int P>
__global__ void __launch_bounds__(kDistThreads, 1)
dist_rank_kernel(const __grid_constant__ Ctx c, const __grid_constant__ DistArgs a, unsigned long long* __restrict__ stats) {
  dist_rank_run<P>(c, a, stats);
}
template <int P>
__global__ void __launch_bounds__(kDistThreads, 1)
dist_topk_kernel(const __grid_constant__ Ctx c, const __grid_constant__ DistArgs a, unsigned long long* __restrict__ stats) {
  dist_topk_run<P>(c, a, stats);
}
__global__ void __launch_bounds__(128)
cdist_true_kernel(const __grid_constant__ Ctx c, const __grid_constant__ DistArgs a, float* __restrict__ dtrue,
                  unsigned long long* __restrict__ stats) {
  dist_true_run<kDistComplex>(c, a, dtrue, stats);
}
__global__ void __launch_bounds__(kDistThreads, 1)
cdist_rank_kernel(const __grid_constant__ Ctx c, const __grid_constant__ DistArgs a, unsigned long long* __restrict__ stats) {
  dist_rank_run<kDistComplex>(c, a, stats);
}
__global__ void __launch_bounds__(kDistThreads, 1)
cdist_topk_kernel(const __grid_constant__ Ctx c, const __grid_constant__ DistArgs a, unsigned long long* __restrict__ stats) {
  dist_topk_run<kDistComplex>(c, a, stats);
}

DistArgs make_args(const float* q, const Key* keys, int M, int N, int dim, int p, bool normalize, int S,
                   const int64_t* ex_off, const int64_t* ex_cols) {
  ADAPM_CHECK(dim >= 4 && dim % 4 == 0, "gather_dist: dim must be a positive multiple of 4");
  ADAPM_CHECK(p == 1 || p == 2 || p == kDistComplex, "gather_dist: p must be 1, 2 or kDistComplex");
  ADAPM_CHECK(p != kDistComplex || !normalize, "gather_dist: the complex metric does not normalise rows");
  ADAPM_CHECK(S >= 1 && S <= kMaxSlices, "gather_dist: bad slice count " << S);
  DistArgs a{};
  a.q = q; a.keys = keys; a.M = M; a.N = N; a.dim = dim; a.p = p; a.S = S; a.normalize = normalize;
  a.ex_off = ex_off; a.ex_cols = ex_cols;
  return a;
}

}  // namespace

int dist_num_slices(CudaBackend& be, int M, int N, int max_tiles_per_cta) {
  const int m_tiles = (M + DB - 1) / DB, n_tiles = (N + DB - 1) / DB;
  if (m_tiles == 0 || n_tiles == 0) return 1;
  int S = (4 * be.num_sms() + m_tiles - 1) / m_tiles;   // about four CTAs per SM
  if (max_tiles_per_cta > 0) S = std::max(S, (n_tiles + max_tiles_per_cta - 1) / max_tiles_per_cta);
  return std::max(1, std::min({S, n_tiles, kMaxSlices}));
}

void gather_dist_rank_count(CudaBackend& be, cudaStream_t stream, const float* q, const Key* keys, int M, int N, int dim,
                            int p, bool normalize, int S, const int64_t* true_col, const int64_t* ex_off,
                            const int64_t* ex_cols, float* dtrue, int64_t* raw, int64_t* filt,
                            unsigned long long* stats) {
  if (M == 0) return;
  ADAPM_CHECK(N > 0, "gather_dist_rank_count: no keys");
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  DistArgs a = make_args(q, keys, M, N, dim, p, normalize, S, ex_off, ex_cols);
  a.true_col = true_col; a.dtrue = dtrue; a.raw = raw; a.filt = filt;
  be.track_stream(stream);
  const int tb = (M * 4 + 127) / 128;
  if (p == 1) dist_true_kernel<1><<<tb, 128, 0, stream>>>(be.ctx(), a, dtrue, stats);
  else if (p == 2) dist_true_kernel<2><<<tb, 128, 0, stream>>>(be.ctx(), a, dtrue, stats);
  else cdist_true_kernel<<<tb, 128, 0, stream>>>(be.ctx(), a, dtrue, stats);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
  const dim3 grid((M + DB - 1) / DB, S);
  if (p == 1) dist_rank_kernel<1><<<grid, kDistThreads, 0, stream>>>(be.ctx(), a, stats);
  else if (p == 2) dist_rank_kernel<2><<<grid, kDistThreads, 0, stream>>>(be.ctx(), a, stats);
  else cdist_rank_kernel<<<grid, kDistThreads, 0, stream>>>(be.ctx(), a, stats);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

void gather_dist_topk(CudaBackend& be, cudaStream_t stream, const float* q, const Key* keys, int M, int N, int dim, int p,
                      bool normalize, int k, int S, const int64_t* ex_off, const int64_t* ex_cols, float* part_v,
                      int* part_c, float* out_v, int64_t* out_i, unsigned long long* stats) {
  if (M == 0) return;
  ADAPM_CHECK(N > 0, "gather_dist_topk: no keys");
  ADAPM_CHECK(k >= 1 && k <= kTopkMax, "gather_dist_topk: k must be in [1, " << kTopkMax << "]");
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  DistArgs a = make_args(q, keys, M, N, dim, p, normalize, S, ex_off, ex_cols);
  a.k = k; a.part_v = part_v; a.part_c = part_c;
  be.track_stream(stream);
  const size_t smem = sizeof(DistSmem) + sizeof(TopkLists);
  set_max_dynamic_smem<dist_topk_kernel<1>>((int)smem);
  set_max_dynamic_smem<dist_topk_kernel<2>>((int)smem);
  set_max_dynamic_smem<cdist_topk_kernel>((int)smem);
  const dim3 grid((M + DB - 1) / DB, S);
  if (p == 1) dist_topk_kernel<1><<<grid, kDistThreads, smem, stream>>>(be.ctx(), a, stats);
  else if (p == 2) dist_topk_kernel<2><<<grid, kDistThreads, smem, stream>>>(be.ctx(), a, stats);
  else cdist_topk_kernel<<<grid, kDistThreads, smem, stream>>>(be.ctx(), a, stats);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
  topk_merge(stream, part_v, part_c, M, S, k, out_v, out_i);
}

}  // namespace cudaops
}  // namespace adapm

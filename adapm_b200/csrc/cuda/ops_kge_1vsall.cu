// KGE 1vsAll training for ComplEx and RESCAL: every query of a batch scored against ALL entities, softmax cross-entropy.
//
// A batch of B triples gives 2 B queries; query q < B is the object query of triple q (given s, answer o), query B + i
// the subject query of triple i (given o, answer s). Their query vectors are the ones of KGE._query (complex_query,
// e_s^T R, R e_o), so that score(q, x) = <q, e_x>. With E the N entity vectors and Q the queries:
//
//     Z  [2B, N] = Q E^T                         scores
//     G  [2B, N] = softmax(Z) - onehot(answer)   loss sum_q logsumexp(Z_q) - Z_q,answer
//     dQ [2B, d] = G E                           (K = N: the long contraction)
//     C  [N, d]  = G^T Q                         candidate gradient of every entity
//
// The three contractions run on the wgmma / TMA tiles of wgmma_utils.cuh (bf16 operands, fp32 accumulation); the score
// matrix and G exist only for one chunk of queries at a time. dQ goes back through the query to the given entity and
// the relation (the chain rule of the reference's ComplEx / RESCAL gradients), L2 is added once per triple, and every
// pulled row gets exactly one AdaGrad update [-eta g / sqrt(a + g^2) | g^2] for the caller's single Push.
//
// Determinism: there is no floating-point atomic anywhere. Z runs on gemm_nt_bf16, whose K (d <= 1024, at most 16
// k-blocks) never takes its atomic split-K path. The long contractions run on gemm_partial_kernel: split z of K writes
// its partial tile to a slice of its own and sum_kernel adds the slices in split order; the split count is a function
// of the shape only (partial_splits), so it is the same on every H100. C sums its chunks in chunk order, every reduction (logsumexp, the loss,
// the sum over a row's occurrences) runs in a fixed order, and every output row has one writer. On one GPU the same
// inputs give bit-identical updates and loss. Kernels, in order (per chunk: z GEMM, lse, grad, dq / c GEMMs and sums):
//   gemm_partial_kernel  P[z] = A B^T over split z's k-blocks (gemm_nt_bf16's tile, tc::tma_tile: TMA producer
//                     warpgroup, two wgmma consumer warpgroups)
//   query_kernel      Qf = queries of the pulled rows (fp32), one warp per query
//   to_bf16_kernel    fp32 rows -> bf16 operand [rows, dpad] and its transpose (chunk-major), 32 x 32 tiles
//   row_lse_kernel    per query: logsumexp over the N scores (one warp, fixed order) and its cross-entropy
//   grad_kernel       Z -> G and G^T (bf16), 32 x 32 tiles
//   sum_kernel        out (+)= P[0] + P[1] + ... (split order)
//   given_kernel      per triple: the gradients of s and o through their queries, plus L2
//   entity_kernel     per entity: C + its occurrences in position order -> AdaGrad update
//   relation_kernel   per pulled relation: its triples in order -> AdaGrad update
//   loss_kernel       *loss += the 2 B cross-entropies, summed in a fixed order
//
// Sampled softmax with shared negatives (kge_shared_core) runs the same rule against short lists instead of all
// entities. The batch is padded to Bp = nch * 128 triples (padding triples are masked); chunk k's list is
// [its 128 subjects | its 128 objects | the S negatives] (Lr columns, padded to a multiple of 8), and each of its 256
// queries is scored against its own list only. The pulled rows are the step's distinct entities and relations. Per
// chunk, as one batched launch each (grid dimension z over chunks, every operand at a fixed row stride, all of K in
// one CTA, so no split-K):
//     Z_k  [256, Lr] = Q_k E_k^T,   G_k = softmax - onehot over the live columns,
//     dQ_k [256, d]  = G_k E_k,     C_k [Lr, d] = G_k^T Q_k
// A column is live unless it is a padding slot, or holds the query's answer without being the answer's own slot.
//   gemm_batched_kernel       P[z] = A_z B_z^T (the tile body of gemm_partial_kernel)
//   gather_bf16_kernel        rows by index -> bf16 operand and / or its chunk-major transpose (lists, queries)
//   kge_shared_lse_kernel     per query: logsumexp over the live columns (one warp, fixed order) and its cross-entropy
//   kge_shared_grad_kernel    Z -> G (query order) and G^T (chunk-major, both sides of a chunk along K)
//   kge_shared_entity_kernel  per distinct entity: its list columns of C in (chunk, column) order, then its
//                             given-entity gradients in position order -> AdaGrad update
// with query_kernel, given_kernel, relation_kernel and loss_kernel as above (batch stride Bp).
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>

#include "group.cuh"
#include "ops.h"
#include "wgmma_utils.cuh"

namespace adapm {
namespace cudaops {

namespace {

enum Model : int { COMPLEX = 0, RESCAL = 1 };

// P[blockIdx.z][M][N] (fp32) = A[M, K] x B[N, K]^T (bf16, K-major) over the k-blocks of split blockIdx.z, one 128 x 128
// tile per CTA. The host picks splits so that none is empty.
__global__ void __launch_bounds__(tc::kGemmThreads, 1)
gemm_partial_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, int M, int N,
                    int K, float* __restrict__ P) {
  using namespace tc;
  const int tile_n = blockIdx.x, tile_m = blockIdx.y;
  const KRange kr = k_split((K + BK<KIND_BF16> - 1) / BK<KIND_BF16>);
  float d[64];
  if (tma_tile<KIND_BF16>(tmap_a, tmap_b, tile_m * BM, tile_n * BN, kr.kb0, kr.num_kb, d))
    store_fragment(d, 1.f, P + (size_t)blockIdx.z * M * N, N, tile_m * BM + frag_row0(threadIdx.x >> 5), tile_n * BN, M,
                   N, threadIdx.x & 31, false);
}

// Batched products over all of K: P[z][M][N] (fp32) = A_z [M, K] x B_z [N, K]^T for z = blockIdx.z, where A_z starts at
// row z a_rows of A and B_z at row (z % nb) b_rows of B (bf16, K-major). A tile that runs past a batch's M or N rows
// reads the next batch's rows (or TMA's zero fill) into output rows and columns that are not stored.
__global__ void __launch_bounds__(tc::kGemmThreads, 1)
gemm_batched_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, int M, int N,
                    int K, int a_rows, int b_rows, int nb, float* __restrict__ P) {
  using namespace tc;
  const int tile_n = blockIdx.x, tile_m = blockIdx.y, z = blockIdx.z;
  float d[64];
  if (tma_tile<KIND_BF16>(tmap_a, tmap_b, z * a_rows + tile_m * BM, (z % nb) * b_rows + tile_n * BN, 0,
                          (K + BK<KIND_BF16> - 1) / BK<KIND_BF16>, d))
    store_fragment(d, 1.f, P + (size_t)z * M * N, N, tile_m * BM + frag_row0(threadIdx.x >> 5), tile_n * BN, M, N,
                   threadIdx.x & 31, false);
}

// Splits of K for gemm_partial: about two CTAs per SM of a 132-SM H100, at least 4 k-blocks per split, at most 64
// splits, none empty. A function of the shape only, so that a step gives the same bits on every H100.
int partial_splits(int M, int N, int K) {
  const int total_kb = (K + 63) / 64;
  const long tiles = (long)((N + tc::BN - 1) / tc::BN) * ((M + tc::BM - 1) / tc::BM);
  const int splits = (int)std::max<long>(1, std::min<long>(264 / tiles, std::min(total_kb / 4, 64)));
  const int kb_per = (total_kb + splits - 1) / splits;
  return (total_kb + kb_per - 1) / kb_per;
}

// P[z] (z < partial_splits(M, N, K)) = the product over split z; K a multiple of 8 (16-byte TMA row pitch).
void gemm_partial(cudaStream_t stream, const void* A, const void* B, int M, int N, int K, float* P) {
  const CUtensorMap ma = tc::make_map("kge_1vsall", A, M, K, tc::BM, tc::KIND_BF16);
  const CUtensorMap mb = tc::make_map("kge_1vsall", B, N, K, tc::BN, tc::KIND_BF16);
  const dim3 grid((N + tc::BN - 1) / tc::BN, (M + tc::BM - 1) / tc::BM, partial_splits(M, N, K));
  tc::launch<gemm_partial_kernel, tc::Ring<tc::STAGES>>(grid, stream, ma, mb, M, N, K, P);
}

// P[z] (z < batches) = A_z B_z^T of gemm_batched_kernel; A holds a_total rows and B b_total rows of K values (K a
// multiple of 8: 16-byte TMA row pitch).
void gemm_batched(cudaStream_t stream, const void* A, long a_total, const void* B, long b_total, int M, int N, int K,
                  int a_rows, int b_rows, int nb, int batches, float* P) {
  const CUtensorMap ma = tc::make_map("kge_shared", A, a_total, K, tc::BM, tc::KIND_BF16);
  const CUtensorMap mb = tc::make_map("kge_shared", B, b_total, K, tc::BN, tc::KIND_BF16);
  const dim3 grid((N + tc::BN - 1) / tc::BN, (M + tc::BM - 1) / tc::BM, batches);
  tc::launch<gemm_batched_kernel, tc::Ring<tc::STAGES>>(grid, stream, ma, mb, M, N, K, a_rows, b_rows, nb, P);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One warp per query q < 2 B: Qf[q][0 .. d) in fp32.
template <int MODEL>
__global__ void __launch_bounds__(256)
query_kernel(const float* __restrict__ R, const Key* __restrict__ s, const Key* __restrict__ o,
             const int32_t* __restrict__ rel, int N, int B, int d, float* __restrict__ Qf) {
  const int lane = threadIdx.x & 31;
  const long q = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (q >= 2L * B) return;
  const bool obj = q < B;
  const int i = obj ? (int)q : (int)(q - B);
  const float* a = R + (size_t)(obj ? s[i] : o[i]) * 2 * d;
  const size_t rl = MODEL == COMPLEX ? 2 * (size_t)d : 2 * (size_t)d * d;
  const float* r = R + (size_t)N * 2 * d + (size_t)rel[i] * rl;
  float* out = Qf + (size_t)q * d;
  if (MODEL == COMPLEX) {
    const int h = d / 2;
    for (int j = lane; j < h; j += 32) {
      const float are = a[j], aim = a[h + j], rre = r[j], rim = r[h + j];
      out[j] = obj ? rre * are - rim * aim : rre * are + rim * aim;
      out[h + j] = obj ? rre * aim + rim * are : rre * aim - rim * are;
    }
  } else {
    for (int j = lane; j < d; j += 32) {
      float acc = 0.f;
      if (obj) for (int k = 0; k < d; ++k) acc += a[k] * r[(size_t)k * d + j];     // (e_s^T R)_j
      else for (int k = 0; k < d; ++k) acc += r[(size_t)j * d + k] * a[k];         // (R e_o)_j
      out[j] = acc;
    }
  }
}

// X [n_rows][ldx] fp32 (first d values) -> Xb [rows][dpad] bf16 and XT bf16 in chunks of W rows: row r, column j at
// XT[(r / W) dpad W + j W + r % W]. Rows >= n_rows and columns >= d are zeros. 32 x 8 threads per 32 x 32 tile.
__global__ void __launch_bounds__(256)
to_bf16_kernel(const float* __restrict__ X, int ldx, int n_rows, int rows, int d, int dpad, int W,
               __nv_bfloat16* __restrict__ Xb, __nv_bfloat16* __restrict__ XT) {
  __shared__ __nv_bfloat16 tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int j0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int rl = ty + 8 * k, r = r0 + rl, j = j0 + tx;
    const float x = r < n_rows && j < d ? X[(size_t)r * ldx + j] : 0.f;
    const __nv_bfloat16 b = __float2bfloat16(x);
    if (r < rows && j < dpad) Xb[(size_t)r * dpad + j] = b;
    tile[rl][tx] = b;
  }
  __syncthreads();
  const int r = r0 + tx;
  if (r >= rows) return;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int j = j0 + ty + 8 * k;
    if (j < dpad) XT[(size_t)(r / W) * dpad * W + (size_t)j * W + r % W] = tile[tx][ty + 8 * k];
  }
}

__device__ __forceinline__ Key answer_of(long q, const Key* s, const Key* o, int B) { return q < B ? o[q] : s[q - B]; }

// One warp per chunk row b (query q0 + b): lse[b] = logsumexp of the N scores, qloss[q] = lse - score of the answer.
__global__ void __launch_bounds__(256)
row_lse_kernel(const float* __restrict__ S, int N, int chunk, int q0, int B, const Key* __restrict__ s,
               const Key* __restrict__ o, float* __restrict__ lse, float* __restrict__ qloss) {
  const int lane = threadIdx.x & 31;
  const int b = (int)(((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const long q = (long)q0 + b;
  if (b >= chunk || q >= 2L * B) return;
  const float* z = S + (size_t)b * N;
  float m = -INFINITY;
  for (int j = lane; j < N; j += 32) m = fmaxf(m, z[j]);
  m = warp_max(m);
  float t = 0.f;
  for (int j = lane; j < N; j += 32) t += expf(z[j] - m);
  t = warp_sum(t);
  const float l = m + logf(t);
  if (lane == 0) {
    lse[b] = l;
    qloss[q] = l - z[answer_of(q, s, o, B)];
  }
}

// Z -> G = softmax - onehot: Gb [chunk][Npad] and GbT [N][chunk] (bf16); rows past 2 B and columns past N are zeros.
__global__ void __launch_bounds__(256)
grad_kernel(const float* __restrict__ S, const float* __restrict__ lse, int N, int Npad, int chunk, int q0, int B,
            const Key* __restrict__ s, const Key* __restrict__ o, __nv_bfloat16* __restrict__ Gb,
            __nv_bfloat16* __restrict__ GbT) {
  __shared__ __nv_bfloat16 tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int n0 = blockIdx.x * 32, b0 = blockIdx.y * 32;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int bl = ty + 8 * k, b = b0 + bl, n = n0 + tx;
    const long q = (long)q0 + b;
    float g = 0.f;
    if (q < 2L * B && n < N) g = expf(S[(size_t)b * N + n] - lse[b]) - (answer_of(q, s, o, B) == n ? 1.f : 0.f);
    const __nv_bfloat16 gb = __float2bfloat16(g);
    if (n < Npad) Gb[(size_t)b * Npad + n] = gb;
    tile[bl][tx] = gb;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int n = n0 + ty + 8 * k;
    if (n < N) GbT[(size_t)n * chunk + b0 + tx] = tile[tx][ty + 8 * k];
  }
}

// out[i] = (accumulate ? out[i] : 0) + (P[0][i] + P[1][i] + ... + P[splits - 1][i])
__global__ void __launch_bounds__(256)
sum_kernel(const float* __restrict__ P, int splits, long n, bool accumulate, float* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float t = P[i];
  for (int z = 1; z < splits; ++z) t += P[(size_t)z * n + i];
  out[i] = accumulate ? out[i] + t : t;
}

// One warp per triple i: GS[2 i] = the subject's gradient through the object query + gamma_e e_s, GS[2 i + 1] = the
// object's gradient through the subject query + gamma_e e_o.
template <int MODEL>
__global__ void __launch_bounds__(256)
given_kernel(const float* __restrict__ R, const Key* __restrict__ s, const Key* __restrict__ o,
             const int32_t* __restrict__ rel, const float* __restrict__ dq, int N, int B, int d, int dpad, float gamma_e,
             float* __restrict__ GS) {
  const int lane = threadIdx.x & 31;
  const long i = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= B) return;
  const float* es = R + (size_t)s[i] * 2 * d;
  const float* eo = R + (size_t)o[i] * 2 * d;
  const size_t rl = MODEL == COMPLEX ? 2 * (size_t)d : 2 * (size_t)d * d;
  const float* r = R + (size_t)N * 2 * d + (size_t)rel[i] * rl;
  const float* dqo = dq + (size_t)i * dpad;          // object query of triple i
  const float* dqs = dq + (size_t)(B + i) * dpad;    // subject query
  float* gs = GS + (size_t)(2 * i) * d;
  float* go = gs + d;
  if (MODEL == COMPLEX) {
    const int h = d / 2;
    for (int j = lane; j < h; j += 32) {
      const float rre = r[j], rim = r[h + j];
      const float a = dqo[j], b = dqo[h + j], a2 = dqs[j], b2 = dqs[h + j];
      gs[j] = (rre * a + rim * b) + gamma_e * es[j];
      gs[h + j] = (rre * b - rim * a) + gamma_e * es[h + j];
      go[j] = (rre * a2 - rim * b2) + gamma_e * eo[j];
      go[h + j] = (rim * a2 + rre * b2) + gamma_e * eo[h + j];
    }
  } else {
    for (int j = lane; j < d; j += 32) {
      float ts = 0.f, to = 0.f;
      for (int k = 0; k < d; ++k) {
        ts += r[(size_t)j * d + k] * dqo[k];      // (R dq^o)_j
        to += r[(size_t)k * d + j] * dqs[k];      // (R^T dq^s)_j
      }
      gs[j] = ts + gamma_e * es[j];
      go[j] = to + gamma_e * eo[j];
    }
  }
}

__device__ __forceinline__ void adagrad(float g, float a, float eta, float* u, float* ua) {
  *u = g == 0.f ? 0.f : -eta * g / sqrtf(a + g * g);
  *ua = g * g;
}

// One warp per entity j: g = C[j] + its occurrences GS[p] in position order; U row j = AdaGrad update.
__global__ void __launch_bounds__(256)
entity_kernel(const float* __restrict__ R, const float* __restrict__ C, const float* __restrict__ GS,
              const int64_t* __restrict__ ent_off, const int32_t* __restrict__ ent_pos, int N, int d, int dpad, float eta,
              float* __restrict__ U) {
  const int lane = threadIdx.x & 31;
  const long j = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (j >= N) return;
  const int64_t p0 = ent_off[j], p1 = ent_off[j + 1];
  const float* row = R + (size_t)j * 2 * d;
  float* out = U + (size_t)j * 2 * d;
  for (int k = lane; k < d; k += 32) {
    float g = C[(size_t)j * dpad + k];
    for (int64_t p = p0; p < p1; ++p) g += GS[(size_t)ent_pos[p] * d + k];
    adagrad(g, row[d + k], eta, out + k, out + d + k);
  }
}

// One CTA per pulled relation u: g = sum over its triples, in order, of (gradient through both queries + gamma_r r).
template <int MODEL>
__global__ void __launch_bounds__(256)
relation_kernel(const float* __restrict__ R, const Key* __restrict__ s, const Key* __restrict__ o,
                const int64_t* __restrict__ rel_off, const int32_t* __restrict__ rel_pos, const float* __restrict__ dq,
                int N, int B, int d, int dpad, float eta, float gamma_r, float* __restrict__ U) {
  const int u = blockIdx.x;
  const int rd = MODEL == COMPLEX ? d : d * d;
  const size_t base = (size_t)N * 2 * d + (size_t)u * 2 * rd;
  const float* row = R + base;
  float* out = U + base;
  const int64_t t0 = rel_off[u], t1 = rel_off[u + 1];
  for (int k = threadIdx.x; k < rd; k += blockDim.x) {
    float g = 0.f;
    for (int64_t t = t0; t < t1; ++t) {
      const int i = rel_pos[t];
      const float* es = R + (size_t)s[i] * 2 * d;
      const float* eo = R + (size_t)o[i] * 2 * d;
      const float* dqo = dq + (size_t)i * dpad;
      const float* dqs = dq + (size_t)(B + i) * dpad;
      float v;
      if (MODEL == COMPLEX) {
        const int h = d / 2, j = k < h ? k : k - h;
        const float a = dqo[j], b = dqo[h + j], a2 = dqs[j], b2 = dqs[h + j];
        const float sre = es[j], sim = es[h + j], ore = eo[j], oim = eo[h + j];
        v = k < h ? (sre * a + sim * b) + (ore * a2 + oim * b2) : (sre * b - sim * a) + (oim * a2 - ore * b2);
      } else {
        const int m = k / d, l = k - m * d;
        v = es[m] * dqo[l] + dqs[m] * eo[l];
      }
      g += v + gamma_r * row[k];
    }
    adagrad(g, row[rd + k], eta, out + k, out + rd + k);
  }
}

__global__ void __launch_bounds__(32) loss_kernel(const float* __restrict__ qloss, int n, float* __restrict__ loss) {
  float t = 0.f;
  for (int i = threadIdx.x; i < n; i += 32) t += qloss[i];
  t = warp_sum(t);
  if (threadIdx.x == 0) *loss += t;
}

// ------------------------------------------------------------------ shared negatives (kge_shared_core)
// Rows idx[r] (r < rows; row r itself when idx is null; zeros when idx[r] < 0) of X [.][ldx] fp32, first d values ->
// Xb [rows][dpad] bf16 and XT in chunks of W rows: row r, column j at XT[(r / W) dpad W + j W + r % W]. A null output
// is skipped; columns past d are zeros. 32 x 8 threads per 32 x 32 tile.
__global__ void __launch_bounds__(256)
gather_bf16_kernel(const float* __restrict__ X, int ldx, const Key* __restrict__ idx, int rows, int d, int dpad, int W,
                   __nv_bfloat16* __restrict__ Xb, __nv_bfloat16* __restrict__ XT) {
  __shared__ __nv_bfloat16 tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int j0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int rl = ty + 8 * k, r = r0 + rl, j = j0 + tx;
    const Key src = r < rows ? (idx ? idx[r] : r) : -1;
    const __nv_bfloat16 b = __float2bfloat16(src >= 0 && j < d ? X[(size_t)src * ldx + j] : 0.f);
    if (Xb && r < rows && j < dpad) Xb[(size_t)r * dpad + j] = b;
    tile[rl][tx] = b;
  }
  __syncthreads();
  const int r = r0 + tx;
  if (!XT || r >= rows) return;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int j = j0 + ty + 8 * k;
    if (j < dpad) XT[(size_t)(r / W) * dpad * W + (size_t)j * W + r % W] = tile[tx][ty + 8 * k];
  }
}

// Query q < 2 Bp of the padded batch (object queries, then subject queries; triple i sits in chunk i / 128 at slot
// i % 128): its answer, and its positive column in the chunk's list [subjects | objects | negatives].
struct SharedQuery {
  int i, pos;
  Key ans;
  __device__ __forceinline__ SharedQuery(long q, int Bp, const Key* s, const Key* o) {
    const bool obj = q < Bp;
    i = obj ? (int)q : (int)(q - Bp);
    ans = obj ? o[i] : s[i];
    pos = (obj ? kKgeSharedChunk : 0) + i % kKgeSharedChunk;
  }
  // column j (entity c, -1 for a padding slot) takes part in the softmax: not padding, and not another copy of the answer
  __device__ __forceinline__ bool live(Key c, int j) const { return c >= 0 && (j == pos || c != ans); }
};

// One warp per query q < 2 Bp: over its chunk's live columns, lse[q] = logsumexp of the scores Z[q] and qloss[q] = lse -
// the positive column's score; queries of padding triples (i >= B) get zeros.
__global__ void __launch_bounds__(256)
kge_shared_lse_kernel(const float* __restrict__ Z, const Key* __restrict__ cand, const Key* __restrict__ s,
                  const Key* __restrict__ o, int B, int Bp, int Lr, float* __restrict__ lse, float* __restrict__ qloss) {
  const int lane = threadIdx.x & 31;
  const long q = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (q >= 2L * Bp) return;
  const SharedQuery sq(q, Bp, s, o);
  if (sq.i >= B) {
    if (lane == 0) lse[q] = qloss[q] = 0.f;
    return;
  }
  const Key* c = cand + (size_t)(sq.i / kKgeSharedChunk) * Lr;
  const float* z = Z + (size_t)q * Lr;
  float m = -INFINITY;
  for (int j = lane; j < Lr; j += 32)
    if (sq.live(c[j], j)) m = fmaxf(m, z[j]);
  m = warp_max(m);
  float t = 0.f;
  for (int j = lane; j < Lr; j += 32)
    if (sq.live(c[j], j)) t += expf(z[j] - m);
  t = warp_sum(t);
  const float l = m + logf(t);
  if (lane == 0) {
    lse[q] = l;
    qloss[q] = l - z[sq.pos];
  }
}

// Z -> G = softmax - onehot(positive) over the live columns: Gb [2 Bp][Lr] in query order, and GT [nch][Lr][2 * 128]
// whose chunk k holds, per list column, G of the chunk's object queries, then of its subject queries. Masked and padding
// columns and the queries of padding triples are zeros. 32 x 32 tiles (32 queries of one chunk and one side).
__global__ void __launch_bounds__(256)
kge_shared_grad_kernel(const float* __restrict__ Z, const float* __restrict__ lse, const Key* __restrict__ cand,
                   const Key* __restrict__ s, const Key* __restrict__ o, int B, int Bp, int Lr,
                   __nv_bfloat16* __restrict__ Gb, __nv_bfloat16* __restrict__ GT) {
  __shared__ __nv_bfloat16 tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int n0 = blockIdx.x * 32, b0 = blockIdx.y * 32;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int bl = ty + 8 * k, n = n0 + tx;
    const long q = (long)b0 + bl;
    const SharedQuery sq(q, Bp, s, o);
    float g = 0.f;
    if (sq.i < B && n < Lr && sq.live(cand[(size_t)(sq.i / kKgeSharedChunk) * Lr + n], n))
      g = expf(Z[(size_t)q * Lr + n] - lse[q]) - (n == sq.pos ? 1.f : 0.f);
    const __nv_bfloat16 gb = __float2bfloat16(g);
    if (n < Lr) Gb[(size_t)q * Lr + n] = gb;
    tile[bl][tx] = gb;
  }
  __syncthreads();
  const bool obj = b0 < Bp;
  const int i0 = obj ? b0 : b0 - Bp;
  const size_t chunk = (size_t)(i0 / kKgeSharedChunk);
  const int col = (obj ? 0 : kKgeSharedChunk) + i0 % kKgeSharedChunk + tx;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int n = n0 + ty + 8 * k;
    if (n < Lr) GT[(chunk * Lr + n) * (2 * kKgeSharedChunk) + col] = tile[tx][ty + 8 * k];
  }
}

// One warp per distinct entity u: g = its candidate columns' rows of C in (chunk, column) order, then its given-entity
// gradients in position order (occurrence p < nC: row p of C [nch Lr][dpad], else row p - nC of GS [2 Bp][d]);
// U row u = AdaGrad update.
__global__ void __launch_bounds__(256)
kge_shared_entity_kernel(const float* __restrict__ R, const float* __restrict__ C, const float* __restrict__ GS,
                     const int64_t* __restrict__ ent_off, const int32_t* __restrict__ ent_pos, int Ne, int nC, int d,
                     int dpad, float eta, float* __restrict__ U) {
  const int lane = threadIdx.x & 31;
  const long u = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (u >= Ne) return;
  const int64_t p0 = ent_off[u], p1 = ent_off[u + 1];
  const float* row = R + (size_t)u * 2 * d;
  float* out = U + (size_t)u * 2 * d;
  for (int k = lane; k < d; k += 32) {
    float g = 0.f;
    for (int64_t p = p0; p < p1; ++p) {
      const int at = ent_pos[p];
      g += at < nC ? C[(size_t)at * dpad + k] : GS[(size_t)(at - nC) * d + k];
    }
    adagrad(g, row[d + k], eta, out + k, out + d + k);
  }
}

inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }
inline int pad8(int x) { return (x + 7) / 8 * 8; }

// The workspace, carved in this order by kge_1vsall_workspace_bytes and kge_1vsall_core.
struct Layout {
  int dpad, Npad, nch, qrows, split_dq, split_c;
  size_t off[15];
  size_t total;
  Layout(int N, int B, int d, int chunk) {
    dpad = pad8(d);
    Npad = pad8(N);
    nch = (2 * B + chunk - 1) / chunk;
    qrows = nch * chunk;
    split_dq = partial_splits(chunk, dpad, Npad);
    split_c = partial_splits(N, dpad, chunk);
    const size_t parts = std::max((size_t)split_dq * chunk * dpad, (size_t)split_c * N * dpad);
    const size_t bytes[15] = {
        (size_t)Npad * dpad * 2,               //  0 Eb   [Npad][dpad] bf16
        (size_t)dpad * Npad * 2,               //  1 ET   [dpad][Npad] bf16
        (size_t)2 * B * d * 4,                 //  2 Qf   [2B][d] fp32
        (size_t)qrows * dpad * 2,              //  3 Qb   [qrows][dpad] bf16
        (size_t)qrows * dpad * 2,              //  4 QT   [nch][dpad][chunk] bf16
        (size_t)qrows * dpad * 4,              //  5 dq   [qrows][dpad] fp32
        (size_t)N * dpad * 4,                  //  6 C    [N][dpad] fp32
        (size_t)chunk * N * 4,                 //  7 S    [chunk][N] fp32
        (size_t)chunk * 4,                     //  8 lse  [chunk]
        (size_t)2 * B * 4,                     //  9 qloss [2B]
        (size_t)chunk * Npad * 2,              // 10 Gb   [chunk][Npad] bf16
        (size_t)N * chunk * 2,                 // 11 GbT  [N][chunk] bf16
        parts * 4,                             // 12 partial tiles
        (size_t)2 * B * d * 4,                 // 13 GS   [2B][d] fp32
        0};
    total = 0;
    for (int i = 0; i < 15; ++i) { off[i] = total; total += align_up(bytes[i]); }
  }
};

// The workspace of kge_shared_core, carved in this order. Bp: B padded to whole chunks; Lr: the list length 2 * 128 + S
// padded to a multiple of 8 (the K extent of G E).
struct SharedLayout {
  int dpad, Bp, nch, Lr;
  size_t off[13];
  size_t total;
  SharedLayout(int B, int S, int d) {
    dpad = pad8(d);
    nch = (B + kKgeSharedChunk - 1) / kKgeSharedChunk;
    Bp = nch * kKgeSharedChunk;
    Lr = pad8(2 * kKgeSharedChunk + S);
    const size_t q = 2 * (size_t)Bp, lists = (size_t)nch * Lr;
    const size_t bytes[13] = {
        lists * dpad * 2,                      //  0 Eb    [nch Lr][dpad] bf16: chunk k's list rows
        lists * dpad * 2,                      //  1 ET    [nch][dpad][Lr] bf16
        q * d * 4,                             //  2 Qf    [2 Bp][d] fp32
        q * dpad * 2,                          //  3 Qb    [2 Bp][dpad] bf16
        q * dpad * 2,                          //  4 QT    [nch][dpad][2 * 128] bf16
        q * Lr * 4,                            //  5 Z     [2 Bp][Lr] fp32
        q * 4,                                 //  6 lse   [2 Bp]
        q * 4,                                 //  7 qloss [2 Bp]
        q * Lr * 2,                            //  8 Gb    [2 Bp][Lr] bf16
        lists * 2 * kKgeSharedChunk * 2,       //  9 GT    [nch][Lr][2 * 128] bf16
        q * dpad * 4,                          // 10 dq    [2 Bp][dpad] fp32
        lists * dpad * 4,                      // 11 C     [nch Lr][dpad] fp32
        q * d * 4};                            // 12 GS    [2 Bp][d] fp32
    total = 0;
    for (int i = 0; i < 13; ++i) { off[i] = total; total += align_up(bytes[i]); }
  }
};

}  // namespace

size_t kge_1vsall_workspace_bytes(int N, int B, int d, int chunk) {
  return Layout(N, B, d, chunk).total;
}

void kge_1vsall_core(cudaStream_t stream, int model, const float* R, const Key* s, const Key* o, const int32_t* rel,
                     const int64_t* ent_off, const int32_t* ent_pos, const int64_t* rel_off, const int32_t* rel_pos,
                     int N, int nrel, int B, int d, int chunk, float eta, float gamma_e, float gamma_r, void* workspace,
                     float* U, float* loss) {
  ADAPM_CHECK(model == COMPLEX || model == RESCAL, "kge_1vsall: model must be ComplEx (0) or RESCAL (1)");
  ADAPM_CHECK(N > 0 && B > 0 && nrel > 0, "kge_1vsall: empty batch or entity set");
  ADAPM_CHECK(d > 0 && d <= kKge1vsAllMaxDim && (model == RESCAL || d % 2 == 0), "kge_1vsall: embedding dimension out of range");
  ADAPM_CHECK(chunk > 0 && chunk % 128 == 0, "kge_1vsall: the query chunk must be a positive multiple of 128");
  const Layout L(N, B, d, chunk);
  const int dpad = L.dpad, Npad = L.Npad;
  char* w = static_cast<char*>(workspace);
  auto* Eb = reinterpret_cast<__nv_bfloat16*>(w + L.off[0]);
  auto* ET = reinterpret_cast<__nv_bfloat16*>(w + L.off[1]);
  auto* Qf = reinterpret_cast<float*>(w + L.off[2]);
  auto* Qb = reinterpret_cast<__nv_bfloat16*>(w + L.off[3]);
  auto* QT = reinterpret_cast<__nv_bfloat16*>(w + L.off[4]);
  auto* dq = reinterpret_cast<float*>(w + L.off[5]);
  auto* C = reinterpret_cast<float*>(w + L.off[6]);
  auto* S = reinterpret_cast<float*>(w + L.off[7]);
  auto* lse = reinterpret_cast<float*>(w + L.off[8]);
  auto* qloss = reinterpret_cast<float*>(w + L.off[9]);
  auto* Gb = reinterpret_cast<__nv_bfloat16*>(w + L.off[10]);
  auto* GbT = reinterpret_cast<__nv_bfloat16*>(w + L.off[11]);
  auto* P = reinterpret_cast<float*>(w + L.off[12]);
  auto* GS = reinterpret_cast<float*>(w + L.off[13]);
  const unsigned warps_q = (unsigned)((2L * B * 32 + 255) / 256);
  if (model == COMPLEX) query_kernel<COMPLEX><<<warps_q, 256, 0, stream>>>(R, s, o, rel, N, B, d, Qf);
  else query_kernel<RESCAL><<<warps_q, 256, 0, stream>>>(R, s, o, rel, N, B, d, Qf);
  const unsigned jt = (unsigned)((dpad + 31) / 32);
  to_bf16_kernel<<<dim3(jt, (Npad + 31) / 32), 256, 0, stream>>>(R, 2 * d, N, Npad, d, dpad, Npad, Eb, ET);
  to_bf16_kernel<<<dim3(jt, (L.qrows + 31) / 32), 256, 0, stream>>>(Qf, d, 2 * B, L.qrows, d, dpad, chunk, Qb, QT);
  ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH();
  for (int c = 0; c < L.nch; ++c) {
    const int q0 = c * chunk;
    gemm_nt_bf16(stream, Qb + (size_t)q0 * dpad, Eb, chunk, N, dpad, S, N);          // Z = Q E^T     (K = dpad)
    row_lse_kernel<<<chunk * 32 / 256, 256, 0, stream>>>(S, N, chunk, q0, B, s, o, lse, qloss);
    grad_kernel<<<dim3((Npad + 31) / 32, chunk / 32), 256, 0, stream>>>(S, lse, N, Npad, chunk, q0, B, s, o, Gb, GbT);
    gemm_partial(stream, Gb, ET, chunk, dpad, Npad, P);          // dQ = G E      (K = N)
    const long ndq = (long)chunk * dpad;
    sum_kernel<<<(unsigned)((ndq + 255) / 256), 256, 0, stream>>>(P, L.split_dq, ndq, false, dq + (size_t)q0 * dpad);
    gemm_partial(stream, GbT, QT + (size_t)c * dpad * chunk, N, dpad, chunk, P);   // G^T Q (K = chunk)
    const long nc = (long)N * dpad;
    sum_kernel<<<(unsigned)((nc + 255) / 256), 256, 0, stream>>>(P, L.split_c, nc, c > 0, C);
    ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH();
  }
  const unsigned warps_b = (unsigned)(((long)B * 32 + 255) / 256);
  if (model == COMPLEX) given_kernel<COMPLEX><<<warps_b, 256, 0, stream>>>(R, s, o, rel, dq, N, B, d, dpad, gamma_e, GS);
  else given_kernel<RESCAL><<<warps_b, 256, 0, stream>>>(R, s, o, rel, dq, N, B, d, dpad, gamma_e, GS);
  entity_kernel<<<(unsigned)(((long)N * 32 + 255) / 256), 256, 0, stream>>>(R, C, GS, ent_off, ent_pos, N, d, dpad, eta, U);
  if (model == COMPLEX)
    relation_kernel<COMPLEX><<<nrel, 256, 0, stream>>>(R, s, o, rel_off, rel_pos, dq, N, B, d, dpad, eta, gamma_r, U);
  else relation_kernel<RESCAL><<<nrel, 256, 0, stream>>>(R, s, o, rel_off, rel_pos, dq, N, B, d, dpad, eta, gamma_r, U);
  loss_kernel<<<1, 32, 0, stream>>>(qloss, 2 * B, loss);
  ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

size_t kge_shared_workspace_bytes(int B, int S, int d) { return SharedLayout(B, S, d).total; }

void kge_shared_core(cudaStream_t stream, int model, const float* R, const Key* s, const Key* o, const int32_t* rel,
                     const Key* cand, const Key* qorder, const int64_t* ent_off, const int32_t* ent_pos,
                     const int64_t* rel_off, const int32_t* rel_pos, int Ne, int nrel, int B, int S, int d, float eta,
                     float gamma_e, float gamma_r, void* workspace, float* U, float* loss) {
  ADAPM_CHECK(model == COMPLEX || model == RESCAL, "kge_shared: model must be ComplEx (0) or RESCAL (1)");
  ADAPM_CHECK(Ne > 0 && B > 0 && nrel > 0 && S >= 0, "kge_shared: empty batch or entity set");
  ADAPM_CHECK(d > 0 && d <= kKge1vsAllMaxDim && (model == RESCAL || d % 2 == 0), "kge_shared: embedding dimension out of range");
  const SharedLayout L(B, S, d);
  const int dpad = L.dpad, Bp = L.Bp, nch = L.nch, Lr = L.Lr;
  char* w = static_cast<char*>(workspace);
  auto* Eb = reinterpret_cast<__nv_bfloat16*>(w + L.off[0]);
  auto* ET = reinterpret_cast<__nv_bfloat16*>(w + L.off[1]);
  auto* Qf = reinterpret_cast<float*>(w + L.off[2]);
  auto* Qb = reinterpret_cast<__nv_bfloat16*>(w + L.off[3]);
  auto* QT = reinterpret_cast<__nv_bfloat16*>(w + L.off[4]);
  auto* Z = reinterpret_cast<float*>(w + L.off[5]);
  auto* lse = reinterpret_cast<float*>(w + L.off[6]);
  auto* qloss = reinterpret_cast<float*>(w + L.off[7]);
  auto* Gb = reinterpret_cast<__nv_bfloat16*>(w + L.off[8]);
  auto* GT = reinterpret_cast<__nv_bfloat16*>(w + L.off[9]);
  auto* dq = reinterpret_cast<float*>(w + L.off[10]);
  auto* C = reinterpret_cast<float*>(w + L.off[11]);
  auto* GS = reinterpret_cast<float*>(w + L.off[12]);
  const int K2 = 2 * kKgeSharedChunk;          // queries per chunk: the K extent of G^T Q
  const unsigned warps_q = (unsigned)((2L * Bp * 32 + 255) / 256);
  if (model == COMPLEX) query_kernel<COMPLEX><<<warps_q, 256, 0, stream>>>(R, s, o, rel, Ne, Bp, d, Qf);
  else query_kernel<RESCAL><<<warps_q, 256, 0, stream>>>(R, s, o, rel, Ne, Bp, d, Qf);
  const unsigned jt = (unsigned)((dpad + 31) / 32);
  gather_bf16_kernel<<<dim3(jt, (nch * Lr + 31) / 32), 256, 0, stream>>>(R, 2 * d, cand, nch * Lr, d, dpad, Lr, Eb, ET);
  gather_bf16_kernel<<<dim3(jt, 2 * Bp / 32), 256, 0, stream>>>(Qf, d, nullptr, 2 * Bp, d, dpad, 1, Qb, nullptr);
  gather_bf16_kernel<<<dim3(jt, 2 * Bp / 32), 256, 0, stream>>>(Qf, d, qorder, 2 * Bp, d, dpad, K2, nullptr, QT);
  ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH();
  // Z = Q_k E_k^T: one batch per 128 queries of one side of chunk k (z % nch = k), K = dpad
  gemm_batched(stream, Qb, 2L * Bp, Eb, (long)nch * Lr, kKgeSharedChunk, Lr, dpad, kKgeSharedChunk, Lr, nch, 2 * nch, Z);
  kge_shared_lse_kernel<<<warps_q, 256, 0, stream>>>(Z, cand, s, o, B, Bp, Lr, lse, qloss);
  kge_shared_grad_kernel<<<dim3((Lr + 31) / 32, 2 * Bp / 32), 256, 0, stream>>>(Z, lse, cand, s, o, B, Bp, Lr, Gb, GT);
  ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH();
  // dQ = G_k E_k (K = Lr), in query order; C_k = G_k^T Q_k (K = the chunk's 256 queries), [nch Lr][dpad]
  gemm_batched(stream, Gb, 2L * Bp, ET, (long)nch * dpad, kKgeSharedChunk, dpad, Lr, kKgeSharedChunk, dpad, nch, 2 * nch, dq);
  gemm_batched(stream, GT, (long)nch * Lr, QT, (long)nch * dpad, Lr, dpad, K2, Lr, dpad, nch, nch, C);
  const unsigned warps_b = (unsigned)(((long)Bp * 32 + 255) / 256);
  if (model == COMPLEX) given_kernel<COMPLEX><<<warps_b, 256, 0, stream>>>(R, s, o, rel, dq, Ne, Bp, d, dpad, gamma_e, GS);
  else given_kernel<RESCAL><<<warps_b, 256, 0, stream>>>(R, s, o, rel, dq, Ne, Bp, d, dpad, gamma_e, GS);
  kge_shared_entity_kernel<<<(unsigned)(((long)Ne * 32 + 255) / 256), 256, 0, stream>>>(R, C, GS, ent_off, ent_pos, Ne,
                                                                                     nch * Lr, d, dpad, eta, U);
  if (model == COMPLEX)
    relation_kernel<COMPLEX><<<nrel, 256, 0, stream>>>(R, s, o, rel_off, rel_pos, dq, Ne, Bp, d, dpad, eta, gamma_r, U);
  else relation_kernel<RESCAL><<<nrel, 256, 0, stream>>>(R, s, o, rel_off, rel_pos, dq, Ne, Bp, d, dpad, eta, gamma_r, U);
  loss_kernel<<<1, 32, 0, stream>>>(qloss, 2 * Bp, loss);
  ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

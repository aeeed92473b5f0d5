// DCN-v2's low-rank cross network (Wang et al., 2021) for sm_90a, as torchrec's LowRankCrossNet: layer l maps
//   x_{l+1} = x_0 * (W_l (V_l x_l) + b_l) + x_l        V_l [r, N], W_l [N, r], b_l [N]
// where x_0 = [z | e_0 | .. | e_{F-1}] [B, N] is the bottom-MLP output z [B, E] followed by the pooled fields e [B, F, E]
// (N = (F + 1) E). The residual stream x_l is fp32; bf16 appears only where a tensor becomes a GEMM operand.
//
// Every GEMM is the tile pipeline of wgmma_utils.cuh (tma_tile: one 128 x 128 fp32 tile of A B^T per CTA, both
// operands K-major bf16) with one of four epilogues, applied straight to the accumulator fragment:
//   EPI_H      bf16 [M, Ncol], and its transpose [Ncol, pitch] when asked for   (h = x_l V_l^T, dh = P W_l)
//   EPI_CROSS  u = acc + b_l, x_{l+1} = x_0 * u + x_l in fp32 (x_0 read from z and e by column, x_l in place), and
//              when asked for x_{l+1} in bf16, its transpose in bf16 and u in bf16
//   EPI_RESID  acc + G (+ a second addend) in fp32, written to one [B, N] matrix or split by column into dz | de
//   EPI_WGRAD  fp32 partial tiles of the weight gradients, one per k-split, added in split order afterwards
//
// forward (1 + 2 L launches): dcn_stage_kernel writes x_0 in bf16 (and x_0^T); per layer h = x_l V_l^T (EPI_H, h^T
// when training), then the cross GEMM u = h W_l^T (EPI_CROSS).
// backward of layer l, G = dL/dx_{l+1} fp32: dcn_bwd_elem_kernel writes P = G * x_0 in bf16 with P^T, dx_0 (+)= G * u
// and per-CTA column sums of P, which dcn_sum_kernel adds in a fixed order into db_l; dh = P W_l (EPI_H against
// W_l^T [r, N]); dx_l = G + dh V_l (EPI_RESID against V_l^T [N, r]); dW_l = P^T h_l and dV_l = dh^T x_l (EPI_WGRAD on
// the transposed operands, K = B). Layer 0's EPI_RESID adds dx_0's accumulator and writes dz and de.
// No floating-point atomics anywhere: one GPU gives bit-identical outputs and gradients on reruns.
// Transposed operands [*, B] have rows pitch = B rounded up to 8 elements apart (the 16-byte TMA row pitch); their
// tensor maps have B columns, so TMA reads zeros past B and the pad is never written or read.
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
using bf16 = __nv_bfloat16;

constexpr int kTile = 64;              // elementwise kernels: 64 x 64 tiles, 256 threads
constexpr int kElemThreads = 256;
constexpr int kElemRowCtas = 32;       // row CTAs of dcn_bwd_elem_kernel: the column sums of P come in <= 32 partials

// x_0 [B, N] read by column from z [B, E] and e [B, N - E]
struct X0 {
  const float* z;
  const float* e;
  int E, N;
  __device__ __forceinline__ float at(int64_t row, int col) const {
    return col < E ? __ldg(z + row * E + col) : __ldg(e + row * (N - E) + (col - E));
  }
};

// an fp32 [B, N] output split the same way: columns < E to lo [B, E], the others to hi [B, N - E] (E = 0: hi [B, N])
struct Out {
  float* lo;
  float* hi;
  int E, N;
  __device__ __forceinline__ float& at(int64_t row, int col) const {
    return col < E ? lo[row * E + col] : hi[row * (N - E) + (col - E)];
  }
};

int64_t pitch_of(int B) { return ((int64_t)B + 7) / 8 * 8; }

// s[c][r], a tile of kTile columns from c0 and kTile rows from r0, to t[(c0 + c) * pitch + r0 + r] (rows < B, cols < N)
__device__ __forceinline__ void store_transposed(const bf16 (*s)[kTile + 2], bf16* t, int64_t pitch, int r0, int c0,
                                                 int B, int N) {
  for (int i = threadIdx.x; i < kTile * kTile; i += kElemThreads) {
    const int c = i / kTile, r = i % kTile;
    if (c0 + c < N && r0 + r < B) t[(int64_t)(c0 + c) * pitch + r0 + r] = s[c][r];
  }
}

// x_0 -> xb [B, N] bf16 and, when xt is given, xt [N, pitch] bf16. Grid (N / 64, B / 64) tiles.
__global__ void __launch_bounds__(kElemThreads)
dcn_stage_kernel(X0 x0, int B, bf16* __restrict__ xb, bf16* __restrict__ xt, int64_t pitch) {
  __shared__ bf16 s[kTile][kTile + 2];
  const int N = x0.N, c0 = blockIdx.x * kTile, r0 = blockIdx.y * kTile;
  const int tx = threadIdx.x % kTile, col = c0 + tx;
  for (int rr = threadIdx.x / kTile; rr < kTile; rr += kElemThreads / kTile) {
    const int row = r0 + rr;
    bf16 v = __float2bfloat16_rn(0.f);
    if (row < B && col < N) {
      v = __float2bfloat16_rn(x0.at(row, col));
      xb[(int64_t)row * N + col] = v;
    }
    s[tx][rr] = v;
  }
  if (!xt) return;
  __syncthreads();
  store_transposed(s, xt, pitch, r0, c0, B, N);
}

// One pass over G, x_0 and u of a layer: P = G * x_0 -> Pb [B, N] and Pt [N, pitch] in bf16; dx0 = G * u (first, the
// top layer) or dx0 += G * u; part[blockIdx.y][col] = the sum of P over the CTA's rows, in row order. Grid
// (N / 64, <= kElemRowCtas): CTA y takes the row tiles y, y + gridDim.y, ...
__global__ void __launch_bounds__(kElemThreads)
dcn_bwd_elem_kernel(const float* __restrict__ G, X0 x0, const bf16* __restrict__ ub, int B, bool first,
                    float* __restrict__ dx0, bf16* __restrict__ Pb, bf16* __restrict__ Pt, int64_t pitch,
                    float* __restrict__ part) {
  __shared__ bf16 s[kTile][kTile + 2];
  __shared__ float cs[kElemThreads / kTile][kTile];
  const int N = x0.N, c0 = blockIdx.x * kTile;
  const int tx = threadIdx.x % kTile, ty = threadIdx.x / kTile, col = c0 + tx;
  float sum = 0.f;
  for (int r0 = blockIdx.y * kTile; r0 < B; r0 += gridDim.y * kTile) {
    for (int rr = ty; rr < kTile; rr += kElemThreads / kTile) {
      const int row = r0 + rr;
      bf16 v = __float2bfloat16_rn(0.f);
      if (row < B && col < N) {
        const int64_t i = (int64_t)row * N + col;
        const float g = G[i], p = g * x0.at(row, col);
        const float d = g * __bfloat162float(ub[i]);
        v = __float2bfloat16_rn(p);
        Pb[i] = v;
        dx0[i] = first ? d : dx0[i] + d;
        sum += p;
      }
      s[tx][rr] = v;
    }
    __syncthreads();
    store_transposed(s, Pt, pitch, r0, c0, B, N);
    __syncthreads();
  }
  cs[ty][tx] = sum;
  __syncthreads();
  if (threadIdx.x < kTile && col < N)
    part[(int64_t)blockIdx.y * N + col] = cs[0][threadIdx.x] + cs[1][threadIdx.x] + cs[2][threadIdx.x] + cs[3][threadIdx.x];
}

// out[i] = part[0][i] + part[1][i] + ... + part[S - 1][i], in that order
__global__ void __launch_bounds__(256) dcn_sum_kernel(const float* __restrict__ part, int S, int64_t n,
                                                      float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < S; ++k) s += part[k * n + i];
    out[i] = s;
  }
}

enum Epi : int { EPI_H = 0, EPI_CROSS = 1, EPI_RESID = 2, EPI_WGRAD = 3 };

struct EpiArgs {
  int M, Ncol;          // the output [M, Ncol]; Ncol % 8 == 0
  bf16* ob;             // H: [M, Ncol]; CROSS: x_{l+1} (or null)
  bf16* ot;             // H, CROSS: the transpose of ob's values, [Ncol, pitch] (or null)
  int64_t pitch;
  X0 x0;                // CROSS
  const float* bias;    // CROSS: b_l [Ncol]
  const float* xprev;   // CROSS: x_l fp32 [M, Ncol] (null: x_0); may be x
  float* x;             // CROSS: x_{l+1} fp32 [M, Ncol]
  bf16* ub;             // CROSS: u bf16 [M, Ncol] (or null)
  const float* G;       // RESID: [M, Ncol]; may alias out
  const float* add;     // RESID: second addend [M, Ncol] (or null)
  Out out;              // RESID
  float* C;             // WGRAD: [gridDim.z][M, Ncol]
};

__device__ __forceinline__ void st_bf16x2(bf16* p, float a, float b) {
  *reinterpret_cast<uint32_t*>(p) = pack_bf16(a, b);
}

template <int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
dcn_gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, int K,
                const EpiArgs p) {
  const KRange kr = k_split((K + BK<KIND_BF16> - 1) / BK<KIND_BF16>);
  float d[64];
  if (!tma_tile<KIND_BF16>(tmap_a, tmap_b, blockIdx.y * BM, blockIdx.x * BN, kr.kb0, kr.num_kb, d)) return;
  const int lane = threadIdx.x & 31;
  const int row0 = blockIdx.y * BM + frag_row0(threadIdx.x >> 5), col0 = blockIdx.x * BN;
  if constexpr (EPI == EPI_WGRAD) {
    store_fragment(d, 1.f, p.C + (size_t)blockIdx.z * p.M * p.Ncol, p.Ncol, row0, col0, p.M, p.Ncol, lane, false);
    return;
  }
  // fragment layout: see store_fragment; a thread's pairs (col, col + 1) have col even, so col < Ncol covers both
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + (lane >> 2) + 8 * h;
    if (row >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int col = col0 + 8 * j + 2 * (lane & 3);
      if (col >= p.Ncol) continue;
      const int64_t i = (int64_t)row * p.Ncol + col;
      float v0 = d[4 * j + 2 * h], v1 = d[4 * j + 2 * h + 1];
      if constexpr (EPI == EPI_H) {
        st_bf16x2(p.ob + i, v0, v1);
      } else if constexpr (EPI == EPI_CROSS) {
        const float u0 = v0 + __ldg(p.bias + col), u1 = v1 + __ldg(p.bias + col + 1);
        const float a0 = p.x0.at(row, col), a1 = p.x0.at(row, col + 1);
        float x0 = a0, x1 = a1;
        if (p.xprev) {
          const float2 xp = *reinterpret_cast<const float2*>(p.xprev + i);
          x0 = xp.x; x1 = xp.y;
        }
        v0 = fmaf(a0, u0, x0);
        v1 = fmaf(a1, u1, x1);
        *reinterpret_cast<float2*>(p.x + i) = make_float2(v0, v1);
        if (p.ob) st_bf16x2(p.ob + i, v0, v1);
        if (p.ub) st_bf16x2(p.ub + i, u0, u1);
      } else {
        v0 += p.G[i];
        v1 += p.G[i + 1];
        if (p.add) { v0 += p.add[i]; v1 += p.add[i + 1]; }
        p.out.at(row, col) = v0;
        p.out.at(row, col + 1) = v1;
      }
      if (EPI != EPI_RESID && p.ot) {
        p.ot[(int64_t)col * p.pitch + row] = __float2bfloat16_rn(v0);
        p.ot[(int64_t)(col + 1) * p.pitch + row] = __float2bfloat16_rn(v1);
      }
    }
  }
}

// C = A B^T over K: A [a_rows, K], B [b_rows, K] bf16 with rows `pitch` elements apart (0: K), k-blocks split over
// `splits` CTAs per tile (EPI_WGRAD only)
template <int EPI>
void gemm(cudaStream_t stream, const void* A, int64_t a_rows, const void* B, int64_t b_rows, int K, int64_t pitch,
          int splits, const EpiArgs& p) {
  const CUtensorMap ma = make_map("dcn_cross", A, a_rows, K, BM, KIND_BF16, pitch);
  const CUtensorMap mb = make_map("dcn_cross", B, b_rows, K, BN, KIND_BF16, pitch);
  const dim3 grid((p.Ncol + BN - 1) / BN, (p.M + BM - 1) / BM, splits);
  launch<dcn_gemm_kernel<EPI>, Ring<STAGES>>(grid, stream, ma, mb, K, p);
}

void sum_partials(cudaStream_t stream, const float* part, int S, int64_t n, float* out) {
  const int blocks = (int)std::min<int64_t>((n + 255) / 256, 4 * (int64_t)num_sms());
  dcn_sum_kernel<<<blocks, 256, 0, stream>>>(part, S, n, out);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

// k-splits of a weight-gradient GEMM [M, Ncol] with K = B: a split per idle SM pair when the output has few tiles and
// K is long (as gemm_nt_bf16 chooses them), no split left empty
int wgrad_splits(int M, int Ncol, int B) {
  const int total_kb = (B + BK<KIND_BF16> - 1) / BK<KIND_BF16>;
  const long tiles = (long)((M + BM - 1) / BM) * ((Ncol + BN - 1) / BN);
  int splits = 1;
  if (tiles * 2 <= num_sms() && total_kb >= 32) splits = (int)std::min<long>(num_sms() / tiles, total_kb / 8);
  splits = std::max(1, std::min(splits, std::min(total_kb, 64)));
  const int kb_per = (total_kb + splits - 1) / splits;
  return (total_kb + kb_per - 1) / kb_per;
}

// C [M, Ncol] = A [M, B] B [Ncol, B]^T on the transposed operands; with splits, the partial tiles go to ws first
void wgrad(cudaStream_t stream, const void* A, const void* Bt, int M, int Ncol, int B, float* ws, float* C) {
  const int splits = wgrad_splits(M, Ncol, B);
  EpiArgs p{};
  p.M = M;
  p.Ncol = Ncol;
  p.C = splits > 1 ? ws : C;
  gemm<EPI_WGRAD>(stream, A, M, Bt, Ncol, B, pitch_of(B), splits, p);
  if (splits > 1) sum_partials(stream, ws, splits, (int64_t)M * Ncol, C);
}

int elem_row_ctas(int B) { return std::min(kElemRowCtas, (B + kTile - 1) / kTile); }

void check_shape(int B, int E, int N, int r, int L) {
  ADAPM_CHECK(B >= 1 && E >= 1 && N > E && N % E == 0, "dcn_cross: need B >= 1 and N = (F + 1) E with F >= 1");
  ADAPM_CHECK(N % 8 == 0 && r % 8 == 0, "dcn_cross: N and r must be multiples of 8");
  ADAPM_CHECK(L >= 1 && L <= kDcnMaxLayers && r >= kDcnMinRank && r <= kDcnMaxRank,
              "dcn_cross: need 1 <= L <= 8 and 8 <= r <= 1024");
  ADAPM_CHECK((int64_t)B * N < ((int64_t)1 << 31), "dcn_cross: B * N must be < 2^31");
}

}  // namespace

size_t dcn_workspace_floats(int B, int N, int r) {
  const int64_t db = (int64_t)elem_row_ctas(B) * N;
  const int64_t wg = (int64_t)std::max(wgrad_splits(N, r, B), wgrad_splits(r, N, B)) * N * r;
  return (size_t)std::max(db, wg);
}

void dcn_forward(cudaStream_t stream, const float* z, const float* e, int B, int E, int N, int r, int L, const void* V,
                 const void* W, const float* b, void* xb, void* hb, float* x, void* xt, void* ht, void* ub) {
  check_shape(B, E, N, r, L);
  const int64_t pitch = pitch_of(B);
  const X0 x0{z, e, E, N};
  bf16* xb16 = static_cast<bf16*>(xb);
  bf16* xt16 = static_cast<bf16*>(xt);
  bf16* ht16 = static_cast<bf16*>(ht);
  bf16* ub16 = static_cast<bf16*>(ub);
  dcn_stage_kernel<<<dim3((N + kTile - 1) / kTile, (B + kTile - 1) / kTile), kElemThreads, 0, stream>>>(x0, B, xb16,
                                                                                                        xt16, pitch);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
  for (int l = 0; l < L; ++l) {
    EpiArgs p{};
    p.M = B;
    p.Ncol = r;
    p.ob = static_cast<bf16*>(hb);
    p.ot = ht16 ? ht16 + (int64_t)l * r * pitch : nullptr;
    p.pitch = pitch;
    gemm<EPI_H>(stream, xb, B, static_cast<const bf16*>(V) + (int64_t)l * r * N, r, N, 0, 1, p);
    EpiArgs q{};
    q.M = B;
    q.Ncol = N;
    q.x0 = x0;
    q.bias = b + (int64_t)l * N;
    q.xprev = l ? x : nullptr;
    q.x = x;
    q.ob = l + 1 < L ? xb16 : nullptr;
    q.ot = xt16 && l + 1 < L ? xt16 + (int64_t)(l + 1) * N * pitch : nullptr;
    q.pitch = pitch;
    q.ub = ub16 ? ub16 + (int64_t)l * B * N : nullptr;
    gemm<EPI_CROSS>(stream, hb, B, static_cast<const bf16*>(W) + (int64_t)l * N * r, N, r, 0, 1, q);
  }
}

void dcn_backward(cudaStream_t stream, const float* z, const float* e, int B, int E, int N, int r, int L, const void* Vt,
                  const void* Wt, const void* xt, const void* ht, const void* ub, const float* grad_out, float* G,
                  float* dx0, void* Pb, void* Pt, void* dh, void* dht, float* ws, float* dz, float* de, float* dV,
                  float* dW, float* db) {
  check_shape(B, E, N, r, L);
  const int64_t pitch = pitch_of(B);
  const X0 x0{z, e, E, N};
  const int rows = elem_row_ctas(B);
  for (int l = L - 1; l >= 0; --l) {
    const float* g = l == L - 1 ? grad_out : G;
    dcn_bwd_elem_kernel<<<dim3((N + kTile - 1) / kTile, rows), kElemThreads, 0, stream>>>(
        g, x0, static_cast<const bf16*>(ub) + (int64_t)l * B * N, B, l == L - 1, dx0, static_cast<bf16*>(Pb),
        static_cast<bf16*>(Pt), pitch, ws);
    ADAPM_COUNT_LAUNCH();
    ADAPM_CUDA_CHECK(cudaGetLastError());
    sum_partials(stream, ws, rows, N, db + (int64_t)l * N);
    EpiArgs p{};                                          // dh = P W_l
    p.M = B;
    p.Ncol = r;
    p.ob = static_cast<bf16*>(dh);
    p.ot = static_cast<bf16*>(dht);
    p.pitch = pitch;
    gemm<EPI_H>(stream, Pb, B, static_cast<const bf16*>(Wt) + (int64_t)l * r * N, r, N, 0, 1, p);
    EpiArgs q{};                                          // dx_l = G + dh V_l (+ dx_0's accumulator at layer 0)
    q.M = B;
    q.Ncol = N;
    q.G = g;
    q.add = l == 0 ? dx0 : nullptr;
    q.out = l == 0 ? Out{dz, de, E, N} : Out{nullptr, G, 0, N};
    gemm<EPI_RESID>(stream, dh, B, static_cast<const bf16*>(Vt) + (int64_t)l * N * r, N, r, 0, 1, q);
    wgrad(stream, Pt, static_cast<const bf16*>(ht) + (int64_t)l * r * pitch, N, r, B, ws, dW + (int64_t)l * N * r);
    wgrad(stream, dht, static_cast<const bf16*>(xt) + (int64_t)l * N * pitch, r, N, B, ws, dV + (int64_t)l * r * N);
  }
}

}  // namespace cudaops
}  // namespace adapm

// Fused GloVe step (Pennington et al., 2014) for sm_90a: Pull(w_i, c_j) + weighted least squares + AdaGrad + Push in one
// kernel over local HBM / NVLink peers.
//
// Rows hold a word's vector (key 2 w) or its context vector (key 2 w + 1) with the bias in a float4 of its own:
//   [vector (d) | bias, 0, 0, 0 | AdaGrad of the vector (d) | AdaGrad of the bias, 0, 0, 0]
// so the row dimension of the warp-per-positive skeleton (kge_step.cuh) is D = d + 4 and its [emb (D) | acc (D)] push
// (push4) applies unchanged; the three padding elements never receive a gradient and stay 0.
// Rule for one non-zero (i, j, X) with word row (w, b) and context row (c, b~):
//   diff = <w, c> + b + b~ - ln X,  f = (X / x_max)^alpha if X < x_max else 1,  loss = f diff^2 / 2
//   g_w = f diff c,  g_c = f diff w,  g_b = g_b~ = f diff
//   push [-eta g / sqrt(acc + g^2) | g^2] (accumulator as pulled; 0 where g == 0) onto each of the two rows once.
// This is the project's AdaGrad (as for KGE and BPR), not glove.c's, which divides by the old accumulator and clips
// gradients at 100: here every update is bounded by eta, so no clipping is needed.
//
// One warp per non-zero (a warp_step rule with two positives and no negatives); lane l holds float4 l, l + 32, ... of
// both rows. d <= 380 (D <= 384, VPL 1..3) has a float4 body; larger d take the generic path for every non-zero, which
// stages the two rows through the generic Pull / Push path in a per-warp global scratch and runs the scalar body on the
// copies (so does a non-zero with a row in a transitional protocol state at any d).
// Deterministic one-GPU variant (FX): start-of-step reads, fixed-point sums into per-key regions (fx_accum.cuh), one
// loss slot per non-zero, summed in a fixed order (float64).
#include <cuda_runtime.h>

#include "fx_accum.cuh"
#include "kge_step.cuh"
#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {

namespace {

using namespace kge;

// Fixed-point scales of the deterministic mode. |value update| <= eta per push (AdaGrad normalises it): 2^40 leaves
// 2^23 / eta pushes per element and step. The AdaGrad increment of one push is g^2 with |g| <= |f diff| max|row|; it is
// clamped to kFxAdaMax = 2^24 (|g| <= 4096) in this mode only, so that no region can overflow. At 2^28 the region of an
// element holds 2^35 of summed g^2, i.e. 2^11 clamped pushes or 2^35 pushes with |g| <= 1, per step, at a resolution of
// 3.7e-9. With vectors initialised to (U[0,1) - 0.5) / d and ln X <= 20 the first steps have |g| < 1.
constexpr float kFxVal = 1099511627776.f;     // 2^40
constexpr float kFxAda = 268435456.f;         // 2^28
constexpr float kFxAdaMax = 16777216.f;       // 2^24
constexpr int kGloveMaxVpl = 3;               // float4 bodies up to D = 384

struct Args {
  const Key* words;            // word-vector keys (2 i)
  const Key* ctxs;             // context-vector keys (2 j + 1)
  const float* xs;             // co-occurrence values X > 0
  int B, n_neg, d;             // n_neg = 0; d: the row dimension D = vector size + 4
  float eta, x_max, alpha;
  float* scratch;              // generic path: 2 rows per warp
  long long* fx_acc;           // FX: fixed-point regions, per-non-zero loss slots
  const int* fx_cidx;
  float* call_loss;
};

// The step as a warp_step rule: positive (word row, context row). VPL float4 per lane; 0: scalar generic path only.
template <int VPL>
struct Glove {
  static constexpr int kPositives = 2, kMaxDim = kGloveMaxDim + 4, kMaxNeg = 0, kBlocksPerSM = 3;
  static constexpr bool kInPlace = VPL > 0, kStageInSmem = false;
  static __device__ __forceinline__ Key positive(const Args& A, int t, int i) { return i == 0 ? A.words[t] : A.ctxs[t]; }
  static __host__ __device__ __forceinline__ size_t state_bytes(int, int) { return 0; }
  static __host__ __device__ __forceinline__ size_t warp_bytes(int, int) { return 0; }
  static __host__ __device__ __forceinline__ int scratch_rows(int) { return kPositives; }
  static __device__ __forceinline__ int stage_row(int, int i) { return i; }
  template <bool FX, bool GEN>
  static __device__ StepOut body(const Ctx& c, const Args& A, int t, const Rows<2>& rows, bool slow,
                                 const dev::Target* ntg, float* wsm, float* stage);
};

// f diff of a non-zero whose <w, c> + b + b~ is s
__device__ __forceinline__ float weighted_diff(const Args& A, int t, float s, float& loss) {
  const float x = A.xs[t];
  const float diff = s - logf(x);
  const float f = x < A.x_max ? powf(x / A.x_max, A.alpha) : 1.f;
  loss = 0.5f * f * diff * diff;
  return f * diff;
}

// One non-zero: pw / pc its rows (staged copies when slow).
template <int VPL>
template <bool FX, bool GEN>
__device__ __forceinline__ StepOut Glove<VPL>::body(const Ctx&, const Args& A, int t, const Rows<2>& rows, bool slow,
                                                    const dev::Target*, float*, float*) {
  const int lane = threadIdx.x & 31;
  const int D = A.d, d = D - 4, nv = D >> 2, nb = nv - 1;   // float4 nb holds the bias
  float* const pw = rows.p[0];
  float* const pc = rows.p[1];
  long long *fw = nullptr, *fc = nullptr;
  if (FX) {
    fw = fx::region(A.fx_acc, A.fx_cidx, A.words[t], 2 * D);
    fc = fx::region(A.fx_acc, A.fx_cidx, A.ctxs[t], 2 * D);
  }
  float loss;
  if constexpr (VPL == 0 || GEN) {
    float s = 0.f;
    for (int z = lane; z < d; z += 32) s += pw[z] * pc[z];
    const float fd = weighted_diff(A, t, dev::warp_sum(s) + pw[d] + pc[d], loss);
    for (int z = lane; z < D; z += 32) {
      const float gw = z < d ? fd * pc[z] : z == d ? fd : 0.f;
      const float gc = z < d ? fd * pw[z] : z == d ? fd : 0.f;
      const float uw = gw != 0.f ? -A.eta * gw * rsqrtf(pw[D + z] + gw * gw) : 0.f;
      const float uc = gc != 0.f ? -A.eta * gc * rsqrtf(pc[D + z] + gc * gc) : 0.f;
      if (FX) {
        fx::add1(fw, z, D, uw, kFxVal); fx::add1(fw + D, z, D, fminf(gw * gw, kFxAdaMax), kFxAda);
        fx::add1(fc, z, D, uc, kFxVal); fx::add1(fc + D, z, D, fminf(gc * gc, kFxAdaMax), kFxAda);
      } else {
        // staged copies: the generic path pushes [update | g^2]
        pw[z] = uw; pw[D + z] = gw * gw;
        pc[z] = uc; pc[D + z] = gc * gc;
      }
    }
    __syncwarp();
  } else {
    float4 w[VPL], c[VPL];
    load_row<VPL>(pw, nv, lane, w);
    load_row<VPL>(pc, nv, lane, c);
    float s = 0.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int j = lane + 32 * v;
      s += j < nb ? dot4(w[v], c[v]) : j == nb ? w[v].x + c[v].x : 0.f;
    }
    const float fd = weighted_diff(A, t, dev::warp_sum(s), loss);
    const float4 gb = make_float4(fd, 0.f, 0.f, 0.f);
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int j = lane + 32 * v;
      if (j < nv) {
        push4<FX>(pw, D, j, j < nb ? mul4(c[v], fd) : gb, slow, fw, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
        push4<FX>(pc, D, j, j < nb ? mul4(w[v], fd) : gb, slow, fc, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
      }
    }
  }
  return {loss, 0u, 0u, 0ull};
}

template <int VPL, bool FX>
__global__ void __launch_bounds__(kStepThreads, 3)
glove_step_kernel(const __grid_constant__ Ctx c, const __grid_constant__ Args A, float* __restrict__ loss_out,
                  unsigned long long* __restrict__ stats) {
  warp_step<Glove<VPL>, FX>(c, A, loss_out, stats);
}

template <bool FX>
void launch_shape(int vpl, CudaBackend& be, cudaStream_t stream, const Args& A, float* loss_out,
                  unsigned long long* stats) {
  switch (vpl) {
    case 1: launch_step<Glove<1>, glove_step_kernel<1, FX>>(be, stream, A, loss_out, stats); break;
    case 2: launch_step<Glove<2>, glove_step_kernel<2, FX>>(be, stream, A, loss_out, stats); break;
    case 3: launch_step<Glove<3>, glove_step_kernel<3, FX>>(be, stream, A, loss_out, stats); break;
    default: launch_step<Glove<0>, glove_step_kernel<0, FX>>(be, stream, A, loss_out, stats); break;
  }
}

}  // namespace

void glove_step(CudaBackend& be, cudaStream_t stream, const Key* words, const Key* ctxs, const float* xs, int n, int d,
                float eta, float x_max, float alpha, float* loss_out, unsigned long long* stats, bool deterministic) {
  if (n == 0) return;
  ADAPM_CHECK(d % 4 == 0 && d >= 4 && d <= kGloveMaxDim,
              "glove_step: the vector size must be a multiple of 4 in [4, " << kGloveMaxDim << "]");
  const int D = d + 4;
  int vpl = (D / 4 + 31) / 32;
  if (vpl > kGloveMaxVpl) vpl = 0;
  Args A;
  A.words = words; A.ctxs = ctxs; A.xs = xs; A.B = n; A.n_neg = 0; A.d = D;
  A.eta = eta; A.x_max = x_max; A.alpha = alpha;
  // deterministic: every key (word or context row, both 2 D long) gets a [D | D] region
  const fx::Source src[2] = {{words, n, 1}, {ctxs, n, 1}};
  run_step(be, stream, A, deterministic, src, 2, 2 * D, kFxVal, kFxAda, loss_out, [&](auto fx, float* lo) {
    launch_shape<decltype(fx)::value>(vpl, be, stream, A, lo, stats);
  });
}

}  // namespace cudaops
}  // namespace adapm

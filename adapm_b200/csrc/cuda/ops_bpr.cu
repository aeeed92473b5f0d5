// Fused BPR (Bayesian personalised ranking) step of implicit-feedback matrix factorisation for sm_90a: Pull(w_u, h_i,
// negatives) + pairwise logistic loss + L2 + AdaGrad + Push in one kernel over local HBM / NVLink peers.
//
// Rows are the squared-loss MF layout [factors (rank) | AdaGrad (rank)]: user keys and item keys alike. Rule (one
// positive (u, i) with n negative item keys j_1..j_n; w_u, h_i, h_j the start-of-triple factors):
//   x_j = <w_u, h_i> - <w_u, h_j>,  loss = sum_j softplus(-x_j)  (= -log sigmoid(x_j); L2 is not part of the loss)
//   c_j = sigmoid(-x_j),  C = sum_j c_j,  S = sum_j c_j h_j
//   g_u = S - C h_i + lam w_u,  g_i = -C w_u + lam h_i,  g_j = c_j w_u + lam h_j
//   push [-eps g / sqrt(acc + g^2) | g^2] (pulled accumulator; 0 where g == 0): u and i once per positive, every negative
//   once per occurrence (2 + n pushes per positive, counted in stats[3]). Negatives are used as given: one equal to i
//   gives x = 0 and its two contributions to h_i cancel; a repeated negative is pushed once per occurrence.
//
// One warp per positive; lane l holds float4 l, l + 32, ... of a row (VPL float4 per lane, rank <= 128 VPL). w_u, h_i
// and the running S stay in registers while the warp streams the n negative rows once each: load h_j, score it, push it
// and add c_j h_j to S; u and i are pushed at the end, so no row is read twice. The negatives' targets are kept per warp
// in shared memory. Rows in a transitional protocol state are staged through the generic Pull / Push path into a per-warp
// global scratch and run the same code on the copies. Deterministic one-GPU variant (FX): start-of-step reads,
// fixed-point sums into per-key regions (fx_accum.cuh), one loss slot per positive.
// The in-place variant reads each row once, when the warp reaches it: a negative that repeats within the positive, or a
// key that another positive of the step has pushed, is read with the updates already added (Hogwild semantics, as for
// the other in-place steps). The deterministic variant reads unchanged rows.
#include <cuda_runtime.h>

#include <algorithm>

#include "fx_accum.cuh"
#include "kge_step.cuh"
#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {

namespace {

using namespace kge;

// Fixed-point scales of the deterministic mode. |value update| <= eps per push (AdaGrad normalises it): 2^40 leaves
// 2^23 / eps pushes per element and step. One push's gradient is bounded by the factors: c_j <= 1, so an element of g_j
// is at most |w_u| + lam |h_j|, of g_i at most n |w_u| + lam |h_i| and of g_u at most 2 n max|h| + lam |w_u|. The AdaGrad
// increment of one push is clamped to kFxAdaMax = 2^24 (|g| <= 4096) in this mode only, so that no region can overflow;
// factors of magnitude below 4096 / (2 n + 1) (16 at n = 128) never reach the clamp. At 2^28 the region of an element
// holds 2^35 of summed g^2, i.e. 2^11 clamped pushes or 2^35 pushes with |g| <= 1, per step, at a resolution of 3.7e-9.
constexpr float kFxVal = 1099511627776.f;     // 2^40
constexpr float kFxAda = 268435456.f;         // 2^28
constexpr float kFxAdaMax = 16777216.f;       // 2^24

template <int VPL>
__device__ __forceinline__ float dot(const float4 (&a)[VPL], const float4 (&b)[VPL]) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) s += dot4(a[i], b[i]);
  return dev::warp_sum(s);
}

struct Args {
  const Key* users;
  const Key* pos;
  const Key* neg;              // [B, n_neg] item keys
  int B, n_neg, d;             // d: the rank
  float eps, lam;
  float* scratch;              // generic path: 3 rows per warp
  long long* fx_acc;           // FX: fixed-point regions, per-positive loss slots
  const int* fx_cidx;
  float* call_loss;
};

// The step as a warp_step rule (kge_step.cuh): positive (u, i), targets only in shared memory.
template <int VPL>
struct Bpr {
  static constexpr int kPositives = 2, kMaxDim = kBprMaxRank, kMaxNeg = kBprMaxNeg, kBlocksPerSM = 4;
  static constexpr bool kInPlace = true, kStageInSmem = false;
  static __device__ __forceinline__ Key positive(const Args& A, int t, int i) { return i == 0 ? A.users[t] : A.pos[t]; }
  static __host__ __device__ __forceinline__ size_t state_bytes(int, int) { return 0; }
  static __host__ __device__ __forceinline__ size_t warp_bytes(int, int n_neg) {
    return (size_t)n_neg * sizeof(dev::Target);
  }
  static __host__ __device__ __forceinline__ int scratch_rows(int) { return kPositives + 1; }
  static __device__ __forceinline__ int stage_row(int, int i) { return i; }
  static __device__ __forceinline__ bool neg_pushed(const StepOut&, int) { return true; }
  template <bool FX, bool GEN>
  static __device__ StepOut body(const Ctx& c, const Args& A, int t, const Rows<2>& rows, bool slow,
                                 const dev::Target* ntg, float* wsm, float* my_scratch);
};

// One positive and its negatives: pu / pi the positive's rows.
template <int VPL>
template <bool FX, bool GEN>
__device__ __forceinline__ StepOut Bpr<VPL>::body(const Ctx& c, const Args& A, int t, const Rows<2>& rows, bool slow,
                                                  const dev::Target* ntg, float*, float* my_scratch) {
  const int lane = threadIdx.x & 31;
  const int rank = A.d, nv = rank >> 2, n_neg = A.n_neg;
  float* const pu = rows.p[0];
  float* const pi = rows.p[1];
  StepOut out = {0.f, 0u, 0u, 0ull};
  float4 w[VPL], h[VPL], s[VPL], e[VPL];
  load_row<VPL>(pu, nv, lane, w);
  load_row<VPL>(pi, nv, lane, h);
#pragma unroll
  for (int i = 0; i < VPL; ++i) s[i] = f4(0.f);
  const float xui = dot<VPL>(w, h);
  float C = 0.f;

  // ---- the n negatives, one row at a time
  for (int q = 0; q < n_neg; ++q) {
    const Key kn = A.neg[(size_t)t * n_neg + q];
    float* pn = ntg[q].row;
    const bool nslow = !pn;
    if (GEN && nslow) {
      ++out.slow;
      pn = my_scratch + 4 * rank;
      if (!dev::slow_pull(c, kn, pn)) continue;
    }
    load_row<VPL>(pn, nv, lane, e);
    const float x = xui - dot<VPL>(w, e);
    out.loss += softplus(-x);
    const float cq = sigmoid(-x);
    C += cq;
    long long* rg = FX ? fx::region(A.fx_acc, A.fx_cidx, kn, 2 * rank) : nullptr;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int j = lane + 32 * i;
      if (j < nv) push4<FX>(pn, rank, j, add4(mul4(w[i], cq), mul4(e[i], A.lam)), GEN && nslow, rg, nv, A.eps, kFxVal,
                            kFxAda, kFxAdaMax);
      s[i] = add4(s[i], mul4(e[i], cq));
    }
    if (GEN && nslow && !FX) {
      if (dev::slow_push(c, kn, pn)) ++out.upd;
    } else {
      ++out.upd;
    }
  }

  // ---- the positive's rows: g_u = S - C h_i + lam w_u, g_i = -C w_u + lam h_i, one push each
  long long *fu = nullptr, *fi = nullptr;
  if (FX) {
    fu = fx::region(A.fx_acc, A.fx_cidx, A.users[t], 2 * rank);
    fi = fx::region(A.fx_acc, A.fx_cidx, A.pos[t], 2 * rank);
  }
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int j = lane + 32 * i;
    if (j < nv) {
      push4<FX>(pu, rank, j, add4(sub4(s[i], mul4(h[i], C)), mul4(w[i], A.lam)), slow, fu, nv, A.eps, kFxVal, kFxAda,
                kFxAdaMax);
      push4<FX>(pi, rank, j, add4(mul4(w[i], -C), mul4(h[i], A.lam)), slow, fi, nv, A.eps, kFxVal, kFxAda, kFxAdaMax);
    }
  }
  __syncwarp();
  return out;
}

template <int VPL, bool FX>
__global__ void __launch_bounds__(kStepThreads, 1)
mf_bpr_step_kernel(const __grid_constant__ Ctx c, const __grid_constant__ Args A, float* __restrict__ loss_out,
                   unsigned long long* __restrict__ stats) {
  warp_step<Bpr<VPL>, FX>(c, A, loss_out, stats);
}

template <bool FX>
void launch_shape(int vpl, CudaBackend& be, cudaStream_t stream, const Args& A, float* loss_out,
                  unsigned long long* stats) {
  switch (vpl) {
    case 1: launch_step<Bpr<1>, mf_bpr_step_kernel<1, FX>>(be, stream, A, loss_out, stats); break;
    case 2: launch_step<Bpr<2>, mf_bpr_step_kernel<2, FX>>(be, stream, A, loss_out, stats); break;
    case 3: launch_step<Bpr<3>, mf_bpr_step_kernel<3, FX>>(be, stream, A, loss_out, stats); break;
    default: launch_step<Bpr<4>, mf_bpr_step_kernel<4, FX>>(be, stream, A, loss_out, stats); break;
  }
}

}  // namespace

void mf_bpr_step(CudaBackend& be, cudaStream_t stream, const Key* users, const Key* pos, const Key* neg, int B, int n_neg,
                 int rank, float eps, float lam, float* loss_out, unsigned long long* stats, bool deterministic) {
  if (B == 0) return;
  ADAPM_CHECK(rank % 4 == 0 && rank >= 4 && rank <= kBprMaxRank,
              "mf_bpr_step: rank must be a multiple of 4 in [4, " << kBprMaxRank << "]");
  ADAPM_CHECK(n_neg >= 1 && n_neg <= kBprMaxNeg, "mf_bpr_step: the negatives per positive must be in [1, " << kBprMaxNeg
                                                                                                            << "]");
  const int vpl = (rank / 4 + 31) / 32;
  Args A;
  A.users = users; A.pos = pos; A.neg = neg; A.B = B; A.n_neg = n_neg; A.d = rank;
  A.eps = eps; A.lam = lam;
  // deterministic: every key (user or item, both 2 rank long) gets a [rank | rank] region
  const fx::Source src[3] = {{users, B, 1}, {pos, B, 1}, {neg, (long)B * n_neg, 1}};
  run_step(be, stream, A, deterministic, src, 3, 2 * rank, kFxVal, kFxAda, loss_out, [&](auto fx, float* lo) {
    launch_shape<decltype(fx)::value>(vpl, be, stream, A, lo, stats);
  });
}

}  // namespace cudaops
}  // namespace adapm

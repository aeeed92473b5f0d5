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

constexpr int kThreads = 256;
// the backend's step buffer that holds the generic path's staged rows (shared with the KGE steps, never concurrently on
// one stream)
constexpr int kScratchBuf = CudaBackend::kStepBuffers - 1;

// Fixed-point scales of the deterministic mode. |value update| <= eps per push (AdaGrad normalises it): 2^40 leaves
// 2^23 / eps pushes per element and step. One push's gradient is bounded by the factors: c_j <= 1, so an element of g_j
// is at most |w_u| + lam |h_j|, of g_i at most n |w_u| + lam |h_i| and of g_u at most 2 n max|h| + lam |w_u|. The AdaGrad
// increment of one push is clamped to kFxAdaMax = 2^24 (|g| <= 4096) in this mode only, so that no region can overflow;
// factors of magnitude below 4096 / (2 n + 1) (16 at n = 128) never reach the clamp. At 2^28 the region of an element
// holds 2^35 of summed g^2, i.e. 2^11 clamped pushes or 2^35 pushes with |g| <= 1, per step, at a resolution of 3.7e-9.
constexpr float kFxVal = 1099511627776.f;     // 2^40
constexpr float kFxAda = 268435456.f;         // 2^28
constexpr float kFxAdaMax = 16777216.f;       // 2^24

__device__ __forceinline__ float softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoid(float x) {
  const float e = expf(-fabsf(x));
  return x >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
}

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
  int B, n_neg, rank;
  float eps, lam;
  float* scratch;              // generic path: 3 rows per warp
  long long* fx_acc;           // FX: fixed-point regions, per-positive loss slots
  const int* fx_cidx;
  float* call_loss;
};

struct PosOut {
  float loss;
  unsigned upd, slow;
};

// One positive and its negatives. pu / pi: the positive's rows, or (slow) their staged copies in global scratch that are
// pushed through the generic path afterwards. ntg: the negatives' targets (row == nullptr: not resolved). GEN: negatives
// in a transitional state are staged one at a time (only the out-of-line generic path calls slow_pull / slow_push; the
// kernel's own loop has no calls, so nothing it holds is spilled around them).
template <int VPL, bool FX, bool GEN>
__device__ __forceinline__ PosOut positive_body(const Ctx& c, const Args& A, int t, float* pu, float* pi, bool slow,
                                                const dev::Target* ntg, float* my_scratch) {
  const int lane = threadIdx.x & 31;
  const int rank = A.rank, nv = rank >> 2, n_neg = A.n_neg;
  PosOut out = {0.f, 0u, 0u};
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

// Generic path of a positive with a row in a transitional protocol state: the positive's rows are staged through
// slow_pull (and pushed back through slow_push), negatives one at a time. (Out of line: the calls would otherwise make
// the kernel spill everything it holds around them.)
template <int VPL, bool FX>
__device__ __noinline__ PosOut positive_generic(const Ctx& c, const Args& A, int t, float* pu, float* pi,
                                                const dev::Target* ntg, float* my_scratch) {
  const int L = 2 * A.rank;
  const bool slow = !pu || !pi;
  PosOut out = {0.f, 0u, 0u};
  const Key ku = A.users[t], ki = A.pos[t];
  if (slow) {
    out.slow = 1;
    if (!dev::slow_pull(c, ku, my_scratch) || !dev::slow_pull(c, ki, my_scratch + L)) return out;
    pu = my_scratch; pi = my_scratch + L;
  }
  PosOut r = positive_body<VPL, FX, true>(c, A, t, pu, pi, slow, ntg, my_scratch);
  r.slow += out.slow;
  if (slow && !FX) {
    bool ok = dev::slow_push(c, ku, pu);
    ok = dev::slow_push(c, ki, pi) && ok;
    r.upd += ok ? 2 : 0;
  } else {
    r.upd += 2;
  }
  return r;
}

template <int VPL, bool FX>
__global__ void __launch_bounds__(kThreads, 1)
mf_bpr_step_kernel(const __grid_constant__ Ctx c, const __grid_constant__ Args A, float* __restrict__ loss_out,
                   unsigned long long* __restrict__ stats) {
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  extern __shared__ float4 bpr_smem[];
  dev::Target* const ntg = reinterpret_cast<dev::Target*>(bpr_smem) + (size_t)(threadIdx.x >> 5) * A.n_neg;
  float loss_acc = 0.f;
  unsigned n_local = 0, n_remote = 0, n_slow = 0, n_upd = 0;

  for (int t = warp; t < A.B; t += nwarps) {
    // lanes 0 and 1 resolve u and i; lane l resolves negatives l, l + 32, ...
    dev::Target tg;
    tg.row = nullptr; tg.version = nullptr; tg.flag = nullptr;
    if (lane < 2) {
      const Key k = lane == 0 ? A.users[t] : A.pos[t];
      tg = dev::resolve_fast(c, k, class_of_key(c, k), &n_local, &n_remote);
    }
    bool ok = lane >= 2 || tg.row;
    for (int q = lane; q < A.n_neg; q += 32) {
      const Key k = A.neg[(size_t)t * A.n_neg + q];
      const dev::Target nt = dev::resolve_fast(c, k, class_of_key(c, k), &n_local, &n_remote);
      ntg[q] = nt;
      ok = ok && nt.row;
    }
    __syncwarp();
    float* pu = (float*)__shfl_sync(0xffffffffu, (unsigned long long)tg.row, 0);
    float* pi = (float*)__shfl_sync(0xffffffffu, (unsigned long long)tg.row, 1);
    PosOut r;
    if (__all_sync(0xffffffffu, ok)) {
      r = positive_body<VPL, FX, false>(c, A, t, pu, pi, false, ntg, nullptr);
      if (lane < 2) dev::mark_pushed(tg);
      r.upd += 2;
    } else {
      r = positive_generic<VPL, FX>(c, A, t, pu, pi, ntg, A.scratch + (size_t)warp * 6 * A.rank);
      if (lane < 2 && pu && pi) dev::mark_pushed(tg);
    }
    for (int q = lane; q < A.n_neg; q += 32)
      if (ntg[q].row) dev::mark_pushed(ntg[q]);
    __syncwarp();
    n_upd += r.upd;
    n_slow += r.slow;
    if (FX) { if (lane == 0) A.call_loss[t] = r.loss; }
    else loss_acc += r.loss;
  }

  __syncwarp();
  if (!FX && lane == 0 && loss_out) atomicAdd(loss_out, loss_acc);
  unsigned sl = n_local, sr = n_remote;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sl += __shfl_xor_sync(0xffffffffu, sl, o);
    sr += __shfl_xor_sync(0xffffffffu, sr, o);
  }
  if (lane == 0 && stats) {
    if (sl) atomicAdd(stats + 0, (unsigned long long)sl);
    if (sr) atomicAdd(stats + 1, (unsigned long long)sr);
    if (n_slow) atomicAdd(stats + 2, (unsigned long long)n_slow);
    if (n_upd) atomicAdd(stats + 3, (unsigned long long)n_upd);
  }
  dev::cta_exit(c);
}

template <int VPL, bool FX>
void launch(cudaStream_t stream, int blocks, const Ctx& c, const Args& A, float* loss_out, unsigned long long* stats) {
  static bool attr_set = false;
  if (!attr_set) {
    ADAPM_CUDA_CHECK(cudaFuncSetAttribute(mf_bpr_step_kernel<VPL, FX>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)(kThreads / 32 * kBprMaxNeg * sizeof(dev::Target))));
    attr_set = true;
  }
  mf_bpr_step_kernel<VPL, FX><<<blocks, kThreads, kThreads / 32 * A.n_neg * sizeof(dev::Target), stream>>>(c, A, loss_out,
                                                                                                          stats);
}

template <bool FX>
void launch_shape(int vpl, cudaStream_t stream, int blocks, const Ctx& c, const Args& A, float* loss_out,
                  unsigned long long* stats) {
  switch (vpl) {
    case 1: launch<1, FX>(stream, blocks, c, A, loss_out, stats); break;
    case 2: launch<2, FX>(stream, blocks, c, A, loss_out, stats); break;
    case 3: launch<3, FX>(stream, blocks, c, A, loss_out, stats); break;
    default: launch<4, FX>(stream, blocks, c, A, loss_out, stats); break;
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
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  be.track_stream(stream);
  const Ctx& c = be.ctx();
  const int warps_per_block = kThreads / 32;
  const int blocks = std::min((B + warps_per_block - 1) / warps_per_block, be.num_sms() * 4);
  // generic-path scratch (rows in a transitional protocol state): three rows of 2 rank per warp
  float* scratch = static_cast<float*>(
      be.step_buffer(kScratchBuf, (size_t)blocks * warps_per_block * 6 * (size_t)rank * sizeof(float)));
  const int vpl = (rank / 4 + 31) / 32;
  Args A;
  A.users = users; A.pos = pos; A.neg = neg; A.B = B; A.n_neg = n_neg; A.rank = rank;
  A.eps = eps; A.lam = lam; A.scratch = scratch;
  A.fx_acc = nullptr; A.fx_cidx = nullptr; A.call_loss = nullptr;
  if (deterministic) {
    // one GPU, start-of-step reads: every key (user or item, both 2 rank long) gets a [rank | rank] region
    const fx::Source src[3] = {{users, B, 1}, {pos, B, 1}, {neg, (long)B * n_neg, 1}};
    CudaBackend::FxScratch& fxs = fx::begin(be, stream, src, 3, 2 * rank, B);
    A.fx_acc = fxs.acc; A.fx_cidx = fxs.cidx; A.call_loss = fxs.call_loss;
    launch_shape<true>(vpl, stream, blocks, c, A, nullptr, stats);
    ADAPM_COUNT_LAUNCH();
    ADAPM_CUDA_CHECK(cudaGetLastError());
    fx::apply(be, stream, 2 * rank, kFxVal, kFxAda, 0.f, B, loss_out);
    return;
  }
  launch_shape<false>(vpl, stream, blocks, c, A, loss_out, stats);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

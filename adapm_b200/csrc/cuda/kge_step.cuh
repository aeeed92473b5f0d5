// The warp-per-positive steps: TransE, RotatE (ops_transe.cu, ops_rotate.cu) and BPR (ops_bpr.cu) with sampled
// negatives, ComplEx, RESCAL (ops_kge.cu) and squared-loss matrix factorisation (ops_mf.cu) without. Device helpers
// (float4 arithmetic, row loads into a lane's float4 registers, the three-mode AdaGrad push: in place, onto a staged
// copy, into a fixed-point region) and the skeleton the six share: the kernel's loop over positives with its fast /
// generic split (warp_step), the generic path (step_generic) and the host side (launch_step, run_step).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <type_traits>

#include "fx_accum.cuh"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {
namespace kge {

constexpr int kStepThreads = 256;

__device__ __forceinline__ float4 f4(float v) { return make_float4(v, v, v, v); }
__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 sub4(float4 a, float4 b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
__device__ __forceinline__ float4 mul4(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float4 mul4(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float4 fma4(float4 a, float4 b, float4 c) {
  return make_float4(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y), fmaf(a.z, b.z, c.z), fmaf(a.w, b.w, c.w));
}
__device__ __forceinline__ float dot4(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
__device__ __forceinline__ float4 ld4(const float* p, int j) { return *reinterpret_cast<const float4*>(p + 4 * j); }
__device__ __forceinline__ void st4(float* p, int j, float4 v) { *reinterpret_cast<float4*>(p + 4 * j) = v; }

// float4 lane, lane + 32, ... of a row (zeros past nv float4)
template <int VPL>
__device__ __forceinline__ void load_row(const float* row, int nv, int lane, float4 (&v)[VPL]) {
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int j = lane + 32 * i;
    v[i] = j < nv ? dev::ld_row4(row + 4 * j) : f4(0.f);
  }
}

// AdaGrad push of gradient g onto float4 j of a row [emb (d) | acc (d)] whose accumulators a the caller loaded: in place
// (REDs), onto a staged copy (the generic path pushes it afterwards) or into the key's fixed-point region (values scaled
// by fx_val, AdaGrad increments clamped to fx_ada_max and scaled by fx_ada).
template <bool FX>
__device__ __forceinline__ void push4(float* row, int d, int j, float4 g, float4 a, bool staged, long long* region,
                                      int nv, float eta, float fx_val, float fx_ada, float fx_ada_max) {
  const float4 ua = make_float4(g.x * g.x, g.y * g.y, g.z * g.z, g.w * g.w);
  const float4 ue = make_float4(g.x != 0.f ? -eta * g.x * rsqrtf(a.x + ua.x) : 0.f,
                                g.y != 0.f ? -eta * g.y * rsqrtf(a.y + ua.y) : 0.f,
                                g.z != 0.f ? -eta * g.z * rsqrtf(a.z + ua.z) : 0.f,
                                g.w != 0.f ? -eta * g.w * rsqrtf(a.w + ua.w) : 0.f);
  if (FX) {
    fx::add4(region, j, nv, ue, fx_val);
    fx::add4(region + d, j, nv,
             make_float4(fminf(ua.x, fx_ada_max), fminf(ua.y, fx_ada_max), fminf(ua.z, fx_ada_max),
                         fminf(ua.w, fx_ada_max)),
             fx_ada);
  } else if (staged) {
    *reinterpret_cast<float4*>(row + 4 * j) = ue;
    *reinterpret_cast<float4*>(row + d + 4 * j) = ua;
  } else {
    dev::red_row4(row + 4 * j, ue);
    dev::red_row4(row + d + 4 * j, ua);
  }
}
// the same, loading the accumulators after g
template <bool FX>
__device__ __forceinline__ void push4(float* row, int d, int j, float4 g, bool staged, long long* region, int nv,
                                      float eta, float fx_val, float fx_ada, float fx_ada_max) {
  push4<FX>(row, d, j, g, dev::ld_row4(row + d + 4 * j), staged, region, nv, eta, fx_val, fx_ada, fx_ada_max);
}

__device__ __forceinline__ float softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoid(float x) {
  const float e = expf(-fabsf(x));
  return x >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
}

// What one positive adds to its warp's loss and counters. pushed: bit q set when negative q was pushed in place (read
// only by rules whose negatives may push nothing, see Rule::neg_pushed).
struct StepOut {
  float loss;
  unsigned upd, slow;
  unsigned long long pushed;
};

// The positive's NP rows: store rows, nullptr (not resolved) or staged copies.
template <int NP>
struct Rows {
  float* p[NP];
};

// A step has an Args struct (B, n_neg, d, neg = [B, n_neg] keys, scratch, fx_acc, fx_cidx, call_loss and its own; a
// step without negatives has n_neg = 0 and no neg) and a Rule type with
//   kPositives                   NP, the keys of a positive (3: s, r, o; 2: u, i)
//   kMaxDim, kMaxNeg             the largest d and n_neg it takes (kMaxNeg = 0: no negatives, their loops compile away)
//   kInPlace                     false: no body for in-place rows at this shape; no key is resolved and every positive
//                                takes the generic path
//   kBlocksPerSM                 the grid's cap of CTAs per SM
//   kStageInSmem                 the generic path stages the positive's rows at the start of the warp's shared memory
//                                (its state), else in global scratch
//   positive(A, t, i)            key i of positive t
//   state_bytes(d, n_neg)        its own per-warp shared memory; the negatives' targets follow it
//   warp_bytes(d, n_neg)         the per-warp stride: state_bytes + n_neg targets (rounded up as the rule needs)
//   scratch_rows(d)              the generic path's global scratch per warp, in rows of 2 d floats (0 with kStageInSmem)
//   stage_row(d, i)              where positive i's row is staged, in rows of 2 d floats
//   neg_pushed(out, q)           whether negative q was pushed (then its mark follows; only with negatives)
//   body<FX, GEN>(c, A, t, rows, slow, ntg, wsm, stage)
//     one positive and its negatives on rows (slow: they are staged copies that the generic path pushes afterwards);
//     ntg: the negatives' targets (row == nullptr: not resolved); GEN: negatives in a transitional state are staged one
//     at a time after the positive's rows (only the out-of-line generic path calls slow_pull / slow_push; the kernel's
//     own loop has no calls, so nothing it holds is spilled around them). It counts its negatives' pushes and stagings.

// Generic path of a positive with a row in a transitional protocol state: the positive's rows are staged through
// slow_pull into stage and pushed back through slow_push, negatives one at a time. (Out of line: the calls would
// otherwise make the kernel spill everything it holds around them.)
template <class Rule, bool FX, class Args>
__device__ __noinline__ StepOut step_generic(const Ctx& c, const Args& A, int t, Rows<Rule::kPositives> rows,
                                             const dev::Target* ntg, float* wsm, float* stage) {
  constexpr int NP = Rule::kPositives;
  const int L = 2 * A.d;
  bool slow = false;
#pragma unroll
  for (int i = 0; i < NP; ++i) slow = slow || !rows.p[i];
  StepOut out = {0.f, 0u, 0u, 0ull};
  if (slow) {
    out.slow = 1;
#pragma unroll
    for (int i = 0; i < NP; ++i) {
      if (!dev::slow_pull(c, Rule::positive(A, t, i), stage + Rule::stage_row(A.d, i) * L)) return out;
      rows.p[i] = stage + Rule::stage_row(A.d, i) * L;
    }
  }
  StepOut r = Rule::template body<FX, true>(c, A, t, rows, slow, ntg, wsm, stage);
  r.slow += out.slow;
  if (slow && !FX) {
    bool ok = true;
#pragma unroll
    for (int i = 0; i < NP; ++i) ok = dev::slow_push(c, Rule::positive(A, t, i), rows.p[i]) && ok;
    r.upd += ok ? NP : 0;
  } else {
    r.upd += NP;
  }
  return r;
}

// The kernel of a step: one warp per positive. Lanes below NP resolve the positive's keys, lane l the negatives l,
// l + 32, ... (targets kept per warp in shared memory after the rule's state); a positive whose rows all resolved runs
// the rule's body in place, any other the generic path. Completed pushes are marked (positives, then the negatives the
// rule pushed). FX: one loss slot per positive; else the loss is summed into *loss_out. stats: flush_stats.
template <class Rule, bool FX, class Args>
__device__ __forceinline__ void warp_step(const Ctx& c, const Args& A, float* loss_out, unsigned long long* stats) {
  constexpr int NP = Rule::kPositives;
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  extern __shared__ float4 step_smem[];
  unsigned char* const wbase =
      reinterpret_cast<unsigned char*>(step_smem) + (size_t)(threadIdx.x >> 5) * Rule::warp_bytes(A.d, A.n_neg);
  float* const wsm = reinterpret_cast<float*>(wbase);
  dev::Target* const ntg =
      Rule::kMaxNeg > 0 ? reinterpret_cast<dev::Target*>(wbase + Rule::state_bytes(A.d, A.n_neg)) : nullptr;
  float loss_acc = 0.f;
  unsigned n_local = 0, n_remote = 0, n_slow = 0, n_upd = 0;

  for (int t = warp; t < A.B; t += nwarps) {
    dev::Target tg;
    tg.row = nullptr; tg.version = nullptr; tg.flag = nullptr;
    if (Rule::kInPlace && lane < NP) {
      const Key k = Rule::positive(A, t, lane);
      tg = dev::resolve_fast(c, k, class_of_key(c, k), &n_local, &n_remote);
    }
    bool ok = lane >= NP || tg.row;
    if constexpr (Rule::kMaxNeg > 0) {
      for (int q = lane; q < A.n_neg; q += 32) {
        const Key k = A.neg[(size_t)t * A.n_neg + q];
        const dev::Target nt = dev::resolve_fast(c, k, class_of_key(c, k), &n_local, &n_remote);
        ntg[q] = nt;
        ok = ok && nt.row;
      }
      __syncwarp();
    }
    Rows<NP> rows;
#pragma unroll
    for (int i = 0; i < NP; ++i)
      rows.p[i] = Rule::kInPlace ? (float*)__shfl_sync(0xffffffffu, (unsigned long long)tg.row, i) : nullptr;
    StepOut r;
    if constexpr (!Rule::kInPlace) {
      r = step_generic<Rule, FX>(c, A, t, rows, ntg, wsm,
                                 Rule::kStageInSmem ? wsm : A.scratch + (size_t)warp * Rule::scratch_rows(A.d) * 2 * A.d);
    } else if (__all_sync(0xffffffffu, ok)) {
      r = Rule::template body<FX, false>(c, A, t, rows, false, ntg, wsm, nullptr);
      if (lane < NP) dev::mark_pushed(tg);
      r.upd += NP;
    } else {
      r = step_generic<Rule, FX>(c, A, t, rows, ntg, wsm,
                                 Rule::kStageInSmem ? wsm : A.scratch + (size_t)warp * Rule::scratch_rows(A.d) * 2 * A.d);
      bool resolved = true;   // the positive's rows were pushed in place
#pragma unroll
      for (int i = 0; i < NP; ++i) resolved = resolved && rows.p[i];
      if (lane < NP && resolved) dev::mark_pushed(tg);
    }
    if constexpr (Rule::kMaxNeg > 0) {
      for (int q = lane; q < A.n_neg; q += 32)
        if (ntg[q].row && Rule::neg_pushed(r, q)) dev::mark_pushed(ntg[q]);
    }
    __syncwarp();
    n_upd += r.upd;
    n_slow += r.slow;
    if (FX) { if (lane == 0) A.call_loss[t] = r.loss; }
    else loss_acc += r.loss;
  }

  __syncwarp();
  if (!FX && lane == 0 && loss_out) atomicAdd(loss_out, loss_acc);
  dev::flush_stats(stats, n_local, n_remote, n_slow, n_upd);
  dev::cta_exit(c);
}

// Launches Kernel, a warp_step over Rule, on min(ceil(B / 8), Rule::kBlocksPerSM per SM) CTAs with the rule's per-warp
// shared memory (the limit is raised once, to the layout at the rule's largest shape) and its generic-path scratch (in
// the backend's last step buffer, which the steps share and never use concurrently on one stream).
template <class Rule, auto Kernel, class Args>
void launch_step(CudaBackend& be, cudaStream_t stream, Args A, float* loss_out, unsigned long long* stats) {
  const int warps_per_block = kStepThreads / 32;
  const int blocks = std::min((A.B + warps_per_block - 1) / warps_per_block, be.num_sms() * Rule::kBlocksPerSM);
  A.scratch = static_cast<float*>(be.step_buffer(
      CudaBackend::kStepBuffers - 1,
      (size_t)blocks * warps_per_block * Rule::scratch_rows(A.d) * 2 * (size_t)A.d * sizeof(float)));
  set_max_dynamic_smem<Kernel>((int)(warps_per_block * Rule::warp_bytes(Rule::kMaxDim, Rule::kMaxNeg)));
  Kernel<<<blocks, kStepThreads, warps_per_block * Rule::warp_bytes(A.d, A.n_neg), stream>>>(be.ctx(), A, loss_out,
                                                                                             stats);
}

// Host side of a step (A filled but for scratch and the FX fields): float32 rows, then launch(fx, loss_out) with
// fx = std::false_type (in place) or, deterministic (one GPU, start-of-step reads), std::true_type between fx::begin
// over src (regions in units of `unit` values) and fx::apply with the rule's scales.
template <class Args, class Launch>
void run_step(CudaBackend& be, cudaStream_t stream, Args& A, bool deterministic, const fx::Source* src, int n_src,
              int unit, float fx_val, float fx_ada, float* loss_out, Launch&& launch) {
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  be.track_stream(stream);
  A.fx_acc = nullptr; A.fx_cidx = nullptr; A.call_loss = nullptr;
  if (deterministic) {
    CudaBackend::FxScratch& fxs = fx::begin(be, stream, src, n_src, unit, A.B);
    A.fx_acc = fxs.acc; A.fx_cidx = fxs.cidx; A.call_loss = fxs.call_loss;
    launch(std::true_type{}, nullptr);
    ADAPM_COUNT_LAUNCH();
    ADAPM_CUDA_CHECK(cudaGetLastError());
    fx::apply(be, stream, unit, fx_val, fx_ada, 0.f, A.B, loss_out);
    return;
  }
  launch(std::false_type{}, loss_out);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace kge
}  // namespace cudaops
}  // namespace adapm

// Fused TransE training step for sm_90a: Pull(s, r, o, negatives) + distance + margin-ranking gradient + L2 + AdaGrad +
// Push in one kernel over local HBM / NVLink peers.
//
// Rule (one positive triple, neg = [B, 2n] entity keys: the first n replace the object, the last n the subject):
//   e^ = e / max(|e|_2, 1e-12) for entity rows (the store rows are never rescaled), relation rows as they are
//   x = s^ + r - o^,  D = |x|_p (p = 1 or 2),  u = dD/dx = sign(x) (p = 1, sign(0) = 0) or x / |x| (p = 2, 0 at x = 0)
//   loss = sum_j max(0, margin + D_pos - D_neg_j); pair j is active when its term is > 0
//   active object-corrupted pair: s^ += u - u_j, r += u - u_j, o^ -= u, o'^_j += u_j
//   active subject-corrupted pair: s^ += u, r += u - u_j, o^ += u_j - u, s'^_j -= u_j
//   through the normalisation g_e = (g_e^ - e^ (e^ . g_e^)) / max(|e|, 1e-12); + gamma_e s, gamma_r r, gamma_e o (raw rows)
//   push [-eta g / sqrt(acc + g^2) | g^2] (pulled accumulator; 0 where g == 0): s, r and o once per triple with their
//   summed gradients, every negative of an active pair once; inactive negatives push nothing.
// With k active pairs, U_o / U_s the sums of u_j over the active object- / subject-corrupted pairs:
//   g_s^ = k u - U_o,  g_r = k u - U_o - U_s,  g_o^ = U_s - k u
// so a warp keeps a = s^ + r, b = r - o^, x, U_o and U_s on chip while it streams the 2n negative rows one at a time.
//
// One warp per positive triple; lane l holds float4 l, l + 32, ... of a row (VPL float4 per lane, d <= 128 VPL).
// Rows in a transitional protocol state are staged through the generic Pull / Push path into a per-warp global scratch
// and run the same code on the copies. Deterministic one-GPU variant (FX): start-of-step reads, fixed-point sums into
// per-key regions (fx_accum.cuh), one loss slot per triple.
// The in-place variant reads the positive's rows a second time for the projection and L2 at the end of the triple; a
// negative equal to s or o has already added its update to that row by then, and the second read pairs the new values
// with the norm of the first (Hogwild semantics, as for concurrent triples). The deterministic variant reads unchanged rows.
#include <cuda_runtime.h>

#include <algorithm>

#include "fx_accum.cuh"
#include "kge_step.cuh"
#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {

namespace {

constexpr float kNormEps = 1e-12f;

// Fixed-point scales of the deterministic mode. |value update| <= eta per push (AdaGrad normalises it): 2^40 leaves
// 2^23 / eta pushes per element and step. The gradient has no bound as |e| -> 0 (the 1/|e| factor), so the AdaGrad
// increment of one push is clamped to kFxAdaMax = 2^24 (|g| <= 4096) in this mode only; at 2^28 the region of an element
// holds 2^35 of summed g^2, i.e. 2^11 clamped pushes or 2^35 pushes with |g| <= 1, per step, at a resolution of 3.7e-9.
// Unclamped, |g| of one push stays below 4096 while |e| >= 3 n sqrt(d) / 4096 (about 0.1 at n = 6, d = 512): the subject's
// k u - U_o reaches 3 n sqrt(d) in norm before the 1/|e| factor.
constexpr float kFxVal = 1099511627776.f;     // 2^40
constexpr float kFxAda = 268435456.f;         // 2^28
constexpr float kFxAdaMax = 16777216.f;       // 2^24

using namespace kge;

__device__ __forceinline__ float sgn(float v) { return v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f); }

// 1 / max(|v|_2, eps)
template <int VPL>
__device__ __forceinline__ float inv_norm(const float4 (&v)[VPL]) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) s += dot4(v[i], v[i]);
  return 1.f / fmaxf(sqrtf(dev::warp_sum(s)), kNormEps);
}
template <int P, int VPL>
__device__ __forceinline__ float dist(const float4 (&x)[VPL]) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i)
    s += P == 1 ? fabsf(x[i].x) + fabsf(x[i].y) + fabsf(x[i].z) + fabsf(x[i].w) : dot4(x[i], x[i]);
  s = dev::warp_sum(s);
  return P == 1 ? s : sqrtf(s);
}
// dD/dx for D = dist(x)
template <int P>
__device__ __forceinline__ float4 ddx(float4 x, float inv_d) {
  if (P == 1) return make_float4(sgn(x.x), sgn(x.y), sgn(x.z), sgn(x.w));
  return mul4(x, inv_d);
}

// gradient of a raw entity row from the gradient gh of its normalised copy eh = e * inv: (gh - eh (eh . gh)) * inv
template <int VPL>
__device__ __forceinline__ void unnormalise(float4 (&gh)[VPL], const float4 (&e)[VPL], float inv) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) s += dot4(mul4(e[i], inv), gh[i]);
  const float dt = dev::warp_sum(s);
#pragma unroll
  for (int i = 0; i < VPL; ++i) gh[i] = mul4(sub4(gh[i], mul4(mul4(e[i], inv), dt)), inv);
}

struct Args {
  const Key* subj;
  const Key* rel;
  const Key* obj;
  const Key* neg;              // [B, n_neg]
  int B, n_neg, d;
  float margin, eta, gamma_e, gamma_r;
  float* scratch;              // generic path: 4 rows per warp
  long long* fx_acc;           // FX: fixed-point regions, per-triple loss slots
  const int* fx_cidx;
  float* call_loss;
};

// The step as a warp_step rule (kge_step.cuh): positive (s, r, o). Per-warp shared memory: a = s^ + r | b = r - o^ |
// x | U_o | U_s (d each; each lane touches only its own float4s) | the negatives' targets.
template <int VPL, int P>
struct TransE {
  static constexpr int kPositives = 3, kMaxDim = kTransEMaxDim, kMaxNeg = kTransEMaxNeg, kBlocksPerSM = 4;
  static constexpr bool kInPlace = true, kStageInSmem = false;
  static __device__ __forceinline__ Key positive(const Args& A, int t, int i) {
    return i == 0 ? A.subj[t] : (i == 1 ? A.rel[t] : A.obj[t]);
  }
  static __host__ __device__ __forceinline__ size_t state_bytes(int d, int) { return (size_t)5 * d * sizeof(float); }
  static __host__ __device__ __forceinline__ size_t warp_bytes(int d, int n_neg) {
    return state_bytes(d, n_neg) + (size_t)n_neg * sizeof(dev::Target);
  }
  static __host__ __device__ __forceinline__ int scratch_rows(int) { return kPositives + 1; }
  static __device__ __forceinline__ int stage_row(int, int i) { return i; }
  // an inactive pair pushes nothing (n_neg <= 64: one bit per negative)
  static __device__ __forceinline__ bool neg_pushed(const StepOut& r, int q) { return r.pushed >> q & 1ull; }
  template <bool FX, bool GEN>
  static __device__ StepOut body(const Ctx& c, const Args& A, int t, const Rows<3>& rows, bool slow,
                                 const dev::Target* ntg, float* wsm, float* my_scratch);
};

// One positive triple and its negatives: ps / pr / po the positive's rows.
template <int VPL, int P>
template <bool FX, bool GEN>
__device__ __forceinline__ StepOut TransE<VPL, P>::body(const Ctx& c, const Args& A, int t, const Rows<3>& rows,
                                                        bool slow, const dev::Target* ntg, float* wsm,
                                                        float* my_scratch) {
  const int lane = threadIdx.x & 31;
  const int d = A.d, nv = d >> 2, L = 2 * d, n_neg = A.n_neg, half = n_neg >> 1;
  float* const ps = rows.p[0];
  float* const pr = rows.p[1];
  float* const po = rows.p[2];
  StepOut out = {0.f, 0u, 0u, 0ull};
  float* const sa = wsm; float* const sb = wsm + d; float* const sx = wsm + 2 * d;
  float* const suo = wsm + 3 * d; float* const sus = wsm + 4 * d;
  float4 e[VPL], v[VPL];
  load_row<VPL>(ps, nv, lane, e);
  const float inv_s = inv_norm<VPL>(e);
  load_row<VPL>(pr, nv, lane, v);
#pragma unroll
  for (int i = 0; i < VPL; ++i) v[i] = add4(mul4(e[i], inv_s), v[i]);      // a
  load_row<VPL>(po, nv, lane, e);
  const float inv_o = inv_norm<VPL>(e);
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const float4 oh = mul4(e[i], inv_o);
    e[i] = sub4(v[i], oh);                                                  // x
    const int j = lane + 32 * i;
    if (j < nv) {
      st4(sa, j, v[i]); st4(sx, j, e[i]);
      st4(sb, j, sub4(dev::ld_row4(pr + 4 * j), oh));
      st4(suo, j, f4(0.f)); st4(sus, j, f4(0.f));
    }
  }
  const float Dp = dist<P, VPL>(e);
  int k_act = 0;

  // ---- the 2n negatives, one row at a time
  for (int q = 0; q < n_neg; ++q) {
    const Key kn = A.neg[(size_t)t * n_neg + q];
    float* pn = ntg[q].row;
    const bool nslow = !pn;
    if (GEN && nslow) {
      ++out.slow;
      pn = my_scratch + 3 * L;
      if (!dev::slow_pull(c, kn, pn)) continue;
    }
    load_row<VPL>(pn, nv, lane, e);
    const float inv_n = inv_norm<VPL>(e);
    const bool obj_side = q < half;
    const float* base = obj_side ? sa : sb;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int j = lane + 32 * i;
      const float4 w = j < nv ? ld4(base, j) : f4(0.f);
      v[i] = obj_side ? sub4(w, mul4(e[i], inv_n)) : add4(mul4(e[i], inv_n), w);
    }
    const float Dn = dist<P, VPL>(v);
    const float term = A.margin + Dp - Dn;
    if (!(term > 0.f)) continue;                     // inactive pair: nothing to push
    out.loss += term;
    ++k_act;
    const float inv_dn = Dn > 0.f ? 1.f / Dn : 0.f;
    float* const su = obj_side ? suo : sus;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {   // v becomes the gradient of the negative's normalised row
      const int j = lane + 32 * i;
      const float4 un = ddx<P>(v[i], inv_dn);
      if (j < nv) st4(su, j, add4(ld4(su, j), un));
      v[i] = obj_side ? un : mul4(un, -1.f);
    }
    unnormalise<VPL>(v, e, inv_n);
    long long* rg = FX ? fx::region(A.fx_acc, A.fx_cidx, kn, L) : nullptr;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int j = lane + 32 * i;
      if (j < nv) push4<FX>(pn, d, j, v[i], GEN && nslow, rg, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
    }
    if (GEN && nslow && !FX) {
      if (dev::slow_push(c, kn, pn)) ++out.upd;
    } else {
      if (!nslow) out.pushed |= 1ull << q;
      ++out.upd;
    }
  }

  // ---- the positive's rows: summed gradients, L2 on the raw rows, one push each
  const float inv_dp = Dp > 0.f ? 1.f / Dp : 0.f;
  const float kf = (float)k_act;
  long long *fs = nullptr, *fr = nullptr, *fo = nullptr;
  if (FX) {
    fs = fx::region(A.fx_acc, A.fx_cidx, A.subj[t], L); fr = fx::region(A.fx_acc, A.fx_cidx, A.rel[t], L);
    fo = fx::region(A.fx_acc, A.fx_cidx, A.obj[t], L);
  }
  // g_s^ = k u - U_o, g_r = g_s^ - U_s, g_o^ = U_s - k u
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int j = lane + 32 * i;
    v[i] = j < nv ? sub4(mul4(ddx<P>(ld4(sx, j), inv_dp), kf), ld4(suo, j)) : f4(0.f);
  }
  load_row<VPL>(ps, nv, lane, e);
  unnormalise<VPL>(v, e, inv_s);
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int j = lane + 32 * i;
    if (j < nv) push4<FX>(ps, d, j, add4(v[i], mul4(e[i], A.gamma_e)), slow, fs, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
  }
  load_row<VPL>(pr, nv, lane, e);
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int j = lane + 32 * i;
    if (j < nv) {
      const float4 gr = sub4(sub4(mul4(ddx<P>(ld4(sx, j), inv_dp), kf), ld4(suo, j)), ld4(sus, j));
      push4<FX>(pr, d, j, add4(gr, mul4(e[i], A.gamma_r)), slow, fr, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
    }
  }
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int j = lane + 32 * i;
    v[i] = j < nv ? sub4(ld4(sus, j), mul4(ddx<P>(ld4(sx, j), inv_dp), kf)) : f4(0.f);
  }
  load_row<VPL>(po, nv, lane, e);
  unnormalise<VPL>(v, e, inv_o);
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int j = lane + 32 * i;
    if (j < nv) push4<FX>(po, d, j, add4(v[i], mul4(e[i], A.gamma_e)), slow, fo, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
  }
  __syncwarp();
  return out;
}

template <int VPL, int P, bool FX>
__global__ void __launch_bounds__(kStepThreads, 1)
transe_step_kernel(const __grid_constant__ Ctx c, const __grid_constant__ Args A, float* __restrict__ loss_out,
                   unsigned long long* __restrict__ stats) {
  warp_step<TransE<VPL, P>, FX>(c, A, loss_out, stats);
}

template <int VPL, bool FX>
void launch_p(int p, CudaBackend& be, cudaStream_t stream, const Args& A, float* loss_out, unsigned long long* stats) {
  if (p == 1) launch_step<TransE<VPL, 1>, transe_step_kernel<VPL, 1, FX>>(be, stream, A, loss_out, stats);
  else launch_step<TransE<VPL, 2>, transe_step_kernel<VPL, 2, FX>>(be, stream, A, loss_out, stats);
}

template <bool FX>
void launch_shape(int vpl, int p, CudaBackend& be, cudaStream_t stream, const Args& A, float* loss_out,
                  unsigned long long* stats) {
  switch (vpl) {
    case 1: launch_p<1, FX>(p, be, stream, A, loss_out, stats); break;
    case 2: launch_p<2, FX>(p, be, stream, A, loss_out, stats); break;
    case 3: launch_p<3, FX>(p, be, stream, A, loss_out, stats); break;
    default: launch_p<4, FX>(p, be, stream, A, loss_out, stats); break;
  }
}

}  // namespace

void kge_transe_step(CudaBackend& be, cudaStream_t stream, const Key* subj, const Key* rel, const Key* obj,
                     const Key* neg, int B, int n_neg, int d, int p, float margin, float eta, float gamma_e,
                     float gamma_r, float* loss_out, unsigned long long* stats, bool deterministic) {
  if (B == 0) return;
  ADAPM_CHECK(d % 4 == 0 && d >= 4 && d <= kTransEMaxDim, "kge_transe_step: embedding size must be a multiple of 4 in [4, "
                                                              << kTransEMaxDim << "]");
  ADAPM_CHECK(p == 1 || p == 2, "kge_transe_step: p must be 1 or 2");
  ADAPM_CHECK(n_neg >= 0 && n_neg % 2 == 0 && n_neg <= kTransEMaxNeg,
              "kge_transe_step: the negatives per triple must be an even count <= " << kTransEMaxNeg);
  const int vpl = (d / 4 + 31) / 32;
  Args A;
  A.subj = subj; A.rel = rel; A.obj = obj; A.neg = neg; A.B = B; A.n_neg = n_neg; A.d = d;
  A.margin = margin; A.eta = eta; A.gamma_e = gamma_e; A.gamma_r = gamma_r;
  // deterministic: every key (entity or relation, both 2 d long) gets a [d | d] region
  const fx::Source src[4] = {{subj, B, 1}, {rel, B, 1}, {obj, B, 1}, {neg, (long)B * n_neg, 1}};
  run_step(be, stream, A, deterministic, src, 4, 2 * d, kFxVal, kFxAda, loss_out, [&](auto fx, float* lo) {
    launch_shape<decltype(fx)::value>(vpl, p, be, stream, A, lo, stats);
  });
}

}  // namespace cudaops
}  // namespace adapm

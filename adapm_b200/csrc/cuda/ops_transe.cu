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

constexpr int kThreads = 256;
constexpr float kNormEps = 1e-12f;
// the backend's step buffer that holds the generic path's staged rows (the deterministic SGNS step uses buffers 0 - 9)
constexpr int kScratchBuf = CudaBackend::kStepBuffers - 1;

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

struct TripleOut {
  float loss;
  unsigned upd, slow;
};

// One positive triple and its negatives. ps / pr / po: the positive's rows, or (slow) their staged copies in global
// scratch that are pushed through the generic path afterwards. nt0 / nt1: this lane's negatives lane and lane + 32.
// GEN: negatives in a transitional state are staged one at a time (only the out-of-line generic path calls
// slow_pull / slow_push; the kernel's own loop has no calls, so nothing it holds is spilled around them).
template <int VPL, int P, bool FX, bool GEN>
__device__ __forceinline__ TripleOut triple_body(const Ctx& c, const Args& A, int t, float* ps, float* pr, float* po,
                                                 bool slow, const dev::Target& nt0, const dev::Target& nt1, float* wsm,
                                                 float* my_scratch) {
  const int lane = threadIdx.x & 31;
  const int d = A.d, nv = d >> 2, L = 2 * d, n_neg = A.n_neg, half = n_neg >> 1;
  TripleOut out = {0.f, 0u, 0u};
  // per-warp state in shared memory (each lane touches only its own float4s): a = s^ + r | b = r - o^ | x | U_o | U_s
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
  unsigned long long pushed = 0ull;

  // ---- the 2n negatives, one row at a time
  for (int q = 0; q < n_neg; ++q) {
    const Key kn = A.neg[(size_t)t * n_neg + q];
    float* pn = (float*)__shfl_sync(0xffffffffu, (unsigned long long)(q < 32 ? nt0.row : nt1.row), q & 31);
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
      if (!nslow) pushed |= 1ull << q;
      ++out.upd;
    }
  }
  if (pushed >> lane & 1ull) dev::mark_pushed(nt0);
  if (pushed >> (lane + 32) & 1ull) dev::mark_pushed(nt1);

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

// Generic path of a triple with a row in a transitional protocol state: the positive's rows are staged through
// slow_pull (and pushed back through slow_push), negatives one at a time. (Out of line: the calls would otherwise make
// the kernel spill everything it holds around them.)
template <int VPL, int P, bool FX>
__device__ __noinline__ TripleOut triple_generic(const Ctx& c, const Args& A, int t, float* ps, float* pr, float* po,
                                                 const dev::Target nt0, const dev::Target nt1, float* wsm, float* my_scratch) {
  const int L = 2 * A.d;
  const bool slow = !ps || !pr || !po;
  TripleOut out = {0.f, 0u, 0u};
  const Key ks = A.subj[t], kr = A.rel[t], ko = A.obj[t];
  if (slow) {
    out.slow = 1;
    if (!dev::slow_pull(c, ks, my_scratch) || !dev::slow_pull(c, kr, my_scratch + L) ||
        !dev::slow_pull(c, ko, my_scratch + 2 * L))
      return out;
    ps = my_scratch; pr = my_scratch + L; po = my_scratch + 2 * L;
  }
  TripleOut r = triple_body<VPL, P, FX, true>(c, A, t, ps, pr, po, slow, nt0, nt1, wsm, my_scratch);
  r.slow += out.slow;
  if (slow && !FX) {
    bool ok = dev::slow_push(c, ks, ps);
    ok = dev::slow_push(c, kr, pr) && ok;
    ok = dev::slow_push(c, ko, po) && ok;
    r.upd += ok ? 3 : 0;
  } else {
    r.upd += 3;
  }
  return r;
}

template <int VPL, int P, bool FX>
__global__ void __launch_bounds__(kThreads, 1)
transe_step_kernel(const __grid_constant__ Ctx c, const __grid_constant__ Args A, float* __restrict__ loss_out,
                   unsigned long long* __restrict__ stats) {
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  extern __shared__ float4 transe_smem[];
  float* const wsm = reinterpret_cast<float*>(transe_smem) + (size_t)(threadIdx.x >> 5) * 5 * A.d;
  float loss_acc = 0.f;
  unsigned n_local = 0, n_remote = 0, n_slow = 0, n_upd = 0;

  for (int t = warp; t < A.B; t += nwarps) {
    // lanes 0-2 resolve s, r, o; lane l resolves negatives l and l + 32
    dev::Target tg, nt0, nt1;
    tg.row = nullptr; tg.version = nullptr; tg.flag = nullptr;
    nt0 = tg; nt1 = tg;
    if (lane < 3) {
      const Key k = lane == 0 ? A.subj[t] : (lane == 1 ? A.rel[t] : A.obj[t]);
      tg = dev::resolve_fast(c, k, class_of_key(c, k), &n_local, &n_remote);
    }
    bool ok = lane >= 3 || tg.row;
    if (lane < A.n_neg) {
      const Key k = A.neg[(size_t)t * A.n_neg + lane];
      nt0 = dev::resolve_fast(c, k, class_of_key(c, k), &n_local, &n_remote);
      ok = ok && nt0.row;
    }
    if (lane + 32 < A.n_neg) {
      const Key k = A.neg[(size_t)t * A.n_neg + lane + 32];
      nt1 = dev::resolve_fast(c, k, class_of_key(c, k), &n_local, &n_remote);
      ok = ok && nt1.row;
    }
    float* ps = (float*)__shfl_sync(0xffffffffu, (unsigned long long)tg.row, 0);
    float* pr = (float*)__shfl_sync(0xffffffffu, (unsigned long long)tg.row, 1);
    float* po = (float*)__shfl_sync(0xffffffffu, (unsigned long long)tg.row, 2);
    TripleOut r;
    if (__all_sync(0xffffffffu, ok)) {
      r = triple_body<VPL, P, FX, false>(c, A, t, ps, pr, po, false, nt0, nt1, wsm, nullptr);
      if (lane < 3) dev::mark_pushed(tg);
      r.upd += 3;
    } else {
      r = triple_generic<VPL, P, FX>(c, A, t, ps, pr, po, nt0, nt1, wsm, A.scratch + (size_t)warp * 8 * A.d);
      if (lane < 3 && ps && pr && po) dev::mark_pushed(tg);
    }
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

template <int VPL, int P, bool FX>
void launch(cudaStream_t stream, int blocks, const Ctx& c, const Args& A, float* loss_out, unsigned long long* stats) {
  static bool attr_set = false;
  if (!attr_set) {
    ADAPM_CUDA_CHECK(cudaFuncSetAttribute(transe_step_kernel<VPL, P, FX>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          kThreads / 32 * 5 * kTransEMaxDim * (int)sizeof(float)));
    attr_set = true;
  }
  transe_step_kernel<VPL, P, FX><<<blocks, kThreads, kThreads / 32 * 5 * A.d * sizeof(float), stream>>>(c, A, loss_out,
                                                                                                         stats);
}

template <bool FX>
void launch_shape(int vpl, int p, cudaStream_t stream, int blocks, const Ctx& c, const Args& A, float* loss_out,
                  unsigned long long* stats) {
  switch (vpl * 2 + p - 1) {
    case 2: launch<1, 1, FX>(stream, blocks, c, A, loss_out, stats); break;
    case 3: launch<1, 2, FX>(stream, blocks, c, A, loss_out, stats); break;
    case 4: launch<2, 1, FX>(stream, blocks, c, A, loss_out, stats); break;
    case 5: launch<2, 2, FX>(stream, blocks, c, A, loss_out, stats); break;
    case 6: launch<3, 1, FX>(stream, blocks, c, A, loss_out, stats); break;
    case 7: launch<3, 2, FX>(stream, blocks, c, A, loss_out, stats); break;
    case 8: launch<4, 1, FX>(stream, blocks, c, A, loss_out, stats); break;
    default: launch<4, 2, FX>(stream, blocks, c, A, loss_out, stats); break;
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
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  be.track_stream(stream);
  const Ctx& c = be.ctx();
  const int warps_per_block = kThreads / 32;
  const int blocks = std::min((B + warps_per_block - 1) / warps_per_block, be.num_sms() * 4);
  // generic-path scratch (rows in a transitional protocol state): four rows per warp, one of the backend's step buffers
  float* scratch = static_cast<float*>(
      be.step_buffer(kScratchBuf, (size_t)blocks * warps_per_block * 8 * (size_t)d * sizeof(float)));
  const int vpl = (d / 4 + 31) / 32;
  Args A;
  A.subj = subj; A.rel = rel; A.obj = obj; A.neg = neg; A.B = B; A.n_neg = n_neg; A.d = d;
  A.margin = margin; A.eta = eta; A.gamma_e = gamma_e; A.gamma_r = gamma_r; A.scratch = scratch;
  A.fx_acc = nullptr; A.fx_cidx = nullptr; A.call_loss = nullptr;
  if (deterministic) {
    // one GPU, start-of-step reads: every key (entity or relation, both 2 d long) gets a [d | d] region
    const fx::Source src[4] = {{subj, B, 1}, {rel, B, 1}, {obj, B, 1}, {neg, (long)B * n_neg, 1}};
    CudaBackend::FxScratch& fxs = fx::begin(be, stream, src, 4, 2 * d, B);
    A.fx_acc = fxs.acc; A.fx_cidx = fxs.cidx; A.call_loss = fxs.call_loss;
    launch_shape<true>(vpl, p, stream, blocks, c, A, nullptr, stats);
    ADAPM_COUNT_LAUNCH();
    ADAPM_CUDA_CHECK(cudaGetLastError());
    fx::apply(be, stream, 2 * d, kFxVal, kFxAda, 0.f, B, loss_out);
    return;
  }
  launch_shape<false>(vpl, p, stream, blocks, c, A, loss_out, stats);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

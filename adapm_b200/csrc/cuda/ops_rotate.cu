// Fused RotatE training step for sm_90a: Pull(s, r, o, negatives) + complex rotation + sigmoid loss with self-adversarial
// negative weights + AdaGrad + Push in one kernel over local HBM / NVLink peers.
//
// Rows: entities [z (d) | AdaGrad (d)] with z interleaved (re_0, im_0, re_1, im_1, ...), relations [theta (m) | AdaGrad
// (m)], m = d / 2 phases in radians. Rule (one positive triple, neg = [B, 2n] entity keys: the first n replace the object,
// the last n the subject):
//   rho_i = e^{i theta_i},  x = a o rho - b,  D(x) = sum_i |x_i|,  u_i = x_i / |x_i| (0 where |x_i| = 0)
//   positive: x = s o rho - o;  object side j: x_j = s o rho - o'_j;  subject side j: x_j = s'_j o rho - o
//   w_j = softmax_j(alpha (gamma - D_j)) over the n negatives of a side (constants, no gradient)
//   loss = softplus(D+ - gamma) + 1/2 sum_side sum_j w_j softplus(gamma - D_j)
//   dD/da = conj(rho) o u,  dD/db = -u,  dD/dtheta_i = -Im(conj(u_i) a_i rho_i), each scaled by dL/dD:
//   sigma(D+ - gamma) for the positive, -1/2 w_j sigma(gamma - D_j) for negative j; s, r and o sum their terms,
//   every negative gets its own; + gamma_e s and gamma_e o (raw rows, once per triple); phases get no L2
//   push [-eta g / sqrt(acc + g^2) | g^2] (pulled accumulator; 0 where g == 0): s, r and o once per triple, every
//   negative once (3 + 2n pushes per triple, counted in stats[3]).
//
// One warp per positive triple; lane l holds float4 l, l + 32, ... of an entity row (two complex values each, VPL float4
// per lane, d <= 128 VPL) and the matching float2 of phases. cos / sin of the phases are computed once per triple
// (sincosf). The weights of a side depend on all of its distances, so a side is two passes over its n negative rows:
// the distances first (kept per warp in shared memory), then the gradients; negative rows are read twice. A warp keeps
// s o rho, o, (cos, sin) and the summed gradients of s, o and theta in shared memory while it streams the negatives.
// Rows in a transitional protocol state are staged through the generic Pull / Push path into a per-warp global scratch
// and run the same code on the copies. Deterministic one-GPU variant (FX): start-of-step reads, fixed-point sums into
// per-key regions (fx_accum.cuh), one loss slot per triple.
// The in-place variant reads a negative's row again in the second pass; concurrent triples (and this triple's own
// earlier negatives, when a key repeats) may have updated it in between, and the raw s and o rows for L2 are read at the
// end of the triple, after the negatives' pushes (Hogwild semantics, as for concurrent triples). The deterministic
// variant reads unchanged rows.
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

// Fixed-point scales of the deterministic mode. |value update| <= eta per push (AdaGrad normalises it): 2^40 leaves
// 2^23 / eta pushes per element and step. One push's gradient is bounded by the model: an entity element gets at most
// 1 (positive) + 1/2 (the weights of a side sum to 1) from the distance terms plus gamma_e |e|, a phase at most
// 1.5 |s_i|. The AdaGrad increment of one push is still clamped to kFxAdaMax = 2^24 (|g| <= 4096, reached only by rows
// of modulus > 2000) so that no region can overflow; at 2^28 the region of an element holds 2^35 of summed g^2, i.e.
// 2^11 clamped pushes or 2^33 pushes with |g| <= 2, per step, at a resolution of 3.7e-9.
constexpr float kFxVal = 1099511627776.f;     // 2^40
constexpr float kFxAda = 268435456.f;         // 2^28
constexpr float kFxAdaMax = 16777216.f;       // 2^24

// 8-byte row accesses of the phase half (relation rows), coherent with concurrent REDs like dev::ld_row4 / red_row4
__device__ __forceinline__ float2 ld_row2(const float* p) {
  float2 v;
  asm volatile("ld.relaxed.sys.global.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_row2(float* p, float2 v) {
  asm volatile("red.relaxed.sys.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v.x), "f"(v.y) : "memory");
}
__device__ __forceinline__ float2 ld2(const float* p, int j) { return *reinterpret_cast<const float2*>(p + 2 * j); }
__device__ __forceinline__ void st2(float* p, int j, float2 v) { *reinterpret_cast<float2*>(p + 2 * j) = v; }

// a o rho for the two complex values of a float4; cs = (cos_0, sin_0, cos_1, sin_1)
__device__ __forceinline__ float4 rot(float4 a, float4 cs) {
  return make_float4(a.x * cs.x - a.y * cs.y, a.x * cs.y + a.y * cs.x, a.z * cs.z - a.w * cs.w, a.z * cs.w + a.w * cs.z);
}
// conj(rho) o u
__device__ __forceinline__ float4 rot_conj(float4 u, float4 cs) {
  return make_float4(u.x * cs.x + u.y * cs.y, u.y * cs.x - u.x * cs.y, u.z * cs.z + u.w * cs.w, u.w * cs.z - u.z * cs.w);
}
// |x_0| + |x_1| of a float4's two complex values; u = x / |x| per value (0 where |x| = 0)
__device__ __forceinline__ float cabs2(float4 x, float4& u) {
  const float r0 = sqrtf(x.x * x.x + x.y * x.y), r1 = sqrtf(x.z * x.z + x.w * x.w);
  const float i0 = r0 > 0.f ? 1.f / r0 : 0.f, i1 = r1 > 0.f ? 1.f / r1 : 0.f;
  u = make_float4(x.x * i0, x.y * i0, x.z * i1, x.w * i1);
  return r0 + r1;
}
// dD/dtheta of the two values for x = p - b, p = a o rho: -Im(conj(u) p) = u_im p_re - u_re p_im
__device__ __forceinline__ float2 dtheta(float4 u, float4 p) {
  return make_float2(u.y * p.x - u.x * p.y, u.w * p.z - u.z * p.w);
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// AdaGrad push of the phase gradient g onto phases 2j, 2j + 1 of a relation row [theta (m) | acc (m)] (the three modes
// of push4)
template <bool FX>
__device__ __forceinline__ void push2(float* row, int m, int j, float2 g, bool staged, long long* region, float eta) {
  const float2 a = ld_row2(row + m + 2 * j);
  const float2 ua = make_float2(g.x * g.x, g.y * g.y);
  const float2 ue = make_float2(g.x != 0.f ? -eta * g.x * rsqrtf(a.x + ua.x) : 0.f,
                                g.y != 0.f ? -eta * g.y * rsqrtf(a.y + ua.y) : 0.f);
  if (FX) {
    fx::add1(region, 2 * j, m, ue.x, kFxVal);
    fx::add1(region, 2 * j + 1, m, ue.y, kFxVal);
    fx::add1(region + m, 2 * j, m, fminf(ua.x, kFxAdaMax), kFxAda);
    fx::add1(region + m, 2 * j + 1, m, fminf(ua.y, kFxAdaMax), kFxAda);
  } else if (staged) {
    st2(row, j, ue);
    st2(row + m, j, ua);
  } else {
    red_row2(row + 2 * j, ue);
    red_row2(row + m + 2 * j, ua);
  }
}

struct Args {
  const Key* subj;
  const Key* rel;
  const Key* obj;
  const Key* neg;              // [B, n_neg]
  int B, n_neg, d;
  float margin, alpha, eta, gamma_e;
  float* scratch;              // generic path: 4 rows of 2 d per warp
  long long* fx_acc;           // FX: fixed-point regions, per-triple loss slots
  const int* fx_cidx;
  float* call_loss;
};

// The step as a warp_step rule (kge_step.cuh): positive (s, r, o). Per-warp shared memory: s o rho | o | (cos, sin) |
// g_s | g_o (d each) | g_theta (m) | distance / dL/dD of every negative (n_neg) | the negatives' targets.
template <int VPL>
struct RotatE {
  static constexpr int kPositives = 3, kMaxDim = kRotatEMaxDim, kMaxNeg = kRotatEMaxNeg, kBlocksPerSM = 4;
  static constexpr bool kInPlace = true, kStageInSmem = false;
  static __device__ __forceinline__ Key positive(const Args& A, int t, int i) {
    return i == 0 ? A.subj[t] : (i == 1 ? A.rel[t] : A.obj[t]);
  }
  static __host__ __device__ __forceinline__ size_t state_bytes(int d, int n_neg) {
    return (size_t)((5 * d + d / 2 + n_neg + 3) & ~3) * sizeof(float);
  }
  static __host__ __device__ __forceinline__ size_t warp_bytes(int d, int n_neg) {
    return (state_bytes(d, n_neg) + (size_t)n_neg * sizeof(dev::Target) + 15) & ~(size_t)15;
  }
  static __host__ __device__ __forceinline__ int scratch_rows(int) { return kPositives + 1; }
  static __device__ __forceinline__ int stage_row(int, int i) { return i; }
  static __device__ __forceinline__ bool neg_pushed(const StepOut&, int) { return true; }
  template <bool FX, bool GEN>
  static __device__ StepOut body(const Ctx& c, const Args& A, int t, const Rows<3>& rows, bool slow,
                                 const dev::Target* ntg, float* wsm, float* my_scratch);
};

// One positive triple and its negatives: ps / pr / po the positive's rows.
template <int VPL>
template <bool FX, bool GEN>
__device__ __forceinline__ StepOut RotatE<VPL>::body(const Ctx& c, const Args& A, int t, const Rows<3>& rows, bool slow,
                                                     const dev::Target* ntg, float* wsm, float* my_scratch) {
  const int lane = threadIdx.x & 31;
  const int d = A.d, m = d >> 1, nv = d >> 2, L = 2 * d, n_neg = A.n_neg, half = n_neg >> 1;
  float* const ps = rows.p[0];
  float* const pr = rows.p[1];
  float* const po = rows.p[2];
  StepOut out = {0.f, 0u, 0u, 0ull};
  float* const sa = wsm; float* const so = wsm + d; float* const scs = wsm + 2 * d;
  float* const sgs = wsm + 3 * d; float* const sgo = wsm + 4 * d; float* const sgt = wsm + 5 * d;
  float* const swq = sgt + m;
  float4 e[VPL];
  float dp = 0.f;
  load_row<VPL>(ps, nv, lane, e);
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int j = lane + 32 * i;
    if (j < nv) {
      const float2 th = ld_row2(pr + 2 * j);
      float4 cs;
      sincosf(th.x, &cs.y, &cs.x);
      sincosf(th.y, &cs.w, &cs.z);
      const float4 a = rot(e[i], cs), o = dev::ld_row4(po + 4 * j);
      st4(sa, j, a); st4(so, j, o); st4(scs, j, cs);
      st4(sgs, j, f4(0.f)); st4(sgo, j, f4(0.f)); st2(sgt, j, make_float2(0.f, 0.f));
      float4 u;
      dp += cabs2(sub4(a, o), u);
    }
  }
  const float Dp = dev::warp_sum(dp);

  for (int side = 0; side < 2; ++side) {
    const int q0 = side * half, q1 = q0 + half;
    // ---- pass 1: the side's distances
    for (int q = q0; q < q1; ++q) {
      float* pn = ntg[q].row;
      if (GEN && !pn) {
        ++out.slow;
        pn = my_scratch + 3 * L;
        if (!dev::slow_pull(c, A.neg[(size_t)t * n_neg + q], pn)) {
          if (lane == 0) swq[q] = __int_as_float(0x7fc00000);   // NaN: no weight, no push
          continue;
        }
      }
      load_row<VPL>(pn, nv, lane, e);
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        const int j = lane + 32 * i;
        if (j < nv) {
          float4 u;
          s += cabs2(side == 0 ? sub4(ld4(sa, j), e[i]) : sub4(rot(e[i], ld4(scs, j)), ld4(so, j)), u);
        }
      }
      const float Dn = dev::warp_sum(s);
      if (lane == 0) swq[q] = Dn;
    }
    __syncwarp();
    // ---- the side's weights: swq[q] becomes dL/dD_q = -1/2 w_q sigma(gamma - D_q) (NaN stays NaN)
    float zmax = -INFINITY;
    for (int q = q0 + lane; q < q1; q += 32) {
      const float D = swq[q];
      if (D == D) zmax = fmaxf(zmax, A.alpha * (A.margin - D));
    }
    zmax = warp_max(zmax);
    float zsum = 0.f;
    for (int q = q0 + lane; q < q1; q += 32) {
      const float D = swq[q];
      if (D == D) zsum += expf(A.alpha * (A.margin - D) - zmax);
    }
    zsum = dev::warp_sum(zsum);
    float lsum = 0.f;
    for (int q = q0 + lane; q < q1; q += 32) {
      const float D = swq[q];
      if (D == D) {
        const float w = expf(A.alpha * (A.margin - D) - zmax) / zsum;
        lsum += w * softplus(A.margin - D);
        swq[q] = -0.5f * w * sigmoid(A.margin - D);
      }
    }
    out.loss += 0.5f * dev::warp_sum(lsum);
    __syncwarp();
    // ---- pass 2: the gradients, one push per negative
    for (int q = q0; q < q1; ++q) {
      const float cq = swq[q];
      if (cq != cq) continue;
      const Key kn = A.neg[(size_t)t * n_neg + q];
      float* pn = ntg[q].row;
      const bool nslow = !pn;
      if (GEN && nslow) {
        pn = my_scratch + 3 * L;
        if (!dev::slow_pull(c, kn, pn)) continue;
      }
      load_row<VPL>(pn, nv, lane, e);
      long long* rg = FX ? fx::region(A.fx_acc, A.fx_cidx, kn, d) : nullptr;
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        const int j = lane + 32 * i;
        if (j < nv) {
          const float4 cs = ld4(scs, j);
          float4 u, g;
          float2 dt;
          if (side == 0) {            // x = s o rho - o'
            const float4 a = ld4(sa, j);
            cabs2(sub4(a, e[i]), u);
            st4(sgs, j, add4(ld4(sgs, j), mul4(rot_conj(u, cs), cq)));
            dt = dtheta(u, a);
            g = mul4(u, -cq);
          } else {                    // x = s' o rho - o
            const float4 p = rot(e[i], cs);
            cabs2(sub4(p, ld4(so, j)), u);
            st4(sgo, j, sub4(ld4(sgo, j), mul4(u, cq)));
            dt = dtheta(u, p);
            g = mul4(rot_conj(u, cs), cq);
          }
          const float2 gt = ld2(sgt, j);
          st2(sgt, j, make_float2(gt.x + cq * dt.x, gt.y + cq * dt.y));
          push4<FX>(pn, d, j, g, GEN && nslow, rg, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
        }
      }
      if (GEN && nslow && !FX) {
        if (dev::slow_push(c, kn, pn)) ++out.upd;
      } else {
        ++out.upd;
      }
    }
  }

  // ---- the positive's rows: summed gradients, L2 on the raw entity rows, one push each
  const float cp = sigmoid(Dp - A.margin);
  out.loss += softplus(Dp - A.margin);
  long long *fs = nullptr, *fr = nullptr, *fo = nullptr;
  if (FX) {
    fs = fx::region(A.fx_acc, A.fx_cidx, A.subj[t], d); fr = fx::region(A.fx_acc, A.fx_cidx, A.rel[t], d);
    fo = fx::region(A.fx_acc, A.fx_cidx, A.obj[t], d);
  }
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int j = lane + 32 * i;
    if (j < nv) {
      const float4 a = ld4(sa, j), cs = ld4(scs, j);
      float4 u;
      cabs2(sub4(a, ld4(so, j)), u);
      const float4 s_raw = dev::ld_row4(ps + 4 * j);
      push4<FX>(ps, d, j, add4(add4(ld4(sgs, j), mul4(rot_conj(u, cs), cp)), mul4(s_raw, A.gamma_e)), slow, fs, nv,
                A.eta, kFxVal, kFxAda, kFxAdaMax);
      const float2 dt = dtheta(u, a), gt = ld2(sgt, j);
      push2<FX>(pr, m, j, make_float2(gt.x + cp * dt.x, gt.y + cp * dt.y), slow, fr, A.eta);
      const float4 o_raw = dev::ld_row4(po + 4 * j);
      push4<FX>(po, d, j, add4(sub4(ld4(sgo, j), mul4(u, cp)), mul4(o_raw, A.gamma_e)), slow, fo, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
    }
  }
  __syncwarp();
  return out;
}

template <int VPL, bool FX>
__global__ void __launch_bounds__(kStepThreads, 1)
rotate_step_kernel(const __grid_constant__ Ctx c, const __grid_constant__ Args A, float* __restrict__ loss_out,
                   unsigned long long* __restrict__ stats) {
  warp_step<RotatE<VPL>, FX>(c, A, loss_out, stats);
}

template <bool FX>
void launch_shape(int vpl, CudaBackend& be, cudaStream_t stream, const Args& A, float* loss_out,
                  unsigned long long* stats) {
  switch (vpl) {
    case 1: launch_step<RotatE<1>, rotate_step_kernel<1, FX>>(be, stream, A, loss_out, stats); break;
    case 2: launch_step<RotatE<2>, rotate_step_kernel<2, FX>>(be, stream, A, loss_out, stats); break;
    case 3: launch_step<RotatE<3>, rotate_step_kernel<3, FX>>(be, stream, A, loss_out, stats); break;
    default: launch_step<RotatE<4>, rotate_step_kernel<4, FX>>(be, stream, A, loss_out, stats); break;
  }
}

}  // namespace

void kge_rotate_step(CudaBackend& be, cudaStream_t stream, const Key* subj, const Key* rel, const Key* obj,
                     const Key* neg, int B, int n_neg, int d, float margin, float alpha, float eta, float gamma_e,
                     float* loss_out, unsigned long long* stats, bool deterministic) {
  if (B == 0) return;
  ADAPM_CHECK(d % 8 == 0 && d >= 8 && d <= kRotatEMaxDim, "kge_rotate_step: embedding size must be a multiple of 8 in [8, "
                                                              << kRotatEMaxDim << "]");
  ADAPM_CHECK(n_neg >= 2 && n_neg % 2 == 0 && n_neg <= kRotatEMaxNeg,
              "kge_rotate_step: the negatives per triple must be an even count in [2, " << kRotatEMaxNeg << "]");
  const int vpl = (d / 4 + 31) / 32;
  Args A;
  A.subj = subj; A.rel = rel; A.obj = obj; A.neg = neg; A.B = B; A.n_neg = n_neg; A.d = d;
  A.margin = margin; A.alpha = alpha; A.eta = eta; A.gamma_e = gamma_e;
  // deterministic: entity keys get a [d | d] region (2 units), relation keys a [m | m] region (1 unit)
  const fx::Source src[4] = {{subj, B, 2}, {rel, B, 1}, {obj, B, 2}, {neg, (long)B * n_neg, 2}};
  run_step(be, stream, A, deterministic, src, 4, d, kFxVal, kFxAda, loss_out, [&](auto fx, float* lo) {
    launch_shape<decltype(fx)::value>(vpl, be, stream, A, lo, stats);
  });
}

}  // namespace cudaops
}  // namespace adapm

// Fused knowledge-graph-embedding training steps (ComplEx, RESCAL) for sm_90a: Pull(s, r, o) + score +
// BCE gradient + L2 + AdaGrad + Push(s, r, o) in one kernel over local HBM / NVLink peers
// (SURVEY K1 + K8 + K9 + K2 + K14).
//
// Semantics = the reference's Model::train with the ComplEx score
// (apps/knowledge_graph_embeddings.cc:437-531, :832-858, :415-435):
//   score = sum_i  r_re s_re o_re + r_re s_im o_im + r_im s_re o_im - r_im s_im o_re
//   dl    = sigmoid(score) - [positive]
//   d_x   = dl * dscore/dx  (+ gamma * x for positives)
//   push(x, [-eta * d_x / sqrt(acc_x + d_x^2) | d_x^2])        for x in {s, r, o}
// Row layout [embedding(nh) | AdaGrad(nh)], embedding = [real(nh/2) | imag(nh/2)].
// Both steps are warp_step rules without negatives (kge_step.cuh): one warp per training call; the three directory
// lookups are issued by three lanes at once.
//
// Deterministic one-GPU variants (kge_step_fx_kernel, kge_rescal_fx_kernel): every call reads the state at the start of
// the step and adds its updates as fixed-point integers into per-key accumulator regions (fx_accum.cuh), which one
// apply pass adds to the rows; each call's loss goes to its own slot and is summed in a fixed order.
#include <cuda_runtime.h>

#include "fx_accum.cuh"
#include "kge_step.cuh"
#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {

namespace {

using namespace kge;

// Dropout on the pulled copies (reference kge.cc:405-413,478-484: Bernoulli(p) zero, others scaled by 1/(1-p); score,
// gradients and L2 all see the masked copy; the AdaGrad half of a row is untouched). The mask is a pure function of
// (seed, training call, which row of the call, element index) so that the PyTorch reference of the tests can
// reproduce it (ops.kge_dropout_mask mirrors mask_keep bit by bit).
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}
struct Dropout {
  uint32_t seed;
  float p, scale;   // scale = 1 / (1 - p)
  __device__ __forceinline__ float keep(uint32_t call, uint32_t which, uint32_t elem) const {
    const uint32_t u = mix32(mix32(seed + call * 3u + which) ^ (elem * 0x9E3779B9u));
    return ((float)(u >> 8) * (1.0f / 16777216.0f)) >= p ? scale : 0.f;
  }
  __device__ __forceinline__ float4 apply4(float4 v, uint32_t call, uint32_t which, uint32_t elem0) const {
    if (p <= 0.f) return v;
    return make_float4(v.x * keep(call, which, elem0), v.y * keep(call, which, elem0 + 1),
                       v.z * keep(call, which, elem0 + 2), v.w * keep(call, which, elem0 + 3));
  }
};

// Fixed-point scales of the deterministic mode. |value update| <= eta per call (AdaGrad normalises it): 2^40 leaves
// 2^23 / eta calls per element and step. AdaGrad increments are g^2 with g = dl * (sum of products of two embedding
// values) + gamma * x and |dl| < 1: 2^36 leaves 2^27 of summed g^2 per element and step (resolution 1.5e-11). The
// increments are not clamped (kFxAdaMax = +inf).
constexpr float kFxVal = 1099511627776.f;     // 2^40
constexpr float kFxAda = 68719476736.f;       // 2^36
constexpr float kFxAdaMax = INFINITY;
// the largest nh whose three staged rows per warp fit 200 KB of shared memory per CTA
constexpr int kComplexMaxDim = 200 * 1024 / (kStepThreads / 32 * 6 * (int)sizeof(float));
constexpr int kRescalMaxDim = 128;

struct Args {
  const Key* subj;
  const Key* rel;
  const Key* obj;
  const float* labels;
  int B, n_neg, d;             // n_neg = 0; d: nh (ComplEx) or D (RESCAL)
  float eta, gamma_e, gamma_r;
  Dropout de, dr;
  float* scratch;              // RESCAL's generic path: a relation row and two entity rows per warp
  long long* fx_acc;           // FX: fixed-point regions, per-call loss slots
  const int* fx_cidx;
  float* call_loss;
};

// What ComplEx and RESCAL share as warp_step rules: positive (s, r, o), no negatives.
struct TripleRule {
  static constexpr int kPositives = 3, kMaxNeg = 0;
  static __device__ __forceinline__ Key positive(const Args& A, int t, int i) {
    return i == 0 ? A.subj[t] : (i == 1 ? A.rel[t] : A.obj[t]);
  }
};

// g = dl * d + gamma * x
__device__ __forceinline__ float4 grad4(float4 d, float4 x, float dl, float gamma) {
  return make_float4(fmaf(gamma, x.x, dl * d.x), fmaf(gamma, x.y, dl * d.y), fmaf(gamma, x.z, dl * d.z),
                     fmaf(gamma, x.w, dl * d.w));
}
// BCE loss of a call with score sc
__device__ __forceinline__ float bce_loss(float sc, bool pos) {
  const float z = pos ? sc : -sc;
  return __logf(1.f + __expf(-fminf(fmaxf(z, -30.f), 30.f)));
}

// ComplEx. VPLH = float4 vectors per lane per half-embedding (nh/8 float4 per half); VPLH = 0: no float4 body (nh % 8
// != 0 or nh > 512), every call takes the generic path. The generic path stages the three rows in the warp's
// shared memory (6 nh floats per warp, the rule's whole state). The kernels run 2 blocks of 256 threads per SM at 128
// registers, which use the whole register file.
template <int VPLH>
struct ComplEx : TripleRule {
  static constexpr int kMaxDim = kComplexMaxDim, kBlocksPerSM = 8;
  static constexpr bool kInPlace = VPLH > 0, kStageInSmem = true;
  static __host__ __device__ __forceinline__ size_t state_bytes(int nh, int) { return (size_t)6 * nh * sizeof(float); }
  static __host__ __device__ __forceinline__ size_t warp_bytes(int nh, int n_neg) { return state_bytes(nh, n_neg); }
  static __host__ __device__ __forceinline__ int scratch_rows(int) { return 0; }
  static __device__ __forceinline__ int stage_row(int, int i) { return i; }
  template <bool FX, bool GEN>
  static __device__ StepOut body(const Ctx& c, const Args& A, int t, const Rows<3>& rows, bool slow,
                                 const dev::Target* ntg, float* wsm, float* stage);
};

// One call. The generic path (GEN: the three rows are staged in shared memory) runs the scalar body at every VPLH.
template <int VPLH>
template <bool FX, bool GEN>
__device__ __forceinline__ StepOut ComplEx<VPLH>::body(const Ctx&, const Args& A, int t, const Rows<3>& rows, bool,
                                                       const dev::Target*, float*, float*) {
  constexpr int V = VPLH > 0 ? VPLH : 1;
  const int lane = threadIdx.x & 31;
  const int nh = A.d, H = nh >> 1, nvh = H >> 2;
  const uint32_t call = (uint32_t)t;
  float* const ps = rows.p[0];
  float* const pr = rows.p[1];
  float* const po = rows.p[2];
  float4 sre[V], sim[V], rre[V], rim[V], ore[V], oim[V];
  float sc = 0.f;
  if constexpr (VPLH == 0 || GEN) {   // scalar, any nh: dropout on the staged rows themselves
    if (A.de.p > 0.f || A.dr.p > 0.f) {
      for (int i = lane; i < nh; i += 32) {
        if (A.de.p > 0.f) { ps[i] *= A.de.keep(call, 0, (uint32_t)i); po[i] *= A.de.keep(call, 2, (uint32_t)i); }
        if (A.dr.p > 0.f) pr[i] *= A.dr.keep(call, 1, (uint32_t)i);
      }
      __syncwarp();
    }
    for (int i = lane; i < H; i += 32)
      sc += pr[i] * ps[i] * po[i] + pr[i] * ps[H + i] * po[H + i] + pr[H + i] * ps[i] * po[H + i] -
            pr[H + i] * ps[H + i] * po[i];
  } else {
#pragma unroll
    for (int v = 0; v < VPLH; ++v) {
      const int j = lane + 32 * v;
      const bool in = j < nvh;
      sre[v] = in ? dev::ld_row4(ps + 4 * j) : f4(0.f); sim[v] = in ? dev::ld_row4(ps + H + 4 * j) : f4(0.f);
      rre[v] = in ? dev::ld_row4(pr + 4 * j) : f4(0.f); rim[v] = in ? dev::ld_row4(pr + H + 4 * j) : f4(0.f);
      ore[v] = in ? dev::ld_row4(po + 4 * j) : f4(0.f); oim[v] = in ? dev::ld_row4(po + H + 4 * j) : f4(0.f);
      if (in && (A.de.p > 0.f || A.dr.p > 0.f)) {   // dropout on the pulled copies (uniform branch: kernel arguments)
        const uint32_t e = 4u * (uint32_t)j;
        sre[v] = A.de.apply4(sre[v], call, 0, e); sim[v] = A.de.apply4(sim[v], call, 0, (uint32_t)H + e);
        rre[v] = A.dr.apply4(rre[v], call, 1, e); rim[v] = A.dr.apply4(rim[v], call, 1, (uint32_t)H + e);
        ore[v] = A.de.apply4(ore[v], call, 2, e); oim[v] = A.de.apply4(oim[v], call, 2, (uint32_t)H + e);
      }
    }
#pragma unroll
    for (int v = 0; v < VPLH; ++v) {
      const float4 a = fma4(sre[v], ore[v], mul4(sim[v], oim[v]));       // s_re o_re + s_im o_im
      const float4 b = sub4(mul4(sre[v], oim[v]), mul4(sim[v], ore[v]));  // s_re o_im - s_im o_re
      const float4 u = fma4(rre[v], a, mul4(rim[v], b));
      sc += u.x + u.y + u.z + u.w;
    }
  }
  sc = dev::warp_sum(sc);
  const float label = A.labels[t];
  const float dl = 1.f / (1.f + __expf(-sc)) - label;
  const bool pos = label > 0.5f;
  const float ge = pos ? A.gamma_e : 0.f, gr = pos ? A.gamma_r : 0.f;
  long long *fs = nullptr, *fr = nullptr, *fo = nullptr;
  if (FX) {
    fs = fx::region(A.fx_acc, A.fx_cidx, A.subj[t], 2 * nh); fr = fx::region(A.fx_acc, A.fx_cidx, A.rel[t], 2 * nh);
    fo = fx::region(A.fx_acc, A.fx_cidx, A.obj[t], 2 * nh);
  }
  if constexpr (VPLH == 0 || GEN) {
    for (int i = lane; i < H; i += 32) {
      float sre = ps[i], sim = ps[H + i], rre = pr[i], rim = pr[H + i], ore = po[i], oim = po[H + i];
      float d[6] = {rre * ore + rim * oim, rre * oim - rim * ore, sre * ore + sim * oim,
                    sre * oim - sim * ore, rre * sre - rim * sim, rre * sim + rim * sre};
      float x[6] = {sre, sim, rre, rim, ore, oim};
      float gm[6] = {ge, ge, gr, gr, ge, ge};
      float* rw[6] = {ps, ps, pr, pr, po, po};
      long long* rg[6] = {fs, fs, fr, fr, fo, fo};
      int off[6] = {i, H + i, i, H + i, i, H + i};
#pragma unroll
      for (int q = 0; q < 6; ++q) {
        float g = dl * d[q] + gm[q] * x[q];
        float a = rw[q][nh + off[q]];
        float ua = g * g;
        const float ue = -A.eta * g * rsqrtf(a + ua);
        if (FX) {
          fx::add1(rg[q], off[q], nh, ue, kFxVal);
          fx::add1(rg[q] + nh, off[q], nh, ua, kFxAda);
        } else {
          rw[q][off[q]] = ue;
          rw[q][nh + off[q]] = ua;
        }
      }
    }
  } else {
    const int nv = nh >> 2;
#pragma unroll
    for (int v = 0; v < VPLH; ++v) {
      const int j = lane + 32 * v;
      if (j < nvh) {
        // gradients of the trilinear score (reference score_grad)
        const float4 ds_re = fma4(rre[v], ore[v], mul4(rim[v], oim[v]));
        const float4 ds_im = sub4(mul4(rre[v], oim[v]), mul4(rim[v], ore[v]));
        const float4 dr_re = fma4(sre[v], ore[v], mul4(sim[v], oim[v]));
        const float4 dr_im = sub4(mul4(sre[v], oim[v]), mul4(sim[v], ore[v]));
        const float4 do_re = sub4(mul4(rre[v], sre[v]), mul4(rim[v], sim[v]));
        const float4 do_im = fma4(rre[v], sim[v], mul4(rim[v], sre[v]));
        // float4 j of the real half, float4 nvh + j of the imaginary half
        push4<FX>(ps, nh, j, grad4(ds_re, sre[v], dl, ge), false, fs, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
        push4<FX>(ps, nh, nvh + j, grad4(ds_im, sim[v], dl, ge), false, fs, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
        push4<FX>(pr, nh, j, grad4(dr_re, rre[v], dl, gr), false, fr, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
        push4<FX>(pr, nh, nvh + j, grad4(dr_im, rim[v], dl, gr), false, fr, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
        push4<FX>(po, nh, j, grad4(do_re, ore[v], dl, ge), false, fo, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
        push4<FX>(po, nh, nvh + j, grad4(do_im, oim[v], dl, ge), false, fo, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
      }
    }
  }
  return {bce_loss(sc, pos), 0u, 0u, 0ull};
}

template <int VPLH>
__global__ void __maxnreg__(128)
kge_step_kernel(const __grid_constant__ Ctx c, const __grid_constant__ Args A, float* __restrict__ loss_out,
                unsigned long long* __restrict__ stats) {
  warp_step<ComplEx<VPLH>, false>(c, A, loss_out, stats);
}

template <int VPLH>
__global__ void __maxnreg__(128)
kge_step_fx_kernel(const __grid_constant__ Ctx c, const __grid_constant__ Args A, float* __restrict__ loss_out,
                   unsigned long long* __restrict__ stats) {
  warp_step<ComplEx<VPLH>, true>(c, A, loss_out, stats);
}

template <bool FX, int VPLH>
void launch_complex(CudaBackend& be, cudaStream_t stream, const Args& A, float* loss_out, unsigned long long* stats) {
  if constexpr (FX) launch_step<ComplEx<VPLH>, kge_step_fx_kernel<VPLH>>(be, stream, A, loss_out, stats);
  else launch_step<ComplEx<VPLH>, kge_step_kernel<VPLH>>(be, stream, A, loss_out, stats);
}

// ---------------------------------------------------------------------------------------------------------------
// RESCAL (reference kge.cc:895-922): score = s^T R o with a D x D relation matrix (relation row = [R | AdaGrad] of
// 2 D^2 floats), gradients d_s = R o, d_o = R^T s, d_R = s o^T (rank 1). One warp per training call:
//   pass 1  stream R once (16-byte loads, local HBM or NVLink): per float4 a row-dot into ds[i] and four axpy terms
//           into do[j..j+3] (shared-memory accumulators of the warp) -> score = s . ds
//   entity rows: AdaGrad + scalar reductions for s and o
//   pass 2  stream R's values + accumulators again (L2 hits), form dl * s_i * o_j (+ gamma R_ij), AdaGrad, 16-byte
//           reductions into both halves of the relation row
// The generic path stages the relation row and the two entity rows of a call in global scratch.
//
// Deterministic mode (FX, kge_rescal_fx_kernel): pass 1 forms ds and do in a fixed order instead of with shared-memory
// atomics - the G = D/4 float4 of a matrix row are read by G consecutive lanes, 32/G rows per round; ds[i] is the sum of
// its G partial dots (shuffle tree for G a power of two, else lane-ordered), each lane keeps its four do partial sums in
// registers over its rows, and do[j] sums those in row-group order. Updates go to fixed-point accumulator regions
// (relation region [D^2 | D^2], entity regions [D | D]) and each call's loss to its own slot.
constexpr int kRescalFxSmem = 32 + 128;   // extra floats per warp: ds partials [32] | do partials [32/G][D]

// Per-warp shared memory: s[D] | o[D] | ds[D] | do[D] (| FX partials); DET: the kernel's mode.
template <bool DET>
struct Rescal : TripleRule {
  static constexpr int kMaxDim = kRescalMaxDim, kBlocksPerSM = 4;
  static constexpr bool kInPlace = true, kStageInSmem = false;
  static __host__ __device__ __forceinline__ size_t state_bytes(int D, int) {
    return (size_t)(DET ? 4 * D + kRescalFxSmem : 4 * D) * sizeof(float);
  }
  static __host__ __device__ __forceinline__ size_t warp_bytes(int D, int n_neg) { return state_bytes(D, n_neg); }
  // relation row (D rows of 2 D) | s row | o row
  static __host__ __device__ __forceinline__ int scratch_rows(int D) { return D + 2; }
  static __device__ __forceinline__ int stage_row(int D, int i) { return i == 1 ? 0 : D + i / 2; }
  template <bool FX, bool GEN>
  static __device__ StepOut body(const Ctx& c, const Args& A, int t, const Rows<3>& rows, bool slow,
                                 const dev::Target* ntg, float* wsm, float* stage);
};

template <bool DET>
template <bool FX, bool GEN>
__device__ __forceinline__ StepOut Rescal<DET>::body(const Ctx&, const Args& A, int t, const Rows<3>& rows, bool slow,
                                                     const dev::Target*, float* wsm, float*) {
  static_assert(FX == DET, "the shared-memory layout follows the mode");
  const int lane = threadIdx.x & 31;
  const int D = A.d, DD = D * D;
  const int nv = DD >> 2;          // float4 of the relation matrix
  float* const ps = rows.p[0];
  float* const pr = rows.p[1];
  float* const po = rows.p[2];
  float* const sv = wsm; float* const ov = sv + D; float* const dsv = ov + D; float* const dov = dsv + D;
  const float label = A.labels[t];
  const uint32_t cp = (uint32_t)t;
  for (int i = lane; i < D; i += 32) {
    float a = reinterpret_cast<const volatile float*>(ps)[i];
    float b = reinterpret_cast<const volatile float*>(po)[i];
    if (A.de.p > 0.f) { a *= A.de.keep(cp, 0, (uint32_t)i); b *= A.de.keep(cp, 2, (uint32_t)i); }
    sv[i] = a; ov[i] = b; dsv[i] = 0.f; dov[i] = 0.f;
  }
  __syncwarp();
  // ---- pass 1: ds = R o, do = R^T s
  if (FX) {
    const int G = D >> 2, rpr = 32 / G;           // float4 per matrix row, rows per round
    const int rg = lane / G, j = 4 * (lane - rg * G);
    const bool pow2 = (G & (G - 1)) == 0;
    float* dsp = dov + D;                         // [32] partial dots
    float* dop = dsp + 32;                        // [rpr][D] partial do sums
    float4 dacc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i0 = 0; i0 < D; i0 += rpr) {
      const int i = i0 + rg;
      float part = 0.f;
      if (rg < rpr && i < D) {
        const int e = i * D + j;
        float4 r4 = dev::ld_row4(pr + e);
        if (A.dr.p > 0.f) r4 = A.dr.apply4(r4, cp, 1, (uint32_t)e);
        part = r4.x * ov[j] + r4.y * ov[j + 1] + r4.z * ov[j + 2] + r4.w * ov[j + 3];
        const float si = sv[i];
        dacc.x += si * r4.x; dacc.y += si * r4.y; dacc.z += si * r4.z; dacc.w += si * r4.w;
      }
      if (pow2) {                                 // G | 32: fixed shuffle tree inside each group of G lanes
        for (int o = G >> 1; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
        if (lane - rg * G == 0 && i < D) dsv[i] = part;
      } else {
        dsp[lane] = part;
        __syncwarp();
        if (lane < rpr && i0 + lane < D) {
          float acc = 0.f;
          for (int q = 0; q < G; ++q) acc += dsp[lane * G + q];
          dsv[i0 + lane] = acc;
        }
        __syncwarp();
      }
    }
    if (rg < rpr) {
      float* d4 = dop + rg * D + j;
      d4[0] = dacc.x; d4[1] = dacc.y; d4[2] = dacc.z; d4[3] = dacc.w;
    }
    __syncwarp();
    for (int jj = lane; jj < D; jj += 32) {
      float acc = 0.f;
      for (int r = 0; r < rpr; ++r) acc += dop[r * D + jj];
      dov[jj] = acc;
    }
  } else {
    for (int q = lane; q < nv; q += 32) {
      const int e = 4 * q, i = e / D, j = e - i * D;
      float4 r4 = dev::ld_row4(pr + e);
      if (A.dr.p > 0.f) r4 = A.dr.apply4(r4, cp, 1, (uint32_t)e);
      const float si = sv[i];
      atomicAdd(dsv + i, r4.x * ov[j] + r4.y * ov[j + 1] + r4.z * ov[j + 2] + r4.w * ov[j + 3]);
      atomicAdd(dov + j, si * r4.x); atomicAdd(dov + j + 1, si * r4.y);
      atomicAdd(dov + j + 2, si * r4.z); atomicAdd(dov + j + 3, si * r4.w);
    }
  }
  __syncwarp();
  float sc = 0.f;
  for (int i = lane; i < D; i += 32) sc += sv[i] * dsv[i];
  sc = dev::warp_sum(sc);
  const float dl = 1.f / (1.f + __expf(-sc)) - label;
  const bool pos = label > 0.5f;
  const float ge = pos ? A.gamma_e : 0.f, grr = pos ? A.gamma_r : 0.f;
  long long *fs = nullptr, *fr = nullptr, *fo = nullptr;
  if (FX) {   // regions in units of an entity row (2 D): relation regions are D units
    fs = fx::region(A.fx_acc, A.fx_cidx, A.subj[t], 2 * D); fr = fx::region(A.fx_acc, A.fx_cidx, A.rel[t], 2 * D);
    fo = fx::region(A.fx_acc, A.fx_cidx, A.obj[t], 2 * D);
  }
  // ---- entity rows
  for (int i = lane; i < D; i += 32) {
    const float g_s = fmaf(ge, sv[i], dl * dsv[i]), g_o = fmaf(ge, ov[i], dl * dov[i]);
    const float a_s = reinterpret_cast<const volatile float*>(ps)[D + i], a_o = reinterpret_cast<const volatile float*>(po)[D + i];
    const float us = -A.eta * g_s * rsqrtf(a_s + g_s * g_s), uo = -A.eta * g_o * rsqrtf(a_o + g_o * g_o);
    if (FX) {
      fx::add1(fs, i, D, us, kFxVal); fx::add1(fs + D, i, D, g_s * g_s, kFxAda);
      fx::add1(fo, i, D, uo, kFxVal); fx::add1(fo + D, i, D, g_o * g_o, kFxAda);
    } else if (slow) { ps[i] = us; ps[D + i] = g_s * g_s; po[i] = uo; po[D + i] = g_o * g_o; }
    else { mem::red_add(ps + i, us); mem::red_add(ps + D + i, g_s * g_s); mem::red_add(po + i, uo); mem::red_add(po + D + i, g_o * g_o); }
  }
  // ---- pass 2: relation matrix update (rank-1 gradient)
  for (int q = lane; q < nv; q += 32) {
    const int e = 4 * q, i = e / D, j = e - i * D;
    float4 r4 = dev::ld_row4(pr + e);
    if (A.dr.p > 0.f) r4 = A.dr.apply4(r4, cp, 1, (uint32_t)e);
    const float4 a4 = dev::ld_row4(pr + DD + e);
    const float4 g = grad4(make_float4(ov[j], ov[j + 1], ov[j + 2], ov[j + 3]), r4, dl * sv[i], grr);
    push4<FX>(pr, DD, q, g, a4, slow, fr, nv, A.eta, kFxVal, kFxAda, kFxAdaMax);
  }
  return {bce_loss(sc, pos), 0u, 0u, 0ull};
}

__global__ void __launch_bounds__(kStepThreads)
kge_rescal_kernel(const __grid_constant__ Ctx c, const __grid_constant__ Args A, float* __restrict__ loss_out,
                  unsigned long long* __restrict__ stats) {
  warp_step<Rescal<false>, false>(c, A, loss_out, stats);
}

__global__ void __launch_bounds__(kStepThreads)
kge_rescal_fx_kernel(const __grid_constant__ Ctx c, const __grid_constant__ Args A, float* __restrict__ loss_out,
                     unsigned long long* __restrict__ stats) {
  warp_step<Rescal<true>, true>(c, A, loss_out, stats);
}

}  // namespace

// n_calls training calls (s[i], r[i], o[i], label[i]); entity and relation rows must be 2*nh floats.
static Dropout make_dropout(float p, uint64_t seed, uint32_t salt) {
  Dropout d;
  d.p = p > 0.f ? p : 0.f;
  ADAPM_CHECK(d.p < 1.f, "dropout probability must be < 1");
  d.scale = 1.f / (1.f - d.p);
  d.seed = (uint32_t)(seed ^ (seed >> 32)) * 2654435761u + salt;
  return d;
}

void kge_complex_step(CudaBackend& be, cudaStream_t stream, const Key* subj, const Key* rel, const Key* obj,
                      const float* labels, int n_calls, int nh, float eta, float gamma_e, float gamma_r, float* loss_out,
                      unsigned long long* stats, float dropout_e, float dropout_r, uint64_t seed, bool deterministic) {
  if (n_calls == 0) return;
  Args A;
  A.de = make_dropout(dropout_e, seed, 0x11u); A.dr = make_dropout(dropout_r, seed, 0x22u);
  ADAPM_CHECK(nh % 2 == 0, "ComplEx needs an even embedding size");
  ADAPM_CHECK(kStepThreads / 32 * ComplEx<0>::warp_bytes(nh, 0) <= 200 * 1024,
              "kge_complex_step: embedding size too large for the staging buffer");
  int vplh = (nh % 8 == 0) ? (nh / 8 + 31) / 32 : 0;
  if (vplh > 2) vplh = 0;
  A.subj = subj; A.rel = rel; A.obj = obj; A.labels = labels; A.B = n_calls; A.n_neg = 0; A.d = nh;
  A.eta = eta; A.gamma_e = gamma_e; A.gamma_r = gamma_r;
  // deterministic: every key gets a [nh | nh] accumulator region (entity and relation rows alike)
  const fx::Source src[3] = {{subj, n_calls, 1}, {rel, n_calls, 1}, {obj, n_calls, 1}};
  run_step(be, stream, A, deterministic, src, 3, 2 * nh, kFxVal, kFxAda, loss_out, [&](auto fx, float* lo) {
    constexpr bool FX = decltype(fx)::value;
    switch (vplh) {
      case 1: launch_complex<FX, 1>(be, stream, A, lo, stats); break;
      case 2: launch_complex<FX, 2>(be, stream, A, lo, stats); break;
      default: launch_complex<FX, 0>(be, stream, A, lo, stats); break;
    }
  });
}

// RESCAL training calls: entity rows 2*D floats, relation rows 2*D*D floats (D % 4 == 0, D <= 128).
void kge_rescal_step(CudaBackend& be, cudaStream_t stream, const Key* subj, const Key* rel, const Key* obj,
                     const float* labels, int n_calls, int D, float eta, float gamma_e, float gamma_r, float* loss_out,
                     unsigned long long* stats, float dropout_e, float dropout_r, uint64_t seed, bool deterministic) {
  if (n_calls == 0) return;
  ADAPM_CHECK(D % 4 == 0 && D >= 4 && D <= kRescalMaxDim,
              "kge_rescal_step: embedding size must be a multiple of 4 in [4, 128]");
  Args A;
  A.de = make_dropout(dropout_e, seed, 0x11u); A.dr = make_dropout(dropout_r, seed, 0x22u);
  A.subj = subj; A.rel = rel; A.obj = obj; A.labels = labels; A.B = n_calls; A.n_neg = 0; A.d = D;
  A.eta = eta; A.gamma_e = gamma_e; A.gamma_r = gamma_r;
  // deterministic: entity regions [D | D] (one unit), relation regions [D^2 | D^2] (D units)
  const fx::Source src[3] = {{subj, n_calls, 1}, {obj, n_calls, 1}, {rel, n_calls, D}};
  run_step(be, stream, A, deterministic, src, 3, 2 * D, kFxVal, kFxAda, loss_out, [&](auto fx, float* lo) {
    if constexpr (decltype(fx)::value) launch_step<Rescal<true>, kge_rescal_fx_kernel>(be, stream, A, lo, stats);
    else launch_step<Rescal<false>, kge_rescal_kernel>(be, stream, A, lo, stats);
  });
}

}  // namespace cudaops
}  // namespace adapm

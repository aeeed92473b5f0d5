// Fused knowledge-graph-embedding training step (ComplEx) for sm_90a: Pull(s, r, o) + score +
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
// One warp per training call; the three directory lookups are issued by three lanes at once.
//
// Deterministic one-GPU variants (kge_step_fx_kernel, kge_rescal_fx_kernel): every call reads the state at the start of
// the step and adds its updates as fixed-point integers into per-key accumulator regions (fx_accum.cuh), which one
// apply pass adds to the rows; each call's loss goes to its own slot and is summed in a fixed order.
#include <cuda_runtime.h>

#include <map>
#include <mutex>

#include "fx_accum.cuh"
#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float4 f4_mul(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float4 f4_fma(float4 a, float4 b, float4 c) {
  return make_float4(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y), fmaf(a.z, b.z, c.z), fmaf(a.w, b.w, c.w));
}
__device__ __forceinline__ float4 f4_sub(float4 a, float4 b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
__device__ __forceinline__ float f4_hsum(float4 a) { return a.x + a.y + a.z + a.w; }

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
// values) + gamma * x and |dl| < 1: 2^36 leaves 2^27 of summed g^2 per element and step (resolution 1.5e-11).
constexpr float kFxVal = 1099511627776.f;     // 2^40
constexpr float kFxAda = 68719476736.f;       // 2^36

// g = dl * d + (reg ? gamma * x : 0); returns AdaGrad update pair and issues the reductions.
__device__ __forceinline__ void adagrad_push4(float* emb_ptr, float* acc_ptr, float4 d, float4 x, float dl, float gamma,
                                              float eta) {
  float4 g = make_float4(fmaf(gamma, x.x, dl * d.x), fmaf(gamma, x.y, dl * d.y), fmaf(gamma, x.z, dl * d.z),
                         fmaf(gamma, x.w, dl * d.w));
  float4 a = dev::ld_row4(acc_ptr);
  float4 ua = f4_mul(g, g);
  float4 ue = make_float4(-eta * g.x * rsqrtf(a.x + ua.x), -eta * g.y * rsqrtf(a.y + ua.y),
                          -eta * g.z * rsqrtf(a.z + ua.z), -eta * g.w * rsqrtf(a.w + ua.w));
  dev::red_row4(emb_ptr, ue);
  dev::red_row4(acc_ptr, ua);
}
// deterministic mode: the same update, added to float4 jj of the key's accumulator region (halves of h values)
__device__ __forceinline__ void adagrad_fx4(const float* acc_ptr, long long* region, int jj, int h, float4 d, float4 x,
                                            float dl, float gamma, float eta) {
  float4 g = make_float4(fmaf(gamma, x.x, dl * d.x), fmaf(gamma, x.y, dl * d.y), fmaf(gamma, x.z, dl * d.z),
                         fmaf(gamma, x.w, dl * d.w));
  float4 a = dev::ld_row4(acc_ptr);
  float4 ua = f4_mul(g, g);
  float4 ue = make_float4(-eta * g.x * rsqrtf(a.x + ua.x), -eta * g.y * rsqrtf(a.y + ua.y),
                          -eta * g.z * rsqrtf(a.z + ua.z), -eta * g.w * rsqrtf(a.w + ua.w));
  fx::add4(region, jj, h >> 2, ue, kFxVal);
  fx::add4(region + h, jj, h >> 2, ua, kFxAda);
}
// deterministic mode: adds a staged row of updates [value update (h) | AdaGrad update (h)] to the key's region
__device__ __forceinline__ void fx_add_staged(long long* region, const float* stage, int h) {
  for (int i = threadIdx.x & 31; i < 2 * h; i += 32) {
    const int hf = i >= h;
    fx::add1(region + hf * h, i - hf * h, h, stage[i], hf ? kFxAda : kFxVal);
  }
}

// scalar generic path (any nh; also used when a row is in a transitional state): rows staged in smem
template <bool FX>
__device__ __noinline__ float kge_call_generic(const Ctx& c, Key ks, Key kr, Key ko, float label, int nh, float eta,
                                               float gamma_e, float gamma_r, float* stage, bool* applied, uint32_t call,
                                               Dropout de, Dropout dr, long long* fx_acc, const int* fx_cidx) {
  const int lane = threadIdx.x & 31;
  float* S = stage; float* R = stage + 2 * nh; float* O = stage + 4 * nh;
  *applied = false;
  if (!dev::slow_pull(c, ks, S) || !dev::slow_pull(c, kr, R) || !dev::slow_pull(c, ko, O)) return 0.f;
  if (de.p > 0.f || dr.p > 0.f) {
    for (int i = lane; i < nh; i += 32) {
      if (de.p > 0.f) { S[i] *= de.keep(call, 0, (uint32_t)i); O[i] *= de.keep(call, 2, (uint32_t)i); }
      if (dr.p > 0.f) R[i] *= dr.keep(call, 1, (uint32_t)i);
    }
    __syncwarp();
  }
  const int H = nh / 2;
  float sc = 0.f;
  for (int i = lane; i < H; i += 32)
    sc += R[i] * S[i] * O[i] + R[i] * S[H + i] * O[H + i] + R[H + i] * S[i] * O[H + i] - R[H + i] * S[H + i] * O[i];
  sc = dev::warp_sum(sc);
  const float dl = 1.f / (1.f + __expf(-sc)) - label;
  const float ge = label > 0.5f ? gamma_e : 0.f, gr = label > 0.5f ? gamma_r : 0.f;
  for (int i = lane; i < H; i += 32) {
    float sre = S[i], sim = S[H + i], rre = R[i], rim = R[H + i], ore = O[i], oim = O[H + i];
    float d[6] = {rre * ore + rim * oim, rre * oim - rim * ore, sre * ore + sim * oim,
                  sre * oim - sim * ore, rre * sre - rim * sim, rre * sim + rim * sre};
    float x[6] = {sre, sim, rre, rim, ore, oim};
    float gm[6] = {ge, ge, gr, gr, ge, ge};
    float* rows[6] = {S, S, R, R, O, O};
    int off[6] = {i, H + i, i, H + i, i, H + i};
#pragma unroll
    for (int q = 0; q < 6; ++q) {
      float g = dl * d[q] + gm[q] * x[q];
      float a = rows[q][nh + off[q]];
      float ua = g * g;
      rows[q][off[q]] = -eta * g * rsqrtf(a + ua);
      rows[q][nh + off[q]] = ua;
    }
  }
  __syncwarp();
  if (FX) {
    fx_add_staged(fx::region(fx_acc, fx_cidx, ks, 2 * nh), S, nh);
    fx_add_staged(fx::region(fx_acc, fx_cidx, kr, 2 * nh), R, nh);
    fx_add_staged(fx::region(fx_acc, fx_cidx, ko, 2 * nh), O, nh);
    *applied = true;
  } else {
    bool ok = dev::slow_push(c, ks, S);
    ok = dev::slow_push(c, kr, R) && ok;
    ok = dev::slow_push(c, ko, O) && ok;
    *applied = ok;
  }
  float z = label > 0.5f ? sc : -sc;
  return __logf(1.f + __expf(-fminf(fmaxf(z, -30.f), 30.f)));
}

// VPLH = float4 vectors per lane per half-embedding (nh/8 float4 per half); VPLH = 0 -> generic only
// The kernels run 2 blocks of 256 threads per SM at 128 registers, which use the whole register file.
// FX: deterministic mode (kge_step_fx_kernel): start-of-step reads, fixed-point sums into fx_acc, call losses.
template <int VPLH, bool FX>
__device__ __forceinline__ void
kge_step_body(const Ctx& c, const Key* __restrict__ subj, const Key* __restrict__ rel, const Key* __restrict__ obj,
              const float* __restrict__ labels, int n_calls, int nh, float eta, float gamma_e, float gamma_r,
              float* __restrict__ loss_out, unsigned long long* __restrict__ stats, Dropout de, Dropout dr,
              long long* __restrict__ fx_acc, const int* __restrict__ fx_cidx, float* __restrict__ call_loss) {
  extern __shared__ float smem_f[];  // generic path: per warp 6*nh floats
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int warp_in_block = threadIdx.x >> 5;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  float* stage = smem_f + (size_t)warp_in_block * 6 * nh;
  const int H = nh >> 1;
  const int nvh = H >> 2;
  float loss_acc = 0.f;
  unsigned n_local = 0, n_remote = 0, n_slow = 0, n_upd = 0;

  for (int p = warp; p < n_calls; p += nwarps) {
    const Key ks = subj[p], kr = rel[p], ko = obj[p];
    const float label = labels[p];
    dev::Target t;
    t.row = nullptr; t.version = nullptr; t.flag = nullptr;
    if (VPLH > 0 && lane < 3) {
      Key k = lane == 0 ? ks : (lane == 1 ? kr : ko);
      t = dev::resolve_fast(c, k, class_of_key(c, k), &n_local, &n_remote);
    }
    float* ps = (float*)__shfl_sync(0xffffffffu, (unsigned long long)t.row, 0);
    float* pr = (float*)__shfl_sync(0xffffffffu, (unsigned long long)t.row, 1);
    float* po = (float*)__shfl_sync(0xffffffffu, (unsigned long long)t.row, 2);
    if (VPLH == 0 || !ps || !pr || !po) {
      ++n_slow;
      bool applied;
      const float l = kge_call_generic<FX>(c, ks, kr, ko, label, nh, eta, gamma_e, gamma_r, stage, &applied,
                                           (uint32_t)p, de, dr, fx_acc, fx_cidx);
      if (FX) { if (lane == 0) call_loss[p] = l; }
      else loss_acc += l;
      if (applied) n_upd += 3;
      continue;
    }
    constexpr int V = VPLH > 0 ? VPLH : 1;
    float4 sre[V], sim[V], rre[V], rim[V], ore[V], oim[V];
    float sc = 0.f;
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const int j = lane + 32 * v;
      const bool in = j < nvh;
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      sre[v] = in ? dev::ld_row4(ps + 4 * j) : z; sim[v] = in ? dev::ld_row4(ps + H + 4 * j) : z;
      rre[v] = in ? dev::ld_row4(pr + 4 * j) : z; rim[v] = in ? dev::ld_row4(pr + H + 4 * j) : z;
      ore[v] = in ? dev::ld_row4(po + 4 * j) : z; oim[v] = in ? dev::ld_row4(po + H + 4 * j) : z;
      if (in && (de.p > 0.f || dr.p > 0.f)) {   // dropout on the pulled copies (uniform branch: kernel arguments)
        const uint32_t e = 4u * (uint32_t)j, cp = (uint32_t)p;
        sre[v] = de.apply4(sre[v], cp, 0, e); sim[v] = de.apply4(sim[v], cp, 0, (uint32_t)H + e);
        rre[v] = dr.apply4(rre[v], cp, 1, e); rim[v] = dr.apply4(rim[v], cp, 1, (uint32_t)H + e);
        ore[v] = de.apply4(ore[v], cp, 2, e); oim[v] = de.apply4(oim[v], cp, 2, (uint32_t)H + e);
      }
    }
#pragma unroll
    for (int v = 0; v < V; ++v) {
      float4 a = f4_fma(sre[v], ore[v], f4_mul(sim[v], oim[v]));   // s_re o_re + s_im o_im
      float4 b = f4_sub(f4_mul(sre[v], oim[v]), f4_mul(sim[v], ore[v]));  // s_re o_im - s_im o_re
      sc += f4_hsum(f4_fma(rre[v], a, f4_mul(rim[v], b)));
    }
    sc = dev::warp_sum(sc);
    const float dl = 1.f / (1.f + __expf(-sc)) - label;
    const bool pos = label > 0.5f;
    const float ge = pos ? gamma_e : 0.f, gr = pos ? gamma_r : 0.f;
    {
      float z = pos ? sc : -sc;
      const float l = __logf(1.f + __expf(-fminf(fmaxf(z, -30.f), 30.f)));
      if (FX) { if (lane == 0) call_loss[p] = l; }
      else loss_acc += l;
    }
    long long *fs = nullptr, *fr = nullptr, *fo = nullptr;
    if (FX) {
      fs = fx::region(fx_acc, fx_cidx, ks, 2 * nh); fr = fx::region(fx_acc, fx_cidx, kr, 2 * nh);
      fo = fx::region(fx_acc, fx_cidx, ko, 2 * nh);
    }
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const int j = lane + 32 * v;
      if (FX && j < nvh) {
        float4 ds_re = f4_fma(rre[v], ore[v], f4_mul(rim[v], oim[v]));
        float4 ds_im = f4_sub(f4_mul(rre[v], oim[v]), f4_mul(rim[v], ore[v]));
        float4 dr_re = f4_fma(sre[v], ore[v], f4_mul(sim[v], oim[v]));
        float4 dr_im = f4_sub(f4_mul(sre[v], oim[v]), f4_mul(sim[v], ore[v]));
        float4 do_re = f4_sub(f4_mul(rre[v], sre[v]), f4_mul(rim[v], sim[v]));
        float4 do_im = f4_fma(rre[v], sim[v], f4_mul(rim[v], sre[v]));
        // float4 j of the real half, float4 nvh + j of the imaginary half
        adagrad_fx4(ps + nh + 4 * j, fs, j, nh, ds_re, sre[v], dl, ge, eta);
        adagrad_fx4(ps + nh + H + 4 * j, fs, nvh + j, nh, ds_im, sim[v], dl, ge, eta);
        adagrad_fx4(pr + nh + 4 * j, fr, j, nh, dr_re, rre[v], dl, gr, eta);
        adagrad_fx4(pr + nh + H + 4 * j, fr, nvh + j, nh, dr_im, rim[v], dl, gr, eta);
        adagrad_fx4(po + nh + 4 * j, fo, j, nh, do_re, ore[v], dl, ge, eta);
        adagrad_fx4(po + nh + H + 4 * j, fo, nvh + j, nh, do_im, oim[v], dl, ge, eta);
      } else if (j < nvh) {
        // gradients of the trilinear score (reference score_grad)
        float4 ds_re = f4_fma(rre[v], ore[v], f4_mul(rim[v], oim[v]));
        float4 ds_im = f4_sub(f4_mul(rre[v], oim[v]), f4_mul(rim[v], ore[v]));
        float4 dr_re = f4_fma(sre[v], ore[v], f4_mul(sim[v], oim[v]));
        float4 dr_im = f4_sub(f4_mul(sre[v], oim[v]), f4_mul(sim[v], ore[v]));
        float4 do_re = f4_sub(f4_mul(rre[v], sre[v]), f4_mul(rim[v], sim[v]));
        float4 do_im = f4_fma(rre[v], sim[v], f4_mul(rim[v], sre[v]));
        adagrad_push4(ps + 4 * j, ps + nh + 4 * j, ds_re, sre[v], dl, ge, eta);
        adagrad_push4(ps + H + 4 * j, ps + nh + H + 4 * j, ds_im, sim[v], dl, ge, eta);
        adagrad_push4(pr + 4 * j, pr + nh + 4 * j, dr_re, rre[v], dl, gr, eta);
        adagrad_push4(pr + H + 4 * j, pr + nh + H + 4 * j, dr_im, rim[v], dl, gr, eta);
        adagrad_push4(po + 4 * j, po + nh + 4 * j, do_re, ore[v], dl, ge, eta);
        adagrad_push4(po + H + 4 * j, po + nh + H + 4 * j, do_im, oim[v], dl, ge, eta);
      }
    }
    if (lane < 3) dev::mark_pushed(t);
    n_upd += 3;
  }

  __syncwarp();
  if (!FX && lane == 0 && loss_out) atomicAdd(loss_out, loss_acc);
  dev::flush_stats(stats, n_local, n_remote, n_slow, n_upd);
  dev::cta_exit(c);
}

template <int VPLH>
__global__ void __maxnreg__(128)
kge_step_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ subj, const Key* __restrict__ rel,
                const Key* __restrict__ obj, const float* __restrict__ labels, int n_calls, int nh, float eta,
                float gamma_e, float gamma_r, float* __restrict__ loss_out, unsigned long long* __restrict__ stats,
                Dropout de, Dropout dr) {
  kge_step_body<VPLH, false>(c, subj, rel, obj, labels, n_calls, nh, eta, gamma_e, gamma_r, loss_out, stats, de, dr,
                             nullptr, nullptr, nullptr);
}

template <int VPLH>
__global__ void __maxnreg__(128)
kge_step_fx_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ subj, const Key* __restrict__ rel,
                   const Key* __restrict__ obj, const float* __restrict__ labels, int n_calls, int nh, float eta,
                   float gamma_e, float gamma_r, unsigned long long* __restrict__ stats, Dropout de, Dropout dr,
                   long long* __restrict__ fx_acc, const int* __restrict__ fx_cidx, float* __restrict__ call_loss) {
  kge_step_body<VPLH, true>(c, subj, rel, obj, labels, n_calls, nh, eta, gamma_e, gamma_r, nullptr, stats, de, dr,
                            fx_acc, fx_cidx, call_loss);
}

// ---------------------------------------------------------------------------------------------------------------
// RESCAL (reference kge.cc:895-922): score = s^T R o with a D x D relation matrix (relation row = [R | AdaGrad] of
// 2 D^2 floats), gradients d_s = R o, d_o = R^T s, d_R = s o^T (rank 1). One warp per training call:
//   pass 1  stream R once (16-byte loads, local HBM or NVLink): per float4 a row-dot into ds[i] and four axpy terms
//           into do[j..j+3] (shared-memory accumulators of the warp) -> score = s . ds
//   entity rows: AdaGrad + 16-byte reductions for s and o
//   pass 2  stream R's values + accumulators again (L2 hits), form dl * s_i * o_j (+ gamma R_ij), AdaGrad, 16-byte
//           reductions into both halves of the relation row
// Rows in a transitional protocol state go through the generic Pull/Push path with a global scratch buffer.
__device__ __noinline__ bool rescal_slow_rows(const Ctx& c, Key ks, Key kr, Key ko, float* gs, float* gr, float* go) {
  return dev::slow_pull(c, ks, gs) && dev::slow_pull(c, kr, gr) && dev::slow_pull(c, ko, go);
}

// Deterministic mode (FX, kge_rescal_fx_kernel): pass 1 forms ds and do in a fixed order instead of with shared-memory
// atomics - the G = D/4 float4 of a matrix row are read by G consecutive lanes, 32/G rows per round; ds[i] is the sum of
// its G partial dots (shuffle tree for G a power of two, else lane-ordered), each lane keeps its four do partial sums in
// registers over its rows, and do[j] sums those in row-group order. Updates go to fixed-point accumulator regions
// (relation region [D^2 | D^2], entity regions [D | D]) and each call's loss to its own slot.
constexpr int kRescalFxSmem = 32 + 128;   // extra floats per warp: ds partials [32] | do partials [32/G][D]

template <bool FX>
__device__ __forceinline__ void
kge_rescal_body(const Ctx& c, const Key* __restrict__ subj, const Key* __restrict__ rel, const Key* __restrict__ obj,
                const float* __restrict__ labels, int n_calls, int D, float eta, float gamma_e, float gamma_r,
                float* __restrict__ loss_out, unsigned long long* __restrict__ stats, Dropout de, Dropout dr,
                float* __restrict__ scratch, long long* __restrict__ fx_acc, const int* __restrict__ fx_cidx,
                float* __restrict__ call_loss) {
  extern __shared__ float smem_f[];   // per warp: s[D] | o[D] | ds[D] | do[D] (| FX partials)
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  float* sv = smem_f + (size_t)wib * (FX ? 4 * D + kRescalFxSmem : 4 * D);
  float* ov = sv + D; float* dsv = ov + D; float* dov = dsv + D;
  const int DD = D * D;
  const int nv = DD >> 2;          // float4 of the relation matrix
  float* my_scratch = scratch + (size_t)warp * (size_t)(2 * DD + 4 * D);   // generic path: rel row | s row | o row
  float loss_acc = 0.f;
  unsigned n_local = 0, n_remote = 0, n_slow = 0, n_upd = 0;

  for (int p = warp; p < n_calls; p += nwarps) {
    const Key ks = subj[p], kr = rel[p], ko = obj[p];
    const float label = labels[p];
    dev::Target t;
    t.row = nullptr; t.version = nullptr; t.flag = nullptr;
    if (lane < 3) {
      Key k = lane == 0 ? ks : (lane == 1 ? kr : ko);
      t = dev::resolve_fast(c, k, class_of_key(c, k), &n_local, &n_remote);
    }
    float* ps = (float*)__shfl_sync(0xffffffffu, (unsigned long long)t.row, 0);
    float* pr = (float*)__shfl_sync(0xffffffffu, (unsigned long long)t.row, 1);
    float* po = (float*)__shfl_sync(0xffffffffu, (unsigned long long)t.row, 2);
    const bool slow = !ps || !pr || !po;
    if (slow) {   // stage the three rows in global scratch and run the same math on the copies
      ++n_slow;
      float* gr_ = my_scratch; float* gs_ = my_scratch + 2 * DD; float* go_ = gs_ + 2 * D;
      if (!rescal_slow_rows(c, ks, kr, ko, gs_, gr_, go_)) {
        if (FX && lane == 0) call_loss[p] = 0.f;
        continue;
      }
      ps = gs_; pr = gr_; po = go_;
    }
    const uint32_t cp = (uint32_t)p;
    for (int i = lane; i < D; i += 32) {
      float a = reinterpret_cast<const volatile float*>(ps)[i];
      float b = reinterpret_cast<const volatile float*>(po)[i];
      if (de.p > 0.f) { a *= de.keep(cp, 0, (uint32_t)i); b *= de.keep(cp, 2, (uint32_t)i); }
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
          if (dr.p > 0.f) r4 = dr.apply4(r4, cp, 1, (uint32_t)e);
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
            float t = 0.f;
            for (int q = 0; q < G; ++q) t += dsp[lane * G + q];
            dsv[i0 + lane] = t;
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
        float t = 0.f;
        for (int r = 0; r < rpr; ++r) t += dop[r * D + jj];
        dov[jj] = t;
      }
    } else {
      for (int q = lane; q < nv; q += 32) {
        const int e = 4 * q, i = e / D, j = e - i * D;
        float4 r4 = dev::ld_row4(pr + e);
        if (dr.p > 0.f) r4 = dr.apply4(r4, cp, 1, (uint32_t)e);
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
    const float ge = pos ? gamma_e : 0.f, grr = pos ? gamma_r : 0.f;
    {
      float z = pos ? sc : -sc;
      const float l = __logf(1.f + __expf(-fminf(fmaxf(z, -30.f), 30.f)));
      if (FX) { if (lane == 0) call_loss[p] = l; }
      else loss_acc += l;
    }
    long long *fs = nullptr, *fr = nullptr, *fo = nullptr;
    if (FX) {   // regions in units of an entity row (2 D): relation regions are D units
      fs = fx::region(fx_acc, fx_cidx, ks, 2 * D); fr = fx::region(fx_acc, fx_cidx, kr, 2 * D);
      fo = fx::region(fx_acc, fx_cidx, ko, 2 * D);
    }
    // ---- entity rows
    for (int i = lane; i < D; i += 32) {
      const float g_s = fmaf(ge, sv[i], dl * dsv[i]), g_o = fmaf(ge, ov[i], dl * dov[i]);
      const float a_s = reinterpret_cast<const volatile float*>(ps)[D + i], a_o = reinterpret_cast<const volatile float*>(po)[D + i];
      const float us = -eta * g_s * rsqrtf(a_s + g_s * g_s), uo = -eta * g_o * rsqrtf(a_o + g_o * g_o);
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
      if (dr.p > 0.f) r4 = dr.apply4(r4, cp, 1, (uint32_t)e);
      const float4 a4 = dev::ld_row4(pr + DD + e);
      const float w = dl * sv[i];
      const float4 g = make_float4(fmaf(grr, r4.x, w * ov[j]), fmaf(grr, r4.y, w * ov[j + 1]), fmaf(grr, r4.z, w * ov[j + 2]),
                                   fmaf(grr, r4.w, w * ov[j + 3]));
      const float4 ua = f4_mul(g, g);
      const float4 ue = make_float4(-eta * g.x * rsqrtf(a4.x + ua.x), -eta * g.y * rsqrtf(a4.y + ua.y),
                                    -eta * g.z * rsqrtf(a4.z + ua.z), -eta * g.w * rsqrtf(a4.w + ua.w));
      if (FX) { fx::add4(fr, q, nv, ue, kFxVal); fx::add4(fr + DD, q, nv, ua, kFxAda); }
      else if (slow) { *reinterpret_cast<float4*>(pr + e) = ue; *reinterpret_cast<float4*>(pr + DD + e) = ua; }
      else { dev::red_row4(pr + e, ue); dev::red_row4(pr + DD + e, ua); }
    }
    if (FX) {
      if (lane < 3 && !slow) dev::mark_pushed(t);
      n_upd += 3;
    } else if (slow) {
      __syncwarp();
      bool ok = dev::slow_push(c, ks, ps);
      ok = dev::slow_push(c, kr, pr) && ok;
      ok = dev::slow_push(c, ko, po) && ok;
      if (ok) n_upd += 3;
    } else {
      if (lane < 3) dev::mark_pushed(t);
      n_upd += 3;
    }
    __syncwarp();
  }

  __syncwarp();
  if (!FX && lane == 0 && loss_out) atomicAdd(loss_out, loss_acc);
  dev::flush_stats(stats, n_local, n_remote, n_slow, n_upd);
  dev::cta_exit(c);
}

__global__ void __launch_bounds__(kThreads)
kge_rescal_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ subj, const Key* __restrict__ rel,
                  const Key* __restrict__ obj, const float* __restrict__ labels, int n_calls, int D, float eta,
                  float gamma_e, float gamma_r, float* __restrict__ loss_out, unsigned long long* __restrict__ stats,
                  Dropout de, Dropout dr, float* __restrict__ scratch) {
  kge_rescal_body<false>(c, subj, rel, obj, labels, n_calls, D, eta, gamma_e, gamma_r, loss_out, stats, de, dr, scratch,
                         nullptr, nullptr, nullptr);
}

__global__ void __launch_bounds__(kThreads)
kge_rescal_fx_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ subj, const Key* __restrict__ rel,
                     const Key* __restrict__ obj, const float* __restrict__ labels, int n_calls, int D, float eta,
                     float gamma_e, float gamma_r, unsigned long long* __restrict__ stats, Dropout de, Dropout dr,
                     float* __restrict__ scratch, long long* __restrict__ fx_acc, const int* __restrict__ fx_cidx,
                     float* __restrict__ call_loss) {
  kge_rescal_body<true>(c, subj, rel, obj, labels, n_calls, D, eta, gamma_e, gamma_r, nullptr, stats, de, dr, scratch,
                        fx_acc, fx_cidx, call_loss);
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
  const Dropout de = make_dropout(dropout_e, seed, 0x11u), dr = make_dropout(dropout_r, seed, 0x22u);
  ADAPM_CHECK(nh % 2 == 0, "ComplEx needs an even embedding size");
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  be.track_stream(stream);
  const Ctx& c = be.ctx();
  const int warps_per_block = kThreads / 32;
  int blocks = std::min((n_calls + warps_per_block - 1) / warps_per_block, be.num_sms() * 8);
  size_t smem = (size_t)warps_per_block * 6 * nh * sizeof(float);
  ADAPM_CHECK(smem <= 200 * 1024, "kge_complex_step: embedding size too large for the staging buffer");
  const int nvh = nh / 8;
  int vplh = (nh % 8 == 0) ? (nvh + 31) / 32 : 0;
  if (vplh > 2) vplh = 0;
#define ADAPM_LAUNCH_KGE(V)                                                                                    \
  do {                                                                                                         \
    set_max_dynamic_smem<kge_step_kernel<V>>(200 * 1024);                                                      \
    kge_step_kernel<V><<<blocks, kThreads, smem, stream>>>(c, subj, rel, obj, labels, n_calls, nh, eta,        \
                                                           gamma_e, gamma_r, loss_out, stats, de, dr);         \
  } while (0)
#define ADAPM_LAUNCH_KGE_FX(V)                                                                                 \
  do {                                                                                                         \
    set_max_dynamic_smem<kge_step_fx_kernel<V>>(200 * 1024);                                                   \
    kge_step_fx_kernel<V><<<blocks, kThreads, smem, stream>>>(c, subj, rel, obj, labels, n_calls, nh, eta,     \
                                                              gamma_e, gamma_r, stats, de, dr, fxs->acc,       \
                                                              fxs->cidx, fxs->call_loss);                      \
  } while (0)
  if (deterministic) {
    // one GPU, start-of-step reads: every key gets a [nh | nh] accumulator region (entity and relation rows alike)
    const fx::Source src[3] = {{subj, n_calls, 1}, {rel, n_calls, 1}, {obj, n_calls, 1}};
    CudaBackend::FxScratch* fxs = &fx::begin(be, stream, src, 3, 2 * nh, n_calls);
    switch (vplh) {
      case 1: ADAPM_LAUNCH_KGE_FX(1); break;
      case 2: ADAPM_LAUNCH_KGE_FX(2); break;
      default: ADAPM_LAUNCH_KGE_FX(0); break;
    }
    ADAPM_COUNT_LAUNCH();
    ADAPM_CUDA_CHECK(cudaGetLastError());
    fx::apply(be, stream, 2 * nh, kFxVal, kFxAda, 0.f, n_calls, loss_out);
    return;
  }
  switch (vplh) {
    case 1: ADAPM_LAUNCH_KGE(1); break;
    case 2: ADAPM_LAUNCH_KGE(2); break;
    default: ADAPM_LAUNCH_KGE(0); break;
  }
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

// RESCAL training calls: entity rows 2*D floats, relation rows 2*D*D floats (D % 4 == 0, D <= 128).
void kge_rescal_step(CudaBackend& be, cudaStream_t stream, const Key* subj, const Key* rel, const Key* obj,
                     const float* labels, int n_calls, int D, float eta, float gamma_e, float gamma_r, float* loss_out,
                     unsigned long long* stats, float dropout_e, float dropout_r, uint64_t seed, bool deterministic) {
  if (n_calls == 0) return;
  ADAPM_CHECK(D % 4 == 0 && D >= 4 && D <= 128, "kge_rescal_step: embedding size must be a multiple of 4 in [4, 128]");
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  be.track_stream(stream);
  const Ctx& c = be.ctx();
  const Dropout de = make_dropout(dropout_e, seed, 0x11u), dr = make_dropout(dropout_r, seed, 0x22u);
  const int warps_per_block = kThreads / 32;
  const int blocks = std::min((n_calls + warps_per_block - 1) / warps_per_block, be.num_sms() * 4);
  const size_t smem = (size_t)warps_per_block * (deterministic ? 4 * D + kRescalFxSmem : 4 * D) * sizeof(float);
  // generic-path scratch (rows in a transitional protocol state): one relation row + two entity rows per warp
  static std::mutex mu;
  static std::map<int, std::pair<float*, size_t>> scratch_by_dev;
  float* scratch = nullptr;
  {
    std::lock_guard<std::mutex> lk(mu);
    const size_t need = (size_t)blocks * warps_per_block * (size_t)(2 * D * D + 4 * D) * sizeof(float);
    auto& e = scratch_by_dev[be.device()];
    if (e.second < need) {
      if (e.first) cudaFree(e.first);
      ADAPM_CUDA_CHECK(cudaMalloc((void**)&e.first, need));
      e.second = need;
    }
    scratch = e.first;
  }
  if (deterministic) {
    // one GPU, start-of-step reads: entity regions [D | D] (one unit), relation regions [D^2 | D^2] (D units)
    const fx::Source src[3] = {{subj, n_calls, 1}, {obj, n_calls, 1}, {rel, n_calls, D}};
    CudaBackend::FxScratch& fxs = fx::begin(be, stream, src, 3, 2 * D, n_calls);
    kge_rescal_fx_kernel<<<blocks, kThreads, smem, stream>>>(c, subj, rel, obj, labels, n_calls, D, eta, gamma_e,
                                                             gamma_r, stats, de, dr, scratch, fxs.acc, fxs.cidx,
                                                             fxs.call_loss);
    ADAPM_COUNT_LAUNCH();
    ADAPM_CUDA_CHECK(cudaGetLastError());
    fx::apply(be, stream, 2 * D, kFxVal, kFxAda, 0.f, n_calls, loss_out);
    return;
  }
  kge_rescal_kernel<<<blocks, kThreads, smem, stream>>>(c, subj, rel, obj, labels, n_calls, D, eta, gamma_e, gamma_r,
                                                        loss_out, stats, de, dr, scratch);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

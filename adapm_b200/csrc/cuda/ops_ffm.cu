// Field-aware factorisation machines (FFM, as in libffm) on the parameter store for sm_90a. A key's row is
// [w, 0, 0, 0 | V_0 | V_1 | ... | V_{F-1} | AdaGrad of all E values], E = 4 + F k, V_f the key's k-vector for field f.
// One step takes ids [B, F] (the field of ids[b, f] is f) and labels [B].
//
// Forward (one launch, one CTA per example): the example's F rows, resolved through the directory, are staged in
// shared memory, and
//   phi_b = sum_f w[x_bf] + r sum_{f1<f2} <V[x_bf1][f2], V[x_bf2][f1]>,  kappa_b = sigmoid(phi_b) - y_b,
//   loss_b = softplus(phi_b) - y_b phi_b,
// each sum in fp32 in a fixed order. In a step the forward also writes every occurrence's gradient contribution
//   c_(b,f) = [kappa_b + lam w[x_bf], 0, 0, 0 | for f2 != f: kappa_b r V[x_b,f2][f] + lam V[x_bf][f2]; 0 for f2 == f]
// to the workspace. Every read of another key's row (the partner blocks V[x_b,f2][f]) happens here, before any push
// of the step: the later launches read only the workspace and each key's own accumulator.
// Backward (three launches, the radix sort counted as one): the sort, tile and finish passes of grouped_push.cuh, which
// the embedding-bag backward shares, over FfmSource: each key's contributions are added in fp32 in position order.
// Every distinct key gets one push [-eta G / sqrt(acc + G^2) | G^2] (0 where G == 0: the key's own-field block and the
// padding) with one fixed sum, so on one GPU two runs of the same step give bit-identical rows and loss. A last
// one-CTA launch adds the per-example losses in index order.
#include <cuda_runtime.h>

#include "grouped_push.cuh"
#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {

namespace {

using namespace grouped;

constexpr int kFwdThreads = 128;

// ------------------------------------------------------------------------------------------------ forward
// One CTA per example (grid-stride). srow[f * E4 + j]: float4 j of the values of the row of ids[b, f]. Thread f < F
// resolves key f; a key in a transitional state is read three ways by that thread alone (rare). `contrib` null: the
// forward of evaluation, which writes logits only. In a step, the forward also writes the positions b * F + f that
// the radix sort takes as its values.
__global__ void __launch_bounds__(kFwdThreads)
ffm_fwd_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ ids, const float* __restrict__ labels, int B,
               int F, int k, float r, float lam, float* __restrict__ logits, float* __restrict__ loss_ex,
               float* __restrict__ contrib, int* __restrict__ pos, unsigned long long* __restrict__ stats) {
  extern __shared__ float4 srow[];
  __shared__ const float* rowp[kFfmMaxFields];
  __shared__ float red[kFwdThreads / 32];
  __shared__ float s_kappa;
  dev::cta_enter(c);
  const int tid = threadIdx.x, lane = tid & 31;
  const int k4 = k >> 2, E4 = 1 + F * k4, n4 = F * E4;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  Counts n;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    if (tid < F) {
      const Key key = ids[(size_t)b * F + tid];
      const float* p = resolve(c, key, n).row;
      if (!p) {                          // transitional slot (relocation in flight)
        dev::GatherRow gr = locate_row(c, key);
        count_rare(stats, gr.row != nullptr);
        if (gr.row && gr.local) ++n.local; else if (gr.row) ++n.remote;
        do {
          for (int j = 0; j < E4; ++j) srow[tid * E4 + j] = gr.row ? dev::ld_gather4(gr, 4 * j) : zero;
        } while (reread_row(c, key, gr));
      }
      rowp[tid] = p;
      if (pos) pos[b * F + tid] = b * F + tid;
    }
    __syncthreads();
    for (int i = tid; i < n4; i += kFwdThreads) {
      const int f = i / E4;
      const float* p = rowp[f];
      if (p) srow[i] = dev::ld_row4(p + 4 * (i - f * E4));
    }
    __syncthreads();
    // pairs (f1 < f2): thread t takes the flat indices q = f1 * F + f2 = t, t + 128, ...; the warps' sums are added
    // in a fixed tree and order
    float s = 0.f;
    for (int q = tid; q < F * F; q += kFwdThreads) {
      const int f1 = q / F, f2 = q - f1 * F;
      if (f1 >= f2) continue;
      const float4* x = srow + f1 * E4 + 1 + f2 * k4;
      const float4* y = srow + f2 * E4 + 1 + f1 * k4;
      for (int i = 0; i < k4; ++i) {
        const float4 u = x[i], v = y[i];
        s = fmaf(u.x, v.x, s); s = fmaf(u.y, v.y, s); s = fmaf(u.z, v.z, s); s = fmaf(u.w, v.w, s);
      }
    }
    s = dev::warp_sum(s);
    if (lane == 0) red[tid >> 5] = s;
    __syncthreads();
    if (tid == 0) {
      float w = 0.f;
      for (int f = 0; f < F; ++f) w += srow[f * E4].x;
      float pair = 0.f;
#pragma unroll
      for (int i = 0; i < kFwdThreads / 32; ++i) pair += red[i];
      const float phi = fmaf(r, pair, w);
      if (logits) logits[b] = phi;
      if (contrib) {
        const float y = labels[b];
        const float e = __expf(-fabsf(phi));
        loss_ex[b] = fmaxf(phi, 0.f) + log1pf(e) - y * phi;       // softplus(phi) - y phi
        s_kappa = (phi >= 0.f ? 1.f : e) / (1.f + e) - y;          // sigmoid(phi) - y
      }
    }
    __syncthreads();
    if (contrib) {
      const float kappa = s_kappa, kr = kappa * r;
      float4* out = reinterpret_cast<float4*>(contrib) + (size_t)b * n4;
      for (int i = tid; i < n4; i += kFwdThreads) {
        const int f = i / E4, j = i - f * E4;
        const float4 v = srow[i];
        float4 o = zero;
        if (j == 0) {
          o.x = fmaf(lam, v.x, kappa);
        } else {
          const int f2 = (j - 1) / k4;
          if (f2 != f) {
            const float4 p = srow[f2 * E4 + 1 + f * k4 + (j - 1 - f2 * k4)];
            o.x = fmaf(kr, p.x, lam * v.x); o.y = fmaf(kr, p.y, lam * v.y);
            o.z = fmaf(kr, p.z, lam * v.z); o.w = fmaf(kr, p.w, lam * v.w);
          }
        }
        out[i] = o;
      }
    }
    __syncthreads();                     // the next example overwrites srow and rowp
  }
  flush_counts(n, stats);
  dev::cta_exit(c);
}

// ------------------------------------------------------------------------------------------------ backward
// the passes of grouped_push.cuh over FfmSource, which adds row b * F + f of the forward's contributions for the
// occurrence at position b * F + f, with a plain add, and nothing to a key's sum before the push
struct FfmSource {
  const float* contrib;
  struct Item { int pos; };
  __device__ __forceinline__ Item load(int pos) const { return {pos}; }
  __device__ __forceinline__ Item share(const Item& it, unsigned mask, int src, int G) const {
    return {__shfl_sync(mask, it.pos, src, G)};
  }
  __device__ __forceinline__ const float4* row(const Item& it, int E) const {
    return reinterpret_cast<const float4*>(contrib + (size_t)it.pos * E);
  }
  __device__ __forceinline__ void add(float4& a, const float4& x, const Item&) const {
    a.x += x.x; a.y += x.y; a.z += x.z; a.w += x.w;
  }
  template <int VPL>
  __device__ __forceinline__ void before_push(float4 (&)[VPL]) const {}
};

template <int VPL>
__global__ void __launch_bounds__(kThreads, 2)
ffm_grad_tile_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ sk, const int* __restrict__ spos,
                     const FfmSource src, int nnz, int E, int log_g, float eta,
                     float* __restrict__ part, unsigned long long* __restrict__ stats) {
  tile_pass<VPL>(c, sk, spos, src, nnz, E, log_g, eta, part, stats);
}

template <int VPL>
__global__ void __launch_bounds__(kThreads, 2)
ffm_grad_finish_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ sk, int nnz, int E, float eta,
                       const float* __restrict__ part, unsigned long long* __restrict__ stats,
                       const FfmSource src) {
  finish_pass<VPL>(c, sk, nnz, E, eta, part, stats, src);
}

// the step's loss: sum_b loss_ex[b] in a fixed order (one CTA; thread t adds b = t, t + 256, ..., then a fixed tree)
__global__ void __launch_bounds__(kThreads)
ffm_loss_sum_kernel(const float* __restrict__ loss_ex, int B, float* __restrict__ loss) {
  __shared__ float red[kThreads / 32];
  float s = 0.f;
  for (int b = threadIdx.x; b < B; b += kThreads) s += loss_ex[b];
  s = dev::warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < kThreads / 32; ++i) t += red[i];
    *loss = t;
  }
}

// ------------------------------------------------------------------------------------------------ host side
// workspace layout: the sort's and the passes' arrays (grouped::carve_push) | contributions | per-example losses
struct Workspace {
  PushWorkspace g; float* contrib; float* loss_ex; size_t total;
};

Workspace carve(void* base, int B, int F, int k) {
  const int64_t nnz = (int64_t)B * F;
  Carve a{static_cast<char*>(base)};
  Workspace w{};
  w.g = carve_push(a, nnz, 4 + F * k);
  w.contrib = a.take<float>((size_t)nnz * (4 + F * k));
  w.loss_ex = a.take<float>(B);
  w.total = a.off;
  return w;
}

void check_shape(const CudaBackend& be, int64_t B, int F, int k) {
  const Ctx& c = be.ctx();
  ADAPM_CHECK(c.L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  ADAPM_CHECK(F >= 2 && F <= kFfmMaxFields, "ffm: the number of fields must be in [2, " << kFfmMaxFields << "]");
  ADAPM_CHECK(k % 4 == 0 && k >= 4 && k <= kFfmMaxK, "ffm: k must be a multiple of 4 in [4, " << kFfmMaxK << "]");
  ADAPM_CHECK(F * k <= kFfmMaxFk, "ffm: fields * k must be <= " << kFfmMaxFk);
  ADAPM_CHECK(c.L.num_classes == 1 && !c.L.per_key_len && c.L.cls[0].len == (uint32_t)(2 * (4 + F * k)),
              "ffm: every row must be [w, 0, 0, 0 | V (fields * k) | AdaGrad] of 2 * (4 + fields * k) values");
  ADAPM_CHECK(B >= 0 && B * F < ((int64_t)1 << 31), "ffm: batch * fields must be < 2^31");
}

void launch_forward(CudaBackend& be, cudaStream_t stream, const Key* ids, const float* labels, int B, int F, int k,
                    float r, float lam, float* logits, float* loss_ex, float* contrib, int* pos,
                    unsigned long long* stats) {
  const int smem = F * (1 + F * k / 4) * (int)sizeof(float4);
  ADAPM_CUDA_CHECK(cudaFuncSetAttribute(ffm_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 0;
  ADAPM_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ffm_fwd_kernel, kFwdThreads, smem));
  const int blocks = std::max(1, std::min(B, be.num_sms() * std::max(per_sm, 1)));
  ffm_fwd_kernel<<<blocks, kFwdThreads, smem, stream>>>(be.ctx(), ids, labels, B, F, k, r, lam, logits, loss_ex,
                                                         contrib, pos, stats);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace

size_t ffm_workspace_bytes(int B, int F, int k) { return carve(nullptr, B, F, k).total; }

void ffm_forward(CudaBackend& be, cudaStream_t stream, const Key* ids, int B, int F, int k, float r, float* logits,
                 unsigned long long* stats) {
  check_shape(be, B, F, k);
  if (B == 0) return;
  be.track_stream(stream);
  launch_forward(be, stream, ids, nullptr, B, F, k, r, 0.f, logits, nullptr, nullptr, nullptr, stats);
}

void ffm_step(CudaBackend& be, cudaStream_t stream, const Key* ids, const float* labels, int B, int F, int k, float r,
              float eta, float lam, void* workspace, size_t workspace_bytes, float* loss, unsigned long long* stats) {
  check_shape(be, B, F, k);
  ADAPM_CHECK(eta >= 0.f && lam >= 0.f, "ffm: eta and lam must be >= 0");
  if (B == 0) {
    ADAPM_CUDA_CHECK(cudaMemsetAsync(loss, 0, sizeof(float), stream));
    return;
  }
  be.track_stream(stream);
  Workspace w = carve(workspace, B, F, k);
  ADAPM_CHECK(workspace && workspace_bytes >= w.total, "ffm: workspace too small");
  const int n = B * F, E = 4 + F * k;
  launch_forward(be, stream, ids, labels, B, F, k, r, lam, nullptr, w.loss_ex, w.contrib, w.g.pos_in, stats);
  int log_g, vpl;
  lane_shape(E, &log_g, &vpl);
  const FfmSource src{w.contrib};
  switch (vpl) {
#define ADAPM_FFM_BWD(V) \
  case V: sort_and_push<ffm_grad_tile_kernel<V>, ffm_grad_finish_kernel<V>>(be, stream, ids, w.g, src, n, E, log_g, eta, stats); break
    ADAPM_FFM_BWD(1); ADAPM_FFM_BWD(2); ADAPM_FFM_BWD(3); ADAPM_FFM_BWD(4); ADAPM_FFM_BWD(5);
#undef ADAPM_FFM_BWD
    default: ADAPM_CHECK(false, "ffm: bad row length " << E);
  }
  ffm_loss_sum_kernel<<<1, kThreads, 0, stream>>>(w.loss_ex, B, loss);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

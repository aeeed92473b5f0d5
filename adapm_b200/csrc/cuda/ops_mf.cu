// Fused matrix-factorisation SGD step for sm_90a: Pull(w_i, h_j) + error + L2 + AdaGrad + Push
// in one kernel over local HBM / NVLink peers (SURVEY K1 + K10 + K9 + K2).
//
// Update rule = the reference's UpdateNsqlL2Adagrad (apps/mf/update.h:32-70):
//   e = x - <w, h>;  g_w = -(-2 e h + 2 lambda w / nnz_row);  g_h = -(-2 e w + 2 lambda h / nnz_col)
//   push(w, [eps * g_w / sqrt(acc_w + g_w^2 + 1e-6) | g_w^2])   (same for h)
// Row layout [factors(rank) | AdaGrad(rank)] (apps/matrix_factorization.cc:697).
// One warp per non-zero; two lanes resolve the two keys at once.
//
// Deterministic one-GPU variant (mf_step_fx_kernel): every non-zero reads the state at the start of the step and adds
// its updates as fixed-point integers into per-key accumulator regions (fx_accum.cuh), which one apply pass adds to the
// rows; each non-zero's squared error goes to its own slot and is summed in a fixed order (float64).
#include <cuda_runtime.h>

#include "fx_accum.cuh"
#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {

namespace {

constexpr int kThreads = 256;
constexpr float kAdagradEps = 1e-6f;
// Fixed-point scales of the deterministic mode. |factor update| <= eps per non-zero (AdaGrad normalises it): 2^40
// leaves 2^23 / eps non-zeros per element and step. AdaGrad increments are g^2 with g = 2 e h - 2 lambda w / nnz, which
// grows with the error e and so with the data: 2^30 leaves 2^33 (8.6e9) of summed g^2 per element and step, at a
// resolution of 9.3e-10. The loss is summed in float64 from per-non-zero float squared errors.
constexpr float kFxVal = 1099511627776.f;     // 2^40
constexpr float kFxAda = 1073741824.f;        // 2^30

// deterministic mode: adds a staged row of updates [factor update (h) | AdaGrad update (h)] to the key's region
__device__ __forceinline__ void fx_add_staged(long long* region, const float* stage, int h) {
  for (int i = threadIdx.x & 31; i < 2 * h; i += 32) {
    const int hf = i >= h;
    fx::add1(region + hf * h, i - hf * h, h, stage[i], hf ? kFxAda : kFxVal);
  }
}

template <bool FX>
__device__ __noinline__ float mf_generic(const Ctx& c, Key kw, Key kh, float x, float inv_rn, float inv_cn, int rank,
                                         float eps, float lambda, float* stage, bool* applied, long long* fx_acc,
                                         const int* fx_cidx) {
  const int lane = threadIdx.x & 31;
  float* Wv = stage; float* Hv = stage + 2 * rank;
  *applied = false;
  if (!dev::slow_pull(c, kw, Wv) || !dev::slow_pull(c, kh, Hv)) return 0.f;
  float wh = 0.f;
  for (int z = lane; z < rank; z += 32) wh += Wv[z] * Hv[z];
  wh = dev::warp_sum(wh);
  const float e = x - wh;
  const float f1 = -2.f * e, f2 = 2.f * lambda;
  for (int z = lane; z < rank; z += 32) {
    float w = Wv[z], h = Hv[z];
    float gw = -(f1 * h + f2 * w * inv_rn), gh = -(f1 * w + f2 * h * inv_cn);
    float aw = Wv[rank + z], ah = Hv[rank + z];
    Wv[z] = eps * gw * rsqrtf(aw + gw * gw + kAdagradEps); Wv[rank + z] = gw * gw;
    Hv[z] = eps * gh * rsqrtf(ah + gh * gh + kAdagradEps); Hv[rank + z] = gh * gh;
  }
  __syncwarp();
  if (FX) {
    fx_add_staged(fx::region(fx_acc, fx_cidx, kw, 2 * rank), Wv, rank);
    fx_add_staged(fx::region(fx_acc, fx_cidx, kh, 2 * rank), Hv, rank);
    *applied = true;
  } else {
    bool ok = dev::slow_push(c, kw, Wv);
    ok = dev::slow_push(c, kh, Hv) && ok;
    *applied = ok;
  }
  return e * e;
}

// VPL: float4 per lane over `rank` floats; 0 = generic only. FX: deterministic mode (mf_step_fx_kernel).
template <int VPL, bool FX>
__device__ __forceinline__ void
mf_step_body(const Ctx& c, const Key* __restrict__ row_keys, const Key* __restrict__ col_keys,
             const float* __restrict__ xs, const int* __restrict__ row_nnz, const int* __restrict__ col_nnz, int n,
             int rank, float eps, float lambda, float* __restrict__ loss_out, unsigned long long* __restrict__ stats,
             long long* __restrict__ fx_acc, const int* __restrict__ fx_cidx, float* __restrict__ call_loss) {
  extern __shared__ float smem_f[];
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int warp_in_block = threadIdx.x >> 5;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  float* stage = smem_f + (size_t)warp_in_block * 4 * rank;
  const int nvec = rank >> 2;
  float loss_acc = 0.f;
  unsigned n_local = 0, n_remote = 0, n_slow = 0, n_upd = 0;
  for (int p = warp; p < n; p += nwarps) {
    const Key kw = row_keys[p], kh = col_keys[p];
    const float x = xs[p];
    const float inv_rn = 1.f / (float)max(1, row_nnz[p]), inv_cn = 1.f / (float)max(1, col_nnz[p]);
    dev::Target t;
    t.row = nullptr; t.version = nullptr; t.flag = nullptr;
    if (VPL > 0 && lane < 2) {
      Key k = lane == 0 ? kw : kh;
      t = dev::resolve_fast(c, k, class_of_key(c, k), &n_local, &n_remote);
    }
    float* pw = (float*)__shfl_sync(0xffffffffu, (unsigned long long)t.row, 0);
    float* ph = (float*)__shfl_sync(0xffffffffu, (unsigned long long)t.row, 1);
    if (VPL == 0 || !pw || !ph) {
      ++n_slow;
      bool applied;
      const float l = mf_generic<FX>(c, kw, kh, x, inv_rn, inv_cn, rank, eps, lambda, stage, &applied, fx_acc, fx_cidx);
      if (FX) { if (lane == 0) call_loss[p] = l; }
      else loss_acc += l;
      if (applied) n_upd += 2;
      continue;
    }
    constexpr int V = VPL > 0 ? VPL : 1;
    float4 w[V], h[V];
    float wh = 0.f;
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const int j = lane + 32 * v;
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      w[v] = j < nvec ? dev::ld_row4(pw + 4 * j) : z;
      h[v] = j < nvec ? dev::ld_row4(ph + 4 * j) : z;
      wh += w[v].x * h[v].x + w[v].y * h[v].y + w[v].z * h[v].z + w[v].w * h[v].w;
    }
    wh = dev::warp_sum(wh);
    const float e = x - wh;
    if (FX) { if (lane == 0) call_loss[p] = e * e; }
    else loss_acc += e * e;
    const float f1 = -2.f * e, f2 = 2.f * lambda;
    long long *fw = nullptr, *fh = nullptr;
    if (FX) { fw = fx::region(fx_acc, fx_cidx, kw, 2 * rank); fh = fx::region(fx_acc, fx_cidx, kh, 2 * rank); }
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const int j = lane + 32 * v;
      if (j < nvec) {
        float4 aw = dev::ld_row4(pw + rank + 4 * j), ah = dev::ld_row4(ph + rank + 4 * j);
        float4 gw, gh, uw, uh;
        gw.x = -(f1 * h[v].x + f2 * w[v].x * inv_rn); gh.x = -(f1 * w[v].x + f2 * h[v].x * inv_cn);
        gw.y = -(f1 * h[v].y + f2 * w[v].y * inv_rn); gh.y = -(f1 * w[v].y + f2 * h[v].y * inv_cn);
        gw.z = -(f1 * h[v].z + f2 * w[v].z * inv_rn); gh.z = -(f1 * w[v].z + f2 * h[v].z * inv_cn);
        gw.w = -(f1 * h[v].w + f2 * w[v].w * inv_rn); gh.w = -(f1 * w[v].w + f2 * h[v].w * inv_cn);
        float4 qw = make_float4(gw.x * gw.x, gw.y * gw.y, gw.z * gw.z, gw.w * gw.w);
        float4 qh = make_float4(gh.x * gh.x, gh.y * gh.y, gh.z * gh.z, gh.w * gh.w);
        uw.x = eps * gw.x * rsqrtf(aw.x + qw.x + kAdagradEps); uh.x = eps * gh.x * rsqrtf(ah.x + qh.x + kAdagradEps);
        uw.y = eps * gw.y * rsqrtf(aw.y + qw.y + kAdagradEps); uh.y = eps * gh.y * rsqrtf(ah.y + qh.y + kAdagradEps);
        uw.z = eps * gw.z * rsqrtf(aw.z + qw.z + kAdagradEps); uh.z = eps * gh.z * rsqrtf(ah.z + qh.z + kAdagradEps);
        uw.w = eps * gw.w * rsqrtf(aw.w + qw.w + kAdagradEps); uh.w = eps * gh.w * rsqrtf(ah.w + qh.w + kAdagradEps);
        if (FX) {
          fx::add4(fw, j, nvec, uw, kFxVal); fx::add4(fw + rank, j, nvec, qw, kFxAda);
          fx::add4(fh, j, nvec, uh, kFxVal); fx::add4(fh + rank, j, nvec, qh, kFxAda);
        } else {
          dev::red_row4(pw + 4 * j, uw); dev::red_row4(pw + rank + 4 * j, qw);
          dev::red_row4(ph + 4 * j, uh); dev::red_row4(ph + rank + 4 * j, qh);
        }
      }
    }
    if (lane < 2) dev::mark_pushed(t);
    n_upd += 2;
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

template <int VPL>
__global__ void __launch_bounds__(kThreads, 3)
mf_step_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ row_keys, const Key* __restrict__ col_keys,
               const float* __restrict__ xs, const int* __restrict__ row_nnz, const int* __restrict__ col_nnz, int n,
               int rank, float eps, float lambda, float* __restrict__ loss_out, unsigned long long* __restrict__ stats) {
  mf_step_body<VPL, false>(c, row_keys, col_keys, xs, row_nnz, col_nnz, n, rank, eps, lambda, loss_out, stats, nullptr,
                           nullptr, nullptr);
}

template <int VPL>
__global__ void __launch_bounds__(kThreads, 3)
mf_step_fx_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ row_keys, const Key* __restrict__ col_keys,
                  const float* __restrict__ xs, const int* __restrict__ row_nnz, const int* __restrict__ col_nnz, int n,
                  int rank, float eps, float lambda, unsigned long long* __restrict__ stats,
                  long long* __restrict__ fx_acc, const int* __restrict__ fx_cidx, float* __restrict__ call_loss) {
  mf_step_body<VPL, true>(c, row_keys, col_keys, xs, row_nnz, col_nnz, n, rank, eps, lambda, nullptr, stats, fx_acc,
                          fx_cidx, call_loss);
}

}  // namespace

void mf_step(CudaBackend& be, cudaStream_t stream, const Key* row_keys, const Key* col_keys, const float* xs,
             const int* row_nnz, const int* col_nnz, int n, int rank, float eps, float lambda, float* loss_out,
             unsigned long long* stats, bool deterministic) {
  if (n == 0) return;
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  be.track_stream(stream);
  const Ctx& c = be.ctx();
  const int warps_per_block = kThreads / 32;
  int blocks = std::min((n + warps_per_block - 1) / warps_per_block, be.num_sms() * 16);
  size_t smem = (size_t)warps_per_block * 4 * rank * sizeof(float);
  ADAPM_CHECK(smem <= 96 * 1024, "mf_step: rank too large");
  int vpl = (rank % 4 == 0) ? (rank / 4 + 31) / 32 : 0;
  if (vpl > 2) vpl = 0;
#define ADAPM_LAUNCH_MF(V)                                                                                   \
  do {                                                                                                       \
    static bool attr_set = false;                                                                            \
    if (!attr_set) {                                                                                         \
      cudaFuncSetAttribute(mf_step_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);       \
      attr_set = true;                                                                                       \
    }                                                                                                        \
    mf_step_kernel<V><<<blocks, kThreads, smem, stream>>>(c, row_keys, col_keys, xs, row_nnz, col_nnz, n, rank, eps, \
                                                          lambda, loss_out, stats);                          \
  } while (0)
#define ADAPM_LAUNCH_MF_FX(V)                                                                                \
  do {                                                                                                       \
    static bool attr_set = false;                                                                            \
    if (!attr_set) {                                                                                         \
      cudaFuncSetAttribute(mf_step_fx_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);    \
      attr_set = true;                                                                                       \
    }                                                                                                        \
    mf_step_fx_kernel<V><<<blocks, kThreads, smem, stream>>>(c, row_keys, col_keys, xs, row_nnz, col_nnz, n, rank, \
                                                             eps, lambda, stats, fxs.acc, fxs.cidx,          \
                                                             fxs.call_loss);                                 \
  } while (0)
  if (deterministic) {
    // one GPU, start-of-step reads: every key gets a [rank | rank] accumulator region
    const fx::Source src[2] = {{row_keys, n, 1}, {col_keys, n, 1}};
    CudaBackend::FxScratch& fxs = fx::begin(be, stream, src, 2, 2 * rank, n);
    switch (vpl) {
      case 1: ADAPM_LAUNCH_MF_FX(1); break;
      case 2: ADAPM_LAUNCH_MF_FX(2); break;
      default: ADAPM_LAUNCH_MF_FX(0); break;
    }
    ADAPM_COUNT_LAUNCH();
    ADAPM_CUDA_CHECK(cudaGetLastError());
    fx::apply(be, stream, 2 * rank, kFxVal, kFxAda, 0.f, n, loss_out);
    return;
  }
  switch (vpl) {
    case 1: ADAPM_LAUNCH_MF(1); break;
    case 2: ADAPM_LAUNCH_MF(2); break;
    default: ADAPM_LAUNCH_MF(0); break;
  }
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

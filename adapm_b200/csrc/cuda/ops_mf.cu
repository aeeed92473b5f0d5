// Fused matrix-factorisation SGD step for sm_90a: Pull(w_i, h_j) + error + L2 + AdaGrad + Push
// in one kernel over local HBM / NVLink peers (SURVEY K1 + K10 + K9 + K2).
//
// Update rule = the reference's UpdateNsqlL2Adagrad (apps/mf/update.h:32-70):
//   e = x - <w, h>;  g_w = -(-2 e h + 2 lambda w / nnz_row);  g_h = -(-2 e w + 2 lambda h / nnz_col)
//   push(w, [eps * g_w / sqrt(acc_w + g_w^2 + 1e-6) | g_w^2])   (same for h)
// Row layout [factors(rank) | AdaGrad(rank)] (apps/matrix_factorization.cc:697).
// A warp_step rule without negatives (kge_step.cuh): one warp per non-zero; two lanes resolve the two keys at once.
// Ranks with no float4 body (rank % 4 != 0 or rank > 256) take the generic path for every non-zero. The generic path
// stages the two rows in the warp's shared memory and runs the scalar body on them.
//
// Deterministic one-GPU variant (mf_step_fx_kernel): every non-zero reads the state at the start of the step and adds
// its updates as fixed-point integers into per-key accumulator regions (fx_accum.cuh), which one apply pass adds to the
// rows; each non-zero's squared error goes to its own slot and is summed in a fixed order (float64).
#include <cuda_runtime.h>

#include "fx_accum.cuh"
#include "kge_step.cuh"
#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {

namespace {

using namespace kge;

constexpr float kAdagradEps = 1e-6f;
// Fixed-point scales of the deterministic mode. |factor update| <= eps per non-zero (AdaGrad normalises it): 2^40
// leaves 2^23 / eps non-zeros per element and step. AdaGrad increments are g^2 with g = 2 e h - 2 lambda w / nnz, which
// grows with the error e and so with the data: 2^30 leaves 2^33 (8.6e9) of summed g^2 per element and step, at a
// resolution of 9.3e-10. The loss is summed in float64 from per-non-zero float squared errors.
constexpr float kFxVal = 1099511627776.f;     // 2^40
constexpr float kFxAda = 1073741824.f;        // 2^30
// the largest rank whose two staged rows per warp fit 96 KB of shared memory per CTA
constexpr int kMfMaxRank = 96 * 1024 / (kStepThreads / 32 * 4 * (int)sizeof(float));

struct Args {
  const Key* row_keys;
  const Key* col_keys;
  const float* xs;
  const int* row_nnz;
  const int* col_nnz;
  int B, n_neg, d;             // n_neg = 0; d: the rank
  float eps, lambda;
  float* scratch;              // unused: the generic path stages in shared memory
  long long* fx_acc;           // FX: fixed-point regions, per-non-zero loss slots
  const int* fx_cidx;
  float* call_loss;
};

// MF's AdaGrad push of gradient g onto float4 j of a row [factors (rank) | AdaGrad (rank)] whose accumulators a the
// caller loaded: in place (REDs) or into the key's fixed-point region
template <bool FX>
__device__ __forceinline__ void push_mf4(float* row, int rank, int j, float4 g, float4 a, long long* region, int nvec,
                                         float eps) {
  const float4 q = make_float4(g.x * g.x, g.y * g.y, g.z * g.z, g.w * g.w);
  const float4 u = make_float4(eps * g.x * rsqrtf(a.x + q.x + kAdagradEps), eps * g.y * rsqrtf(a.y + q.y + kAdagradEps),
                               eps * g.z * rsqrtf(a.z + q.z + kAdagradEps), eps * g.w * rsqrtf(a.w + q.w + kAdagradEps));
  if (FX) {
    fx::add4(region, j, nvec, u, kFxVal);
    fx::add4(region + rank, j, nvec, q, kFxAda);
  } else {
    dev::red_row4(row + 4 * j, u);
    dev::red_row4(row + rank + 4 * j, q);
  }
}

// The step as a warp_step rule: positive (w, h). VPL float4 per lane over `rank` floats; 0: scalar generic path only.
template <int VPL>
struct Mf {
  static constexpr int kPositives = 2, kMaxDim = kMfMaxRank, kMaxNeg = 0, kBlocksPerSM = 16;
  static constexpr bool kInPlace = VPL > 0, kStageInSmem = true;
  static __device__ __forceinline__ Key positive(const Args& A, int t, int i) {
    return i == 0 ? A.row_keys[t] : A.col_keys[t];
  }
  static __host__ __device__ __forceinline__ size_t state_bytes(int rank, int) {
    return (size_t)4 * rank * sizeof(float);
  }
  static __host__ __device__ __forceinline__ size_t warp_bytes(int rank, int n_neg) { return state_bytes(rank, n_neg); }
  static __host__ __device__ __forceinline__ int scratch_rows(int) { return 0; }
  static __device__ __forceinline__ int stage_row(int, int i) { return i; }
  template <bool FX, bool GEN>
  static __device__ StepOut body(const Ctx& c, const Args& A, int t, const Rows<2>& rows, bool slow,
                                 const dev::Target* ntg, float* wsm, float* stage);
};

// One non-zero: pw / ph its rows. The generic path (GEN: both rows are staged in shared memory) runs the scalar body
// at every VPL.
template <int VPL>
template <bool FX, bool GEN>
__device__ __forceinline__ StepOut Mf<VPL>::body(const Ctx&, const Args& A, int t, const Rows<2>& rows, bool,
                                                 const dev::Target*, float*, float*) {
  constexpr int V = VPL > 0 ? VPL : 1;
  const int lane = threadIdx.x & 31;
  const int rank = A.d, nvec = rank >> 2;
  float* const pw = rows.p[0];
  float* const ph = rows.p[1];
  float4 w[V], h[V];
  float wh = 0.f;
  if constexpr (VPL == 0 || GEN) {
    for (int z = lane; z < rank; z += 32) wh += pw[z] * ph[z];
  } else {
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int j = lane + 32 * v;
      w[v] = j < nvec ? dev::ld_row4(pw + 4 * j) : f4(0.f);
      h[v] = j < nvec ? dev::ld_row4(ph + 4 * j) : f4(0.f);
      wh += w[v].x * h[v].x + w[v].y * h[v].y + w[v].z * h[v].z + w[v].w * h[v].w;
    }
  }
  wh = dev::warp_sum(wh);
  const float e = A.xs[t] - wh;
  const float f1 = -2.f * e, f2 = 2.f * A.lambda;
  const float inv_rn = 1.f / (float)max(1, A.row_nnz[t]), inv_cn = 1.f / (float)max(1, A.col_nnz[t]);
  long long *fw = nullptr, *fh = nullptr;
  if (FX) {
    fw = fx::region(A.fx_acc, A.fx_cidx, A.row_keys[t], 2 * rank);
    fh = fx::region(A.fx_acc, A.fx_cidx, A.col_keys[t], 2 * rank);
  }
  if constexpr (VPL == 0 || GEN) {
    for (int z = lane; z < rank; z += 32) {
      const float w = pw[z], h = ph[z];
      const float gw = -(f1 * h + f2 * w * inv_rn), gh = -(f1 * w + f2 * h * inv_cn);
      const float uw = A.eps * gw * rsqrtf(pw[rank + z] + gw * gw + kAdagradEps);
      const float uh = A.eps * gh * rsqrtf(ph[rank + z] + gh * gh + kAdagradEps);
      if (FX) {
        fx::add1(fw, z, rank, uw, kFxVal); fx::add1(fw + rank, z, rank, gw * gw, kFxAda);
        fx::add1(fh, z, rank, uh, kFxVal); fx::add1(fh + rank, z, rank, gh * gh, kFxAda);
      } else {
        pw[z] = uw; pw[rank + z] = gw * gw;
        ph[z] = uh; ph[rank + z] = gh * gh;
      }
    }
  } else {
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int j = lane + 32 * v;
      if (j < nvec) {
        const float4 aw = dev::ld_row4(pw + rank + 4 * j), ah = dev::ld_row4(ph + rank + 4 * j);
        float4 gw, gh;
        gw.x = -(f1 * h[v].x + f2 * w[v].x * inv_rn); gh.x = -(f1 * w[v].x + f2 * h[v].x * inv_cn);
        gw.y = -(f1 * h[v].y + f2 * w[v].y * inv_rn); gh.y = -(f1 * w[v].y + f2 * h[v].y * inv_cn);
        gw.z = -(f1 * h[v].z + f2 * w[v].z * inv_rn); gh.z = -(f1 * w[v].z + f2 * h[v].z * inv_cn);
        gw.w = -(f1 * h[v].w + f2 * w[v].w * inv_rn); gh.w = -(f1 * w[v].w + f2 * h[v].w * inv_cn);
        push_mf4<FX>(pw, rank, j, gw, aw, fw, nvec, A.eps);
        push_mf4<FX>(ph, rank, j, gh, ah, fh, nvec, A.eps);
      }
    }
  }
  return {e * e, 0u, 0u, 0ull};
}

template <int VPL>
__global__ void __launch_bounds__(kStepThreads, 3)
mf_step_kernel(const __grid_constant__ Ctx c, const __grid_constant__ Args A, float* __restrict__ loss_out,
               unsigned long long* __restrict__ stats) {
  warp_step<Mf<VPL>, false>(c, A, loss_out, stats);
}

template <int VPL>
__global__ void __launch_bounds__(kStepThreads, 3)
mf_step_fx_kernel(const __grid_constant__ Ctx c, const __grid_constant__ Args A, float* __restrict__ loss_out,
                  unsigned long long* __restrict__ stats) {
  warp_step<Mf<VPL>, true>(c, A, loss_out, stats);
}

template <bool FX, int VPL>
void launch_mf(CudaBackend& be, cudaStream_t stream, const Args& A, float* loss_out, unsigned long long* stats) {
  if constexpr (FX) launch_step<Mf<VPL>, mf_step_fx_kernel<VPL>>(be, stream, A, loss_out, stats);
  else launch_step<Mf<VPL>, mf_step_kernel<VPL>>(be, stream, A, loss_out, stats);
}

}  // namespace

void mf_step(CudaBackend& be, cudaStream_t stream, const Key* row_keys, const Key* col_keys, const float* xs,
             const int* row_nnz, const int* col_nnz, int n, int rank, float eps, float lambda, float* loss_out,
             unsigned long long* stats, bool deterministic) {
  if (n == 0) return;
  ADAPM_CHECK(kStepThreads / 32 * Mf<0>::warp_bytes(rank, 0) <= 96 * 1024, "mf_step: rank too large");
  int vpl = (rank % 4 == 0) ? (rank / 4 + 31) / 32 : 0;
  if (vpl > 2) vpl = 0;
  Args A;
  A.row_keys = row_keys; A.col_keys = col_keys; A.xs = xs; A.row_nnz = row_nnz; A.col_nnz = col_nnz;
  A.B = n; A.n_neg = 0; A.d = rank; A.eps = eps; A.lambda = lambda;
  // deterministic: every key gets a [rank | rank] accumulator region
  const fx::Source src[2] = {{row_keys, n, 1}, {col_keys, n, 1}};
  run_step(be, stream, A, deterministic, src, 2, 2 * rank, kFxVal, kFxAda, loss_out, [&](auto fx, float* lo) {
    constexpr bool FX = decltype(fx)::value;
    switch (vpl) {
      case 1: launch_mf<FX, 1>(be, stream, A, lo, stats); break;
      case 2: launch_mf<FX, 2>(be, stream, A, lo, stats); break;
      default: launch_mf<FX, 0>(be, stream, A, lo, stats); break;
    }
  });
}

}  // namespace cudaops
}  // namespace adapm

// word2vec SGNS with SHARED negatives on the tensor cores (SURVEY K7, optional formulation).
//
// The reference draws `negative` fresh negatives for every (center, context) pair (apps/word2vec.cc:682-745): 27 rows
// of 2400 B are touched per pair and the arithmetic is a batch of independent dot products - the fused step kernel
// (ops_sgns_tma.cu) is bound by row traffic, there is nothing for a tensor core to do. With one set of Nn negatives
// shared by the B pairs of a batch the same objective becomes three GEMM-shaped contractions over the SAME operands:
//
//     S   [B, Nn] = E0 [B, d]  x En^T            scores of every center against every shared negative
//     G   [B, Nn] = -sigmoid(S)                  (label 0; negative == the pair's positive target is masked out)
//     dE0 [B, d]  = G x En        + gpos * Ec    center gradient (gpos = 1 - sigmoid(<e0, ec>), the positive target)
//     dEn [Nn, d] = G^T x E0                     negative gradient
//
// i.e. B * Nn sample pairs for 2 B + Nn rows of traffic. All three contractions run on the hand-written wgmma /
// TMA GEMM of this package (ops_gemm_wgmma.cu; bf16 operands, fp32 accumulation); the pieces around them are the
// three kernels of this file:
//   shared_prep_kernel    rows (fp32, as pulled from the store) -> bf16 operand + its transpose (tile transposition
//                         through shared memory), positive-target gradient gpos and its loss
//   shared_grad_kernel    S -> G (bf16) and G^T (bf16), masking, loss
//   shared_update_kernel  AdaGrad (worker-side rule of the reference, word2vec.cc:702-745) -> additive updates
//                         [embedding | AdaGrad] for all 2 B + Nn rows, pushed by the caller with ONE Push
// Rows are gathered / scattered with the store's Pull / Push kernels (every protocol state, local or NVLink), so the
// variant works wherever the fused kernel works. Python: adapm_b200.ops.sgns_shared_step.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "group.cuh"
#include "ops.h"

namespace adapm {
namespace cudaops {

namespace {

constexpr float kMaxExp = 6.f;   // MAX_EXP of the reference: gradients saturate outside [-6, 6]
constexpr int kTile = 32;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// rows[n_rows][2 d] fp32 -> Eb[n_rows][dpad] bf16 (zero padded) and EbT[dpad][ldt] bf16 (column r = row r).
// other != nullptr: gpos[r] = label 1 gradient of <rows[r].e, other[r].e> and its loss.
__global__ void __launch_bounds__(256)
shared_prep_kernel(const float* __restrict__ rows, const float* __restrict__ other, int n_rows, int d, int dpad,
                   __nv_bfloat16* __restrict__ Eb, __nv_bfloat16* __restrict__ EbT, int ldt, float* __restrict__ gpos,
                   float* __restrict__ loss) {
  extern __shared__ __nv_bfloat16 tile[];            // [kTile][dpad + 2]
  const int pitch = dpad + 2;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r0 = blockIdx.x * kTile;
  float loss_acc = 0.f;
  for (int rl = warp; rl < kTile; rl += 8) {
    const int r = r0 + rl;
    float dot = 0.f;
    for (int j = lane; j < dpad; j += 32) {
      float e = 0.f;
      if (r < n_rows && j < d) {
        e = rows[(size_t)r * 2 * d + j];
        if (other) dot += e * other[(size_t)r * 2 * d + j];
      }
      const __nv_bfloat16 b = __float2bfloat16(e);
      tile[rl * pitch + j] = b;
      if (r < n_rows) Eb[(size_t)r * dpad + j] = b;
    }
    if (other && r < n_rows) {
      const float f = warp_sum(dot);
      if (lane == 0) {
        gpos[r] = f > kMaxExp ? 0.f : (f < -kMaxExp ? 1.f : 1.f - 1.f / (1.f + __expf(-f)));
        loss_acc += __logf(1.f + __expf(-fminf(fmaxf(f, -kMaxExp), kMaxExp)));
      }
    }
  }
  __syncthreads();
  if (r0 + lane < ldt) {
    for (int j = warp; j < dpad; j += 8) EbT[(size_t)j * ldt + r0 + lane] = tile[lane * pitch + j];
  }
  if (other && lane == 0 && loss_acc != 0.f) atomicAdd(loss, loss_acc);
}

// S[B][Nn] -> Gb[B][Nn], GbT[Nn][B] (bf16): G = -sigmoid(S), saturated like the reference; a shared negative that IS the
// pair's positive target does not count (reference: `if (target == word) continue`).
__global__ void __launch_bounds__(256)
shared_grad_kernel(const float* __restrict__ S, const Key* __restrict__ contexts, const Key* __restrict__ negs, int B, int Nn,
                   __nv_bfloat16* __restrict__ Gb, __nv_bfloat16* __restrict__ GbT, float* __restrict__ loss) {
  __shared__ float tile[kTile][kTile + 1];
  __shared__ float red[8];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;     // 32 x 8
  const int n0 = blockIdx.x * kTile, b0 = blockIdx.y * kTile;
  const Key nk = negs[n0 + tx];
  float loss_acc = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int bl = ty + 8 * i, b = b0 + bl;
    const float s = S[(size_t)b * Nn + n0 + tx];
    float g = 0.f;
    if (contexts[b] != nk) {
      g = s > kMaxExp ? -1.f : (s < -kMaxExp ? 0.f : -1.f / (1.f + __expf(-s)));
      loss_acc += __logf(1.f + __expf(fminf(fmaxf(s, -kMaxExp), kMaxExp)));
    }
    Gb[(size_t)b * Nn + n0 + tx] = __float2bfloat16(g);
    tile[bl][tx] = g;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int nl = ty + 8 * i;
    GbT[(size_t)(n0 + nl) * B + b0 + tx] = __float2bfloat16(tile[tx][nl]);
  }
  loss_acc = warp_sum(loss_acc);
  if (tx == 0) red[ty] = loss_acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i];
    atomicAdd(loss, t);
  }
}

// One warp per row of R = [centers (B) | contexts (B) | negatives (Nn)] x [embedding (d) | AdaGrad (d)]:
// U = [alpha * g * rsqrt(a + g^2) | g^2]   (AdaGrad with the accumulator read before the update, like the fused kernel)
__global__ void __launch_bounds__(256)
shared_update_kernel(const float* __restrict__ R, const float* __restrict__ dE0, const float* __restrict__ dEn,
                     const float* __restrict__ gpos, int B, int Nn, int d, int dpad, float alpha, float* __restrict__ U) {
  const int lane = threadIdx.x & 31;
  const long r = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= 2L * B + Nn) return;
  const float* row = R + (size_t)r * 2 * d;
  float* out = U + (size_t)r * 2 * d;
  const float* mat = nullptr;      // GEMM part of the gradient
  const float* peer = nullptr;     // the pair's other row (positive-target part)
  float gp = 0.f;
  if (r < B) { mat = dE0 + (size_t)r * dpad; peer = R + (size_t)(B + r) * 2 * d; gp = gpos[r]; }
  else if (r < 2L * B) { peer = R + (size_t)(r - B) * 2 * d; gp = gpos[r - B]; }
  else mat = dEn + (size_t)(r - 2L * B) * dpad;
  for (int j = lane; j < d; j += 32) {
    float g = mat ? mat[j] : 0.f;
    if (peer) g += gp * peer[j];
    const float ua = g * g;
    out[j] = alpha * g * rsqrtf(row[d + j] + ua);
    out[d + j] = ua;
  }
}

inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace

size_t sgns_shared_workspace_bytes(int B, int Nn, int d) {
  const size_t dpad = (size_t)((d + 7) / 8) * 8;
  size_t n = 0;
  n += align_up((size_t)B * dpad * 2);      // E0b
  n += align_up(dpad * (size_t)B * 2);      // E0bT
  n += align_up((size_t)Nn * dpad * 2);     // Nb
  n += align_up(dpad * (size_t)Nn * 2);     // NbT
  n += align_up((size_t)B * Nn * 4);        // S
  n += align_up((size_t)B * Nn * 2);        // Gb
  n += align_up((size_t)Nn * B * 2);        // GbT
  n += align_up((size_t)B * dpad * 4);      // dE0
  n += align_up((size_t)Nn * dpad * 4);     // dEn
  n += align_up((size_t)B * 4);             // gpos
  return n;
}

// R: pulled rows [2 B + Nn][2 d] in the order centers | contexts | shared negatives; U: the additive updates, same order.
void sgns_shared_core(cudaStream_t stream, const float* R, const Key* contexts, const Key* negs, int B, int Nn, int d,
                      float alpha, void* workspace, float* U, float* loss) {
  ADAPM_CHECK(B > 0 && Nn > 0 && B % kTile == 0 && Nn % kTile == 0, "sgns_shared: batch and negative count must be multiples of 32");
  ADAPM_CHECK(d > 0 && d <= 512, "sgns_shared: embedding dimension out of range");
  const int dpad = ((d + 7) / 8) * 8;
  char* p = static_cast<char*>(workspace);
  auto take = [&](size_t bytes) { char* q = p; p += align_up(bytes); return q; };
  auto* E0b = reinterpret_cast<__nv_bfloat16*>(take((size_t)B * dpad * 2));
  auto* E0bT = reinterpret_cast<__nv_bfloat16*>(take((size_t)dpad * B * 2));
  auto* Nb = reinterpret_cast<__nv_bfloat16*>(take((size_t)Nn * dpad * 2));
  auto* NbT = reinterpret_cast<__nv_bfloat16*>(take((size_t)dpad * Nn * 2));
  auto* S = reinterpret_cast<float*>(take((size_t)B * Nn * 4));
  auto* Gb = reinterpret_cast<__nv_bfloat16*>(take((size_t)B * Nn * 2));
  auto* GbT = reinterpret_cast<__nv_bfloat16*>(take((size_t)Nn * B * 2));
  auto* dE0 = reinterpret_cast<float*>(take((size_t)B * dpad * 4));
  auto* dEn = reinterpret_cast<float*>(take((size_t)Nn * dpad * 4));
  auto* gpos = reinterpret_cast<float*>(take((size_t)B * 4));
  const size_t tile_smem = (size_t)kTile * (dpad + 2) * sizeof(__nv_bfloat16);
  const float* Rc = R;
  const float* Rp = R + (size_t)B * 2 * d;
  const float* Rn = R + (size_t)2 * B * 2 * d;
  shared_prep_kernel<<<B / kTile, 256, tile_smem, stream>>>(Rc, Rp, B, d, dpad, E0b, E0bT, B, gpos, loss);
  shared_prep_kernel<<<Nn / kTile, 256, tile_smem, stream>>>(Rn, nullptr, Nn, d, dpad, Nb, NbT, Nn, nullptr, nullptr);
  ADAPM_COUNT_LAUNCH(); ADAPM_COUNT_LAUNCH();
  gemm_nt_bf16(stream, E0b, Nb, B, Nn, dpad, S, Nn);                     // S = E0 En^T
  shared_grad_kernel<<<dim3(Nn / kTile, B / kTile), 256, 0, stream>>>(S, contexts, negs, B, Nn, Gb, GbT, loss);
  ADAPM_COUNT_LAUNCH();
  gemm_nt_bf16(stream, Gb, NbT, B, dpad, Nn, dE0, dpad);                 // dE0 = G En      (K = Nn)
  gemm_nt_bf16(stream, GbT, E0bT, Nn, dpad, B, dEn, dpad);               // dEn = G^T E0    (K = B)
  const long rows = 2L * B + Nn;
  shared_update_kernel<<<(unsigned)((rows * 32 + 255) / 256), 256, 0, stream>>>(R, dE0, dEn, gpos, B, Nn, d, dpad, alpha, U);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

// DLRM's pairwise dot interaction (Naumov et al., 2019) for sm_90a: forward and backward, one launch each.
//
// Per example b, T = [z_b; e_b,0; ...; e_b,F-1] is the (F + 1) x E matrix of the bottom-MLP output z [B, E] and the F
// pooled field embeddings e [B, F, E] (the rows of e are read in place: no cat). With N = F + 1, P = F (F + 1) / 2 and
// W = E + P rounded up to a multiple of 8, the forward writes
//   R[b, :E] = z_b,   R[b, E + p] = <T_i, T_j> for the p-th pair (i, j), 0 <= j < i <= F, row-major
//   (p = i (i - 1) / 2 + j: the order of torch.tril_indices(N, N, -1)),   R[b, E + P:] = 0.
// The backward, for the gradient dR of R, writes (dZ_ij = dR[b, E + p(max(i, j), min(i, j))], dZ_ii = 0)
//   dT_i = sum_j dZ_ij T_j (j = 0 .. N - 1 in order),   dz = dR[:, :E] + dT_0,   de_f = dT_{f + 1}.
//
// One CTA per example. Its T is staged in shared memory by 16-byte cp.async copies (the whole example's bytes are in
// flight at once; several CTAs per SM keep HBM busy while others compute). Every output element is summed by one
// owner in a fixed order in fp32, without atomics, so two runs give bit-identical R, dz and de.
//   forward:  the lower triangle of T T^T in 4 x 4 tiles of rows; a tile belongs to 8 lanes that split E (lane s
//             takes the float4 columns s, s + 8, ...), each lane sums its columns in order and the 8 partial sums are
//             added by a fixed xor butterfly. R's row is assembled in shared memory and written with float4 stores.
//   backward: dZ (symmetric, zero diagonal, N x NP with NP = N rounded up to 4) is built in shared memory from dR; a
//             thread owns 4 rows x 4 columns of dT and adds dZ_ij T_j for j in order (dZ's row j read as a float4
//             broadcast, T_j as a float4).
#include <cuda_runtime.h>

#include "group.cuh"
#include "ops.h"

namespace adapm {
namespace cudaops {

namespace {

constexpr int kDlrmThreads = 128;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  const unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem) : "memory");
}

__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

// T of example b into shared memory: row 0 = z[b], rows 1..F = e[b] (N rows of E floats, dense)
__device__ __forceinline__ void stage_t(float* t, const float* __restrict__ z, const float* __restrict__ e, int b, int F,
                                        int E) {
  const int E4 = E >> 2;
  const float4* zs = reinterpret_cast<const float4*>(z + (size_t)b * E);
  const float4* es = reinterpret_cast<const float4*>(e + (size_t)b * F * E);
  float4* ts = reinterpret_cast<float4*>(t);
  for (int i = threadIdx.x; i < (F + 1) * E4; i += blockDim.x) cp_async16(ts + i, i < E4 ? zs + i : es + (i - E4));
}

__device__ __forceinline__ float dot4(const float4& a, const float4& b, float acc) {
  acc = fmaf(a.x, b.x, acc);
  acc = fmaf(a.y, b.y, acc);
  acc = fmaf(a.z, b.z, acc);
  return fmaf(a.w, b.w, acc);
}

__global__ void __launch_bounds__(kDlrmThreads)
dlrm_interaction_fwd_kernel(const float* __restrict__ z, const float* __restrict__ e, int F, int E, int W,
                            float* __restrict__ R) {
  extern __shared__ float4 smem4[];
  const int N = F + 1, E4 = E >> 2, NB = (N + 3) >> 2;
  const int b = blockIdx.x;
  float* t = reinterpret_cast<float*>(smem4);          // [N][E]
  float* row = t + (size_t)N * E;                       // [W]: the output row
  stage_t(t, z, e, b, F, E);
  cp_async_wait_all();
  __syncthreads();

  const int sub = threadIdx.x & 7;
  const unsigned group = 0xffu << (threadIdx.x & 24);   // the 8 lanes of a tile (the loop may end early for a warp)
  const int ntiles = NB * (NB + 1) / 2;
  for (int tile = threadIdx.x >> 3; tile < ntiles; tile += kDlrmThreads >> 3) {
    int I = (int)((sqrtf(8.f * tile + 1.f) - 1.f) * 0.5f);   // tile = I (I + 1) / 2 + J, J <= I
    while (I * (I + 1) / 2 > tile) --I;
    while ((I + 1) * (I + 2) / 2 <= tile) ++I;
    const int J = tile - I * (I + 1) / 2;
    const float4* ra[4];
    const float4* rb[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {                       // rows past N alias row N - 1; their sums are not written
      ra[r] = reinterpret_cast<const float4*>(t + (size_t)min(4 * I + r, N - 1) * E);
      rb[r] = reinterpret_cast<const float4*>(t + (size_t)min(4 * J + r, N - 1) * E);
    }
    float acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
    for (int k = sub; k < E4; k += 8) {
      float4 a[4], bb[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) { a[r] = ra[r][k]; bb[r] = rb[r][k]; }
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = dot4(a[r], bb[c], acc[r][c]);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float v = acc[r][c];
        v += __shfl_xor_sync(group, v, 4, 8);
        v += __shfl_xor_sync(group, v, 2, 8);
        v += __shfl_xor_sync(group, v, 1, 8);
        const int i = 4 * I + r, j = 4 * J + c;
        if (((r * 4 + c) & 7) == sub && j < i && i < N) row[E + i * (i - 1) / 2 + j] = v;
      }
  }
  const int P = F * N / 2;
  for (int k = threadIdx.x; k < W; k += blockDim.x) {
    if (k < E) row[k] = t[k];
    else if (k >= E + P) row[k] = 0.f;
  }
  __syncthreads();
  float4* out = reinterpret_cast<float4*>(R + (size_t)b * W);
  const float4* src = reinterpret_cast<const float4*>(row);
  for (int k = threadIdx.x; k < (W >> 2); k += blockDim.x) out[k] = src[k];
}

__global__ void __launch_bounds__(kDlrmThreads)
dlrm_interaction_bwd_kernel(const float* __restrict__ dR, const float* __restrict__ z, const float* __restrict__ e,
                            int F, int E, int W, float* __restrict__ dz, float* __restrict__ de) {
  extern __shared__ float4 smem4[];
  const int N = F + 1, E4 = E >> 2, NB = (N + 3) >> 2, NP = 4 * NB;
  const int b = blockIdx.x;
  float* t = reinterpret_cast<float*>(smem4);          // [N][E]
  float* g = t + (size_t)N * E;                         // [N][NP]: dZ, zero on the diagonal and past column N - 1
  stage_t(t, z, e, b, F, E);
  const float* dr = dR + (size_t)b * W;
  for (int k = threadIdx.x; k < N * NP; k += blockDim.x) {
    const int i = k / NP, j = k - i * NP;
    float v = 0.f;
    if (j < N && j != i) {
      const int hi = max(i, j), lo = min(i, j);
      v = __ldg(dr + E + hi * (hi - 1) / 2 + lo);
    }
    g[k] = v;
  }
  cp_async_wait_all();
  __syncthreads();

  const float4* t4 = reinterpret_cast<const float4*>(t);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (int item = threadIdx.x; item < NB * E4; item += blockDim.x) {
    const int I = item / E4, k = item - I * E4;
    float4 acc[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) acc[r] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < N; ++j) {
      const float4 x = t4[(size_t)j * E4 + k];
      const float4 w = g4[j * NB + I];                  // dZ_{4I + r, j} = dZ_{j, 4I + r}
      const float wr[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        acc[r].x = fmaf(wr[r], x.x, acc[r].x);
        acc[r].y = fmaf(wr[r], x.y, acc[r].y);
        acc[r].z = fmaf(wr[r], x.z, acc[r].z);
        acc[r].w = fmaf(wr[r], x.w, acc[r].w);
      }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = 4 * I + r;
      if (i == 0) {
        const float4 d = reinterpret_cast<const float4*>(dr)[k];
        reinterpret_cast<float4*>(dz + (size_t)b * E)[k] =
            make_float4(d.x + acc[r].x, d.y + acc[r].y, d.z + acc[r].z, d.w + acc[r].w);
      } else if (i < N) {
        reinterpret_cast<float4*>(de + ((size_t)b * F + (i - 1)) * E)[k] = acc[r];
      }
    }
  }
}

void check_shape(int64_t B, int F, int E, int W) {
  ADAPM_CHECK(F >= 1 && F + 1 <= kDlrmMaxRows, "dlrm_interaction: need 1 <= F and F + 1 <= " << kDlrmMaxRows);
  ADAPM_CHECK(E % 4 == 0 && E >= 4 && E <= kDlrmMaxDim, "dlrm_interaction: E must be a multiple of 4 in [4, 512]");
  ADAPM_CHECK(W == (E + F * (F + 1) / 2 + 7) / 8 * 8, "dlrm_interaction: W must be E + F (F + 1) / 2 rounded up to 8");
  ADAPM_CHECK(B >= 0 && B * W < ((int64_t)1 << 31), "dlrm_interaction: B * W must be < 2^31");
}

template <class K>
void set_smem(K kernel, size_t smem) {
  if (smem > 48 * 1024)
    ADAPM_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
}

}  // namespace

void dlrm_interaction_forward(cudaStream_t stream, const float* z, const float* e, int64_t B, int F, int E, int W,
                              float* R) {
  check_shape(B, F, E, W);
  if (B == 0) return;
  const size_t smem = ((size_t)(F + 1) * E + W) * sizeof(float);
  set_smem(dlrm_interaction_fwd_kernel, smem);
  dlrm_interaction_fwd_kernel<<<(unsigned)B, kDlrmThreads, smem, stream>>>(z, e, F, E, W, R);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

void dlrm_interaction_backward(cudaStream_t stream, const float* dR, const float* z, const float* e, int64_t B, int F,
                               int E, int W, float* dz, float* de) {
  check_shape(B, F, E, W);
  if (B == 0) return;
  const int N = F + 1, NP = (N + 3) / 4 * 4;
  const size_t smem = ((size_t)N * E + (size_t)N * NP) * sizeof(float);
  set_smem(dlrm_interaction_bwd_kernel, smem);
  dlrm_interaction_bwd_kernel<<<(unsigned)B, kDlrmThreads, smem, stream>>>(dR, z, e, F, E, W, dz, de);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

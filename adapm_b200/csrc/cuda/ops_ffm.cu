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
// Backward (three launches, the radix sort counted as one), the skeleton of ops_embbag.cu's:
//   1. sort:   cub radix sort of (key, position b * F + f); stable, so every key's occurrences stay in position order
//   2. tile:   the sorted occurrences are cut into tiles of kTile; one lane group per tile sums each key's run of
//              contributions in fp32 in position order. A run inside the tile is pushed right away; a run that crosses
//              a tile boundary leaves one partial sum per tile it touches
//   3. finish: one warp per run that crosses a boundary adds its partials in tile order and pushes.
// Every distinct key gets one push [-eta G / sqrt(acc + G^2) | G^2] (0 where G == 0: the key's own-field block and the
// padding) with one fixed sum, so on one GPU two runs of the same step give bit-identical rows and loss. A last
// one-CTA launch adds the per-example losses in index order.
#include <cuda_runtime.h>

#include <cub/cub.cuh>

#include "grouped_push.cuh"
#include "ops.h"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {

namespace {

using namespace grouped;

constexpr int kFwdThreads = 128;
constexpr int kThreads = 256;
constexpr int kTile = 32;     // sorted occurrences per lane group in the tile pass

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
// 2. one group per tile of kTile sorted occurrences. part[t][0]: the partial of the run that was open at the tile's
// start (it began in an earlier tile); part[t][1]: the partial of a run that begins in the tile and crosses its end.
template <int VPL>
__global__ void __launch_bounds__(kThreads, 2)
ffm_grad_tile_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ sk, const int* __restrict__ spos,
                     const float* __restrict__ contrib, int nnz, int E, int log_g, float eta, float* __restrict__ part,
                     unsigned long long* __restrict__ stats) {
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int G = 1 << log_g;
  const int sub = lane & (G - 1);
  const unsigned mask = group_mask(lane, log_g);
  const int E4 = E >> 2;
  const int n_tiles = (nnz + kTile - 1) / kTile;
  const int groups_per_warp = 32 >> log_g;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  Counts n;
  for (int wt = warp * groups_per_warp; wt < n_tiles; wt += nwarps * groups_per_warp) {
    const int t = wt + (lane >> log_g);
    if (t >= n_tiles) continue;          // (group-uniform; the shuffles below only involve the group)
    const int lo = t * kTile, hi = min(nnz, lo + kTile);
    Key cur = sk[lo];
    bool open_before = lo > 0 && sk[lo - 1] == cur;
    float4 acc[VPL];
#pragma unroll
    for (int v = 0; v < VPL; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int p0 = lo; p0 <= hi; p0 += G) {
      // lane `sub` loads occurrence p0 + sub; position hi is the end of the last run
      Key kk = -1;
      int pp = 0;
      if (p0 + sub < hi) { kk = sk[p0 + sub]; pp = spos[p0 + sub]; }
      const int cnt = min(G, hi + 1 - p0);
      for (int u = 0; u < cnt; ++u) {
        const Key k = (Key)__shfl_sync(mask, (long long)kk, u, G);
        const int pu = __shfl_sync(mask, pp, u, G);
        if (k != cur) {                  // the run of `cur` ends here (k == -1: at the tile's end)
          const bool crosses = k == -1 && hi < nnz && sk[hi] == cur;
          if (open_before || crosses) {
            float* dst = part + ((size_t)t * 2 + (open_before ? 0 : 1)) * E;
#pragma unroll
            for (int v = 0; v < VPL; ++v) {
              const int j = sub + G * v;
              if (j < E4) reinterpret_cast<float4*>(dst)[j] = acc[v];
            }
          } else {
            push_update<VPL>(c, cur, acc, E, sub, G, mask, eta, n, stats);
          }
          if (k == -1) break;
          cur = k;
          open_before = false;
#pragma unroll
          for (int v = 0; v < VPL; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        const float4* cr = reinterpret_cast<const float4*>(contrib + (size_t)pu * E);
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int j = sub + G * v;
          if (j < E4) {
            const float4 x = __ldg(cr + j);
            acc[v].x += x.x; acc[v].y += x.y; acc[v].z += x.z; acc[v].w += x.w;
          }
        }
      }
    }
  }
  __syncwarp();
  flush_counts(n, stats);
  dev::cta_exit(c);
}

// 3. one warp per tile boundary q = i * kTile: if a run crosses q and does not cross q - kTile, the warp owns it: its
// partials part[i - 1][1], part[i][0], part[i + 1][0], ... are added in tile order, and the key is pushed.
template <int VPL>
__global__ void __launch_bounds__(kThreads, 2)
ffm_grad_finish_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ sk, int nnz, int E, float eta,
                       const float* __restrict__ part, unsigned long long* __restrict__ stats) {
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int E4 = E >> 2;
  const int n_tiles = (nnz + kTile - 1) / kTile;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  Counts n;
  for (int i = 1 + warp; i < n_tiles; i += nwarps) {
    const int q = i * kTile;
    const Key k = sk[q];
    if (sk[q - 1] != k || (q - kTile - 1 >= 0 && sk[q - kTile - 1] == k)) continue;   // (warp-uniform)
    float4 acc[VPL];
    const float* p0 = part + ((size_t)(i - 1) * 2 + 1) * E;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int j = lane + 32 * v;
      acc[v] = j < E4 ? reinterpret_cast<const float4*>(p0)[j] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int t = i;; ++t) {
      const float* pt = part + (size_t)t * 2 * E;
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int j = lane + 32 * v;
        if (j < E4) {
          const float4 x = reinterpret_cast<const float4*>(pt)[j];
          acc[v].x += x.x; acc[v].y += x.y; acc[v].z += x.z; acc[v].w += x.w;
        }
      }
      const int e = (t + 1) * kTile;
      if (e >= nnz || sk[e] != k) break;
    }
    push_update<VPL>(c, k, acc, E, lane, 32, 0xffffffffu, eta, n, stats);
  }
  flush_counts(n, stats);
  dev::cta_exit(c);
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
// workspace layout: sorted keys | positions (in, out) | contributions | tile partials | per-example losses | sort scratch
struct Workspace {
  Key* sk; int* pos_in; int* pos_out; float* contrib; float* part; float* loss_ex; void* sort_tmp; size_t sort_bytes;
  size_t total;
};

Workspace carve(void* base, int B, int F, int k) {
  Workspace w{};
  const int64_t nnz = (int64_t)B * F;
  const int E = 4 + F * k;
  size_t sort_bytes = 0;
  ADAPM_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const unsigned long long*)nullptr,
                                                   (unsigned long long*)nullptr, (const int*)nullptr, (int*)nullptr,
                                                   (int)nnz, 0, 64));
  const size_t n_tiles = (size_t)(nnz + kTile - 1) / kTile;
  char* p = static_cast<char*>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) { char* q = p ? p + off : nullptr; off += align_up(bytes); return q; };
  w.sk = reinterpret_cast<Key*>(take((size_t)nnz * sizeof(Key)));
  w.pos_in = reinterpret_cast<int*>(take((size_t)nnz * sizeof(int)));
  w.pos_out = reinterpret_cast<int*>(take((size_t)nnz * sizeof(int)));
  w.contrib = reinterpret_cast<float*>(take((size_t)nnz * E * sizeof(float)));
  w.part = reinterpret_cast<float*>(take(n_tiles * 2 * E * sizeof(float)));
  w.loss_ex = reinterpret_cast<float*>(take((size_t)B * sizeof(float)));
  w.sort_tmp = take(sort_bytes);
  w.sort_bytes = sort_bytes;
  w.total = off;
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
  const Ctx& c = be.ctx();
  Workspace w = carve(workspace, B, F, k);
  ADAPM_CHECK(workspace && workspace_bytes >= w.total, "ffm: workspace too small");
  const int n = B * F, E = 4 + F * k;
  launch_forward(be, stream, ids, labels, B, F, k, r, lam, nullptr, w.loss_ex, w.contrib, w.pos_in, stats);
  size_t sort_bytes = w.sort_bytes;
  ADAPM_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(w.sort_tmp, sort_bytes, reinterpret_cast<const unsigned long long*>(ids),
                                                   reinterpret_cast<unsigned long long*>(w.sk), w.pos_in, w.pos_out, n, 0,
                                                   key_bits(c.L.num_keys), stream));
  ADAPM_COUNT_LAUNCH();   // (the sort counts as one launch; cub runs one or more kernels, depending on nnz and the bits)
  int log_g, vpl;
  lane_shape(E, &log_g, &vpl);
  const int n_tiles = (n + kTile - 1) / kTile;
  const int tiles_per_block = (kThreads / 32) << (5 - log_g);
  const int tile_blocks = std::max(1, std::min((n_tiles + tiles_per_block - 1) / tiles_per_block, be.num_sms() * 16));
  const int fin_blocks = std::max(1, std::min((n_tiles + kThreads / 32 - 1) / (kThreads / 32), be.num_sms() * 8));
  switch (vpl) {
#define ADAPM_FFM_BWD(V)                                                                                             \
  case V:                                                                                                            \
    ffm_grad_tile_kernel<V><<<tile_blocks, kThreads, 0, stream>>>(c, w.sk, w.pos_out, w.contrib, n, E, log_g, eta,   \
                                                                  w.part, stats);                                    \
    ADAPM_COUNT_LAUNCH();                                                                                            \
    ffm_grad_finish_kernel<V><<<fin_blocks, kThreads, 0, stream>>>(c, w.sk, n, E, eta, w.part, stats);               \
    ADAPM_COUNT_LAUNCH();                                                                                            \
    break
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

// Fused word2vec SGNS step for sm_90a: Pull + dot/sigmoid + AdaGrad + Push in ONE kernel,
// reading rows from and reducing updates into whichever HBM currently holds each key
// (local slab, local replica, or a peer GPU over NVLink) - SURVEY K1+K7+K9+K2.
//
// Semantics follow the reference's inner loop (apps/word2vec.cc:682-745) and its worker-side
// AdaGrad (apps/word2vec.cc:420-429): for a (center, context) pair
//   e0 = row(syn0[center]).emb
//   for target in {context (label 1)} U {neg negatives (label 0)}:   (negatives == context are skipped)
//       f = <e0, row(syn1[target]).emb>;  g = label - sigmoid(f)  (|f| > 6 saturates)
//       grad0 += g * e1;  grad1 = g * e0
//       push(target, [alpha*grad1/sqrt(acc1 + grad1^2) | grad1^2])
//   push(center, [alpha*grad0/sqrt(acc0 + grad0^2) | grad0^2])
// Row layout = [embedding(d) | AdaGrad accumulator(d)] (apps/word2vec.cc:1101).
//
// One warp owns one pair. The directory lookups of all (1+neg) targets are issued by different
// lanes at once (one dependent-load chain instead of 1+neg), then rows stream through 16-byte
// loads and 16-byte vector reductions (red.global.add.v4.f32).
#include <cuda_runtime.h>

#include "ops.h"
#include "pm_kernels.cuh"
#include "sgns_common.cuh"

namespace adapm {
namespace cudaops {

namespace {

constexpr int kThreads = 256;
using sgns::kMaxExp;

using dev::Target;
using dev::warp_sum;

__device__ __forceinline__ Target resolve_fast(const Ctx& c, Key key, unsigned* n_local, unsigned* n_remote) {
  return dev::resolve_fast(c, key, 0, n_local, n_remote);
}

using sgns::slow_target;

using dev::slow_pull;
using dev::slow_push;

// VPL = float4 vectors per lane covering d floats: VPL = ceil(d / 128)
// 2 blocks/SM: 128 registers and no spills (3 blocks/SM would cap the kernel at 80 registers, and it spills there)
template <int VPL>
__global__ void __launch_bounds__(kThreads, 2)
sgns_step_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ centers, const Key* __restrict__ contexts,
                 const Key* __restrict__ negatives, int n_pairs, int neg, int d, float alpha,
                 float* __restrict__ loss_out, unsigned long long* __restrict__ stats) {
  extern __shared__ float smem_f[];  // slow-path scratch: per warp 4*d floats
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int warp_in_block = threadIdx.x >> 5;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int nvec = d >> 2;  // float4 per half row
  float* stage = smem_f + (size_t)warp_in_block * 4 * d;
  float* e0s = stage + 2 * d;
  float* g0s = stage + 3 * d;
  float loss_acc = 0.f;
  unsigned n_local = 0, n_remote = 0, n_slow = 0, n_upd = 0;
  const int n_targets = neg + 1;

  for (int p = warp; p < n_pairs; p += nwarps) {
    const Key ckey = centers[p];
    const Key pos_key = contexts[p];
    // ---- resolve the center (lane 0) and the first 31 targets (lanes 1..31) in parallel:
    //      one dependent-load chain (slot -> state [-> peer slot -> peer state]) for all of them
    Key my_key = -1;
    Target my_t;
    my_t.row = nullptr; my_t.version = nullptr; my_t.flag = nullptr;
    if (lane == 0) my_key = ckey;
    else if (lane - 1 < n_targets) my_key = (lane == 1) ? pos_key : negatives[(size_t)p * neg + (lane - 2)];
    if (my_key >= 0) my_t = resolve_fast(c, my_key, &n_local, &n_remote);

    // ---- center row
    float* c_row = (float*)__shfl_sync(0xffffffffu, (unsigned long long)my_t.row, 0);
    const bool c_slow = (c_row == nullptr);
    bool have_slow = false;
    float4 e0[VPL], g0[VPL];
    if (c_slow) {
      ++n_slow;
      if (!slow_pull(c, ckey, stage)) continue;
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        int j = lane + v * 32;
        e0[v] = j < nvec ? reinterpret_cast<float4*>(stage)[j] : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      __syncwarp();
    } else {
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        int j = lane + v * 32;
        e0[v] = j < nvec ? dev::ld_row4(c_row + 4 * j) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int v = 0; v < VPL; ++v) g0[v] = make_float4(0.f, 0.f, 0.f, 0.f);

    // ---- targets
    for (int t = 0; t < n_targets; ++t) {
      Key tkey;
      float* t_row; uint32_t* t_ver; uint8_t* t_flag;
      if (t < 31) {
        tkey = (Key)__shfl_sync(0xffffffffu, (unsigned long long)my_key, t + 1);
        t_row = (float*)__shfl_sync(0xffffffffu, (unsigned long long)my_t.row, t + 1);
        t_ver = (uint32_t*)__shfl_sync(0xffffffffu, (unsigned long long)my_t.version, t + 1);
        t_flag = (uint8_t*)__shfl_sync(0xffffffffu, (unsigned long long)my_t.flag, t + 1);
      } else {  // more than 31 targets: resolve the rest one by one
        tkey = negatives[(size_t)p * neg + (t - 1)];
        Target tt;
        tt.row = nullptr; tt.version = nullptr; tt.flag = nullptr;
        if (lane == 0) tt = resolve_fast(c, tkey, &n_local, &n_remote);
        t_row = (float*)__shfl_sync(0xffffffffu, (unsigned long long)tt.row, 0);
        t_ver = (uint32_t*)__shfl_sync(0xffffffffu, (unsigned long long)tt.version, 0);
        t_flag = (uint8_t*)__shfl_sync(0xffffffffu, (unsigned long long)tt.flag, 0);
      }
      const float label = (t == 0) ? 1.f : 0.f;
      if (t > 0 && tkey == pos_key) continue;  // reference: negative == positive target is skipped

      if (t_row == nullptr) {
        // transitional key: out-of-line generic path through shared memory
        ++n_slow;
        if (!have_slow) {
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            int j = lane + v * 32;
            if (j < nvec) {
              reinterpret_cast<float4*>(e0s)[j] = e0[v];
              reinterpret_cast<float4*>(g0s)[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
          }
          __syncwarp();
          have_slow = true;
        }
        bool applied;
        loss_acc += slow_target(c, tkey, label, alpha, d, stage, e0s, g0s, &applied);
        if (applied) ++n_upd;
        continue;
      }

      float4 e1[VPL], a1[VPL];
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        int j = lane + v * 32;
        e1[v] = j < nvec ? dev::ld_row4(t_row + 4 * j) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        int j = lane + v * 32;
        a1[v] = j < nvec ? dev::ld_row4(t_row + d + 4 * j) : make_float4(1.f, 1.f, 1.f, 1.f);
      }
      float f = 0.f;
#pragma unroll
      for (int v = 0; v < VPL; ++v) f += e0[v].x * e1[v].x + e0[v].y * e1[v].y + e0[v].z * e1[v].z + e0[v].w * e1[v].w;
      f = warp_sum(f);
      float gs;
      if (f > kMaxExp) gs = label - 1.f;
      else if (f < -kMaxExp) gs = label;
      else gs = label - 1.f / (1.f + __expf(-f));
      {  // monitoring loss: -log sigmoid(+-f), clamped like the gradient
        float z = label > 0.5f ? f : -f;
        z = fminf(fmaxf(z, -kMaxExp), kMaxExp);
        loss_acc += __logf(1.f + __expf(-z));
      }
      // AdaGrad step for the target row (uses the pulled accumulator, like the reference) fused with
      // the push: 16-byte vector reductions into the owner's / replica's row
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        int j = lane + v * 32;
        g0[v].x += gs * e1[v].x; g0[v].y += gs * e1[v].y; g0[v].z += gs * e1[v].z; g0[v].w += gs * e1[v].w;
        float4 gr = make_float4(gs * e0[v].x, gs * e0[v].y, gs * e0[v].z, gs * e0[v].w);
        float4 ua = make_float4(gr.x * gr.x, gr.y * gr.y, gr.z * gr.z, gr.w * gr.w);
        float4 ue;
        ue.x = alpha * gr.x * rsqrtf(a1[v].x + ua.x);
        ue.y = alpha * gr.y * rsqrtf(a1[v].y + ua.y);
        ue.z = alpha * gr.z * rsqrtf(a1[v].z + ua.z);
        ue.w = alpha * gr.w * rsqrtf(a1[v].w + ua.w);
        if (j < nvec) { dev::red_row4(t_row + 4 * j, ue); dev::red_row4(t_row + d + 4 * j, ua); }
      }
      if (lane == 0) {
        if (t_ver) mem::red_add(t_ver, 1u);
        if (t_flag) *t_flag = (uint8_t)1;
      }
      ++n_upd;
    }

    // ---- center update
    if (have_slow) {
      __syncwarp();
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        int j = lane + v * 32;
        if (j < nvec) {
          float4 q = reinterpret_cast<float4*>(g0s)[j];
          g0[v].x += q.x; g0[v].y += q.y; g0[v].z += q.z; g0[v].w += q.w;
        }
      }
      __syncwarp();
    }
    if (c_slow) {
      // accumulator half of the center row is still in stage[d..2d) only if no slow target overwrote it:
      // re-pull to be safe, then push through the generic path
      if (slow_pull(c, ckey, stage)) {
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          int j = lane + v * 32;
          if (j < nvec) {
            float4 a0 = reinterpret_cast<float4*>(stage + d)[j];
            float4 ua = make_float4(g0[v].x * g0[v].x, g0[v].y * g0[v].y, g0[v].z * g0[v].z, g0[v].w * g0[v].w);
            float4 ue;
            ue.x = alpha * g0[v].x * rsqrtf(a0.x + ua.x);
            ue.y = alpha * g0[v].y * rsqrtf(a0.y + ua.y);
            ue.z = alpha * g0[v].z * rsqrtf(a0.z + ua.z);
            ue.w = alpha * g0[v].w * rsqrtf(a0.w + ua.w);
            reinterpret_cast<float4*>(stage)[j] = ue;
            reinterpret_cast<float4*>(stage + d)[j] = ua;
          }
        }
        if (slow_push(c, ckey, stage)) ++n_upd;
      }
    } else {
      uint32_t* c_ver = (uint32_t*)__shfl_sync(0xffffffffu, (unsigned long long)my_t.version, 0);
      uint8_t* c_flag = (uint8_t*)__shfl_sync(0xffffffffu, (unsigned long long)my_t.flag, 0);
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        int j = lane + v * 32;
        if (j < nvec) {
          float4 a0 = dev::ld_row4(c_row + d + 4 * j);
          float4 ua = make_float4(g0[v].x * g0[v].x, g0[v].y * g0[v].y, g0[v].z * g0[v].z, g0[v].w * g0[v].w);
          float4 ue;
          ue.x = alpha * g0[v].x * rsqrtf(a0.x + ua.x);
          ue.y = alpha * g0[v].y * rsqrtf(a0.y + ua.y);
          ue.z = alpha * g0[v].z * rsqrtf(a0.z + ua.z);
          ue.w = alpha * g0[v].w * rsqrtf(a0.w + ua.w);
          dev::red_row4(c_row + 4 * j, ue);
          dev::red_row4(c_row + d + 4 * j, ua);
        }
      }
      if (lane == 0) {
        if (c_ver) mem::red_add(c_ver, 1u);
        if (c_flag) *c_flag = (uint8_t)1;
      }
      ++n_upd;
    }
  }

  // ---- per-warp results
  __syncwarp();
  if (lane == 0 && loss_out) atomicAdd(loss_out, loss_acc);
  dev::flush_stats(stats, n_local, n_remote, n_slow, n_upd);
  dev::cta_exit(c);
}

}  // namespace

// keys are int64 device pointers; negatives has n_pairs*neg entries. loss_out (1 float) and
// stats (4 x u64: local rows, remote rows, slow-path rows, updates applied) are accumulated.
void sgns_step(CudaBackend& be, cudaStream_t stream, const Key* centers, const Key* contexts, const Key* negatives,
               int n_pairs, int neg, int d, float alpha, float* loss_out, unsigned long long* stats, int impl) {
  const Ctx& c = be.ctx();
  ADAPM_CHECK(c.L.num_classes == 1 && (int)c.L.cls[0].len == 2 * d, "sgns_step: store rows must be 2*embed_dim floats");
  ADAPM_CHECK(d % 4 == 0 && d <= 512, "sgns_step: embed_dim must be a multiple of 4 and <= 512");
  ADAPM_CHECK(neg >= 0, "sgns_step: negative must be >= 0");
  if (n_pairs == 0) return;
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  be.track_stream(stream);
  if ((impl == 0 || impl == 2) && sgns_step_tma(be, stream, centers, contexts, negatives, n_pairs, neg, d, alpha, loss_out, stats)) return;
  // auto falls back to the register kernel (in place, also on one GPU); an explicit tma request does not
  ADAPM_CHECK(impl != 2, "sgns_step: impl=\"tma\" takes embed_dim <= 336 and negative <= 30, got embed_dim "
                             << d << ", negative " << neg << " (impl=\"auto\" runs the in-place register kernel)");
  const int vpl = (d / 4 + 31) / 32;
  const int warps_per_block = kThreads / 32;
  int blocks = std::min((n_pairs + warps_per_block - 1) / warps_per_block, be.num_sms() * 8);
  size_t smem = (size_t)warps_per_block * 4 * d * sizeof(float);
#define ADAPM_LAUNCH_SGNS(V)                                                                             \
  do {                                                                                                   \
    set_max_dynamic_smem<sgns_step_kernel<V>>(96 * 1024);                                                \
    sgns_step_kernel<V><<<blocks, kThreads, smem, stream>>>(c, centers, contexts, negatives, n_pairs, neg, d, \
                                                           alpha, loss_out, stats);                     \
  } while (0)
  switch (vpl) {
    case 1: ADAPM_LAUNCH_SGNS(1); break;
    case 2: ADAPM_LAUNCH_SGNS(2); break;
    case 3: ADAPM_LAUNCH_SGNS(3); break;
    default: ADAPM_LAUNCH_SGNS(4); break;
  }
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

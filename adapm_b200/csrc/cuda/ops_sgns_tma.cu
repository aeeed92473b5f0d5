// SGNS step, TMA-prefetch variant (sm_90a): same semantics as ops_sgns.cu, but the target rows of a
// pair stream through a per-warp shared-memory ring that is filled by the TMA engine
// (cp.async.bulk global -> shared, completion on an mbarrier) several targets ahead of the math.
//
// Why: the LDG variant keeps one target (2 x 1200 B per warp) in flight per warp and is register
// limited to 16 warps/SM -> ~48 KB in flight per SM, latency bound (ncu: DRAM 42 %, L2 49 %).
// Here rows never occupy registers while in flight: 16 warps/SM x RING (4) rows x 2400 B = 150 KB per SM.
//   lane 0      : mbarrier.arrive.expect_tx + cp.async.bulk (UBLKCP) for target t + RING - 1
//   whole warp  : mbarrier.try_wait, LDS.128 the row from shared memory, dot / sigmoid / AdaGrad,
//                 the update overwrites the consumed ring slot
//   lane 0      : cp.reduce.async.bulk (UBLKRED) of that slot into the row's home (local HBM or NVLink peer)
// The deterministic one-GPU step (sgns_step_det) runs the same body as a score pass that loads only the targets'
// embedding halves and writes no row, then groups the step's contributions by key and lets one warp per row gather them
// as fixed-point integer sums.
// The TMA engine reads rows that live on a peer GPU through their NVLink-mapped addresses as well;
// rows in a transitional protocol state take the generic out-of-line path.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>

#include <cub/cub.cuh>

#include "fx_accum.cuh"
#include "ops.h"
#include "pm_kernels.cuh"
#include "sgns_common.cuh"

namespace adapm {
namespace cudaops {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int RING = 4;
using sgns::kMaxExp;

using dev::Target;
using dev::warp_sum;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
  } while (!ok);
}
// 1-D bulk copy global -> shared through the TMA engine; completes `bytes` on the mbarrier
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// Bulk reduction shared -> global through the TMA engine (cp.reduce.async.bulk ... add.f32): ONE instruction adds a whole
// staged row (element-wise atomic at the row's home L2, local HBM or NVLink peer) instead of row_bytes / 16 RED.128
// issued by the warp. Completion is tracked with bulk async-groups of the issuing thread.
__device__ __forceinline__ void bulk_red_s2g(float* dst, const void* src, uint32_t bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;"
               ::"l"(dst), "r"(smem_u32(src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() {   // all but the N youngest groups have read their source
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// dev::mark_pushed on the packed (mark pointer, kind bit) form of a Target
__device__ __forceinline__ void mark_pushed(void* mark, int bits) {
  if (!mark) return;
  if (bits & 2) *static_cast<uint8_t*>(mark) = (uint8_t)1;
  else mem::red_add(static_cast<uint32_t*>(mark), 1u);
}

// Deterministic step (one GPU): every contribution is rounded to fixed point, |embedding update| <= alpha per
// contribution (AdaGrad normalises it), AdaGrad increments are squared gradients: 2^40 / 2^36 leave 2^23 / 2^27 of range
// per element and step. The loss is a fixed-point sum too: 2^32 leaves 2^31 of summed loss per step.
constexpr float kFxEmb = 1099511627776.f;     // 2^40
constexpr float kFxAda = 68719476736.f;       // 2^36
constexpr float kFxLoss = 4294967296.f;       // 2^32
// Entry x = p * (neg + 2) + s of a step: s = 0 the center of pair p, s = 1 its context, s >= 2 negative s - 2.
// gs[x] of an entry that adds nothing (negative == context, generic-path target or center, skipped pair). A real gs is
// in [-1, 1] or NaN; 0 is a real gs (and a center entry's "valid" mark), so it cannot be the marker.
constexpr float kNoEntry = __builtin_huge_valf();

// What the score pass (SCORE) of the deterministic step writes for the gather pass besides gs and the loss (the
// step body takes those as separate arguments).
struct ScoreOut {
  float* g0;                     // [n_pairs x d] the pair's center gradient
  float* snap;                   // [distinct centers x d] start-of-step embedding of each center, by compact id
                                 // (the deterministic step keeps it right after g0 in one buffer)
  int* pcid;                     // [n_pairs] compact id of the pair's center
};

struct WarpSmem {
  unsigned long long bar[RING];
};

// VPL = float4 per lane over d floats. MAXREG is the register budget: the kernel runs 2 blocks of 256 threads per SM;
// 128 registers use the whole register file, 104 leave 12 K registers per SM free so that one block of the
// sync-round kernels (40 registers x 256 threads) can be co-resident instead of waiting for a step block to retire.
// (A variant that summed rows whose relocation to this rank is in flight inside the kernel - local row + source row -
// instead of taking the out-of-line generic path for them was measured on 2 GPUs and removed: no gain, 2 x the
// instantiations.)
// In place (BULK): the updates of a target leave as ONE TMA bulk reduction per row: the warp overwrites the consumed ring
// slot with [embedding update | AdaGrad update] and lane 0 issues cp.reduce.async.bulk from it; the slot is reloaded one
// target later, after the reduction has read it (prefetch distance RING - 1).
// SCORE: score pass of the deterministic one-GPU step (sgns_score_tma_kernel, its own kernel so that the in-place
// variants keep their register allocation). It reads start-of-step rows only - the embedding half of each target - and
// writes no store row: per pair the center gradient g0, per target gs, and each center's embedding (ScoreOut). The
// gather pass forms and applies every row's update from these.
template <int VPL, bool SCORE>
__device__ __forceinline__ void
sgns_step_tma_body(const Ctx& c, const Key* __restrict__ centers, const Key* __restrict__ contexts,
                   const Key* __restrict__ negatives, int n_pairs, int neg, int d, float alpha,
                   float* __restrict__ loss_out, unsigned long long* __restrict__ stats,
                   const int* __restrict__ cidx, float* __restrict__ gs_buf, unsigned long long* __restrict__ fx_loss,
                   const ScoreOut& so) {
  constexpr bool BULK = !SCORE;
  // per warp: RING row buffers of 2*d floats (16-byte aligned) | generic-path scratch is carved from the ring
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ WarpSmem wsm[kWarps];
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int warp = blockIdx.x * kWarps + wib;       // launched with kThreads threads: the compile-time warp count lets
  const int nwarps = gridDim.x * kWarps;             // ptxas rematerialise the grid stride instead of spilling it
  const int nvec = d >> 2;
  const uint32_t row_bytes = (uint32_t)(2 * d * sizeof(float));
  const uint32_t load_bytes = SCORE ? (uint32_t)(d * sizeof(float)) : row_bytes;   // SCORE: embedding half only
  const size_t buf_floats = ((size_t)2 * d + 31) & ~(size_t)31;  // keep every ring slot 128-byte aligned
  float* ring = reinterpret_cast<float*>(smem_raw) + (size_t)wib * (RING + 1) * buf_floats;
  float* scratch = ring + (size_t)RING * buf_floats;             // e0s | g0s for the generic path (2*d floats)
  unsigned long long* bars = wsm[wib].bar;
  if (lane == 0) {
    for (int r = 0; r < RING; ++r) mbar_init(&bars[r], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncwarp();
  uint32_t issued = 0, consumed = 0;   // ring counters (buffer = n % RING, phase parity = (n / RING) & 1)
  float loss_acc = 0.f;
  unsigned n_local = 0, n_remote = 0, n_slow = 0, n_upd = 0;
  const int n_targets = neg + 1;

  for (int p = warp; p < n_pairs; p += nwarps) {
    const Key ckey = centers[p];
    const Key pos_key = contexts[p];
    // ---- resolve center (lane 0) + up to 31 targets (lanes 1..31) with one dependent-load chain
    Key my_key = -1;
    // what this lane resolved: the row, and what marks a completed push of it - resolve_fast sets at most one of the
    // version counter (owned row) and the dirty byte (replica), so one pointer + a kind bit hold it (frees registers)
    float* my_row = nullptr;
    void* my_mark = nullptr;
    int my_bits = 0;                     // bit 1: my_mark is a replica dirty byte,
                                         // bits 2..: the center's compact id (SCORE, lane 0)
    if (lane == 0) my_key = ckey;
    else if (lane - 1 < n_targets) my_key = (lane == 1) ? pos_key : negatives[(size_t)p * neg + (lane - 2)];
    if (my_key >= 0) {
      const Target tg = dev::resolve_fast(c, my_key, 0, &n_local, &n_remote);
      my_row = tg.row;
      my_mark = tg.flag ? (void*)tg.flag : (void*)tg.version;
      my_bits = (tg.flag ? 2 : 0) | (SCORE && lane == 0 ? __ldg(cidx + my_key) << 2 : 0);
    }
    // target t (0-based) -> lane t+1 (only pairs with <= 31 targets use this kernel)
    auto issue = [&](int t) {
      const int b = issued % RING;
      float* buf = ring + (size_t)b * buf_floats;
      const Key tkey = (Key)__shfl_sync(0xffffffffu, (unsigned long long)my_key, t + 1);
      float* row = (float*)__shfl_sync(0xffffffffu, (unsigned long long)my_row, t + 1);
      const bool skip = (t > 0 && tkey == pos_key) || row == nullptr;
      if (skip) {
        if (lane == 0) mbar_arrive(&bars[b]);            // nothing to load: complete the phase
      } else if (lane == 0) {
        // local HBM row - or a peer's row: the TMA engine reads NVLink-mapped addresses as well
        if (BULK) bulk_wait_read<1>();   // the reduction that used this slot (issued one target ago) has read it
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // order earlier LDS of this slot before the TMA write
        mbar_expect_tx(&bars[b], load_bytes);
        bulk_g2s(buf, row, load_bytes, &bars[b]);
      }
      ++issued;
    };

    // ---- center row (registers)
    float* c_row = (float*)__shfl_sync(0xffffffffu, (unsigned long long)my_row, 0);
    const bool c_slow = (c_row == nullptr);
    float4 e0[VPL], g0[VPL];
    // prefetch the first RING (BULK: RING - 1) targets before touching the center row
    constexpr int DIST = BULK ? RING - 1 : RING;
    if (BULK) { if (lane == 0) bulk_wait_read<0>(); __syncwarp(); }   // the previous pair's reductions have read ring + scratch
    const int pre = n_targets < DIST ? n_targets : DIST;
    for (int t = 0; t < pre; ++t) issue(t);
    if (c_slow) {
      ++n_slow;
      if (!dev::slow_pull(c, ckey, scratch)) {
        // drain the ring so that the barrier phases stay in step, then skip the pair
        for (int t = 0; t < pre; ++t) { mbar_wait(&bars[consumed % RING], (consumed / RING) & 1u); ++consumed; }
        for (int t = pre; t < n_targets; ++t) { issue(t); mbar_wait(&bars[consumed % RING], (consumed / RING) & 1u); ++consumed; }
        (void)DIST;
        if (SCORE) for (int s = lane; s < neg + 2; s += 32) gs_buf[(size_t)p * (neg + 2) + s] = kNoEntry;
        continue;
      }
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        int j = lane + v * 32;
        e0[v] = j < nvec ? reinterpret_cast<float4*>(scratch)[j] : make_float4(0.f, 0.f, 0.f, 0.f);
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
    bool have_slow = false;
    if (SCORE) {                           // the center's start-of-step embedding, for the gather pass
      const int cid = __shfl_sync(0xffffffffu, my_bits, 0) >> 2;
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        int j = lane + v * 32;
        if (j < nvec) reinterpret_cast<float4*>(so.snap + (size_t)cid * d)[j] = e0[v];
      }
      if (lane == 0) so.pcid[p] = cid;
    }

    // ---- targets
    for (int t = 0; t < n_targets; ++t) {
      const int b = consumed % RING;
      float* buf = ring + (size_t)b * buf_floats;
      const Key tkey = (Key)__shfl_sync(0xffffffffu, (unsigned long long)my_key, t + 1);
      float* t_row = (float*)__shfl_sync(0xffffffffu, (unsigned long long)my_row, t + 1);
      mbar_wait(&bars[b], (consumed / RING) & 1u);
      ++consumed;
      const float label = (t == 0) ? 1.f : 0.f;
      const bool dup = (t > 0 && tkey == pos_key);  // reference: negative == positive target is skipped
      float gs_out = kNoEntry;                       // SCORE: what the gather pass adds for this target
      if (!dup && t_row == nullptr) {
        ++n_slow;
        float* e0s = scratch; float* g0s = scratch + d;
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
        loss_acc += sgns::slow_target(c, tkey, label, alpha, d, buf, e0s, g0s, &applied);  // ring slot b is free: use it as stage
        if (applied) ++n_upd;
      } else if (!dup) {
        float4 e1[VPL];
        float f = 0.f;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          int j = lane + v * 32;
          e1[v] = j < nvec ? reinterpret_cast<const float4*>(buf)[j] : make_float4(0.f, 0.f, 0.f, 0.f);
          f += e0[v].x * e1[v].x + e0[v].y * e1[v].y + e0[v].z * e1[v].z + e0[v].w * e1[v].w;
        }
        f = warp_sum(f);
        float gs;
        if (f > kMaxExp) gs = label - 1.f;
        else if (f < -kMaxExp) gs = label;
        else gs = label - 1.f / (1.f + __expf(-f));
        {
          float z = label > 0.5f ? f : -f;
          z = fminf(fmaxf(z, -kMaxExp), kMaxExp);
          loss_acc += __logf(1.f + __expf(-z));
        }
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          int j = lane + v * 32;
          if (j < nvec) {
            if (SCORE) {                  // the gather pass forms the target's update from gs
              g0[v].x += gs * e1[v].x; g0[v].y += gs * e1[v].y; g0[v].z += gs * e1[v].z; g0[v].w += gs * e1[v].w;
              continue;
            }
            float4 a1 = reinterpret_cast<const float4*>(buf + d)[j];
            g0[v].x += gs * e1[v].x; g0[v].y += gs * e1[v].y; g0[v].z += gs * e1[v].z; g0[v].w += gs * e1[v].w;
            float4 gr = make_float4(gs * e0[v].x, gs * e0[v].y, gs * e0[v].z, gs * e0[v].w);
            float4 ua = make_float4(gr.x * gr.x, gr.y * gr.y, gr.z * gr.z, gr.w * gr.w);
            float4 ue;
            ue.x = alpha * gr.x * rsqrtf(a1.x + ua.x);
            ue.y = alpha * gr.y * rsqrtf(a1.y + ua.y);
            ue.z = alpha * gr.z * rsqrtf(a1.z + ua.z);
            ue.w = alpha * gr.w * rsqrtf(a1.w + ua.w);
            // stage the update in place of the consumed row
            reinterpret_cast<float4*>(buf)[j] = ue;
            reinterpret_cast<float4*>(buf + d)[j] = ua;
          }
        }
        gs_out = gs;
        if (BULK) {
          __syncwarp();
          if (lane == 0) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the staged update is visible to the TMA engine
            bulk_red_s2g(t_row, buf, row_bytes);
          }
        }
        if (lane == t + 1) mark_pushed(my_mark, my_bits);
        ++n_upd;
      }
      if (SCORE && lane == 0) gs_buf[(size_t)p * (neg + 2) + 1 + t] = gs_out;
      // exactly one bulk group per target (empty for skipped / generic-path targets): "all but the youngest group"
      // below always means "the reduction that used the slot of the previous target"
      if (BULK && lane == 0) bulk_commit();
      __syncwarp();                       // all lanes are done reading ring slot b
      if (t + DIST < n_targets) issue(t + DIST);
    }

    // ---- center update
    if (have_slow) {
      const float* g0s = scratch + d;
      __syncwarp();
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        int j = lane + v * 32;
        if (j < nvec) {
          float4 q = reinterpret_cast<const float4*>(g0s)[j];
          g0[v].x += q.x; g0[v].y += q.y; g0[v].z += q.z; g0[v].w += q.w;
        }
      }
      __syncwarp();
    }
    if (c_slow) {
      float* stage = ring;  // every ring slot is free here; 2*d floats needed
      if (dev::slow_pull(c, ckey, stage)) {
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
        if (dev::slow_push(c, ckey, stage)) ++n_upd;
      }
      if (SCORE && lane == 0) gs_buf[(size_t)p * (neg + 2)] = kNoEntry;
    } else if (SCORE) {                   // the gather pass applies g0 to the center row
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        int j = lane + v * 32;
        if (j < nvec) reinterpret_cast<float4*>(so.g0 + (size_t)p * d)[j] = g0[v];
      }
      if (lane == 0) gs_buf[(size_t)p * (neg + 2)] = 0.f;
      if (lane == 0) mark_pushed(my_mark, my_bits);
      ++n_upd;
    } else {
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
          reinterpret_cast<float4*>(scratch)[j] = ue;
          reinterpret_cast<float4*>(scratch + d)[j] = ua;
        }
      }
      if (BULK) {
        __syncwarp();
        if (lane == 0) {
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          bulk_red_s2g(c_row, scratch, row_bytes);
          bulk_commit();
        }
      }
      if (lane == 0) mark_pushed(my_mark, my_bits);
      ++n_upd;
    }
    __syncwarp();
  }
  if (BULK) { if (lane == 0) bulk_wait_all(); __syncwarp(); }   // every bulk reduction has been performed before the CTA leaves

  __syncwarp();
  if (SCORE && lane == 0) atomicAdd(fx_loss, (unsigned long long)__float2ll_rn(loss_acc * kFxLoss));
  else if (lane == 0 && loss_out) atomicAdd(loss_out, loss_acc);
  unsigned sum_local = n_local, sum_remote = n_remote;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum_local += __shfl_xor_sync(0xffffffffu, sum_local, o);
    sum_remote += __shfl_xor_sync(0xffffffffu, sum_remote, o);
  }
  if (lane == 0 && stats) {
    if (sum_local) atomicAdd(stats + 0, (unsigned long long)sum_local);
    if (sum_remote) atomicAdd(stats + 1, (unsigned long long)sum_remote);
    if (n_slow) atomicAdd(stats + 2, (unsigned long long)n_slow);
    if (n_upd) atomicAdd(stats + 3, (unsigned long long)n_upd);
  }
  dev::cta_exit(c);
}

template <int VPL, int MAXREG>
__global__ void __maxnreg__(MAXREG)
sgns_step_tma_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ centers, const Key* __restrict__ contexts,
                     const Key* __restrict__ negatives, int n_pairs, int neg, int d, float alpha,
                     float* __restrict__ loss_out, unsigned long long* __restrict__ stats) {
  sgns_step_tma_body<VPL, false>(c, centers, contexts, negatives, n_pairs, neg, d, alpha, loss_out, stats, nullptr,
                                 nullptr, nullptr, ScoreOut{});
}

template <int VPL>
__global__ void __maxnreg__(128)
sgns_score_tma_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ centers, const Key* __restrict__ contexts,
                      const Key* __restrict__ negatives, int n_pairs, int neg, int d, float alpha,
                      unsigned long long* __restrict__ stats, const int* __restrict__ cidx,
                      float* __restrict__ gs_buf, unsigned long long* __restrict__ fx_loss,
                      const __grid_constant__ ScoreOut so) {
  // (cidx, gs_buf and fx_loss are restrict arguments as the in-place kernel's are: the same alias scopes keep the
  // in-place instantiations' code unchanged)
  sgns_step_tma_body<VPL, true>(c, centers, contexts, negatives, n_pairs, neg, d, alpha, nullptr, stats, cidx, gs_buf,
                                fx_loss, so);
}

// ---- deterministic one-GPU step: index, score, group by key, gather
// The contributions of a step are grouped by key (CSR: off / list / kid), so that each row is updated by the one warp
// that owns it and no accumulator per key and element is needed. Integer sums do not depend on the order of their
// terms, so the grouping may differ from run to run and the rows and loss do not.

__device__ __forceinline__ Key entry_key(const Key* centers, const Key* contexts, const Key* negatives, int neg, int p,
                                         int s) {
  return s == 0 ? centers[p] : (s == 1 ? contexts[p] : negatives[(size_t)p * neg + (s - 2)]);
}
// a negative equal to the pair's context adds nothing (the step skips it); neither does a negative key
__device__ __forceinline__ bool entry_counts(const Key* contexts, int p, int s, Key k) {
  return k >= 0 && !(s >= 2 && k == contexts[p]);
}

// the key's row in this GPU's store (one GPU: rows do not move during a step)
__device__ __forceinline__ float* home_row(const Ctx& c, Key k) {
  const int32_t slot = __ldcg(slot_of(c, c.rank) + k);
  return slot >= 0 ? row_ptr<float>(c, c.rank, class_of_key(c, k), (uint32_t)slot) : nullptr;
}

// Gives every key of slots [first_slot, first_slot + n_slots) of each pair a compact id (cidx[key], keys[id]) and
// looks its row up once (rowp[id]). Run over the centers first, so that the centers' ids are 0 .. distinct centers - 1.
__global__ void sgns_det_index_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ centers,
                                      const Key* __restrict__ contexts, const Key* __restrict__ negatives, int n_pairs,
                                      int neg, int first_slot, int n_slots, int* __restrict__ cidx,
                                      Key* __restrict__ keys, float** __restrict__ rowp,
                                      unsigned int* __restrict__ count) {
  const long n = (long)n_pairs * n_slots;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int p = (int)(i / n_slots), s = first_slot + (int)(i % n_slots);
    const Key k = entry_key(centers, contexts, negatives, neg, p, s);
    // (the plain load skips the atomic for keys that are already claimed: hot keys appear thousands of times)
    if (k >= 0 && cidx[k] == -1 && atomicCAS(cidx + k, -1, -2) == -1) {
      const unsigned r = atomicAdd(count, 1u);
      keys[r] = k;
      rowp[r] = home_row(c, k);
      cidx[k] = (int)r;
    }
  }
}

// What one contribution (CSR position) adds to its key's row: g times vector vec of the step's vector buffer, which holds
// the pairs' center gradients g0 (rows 0 .. n_pairs - 1) followed by the centers' start-of-step embeddings (rows
// n_pairs + compact id). g is 1 for a center (its gradient is g0 itself), gs for a target, kNoEntry for nothing.
struct alignas(8) GatherDesc {
  float g;
  int vec;
};

// SCATTER = false: cnt[id] = entries of key id. SCATTER = true: desc / kid of CSR position off[id] + i, i < cnt[id],
// describe the entries of key id (from the score pass's gs and pcid); counts cnt back down to zero.
template <bool SCATTER>
__global__ void sgns_det_group_kernel(const Key* __restrict__ centers, const Key* __restrict__ contexts,
                                      const Key* __restrict__ negatives, int n_pairs, int neg,
                                      const int* __restrict__ cidx, int* __restrict__ cnt, const int* __restrict__ off,
                                      int* __restrict__ kid, const float* __restrict__ gsb,
                                      const int* __restrict__ pcid, GatherDesc* __restrict__ desc) {
  const int n = n_pairs * (neg + 2);
  for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < n; x += gridDim.x * blockDim.x) {
    const int p = x / (neg + 2), s = x - p * (neg + 2);
    const Key k = entry_key(centers, contexts, negatives, neg, p, s);
    if (!entry_counts(contexts, p, s, k)) continue;
    const int id = __ldg(cidx + k);
    if (!SCATTER) {
      atomicAdd(cnt + id, 1);
    } else {
      const int q = __ldg(off + id) + atomicSub(cnt + id, 1) - 1;
      const float gx = __ldg(gsb + x);
      GatherDesc e;
      if (s == 0) {
        e.g = gx == kNoEntry ? kNoEntry : 1.f;
        e.vec = p;
      } else {
        e.g = gx;
        e.vec = gx == kNoEntry ? 0 : n_pairs + __ldg(pcid + p);
      }
      desc[q] = e;
      kid[q] = id;
    }
  }
}

// The fixed-point terms of one element of one contribution (gr = gs * e0 of a target, g0 of a center; a = the row's
// AdaGrad value at the start of the step), with the expressions of the in-place step.
__device__ __forceinline__ void fx_terms(float gr, float a, float alpha, long long& se, long long& sa) {
  const float ua = gr * gr;
  const float ue = alpha * gr * rsqrtf(a + ua);
  se += __float2ll_rn(ue * kFxEmb);
  sa += __float2ll_rn(ua * kFxAda);
}

// Gather pass: warp w works on CSR positions [w R, (w + 1) R). A key with at most R entries ("light") belongs wholly to
// the warp whose range holds its first entry, which adds its sums to the row (one writer per row). A longer ("heavy")
// key is shared by the warps whose ranges it spans: each adds its int64 partial sums to the key's partial row - the
// one of the first range boundary inside the key's entries - and sgns_det_finish_kernel applies it.
// Within each half of a partial row, element 4j + c sits at c * d/4 + j (fx::pos), so a warp's atomics are contiguous.
//
// The warp first finds all keys of its range at once: the CSR is ordered by compact id, so a lane per position sees
// where a key starts, and the keys' extents and rows are looked up together. It stages them and the range's entry
// descriptors in shared memory. Rows and vectors then stream through two per-warp rings that the TMA engine fills
// (cp.async.bulk, completion on an mbarrier) ahead of the math, as in the score pass: while the warp sums one key, the
// rows of the next kGatherRows - 1 keys and the vectors of the next kGatherVecs entries are in flight. A light key's
// update is written back from registers.
// Little's law at d = 300 (2400-byte rows, 1200-byte vectors): 2 rows + 4 vectors = 9.6 KB in flight per warp, and
// 16 warps per SM (2 blocks of 256 threads, 110 KB of shared memory and at most 128 registers each) keep about 150 KB
// in flight per SM, 77 KB of it rows from HBM; 3.35 TB/s over 132 SMs needs about 25 KB per microsecond of latency.
// Two blocks fit per SM up to d = 308; wider rows (up to d = 336, the widest the deterministic step takes) run one.
constexpr int kGatherRange = 64;
constexpr int kGatherRows = 3;                   // row ring slots
constexpr int kGatherVecs = 4;                   // vector ring slots
constexpr int kGatherDescs = 2 * kGatherRange;   // staged descriptors: the range and the rest of its last light key

// shared memory of one gather warp: row ring | vector ring | descriptors | per key: row, start if heavy, end
__host__ __device__ constexpr size_t gather_warp_bytes(int d) {
  return ((size_t)kGatherRows * 2 * d + (size_t)kGatherVecs * d) * sizeof(float) + kGatherDescs * sizeof(GatherDesc) +
         kGatherRange * (sizeof(float*) + 2 * sizeof(int));
}

template <int VPL>
__global__ void __launch_bounds__(256, 2)
sgns_det_gather_kernel(const __grid_constant__ Ctx c, float* const* __restrict__ rowp, const int* __restrict__ off,
                       int n_ids, const int* __restrict__ kid, const GatherDesc* __restrict__ desc,
                       const float* __restrict__ vecs, int d, float alpha, long long* __restrict__ part) {
  constexpr int R = kGatherRange, NR = kGatherRows, NV = kGatherVecs;
  constexpr unsigned kAll = 0xffffffffu;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ unsigned long long bars[kWarps][NR + NV];
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int nvec = d >> 2;
  const int total = off[n_ids];
  const int q0 = (int)(blockIdx.x * kWarps + wib) * R;
  if (q0 < total) {
    const int q1 = min(q0 + R, total);
    float* rring = reinterpret_cast<float*>(smem_raw + (size_t)wib * gather_warp_bytes(d));
    float* vring = rring + (size_t)NR * 2 * d;
    GatherDesc* dsm = reinterpret_cast<GatherDesc*>(vring + (size_t)NV * d);   // dsm[i]: CSR position q0 + i
    float** krow = reinterpret_cast<float**>(dsm + kGatherDescs);              // key k of the warp: its row,
    int* kheavy = reinterpret_cast<int*>(krow + R);                            // its first entry if heavy, else -1,
    int* kend = kheavy + R;                                                    // and the end of its entries here
    unsigned long long* rbar = bars[wib];
    unsigned long long* vbar = rbar + NR;
    if (lane == 0) {
      for (int r = 0; r < NR + NV; ++r) mbar_init(&rbar[r], 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }

    // ---- the keys of the range: lane l looks at positions q0 + l and q0 + 32 + l
    const int ida = q0 + lane < q1 ? __ldg(kid + q0 + lane) : -1;
    const int idb = q0 + 32 + lane < q1 ? __ldg(kid + q0 + 32 + lane) : -1;
    for (int i = lane; i < kGatherDescs && q0 + i < total; i += 32) dsm[i] = desc[q0 + i];
    const int prev_a = __shfl_up_sync(kAll, ida, 1), last_a = __shfl_sync(kAll, ida, 31);
    const int prev_b = __shfl_up_sync(kAll, idb, 1);
    // a key that starts at this position: its row, where its entries end in this warp, its first entry if heavy;
    // false for the rest of a light key that an earlier range owns
    auto key_at = [&](int id, bool start, float*& row, int& end, int& heavy_start) {
      if (!start) return false;
      const int s = __ldg(off + id), e = __ldg(off + id + 1);
      row = rowp[id];
      const bool heavy = e - s > R;
      end = heavy ? min(e, q1) : e;
      heavy_start = heavy ? s : -1;
      return heavy || s >= q0;
    };
    float *row_a = nullptr, *row_b = nullptr;
    int end_a = 0, end_b = 0, hs_a = -1, hs_b = -1;
    const bool in_a = key_at(ida, ida >= 0 && (lane == 0 || ida != prev_a), row_a, end_a, hs_a);
    const bool in_b = key_at(idb, idb >= 0 && idb != (lane == 0 ? last_a : prev_b), row_b, end_b, hs_b);
    const int qa = __shfl_sync(kAll, in_a ? q0 : end_a, 0);   // the first entry of the warp's first key
    const unsigned ma = __ballot_sync(kAll, in_a), mb = __ballot_sync(kAll, in_b);
    const unsigned below = (1u << lane) - 1u;
    const int nk = __popc(ma) + __popc(mb);
    if (in_a) {
      const int k = __popc(ma & below);
      krow[k] = row_a; kheavy[k] = hs_a; kend[k] = end_a;
    }
    if (in_b) {
      const int k = __popc(ma) + __popc(mb & below);
      krow[k] = row_b; kheavy[k] = hs_b; kend[k] = end_b;
    }
    __syncwarp();

    if (nk > 0) {
      // entries i = 0 .. ne - 1 of the warp are CSR positions qa + i, key after key
      const int ne = kend[nk - 1] - qa;
      const GatherDesc* dw = dsm + (qa - q0);
      auto issue_row = [&](int k) {      // the row of key k into row slot k % NR (a heavy key: its AdaGrad half only)
        if (lane != 0) return;
        const int b = k % NR;
        const float* row = krow[k];
        if (!row) {
          mbar_arrive(&rbar[b]);           // nothing to load: complete the phase
          return;
        }
        const int h = kheavy[k] >= 0 ? d : 0;
        const uint32_t bytes = (uint32_t)((2 * d - h) * sizeof(float));
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // earlier LDS of the slot before the TMA write
        mbar_expect_tx(&rbar[b], bytes);
        bulk_g2s(rring + (size_t)b * 2 * d + h, row + h, bytes, &rbar[b]);
      };
      auto issue_vec = [&](int i) {      // the vector of entry i into vector slot i % NV
        if (lane != 0) return;
        const int b = i % NV;
        const GatherDesc e = dw[i];
        if (e.g == kNoEntry) {
          mbar_arrive(&vbar[b]);
          return;
        }
        const uint32_t bytes = (uint32_t)(d * sizeof(float));
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_expect_tx(&vbar[b], bytes);
        bulk_g2s(vring + (size_t)b * d, vecs + (size_t)e.vec * d, bytes, &vbar[b]);
      };
      for (int k = 0; k < min(nk, NR); ++k) issue_row(k);
      for (int i = 0; i < min(ne, NV); ++i) issue_vec(i);

      int i = 0;
      for (int k = 0; k < nk; ++k) {
        const int b = k % NR;
        const float* rs = rring + (size_t)b * 2 * d;
        float* row = krow[k];
        const int heavy_start = kheavy[k];
        const int ie_end = kend[k] - qa;
        mbar_wait(&rbar[b], (uint32_t)(k / NR) & 1u);
        float4 a[VPL];
        long long se[VPL][4], sa[VPL][4];
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int j = lane + v * 32;
          a[v] = (j < nvec && row) ? reinterpret_cast<const float4*>(rs + d)[j] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int q = 0; q < 4; ++q) se[v][q] = sa[v][q] = 0;
        }
        for (; i < ie_end; ++i) {
          const int vb = i % NV;
          const float g = dw[i].g;
          mbar_wait(&vbar[vb], (uint32_t)(i / NV) & 1u);
          if (g != kNoEntry) {
            const float4* vs = reinterpret_cast<const float4*>(vring + (size_t)vb * d);
#pragma unroll
            for (int v = 0; v < VPL; ++v) {
              const int j = lane + v * 32;
              if (j < nvec) {
                const float4 ev = vs[j];
                fx_terms(g * ev.x, a[v].x, alpha, se[v][0], sa[v][0]);
                fx_terms(g * ev.y, a[v].y, alpha, se[v][1], sa[v][1]);
                fx_terms(g * ev.z, a[v].z, alpha, se[v][2], sa[v][2]);
                fx_terms(g * ev.w, a[v].w, alpha, se[v][3], sa[v][3]);
              }
            }
          }
          __syncwarp();                    // every lane has read vector slot vb
          if (i + NV < ne) issue_vec(i + NV);
        }
        if (heavy_start >= 0) {
          unsigned long long* pr = reinterpret_cast<unsigned long long*>(part + (size_t)(heavy_start / R + 1) * (2 * d));
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            const int j = lane + v * 32;
            if (j < nvec) {
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                if (se[v][q]) atomicAdd(pr + q * nvec + j, (unsigned long long)se[v][q]);
                if (sa[v][q]) atomicAdd(pr + d + q * nvec + j, (unsigned long long)sa[v][q]);
              }
            }
          }
        } else if (row) {
          // row += sum / scale; a zero sum leaves the element as it is (a -0.0 stays -0.0)
          const double ie = 1.0 / (double)kFxEmb, ia = 1.0 / (double)kFxAda;
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            const int j = lane + v * 32;
            if (j < nvec) {
              float4 r = reinterpret_cast<const float4*>(rs)[j];
              float4 na = a[v];
              float* rp = &r.x;
              float* ap = &na.x;
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                if (se[v][q]) rp[q] += (float)((double)se[v][q] * ie);
                if (sa[v][q]) ap[q] += (float)((double)sa[v][q] * ia);
              }
              reinterpret_cast<float4*>(row)[j] = r;
              reinterpret_cast<float4*>(row + d)[j] = na;
            }
          }
        }
        __syncwarp();                      // every lane has read row slot b
        if (k + NR < nk) issue_row(k + NR);
      }
    }
  }
  dev::cta_exit(c);
}

// After the gather pass: adds the partial rows of the heavy keys to their rows and clears them, gives every key of the
// step its id -1 back, and moves the step's fixed-point loss into loss_out (block 0).
__global__ void sgns_det_finish_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ keys,
                                       float* const* __restrict__ rowp,
                                       const int* __restrict__ off, int n_ids, const int* __restrict__ kid, int d,
                                       long long* __restrict__ part, int* __restrict__ cidx,
                                       const unsigned int* __restrict__ count, unsigned long long* __restrict__ fx_loss,
                                       float* __restrict__ loss_out) {
  constexpr int R = kGatherRange;
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const long long v = (long long)*fx_loss;
    *fx_loss = 0ull;
    if (loss_out) *loss_out += (float)((double)v / (double)kFxLoss);
  }
  const unsigned n_keys = *count;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n_keys; i += gridDim.x * blockDim.x) cidx[keys[i]] = -1;
  const int total = off[n_ids];
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int b = 1 + (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); b * R < total; b += nwarps) {
    const int id = kid[b * R];
    const int s = off[id], e = off[id + 1];
    if (e - s <= R || s / R + 1 != b) continue;     // not the first boundary inside a heavy key
    float* row = rowp[id];
    long long* pr = part + (size_t)b * (2 * d);
    for (int hf = 0; hf < 2; ++hf) {
      const double inv = 1.0 / (double)(hf ? kFxAda : kFxEmb);
      for (int i = lane; i < d; i += 32) {
        const long long v = pr[(size_t)hf * d + i];
        if (v) {
          if (row) row[(size_t)hf * d + fx::elem(i, d)] += (float)((double)v * inv);
          pr[(size_t)hf * d + i] = 0;
        }
      }
    }
  }
  dev::cta_exit(c);
}

// the backend's step buffers (CudaBackend::step_buffer) that the deterministic step uses
enum StepBuf { kBufGs, kBufVec, kBufPcid, kBufCnt, kBufOff, kBufDesc, kBufKid, kBufPart, kBufScan, kBufRowp };
static_assert(kBufRowp < CudaBackend::kStepBuffers, "step buffers");

// The deterministic one-GPU step: index -> score -> count, scan, scatter -> gather -> finish, all on `stream`.
void sgns_step_det(CudaBackend& be, cudaStream_t stream, const Key* centers, const Key* contexts, const Key* negatives,
                   int n_pairs, int neg, int d, float alpha, float* loss_out, unsigned long long* stats, int vpl,
                   int score_blocks, size_t score_smem) {
  const Ctx& c = be.ctx();
  const int n_entries = n_pairs * (neg + 2);
  const size_t num_keys = (size_t)c.L.num_keys;
  const int n_ids = (int)std::min<size_t>((size_t)n_entries, num_keys);          // bound on the step's distinct keys
  const size_t n_centers = std::min<size_t>((size_t)n_pairs, num_keys);
  const int n_ranges = (n_entries + kGatherRange - 1) / kGatherRange;
  CudaBackend::FxScratch& fx = be.fx_scratch(0, (size_t)n_ids, 0);
  float* gsb = static_cast<float*>(be.step_buffer(kBufGs, (size_t)n_entries * sizeof(float)));
  ScoreOut so;
  // one vector buffer: g0 of every pair, then the centers' snapshots (GatherDesc::vec is a row of it)
  so.g0 = static_cast<float*>(be.step_buffer(kBufVec, ((size_t)n_pairs + n_centers) * d * sizeof(float)));
  so.snap = so.g0 + (size_t)n_pairs * d;
  so.pcid = static_cast<int*>(be.step_buffer(kBufPcid, (size_t)n_pairs * sizeof(int)));
  int* cnt = static_cast<int*>(be.step_buffer(kBufCnt, ((size_t)n_ids + 1) * sizeof(int)));    // zero between steps
  int* off = static_cast<int*>(be.step_buffer(kBufOff, ((size_t)n_ids + 1) * sizeof(int)));
  GatherDesc* desc = static_cast<GatherDesc*>(be.step_buffer(kBufDesc, (size_t)n_entries * sizeof(GatherDesc)));
  int* kid = static_cast<int*>(be.step_buffer(kBufKid, (size_t)n_entries * sizeof(int)));
  long long* part = static_cast<long long*>(                                            // zero between steps
      be.step_buffer(kBufPart, ((size_t)n_ranges + 1) * 2 * d * sizeof(long long)));
  float** rowp = static_cast<float**>(be.step_buffer(kBufRowp, (size_t)n_ids * sizeof(float*)));
  size_t scan_bytes = 0;
  ADAPM_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, cnt, off, n_ids + 1, stream));
  void* scan_tmp = be.step_buffer(kBufScan, scan_bytes);

  const int grid_n = be.num_sms() * 8;
  auto blocks_for = [&](long n) { return (int)std::max<long>(1, std::min<long>((n + 255) / 256, grid_n)); };
  ADAPM_CUDA_CHECK(cudaMemsetAsync(fx.count, 0, 2 * sizeof(unsigned int), stream));
  sgns_det_index_kernel<<<blocks_for(n_pairs), 256, 0, stream>>>(c, centers, contexts, negatives, n_pairs, neg, 0, 1,
                                                                  fx.cidx, fx.keys, rowp, fx.count);
  ADAPM_COUNT_LAUNCH();
  sgns_det_index_kernel<<<blocks_for((long)n_pairs * (neg + 1)), 256, 0, stream>>>(
      c, centers, contexts, negatives, n_pairs, neg, 1, neg + 1, fx.cidx, fx.keys, rowp, fx.count);
  ADAPM_COUNT_LAUNCH();
#define ADAPM_LAUNCH_SCORE(V)                                                                                  \
  do {                                                                                                         \
    static bool attr_set = false;                                                                              \
    if (!attr_set) {                                                                                           \
      cudaFuncSetAttribute(sgns_score_tma_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024); \
      attr_set = true;                                                                                         \
    }                                                                                                          \
    sgns_score_tma_kernel<V><<<score_blocks, kThreads, score_smem, stream>>>(c, centers, contexts, negatives,  \
                                                                             n_pairs, neg, d, alpha, stats, fx.cidx, \
                                                                             gsb, fx.loss, so);                  \
  } while (0)
  switch (vpl) {
    case 1: ADAPM_LAUNCH_SCORE(1); break;
    case 2: ADAPM_LAUNCH_SCORE(2); break;
    default: ADAPM_LAUNCH_SCORE(3); break;
  }
#undef ADAPM_LAUNCH_SCORE
  ADAPM_COUNT_LAUNCH();
  sgns_det_group_kernel<false><<<blocks_for(n_entries), 256, 0, stream>>>(centers, contexts, negatives, n_pairs, neg,
                                                                           fx.cidx, cnt, off, kid, gsb, so.pcid, desc);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, cnt, off, n_ids + 1, stream));
  ADAPM_COUNT_LAUNCH();
  ADAPM_COUNT_LAUNCH();   // (the scan is two kernels)
  sgns_det_group_kernel<true><<<blocks_for(n_entries), 256, 0, stream>>>(centers, contexts, negatives, n_pairs, neg,
                                                                          fx.cidx, cnt, off, kid, gsb, so.pcid, desc);
  ADAPM_COUNT_LAUNCH();
  const int gather_blocks = (n_ranges + kWarps - 1) / kWarps;
  const auto gather = vpl == 1 ? sgns_det_gather_kernel<1> : vpl == 2 ? sgns_det_gather_kernel<2> : sgns_det_gather_kernel<3>;
  static bool gather_attr_set[4] = {};
  if (!gather_attr_set[vpl]) {          // room for the largest row of this VPL (d = 128 VPL)
    ADAPM_CUDA_CHECK(cudaFuncSetAttribute(gather, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)(kWarps * gather_warp_bytes(128 * vpl))));
    gather_attr_set[vpl] = true;
  }
  gather<<<gather_blocks, kThreads, kWarps * gather_warp_bytes(d), stream>>>(c, rowp, off, n_ids, kid, desc, so.g0, d,
                                                                             alpha, part);
  ADAPM_COUNT_LAUNCH();
  sgns_det_finish_kernel<<<blocks_for(n_entries), 256, 0, stream>>>(c, fx.keys, rowp, off, n_ids, kid, d, part, fx.cidx,
                                                                     fx.count, fx.loss, loss_out);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace

// Returns false if this variant does not support the shape (the caller falls back to the LDG kernel).
bool sgns_step_tma(CudaBackend& be, cudaStream_t stream, const Key* centers, const Key* contexts, const Key* negatives,
                   int n_pairs, int neg, int d, float alpha, float* loss_out, unsigned long long* stats) {
  if (neg + 1 > 31 || d % 4 != 0 || d > 384) return false;
  const Ctx& c = be.ctx();
  const int vpl = (d / 4 + 31) / 32;
  const size_t buf_floats = ((size_t)2 * d + 31) & ~(size_t)31;
  // Block shape: 256 threads x 2 blocks = 16 warps per SM (two blocks of 128 registers fill the register file; the
  // ring of 5 row buffers per warp keeps enough 2400-byte rows in flight to be memory-bound).
  const int threads = kThreads;
  const int warps = threads / 32;
  const size_t smem = (size_t)warps * (RING + 1) * buf_floats * sizeof(float) + 128;
  if (smem > 110 * 1024) return false;  // keep 2 blocks per SM
  int blocks = std::min((n_pairs + warps - 1) / warps, be.num_sms() * 12);
  // register budget: 128 (single GPU: nothing to share the SMs with) or 104 (multi GPU)
  const bool lean = c.L.world > 1;
  // In-place updates leave as TMA bulk reductions: measured +2.6 % on one GPU against RED.128 from the warp, and the
  // warp's LSU slots stay free for the sync round's kernels. (A software-pipelined target loop - score of target t+1
  // during the update of target t - was measured too: no gain at 128 registers, -5 % at 104: the kernel is not bound by
  // the per-warp dependency chain.)
  // One GPU: deterministic step (score pass + updates grouped by key, see sgns_step_det), so that the same inputs give
  // the same rows and loss in every run; ADAPM_SGNS_DETERMINISTIC=0 selects in-place (Hogwild) updates. Several GPUs:
  // rows move between ranks during the step and are updated in place.
  static const bool det_env = [] { const char* e = getenv("ADAPM_SGNS_DETERMINISTIC"); return !e || atoi(e) != 0; }();
  const long n_src = (long)n_pairs * (neg + 2);
  ADAPM_CHECK(n_src < (1L << 29), "sgns_step: too many keys in one step");   // (entry or key id << 2 fits an int)
  if (det_env && c.L.world == 1) {
    sgns_step_det(be, stream, centers, contexts, negatives, n_pairs, neg, d, alpha, loss_out, stats, vpl, blocks, smem);
    return true;
  }
#define ADAPM_LAUNCH_TMA2(V, R)                                                                                 \
  do {                                                                                                          \
    static bool attr_set = false;                                                                               \
    if (!attr_set) {                                                                                            \
      cudaFuncSetAttribute(sgns_step_tma_kernel<V, R>, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024);  \
      attr_set = true;                                                                                          \
    }                                                                                                           \
    sgns_step_tma_kernel<V, R><<<blocks, threads, smem, stream>>>(c, centers, contexts, negatives, n_pairs, neg, d, \
                                                                  alpha, loss_out, stats);                      \
  } while (0)
#define ADAPM_LAUNCH_TMA(V)              \
  do {                                   \
    if (lean) ADAPM_LAUNCH_TMA2(V, 104); \
    else ADAPM_LAUNCH_TMA2(V, 128);      \
  } while (0)
  switch (vpl) {
    case 1: ADAPM_LAUNCH_TMA(1); break;
    case 2: ADAPM_LAUNCH_TMA(2); break;
    default: ADAPM_LAUNCH_TMA(3); break;
  }
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
  return true;
}

}  // namespace cudaops
}  // namespace adapm

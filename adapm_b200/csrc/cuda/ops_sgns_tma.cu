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
// (The deterministic one-GPU kernel adds its updates to fixed-point accumulators instead and prefetches RING targets.)
// The TMA engine reads rows that live on a peer GPU through their NVLink-mapped addresses as well;
// rows in a transitional protocol state take the generic out-of-line path.
#include <cuda_runtime.h>

#include <cstdlib>

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

// Deterministic accumulation (one GPU, fx_accum.cuh): |embedding update| <= alpha per contribution (AdaGrad normalises
// it), AdaGrad increments are squared gradients: 2^40 / 2^36 leave 2^23 / 2^27 of range per element and step. The
// loss is a fixed-point sum too: 2^32 leaves 2^31 of summed loss per step.
constexpr float kFxEmb = 1099511627776.f;     // 2^40
constexpr float kFxAda = 68719476736.f;       // 2^36
constexpr float kFxLoss = 4294967296.f;       // 2^32
using fx::add4;

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
// FX: deterministic one-GPU variant (fixed-point accumulation, see kFxEmb); instantiated as its own kernel
// (sgns_step_tma_fx_kernel) so that the in-place variants keep their register allocation.
template <int VPL, bool FX>
__device__ __forceinline__ void
sgns_step_tma_body(const Ctx& c, const Key* __restrict__ centers, const Key* __restrict__ contexts,
                   const Key* __restrict__ negatives, int n_pairs, int neg, int d, float alpha,
                   float* __restrict__ loss_out, unsigned long long* __restrict__ stats,
                   long long* __restrict__ fx_acc, const int* __restrict__ fx_cidx,
                   unsigned long long* __restrict__ fx_loss) {
  constexpr bool BULK = !FX;
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
                                         // bits 2..: the key's accumulator row (deterministic mode)
    if (lane == 0) my_key = ckey;
    else if (lane - 1 < n_targets) my_key = (lane == 1) ? pos_key : negatives[(size_t)p * neg + (lane - 2)];
    if (my_key >= 0) {
      const Target tg = dev::resolve_fast(c, my_key, 0, &n_local, &n_remote);
      my_row = tg.row;
      my_mark = tg.flag ? (void*)tg.flag : (void*)tg.version;
      my_bits = (tg.flag ? 2 : 0) | (FX ? __ldg(fx_cidx + my_key) << 2 : 0);
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
        mbar_expect_tx(&bars[b], row_bytes);
        bulk_g2s(buf, row, row_bytes, &bars[b]);
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

    // ---- targets
    for (int t = 0; t < n_targets; ++t) {
      const int b = consumed % RING;
      float* buf = ring + (size_t)b * buf_floats;
      const Key tkey = (Key)__shfl_sync(0xffffffffu, (unsigned long long)my_key, t + 1);
      float* t_row = (float*)__shfl_sync(0xffffffffu, (unsigned long long)my_row, t + 1);
      // (shuffled here, with the whole warp converged: the update loop below runs on a subset of the lanes)
      long long* fx_t = FX ? fx_acc + (size_t)(__shfl_sync(0xffffffffu, my_bits, t + 1) >> 2) * (2 * d) : nullptr;
      mbar_wait(&bars[b], (consumed / RING) & 1u);
      ++consumed;
      const float label = (t == 0) ? 1.f : 0.f;
      const bool dup = (t > 0 && tkey == pos_key);  // reference: negative == positive target is skipped
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
            float4 a1 = reinterpret_cast<const float4*>(buf + d)[j];
            g0[v].x += gs * e1[v].x; g0[v].y += gs * e1[v].y; g0[v].z += gs * e1[v].z; g0[v].w += gs * e1[v].w;
            float4 gr = make_float4(gs * e0[v].x, gs * e0[v].y, gs * e0[v].z, gs * e0[v].w);
            float4 ua = make_float4(gr.x * gr.x, gr.y * gr.y, gr.z * gr.z, gr.w * gr.w);
            float4 ue;
            ue.x = alpha * gr.x * rsqrtf(a1.x + ua.x);
            ue.y = alpha * gr.y * rsqrtf(a1.y + ua.y);
            ue.z = alpha * gr.z * rsqrtf(a1.z + ua.z);
            ue.w = alpha * gr.w * rsqrtf(a1.w + ua.w);
            if (FX) {                     // deterministic mode: fixed-point sums, applied after the step
              add4(fx_t, j, nvec, ue, kFxEmb);
              add4(fx_t + d, j, nvec, ua, kFxAda);
            } else {                      // stage the update in place of the consumed row
              reinterpret_cast<float4*>(buf)[j] = ue;
              reinterpret_cast<float4*>(buf + d)[j] = ua;
            }
          }
        }
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
    } else {
      long long* fx_c = FX ? fx_acc + (size_t)(__shfl_sync(0xffffffffu, my_bits, 0) >> 2) * (2 * d) : nullptr;
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
          if (FX) {
            add4(fx_c, j, nvec, ue, kFxEmb);
            add4(fx_c + d, j, nvec, ua, kFxAda);
          } else {
            reinterpret_cast<float4*>(scratch)[j] = ue;
            reinterpret_cast<float4*>(scratch + d)[j] = ua;
          }
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
  if (FX && lane == 0) atomicAdd(fx_loss, (unsigned long long)__float2ll_rn(loss_acc * kFxLoss));
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
                                 nullptr, nullptr);
}

template <int VPL>
__global__ void __maxnreg__(128)
sgns_step_tma_fx_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ centers, const Key* __restrict__ contexts,
                        const Key* __restrict__ negatives, int n_pairs, int neg, int d, float alpha,
                        unsigned long long* __restrict__ stats, long long* __restrict__ fx_acc,
                        const int* __restrict__ fx_cidx, unsigned long long* __restrict__ fx_loss) {
  sgns_step_tma_body<VPL, true>(c, centers, contexts, negatives, n_pairs, neg, d, alpha, nullptr, stats, fx_acc, fx_cidx,
                                fx_loss);
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
  // One GPU: deterministic step (fixed-point accumulation + apply pass), so that the same inputs give the same rows
  // and loss in every run; ADAPM_SGNS_DETERMINISTIC=0 selects in-place (Hogwild) updates. Several GPUs: rows move
  // between ranks during the step and are updated in place.
  static const bool det_env = [] { const char* e = getenv("ADAPM_SGNS_DETERMINISTIC"); return !e || atoi(e) != 0; }();
  const long n_src = (long)n_pairs * (neg + 2);
  ADAPM_CHECK(n_src < (1L << 29), "sgns_step: too many keys in one step");   // (row index << 2 fits an int)
  CudaBackend::FxScratch* fxs = nullptr;
  if (det_env && c.L.world == 1) {   // every key of the step gets an accumulator region of 2 d (one unit)
    const fx::Source src[3] = {{centers, n_pairs, 1}, {contexts, n_pairs, 1}, {negatives, (long)n_pairs * neg, 1}};
    fxs = &fx::begin(be, stream, src, 3, 2 * d);
  }
  long long* fx_acc = fxs ? fxs->acc : nullptr;
  const int* fx_cidx = fxs ? fxs->cidx : nullptr;
  unsigned long long* fx_loss = fxs ? fxs->loss : nullptr;
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
#define ADAPM_LAUNCH_TMA_FX(V)                                                                                  \
  do {                                                                                                          \
    static bool attr_set = false;                                                                               \
    if (!attr_set) {                                                                                            \
      cudaFuncSetAttribute(sgns_step_tma_fx_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024); \
      attr_set = true;                                                                                          \
    }                                                                                                           \
    sgns_step_tma_fx_kernel<V><<<blocks, threads, smem, stream>>>(c, centers, contexts, negatives, n_pairs, neg, d, \
                                                                  alpha, stats, fx_acc, fx_cidx, fx_loss);      \
  } while (0)
  if (fxs) {
    switch (vpl) {
      case 1: ADAPM_LAUNCH_TMA_FX(1); break;
      case 2: ADAPM_LAUNCH_TMA_FX(2); break;
      default: ADAPM_LAUNCH_TMA_FX(3); break;
    }
  } else {
    switch (vpl) {
      case 1: ADAPM_LAUNCH_TMA(1); break;
      case 2: ADAPM_LAUNCH_TMA(2); break;
      default: ADAPM_LAUNCH_TMA(3); break;
    }
  }
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
  if (fxs) fx::apply(be, stream, 2 * d, kFxEmb, kFxAda, kFxLoss, 0, loss_out);
  return true;
}

}  // namespace cudaops
}  // namespace adapm

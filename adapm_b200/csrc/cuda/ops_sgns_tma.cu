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
// The deterministic one-GPU step (det_step in sgns_det.cuh, with the entry source SgnsEntries) runs the same body as a
// score pass that loads the targets' embedding halves, then groups the step's contributions by key and lets one warp
// per row gather them as fixed-point integer sums.
// A key with a single entry in the step (two thirds of the keys at the benchmark's shape) skips the grouping: the score
// pass loads its whole row and writes the update back itself, with the gather pass's fixed-point arithmetic.
// The TMA engine reads rows that live on a peer GPU through their NVLink-mapped addresses as well;
// rows in a transitional protocol state take the generic out-of-line path.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>

#include <cub/cub.cuh>
#include <thrust/iterator/transform_iterator.h>

#include "fx_accum.cuh"
#include "ops.h"
#include "pm_kernels.cuh"
#include "sgns_common.cuh"
#include "sgns_det.cuh"

namespace adapm {
namespace cudaops {

namespace {

constexpr int RING = 4;
using sgns::kMaxExp;

using dev::Target;
using dev::warp_sum;

// What the score pass (SCORE) of the deterministic step writes for the gather pass besides gs and the loss (the
// step body takes those as separate arguments).
struct ScoreOut {
  float* g0;                     // [n_pairs x d] the pair's center gradient
  float* snap;                   // [distinct centers x d] start-of-step embedding of each center, by compact id
                                 // (the deterministic step keeps it right after g0 in one buffer)
  int* pcid;                     // [n_pairs] compact id of the pair's center
  const int* cnt;                // [distinct keys] entries of each key in the step, by compact id: the score pass
                                 // applies a key with one entry itself
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
// variants keep their register allocation). It reads start-of-step rows - the embedding half of each target - and
// writes per pair the center gradient g0, per target gs, and each center's embedding (ScoreOut). The gather pass forms
// and applies the rows' updates from these. A key whose only entry in the step is this pair's (ScoreOut::cnt) is the
// exception: no other warp reads or writes its row during the step, so the warp loads the whole row (target) or its
// AdaGrad half (center), applies the one term exactly as the gather pass would (fx_apply_one) and stores the row.
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
    int my_bits = 0;                     // bit 0: the key's only entry in the step is this one (SCORE),
                                         // bit 1: my_mark is a replica dirty byte,
                                         // bits 2..: the center's compact id (SCORE, lane 0)
    if (lane == 0) my_key = ckey;
    else if (lane - 1 < n_targets) my_key = (lane == 1) ? pos_key : negatives[(size_t)p * neg + (lane - 2)];
    if (my_key >= 0) {
      int cid = 0, n_entries = 0;
      if (SCORE) {                       // (a chain of its own, next to resolve_fast's)
        cid = __ldg(cidx + my_key);
        n_entries = __ldg(so.cnt + cid);
      }
      const Target tg = dev::resolve_fast(c, my_key, 0, &n_local, &n_remote);
      my_row = tg.row;
      my_mark = tg.flag ? (void*)tg.flag : (void*)tg.version;
      const bool dup = lane >= 2 && my_key == pos_key;   // a negative equal to the context is no entry
      my_bits = (tg.flag ? 2 : 0) | (SCORE && lane == 0 ? cid << 2 : 0) | (SCORE && n_entries == 1 && !dup ? 1 : 0);
    }
    // SCORE: lane l's key has one entry in the step, and it is this pair's: no other warp reads or writes its row during
    // the step, so this warp loads the whole row and writes its update back (the gather pass does not see the key)
    const unsigned single = SCORE ? __ballot_sync(0xffffffffu, my_bits & 1) : 0u;
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
        const uint32_t bytes = (single >> (t + 1)) & 1u ? row_bytes : load_bytes;
        mbar_expect_tx(&bars[b], bytes);
        bulk_g2s(buf, row, bytes, &bars[b]);
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
        const bool one = (single >> (t + 1)) & 1u;   // SCORE: the slot holds the whole row, which this warp updates
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
              if (one) {                  // ... unless its key has this one entry: gs * e0 as the gather pass adds it
                float4 a1 = reinterpret_cast<const float4*>(buf + d)[j];
                fx_apply_one(e1[v].x, a1.x, gs * e0[v].x, alpha);
                fx_apply_one(e1[v].y, a1.y, gs * e0[v].y, alpha);
                fx_apply_one(e1[v].z, a1.z, gs * e0[v].z, alpha);
                fx_apply_one(e1[v].w, a1.w, gs * e0[v].w, alpha);
                reinterpret_cast<float4*>(t_row)[j] = e1[v];
                reinterpret_cast<float4*>(t_row + d)[j] = a1;
              }
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
      if (single & 1u) {                  // ... unless this pair is the center's one entry: 1 * g0 as the gather adds it
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          int j = lane + v * 32;
          if (j < nvec) {
            float4 r = e0[v];
            float4 a0 = dev::ld_row4(c_row + d + 4 * j);
            fx_apply_one(r.x, a0.x, g0[v].x, alpha);
            fx_apply_one(r.y, a0.y, g0[v].y, alpha);
            fx_apply_one(r.z, a0.z, g0[v].z, alpha);
            fx_apply_one(r.w, a0.w, g0[v].w, alpha);
            reinterpret_cast<float4*>(c_row)[j] = r;
            reinterpret_cast<float4*>(c_row + d)[j] = a0;
          }
        }
      } else {
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          int j = lane + v * 32;
          if (j < nvec) reinterpret_cast<float4*>(so.g0 + (size_t)p * d)[j] = g0[v];
        }
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
  dev::flush_stats(stats, n_local, n_remote, n_slow, n_upd);
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

// ---- the deterministic one-GPU step (det_step, sgns_det.cuh)
// Entry x = p * (neg + 2) + s: s = 0 the center of pair p, s = 1 its context, s >= 2 negative s - 2. The center adds
// 1 * the pair's center gradient g0 (vector row p); a target adds gs * the center's start-of-step embedding (vector row
// n_pairs + the center's compact id).
struct SgnsEntries {
  const Key* __restrict__ centers;
  const Key* __restrict__ contexts;
  const Key* __restrict__ negatives;
  int n_pairs, neg;
  const int* __restrict__ pcid;  // [n_pairs] the compact id of the pair's center (ScoreOut::pcid)
  float* gs;                     // [n_pairs x (neg + 2)] gs of each target; 0 or kNoEntry: whether the center adds g0
  static constexpr int kFirstSlots = 1;          // the centers first: their compact ids are the rows of ScoreOut::snap
  static constexpr bool kSinglesInScore = true;
  __host__ __device__ int items() const { return n_pairs; }
  __host__ __device__ int per() const { return neg + 2; }
  __device__ __forceinline__ Key key(int p, int s) const {
    return s == 0 ? centers[p] : (s == 1 ? contexts[p] : negatives[(size_t)p * neg + (s - 2)]);
  }
  // a negative equal to the pair's context adds nothing (the step skips it); neither does a negative key
  __device__ __forceinline__ bool counts(int p, int s, Key k) const { return k >= 0 && !(s >= 2 && k == contexts[p]); }
  __device__ __forceinline__ GatherDesc desc(int p, int s, int x) const {
    const float g = __ldg(gs + x);
    if (s == 0) return {g == kNoEntry ? kNoEntry : 1.f, p};
    return {g, g == kNoEntry ? 0 : n_pairs + __ldg(pcid + p)};
  }
};

__global__ void sgns_det_index_kernel(const __grid_constant__ Ctx c, const __grid_constant__ SgnsEntries src,
                                      int first_slot, int n_slots, int* __restrict__ cidx, Key* __restrict__ keys,
                                      float** __restrict__ rowp, unsigned int* __restrict__ count) {
  det_index(c, src, first_slot, n_slots, cidx, keys, rowp, count);
}

template <bool SCATTER>
__global__ void sgns_det_group_kernel(const __grid_constant__ SgnsEntries src, const int* __restrict__ cidx,
                                      int* __restrict__ cnt, const int* __restrict__ off, int* __restrict__ kid,
                                      GatherDesc* __restrict__ desc) {
  det_group<SCATTER>(src, cidx, cnt, off, kid, desc);
}

}  // namespace

// Returns false if this variant does not support the shape: neg + 1 > 31, or d >= 340, where the ring of 5 row buffers
// per warp no longer fits two blocks per SM. sgns_step then falls back to the LDG kernel (impl auto) or raises (impl tma).
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
  // One GPU: deterministic step (score pass + updates grouped by key, det_step), so that the same inputs give
  // the same rows and loss in every run; ADAPM_SGNS_DETERMINISTIC=0 selects in-place (Hogwild) updates. Several GPUs:
  // rows move between ranks during the step and are updated in place.
  static const bool det_env = [] { const char* e = getenv("ADAPM_SGNS_DETERMINISTIC"); return !e || atoi(e) != 0; }();
  const long n_src = (long)n_pairs * (neg + 2);
  ADAPM_CHECK(n_src < (1L << 29), "sgns_step: too many keys in one step");   // (entry or key id << 2 fits an int)
  if (det_env && c.L.world == 1) {
    int* pcid = static_cast<int*>(be.step_buffer(kBufPcid, (size_t)n_pairs * sizeof(int)));
    const SgnsEntries src{centers, contexts, negatives, n_pairs, neg, pcid, nullptr};
    // vector buffer: g0 of every pair, then the snapshots of the distinct centers
    const size_t n_centers = std::min<size_t>((size_t)n_pairs, (size_t)c.L.num_keys);
    det_step<sgns_det_index_kernel, sgns_det_group_kernel<false>, sgns_det_group_kernel<true>>(
        be, stream, src, n_pairs + n_centers, d, alpha, vpl, loss_out,
        [&](float* gs, float* vecs, const int* cnt, CudaBackend::FxScratch& fx) {
          const ScoreOut so{vecs, vecs + (size_t)n_pairs * d, pcid, cnt};
          by_vpl(vpl, [&](auto v) {
            constexpr auto score = sgns_score_tma_kernel<decltype(v)::value>;
            set_max_dynamic_smem<score>(110 * 1024);
            score<<<blocks, kThreads, smem, stream>>>(c, centers, contexts, negatives, n_pairs, neg, d, alpha, stats,
                                                      fx.cidx, gs, fx.loss, so);
          });
        });
    return true;
  }
#define ADAPM_LAUNCH_TMA2(V, R)                                                                                 \
  do {                                                                                                          \
    set_max_dynamic_smem<sgns_step_tma_kernel<V, R>>(110 * 1024);                                               \
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

namespace {
// CSR positions of a key with c entries
struct GatheredEntries {
  bool singles_in_score;
  __host__ __device__ int operator()(int c) const { return singles_in_score && c == 1 ? 0 : c; }
};
}  // namespace

void det_scan(void* tmp, size_t& bytes, const int* cnt, int* off, int n, bool singles_in_score, cudaStream_t stream) {
  const auto gathered = thrust::make_transform_iterator(cnt, GatheredEntries{singles_in_score});
  ADAPM_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(tmp, bytes, gathered, off, n, stream));
}

}  // namespace cudaops
}  // namespace adapm

// word2vec CBOW step (continuous bag of words, word2vec.c's default architecture) with negative sampling and
// per-contribution AdaGrad, on the parameter store. Rows and keys are as for SGNS: syn0[w] = 2w, syn1[w] = 2w + 1, a row
// is [embedding d | AdaGrad d]. One window = one centre (syn1 key) and up to 32 context occurrences (syn0 keys, -1 =
// padding); every window reads the rows as they were at the start of the step:
//   h = (1 / C) sum_c syn0[c].emb        over the C context occurrences (a repeated word counts every time)
//   targets syn1[centre] (label 1) and syn1[neg_j] (label 0; a negative equal to the centre is skipped)
//   g_t = label - sigmoid(h . t.emb), saturated at |f| > 6; neu1e = sum_t g_t t.emb
//   syn1[t] += [alpha g_t h / sqrt(a_t + (g_t h)^2) | (g_t h)^2]       one push per (window, target)
//   syn0[c] += [alpha neu1e / sqrt(a_c + neu1e^2) | neu1e^2]          one push per context occurrence
// A window with centre < 0 or no context does nothing.
//
// Hierarchical softmax (word2vec.c's -hs 1) is the same body with another target source. The centre's syn1 key 2w + 1
// names the word w whose Huffman path supplies the targets: lane j gets inner node nodes[offsets[w] + j] (row
// syn1_key(node) = 2 node + 1) with label 1 - bit j of codes[w], for j < len(w) <= 32. A node with |f| >= 6 gets no
// update and adds nothing to neu1e (word2vec.c and gensim skip it); its loss term is counted. The skip-gram form is an
// item with one context. The root is on every path, so in the deterministic step it takes one contribution per item:
// its AdaGrad half gains sum over the step's items of (g h)^2 per element, which must stay below 2^27 (|g h| < 1 per
// item keeps it there for B < 2^27 items; h is a mean of embeddings, |h| < 1 in practice).
//
// Two paths, selected by the world size:
//  * in place (several GPUs; on one GPU on request): cbow_step_kernel, one warp per window. The lanes resolve the
//    contexts and the targets through the directory at once. The window's rows stream through a per-warp shared-memory
//    ring that the TMA engine fills (cp.async.bulk, completion on an mbarrier) RING - 1 items ahead of the math, as in
//    the SGNS step (ops_sgns_tma.cu): first the contexts' embedding halves (h), then the targets' whole rows (each
//    target's update overwrites its consumed slot and leaves as one bulk reduction, cp.reduce.async.bulk), then the
//    contexts' AdaGrad halves (each context occurrence's update leaves the same way). Rows in a transitional protocol
//    state take the generic out-of-line path. Updates of other windows land while the step runs (Hogwild); so do the
//    pushes of a context repeated within one window.
//  * deterministic (one GPU): cbow_score_kernel, the same body as a score pass that loads only embedding halves and
//    writes per window h and neu1e ([h rows | neu1e rows]), per (window, target) g_t, and the loss. Each target
//    contribution is then GatherDesc{g_t, h row} and each context occurrence GatherDesc{1, neu1e row}: grouped by key,
//    they go through the gather and finish passes of the deterministic SGNS step (sgns_det.cuh), which sum them in
//    fixed point. Runs give bit-identical rows and loss. The scales are the SGNS step's: 2^23 of summed embedding update
//    and 2^27 of summed AdaGrad increment per element and step. A word that is a context in n windows of a step adds
//    n neu1e^2 terms to its AdaGrad half, so n |neu1e|^2 must stay below 2^27 (n = 10 000: |neu1e| < 115).
#include <cuda_runtime.h>

#include <algorithm>

#include <cub/cub.cuh>

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

// What the score pass writes besides the loss.
struct CbowScoreOut {
  float* vecs;                   // [2 B x d]: h of window w at row w, neu1e at row B + w
  float* gs;                     // [B x n_t]: g of target t of window w, kNoEntry if the target adds nothing
};

// Where a window's targets come from. n_t(): target slots per window. target(): lane l's target key (-1: none) of a
// window with centre ckey >= 0, filling the window's Item. label(): target s's label. slow_key(): target s's key again,
// for the generic path. entry_key() / entry_counts(): entry s < n_t() of the deterministic step's index and group
// kernels (entry_key also gives the contexts' entries), which skip entries for which entry_counts() is false.
//
// Negative sampling: the centre (label 1) and the negatives (label 0; one equal to the centre is skipped); the gradient
// saturates at |f| > 6.
struct NegTargets {
  const Key* __restrict__ negatives;
  int neg;
  static constexpr bool kSkipSaturated = false;
  struct Item {};
  __host__ __device__ __forceinline__ int n_t() const { return neg + 1; }
  __device__ __forceinline__ Key target(Item&, Key ckey, int w, int lane, int n_t) const {
    Key tk = lane == 0 ? ckey : (lane < n_t ? negatives[(size_t)w * neg + lane - 1] : -1);
    if (lane > 0 && tk == ckey) tk = -1;
    return tk;
  }
  __device__ __forceinline__ float label(const Item&, int s) const { return s == 0 ? 1.f : 0.f; }
  __device__ __forceinline__ Key slow_key(Key ckey, int w, int s) const {
    return s == 0 ? ckey : negatives[(size_t)w * neg + s - 1];
  }
  __device__ __forceinline__ Key entry_key(const Key* centers, const Key* contexts, int nc, int w, int s) const {
    const int n_t = neg + 1;
    return s == 0 ? centers[w] : (s < n_t ? negatives[(size_t)w * neg + s - 1] : contexts[(size_t)w * nc + s - n_t]);
  }
  // what adds nothing: a key < 0, every entry of a window whose centre is < 0, a negative equal to the centre
  __device__ __forceinline__ bool entry_counts(const Key* centers, int w, int s, Key k) const {
    const Key ck = centers[w];
    return k >= 0 && ck >= 0 && !(s >= 1 && s <= neg && k == ck);
  }
};

// Hierarchical softmax: the Huffman path of the centre's word (offsets [n_words + 1], nodes, codes [n_words]: the CSR of
// the tree, root first). A centre whose word is not in the tree has no targets.
struct PathTargets {
  const int64_t* __restrict__ offsets;
  const int32_t* __restrict__ nodes;
  const uint32_t* __restrict__ codes;
  int n_words;
  int max_len;
  static constexpr bool kSkipSaturated = true;
  struct Item { uint32_t code; };
  __host__ __device__ __forceinline__ int n_t() const { return max_len; }
  __device__ __forceinline__ Key node_key(Key ckey, int s) const {   // -1 past the end of the path
    const Key word = ckey >> 1;
    if (word >= n_words) return -1;
    const int64_t o = offsets[word];
    return s < offsets[word + 1] - o ? 2 * (Key)nodes[o + s] + 1 : -1;
  }
  __device__ __forceinline__ Key target(Item& it, Key ckey, int, int lane, int) const {
    it.code = (ckey >> 1) < n_words ? codes[ckey >> 1] : 0u;
    return node_key(ckey, lane);
  }
  __device__ __forceinline__ float label(const Item& it, int s) const { return (it.code >> s) & 1u ? 0.f : 1.f; }
  __device__ __forceinline__ Key slow_key(Key ckey, int, int s) const { return node_key(ckey, s); }
  __device__ __forceinline__ Key entry_key(const Key* centers, const Key* contexts, int nc, int w, int s) const {
    if (s >= max_len) return contexts[(size_t)w * nc + s - max_len];
    const Key ck = centers[w];
    return ck >= 0 ? node_key(ck, s) : -1;
  }
  __device__ __forceinline__ bool entry_counts(const Key* centers, int w, int, Key k) const {
    return k >= 0 && centers[w] >= 0;
  }
};

// Lane-resolved window: lane l holds context occurrence l and target l (ts.target(.., l, ..)).
// bits: 1 context present, 2 its mark is a replica dirty byte, 4 target present, 8 its mark is a dirty byte.
template <int VPL, bool SCORE, class Src>
__device__ __forceinline__ void
cbow_step_body(const Ctx& c, const Key* __restrict__ centers, const Key* __restrict__ contexts, const Src& ts,
               int n_win, int nc, int d, float alpha,
               float* __restrict__ loss_out, unsigned long long* __restrict__ stats,
               unsigned long long* __restrict__ fx_loss, const CbowScoreOut& so) {
  constexpr bool BULK = !SCORE;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ unsigned long long wbar[kWarps][RING];
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int warp = blockIdx.x * kWarps + wib;
  const int nwarps = gridDim.x * kWarps;
  const int nvec = d >> 2;
  const int n_t = ts.n_t();
  const uint32_t half_bytes = (uint32_t)(d * sizeof(float));
  const uint32_t row_bytes = 2 * half_bytes;
  const size_t buf_floats = ((size_t)2 * d + 31) & ~(size_t)31;  // keep every ring slot 128-byte aligned
  float* ring = reinterpret_cast<float*>(smem_raw) + (size_t)wib * (RING + 1) * buf_floats;
  float* scratch = ring + (size_t)RING * buf_floats;             // h | neu1e of generic-path targets (2 d floats)
  unsigned long long* bars = wbar[wib];
  if (lane == 0) {
    for (int r = 0; r < RING; ++r) mbar_init(&bars[r], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncwarp();
  uint32_t issued = 0, consumed = 0;   // ring counters (slot = n % RING, phase parity = (n / RING) & 1)
  float loss_acc = 0.f;
  unsigned n_local = 0, n_remote = 0, n_slow = 0, n_upd = 0;

  for (int w = warp; w < n_win; w += nwarps) {
    const Key ckey = centers[w];
    float my_gs = kNoEntry;                       // SCORE: g of this lane's target
    float* x_row = nullptr;
    void* x_mark = nullptr;
    float* t_row = nullptr;
    void* t_mark = nullptr;
    int bits = 0;
    typename Src::Item it{};
    if (ckey >= 0) {
      const Key xk = lane < nc ? contexts[(size_t)w * nc + lane] : -1;
      const Key tk = ts.target(it, ckey, w, lane, n_t);
      if (xk >= 0) {
        const Target tg = dev::resolve_fast(c, xk, 0, &n_local, &n_remote);
        x_row = tg.row;
        x_mark = tg.flag ? (void*)tg.flag : (void*)tg.version;
        bits |= 1 | (tg.flag ? 2 : 0);
      }
      if (tk >= 0) {
        const Target tg = dev::resolve_fast(c, tk, 0, &n_local, &n_remote);
        t_row = tg.row;
        t_mark = tg.flag ? (void*)tg.flag : (void*)tg.version;
        bits |= 4 | (tg.flag ? 8 : 0);
      }
      // the score pass runs on one GPU, where every row is at home: a key without a row adds nothing there
      if (SCORE && !x_row) bits &= ~3;
      if (SCORE && !t_row) bits &= ~12;
    }
    const unsigned xmask = __ballot_sync(0xffffffffu, bits & 1);
    const unsigned tmask = __ballot_sync(0xffffffffu, bits & 4);
    const int n_x = __popc(xmask), n_tt = __popc(tmask);
    if (n_x == 0 || n_tt == 0) {
      if (SCORE && lane < n_t) so.gs[(size_t)w * n_t + lane] = kNoEntry;
      if (SCORE && n_x > 0) {           // contexts but no target: h and neu1e are zero (the gather adds zero updates)
        for (int j = lane; j < nvec; j += 32) {
          reinterpret_cast<float4*>(so.vecs + (size_t)w * d)[j] = make_float4(0.f, 0.f, 0.f, 0.f);
          reinterpret_cast<float4*>(so.vecs + ((size_t)n_win + w) * d)[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
      if (n_x == 0) continue;
      if (SCORE) { n_upd += n_x; continue; }
    }
    // ring items: contexts' embedding halves (n_x), targets (n_tt), in place also contexts' AdaGrad halves (n_x)
    const int n_items = n_x + n_tt + (BULK ? n_x : 0);
    auto item_lane = [&](int i) -> int {
      if (i < n_x) return __fns(xmask, 0, i + 1);
      if (i < n_x + n_tt) return __fns(tmask, 0, i - n_x + 1);
      return __fns(xmask, 0, i - n_x - n_tt + 1);
    };
    auto issue = [&](int i) {
      const int b = issued % RING;
      float* buf = ring + (size_t)b * buf_floats;
      const int src = item_lane(i);
      const bool tgt = i >= n_x && i < n_x + n_tt;
      float* xr = (float*)__shfl_sync(0xffffffffu, (unsigned long long)x_row, src);
      float* tr = (float*)__shfl_sync(0xffffffffu, (unsigned long long)t_row, src);
      float* row = tgt ? tr : xr;
      if (lane == 0) {
        if (row == nullptr) {
          mbar_arrive(&bars[b]);                 // generic path: nothing to load, complete the phase
        } else {
          if (BULK) bulk_wait_read<1>();         // the reduction that used this slot (one item ago) has read it
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          const bool ada = i >= n_x + n_tt;      // a context's AdaGrad half, into the slot's second half
          const uint32_t bytes = tgt ? (SCORE ? half_bytes : row_bytes) : half_bytes;
          mbar_expect_tx(&bars[b], bytes);
          bulk_g2s(ada ? buf + d : buf, ada ? row + d : row, bytes, &bars[b]);
        }
      }
      ++issued;
    };
    // the generic path stages rows in the consumed slot, which no load fills: wait until no reduction reads it
    auto slot_free = [&] { if (BULK) { if (lane == 0) bulk_wait_read<0>(); __syncwarp(); } };
    constexpr int DIST = BULK ? RING - 1 : RING;
    if (BULK) { if (lane == 0) bulk_wait_read<0>(); __syncwarp(); }   // the previous window's reductions have read the ring
    for (int i = 0; i < min(n_items, DIST); ++i) issue(i);

    // nu sums the contexts' embeddings first; h then lives in scratch[0, d) (shared memory: one register array per lane
    // instead of two) and nu becomes neu1e; scratch[d, 2d) sums the neu1e terms of generic-path targets
    float4 nu[VPL];
#pragma unroll
    for (int v = 0; v < VPL; ++v) nu[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    bool have_slow = false;
    for (int i = 0; i < n_items; ++i) {
      const int b = consumed % RING;
      float* buf = ring + (size_t)b * buf_floats;
      const int src = item_lane(i);
      mbar_wait(&bars[b], (consumed / RING) & 1u);
      ++consumed;
      if (i < n_x) {
        // ---- context i: its embedding into h
        const float* xr = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)x_row, src);
        bool ok = true;
        if (xr == nullptr) {
          ++n_slow;
          slot_free();
          ok = dev::slow_pull(c, contexts[(size_t)w * nc + src], buf);   // ring slot b is free: use it as stage
        }
        if (ok) {
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            const int j = lane + v * 32;
            if (j < nvec) {
              const float4 e = reinterpret_cast<const float4*>(buf)[j];
              nu[v].x += e.x; nu[v].y += e.y; nu[v].z += e.z; nu[v].w += e.w;
            }
          }
        }
        if (i == n_x - 1) {
          const float inv = 1.f / (float)n_x;
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            const int j = lane + v * 32;
            if (j < nvec) {
              const float4 h = make_float4(nu[v].x * inv, nu[v].y * inv, nu[v].z * inv, nu[v].w * inv);
              reinterpret_cast<float4*>(scratch)[j] = h;
              reinterpret_cast<float4*>(scratch + d)[j] = make_float4(0.f, 0.f, 0.f, 0.f);
              if (SCORE) reinterpret_cast<float4*>(so.vecs + (size_t)w * d)[j] = h;
            }
            nu[v] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
          __syncwarp();
        }
      } else if (i < n_x + n_tt) {
        // ---- target: score against h, g, neu1e, the target's update
        const float* tr = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)t_row, src);
        const float label = ts.label(it, src);
        if (BULK && tr == nullptr) {
          ++n_slow;
          slot_free();
          have_slow = true;
          const Key tk = ts.slow_key(ckey, w, src);
          bool applied;
          loss_acc += sgns::slow_target<Src::kSkipSaturated>(c, tk, label, alpha, d, buf, scratch, scratch + d,
                                                             &applied);
          if (applied) ++n_upd;
        } else {
          float f = 0.f;
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            const int j = lane + v * 32;
            if (j < nvec) {
              const float4 e = reinterpret_cast<const float4*>(buf)[j];
              const float4 h = reinterpret_cast<const float4*>(scratch)[j];
              f += h.x * e.x + h.y * e.y + h.z * e.z + h.w * e.w;
            }
          }
          f = warp_sum(f);
          float gs;
          bool skip = false;                       // hierarchical softmax: |f| >= 6 adds nothing
          if constexpr (Src::kSkipSaturated) {
            skip = fabsf(f) >= kMaxExp;
            gs = label - 1.f / (1.f + __expf(-f));
          } else if (f > kMaxExp) gs = label - 1.f;
          else if (f < -kMaxExp) gs = label;
          else gs = label - 1.f / (1.f + __expf(-f));
          {
            float z = label > 0.5f ? f : -f;
            z = fminf(fmaxf(z, -kMaxExp), kMaxExp);
            loss_acc += __logf(1.f + __expf(-z));
          }
          if (!skip) {
#pragma unroll
            for (int v = 0; v < VPL; ++v) {
              const int j = lane + v * 32;
              if (j < nvec) {
                const float4 e = reinterpret_cast<const float4*>(buf)[j];
                nu[v].x += gs * e.x; nu[v].y += gs * e.y; nu[v].z += gs * e.z; nu[v].w += gs * e.w;
                if (BULK) {
                  const float4 a = reinterpret_cast<const float4*>(buf + d)[j];
                  const float4 h = reinterpret_cast<const float4*>(scratch)[j];
                  const float4 gr = make_float4(gs * h.x, gs * h.y, gs * h.z, gs * h.w);
                  const float4 ua = make_float4(gr.x * gr.x, gr.y * gr.y, gr.z * gr.z, gr.w * gr.w);
                  float4 ue;
                  ue.x = alpha * gr.x * rsqrtf(a.x + ua.x);
                  ue.y = alpha * gr.y * rsqrtf(a.y + ua.y);
                  ue.z = alpha * gr.z * rsqrtf(a.z + ua.z);
                  ue.w = alpha * gr.w * rsqrtf(a.w + ua.w);
                  reinterpret_cast<float4*>(buf)[j] = ue;      // stage the update in place of the consumed row
                  reinterpret_cast<float4*>(buf + d)[j] = ua;
                }
              }
            }
            if (BULK) {
              __syncwarp();
              if (lane == 0) {
                // the staged update is visible to the TMA engine
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                bulk_red_s2g(const_cast<float*>(tr), buf, row_bytes);
              }
            }
            if (lane == src) { mark_pushed(t_mark, bits >> 2); my_gs = gs; }
            ++n_upd;
          }
        }
        if (i == n_x + n_tt - 1) {
          if (have_slow) {                 // neu1e of the targets that took the generic path
            __syncwarp();
#pragma unroll
            for (int v = 0; v < VPL; ++v) {
              const int j = lane + v * 32;
              if (j < nvec) {
                const float4 q = reinterpret_cast<const float4*>(scratch + d)[j];
                nu[v].x += q.x; nu[v].y += q.y; nu[v].z += q.z; nu[v].w += q.w;
              }
            }
          }
          if (SCORE) {
#pragma unroll
            for (int v = 0; v < VPL; ++v) {
              const int j = lane + v * 32;
              if (j < nvec) reinterpret_cast<float4*>(so.vecs + ((size_t)n_win + w) * d)[j] = nu[v];
            }
            n_upd += n_x;                  // the gather pass applies neu1e to every context occurrence
            if ((xmask >> lane) & 1) mark_pushed(x_mark, bits);
          }
        }
      } else {
        // ---- context occurrence (in place): neu1e against its AdaGrad half
        float* xr = (float*)__shfl_sync(0xffffffffu, (unsigned long long)x_row, src);
        if (xr == nullptr) {
          ++n_slow;
          slot_free();
          const Key xk = contexts[(size_t)w * nc + src];
          if (dev::slow_pull(c, xk, buf)) {
#pragma unroll
            for (int v = 0; v < VPL; ++v) {
              const int j = lane + v * 32;
              if (j < nvec) {
                const float4 a = reinterpret_cast<const float4*>(buf + d)[j];
                const float4 ua = make_float4(nu[v].x * nu[v].x, nu[v].y * nu[v].y, nu[v].z * nu[v].z, nu[v].w * nu[v].w);
                float4 ue;
                ue.x = alpha * nu[v].x * rsqrtf(a.x + ua.x);
                ue.y = alpha * nu[v].y * rsqrtf(a.y + ua.y);
                ue.z = alpha * nu[v].z * rsqrtf(a.z + ua.z);
                ue.w = alpha * nu[v].w * rsqrtf(a.w + ua.w);
                reinterpret_cast<float4*>(buf)[j] = ue;
                reinterpret_cast<float4*>(buf + d)[j] = ua;
              }
            }
            if (dev::slow_push(c, xk, buf)) ++n_upd;
          }
        } else {
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            const int j = lane + v * 32;
            if (j < nvec) {
              const float4 a = reinterpret_cast<const float4*>(buf + d)[j];
              const float4 ua = make_float4(nu[v].x * nu[v].x, nu[v].y * nu[v].y, nu[v].z * nu[v].z, nu[v].w * nu[v].w);
              float4 ue;
              ue.x = alpha * nu[v].x * rsqrtf(a.x + ua.x);
              ue.y = alpha * nu[v].y * rsqrtf(a.y + ua.y);
              ue.z = alpha * nu[v].z * rsqrtf(a.z + ua.z);
              ue.w = alpha * nu[v].w * rsqrtf(a.w + ua.w);
              reinterpret_cast<float4*>(buf)[j] = ue;
              reinterpret_cast<float4*>(buf + d)[j] = ua;
            }
          }
          __syncwarp();
          if (lane == 0) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            bulk_red_s2g(xr, buf, row_bytes);
          }
          if (lane == src) mark_pushed(x_mark, bits);
          ++n_upd;
        }
      }
      // exactly one bulk group per item (empty unless a reduction was issued): "all but the youngest group" in issue()
      // always means "the reduction that used the slot of the previous item"
      if (BULK && lane == 0) bulk_commit();
      __syncwarp();                        // all lanes are done with ring slot b
      if (i + DIST < n_items) issue(i + DIST);
    }
    if (SCORE && lane < n_t) so.gs[(size_t)w * n_t + lane] = my_gs;
  }
  if (BULK) { if (lane == 0) bulk_wait_all(); __syncwarp(); }   // every bulk reduction has been performed

  __syncwarp();
  if (SCORE && lane == 0) atomicAdd(fx_loss, (unsigned long long)__float2ll_rn(loss_acc * kFxLoss));
  else if (lane == 0 && loss_out) atomicAdd(loss_out, loss_acc);
  dev::flush_stats(stats, n_local, n_remote, n_slow, n_upd);
  dev::cta_exit(c);
}

// In place: 104 registers, so that one block of the sync round's kernels fits next to two step blocks per SM.
template <int VPL>
__global__ void __maxnreg__(104)
cbow_step_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ centers, const Key* __restrict__ contexts,
                 const Key* __restrict__ negatives, int n_win, int nc, int neg, int d, float alpha,
                 float* __restrict__ loss_out, unsigned long long* __restrict__ stats) {
  cbow_step_body<VPL, false>(c, centers, contexts, NegTargets{negatives, neg}, n_win, nc, d, alpha, loss_out, stats,
                             nullptr, CbowScoreOut{});
}

template <int VPL>
__global__ void __maxnreg__(128)
cbow_score_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ centers, const Key* __restrict__ contexts,
                  const Key* __restrict__ negatives, int n_win, int nc, int neg, int d,
                  unsigned long long* __restrict__ stats, unsigned long long* __restrict__ fx_loss,
                  const __grid_constant__ CbowScoreOut so) {
  cbow_step_body<VPL, true>(c, centers, contexts, NegTargets{negatives, neg}, n_win, nc, d, 0.f, nullptr, stats, fx_loss,
                            so);
}

template <int VPL>
__global__ void __maxnreg__(104)
hs_step_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ centers, const Key* __restrict__ contexts,
               const __grid_constant__ PathTargets ts, int n_win, int nc, int d, float alpha,
               float* __restrict__ loss_out, unsigned long long* __restrict__ stats) {
  cbow_step_body<VPL, false>(c, centers, contexts, ts, n_win, nc, d, alpha, loss_out, stats, nullptr, CbowScoreOut{});
}

template <int VPL>
__global__ void __maxnreg__(128)
hs_score_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ centers, const Key* __restrict__ contexts,
                const __grid_constant__ PathTargets ts, int n_win, int nc, int d, unsigned long long* __restrict__ stats,
                unsigned long long* __restrict__ fx_loss, const __grid_constant__ CbowScoreOut so) {
  cbow_step_body<VPL, true>(c, centers, contexts, ts, n_win, nc, d, 0.f, nullptr, stats, fx_loss, so);
}

// ---- deterministic one-GPU step: index, score, group by key, gather (sgns_det.cuh)
// Entry x = w * (n_t + nc) + s of a step: s < n_t target s of window w, else context occurrence s - n_t
// (Src::entry_key, Src::entry_counts).

// Gives every key of the step's entries a compact id (cidx[key], keys[id]) and looks its row up once (rowp[id]).
template <class Src>
__device__ __forceinline__ void det_index_body(const Ctx& c, const Key* __restrict__ centers,
                                               const Key* __restrict__ contexts, const Src& ts, int n_win, int nc,
                                               int* __restrict__ cidx, Key* __restrict__ keys,
                                               float** __restrict__ rowp, unsigned int* __restrict__ count) {
  const int per = ts.n_t() + nc;
  const long n = (long)n_win * per;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int w = (int)(i / per), s = (int)(i % per);
    const Key k = ts.entry_key(centers, contexts, nc, w, s);
    // (the plain load skips the atomic for keys that are already claimed: frequent words appear thousands of times)
    if (k >= 0 && cidx[k] == -1 && atomicCAS(cidx + k, -1, -2) == -1) {
      const unsigned r = atomicAdd(count, 1u);
      keys[r] = k;
      rowp[r] = home_row(c, k);
      cidx[k] = (int)r;
    }
  }
}

// SCATTER = false: cnt[id] = entries of key id. SCATTER = true: desc / kid of CSR position off[id] + i, i < cnt[id],
// describe the entries of key id; counts cnt back down to zero. A target adds g_t times the window's h (vector row w),
// a context occurrence 1 times the window's neu1e (vector row n_win + w).
template <bool SCATTER, class Src>
__device__ __forceinline__ void det_group_body(const Key* __restrict__ centers, const Key* __restrict__ contexts,
                                               const Src& ts, int n_win, int nc, const int* __restrict__ cidx,
                                               int* __restrict__ cnt, const int* __restrict__ off,
                                               int* __restrict__ kid, const float* __restrict__ gsb,
                                               GatherDesc* __restrict__ desc) {
  const int n_t = ts.n_t(), per = n_t + nc;
  const long n = (long)n_win * per;
  for (long x = (long)blockIdx.x * blockDim.x + threadIdx.x; x < n; x += (long)gridDim.x * blockDim.x) {
    const int w = (int)(x / per), s = (int)(x - (long)w * per);
    const Key k = ts.entry_key(centers, contexts, nc, w, s);
    if (!ts.entry_counts(centers, w, s, k)) continue;
    const int id = __ldg(cidx + k);
    if (!SCATTER) {
      atomicAdd(cnt + id, 1);
    } else {
      const int q = __ldg(off + id) + atomicSub(cnt + id, 1) - 1;
      GatherDesc e;
      if (s < n_t) {
        e.g = __ldg(gsb + (size_t)w * n_t + s);
        e.vec = e.g == kNoEntry ? 0 : w;
      } else {
        e.g = 1.f;
        e.vec = n_win + w;
      }
      desc[q] = e;
      kid[q] = id;
    }
  }
}

__global__ void cbow_det_index_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ centers,
                                      const Key* __restrict__ contexts, const Key* __restrict__ negatives, int n_win,
                                      int nc, int neg, int* __restrict__ cidx, Key* __restrict__ keys,
                                      float** __restrict__ rowp, unsigned int* __restrict__ count) {
  det_index_body(c, centers, contexts, NegTargets{negatives, neg}, n_win, nc, cidx, keys, rowp, count);
}
__global__ void hs_det_index_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ centers,
                                    const Key* __restrict__ contexts, const __grid_constant__ PathTargets ts, int n_win,
                                    int nc, int* __restrict__ cidx, Key* __restrict__ keys, float** __restrict__ rowp,
                                    unsigned int* __restrict__ count) {
  det_index_body(c, centers, contexts, ts, n_win, nc, cidx, keys, rowp, count);
}

template <bool SCATTER>
__global__ void cbow_det_group_kernel(const Key* __restrict__ centers, const Key* __restrict__ contexts,
                                      const Key* __restrict__ negatives, int n_win, int nc, int neg,
                                      const int* __restrict__ cidx, int* __restrict__ cnt, const int* __restrict__ off,
                                      int* __restrict__ kid, const float* __restrict__ gsb,
                                      GatherDesc* __restrict__ desc) {
  det_group_body<SCATTER>(centers, contexts, NegTargets{negatives, neg}, n_win, nc, cidx, cnt, off, kid, gsb, desc);
}
template <bool SCATTER>
__global__ void hs_det_group_kernel(const Key* __restrict__ centers, const Key* __restrict__ contexts,
                                    const __grid_constant__ PathTargets ts, int n_win, int nc,
                                    const int* __restrict__ cidx, int* __restrict__ cnt, const int* __restrict__ off,
                                    int* __restrict__ kid, const float* __restrict__ gsb,
                                    GatherDesc* __restrict__ desc) {
  det_group_body<SCATTER>(centers, contexts, ts, n_win, nc, cidx, cnt, off, kid, gsb, desc);
}

// The kernels of one target source.
template <class Src> struct StepKernels;
template <> struct StepKernels<NegTargets> {
  template <int V> static void step(int blocks, size_t smem, cudaStream_t st, const Ctx& c, const Key* centers,
                                    const Key* contexts, const NegTargets& ts, int n_win, int nc, int d, float alpha,
                                    float* loss_out, unsigned long long* stats) {
    set_max_dynamic_smem<cbow_step_kernel<V>>(110 * 1024);
    cbow_step_kernel<V><<<blocks, kThreads, smem, st>>>(c, centers, contexts, ts.negatives, n_win, nc, ts.neg, d, alpha,
                                                        loss_out, stats);
  }
  template <int V> static void score(int blocks, size_t smem, cudaStream_t st, const Ctx& c, const Key* centers,
                                     const Key* contexts, const NegTargets& ts, int n_win, int nc, int d,
                                     unsigned long long* stats, unsigned long long* fx_loss, const CbowScoreOut& so) {
    set_max_dynamic_smem<cbow_score_kernel<V>>(110 * 1024);
    cbow_score_kernel<V><<<blocks, kThreads, smem, st>>>(c, centers, contexts, ts.negatives, n_win, nc, ts.neg, d, stats,
                                                         fx_loss, so);
  }
  static void index(int blocks, cudaStream_t st, const Ctx& c, const Key* centers, const Key* contexts,
                    const NegTargets& ts, int n_win, int nc, int* cidx, Key* keys, float** rowp, unsigned int* count) {
    cbow_det_index_kernel<<<blocks, 256, 0, st>>>(c, centers, contexts, ts.negatives, n_win, nc, ts.neg, cidx, keys,
                                                  rowp, count);
  }
  template <bool SCATTER> static void group(int blocks, cudaStream_t st, const Key* centers, const Key* contexts,
                                            const NegTargets& ts, int n_win, int nc, const int* cidx, int* cnt,
                                            const int* off, int* kid, const float* gsb, GatherDesc* desc) {
    cbow_det_group_kernel<SCATTER><<<blocks, 256, 0, st>>>(centers, contexts, ts.negatives, n_win, nc, ts.neg, cidx, cnt,
                                                           off, kid, gsb, desc);
  }
};
template <> struct StepKernels<PathTargets> {
  template <int V> static void step(int blocks, size_t smem, cudaStream_t st, const Ctx& c, const Key* centers,
                                    const Key* contexts, const PathTargets& ts, int n_win, int nc, int d, float alpha,
                                    float* loss_out, unsigned long long* stats) {
    set_max_dynamic_smem<hs_step_kernel<V>>(110 * 1024);
    hs_step_kernel<V><<<blocks, kThreads, smem, st>>>(c, centers, contexts, ts, n_win, nc, d, alpha, loss_out, stats);
  }
  template <int V> static void score(int blocks, size_t smem, cudaStream_t st, const Ctx& c, const Key* centers,
                                     const Key* contexts, const PathTargets& ts, int n_win, int nc, int d,
                                     unsigned long long* stats, unsigned long long* fx_loss, const CbowScoreOut& so) {
    set_max_dynamic_smem<hs_score_kernel<V>>(110 * 1024);
    hs_score_kernel<V><<<blocks, kThreads, smem, st>>>(c, centers, contexts, ts, n_win, nc, d, stats, fx_loss, so);
  }
  static void index(int blocks, cudaStream_t st, const Ctx& c, const Key* centers, const Key* contexts,
                    const PathTargets& ts, int n_win, int nc, int* cidx, Key* keys, float** rowp, unsigned int* count) {
    hs_det_index_kernel<<<blocks, 256, 0, st>>>(c, centers, contexts, ts, n_win, nc, cidx, keys, rowp, count);
  }
  template <bool SCATTER> static void group(int blocks, cudaStream_t st, const Key* centers, const Key* contexts,
                                            const PathTargets& ts, int n_win, int nc, const int* cidx, int* cnt,
                                            const int* off, int* kid, const float* gsb, GatherDesc* desc) {
    hs_det_group_kernel<SCATTER><<<blocks, 256, 0, st>>>(centers, contexts, ts, n_win, nc, cidx, cnt, off, kid, gsb,
                                                         desc);
  }
};

template <class Src>
void cbow_step_det(CudaBackend& be, cudaStream_t stream, const Key* centers, const Key* contexts, const Src& ts,
                   int n_win, int nc, int d, float alpha, float* loss_out, unsigned long long* stats, int vpl,
                   int score_blocks, size_t smem) {
  using K = StepKernels<Src>;
  const Ctx& c = be.ctx();
  const int n_t = ts.n_t();
  const int n_entries = n_win * (n_t + nc);
  const int n_ids = (int)std::min<size_t>((size_t)n_entries, (size_t)c.L.num_keys);   // bound on the distinct keys
  const int n_ranges = (n_entries + kGatherRange - 1) / kGatherRange;
  CudaBackend::FxScratch& fx = be.fx_scratch(0, (size_t)n_ids, 0);
  CbowScoreOut so;
  so.gs = static_cast<float*>(be.step_buffer(kBufGs, (size_t)n_win * n_t * sizeof(float)));
  so.vecs = static_cast<float*>(be.step_buffer(kBufVec, (size_t)2 * n_win * d * sizeof(float)));
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
  K::index(blocks_for(n_entries), stream, c, centers, contexts, ts, n_win, nc, fx.cidx, fx.keys, rowp, fx.count);
  ADAPM_COUNT_LAUNCH();
  switch (vpl) {
    case 1: K::template score<1>(score_blocks, smem, stream, c, centers, contexts, ts, n_win, nc, d, stats, fx.loss, so); break;
    case 2: K::template score<2>(score_blocks, smem, stream, c, centers, contexts, ts, n_win, nc, d, stats, fx.loss, so); break;
    default: K::template score<3>(score_blocks, smem, stream, c, centers, contexts, ts, n_win, nc, d, stats, fx.loss, so); break;
  }
  ADAPM_COUNT_LAUNCH();
  K::template group<false>(blocks_for(n_entries), stream, centers, contexts, ts, n_win, nc, fx.cidx, cnt, off, kid, so.gs,
                           desc);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, cnt, off, n_ids + 1, stream));
  ADAPM_COUNT_LAUNCH();
  ADAPM_COUNT_LAUNCH();   // (the scan is two kernels)
  K::template group<true>(blocks_for(n_entries), stream, centers, contexts, ts, n_win, nc, fx.cidx, cnt, off, kid, so.gs,
                          desc);
  ADAPM_COUNT_LAUNCH();
  det_gather_finish(be, stream, vpl, rowp, off, n_ids, kid, desc, so.vecs, d, alpha, part, n_ranges,
                    blocks_for(n_entries), fx, loss_out);
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

// One step of either target source: the deterministic step or one in-place launch. The caller checks the arguments.
template <class Src>
void run_step(CudaBackend& be, cudaStream_t stream, const Key* centers, const Key* contexts, const Src& ts, int n_win,
              int nc, int d, float alpha, float* loss_out, unsigned long long* stats, bool deterministic) {
  const int vpl = (d / 4 + 31) / 32;
  const size_t buf_floats = ((size_t)2 * d + 31) & ~(size_t)31;
  const size_t smem = (size_t)kWarps * (RING + 1) * buf_floats * sizeof(float) + 128;   // <= 110 KB: 2 blocks per SM
  const int blocks = std::min((n_win + kWarps - 1) / kWarps, be.num_sms() * 12);
  if (deterministic) {
    cbow_step_det(be, stream, centers, contexts, ts, n_win, nc, d, alpha, loss_out, stats, vpl, blocks, smem);
    return;
  }
  using K = StepKernels<Src>;
  const Ctx& c = be.ctx();
  switch (vpl) {
    case 1: K::template step<1>(blocks, smem, stream, c, centers, contexts, ts, n_win, nc, d, alpha, loss_out, stats); break;
    case 2: K::template step<2>(blocks, smem, stream, c, centers, contexts, ts, n_win, nc, d, alpha, loss_out, stats); break;
    default: K::template step<3>(blocks, smem, stream, c, centers, contexts, ts, n_win, nc, d, alpha, loss_out, stats); break;
  }
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace

void cbow_step(CudaBackend& be, cudaStream_t stream, const Key* centers, const Key* contexts, const Key* negatives,
               int n_win, int nc, int neg, int d, float alpha, float* loss_out, unsigned long long* stats,
               bool deterministic) {
  ADAPM_CHECK(d % 4 == 0 && d >= 4 && d <= kCbowMaxDim, "cbow_step: embed_dim must be a multiple of 4 in [4, 336]");
  ADAPM_CHECK(neg >= 0 && neg + 1 <= kCbowMaxTargets, "cbow_step: 1 + negative must be at most 32");
  ADAPM_CHECK(nc >= 1 && nc <= kCbowMaxContexts, "cbow_step: 1 to 32 context columns");
  ADAPM_CHECK(!deterministic || be.ctx().L.world == 1, "cbow_step: the deterministic step needs a single-GPU store");
  if (n_win <= 0) return;
  ADAPM_CHECK((long)n_win * (neg + 1 + nc) < (1L << 30), "cbow_step: too many keys in one step");
  run_step(be, stream, centers, contexts, NegTargets{negatives, neg}, n_win, nc, d, alpha, loss_out, stats,
           deterministic);
}

void hs_step(CudaBackend& be, cudaStream_t stream, const Key* centers, const Key* contexts, int n_items, int nc,
             const int64_t* offsets, const int32_t* nodes, const uint32_t* codes, int n_words, int max_len, int d,
             float alpha, float* loss_out, unsigned long long* stats, bool deterministic) {
  ADAPM_CHECK(d % 4 == 0 && d >= 4 && d <= kCbowMaxDim, "hs_step: embed_dim must be a multiple of 4 in [4, 336]");
  ADAPM_CHECK(max_len >= 1 && max_len <= kCbowMaxTargets, "hs_step: the tree's paths must be 1 to 32 nodes long");
  ADAPM_CHECK(n_words >= 2, "hs_step: the tree needs at least 2 words");
  ADAPM_CHECK(nc >= 1 && nc <= kCbowMaxContexts, "hs_step: 1 to 32 context columns");
  ADAPM_CHECK(!deterministic || be.ctx().L.world == 1, "hs_step: the deterministic step needs a single-GPU store");
  if (n_items <= 0) return;
  ADAPM_CHECK((long)n_items * (max_len + nc) < (1L << 30), "hs_step: too many keys in one step");
  run_step(be, stream, centers, contexts, PathTargets{offsets, nodes, codes, n_words, max_len}, n_items, nc, d, alpha,
           loss_out, stats, deterministic);
}

}  // namespace cudaops
}  // namespace adapm

// The deterministic one-GPU word2vec steps (SGNS: ops_sgns_tma.cu; CBOW and hierarchical softmax: ops_cbow.cu) and the
// TMA rings of their kernels: mbarrier and bulk-copy helpers, the fixed-point scales, and one implementation of every
// pass but the score pass. det_step runs a step: det_index gives each key a compact id, the op's score pass reads
// start-of-step rows, det_group counts each key's entries and (after a scan) scatters them into a CSR grouped by key,
// and the gather and finish passes apply them. The passes are generic over an entry source, which says what each entry
// of the step is. The score pass describes every contribution to a row as GatherDesc{g, vec}: the row gains
// AdaGrad(g * vecs[vec]) in fixed point against its start-of-step accumulator. (The SGNS score pass applies a row with
// a single contribution itself, with the same arithmetic: fx_apply_one.)
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <type_traits>

#include "cuda_backend.h"
#include "fx_accum.cuh"
#include "pm_kernels.cuh"

namespace adapm {
namespace cudaops {

// off[0 .. n) = exclusive sum of the CSR positions of keys with cnt[0 .. n) entries (none for a key with one entry if
// singles_in_score); tmp null: sets bytes. Defined in ops_sgns_tma.cu, so that the extension carries one copy of cub's
// scan for all the steps.
void det_scan(void* tmp, size_t& bytes, const int* cnt, int* off, int n, bool singles_in_score, cudaStream_t stream);

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

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
// The g a score pass writes for an entry that adds nothing (a skipped target, a generic-path row, a skipped item). A
// real g is in [-1, 1] or NaN; 0 is a real g (and an SGNS center entry's "valid" mark), so it cannot be the marker.
constexpr float kNoEntry = __builtin_huge_valf();

// the key's row in this GPU's store (one GPU: rows do not move during a step)
__device__ __forceinline__ float* home_row(const Ctx& c, Key k) {
  const int32_t slot = __ldcg(slot_of(c, c.rank) + k);
  return slot >= 0 ? row_ptr<float>(c, c.rank, class_of_key(c, k), (uint32_t)slot) : nullptr;
}

// What one contribution (CSR position) adds to its key's row: g times row vec of the step's vector buffer, which the
// score pass fills (the entry source's desc() says which row); g = kNoEntry: nothing.
struct alignas(8) GatherDesc {
  float g;
  int vec;
};

// The fixed-point terms of one element of one contribution (gr = gs * e0 of a target, g0 of a center; a = the row's
// AdaGrad value at the start of the step), with the expressions of the in-place step. a + gr * gr is rounded twice (no
// FMA), so that every caller computes the same terms.
__device__ __forceinline__ void fx_terms(float gr, float a, float alpha, long long& se, long long& sa) {
  const float ua = __fmul_rn(gr, gr);
  const float ue = alpha * gr * rsqrtf(__fadd_rn(a, ua));
  se += __float2ll_rn(ue * kFxEmb);
  sa += __float2ll_rn(ua * kFxAda);
}
// row element r and its AdaGrad value a += their summed terms; a zero sum leaves the element as it is (a -0.0 stays -0.0)
__device__ __forceinline__ void fx_apply(float& r, float& a, long long se, long long sa) {
  if (se) r += (float)((double)se * (1.0 / (double)kFxEmb));
  if (sa) a += (float)((double)sa * (1.0 / (double)kFxAda));
}
// An element of a row with one contribution in the step gets exactly what the gather pass would give it: the score
// pass applies such rows itself.
__device__ __forceinline__ void fx_apply_one(float& r, float& a, float gr, float alpha) {
  long long se = 0, sa = 0;
  fx_terms(gr, a, alpha, se, sa);
  fx_apply(r, a, se, sa);
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
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            const int j = lane + v * 32;
            if (j < nvec) {
              float4 r = reinterpret_cast<const float4*>(rs)[j];
              float4 na = a[v];
              float* rp = &r.x;
              float* ap = &na.x;
#pragma unroll
              for (int q = 0; q < 4; ++q) fx_apply(rp[q], ap[q], se[v][q], sa[v][q]);
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
// Launches the gather pass over the n_ranges ranges of kGatherRange CSR positions and the finish pass (finish_blocks
// blocks of 256 threads) on `stream`: 2 launches.
inline void det_gather_finish(CudaBackend& be, cudaStream_t stream, int vpl, float* const* rowp, const int* off, int n_ids,
                              const int* kid, const GatherDesc* desc, const float* vecs, int d, float alpha,
                              long long* part, int n_ranges, int finish_blocks, CudaBackend::FxScratch& fx,
                              float* loss_out) {
  const Ctx& c = be.ctx();
  const int gather_blocks = (n_ranges + kWarps - 1) / kWarps;
  const auto gather = vpl == 1 ? sgns_det_gather_kernel<1> : vpl == 2 ? sgns_det_gather_kernel<2> : sgns_det_gather_kernel<3>;
  static bool gather_attr_set[4] = {};
  if (!gather_attr_set[vpl]) {          // room for the largest row of this VPL (d = 128 VPL)
    ADAPM_CUDA_CHECK(cudaFuncSetAttribute(gather, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)(kWarps * gather_warp_bytes(128 * vpl))));
    gather_attr_set[vpl] = true;
  }
  gather<<<gather_blocks, kThreads, kWarps * gather_warp_bytes(d), stream>>>(c, rowp, off, n_ids, kid, desc, vecs, d,
                                                                             alpha, part);
  ADAPM_COUNT_LAUNCH();
  sgns_det_finish_kernel<<<finish_blocks, 256, 0, stream>>>(c, fx.keys, rowp, off, n_ids, kid, d, part, fx.cidx,
                                                            fx.count, fx.loss, loss_out);
  ADAPM_COUNT_LAUNCH();
}

// ---- Before the gather: the step's entries are grouped by key (CSR: off / kid / desc), so that one warp owns each row
// and no accumulator per key and element is needed. Integer sums do not depend on the order of their terms, so the
// grouping may differ from run to run and the rows and loss do not. An entry source (a struct passed by value to the
// index and group kernels) says what entry x = i * per() + s of item i of the step is:
//   int items() const, int per() const        items of the step, entries per item
//   Key key(int i, int s) const                the entry's key (< 0: none)
//   bool counts(int i, int s, Key k) const     whether the entry adds anything to row k
//   GatherDesc desc(int i, int s, int x) const what it adds, from what the score pass wrote
//   float* gs                                  the score pass's g of each entry (det_step carves it, at most one per
//                                              entry; the layout is the source's)
//   static constexpr int kFirstSlots           slots [0, kFirstSlots) of every item are indexed first, so that their
//                                              keys get the compact ids 0 .. distinct - 1
//   static constexpr bool kSinglesInScore      the score pass applies a key with one entry itself: the key gets no CSR
//                                              position

// Gives every key of slots [first, first + n_slots) of each item a compact id (cidx[key], keys[id]) and looks its row
// up once (rowp[id]). cidx[key] goes -1 (no id) -> -2 (being claimed) -> id; the plain load skips the atomic for keys
// that are already claimed (frequent words appear thousands of times in a step).
template <class Src>
__device__ __forceinline__ void det_index(const Ctx& c, const Src& src, int first, int n_slots, int* __restrict__ cidx,
                                          Key* __restrict__ keys, float** __restrict__ rowp,
                                          unsigned int* __restrict__ count) {
  const int n = src.items() * n_slots;
  for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < n; x += gridDim.x * blockDim.x) {
    const int i = x / n_slots;
    const Key k = src.key(i, first + (x - i * n_slots));
    if (k >= 0 && cidx[k] == -1 && atomicCAS(cidx + k, -1, -2) == -1) {
      const unsigned r = atomicAdd(count, 1u);
      keys[r] = k;
      rowp[r] = home_row(c, k);
      cidx[k] = (int)r;
    }
  }
}

// SCATTER = false: cnt[id] = entries of key id. SCATTER = true: desc / kid of CSR positions off[id] + j, j < cnt[id],
// describe the entries of key id, and cnt counts back down to zero for the next step; a key without CSR positions
// (kSinglesInScore) has its count cleared.
template <bool SCATTER, class Src>
__device__ __forceinline__ void det_group(const Src& src, const int* __restrict__ cidx, int* __restrict__ cnt,
                                          const int* __restrict__ off, int* __restrict__ kid,
                                          GatherDesc* __restrict__ desc) {
  const int per = src.per();
  const int n = src.items() * per;
  for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < n; x += gridDim.x * blockDim.x) {
    const int i = x / per, s = x - i * per;
    const Key k = src.key(i, s);
    if (!src.counts(i, s, k)) continue;
    const int id = __ldg(cidx + k);
    if (!SCATTER) {
      atomicAdd(cnt + id, 1);
      continue;
    }
    const int q0 = __ldg(off + id);
    if (Src::kSinglesInScore && __ldg(off + id + 1) == q0) {
      cnt[id] = 0;
      continue;
    }
    const int q = q0 + atomicSub(cnt + id, 1) - 1;
    desc[q] = src.desc(i, s, x);
    kid[q] = id;
  }
}

// f(std::integral_constant<int, VPL>) for the float4-per-lane count of a row (1, 2 or 3)
template <class F>
void by_vpl(int vpl, F&& f) {
  switch (vpl) {
    case 1: f(std::integral_constant<int, 1>{}); break;
    case 2: f(std::integral_constant<int, 2>{}); break;
    default: f(std::integral_constant<int, 3>{}); break;
  }
}

// The deterministic one-GPU step of entry source src on `stream`: index (kFirstSlots first), score, count, scan,
// scatter, gather, finish - 9 launches with kFirstSlots, else 8. Index, Count and Scatter are the source's det_index,
// det_group<false> and det_group<true> kernels. score(gs, vecs, cnt, fx) launches the op's score pass (one kernel) with
// the buffers carved here: the entries' g, the vector buffer (vec_rows rows of d floats) that the descriptors point
// into, and each key's entry count by compact id. A kSinglesInScore pass reads the counts, so it runs after the scan;
// any other runs right after the index, and the host enqueues the short count and scan passes while the GPU runs it.
// The caller checks that the step's entries fit an int.
template <auto Index, auto Count, auto Scatter, class Src, class Score>
void det_step(CudaBackend& be, cudaStream_t stream, Src src, size_t vec_rows, int d, float alpha, int vpl,
              float* loss_out, Score&& score) {
  const Ctx& c = be.ctx();
  const int n_entries = src.items() * src.per();
  const int n_ids = (int)std::min<size_t>((size_t)n_entries, (size_t)c.L.num_keys);   // bound on the distinct keys
  const int n_ranges = (n_entries + kGatherRange - 1) / kGatherRange;
  CudaBackend::FxScratch& fx = be.fx_scratch(0, (size_t)n_ids, 0);
  src.gs = static_cast<float*>(be.step_buffer(kBufGs, (size_t)n_entries * sizeof(float)));
  float* vecs = static_cast<float*>(be.step_buffer(kBufVec, vec_rows * d * sizeof(float)));
  int* cnt = static_cast<int*>(be.step_buffer(kBufCnt, ((size_t)n_ids + 1) * sizeof(int)));    // zero between steps
  int* off = static_cast<int*>(be.step_buffer(kBufOff, ((size_t)n_ids + 1) * sizeof(int)));
  GatherDesc* desc = static_cast<GatherDesc*>(be.step_buffer(kBufDesc, (size_t)n_entries * sizeof(GatherDesc)));
  int* kid = static_cast<int*>(be.step_buffer(kBufKid, (size_t)n_entries * sizeof(int)));
  long long* part = static_cast<long long*>(                                            // zero between steps
      be.step_buffer(kBufPart, ((size_t)n_ranges + 1) * 2 * d * sizeof(long long)));
  float** rowp = static_cast<float**>(be.step_buffer(kBufRowp, (size_t)n_ids * sizeof(float*)));
  size_t scan_bytes = 0;
  det_scan(nullptr, scan_bytes, cnt, off, n_ids + 1, Src::kSinglesInScore, stream);
  void* scan_tmp = be.step_buffer(kBufScan, scan_bytes);

  const int grid_n = be.num_sms() * 8;
  auto blocks_for = [&](long n) { return (int)std::max<long>(1, std::min<long>((n + 255) / 256, grid_n)); };
  ADAPM_CUDA_CHECK(cudaMemsetAsync(fx.count, 0, 2 * sizeof(unsigned int), stream));
  constexpr int first = Src::kFirstSlots;
  if (first > 0) {
    Index<<<blocks_for((long)src.items() * first), 256, 0, stream>>>(c, src, 0, first, fx.cidx, fx.keys, rowp,
                                                                     fx.count);
    ADAPM_COUNT_LAUNCH();
  }
  Index<<<blocks_for((long)src.items() * (src.per() - first)), 256, 0, stream>>>(c, src, first, src.per() - first,
                                                                                 fx.cidx, fx.keys, rowp, fx.count);
  ADAPM_COUNT_LAUNCH();
  if constexpr (!Src::kSinglesInScore) {
    score(src.gs, vecs, static_cast<const int*>(cnt), fx);
    ADAPM_COUNT_LAUNCH();
  }
  Count<<<blocks_for(n_entries), 256, 0, stream>>>(src, fx.cidx, cnt, off, kid, desc);
  ADAPM_COUNT_LAUNCH();
  det_scan(scan_tmp, scan_bytes, cnt, off, n_ids + 1, Src::kSinglesInScore, stream);
  ADAPM_COUNT_LAUNCH();
  ADAPM_COUNT_LAUNCH();   // (the scan is two kernels)
  if constexpr (Src::kSinglesInScore) {
    score(src.gs, vecs, static_cast<const int*>(cnt), fx);
    ADAPM_COUNT_LAUNCH();
  }
  Scatter<<<blocks_for(n_entries), 256, 0, stream>>>(src, fx.cidx, cnt, off, kid, desc);
  ADAPM_COUNT_LAUNCH();
  det_gather_finish(be, stream, vpl, rowp, off, n_ids, kid, desc, vecs, d, alpha, part, n_ranges, blocks_for(n_entries),
                    fx, loss_out);
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace
}  // namespace cudaops
}  // namespace adapm

// Paragraph-vector (doc2vec) inference for sm_90a: one new vector per document, trained against frozen store rows.
//
// Document m has the words w_0 .. w_{L-1} (tokens[offsets[m] .. offsets[m + 1])) and the caller's id t = doc_ids[m].
// With base = mix64(mix64(seed) ^ t):
//   initial state  v_k = (u_k - 0.5) / d with u_k = (mix64(base ^ (2^63 | k)) >> 40) 2^-24, a_k = 1e-6;
//   epoch seed     es = mix64(base ^ (2^62 | e)); draw n of the epoch is the sampler's hash with seed es, try 0
//                  (mix64(es ^ n * 0x9E3779B97F4A7C15) into draw_key), so ops.sample_keys_reference replays it;
//   PV-DM shrink   b = mix64(mix64(es) ^ i) mod window at position i.
// Each epoch visits the positions in order. Targets: syn1(w_i) with label 1, then the draws i * negative + j with label
// 0 (a draw equal to the positive is skipped). Input h = v (PV-DBOW) or (v + the syn0 rows of the positions i' != i
// with |i' - i| <= window - b) / (1 + C) (PV-DM, mean). g = label - sigmoid(h . row), saturated at |f| > 6 as in
// training, neu1e = sum g row, then v += alpha_e neu1e / sqrt(a + neu1e^2) and a += neu1e^2. The summed logistic loss
// is added to *loss. Store rows are only read; (v | a) lives in state [M, 2d] between the per-epoch launches.
//
// One warp per document: lane l holds the float4 chunks l, l + 32, l + 64 of v, a, h and neu1e in registers (d <= 336).
// A position's keys are resolved in parallel, one per lane (resolve_fast, then gather_locate for keys in a transitional
// state), and each row is read by the whole warp through ld_gather4 / gather_reread, so peer rows, replicas and keys
// in flight read correctly. Targets go in groups of four, so four rows are in flight and four dot products reduce
// together. A document's result depends on its words, its id, the seed and the rows only: not on the batch it is in.
#include <cuda_runtime.h>

#include <cmath>

#include "hash.cuh"
#include "ops.h"
#include "pm_kernels.cuh"
#include "sampler_draw.cuh"

namespace adapm {
namespace cudaops {

namespace {

constexpr int kDocWarps = 4;      // documents per CTA
constexpr int kVecs = 3;          // float4 chunks per lane: d <= 4 * 32 * 3
constexpr int kGroup = 4;         // target rows in flight

struct InferArgs {
  Ctx c;
  const int64_t* tokens;
  const int64_t* offsets;
  const int64_t* doc_ids;
  int64_t M;
  int d, negative, window, epoch;
  float alpha;
  uint64_t seed;
  int kind;
  const float* prob;
  const int32_t* alias;
  int64_t n_table;
  double lg;
  Key first, stride;
  float* state;
  float* loss;
  unsigned long long* stats;      // [3]: stats[2] += rows that could not be resolved (read as zeros)
};

__device__ __forceinline__ dev::GatherRow shfl_row(const dev::GatherRow& r, int src) {
  dev::GatherRow o;
  o.row = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)r.row, src);
  o.base = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)r.base, src);
  o.row2 = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)r.row2, src);
  o.meta_ptr = (const uint32_t*)__shfl_sync(0xffffffffu, (unsigned long long)r.meta_ptr, src);
  o.meta_val = __shfl_sync(0xffffffffu, r.meta_val, src);
  o.local = false;
  return o;
}

// one lane: where key's row is read
__device__ __forceinline__ dev::GatherRow locate(const Ctx& c, Key key, unsigned* n_bad) {
  unsigned nl = 0, nr = 0;
  dev::GatherRow r = {nullptr, nullptr, nullptr, nullptr, 0u, false};
  r.row = dev::resolve_fast(c, key, class_of_key(c, key), &nl, &nr).row;
  if (!r.row) {
    r = dev::gather_locate(c, key);
    if (!r.row) ++*n_bad;
  }
  return r;
}

// the whole warp: this lane's chunks of the row of `key` (zeros if it could not be resolved)
__device__ __forceinline__ void load_row(const Ctx& c, Key key, dev::GatherRow& r, int d, int lane, float4 (&x)[kVecs]) {
  do {
#pragma unroll
    for (int q = 0; q < kVecs; ++q) {
      const int k = 4 * (lane + 32 * q);
      x[q] = (r.row && k < d) ? dev::ld_gather4(r, k) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  } while (dev::gather_reread(c, key, r));
}

__device__ __forceinline__ float dot4(const float4& a, const float4& b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }

__device__ __forceinline__ void axpy4(float4& y, float g, const float4& x) {
  y.x += g * x.x; y.y += g * x.y; y.z += g * x.z; y.w += g * x.w;
}

template <bool DM>
__global__ void __launch_bounds__(32 * kDocWarps, 1) doc2vec_infer_kernel(const __grid_constant__ InferArgs p) {
  const Ctx& c = p.c;
  dev::cta_enter(c);   // the warps read store rows through the directory: count this CTA in the grace epoch
  const int lane = threadIdx.x & 31;
  const int64_t m = (int64_t)blockIdx.x * kDocWarps + (threadIdx.x >> 5);
  unsigned n_bad = 0;
  if (m < p.M) {
    const int d = p.d;
    const int64_t* w = p.tokens + __ldg(p.offsets + m);
    const int L = (int)(__ldg(p.offsets + m + 1) - __ldg(p.offsets + m));
    const uint64_t base = mix64(mix64(p.seed) ^ (uint64_t)__ldg(p.doc_ids + m));
    const uint64_t es = mix64(base ^ ((1ull << 62) | (uint64_t)p.epoch));
    const uint64_t shrink_seed = mix64(es);
    float* st = p.state + m * 2 * (int64_t)d;
    float4 v[kVecs], a[kVecs];
#pragma unroll
    for (int q = 0; q < kVecs; ++q) {
      const int k = 4 * (lane + 32 * q);
      // chunks past d stay v = 0 with a > 0: their neu1e is 0, so their update is 0 / sqrt(a) = 0, never 0 / 0
      v[q] = make_float4(0.f, 0.f, 0.f, 0.f);
      a[q] = make_float4(1e-6f, 1e-6f, 1e-6f, 1e-6f);
      if (k >= d) continue;
      if (p.epoch == 0) {
        float u[4];
#pragma unroll
        for (int e = 0; e < 4; ++e)
          u[e] = ((float)(uint32_t)(mix64(base ^ ((1ull << 63) | (uint64_t)(k + e))) >> 40) * 0x1p-24f - 0.5f) / (float)d;
        v[q] = make_float4(u[0], u[1], u[2], u[3]);
      } else {
        v[q] = *reinterpret_cast<const float4*>(st + k);
        a[q] = *reinterpret_cast<const float4*>(st + d + k);
      }
    }
    const int NT = 1 + p.negative;
    float loss = 0.f;
    for (int i = 0; i < L; ++i) {
      // ---- keys of this position, one per lane: lane j < NT the target j, lane j < C (PV-DM) context j
      const Key pos_key = 2 * __ldg(w + i) + 1;
      Key tkey = pos_key;
      if (lane >= 1 && lane < NT) {
        const uint64_t n = (uint64_t)i * (uint64_t)p.negative + (uint64_t)(lane - 1);
        tkey = draw_key(p.kind, p.prob, p.alias, p.n_table, p.lg, p.first, p.stride,
                        mix64(es ^ (n * 0x9E3779B97F4A7C15ULL)));
      }
      const bool tvalid = lane < NT && (lane == 0 || tkey != pos_key);
      const dev::GatherRow trow = tvalid ? locate(c, tkey, &n_bad) : dev::GatherRow{nullptr, nullptr, nullptr, nullptr, 0u, false};
      float4 h[kVecs];
#pragma unroll
      for (int q = 0; q < kVecs; ++q) h[q] = v[q];
      if (DM) {
        const int r = p.window - (int)(mix64(shrink_seed ^ (uint64_t)i) % (uint64_t)p.window);
        const int lo = max(0, i - r), hi = min(L, i + r + 1);
        const int C = hi - lo - 1;
        const int ip = lo + lane + (lo + lane >= i ? 1 : 0);   // lane j's context position
        const Key ckey = lane < C ? 2 * __ldg(w + ip) : 0;
        const dev::GatherRow crow = lane < C ? locate(c, ckey, &n_bad) : dev::GatherRow{nullptr, nullptr, nullptr, nullptr, 0u, false};
        for (int j = 0; j < C; ++j) {
          const Key kj = __shfl_sync(0xffffffffu, ckey, j);
          dev::GatherRow rj = shfl_row(crow, j);
          float4 x[kVecs];
          load_row(c, kj, rj, d, lane, x);
#pragma unroll
          for (int q = 0; q < kVecs; ++q) axpy4(h[q], 1.f, x[q]);
        }
        const float n1 = (float)(1 + C);
#pragma unroll
        for (int q = 0; q < kVecs; ++q) { h[q].x /= n1; h[q].y /= n1; h[q].z /= n1; h[q].w /= n1; }
      }
      // ---- targets, kGroup rows in flight
      float4 neu[kVecs];
#pragma unroll
      for (int q = 0; q < kVecs; ++q) neu[q] = make_float4(0.f, 0.f, 0.f, 0.f);
      const unsigned valid_mask = __ballot_sync(0xffffffffu, tvalid);
      for (int j0 = 0; j0 < NT; j0 += kGroup) {
        float4 x[kGroup][kVecs];
        float f[kGroup];
#pragma unroll
        for (int u = 0; u < kGroup; ++u) {
          const int j = j0 + u;
          const Key kj = __shfl_sync(0xffffffffu, tkey, j & 31);
          dev::GatherRow rj = shfl_row(trow, j & 31);
          if (j < NT && ((valid_mask >> j) & 1u)) {
            load_row(c, kj, rj, d, lane, x[u]);
          } else {
#pragma unroll
            for (int q = 0; q < kVecs; ++q) x[u][q] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
          f[u] = 0.f;
#pragma unroll
          for (int q = 0; q < kVecs; ++q) f[u] += dot4(h[q], x[u][q]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
          for (int u = 0; u < kGroup; ++u) f[u] += __shfl_xor_sync(0xffffffffu, f[u], o);
        }
#pragma unroll
        for (int u = 0; u < kGroup; ++u) {
          const int j = j0 + u;
          if (j >= NT || !((valid_mask >> j) & 1u)) continue;
          const float label = j == 0 ? 1.f : 0.f;
          const float g = f[u] > 6.f ? label - 1.f : (f[u] < -6.f ? label : label - 1.f / (1.f + expf(-f[u])));
          const float z = fminf(6.f, fmaxf(-6.f, j == 0 ? f[u] : -f[u]));
          loss += log1pf(expf(-z));
#pragma unroll
          for (int q = 0; q < kVecs; ++q) axpy4(neu[q], g, x[u][q]);
        }
      }
      // ---- AdaGrad update of the document vector
#pragma unroll
      for (int q = 0; q < kVecs; ++q) {
        const float4 g = neu[q];
        const float4 g2 = make_float4(g.x * g.x, g.y * g.y, g.z * g.z, g.w * g.w);
        v[q].x += p.alpha * g.x / sqrtf(a[q].x + g2.x);
        v[q].y += p.alpha * g.y / sqrtf(a[q].y + g2.y);
        v[q].z += p.alpha * g.z / sqrtf(a[q].z + g2.z);
        v[q].w += p.alpha * g.w / sqrtf(a[q].w + g2.w);
        a[q].x += g2.x; a[q].y += g2.y; a[q].z += g2.z; a[q].w += g2.w;
      }
    }
#pragma unroll
    for (int q = 0; q < kVecs; ++q) {
      const int k = 4 * (lane + 32 * q);
      if (k >= d) continue;
      *reinterpret_cast<float4*>(st + k) = v[q];
      *reinterpret_cast<float4*>(st + d + k) = a[q];
    }
    if (lane == 0 && p.loss && L > 0) atomicAdd(p.loss, loss);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n_bad += __shfl_xor_sync(0xffffffffu, n_bad, o);
  if (lane == 0 && n_bad && p.stats) atomicAdd(p.stats + 2, (unsigned long long)n_bad);
  dev::cta_exit(c);
}

}  // namespace

void doc2vec_infer_epoch(CudaBackend& be, cudaStream_t stream, const int64_t* tokens, const int64_t* offsets,
                         const int64_t* doc_ids, int64_t M, bool dm, int d, int negative, int window, int epoch,
                         float alpha, uint64_t seed, int kind, const float* prob, const int32_t* alias, int64_t n_table,
                         Key first, Key stride, float* state, float* loss, unsigned long long* stats) {
  ADAPM_CHECK(d >= 4 && d <= kDoc2VecMaxDim && d % 4 == 0,
              "doc2vec_infer: embed_dim must be a multiple of 4 in [4, " << kDoc2VecMaxDim << "], got " << d);
  ADAPM_CHECK(negative >= 1 && 1 + negative <= kDoc2VecMaxTargets,
              "doc2vec_infer: negative must be in [1, " << kDoc2VecMaxTargets - 1 << "], got " << negative);
  ADAPM_CHECK(!dm || (window >= 1 && window <= kDoc2VecMaxWindow),
              "doc2vec_infer: PV-DM needs 1 <= window <= " << kDoc2VecMaxWindow << ", got " << window);
  ADAPM_CHECK(be.ctx().L.val_bytes == 4, "the fused ops need float32 rows (Options::dtype)");
  ADAPM_CHECK(n_table >= 1 && n_table < (kind == 0 ? ((int64_t)1 << 31) : ((int64_t)1 << 32)),
              "doc2vec_infer: bad sampler table size " << n_table);
  ADAPM_CHECK(M >= 0 && M < ((int64_t)1 << 31) * kDocWarps, "doc2vec_infer: too many documents in one call: " << M);
  if (M == 0) return;
  be.track_stream(stream);
  InferArgs a{be.ctx(), tokens, offsets, doc_ids, M, d, negative, dm ? window : 1, epoch, alpha, seed, kind, prob,
              alias, n_table, std::log((double)(n_table + 1)), first, stride, state, loss, stats};
  const int blocks = (int)((M + kDocWarps - 1) / kDocWarps);
  if (dm) doc2vec_infer_kernel<true><<<blocks, 32 * kDocWarps, 0, stream>>>(a);
  else doc2vec_infer_kernel<false><<<blocks, 32 * kDocWarps, 0, stream>>>(a);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

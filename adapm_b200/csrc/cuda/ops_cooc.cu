// GloVe's co-occurrence matrix (glove.c's cooccur.c) of an encoded corpus, counted on the device for sm_90a.
//
// X[a][b] sums 1 / k over every pair of positions of one sentence where word a comes k <= window positions before word
// b (1 instead of 1 / k without distance weighting), and with symmetric also X[b][a]. Every weight is an integer
// numerator over Lw = lcm(1..window) (<= 720720 at window 16; Lw = 1 without distance weighting); the numerators are
// summed in 64-bit integers and each sum is divided by Lw once at the end (in float64, then rounded to float32). The
// result therefore depends on nothing but the corpus: not on the chunking, the launch configuration or the order of
// the sums. A rank keeps only rows a with a % world == rank, so `world` ranks that each count the whole corpus build
// disjoint row partitions of the full matrix without communicating.
//
// The tokens are processed in chunks whose working set fits max_bytes next to the running result:
//   room      per token, how many later positions of its sentence are within the window (uint8, whole corpus, once)
//   count     per token of the chunk, the entries it makes (int32), then an exclusive scan (cub) for their positions
//   expand    the entries (key a * V + b as uint64, numerator as uint32), in token order
//   sort      cub radix sort of the entries by key (only the bits V * V needs)
//   reduce    cub reduce-by-key into (key, int64 sum): the chunk's matrix, sorted
//   merge     cub merge with the running result, then reduce-by-key again (a key appears at most twice)
// A chunk starts at the size the budget allows at the worst case of window * (1 + symmetric) entries per token, or at
// the last chunk's measured rate; a chunk whose count exceeds the budget is shrunk and counted again.
#include <cuda_runtime.h>

#include <cub/cub.cuh>

#include <algorithm>
#include <numeric>

#include "group.cuh"
#include "ops.h"

namespace adapm {
namespace cudaops {

namespace {

constexpr int kThreads = 256;

// Device memory freed on scope exit (the call's working set; nothing outlives run() but the result).
template <class T>
struct Buf {
  T* p = nullptr;
  size_t n = 0;
  Buf() = default;
  explicit Buf(size_t count) : n(count) {
    if (count) ADAPM_CUDA_CHECK(cudaMalloc(&p, count * sizeof(T)));
  }
  Buf(const Buf&) = delete;
  Buf& operator=(const Buf&) = delete;
  Buf(Buf&& o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
  Buf& operator=(Buf&& o) noexcept {
    if (this != &o) { release(); p = o.p; n = o.n; o.p = nullptr; o.n = 0; }
    return *this;
  }
  ~Buf() { release(); }
  void release() {
    if (p) cudaFree(p);
    p = nullptr; n = 0;
  }
};

struct Params {
  const int32_t* tok;
  const uint8_t* room;
  int64_t t0, n;               // the chunk: tokens [t0, t0 + n)
  uint64_t V;
  uint32_t lw;                 // numerator of distance k: lw / k (distance weighting) or 1
  int rank, world;
  bool sym, dw;
};

__global__ void __launch_bounds__(kThreads)
cooc_room_kernel(const int64_t* __restrict__ off, int64_t ns, int64_t n_tokens, int window, uint8_t* __restrict__ room) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n_tokens; p += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = ns;                    // the sentence s with off[s] <= p < off[s + 1]
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) >> 1;
      if (__ldg(off + mid) <= p) lo = mid; else hi = mid;
    }
    room[p] = (uint8_t)min((int64_t)window, __ldg(off + lo + 1) - 1 - p);
  }
}

__device__ __forceinline__ bool mine(const Params& P, int32_t w) { return (int)((uint32_t)w % (uint32_t)P.world) == P.rank; }

__global__ void __launch_bounds__(kThreads)
cooc_count_kernel(const Params P, int32_t* __restrict__ cnt) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P.n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = P.t0 + i;
    const int r = P.room[p];
    const int a = P.tok[p];
    int c = mine(P, a) ? r : 0;
    if (P.sym)
      for (int k = 1; k <= r; ++k) c += mine(P, P.tok[p + k]);
    cnt[i] = c;
  }
}

__global__ void __launch_bounds__(kThreads)
cooc_expand_kernel(const Params P, const int32_t* __restrict__ pos, uint64_t* __restrict__ keys,
                   uint32_t* __restrict__ nums) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P.n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = P.t0 + i;
    const int r = P.room[p];
    const int32_t a = P.tok[p];
    const bool ma = mine(P, a);
    int64_t o = pos[i];
    for (int k = 1; k <= r; ++k) {
      const int32_t b = P.tok[p + k];
      const uint32_t num = P.dw ? P.lw / (uint32_t)k : 1u;
      if (ma) { keys[o] = (uint64_t)a * P.V + (uint64_t)b; nums[o] = num; ++o; }
      if (P.sym && mine(P, b)) { keys[o] = (uint64_t)b * P.V + (uint64_t)a; nums[o] = num; ++o; }
    }
  }
}

__global__ void __launch_bounds__(kThreads)
cooc_finish_kernel(const uint64_t* __restrict__ keys, const long long* __restrict__ sums, int64_t n, uint64_t V,
                   double lw, int32_t* __restrict__ rows, int32_t* __restrict__ cols, float* __restrict__ x) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t k = keys[i];
    rows[i] = (int32_t)(k / V);
    cols[i] = (int32_t)(k % V);
    x[i] = __double2float_rn(__ddiv_rn((double)sums[i], lw));
  }
}

struct Widen {
  __host__ __device__ __forceinline__ long long operator()(uint32_t v) const { return (long long)v; }
};
struct Add {
  __host__ __device__ __forceinline__ long long operator()(long long a, long long b) const { return a + b; }
};
struct Less {
  __host__ __device__ __forceinline__ bool operator()(uint64_t a, uint64_t b) const { return a < b; }
};

int grid_for(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + kThreads - 1) / kThreads, 1 << 16)); }

int key_bits(uint64_t V) {
  const uint64_t top = V * V - 1;
  int b = 1;
  while (b < 64 && (top >> b)) ++b;
  return b;
}

// The result so far: unique sorted keys and their numerator sums.
struct Matrix {
  Buf<uint64_t> keys;
  Buf<long long> sums;
  int64_t n = 0;
};

}  // namespace

struct Cooccurrence::Impl {
  cudaStream_t stream;
  const int32_t* tokens;
  int64_t n_tokens;
  const int64_t* offsets;
  int64_t n_sentences;
  uint64_t V;
  int window;
  bool sym, dw;
  int rank, world;
  int64_t max_bytes;
  Matrix result;

  int64_t fetch(const int32_t* p) const {
    int32_t v = 0;
    ADAPM_CUDA_CHECK(cudaMemcpyAsync(&v, p, sizeof(v), cudaMemcpyDeviceToHost, stream));
    ADAPM_CUDA_CHECK(cudaStreamSynchronize(stream));
    return v;
  }
  int64_t fetch(const int64_t* p) const {
    int64_t v = 0;
    ADAPM_CUDA_CHECK(cudaMemcpyAsync(&v, p, sizeof(v), cudaMemcpyDeviceToHost, stream));
    ADAPM_CUDA_CHECK(cudaStreamSynchronize(stream));
    return v;
  }

  // the sorted, reduced (key, sum) pairs of keys / nums [0, E) into out (room for E entries)
  void sort_reduce(cub::DoubleBuffer<uint64_t>& k, cub::DoubleBuffer<uint32_t>& v, int64_t E, Matrix& out) {
    size_t bytes = 0;
    const int bits = key_bits(V);
    ADAPM_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, k, v, (int)E, 0, bits, stream));
    {
      Buf<char> tmp(bytes);
      ADAPM_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(tmp.p, bytes, k, v, (int)E, 0, bits, stream));
      ADAPM_COUNT_LAUNCH();
    }
    cub::TransformInputIterator<long long, Widen, const uint32_t*> wide(v.Current(), Widen{});
    Buf<int64_t> nr(1);
    bytes = 0;
    ADAPM_CUDA_CHECK(cub::DeviceReduce::ReduceByKey(nullptr, bytes, k.Current(), out.keys.p, wide, out.sums.p, nr.p,
                                                    Add{}, E, stream));
    Buf<char> tmp(bytes);
    ADAPM_CUDA_CHECK(cub::DeviceReduce::ReduceByKey(tmp.p, bytes, k.Current(), out.keys.p, wide, out.sums.p, nr.p, Add{},
                                                    E, stream));
    ADAPM_COUNT_LAUNCH();
    out.n = fetch(nr.p);
  }

  // result += c (both sorted and unique)
  void merge(Matrix& c) {
    if (result.n == 0) { result = std::move(c); return; }
    const int64_t n = result.n + c.n;
    ADAPM_CHECK(n < (int64_t)INT32_MAX, "glove_cooccurrence: more than 2^31 entries to merge");
    Matrix m;
    m.keys = Buf<uint64_t>(n);
    m.sums = Buf<long long>(n);
    size_t bytes = 0;
    ADAPM_CUDA_CHECK(cub::DeviceMerge::MergePairs(nullptr, bytes, result.keys.p, result.sums.p, (int)result.n, c.keys.p,
                                                  c.sums.p, (int)c.n, m.keys.p, m.sums.p, Less{}, stream));
    {
      Buf<char> tmp(bytes);
      ADAPM_CUDA_CHECK(cub::DeviceMerge::MergePairs(tmp.p, bytes, result.keys.p, result.sums.p, (int)result.n, c.keys.p,
                                                    c.sums.p, (int)c.n, m.keys.p, m.sums.p, Less{}, stream));
      ADAPM_COUNT_LAUNCH();
      ADAPM_CUDA_CHECK(cudaStreamSynchronize(stream));
    }
    result = Matrix();
    c = Matrix();
    Matrix r;
    r.keys = Buf<uint64_t>(n);
    r.sums = Buf<long long>(n);
    Buf<int64_t> nr(1);
    bytes = 0;
    ADAPM_CUDA_CHECK(cub::DeviceReduce::ReduceByKey(nullptr, bytes, m.keys.p, r.keys.p, m.sums.p, r.sums.p, nr.p, Add{}, n,
                                                    stream));
    Buf<char> tmp(bytes);
    ADAPM_CUDA_CHECK(cub::DeviceReduce::ReduceByKey(tmp.p, bytes, m.keys.p, r.keys.p, m.sums.p, r.sums.p, nr.p, Add{}, n,
                                                    stream));
    ADAPM_COUNT_LAUNCH();
    r.n = fetch(nr.p);
    result = std::move(r);
  }
};

Cooccurrence::Cooccurrence(cudaStream_t stream, const int32_t* tokens, int64_t n_tokens, const int64_t* offsets,
                           int64_t n_sentences, int64_t V, int window, bool symmetric, bool distance_weighting, int rank,
                           int world, int64_t max_bytes) {
  ADAPM_CHECK(window >= 1 && window <= kCoocMaxWindow, "glove_cooccurrence: window must be in [1, " << kCoocMaxWindow << "]");
  ADAPM_CHECK(world >= 1 && rank >= 0 && rank < world, "glove_cooccurrence: bad rank / world");
  ADAPM_CHECK(V >= 1 && V <= INT32_MAX, "glove_cooccurrence: the vocabulary must have 1 .. 2^31 - 1 words");
  ADAPM_CHECK(n_tokens >= 0 && n_sentences >= 0 && max_bytes > 0, "glove_cooccurrence: bad sizes");
  impl_ = new Impl{stream, tokens, n_tokens, offsets, n_sentences, (uint64_t)V, window, symmetric, distance_weighting,
                   rank, world, max_bytes, Matrix()};
  if (distance_weighting)
    for (int k = 2; k <= window; ++k) lw_ = std::lcm(lw_, (int64_t)k);
}

Cooccurrence::~Cooccurrence() { delete impl_; }

int64_t Cooccurrence::run() {
  Impl& I = *impl_;
  cudaStream_t s = I.stream;
  I.result = Matrix();
  chunks_ = 0;
  if (I.n_tokens == 0 || I.n_sentences == 0) return 0;
  Buf<uint8_t> room((size_t)I.n_tokens);
  cooc_room_kernel<<<grid_for(I.n_tokens), kThreads, 0, s>>>(I.offsets, I.n_sentences, I.n_tokens, I.window, room.p);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
  Params P{I.tokens, room.p, 0, 0, I.V, (uint32_t)lw_, I.rank, I.world, I.sym, I.dw};

  // Budget: the room array and cub's temporary storage, then two phases that must each fit what is left. Counting,
  // sorting and reducing a chunk of T tokens with E entries holds the result (16 bytes a non-zero), two int32 per
  // token and 40 bytes per entry (keys and numerators double-buffered, the reduced chunk); merging holds the result,
  // the reduced chunk and two merged copies, at most 32 bytes per non-zero of the result and per entry of the chunk.
  constexpr int64_t kSlack = 64 << 20;
  const int64_t avail = I.max_bytes - I.n_tokens - kSlack;
  const double worst = (double)I.window * (I.sym ? 2 : 1);
  double rate = worst;                                // entries per token the next chunk is sized for
  for (int64_t t0 = 0; t0 < I.n_tokens;) {
    const int64_t nr = I.result.n;
    auto fits = [&](int64_t T, int64_t E) { return 16 * nr + 8 * T + 40 * E <= avail && 32 * (nr + E) <= avail; };
    const double by_sort = (double)(avail - 16 * nr) / (8.0 + 40.0 * rate);
    const double by_merge = ((double)avail / 32.0 - (double)nr) / rate;
    int64_t T = (int64_t)std::min({(double)(I.n_tokens - t0), by_sort, by_merge, (double)INT32_MAX / worst});
    ADAPM_CHECK(T >= 1, "glove_cooccurrence: max_bytes = " << I.max_bytes << " is too small for a corpus of "
                                                          << I.n_tokens << " tokens and the " << nr
                                                          << " non-zeros counted so far");
    int64_t E = 0;
    Buf<int32_t> cnt, pos;
    for (;;) {
      P.t0 = t0; P.n = T;
      cnt = Buf<int32_t>((size_t)T);
      pos = Buf<int32_t>((size_t)T);
      cooc_count_kernel<<<grid_for(T), kThreads, 0, s>>>(P, cnt.p);
      ADAPM_COUNT_LAUNCH();
      ADAPM_CUDA_CHECK(cudaGetLastError());
      size_t bytes = 0;
      ADAPM_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, bytes, cnt.p, pos.p, (int)T, s));
      {
        Buf<char> tmp(bytes);
        ADAPM_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, cnt.p, pos.p, (int)T, s));
        ADAPM_COUNT_LAUNCH();
      }
      E = I.fetch(pos.p + T - 1) + I.fetch(cnt.p + T - 1);
      if (fits(T, E)) break;
      ADAPM_CHECK(T > 1, "glove_cooccurrence: max_bytes = " << I.max_bytes << " is too small");
      T = std::max<int64_t>(1, T / 2);
    }
    rate = std::min(worst, 1.1 * (double)E / (double)T + 1e-3);
    ++chunks_;
    if (E > 0) {
      Matrix c;
      c.keys = Buf<uint64_t>(E);
      c.sums = Buf<long long>(E);
      {
        Buf<uint64_t> k0(E), k1(E);
        Buf<uint32_t> v0(E), v1(E);
        cooc_expand_kernel<<<grid_for(T), kThreads, 0, s>>>(P, pos.p, k0.p, v0.p);
        ADAPM_COUNT_LAUNCH();
        ADAPM_CUDA_CHECK(cudaGetLastError());
        cub::DoubleBuffer<uint64_t> kb(k0.p, k1.p);
        cub::DoubleBuffer<uint32_t> vb(v0.p, v1.p);
        I.sort_reduce(kb, vb, E, c);
      }
      cnt.release();
      pos.release();
      I.merge(c);
    }
    t0 += T;
  }
  ADAPM_CUDA_CHECK(cudaStreamSynchronize(s));
  return I.result.n;
}

void Cooccurrence::write(int32_t* rows, int32_t* cols, float* x) const {
  const Impl& I = *impl_;
  const int64_t n = I.result.n;
  if (n == 0) return;
  cooc_finish_kernel<<<grid_for(n), kThreads, 0, I.stream>>>(I.result.keys.p, I.result.sums.p, n, I.V, (double)lw_, rows,
                                                            cols, x);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace cudaops
}  // namespace adapm

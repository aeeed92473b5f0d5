// Index and apply passes of the deterministic one-GPU steps (see fx_accum.cuh).
#include "fx_accum.cuh"

#include <algorithm>
#include <map>

#include "pm_kernels.cuh"

namespace adapm {
namespace fx {

namespace {

struct Sources {
  Source s[4];
};

// Gives every key of the step a region of its own length: region offset = running total of the units handed out, or
// r * units when every source has the same row length (uniform > 0: no second atomic on one counter).
__global__ void fx_index_kernel(Sources src, int uniform, int* __restrict__ cidx, Key* __restrict__ keys,
                                int2* __restrict__ rows, unsigned int* __restrict__ count) {
  const long n0 = src.s[0].n, n1 = n0 + src.s[1].n, n2 = n1 + src.s[2].n, n = n2 + src.s[3].n;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    // (selected with conditionals: an indexed access would copy the sources to local memory)
    const Key k = i < n0 ? src.s[0].keys[i]
                : (i < n1 ? src.s[1].keys[i - n0] : (i < n2 ? src.s[2].keys[i - n1] : src.s[3].keys[i - n2]));
    if (k >= 0 && atomicCAS(cidx + k, -1, -2) == -1) {
      const int units = i < n0 ? src.s[0].units
                      : (i < n1 ? src.s[1].units : (i < n2 ? src.s[2].units : src.s[3].units));
      const unsigned r = atomicAdd(count, 1u);
      const unsigned off = uniform ? r * (unsigned)uniform : atomicAdd(count + 1, (unsigned)units);
      keys[r] = k;
      rows[r] = make_int2((int)off, units);
      cidx[k] = (int)off;
    }
  }
}

// One warp per region: adds its fixed-point sums to the key's store row (one writer per row), clears the region and
// the key's offset. Block 0 first moves the step's loss into loss_out.
__global__ void fx_apply_kernel(const __grid_constant__ Ctx c, int unit, const Key* __restrict__ keys,
                                const int2* __restrict__ rows, const unsigned int* __restrict__ count,
                                int* __restrict__ cidx, long long* __restrict__ acc, float scale_val, float scale_ada,
                                unsigned long long* __restrict__ fx_loss, float fx_loss_scale,
                                const float* __restrict__ call_loss, long n_calls, float* __restrict__ loss_out) {
  __shared__ double part[256];
  dev::cta_enter(c);
  const int lane = threadIdx.x & 31;
  if (blockIdx.x == 0) {
    if (fx_loss_scale > 0.f) {
      if (threadIdx.x == 0) {
        const long long v = (long long)*fx_loss;
        *fx_loss = 0ull;
        if (loss_out) *loss_out += (float)((double)v / (double)fx_loss_scale);
      }
    } else if (n_calls > 0) {
      // fixed order: thread t sums calls t, t + 256, ... in float64, then a fixed tree over the threads
      double s = 0.0;
      for (long i = threadIdx.x; i < n_calls; i += blockDim.x) s += (double)call_loss[i];
      part[threadIdx.x] = s;
      __syncthreads();
      for (int o = blockDim.x / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) part[threadIdx.x] += part[threadIdx.x + o];
        __syncthreads();
      }
      if (threadIdx.x == 0 && loss_out) *loss_out += (float)part[0];
    }
  }
  const unsigned n = *count;
  const unsigned nwarps = (gridDim.x * blockDim.x) >> 5;
  for (unsigned r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += nwarps) {
    const Key k = keys[r];
    const int2 rg = rows[r];
    const int h = rg.y * unit / 2;
    const int32_t slot = __ldcg(slot_of(c, c.rank) + k);
    long long* a = acc + (size_t)rg.x * unit;
    float* row = slot >= 0 ? row_ptr<float>(c, c.rank, class_of_key(c, k), (uint32_t)slot) : nullptr;
    for (int hf = 0; hf < 2; ++hf) {
      const double inv = 1.0 / (double)(hf ? scale_ada : scale_val);
      for (int i = lane; i < h; i += 32) {
        const long long v = a[(size_t)hf * h + i];
        if (v) {
          if (row) row[(size_t)hf * h + elem(i, h)] += (float)((double)v * inv);
          a[(size_t)hf * h + i] = 0;
        }
      }
    }
    if (lane == 0) cidx[k] = -1;
  }
  dev::cta_exit(c);
}

}  // namespace

CudaBackend::FxScratch& begin(CudaBackend& be, cudaStream_t stream, const Source* src, int n_src, int unit,
                              long n_calls) {
  ADAPM_CHECK(n_src >= 1 && n_src <= 4, "fx::begin: 1 to 4 key sources");
  ADAPM_CHECK(be.ctx().L.world == 1, "deterministic steps need a single-GPU server (world == 1)");
  // scratch bound: per row length, min(keys of the step, keys of that length in the store)
  std::map<int, long> by_units;
  Sources s{};
  long n_all = 0;
  for (int q = 0; q < n_src; ++q) {
    s.s[q] = src[q];
    by_units[src[q].units] += src[q].n;
    n_all += src[q].n;
  }
  size_t rows = 0, units = 0;
  for (const auto& kv : by_units) {
    const size_t r = std::min<size_t>((size_t)kv.second, be.keys_with_len((uint32_t)(kv.first * unit)));
    rows += r;
    units += r * (size_t)kv.first;
  }
  ADAPM_CHECK(units < (1ull << 31), "deterministic step: too many accumulator units in one step");
  CudaBackend::FxScratch& fx = be.fx_scratch(std::max<size_t>(units, 1) * unit, std::max<size_t>(rows, 1),
                                             (size_t)std::max<long>(n_calls, 0));
  ADAPM_CUDA_CHECK(cudaMemsetAsync(fx.count, 0, 2 * sizeof(unsigned int), stream));
  fx_index_kernel<<<(int)std::max<long>(1, std::min<long>((n_all + 255) / 256, be.num_sms() * 8L)), 256, 0, stream>>>(
      s, by_units.size() == 1 ? src[0].units : 0, fx.cidx, fx.keys, fx.rows, fx.count);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
  fx.step_rows = rows;
  return fx;
}

void apply(CudaBackend& be, cudaStream_t stream, int unit, float scale_val, float scale_ada, float fx_loss_scale,
           long n_calls, float* loss_out) {
  CudaBackend::FxScratch& fx = be.fx_scratch(0, 0, 0);
  const int blocks = (int)std::max<size_t>(1, std::min<size_t>((fx.step_rows + 7) / 8, (size_t)be.num_sms() * 16));
  fx_apply_kernel<<<blocks, 256, 0, stream>>>(be.ctx(), unit, fx.keys, fx.rows, fx.count, fx.cidx, fx.acc,
                                                     scale_val, scale_ada, fx.loss, fx_loss_scale, fx.call_loss,
                                                     n_calls, loss_out);
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

}  // namespace fx
}  // namespace adapm

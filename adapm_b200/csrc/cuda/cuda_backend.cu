// Generic parameter-manager kernels for sm_90a and their host driver.
//
// Kernel inventory (SURVEY 2.5 numbering):
//   K1  pull_kernel        batched gather: in-kernel directory lookup, local HBM rows or
//                          NVLink peer loads in the same kernel
//   K2  push_kernel        batched scatter-add / set: local or peer reductions (REDG over NVLink)
//   K3  phase_a_kernel     replica delta extract + reduce to owner (+ L2-norm threshold, K5)
//   K6  phase_b_kernel     owner-side relocate/replicate decision + directory broadcast
//   K4  phase_c_kernel     replica refresh / relocation transfer / drop
//       register_kernel    intent registration (placeholder replicas)
#include "cuda_backend.h"

#include <cstring>
#include <sstream>
#include <type_traits>

#include "pm_kernels.cuh"

namespace adapm {

namespace {

constexpr int kThreads = 256;
constexpr int kWarpsPerBlock = kThreads / 32;

__global__ void init_uniform_kernel(const __grid_constant__ Ctx c) {
  const int me = c.rank;
  const int64_t K = c.L.num_keys;
  const int world = c.L.world;
  uint8_t* dir = dir_of(c, me);
  int32_t* so = slot_of(c, me);
  uint32_t* meta = meta_of(c, me);
  int64_t* skey = slot_key_of(c, me);
  for (int64_t key = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; key < K; key += (int64_t)gridDim.x * blockDim.x) {
    int home = (int)(key % world);
    dir[key] = (uint8_t)home;
    if (home == me) {
      uint32_t s = (uint32_t)(key / world);
      so[key] = (int32_t)s;
      meta[s] = meta_make(S_OWNED, 0, 1);
      skey[s] = key;
    } else {
      so[key] = -1;
    }
  }
  // free stack: slots [n_home, cap) in ascending pop order
  const int64_t n_home = K / world + ((K % world) > me ? 1 : 0);
  const int64_t cap = c.L.cls[0].cap;
  int32_t* stack = at<int32_t>(c, me, c.L.cls[0].free_off);
  const int64_t n_free = cap - n_home;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_free; i += (int64_t)gridDim.x * blockDim.x)
    stack[i] = (int32_t)(cap - 1 - i);
  if (blockIdx.x == 0 && threadIdx.x == 0) free_top_of(c, me)[0] = (int32_t)n_free;
}

// ------------------------------------------------------------------------------ K1
// (templated on the value type: float32 rows take the 16-byte fast paths, float64 / int64 rows - the reference's
// `double` applications and its exact `long` contract tests - the element-wise protocol path)
template <class Val>
__global__ void __launch_bounds__(kThreads)
pull_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ keys, size_t n, Val* __restrict__ out,
            const int64_t* __restrict__ offsets, uint32_t uniform_len, int local_only, uint8_t* ok,
            unsigned long long* result) {
  WarpGroup g;
  dev::cta_enter(c);
  const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  unsigned nl = 0, nr = 0, nf = 0;
  for (size_t i = warp; i < n; i += nwarps) {
    const Key key = keys[i];
    Val* o = out + (offsets ? (size_t)offsets[i] : i * (size_t)uniform_len);
    bool good = false, local = false;
    if (key >= 0 && key < c.L.num_keys) {
      const uint32_t len = key_len(c, key, class_of_key(c, key));
      // fast path: directly readable row, 16-byte vectorised
      for (int attempt = 0; attempt < 1024 && !good; ++attempt) {
        PullLoc<Val> loc = locate_pull<Val>(c, g, key, local_only != 0);
        if (loc.kind == LOC_FAIL) break;
        bool fast = false;
        if constexpr (std::is_same<Val, float>::value) {
          if (loc.kind == LOC_DIRECT && (len & 3u) == 0 && ((((uintptr_t)loc.row) | ((uintptr_t)o)) & 15u) == 0) {
            for (uint32_t j = g.lane() * 4; j < len; j += 128) {
              float4 v = dev::ld_row4(loc.row + j);
              *reinterpret_cast<float4*>(o + j) = v;
            }
            fast = true;
          }
        }
        good = fast || read_row(g, loc, o, len);
        local = loc.local;
      }
    }
    if (ok && g.lane() == 0) ok[i] = good ? 1 : 0;
    if (!good) ++nf; else if (local) ++nl; else ++nr;
  }
  if (g.lane() == 0) {
    if (result) {
      if (nl) atomicAdd(result + 0, (unsigned long long)nl);
      if (nr) atomicAdd(result + 1, (unsigned long long)nr);
      if (nf) atomicAdd(result + 2, (unsigned long long)nf);
    }
    uint64_t* cn = counters_of(c, c.rank);
    if (nl) atomicAdd((unsigned long long*)(cn + C_PULL_LOCAL), (unsigned long long)nl);
    if (nr) atomicAdd((unsigned long long*)(cn + C_PULL_REMOTE), (unsigned long long)nr);
    // a local_only miss (PullIfLocal, local sampling) is an ordinary outcome, not a protocol error (cpu backend: same)
    if (nf && !local_only) atomicAdd((unsigned long long*)(cn + C_PROTOCOL_ERRORS), (unsigned long long)nf);
  }
  dev::cta_exit(c);
}

// ------------------------------------------------------------------------------ K2
template <class Val>
__global__ void __launch_bounds__(kThreads)
push_kernel(const __grid_constant__ Ctx c, const Key* __restrict__ keys, size_t n, const Val* __restrict__ vals,
            const int64_t* __restrict__ offsets, uint32_t uniform_len, int set, unsigned long long* result,
            uint8_t* __restrict__ todo) {
  WarpGroup g;
  dev::cta_enter(c);
  const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  unsigned nl = 0, nr = 0, nf = 0, nretry = 0;
  for (size_t i = warp; i < n; i += nwarps) {
    if (todo && !todo[i]) continue;   // Set with retry: this key is already done
    const Key key = keys[i];
    const Val* v = vals + (offsets ? (size_t)offsets[i] : i * (size_t)uniform_len);
    bool good = false, local = false;
    if (key >= 0 && key < c.L.num_keys) {
      if (set) {
        const int r = set_key<Val>(c, g, key, v, &local);
        if (r == SET_RETRY && todo) { ++nretry; continue; }   // relocation in flight: the host repeats it after a round
        good = r == SET_OK;
      } else {
        const uint32_t len = key_len(c, key, class_of_key(c, key));
        PushLoc<Val> loc = locate_push<Val>(c, g, key);
        if (loc.row) {
          bool fast = false;
          if constexpr (std::is_same<Val, float>::value) {
            if ((len & 3u) == 0 && ((((uintptr_t)loc.row) | ((uintptr_t)v)) & 15u) == 0) {
              for (uint32_t j = g.lane() * 4; j < len; j += 128)
                dev::red_row4(loc.row + j, *reinterpret_cast<const float4*>(v + j));
              fast = true;
            }
          }
          if (!fast)
            for (uint32_t j = g.lane(); j < len; j += 32) mem::red_add(loc.row + j, v[j]);
          if (g.lane() == 0) {
            if (loc.version) mem::red_add(loc.version, 1u);
            if (loc.flag) mem::st_relaxed(loc.flag, (uint8_t)1);
          }
          good = true;
          local = loc.local;
        }
      }
    }
    if (todo && g.lane() == 0) todo[i] = 0;
    if (!good) ++nf; else if (local) ++nl; else ++nr;
  }
  if (g.lane() == 0) {
    if (result) {
      if (nl) atomicAdd(result + 0, (unsigned long long)nl);
      if (nr) atomicAdd(result + 1, (unsigned long long)nr);
      if (nf) atomicAdd(result + 2, (unsigned long long)nf);
      if (nretry) atomicAdd(result + 3, (unsigned long long)nretry);
    }
    uint64_t* cn = counters_of(c, c.rank);
    if (nl) atomicAdd((unsigned long long*)(cn + C_PUSH_LOCAL), (unsigned long long)nl);
    if (nr) atomicAdd((unsigned long long*)(cn + C_PUSH_REMOTE), (unsigned long long)nr);
    if (nf) atomicAdd((unsigned long long*)(cn + C_PROTOCOL_ERRORS), (unsigned long long)nf);
  }
  dev::cta_exit(c);
}

__global__ void peek_kernel(const __grid_constant__ Ctx c, const Key* keys, size_t n, uint8_t* state_out, uint8_t* owner_out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Key k = keys[i];
  int32_t s = mem::ld_relaxed(slot_of(c, c.rank) + k);
  state_out[i] = s >= 0 ? (uint8_t)meta_state(mem::ld_acquire(meta_of(c, c.rank) + s)) : (uint8_t)S_FREE;
  owner_out[i] = mem::ld_relaxed(dir_of(c, c.rank) + k);
}

// ------------------------------------------------------------------------------ sync round
// All round kernels read their parameters from a device-resident RoundDev (cuda_backend.h): the host uploads it once
// per round, the first cross-rank barrier of the round fills in what the ranks agreed on (sweep / stop).
template <class Val>
__global__ void register_kernel(const __grid_constant__ Ctx c, const IntentRec* recs, const RoundDev* __restrict__ rd,
                                uint8_t* status) {
  if (rd->stop) return;
  const size_t n = rd->n_recs;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int st = register_intent<Val>(c, recs[i], rd->rp.clocks);
  status[i] = (uint8_t)st;
  if (st == 0) count(c, C_INTENTS_REGISTERED);
  else if (st == 1) count(c, C_INTENTS_DEFERRED);
}

// Phase A / C run as two kernels: (1) a streaming scan over the slot states compacts the slots that
// need work into a worklist (replica slots are allocated contiguously, so a static slot->warp mapping
// would leave most warps idle), (2) one warp per worklist item, grid-strided, so that the long
// dependent-load chains of many slots overlap.
template <int PHASE>
__global__ void __launch_bounds__(kThreads) phase_scan_kernel(const __grid_constant__ Ctx c, const RoundDev* __restrict__ rd,
                                                              SlotWork* __restrict__ worklist,
                                                              unsigned int* __restrict__ count) {
  if (rd->stop) return;
  const RoundParams& rp = rd->rp;
  const uint32_t S = c.L.total_slots;
  const uint32_t* meta = meta_of(c, c.rank);
  const int lane = threadIdx.x & 31;
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < ((S + 31u) & ~31u); s += gridDim.x * blockDim.x) {
    bool hit = false;
    if (s < S) {
      uint32_t st = meta_state(__ldcg(meta + s));
      if (st != S_FREE && st != S_OWNED) hit = (PHASE == 0) ? phase_a_wants(c, s, rp) : phase_c_wants(c, s, rp);
    }
    unsigned mask = __ballot_sync(0xffffffffu, hit);
    if (mask) {
      unsigned base = 0;
      if (lane == 0) base = atomicAdd(count, (unsigned)__popc(mask));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (hit) worklist[base + __popc(mask & ((1u << lane) - 1u))].slot = s;
    }
  }
}

// resolve / commit: one thread per worklist entry (all the metadata work, including the NVLink metadata loads: a
// thread-per-slot pass keeps as many of them in flight as there are entries). STEP 0 = resolve, 1 = commit.
template <class Val, int PHASE, int STEP>
__global__ void __launch_bounds__(kThreads) phase_meta_kernel(const __grid_constant__ Ctx c, const RoundDev* __restrict__ rd,
                                                              SlotWork* __restrict__ worklist,
                                                              const unsigned int* __restrict__ count) {
  if (rd->stop) return;
  const unsigned n = *count;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (PHASE == 0) {
      if (STEP == 0) phase_a_resolve<Val>(c, worklist[i], rd->rp); else phase_a_commit<Val>(c, worklist[i]);
    } else {
      if (STEP == 0) phase_c_resolve<Val>(c, worklist[i], rd->rp); else phase_c_commit<Val>(c, worklist[i]);
    }
  }
}

// row pass: one warp per worklist entry that has a row operation; 16-byte loads / reductions only, no metadata, no
// fence (the kernel boundary orders it against resolve and commit). 128-thread blocks at <= 64 registers: one block
// fits into the registers a lean training kernel (104 x 512) leaves free per SM, so the pass runs NEXT to the
// training kernels instead of taking one of their two block slots.
constexpr int kWorkThreads = 128;
constexpr int kWorkMinBlocks = 6;   // <= 80 registers x 128 threads = 10 K of the 12 K registers a lean training kernel leaves free per SM
template <class Val>
__global__ void __launch_bounds__(kWorkThreads, kWorkMinBlocks) phase_row_kernel(const __grid_constant__ Ctx c,
                                                                              const RoundDev* __restrict__ rd,
                                                                              SlotWork* __restrict__ worklist,
                                                                              const unsigned int* __restrict__ count) {
  if (rd->stop) return;
  WarpGroup g;
  const unsigned n = *count;
  const unsigned warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned nwarps = (gridDim.x * blockDim.x) >> 5;
  for (unsigned i = warp; i < n; i += nwarps) {
    if (worklist[i].op != OP_NONE) row_op_execute<Val>(c, g, worklist[i]);
    __syncwarp();
  }
}

// Phase B: (1) a streaming scan compacts the owned slots that can relocate in this round (exactly one requester) into
// the worklist, (2) one THREAD per candidate decides and announces the new owner: the two NVLink round trips of a
// relocation (target slot id, target state) overlap across tens of thousands of threads instead of queueing up inside
// a few grid-striding ones.
__global__ void __launch_bounds__(kThreads) phase_b_scan_kernel(const __grid_constant__ Ctx c, const RoundDev* __restrict__ rd,
                                                                SlotWork* __restrict__ worklist,
                                                                unsigned int* __restrict__ count) {
  if (rd->stop) return;
  const uint32_t S = c.L.total_slots;
  const uint64_t* want = want_of(c, c.rank);
  const int lane = threadIdx.x & 31;
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < ((S + 31u) & ~31u); s += gridDim.x * blockDim.x) {
    const bool hit = s < S && __ldcg(want + s) != 0 && phase_b_candidate(c, s);
    const unsigned mask = __ballot_sync(0xffffffffu, hit);
    if (mask) {
      unsigned base = 0;
      if (lane == 0) base = atomicAdd(count, (unsigned)__popc(mask));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (hit) worklist[base + __popc(mask & ((1u << lane) - 1u))].slot = s;
    }
  }
}
__global__ void __launch_bounds__(kThreads) phase_b_kernel(const __grid_constant__ Ctx c, const RoundDev* __restrict__ rd,
                                                           const SlotWork* __restrict__ worklist,
                                                           const unsigned int* __restrict__ count) {
  if (rd->stop) return;
  const unsigned n = *count;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    phase_b_slot(c, worklist[i].slot, rd->rp);
}

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Cross-rank barrier on the device (layout.h: SyncArea). One thread per rank: publish my arrival (and, for the first
// barrier of a round, my stop/sweep request word) in that rank's area with a system-scope release store over NVLink,
// then wait until that rank's arrival shows up in my own area. No host thread is involved: the round is ONE enqueue.
// Every wait is bounded (timeout_ns, and the host's abort word in mapped pinned memory): a dead peer produces an
// error code in RoundDev, never a kernel that spins forever.
__global__ void __launch_bounds__(64) xbar_kernel(const __grid_constant__ Ctx c, uint32_t seq, uint32_t parity, RoundDev* rd,
                                                  int gather, const volatile uint32_t* abort_word,
                                                  unsigned long long timeout_ns) {
  if (!gather && rd->stop) return;   // all ranks agreed to stop in the first barrier of this round
  const int r = threadIdx.x;
  const int me = c.rank;
  __shared__ uint32_t failed;
  if (r == 0) failed = 0;
  __syncthreads();
  if (r < c.L.world) {
    __threadfence_system();          // everything the earlier kernels of this round wrote (anywhere) is performed
    if (c.mc_heap) {
      // NVSwitch multicast: ONE multimem store per word reaches the sync area of every rank (incl. this one)
      if (r == 0) {
        const uint64_t area = c.L.off_sync;
        // my request word stays in MY heap; after the barrier every rank reduces the words of all ranks in the switch
        if (gather) mem::st_relaxed(&sync_area_of(c, me)->my_flag[parity], rd->my_flags);
        __threadfence_system();
        dev::multimem_st_release_u32(at_all<char>(c, area + offsetof(SyncArea, bar_arrive) + me * 4u), seq);
      }
    } else {
      SyncArea* theirs = sync_area_of(c, r);
      if (gather) mem::st_relaxed(&theirs->flag_word[parity][me], rd->my_flags);
      mem::st_release(&theirs->bar_arrive[me], seq);
    }
    const uint32_t* mine = &sync_area_of(c, me)->bar_arrive[r];
    const unsigned long long t0 = global_ns();
    unsigned spins = 0;
    while ((int32_t)(mem::ld_acquire(mine) - seq) < 0) {
      __nanosleep(100);
      if ((++spins & 63u) == 0 && ((abort_word && *abort_word) || global_ns() - t0 > timeout_ns)) { failed = 1; break; }
    }
  }
  __syncthreads();
  if (r == 0) {
    if (failed) rd->error = 1;
    if (gather) {
      uint32_t all_stop = 1, any_sweep = 0;
      if (c.mc_heap) {   // stop = AND, sweep = OR over the ranks' words: two multimem.ld_reduce (in-switch reductions)
        const void* mcw = at_all<char>(c, c.L.off_sync + offsetof(SyncArea, my_flag) + parity * 4u);
        all_stop = dev::multimem_ld_and_u32(mcw) & 1u;
        any_sweep = (dev::multimem_ld_or_u32(mcw) >> 1) & 1u;
      } else {
        const uint32_t* w = sync_area_of(c, me)->flag_word[parity];
        for (int k = 0; k < c.L.world; ++k) {
          const uint32_t f = mem::ld_relaxed(w + k);
          all_stop &= f & 1u;
          any_sweep |= (f >> 1) & 1u;
        }
      }
      rd->stop = (all_stop && !failed) ? 1u : 0u;
      rd->any_sweep = any_sweep;
      rd->rp.sweep = (int32_t)any_sweep;
    }
    __threadfence_system();
  }
}

// Grace period on the device: flip the epoch, wait until every CTA that registered on the old side (and may have
// read the directory before phase B changed it) has left. Replaces one event record + host wait per tracked stream.
__global__ void grace_kernel(const __grid_constant__ Ctx c, RoundDev* rd, const volatile uint32_t* abort_word,
                             unsigned long long timeout_ns) {
  if (rd->stop) return;
  SyncArea* sa = sync_area_of(c, c.rank);
  const uint32_t old = mem::ld_relaxed(&sa->epoch);
  mem::st_release(&sa->epoch, old + 1u);
  __threadfence();
  const unsigned long long t0 = global_ns();
  unsigned spins = 0;
  while (mem::ld_acquire(&sa->active[old & 1u]) != 0u) {
    __nanosleep(200);
    if ((++spins & 63u) == 0 && ((abort_word && *abort_word) || global_ns() - t0 > timeout_ns)) { rd->error = 2; break; }
  }
  __threadfence_system();
}

}  // namespace

// run `...` with the alias Val bound to the value type of the store (Options::dtype)
#define ADAPM_DISPATCH_VAL(vb_is_int, vbytes, ...)                  \
  do {                                                              \
    if ((vbytes) == 4) { using Val = float; __VA_ARGS__; }          \
    else if (vb_is_int) { using Val = int64_t; __VA_ARGS__; }       \
    else { using Val = double; __VA_ARGS__; }                       \
  } while (0)

std::atomic<uint64_t>& kernel_launch_counter() {
  static std::atomic<uint64_t> c{0};
  return c;
}

// =============================================================================== host side
void CudaBackend::use_device() const { ADAPM_CUDA_CHECK(cudaSetDevice(device_)); }

CudaBackend::CudaBackend(const Options& opt, const Layout& L, std::shared_ptr<Fabric> fabric) : fabric_(fabric) {
  memset(&ctx_, 0, sizeof(ctx_));
  ctx_.L = L;
  ctx_.rank = opt.rank;
  ctx_.technique = (int)opt.techniques;
  int_rows_ = opt.dtype == "int64";
  fabric_->allocate_heaps(L.heap_bytes);
  device_ = fabric_->device();
  use_device();
  for (int r = 0; r < L.world; ++r) ctx_.heap[r] = fabric_->heap(r);
  ctx_.mc_heap = fabric_->mc_heap();
  if (const char* e = getenv("ADAPM_MULTICAST_BARRIER")) { if (atoi(e) == 0) ctx_.mc_heap = nullptr; }
  cudaDeviceProp prop;
  ADAPM_CUDA_CHECK(cudaGetDeviceProperties(&prop, device_));
  num_sms_ = prop.multiProcessorCount;
  if (const char* e = getenv("ADAPM_SYNC_TRACE")) trace_on_ = atoi(e) != 0;
  int lo = 0, hi = 0;
  ADAPM_CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  ADAPM_CUDA_CHECK(cudaStreamCreateWithPriority(&sync_stream_, cudaStreamNonBlocking, hi));
  worker_streams_.resize(opt.workers);
  for (int w = 0; w < opt.workers; ++w) {
    ADAPM_CUDA_CHECK(cudaStreamCreateWithFlags(&worker_streams_[w], cudaStreamNonBlocking));
    tracked_.insert(worker_streams_[w]);
    staging_.emplace_back(new Staging());
  }
  ADAPM_CUDA_CHECK(cudaMalloc((void**)&worklist_, (size_t)(L.total_slots + 32) * sizeof(SlotWork)));
  ADAPM_CUDA_CHECK(cudaMalloc((void**)&work_count_, 64));
  ADAPM_CUDA_CHECK(cudaMalloc((void**)&round_dev_, sizeof(RoundDev)));
  ADAPM_CUDA_CHECK(cudaMemset(round_dev_, 0, sizeof(RoundDev)));
  ADAPM_CUDA_CHECK(cudaHostAlloc((void**)&round_host_, 2 * sizeof(RoundDev), cudaHostAllocDefault));
  memset(round_host_, 0, 2 * sizeof(RoundDev));
  ADAPM_CUDA_CHECK(cudaHostAlloc((void**)&abort_word_, 64, cudaHostAllocMapped));
  *abort_word_ = 0;
  ADAPM_CUDA_CHECK(cudaEventCreateWithFlags(&round_done_, cudaEventDisableTiming));
  // The device-resident round needs the ranks' kernels to run concurrently (a barrier kernel waits for its peers'
  // barrier kernels): guaranteed with one process and GPU per rank. Logical ranks that share ONE device (inproc fabric,
  // the single-GPU tests) can starve each other - any implicitly synchronising call of one rank's host thread
  // (cudaFree, cudaDeviceSynchronize, ...) waits for another rank's waiting barrier - so they default to the
  // host-sequenced round; ADAPM_DEVICE_ROUND=1 / ADAPM_HOST_ROUND=1 force either.
  fused_round_ = L.world > 1 && fabric_->peers_are_processes();
  if (const char* e = getenv("ADAPM_DEVICE_ROUND")) fused_round_ = L.world > 1 && atoi(e) != 0;
  if (const char* e = getenv("ADAPM_HOST_ROUND")) fused_round_ = fused_round_ && atoi(e) == 0;
  dev_timeout_ns_ = (unsigned long long)(std::min(opt.wait_timeout_s, 20.0) * 1e9);
}

CudaBackend::FxScratch& CudaBackend::fx_scratch(size_t acc_len, size_t rows, size_t calls) {
  use_device();
  if (!fx_.cidx) {
    const size_t nk = (size_t)ctx_.L.num_keys;
    ADAPM_CUDA_CHECK(cudaMalloc((void**)&fx_.cidx, nk * sizeof(int)));
    ADAPM_CUDA_CHECK(cudaMemset(fx_.cidx, 0xff, nk * sizeof(int)));
    ADAPM_CUDA_CHECK(cudaMalloc((void**)&fx_.count, 2 * sizeof(unsigned int)));
    ADAPM_CUDA_CHECK(cudaMalloc((void**)&fx_.loss, sizeof(unsigned long long)));
    ADAPM_CUDA_CHECK(cudaMemset(fx_.loss, 0, sizeof(unsigned long long)));
  }
  // (the regions are all zero between steps, so a larger buffer replaces the old one without a copy)
  if (acc_len > fx_.acc_len) {
    if (fx_.acc) ADAPM_CUDA_CHECK(cudaFree(fx_.acc));
    ADAPM_CUDA_CHECK(cudaMalloc((void**)&fx_.acc, acc_len * sizeof(long long)));
    ADAPM_CUDA_CHECK(cudaMemset(fx_.acc, 0, acc_len * sizeof(long long)));
    fx_.acc_len = acc_len;
  }
  if (rows > fx_.rows_cap) {
    if (fx_.keys) { ADAPM_CUDA_CHECK(cudaFree(fx_.keys)); ADAPM_CUDA_CHECK(cudaFree(fx_.rows)); }
    ADAPM_CUDA_CHECK(cudaMalloc((void**)&fx_.keys, rows * sizeof(Key)));
    ADAPM_CUDA_CHECK(cudaMalloc((void**)&fx_.rows, rows * sizeof(int2)));
    fx_.rows_cap = rows;
  }
  if (calls > fx_.calls_cap) {
    if (fx_.call_loss) ADAPM_CUDA_CHECK(cudaFree(fx_.call_loss));
    ADAPM_CUDA_CHECK(cudaMalloc((void**)&fx_.call_loss, calls * sizeof(float)));
    fx_.calls_cap = calls;
  }
  return fx_;
}

void* CudaBackend::step_buffer(int i, size_t bytes) {
  auto& b = step_bufs_.at((size_t)i);
  if (bytes > b.second) {
    use_device();
    if (b.first) ADAPM_CUDA_CHECK(cudaFree(b.first));
    ADAPM_CUDA_CHECK(cudaMalloc(&b.first, bytes));
    ADAPM_CUDA_CHECK(cudaMemset(b.first, 0, bytes));
    b.second = bytes;
  }
  return b.first;
}

size_t CudaBackend::keys_with_len(uint32_t len) {
  if (key_len_.empty()) return (size_t)ctx_.L.num_keys;
  if (keys_by_len_.empty())
    for (uint32_t l : key_len_) ++keys_by_len_[l];
  auto it = keys_by_len_.find(len);
  return it == keys_by_len_.end() ? 0 : it->second;
}

CudaBackend::~CudaBackend() {
  cudaSetDevice(device_);
  cudaDeviceSynchronize();
  for (auto& st : staging_) { if (st->host) cudaFreeHost(st->host); if (st->dev) cudaFree(st->dev); }
  if (sync_staging_.host) cudaFreeHost(sync_staging_.host);
  if (sync_staging_.dev) cudaFree(sync_staging_.dev);
  if (worklist_) cudaFree(worklist_);
  if (work_count_) cudaFree(work_count_);
  if (round_dev_) cudaFree(round_dev_);
  if (round_host_) cudaFreeHost(round_host_);
  if (abort_word_) cudaFreeHost(abort_word_);
  if (recs_dev_) cudaFree(recs_dev_);
  if (recs_host_) cudaFreeHost(recs_host_);
  if (status_dev_) cudaFree(status_dev_);
  if (status_host_) cudaFreeHost(status_host_);
  if (fx_.acc) cudaFree(fx_.acc);
  if (fx_.cidx) cudaFree(fx_.cidx);
  if (fx_.keys) cudaFree(fx_.keys);
  if (fx_.rows) cudaFree(fx_.rows);
  if (fx_.call_loss) cudaFree(fx_.call_loss);
  if (fx_.count) cudaFree(fx_.count);
  if (fx_.loss) cudaFree(fx_.loss);
  for (auto& b : step_bufs_) if (b.first) cudaFree(b.first);
  if (round_done_) cudaEventDestroy(round_done_);
  for (auto& kv : tickets_) cudaEventDestroy(kv.second);
  for (auto e : event_pool_) cudaEventDestroy(e);
  for (auto s : worker_streams_) cudaStreamDestroy(s);
  if (sync_stream_) cudaStreamDestroy(sync_stream_);
}

void CudaBackend::ensure_staging(Staging& st, size_t bytes) {
  if (st.bytes >= bytes) return;
  size_t nb = std::max<size_t>(bytes * 2, 1 << 20);
  if (st.host) { ADAPM_CUDA_CHECK(cudaFreeHost(st.host)); st.host = nullptr; }
  if (st.dev) { ADAPM_CUDA_CHECK(cudaFree(st.dev)); st.dev = nullptr; }
  ADAPM_CUDA_CHECK(cudaMallocHost((void**)&st.host, nb));
  ADAPM_CUDA_CHECK(cudaMalloc((void**)&st.dev, nb));
  st.bytes = nb;
}

void CudaBackend::init_store(const std::vector<uint8_t>& key_class, const std::vector<uint32_t>& key_lens) {
  use_device();
  const Layout& L = ctx_.L;
  const int me = ctx_.rank;
  if (L.num_classes == 1) {
    init_uniform_kernel<<<num_sms_ * 4, 256, 0, sync_stream_>>>(ctx_);
    ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
  } else {
    // multi-class: build the tables on the host (cold path) and upload
    std::vector<uint8_t> dir(L.num_keys);
    std::vector<int32_t> so(L.num_keys, -1);
    std::vector<uint32_t> meta(L.total_slots, 0);
    std::vector<int64_t> skey(L.total_slots, 0);
    std::vector<uint32_t> next(L.num_classes);
    for (int k = 0; k < L.num_classes; ++k) next[k] = L.cls[k].slot_begin;
    key_len_.resize(L.num_keys);
    for (int64_t key = 0; key < L.num_keys; ++key) {
      int home = (int)(key % L.world);
      dir[key] = (uint8_t)home;
      key_len_[key] = L.per_key_len ? key_lens[key] : L.cls[key_class[key]].len;
      if (home == me) {
        uint32_t s = next[key_class[key]]++;
        so[key] = (int32_t)s;
        meta[s] = meta_make(S_OWNED, 0, 1);
        skey[s] = key;
      }
    }
    char* h = ctx_.heap[me];
    ADAPM_CUDA_CHECK(cudaMemcpy(h + L.off_dir, dir.data(), dir.size(), cudaMemcpyHostToDevice));
    ADAPM_CUDA_CHECK(cudaMemcpy(h + L.off_slot_of, so.data(), so.size() * 4, cudaMemcpyHostToDevice));
    ADAPM_CUDA_CHECK(cudaMemcpy(h + L.off_key_class, key_class.data(), key_class.size(), cudaMemcpyHostToDevice));
    if (L.per_key_len) ADAPM_CUDA_CHECK(cudaMemcpy(h + L.off_key_len, key_lens.data(), key_lens.size() * 4, cudaMemcpyHostToDevice));
    ADAPM_CUDA_CHECK(cudaMemcpy(h + L.off_meta, meta.data(), meta.size() * 4, cudaMemcpyHostToDevice));
    ADAPM_CUDA_CHECK(cudaMemcpy(h + L.off_slot_key, skey.data(), skey.size() * 8, cudaMemcpyHostToDevice));
    int32_t tops[MAX_CLASSES] = {0};
    for (int k = 0; k < L.num_classes; ++k) {
      std::vector<int32_t> stack;
      uint32_t end = L.cls[k].slot_begin + L.cls[k].cap;
      for (uint32_t s = end; s-- > next[k];) stack.push_back((int32_t)s);
      tops[k] = (int32_t)stack.size();
      if (!stack.empty())
        ADAPM_CUDA_CHECK(cudaMemcpy(h + L.cls[k].free_off, stack.data(), stack.size() * 4, cudaMemcpyHostToDevice));
    }
    ADAPM_CUDA_CHECK(cudaMemcpy(h + L.off_free_top, tops, sizeof(tops), cudaMemcpyHostToDevice));
  }
  ADAPM_CUDA_CHECK(cudaStreamSynchronize(sync_stream_));
  ADAPM_CUDA_CHECK(cudaDeviceSynchronize());
  fabric_->node_barrier("init_store");
}

void CudaBackend::track_stream(cudaStream_t s) {
  std::lock_guard<std::mutex> lk(streams_mu_);
  tracked_.insert(s);
}

uint64_t CudaBackend::record_ticket(cudaStream_t s) {
  cudaEvent_t ev;
  {
    std::lock_guard<std::mutex> lk(tickets_mu_);
    if (!event_pool_.empty()) { ev = event_pool_.back(); event_pool_.pop_back(); }
    else ADAPM_CUDA_CHECK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  }
  ADAPM_CUDA_CHECK(cudaEventRecord(ev, s));
  std::lock_guard<std::mutex> lk(tickets_mu_);
  uint64_t t = next_ticket_++;
  tickets_[t] = ev;
  return t;
}

void CudaBackend::wait_ticket(uint64_t t) {
  cudaEvent_t ev;
  {
    std::lock_guard<std::mutex> lk(tickets_mu_);
    auto it = tickets_.find(t);
    if (it == tickets_.end()) return;
    ev = it->second;
  }
  ADAPM_CUDA_CHECK(cudaEventSynchronize(ev));
  std::lock_guard<std::mutex> lk(tickets_mu_);
  auto it = tickets_.find(t);
  if (it != tickets_.end()) { event_pool_.push_back(it->second); tickets_.erase(it); }
}

bool CudaBackend::ticket_done(uint64_t t) {
  std::lock_guard<std::mutex> lk(tickets_mu_);
  auto it = tickets_.find(t);
  if (it == tickets_.end()) return true;
  cudaError_t e = cudaEventQuery(it->second);
  if (e == cudaErrorNotReady) return false;
  ADAPM_CUDA_CHECK(e);
  event_pool_.push_back(it->second);
  tickets_.erase(it);
  return true;
}

void CudaBackend::wait_worker(int worker) {
  use_device();
  ADAPM_CUDA_CHECK(cudaStreamSynchronize(worker_streams_[worker]));
  std::vector<cudaStream_t> ss;
  {
    std::lock_guard<std::mutex> lk(streams_mu_);
    ss.assign(tracked_.begin(), tracked_.end());
  }
  for (auto s : ss) ADAPM_CUDA_CHECK(cudaStreamSynchronize(s));
}

static inline int grid_for_warps(size_t n_items, int num_sms) {
  size_t blocks = (n_items + kWarpsPerBlock - 1) / kWarpsPerBlock;
  size_t cap = (size_t)num_sms * 8;
  return (int)std::max<size_t>(1, std::min(blocks, cap));
}

uint64_t CudaBackend::pull(int worker, const Key* keys, size_t n, void* vals, bool local_only, uint8_t* ok,
                           OpResult* res, const IoDesc& io) {
  use_device();
  if (n == 0) { if (res) *res = OpResult(); return 0; }
  const Layout& L = ctx_.L;
  const bool uniform = L.num_classes == 1;
  if (io.on_device) {
    ADAPM_CHECK(uniform || io.offsets, "device-pointer pull on a mixed-length store needs per-key value offsets");
    cudaStream_t s = resolve_stream(worker, io);
    ADAPM_DISPATCH_VAL(int_rows_, L.val_bytes, pull_kernel<Val><<<grid_for_warps(n, num_sms_), kThreads, 0, s>>>(
        ctx_, keys, n, (Val*)vals, uniform ? nullptr : io.offsets, L.cls[0].len, local_only ? 1 : 0, ok, nullptr));
    ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
    return record_ticket(s);
  }
  // host pointers: stage through pinned memory on the worker's stream, synchronous
  Staging& st = *staging_[worker];
  std::lock_guard<std::mutex> lk(st.mu);
  cudaStream_t s = worker_streams_[worker];
  const size_t o_keys = 0;
  const size_t o_offs = align_up(o_keys + n * 8, 256);
  const size_t o_res = align_up(o_offs + n * 8, 256);
  const size_t o_ok = align_up(o_res + 64, 256);
  const size_t o_vals = align_up(o_ok + n, 256);
  // rows are concatenated in key order, so for mixed lengths the output offsets are a prefix sum
  // over the key lengths (host mirror of the class table, built in init_store)
  size_t bytes_vals;
  std::vector<int64_t> prefix;
  if (uniform) bytes_vals = n * (size_t)L.cls[0].len * L.val_bytes;
  else {
    prefix.resize(n);
    size_t acc = 0;
    for (size_t i = 0; i < n; ++i) {
      ADAPM_CHECK(keys[i] >= 0 && keys[i] < L.num_keys, "[ERROR] Pull key " << keys[i] << ", which is outside the configured key range [0," << L.num_keys << ")");
      prefix[i] = (int64_t)acc;
      acc += (size_t)key_len_[keys[i]];
    }
    bytes_vals = acc * L.val_bytes;
  }
  ensure_staging(st, o_vals + bytes_vals + 256);
  memcpy(st.host + o_keys, keys, n * 8);
  if (!uniform) memcpy(st.host + o_offs, prefix.data(), n * 8);
  memset(st.host + o_res, 0, 64);
  ADAPM_CUDA_CHECK(cudaMemcpyAsync(st.dev, st.host, o_ok, cudaMemcpyHostToDevice, s));
  ADAPM_DISPATCH_VAL(int_rows_, L.val_bytes, pull_kernel<Val><<<grid_for_warps(n, num_sms_), kThreads, 0, s>>>(
      ctx_, (const Key*)(st.dev + o_keys), n, (Val*)(st.dev + o_vals), uniform ? nullptr : (const int64_t*)(st.dev + o_offs),
      L.cls[0].len, local_only ? 1 : 0, (uint8_t*)(st.dev + o_ok), (unsigned long long*)(st.dev + o_res)));
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
  ADAPM_CUDA_CHECK(cudaMemcpyAsync(st.host + o_res, st.dev + o_res, (o_vals - o_res) + bytes_vals, cudaMemcpyDeviceToHost, s));
  ADAPM_CUDA_CHECK(cudaStreamSynchronize(s));
  const unsigned long long* r = (const unsigned long long*)(st.host + o_res);
  if (res) { res->n_local = r[0]; res->n_remote = r[1]; res->n_failed = r[2]; }
  if (ok) memcpy(ok, st.host + o_ok, n);
  // copy only rows that were actually read (local_only misses leave garbage)
  memcpy(vals, st.host + o_vals, bytes_vals);
  return 0;
}

uint64_t CudaBackend::push(int worker, const Key* keys, size_t n, const void* vals, bool set, OpResult* res,
                           const IoDesc& io, uint8_t* todo) {
  use_device();
  if (n == 0) { if (res) *res = OpResult(); return 0; }
  const Layout& L = ctx_.L;
  const bool uniform = L.num_classes == 1;
  if (io.on_device) {
    ADAPM_CHECK(uniform || io.offsets, "device-pointer push on a mixed-length store needs per-key value offsets");
    cudaStream_t s = resolve_stream(worker, io);
    if (!todo) {
      ADAPM_DISPATCH_VAL(int_rows_, L.val_bytes, push_kernel<Val><<<grid_for_warps(n, num_sms_), kThreads, 0, s>>>(
          ctx_, keys, n, (const Val*)vals, uniform ? nullptr : io.offsets, L.cls[0].len, set ? 1 : 0, nullptr, nullptr));
      ADAPM_COUNT_LAUNCH();
      ADAPM_CUDA_CHECK(cudaGetLastError());
      return record_ticket(s);
    }
    // Set with retry: keys and values stay on the device, the todo mask and the counts go through pinned memory;
    // synchronous (the caller decides from the counts whether to repeat after the next sync round)
    Staging& st = *staging_[worker];
    std::lock_guard<std::mutex> lk(st.mu);
    const size_t o_todo = 256;
    ensure_staging(st, o_todo + n + 256);
    memset(st.host, 0, 64);
    memcpy(st.host + o_todo, todo, n);
    ADAPM_CUDA_CHECK(cudaMemcpyAsync(st.dev, st.host, o_todo + n, cudaMemcpyHostToDevice, s));
    ADAPM_DISPATCH_VAL(int_rows_, L.val_bytes, push_kernel<Val><<<grid_for_warps(n, num_sms_), kThreads, 0, s>>>(
        ctx_, keys, n, (const Val*)vals, uniform ? nullptr : io.offsets, L.cls[0].len, set ? 1 : 0, (unsigned long long*)st.dev,
        (uint8_t*)(st.dev + o_todo)));
    ADAPM_COUNT_LAUNCH();
    ADAPM_CUDA_CHECK(cudaGetLastError());
    ADAPM_CUDA_CHECK(cudaMemcpyAsync(st.host, st.dev, o_todo + n, cudaMemcpyDeviceToHost, s));
    ADAPM_CUDA_CHECK(cudaStreamSynchronize(s));
    const unsigned long long* r = (const unsigned long long*)st.host;
    if (res) { res->n_local = r[0]; res->n_remote = r[1]; res->n_failed = r[2]; res->n_retry = r[3]; }
    memcpy(todo, st.host + o_todo, n);
    return 0;
  }
  Staging& st = *staging_[worker];
  std::lock_guard<std::mutex> lk(st.mu);
  cudaStream_t s = worker_streams_[worker];
  std::vector<int64_t> prefix;
  size_t bytes_vals;
  if (uniform) bytes_vals = n * (size_t)L.cls[0].len * L.val_bytes;
  else {
    prefix.resize(n);
    size_t acc = 0;
    for (size_t i = 0; i < n; ++i) {
      ADAPM_CHECK(keys[i] >= 0 && keys[i] < L.num_keys, "[ERROR] Push key " << keys[i] << ", which is outside the configured key range [0," << L.num_keys << ")");
      prefix[i] = (int64_t)acc;
      acc += (size_t)key_len_[keys[i]];
    }
    bytes_vals = acc * L.val_bytes;
  }
  const size_t o_keys = 0;
  const size_t o_offs = align_up(o_keys + n * 8, 256);
  const size_t o_res = align_up(o_offs + n * 8, 256);
  const size_t o_todo = align_up(o_res + 64, 256);
  const size_t o_vals = align_up(o_todo + (todo ? n : 0), 256);
  ensure_staging(st, o_vals + bytes_vals + 256);
  memcpy(st.host + o_keys, keys, n * 8);
  if (!uniform) memcpy(st.host + o_offs, prefix.data(), n * 8);
  memset(st.host + o_res, 0, 64);
  if (todo) memcpy(st.host + o_todo, todo, n);
  memcpy(st.host + o_vals, vals, bytes_vals);
  ADAPM_CUDA_CHECK(cudaMemcpyAsync(st.dev, st.host, o_vals + bytes_vals, cudaMemcpyHostToDevice, s));
  ADAPM_DISPATCH_VAL(int_rows_, L.val_bytes, push_kernel<Val><<<grid_for_warps(n, num_sms_), kThreads, 0, s>>>(
      ctx_, (const Key*)(st.dev + o_keys), n, (const Val*)(st.dev + o_vals), uniform ? nullptr : (const int64_t*)(st.dev + o_offs),
      L.cls[0].len, set ? 1 : 0, (unsigned long long*)(st.dev + o_res), todo ? (uint8_t*)(st.dev + o_todo) : nullptr));
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
  ADAPM_CUDA_CHECK(cudaMemcpyAsync(st.host + o_res, st.dev + o_res, (o_todo - o_res) + (todo ? n : 0), cudaMemcpyDeviceToHost, s));
  ADAPM_CUDA_CHECK(cudaStreamSynchronize(s));
  const unsigned long long* r = (const unsigned long long*)(st.host + o_res);
  if (res) { res->n_local = r[0]; res->n_remote = r[1]; res->n_failed = r[2]; res->n_retry = r[3]; }
  if (todo) memcpy(todo, st.host + o_todo, n);
  return 0;
}

void CudaBackend::peek_states(const Key* keys, size_t n, uint8_t* state_out, uint8_t* owner_out) {
  use_device();
  if (n == 0) return;
  std::lock_guard<std::mutex> lk(sync_staging_.mu);
  const size_t o_st = align_up(n * 8, 256), o_ow = align_up(o_st + n, 256);
  ensure_staging(sync_staging_, o_ow + n + 256);
  Staging& st = sync_staging_;
  memcpy(st.host, keys, n * 8);
  cudaStream_t s = worker_streams_[0];
  ADAPM_CUDA_CHECK(cudaMemcpyAsync(st.dev, st.host, n * 8, cudaMemcpyHostToDevice, s));
  peek_kernel<<<(int)((n + 255) / 256), 256, 0, s>>>(ctx_, (const Key*)st.dev, n, (uint8_t*)(st.dev + o_st), (uint8_t*)(st.dev + o_ow));
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
  ADAPM_CUDA_CHECK(cudaMemcpyAsync(st.host + o_st, st.dev + o_st, o_ow + n - o_st, cudaMemcpyDeviceToHost, s));
  ADAPM_CUDA_CHECK(cudaStreamSynchronize(s));
  memcpy(state_out, st.host + o_st, n);
  memcpy(owner_out, st.host + o_ow, n);
}

bool CudaBackend::key_is_local(Key k) {
  uint8_t st, ow;
  peek_states(&k, 1, &st, &ow);
  return st == S_OWNED || st == S_REPLICA || st == S_INCOMING_REPLICA;
}

void CudaBackend::upload_round(const RoundParams& rp, uint32_t n_recs, uint32_t flags) {
  RoundDev& h = round_host_[0];
  h.rp = rp;
  h.n_recs = n_recs;
  h.my_flags = flags;
  h.stop = 0; h.any_sweep = 0; h.error = 0;
  ADAPM_CUDA_CHECK(cudaMemcpyAsync(round_dev_, &h, sizeof(RoundDev), cudaMemcpyHostToDevice, sync_stream_));
}

// ---- host-sequenced round (ADAPM_HOST_ROUND=1): the sync thread waits for every phase and the ranks meet at
// control-plane barriers; the kernels are the same as in the device-resident round
void CudaBackend::register_intents(const IntentRec* recs, size_t n, const RoundParams& rp, uint8_t* status) {
  use_device();
  if (n == 0) return;
  std::lock_guard<std::mutex> lk(sync_staging_.mu);
  const size_t o_st = align_up(n * sizeof(IntentRec), 256);
  ensure_staging(sync_staging_, o_st + n + 256);
  Staging& st = sync_staging_;
  memcpy(st.host, recs, n * sizeof(IntentRec));
  TraceScope ts_(this, "register", sync_stream_);
  upload_round(rp, (uint32_t)n, 0);
  ADAPM_CUDA_CHECK(cudaMemcpyAsync(st.dev, st.host, n * sizeof(IntentRec), cudaMemcpyHostToDevice, sync_stream_));
  ADAPM_DISPATCH_VAL(int_rows_, ctx_.L.val_bytes, register_kernel<Val><<<(int)((n + 255) / 256), 256, 0, sync_stream_>>>(
      ctx_, (const IntentRec*)st.dev, round_dev_, (uint8_t*)(st.dev + o_st)));
  ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
  ADAPM_CUDA_CHECK(cudaMemcpyAsync(st.host + o_st, st.dev + o_st, n, cudaMemcpyDeviceToHost, sync_stream_));
  ADAPM_CUDA_CHECK(cudaStreamSynchronize(sync_stream_));
  memcpy(status, st.host + o_st, n);
}

void CudaBackend::launch_phase(int phase) {
  if (phase == 1) {
    unsigned int* wc = work_count_ + 2;
    ADAPM_CUDA_CHECK(cudaMemsetAsync(wc, 0, sizeof(unsigned int), sync_stream_));
    {
      TraceScope t_(this, "B.scan", sync_stream_);
      phase_b_scan_kernel<<<num_sms_, kThreads, 0, sync_stream_>>>(ctx_, round_dev_, worklist_, wc);
    }
    // one thread per candidate: the grid is sized for the worst case seen so far (the count lives on the device)
    {
      TraceScope t_(this, "B.decide", sync_stream_);
      phase_b_kernel<<<num_sms_ * 4, kThreads, 0, sync_stream_>>>(ctx_, round_dev_, worklist_, wc);
    }
    ADAPM_COUNT_LAUNCH();
    ADAPM_COUNT_LAUNCH();
    ADAPM_CUDA_CHECK(cudaGetLastError());
    return;
  }
  unsigned int* wc = work_count_ + (phase == 0 ? 0 : 1);   // one counter per phase (read back by the kernel timeline)
  ADAPM_CUDA_CHECK(cudaMemsetAsync(wc, 0, sizeof(unsigned int), sync_stream_));
  if (phase == 0) {
    { TraceScope t_(this, "A.scan", sync_stream_); phase_scan_kernel<0><<<num_sms_, kThreads, 0, sync_stream_>>>(ctx_, round_dev_, worklist_, wc); }
    {
      TraceScope t_(this, "A.resolve", sync_stream_);
      ADAPM_DISPATCH_VAL(int_rows_, ctx_.L.val_bytes,
                         phase_meta_kernel<Val, 0, 0><<<num_sms_, kThreads, 0, sync_stream_>>>(ctx_, round_dev_, worklist_, wc));
    }
    {
      TraceScope t_(this, "A.row", sync_stream_);
      ADAPM_DISPATCH_VAL(int_rows_, ctx_.L.val_bytes,
                         phase_row_kernel<Val><<<num_sms_, kWorkThreads, 0, sync_stream_>>>(ctx_, round_dev_, worklist_, wc));
    }
    {
      TraceScope t_(this, "A.commit", sync_stream_);
      ADAPM_DISPATCH_VAL(int_rows_, ctx_.L.val_bytes,
                         phase_meta_kernel<Val, 0, 1><<<num_sms_, kThreads, 0, sync_stream_>>>(ctx_, round_dev_, worklist_, wc));
    }
  } else {
    { TraceScope t_(this, "C.scan", sync_stream_); phase_scan_kernel<1><<<num_sms_, kThreads, 0, sync_stream_>>>(ctx_, round_dev_, worklist_, wc); }
    {
      TraceScope t_(this, "C.resolve", sync_stream_);
      ADAPM_DISPATCH_VAL(int_rows_, ctx_.L.val_bytes,
                         phase_meta_kernel<Val, 1, 0><<<num_sms_, kThreads, 0, sync_stream_>>>(ctx_, round_dev_, worklist_, wc));
    }
    {
      TraceScope t_(this, "C.row", sync_stream_);
      ADAPM_DISPATCH_VAL(int_rows_, ctx_.L.val_bytes,
                         phase_row_kernel<Val><<<num_sms_, kWorkThreads, 0, sync_stream_>>>(ctx_, round_dev_, worklist_, wc));
    }
    {
      TraceScope t_(this, "C.commit", sync_stream_);
      ADAPM_DISPATCH_VAL(int_rows_, ctx_.L.val_bytes,
                         phase_meta_kernel<Val, 1, 1><<<num_sms_, kThreads, 0, sync_stream_>>>(ctx_, round_dev_, worklist_, wc));
    }
  }
  for (int i = 0; i < 4; ++i) ADAPM_COUNT_LAUNCH();
  ADAPM_CUDA_CHECK(cudaGetLastError());
}

void CudaBackend::phase_a(const RoundParams& rp) {
  use_device();
  upload_round(rp, 0, 0);
  launch_phase(0);
}
void CudaBackend::phase_b(const RoundParams&) {
  use_device();
  launch_phase(1);
}
void CudaBackend::phase_c(const RoundParams&) {
  use_device();
  launch_phase(2);
}

// ---- device-resident round: ONE enqueue per round, nothing in it waits for the host.
//   upload {params, intent records} -> barrier 1 (+ stop/sweep agreement) -> register -> phase A -> barrier 2 ->
//   phase B -> barrier 3 -> grace (epoch flip + drain) -> barrier 4 -> phase C -> download {agreement, status}
// The ranks run the same sequence in lock-step; the barrier numbers derive from the round count.
RoundOutcome CudaBackend::fused_round(const RoundRequest& rq) {
  use_device();
  cudaStream_t s = sync_stream_;
  const size_t n = rq.n_recs;
  if (n > recs_cap_) {
    const size_t cap = std::max<size_t>(2 * n, 1 << 16);
    if (recs_dev_) { cudaFree(recs_dev_); cudaFreeHost(recs_host_); cudaFree(status_dev_); cudaFreeHost(status_host_); }
    ADAPM_CUDA_CHECK(cudaMalloc((void**)&recs_dev_, cap * sizeof(IntentRec)));
    ADAPM_CUDA_CHECK(cudaHostAlloc((void**)&recs_host_, cap * sizeof(IntentRec), cudaHostAllocDefault));
    ADAPM_CUDA_CHECK(cudaMalloc((void**)&status_dev_, cap));
    ADAPM_CUDA_CHECK(cudaHostAlloc((void**)&status_host_, cap, cudaHostAllocDefault));
    recs_cap_ = cap;
  }
  upload_round(rq.rp, (uint32_t)n, (rq.want_stop ? 1u : 0u) | (rq.want_sweep ? 2u : 0u));
  if (n) {
    memcpy(recs_host_, rq.recs, n * sizeof(IntentRec));
    ADAPM_CUDA_CHECK(cudaMemcpyAsync(recs_dev_, recs_host_, n * sizeof(IntentRec), cudaMemcpyHostToDevice, s));
  }
  const uint32_t seq0 = (uint32_t)(fused_rounds_ * 4);
  const uint32_t parity = (uint32_t)(fused_rounds_ & 1);
  uint32_t* abort_dev = nullptr;
  ADAPM_CUDA_CHECK(cudaHostGetDevicePointer((void**)&abort_dev, abort_word_, 0));
  auto xbar = [&](uint32_t k, int gather) {
    TraceScope ts_(this, "xbar", s);
    xbar_kernel<<<1, 64, 0, s>>>(ctx_, seq0 + k, parity, round_dev_, gather, abort_dev, dev_timeout_ns_);
    ADAPM_COUNT_LAUNCH();
  };
  xbar(1, 1);
  if (n) {
    TraceScope ts_(this, "register", s);
    ADAPM_DISPATCH_VAL(int_rows_, ctx_.L.val_bytes, register_kernel<Val><<<(int)((n + 255) / 256), 256, 0, s>>>(ctx_, recs_dev_, round_dev_, status_dev_));
    ADAPM_COUNT_LAUNCH();
  }
  launch_phase(0);
  xbar(2, 0);
  launch_phase(1);
  xbar(3, 0);
  {
    TraceScope ts_(this, "grace", s);
    grace_kernel<<<1, 1, 0, s>>>(ctx_, round_dev_, abort_dev, dev_timeout_ns_);
    ADAPM_COUNT_LAUNCH();
  }
  xbar(4, 0);
  launch_phase(2);
  ADAPM_CUDA_CHECK(cudaGetLastError());
  ADAPM_CUDA_CHECK(cudaMemcpyAsync(&round_host_[1], round_dev_, sizeof(RoundDev), cudaMemcpyDeviceToHost, s));
  if (trace_on_) ADAPM_CUDA_CHECK(cudaMemcpyAsync(abort_word_ + 4, work_count_, 2 * sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
  if (n) ADAPM_CUDA_CHECK(cudaMemcpyAsync(status_host_, status_dev_, n, cudaMemcpyDeviceToHost, s));
  ADAPM_CUDA_CHECK(cudaEventRecord(round_done_, s));
  ++fused_rounds_;
  // wait for the round; a failed peer (the failure detector breaks the control-plane barriers) aborts the device waits
  ControlBlock* ctl = fabric_->control();
  unsigned spins = 0;
  for (;;) {
    cudaError_t e = cudaEventQuery(round_done_);
    if (e == cudaSuccess) break;
    if (e != cudaErrorNotReady) ADAPM_CUDA_CHECK(e);
    if (++spins < 2000) std::this_thread::yield();
    else std::this_thread::sleep_for(std::chrono::microseconds(20));
    if ((spins & 255u) == 0 && ctl->sync_barrier.broken.load(std::memory_order_relaxed)) *abort_word_ = 1;
  }
  const RoundDev& res = round_host_[1];
  if (trace_on_) {
    std::lock_guard<std::mutex> lk(trace_mu_);
    if (trace_counts_.size() < ((size_t)1 << 20)) trace_counts_.push_back({(uint32_t)n, abort_word_[4], abort_word_[5]});
  }
  if (res.error) {
    ctl->sync_barrier.broken.store(1);
    throw Error(res.error == 1 ? "sync round: a device-side cross-rank barrier timed out or was aborted (a peer died or hangs)"
                               : "sync round: the grace period did not end (a kernel that touches the store hangs)");
  }
  if (n && rq.status) memcpy(rq.status, status_host_, n);
  RoundOutcome out;
  out.all_stop = res.stop != 0;
  out.any_sweep = res.any_sweep != 0;
  return out;
}
// ---------------------------------------------------------------------------------------- kernel timeline
CudaBackend::TraceScope::TraceScope(CudaBackend* be, const char* name, cudaStream_t st) : b(be), idx(-1), s(st) {
  if (!b->trace_on_) return;
  std::lock_guard<std::mutex> lk(b->trace_mu_);
  if (b->trace_.size() >= (size_t)1 << 20) return;
  if (!b->trace_base_) {
    cudaEventCreate(&b->trace_base_);
    cudaEventRecord(b->trace_base_, s);
  }
  TraceRec r;
  r.name = name;
  cudaEventCreate(&r.a);
  cudaEventCreate(&r.b);
  cudaEventRecord(r.a, s);
  idx = (int)b->trace_.size();
  b->trace_.push_back(r);
}
CudaBackend::TraceScope::~TraceScope() {
  if (idx < 0) return;
  std::lock_guard<std::mutex> lk(b->trace_mu_);
  cudaEventRecord(b->trace_[idx].b, s);
}
void CudaBackend::trace_mark(const char* name, void* stream) {
  if (!trace_on_) return;
  use_device();
  TraceScope t(this, name, (cudaStream_t)stream);
}
void CudaBackend::dump_trace(const std::string& path) {
  if (!trace_on_) return;
  use_device();
  cudaDeviceSynchronize();
  std::lock_guard<std::mutex> lk(trace_mu_);
  FILE* f = fopen(path.c_str(), "w");
  if (!f) return;
  fprintf(f, "name\tstart_ms\tend_ms\n");
  for (auto& r : trace_) {
    float a = 0, b = 0;
    if (cudaEventElapsedTime(&a, trace_base_, r.a) != cudaSuccess) { cudaGetLastError(); continue; }
    if (cudaEventElapsedTime(&b, trace_base_, r.b) != cudaSuccess) { cudaGetLastError(); b = a; }
    fprintf(f, "%s\t%.4f\t%.4f\n", r.name, a, b);
    cudaEventDestroy(r.a);
    cudaEventDestroy(r.b);
  }
  fclose(f);
  trace_.clear();
  if (!trace_counts_.empty()) {   // per round: intent records registered, phase A worklist, phase C worklist
    FILE* g = fopen((path + ".counts").c_str(), "w");
    if (g) {
      fprintf(g, "recs\tworkA\tworkC\n");
      for (auto& c3 : trace_counts_) fprintf(g, "%u\t%u\t%u\n", c3[0], c3[1], c3[2]);
      fclose(g);
    }
    trace_counts_.clear();
  }
}

void CudaBackend::round_fence() {
  use_device();
  ADAPM_CUDA_CHECK(cudaStreamSynchronize(sync_stream_));
}

void CudaBackend::grace() {
  use_device();
  std::vector<cudaStream_t> ss;
  {
    std::lock_guard<std::mutex> lk(streams_mu_);
    ss.assign(tracked_.begin(), tracked_.end());
  }
  // One event per stream: everything enqueued before this point (which may have read the old
  // directory) must have finished before the relocation transfers start.
  std::vector<cudaEvent_t> evs(ss.size());
  for (size_t i = 0; i < ss.size(); ++i) {
    ADAPM_CUDA_CHECK(cudaEventCreateWithFlags(&evs[i], cudaEventDisableTiming));
    ADAPM_CUDA_CHECK(cudaEventRecord(evs[i], ss[i]));
  }
  for (size_t i = 0; i < ss.size(); ++i) {
    ADAPM_CUDA_CHECK(cudaEventSynchronize(evs[i]));
    cudaEventDestroy(evs[i]);
  }
}

void CudaBackend::read_counters(uint64_t* out) {
  use_device();
  ADAPM_CUDA_CHECK(cudaMemcpy(out, ctx_.heap[ctx_.rank] + ctx_.L.off_counters, C_NUM_COUNTERS * 8, cudaMemcpyDeviceToHost));
}
void CudaBackend::read_heap(uint64_t off, void* dst, size_t bytes) {
  use_device();
  ADAPM_CUDA_CHECK(cudaMemcpy(dst, ctx_.heap[ctx_.rank] + off, bytes, cudaMemcpyDeviceToHost));
}
void CudaBackend::reset_counters() {
  use_device();
  ADAPM_CUDA_CHECK(cudaMemset(ctx_.heap[ctx_.rank] + ctx_.L.off_counters, 0, C_NUM_COUNTERS * 8));
}

std::unique_ptr<Backend> make_cuda_backend(const Options& opt, const Layout& L, std::shared_ptr<Fabric> fabric) {
  return std::unique_ptr<Backend>(new CudaBackend(opt, L, fabric));
}

}  // namespace adapm

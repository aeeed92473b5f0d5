// CudaBackend: the GPU executor of the protocol. One instance per rank = per GPU.
// Heaps are peer-mapped device allocations (VMM handles + NVLS multicast or CUDA IPC across
// processes - fabric.cc; peer access inside one process); every kernel receives the Ctx by value and dereferences peer heaps
// directly, so Pull = NVLink loads, Push = NVLink reductions (REDG), directory updates =
// NVLink stores - all issued from inside the kernels.
#pragma once
#include <cuda_runtime.h>

#include <array>
#include <mutex>
#include <set>
#include <unordered_map>

#include "../adapm/store.h"

namespace adapm {

// number of kernels this library launched in this process (bench.py reports it as gpu_launches)
std::atomic<uint64_t>& kernel_launch_counter();
#define ADAPM_COUNT_LAUNCH() (::adapm::kernel_launch_counter().fetch_add(1, std::memory_order_relaxed))

// Device-resident parameters and results of the round in flight: uploaded by the host once per round; the first
// cross-rank barrier of the round fills in what the ranks agreed on.
struct RoundDev {
  RoundParams rp;
  uint32_t n_recs;
  uint32_t my_flags;    // in : bit 0 = this rank wants to stop, bit 1 = this rank wants a guaranteed-propagation round
  uint32_t stop;        // out: every rank wants to stop -> the rest of the round is skipped on all ranks
  uint32_t any_sweep;   // out
  uint32_t error;       // out: 1 = a cross-rank barrier, 2 = the grace period timed out / was aborted
  uint32_t pad[3];
};

class CudaBackend : public Backend {
 public:
  CudaBackend(const Options& opt, const Layout& L, std::shared_ptr<Fabric> fabric);
  ~CudaBackend() override;

  const Ctx& ctx() const override { return ctx_; }
  bool is_cuda() const override { return true; }
  void init_store(const std::vector<uint8_t>& key_class, const std::vector<uint32_t>& key_lens) override;

  uint64_t pull(int worker, const Key* keys, size_t n, void* vals, bool local_only, uint8_t* ok, OpResult* res,
                const IoDesc& io) override;
  uint64_t push(int worker, const Key* keys, size_t n, const void* vals, bool set, OpResult* res,
                const IoDesc& io, uint8_t* todo = nullptr) override;
  void wait_ticket(uint64_t t) override;
  bool ticket_done(uint64_t t) override;
  void wait_worker(int worker) override;
  bool key_is_local(Key k) override;
  void peek_states(const Key* keys, size_t n, uint8_t* state_out, uint8_t* owner_out) override;

  void register_intents(const IntentRec* recs, size_t n, const RoundParams& rp, uint8_t* status) override;
  void phase_a(const RoundParams& rp) override;
  void phase_b(const RoundParams& rp) override;
  void phase_c(const RoundParams& rp) override;
  void round_fence() override;
  void grace() override;
  bool has_fused_round() const override { return fused_round_; }
  RoundOutcome fused_round(const RoundRequest& rq) override;
  void read_counters(uint64_t* out) override;
  void reset_counters() override;
  void read_heap(uint64_t off, void* dst, size_t bytes) override;

  // ---- used by the fused application kernels (cuda/ops_*.cu)
  int device() const { return device_; }
  cudaStream_t worker_stream(int w) const { return worker_streams_[w]; }
  cudaStream_t sync_stream() const { return sync_stream_; }
  void track_stream(cudaStream_t s);            // streams that launch kernels touching the store
  uint64_t record_ticket(cudaStream_t s);       // completion ticket for work enqueued so far on s
  cudaStream_t resolve_stream(int worker, const IoDesc& io) {
    cudaStream_t s = io.has_stream ? (cudaStream_t)io.stream : worker_streams_[worker];
    track_stream(s);
    return s;
  }
  int num_sms() const { return num_sms_; }
  // device scratch of the deterministic one-GPU steps (fx_accum.cuh), owned by the backend, grown on demand: fixed-point
  // accumulator regions, the region offset of every key touched by the step (-1 = none) and the step's regions
  struct FxScratch {
    long long* acc = nullptr;          // [acc_len], zero between steps
    size_t acc_len = 0;
    int* cidx = nullptr;               // [num_keys] region offset in units
    Key* keys = nullptr;               // [rows] key of region r
    int2* rows = nullptr;              // [rows] (offset, length) of region r, in units
    size_t rows_cap = 0;
    size_t step_rows = 0;              // bound on the regions of the current step
    unsigned int* count = nullptr;     // [2]: regions of the current step, units handed out
    unsigned long long* loss = nullptr;   // fixed-point loss (SGNS)
    float* call_loss = nullptr;        // [calls] loss of every call of the step (KGE, MF)
    size_t calls_cap = 0;
  };
  FxScratch& fx_scratch(size_t acc_len, size_t rows, size_t calls);
  // number of keys whose rows have `len` values (every key for a store of one row length)
  size_t keys_with_len(uint32_t len);
  // device buffer i (< kStepBuffers) of at least `bytes`, grown on demand and zero-filled when it grows (a buffer that
  // its user leaves zero stays zero); scratch of the deterministic one-GPU SGNS step (ops_sgns_tma.cu, buffers 0 - 9)
  // and of the TransE step's generic path (ops_transe.cu, buffer 11)
  static constexpr int kStepBuffers = 12;
  void* step_buffer(int i, size_t bytes);

  // ---- kernel timeline: CUDA events around every sync-round kernel plus user marks, all relative to one base
  // event, so that the round's kernels and the training kernels of other streams land on one time axis
  void trace_mark(const char* name, void* stream) override;
  void dump_trace(const std::string& path) override;
  struct TraceScope {
    TraceScope(CudaBackend* b, const char* name, cudaStream_t s);
    ~TraceScope();
    CudaBackend* b; int idx; cudaStream_t s;
  };

 private:
  struct Staging {
    char* host = nullptr;
    char* dev = nullptr;
    size_t bytes = 0;
    std::mutex mu;
  };
  void ensure_staging(Staging& st, size_t bytes);
  void use_device() const;

  std::shared_ptr<Fabric> fabric_;
  Ctx ctx_;
  bool int_rows_ = false;   // Options::dtype == int64 (8-byte rows are float64 otherwise)
  int device_ = 0;
  // The sync-round kernels run one block per SM. The round runs on a high-priority stream next to the training
  // kernels: a small footprint lets it share the SMs with them instead of displacing them.
  int num_sms_ = 132;
  struct TraceRec { const char* name; cudaEvent_t a, b; };
  bool trace_on_ = false;        // ADAPM_SYNC_TRACE
  cudaEvent_t trace_base_ = nullptr;
  std::vector<TraceRec> trace_;
  std::vector<std::array<uint32_t, 3>> trace_counts_;
  std::mutex trace_mu_;
  cudaStream_t sync_stream_ = nullptr;
  std::vector<cudaStream_t> worker_streams_;
  std::vector<std::unique_ptr<Staging>> staging_;  // per worker
  Staging sync_staging_;
  std::mutex streams_mu_;
  std::set<cudaStream_t> tracked_;
  std::mutex tickets_mu_;
  std::unordered_map<uint64_t, cudaEvent_t> tickets_;
  std::vector<cudaEvent_t> event_pool_;
  uint64_t next_ticket_ = 1;
  SlotWork* worklist_ = nullptr;       // slots that need work in the current phase (device), one record each
  unsigned int* work_count_ = nullptr;
  // device-resident round (default for world > 1; ADAPM_HOST_ROUND=1 selects the host-sequenced round)
  void upload_round(const RoundParams& rp, uint32_t n_recs, uint32_t flags);
  void launch_phase(int phase);   // 0 = A, 1 = B, 2 = C
  bool fused_round_ = false;
  RoundDev* round_dev_ = nullptr;      // device
  RoundDev* round_host_ = nullptr;     // pinned: [0] = upload staging, [1] = results
  uint32_t* abort_word_ = nullptr;     // pinned + mapped: set by the host to break device-side waits
  IntentRec* recs_dev_ = nullptr;
  IntentRec* recs_host_ = nullptr;     // pinned
  uint8_t* status_dev_ = nullptr;
  uint8_t* status_host_ = nullptr;     // pinned
  size_t recs_cap_ = 0;
  cudaEvent_t round_done_ = nullptr;
  uint64_t fused_rounds_ = 0;          // barrier sequence numbers derive from it (same on every rank)
  unsigned long long dev_timeout_ns_ = 20ull * 1000000000ull;
  std::vector<uint32_t> key_len_;   // host mirror of per-key lengths (mixed-length stores only)
  FxScratch fx_;
  std::array<std::pair<void*, size_t>, kStepBuffers> step_bufs_{};
  std::unordered_map<uint32_t, size_t> keys_by_len_;   // keys_with_len cache (mixed-length stores)
};

}  // namespace adapm

// Fabric: how ranks find each other's control block and symmetric heaps.
//
//   inproc  ranks are objects/threads of one process (CPU tests; several logical ranks
//           on one GPU); heaps are plain allocations visible to everybody.
//   shm     one process per rank on one host (the torchrun model). The control block is
//           a POSIX shm segment. CPU heaps are shm segments mapped by every rank; CUDA
//           heaps are VMM allocations (cuMemCreate) whose handles travel as POSIX file
//           descriptors over a unix datagram socket (SCM_RIGHTS, once at start-up), are
//           mapped by every peer and bound to an NVLS multicast object when the devices
//           support it; cudaMalloc + CUDA IPC is the fallback. Peers read and write the
//           heaps directly over NVLink/NVSwitch.
//
// This is the GPU-native stand-in for ZMQVan + Van + Postoffice node management
// (include/zmq_van.h:30-250, src/van.cc:267-357): no data ever travels through a socket
// and there is no message (de)serialisation anywhere.
#pragma once
#include <atomic>
#include <memory>
#include <thread>
#include <string>
#include <vector>
#include "config.h"
#include "control.h"

namespace adapm {

class Fabric {
 public:
  static std::shared_ptr<Fabric> create(const Options& opt);
  virtual ~Fabric() {}

  ControlBlock* control() { return ctl_; }
  int rank() const { return rank_; }
  int world() const { return world_; }
  bool cuda() const { return cuda_; }
  bool peers_are_processes() const { return peers_are_processes_; }   // one process (and GPU) per rank
  int device() const { return device_; }

  // Collective: allocate `bytes` for this rank (zero-filled) and map all peers' heaps.
  virtual void allocate_heaps(uint64_t bytes) = 0;
  char* heap(int r) const { return heaps_[r]; }
  // NVLS multicast mapping of the heaps (cuda, one process per GPU, NVSwitch): a store / reduction to mc_heap() + off
  // reaches offset `off` of EVERY rank's heap in one NVLink transaction. nullptr when the box has no multicast support.
  char* mc_heap() const { return mc_heap_; }

  void node_barrier(const char* what) {
    ctl_->node_barrier.wait(world_, timeout_s_, what);
  }

  // Failure detector (the reference's heartbeat skeleton, van.cc:529-548, made effective): a thread that checks
  // every `period_ms` whether the processes of the other ranks are still alive; a dead peer breaks all barriers so
  // that every blocked call on this rank raises instead of waiting for the watchdog timeout. No-op for in-process
  // ranks. stop_failure_detector() is called before the last shutdown barrier (peers exit at different times).
  void start_failure_detector(int period_ms = 200);
  void stop_failure_detector();
  int dead_peer() const { return dead_peer_.load(); }   // -1: none detected

 protected:
  ControlBlock* ctl_ = nullptr;
  int rank_ = 0, world_ = 1, device_ = -1;
  bool cuda_ = false;
  double timeout_s_ = 300;
  std::vector<char*> heaps_;
  char* mc_heap_ = nullptr;
  bool peers_are_processes_ = false;
  std::thread fd_thread_;
  std::atomic<bool> fd_stop_{false};
  std::atomic<int> dead_peer_{-1};
};

bool fabric_fdpass_selftest();   // unit test hook of the descriptor channel between ranks (fabric.cc)

// device helpers implemented in cuda/device_mem.cu (only linked in the cuda build)
namespace cudamem {
bool available();
int device_count();
void set_device(int dev);
char* alloc_zeroed(uint64_t bytes);               // cudaMalloc + memset
void free_dev(char* p);
void export_handle(char* p, unsigned char* out128);   // cudaIpcGetMemHandle
char* import_handle(const unsigned char* in128);      // cudaIpcOpenMemHandle
void close_handle(char* p);
void enable_peer(int my_dev, int peer_dev);

// ---- CUDA virtual memory management (cuMemCreate / cuMemMap) + NVLS multicast objects (cuMulticastCreate), used by
// the shm fabric when the driver supports them: the heap of a rank is ONE physical allocation that peers import through
// a POSIX file descriptor (sent over a unix socket) and that is bound to a multicast object spanning all ranks.
// All driver entry points are resolved at run time (cudaGetDriverEntryPoint): no link-time dependency on libcuda.
struct VmmHeap {
  char* va = nullptr;          // mapping in this process
  uint64_t size = 0;           // padded to the allocation / multicast granularity
  unsigned long long handle = 0;   // CUmemGenericAllocationHandle
};
bool vmm_supported(int dev, bool* multicast);        // VMM + POSIX-fd handles (and multicast objects) on this device
uint64_t vmm_granularity(int dev, int world, bool multicast);
VmmHeap vmm_alloc(int dev, uint64_t size);           // zero-filled, mapped read/write for `dev`
int vmm_export_fd(const VmmHeap& h);
VmmHeap vmm_import_fd(int dev, int fd, uint64_t size);   // peer's allocation mapped read/write for `dev` (closes fd)
void vmm_free(VmmHeap& h);
// multicast object: created by one rank, imported by the others through an fd, every rank adds its device, then binds
// its heap and maps the object
unsigned long long mc_create(int world, uint64_t size, int* fd_out);
unsigned long long mc_import_fd(int fd);
void mc_add_device(unsigned long long mc, int dev);
char* mc_bind_and_map(unsigned long long mc, int dev, const VmmHeap& heap);
void mc_unmap(unsigned long long mc, int dev, char* va, uint64_t size);
}  // namespace cudamem

}  // namespace adapm

// Device memory helpers behind fabric.h's cudamem namespace: heap allocation, the NVLink/NVSwitch
// peer mapping between one-process-per-GPU ranks (VMM allocations exported as file descriptors,
// NVLS multicast objects; CUDA IPC export/import as the fallback) and peer access between devices
// of one process. The driver API is resolved at run time (cudaGetDriverEntryPoint): no libcuda link.
#include <cuda_runtime.h>
#include <cstring>
#include <sstream>
#include "../adapm/fabric.h"
#include "group.cuh"

namespace adapm {
namespace cudamem {

bool available() {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) { cudaGetLastError(); return false; }
  return n > 0;
}
int device_count() {
  int n = 0;
  ADAPM_CUDA_CHECK(cudaGetDeviceCount(&n));
  return n;
}
void set_device(int dev) { ADAPM_CUDA_CHECK(cudaSetDevice(dev)); }
char* alloc_zeroed(uint64_t bytes) {
  void* p = nullptr;
  ADAPM_CUDA_CHECK(cudaMalloc(&p, bytes));
  ADAPM_CUDA_CHECK(cudaMemset(p, 0, bytes));
  ADAPM_CUDA_CHECK(cudaDeviceSynchronize());
  return (char*)p;
}
void free_dev(char* p) { cudaFree(p); }
void export_handle(char* p, unsigned char* out128) {
  static_assert(sizeof(cudaIpcMemHandle_t) <= 128, "ipc handle size");
  cudaIpcMemHandle_t h;
  ADAPM_CUDA_CHECK(cudaIpcGetMemHandle(&h, p));
  memset(out128, 0, 128);
  memcpy(out128, &h, sizeof(h));
}
char* import_handle(const unsigned char* in128) {
  cudaIpcMemHandle_t h;
  memcpy(&h, in128, sizeof(h));
  void* p = nullptr;
  ADAPM_CUDA_CHECK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  return (char*)p;
}
void close_handle(char* p) { cudaIpcCloseMemHandle(p); }
void enable_peer(int my_dev, int peer_dev) {
  if (my_dev == peer_dev) return;
  int can = 0;
  ADAPM_CUDA_CHECK(cudaDeviceCanAccessPeer(&can, my_dev, peer_dev));
  if (!can) throw Error("device " + std::to_string(my_dev) + " cannot access peer " + std::to_string(peer_dev) + " (no NVLink/P2P path)");
  cudaError_t e = cudaDeviceEnablePeerAccess(peer_dev, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return; }
  ADAPM_CUDA_CHECK(e);
}

}  // namespace cudamem
}  // namespace adapm

// ------------------------------------------------------------------------------------------------------------------
// Virtual memory management + NVLS multicast (driver API, resolved at run time)
#include <cuda.h>
#include <unistd.h>

namespace adapm {
namespace cudamem {

namespace {

template <class F> F driver_fn(const char* name) {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qr;
  cudaError_t e = cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &qr);
  if (e != cudaSuccess || qr != cudaDriverEntryPointSuccess || !fn) {
    cudaGetLastError();
    return nullptr;
  }
  return reinterpret_cast<F>(fn);
}

struct DriverApi {
  CUresult (*DeviceGet)(CUdevice*, int) = nullptr;
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice) = nullptr;
  CUresult (*GetErrorString)(CUresult, const char**) = nullptr;
  CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*MemRelease)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*MemAddressFree)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*MemUnmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
  CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long) = nullptr;
  CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType) = nullptr;
  CUresult (*MulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*) = nullptr;
  CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice) = nullptr;
  CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long) = nullptr;
  CUresult (*MulticastUnbind)(CUmemGenericAllocationHandle, CUdevice, size_t, size_t) = nullptr;
  CUresult (*MulticastGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags) = nullptr;
  bool ok = false, mc_ok = false;
};

const DriverApi& drv() {
  static const DriverApi api = [] {
    DriverApi a;
    cudaFree(0);   // make sure the runtime (and with it the driver) is initialised
#define ADAPM_DRV(field, name) a.field = driver_fn<decltype(a.field)>(name)
    ADAPM_DRV(DeviceGet, "cuDeviceGet");
    ADAPM_DRV(DeviceGetAttribute, "cuDeviceGetAttribute");
    ADAPM_DRV(GetErrorString, "cuGetErrorString");
    ADAPM_DRV(MemCreate, "cuMemCreate");
    ADAPM_DRV(MemRelease, "cuMemRelease");
    ADAPM_DRV(MemAddressReserve, "cuMemAddressReserve");
    ADAPM_DRV(MemAddressFree, "cuMemAddressFree");
    ADAPM_DRV(MemMap, "cuMemMap");
    ADAPM_DRV(MemUnmap, "cuMemUnmap");
    ADAPM_DRV(MemSetAccess, "cuMemSetAccess");
    ADAPM_DRV(MemGetAllocationGranularity, "cuMemGetAllocationGranularity");
    ADAPM_DRV(MemExportToShareableHandle, "cuMemExportToShareableHandle");
    ADAPM_DRV(MemImportFromShareableHandle, "cuMemImportFromShareableHandle");
    ADAPM_DRV(MulticastCreate, "cuMulticastCreate");
    ADAPM_DRV(MulticastAddDevice, "cuMulticastAddDevice");
    ADAPM_DRV(MulticastBindMem, "cuMulticastBindMem");
    ADAPM_DRV(MulticastUnbind, "cuMulticastUnbind");
    ADAPM_DRV(MulticastGetGranularity, "cuMulticastGetGranularity");
#undef ADAPM_DRV
    a.ok = a.DeviceGet && a.DeviceGetAttribute && a.MemCreate && a.MemRelease && a.MemAddressReserve && a.MemAddressFree &&
           a.MemMap && a.MemUnmap && a.MemSetAccess && a.MemGetAllocationGranularity && a.MemExportToShareableHandle &&
           a.MemImportFromShareableHandle;
    a.mc_ok = a.ok && a.MulticastCreate && a.MulticastAddDevice && a.MulticastBindMem && a.MulticastGetGranularity;
    return a;
  }();
  return api;
}

#define ADAPM_CU_CHECK(expr)                                                                    \
  do {                                                                                          \
    CUresult _r = (expr);                                                                       \
    if (_r != CUDA_SUCCESS) {                                                                   \
      const char* _s = nullptr;                                                                 \
      if (drv().GetErrorString) drv().GetErrorString(_r, &_s);                                  \
      std::ostringstream _os;                                                                   \
      _os << "[adapm] CUDA driver error " << (int)_r << " (" << (_s ? _s : "?") << ") at "      \
          << __FILE__ << ":" << __LINE__ << ": " #expr;                                         \
      throw ::adapm::Error(_os.str());                                                          \
    }                                                                                           \
  } while (0)

CUmemAllocationProp alloc_prop(int dev) {
  CUmemAllocationProp p;
  memset(&p, 0, sizeof(p));
  p.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  p.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  p.location.id = dev;
  p.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  return p;
}

char* map_handle(int dev, CUmemGenericAllocationHandle h, uint64_t size, uint64_t align) {
  CUdeviceptr va = 0;
  ADAPM_CU_CHECK(drv().MemAddressReserve(&va, size, align, 0, 0));
  ADAPM_CU_CHECK(drv().MemMap(va, size, 0, h, 0));
  CUmemAccessDesc ad;
  memset(&ad, 0, sizeof(ad));
  ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  ad.location.id = dev;
  ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  ADAPM_CU_CHECK(drv().MemSetAccess(va, size, &ad, 1));
  return reinterpret_cast<char*>(va);
}

}  // namespace

bool vmm_supported(int dev, bool* multicast) {
  if (multicast) *multicast = false;
  const DriverApi& a = drv();
  if (!a.ok) return false;
  CUdevice d;
  if (a.DeviceGet(&d, dev) != CUDA_SUCCESS) return false;
  int vmm = 0, fd = 0, mc = 0;
  a.DeviceGetAttribute(&vmm, CU_DEVICE_ATTRIBUTE_VIRTUAL_MEMORY_MANAGEMENT_SUPPORTED, d);
  a.DeviceGetAttribute(&fd, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, d);
  if (a.mc_ok) a.DeviceGetAttribute(&mc, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, d);
  if (multicast) *multicast = mc != 0;
  return vmm != 0 && fd != 0;
}

uint64_t vmm_granularity(int dev, int world, bool multicast) {
  CUmemAllocationProp p = alloc_prop(dev);
  size_t g = 0;
  ADAPM_CU_CHECK(drv().MemGetAllocationGranularity(&g, &p, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
  if (multicast) {
    CUmulticastObjectProp mp;
    memset(&mp, 0, sizeof(mp));
    mp.numDevices = (unsigned)world;
    mp.size = g;
    mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t mg = 0;
    // (the RECOMMENDED multicast granularity can be far larger; the minimum - 2 MB - is what binding requires)
    ADAPM_CU_CHECK(drv().MulticastGetGranularity(&mg, &mp, CU_MULTICAST_GRANULARITY_MINIMUM));
    if (mg > g) g = mg;
  }
  return g;
}

VmmHeap vmm_alloc(int dev, uint64_t size) {
  VmmHeap h;
  CUmemAllocationProp p = alloc_prop(dev);
  CUmemGenericAllocationHandle hd;
  ADAPM_CU_CHECK(drv().MemCreate(&hd, size, &p, 0));
  h.handle = hd;
  h.size = size;
  h.va = map_handle(dev, hd, size, 2ull << 20);
  ADAPM_CUDA_CHECK(cudaMemset(h.va, 0, size));
  ADAPM_CUDA_CHECK(cudaDeviceSynchronize());
  return h;
}

int vmm_export_fd(const VmmHeap& h) {
  int fd = -1;
  ADAPM_CU_CHECK(drv().MemExportToShareableHandle(&fd, (CUmemGenericAllocationHandle)h.handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
  return fd;
}

VmmHeap vmm_import_fd(int dev, int fd, uint64_t size) {
  VmmHeap h;
  CUmemGenericAllocationHandle hd;
  ADAPM_CU_CHECK(drv().MemImportFromShareableHandle(&hd, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
  close(fd);
  h.handle = hd;
  h.size = size;
  h.va = map_handle(dev, hd, size, 2ull << 20);
  return h;
}

void vmm_free(VmmHeap& h) {
  if (!h.va) return;
  drv().MemUnmap((CUdeviceptr)h.va, h.size);
  drv().MemAddressFree((CUdeviceptr)h.va, h.size);
  drv().MemRelease((CUmemGenericAllocationHandle)h.handle);
  h.va = nullptr;
}

unsigned long long mc_create(int world, uint64_t size, int* fd_out) {
  CUmulticastObjectProp mp;
  memset(&mp, 0, sizeof(mp));
  mp.numDevices = (unsigned)world;
  mp.size = size;
  mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  CUmemGenericAllocationHandle mc;
  ADAPM_CU_CHECK(drv().MulticastCreate(&mc, &mp));
  int fd = -1;
  ADAPM_CU_CHECK(drv().MemExportToShareableHandle(&fd, mc, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
  *fd_out = fd;
  return mc;
}

unsigned long long mc_import_fd(int fd) {
  CUmemGenericAllocationHandle mc;
  ADAPM_CU_CHECK(drv().MemImportFromShareableHandle(&mc, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
  close(fd);
  return mc;
}

void mc_add_device(unsigned long long mc, int dev) {
  CUdevice d;
  ADAPM_CU_CHECK(drv().DeviceGet(&d, dev));
  ADAPM_CU_CHECK(drv().MulticastAddDevice((CUmemGenericAllocationHandle)mc, d));
}

char* mc_bind_and_map(unsigned long long mc, int dev, const VmmHeap& heap) {
  ADAPM_CU_CHECK(drv().MulticastBindMem((CUmemGenericAllocationHandle)mc, 0, (CUmemGenericAllocationHandle)heap.handle, 0, heap.size, 0));
  return map_handle(dev, (CUmemGenericAllocationHandle)mc, heap.size, 2ull << 20);
}

void mc_unmap(unsigned long long mc, int dev, char* va, uint64_t size) {
  if (va) {
    drv().MemUnmap((CUdeviceptr)va, size);
    drv().MemAddressFree((CUdeviceptr)va, size);
  }
  CUdevice d;
  if (drv().MulticastUnbind && drv().DeviceGet(&d, dev) == CUDA_SUCCESS) drv().MulticastUnbind((CUmemGenericAllocationHandle)mc, d, 0, size);
  drv().MemRelease((CUmemGenericAllocationHandle)mc);
}

}  // namespace cudamem
}  // namespace adapm

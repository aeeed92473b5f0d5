// Probe: does this box support NVLS multicast objects (cuMulticastCreate) between 2+ GPUs, and do multimem.st /
// multimem.ld_reduce / multimem.red work on them? Single process, one context per device.
//   nvcc -gencode arch=compute_90a,code=sm_90a -o mc_probe mc_probe.cu -lcuda
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>
#define CK(x) do { CUresult r_ = (x); if (r_ != CUDA_SUCCESS) { const char* s_; cuGetErrorString(r_, &s_); \
  printf("FAIL %s -> %d %s (line %d)\n", #x, (int)r_, s_ ? s_ : "?", __LINE__); return 1; } } while (0)
#define CR(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("FAIL %s -> %s (line %d)\n", #x, cudaGetErrorString(e_), __LINE__); return 1; } } while (0)

__global__ void mc_store(float* mc, int n, float v) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i * 4 < n)
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc + 4 * i), "f"(v), "f"(v + 1),
                 "f"(v + 2), "f"(v + 3) : "memory");
}
__global__ void mc_red(float* mc, int n, float v) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i * 4 < n) asm volatile("multimem.red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc + 4 * i), "f"(v), "f"(v), "f"(v), "f"(v) : "memory");
}
__global__ void mc_ldreduce(const float* mc, float* out, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i * 4 < n) {
    float a, b, c, d;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(a), "=f"(b), "=f"(c), "=f"(d) : "l"(mc + 4 * i) : "memory");
    out[4 * i] = a; out[4 * i + 1] = b; out[4 * i + 2] = c; out[4 * i + 3] = d;
  }
}
__global__ void fill(float* p, int n, float v) { int i = blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] = v; }

int main() {
  CK(cuInit(0));
  int ndev = 0; CK(cuDeviceGetCount(&ndev));
  printf("devices: %d\n", ndev);
  for (int d = 0; d < ndev; ++d) {
    CUdevice dev; CK(cuDeviceGet(&dev, d));
    int mc = 0, vmm = 0, fab = 0, fd = 0;
    cuDeviceGetAttribute(&mc, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev);
    cuDeviceGetAttribute(&vmm, CU_DEVICE_ATTRIBUTE_VIRTUAL_MEMORY_MANAGEMENT_SUPPORTED, dev);
    cuDeviceGetAttribute(&fab, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_FABRIC_SUPPORTED, dev);
    cuDeviceGetAttribute(&fd, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, dev);
    printf("dev %d: multicast=%d vmm=%d fabric_handle=%d posix_fd_handle=%d\n", d, mc, vmm, fab, fd);
  }
  if (ndev < 2) { printf("RESULT single device: multicast object needs >= 2 devices, attribute only\n"); return 0; }
  const int N = ndev < 8 ? ndev : 8;
  const size_t want = 4 << 20;
  CUmulticastObjectProp mp = {};
  mp.numDevices = N; mp.size = want; mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  size_t gran = 0, gran_rec = 0;
  CK(cuMulticastGetGranularity(&gran, &mp, CU_MULTICAST_GRANULARITY_MINIMUM));
  CK(cuMulticastGetGranularity(&gran_rec, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED));
  printf("multicast granularity min=%zu recommended=%zu\n", gran, gran_rec);
  size_t size = (want + gran_rec - 1) / gran_rec * gran_rec;
  mp.size = size;
  CUmemGenericAllocationHandle mch;
  CK(cuMulticastCreate(&mch, &mp));
  std::vector<CUmemGenericAllocationHandle> mem(N);
  std::vector<CUdeviceptr> uc(N), mcva(N);
  for (int d = 0; d < N; ++d) { CUdevice dev; CK(cuDeviceGet(&dev, d)); CK(cuMulticastAddDevice(mch, dev)); }
  for (int d = 0; d < N; ++d) {
    CR(cudaSetDevice(d)); CR(cudaFree(0));
    CUmemAllocationProp ap = {};
    ap.type = CU_MEM_ALLOCATION_TYPE_PINNED; ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE; ap.location.id = d;
    ap.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t g2 = 0; CK(cuMemGetAllocationGranularity(&g2, &ap, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
    if (d == 0) printf("mem granularity recommended=%zu\n", g2);
    CK(cuMemCreate(&mem[d], size, &ap, 0));
    CK(cuMulticastBindMem(mch, 0, mem[d], 0, size, 0));
    CUmemAccessDesc ad = {}; ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE; ad.location.id = d; ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    CK(cuMemAddressReserve(&uc[d], size, g2, 0, 0)); CK(cuMemMap(uc[d], size, 0, mem[d], 0)); CK(cuMemSetAccess(uc[d], size, &ad, 1));
    CK(cuMemAddressReserve(&mcva[d], size, gran_rec, 0, 0)); CK(cuMemMap(mcva[d], size, 0, mch, 0)); CK(cuMemSetAccess(mcva[d], size, &ad, 1));
  }
  const int n = 1 << 16;
  for (int d = 0; d < N; ++d) { CR(cudaSetDevice(d)); fill<<<n / 256, 256>>>((float*)uc[d], n, 0.f); CR(cudaDeviceSynchronize()); }
  CR(cudaSetDevice(0));
  mc_store<<<n / 4 / 256, 256>>>((float*)mcva[0], n, 5.f); CR(cudaDeviceSynchronize());
  for (int d = 0; d < N; ++d) {
    CR(cudaSetDevice(d));
    mc_red<<<n / 4 / 256, 256>>>((float*)mcva[d], n, 1.f); CR(cudaDeviceSynchronize());
  }
  bool ok = true;
  for (int d = 0; d < N; ++d) {
    CR(cudaSetDevice(d));
    float h[8]; CR(cudaMemcpy(h, (void*)uc[d], sizeof(h), cudaMemcpyDeviceToHost));
    printf("dev %d after multimem.st(5..8) + %d x multimem.red(+1): %g %g %g %g\n", d, N, h[0], h[1], h[2], h[3]);
    ok = ok && h[0] == 5.f + N && h[3] == 8.f + N;
  }
  CR(cudaSetDevice(N - 1));
  float* out; CR(cudaMalloc(&out, n * 4));
  mc_ldreduce<<<n / 4 / 256, 256>>>((const float*)mcva[N - 1], out, n); CR(cudaDeviceSynchronize());
  float h[4]; CR(cudaMemcpy(h, out, sizeof(h), cudaMemcpyDeviceToHost));
  printf("multimem.ld_reduce.add on dev %d: %g (expect %g)\n", N - 1, h[0], (5.f + N) * N);
  ok = ok && h[0] == (5.f + N) * N;
  printf("RESULT multicast %s\n", ok ? "WORKS" : "MISMATCH");
  return 0;
}

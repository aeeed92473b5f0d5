// Memory primitives shared by the CPU executor and the sm_90a kernels.
//
// The parameter manager talks to peers through *memory semantics*: a peer's heap
// is mapped into this address space (POSIX shm on CPU, CUDA IPC / NVLink peer
// mapping on the GPU) and every protocol step is a load, store, or reduction on such
// a pointer. On the device all cross-rank accesses use system scope so that they
// are coherent over NVLink; on the host they are __atomic builtins.
#pragma once
#include "base.h"

#if !defined(__CUDA_ARCH__)
#include <sched.h>
#endif

namespace adapm {
namespace mem {

#if defined(__CUDA_ARCH__)
// ---------------------------------------------------------------- device (sm_90a)
ADAPM_D uint32_t ld_acquire(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
ADAPM_D void st_release(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// release store to memory of THIS GPU (device scope, see fence_local)
ADAPM_D void st_release_local(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
ADAPM_D void st_release(int32_t* p, int32_t v) {
  asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
ADAPM_D uint32_t ld_relaxed(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
ADAPM_D int32_t ld_relaxed(const int32_t* p) {
  int32_t v;
  asm volatile("ld.relaxed.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
ADAPM_D void st_relaxed(int32_t* p, int32_t v) {
  asm volatile("st.relaxed.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
ADAPM_D void st_relaxed(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
ADAPM_D uint8_t ld_relaxed(const uint8_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u8 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return (uint8_t)v;
}
ADAPM_D void st_relaxed(uint8_t* p, uint8_t v) {
  asm volatile("st.relaxed.sys.global.u8 [%0], %1;" ::"l"(p), "r"((uint32_t)v) : "memory");
}
ADAPM_D uint64_t ld_relaxed(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
ADAPM_D int64_t ld_relaxed(const int64_t* p) {
  int64_t v;
  asm volatile("ld.relaxed.sys.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
ADAPM_D void st_relaxed(uint64_t* p, uint64_t v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
ADAPM_D void st_relaxed(int64_t* p, int64_t v) {
  asm volatile("st.relaxed.sys.global.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
ADAPM_D float ld_relaxed(const float* p) {
  float v;
  asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}
ADAPM_D double ld_relaxed(const double* p) {
  double v;
  asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}
ADAPM_D void st_relaxed(float* p, float v) {
  asm volatile("st.relaxed.sys.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
ADAPM_D void st_relaxed(double* p, double v) {
  asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
ADAPM_D uint32_t fetch_add(uint32_t* p, uint32_t v) { return atomicAdd_system(p, v); }
ADAPM_D int32_t fetch_add(int32_t* p, int32_t v) { return atomicAdd_system(p, v); }
ADAPM_D uint64_t fetch_or(uint64_t* p, uint64_t v) {
  return (uint64_t)atomicOr_system((unsigned long long*)p, (unsigned long long)v);
}
ADAPM_D uint64_t fetch_and(uint64_t* p, uint64_t v) {
  return (uint64_t)atomicAnd_system((unsigned long long*)p, (unsigned long long)v);
}
ADAPM_D uint64_t exchange(uint64_t* p, uint64_t v) {
  return (uint64_t)atomicExch_system((unsigned long long*)p, (unsigned long long)v);
}
// fire-and-forget reductions (REDG; over NVLink for peer pointers)
ADAPM_D void red_add(float* p, float v) {
  asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
ADAPM_D void red_add(double* p, double v) {
  asm volatile("red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
ADAPM_D void red_add(int64_t* p, int64_t v) {
  asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
ADAPM_D void red_add(uint64_t* p, uint64_t v) {
  asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
ADAPM_D void red_add(uint32_t* p, uint32_t v) {
  asm volatile("red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// no-return bit operations (RED.OR / RED.AND over NVLink: nothing to wait for)
ADAPM_D void red_or(uint64_t* p, uint64_t v) {
  asm volatile("red.relaxed.sys.global.or.b64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
ADAPM_D void red_and(uint64_t* p, uint64_t v) {
  asm volatile("red.relaxed.sys.global.and.b64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// 16-byte row accesses (local HBM or an NVLink peer: same instructions)
struct alignas(16) F4 { float x, y, z, w; };
ADAPM_D F4 ld_relaxed4(const float* p) {
  float x, y, z, w;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(x), "=f"(y), "=f"(z), "=f"(w) : "l"(p) : "memory");
  F4 v; v.x = x; v.y = y; v.z = z; v.w = w;
  return v;
}
ADAPM_D void st_relaxed4(float* p, F4 v) {
  asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
ADAPM_D void red_add4(float* p, F4 v) {
  asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}
ADAPM_D void fence() { __threadfence_system(); }
// Orders this thread's accesses to memory of THIS GPU: device scope is enough even towards peers, which reach local
// memory through this GPU's L2 (the point of coherence). MEMBAR.SYS additionally waits for everything the thread has
// outstanding towards peers / the host - measured at tens of microseconds per fence next to a training kernel that
// keeps the SM's memory pipes full of NVLink reductions, i.e. unusable in a per-slot sequence.
ADAPM_D void fence_local() { __threadfence(); }
ADAPM_D void cpu_relax() { __nanosleep(64); }

#else
// ---------------------------------------------------------------- host
template <class T> inline T ld_acquire(const T* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
template <class T> inline void st_release(T* p, T v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
template <class T> inline void st_release_local(T* p, T v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
template <class T> inline T ld_relaxed(const T* p) { return __atomic_load_n(p, __ATOMIC_RELAXED); }
template <class T> inline void st_relaxed(T* p, T v) { __atomic_store_n(p, v, __ATOMIC_RELAXED); }
inline float ld_relaxed(const float* p) {
  uint32_t u = __atomic_load_n(reinterpret_cast<const uint32_t*>(p), __ATOMIC_RELAXED);
  float f; __builtin_memcpy(&f, &u, 4); return f;
}
inline double ld_relaxed(const double* p) {
  uint64_t u = __atomic_load_n(reinterpret_cast<const uint64_t*>(p), __ATOMIC_RELAXED);
  double f; __builtin_memcpy(&f, &u, 8); return f;
}
inline void st_relaxed(float* p, float v) {
  uint32_t u; __builtin_memcpy(&u, &v, 4);
  __atomic_store_n(reinterpret_cast<uint32_t*>(p), u, __ATOMIC_RELAXED);
}
inline void st_relaxed(double* p, double v) {
  uint64_t u; __builtin_memcpy(&u, &v, 8);
  __atomic_store_n(reinterpret_cast<uint64_t*>(p), u, __ATOMIC_RELAXED);
}
template <class T> inline T fetch_add(T* p, T v) { return __atomic_fetch_add(p, v, __ATOMIC_ACQ_REL); }
inline uint64_t fetch_or(uint64_t* p, uint64_t v) { return __atomic_fetch_or(p, v, __ATOMIC_ACQ_REL); }
inline uint64_t fetch_and(uint64_t* p, uint64_t v) { return __atomic_fetch_and(p, v, __ATOMIC_ACQ_REL); }
inline uint64_t exchange(uint64_t* p, uint64_t v) { return __atomic_exchange_n(p, v, __ATOMIC_ACQ_REL); }
inline void red_or(uint64_t* p, uint64_t v) { __atomic_fetch_or(p, v, __ATOMIC_ACQ_REL); }
inline void red_and(uint64_t* p, uint64_t v) { __atomic_fetch_and(p, v, __ATOMIC_ACQ_REL); }
inline void red_add(int64_t* p, int64_t v) { __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline void red_add(uint64_t* p, uint64_t v) { __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline void red_add(uint32_t* p, uint32_t v) { __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline void red_add(float* p, float v) {
  uint32_t* u = reinterpret_cast<uint32_t*>(p);
  uint32_t old = __atomic_load_n(u, __ATOMIC_RELAXED);
  for (;;) {
    float f; __builtin_memcpy(&f, &old, 4);
    f += v;
    uint32_t nu; __builtin_memcpy(&nu, &f, 4);
    if (__atomic_compare_exchange_n(u, &old, nu, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) return;
  }
}
inline void red_add(double* p, double v) {
  uint64_t* u = reinterpret_cast<uint64_t*>(p);
  uint64_t old = __atomic_load_n(u, __ATOMIC_RELAXED);
  for (;;) {
    double f; __builtin_memcpy(&f, &old, 8);
    f += v;
    uint64_t nu; __builtin_memcpy(&nu, &f, 8);
    if (__atomic_compare_exchange_n(u, &old, nu, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) return;
  }
}
inline void fence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
inline void fence_local() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
inline void cpu_relax() { sched_yield(); }
#endif

}  // namespace mem
}  // namespace adapm

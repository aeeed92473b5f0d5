// Device-side building blocks of the parameter manager that the generic kernels
// (cuda_backend.cu) and the fused application kernels (ops_*.cu) share.
#pragma once
#include <cuda_runtime.h>
#include "group.cuh"

namespace adapm {
namespace dev {

// 16-byte row accesses. Rows may live in a peer GPU's HBM (NVLink) - the same
// instructions work on both; `relaxed.sys` keeps them coherent with concurrent REDs.
__device__ __forceinline__ float4 ld_row4(const float* p) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
// weak 16-byte load through L1/L2 (local rows that are not re-read after a remote write in
// the same kernel)
__device__ __forceinline__ float4 ld_row4_weak(const float* p) {
  return __ldcg(reinterpret_cast<const float4*>(p));
}
// NVLS multicast stores (the address is the multicast alias of a heap offset: the switch replicates the store into
// every rank's heap)
__device__ __forceinline__ void multimem_st_u32(void* mc, uint32_t v) {
  asm volatile("multimem.st.relaxed.sys.global.u32 [%0], %1;" ::"l"(mc), "r"(v) : "memory");
}
__device__ __forceinline__ void multimem_st_release_u32(void* mc, uint32_t v) {
  asm volatile("multimem.st.release.sys.global.u32 [%0], %1;" ::"l"(mc), "r"(v) : "memory");
}
// in-switch reductions over the same heap offset of all ranks (multimem.ld_reduce -> SASS LDGMC)
__device__ __forceinline__ uint32_t multimem_ld_or_u32(const void* mc) {
  uint32_t v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.or.b32 %0, [%1];" : "=r"(v) : "l"(mc) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t multimem_ld_and_u32(const void* mc) {
  uint32_t v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.and.b32 %0, [%1];" : "=r"(v) : "l"(mc) : "memory");
  return v;
}
__device__ __forceinline__ void multimem_st_f32x4(float* mc, float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}
__device__ __forceinline__ void red_row4(float* p, float4 v) {
  asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w)
               : "memory");
}

// Grace-period registration (layout.h: SyncArea). Every CTA of a kernel that reads the directory / touches rows brackets
// its work with cta_enter / cta_exit: it is counted in active[epoch & 1] while it runs. The sync round flips the epoch
// after it announced new owners (phase B) and waits until the old side has drained: everything that may still act on
// the old directory is done before the relocation transfers start (phase C). One atomic pair per CTA; nothing on a
// single-rank store. All threads of the CTA must call both (they contain __syncthreads()).
__device__ __forceinline__ uint32_t& cta_epoch_ref() {
  __shared__ uint32_t cta_epoch_;
  return cta_epoch_;
}
// (out of line on purpose: the fused kernels sit exactly at their register budget)
static __device__ __noinline__ void cta_register(SyncArea* sa) {
  for (;;) {
    const uint32_t e = mem::ld_acquire(&sa->epoch);
    atomicAdd(&sa->active[e & 1u], 1u);
    __threadfence();
    if (mem::ld_acquire(&sa->epoch) == e) { cta_epoch_ref() = e; break; }
    atomicSub(&sa->active[e & 1u], 1u);   // the round flipped the epoch in between: register on the new side
  }
}
__device__ __forceinline__ void cta_deregister(SyncArea* sa) {
  __threadfence_system();   // this CTA's reductions (local or NVLink) are performed before it counts as gone
  atomicSub(&sa->active[cta_epoch_ref() & 1u], 1u);
}
__device__ __forceinline__ void cta_enter(const Ctx& c) {
  if (c.L.world == 1) return;
  if (threadIdx.x == 0 && threadIdx.y == 0 && threadIdx.z == 0) cta_register(sync_area_of(c, c.rank));
  __syncthreads();
}
__device__ __forceinline__ void cta_exit(const Ctx& c) {
  if (c.L.world == 1) return;
  __syncthreads();
  if (threadIdx.x == 0 && threadIdx.y == 0 && threadIdx.z == 0) cta_deregister(sync_area_of(c, c.rank));
}

// Warp-cooperative: where does `key` live for a read? Wraps protocol.h's locate_pull and
// returns raw pointers. All lanes get the same answer.
struct RowRef {
  const float* row;    // DIRECT: the row; SUM3: target row
  const float* base;   // SUM3 only
  const float* row2;   // SUM3 only
  const uint32_t* meta_ptr;
  uint32_t meta_val;
  int kind;            // LocKind
  bool local;
};

__device__ __forceinline__ RowRef locate_read(const Ctx& c, Key key) {
  WarpGroup g;
  PullLoc<float> l = locate_pull<float>(c, g, key, false);
  RowRef r;
  r.row = l.row; r.base = l.base; r.row2 = l.row2; r.meta_ptr = l.meta_ptr; r.meta_val = l.meta_val;
  r.kind = l.kind; r.local = l.local;
  return r;
}

// Fast local probe used by hot kernels: returns the row pointer if `key` is usable from local
// HBM (owned or valid replica), nullptr otherwise. One lane's worth of work (no shuffles).
__device__ __forceinline__ float* local_row_or_null(const Ctx& c, Key key, uint32_t* state_out, int32_t* slot_out) {
  int32_t s = __ldcg(slot_of(c, c.rank) + key);
  if (s < 0) return nullptr;
  uint32_t st = meta_state(mem::ld_acquire(meta_of(c, c.rank) + s));
  if (state_out) *state_out = st;
  if (slot_out) *slot_out = s;
  if (st == S_OWNED || st == S_REPLICA || st == S_INCOMING_REPLICA) return row_ptr<float>(c, c.rank, class_of_key(c, key), (uint32_t)s);
  return nullptr;
}

// A key resolved to a directly usable row. `row == nullptr` means the key is in a transitional
// protocol state and must go through the generic (out-of-line) path.
struct Target {
  float* row;
  uint32_t* version;  // owner version counter (may be remote) or nullptr
  uint8_t* flag;      // replica dirty byte or nullptr
};

// Single-lane fast path: local owned / local replica / local incoming-replica / remote owned.
__device__ __forceinline__ Target resolve_fast(const Ctx& c, Key key, int cls, unsigned* n_local, unsigned* n_remote) {
  Target t;
  t.row = nullptr; t.version = nullptr; t.flag = nullptr;
  const int me = c.rank;
  int32_t s = __ldcg(slot_of(c, me) + key);
  if (s >= 0) {
    uint32_t st = meta_state(__ldcg(meta_of(c, me) + s));
    if (st == S_OWNED || st == S_INCOMING_REPLICA) {
      t.row = row_ptr<float>(c, me, cls, (uint32_t)s); t.version = version_of(c, me) + s; ++*n_local;
      return t;
    }
    if (st == S_REPLICA) {
      t.row = row_ptr<float>(c, me, cls, (uint32_t)s); t.flag = dirty_of(c, me) + s; ++*n_local;
      return t;
    }
    if (st == S_INCOMING || st == S_FINALIZING) return t;  // needs the 3-way read: slow path
    // REPLICA_PENDING / OUTGOING / DEAD / DROPPING: not usable locally -> go to the owner
  }
  if (c.L.world == 1) return t;
  int o = (int)__ldcg(dir_of(c, me) + key);
  if (o == me) return t;
  int32_t ps = mem::ld_relaxed(slot_of(c, o) + key);  // NVLink load
  if (ps < 0) return t;
  uint32_t pst = meta_state(mem::ld_relaxed(meta_of(c, o) + ps));
  if (pst != S_OWNED) return t;
  t.row = row_ptr<float>(c, o, cls, (uint32_t)ps); t.version = version_of(c, o) + ps; ++*n_remote;
  return t;
}

// Rows for the gather threads of the GEMM kernels (one thread per row: ops_gather_gemm.cu, ops_topk.cu). `base` set: the
// key's relocation is in flight and its value is row - base + row2 (locate_pull's three-way read), valid while
// *meta_ptr still holds meta_val. row == nullptr: the key could not be resolved.
struct GatherRow {
  const float* row;
  const float* base;
  const float* row2;
  const uint32_t* meta_ptr;
  uint32_t meta_val;
  bool local;
};

// For keys that resolve_fast leaves open: protocol.h's locate_pull with a one-lane group follows a relocation source to
// the new owner, reads an INCOMING slot three ways and waits out FINALIZING - none of which needs the sync round to
// progress, so a CTA that the round's grace period waits for cannot wait for the round.
static __device__ __noinline__ GatherRow gather_locate(const Ctx& c, Key key) {
  LaneGroup g;
  const PullLoc<float> l = locate_pull<float>(c, g, key, false);
  GatherRow r;
  r.row = l.kind == LOC_FAIL ? nullptr : l.row;
  r.base = l.kind == LOC_SUM3 ? l.base : nullptr;
  r.row2 = l.row2; r.meta_ptr = l.meta_ptr; r.meta_val = l.meta_val; r.local = l.local;
  return r;
}

__device__ __forceinline__ float4 ld_gather4(const GatherRow& r, int k) {
  float4 v = ld_row4(r.row + k);
  if (r.base) {
    const float4 b = ld_row4(r.base + k), s = ld_row4(r.row2 + k);
    v.x = v.x - b.x + s.x; v.y = v.y - b.y + s.y; v.z = v.z - b.z + s.z; v.w = v.w - b.w + s.w;
  }
  return v;
}

// After a three-way read: did the transfer complete in between (the values read may mix both sides)? Then re-locate.
__device__ __forceinline__ bool gather_reread(const Ctx& c, Key key, GatherRow& r) {
  if (!r.base) return false;
  mem::fence();
  if (mem::ld_acquire(r.meta_ptr) == r.meta_val) return false;
  r = gather_locate(c, key);
  return true;
}

// lane 0 marks a completed fast-path push
__device__ __forceinline__ void mark_pushed(const Target& t) {
  if (t.version) mem::red_add(t.version, 1u);
  if (t.flag) *t.flag = (uint8_t)1;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// End of a fused step's kernel, all lanes of the warp: stats[0..3] += (local rows, peer rows, slow-path rows, pushes).
// The resolve counts are per lane and summed over the warp; n_slow and n_upd are warp-uniform and lane 0's are added.
__device__ __forceinline__ void flush_stats(unsigned long long* stats, unsigned n_local, unsigned n_remote,
                                            unsigned n_slow, unsigned n_upd) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    n_local += __shfl_xor_sync(0xffffffffu, n_local, o);
    n_remote += __shfl_xor_sync(0xffffffffu, n_remote, o);
  }
  if ((threadIdx.x & 31) == 0 && stats) {
    if (n_local) atomicAdd(stats + 0, (unsigned long long)n_local);
    if (n_remote) atomicAdd(stats + 1, (unsigned long long)n_remote);
    if (n_slow) atomicAdd(stats + 2, (unsigned long long)n_slow);
    if (n_upd) atomicAdd(stats + 3, (unsigned long long)n_upd);
  }
}

// generic out-of-line fallbacks (warp-cooperative)
static __device__ __noinline__ bool slow_pull(const Ctx& c, Key key, float* stage) {
  WarpGroup g;
  bool ok = pull_key<float>(c, g, key, stage, false, nullptr);
  __syncwarp();
  return ok;
}
static __device__ __noinline__ bool slow_push(const Ctx& c, Key key, const float* stage) {
  WarpGroup g;
  __syncwarp();
  bool ok = push_key<float>(c, g, key, stage, nullptr);
  __syncwarp();
  return ok;
}

}  // namespace dev
}  // namespace adapm

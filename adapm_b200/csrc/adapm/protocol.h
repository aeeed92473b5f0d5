// The parameter-management protocol, written once for host and device.
//
// Every function here is a per-key / per-slot step executed by a "group" of lanes:
// one CPU thread (HostGroup) or one 32-wide warp (WarpGroup, see cuda/group.cuh).
// The CPU executor and the sm_90a kernels both instantiate this file, so the CPU
// contract tests exercise the exact state machine that runs on the GPU.
//
// What it replaces in the reference (studied, not copied):
//   worker fast path       coloc_kv_worker.h:120-318, coloc_kv_server_handle.h:346-478
//   intent registration    coloc_kv_server_handle.h:484-532, sync_manager.h:257-286
//   replica delta / drop   coloc_kv_server_handle.h:601-662         (phase A)
//   relocate-vs-replicate  sync_manager.h:553-739                   (phase B)
//   refresh / upgrade      coloc_kv_server_handle.h:776-840         (phase C)
// Instead of SYNC / SYNC_FORWARD / response messages, a sync round is three passes
// over the slots separated by barriers; all cross-rank traffic is peer loads,
// stores and reductions. Relocation is made exact without locks by a grace period
// (all worker kernels that may have read the old directory have drained) between
// the ownership announcement (phase B) and the transfer (phase C).
#pragma once
#include "layout.h"

namespace adapm {

struct HostGroup {
  ADAPM_HD int lane() const { return 0; }
  ADAPM_HD int size() const { return 1; }
  ADAPM_HD bool any(bool p) const { return p; }
  ADAPM_HD void sync() const {}
  ADAPM_HD uint32_t bcast(uint32_t v) const { return v; }
  ADAPM_HD int32_t bcast(int32_t v) const { return v; }
  ADAPM_HD uint64_t bcast(uint64_t v) const { return v; }
  ADAPM_HD uint32_t bcast_from(uint32_t v, int) const { return v; }
  ADAPM_HD double sum(double v) const { return v; }
};

constexpr int kMaxAttempts = 1 << 16;

enum LocKind : int { LOC_FAIL = 0, LOC_DIRECT = 1, LOC_SUM3 = 2 };

template <class Val> struct PullLoc {
  int kind;
  bool local;               // served from this rank's memory only
  const Val* row;           // DIRECT: the row; SUM3: target row
  const Val* base;          // SUM3: target base
  const Val* row2;          // SUM3: source (old owner) row
  const uint32_t* meta_ptr; // SUM3: seqlock word to re-validate
  uint32_t meta_val;
};

template <class Val> struct PushLoc {
  Val* row;          // nullptr on failure
  uint32_t* version; // owner version counter to bump (nullptr for replica pushes)
  uint8_t* flag;     // replica dirty flag (nullptr otherwise)
  bool local;
  int owner;
};

// ---------------------------------------------------------------------------------------
// locate: where does a Pull of `key` read from?   (all lanes compute the same result)
template <class Val, class G>
ADAPM_HD PullLoc<Val> locate_pull(const Ctx& c, const G& g, Key key, bool local_only) {
  PullLoc<Val> r;
  r.kind = LOC_FAIL; r.local = false; r.row = nullptr; r.base = nullptr; r.row2 = nullptr;
  r.meta_ptr = nullptr; r.meta_val = 0;
  const int me = c.rank;
  const int cls = class_of_key(c, key);
  for (int attempt = 0; attempt < kMaxAttempts; ++attempt) {
    int32_t s = g.bcast(g.lane() == 0 ? mem::ld_relaxed(slot_of(c, me) + key) : 0);
    if (s >= 0) {
      uint32_t m = g.bcast(g.lane() == 0 ? mem::ld_acquire(meta_of(c, me) + s) : 0u);
      uint32_t st = meta_state(m);
      if (st == S_OWNED || st == S_REPLICA || st == S_INCOMING_REPLICA) {
        // INCOMING_REPLICA: the slot was a usable replica when the owner handed the key over;
        // until the transfer is finalized it keeps serving local reads with replica semantics
        r.kind = LOC_DIRECT; r.local = true; r.row = row_ptr<Val>(c, me, cls, s);
        return r;
      }
      if (st == S_INCOMING && !local_only) {
        int src = (int)meta_peer(m);
        // while INCOMING, ver_seen holds the source's slot id (written by the old owner in phase B)
        int32_t ss = (int32_t)g.bcast(g.lane() == 0 ? mem::ld_relaxed(ver_seen_of(c, me) + s) : 0u);
        if (ss >= 0) {
          r.kind = LOC_SUM3; r.local = false;
          r.row = row_ptr<Val>(c, me, cls, s); r.base = base_ptr<Val>(c, me, cls, s);
          r.row2 = row_ptr<Val>(c, src, cls, ss);
          r.meta_ptr = meta_of(c, me) + s; r.meta_val = m;
          return r;
        }
      }
      if (st == S_FINALIZING && !local_only) { mem::cpu_relax(); continue; }
      // REPLICA_PENDING / OUTGOING / DEAD / DROPPING: not usable locally
    }
    if (local_only) return r;
    int o = (int)g.bcast((uint32_t)(g.lane() == 0 ? mem::ld_relaxed(dir_of(c, me) + key) : 0));
    if (o == me) { mem::cpu_relax(); continue; }  // directory in flux
    bool retry = false;
    for (int hop = 0; hop < 4; ++hop) {
      int32_t ps = g.bcast(g.lane() == 0 ? mem::ld_relaxed(slot_of(c, o) + key) : 0);
      if (ps < 0) { retry = true; break; }
      uint32_t pm = g.bcast(g.lane() == 0 ? mem::ld_acquire(meta_of(c, o) + ps) : 0u);
      uint32_t pst = meta_state(pm);
      if (pst == S_OWNED) {
        r.kind = LOC_DIRECT; r.local = false; r.row = row_ptr<Val>(c, o, cls, ps);
        return r;
      }
      if (state_is_incoming(pst)) {
        int src = (int)meta_peer(pm);
        int32_t ss = (int32_t)g.bcast(g.lane() == 0 ? mem::ld_relaxed(ver_seen_of(c, o) + ps) : 0u);
        if (ss < 0) { retry = true; break; }
        r.kind = LOC_SUM3; r.local = false;
        r.row = row_ptr<Val>(c, o, cls, ps); r.base = base_ptr<Val>(c, o, cls, ps);
        r.row2 = row_ptr<Val>(c, src, cls, ss);
        r.meta_ptr = meta_of(c, o) + ps; r.meta_val = pm;
        return r;
      }
      if (pst == S_OUTGOING || pst == S_DEAD) { o = (int)meta_peer(pm); if (o == me) { retry = true; break; } continue; }
      retry = true; break;  // FINALIZING or a stale directory entry
    }
    if (retry) { mem::cpu_relax(); continue; }
  }
  return r;
}

// Row loops run in batches: all loads of a batch are issued before their first use, so that a warp keeps kRowBatch
// independent (possibly NVLink) loads in flight. Written element-by-element they serialise on one dependent round
// trip per element (system-scope loads are not reordered): 19 round trips for a 600-float row.
constexpr int kRowBatch = 8;
#if defined(__CUDA_ARCH__)
#define ADAPM_UNROLL _Pragma("unroll")
#else
#define ADAPM_UNROLL
#endif
#define ADAPM_ROW_BATCHES(g, len) for (uint32_t i0_ = (g).lane(); i0_ < (len); i0_ += (g).size() * kRowBatch)
#define ADAPM_ROW_ELEMS(g, len, u, i) \
  ADAPM_UNROLL for (int u = 0; u < kRowBatch; ++u) \
    for (uint32_t i = i0_ + (uint32_t)u * (g).size(); i < (len); i = 0xffffffffu)

// ---------------------------------------------------------------------------------------
// Row primitives of the sync round: the only loops over row elements. On the device, float rows whose length is a
// multiple of 4 take the 16-byte path (LDG.128 / REDG.F32x4 / STG.128, local HBM or an NVLink peer alike) with
// kVecBatch independent 16-byte accesses per lane in flight: a 600-float word2vec row is ONE batch per array, i.e. one
// NVLink round trip instead of the 19 dependent ones of an element-wise loop.
#ifndef ADAPM_VEC_BATCH
#define ADAPM_VEC_BATCH 5
#endif
constexpr int kVecBatch = ADAPM_VEC_BATCH;
// (out of line on the device: the primitives are called from several branches of the slot functions; inlined, their
// batches of 16-byte registers pushed the round kernels into spills)
#if defined(__CUDA_ARCH__) && !defined(ADAPM_ROW_INLINE)
#define ADAPM_ROWFN __device__ __noinline__
#elif defined(__CUDA_ARCH__)
#define ADAPM_ROWFN __device__ __forceinline__
#else
#define ADAPM_ROWFN inline
#endif
#if defined(__CUDA_ARCH__)
template <class Val> ADAPM_D bool row_vec_ok(uint32_t, const void*, const void*, const void*) { return false; }
template <> ADAPM_D bool row_vec_ok<float>(uint32_t len, const void* a, const void* b, const void* c) {
#ifdef ADAPM_NO_VEC   // debugging: element-wise loops only
  return false;
#endif
  return (len & 3u) == 0 && ((((uintptr_t)a) | ((uintptr_t)b) | ((uintptr_t)c)) & 15u) == 0;
}
#define ADAPM_VEC_BATCHES(g, nv) for (uint32_t j0_ = (g).lane(); j0_ < (nv); j0_ += (g).size() * kVecBatch)
#define ADAPM_VEC_ELEMS(g, nv, u, j) \
  _Pragma("unroll") for (int u = 0; u < kVecBatch; ++u) \
    if (const uint32_t j = j0_ + (uint32_t)u * 32u; j < (nv))
ADAPM_D bool f4_ne(const mem::F4& a, const mem::F4& b) { return a.x != b.x || a.y != b.y || a.z != b.z || a.w != b.w; }
ADAPM_D mem::F4 f4_sub(const mem::F4& a, const mem::F4& b) { mem::F4 r; r.x = a.x - b.x; r.y = a.y - b.y; r.z = a.z - b.z; r.w = a.w - b.w; return r; }
#endif

// dst += (src - ref) where they differ; ref := (rebase ? src : 0).  Used by the refresh (dst = replica row,
// ref = replica base, src = owner row or its published mirror) and by the relocation finalize (rebase = false).
// Returns (via *ref_nonzero) whether any ref element was non-zero.
template <class Val, class G>
ADAPM_ROWFN void row_fold(const G& g, Val* dst, Val* ref, const Val* src, uint32_t len, bool rebase, bool* ref_nonzero) {
  bool bnz = false;
#if defined(__CUDA_ARCH__)
  if (row_vec_ok<Val>(len, dst, ref, src)) {
    float* d = reinterpret_cast<float*>(dst); float* r = reinterpret_cast<float*>(ref);
    const float* s = reinterpret_cast<const float*>(src);
    const uint32_t nv = len >> 2;
    ADAPM_VEC_BATCHES(g, nv) {
      mem::F4 S[kVecBatch], b[kVecBatch];
      ADAPM_VEC_ELEMS(g, nv, u, j) S[u] = mem::ld_relaxed4(s + 4 * j);
      ADAPM_VEC_ELEMS(g, nv, u, j) b[u] = mem::ld_relaxed4(r + 4 * j);
      ADAPM_VEC_ELEMS(g, nv, u, j) {
        const mem::F4 z = {0.f, 0.f, 0.f, 0.f};
        bnz = bnz || f4_ne(b[u], z);
        if (f4_ne(S[u], b[u])) {
          mem::red_add4(d + 4 * j, f4_sub(S[u], b[u]));
          if (rebase) mem::st_relaxed4(r + 4 * j, S[u]);
        }
        if (!rebase && f4_ne(b[u], z)) mem::st_relaxed4(r + 4 * j, z);
      }
    }
    if (ref_nonzero) *ref_nonzero = g.any(bnz);
    return;
  }
#endif
  ADAPM_ROW_BATCHES(g, len) {
    Val S[kRowBatch], b[kRowBatch];
    ADAPM_ROW_ELEMS(g, len, u, i) S[u] = mem::ld_relaxed(src + i);
    ADAPM_ROW_ELEMS(g, len, u, i) b[u] = mem::ld_relaxed(ref + i);
    ADAPM_ROW_ELEMS(g, len, u, i) {
      bnz = bnz || b[u] != (Val)0;
      if (S[u] != b[u]) {
        mem::red_add(dst + i, (Val)(S[u] - b[u]));
        if (rebase) mem::st_relaxed(ref + i, S[u]);
      }
      if (!rebase && b[u] != (Val)0) mem::st_relaxed(ref + i, (Val)0);
    }
  }
  if (ref_nonzero) *ref_nonzero = g.any(bnz);
}

// out += (row - base) where they differ (reductions into the owner's row); base := row if `rebase`.
// Returns true if any element differed. (`all`: sys.sync.threshold < 0 - nothing changes for equal elements.)
template <class Val, class G>
ADAPM_ROWFN bool row_ship(const G& g, const Val* row, Val* base, Val* out, uint32_t len, bool rebase) {
  bool nz = false;
#if defined(__CUDA_ARCH__)
  if (row_vec_ok<Val>(len, row, base, out)) {
    const float* w = reinterpret_cast<const float*>(row); float* r = reinterpret_cast<float*>(base);
    float* o = reinterpret_cast<float*>(out);
    const uint32_t nv = len >> 2;
    ADAPM_VEC_BATCHES(g, nv) {
      mem::F4 v[kVecBatch], b[kVecBatch];
      ADAPM_VEC_ELEMS(g, nv, u, j) v[u] = mem::ld_relaxed4(w + 4 * j);
      ADAPM_VEC_ELEMS(g, nv, u, j) b[u] = mem::ld_relaxed4(r + 4 * j);
      ADAPM_VEC_ELEMS(g, nv, u, j) {
        if (f4_ne(v[u], b[u])) {
          mem::red_add4(o + 4 * j, f4_sub(v[u], b[u]));
          if (rebase) mem::st_relaxed4(r + 4 * j, v[u]);
          nz = true;
        }
      }
    }
    return g.any(nz);
  }
#endif
  ADAPM_ROW_BATCHES(g, len) {
    Val v[kRowBatch], b[kRowBatch];
    ADAPM_ROW_ELEMS(g, len, u, i) v[u] = mem::ld_relaxed(row + i);
    ADAPM_ROW_ELEMS(g, len, u, i) b[u] = mem::ld_relaxed(base + i);
    ADAPM_ROW_ELEMS(g, len, u, i) {
      const Val d = v[u] - b[u];
      if (d != (Val)0) {
        mem::red_add(out + i, d);
        if (rebase) mem::st_relaxed(base + i, v[u]);
        nz = true;
      }
    }
  }
  return g.any(nz);
}

// sum over (row - base)^2   (sys.sync.threshold > 0: ship a replica delta only if its L2 norm is large enough)
template <class Val, class G>
ADAPM_ROWFN double row_delta_norm2(const G& g, const Val* row, const Val* base, uint32_t len) {
  double acc = 0;
#if defined(__CUDA_ARCH__)
  if (row_vec_ok<Val>(len, row, base, row)) {
    const float* w = reinterpret_cast<const float*>(row); const float* r = reinterpret_cast<const float*>(base);
    const uint32_t nv = len >> 2;
    float a = 0.f;
    ADAPM_VEC_BATCHES(g, nv) {
      mem::F4 v[kVecBatch], b[kVecBatch];
      ADAPM_VEC_ELEMS(g, nv, u, j) v[u] = mem::ld_relaxed4(w + 4 * j);
      ADAPM_VEC_ELEMS(g, nv, u, j) b[u] = mem::ld_relaxed4(r + 4 * j);
      ADAPM_VEC_ELEMS(g, nv, u, j) {
        const mem::F4 d = f4_sub(v[u], b[u]);
        a += d.x * d.x + d.y * d.y + d.z * d.z + d.w * d.w;
      }
    }
    return g.sum((double)a);
  }
#endif
  ADAPM_ROW_BATCHES(g, len) {
    Val v[kRowBatch];
    ADAPM_ROW_ELEMS(g, len, u, i) v[u] = mem::ld_relaxed(row + i);
    ADAPM_ROW_ELEMS(g, len, u, i) v[u] -= mem::ld_relaxed(base + i);
    ADAPM_ROW_ELEMS(g, len, u, i) acc += (double)v[u] * (double)v[u];
  }
  return g.sum(acc);
}

// row := 0, base := 0   (a slot goes back to the pool with all-zero rows: register_intent relies on it)
template <class Val, class G>
ADAPM_ROWFN void row_clear(const G& g, Val* row, Val* base, uint32_t len) {
#if defined(__CUDA_ARCH__)
  if (row_vec_ok<Val>(len, row, base, row)) {
    const mem::F4 z = {0.f, 0.f, 0.f, 0.f};
    for (uint32_t j = g.lane(); j < (len >> 2); j += g.size()) {
      mem::st_relaxed4(reinterpret_cast<float*>(row) + 4 * j, z);
      mem::st_relaxed4(reinterpret_cast<float*>(base) + 4 * j, z);
    }
    return;
  }
#endif
  for (uint32_t i = g.lane(); i < len; i += g.size()) {
    mem::st_relaxed(row + i, (Val)0);
    mem::st_relaxed(base + i, (Val)0);
  }
}

// dst := src  (len values; owner row -> published mirror row)
template <class Val, class G>
ADAPM_ROWFN void row_copy(const G& g, Val* dst, const Val* src, uint32_t len) {
#if defined(__CUDA_ARCH__)
  if (row_vec_ok<Val>(len, dst, src, src)) {
    float* d = reinterpret_cast<float*>(dst); const float* s = reinterpret_cast<const float*>(src);
    const uint32_t nv = len >> 2;
    ADAPM_VEC_BATCHES(g, nv) {
      mem::F4 v[kVecBatch];
      ADAPM_VEC_ELEMS(g, nv, u, j) v[u] = mem::ld_relaxed4(s + 4 * j);
      ADAPM_VEC_ELEMS(g, nv, u, j) mem::st_relaxed4(d + 4 * j, v[u]);
    }
    return;
  }
#endif
  for (uint32_t i = g.lane(); i < len; i += g.size()) mem::st_relaxed(dst + i, mem::ld_relaxed(src + i));
}

// Copy the located row into `out` (len values). Returns false if a SUM3 read raced with the
// finalize step and must be retried by the caller.
template <class Val, class G>
ADAPM_HD bool read_row(const G& g, const PullLoc<Val>& loc, Val* out, uint32_t len) {
  if (loc.kind == LOC_DIRECT) {
    // (element-wise on purpose: read_row / push_key are inlined into the out-of-line paths of the fused training
    // kernels, whose register budget must not grow; the batched form is for the round kernels)
    for (uint32_t i = g.lane(); i < len; i += g.size()) out[i] = mem::ld_relaxed(loc.row + i);
    return true;
  }
  for (uint32_t i = g.lane(); i < len; i += g.size())
    out[i] = mem::ld_relaxed(loc.row + i) - mem::ld_relaxed(loc.base + i) + mem::ld_relaxed(loc.row2 + i);
  mem::fence();
  uint32_t m2 = g.bcast(g.lane() == 0 ? mem::ld_acquire(loc.meta_ptr) : 0u);
  return m2 == loc.meta_val;
}

template <class Val, class G>
ADAPM_HD bool pull_key(const Ctx& c, const G& g, Key key, Val* out, bool local_only, bool* was_local) {
  const uint32_t len = key_len(c, key, class_of_key(c, key));
  for (int attempt = 0; attempt < kMaxAttempts; ++attempt) {
    PullLoc<Val> loc = locate_pull<Val>(c, g, key, local_only);
    if (loc.kind == LOC_FAIL) return false;
    if (read_row(g, loc, out, len)) {
      if (was_local) *was_local = loc.local;
      if (c.L.off_access && g.lane() == 0) {  // per-key locality statistics (PS_LOCALITY_STATS equivalent)
        uint32_t* acc = at<uint32_t>(c, c.rank, c.L.off_access) + 2 * (size_t)key;
        mem::red_add(acc, 1u);
        if (loc.local) mem::red_add(acc + 1, 1u);
      }
      return true;
    }
    mem::cpu_relax();
  }
  return false;
}

// ---------------------------------------------------------------------------------------
// locate: where does a Push (additive) of `key` go?
template <class Val, class G>
ADAPM_HD PushLoc<Val> locate_push(const Ctx& c, const G& g, Key key) {
  PushLoc<Val> r;
  r.row = nullptr; r.version = nullptr; r.flag = nullptr; r.local = false; r.owner = -1;
  const int me = c.rank;
  const int cls = class_of_key(c, key);
  for (int attempt = 0; attempt < kMaxAttempts; ++attempt) {
    int32_t s = g.bcast(g.lane() == 0 ? mem::ld_relaxed(slot_of(c, me) + key) : 0);
    if (s >= 0) {
      uint32_t st = meta_state(g.bcast(g.lane() == 0 ? mem::ld_acquire(meta_of(c, me) + s) : 0u));
      if (st == S_OWNED || state_is_incoming(st) || st == S_FINALIZING) {
        r.row = row_ptr<Val>(c, me, cls, s); r.version = version_of(c, me) + s;
        r.local = true; r.owner = me;
        return r;
      }
      if (st == S_REPLICA) {
        r.row = row_ptr<Val>(c, me, cls, s); r.flag = dirty_of(c, me) + s;
        r.local = true; r.owner = -1;
        return r;
      }
    }
    int o = (int)g.bcast((uint32_t)(g.lane() == 0 ? mem::ld_relaxed(dir_of(c, me) + key) : 0));
    if (o == me) { mem::cpu_relax(); continue; }
    int32_t ps = g.bcast(g.lane() == 0 ? mem::ld_relaxed(slot_of(c, o) + key) : 0);
    if (ps < 0) { mem::cpu_relax(); continue; }
    uint32_t pst = meta_state(g.bcast(g.lane() == 0 ? mem::ld_acquire(meta_of(c, o) + ps) : 0u));
    // OWNED / INCOMING / FINALIZING accept adds; OUTGOING still accepts adds until the grace
    // period of the announcing round has passed (we are inside it, or we would see the new dir).
    // REPLICA / REPLICA_PENDING with dir == o happens for a moment when the directory store
    // overtakes the INCOMING store: the row is the accumulator of the incoming owner -> valid.
    if (pst == S_FREE || pst == S_DEAD || pst == S_DROPPING) { mem::cpu_relax(); continue; }
    r.row = row_ptr<Val>(c, o, cls, ps); r.version = version_of(c, o) + ps;
    r.local = false; r.owner = o;
    return r;
  }
  return r;
}

template <class Val, class G>
ADAPM_HD bool push_key(const Ctx& c, const G& g, Key key, const Val* vals, bool* was_local) {
  const uint32_t len = key_len(c, key, class_of_key(c, key));
  PushLoc<Val> loc = locate_push<Val>(c, g, key);
  if (!loc.row) return false;
  for (uint32_t i = g.lane(); i < len; i += g.size()) mem::red_add(loc.row + i, vals[i]);
  if (g.lane() == 0) {
    if (loc.version) mem::red_add(loc.version, 1u);
    if (loc.flag) mem::st_relaxed(loc.flag, (uint8_t)1);
  }
  if (was_local) *was_local = loc.local;
  return true;
}

// Set (assignment) goes to the owner's row. Mirrors the reference's `set` flag of Push
// (coloc_kv_worker.h:223-239, coloc_kv_server_handle.h:404-415); on a replica the reference
// only asserts, we route the store to the owner and re-base the local replica.
// A key whose relocation is in flight cannot be assigned exactly (its value is spread over two rows until phase C
// folds them). The op must NOT wait for that inside a grace-tracked kernel / op - the grace period waits for the op -
// so set_key reports SET_RETRY and the caller (Worker::Push) repeats the key after the next sync round.
enum SetResult : int { SET_FAIL = 0, SET_OK = 1, SET_RETRY = 2 };
template <class Val, class G>
ADAPM_HD int set_key(const Ctx& c, const G& g, Key key, const Val* vals, bool* was_local) {
  const int me = c.rank;
  const int cls = class_of_key(c, key);
  const uint32_t len = key_len(c, key, cls);
  for (int attempt = 0; attempt < 256; ++attempt) {
    int32_t s = g.bcast(g.lane() == 0 ? mem::ld_relaxed(slot_of(c, me) + key) : 0);
    uint32_t st = S_FREE;
    if (s >= 0) st = meta_state(g.bcast(g.lane() == 0 ? mem::ld_acquire(meta_of(c, me) + s) : 0u));
    if (st == S_OWNED) {
      Val* row = row_ptr<Val>(c, me, cls, s);
      for (uint32_t i = g.lane(); i < len; i += g.size()) mem::st_relaxed(row + i, vals[i]);
      if (g.lane() == 0) mem::red_add(version_of(c, me) + s, 1u);
      if (was_local) *was_local = true;
      return SET_OK;
    }
    if (state_is_incoming(st) || st == S_FINALIZING) return SET_RETRY;   // transfer in flight: after the next round
    int o = (int)g.bcast((uint32_t)(g.lane() == 0 ? mem::ld_relaxed(dir_of(c, me) + key) : 0));
    if (o == me) { mem::cpu_relax(); continue; }   // directory store and state word are a few stores apart
    int32_t ps = g.bcast(g.lane() == 0 ? mem::ld_relaxed(slot_of(c, o) + key) : 0);
    if (ps < 0) { mem::cpu_relax(); continue; }
    uint32_t pst = meta_state(g.bcast(g.lane() == 0 ? mem::ld_acquire(meta_of(c, o) + ps) : 0u));
    if (pst != S_OWNED) return SET_RETRY;
    Val* row = row_ptr<Val>(c, o, cls, ps);
    for (uint32_t i = g.lane(); i < len; i += g.size()) mem::st_relaxed(row + i, vals[i]);
    if (g.lane() == 0) mem::red_add(version_of(c, o) + ps, 1u);
    if (st == S_REPLICA) {  // keep the local replica coherent with the assignment
      Val* lrow = row_ptr<Val>(c, me, cls, s);
      Val* lbase = base_ptr<Val>(c, me, cls, s);
      for (uint32_t i = g.lane(); i < len; i += g.size()) {
        mem::st_relaxed(lrow + i, vals[i]);
        mem::st_relaxed(lbase + i, vals[i]);
      }
    }
    if (was_local) *was_local = false;
    return SET_OK;
  }
  return SET_RETRY;
}

// ---------------------------------------------------------------------------------------
// helpers for the sync round
ADAPM_HD bool intent_active(const Ctx& c, uint32_t s, const Clock* clocks) {
  const int64_t* ie = intent_end_of(c, c.rank) + (size_t)s * c.L.workers;
  for (int w = 0; w < c.L.workers; ++w)
    if (mem::ld_relaxed(ie + w) > clocks[w]) return true;
  return false;
}

ADAPM_HD void atomic_max_i64(int64_t* p, int64_t v) {
#if defined(__CUDA_ARCH__)
  atomicMax((long long*)p, (long long)v);
#else
  int64_t old = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (old < v && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
#endif
}
ADAPM_HD int32_t cas_i32(int32_t* p, int32_t expect, int32_t desired) {
#if defined(__CUDA_ARCH__)
  return atomicCAS_system(p, expect, desired);
#else
  __atomic_compare_exchange_n(p, &expect, desired, false, __ATOMIC_ACQ_REL, __ATOMIC_ACQUIRE);
  return expect;
#endif
}

ADAPM_HD int32_t alloc_slot(const Ctx& c, int cls) {
  int32_t* top = free_top_of(c, c.rank) + cls;
  int32_t idx = mem::fetch_add(top, (int32_t)-1) - 1;
  if (idx < 0) { mem::fetch_add(top, (int32_t)1); return -1; }
  const int32_t* stack = at<int32_t>(c, c.rank, c.L.cls[cls].free_off);
  return mem::ld_relaxed(stack + idx);
}
ADAPM_HD void free_slot(const Ctx& c, int cls, int32_t slot) {
  int32_t* top = free_top_of(c, c.rank) + cls;
  int32_t idx = mem::fetch_add(top, (int32_t)1);
  int32_t* stack = at<int32_t>(c, c.rank, c.L.cls[cls].free_off);
  mem::st_relaxed(stack + idx, slot);
}

// Register one intent record (phase A, step 1). Executed by ONE lane.
// Returns 0 = registered, 1 = deferred to the next round, 2 = dropped (expired / no memory).
template <class Val>
ADAPM_HD int register_intent(const Ctx& c, const IntentRec& rec, const Clock* clocks) {
  const int me = c.rank;
  const Key key = rec.key;
  if (rec.end <= clocks[rec.worker]) return 2;  // already expired
  int32_t s = mem::ld_relaxed(slot_of(c, me) + key);
  bool claimed = false;
  if (s >= 0) {
    // a relocation source slot (OUTGOING/DEAD) no longer represents the key on this rank:
    // the key gets a fresh placeholder, the old row stays readable until it is recycled
    uint32_t st0 = meta_state(mem::ld_acquire(meta_of(c, me) + s));
    if (st0 == S_OUTGOING || st0 == S_DEAD) {
      int32_t prev = cas_i32(slot_of(c, me) + key, s, -2);
      if (prev != s) return 1;
      claimed = true;
      s = -1;
    }
  }
  if (s == -1) {
    // claim the key so that concurrent records for the same key do not allocate twice
    if (!claimed) {
      int32_t prev = cas_i32(slot_of(c, me) + key, -1, -2);
      if (prev != -1) return 1;
    }
    const int cls = class_of_key(c, key);
    int32_t ns = alloc_slot(c, cls);
    if (ns < 0) {
      // pool exhausted: give the claim back and retry in a later round (slots free up as replicas expire)
      mem::st_relaxed(slot_of(c, me) + key, (int32_t)-1);
      count(c, C_ALLOC_FAIL);
      return 1;
    }
    // row and base of a free slot are all-zero: the heap starts zeroed and phase C clears a slot before it returns
    // it to the pool (warp-cooperative, coalesced) - a single lane zeroing 2 x len values here was the most
    // expensive part of the round
    int64_t* ie = intent_end_of(c, me) + (size_t)ns * c.L.workers;
    for (int w = 0; w < c.L.workers; ++w) mem::st_relaxed(ie + w, (int64_t)0);
    mem::st_relaxed(ie + rec.worker, rec.end);
    mem::st_relaxed(slot_key_of(c, me) + ns, (int64_t)key);
    mem::st_relaxed(version_of(c, me) + ns, 0u);
    mem::st_relaxed(ver_seen_of(c, me) + ns, 0xffffffffu);
    mem::st_relaxed(want_of(c, me) + ns, (uint64_t)0);
    mem::st_relaxed(flags_of(c, me) + ns, (uint8_t)0);
    mem::st_relaxed(dirty_of(c, me) + ns, (uint8_t)0);
    mem::st_relaxed(want_owner_of(c, me) + ns, (uint8_t)0xff);
    uint32_t m = mem::ld_relaxed(meta_of(c, me) + ns);
    mem::fence();
    mem::st_release(meta_of(c, me) + ns, meta_next(m, S_REPLICA_PENDING, 0));
    mem::st_release(slot_of(c, me) + key, ns);
    return 0;
  }
  if (s < 0) return 1;  // being allocated by a concurrent record
  uint32_t st = meta_state(mem::ld_acquire(meta_of(c, me) + s));
  if (st == S_OWNED || st == S_REPLICA || st == S_REPLICA_PENDING || state_is_incoming(st)) {
    atomic_max_i64(intent_end_of(c, me) + (size_t)s * c.L.workers + rec.worker, rec.end);
    return 0;
  }
  return 1;  // OUTGOING / DEAD / DROPPING / FINALIZING: retry after the slot is recycled
}

struct RoundParams {
  Clock clocks[MAX_LOCAL_WORKERS];
  double threshold;     // sys.sync.threshold: -1 all, 0 non-zero, >0 L2 norm, inf = never
  int32_t sweep;        // full sweep: ignore dirty hints / versions for every slot (WaitSync: guaranteed propagation)
  uint32_t round_no;    // same on every rank (rounds run in lock-step)
  int32_t sweep_period; // rolling sweep: slot s is swept in the rounds with (s + round_no) % sweep_period == 0
  int32_t idle_period;  // idle replicas (no local push, intent active) check the owner's version every n-th round
};

ADAPM_HD bool round_due(uint32_t s, uint32_t round_no, int32_t period) {
  return period <= 1 || ((s + round_no) % (uint32_t)period) == 0u;
}
ADAPM_HD bool slot_swept(uint32_t s, const RoundParams& rp) {
  return rp.sweep != 0 || (rp.sweep_period > 0 && round_due(s, rp.round_no, rp.sweep_period));
}

// Which slots does phase A have to visit? ONE lane, local reads only (the compaction scan of the CUDA backend and
// the slot loop of the CPU backend use it). An idle replica - intent active, no local push since the last
// round, want-bit already standing at the current owner - needs nothing in phase A.
ADAPM_HD bool phase_a_wants(const Ctx& c, uint32_t s, const RoundParams& rp) {
  const int me = c.rank;
  const uint32_t st = meta_state(mem::ld_relaxed(meta_of(c, me) + s));
  if (st == S_REPLICA_PENDING) return true;
  if (st != S_REPLICA) return false;
  if (mem::ld_relaxed(dirty_of(c, me) + s) != 0) return true;
  if (slot_swept(s, rp)) return true;
  if (!intent_active(c, s, rp.clocks)) return true;
  if (!(mem::ld_relaxed(flags_of(c, me) + s) & F_WANT_SET)) return true;
  const Key key = mem::ld_relaxed(slot_key_of(c, me) + s);
  return mem::ld_relaxed(dir_of(c, me) + key) != mem::ld_relaxed(want_owner_of(c, me) + s);  // owner changed
}
// ... and phase C: everything in a transitional state, replicas that phase A visited, and a rolling share
// of the idle replicas (owner version check).
ADAPM_HD bool phase_c_wants(const Ctx& c, uint32_t s, const RoundParams& rp) {
  const int me = c.rank;
  const uint32_t st = meta_state(mem::ld_relaxed(meta_of(c, me) + s));
  if (st == S_FREE || st == S_OWNED) return false;
  if (st != S_REPLICA) return true;
  if (mem::ld_relaxed(flags_of(c, me) + s) & F_REQUESTED) return true;
  return slot_swept(s, rp) || round_due(s, rp.round_no, rp.idle_period);
}

// ---------------------------------------------------------------------------------------
// Phases A and C are written as THREE steps per slot, so that the device can run each step as its own grid-wide pass:
//   resolve  (one lane per slot)   all the metadata work: states, directory, owner slot, versions - including the
//                                  remote (NVLink) metadata loads, of which a thread-per-slot pass keeps 100 000s in flight;
//                                  produces at most one row operation (SlotWork::op with its three row pointers)
//   row op   (one group per slot)  the only step that touches row data: 16-byte loads / reductions, no metadata, no fence
//   commit   (one lane per slot)   versions, flags, state transitions, slot recycling
// The kernel boundaries between the passes order them (plus the cross-rank barriers of the round); on the CPU the three
// steps of a slot run back to back. Nothing in here spins or waits.
enum RowOpKind : uint8_t { OP_NONE = 0, OP_SHIP = 1, OP_FINALIZE = 2, OP_REFRESH = 3, OP_DROP = 4, OP_CLEAR = 5 };
constexpr uint8_t W_ACTIVE = 1, W_NZ = 2, W_REF_NONZERO = 4, W_SKIP_COMMIT = 8, W_WAS_PENDING = 16;

struct SlotWork {
  uint32_t slot;
  uint32_t m;       // the slot's meta word as left by resolve
  int32_t ps;       // the key's slot at the peer (owner / relocation source)
  uint32_t v;       // owner version seen by resolve (refresh)
  uint32_t len;
  uint8_t st;       // slot state seen by resolve
  uint8_t peer;     // owner / source rank
  uint8_t op;       // RowOpKind
  uint8_t flags;    // W_*
  int32_t cls;
  float thresh2;    // OP_SHIP: ship only if |row - base|^2 >= thresh2 (0 = always)
  Key key;
  void* dst;        // OP_SHIP: owner row (reduction target) | FINALIZE/REFRESH: local row | DROP: owner row | CLEAR: local row
  void* ref;        // local base row
  const void* src;  // OP_SHIP/DROP: local row | FINALIZE: source rank's row | REFRESH: owner row (or its published mirror)
};

// The key's slot id at its owner `o` as seen from holder slot `s`: cached next to the standing want-bit (the owner's
// slot of a key cannot change while it stays the owner), otherwise ONE NVLink load.
ADAPM_HD int32_t owner_slot_of(const Ctx& c, uint32_t s, Key key, int o) {
  const int me = c.rank;
  if ((mem::ld_relaxed(flags_of(c, me) + s) & F_WANT_SET) && (int)mem::ld_relaxed(want_owner_of(c, me) + s) == o)
    return mem::ld_relaxed(peer_slot_of(c, me) + s);
  return mem::ld_relaxed(slot_of(c, o) + key);
}

// ---- Phase A: replicas ship their deltas to the owners, expired replicas start dropping, live ones (re)request.
// In steady state (want-bit standing, owner unchanged) this issues only fire-and-forget reductions over NVLink.
template <class Val>
ADAPM_HD void phase_a_resolve(const Ctx& c, SlotWork& w, const RoundParams& rp) {
  const int me = c.rank;
  const uint32_t s = w.slot;
  w.op = OP_NONE; w.flags = W_SKIP_COMMIT; w.ps = -1; w.v = 0; w.thresh2 = 0.f;
  const uint32_t m = mem::ld_acquire(meta_of(c, me) + s);
  const uint32_t st = meta_state(m);
  w.m = m; w.st = (uint8_t)st;
  if (st != S_REPLICA && st != S_REPLICA_PENDING) return;
  const Key key = mem::ld_relaxed(slot_key_of(c, me) + s);
  const int cls = class_of_key(c, key);
  const uint32_t len = key_len(c, key, cls);
  const bool active = intent_active(c, s, rp.clocks);
  const int o = (int)mem::ld_relaxed(dir_of(c, me) + key);
  int32_t ps = -1;
  if (o != me) ps = owner_slot_of(c, s, key, o);
  if (ps < 0) { count(c, C_PROTOCOL_ERRORS); return; }
  w.key = key; w.cls = cls; w.len = len; w.peer = (uint8_t)o; w.ps = ps;
  w.flags = active ? W_ACTIVE : 0;
  if (st == S_REPLICA) {
    uint8_t* dp = dirty_of(c, me) + s;
    const uint8_t f = mem::ld_relaxed(dp);
    const bool swept = slot_swept(s, rp);
    const bool consider = (f != 0) || swept || !active;
    const bool never = rp.threshold > 1e300;  // inf: replicas never synchronise (except on drop)
    if (consider && (!never || !active)) {
      // clear the hint BEFORE the row is read (next pass): a push that lands later sets it again
      mem::st_relaxed(dp, (uint8_t)0);
      w.op = OP_SHIP;
      w.src = row_ptr<Val>(c, me, cls, s);
      w.ref = base_ptr<Val>(c, me, cls, s);
      w.dst = row_ptr<Val>(c, o, cls, ps);
      if (rp.threshold > 0 && active && !swept) w.thresh2 = (float)(rp.threshold * rp.threshold);
    }
  }
}

template <class Val>
ADAPM_HD void phase_a_commit(const Ctx& c, const SlotWork& w) {
  if (w.flags & W_SKIP_COMMIT) return;
  const int me = c.rank;
  const uint32_t s = w.slot;
  const int o = w.peer;
  const int32_t ps = w.ps;
  if (w.op == OP_SHIP && (w.flags & W_NZ)) {
    // the owner's version counts applied updates; this replica accounts for its own bump locally, so that in
    // phase C "owner version == ver_seen" still means "nothing but my own deltas arrived" (no round trip)
    mem::red_add(version_of(c, o) + ps, 1u);
    uint32_t* vs = ver_seen_of(c, me) + s;
    mem::st_relaxed(vs, mem::ld_relaxed(vs) + 1u);
    count(c, C_DELTAS_SHIPPED);
  }
  uint8_t* fl = flags_of(c, me) + s;
  uint8_t* wo = want_owner_of(c, me) + s;
  if (!(w.flags & W_ACTIVE)) {
    // withdraw the standing request (the bit lives in the mask of the owner it was sent to; a relocation resets it)
    const uint8_t f = mem::ld_relaxed(fl);
    if ((f & F_WANT_SET) && (int)mem::ld_relaxed(wo) == o) mem::red_and(want_of(c, o) + ps, ~((uint64_t)1 << me));
    mem::st_relaxed(wo, (uint8_t)0xff);
    mem::st_relaxed(fl, (uint8_t)(f & ~(F_REQUESTED | F_WANT_SET)));
    mem::st_release(meta_of(c, me) + s, meta_next(w.m, S_DROPPING, 0));
    return;
  }
  // the request is sticky: it stands in the owner's want-mask until this rank drops the replica
  uint8_t f = mem::ld_relaxed(fl);
  if (!(f & F_WANT_SET) || (int)mem::ld_relaxed(wo) != o) {
    mem::red_or(want_of(c, o) + ps, (uint64_t)1 << me);
    mem::st_relaxed(peer_slot_of(c, me) + s, ps);
    mem::st_relaxed(wo, (uint8_t)o);
    f |= F_WANT_SET;
  }
  mem::st_relaxed(fl, (uint8_t)(f | F_REQUESTED));
}

// Phase B, filter (ONE lane, local reads only): can this owned slot relocate at all in this round? The standing (sticky)
// want-bits make every replicated key a hit of a plain "want != 0" test in every round; relocation needs exactly one
// requester (technique `all`), which only a few slots satisfy - the device compacts those into a worklist.
ADAPM_HD bool phase_b_candidate(const Ctx& c, uint32_t s) {
  uint64_t mask = mem::ld_relaxed(want_of(c, c.rank) + s);
  if (mask == 0) return false;
  mask &= ~((uint64_t)1 << c.rank);
  if (mask == 0) return false;
  if (c.technique == (int)MgmtTechniques::REPLICATION_ONLY) return false;
  if (c.technique == (int)MgmtTechniques::RELOCATION_ONLY) return true;
  return (mask & (mask - 1)) == 0;   // exactly one requester
}

// Phase B: the owner decides relocate vs replicate for one owned slot (ONE lane).
// Decision rule = reference sync_manager.h:615-641: relocate iff no worker on the owner and no
// other node has intent; the technique switch forces one side.
ADAPM_HD void phase_b_slot(const Ctx& c, uint32_t s, const RoundParams& rp) {
  const int me = c.rank;
  uint64_t* wp = want_of(c, me) + s;
  if (mem::ld_relaxed(wp) == 0) return;
  uint32_t* mp = meta_of(c, me) + s;
  uint32_t m = mem::ld_acquire(mp);
  uint64_t mask = mem::ld_relaxed(wp);   // sticky: holders clear their own bit when they drop the replica
  if (meta_state(m) != S_OWNED || mask == 0) return;
  mask &= ~((uint64_t)1 << me);
  if (mask == 0) return;
  const Key key = mem::ld_relaxed(slot_key_of(c, me) + s);
  bool relocate;
  if (c.technique == (int)MgmtTechniques::REPLICATION_ONLY) relocate = false;
  else if (c.technique == (int)MgmtTechniques::RELOCATION_ONLY) relocate = true;
  else {
    int pc = 0; for (uint64_t t = mask; t; t &= t - 1) ++pc;
    relocate = (pc == 1) && !intent_active(c, s, rp.clocks);
  }
  if (!relocate) return;
  int dst = 0; while (!((mask >> dst) & 1)) ++dst;
  int32_t ds = mem::ld_relaxed(slot_of(c, dst) + key);
  if (ds < 0) { count(c, C_PROTOCOL_ERRORS); return; }
  uint32_t* dmp = meta_of(c, dst) + ds;
  uint32_t dm = mem::ld_acquire(dmp);
  uint32_t dst_state = meta_state(dm);
  if (dst_state != S_REPLICA && dst_state != S_REPLICA_PENDING) return;
  mem::st_relaxed(ver_seen_of(c, dst) + ds, (uint32_t)s);  // source slot id for SUM3 readers / finalize
  mem::fence();
  mem::st_release(dmp, meta_next(dm, dst_state == S_REPLICA ? S_INCOMING_REPLICA : S_INCOMING, (uint32_t)me));
  mem::st_release(mp, meta_next(m, S_OUTGOING, (uint32_t)dst));
  mem::st_relaxed(wp, (uint64_t)0);   // the only requester becomes the owner: nothing stands against this slot any more
  mem::fence();
  for (int r = 0; r < c.L.world; ++r) mem::st_relaxed(dir_of(c, r) + key, (uint8_t)dst);
  count(c, C_RELOCATIONS);
}

// ---- Phase C: transfers, refreshes, drops.  (after the grace period)
template <class Val>
ADAPM_HD void phase_c_resolve(const Ctx& c, SlotWork& w, const RoundParams& rp) {
  const int me = c.rank;
  const uint32_t s = w.slot;
  w.op = OP_NONE; w.flags = W_SKIP_COMMIT; w.ps = -1; w.v = 0; w.thresh2 = 0.f;
  uint32_t* mp = meta_of(c, me) + s;
  const uint32_t m = mem::ld_acquire(mp);
  const uint32_t st = meta_state(m);
  w.m = m; w.st = (uint8_t)st;
  if (st == S_FREE || st == S_OWNED) return;
  const Key key = mem::ld_relaxed(slot_key_of(c, me) + s);
  const int cls = class_of_key(c, key);
  const uint32_t len = key_len(c, key, cls);
  w.key = key; w.cls = cls; w.len = len;
  uint8_t* fl = flags_of(c, me) + s;
  if (state_is_incoming(st)) {
    const int src = (int)meta_peer(m);
    const int32_t ss = (int32_t)mem::ld_relaxed(ver_seen_of(c, me) + s);
    if (ss < 0) { count(c, C_PROTOCOL_ERRORS); return; }
    // (the slot stays INCOMING - readable as row - base + source row - until the row pass folds it: FINALIZING, during
    // which readers have to wait, only lasts for the few microseconds of that one row operation)
    w.peer = (uint8_t)src; w.ps = ss;
    w.op = OP_FINALIZE; w.flags = 0;
    w.dst = row_ptr<Val>(c, me, cls, s); w.ref = base_ptr<Val>(c, me, cls, s); w.src = row_ptr<Val>(c, src, cls, ss);
    return;
  }
  if (st == S_REPLICA || st == S_REPLICA_PENDING) {
    const uint8_t f = mem::ld_relaxed(fl);
    const bool requested = (f & F_REQUESTED) != 0;
    if (requested) mem::st_relaxed(fl, (uint8_t)(f & ~F_REQUESTED));
    if (st == S_REPLICA_PENDING && !requested) return;  // the owner has not seen the request yet
    if (c.technique == (int)MgmtTechniques::RELOCATION_ONLY) return;
    const int o = (int)mem::ld_relaxed(dir_of(c, me) + key);
    if (o == me) return;
    const int32_t ps = owner_slot_of(c, s, key, o);
    if (ps < 0) return;
    // owner state word and version: two independent loads, one NVLink round trip
    const uint32_t pm = mem::ld_relaxed(meta_of(c, o) + ps);
    const uint32_t v = mem::ld_relaxed(version_of(c, o) + ps);
    if (meta_state(pm) != S_OWNED) return;  // owner is mid-relocation: ask again next round
    const uint32_t seen = mem::ld_relaxed(ver_seen_of(c, me) + s);
    if (st == S_REPLICA && v == seen && !slot_swept(s, rp)) return;
    w.peer = (uint8_t)o; w.ps = ps; w.v = v;
    w.op = OP_REFRESH; w.flags = (st == S_REPLICA_PENDING) ? W_WAS_PENDING : 0;
    w.dst = row_ptr<Val>(c, me, cls, s); w.ref = base_ptr<Val>(c, me, cls, s); w.src = row_ptr<Val>(c, o, cls, ps);
    return;
  }
  if (st == S_DROPPING) {
    const int o = (int)mem::ld_relaxed(dir_of(c, me) + key);
    int32_t ps = -1;
    if (o != me) ps = mem::ld_relaxed(slot_of(c, o) + key);
    w.peer = (uint8_t)o; w.ps = ps; w.flags = 0;
    w.src = row_ptr<Val>(c, me, cls, s); w.ref = base_ptr<Val>(c, me, cls, s);
    if (ps >= 0) { w.op = OP_DROP; w.dst = row_ptr<Val>(c, o, cls, ps); }
    else { count(c, C_PROTOCOL_ERRORS); w.op = OP_CLEAR; w.dst = const_cast<void*>(w.src); }
    return;
  }
  if (st == S_OUTGOING) {
    mem::st_release(mp, meta_next(m, S_DEAD, meta_peer(m)));
    return;
  }
  if (st == S_DEAD) {
    w.op = OP_CLEAR; w.flags = 0;
    w.dst = row_ptr<Val>(c, me, cls, s); w.ref = base_ptr<Val>(c, me, cls, s); w.src = w.dst;
    return;
  }
}

template <class Val>
ADAPM_HD void phase_c_commit(const Ctx& c, const SlotWork& w) {
  if (w.flags & W_SKIP_COMMIT) return;
  const int me = c.rank;
  const uint32_t s = w.slot;
  uint32_t* mp = meta_of(c, me) + s;
  if (w.op == OP_FINALIZE) return;   // committed by the row operation itself (finalize_row)
  if (w.op == OP_REFRESH) {
    mem::st_relaxed(ver_seen_of(c, me) + s, w.v);
    count(c, C_REFRESHES);
    if (w.flags & W_WAS_PENDING) {
      mem::st_release(mp, meta_next(w.m, S_REPLICA, 0));
      count(c, C_REPLICA_SETUPS);
    }
    return;
  }
  if (w.op == OP_DROP || (w.op == OP_CLEAR && w.st == S_DROPPING)) {
    if (w.op == OP_DROP && (w.flags & W_NZ)) mem::red_add(version_of(c, w.peer) + w.ps, 1u);
    mem::st_release(slot_of(c, me) + w.key, (int32_t)-1);
    mem::st_release(mp, meta_next(w.m, S_FREE, 0));
    free_slot(c, w.cls, (int32_t)s);
    count(c, C_REPLICA_DROPS);
    return;
  }
  if (w.op == OP_CLEAR) {   // DEAD relocation source
    // the key may already have a fresh slot on this rank (it was requested back)
    cas_i32(slot_of(c, me) + w.key, (int32_t)s, (int32_t)-1);
    mem::st_release(mp, meta_next(w.m, S_FREE, 0));
    free_slot(c, w.cls, (int32_t)s);
    return;
  }
}

// Relocation transfer of one slot: fold the source row into the local one and take over the ownership - as ONE short
// per-slot sequence (state FINALIZING only while it runs), because readers of an in-flight key have to wait it out.
template <class Val, class G>
ADAPM_HD void finalize_row(const Ctx& c, const G& g, SlotWork& w) {
  const int me = c.rank;
  const uint32_t s = w.slot;
  uint32_t* mp = meta_of(c, me) + s;
  const uint32_t m1 = meta_next(w.m, S_FINALIZING, (uint32_t)w.peer);
  if (g.lane() == 0) mem::st_release_local(mp, m1);   // readers of row - base + source row re-validate this word
  // (everything this sequence WRITES is local memory - state word, row, base - so device-scope fences order it for
  //  local and, through this GPU's L2, for remote readers)
  mem::fence_local(); g.sync();
  bool rnz = false;
  row_fold<Val>(g, reinterpret_cast<Val*>(w.dst), reinterpret_cast<Val*>(w.ref), reinterpret_cast<const Val*>(w.src), w.len,
                false, &rnz);
  mem::fence_local(); g.sync();
  if (g.lane() == 0) {
    // invariant used by the in-kernel read of in-flight rows (pm_kernels.cuh: value = local row + source row): a
    // placeholder that became the relocation target (INCOMING, not INCOMING_REPLICA) has an all-zero base
    if (w.st == S_INCOMING && rnz) count(c, C_PROTOCOL_ERRORS);
    const uint32_t sv = mem::ld_relaxed(version_of(c, w.peer) + w.ps);
    mem::red_add(version_of(c, me) + s, sv + 1u);
    mem::st_relaxed(ver_seen_of(c, me) + s, 0xffffffffu);
    mem::st_relaxed(flags_of(c, me) + s, (uint8_t)0);
    mem::st_relaxed(want_owner_of(c, me) + s, (uint8_t)0xff);
    mem::st_release_local(mp, meta_next(m1, S_OWNED, 0));
  }
}

// The row operation of one slot (one group of lanes; the only code of the round that touches row data).
template <class Val, class G>
ADAPM_HD void row_op_execute(const Ctx& c, const G& g, SlotWork& w) {
  Val* dst = reinterpret_cast<Val*>(w.dst);
  Val* ref = reinterpret_cast<Val*>(w.ref);
  const Val* src = reinterpret_cast<const Val*>(w.src);
  uint8_t out = 0;
  switch (w.op) {
    case OP_SHIP: {
      bool ship = true;
      if (w.thresh2 > 0.f) ship = row_delta_norm2<Val>(g, src, ref, w.len) >= (double)w.thresh2;
      if (ship && row_ship<Val>(g, src, ref, dst, w.len, true)) out = W_NZ;
      break;
    }
    case OP_FINALIZE:
      finalize_row<Val>(c, g, w);
      break;
    case OP_REFRESH:
      row_fold<Val>(g, dst, ref, src, w.len, true, (bool*)nullptr);
      break;
    case OP_DROP:
      if (row_ship<Val>(g, src, ref, dst, w.len, false)) out = W_NZ;
      row_clear<Val>(g, const_cast<Val*>(src), ref, w.len);   // a slot returns to the pool with all-zero row and base
      break;
    case OP_CLEAR:
      row_clear<Val>(g, dst, ref, w.len);
      break;
    default: break;
  }
  if (out && g.lane() == 0) w.flags |= out;
}

// Intent pre-pass for one key (ONE lane, any thread, any time): if the key already has a usable local slot, extending
// the intent is just an atomic max on the slot's end clock - the sync round only reads the end clocks. Returns false
// when the key needs the sync thread (no slot yet, or the slot is on its way out).
ADAPM_HD bool extend_intent_if_local(const Ctx& c, Key key, int worker, Clock end) {
  const int32_t s = mem::ld_relaxed(slot_of(c, c.rank) + key);
  if (s < 0) return false;
  const uint32_t m = mem::ld_acquire(meta_of(c, c.rank) + s);
  const uint32_t st = meta_state(m);
  if (!(st == S_OWNED || st == S_REPLICA || st == S_REPLICA_PENDING || state_is_incoming(st))) return false;
  atomic_max_i64(intent_end_of(c, c.rank) + (size_t)s * c.L.workers + worker, end);
  // The sync round may have decided to drop this replica / to hand the key over (or may even have recycled the slot
  // for another key) between the state check and the atomic max: the extension is then not (reliably) seen. Re-read:
  // only an unchanged slot of this very key counts; everything else goes through the host path, which cannot lose it.
  mem::fence();
  const uint32_t m2 = mem::ld_acquire(meta_of(c, c.rank) + s);
  const uint32_t st2 = meta_state(m2);
  const bool still = (st2 == S_OWNED || st2 == S_REPLICA || st2 == S_REPLICA_PENDING || state_is_incoming(st2)) &&
                     (meta_seq(m2) == meta_seq(m) || st2 == st) &&
                     mem::ld_relaxed(slot_key_of(c, c.rank) + s) == key &&
                     mem::ld_relaxed(slot_of(c, c.rank) + key) == s;
  return still;
}

// Is `key` usable from local memory right now (owned or usable replica)?  (PullIfLocal / local sampling)
ADAPM_HD bool is_local(const Ctx& c, Key key) {
  int32_t s = mem::ld_relaxed(slot_of(c, c.rank) + key);
  if (s < 0) return false;
  uint32_t st = meta_state(mem::ld_acquire(meta_of(c, c.rank) + s));
  return st == S_OWNED || st == S_REPLICA || st == S_INCOMING_REPLICA;
}

}  // namespace adapm

// Symmetric-heap layout of one rank's parameter store.
//
// Every rank allocates ONE heap with the SAME layout; peers map each other's heaps
// (POSIX shm on CPU, CUDA-IPC/NVLink on the GPUs), so any per-key or per-slot field of
// any rank is `heap[rank] + offset`. This replaces the reference's
// vector<unique_ptr<Parameter>> + 16384 mutexes (coloc_kv_server_handle.h:122-152,
// :1069-1083) and its Addressbook (addressbook.h:30-176): the ownership directory
// `dir[key]` is fully replicated on every rank and updated by the relocating owner
// with peer stores, so there is no home-node forwarding.
#pragma once
#include "base.h"
#include "atomics.h"

namespace adapm {

struct ClassInfo {
  uint32_t len;         // values per slot of this size class (= the row length of its keys unless Layout::per_key_len)
  uint32_t cap;         // slots of this class per rank
  uint32_t slot_begin;  // first global slot id of this class
  uint32_t pad;
  uint64_t rows_off;    // Val[cap][len]   current value (owner: main copy; replica: base + local delta)
  uint64_t base_off;    // Val[cap][len]   replica sync state ("state at last sync")
  uint64_t free_off;    // int32[cap]      free-slot stack
};

struct Layout {
  int64_t num_keys;
  int32_t world;
  int32_t num_classes;
  int32_t workers;       // local workers per rank
  uint32_t total_slots;
  uint32_t val_bytes;    // sizeof(Val)
  uint32_t pad;
  uint64_t off_dir;        // uint8[num_keys]   owner rank of each key (replicated directory)
  uint64_t off_slot_of;    // int32[num_keys]   local slot of a key, -1 = not resident
  uint64_t off_key_class;  // uint8[num_keys]   size class (only if num_classes > 1)
  uint64_t off_key_len;    // uint32[num_keys]  row length of every key (only if per_key_len: more distinct value
                           //                   lengths than size classes, so a class holds keys of different lengths)
  uint64_t off_meta;       // uint32[S]         state | peer | seq
  uint64_t off_version;    // uint32[S]         owner: #pushes applied
  uint64_t off_ver_seen;   // uint32[S]         replica: owner version at last refresh
  uint64_t off_want;       // uint64[S]         owner: ranks that hold a replica / placeholder of the key (sticky bits)
  uint64_t off_want_owner; // uint8[S]          holder: the owner whose want-mask carries this rank's bit (0xff none)
  uint64_t off_peer_slot;  // int32[S]          holder: the key's slot id at want_owner (valid while dir[key] == want_owner)
  uint64_t off_slot_key;   // int64[S]
  uint64_t off_intent_end; // int64[S*workers]  end clock of the local intents
  uint64_t off_flags;      // uint8[S]          F_REQUESTED (sync thread only)
  uint64_t off_dirty;      // uint8[S]          replica got local pushes since the last delta ship (blind store 1)
  uint64_t off_free_top;   // int32[MAX_CLASSES]
  uint64_t off_counters;   // uint64[C_NUM_COUNTERS]
  uint64_t off_access;     // uint32[2*num_keys] (accesses, local accesses) - only if locality stats are on, else 0
  uint64_t off_sync;       // SyncArea: device-side round state (grace epochs, cross-rank barrier flags)
  uint32_t locality_stats; // PS_LOCALITY_STATS equivalent (run-time switch sys.stats.locality)
  uint32_t per_key_len;    // 1: row lengths come from off_key_len, the class only fixes the slot stride
  ClassInfo cls[MAX_CLASSES];
  uint64_t heap_bytes;
};

// Device-side state of the sync round (one per rank, in the heap, written by peers):
//  * grace epochs: every CTA of a kernel that touches the store registers in active[epoch & 1] for its lifetime;
//    the round flips the epoch after phase B and waits until the old side has drained (an RCU grace period:
//    everything that may have read the old directory is done) - no host involvement, no stream events;
//  * cross-rank barrier: rank r's barrier kernel stores the barrier sequence number into bar_arrive[r] of EVERY
//    rank's area (st.release.sys over NVLink) and then waits until all entries of its own area reached it;
//  * flag exchange: the first barrier of a round also carries one word per rank (stop / sweep requests), so the
//    ranks agree on them without a host barrier.
struct SyncArea {
  uint32_t epoch;
  uint32_t active[2];
  uint32_t pad0[29];
  uint32_t bar_arrive[MAX_RANKS];
  uint32_t flag_word[2][MAX_RANKS];   // [round parity][rank]            (unicast exchange)
  uint32_t my_flag[2];                // [round parity] this rank's word (multicast: reduced in the switch by the readers)
  uint32_t pad1[30];
};

struct IntentRec {
  int64_t key;
  int64_t end;
  int32_t worker;
  int32_t pad;
};

// The execution context handed to every kernel / CPU loop (by value).
struct Ctx {
  Layout L;
  int32_t rank;
  int32_t technique;    // MgmtTechniques
  char* heap[MAX_RANKS];
  // NVLS multicast mapping of the heaps (cuda, NVSwitch, one process per GPU; nullptr otherwise): a multimem store /
  // reduction to mc_heap + off reaches offset `off` of EVERY rank's heap with one NVLink transaction
  char* mc_heap;
};

template <class T> ADAPM_HD T* at(const Ctx& c, int r, uint64_t off) {
  return reinterpret_cast<T*>(c.heap[r] + off);
}
template <class T> ADAPM_HD T* at_all(const Ctx& c, uint64_t off) {   // the multicast alias of `off` (mc_heap != nullptr)
  return reinterpret_cast<T*>(c.mc_heap + off);
}
ADAPM_HD uint8_t* dir_of(const Ctx& c, int r) { return at<uint8_t>(c, r, c.L.off_dir); }
ADAPM_HD int32_t* slot_of(const Ctx& c, int r) { return at<int32_t>(c, r, c.L.off_slot_of); }
ADAPM_HD uint32_t* meta_of(const Ctx& c, int r) { return at<uint32_t>(c, r, c.L.off_meta); }
ADAPM_HD uint32_t* version_of(const Ctx& c, int r) { return at<uint32_t>(c, r, c.L.off_version); }
ADAPM_HD uint32_t* ver_seen_of(const Ctx& c, int r) { return at<uint32_t>(c, r, c.L.off_ver_seen); }
ADAPM_HD uint64_t* want_of(const Ctx& c, int r) { return at<uint64_t>(c, r, c.L.off_want); }
ADAPM_HD int64_t* slot_key_of(const Ctx& c, int r) { return at<int64_t>(c, r, c.L.off_slot_key); }
ADAPM_HD int64_t* intent_end_of(const Ctx& c, int r) { return at<int64_t>(c, r, c.L.off_intent_end); }
ADAPM_HD uint8_t* flags_of(const Ctx& c, int r) { return at<uint8_t>(c, r, c.L.off_flags); }
ADAPM_HD uint8_t* dirty_of(const Ctx& c, int r) { return at<uint8_t>(c, r, c.L.off_dirty); }
ADAPM_HD uint8_t* want_owner_of(const Ctx& c, int r) { return at<uint8_t>(c, r, c.L.off_want_owner); }
ADAPM_HD int32_t* peer_slot_of(const Ctx& c, int r) { return at<int32_t>(c, r, c.L.off_peer_slot); }
ADAPM_HD int32_t* free_top_of(const Ctx& c, int r) { return at<int32_t>(c, r, c.L.off_free_top); }
ADAPM_HD uint64_t* counters_of(const Ctx& c, int r) { return at<uint64_t>(c, r, c.L.off_counters); }
ADAPM_HD SyncArea* sync_area_of(const Ctx& c, int r) { return at<SyncArea>(c, r, c.L.off_sync); }

ADAPM_HD int class_of_key(const Ctx& c, Key k) {
  if (c.L.num_classes == 1) return 0;
  return at<uint8_t>(c, c.rank, c.L.off_key_class)[k];
}
// number of values of `key`'s row (<= the slot stride of its size class)
ADAPM_HD uint32_t key_len(const Ctx& c, Key k, int cls) {
  if (c.L.per_key_len) return at<uint32_t>(c, c.rank, c.L.off_key_len)[k];
  return c.L.cls[cls].len;
}
template <class Val> ADAPM_HD Val* row_ptr(const Ctx& c, int r, int cls, uint32_t slot) {
  const ClassInfo& ci = c.L.cls[cls];
  return reinterpret_cast<Val*>(c.heap[r] + ci.rows_off) + (size_t)(slot - ci.slot_begin) * ci.len;
}
template <class Val> ADAPM_HD Val* base_ptr(const Ctx& c, int r, int cls, uint32_t slot) {
  const ClassInfo& ci = c.L.cls[cls];
  return reinterpret_cast<Val*>(c.heap[r] + ci.base_off) + (size_t)(slot - ci.slot_begin) * ci.len;
}
ADAPM_HD void count(const Ctx& c, int which, uint64_t n = 1) {
  mem::red_add(counters_of(c, c.rank) + which, n);
}

}  // namespace adapm

// Base types of the GPU-native parameter manager.
//
// Parity with the reference's include/ps/base.h:1-65 (Key, Clock, CLOCK_MAX,
// WORKER_FINISHED, WINDOW_MAX, Version, MgmtTechniques, LOCAL). The reference
// defaults Key to uint64_t and its bindings to int64_t (bindings.cc:8); we use
// int64_t everywhere so that torch.int64 tensors are keys without a cast.
#pragma once
#include <cstdint>
#include <cstddef>
#include <limits>

#if defined(__CUDACC__)
#define ADAPM_HD __host__ __device__ __forceinline__
#define ADAPM_D __device__ __forceinline__
#else
#define ADAPM_HD inline
#define ADAPM_D inline
#endif

namespace adapm {

using Key = int64_t;
using Clock = int64_t;
using Version = uint32_t;
using SampleID = int64_t;

constexpr Clock CLOCK_MAX = std::numeric_limits<Clock>::max();
constexpr Clock WORKER_FINISHED = CLOCK_MAX;   // clock of a worker that has finalized
constexpr Clock WINDOW_MAX = CLOCK_MAX / 4;    // "act on every intent right away"
constexpr int LOCAL = -1;                      // timestamp of an op that completed locally/inline

constexpr int MAX_RANKS = 64;          // want-mask is one 64-bit word per slot
constexpr int MAX_CLASSES = 32;        // size classes of the row slabs (any number of distinct value lengths maps onto them)
constexpr int MAX_LOCAL_WORKERS = 16;  // logical workers per rank (per GPU)

// Which management techniques the sync engine may use (reference base.h:54).
enum class MgmtTechniques : int { ALL = 0, REPLICATION_ONLY = 1, RELOCATION_ONLY = 2 };

// Slot life cycle. One slot = one row of one length class on one rank.
//   OWNED            this rank holds the main copy
//   REPLICA_PENDING  placeholder created by an intent; not usable until first refresh
//                    (reference: replica with version == -1)
//   REPLICA          usable replica; row = base + local unsynced delta
//   INCOMING         relocation target before the transfer is finalized;
//                    logical value = row - base + src.row
//   FINALIZING       transient inside the finalize kernel (readers spin/retry)
//   OUTGOING         relocation source; row stays valid until the grace period ends
//   DEAD             relocation source after the transfer; freed one round later
//   DROPPING         replica whose intent expired; freed after the grace period
enum SlotState : uint32_t {
  S_FREE = 0, S_OWNED = 1, S_REPLICA_PENDING = 2, S_REPLICA = 3, S_INCOMING = 4,
  S_FINALIZING = 5, S_OUTGOING = 6, S_DEAD = 7, S_DROPPING = 8,
  S_INCOMING_REPLICA = 9   // INCOMING whose slot was a usable replica: local reads keep working
};
ADAPM_HD bool state_is_incoming(uint32_t st) { return st == 4u || st == 9u; }

// meta word: state | peer<<8 | seq<<16   (seq bumps on every transition; seqlock for readers)
ADAPM_HD uint32_t meta_make(uint32_t state, uint32_t peer, uint32_t seq) {
  return (state & 0xffu) | ((peer & 0xffu) << 8) | ((seq & 0xffffu) << 16);
}
ADAPM_HD uint32_t meta_state(uint32_t m) { return m & 0xffu; }
ADAPM_HD uint32_t meta_peer(uint32_t m) { return (m >> 8) & 0xffu; }
ADAPM_HD uint32_t meta_seq(uint32_t m) { return (m >> 16) & 0xffffu; }
ADAPM_HD uint32_t meta_next(uint32_t m, uint32_t state, uint32_t peer) {
  return meta_make(state, peer, meta_seq(m) + 1);
}

// slot flag bits (one byte per slot)
constexpr uint8_t F_REQUESTED = 2;  // phase A visited this replica in the current round (refresh it in phase C)
constexpr uint8_t F_WANT_SET = 4;   // this rank's bit is set in the want-mask of the owner named by want_owner[slot]

// Counters written by the PM kernels / loops (one block per rank, in the heap).
enum Counter : int {
  C_PULL_LOCAL = 0, C_PULL_REMOTE, C_PUSH_LOCAL, C_PUSH_REMOTE,
  C_RELOCATIONS, C_REPLICA_SETUPS, C_REPLICA_DROPS, C_REFRESHES, C_DELTAS_SHIPPED,
  C_INTENTS_REGISTERED, C_INTENTS_DEFERRED, C_ALLOC_FAIL, C_PROTOCOL_ERRORS,
  C_NUM_COUNTERS = 32
};

}  // namespace adapm

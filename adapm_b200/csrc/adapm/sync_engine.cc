// SyncEngine: one background thread per rank that drives the sync rounds.
//
// A round (all ranks in lock-step, separated by control-plane barriers):
//   0. publish stop/sweep flags, barrier, agree on stop/sweep
//   1. act on intents whose start clock falls into the estimated window (ActionTimer),
//      i.e. create placeholder replicas                     [register_intents]
//   2. phase A: replicas ship deltas to owners, expired replicas start dropping,
//      live replicas request a refresh                      [barrier]
//   3. phase B: owners decide relocate vs replicate and announce new owners
//      in every rank's directory                            [barrier]
//   4. grace period: all worker ops that may have used the old directory drain [barrier]
//   5. phase C: relocation transfers, replica refreshes, drops
// Reference equivalent: SyncManager::thread/startSync/ProcessSyncMessage
// (sync_manager.h:291-382,452-520,544-799); message round trips became barriers.
#include "node.h"
#include "nvtx.h"

#include <algorithm>
#include <sstream>

namespace adapm {

SyncEngine::SyncEngine(Server* server)
    : server_(server),
      timer_(server->options().workers, server->options().timing_initial_estimate, server->options().timing_autotune,
             server->options().timing_smoothing_factor, server->options().timing_buffer_quantile),
      heaps_(server->options().workers) {}

SyncEngine::~SyncEngine() {
  if (thread_.joinable()) {
    try { request_stop_and_join(); } catch (...) {}
  }
}

void SyncEngine::start() {
  if (server_->num_servers() == 1) return;  // nothing to synchronise
  last_run_ = std::chrono::steady_clock::now();
  thread_ = std::thread([this] {
    try {
      loop();
    } catch (const std::exception& e) {
      ALOG("[adapm] rank " << server_->my_rank() << " sync thread died: " << e.what());
      server_->control()->sync_barrier.broken.store(1);
      server_->control()->node_barrier.broken.store(1);
      server_->control()->worker_barrier.broken.store(1);
    }
  });
}

void SyncEngine::request_stop_and_join() {
  if (!thread_.joinable()) return;
  server_->my_control().stop_requested.store(1, std::memory_order_release);
  thread_.join();
}

void SyncEngine::enqueue(FutureIntent&& fi) {
  std::lock_guard<std::mutex> lk(in_mu_);
  incoming_.push_back(std::move(fi));
}

std::shared_ptr<std::vector<Key>> SyncEngine::acquire_key_buffer() {
  {
    std::lock_guard<std::mutex> lk(pool_mu_);
    if (!key_pool_.empty()) {
      auto b = std::move(key_pool_.back());
      key_pool_.pop_back();
      return b;
    }
  }
  return std::make_shared<std::vector<Key>>();
}

uint64_t SyncEngine::rounds_done() const {
  return server_->my_control().rounds_done.load(std::memory_order_acquire);
}

void SyncEngine::wait_sync() {
  if (server_->num_servers() == 1) return;
  RankControl& rc = server_->my_control();
  uint64_t target = rc.rounds_done.load(std::memory_order_acquire) + 2;
  // ask for (at least) two guaranteed-propagation rounds
  int32_t cur = rc.sweep_requested.load();
  while (cur < 2 && !rc.sweep_requested.compare_exchange_weak(cur, 2)) {}
  auto t0 = std::chrono::steady_clock::now();
  int spins = 0;
  // ... and keep waiting (bounded) while intents of this rank are still deferred, e.g. because a key's old
  // slot has to be recycled first or the pool is momentarily full
  int extensions = 0;
  for (;;) {
    const uint64_t done = rc.rounds_done.load(std::memory_order_acquire);
    if (done >= target) {
      if (deferred_pending_.load(std::memory_order_acquire) == 0 || extensions >= 4) break;
      target = done + 2;   // the deferred records register in the next round; wait until that round is complete
      ++extensions;
      int32_t c2 = rc.sweep_requested.load();
      while (c2 < 2 && !rc.sweep_requested.compare_exchange_weak(c2, 2)) {}
    }
    if (++spins < 50) std::this_thread::yield();
    else std::this_thread::sleep_for(std::chrono::microseconds(50));
    if ((spins & 4095) == 0) {
      double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      ADAPM_CHECK(el < server_->options().wait_timeout_s, "watchdog: WaitSync timed out (sync thread or a peer is dead)");
      ADAPM_CHECK(!server_->control()->sync_barrier.broken.load(), "WaitSync: sync barrier broken by a failed peer");
    }
  }
}

void SyncEngine::collect_intents(const std::vector<Clock>& clocks, const std::vector<Clock>& windows) {
  {
    std::lock_guard<std::mutex> lk(in_mu_);
    while (!incoming_.empty()) {
      FutureIntent fi = std::move(incoming_.front());
      incoming_.pop_front();
      ++intents_seen_;
      heaps_[fi.worker].push(std::move(fi));
    }
  }
  recs_.clear();
  recs_.swap(deferred_);  // retry what could not be registered last round
  // Records of one round are merged per (key, worker): a key that occurs in several of the intents that become
  // relevant in this round (with a long look-ahead: most hot keys, once per batch) is registered once, with the
  // latest end clock. O(1) per record with a round-stamped table (8 B per key; skipped for very large key spaces).
  const bool merge = server_->num_keys() <= ((int64_t)1 << 25) && heaps_.size() == 1;
  if (merge) {
    // one 8-byte entry per key: round stamp << 32 | index of the key's record in recs_
    if (rec_tab_.empty()) rec_tab_.assign((size_t)server_->num_keys(), 0ull);
    if (++rec_epoch_ == 0) { std::fill(rec_tab_.begin(), rec_tab_.end(), 0ull); rec_epoch_ = 1; }
    for (size_t i = 0; i < recs_.size(); ++i) rec_tab_[(size_t)recs_[i].key] = ((uint64_t)rec_epoch_ << 32) | (uint32_t)i;
  }
  const bool tracing = server_->tracing();
  for (size_t w = 0; w < heaps_.size(); ++w) {
    auto& h = heaps_[w];
    const Clock clk = clocks[w];
    if (clk == WORKER_FINISHED) { while (!h.empty()) h.pop(); continue; }
    const Clock horizon = (windows[w] >= WINDOW_MAX || clk > CLOCK_MAX - windows[w]) ? CLOCK_MAX : clk + windows[w];
    // the intents that become relevant now, latest first: with the usual "one intent per future step" pattern the
    // first occurrence of a key then already carries the latest end clock and duplicates are a pure table hit
    due_.clear();
    while (!h.empty() && h.top().start <= horizon) {
      due_.push_back(h.top());
      h.pop();
    }
    for (size_t di = due_.size(); di-- > 0;) {
      const FutureIntent& fi = due_[di];
      if (fi.end > clk) {
        std::vector<Key>& ks = *fi.keys;
        if (merge) {
          // duplicates inside one intent merge like duplicates across intents: one table access per key, prefetched
          // (the table is far larger than the caches and the keys are random)
          const size_t n = ks.size();
          const Key* kp = ks.data();
          const uint64_t stamp = (uint64_t)rec_epoch_ << 32;
          for (size_t i = 0; i < n; ++i) {
            if (i + 12 < n) __builtin_prefetch(&rec_tab_[(size_t)kp[i + 12]], 1, 0);
            const Key k = kp[i];
            uint64_t& e = rec_tab_[(size_t)k];
            if ((e >> 32) == rec_epoch_) {
              IntentRec& prev = recs_[(size_t)(uint32_t)e];
              if (fi.end > prev.end) prev.end = fi.end;
              continue;
            }
            e = stamp | (uint32_t)recs_.size();
            IntentRec r;
            r.key = k; r.end = fi.end; r.worker = (int32_t)w; r.pad = 0;
            recs_.push_back(r);
            if (tracing && (server_->trace_all_ || server_->traced_.count(k))) server_->trace(k, TraceEvent::INTENT_START);
          }
        } else {
          // the reference dedupes in Intent() (coloc_kv_worker.h:394-401); here it happens off the
          // worker thread, once per batch
          if (ks.size() > 1) {
            const int64_t nk = server_->num_keys();
            if (nk <= (int64_t)1 << 25) {
              // O(n) dedupe with an epoch-stamped table (4 B per key) instead of a sort
              if (seen_epoch_.empty()) seen_epoch_.assign((size_t)nk, 0u);
              if (++epoch_ == 0) { std::fill(seen_epoch_.begin(), seen_epoch_.end(), 0u); epoch_ = 1; }
              size_t m = 0;
              for (size_t i = 0; i < ks.size(); ++i) {
                const Key k = ks[i];
                if (seen_epoch_[(size_t)k] != epoch_) { seen_epoch_[(size_t)k] = epoch_; ks[m++] = k; }
              }
              ks.resize(m);
            } else {
              std::sort(ks.begin(), ks.end());
              ks.erase(std::unique(ks.begin(), ks.end()), ks.end());
            }
          }
          for (Key k : ks) {
            IntentRec r;
            r.key = k; r.end = fi.end; r.worker = (int32_t)w; r.pad = 0;
            recs_.push_back(r);
            if (tracing && (server_->trace_all_ || server_->traced_.count(k))) server_->trace(k, TraceEvent::INTENT_START);
          }
        }
      }
    }
    for (FutureIntent& fi : due_) {   // recycle the key buffers
      std::shared_ptr<std::vector<Key>> done = std::move(fi.keys);
      if (done && done.use_count() == 1) {
        std::lock_guard<std::mutex> lk(pool_mu_);
        if (key_pool_.size() < 64) key_pool_.push_back(std::move(done));
      }
    }
    due_.clear();
  }
}

void SyncEngine::round(bool sweep) {
  const Options& opt = server_->options();
  Backend& be = server_->backend();
  ControlBlock* ctl = server_->control();
  const int world = opt.world;
  const double to = opt.wait_timeout_s;

  std::vector<Clock> clocks = server_->worker_clocks();
  std::vector<Clock> windows(clocks.size(), WINDOW_MAX);
  if (opt.time_intent_actions) windows = timer_.estimate_windows_and_tune(clocks, round_no_.load(std::memory_order_relaxed));

  RoundParams rp;
  memset(&rp, 0, sizeof(rp));
  for (size_t w = 0; w < clocks.size(); ++w) rp.clocks[w] = clocks[w];
  rp.threshold = opt.sync_threshold;
  rp.sweep = sweep ? 1 : 0;
  rp.round_no = (uint32_t)round_no_.load(std::memory_order_relaxed);
  rp.sweep_period = opt.sweep_period;
  rp.idle_period = opt.idle_period;

  sw_register_.resume();
  sw_collect_.resume();
  collect_intents(clocks, windows);
  sw_collect_.stop();
  if (!recs_.empty()) {
    status_.assign(recs_.size(), 0);
    be.register_intents(recs_.data(), recs_.size(), rp, status_.data());
    for (size_t i = 0; i < recs_.size(); ++i) {
      if (status_[i] == 1) deferred_.push_back(recs_[i]);
      else if (status_[i] == 0) ++recs_registered_;
    }
  }
  deferred_pending_.store(deferred_.size(), std::memory_order_release);
  sw_register_.stop();

  sw_phase_a_.resume();
  {
    ADAPM_NVTX("adapm::sync::phase_a");
    be.phase_a(rp);
    be.round_fence();
  }
  sw_phase_a_.stop();
  sw_barriers_.resume(); ctl->sync_barrier.wait(world, to, "sync round: after phase A"); sw_barriers_.stop();

  sw_phase_b_.resume();
  {
    ADAPM_NVTX("adapm::sync::phase_b");
    be.phase_b(rp);
    be.round_fence();
  }
  sw_phase_b_.stop();
  sw_barriers_.resume(); ctl->sync_barrier.wait(world, to, "sync round: after phase B"); sw_barriers_.stop();

  sw_grace_.resume();
  {
    ADAPM_NVTX("adapm::sync::grace");
    be.grace();
  }
  sw_grace_.stop();
  sw_barriers_.resume(); ctl->sync_barrier.wait(world, to, "sync round: grace"); sw_barriers_.stop();

  sw_phase_c_.resume();
  {
    ADAPM_NVTX("adapm::sync::phase_c");
    be.phase_c(rp);
    be.round_fence();
  }
  sw_phase_c_.stop();
  if (server_->tracing()) server_->observe_traced_keys();
}

// Pacing of the rounds (reference wait_none / wait_period / wait_interval, sync_manager.h:385-411) plus a cadence floor
// in worker clocks.
//
// The work of a round is "every replica that changed since the previous round"; with many ranks the hot replicas change
// within a step or two, so that set saturates and a round costs the same whether it comes after 2 steps or after 20.
// Under load the rounds pace themselves (a round takes longer than min_clocks steps), but after any gap in the step
// stream (barrier, checkpoint, loader stall) the engine would otherwise restart with a burst of short-interval rounds,
// each refreshing the whole hot set again (more refresh traffic per step and slower steps right after the gap).
// Requests that wait for rounds (WaitSync, shutdown) are served at
// once, and without clock progress a round starts every min_clocks_wait_ms so that intents and evictions never starve.
void SyncEngine::pace(bool device_round) {
  ADAPM_NVTX("adapm::sync::pace");
  const Options& opt = server_->options();
  RankControl& rc = server_->my_control();
  sw_pausing_.resume();
  auto fastest_clock = [&] {
    Clock m = 0;
    for (Clock c : server_->worker_clocks()) if (c != WORKER_FINISHED && c > m) m = c;
    return m;
  };
  // somebody waits for rounds (WaitSync, shutdown) - on ANY rank: a round is collective, so a peer's request is as urgent
  // as my own (the requests live in the shared control block)
  ControlBlock* ctl = server_->control();
  const int world = opt.world;
  auto urgent = [&] {
    if (rc.sweep_requested.load() > 0 || rc.stop_requested.load() > 0) return true;
    for (int r = 0; r < world; ++r) {
      if (ctl->ranks[r].sweep_requested.load(std::memory_order_relaxed) > 0 ||
          ctl->ranks[r].stop_requested.load(std::memory_order_relaxed) > 0) return true;
    }
    return false;
  };
  if (round_no_ > 0 && !urgent()) {
    if (opt.sync_pause_ms > 0) {
      std::this_thread::sleep_for(std::chrono::milliseconds(opt.sync_pause_ms));
    } else if (opt.sync_max_per_sec > 0) {
      auto target = last_run_ + std::chrono::nanoseconds((int64_t)(1e9 / opt.sync_max_per_sec));
      if (std::chrono::steady_clock::now() < target) std::this_thread::sleep_until(target);
    }
    const int min_clocks = opt.sync_min_clocks >= 0 ? opt.sync_min_clocks : (device_round ? 8 : 0);
    if (min_clocks > 0) {
      const auto deadline = last_run_ + std::chrono::milliseconds(std::max(1, opt.sync_min_clocks_wait_ms));
      while (std::chrono::steady_clock::now() < deadline) {
        if (fastest_clock() - last_round_clock_ >= (Clock)min_clocks || urgent()) break;
        std::this_thread::sleep_for(std::chrono::microseconds(100));
      }
    }
  }
  last_run_ = std::chrono::steady_clock::now();
  last_round_clock_ = fastest_clock();
  sw_pausing_.stop();
}

// The same loop for backends that run a whole round by themselves (cuda: device-side barriers, grace period and
// stop/sweep agreement - the round is one enqueue): this thread only feeds intents and reads the outcome back.
void SyncEngine::loop_fused() {
  const Options& opt = server_->options();
  Backend& be = server_->backend();
  RankControl& rc = server_->my_control();
  sw_total_.start();
  for (;;) {
    pace(/*device_round=*/true);

    RoundRequest rq;
    rq.want_stop = rc.stop_requested.load(std::memory_order_acquire) != 0;
    rq.want_sweep = rc.sweep_requested.load(std::memory_order_acquire) > 0;
    std::vector<Clock> clocks = server_->worker_clocks();
    std::vector<Clock> windows(clocks.size(), WINDOW_MAX);
    if (opt.time_intent_actions) windows = timer_.estimate_windows_and_tune(clocks, round_no_.load(std::memory_order_relaxed));
    memset(&rq.rp, 0, sizeof(rq.rp));
    for (size_t w = 0; w < clocks.size(); ++w) rq.rp.clocks[w] = clocks[w];
    rq.rp.threshold = opt.sync_threshold;
    rq.rp.round_no = (uint32_t)round_no_.load(std::memory_order_relaxed);
    rq.rp.sweep_period = opt.sweep_period;
    rq.rp.idle_period = opt.idle_period;

    sw_register_.resume();
    sw_collect_.resume();
    {
      ADAPM_NVTX("adapm::sync::collect_intents");
      collect_intents(clocks, windows);
    }
    sw_collect_.stop();
    sw_register_.stop();
    status_.assign(recs_.size(), 0);
    rq.recs = recs_.data();
    rq.n_recs = recs_.size();
    rq.status = status_.data();

    sw_phase_a_.resume();   // (the whole device round is accounted here)
    RoundOutcome out;
    {
      ADAPM_NVTX("adapm::sync::device_round");
      out = be.fused_round(rq);
    }
    sw_phase_a_.stop();
    if (out.all_stop) break;
    for (size_t i = 0; i < recs_.size(); ++i) {
      if (status_[i] == 1) deferred_.push_back(recs_[i]);
      else if (status_[i] == 0) ++recs_registered_;
    }
    deferred_pending_.store(deferred_.size(), std::memory_order_release);
    if (server_->tracing()) server_->observe_traced_keys();

    if (rq.want_sweep) {
      int32_t cur = rc.sweep_requested.load();
      while (cur > 0 && !rc.sweep_requested.compare_exchange_weak(cur, cur - 1)) {}
    }
    ++round_no_;
    rc.rounds_done.fetch_add(1, std::memory_order_acq_rel);
  }
  sw_total_.stop();
}

void SyncEngine::loop() {
  if (server_->backend().has_fused_round()) { fused_ = true; loop_fused(); return; }
  const Options& opt = server_->options();
  ControlBlock* ctl = server_->control();
  RankControl& rc = server_->my_control();
  const int world = opt.world;
  sw_total_.start();
  for (;;) {
    // ---- pacing (reference wait_none / wait_period / wait_interval, sync_manager.h:385-411)
    pace(/*device_round=*/false);

    // ---- agree on stop / sweep
    rc.snap_stop.store(rc.stop_requested.load(std::memory_order_acquire));
    rc.snap_sweep.store(rc.sweep_requested.load(std::memory_order_acquire) > 0 ? 1 : 0);
    sw_barriers_.resume();
    ctl->sync_barrier.wait(world, opt.wait_timeout_s, "sync round: start");
    sw_barriers_.stop();
    bool all_stop = true, any_sweep = false;
    for (int r = 0; r < world; ++r) {
      all_stop = all_stop && ctl->ranks[r].snap_stop.load() != 0;
      any_sweep = any_sweep || ctl->ranks[r].snap_sweep.load() != 0;
    }
    if (all_stop) break;

    round(any_sweep);

    if (rc.snap_sweep.load()) {
      int32_t cur = rc.sweep_requested.load();
      while (cur > 0 && !rc.sweep_requested.compare_exchange_weak(cur, cur - 1)) {}
    }
    ++round_no_;
    rc.rounds_done.fetch_add(1, std::memory_order_acq_rel);
  }
  sw_total_.stop();
}

std::string SyncEngine::report() const {
  std::ostringstream os;
  double tot = sw_total_.elapsed_s();
  const uint64_t rounds = round_no_.load(std::memory_order_relaxed);
  os << "[rank " << server_->my_rank() << "] sync: " << rounds << " rounds in " << tot << "s ("
     << (tot > 0 ? rounds / tot : 0) << "/s), intents " << intents_seen_.load() << " (" << recs_registered_.load()
     << " key registrations), clocks/round estimate " << timer_.avg_estimate() << "; time: pausing "
     << sw_pausing_.elapsed_s() << "s, register " << sw_register_.elapsed_s() << "s (of which host-side intent collection "
     << sw_collect_.elapsed_s() << "s), " << (fused_ ? "device round (enqueue + wait) " : "phaseA ")
     << sw_phase_a_.elapsed_s() << "s, phaseB " << sw_phase_b_.elapsed_s() << "s, grace " << sw_grace_.elapsed_s()
     << "s, phaseC " << sw_phase_c_.elapsed_s() << "s, barriers " << sw_barriers_.elapsed_s() << "s";
  return os.str();
}

}  // namespace adapm

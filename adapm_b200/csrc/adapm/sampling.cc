// Sampling support: naive / preloc / pool / local schemes (parity: include/ps/sampling.h).
//
//   naive   draw K keys at PrepareSample, PullSample = ordinary Pull of the next n keys
//   preloc  naive + Intent(keys, start, end) so the sync rounds pre-localise them
//   pool    keys are drawn from a shared per-node pool that is reshuffled `reuse` times
//           before it is redrawn (implemented as documented in the reference; its own
//           pool draw is unreachable, SURVEY 7.5) + Intent like preloc
//   local   nothing at PrepareSample; PullSample rejects draws until a key is resident
//           locally (or, for a declared contiguous key range, walks upward to the next
//           resident key). Never communicates; does not preserve the distribution.
#include <cmath>
#include <cstdint>

#include "node.h"

namespace adapm {

namespace {

class UniformDist : public KeyDistribution {
 public:
  UniformDist(Key mn, Key mx) : d_(mn, mx - 1) { min_key = mn; max_key = mx; name = "uniform"; }
  Key draw(std::mt19937_64& rng) override { return d_(rng); }
 private:
  std::uniform_int_distribution<Key> d_;
};

// key = floor(exp(u * ln(max-min+1)) + min - 1), u ~ U[0,1)   (reference bindings.cc:72-76)
class LogUniformDist : public KeyDistribution {
 public:
  LogUniformDist(Key mn, Key mx) : u_(0.0, 1.0) { min_key = mn; max_key = mx; name = "log-uniform"; lg_ = std::log((long double)(mx - mn + 1)); }
  Key draw(std::mt19937_64& rng) override {
    Key k = (Key)(std::exp(u_(rng) * lg_) + (long double)min_key - 1);
    if (k < min_key) k = min_key;
    if (k >= max_key) k = max_key - 1;
    return k;
  }
 private:
  std::uniform_real_distribution<long double> u_;
  long double lg_;
};

// Walker alias table over n keys: key_i = first_key + i * stride, P(i) ~ weights[i].
class AliasDist : public KeyDistribution {
 public:
  AliasDist(const double* w, int64_t n, Key first, Key stride) : n_(n), first_(first), stride_(stride), prob_(n), alias_(n), u_(0.0, 1.0) {
    name = "alias";
    if (stride == 1) { min_key = first; max_key = first + n; }
    build_alias_table(w, n, prob_.data(), alias_.data());
  }
  Key draw(std::mt19937_64& rng) override {
    int64_t i = (int64_t)(u_(rng) * n_);
    if (i >= n_) i = n_ - 1;
    int64_t j = u_(rng) < prob_[i] ? i : alias_[i];
    return first_ + j * stride_;
  }
 private:
  int64_t n_;
  Key first_, stride_;
  std::vector<float> prob_;
  std::vector<int32_t> alias_;
  std::uniform_real_distribution<double> u_;
};

class CallbackDist : public KeyDistribution {
 public:
  CallbackDist(std::function<Key()> fn, Key mn, Key mx) : fn_(std::move(fn)) { min_key = mn; max_key = mx; name = "callback"; }
  Key draw(std::mt19937_64&) override {
    std::lock_guard<std::mutex> lk(mu_);  // app callbacks are not assumed to be thread-safe
    return fn_();
  }
 private:
  std::function<Key()> fn_;
  std::mutex mu_;
};

}  // namespace

void build_alias_table(const double* w, int64_t n, float* prob, int32_t* alias) {
  ADAPM_CHECK(n >= 1, "alias table: needs at least one weight");
  ADAPM_CHECK(n <= INT32_MAX, "alias table: " << n << " weights, at most " << INT32_MAX << " fit the int32 alias");
  double sum = 0;
  for (int64_t i = 0; i < n; ++i) {
    // a negative weight yields prob < 0 and an infinite one prob = 0 for every other key: both draw garbage silently
    ADAPM_CHECK(std::isfinite(w[i]) && w[i] >= 0, "alias table: weight " << i << " is " << w[i]
                                                                          << ", weights must be finite and >= 0");
    sum += w[i];
  }
  ADAPM_CHECK(std::isfinite(sum), "alias table: the weights' sum overflows a double");
  ADAPM_CHECK(sum > 0, "alias table: weights sum to zero");
  std::vector<double> p(n);
  std::vector<int64_t> small, large;
  for (int64_t i = 0; i < n; ++i) { p[i] = w[i] * n / sum; (p[i] < 1.0 ? small : large).push_back(i); }
  while (!small.empty() && !large.empty()) {
    int64_t s = small.back(); small.pop_back();
    int64_t l = large.back(); large.pop_back();
    prob[s] = (float)p[s]; alias[s] = (int32_t)l;
    p[l] = p[l] + p[s] - 1.0;
    (p[l] < 1.0 ? small : large).push_back(l);
  }
  for (int64_t i : large) { prob[i] = 1.f; alias[i] = (int32_t)i; }
  for (int64_t i : small) { prob[i] = 1.f; alias[i] = (int32_t)i; }
}

std::shared_ptr<KeyDistribution> make_uniform_distribution(Key mn, Key mx) {
  ADAPM_CHECK(mx > mn, "uniform distribution needs max > min");
  return std::make_shared<UniformDist>(mn, mx);
}
std::shared_ptr<KeyDistribution> make_log_uniform_distribution(Key mn, Key mx) {
  ADAPM_CHECK(mx > mn, "log-uniform distribution needs max > min");
  return std::make_shared<LogUniformDist>(mn, mx);
}
std::shared_ptr<KeyDistribution> make_alias_distribution(const double* w, int64_t n, Key first, Key stride) {
  ADAPM_CHECK(n > 0, "alias distribution needs at least one weight");
  return std::make_shared<AliasDist>(w, n, first, stride);
}
std::shared_ptr<KeyDistribution> make_callback_distribution(std::function<Key()> fn, Key mn, Key mx) {
  return std::make_shared<CallbackDist>(std::move(fn), mn, mx);
}

Sampling::Sampling(Server* server, std::shared_ptr<KeyDistribution> dist, const std::string& scheme, bool wr)
    : server_(server), dist_(dist), scheme_(scheme), with_replacement_(wr), mu_(server->num_workers()),
      samples_(server->num_workers()), id_counter_(server->num_workers(), 1), predrawn_(server->num_workers()),
      used_wor_(server->num_workers()) {
  ADAPM_CHECK(scheme == "naive" || scheme == "preloc" || scheme == "pool" || scheme == "local",
              "Unknown sampling scheme '" << scheme << "'");
  for (int w = 0; w < server->num_workers(); ++w)
    rng_.emplace_back((uint64_t)server->my_rank() * 7919u + (uint64_t)w * 104729u + 17u);
  pool_rng_.seed((uint64_t)server->my_rank() * 31u + 5u);
  if (scheme_ == "pool") {
    ADAPM_CHECK(server->options().sampling_pool_size > 0 && server->options().sampling_reuse > 0,
                "pool sampling needs sampling.pool_size > 0 and sampling.reuse > 0");
    ADAPM_CHECK(with_replacement_, "pool sampling supports only with-replacement sampling");
    pool_.resize(server->options().sampling_pool_size);
    pool_pos_ = pool_.size();
    pool_uses_ = server->options().sampling_reuse;
  }
}

void Sampling::draw(Key* out, size_t n, std::mt19937_64& rng) {
  if (with_replacement_) {
    for (size_t i = 0; i < n; ++i) out[i] = dist_->draw(rng);
  } else {
    std::unordered_set<Key> seen;
    size_t i = 0;
    size_t tries = 0;
    while (i < n) {
      Key k = dist_->draw(rng);
      if (seen.insert(k).second) out[i++] = k;
      ADAPM_CHECK(++tries < 1000 * (n + 10), "without-replacement sampling cannot find " << n << " distinct keys");
    }
  }
}

void Sampling::draw_from_pool(Key* out, size_t n) {
  std::lock_guard<std::mutex> lk(pool_mu_);
  for (size_t i = 0; i < n; ++i) {
    if (pool_pos_ >= pool_.size()) {
      ++pool_uses_;
      if (pool_uses_ < (size_t)server_->options().sampling_reuse) {
        std::shuffle(pool_.begin(), pool_.end(), pool_rng_);
      } else {
        for (auto& k : pool_) k = dist_->draw(pool_rng_);
        pool_uses_ = 0;
      }
      pool_pos_ = 0;
    }
    out[i] = pool_[pool_pos_++];
  }
}

SampleID Sampling::prepare_sample(size_t K, int worker, Clock start, Clock end) {
  std::lock_guard<std::mutex> lk(mu_[worker]);
  SampleID id = id_counter_[worker]++;
  if (scheme_ == "local") {
    if (!with_replacement_) used_wor_[worker].emplace(id, std::unordered_set<Key>());
    return id;
  }
  Sample s;
  s.K = K;
  s.keys.resize(K);
  if (scheme_ == "pool") draw_from_pool(s.keys.data(), K);
  else draw(s.keys.data(), K, rng_[worker]);
  if (scheme_ == "preloc" || scheme_ == "pool") {
    Worker* w = nullptr;
    {
      std::lock_guard<std::mutex> lk2(server_->mu_);
      w = server_->workers_[worker];
    }
    if (w) w->Intent(s.keys.data(), s.keys.size(), start, end);
  }
  samples_[worker].emplace(id, std::move(s));
  return id;
}

Key Sampling::next_local(int worker, Worker& w, void* vals, std::unordered_set<Key>* exclude) {
  auto& q = predrawn_[worker];
  auto refill = [&] {
    size_t b = (size_t)std::max<int64_t>(1, server_->options().sampling_batch_size);
    for (size_t z = 0; z < b; ++z) q.push_back(dist_->draw(rng_[worker]));
  };
  const bool ranged = dist_->max_key > dist_->min_key;
  uint64_t guard = 0;
  for (;;) {
    if (q.empty()) refill();
    Key k = q.front();
    q.pop_front();
    if (!ranged) {
      if (exclude && exclude->count(k)) continue;
      ++checks_;
      if (w.PullIfLocal(k, vals)) return k;
      ADAPM_CHECK(++guard < (1ull << 26), "local sampling cannot find a local key");
    } else {
      // memory-friendly variant: walk upward from the drawn key to the next resident key
      const Key mn = dist_->min_key, mx = dist_->max_key;
      for (Key steps = 0; steps <= (mx - mn); ++steps) {
        if (!(exclude && exclude->count(k))) {
          if (server_->is_local(k)) {
            ++checks_;
            if (w.PullIfLocal(k, vals)) return k;
          }
        }
        if (++k >= mx) k = mn;
      }
      ADAPM_CHECK(false, "local sampling: no (unused) local key in [" << mn << "," << mx << ")");
    }
  }
}

int Sampling::pull_sample(SampleID id, Key* keys, size_t n, void* vals, Worker& w) {
  const int worker = w.id();
  if (scheme_ == "local") {
    ++pulls_;
    std::unordered_set<Key>* excl = nullptr;
    if (!with_replacement_) {
      std::lock_guard<std::mutex> lk(mu_[worker]);
      auto it = used_wor_[worker].find(id);
      ADAPM_CHECK(it != used_wor_[worker].end(), "Invalid sample id " << server_->my_rank() << "::" << worker << "::" << id);
      excl = &it->second;
    }
    char* out = reinterpret_cast<char*>(vals);
    const size_t vb = server_->backend().ctx().L.val_bytes;
    for (size_t i = 0; i < n; ++i) {
      keys[i] = next_local(worker, w, out, excl);
      if (excl) excl->insert(keys[i]);
      out += server_->get_len(keys[i]) * vb;
    }
    return LOCAL;
  }
  {
    std::lock_guard<std::mutex> lk(mu_[worker]);
    auto it = samples_[worker].find(id);
    ADAPM_CHECK(it != samples_[worker].end(), "Invalid sample id " << server_->my_rank() << "::" << worker << "::" << id);
    Sample& s = it->second;
    ADAPM_CHECK(s.used + n <= s.K, "sample " << id << " has only " << (s.K - s.used) << " keys left, requested " << n);
    for (size_t i = 0; i < n; ++i) keys[i] = s.keys[s.used + i];
    s.used += n;
  }
  return w.Pull(keys, n, vals);
}

void Sampling::finish_sample(SampleID id, int worker) {
  std::lock_guard<std::mutex> lk(mu_[worker]);
  samples_[worker].erase(id);
  used_wor_[worker].erase(id);
}

}  // namespace adapm

#include "corpus.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <fstream>
#include <limits>
#include <stdexcept>
#include <string_view>
#include <unordered_map>

#include "log.h"

namespace adapm {

namespace {

inline bool is_space(char c) { return c == ' ' || c == '\n' || c == '\t' || c == '\r' || c == '\v' || c == '\f'; }

std::string read_file(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  ADAPM_CHECK(f.good(), "cannot open corpus file '" << path << "'");
  f.seekg(0, std::ios::end);
  const std::streamoff n = f.tellg();
  f.seekg(0, std::ios::beg);
  std::string s((size_t)n, '\0');
  f.read(&s[0], n);
  return s;
}

// calls fn(line_no, begin, end) for every line (without the terminator)
template <class F>
void for_each_line(const std::string& buf, F&& fn) {
  size_t b = 0;
  int64_t li = 0;
  const size_t n = buf.size();
  while (b < n) {
    size_t e = buf.find('\n', b);
    if (e == std::string::npos) e = n;
    fn(li++, b, e);
    b = e + 1;
  }
}

template <class F>
void for_each_word(const std::string& buf, size_t b, size_t e, F&& fn) {
  size_t i = b;
  while (i < e) {
    while (i < e && is_space(buf[i])) ++i;
    size_t j = i;
    while (j < e && !is_space(buf[j])) ++j;
    if (j > i) fn(std::string_view(buf.data() + i, j - i));
    i = j;
  }
}

// splitmix64 / xorshift: small, fast, reproducible across platforms
struct Rng {
  uint64_t s;
  explicit Rng(uint64_t seed) : s(seed ? seed : 0x9E3779B97F4A7C15ull) {}
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  double uniform() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
};

}  // namespace

struct Corpus::Index {
  std::unordered_map<std::string, int32_t> map;
};

std::shared_ptr<Corpus> Corpus::build(const std::string& path, int64_t min_count) {
  const std::string buf = read_file(path);
  struct Ent { int64_t count, first; };
  std::unordered_map<std::string_view, Ent> cnt;
  cnt.reserve(1 << 16);
  int64_t lines = 0, order = 0;
  for_each_line(buf, [&](int64_t, size_t b, size_t e) {
    ++lines;
    for_each_word(buf, b, e, [&](std::string_view w) {
      auto it = cnt.find(w);
      if (it == cnt.end()) cnt.emplace(w, Ent{1, order++});
      else ++it->second.count;
    });
  });
  std::vector<std::pair<std::string_view, Ent>> items;
  items.reserve(cnt.size());
  for (auto& p : cnt)
    if (p.second.count >= min_count) items.push_back(p);
  std::sort(items.begin(), items.end(), [](const auto& a, const auto& b) {
    if (a.second.count != b.second.count) return a.second.count > b.second.count;
    return a.second.first < b.second.first;   // ties: first occurrence first (a stable sort of the insertion order)
  });
  auto c = std::make_shared<Corpus>();
  c->words_.reserve(items.size() + 1);
  c->counts_.reserve(items.size() + 1);
  c->words_.push_back("</s>");
  c->counts_.push_back(std::max<int64_t>(1, lines));
  for (auto& p : items) {
    c->words_.emplace_back(p.first);
    c->counts_.push_back(p.second.count);
  }
  c->index_words();
  return c;
}

std::shared_ptr<Corpus> Corpus::from_vocab(std::vector<std::string> words, std::vector<int64_t> counts) {
  ADAPM_CHECK(words.size() == counts.size() && !words.empty(), "vocabulary: words and counts must have the same length");
  auto c = std::make_shared<Corpus>();
  c->words_ = std::move(words);
  c->counts_ = std::move(counts);
  c->index_words();
  return c;
}

void Corpus::index_words() {
  index_ = std::make_shared<Index>();
  index_->map.reserve(words_.size() * 2);
  for (size_t i = 0; i < words_.size(); ++i) index_->map.emplace(words_[i], (int32_t)i);
}

int64_t Corpus::lookup(const std::string& w) const {
  auto it = index_->map.find(w);
  return it == index_->map.end() ? -1 : it->second;
}

void Corpus::encode(const std::string& path, int rank, int world) {
  ADAPM_CHECK(world >= 1 && rank >= 0 && rank < world, "corpus: bad rank/world");
  const std::string buf = read_file(path);
  tokens_.clear();
  sent_off_.assign(1, 0);
  sent_line_.clear();
  num_lines_ = 0;
  std::string tmp;
  for_each_line(buf, [&](int64_t li, size_t b, size_t e) {
    num_lines_ = li + 1;
    if (li % world != rank) return;
    const size_t before = tokens_.size();
    for_each_word(buf, b, e, [&](std::string_view w) {
      tmp.assign(w.data(), w.size());
      auto it = index_->map.find(tmp);
      if (it != index_->map.end()) tokens_.push_back(it->second);
    });
    if (tokens_.size() > before) {
      sent_off_.push_back((int64_t)tokens_.size());
      sent_line_.push_back(li);
    }
  });
}

// ------------------------------------------------------------------------------------- batch streams
KeyBatchStream::KeyBatchStream(std::shared_ptr<Corpus> corpus, int window, double subsample, uint64_t seed,
                               int64_t batch_keys, int queue_depth)
    : corpus_(std::move(corpus)), window_(window), subsample_(subsample), seed_(seed), batch_keys_(batch_keys),
      key_space_(2 * corpus_->vocab_size()) {
  ADAPM_CHECK(window_ >= 1 && batch_keys_ >= 1 && queue_depth >= 1, "batch stream: bad window / batch size / queue depth");
  ring_.resize((size_t)queue_depth);
  for (auto& sl : ring_) sl.keys.resize((size_t)batch_keys_);
}

void KeyBatchStream::stop() {
  {
    std::lock_guard<std::mutex> lk(mu_);
    abort_ = true;
  }
  cv_put_.notify_all();
  cv_get_.notify_all();
  if (thread_.joinable()) thread_.join();
  abort_ = false;
}

void KeyBatchStream::start_epoch(uint64_t epoch) {
  stop();
  {
    std::lock_guard<std::mutex> lk(mu_);
    head_ = tail_ = count_ = 0;
    done_ = false;
  }
  thread_ = std::thread([this, epoch] { run(epoch); });
}

template <class F>
bool KeyBatchStream::walk(uint64_t epoch, F&& fn) {
  Rng rng(seed_ * 0x2545F4914F6CDD1Dull + epoch * 0x9E3779B97F4A7C15ull + 1);
  const int32_t* tok = corpus_->tokens();
  const int64_t* off = corpus_->sentence_offsets();
  const int64_t ns = corpus_->num_sentences();
  const std::vector<int64_t>& counts = corpus_->counts();
  double total = 0;
  for (int64_t c : counts) total += (double)c;
  // keep probability per word (word2vec.c rule): (sqrt(f / t) + 1) * t / f
  std::vector<float> keep;
  if (subsample_ > 0) {
    keep.resize(counts.size());
    for (size_t i = 0; i < counts.size(); ++i) {
      const double fr = (double)counts[i] / total;
      keep[i] = (float)((std::sqrt(fr / subsample_) + 1.0) * subsample_ / fr);
    }
  }
  std::vector<int32_t> s;
  for (int64_t si = 0; si < ns; ++si) {
    s.clear();
    for (int64_t t = off[si]; t < off[si + 1]; ++t) {
      const int32_t w = tok[t];
      if (subsample_ > 0 && keep[(size_t)w] < 1.f && rng.uniform() >= keep[(size_t)w]) continue;
      s.push_back(w);
    }
    const int64_t L = (int64_t)s.size();
    if (L < 2) continue;
    sentence_ = si;
    for (int64_t pos = 0; pos < L; ++pos) {
      const int64_t b = (int64_t)(rng.next() % (uint64_t)window_);   // window shrink in [0, window)
      const int64_t r = window_ - b;
      const int64_t lo = std::max<int64_t>(0, pos - r), hi = std::min<int64_t>(L, pos + r + 1);
      if (!fn(s, pos, lo, hi)) return false;
    }
  }
  return true;
}

bool KeyBatchStream::publish(std::vector<Key>& cur, int64_t valid) {
  // distinct keys of the batch (before taking the lock: this is the expensive part)
  if (seen_.empty()) seen_.assign((size_t)key_space_, 0u);
  if (++seen_epoch_ == 0) { std::fill(seen_.begin(), seen_.end(), 0u); seen_epoch_ = 1; }
  uniq_.clear();
  for (int64_t i = 0; i < batch_keys_; ++i) {
    const Key k = cur[(size_t)i];
    if (k >= 0 && seen_[(size_t)k] != seen_epoch_) { seen_[(size_t)k] = seen_epoch_; uniq_.push_back(k); }
  }
  std::unique_lock<std::mutex> lk(mu_);
  cv_put_.wait(lk, [&] { return count_ < ring_.size() || abort_; });
  if (abort_) return false;
  Slot& sl = ring_[tail_];
  sl.keys.swap(cur);
  sl.uniq.swap(uniq_);
  sl.valid = valid;
  tail_ = (tail_ + 1) % ring_.size();
  ++count_;
  produced_.fetch_add((uint64_t)valid);
  lk.unlock();
  cv_get_.notify_one();
  return true;
}

void KeyBatchStream::finish() {
  {
    std::lock_guard<std::mutex> lk(mu_);
    done_ = true;
  }
  cv_get_.notify_all();
}

int64_t KeyBatchStream::next_with_unique(Key* out, Key* uniq, int64_t* n_uniq) {
  std::unique_lock<std::mutex> lk(mu_);
  cv_get_.wait(lk, [&] { return count_ > 0 || done_ || abort_; });
  if (count_ == 0) return 0;
  Slot& sl = ring_[head_];
  const int64_t valid = sl.valid;
  lk.unlock();
  memcpy(out, sl.keys.data(), (size_t)batch_keys_ * sizeof(Key));   // the slot stays reserved while we copy
  if (uniq) {
    memcpy(uniq, sl.uniq.data(), sl.uniq.size() * sizeof(Key));
    *n_uniq = (int64_t)sl.uniq.size();
  }
  lk.lock();
  head_ = (head_ + 1) % ring_.size();
  --count_;
  lk.unlock();
  cv_put_.notify_one();
  return valid;
}

// ------------------------------------------------------------------------------------- pair stream
PairStream::PairStream(std::shared_ptr<Corpus> corpus, int window, double subsample, int64_t batch_pairs, uint64_t seed,
                       int queue_depth)
    : KeyBatchStream(std::move(corpus), window, subsample, seed, 2 * batch_pairs, queue_depth), batch_(batch_pairs) {
  ADAPM_CHECK(batch_ >= 1, "PairStream: bad window / batch size / queue depth");
}

PairStream::~PairStream() { stop(); }

void PairStream::run(uint64_t epoch) {
  std::vector<Key> cur((size_t)(2 * batch_));
  int64_t n = 0;
  auto publish_pairs = [&](int64_t valid) -> bool {
    if (valid < batch_) {   // pad a short last batch by repeating its pairs (fixed-size batches for the fused kernel)
      for (int64_t i = valid; i < batch_; ++i) {
        cur[(size_t)i] = cur[(size_t)(i % valid)];
        cur[(size_t)(batch_ + i)] = cur[(size_t)(batch_ + i % valid)];
      }
    }
    return publish(cur, valid);
  };
  const bool ok = walk(epoch, [&](const std::vector<int32_t>& s, int64_t pos, int64_t lo, int64_t hi) {
    const Key target = 2 * (Key)s[(size_t)pos] + 1;               // syn1 key of the centre word
    for (int64_t j = lo; j < hi; ++j) {
      if (j == pos) continue;
      cur[(size_t)n] = 2 * (Key)s[(size_t)j];                       // syn0 key of the context word
      cur[(size_t)(batch_ + n)] = target;
      if (++n == batch_) {
        n = 0;
        if (!publish_pairs(batch_)) return false;
      }
    }
    return true;
  });
  if (ok && n > 0) publish_pairs(n);
  finish();
}

int64_t PairStream::next(Key* out) { return next_with_unique(out, nullptr, nullptr); }

// ------------------------------------------------------------------------------------- window stream
WindowStream::WindowStream(std::shared_ptr<Corpus> corpus, int window, double subsample, int64_t batch_windows,
                           uint64_t seed, int queue_depth)
    : KeyBatchStream(std::move(corpus), window, subsample, seed, batch_windows * (1 + 2 * (int64_t)window), queue_depth),
      batch_(batch_windows) {
  ADAPM_CHECK(window >= 1 && window <= kMaxWindow, "WindowStream: window must be in [1, 16]");
}

WindowStream::~WindowStream() { stop(); }

void WindowStream::run(uint64_t epoch) {
  const int64_t cols = columns();
  std::vector<Key> cur((size_t)batch_keys_);
  int64_t n = 0;
  const bool ok = walk(epoch, [&](const std::vector<int32_t>& s, int64_t pos, int64_t lo, int64_t hi) {
    Key* r = cur.data() + n * cols;
    r[0] = 2 * (Key)s[(size_t)pos] + 1;                              // syn1 key of the centre word
    int64_t k = 1;
    for (int64_t j = lo; j < hi; ++j)
      if (j != pos) r[k++] = 2 * (Key)s[(size_t)j];                   // syn0 keys of the context words
    std::fill(r + k, r + cols, (Key)-1);
    if (++n == batch_) {
      n = 0;
      return publish(cur, batch_);
    }
    return true;
  });
  if (ok && n > 0) {         // pad a short last batch with windows that train nothing
    std::fill(cur.begin() + n * cols, cur.end(), (Key)-1);
    publish(cur, n);
  }
  finish();
}

// ------------------------------------------------------------------------------------- document streams
DocPairStream::DocPairStream(std::shared_ptr<Corpus> corpus, int window, double subsample, int64_t batch_pairs,
                             uint64_t seed, bool dbow_words, int queue_depth)
    : KeyBatchStream(std::move(corpus), window, subsample, seed, 2 * batch_pairs, queue_depth), batch_(batch_pairs),
      words_(dbow_words) {
  ADAPM_CHECK(batch_ >= 1, "DocPairStream: bad batch size");
  key_space_ = 2 * corpus_->vocab_size() + corpus_->num_lines();
}

DocPairStream::~DocPairStream() { stop(); }

void DocPairStream::run(uint64_t epoch) {
  std::vector<Key> cur((size_t)(2 * batch_));
  const int64_t* lines = corpus_->sentence_lines();
  const Key doc0 = 2 * (Key)corpus_->vocab_size();
  int64_t n = 0;
  auto publish_pairs = [&](int64_t valid) -> bool {
    for (int64_t i = valid; i < batch_; ++i) {   // pad a short last batch by repeating its pairs, as PairStream does
      cur[(size_t)i] = cur[(size_t)(i % valid)];
      cur[(size_t)(batch_ + i)] = cur[(size_t)(batch_ + i % valid)];
    }
    return publish(cur, valid);
  };
  auto emit = [&](Key input, Key target) -> bool {
    cur[(size_t)n] = input;
    cur[(size_t)(batch_ + n)] = target;
    if (++n < batch_) return true;
    n = 0;
    return publish_pairs(batch_);
  };
  const bool ok = walk(epoch, [&](const std::vector<int32_t>& s, int64_t pos, int64_t lo, int64_t hi) {
    const Key target = 2 * (Key)s[(size_t)pos] + 1;
    if (!emit(doc0 + lines[sentence_], target)) return false;
    if (words_)
      for (int64_t j = lo; j < hi; ++j)
        if (j != pos && !emit(2 * (Key)s[(size_t)j], target)) return false;
    return true;
  });
  if (ok && n > 0) publish_pairs(n);
  finish();
}

DocWindowStream::DocWindowStream(std::shared_ptr<Corpus> corpus, int window, double subsample, int64_t batch_windows,
                                 uint64_t seed, int queue_depth)
    : KeyBatchStream(std::move(corpus), window, subsample, seed, batch_windows * (2 + 2 * (int64_t)window), queue_depth),
      batch_(batch_windows) {
  ADAPM_CHECK(window >= 1 && window <= kMaxWindow, "DocWindowStream: window must be in [1, 15]");
  key_space_ = 2 * corpus_->vocab_size() + corpus_->num_lines();
}

DocWindowStream::~DocWindowStream() { stop(); }

void DocWindowStream::run(uint64_t epoch) {
  const int64_t cols = columns();
  const int64_t* lines = corpus_->sentence_lines();
  const Key doc0 = 2 * (Key)corpus_->vocab_size();
  std::vector<Key> cur((size_t)batch_keys_);
  int64_t n = 0;
  const bool ok = walk(epoch, [&](const std::vector<int32_t>& s, int64_t pos, int64_t lo, int64_t hi) {
    Key* r = cur.data() + n * cols;
    r[0] = 2 * (Key)s[(size_t)pos] + 1;
    r[1] = doc0 + lines[sentence_];
    int64_t k = 2;
    for (int64_t j = lo; j < hi; ++j)
      if (j != pos) r[k++] = 2 * (Key)s[(size_t)j];
    std::fill(r + k, r + cols, (Key)-1);
    if (++n == batch_) {
      n = 0;
      return publish(cur, batch_);
    }
    return true;
  });
  if (ok && n > 0) {
    std::fill(cur.begin() + n * cols, cur.end(), (Key)-1);
    publish(cur, n);
  }
  finish();
}

HuffmanTree huffman_tree(const double* counts, int64_t n) {
  if (n < 2) throw std::invalid_argument("huffman_tree: needs at least 2 words, got " + std::to_string(n));
  if (n > INT32_MAX / 2) throw std::invalid_argument("huffman_tree: too many words");
  for (int64_t w = 0; w < n; ++w)
    if (!(counts[w] > 0) || !std::isfinite(counts[w]))
      throw std::invalid_argument("huffman_tree: count of word " + std::to_string(w) + " is not a positive number");
  // leaf p < n is the word order[p] (count descending, ties by id); node n + a is the a-th merge (inner node a)
  std::vector<int32_t> order(n);
  for (int64_t w = 0; w < n; ++w) order[w] = (int32_t)w;
  std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return counts[a] > counts[b]; });
  std::vector<double> cnt(2 * n, std::numeric_limits<double>::infinity());
  for (int64_t p = 0; p < n; ++p) cnt[p] = counts[order[p]];
  std::vector<int32_t> parent(2 * n - 1, -1);
  std::vector<uint8_t> bit(2 * n - 1, 0);
  int64_t pos1 = n - 1, pos2 = n;     // the smallest unmerged leaf, the oldest unmerged inner node
  auto take = [&]() {
    if (pos1 >= 0 && cnt[pos1] < cnt[pos2]) return pos1--;
    return pos2++;
  };
  for (int64_t a = 0; a < n - 1; ++a) {
    const int64_t m1 = take(), m2 = take();
    cnt[n + a] = cnt[m1] + cnt[m2];
    parent[m1] = parent[m2] = (int32_t)(n + a);
    bit[m2] = 1;
  }
  // depths top-down: a parent is always created after its children
  std::vector<int32_t> depth(2 * n - 1, 0);
  for (int64_t v = 2 * n - 3; v >= 0; --v) depth[v] = depth[parent[v]] + 1;
  HuffmanTree t;
  t.offsets.assign(n + 1, 0);
  for (int64_t p = 0; p < n; ++p) t.max_len = std::max(t.max_len, depth[p]);
  if (t.max_len > kMaxHuffmanDepth)
    throw std::invalid_argument("huffman_tree: the tree is " + std::to_string(t.max_len) + " levels deep, more than " +
                                std::to_string(kMaxHuffmanDepth));
  for (int64_t p = 0; p < n; ++p) t.offsets[order[p] + 1] = depth[p];
  for (int64_t w = 0; w < n; ++w) t.offsets[w + 1] += t.offsets[w];
  t.nodes.resize(t.offsets[n]);
  t.codes.assign(n, 0u);
  for (int64_t p = 0; p < n; ++p) {
    const int32_t w = order[p];
    int64_t v = p;
    for (int j = depth[p] - 1; j >= 0; --j) {     // walk up: the node at depth j is v's parent
      t.nodes[t.offsets[w] + j] = (int32_t)(parent[v] - n);
      t.codes[w] |= (uint32_t)bit[v] << j;
      v = parent[v];
    }
  }
  return t;
}

}  // namespace adapm

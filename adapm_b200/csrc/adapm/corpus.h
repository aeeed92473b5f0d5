// Native data loader for the word2vec application: vocabulary building, corpus encoding and a background
// (center, context) pair generator that fills fixed-size key batches.
//
// Capability parity with the corpus handling of the reference application (apps/word2vec.cc:147-364 vocabulary hash /
// sort / min_count pruning, :563-606 reading sentences ahead, :672-690 window shrinking, frequent-word subsampling),
// re-shaped for a GPU consumer: a GPU trains 32 768 pairs in a few ms, i.e. the loader has to deliver millions of pairs/s per
// GPU, so batches are produced by a C++ thread into a bounded ring of buffers while the previous batches train.
#pragma once
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include "base.h"

namespace adapm {

class Corpus {
 public:
  // Pass 1: whitespace-tokenise `path`, count words, keep those with count >= min_count, order by count
  // (descending, ties by first occurrence). Word 0 is the sentence delimiter "</s>" (count = number of lines).
  static std::shared_ptr<Corpus> build(const std::string& path, int64_t min_count);
  // ... or adopt an existing vocabulary (vocab_retrieve)
  static std::shared_ptr<Corpus> from_vocab(std::vector<std::string> words, std::vector<int64_t> counts);

  // Pass 2: encode this rank's share of the file (line i belongs to rank i % world) as word ids.
  void encode(const std::string& path, int rank, int world);

  const std::vector<std::string>& words() const { return words_; }
  const std::vector<int64_t>& counts() const { return counts_; }
  int64_t vocab_size() const { return (int64_t)words_.size(); }
  int64_t num_tokens() const { return (int64_t)tokens_.size(); }
  int64_t num_sentences() const { return (int64_t)sent_off_.size() - 1; }
  const int32_t* tokens() const { return tokens_.data(); }
  const int64_t* sentence_offsets() const { return sent_off_.data(); }
  int64_t lookup(const std::string& w) const;   // -1 if unknown

 private:
  void index_words();
  std::vector<std::string> words_;
  std::vector<int64_t> counts_;
  std::vector<int32_t> tokens_;      // in-vocabulary word ids of this rank's sentences, concatenated
  std::vector<int64_t> sent_off_;    // sentence s = tokens_[sent_off_[s] .. sent_off_[s+1])
  struct Index;
  std::shared_ptr<Index> index_;
};

// Produces [2, batch_pairs] key batches (row 0: syn0 key of the context word = 2*w, row 1: syn1 key of the centre
// word = 2*w + 1) for one epoch over the encoded sentences, on a background thread.
class PairStream {
 public:
  PairStream(std::shared_ptr<Corpus> corpus, int window, double subsample, int64_t batch_pairs, uint64_t seed,
             int queue_depth = 8);
  ~PairStream();
  void start_epoch(uint64_t epoch);
  // Copies the next batch into out[2 * batch_pairs]; returns the number of valid pairs (a short last batch is padded
  // by repeating its pairs), 0 at the end of the epoch.
  int64_t next(Key* out);
  // Same, and also writes the distinct keys of the batch (what Intent() should be called with: the deduplication
  // happens here, on the loader thread, instead of on the sync thread) into uniq[0 .. *n_uniq); uniq holds 2*batch.
  int64_t next_with_unique(Key* out, Key* uniq, int64_t* n_uniq);
  int64_t batch_pairs() const { return batch_; }
  uint64_t pairs_produced() const { return produced_.load(); }

 private:
  void run(uint64_t epoch);
  void stop();
  struct Slot { std::vector<Key> keys, uniq; int64_t valid = 0; };
  std::vector<uint32_t> seen_;   // producer thread: round-stamped table for the per-batch deduplication
  uint32_t seen_epoch_ = 0;

  std::shared_ptr<Corpus> corpus_;
  int window_;
  double subsample_;
  int64_t batch_;
  uint64_t seed_;
  std::vector<Slot> ring_;
  size_t head_ = 0, tail_ = 0, count_ = 0;   // ring state (mu_)
  bool done_ = true, abort_ = false;
  std::mutex mu_;
  std::condition_variable cv_put_, cv_get_;
  std::thread thread_;
  std::atomic<uint64_t> produced_{0};
};

}  // namespace adapm

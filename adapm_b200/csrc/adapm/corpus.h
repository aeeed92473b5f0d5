// Native data loader for the word2vec application: vocabulary building, corpus encoding and background generators of
// fixed-size key batches: (center, context) pairs for skip-gram, windows for CBOW.
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

// Huffman coding of a vocabulary for hierarchical softmax, built like word2vec.c's CreateBinaryTree so that trees match
// word2vec.c and gensim for the same counts: words ordered by count (descending, ties by word id), the two-queue O(V)
// merge, inner nodes numbered 0 .. V-2 in creation order (the root is V-2), code bit 1 for the second-smallest child of
// each merge. Word w's path is nodes[offsets[w] .. offsets[w + 1]), root first, and bit j of codes[w] is its code bit
// at depth j. Throws std::invalid_argument for V < 2, a count that is not > 0, or a path longer than kMaxHuffmanDepth.
constexpr int kMaxHuffmanDepth = 32;
struct HuffmanTree {
  std::vector<int64_t> offsets;    // [V + 1]
  std::vector<int32_t> nodes;      // [sum of the path lengths]
  std::vector<uint32_t> codes;     // [V]
  int max_len = 0;
};
HuffmanTree huffman_tree(const double* counts, int64_t n);

class Corpus {
 public:
  // Pass 1: whitespace-tokenise `path`, count words, keep those with count >= min_count, order by count
  // (descending, ties by first occurrence). Word 0 is the sentence delimiter "</s>" (count = number of lines).
  static std::shared_ptr<Corpus> build(const std::string& path, int64_t min_count);
  // ... or adopt an existing vocabulary (vocab_retrieve)
  static std::shared_ptr<Corpus> from_vocab(std::vector<std::string> words, std::vector<int64_t> counts);

  // Pass 2: encode this rank's share of the file (line i belongs to rank i % world) as word ids. Lines without an
  // in-vocabulary word are skipped; sentence_lines() keeps the 0-based file line of every encoded sentence.
  void encode(const std::string& path, int rank, int world);

  const std::vector<std::string>& words() const { return words_; }
  const std::vector<int64_t>& counts() const { return counts_; }
  int64_t vocab_size() const { return (int64_t)words_.size(); }
  int64_t num_tokens() const { return (int64_t)tokens_.size(); }
  int64_t num_sentences() const { return (int64_t)sent_off_.size() - 1; }
  const int32_t* tokens() const { return tokens_.data(); }
  const int64_t* sentence_offsets() const { return sent_off_.data(); }
  const int64_t* sentence_lines() const { return sent_line_.data(); }
  int64_t num_lines() const { return num_lines_; }   // lines of the encoded file, every rank's
  int64_t lookup(const std::string& w) const;   // -1 if unknown

 private:
  void index_words();
  std::vector<std::string> words_;
  std::vector<int64_t> counts_;
  std::vector<int32_t> tokens_;      // in-vocabulary word ids of this rank's sentences, concatenated
  std::vector<int64_t> sent_off_;    // sentence s = tokens_[sent_off_[s] .. sent_off_[s+1])
  std::vector<int64_t> sent_line_;   // sentence s is line sent_line_[s] of the file
  int64_t num_lines_ = 0;
  struct Index;
  std::shared_ptr<Index> index_;
};

// Background producer of fixed-size key batches: a C++ thread fills a bounded ring of slots while the consumer trains
// on earlier batches. Each slot also carries the batch's distinct keys (what Intent() should be called with: the
// deduplication happens on the loader thread instead of the sync thread).
class KeyBatchStream {
 public:
  virtual ~KeyBatchStream() = default;
  void start_epoch(uint64_t epoch);
  // Copies the next batch into out[batch_keys]; returns its number of valid items (pairs or windows), 0 at the end of
  // the epoch. With uniq: also writes the batch's distinct keys (>= 0) into uniq[0 .. *n_uniq); uniq holds batch_keys.
  int64_t next_with_unique(Key* out, Key* uniq, int64_t* n_uniq);

 protected:
  KeyBatchStream(std::shared_ptr<Corpus> corpus, int window, double subsample, uint64_t seed, int64_t batch_keys,
                 int queue_depth);
  void stop();   // derived classes call it in their destructor: the thread runs their run()
  virtual void run(uint64_t epoch) = 0;
  // Walks this rank's sentences for one epoch with word2vec.c's frequent-word subsampling and window shrinking:
  // fn(s, pos, lo, hi) for every position pos of every subsampled sentence s with at least two words, whose context is
  // s[lo, hi) without pos. Returns false as soon as fn does.
  template <class F> bool walk(uint64_t epoch, F&& fn);
  // Publishes cur[0 .. batch_keys) (swapped out) with `valid` items; false if the stream was stopped.
  bool publish(std::vector<Key>& cur, int64_t valid);
  void finish();   // end of the epoch

  std::shared_ptr<Corpus> corpus_;
  int window_;
  double subsample_;
  uint64_t seed_;
  int64_t batch_keys_;
  int64_t key_space_;           // keys are < key_space_ (the deduplication table's size): 2 |V| unless a stream adds keys
  int64_t sentence_ = -1;       // inside walk()'s fn: the index of the sentence being walked
  std::atomic<uint64_t> produced_{0};

 private:
  struct Slot { std::vector<Key> keys, uniq; int64_t valid = 0; };
  std::vector<uint32_t> seen_;   // producer thread: round-stamped table for the per-batch deduplication
  uint32_t seen_epoch_ = 0;
  std::vector<Key> uniq_;
  std::vector<Slot> ring_;
  size_t head_ = 0, tail_ = 0, count_ = 0;   // ring state (mu_)
  bool done_ = true, abort_ = false;
  std::mutex mu_;
  std::condition_variable cv_put_, cv_get_;
  std::thread thread_;
};

// Produces [2, batch_pairs] key batches (row 0: syn0 key of the context word = 2*w, row 1: syn1 key of the centre
// word = 2*w + 1) for one epoch over the encoded sentences, on a background thread.
class PairStream : public KeyBatchStream {
 public:
  PairStream(std::shared_ptr<Corpus> corpus, int window, double subsample, int64_t batch_pairs, uint64_t seed,
             int queue_depth = 8);
  ~PairStream() override;
  // Copies the next batch into out[2 * batch_pairs]; returns the number of valid pairs (a short last batch is padded
  // by repeating its pairs), 0 at the end of the epoch.
  int64_t next(Key* out);
  int64_t batch_pairs() const { return batch_; }
  uint64_t pairs_produced() const { return produced_.load(); }

 private:
  void run(uint64_t epoch) override;
  int64_t batch_;
};

// Produces CBOW window batches [batch_windows, 1 + 2 * window]: column 0 the syn1 key of the centre word, then the syn0
// keys of its context words in sentence order, padded with -1. The rng draws (subsampling, window shrink) are
// PairStream's: for the same seed and epoch, expanding every window into (context, centre) pairs gives exactly the
// pairs of PairStream. A short last batch is padded with windows whose centre is -1. window <= 16.
class WindowStream : public KeyBatchStream {
 public:
  static constexpr int kMaxWindow = 16;
  WindowStream(std::shared_ptr<Corpus> corpus, int window, double subsample, int64_t batch_windows, uint64_t seed,
               int queue_depth = 8);
  ~WindowStream() override;
  int64_t batch_windows() const { return batch_; }
  int64_t columns() const { return 1 + 2 * (int64_t)window_; }
  uint64_t windows_produced() const { return produced_.load(); }

 private:
  void run(uint64_t epoch) override;
  int64_t batch_;
};

// Paragraph-vector (doc2vec) streams. Sentence s of the corpus is the document on file line l = sentence_lines()[s],
// whose key is 2 |V| + l. Both walk the corpus with PairStream's draws (subsampling and window shrink), so they relate
// to the word streams exactly:
//  - DocPairStream: [2, batch_pairs] pairs for PV-DBOW. For every walked position it emits (doc key, syn1 key of the
//    word) and then, with dbow_words, the position's skip-gram pairs in PairStream's order. Removing the document pairs
//    leaves PairStream's pairs. A short last batch is padded by repeating its pairs.
//  - DocWindowStream: [batch_windows, 2 + 2 window] windows for PV-DM: the centre's syn1 key, the doc key, then the
//    contexts as WindowStream lays them out. Removing column 1 leaves WindowStream's windows. window <= 15; a short
//    last batch is padded with windows whose centre is -1.
class DocPairStream : public KeyBatchStream {
 public:
  DocPairStream(std::shared_ptr<Corpus> corpus, int window, double subsample, int64_t batch_pairs, uint64_t seed,
                bool dbow_words, int queue_depth = 8);
  ~DocPairStream() override;
  int64_t batch_pairs() const { return batch_; }

 private:
  void run(uint64_t epoch) override;
  int64_t batch_;
  bool words_;
};

class DocWindowStream : public KeyBatchStream {
 public:
  static constexpr int kMaxWindow = 15;
  DocWindowStream(std::shared_ptr<Corpus> corpus, int window, double subsample, int64_t batch_windows, uint64_t seed,
                  int queue_depth = 8);
  ~DocWindowStream() override;
  int64_t batch_windows() const { return batch_; }
  int64_t columns() const { return 2 + 2 * (int64_t)window_; }

 private:
  void run(uint64_t epoch) override;
  int64_t batch_;
};

}  // namespace adapm

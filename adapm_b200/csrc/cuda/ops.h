// C++ entry points of the fused application kernels (implemented in ops_*.cu, bound to
// Python in ops_bind.cc).
#pragma once
#include <cstdint>
#include <vector>
#include "cuda_backend.h"

namespace adapm { class Worker; }

namespace adapm {
namespace cudaops {

// word2vec SGNS: fused pull + score + AdaGrad + push   (ops_sgns.cu)
// impl: 0 = auto, 1 = LDG variant (ops_sgns.cu), 2 = TMA-prefetch variant (ops_sgns_tma.cu)
void sgns_step(CudaBackend& be, cudaStream_t stream, const Key* centers, const Key* contexts, const Key* negatives,
               int n_pairs, int neg, int d, float alpha, float* loss_out, unsigned long long* stats, int impl = 0);
bool sgns_step_tma(CudaBackend& be, cudaStream_t stream, const Key* centers, const Key* contexts, const Key* negatives,
                   int n_pairs, int neg, int d, float alpha, float* loss_out, unsigned long long* stats);

// word2vec CBOW (ops_cbow.cu): one window per centre[i] with contexts[i * nc .. (i + 1) * nc) (syn0 keys, -1 = padding)
// and negatives[i * neg .. (i + 1) * neg) (syn1 keys); rows [embedding d | AdaGrad d]. d % 4 == 0, 4 <= d <= 336,
// 1 + neg <= 32, nc <= 32. deterministic (one GPU only): start-of-step reads, updates grouped by key and summed in fixed
// point (8 launches, the scan counted as two), bit-identical runs; else one kernel that adds the updates in place.
// stats: (local rows, remote rows, slow-path rows, updates), accumulated.
constexpr int kCbowMaxDim = 336;
constexpr int kCbowMaxTargets = 32;
constexpr int kCbowMaxContexts = 32;
void cbow_step(CudaBackend& be, cudaStream_t stream, const Key* centers, const Key* contexts, const Key* negatives,
               int n_win, int nc, int neg, int d, float alpha, float* loss_out, unsigned long long* stats,
               bool deterministic);

// word2vec SGNS with shared negatives on the tensor cores (ops_sgns_shared.cu): three wgmma GEMMs + three elementwise
// kernels between ONE Pull and ONE Push of the rows [centers | contexts | shared negatives].
size_t sgns_shared_workspace_bytes(int B, int Nn, int d);
void sgns_shared_core(cudaStream_t stream, const float* R, const Key* contexts, const Key* negs, int B, int Nn, int d,
                      float alpha, void* workspace, float* U, float* loss);

// key sampling (ops_sampler.cu). kind: 0 alias table, 1 uniform, 2 log-uniform
void sample_keys(CudaBackend& be, cudaStream_t stream, int kind, const float* prob, const int32_t* alias,
                 int64_t n_table, Key first, Key stride, Key* out, int64_t n, uint64_t seed, bool local_only,
                 int max_tries, unsigned long long* stats);

// Intent pre-pass (ops_intent.cu): extends the intent end clock of keys that already have a usable local slot on the
// device and writes the other keys to out_keys[0 .. *out_count) (out_count must be zero on entry).
void intent_prepass(CudaBackend& be, cudaStream_t stream, const Key* keys, int64_t n, Clock end, int worker, Key* out_keys,
                    unsigned int* out_count);

// deterministic = true (one GPU only): every call reads the state at the start of the step and the updates are summed
// in fixed point and applied once per row after the step (fx_accum.cuh), so the same inputs give the same rows and
// loss in every run; false: one kernel that adds the updates in place (default).
// knowledge-graph embeddings, ComplEx: fused pull + score + BCE/L2 gradient + AdaGrad + push (ops_kge.cu)
void kge_complex_step(CudaBackend& be, cudaStream_t stream, const Key* subj, const Key* rel, const Key* obj,
                      const float* labels, int n_calls, int nh, float eta, float gamma_e, float gamma_r, float* loss_out,
                      unsigned long long* stats, float dropout_e = 0.f, float dropout_r = 0.f, uint64_t seed = 0,
                      bool deterministic = false);
// RESCAL: fused pull + s^T R o + rank-1 relation gradient + AdaGrad + push (ops_kge.cu); relation rows are 2*D*D floats
void kge_rescal_step(CudaBackend& be, cudaStream_t stream, const Key* subj, const Key* rel, const Key* obj,
                     const float* labels, int n_calls, int D, float eta, float gamma_e, float gamma_r, float* loss_out,
                     unsigned long long* stats, float dropout_e = 0.f, float dropout_r = 0.f, uint64_t seed = 0,
                     bool deterministic = false);

// TransE: fused pull + L1/L2 distance + margin-ranking gradient + AdaGrad + push (ops_transe.cu). One positive triple
// per (subj[i], rel[i], obj[i]) with neg[i * n_neg .. (i + 1) * n_neg) entity keys: the first half replaces the object,
// the second the subject. Entity and relation rows are [embedding (d) | AdaGrad (d)], d % 4 == 0, 4 <= d <= 512;
// entity rows are normalised on read. p = 1 or 2, n_neg <= 64. stats[3] counts the pushes issued.
constexpr int kTransEMaxDim = 512;
constexpr int kTransEMaxNeg = 64;
void kge_transe_step(CudaBackend& be, cudaStream_t stream, const Key* subj, const Key* rel, const Key* obj,
                     const Key* neg, int B, int n_neg, int d, int p, float margin, float eta, float gamma_e,
                     float gamma_r, float* loss_out, unsigned long long* stats, bool deterministic = false);

// RotatE: fused pull + complex rotation + sigmoid loss with self-adversarial negative weights + AdaGrad + push
// (ops_rotate.cu). Triples and negatives as for TransE. Entity rows are [z (d) | AdaGrad (d)] with z interleaved
// (re, im), relation rows [phases (d / 2) | AdaGrad (d / 2)]; d % 8 == 0, 8 <= d <= 512, 2 <= n_neg <= 256.
// stats[3] counts the pushes issued (3 + n_neg per triple).
constexpr int kRotatEMaxDim = 512;
constexpr int kRotatEMaxNeg = 256;
void kge_rotate_step(CudaBackend& be, cudaStream_t stream, const Key* subj, const Key* rel, const Key* obj,
                     const Key* neg, int B, int n_neg, int d, float margin, float alpha, float eta, float gamma_e,
                     float* loss_out, unsigned long long* stats, bool deterministic = false);

// matrix factorisation: fused pull + error + L2 + AdaGrad + push (ops_mf.cu)
void mf_step(CudaBackend& be, cudaStream_t stream, const Key* row_keys, const Key* col_keys, const float* xs,
             const int* row_nnz, const int* col_nnz, int n, int rank, float eps, float lambda, float* loss_out,
             unsigned long long* stats, bool deterministic = false);

// implicit-feedback matrix factorisation: fused pull + BPR loss over sampled negatives + L2 + AdaGrad + push
// (ops_bpr.cu). One positive (users[i], pos[i]) per i with neg[i * n_neg .. (i + 1) * n_neg) item keys; rows
// [factors (rank) | AdaGrad (rank)], rank % 4 == 0, 4 <= rank <= 512, 1 <= n_neg <= 256. stats[3] counts the pushes
// issued (2 + n_neg per positive).
constexpr int kBprMaxRank = 512;
constexpr int kBprMaxNeg = 256;
void mf_bpr_step(CudaBackend& be, cudaStream_t stream, const Key* users, const Key* pos, const Key* neg, int B, int n_neg,
                 int rank, float eps, float lam, float* loss_out, unsigned long long* stats, bool deterministic = false);

// alternating least squares for matrix factorisation (ops_als.cu). Target targets[t] (distinct) has the entries
// others[offsets[t] .. offsets[t + 1]) with weights a, b; rows [factors (rank) | AdaGrad (rank)], rank % 4 == 0,
// 4 <= rank <= 128. One CTA per target, in the given order: A = gram + lam I + sum_e a_e h_e h_e^T, r = sum_e b_e h_e,
// w <- A^{-1} r pushed as [w_new - w_old | 0]; a pivot <= 0 leaves the target unchanged. gram: [rank, rank] or null.
// stats: (other rows local, other rows from peers, slow-path rows, rows solved), accumulated. 1 launch.
constexpr int kAlsMaxRank = 128;
void als_solve(CudaBackend& be, cudaStream_t stream, const Key* targets, const int64_t* offsets, const Key* others,
               const float* a, const float* b, int n, int rank, float lam, const float* gram, unsigned long long* stats);
// G[rank, rank] = sum over keys[0 .. n) of h h^T (factor halves): partials of 1024 keys added in index order,
// bit-identical from call to call and wherever the rows live. 2 launches.
void als_gram(CudaBackend& be, cudaStream_t stream, const Key* keys, int64_t n, int rank, float* G);

// wgmma/TMA GEMM: C[M,N] fp32 = A[M,K] bf16 x B[N,K]^T bf16 (ops_gemm_wgmma.cu)
void gemm_nt_bf16(cudaStream_t stream, const void* A, const void* B, int M, int N, int K, float* C, int ldc);
void gemm_nt_e4m3(cudaStream_t stream, const void* A, const void* B, int M, int N, int K, float* C, int ldc, float alpha);
// same GEMM with the ranking epilogue: rank_out[row] += #{col != true_col[row] : score > true_score[row]}
void gemm_nt_bf16_rank_count(cudaStream_t stream, const void* A, const void* B, int M, int N, int K,
                             const float* true_score, const int* true_col, int* rank_out);

// fused gather (local HBM / NVLink peers, through the directory) + wgmma GEMM (ops_gather_gemm.cu):
// C[M,N] = Q[M,K] (bf16, row pitch ldq) x rows(keys[0..N))[0..K)^T, rows read from the parameter store
void gather_gemm(CudaBackend& be, cudaStream_t stream, const void* Q, const Key* keys, int M, int N, int K, int ldq, float* C,
                 int ldc, unsigned long long* stats);
void gather_gemm_rank_count(CudaBackend& be, cudaStream_t stream, const void* Q, const Key* keys, int M, int N, int K, int ldq,
                            const float* true_score, const int* true_col, int* rank_out, unsigned long long* stats);

// top-k retrieval on the tensor cores (ops_topk.cu): per query row the k best columns of Q x E^T (fp32 wgmma scores,
// times col_scale[j] when given; score descending, ties to the smaller column; columns in the row's CSR exclusion list
// ex_cols[ex_off[i] .. ex_off[i+1]) skipped; (-inf, -1) padding). The tile kernels write sorted partial lists of S
// N-slices into part_v / part_c [M, S, k]; a merge kernel writes out_v [M, k] and out_i [M, k].
constexpr int kTopkMax = 64;
int topk_num_slices(int M, int N, int max_tiles_per_cta);   // S for the grid; max_tiles_per_cta <= 0: unbounded
void gemm_nt_topk(cudaStream_t stream, const void* A, const void* B, int M, int N, int K, int k, int S,
                  const float* col_scale, const int64_t* ex_off, const int64_t* ex_cols, float* part_v, int* part_c,
                  float* out_v, int64_t* out_i);
// the same with E = rows(keys[0..N))[0..K) gathered from the parameter store (as gather_gemm); out_i are positions in keys
void gather_gemm_topk(CudaBackend& be, cudaStream_t stream, const void* Q, const Key* keys, int M, int N, int K, int ldq,
                      int k, int S, const float* col_scale, const int64_t* ex_off, const int64_t* ex_cols, float* part_v,
                      int* part_c, float* out_v, int64_t* out_i, unsigned long long* stats);
// merges S sorted partial lists per row (part_v / part_c [M, S, k], column -1 = padding) into out_v / out_i [M, k]
// with the order above
void topk_merge(cudaStream_t stream, const float* part_v, const int* part_c, int M, int S, int k, float* out_v,
                int64_t* out_i);

// distance ranking and top-k against parameter-store rows on the CUDA cores (ops_dist.cu): D(i, j) = |q_i - e_j|_p,
// p = 1 or 2, e_j = the first dim values of store row keys[j] (dim % 4 == 0), divided by max(|e_j|_2, 1e-12) when
// normalize; p = kDistComplex: the sum of complex moduli sum_k |(q - e)_{2k} + i (q - e)_{2k+1}| (never normalised);
// each distance is an fp32 sum over the dim elements in order, bit-identical whichever CTA computes it.
// Grid (M / 64 tiles) x S column slices. stats: (local rows, peer rows, rows that could not be resolved), accumulated.
constexpr int kDistComplex = 3;
int dist_num_slices(CudaBackend& be, int M, int N, int max_tiles_per_cta);   // max_tiles_per_cta <= 0: unbounded
// dtrue[i] = D(i, true_col[i]); raw[i] += #{j != true_col[i] : D(i, j) < dtrue[i]}; filt[i] the same without the
// columns ex_cols[ex_off[i] .. ex_off[i + 1]) (raw, filt zeroed by the caller). 2 launches.
void gather_dist_rank_count(CudaBackend& be, cudaStream_t stream, const float* q, const Key* keys, int M, int N, int dim,
                            int p, bool normalize, int S, const int64_t* true_col, const int64_t* ex_off,
                            const int64_t* ex_cols, float* dtrue, int64_t* raw, int64_t* filt,
                            unsigned long long* stats);
// per row the k (<= 64) columns of smallest distance: out_v = -D, out_i = column; ties to the smaller column, NaN never
// selected, (-inf, -1) padding; exclusions as above. 2 launches (tiles, merge).
void gather_dist_topk(CudaBackend& be, cudaStream_t stream, const float* q, const Key* keys, int M, int N, int dim, int p,
                      bool normalize, int k, int S, const int64_t* ex_off, const int64_t* ex_cols, float* part_v,
                      int* part_c, float* out_v, int64_t* out_i, unsigned long long* stats);

// multi-hot embedding bags over rows [embedding (E) | AdaGrad (E)] (ops_embbag.cu). CSR bags: keys[nnz],
// offsets[nbags + 1], optional weights[nnz]; mean: divide by the bag length. stats: int64[5] accumulated with (local
// rows, peer rows, slow-path rows, rows updated, rows that could not be resolved).
// forward (1 launch): out[nbags, E] = pooled rows, each bag summed in fp32 in key order.
// backward (4 launches, the radix sort counted as one): G_k = grad_scale * sum over the occurrences of k of
// c_i * grad_out[bag(i)] in position order, then push [-lr G / sqrt(acc + G^2) | G^2] once per distinct key.
constexpr int kEmbBagMaxDim = 512;
size_t embedding_bag_workspace_bytes(int64_t nnz, int64_t nbags, int E);
void embedding_bag_forward(CudaBackend& be, cudaStream_t stream, const Key* keys, const int64_t* offsets,
                           const float* weights, int64_t nnz, int nbags, int E, bool mean, float* out,
                           unsigned long long* stats);
void embedding_bag_backward(CudaBackend& be, cudaStream_t stream, const Key* keys, const int64_t* offsets,
                            const float* weights, int64_t nnz, int nbags, int E, bool mean, const float* grad_out,
                            float lr, float grad_scale, void* workspace, size_t workspace_bytes,
                            unsigned long long* stats);

// Native step driver of the word2vec SGNS loop (ops_train_loop.cu)
struct SgnsLoopConfig {
  int batch_pairs = 0, negative = 0, embed_dim = 0, read_ahead = 0, max_inflight = 3, rank = 0;
  bool signal_intent = true, local_only = false;
  int64_t model_seed = 0;
  int sampler_kind = 0;
  const float* prob = nullptr;
  const int32_t* alias = nullptr;
  int64_t n_table = 0;
  Key first_key = 0, key_stride = 1;
  unsigned long long* sampler_stats = nullptr;
};
class SgnsLoop {
 public:
  SgnsLoop(Worker* worker, CudaBackend* be, const SgnsLoopConfig& cfg);
  ~SgnsLoop();
  void run(cudaStream_t stream, int64_t first, int64_t n, bool resident, const std::vector<uintptr_t>& batches,
           const std::vector<uintptr_t>& intent_keys, const std::vector<int64_t>& intent_counts, float* loss_dev,
           float* loss_host, unsigned long long* stats, int64_t step_no0, float alpha);

 private:
  Worker* w_;
  CudaBackend* be_;
  SgnsLoopConfig c_;
  int depth_ = 0;
  std::vector<Key*> key_bufs_;
  std::vector<cudaEvent_t> copied_, done_;
  std::vector<bool> done_valid_;
  Key* neg_ = nullptr;
  cudaStream_t copy_stream_ = nullptr;
};

}  // namespace cudaops
}  // namespace adapm

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
// word2vec hierarchical softmax (ops_cbow.cu, the CBOW body with Huffman-path targets): item i has the syn1 key
// centers[i] = 2w + 1 (< 0: nothing) and the syn0 contexts[i * nc .. (i + 1) * nc) (-1 = padding); its targets are the
// inner nodes nodes[offsets[w] .. offsets[w + 1]) of word w's path (rows 2 node + 1), labelled 1 - bit j of codes[w];
// a node with |f| >= 6 is skipped. Shapes, stats and the two paths as for cbow_step; max_len (the longest path) <= 32.
void hs_step(CudaBackend& be, cudaStream_t stream, const Key* centers, const Key* contexts, int n_items, int nc,
             const int64_t* offsets, const int32_t* nodes, const uint32_t* codes, int n_words, int max_len, int d,
             float alpha, float* loss_out, unsigned long long* stats, bool deterministic);

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

// KGE 1vsAll training for ComplEx (model 0) and RESCAL (model 1) on pulled rows (ops_kge_1vsall.cu): every query
// (s, r, ?) and (?, r, o) of the B triples against all N entities with a softmax cross-entropy loss. R: the pulled rows
// [N entity rows (2 d) | nrel relation rows (2 d or 2 d d)]; s, o: entity ids, rel: the triple's relation as an index
// into the pulled relations; ent_off [N + 1] / ent_pos: per entity, the positions p (2 i: subject of triple i, 2 i + 1:
// object) in ascending order; rel_off [nrel + 1] / rel_pos: per pulled relation, its triples in ascending order.
// U: the additive updates [-eta g / sqrt(a + g^2) | g^2] of every pulled row, for one Push. Queries run in chunks of
// `chunk` (a multiple of 128) rows; the workspace holds kge_1vsall_workspace_bytes(...). No floating-point atomics: on
// one GPU the same inputs give bit-identical updates and loss. *loss += sum of the 2 B cross-entropies.
constexpr int kKge1vsAllMaxDim = 1024;
size_t kge_1vsall_workspace_bytes(int N, int B, int d, int chunk);
void kge_1vsall_core(cudaStream_t stream, int model, const float* R, const Key* s, const Key* o, const int32_t* rel,
                     const int64_t* ent_off, const int32_t* ent_pos, const int64_t* rel_off, const int32_t* rel_pos,
                     int N, int nrel, int B, int d, int chunk, float eta, float gamma_e, float gamma_r, void* workspace,
                     float* U, float* loss);

// KGE sampled-softmax training for ComplEx and RESCAL on pulled rows (ops_kge_1vsall.cu): the B triples in chunks of
// kKgeSharedChunk; chunk k scores its object queries (s, r, ?) and subject queries (?, r, o) against one list
// [its subjects | its objects | the S shared negatives] with a softmax cross-entropy. R: the pulled rows [Ne entity rows
// (2 d) | nrel relation rows]; s, o, rel: [Bp] indices into them, Bp = B padded to whole chunks (padding triples are
// masked out of the loss and left out of every CSR); cand [nch][Lr]: the lists as entity indices, -1 for padding slots,
// Lr = 2 * 128 + S padded to a multiple of 8; qorder [nch][2 * 128]: the queries of chunk k, object queries first, as
// indices q < 2 Bp (object query of triple i: i, subject query: Bp + i). ent_off [Ne + 1] / ent_pos: per entity, its
// occurrences in ascending order, p < nch * Lr the list column k * Lr + j, else the given entity of position
// p - nch * Lr (2 i: subject of triple i, 2 i + 1: object); rel_off / rel_pos as in kge_1vsall_core. U: one AdaGrad
// update per pulled row. No floating-point atomics. *loss += the 2 B cross-entropies.
constexpr int kKgeSharedChunk = 128;
size_t kge_shared_workspace_bytes(int B, int S, int d);
void kge_shared_core(cudaStream_t stream, int model, const float* R, const Key* s, const Key* o, const int32_t* rel,
                     const Key* cand, const Key* qorder, const int64_t* ent_off, const int32_t* ent_pos,
                     const int64_t* rel_off, const int32_t* rel_pos, int Ne, int nrel, int B, int S, int d, float eta,
                     float gamma_e, float gamma_r, void* workspace, float* U, float* loss);

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

// GloVe: fused pull + weighted least squares + AdaGrad + push (ops_glove.cu). One non-zero (words[i], ctxs[i], xs[i])
// per i: the keys of a word row and a context row, X > 0. Rows [vector (d) | bias, 0, 0, 0 | AdaGrad (d + 4)],
// d % 4 == 0, 4 <= d <= 508. stats[3] counts the pushes issued (2 per non-zero).
constexpr int kGloveMaxDim = 508;
void glove_step(CudaBackend& be, cudaStream_t stream, const Key* words, const Key* ctxs, const float* xs, int n, int d,
                float eta, float x_max, float alpha, float* loss_out, unsigned long long* stats,
                bool deterministic = false);

// GloVe co-occurrence counts of an encoded corpus on the device (ops_cooc.cu): tokens[0 .. n_tokens) int32 word ids in
// [0, V), sentence s = tokens[offsets[s] .. offsets[s + 1]). For every pair of positions of one sentence where word a
// comes k <= window positions before word b, X[a][b] += 1 / k (1 without distance weighting), and with symmetric also
// X[b][a]; only rows a with a % world == rank are kept. Sums are exact: integer numerators over lcm(1..window) in 64
// bits, divided once at the end. Processed in token chunks so that the device memory of the call stays within
// max_bytes; run() returns the number of non-zeros, write() stores them sorted by (row, col).
constexpr int kCoocMaxWindow = 16;
class Cooccurrence {
 public:
  Cooccurrence(cudaStream_t stream, const int32_t* tokens, int64_t n_tokens, const int64_t* offsets, int64_t n_sentences,
               int64_t V, int window, bool symmetric, bool distance_weighting, int rank, int world, int64_t max_bytes);
  ~Cooccurrence();
  int64_t run();
  void write(int32_t* rows, int32_t* cols, float* x) const;
  int chunks() const { return chunks_; }
  int64_t denominator() const { return lw_; }

 private:
  struct Impl;
  Impl* impl_;
  int chunks_ = 0;
  int64_t lw_ = 1;
};

// paragraph-vector (doc2vec) inference (ops_doc2vec.cu; the rule is in its header): one epoch e of the documents
// tokens[offsets[m] .. offsets[m + 1]) (word ids) with ids doc_ids[m], each trained on its own row of state [M, 2 d]
// (embedding | AdaGrad; written at e = 0, read and written after) against the read-only store rows; negatives drawn by
// the sampler table (kind, prob, alias, n_table, first, stride) as ops_sampler.cu draws them. loss (may be null) +=
// the summed logistic loss; stats[2] += rows that could not be resolved. Limits: d a multiple of 4 in [4, 336],
// 1 <= negative <= 31, PV-DM window in [1, 15]. One launch.
constexpr int kDoc2VecMaxDim = 336;
constexpr int kDoc2VecMaxTargets = 32;
constexpr int kDoc2VecMaxWindow = 15;
constexpr int kDoc2VecMaxWords = 10000;
void doc2vec_infer_epoch(CudaBackend& be, cudaStream_t stream, const int64_t* tokens, const int64_t* offsets,
                         const int64_t* doc_ids, int64_t M, bool dm, int d, int negative, int window, int epoch,
                         float alpha, uint64_t seed, int kind, const float* prob, const int32_t* alias, int64_t n_table,
                         Key first, Key stride, float* state, float* loss, unsigned long long* stats);

// node2vec / DeepWalk random walks on a CSR graph (ops_walk.cu; the rule is in its header): walk w starts at
// starts[w] and is numbered walk_nos[w]; out [n_walks, L] int64, -1 after a node without out-edges. cumw: the inclusive
// prefix sums of the quantised weights per node (null: unweighted). second_order: rejection sampling with the 24-bit
// acceptance thresholds of alpha = 1 / p (return), 1 (x in N(t)) and 1 / q (outward); else first order. 1 launch.
void node2vec_walks(cudaStream_t stream, const int64_t* offsets, const int32_t* nbrs, const int64_t* cumw,
                    const int64_t* starts, const int64_t* walk_nos, int64_t n_walks, int L, uint64_t seed,
                    uint64_t epoch, uint32_t thr_return, uint32_t thr_in, uint32_t thr_out, bool second_order,
                    int64_t* out);
// skip-gram pairs of walks [n_walks, L] (ops_walk.cu): walk_pair_ends writes each position's pair count to counts
// and their inclusive scan to ends (cub, temp of walk_pair_scan_bytes(n_walks * L) bytes; 2 launches);
// walk_pairs_write then stores the ends[last] pairs as out [2, n_pairs] (1 launch).
size_t walk_pair_scan_bytes(int64_t n_items);
void walk_pair_ends(cudaStream_t stream, const int64_t* walks, int64_t n_walks, int L, int window, uint64_t seed,
                    int64_t* counts, int64_t* ends, void* temp, size_t temp_bytes);
void walk_pairs_write(cudaStream_t stream, const int64_t* walks, int64_t n_walks, int L, int window, uint64_t seed,
                      const int64_t* ends, int64_t n_pairs, Key* out);

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
// DLRM dot interaction (ops_dlrm.cu), fp32, one launch each way. z [B, E], e [B, F, E] (the pooled bags in place),
// R [B, W] with W = E + F (F + 1) / 2 rounded up to 8: R = [z | <T_i, T_j> for j < i, row-major | 0] where
// T = [z; e_0 .. e_{F-1}]. backward: dz = dR[:, :E] + dT_0, de_f = dT_{f+1} with dT_i = sum_{j != i} dZ_ij T_j.
// 1 <= F, F + 1 <= 64, E % 4 == 0 in [4, 512], B * W < 2^31; 16-byte aligned pointers. Bit-identical reruns.
constexpr int kDlrmMaxRows = 64;
constexpr int kDlrmMaxDim = 512;
void dlrm_interaction_forward(cudaStream_t stream, const float* z, const float* e, int64_t B, int F, int E, int W,
                              float* R);
void dlrm_interaction_backward(cudaStream_t stream, const float* dR, const float* z, const float* e, int64_t B, int F,
                               int E, int W, float* dz, float* de);

// DCN-v2 low-rank cross network (ops_dcn.cu): x_{l+1} = x_0 * (W_l (V_l x_l) + b_l) + x_l, x_0 = [z | e] [B, N] from
// z [B, E] and e [B, F, E] (N = (F + 1) E); V [L, r, N], W [L, N, r] (and the backward's Vt [L, N, r], Wt [L, r, N]) bf16,
// b [L, N] fp32. N % 8 == 0, r % 8 == 0, 8 <= r <= 1024, 1 <= L <= 8, B * N < 2^31. Transposed buffers [*, pitch] have
// pitch = B rounded up to 8. forward (1 + 2 L launches): x [B, N] fp32 = x_L; xb [B, N], hb [B, r] bf16 scratch; when
// training (xt non-null) also xt [L, N, pitch] = x_l^T, ht [L, r, pitch] = h_l^T and ub [L, B, N] = u_l in bf16 for the
// backward. backward: grad_out [B, N]; G, dx0 [B, N] fp32, Pb [B, N], Pt [N, pitch], dh [B, r], dht [r, pitch] bf16 and
// ws (dcn_workspace_floats) scratch; writes dz, de, dV [L, r, N], dW [L, N, r], db [L, N]. No floating-point atomics:
// bit-identical reruns on one GPU.
constexpr int kDcnMaxLayers = 8;
constexpr int kDcnMinRank = 8;
constexpr int kDcnMaxRank = 1024;
size_t dcn_workspace_floats(int B, int N, int r);
void dcn_forward(cudaStream_t stream, const float* z, const float* e, int B, int E, int N, int r, int L, const void* V,
                 const void* W, const float* b, void* xb, void* hb, float* x, void* xt, void* ht, void* ub);
void dcn_backward(cudaStream_t stream, const float* z, const float* e, int B, int E, int N, int r, int L, const void* Vt,
                  const void* Wt, const void* xt, const void* ht, const void* ub, const float* grad_out, float* G,
                  float* dx0, void* Pb, void* Pt, void* dh, void* dht, float* ws, float* dz, float* de, float* dV,
                  float* dW, float* db);

constexpr int kEmbBagMaxDim = 512;
size_t embedding_bag_workspace_bytes(int64_t nnz, int E);
void embedding_bag_forward(CudaBackend& be, cudaStream_t stream, const Key* keys, const int64_t* offsets,
                           const float* weights, int64_t nnz, int nbags, int E, bool mean, float* out,
                           unsigned long long* stats);
void embedding_bag_backward(CudaBackend& be, cudaStream_t stream, const Key* keys, const int64_t* offsets,
                            const float* weights, int64_t nnz, int nbags, int E, bool mean, const float* grad_out,
                            float lr, float grad_scale, void* workspace, size_t workspace_bytes,
                            unsigned long long* stats);

// field-aware factorisation machines (ops_ffm.cu) over rows [w, 0, 0, 0 | V_0 .. V_{F-1} (k each) | AdaGrad], E =
// 4 + F k values: ids [B, F] (the field of ids[b, f] is f), labels [B]; 2 <= F <= 64, k a multiple of 4 in [4, 32],
// F k <= 512, B F < 2^31. stats: int64[5] accumulated with (local rows, peer rows, slow-path rows, rows updated, rows
// that could not be resolved).
// forward (1 launch): logits[b] = phi_b = sum_f w[x_bf] + r sum_{f1<f2} <V[x_bf1][f2], V[x_bf2][f1]>.
// step (5 launches, the radix sort counted as one): phi from the rows at the start of the step; per distinct key the
// sum over its occurrences (b, f), in position order, of [kappa_b + lam w | 0 | kappa_b r V[x_b,f2][f] + lam V_f2 for
// f2 != f], kappa_b = sigmoid(phi_b) - y_b, pushed once as [-eta G / sqrt(acc + G^2) | G^2]; *loss = sum_b
// softplus(phi_b) - y_b phi_b.
constexpr int kFfmMaxFields = 64;
constexpr int kFfmMaxK = 32;
constexpr int kFfmMaxFk = 512;
size_t ffm_workspace_bytes(int B, int F, int k);
void ffm_forward(CudaBackend& be, cudaStream_t stream, const Key* ids, int B, int F, int k, float r, float* logits,
                 unsigned long long* stats);
void ffm_step(CudaBackend& be, cudaStream_t stream, const Key* ids, const float* labels, int B, int F, int k, float r,
              float eta, float lam, void* workspace, size_t workspace_bytes, float* loss, unsigned long long* stats);

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

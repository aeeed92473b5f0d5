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

// matrix factorisation: fused pull + error + L2 + AdaGrad + push (ops_mf.cu)
void mf_step(CudaBackend& be, cudaStream_t stream, const Key* row_keys, const Key* col_keys, const float* xs,
             const int* row_nnz, const int* col_nnz, int n, int rank, float eps, float lambda, float* loss_out,
             unsigned long long* stats, bool deterministic = false);

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

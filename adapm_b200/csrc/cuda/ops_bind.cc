// Python bindings of the fused application kernels. Tensors are passed as raw device
// addresses (see adapm_b200/ops/__init__.py for the torch-facing wrappers).
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include "ops.h"

namespace py = pybind11;

namespace adapm {
namespace cudaops {

namespace {
template <class T> T* ptr(uintptr_t a) { return reinterpret_cast<T*>(a); }
CudaBackend& backend_of(uintptr_t handle) {
  Backend* b = reinterpret_cast<Backend*>(handle);
  ADAPM_CHECK(b && b->is_cuda(), "this op needs a server with backend='cuda'");
  return *static_cast<CudaBackend*>(b);
}
}  // namespace

void bind(py::module_& m) {
  m.def("sgns_step", [](uintptr_t be, uintptr_t stream, uintptr_t centers, uintptr_t contexts, uintptr_t negatives,
                        int n_pairs, int neg, int d, float alpha, uintptr_t loss, uintptr_t stats, int impl) {
    sgns_step(backend_of(be), (cudaStream_t)stream, ptr<const Key>(centers), ptr<const Key>(contexts),
              ptr<const Key>(negatives), n_pairs, neg, d, alpha, ptr<float>(loss), ptr<unsigned long long>(stats), impl);
  });
  m.attr("cbow_max_dim") = kCbowMaxDim;
  m.attr("cbow_max_targets") = kCbowMaxTargets;
  m.attr("cbow_max_contexts") = kCbowMaxContexts;
  m.def("cbow_step", [](uintptr_t be, uintptr_t stream, uintptr_t centers, uintptr_t contexts, uintptr_t negatives,
                        int n_win, int nc, int neg, int d, float alpha, uintptr_t loss, uintptr_t stats,
                        bool deterministic) {
    cbow_step(backend_of(be), (cudaStream_t)stream, ptr<const Key>(centers), ptr<const Key>(contexts),
              ptr<const Key>(negatives), n_win, nc, neg, d, alpha, ptr<float>(loss), ptr<unsigned long long>(stats),
              deterministic);
  });
  m.def("sample_keys", [](uintptr_t be, uintptr_t stream, int kind, uintptr_t prob, uintptr_t alias, int64_t n_table,
                          Key first, Key stride, uintptr_t out, int64_t n, uint64_t seed, bool local_only, int max_tries,
                          uintptr_t stats) {
    sample_keys(backend_of(be), (cudaStream_t)stream, kind, ptr<const float>(prob), ptr<const int32_t>(alias), n_table,
                first, stride, ptr<Key>(out), n, seed, local_only, max_tries, ptr<unsigned long long>(stats));
  });
  m.def("intent_prepass", [](uintptr_t be, uintptr_t stream, uintptr_t keys, int64_t n, int64_t end, int worker, uintptr_t out_keys,
                             uintptr_t out_count) {
    intent_prepass(backend_of(be), (cudaStream_t)stream, ptr<const Key>(keys), n, (Clock)end, worker, ptr<Key>(out_keys),
                   ptr<unsigned int>(out_count));
  });
  m.def("kge_complex_step", [](uintptr_t be, uintptr_t stream, uintptr_t s, uintptr_t r, uintptr_t o, uintptr_t labels,
                               int n, int nh, float eta, float gamma_e, float gamma_r, uintptr_t loss, uintptr_t stats,
                               float dropout_e, float dropout_r, uint64_t seed, bool deterministic) {
    kge_complex_step(backend_of(be), (cudaStream_t)stream, ptr<const Key>(s), ptr<const Key>(r), ptr<const Key>(o),
                     ptr<const float>(labels), n, nh, eta, gamma_e, gamma_r, ptr<float>(loss),
                     ptr<unsigned long long>(stats), dropout_e, dropout_r, seed, deterministic);
  });
  m.def("kge_rescal_step", [](uintptr_t be, uintptr_t stream, uintptr_t s, uintptr_t r, uintptr_t o, uintptr_t labels,
                              int n, int D, float eta, float gamma_e, float gamma_r, uintptr_t loss, uintptr_t stats,
                              float dropout_e, float dropout_r, uint64_t seed, bool deterministic) {
    kge_rescal_step(backend_of(be), (cudaStream_t)stream, ptr<const Key>(s), ptr<const Key>(r), ptr<const Key>(o),
                    ptr<const float>(labels), n, D, eta, gamma_e, gamma_r, ptr<float>(loss),
                    ptr<unsigned long long>(stats), dropout_e, dropout_r, seed, deterministic);
  });
  m.def("mf_step", [](uintptr_t be, uintptr_t stream, uintptr_t rows, uintptr_t cols, uintptr_t xs, uintptr_t rn,
                      uintptr_t cn, int n, int rank, float eps, float lambda, uintptr_t loss, uintptr_t stats,
                      bool deterministic) {
    mf_step(backend_of(be), (cudaStream_t)stream, ptr<const Key>(rows), ptr<const Key>(cols), ptr<const float>(xs),
            ptr<const int>(rn), ptr<const int>(cn), n, rank, eps, lambda, ptr<float>(loss),
            ptr<unsigned long long>(stats), deterministic);
  });
  m.def("sgns_shared_workspace_bytes", [](int B, int Nn, int d) { return sgns_shared_workspace_bytes(B, Nn, d); });
  m.def("sgns_shared_core", [](uintptr_t stream, uintptr_t R, uintptr_t contexts, uintptr_t negs, int B, int Nn, int d, float alpha,
                               uintptr_t ws, uintptr_t U, uintptr_t loss) {
    sgns_shared_core((cudaStream_t)stream, ptr<const float>(R), ptr<const Key>(contexts), ptr<const Key>(negs), B, Nn, d, alpha,
                     ptr<void>(ws), ptr<float>(U), ptr<float>(loss));
  });
  m.def("gemm_nt_bf16", [](uintptr_t stream, uintptr_t A, uintptr_t B, int M, int N, int K, uintptr_t C, int ldc) {
    gemm_nt_bf16((cudaStream_t)stream, ptr<const void>(A), ptr<const void>(B), M, N, K, ptr<float>(C), ldc);
  });
  m.def("gemm_nt_e4m3", [](uintptr_t stream, uintptr_t A, uintptr_t B, int M, int N, int K, uintptr_t C, int ldc, float alpha) {
    gemm_nt_e4m3((cudaStream_t)stream, ptr<const void>(A), ptr<const void>(B), M, N, K, ptr<float>(C), ldc, alpha);
  });
  m.def("gemm_nt_bf16_rank_count", [](uintptr_t stream, uintptr_t A, uintptr_t B, int M, int N, int K, uintptr_t ts,
                                      uintptr_t tc, uintptr_t rank) {
    gemm_nt_bf16_rank_count((cudaStream_t)stream, ptr<const void>(A), ptr<const void>(B), M, N, K, ptr<const float>(ts),
                            ptr<const int>(tc), ptr<int>(rank));
  });
  m.def("gather_gemm", [](uintptr_t be, uintptr_t stream, uintptr_t Q, uintptr_t keys, int M, int N, int K, int ldq,
                          uintptr_t C, int ldc, uintptr_t stats) {
    gather_gemm(backend_of(be), (cudaStream_t)stream, ptr<const void>(Q), ptr<const Key>(keys), M, N, K, ldq, ptr<float>(C),
                ldc, ptr<unsigned long long>(stats));
  });
  m.def("gather_gemm_rank_count", [](uintptr_t be, uintptr_t stream, uintptr_t Q, uintptr_t keys, int M, int N, int K,
                                     int ldq, uintptr_t ts, uintptr_t tc, uintptr_t rank, uintptr_t stats) {
    gather_gemm_rank_count(backend_of(be), (cudaStream_t)stream, ptr<const void>(Q), ptr<const Key>(keys), M, N, K, ldq,
                           ptr<const float>(ts), ptr<const int>(tc), ptr<int>(rank), ptr<unsigned long long>(stats));
  });
  m.attr("topk_max_k") = kTopkMax;
  m.def("topk_num_slices", [](int M, int N, int max_tiles_per_cta) { return topk_num_slices(M, N, max_tiles_per_cta); });
  m.def("gemm_nt_topk", [](uintptr_t stream, uintptr_t A, uintptr_t B, int M, int N, int K, int k, int S, uintptr_t col_scale,
                           uintptr_t ex_off, uintptr_t ex_cols, uintptr_t part_v, uintptr_t part_c, uintptr_t out_v,
                           uintptr_t out_i) {
    gemm_nt_topk((cudaStream_t)stream, ptr<const void>(A), ptr<const void>(B), M, N, K, k, S, ptr<const float>(col_scale),
                 ptr<const int64_t>(ex_off), ptr<const int64_t>(ex_cols), ptr<float>(part_v), ptr<int>(part_c),
                 ptr<float>(out_v), ptr<int64_t>(out_i));
  });
  m.def("gather_gemm_topk", [](uintptr_t be, uintptr_t stream, uintptr_t Q, uintptr_t keys, int M, int N, int K, int ldq,
                               int k, int S, uintptr_t col_scale, uintptr_t ex_off, uintptr_t ex_cols, uintptr_t part_v,
                               uintptr_t part_c, uintptr_t out_v, uintptr_t out_i, uintptr_t stats) {
    gather_gemm_topk(backend_of(be), (cudaStream_t)stream, ptr<const void>(Q), ptr<const Key>(keys), M, N, K, ldq, k, S,
                     ptr<const float>(col_scale), ptr<const int64_t>(ex_off), ptr<const int64_t>(ex_cols), ptr<float>(part_v),
                     ptr<int>(part_c), ptr<float>(out_v), ptr<int64_t>(out_i), ptr<unsigned long long>(stats));
  });
  m.attr("transe_max_dim") = kTransEMaxDim;
  m.attr("transe_max_neg") = kTransEMaxNeg;
  m.def("kge_transe_step", [](uintptr_t be, uintptr_t stream, uintptr_t s, uintptr_t r, uintptr_t o, uintptr_t neg, int B,
                              int n_neg, int d, int p, float margin, float eta, float gamma_e, float gamma_r, uintptr_t loss,
                              uintptr_t stats, bool deterministic) {
    kge_transe_step(backend_of(be), (cudaStream_t)stream, ptr<const Key>(s), ptr<const Key>(r), ptr<const Key>(o),
                    ptr<const Key>(neg), B, n_neg, d, p, margin, eta, gamma_e, gamma_r, ptr<float>(loss),
                    ptr<unsigned long long>(stats), deterministic);
  });
  m.attr("rotate_max_dim") = kRotatEMaxDim;
  m.attr("rotate_max_neg") = kRotatEMaxNeg;
  m.def("kge_rotate_step", [](uintptr_t be, uintptr_t stream, uintptr_t s, uintptr_t r, uintptr_t o, uintptr_t neg, int B,
                              int n_neg, int d, float margin, float alpha, float eta, float gamma_e, uintptr_t loss,
                              uintptr_t stats, bool deterministic) {
    kge_rotate_step(backend_of(be), (cudaStream_t)stream, ptr<const Key>(s), ptr<const Key>(r), ptr<const Key>(o),
                    ptr<const Key>(neg), B, n_neg, d, margin, alpha, eta, gamma_e, ptr<float>(loss),
                    ptr<unsigned long long>(stats), deterministic);
  });
  m.attr("bpr_max_rank") = kBprMaxRank;
  m.attr("bpr_max_neg") = kBprMaxNeg;
  m.def("mf_bpr_step", [](uintptr_t be, uintptr_t stream, uintptr_t users, uintptr_t pos, uintptr_t neg, int B, int n_neg,
                          int rank, float eps, float lam, uintptr_t loss, uintptr_t stats, bool deterministic) {
    mf_bpr_step(backend_of(be), (cudaStream_t)stream, ptr<const Key>(users), ptr<const Key>(pos), ptr<const Key>(neg), B,
                n_neg, rank, eps, lam, ptr<float>(loss), ptr<unsigned long long>(stats), deterministic);
  });
  m.attr("als_max_rank") = kAlsMaxRank;
  m.def("als_solve", [](uintptr_t be, uintptr_t stream, uintptr_t targets, uintptr_t offsets, uintptr_t others,
                        uintptr_t a, uintptr_t b, int n, int rank, float lam, uintptr_t gram, uintptr_t stats) {
    als_solve(backend_of(be), (cudaStream_t)stream, ptr<const Key>(targets), ptr<const int64_t>(offsets),
              ptr<const Key>(others), ptr<const float>(a), ptr<const float>(b), n, rank, lam, ptr<const float>(gram),
              ptr<unsigned long long>(stats));
  });
  m.def("als_gram", [](uintptr_t be, uintptr_t stream, uintptr_t keys, int64_t n, int rank, uintptr_t G) {
    als_gram(backend_of(be), (cudaStream_t)stream, ptr<const Key>(keys), n, rank, ptr<float>(G));
  });
  m.def("dist_num_slices", [](uintptr_t be, int M, int N, int max_tiles_per_cta) {
    return dist_num_slices(backend_of(be), M, N, max_tiles_per_cta);
  });
  m.def("gather_dist_rank_count", [](uintptr_t be, uintptr_t stream, uintptr_t q, uintptr_t keys, int M, int N, int dim,
                                     int p, bool normalize, int S, uintptr_t true_col, uintptr_t ex_off, uintptr_t ex_cols,
                                     uintptr_t dtrue, uintptr_t raw, uintptr_t filt, uintptr_t stats) {
    gather_dist_rank_count(backend_of(be), (cudaStream_t)stream, ptr<const float>(q), ptr<const Key>(keys), M, N, dim, p,
                           normalize, S, ptr<const int64_t>(true_col), ptr<const int64_t>(ex_off),
                           ptr<const int64_t>(ex_cols), ptr<float>(dtrue), ptr<int64_t>(raw), ptr<int64_t>(filt),
                           ptr<unsigned long long>(stats));
  });
  m.def("gather_dist_topk", [](uintptr_t be, uintptr_t stream, uintptr_t q, uintptr_t keys, int M, int N, int dim, int p,
                               bool normalize, int k, int S, uintptr_t ex_off, uintptr_t ex_cols, uintptr_t part_v,
                               uintptr_t part_c, uintptr_t out_v, uintptr_t out_i, uintptr_t stats) {
    gather_dist_topk(backend_of(be), (cudaStream_t)stream, ptr<const float>(q), ptr<const Key>(keys), M, N, dim, p,
                     normalize, k, S, ptr<const int64_t>(ex_off), ptr<const int64_t>(ex_cols), ptr<float>(part_v),
                     ptr<int>(part_c), ptr<float>(out_v), ptr<int64_t>(out_i), ptr<unsigned long long>(stats));
  });
  m.attr("embedding_bag_max_dim") = kEmbBagMaxDim;
  m.def("embedding_bag_workspace_bytes", [](int64_t nnz, int64_t nbags, int E) {
    return embedding_bag_workspace_bytes(nnz, nbags, E);
  });
  m.def("embedding_bag_forward", [](uintptr_t be, uintptr_t stream, uintptr_t keys, uintptr_t offsets, uintptr_t weights,
                                    int64_t nnz, int nbags, int E, bool mean, uintptr_t out, uintptr_t stats) {
    embedding_bag_forward(backend_of(be), (cudaStream_t)stream, ptr<const Key>(keys), ptr<const int64_t>(offsets),
                          ptr<const float>(weights), nnz, nbags, E, mean, ptr<float>(out), ptr<unsigned long long>(stats));
  });
  m.def("embedding_bag_backward", [](uintptr_t be, uintptr_t stream, uintptr_t keys, uintptr_t offsets, uintptr_t weights,
                                     int64_t nnz, int nbags, int E, bool mean, uintptr_t grad_out, float lr,
                                     float grad_scale, uintptr_t ws, size_t ws_bytes, uintptr_t stats) {
    embedding_bag_backward(backend_of(be), (cudaStream_t)stream, ptr<const Key>(keys), ptr<const int64_t>(offsets),
                           ptr<const float>(weights), nnz, nbags, E, mean, ptr<const float>(grad_out), lr, grad_scale,
                           ptr<void>(ws), ws_bytes, ptr<unsigned long long>(stats));
  });
  py::class_<SgnsLoop>(m, "SgnsLoop")
      .def(py::init([](uintptr_t worker, uintptr_t be, int batch_pairs, int negative, int embed_dim, int read_ahead,
                       int max_inflight, int rank, bool signal_intent, bool local_only, int64_t model_seed, int sampler_kind,
                       uintptr_t prob, uintptr_t alias, int64_t n_table, Key first_key, Key key_stride, uintptr_t sampler_stats) {
        SgnsLoopConfig c;
        c.batch_pairs = batch_pairs; c.negative = negative; c.embed_dim = embed_dim; c.read_ahead = read_ahead;
        c.max_inflight = max_inflight; c.rank = rank; c.signal_intent = signal_intent; c.local_only = local_only;
        c.model_seed = model_seed; c.sampler_kind = sampler_kind; c.prob = ptr<const float>(prob);
        c.alias = ptr<const int32_t>(alias); c.n_table = n_table; c.first_key = first_key; c.key_stride = key_stride;
        c.sampler_stats = ptr<unsigned long long>(sampler_stats);
        return new SgnsLoop(reinterpret_cast<Worker*>(worker), &backend_of(be), c);
      }))
      .def("run", [](SgnsLoop& l, uintptr_t stream, int64_t first, int64_t n, bool resident, std::vector<uintptr_t> batches,
                     std::vector<uintptr_t> intent_keys, std::vector<int64_t> intent_counts, uintptr_t loss_dev,
                     uintptr_t loss_host, uintptr_t stats, int64_t step_no0, float alpha) {
        py::gil_scoped_release rel;
        l.run((cudaStream_t)stream, first, n, resident, batches, intent_keys, intent_counts, ptr<float>(loss_dev),
              ptr<float>(loss_host), ptr<unsigned long long>(stats), step_no0, alpha);
      });
  m.def("kernel_launches", [] { return kernel_launch_counter().load(); });
  m.def("track_stream", [](uintptr_t be, uintptr_t stream) { backend_of(be).track_stream((cudaStream_t)stream); });
}

}  // namespace cudaops
}  // namespace adapm

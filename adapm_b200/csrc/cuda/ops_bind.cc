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
  m.def("hs_step", [](uintptr_t be, uintptr_t stream, uintptr_t centers, uintptr_t contexts, int n_items, int nc,
                      uintptr_t offsets, uintptr_t nodes, uintptr_t codes, int n_words, int max_len, int d, float alpha,
                      uintptr_t loss, uintptr_t stats, bool deterministic) {
    hs_step(backend_of(be), (cudaStream_t)stream, ptr<const Key>(centers), ptr<const Key>(contexts), n_items, nc,
            ptr<const int64_t>(offsets), ptr<const int32_t>(nodes), ptr<const uint32_t>(codes), n_words, max_len, d,
            alpha, ptr<float>(loss), ptr<unsigned long long>(stats), deterministic);
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
  m.def("kge_1vsall_workspace_bytes", [](int N, int B, int d, int chunk) { return kge_1vsall_workspace_bytes(N, B, d, chunk); });
  m.def("kge_1vsall_core", [](uintptr_t stream, int model, uintptr_t R, uintptr_t s, uintptr_t o, uintptr_t rel,
                              uintptr_t ent_off, uintptr_t ent_pos, uintptr_t rel_off, uintptr_t rel_pos, int N, int nrel,
                              int B, int d, int chunk, float eta, float gamma_e, float gamma_r, uintptr_t ws, uintptr_t U,
                              uintptr_t loss) {
    kge_1vsall_core((cudaStream_t)stream, model, ptr<const float>(R), ptr<const Key>(s), ptr<const Key>(o),
                    ptr<const int32_t>(rel), ptr<const int64_t>(ent_off), ptr<const int32_t>(ent_pos),
                    ptr<const int64_t>(rel_off), ptr<const int32_t>(rel_pos), N, nrel, B, d, chunk, eta, gamma_e, gamma_r,
                    ptr<void>(ws), ptr<float>(U), ptr<float>(loss));
  });
  m.def("kge_shared_workspace_bytes", [](int B, int S, int d) { return kge_shared_workspace_bytes(B, S, d); });
  m.def("kge_shared_core", [](uintptr_t stream, int model, uintptr_t R, uintptr_t s, uintptr_t o, uintptr_t rel,
                              uintptr_t cand, uintptr_t qorder, uintptr_t ent_off, uintptr_t ent_pos, uintptr_t rel_off,
                              uintptr_t rel_pos, int Ne, int nrel, int B, int S, int d, float eta, float gamma_e,
                              float gamma_r, uintptr_t ws, uintptr_t U, uintptr_t loss) {
    kge_shared_core((cudaStream_t)stream, model, ptr<const float>(R), ptr<const Key>(s), ptr<const Key>(o),
                    ptr<const int32_t>(rel), ptr<const Key>(cand), ptr<const Key>(qorder), ptr<const int64_t>(ent_off),
                    ptr<const int32_t>(ent_pos), ptr<const int64_t>(rel_off), ptr<const int32_t>(rel_pos), Ne, nrel, B,
                    S, d, eta, gamma_e, gamma_r, ptr<void>(ws), ptr<float>(U), ptr<float>(loss));
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
  m.attr("glove_max_dim") = kGloveMaxDim;
  m.def("glove_step", [](uintptr_t be, uintptr_t stream, uintptr_t words, uintptr_t ctxs, uintptr_t xs, int n, int d,
                         float eta, float x_max, float alpha, uintptr_t loss, uintptr_t stats, bool deterministic) {
    glove_step(backend_of(be), (cudaStream_t)stream, ptr<const Key>(words), ptr<const Key>(ctxs), ptr<const float>(xs), n,
               d, eta, x_max, alpha, ptr<float>(loss), ptr<unsigned long long>(stats), deterministic);
  });
  m.attr("cooc_max_window") = kCoocMaxWindow;
  py::class_<Cooccurrence>(m, "Cooccurrence")
      .def(py::init([](uintptr_t stream, uintptr_t tokens, int64_t n_tokens, uintptr_t offsets, int64_t n_sentences,
                       int64_t V, int window, bool symmetric, bool distance_weighting, int rank, int world,
                       int64_t max_bytes) {
        return new Cooccurrence((cudaStream_t)stream, ptr<const int32_t>(tokens), n_tokens, ptr<const int64_t>(offsets),
                                n_sentences, V, window, symmetric, distance_weighting, rank, world, max_bytes);
      }))
      .def("run", [](Cooccurrence& c) {
        py::gil_scoped_release rel;
        return c.run();
      })
      .def("write", [](const Cooccurrence& c, uintptr_t rows, uintptr_t cols, uintptr_t x) {
        c.write(ptr<int32_t>(rows), ptr<int32_t>(cols), ptr<float>(x));
      })
      .def("chunks", &Cooccurrence::chunks)
      .def("denominator", &Cooccurrence::denominator);
  m.attr("doc2vec_max_dim") = kDoc2VecMaxDim;
  m.attr("doc2vec_max_targets") = kDoc2VecMaxTargets;
  m.attr("doc2vec_max_window") = kDoc2VecMaxWindow;
  m.attr("doc2vec_max_words") = kDoc2VecMaxWords;
  m.def("doc2vec_infer_epoch", [](uintptr_t be, uintptr_t stream, uintptr_t tokens, uintptr_t offsets, uintptr_t doc_ids,
                                  int64_t M, bool dm, int d, int negative, int window, int epoch, float alpha,
                                  uint64_t seed, int kind, uintptr_t prob, uintptr_t alias, int64_t n_table, int64_t first,
                                  int64_t stride, uintptr_t state, uintptr_t loss, uintptr_t stats) {
    doc2vec_infer_epoch(backend_of(be), (cudaStream_t)stream, ptr<const int64_t>(tokens), ptr<const int64_t>(offsets),
                        ptr<const int64_t>(doc_ids), M, dm, d, negative, window, epoch, alpha, seed, kind,
                        ptr<const float>(prob), ptr<const int32_t>(alias), n_table, first, stride, ptr<float>(state),
                        ptr<float>(loss), ptr<unsigned long long>(stats));
  });
  m.def("node2vec_walks", [](uintptr_t stream, uintptr_t offsets, uintptr_t nbrs, uintptr_t cumw, uintptr_t starts,
                             uintptr_t walk_nos, int64_t n_walks, int L, uint64_t seed, uint64_t epoch,
                             uint32_t thr_return, uint32_t thr_in, uint32_t thr_out, bool second_order, uintptr_t out) {
    node2vec_walks((cudaStream_t)stream, ptr<const int64_t>(offsets), ptr<const int32_t>(nbrs), ptr<const int64_t>(cumw),
                   ptr<const int64_t>(starts), ptr<const int64_t>(walk_nos), n_walks, L, seed, epoch, thr_return, thr_in,
                   thr_out, second_order, ptr<int64_t>(out));
  });
  m.def("walk_pair_scan_bytes", [](int64_t n_items) { return walk_pair_scan_bytes(n_items); });
  m.def("walk_pair_ends", [](uintptr_t stream, uintptr_t walks, int64_t n_walks, int L, int window, uint64_t seed,
                             uintptr_t counts, uintptr_t ends, uintptr_t temp, size_t temp_bytes) {
    walk_pair_ends((cudaStream_t)stream, ptr<const int64_t>(walks), n_walks, L, window, seed, ptr<int64_t>(counts),
                   ptr<int64_t>(ends), ptr<void>(temp), temp_bytes);
  });
  m.def("walk_pairs_write", [](uintptr_t stream, uintptr_t walks, int64_t n_walks, int L, int window, uint64_t seed,
                               uintptr_t ends, int64_t n_pairs, uintptr_t out) {
    walk_pairs_write((cudaStream_t)stream, ptr<const int64_t>(walks), n_walks, L, window, seed, ptr<const int64_t>(ends),
                     n_pairs, ptr<Key>(out));
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
  m.def("embedding_bag_workspace_bytes", [](int64_t nnz, int E) {
    return embedding_bag_workspace_bytes(nnz, E);
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
  m.attr("dlrm_max_rows") = kDlrmMaxRows;
  m.attr("dlrm_max_dim") = kDlrmMaxDim;
  m.def("dlrm_interaction_forward", [](uintptr_t stream, uintptr_t z, uintptr_t e, int64_t B, int F, int E, int W,
                                       uintptr_t R) {
    dlrm_interaction_forward((cudaStream_t)stream, ptr<const float>(z), ptr<const float>(e), B, F, E, W, ptr<float>(R));
  });
  m.def("dlrm_interaction_backward", [](uintptr_t stream, uintptr_t dR, uintptr_t z, uintptr_t e, int64_t B, int F,
                                        int E, int W, uintptr_t dz, uintptr_t de) {
    dlrm_interaction_backward((cudaStream_t)stream, ptr<const float>(dR), ptr<const float>(z), ptr<const float>(e), B,
                              F, E, W, ptr<float>(dz), ptr<float>(de));
  });
  m.attr("dcn_max_layers") = kDcnMaxLayers;
  m.attr("dcn_min_rank") = kDcnMinRank;
  m.attr("dcn_max_rank") = kDcnMaxRank;
  m.def("dcn_workspace_floats", [](int B, int N, int r) { return dcn_workspace_floats(B, N, r); });
  m.def("dcn_forward", [](uintptr_t stream, uintptr_t z, uintptr_t e, int B, int E, int N, int r, int L, uintptr_t V,
                          uintptr_t W, uintptr_t b, uintptr_t xb, uintptr_t hb, uintptr_t x, uintptr_t xt, uintptr_t ht,
                          uintptr_t ub) {
    dcn_forward((cudaStream_t)stream, ptr<const float>(z), ptr<const float>(e), B, E, N, r, L, ptr<const void>(V),
                ptr<const void>(W), ptr<const float>(b), ptr<void>(xb), ptr<void>(hb), ptr<float>(x), ptr<void>(xt),
                ptr<void>(ht), ptr<void>(ub));
  });
  m.def("dcn_backward", [](uintptr_t stream, uintptr_t z, uintptr_t e, int B, int E, int N, int r, int L, uintptr_t Vt,
                           uintptr_t Wt, uintptr_t xt, uintptr_t ht, uintptr_t ub, uintptr_t grad_out, uintptr_t G,
                           uintptr_t dx0, uintptr_t Pb, uintptr_t Pt, uintptr_t dh, uintptr_t dht, uintptr_t ws,
                           uintptr_t dz, uintptr_t de, uintptr_t dV, uintptr_t dW, uintptr_t db) {
    dcn_backward((cudaStream_t)stream, ptr<const float>(z), ptr<const float>(e), B, E, N, r, L, ptr<const void>(Vt),
                 ptr<const void>(Wt), ptr<const void>(xt), ptr<const void>(ht), ptr<const void>(ub),
                 ptr<const float>(grad_out), ptr<float>(G), ptr<float>(dx0), ptr<void>(Pb), ptr<void>(Pt),
                 ptr<void>(dh), ptr<void>(dht), ptr<float>(ws), ptr<float>(dz), ptr<float>(de), ptr<float>(dV),
                 ptr<float>(dW), ptr<float>(db));
  });
  m.attr("ffm_max_fields") = kFfmMaxFields;
  m.attr("ffm_max_k") = kFfmMaxK;
  m.attr("ffm_max_fk") = kFfmMaxFk;
  m.def("ffm_workspace_bytes", [](int B, int F, int k) { return ffm_workspace_bytes(B, F, k); });
  m.def("ffm_forward", [](uintptr_t be, uintptr_t stream, uintptr_t ids, int B, int F, int k, float r, uintptr_t logits,
                          uintptr_t stats) {
    ffm_forward(backend_of(be), (cudaStream_t)stream, ptr<const Key>(ids), B, F, k, r, ptr<float>(logits),
                ptr<unsigned long long>(stats));
  });
  m.def("ffm_step", [](uintptr_t be, uintptr_t stream, uintptr_t ids, uintptr_t labels, int B, int F, int k, float r,
                       float eta, float lam, uintptr_t ws, size_t ws_bytes, uintptr_t loss, uintptr_t stats) {
    ffm_step(backend_of(be), (cudaStream_t)stream, ptr<const Key>(ids), ptr<const float>(labels), B, F, k, r, eta, lam,
             ptr<void>(ws), ws_bytes, ptr<float>(loss), ptr<unsigned long long>(stats));
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

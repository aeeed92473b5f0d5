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

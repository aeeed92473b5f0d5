// The host side of grouped_push.cuh that needs cub: the workspace of the sort and the sort itself, in one translation
// unit so that the extension carries one set of cub's radix-sort kernels for the embedding-bag and FFM backwards.
#include <cuda_runtime.h>

#include <cub/cub.cuh>

#include "grouped_push.cuh"

namespace adapm {
namespace cudaops {
namespace grouped {

PushWorkspace carve_push(Carve& a, int64_t nnz, int E) {
  PushWorkspace w{};
  ADAPM_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, w.sort_bytes, (const unsigned long long*)nullptr,
                                                   (unsigned long long*)nullptr, (const int*)nullptr, (int*)nullptr,
                                                   (int)nnz, 0, 64));
  const size_t n_tiles = (size_t)(nnz + kTile - 1) / kTile;
  w.sk = a.take<Key>(nnz);
  w.pos_in = a.take<int>(nnz);
  w.pos_out = a.take<int>(nnz);
  w.part = a.take<float>(n_tiles * 2 * E);
  w.sort_tmp = a.take<char>(w.sort_bytes);
  return w;
}

void sort_pairs(CudaBackend& be, cudaStream_t stream, const Key* keys, const PushWorkspace& w, int nnz) {
  size_t sort_bytes = w.sort_bytes;
  ADAPM_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(w.sort_tmp, sort_bytes, reinterpret_cast<const unsigned long long*>(keys),
                                                   reinterpret_cast<unsigned long long*>(w.sk), w.pos_in, w.pos_out, nnz, 0,
                                                   key_bits(be.ctx().L.num_keys), stream));
}

}  // namespace grouped
}  // namespace cudaops
}  // namespace adapm

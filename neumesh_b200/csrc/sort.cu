// Stable key-value radix sort shared by the deterministic reductions (csrc/train.cu's vertex-table scatter,
// nmb_vertex_normals' corner lists).  Kept in its own translation unit so that the kernels of the files that call it do
// not change with the sort's instantiation.
#include <cub/cub.cuh>

#include "common.cuh"

namespace nmb {

cudaError_t sort_pairs_u32(void* tmp, size_t& tmp_bytes, const uint32_t* key_in, uint32_t* key_out,
                           const int32_t* val_in, int32_t* val_out, int n, int end_bit, cudaStream_t stream) {
  return cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, key_in, key_out, val_in, val_out, n, 0, end_bit, stream);
}

}  // namespace nmb

// The edges of a triangle mesh as fnr_measure.cu and fnr_decimate.cu both find them: half-edge k of face f runs from
// corner k to corner (k + 1) % 3 and is keyed min * V + max; one stable radix sort of the 3F keys (with whatever the
// caller carries along as values) makes each edge a run of equal keys, in key order.
#pragma once
#include <cub/cub.cuh>
#include <cstdint>

namespace fnr {

__device__ __forceinline__ unsigned long long half_edge_key(unsigned long long a, unsigned long long b, unsigned long long V) {
  return (a < b ? a : b) * V + (a < b ? b : a);
}

inline int bits_for(unsigned long long n) {  // bits that hold every value below n
  int b = 1;
  while (b < 64 && (n - 1) >> b) ++b;
  return b;
}

// The sort of the E = 3F half-edge keys of a mesh of V vertices (E within int); a null temp queries its size.
template <class Value>
cudaError_t sort_half_edges(void* temp, size_t& temp_bytes, const unsigned long long* keys_in, unsigned long long* keys_out,
                            const Value* values_in, Value* values_out, long long E, long long V, cudaStream_t st) {
  return cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys_in, keys_out, values_in, values_out, (int)E, 0,
                                         bits_for((unsigned long long)V * (unsigned long long)V), st);
}

}  // namespace fnr

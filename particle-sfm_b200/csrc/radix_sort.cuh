// radix_sort.cuh — the CUB radix sort of key/value double buffers the stages share.  Kept out of psfm_common.cuh
// so that only the units that sort include CUB.
#pragma once
#include <cub/device/device_radix_sort.cuh>

#include "psfm_common.cuh"

namespace psfm {

// stable sort of n (key, value) pairs on the key bits [0, end_bit); the result is in keys.Current() / vals.Current().
// The scratch is stream-ordered when a stream is given.
template <typename K, typename V, typename NumT>
void sort_pairs(cub::DoubleBuffer<K>& keys, cub::DoubleBuffer<V>& vals, NumT n, int end_bit, cudaStream_t st = nullptr) {
  size_t bytes = 0;
  PSFM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys, vals, n, 0, end_bit, st));
  DBuf<unsigned char> tmp;
  tmp.alloc(bytes, st);
  PSFM_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, bytes, keys, vals, n, 0, end_bit, st));
  PSFM_LAUNCH_CHECK();
}

// number of bits the radix sort looks at for keys in [0, max_key], at least 1
inline int key_bits(unsigned long long max_key) {
  int b = 1;
  while (b < 64 && (max_key >> b)) ++b;
  return b;
}

}  // namespace psfm

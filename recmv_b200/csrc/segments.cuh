// Deterministic segmented sums without float atomics: items are keyed by the slot they add to, a stable CUB radix
// sort groups each slot's items in increasing item order, and segment_bounds_kernel finds every slot's [begin, end)
// range in the sorted list.  One thread per slot then sums its range in order, so the result is bit-identical from
// run to run and independent of the SM count.  Used by the vertex normals (shade.cu) and the KNN backward (knn.cu).
#pragma once
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"

namespace recmv {
namespace {

constexpr int kSegThreads = 256;

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

inline int key_bits(unsigned max_key) {   // bits that hold the keys 0..max_key
  int bits = 1;
  while (bits < 32 && (1ull << bits) <= (unsigned long long)max_key) ++bits;
  return bits;
}

// CUB's temporary storage for the sort of M pairs with keys in [0, max_key]; the same query in the size call and in
// the run.
inline int sort_temp_bytes(long long M, unsigned max_key, size_t* bytes) {
  *bytes = 0;
  if (M == 0) return RECMV_OK;
  const cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, *bytes, (const unsigned*)nullptr, (unsigned*)nullptr,
                                                        (const unsigned*)nullptr, (unsigned*)nullptr, (int)M, 0,
                                                        key_bits(max_key));
  return e == cudaSuccess ? RECMV_OK : (int)e;
}

// Stable sort of M (key, value) pairs; temp holds sort_temp_bytes(M, max_key).  Counts as one library launch.
inline int sort_pairs(void* temp, const unsigned* keys_in, unsigned* keys_out, const unsigned* vals_in,
                      unsigned* vals_out, long long M, unsigned max_key, cudaStream_t st) {
  size_t bytes = 0;
  int s = sort_temp_bytes(M, max_key, &bytes);
  if (s) return s;
  const cudaError_t e = cub::DeviceRadixSort::SortPairs(temp, bytes, keys_in, keys_out, vals_in, vals_out, (int)M, 0,
                                                        key_bits(max_key), st);
  if (e != cudaSuccess) return (int)e;
  return launch_status();
}

// The [beg, end) range of every slot k < S in the sorted keys; keys >= S (invalid items) are skipped.  beg and end
// must be zero beforehand, so a slot with no items keeps the empty range [0, 0).
__global__ void __launch_bounds__(kSegThreads) segment_bounds_kernel(const unsigned* __restrict__ keys, long long M,
                                                                      unsigned S, int* __restrict__ beg,
                                                                      int* __restrict__ end) {
  const long long i = blockIdx.x * (long long)kSegThreads + threadIdx.x;
  if (i >= M) return;
  const unsigned k = keys[i];
  if (k >= S) return;
  if (i == 0 || keys[i - 1] != k) beg[k] = (int)i;
  if (i == M - 1 || keys[i + 1] != k) end[k] = (int)(i + 1);
}

}  // namespace
}  // namespace recmv

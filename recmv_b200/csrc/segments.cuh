// Deterministic segmented sums without float atomics: items are keyed by the slot they add to, a stable CUB radix
// sort groups each slot's items in increasing item order, and segment_bounds_kernel finds every slot's [begin, end)
// range in the sorted list.  One thread per slot then sums its range in order, so the result is bit-identical from
// run to run and independent of the SM count.  Used by the vertex normals (shade.cu) and the KNN backward (knn.cu).
// The vertex-face incidence (vertex_faces.cu) uses the corner keys and the pair sort without the sums; the mesh
// adjacency (nricp.cu) uses the 64-bit key sort alone.
#pragma once
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "workspace.cuh"

namespace recmv {
namespace {

constexpr int kSegThreads = 256;

template <class K>
int key_bits(K max_key) {   // bits that hold the keys 0..max_key
  int bits = 1;
  while (bits < 8 * (int)sizeof(K) && (1ull << bits) <= (unsigned long long)max_key) ++bits;
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

// The same two calls for a sort of M keys alone.  Templates, so that only a file that sorts keys instantiates CUB's
// kernels for them.
template <class K>
int sort_keys_temp_bytes(long long M, K max_key, size_t* bytes) {
  *bytes = 0;
  if (M == 0) return RECMV_OK;
  const cudaError_t e =
      cub::DeviceRadixSort::SortKeys(nullptr, *bytes, (const K*)nullptr, (K*)nullptr, (int)M, 0, key_bits(max_key));
  return e == cudaSuccess ? RECMV_OK : (int)e;
}

template <class K>
int sort_keys(void* temp, const K* in, K* out, long long M, K max_key, cudaStream_t st) {
  size_t bytes = 0;
  int s = sort_keys_temp_bytes(M, max_key, &bytes);
  if (s) return s;
  const cudaError_t e = cub::DeviceRadixSort::SortKeys(temp, bytes, in, out, (int)M, 0, key_bits(max_key), st);
  if (e != cudaSuccess) return (int)e;
  return launch_status();
}

// The workspace of a segmented sum of M items into S slots: the sort's keys and values, the slots' [beg, end) ranges
// and, last, CUB's temporary storage, whose sort_temp_bytes the size query adds to the bytes taken.
struct SegmentWs {
  unsigned *keys_in, *keys_out, *vals_in, *vals_out;
  int *beg, *end;
  size_t ranges_bytes;   // beg and end, which are cleared together
  void* temp;
};

inline SegmentWs segment_layout(Carve& c, long long M, long long S) {
  SegmentWs w;
  w.keys_in = c.take<unsigned>(M);
  w.keys_out = c.take<unsigned>(M);
  w.vals_in = c.take<unsigned>(M);
  w.vals_out = c.take<unsigned>(M);
  const size_t ranges = c.used;
  w.beg = c.take<int>(S);
  w.end = c.take<int>(S);
  w.ranges_bytes = c.used - ranges;
  w.temp = c.take<char>(0, 1);
  return w;
}

// One thread per (face, corner) e = 3 f + k of faces [F,3], M = 3 F: key = the corner's vertex, or V for every corner
// of a face with an index outside [0, V) (so such faces sort last), value e.  bad (or nullptr) is set to 1 when any
// face has such an index.
__global__ void __launch_bounds__(kSegThreads) corner_keys_kernel(const long long* __restrict__ faces, long long M,
                                                                   int V, unsigned* __restrict__ keys,
                                                                   unsigned* __restrict__ vals, int* __restrict__ bad) {
  const long long e = blockIdx.x * (long long)kSegThreads + threadIdx.x;
  if (e >= M) return;
  const long long f = e / 3;
  const long long a = faces[3 * f], b = faces[3 * f + 1], c = faces[3 * f + 2];
  const bool ok = a >= 0 && a < V && b >= 0 && b < V && c >= 0 && c < V;
  keys[e] = ok ? (unsigned)faces[e] : (unsigned)V;
  vals[e] = (unsigned)e;
  if (!ok && bad) *bad = 1;
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

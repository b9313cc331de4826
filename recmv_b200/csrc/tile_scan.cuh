// Single-CTA exclusive scan shared by the binned rasterizers (raster.cu, points_raster.cu).
#pragma once

namespace recmv {
namespace {

constexpr int kScanThreads = 1024;

// Exclusive scan of counts[0..n).  offsets[i] is the first list entry of bin i (offsets[n] = total); cursor[i] starts
// there when cursor is not NULL.  The total goes to counters[2] (saturated at INT32_MAX) and counters[3] = total >
// capacity.  One CTA: n is at most a few hundred thousand.
__global__ void __launch_bounds__(kScanThreads) raster_scan_kernel(const int* __restrict__ tile_counts, int ntiles,
                                                                   long long* __restrict__ offsets,
                                                                   long long* __restrict__ cursor, long long capacity,
                                                                   int* __restrict__ counters) {
  __shared__ long long warp_sums[32];
  __shared__ long long carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int base = 0; base < ntiles; base += kScanThreads) {
    const int i = base + threadIdx.x;
    const long long v = i < ntiles ? tile_counts[i] : 0;
    long long inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const long long t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
      const long long w = warp_sums[lane];
      long long wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const long long t = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += t; }
      warp_sums[lane] = wi - w;
    }
    __syncthreads();
    const long long carry = carry_s;
    if (i < ntiles) {
      offsets[i] = carry + warp_sums[wid] + inc - v;
      if (cursor) cursor[i] = offsets[i];
    }
    __syncthreads();
    if (threadIdx.x == kScanThreads - 1) carry_s = carry + warp_sums[31] + inc;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const long long total = carry_s;
    offsets[ntiles] = total;
    counters[2] = total > 0x7fffffffLL ? 0x7fffffff : (int)total;
    counters[3] = total > capacity ? 1 : 0;
  }
}

}  // namespace
}  // namespace recmv

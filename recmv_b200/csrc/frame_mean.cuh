// The deterministic per-frame mean of the photometric terms (frame_loss.cu, DESIGN section 1k):
//   L = (1/N) sum_b [ sum_{i in b, included} e_i / max(1, n_b) ],
// torch_scatter's `scatter(e, b, reduce='mean', dim_size=N).mean()` with an empty frame contributing 0.  Rows are cut
// into fixed chunks of kChunkRows; each chunk's per-frame sums (f64) and counts go to the workspace, and one CTA
// combines them per frame in chunk order.  No float atomics, and the partition does not depend on the launch, so the
// value is bit-identical from run to run.  A row whose frame lies outside [0, N) contributes nothing.
#pragma once

namespace recmv {
namespace {

constexpr int kMeanThreads = 256;
constexpr int kRowsPerThread = 4;
constexpr int kChunkRows = kMeanThreads * kRowsPerThread;

// Sum of v over the block in a fixed tree order; the result is valid in thread 0.  red has kMeanThreads / 32 slots.
__device__ __forceinline__ double block_sum(double v, double* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();                        // red is free again
  if (lane == 0) red[wid] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kMeanThreads / 32; ++w) s += red[w];
  return s;
}

__device__ __forceinline__ int block_count(int v, int* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  int s = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kMeanThreads / 32; ++w) s += red[w];
  return s;
}

// One CTA per chunk.  row(i, &e, &b) gives row i's term and frame (b < 0 or b >= N: not included).
// part_sum / part_cnt [chunks, N].
template <class Row>
__device__ __forceinline__ void chunk_partials(const Row& row, long long M, int N, double* __restrict__ part_sum,
                                               int* __restrict__ part_cnt) {
  __shared__ double red_d[kMeanThreads / 32];
  __shared__ int red_i[kMeanThreads / 32];
  double e[kRowsPerThread];
  int b[kRowsPerThread];
  const long long c0 = (long long)blockIdx.x * kChunkRows;
#pragma unroll
  for (int k = 0; k < kRowsPerThread; ++k) {
    const long long i = c0 + k * kMeanThreads + threadIdx.x;
    e[k] = 0.0;
    b[k] = -1;
    if (i < M) row(i, e[k], b[k]);
    if (b[k] >= N) b[k] = -1;
  }
  for (int f = 0; f < N; ++f) {
    double s = 0.0;
    int n = 0;
#pragma unroll
    for (int k = 0; k < kRowsPerThread; ++k)
      if (b[k] == f) { s += e[k]; ++n; }
    s = block_sum(s, red_d);
    n = block_count(n, red_i);
    if (threadIdx.x == 0) {
      part_sum[(size_t)blockIdx.x * N + f] = s;
      part_cnt[(size_t)blockIdx.x * N + f] = n;
    }
  }
}

// One CTA: per frame, the chunk partials summed in chunk order (strided by thread, then the block tree), then
// L = (1/N) sum_b S_b / max(1, n_b) in frame order, rounded once.
__device__ __forceinline__ void finish_mean(const double* __restrict__ part_sum, const int* __restrict__ part_cnt,
                                            int chunks, int N, float* __restrict__ loss, int* __restrict__ counts) {
  __shared__ double red_d[kMeanThreads / 32];
  __shared__ int red_i[kMeanThreads / 32];
  double L = 0.0;
  for (int f = 0; f < N; ++f) {
    double s = 0.0;
    int n = 0;
    for (int c = threadIdx.x; c < chunks; c += kMeanThreads) {
      s += part_sum[(size_t)c * N + f];
      n += part_cnt[(size_t)c * N + f];
    }
    s = block_sum(s, red_d);
    n = block_count(n, red_i);
    if (threadIdx.x == 0) {
      counts[f] = n;
      L += s / (double)(n > 1 ? n : 1);
    }
  }
  if (threadIdx.x == 0) *loss = __double2float_rn(N > 0 ? L / (double)N : 0.0);
}

// g / (N max(1, n_b)) of the upstream gradient g, for a row of frame b in [0, N)
__device__ __forceinline__ double frame_scale(const float* grad_loss, const int* counts, int N, int b) {
  const int n = counts[b];
  return (double)__ldg(grad_loss) / ((double)N * (double)(n > 1 ? n : 1));
}

}  // namespace
}  // namespace recmv

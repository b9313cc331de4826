// Pieces of the ordered compactions that emit training rays (fragments.cu, train_rays.cu): the exclusive scan of
// per-block counts and CameraMine.view_rays in fp32.
#pragma once

namespace recmv {
namespace {

// In-place exclusive scan of counts[0..n) by one CTA of 1024 threads; the total goes to *total.  n is at most a few
// hundred thousand (one count per block of rows).
__device__ __forceinline__ void scan_block_counts(int* __restrict__ counts, int n, int* __restrict__ total) {
  __shared__ int warp_sums[32];
  __shared__ int carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int base = 0; base < n; base += 1024) {
    const int b = base + threadIdx.x;
    const int v = b < n ? counts[b] : 0;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
      const int w = warp_sums[lane];
      int wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += t; }
      warp_sums[lane] = wi - w;
    }
    __syncthreads();
    const int carry = carry_s;
    if (b < n) counts[b] = carry + warp_sums[wid] + inc - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = carry + warp_sums[31] + inc;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry_s;
}

// CameraMine.view_rays (model/CameraMine.py:146-167) of pixel (x, y) = (col, row) with ps = (x, y, 1): every operation
// rounded separately, as the torch expression does.  R row-major; rays = v @ R^T -> out_i = sum_j v_j R[i][j].
__device__ __forceinline__ void view_ray(float fx, float fy, float px, float py, const float* R, float x, float y,
                                         float* out) {
  float v0 = __fadd_rn(__fdiv_rn(-x, fx), __fdiv_rn(px, fx));
  float v1 = __fadd_rn(__fdiv_rn(-y, fy), __fdiv_rn(py, fy));
  float v2 = 1.f;
  const float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(v0, v0), __fmul_rn(v1, v1)), __fmul_rn(v2, v2)));
  v0 = __fdiv_rn(v0, nrm); v1 = __fdiv_rn(v1, nrm); v2 = __fdiv_rn(v2, nrm);
#pragma unroll
  for (int i = 0; i < 3; ++i)
    out[i] = __fadd_rn(__fadd_rn(__fmul_rn(v0, R[3 * i]), __fmul_rn(v1, R[3 * i + 1])), __fmul_rn(v2, R[3 * i + 2]));
}

}  // namespace
}  // namespace recmv

// 3x3 singular value decomposition, one matrix per thread, entirely in registers.
// Replaces the deformation regulariser's `torch.svd(Jacobs.cpu())` (engineer/networks/OptimGarmentNetwork.py:1148 -- the
// reference moves the [N,3,3] Jacobians to the host because "the gpu svd is too slow", then copies the singular values
// back) and its backward (autograd of the LAPACK call, again through host memory).
//
// Algorithm: one-sided Jacobi (Hestenes).  The columns of J are rotated pairwise until mutually orthogonal; the rotations
// accumulate in V, the column norms are the singular values and the normalised columns are U:  J = U diag(S) V^T.
// Working on J directly (not on J^T J) keeps small singular values to full relative accuracy.  Output follows torch.svd:
// S descending; the signs of matching U / V columns are arbitrary (they are in LAPACK too) -- callers that differentiate
// use S only (the reference's loss is a function of log S), for which  dJ = U diag(dS) V^T.
// HBM-bound: 36 B read, 84 B written per matrix (12 B if only S is asked for).
#include "common.cuh"

namespace recmv {
namespace {

constexpr int kSvdThreads = 128;
constexpr int kSvdSweeps = 10;   // fp32 converges in 4-5 sweeps (quadratic); the loop exits early per thread

__device__ __forceinline__ void rotate_pair(float (&a)[3][3], float (&v)[3][3], int p, int q, bool& rotated) {
  // columns p, q of a (a[row][col])
  const float alpha = a[0][p] * a[0][p] + a[1][p] * a[1][p] + a[2][p] * a[2][p];
  const float beta = a[0][q] * a[0][q] + a[1][q] * a[1][q] + a[2][q] * a[2][q];
  const float gamma = a[0][p] * a[0][q] + a[1][p] * a[1][q] + a[2][p] * a[2][q];
  // sqrt(alpha) sqrt(beta), not sqrt(alpha beta): the product is a fourth power of the entries and overflows from 1e10
  if (fabsf(gamma) <= 1e-7f * (sqrtf(alpha) * sqrtf(beta)) || gamma == 0.f) return;
  rotated = true;
  const float zeta = (beta - alpha) / (2.f * gamma);
  const float t = copysignf(1.f, zeta) / (fabsf(zeta) + sqrtf(1.f + zeta * zeta));
  const float c = rsqrtf(1.f + t * t), s = c * t;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const float ap = a[r][p], aq = a[r][q];
    a[r][p] = c * ap - s * aq;
    a[r][q] = s * ap + c * aq;
    const float vp = v[r][p], vq = v[r][q];
    v[r][p] = c * vp - s * vq;
    v[r][q] = s * vp + c * vq;
  }
}

__device__ __forceinline__ void swap_cols(float (&a)[3][3], float (&v)[3][3], float (&s)[3], int p, int q) {
  if (s[p] >= s[q]) return;
  const float ts = s[p]; s[p] = s[q]; s[q] = ts;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    float t = a[r][p]; a[r][p] = a[r][q]; a[r][q] = t;
    t = v[r][p]; v[r][p] = v[r][q]; v[r][q] = t;
  }
}

__device__ __forceinline__ void any_perpendicular(const float (&u)[3], float (&w)[3]) {
  // unit vector orthogonal to the unit vector u: cross with the axis u is least aligned with
  const float ax = fabsf(u[0]), ay = fabsf(u[1]), az = fabsf(u[2]);
  float e[3] = {0.f, 0.f, 0.f};
  if (ax <= ay && ax <= az) e[0] = 1.f; else if (ay <= az) e[1] = 1.f; else e[2] = 1.f;
  w[0] = u[1] * e[2] - u[2] * e[1];
  w[1] = u[2] * e[0] - u[0] * e[2];
  w[2] = u[0] * e[1] - u[1] * e[0];
  const float inv = rsqrtf(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  w[0] *= inv; w[1] *= inv; w[2] *= inv;
}

__global__ void __launch_bounds__(kSvdThreads) svd3_kernel(const float* __restrict__ J, long long N, float* __restrict__ U,
                                                           float* __restrict__ S, float* __restrict__ V) {
  const long long i = blockIdx.x * (long long)kSvdThreads + threadIdx.x;
  if (i >= N) return;
  float a[3][3], v[3][3] = {{1.f, 0.f, 0.f}, {0.f, 1.f, 0.f}, {0.f, 0.f, 1.f}};
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) a[r][c] = __ldg(J + i * 9 + r * 3 + c);
#pragma unroll 1
  for (int sweep = 0; sweep < kSvdSweeps; ++sweep) {
    bool rotated = false;
    rotate_pair(a, v, 0, 1, rotated);
    rotate_pair(a, v, 0, 2, rotated);
    rotate_pair(a, v, 1, 2, rotated);
    if (!rotated) break;
  }
  float s[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) s[c] = sqrtf(a[0][c] * a[0][c] + a[1][c] * a[1][c] + a[2][c] * a[2][c]);
  swap_cols(a, v, s, 0, 1);
  swap_cols(a, v, s, 0, 2);
  swap_cols(a, v, s, 1, 2);
  S[i * 3 + 0] = s[0]; S[i * 3 + 1] = s[1]; S[i * 3 + 2] = s[2];
  if (V) {
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) V[i * 9 + r * 3 + c] = v[r][c];
  }
  if (U) {
    // normalised columns; columns of (numerically) zero singular values are completed to an orthonormal basis
    const float tiny = 1e-30f + 1e-7f * s[0];
    float u[3][3];   // u[col][row]
    if (s[0] > 1e-30f) {
      const float inv = 1.f / s[0];
      u[0][0] = a[0][0] * inv; u[0][1] = a[1][0] * inv; u[0][2] = a[2][0] * inv;
    } else {
      u[0][0] = 1.f; u[0][1] = 0.f; u[0][2] = 0.f;
    }
    if (s[1] > tiny) {
      const float inv = 1.f / s[1];
      u[1][0] = a[0][1] * inv; u[1][1] = a[1][1] * inv; u[1][2] = a[2][1] * inv;
    } else {
      any_perpendicular(u[0], u[1]);
    }
    if (s[2] > tiny) {
      const float inv = 1.f / s[2];
      u[2][0] = a[0][2] * inv; u[2][1] = a[1][2] * inv; u[2][2] = a[2][2] * inv;
    } else {
      u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
      u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
      u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
    }
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) U[i * 9 + r * 3 + c] = u[c][r];
  }
}

// dJ = U diag(dS) V^T
__global__ void __launch_bounds__(kSvdThreads) svd3_backward_s_kernel(const float* __restrict__ U, const float* __restrict__ V,
                                                                      const float* __restrict__ dS, long long N,
                                                                      float* __restrict__ dJ) {
  const long long i = blockIdx.x * (long long)kSvdThreads + threadIdx.x;
  if (i >= N) return;
  float u[9], v[9], g[3];
#pragma unroll
  for (int e = 0; e < 9; ++e) { u[e] = __ldg(U + i * 9 + e); v[e] = __ldg(V + i * 9 + e); }
#pragma unroll
  for (int e = 0; e < 3; ++e) g[e] = __ldg(dS + i * 3 + e);
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c)
      dJ[i * 9 + r * 3 + c] = u[r * 3 + 0] * g[0] * v[c * 3 + 0] + u[r * 3 + 1] * g[1] * v[c * 3 + 1] + u[r * 3 + 2] * g[2] * v[c * 3 + 2];
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_svd3x3(const float* J, int64_t N, float* U, float* S, float* V, recmv_stream_t stream) {
  if (N < 0) return RECMV_E_SHAPE;
  if (N == 0) return RECMV_OK;
  if (!J || !S) return RECMV_E_NULL;
  svd3_kernel<<<(unsigned)((N + kSvdThreads - 1) / kSvdThreads), kSvdThreads, 0, (cudaStream_t)stream>>>(J, N, U, S, V);
  return launch_status();
}

extern "C" int recmv_svd3x3_backward_s(const float* U, const float* V, const float* dS, int64_t N, float* dJ,
                                       recmv_stream_t stream) {
  if (N < 0) return RECMV_E_SHAPE;
  if (N == 0) return RECMV_OK;
  if (!U || !V || !dS || !dJ) return RECMV_E_NULL;
  svd3_backward_s_kernel<<<(unsigned)((N + kSvdThreads - 1) / kSvdThreads), kSvdThreads, 0, (cudaStream_t)stream>>>(U, V, dS, N, dJ);
  return launch_status();
}

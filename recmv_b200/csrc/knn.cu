// Nearest neighbour of every point of one cloud in a second cloud (DESIGN section 1e): the K = 1 `knn_points` behind
// `chamfer_distance` and the feature-curve loss `fl_proj_loss`.  Replaces pytorch3d's KNN extension.
//
// Forward, p1 [N,P1,D] queries against p2 [N,P2,D] candidates, D = 2 or 3, optional device lengths clamped to [0, P]:
//   d = (dx*dx + dy*dy) [+ dz*dz], dx = x1 - x2, every operation rounded in fp32 in that order (no FMA contraction).
//   The smallest d wins, on equal d the lower index j: the lexicographic (d, j) minimum.  d >= 0 (or NaN), so its bit
//   pattern orders like its value and the key float_bits(d) << 32 | j orders like (d, j).
//   1. knn_scan_kernel   one thread per query; the block stages 256 candidates at a time in shared memory and keeps
//                        its best (d, j) in registers.  When the queries alone do not fill the SMs the grid also splits
//                        P2 into S ranges, each writing its own key slot -- no atomics.
//   2. knn_final_kernel  one thread per query: the minimum key over the S slots (order-free, so the result does not
//                        depend on S, the launch shape or the SM count), then dists / idx and the padding
//                        (dists = 0, idx = -1 for i >= lengths1[n] or lengths2[n] == 0).
//
// Backward from grad_dists g [N,P1]:  dp1_i = 2 g_i (p1_i - p2_idx_i),  dp2_j = -sum_{i: idx_i = j} dp1_i summed in
// increasing i -- the segmented sum of segments.cuh: knn_grad_p1_kernel also keys every query by its candidate, a
// stable radix sort groups each candidate's queries in increasing i, and knn_grad_p2_kernel sums them in that order.
// Entries with idx = -1 contribute nothing.  No float atomics: bit-identical from run to run and on any GPU.
#include "common.cuh"
#include "segments.cuh"

namespace recmv {
namespace {

constexpr int kKnnThreads = 256;   // queries per block = candidates per shared-memory tile
constexpr int kMaxSplits = 64;
constexpr int kScanBlocksPerSm = 8;

template <int D> struct Stage;
template <> struct Stage<2> {
  using T = float2;
  static __device__ __forceinline__ T load(const float* p) { return make_float2(p[0], p[1]); }
};
template <> struct Stage<3> {
  using T = float4;
  static __device__ __forceinline__ T load(const float* p) { return make_float4(p[0], p[1], p[2], 0.f); }
};

__device__ __forceinline__ float dist(const float2& q, const float2& c) {
  const float dx = __fsub_rn(q.x, c.x), dy = __fsub_rn(q.y, c.y);
  return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
}
__device__ __forceinline__ float dist(const float4& q, const float4& c) {
  const float dx = __fsub_rn(q.x, c.x), dy = __fsub_rn(q.y, c.y), dz = __fsub_rn(q.z, c.z);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ int clamp_len(const long long* __restrict__ len, int n, int P) {
  if (!len) return P;
  const long long v = len[n];
  return v < 0 ? 0 : (v > P ? P : (int)v);
}

// grid.x = N * query blocks, grid.y = S splits of `chunk` candidates (a multiple of kKnnThreads).
// keys [S][N*P1]: slot s holds the best key of candidates [s*chunk, (s+1)*chunk) within lengths2.
template <int D>
__global__ void __launch_bounds__(kKnnThreads) knn_scan_kernel(const float* __restrict__ p1,
                                                                const float* __restrict__ p2,
                                                                const long long* __restrict__ len1,
                                                                const long long* __restrict__ len2, int P1, int P2,
                                                                int qblocks, int chunk, long long NP1,
                                                                unsigned long long* __restrict__ keys) {
  using T = typename Stage<D>::T;
  __shared__ T tile[kKnnThreads];
  const int n = blockIdx.x / qblocks;
  const int i0 = (blockIdx.x - n * qblocks) * kKnnThreads;
  const int L1 = clamp_len(len1, n, P1);
  if (i0 >= L1) return;   // block-uniform: no query of this block is live
  const int L2 = clamp_len(len2, n, P2);
  const int i = i0 + threadIdx.x;
  const bool live = i < L1;
  const T q = Stage<D>::load(p1 + ((long long)n * P1 + (live ? i : i0)) * D);
  const int c0 = blockIdx.y * chunk;
  const int c1 = min(c0 + chunk, L2);
  // a key of all ones loses to every candidate whose d is not a NaN with every bit set; bj starts at the range's
  // first index, so even then a non-empty range reports an index inside it
  unsigned bu = 0xffffffffu;
  int bj = c0;
  const float* src = p2 + (long long)n * P2 * D;
  for (int t0 = c0; t0 < c1; t0 += kKnnThreads) {
    const int j = t0 + threadIdx.x;
    if (j < c1) tile[threadIdx.x] = Stage<D>::load(src + (long long)j * D);
    __syncthreads();
    const int cnt = min(kKnnThreads, c1 - t0);
    if (cnt == kKnnThreads) {
#pragma unroll 8
      for (int k = 0; k < kKnnThreads; ++k) {
        const unsigned u = __float_as_uint(dist(q, tile[k]));
        if (u < bu) { bu = u; bj = t0 + k; }
      }
    } else {
      for (int k = 0; k < cnt; ++k) {
        const unsigned u = __float_as_uint(dist(q, tile[k]));
        if (u < bu) { bu = u; bj = t0 + k; }
      }
    }
    __syncthreads();
  }
  if (live) keys[blockIdx.y * NP1 + (long long)n * P1 + i] = ((unsigned long long)bu << 32) | (unsigned)bj;
}

__global__ void __launch_bounds__(kKnnThreads) knn_final_kernel(const unsigned long long* __restrict__ keys, int S,
                                                                 const long long* __restrict__ len1,
                                                                 const long long* __restrict__ len2, int P1, int P2,
                                                                 long long NP1, float* __restrict__ dists,
                                                                 long long* __restrict__ idx) {
  const long long gid = blockIdx.x * (long long)kKnnThreads + threadIdx.x;
  if (gid >= NP1) return;
  const int n = (int)(gid / P1), i = (int)(gid - (long long)n * P1);
  if (i >= clamp_len(len1, n, P1) || clamp_len(len2, n, P2) == 0) {
    dists[gid] = 0.f;
    idx[gid] = -1;
    return;
  }
  unsigned long long best = keys[gid];
  for (int s = 1; s < S; ++s) best = min(best, keys[s * NP1 + gid]);
  dists[gid] = __uint_as_float((unsigned)(best >> 32));
  idx[gid] = (long long)(unsigned)best;
}

// dp1 of every query, and its sort item: key n*P2 + j (N*P2 when it has no neighbour), value = its row n*P1 + i
template <int D>
__global__ void __launch_bounds__(kKnnThreads) knn_grad_p1_kernel(const float* __restrict__ p1,
                                                                   const float* __restrict__ p2,
                                                                   const long long* __restrict__ idx,
                                                                   const float* __restrict__ grad, int P1, int P2,
                                                                   long long NP1, unsigned invalid,
                                                                   float* __restrict__ dp1, unsigned* __restrict__ keys,
                                                                   unsigned* __restrict__ vals) {
  const long long gid = blockIdx.x * (long long)kKnnThreads + threadIdx.x;
  if (gid >= NP1) return;
  const long long n = gid / P1;
  const long long j = idx[gid];
  const bool ok = j >= 0 && j < P2;
  const float g2 = __fmul_rn(2.f, grad[gid]);
  const float* a = p1 + gid * D;
  if (ok) {   // p2 is only read here: with P2 == 0 it may be NULL
    const float* b = p2 + (n * P2 + j) * D;
#pragma unroll
    for (int c = 0; c < D; ++c) dp1[gid * D + c] = __fmul_rn(g2, __fsub_rn(a[c], b[c]));
  } else {
#pragma unroll
    for (int c = 0; c < D; ++c) dp1[gid * D + c] = 0.f;
  }
  if (keys) {
    keys[gid] = ok ? (unsigned)(n * P2 + j) : invalid;
    vals[gid] = (unsigned)gid;
  }
}

// one thread per candidate (n, j): dp2 = -(sum of dp1 over its queries, in increasing i)
template <int D>
__global__ void __launch_bounds__(kKnnThreads) knn_grad_p2_kernel(const float* __restrict__ dp1,
                                                                   const unsigned* __restrict__ vals,
                                                                   const int* __restrict__ beg,
                                                                   const int* __restrict__ end, long long NP2,
                                                                   float* __restrict__ dp2) {
  const long long gid = blockIdx.x * (long long)kKnnThreads + threadIdx.x;
  if (gid >= NP2) return;
  float acc[D];
#pragma unroll
  for (int c = 0; c < D; ++c) acc[c] = 0.f;
  const int e1 = end[gid];
  for (int k = beg[gid]; k < e1; ++k) {
    const float* g = dp1 + (long long)vals[k] * D;
#pragma unroll
    for (int c = 0; c < D; ++c) acc[c] = __fadd_rn(acc[c], g[c]);
  }
#pragma unroll
  for (int c = 0; c < D; ++c) dp2[gid * D + c] = -acc[c];
}

// Splits of P2: enough (query block, split) pairs for two waves of kScanBlocksPerSm blocks per SM, each split a whole
// number of tiles.  Depends only on the shape and the SM count, so the size query and the run agree.
void plan(int N, long long P1, long long P2, int* S, int* chunk) {
  const long long qb = (P1 + kKnnThreads - 1) / kKnnThreads * N;
  const long long tiles = (P2 + kKnnThreads - 1) / kKnnThreads;
  const long long want = 2LL * kScanBlocksPerSm * num_sms();
  long long s = qb > 0 ? (want + qb - 1) / qb : 1;
  s = s < 1 ? 1 : s;
  s = s > kMaxSplits ? kMaxSplits : s;
  s = s > tiles ? (tiles > 0 ? tiles : 1) : s;
  const long long per = (tiles + s - 1) / s;   // tiles per split
  *chunk = (int)((per > 0 ? per : 1) * kKnnThreads);
  *S = tiles > 0 ? (int)((tiles + per - 1) / per) : 1;
}

int check_shape(int N, long long P1, long long P2) {
  if (N < 0 || P1 < 0 || P2 < 0) return RECMV_E_SHAPE;
  // int point indices, unsigned sort keys n*P2 + j up to the sentinel N*P2, int list positions
  if (P1 >= 0x7fffffffLL || P2 >= 0x7fffffffLL || (long long)N * P1 >= 0x7fffffffLL ||
      (long long)N * P2 >= 0xffffffffLL)
    return RECMV_E_RANGE;
  return RECMV_OK;
}

struct BackwardWs {
  unsigned *keys_in, *keys_out, *vals_in, *vals_out;
  int *beg, *end;
  void* temp;
};

BackwardWs carve(void* ws, long long M, long long NP2) {
  BackwardWs w;
  char* p = (char*)ws;
  w.keys_in = (unsigned*)p; p += align256((size_t)M * 4);
  w.keys_out = (unsigned*)p; p += align256((size_t)M * 4);
  w.vals_in = (unsigned*)p; p += align256((size_t)M * 4);
  w.vals_out = (unsigned*)p; p += align256((size_t)M * 4);
  w.beg = (int*)p; p += align256((size_t)NP2 * 4);
  w.end = (int*)p; p += align256((size_t)NP2 * 4);
  w.temp = p;
  return w;
}

template <int D>
int nearest(const float* p1, const float* p2, const long long* l1, const long long* l2, int N, int P1, int P2,
            void* ws, float* dists, long long* idx, cudaStream_t st) {
  int S, chunk;
  plan(N, P1, P2, &S, &chunk);
  const int qb = (P1 + kKnnThreads - 1) / kKnnThreads;
  const long long NP1 = (long long)N * P1;
  unsigned long long* keys = (unsigned long long*)ws;
  knn_scan_kernel<D><<<dim3((unsigned)((long long)N * qb), (unsigned)S), kKnnThreads, 0, st>>>(
      p1, p2, l1, l2, P1, P2, qb, chunk, NP1, keys);
  int s = launch_status();
  if (s) return s;
  knn_final_kernel<<<(unsigned)((NP1 + kKnnThreads - 1) / kKnnThreads), kKnnThreads, 0, st>>>(keys, S, l1, l2, P1, P2,
                                                                                            NP1, dists, idx);
  return launch_status();
}

template <int D>
int nearest_backward(const float* p1, const float* p2, const long long* idx, const float* grad, int N, int P1, int P2,
                     void* ws, float* dp1, float* dp2, cudaStream_t st) {
  const long long M = (long long)N * P1, NP2 = (long long)N * P2;
  BackwardWs w = carve(ws, M, NP2);
  if (M > 0) {
    knn_grad_p1_kernel<D><<<(unsigned)((M + kKnnThreads - 1) / kKnnThreads), kKnnThreads, 0, st>>>(
        p1, p2, idx, grad, P1, P2, M, (unsigned)NP2, dp1, dp2 ? w.keys_in : nullptr, w.vals_in);
    int s = launch_status();
    if (s) return s;
  }
  if (!dp2 || NP2 == 0) return RECMV_OK;
  cudaError_t e = cudaMemsetAsync(w.beg, 0, 2 * align256((size_t)NP2 * 4), st);   // beg and end: empty ranges
  if (e != cudaSuccess) return (int)e;
  if (M > 0) {
    int s = sort_pairs(w.temp, w.keys_in, w.keys_out, w.vals_in, w.vals_out, M, (unsigned)NP2, st);
    if (s) return s;
    segment_bounds_kernel<<<(unsigned)((M + kSegThreads - 1) / kSegThreads), kSegThreads, 0, st>>>(
        w.keys_out, M, (unsigned)NP2, w.beg, w.end);
    s = launch_status();
    if (s) return s;
  }
  knn_grad_p2_kernel<D><<<(unsigned)((NP2 + kKnnThreads - 1) / kKnnThreads), kKnnThreads, 0, st>>>(
      dp1, w.vals_out, w.beg, w.end, NP2, dp2);
  return launch_status();
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_knn_workspace_bytes(int N, int64_t P1, int64_t P2, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  int s = check_shape(N, P1, P2);
  if (s) return s;
  int S, chunk;
  plan(N, P1, P2, &S, &chunk);
  const long long M = (long long)N * P1, NP2 = (long long)N * P2;
  size_t temp = 0;
  s = sort_temp_bytes(M, (unsigned)NP2, &temp);
  if (s) return s;
  const size_t fwd = (size_t)S * (size_t)M * 8;
  const size_t bwd = 4 * align256((size_t)M * 4) + 2 * align256((size_t)NP2 * 4) + temp;
  *bytes = fwd > bwd ? fwd : bwd;
  return RECMV_OK;
}

extern "C" int recmv_knn_nearest(const float* p1, const float* p2, const int64_t* lengths1, const int64_t* lengths2,
                                 int N, int64_t P1, int64_t P2, int D, void* workspace, float* out_dists,
                                 int64_t* out_idx, recmv_stream_t stream) {
  int s = check_shape(N, P1, P2);
  if (s) return s;
  if (D != 2 && D != 3) return RECMV_E_SHAPE;
  if ((long long)N * P1 == 0) return RECMV_OK;
  if (!p1 || !workspace || !out_dists || !out_idx || (P2 > 0 && !p2)) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  const long long *l1 = (const long long*)lengths1, *l2 = (const long long*)lengths2;
  if (D == 2) return nearest<2>(p1, p2, l1, l2, N, (int)P1, (int)P2, workspace, out_dists, (long long*)out_idx, st);
  return nearest<3>(p1, p2, l1, l2, N, (int)P1, (int)P2, workspace, out_dists, (long long*)out_idx, st);
}

extern "C" int recmv_knn_nearest_backward(const float* p1, const float* p2, const int64_t* idx,
                                          const float* grad_dists, int N, int64_t P1, int64_t P2, int D,
                                          void* workspace, float* grad_p1, float* grad_p2, recmv_stream_t stream) {
  int s = check_shape(N, P1, P2);
  if (s) return s;
  if (D != 2 && D != 3) return RECMV_E_SHAPE;
  const long long M = (long long)N * P1, NP2 = (long long)N * P2;
  if (M == 0 && (!grad_p2 || NP2 == 0)) return RECMV_OK;
  // an empty candidate cloud (P2 == 0) may come as NULL, as in the forward: no query has a neighbour to read
  if (!workspace || (M > 0 && (!p1 || (P2 > 0 && !p2) || !idx || !grad_dists || !grad_p1))) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  if (D == 2)
    return nearest_backward<2>(p1, p2, (const long long*)idx, grad_dists, N, (int)P1, (int)P2, workspace, grad_p1,
                               grad_p2, st);
  return nearest_backward<3>(p1, p2, (const long long*)idx, grad_dists, N, (int)P1, (int)P2, workspace, grad_p1,
                             grad_p2, st);
}

// Template registration by non-rigid ICP (DESIGN section 1f): the mesh adjacency and the fused inner step of
// `NRICP_Optimizer_AdamW`.  Replaces the per-iteration torch graph of the reference's inner loop (Local_Affine warp,
// edge stiffness, pytorch3d's `Meshes` + `mesh_laplacian_smoothing`, autograd and `AdamW(amsgrad=True)`).
//
// Adjacency of faces [F,3] over V vertices, no host read (every capacity follows from F):
//   1. adj_side_keys_kernel  one thread per face side (3F): key lo*V + hi of the sorted pair, V*V for a face with an
//                            index outside [0, V); also clears the boundary flags;
//   2. CUB radix sort        of the 3F side keys;
//   3. adj_mark_kernel       run-length marking: the first side of each run is an edge of E and emits its two
//                            directed keys lo*V + hi and hi*V + lo (V*V elsewhere); a run of length 1 marks both
//                            endpoints as boundary;
//   4. CUB radix sort        of the 6F directed keys: row-major order, neighbours ascending within a row;
//   5. adj_csr_kernel        row_ptr[r] = the first directed key >= r*V (binary search), deg, col = key mod V.
//   A self side (a, a) of a repeated-index face gives the edge (a, a), which appears twice in row a, as both
//   directions of pytorch3d's COO adjacency do.
//
// Inner step, X [V,3,4] = [A | b] per vertex, two launches and no float atomics:
//   1. nricp_grad_kernel    one thread per vertex: v_i, the warped normal and the gate w_i, the data residual
//                           r_i = w_i (v_i - c_i), the Laplacian Lv_i and u_i = Lv_i / |Lv_i|, the stiffness sum
//                           K_i = sum_j (X_i - X_j) G2; per-block partials of the data, stiffness, |Lv| and gate sums
//                           in a fixed shared-memory tree;
//   2. nricp_update_kernel  every block reduces the partials in the same fixed order (one warp, float64), so the
//                           sums depend on V only, never on the SM count; then per vertex the gradient
//                           dv_i = 2 s r_i + (lw / V)(sum_j u_j / deg_j - u_i), dX_i = dv_i [x_i; 1]^T + 2 s sw K_i
//                           with s = 1 / (2 sqrt(S)), and the AMSGrad-AdamW update of X and its three moment arrays.
//   Pass 1 reads every neighbour's X_j and pass 2 every neighbour's u_j before any vertex is updated.
#include <math.h>

#include "common.cuh"
#include "segments.cuh"

namespace recmv {
namespace {

constexpr int kAdjThreads = 256;
constexpr int kNricpThreads = 256;

inline int key_bits64(unsigned long long max_key) {
  int bits = 1;
  while (bits < 64 && (1ull << bits) <= max_key) ++bits;
  return bits;
}

inline int sort_keys64_temp(long long M, unsigned long long max_key, size_t* bytes) {
  *bytes = 0;
  if (M == 0) return RECMV_OK;
  const cudaError_t e = cub::DeviceRadixSort::SortKeys(nullptr, *bytes, (const unsigned long long*)nullptr,
                                                       (unsigned long long*)nullptr, (int)M, 0, key_bits64(max_key));
  return e == cudaSuccess ? RECMV_OK : (int)e;
}

inline int sort_keys64(void* temp, const unsigned long long* in, unsigned long long* out, long long M,
                       unsigned long long max_key, cudaStream_t st) {
  size_t bytes = 0;
  int s = sort_keys64_temp(M, max_key, &bytes);
  if (s) return s;
  const cudaError_t e =
      cub::DeviceRadixSort::SortKeys(temp, bytes, in, out, (int)M, 0, key_bits64(max_key), st);
  if (e != cudaSuccess) return (int)e;
  return launch_status();
}

__global__ void __launch_bounds__(kAdjThreads) adj_side_keys_kernel(const long long* __restrict__ faces, long long M,
                                                                     long long V, unsigned long long* __restrict__ keys,
                                                                     uint8_t* __restrict__ boundary) {
  const long long t = blockIdx.x * (long long)kAdjThreads + threadIdx.x;
  if (t < V) boundary[t] = 0;
  if (t >= M) return;
  const long long f = t / 3, k = t - 3 * f;
  const long long* fc = faces + 3 * f;
  const long long a = fc[0], b = fc[1], c = fc[2];
  const bool ok = a >= 0 && a < V && b >= 0 && b < V && c >= 0 && c < V;
  const long long p = fc[k], q = fc[k == 2 ? 0 : k + 1];
  keys[t] = ok ? (unsigned long long)(p < q ? p * V + q : q * V + p) : (unsigned long long)V * V;
}

__global__ void __launch_bounds__(kAdjThreads) adj_mark_kernel(const unsigned long long* __restrict__ sides,
                                                                long long M, long long V,
                                                                unsigned long long* __restrict__ dir,
                                                                uint8_t* __restrict__ boundary) {
  const long long i = blockIdx.x * (long long)kAdjThreads + threadIdx.x;
  if (i >= M) return;
  const unsigned long long none = (unsigned long long)V * V;
  const unsigned long long k = sides[i];
  const bool first = i == 0 || sides[i - 1] != k;
  if (k < none && first) {
    const unsigned long long lo = k / (unsigned long long)V, hi = k - lo * (unsigned long long)V;
    dir[2 * i] = k;
    dir[2 * i + 1] = hi * (unsigned long long)V + lo;
    if (i == M - 1 || sides[i + 1] != k) {   // the side occurs once among the 3F sides
      boundary[lo] = 1;
      boundary[hi] = 1;
    }
  } else {
    dir[2 * i] = none;
    dir[2 * i + 1] = none;
  }
}

__device__ __forceinline__ long long lower_bound64(const unsigned long long* __restrict__ a, long long n,
                                                   unsigned long long x) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(kAdjThreads) adj_csr_kernel(const unsigned long long* __restrict__ dir, long long M2,
                                                               long long V, int* __restrict__ row_ptr,
                                                               int* __restrict__ col, int* __restrict__ deg) {
  const long long t = blockIdx.x * (long long)kAdjThreads + threadIdx.x;
  const unsigned long long none = (unsigned long long)V * V;
  if (t <= V) {
    const long long b = lower_bound64(dir, M2, (unsigned long long)t * V);
    row_ptr[t] = (int)b;
    if (t < V) deg[t] = (int)(lower_bound64(dir, M2, (unsigned long long)(t + 1) * V) - b);
  }
  if (t < M2) {
    const unsigned long long k = dir[t];
    col[t] = k < none ? (int)(k % (unsigned long long)V) : -1;
  }
}

struct AdjWs {
  unsigned long long *a, *b;
  void* temp;
};

AdjWs carve_adj(void* ws, long long F) {
  AdjWs w;
  char* p = (char*)ws;
  w.a = (unsigned long long*)p; p += align256((size_t)F * 6 * 8);
  w.b = (unsigned long long*)p; p += align256((size_t)F * 6 * 8);
  w.temp = p;
  return w;
}

int adj_shape(long long V, long long F) {
  if (V < 0 || F < 0) return RECMV_E_SHAPE;
  if (V >= 0x7fffffffLL || 6 * F >= 0x7fffffffLL) return RECMV_E_RANGE;   // int row pointers and CUB item counts
  return RECMV_OK;
}

// ---- the inner step --------------------------------------------------------------------------------------------

// v = A x + b of the row-major [3][4] matrix X
__device__ __forceinline__ void warp_point(const float* __restrict__ X, float x0, float x1, float x2, float v[3]) {
#pragma unroll
  for (int r = 0; r < 3; ++r) v[r] = X[4 * r] * x0 + X[4 * r + 1] * x1 + X[4 * r + 2] * x2 + X[4 * r + 3];
}

// n' = inv(A)^T n with the FastMinv rule; false (and n' = 0) when |det A| < 1e-4
__device__ __forceinline__ bool warp_normal(const float* __restrict__ X, const float* __restrict__ n, float o[3]) {
  const float m[9] = {X[0], X[1], X[2], X[4], X[5], X[6], X[8], X[9], X[10]};
  float inv[9];
  const bool ok = inv3x3<float>(m, inv);
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = inv[c] * n[0] + inv[3 + c] * n[1] + inv[6 + c] * n[2];
  return ok;
}

__global__ void __launch_bounds__(kNricpThreads) nricp_warp_kernel(const float* __restrict__ X,
                                                                    const float* __restrict__ x,
                                                                    const float* __restrict__ n, long long V,
                                                                    float* __restrict__ out_v,
                                                                    float* __restrict__ out_n,
                                                                    uint8_t* __restrict__ out_ok) {
  const long long i = blockIdx.x * (long long)kNricpThreads + threadIdx.x;
  if (i >= V) return;
  float Xi[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) Xi[k] = X[12 * i + k];
  float v[3];
  warp_point(Xi, x[3 * i], x[3 * i + 1], x[3 * i + 2], v);
#pragma unroll
  for (int r = 0; r < 3; ++r) out_v[3 * i + r] = v[r];
  if (out_n || out_ok) {
    const float ni[3] = {n[3 * i], n[3 * i + 1], n[3 * i + 2]};
    float o[3];
    const bool ok = warp_normal(Xi, ni, o);
    if (out_n) {
#pragma unroll
      for (int r = 0; r < 3; ++r) out_n[3 * i + r] = o[r];
    }
    if (out_ok) out_ok[i] = ok ? 1 : 0;
  }
}

// one vertex per thread; part[block] = (data sum, stiffness sum over directed edges, sum |Lv|, gate count)
__global__ void __launch_bounds__(kNricpThreads) nricp_grad_kernel(
    const float* __restrict__ X, const float* __restrict__ x, const float* __restrict__ n,
    const float* __restrict__ tv, const float* __restrict__ tn, const long long* __restrict__ idx, long long T,
    const int* __restrict__ row_ptr, const int* __restrict__ col, const uint8_t* __restrict__ boundary, int V,
    float threshold, float gamma, float* __restrict__ u_out, float* __restrict__ r_out, float* __restrict__ K_out,
    float4* __restrict__ part) {
  __shared__ float4 red[kNricpThreads];
  const int i = blockIdx.x * kNricpThreads + threadIdx.x;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < V) {
    float Xi[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) Xi[k] = X[12 * (long long)i + k];
    float v[3];
    warp_point(Xi, x[3 * i], x[3 * i + 1], x[3 * i + 2], v);
    // gate and data residual
    const float ni[3] = {n[3 * i], n[3 * i + 1], n[3 * i + 2]};
    float np[3];
    const bool ok = warp_normal(Xi, ni, np);
    const long long j = idx[i];
    float res[3] = {0.f, 0.f, 0.f};
    bool w = false;
    if (j >= 0 && j < T) {
      const float* c = tv + 3 * j;
      const float* m = tn + 3 * j;
      const float dot = m[0] * np[0] + m[1] * np[1] + m[2] * np[2];
      const float mm = m[0] * m[0] + m[1] * m[1] + m[2] * m[2];
      const float nn = np[0] * np[0] + np[1] * np[1] + np[2] * np[2];
      const float cs = dot / sqrtf(fmaxf(mm * nn, 1e-16f));
      w = !boundary[i] && ok && cs > threshold;
      if (w) {
#pragma unroll
        for (int r = 0; r < 3; ++r) res[r] = v[r] - c[r];
      }
    }
    acc.x = res[0] * res[0] + res[1] * res[1] + res[2] * res[2];
    acc.w = w ? 1.f : 0.f;
    // Laplacian and stiffness over the sorted neighbours
    const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
    float sv[3] = {0.f, 0.f, 0.f}, K[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) K[k] = 0.f;
    float stiff = 0.f;
    const float g2 = gamma * gamma;
    for (int e = e0; e < e1; ++e) {
      const long long nb = col[e];
      const float* Xj = X + 12 * nb;
      float Xv[12];
#pragma unroll
      for (int k = 0; k < 12; ++k) Xv[k] = Xj[k];
      float vj[3];
      warp_point(Xv, x[3 * nb], x[3 * nb + 1], x[3 * nb + 2], vj);
#pragma unroll
      for (int r = 0; r < 3; ++r) sv[r] += vj[r];
#pragma unroll
      for (int k = 0; k < 12; ++k) {
        const float d = Xi[k] - Xv[k];
        const float dg = (k & 3) == 3 ? d * gamma : d;
        stiff += dg * dg;
        K[k] += (k & 3) == 3 ? d * g2 : d;
      }
    }
    const int deg = e1 - e0;
    float Lv[3];
    const float inv_deg = deg > 0 ? 1.f / (float)deg : 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) Lv[r] = sv[r] * inv_deg - v[r];
    const float ln = sqrtf(Lv[0] * Lv[0] + Lv[1] * Lv[1] + Lv[2] * Lv[2]);
    const float il = ln > 0.f ? 1.f / ln : 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      u_out[3 * (long long)i + r] = Lv[r] * il;
      r_out[3 * (long long)i + r] = res[r];
    }
#pragma unroll
    for (int k = 0; k < 12; ++k) K_out[12 * (long long)i + k] = K[k];
    acc.y = stiff;
    acc.z = ln;
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = kNricpThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      const float4 a = red[threadIdx.x], b = red[threadIdx.x + s];
      red[threadIdx.x] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = red[0];
}

struct AdamConst {
  float decay;       // 1 - lr * weight_decay
  float beta1, beta2, one_minus_beta1, one_minus_beta2;
  float step_size;   // lr / (1 - beta1^t)
  float bc2_sqrt;    // sqrt(1 - beta2^t)
  float eps;
  int first;         // t == 1: the moments start from zero (a new optimizer every epoch)
};

__global__ void __launch_bounds__(kNricpThreads) nricp_update_kernel(
    const float* __restrict__ x, const int* __restrict__ row_ptr, const int* __restrict__ col,
    const float* __restrict__ u, const float* __restrict__ r, const float* __restrict__ K,
    const float4* __restrict__ part, int nb, int V, float sw, float lw, AdamConst ad, float* __restrict__ X,
    float* __restrict__ m1, float* __restrict__ m2, float* __restrict__ vmax, float* __restrict__ stats) {
  __shared__ float coef[3];   // 2 s, 2 s sw, lw / V
  if (threadIdx.x < 32) {
    // every block sums the partials in the same order: lane l takes l, l + 32, ..., then a fixed butterfly
    double d = 0.0, st = 0.0, lp = 0.0, cnt = 0.0;
    for (int b = threadIdx.x; b < nb; b += 32) {
      const float4 p = part[b];
      d += p.x; st += p.y; lp += p.z; cnt += p.w;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      d += __shfl_xor_sync(0xffffffffu, d, o);
      st += __shfl_xor_sync(0xffffffffu, st, o);
      lp += __shfl_xor_sync(0xffffffffu, lp, o);
      cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if (threadIdx.x == 0) {
      const double stiff = 0.5 * st * (double)sw;   // every edge of E was summed from both ends
      const double S = d + stiff;
      const double lap = (double)lw * lp / (double)V;
      const float s2 = 1.f / sqrtf((float)S);      // 2 s; +inf at S = 0, as the sqrt backward gives
      coef[0] = s2;
      coef[1] = s2 * sw;
      coef[2] = lw / (float)V;
      if (blockIdx.x == 0) {
        stats[0] = (float)d;
        stats[1] = (float)stiff;
        stats[2] = (float)lap;
        stats[3] = (float)(sqrt(S) + lap);
        stats[4] = (float)cnt;
        stats[5] = (float)S;
        stats[6] = 0.f;
        stats[7] = 0.f;
      }
    }
  }
  __syncthreads();
  const int i = blockIdx.x * kNricpThreads + threadIdx.x;
  if (i >= V) return;
  const float c_data = coef[0], c_stiff = coef[1], c_lap = coef[2];
  float lu[3] = {0.f, 0.f, 0.f};
  const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
  for (int e = e0; e < e1; ++e) {
    const int j = col[e];
    const float inv_dj = 1.f / (float)(row_ptr[j + 1] - row_ptr[j]);   // j has i as a neighbour: deg_j >= 1
#pragma unroll
    for (int c = 0; c < 3; ++c) lu[c] += u[3 * (long long)j + c] * inv_dj;
  }
  float dv[3];
#pragma unroll
  for (int c = 0; c < 3; ++c)
    dv[c] = c_data * r[3 * (long long)i + c] + c_lap * (lu[c] - u[3 * (long long)i + c]);
  const float xh[4] = {x[3 * (long long)i], x[3 * (long long)i + 1], x[3 * (long long)i + 2], 1.f};
#pragma unroll
  for (int k = 0; k < 12; ++k) {
    const long long o = 12 * (long long)i + k;
    const float g = dv[k >> 2] * xh[k & 3] + c_stiff * K[o];
    const float p = X[o] * ad.decay;
    const float a = ad.first ? ad.one_minus_beta1 * g : m1[o] + ad.one_minus_beta1 * (g - m1[o]);
    const float b = ad.first ? ad.one_minus_beta2 * (g * g) : m2[o] * ad.beta2 + ad.one_minus_beta2 * (g * g);
    const float mx = ad.first ? b : fmaxf(vmax[o], b);
    const float denom = sqrtf(mx) / ad.bc2_sqrt + ad.eps;
    X[o] = p - ad.step_size * (a / denom);
    m1[o] = a;
    m2[o] = b;
    vmax[o] = mx;
  }
}

struct StepWs {
  float *u, *r, *K;
  float4* part;
};

int step_blocks(long long V) { return (int)((V + kNricpThreads - 1) / kNricpThreads); }

StepWs carve_step(void* ws, long long V) {
  StepWs w;
  char* p = (char*)ws;
  w.u = (float*)p; p += align256((size_t)V * 12);
  w.r = (float*)p; p += align256((size_t)V * 12);
  w.K = (float*)p; p += align256((size_t)V * 48);
  w.part = (float4*)p;
  return w;
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_mesh_adjacency_workspace_bytes(int64_t V, int64_t F, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  int s = adj_shape(V, F);
  if (s) return s;
  const unsigned long long none = (unsigned long long)V * V;
  size_t t1 = 0, t2 = 0;
  s = sort_keys64_temp(3 * F, none, &t1);
  if (s) return s;
  s = sort_keys64_temp(6 * F, none, &t2);
  if (s) return s;
  *bytes = 2 * align256((size_t)F * 6 * 8) + (t1 > t2 ? t1 : t2);
  return RECMV_OK;
}

extern "C" int recmv_mesh_adjacency(const int64_t* faces, int64_t F, int64_t V, void* workspace, int32_t* row_ptr,
                                    int32_t* col, int32_t* deg, uint8_t* boundary, recmv_stream_t stream) {
  int s = adj_shape(V, F);
  if (s) return s;
  if (!row_ptr || (V > 0 && (!deg || !boundary)) || (F > 0 && (!faces || !col || !workspace))) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  const long long M = 3 * F, M2 = 6 * F;
  const unsigned long long none = (unsigned long long)V * V;
  AdjWs w = carve_adj(workspace, F);
  if (M > 0) {
    const long long n1 = M > V ? M : V;
    adj_side_keys_kernel<<<(unsigned)((n1 + kAdjThreads - 1) / kAdjThreads), kAdjThreads, 0, st>>>(
        (const long long*)faces, M, V, w.a, boundary);
    s = launch_status();
    if (s) return s;
    s = sort_keys64(w.temp, w.a, w.b, M, none, st);
    if (s) return s;
    adj_mark_kernel<<<(unsigned)((M + kAdjThreads - 1) / kAdjThreads), kAdjThreads, 0, st>>>(w.b, M, V, w.a,
                                                                                            boundary);
    s = launch_status();
    if (s) return s;
    s = sort_keys64(w.temp, w.a, w.b, M2, none, st);
    if (s) return s;
  } else if (V > 0) {
    cudaError_t e = cudaMemsetAsync(boundary, 0, (size_t)V, st);
    if (e != cudaSuccess) return (int)e;
  }
  const long long n2 = M2 > V + 1 ? M2 : V + 1;
  adj_csr_kernel<<<(unsigned)((n2 + kAdjThreads - 1) / kAdjThreads), kAdjThreads, 0, st>>>(w.b, M2, V, row_ptr, col,
                                                                                          deg);
  return launch_status();
}

extern "C" int recmv_nricp_warp(const float* X, const float* x, const float* normals, int64_t V, float* out_v,
                                float* out_n, uint8_t* out_ok, recmv_stream_t stream) {
  if (V < 0) return RECMV_E_SHAPE;
  if (V >= 0x7fffffffLL) return RECMV_E_RANGE;
  if (V == 0) return RECMV_OK;
  if (!X || !x || !out_v || ((out_n || out_ok) && !normals)) return RECMV_E_NULL;
  nricp_warp_kernel<<<(unsigned)((V + kNricpThreads - 1) / kNricpThreads), kNricpThreads, 0, (cudaStream_t)stream>>>(
      X, x, normals, V, out_v, out_n, out_ok);
  return launch_status();
}

extern "C" int recmv_nricp_workspace_bytes(int64_t V, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  if (V < 0) return RECMV_E_SHAPE;
  if (V >= 0x7fffffffLL) return RECMV_E_RANGE;
  *bytes = 2 * align256((size_t)V * 12) + align256((size_t)V * 48) + align256((size_t)step_blocks(V) * 16);
  return RECMV_OK;
}

extern "C" int recmv_nricp_step(const float* x, const float* normals, const float* target_v, const float* target_n,
                                int64_t T, const int64_t* corr_idx, const int32_t* row_ptr, const int32_t* col,
                                const uint8_t* boundary, int64_t V, const recmv_nricp_params_t* prm, float* X,
                                float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq, void* workspace,
                                float* stats, recmv_stream_t stream) {
  if (V < 0 || T < 0) return RECMV_E_SHAPE;
  if (V >= 0x7fffffffLL) return RECMV_E_RANGE;
  if (!prm || !stats) return RECMV_E_NULL;
  if (prm->step < 1) return RECMV_E_SHAPE;
  if (V == 0) return RECMV_E_SHAPE;   // the loss divides by V
  if (!x || !normals || !corr_idx || !row_ptr || !col || !boundary || !X || !exp_avg || !exp_avg_sq ||
      !max_exp_avg_sq || !workspace || (T > 0 && (!target_v || !target_n)))
    return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  StepWs w = carve_step(workspace, V);
  const int nb = step_blocks(V);
  nricp_grad_kernel<<<nb, kNricpThreads, 0, st>>>(X, x, normals, target_v, target_n, (const long long*)corr_idx, T,
                                                  row_ptr, col, boundary, (int)V, prm->threshold, prm->gamma, w.u,
                                                  w.r, w.K, w.part);
  int s = launch_status();
  if (s) return s;
  // torch.optim.AdamW's scalars, formed in double as its single-tensor step forms them
  const double t = (double)prm->step;
  AdamConst ad;
  ad.decay = (float)(1.0 - (double)prm->lr * (double)prm->weight_decay);
  ad.beta1 = prm->beta1;
  ad.beta2 = prm->beta2;
  ad.one_minus_beta1 = (float)(1.0 - (double)prm->beta1);
  ad.one_minus_beta2 = (float)(1.0 - (double)prm->beta2);
  ad.step_size = (float)((double)prm->lr / (1.0 - pow((double)prm->beta1, t)));
  ad.bc2_sqrt = (float)sqrt(1.0 - pow((double)prm->beta2, t));
  ad.eps = prm->eps;
  ad.first = prm->step == 1;
  nricp_update_kernel<<<nb, kNricpThreads, 0, st>>>(x, row_ptr, col, w.u, w.r, w.K, w.part, nb, (int)V,
                                                    prm->stiffness_weight, prm->laplacian_weight, ad, X, exp_avg,
                                                    exp_avg_sq, max_exp_avg_sq, stats);
  return launch_status();
}

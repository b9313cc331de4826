// Laplacian editing of a garment template (DESIGN section 1g): the solve of `Laplacian_Optimizer`,
//   argmin_y |L y - L x|^2 + c |P y - u|^2   <=>   A y = b,  A = L^T L + c P^T P,  b = L^T L x + c P^T u,
// with L the uniform Laplacian D^-1 Adj - I of the CSR adjacency of csrc/nricp.cu and P the selection of the M
// constrained vertices.  Replaces the reference's dense inv(L^T W L) L^T W t.  Matrix-free Jacobi-preconditioned CG in
// float64, the three columns in lockstep, started at y0 = x; three launches and no host read:
//   1. lap_setup_kernel   one thread per vertex: b, the exact diagonal of A, r0 = c P^T (u - P x) (zero wherever no
//                         constraint reaches, so an unconstrained component keeps y = x exactly), z0 = p0 = r0 / diag;
//                         chunk partials of |b|^2, r.z, r.r; the count of skipped constraints;
//   2. lap_pcg_kernel     one cooperative kernel for all iterations: w = L p | q = L^T w + c cnt p, p.q | y, r, z,
//                         r.z, r.r | beta, p = z + beta p, each phase ended by a grid sync;
//   3. lap_finalize_kernel the optional zero-diagonal smoothing and the fp32 store.
// Determinism: the partial sums are over fixed 256-vertex chunks whatever the grid, and every block reduces all the
// chunk partials itself in the same fixed order, so every block holds the same scalars, takes the same branch at the
// stop test (no block can miss a grid sync) and the result is bit-identical across runs and grid sizes.  No atomics.
#include <cooperative_groups.h>
#include <math.h>

#include "common.cuh"
#include "segments.cuh"

namespace cg = cooperative_groups;

namespace recmv {
namespace {

constexpr int kLapThreads = 256;   // threads per block = vertices per reduction chunk
constexpr int kParts = 9;          // per chunk: slot 0-2 |b|^2 then p.q, 3-5 r.z, 6-8 r.r (one per column)

struct LapWs {
  double *y[3], *r[3], *p[3], *w[3], *q[3];   // [V] per column
  double* inv_deg;                            // [V] 1 / deg_i, 0 at deg_i = 0
  double* dinv;                               // [V] 1 / A_ii (0 where A_ii = 0: such a vertex is decoupled)
  double* cc;                                 // [V] c * (number of constraints on the vertex)
  double* part;                               // [chunks][kParts]
};

__host__ __device__ __forceinline__ long long lap_chunks(long long V) { return (V + kLapThreads - 1) / kLapThreads; }

size_t lap_ws_bytes(long long V) {
  const long long nc = lap_chunks(V);
  return 18 * align256((size_t)V * 8) + align256((size_t)(nc > 0 ? nc : 1) * kParts * 8);   // one block at V = 0
}

LapWs carve_lap(void* ws, long long V) {
  LapWs w;
  char* p = (char*)ws;
  const size_t vec = align256((size_t)V * 8);
  double** vecs[5] = {w.y, w.r, w.p, w.w, w.q};
  for (int a = 0; a < 5; ++a)
    for (int k = 0; k < 3; ++k, p += vec) vecs[a][k] = (double*)p;
  w.inv_deg = (double*)p; p += vec;
  w.dinv = (double*)p; p += vec;
  w.cc = (double*)p; p += vec;
  w.part = (double*)p;
  return w;
}

__device__ __forceinline__ long long lower_bound_idx(const long long* a, long long n, long long x) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// 1 / x from the hardware approximation and two Newton steps, within an ulp of the quotient.  A double division or
// sqrt would call a slow-path routine, and registers live across that call spill.  0 and inf give NaN.
__device__ __forceinline__ double rcp64(double x) {
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  y = fma(y, fma(-x, y, 1.0), y);
  return fma(y, fma(-x, y, 1.0), y);
}

// sqrt(v) for the stats record, the same way
__device__ __forceinline__ double sqrt64(double v) {
  if (v == 0.0) return 0.0;
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(v));
  y = y * fma(-0.5 * v * y, y, 1.5);
  y = y * fma(-0.5 * v * y, y, 1.5);
  return v * y;
}

// v[0..2] summed over the block's threads in a fixed shared-memory tree; every thread gets the sums
__device__ __forceinline__ void block_sum3(double v[3], double (*red)[kLapThreads]) {
  const int t = threadIdx.x;
#pragma unroll
  for (int k = 0; k < 3; ++k) red[k][t] = v[k];
  __syncthreads();
  for (int s = kLapThreads / 2; s > 0; s >>= 1) {
    if (t < s) {
#pragma unroll
      for (int k = 0; k < 3; ++k) red[k][t] += red[k][t + s];
    }
    __syncthreads();
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) v[k] = red[k][0];
  __syncthreads();   // red is reused by the next call
}

// the chunk partials of slots off..off+2, summed in an order fixed by the chunk count alone
__device__ __forceinline__ void reduce_parts(const double* part, long long nc, int off, double out[3],
                                             double (*red)[kLapThreads]) {
  out[0] = out[1] = out[2] = 0.0;
  for (long long c = threadIdx.x; c < nc; c += kLapThreads) {
#pragma unroll
    for (int k = 0; k < 3; ++k) out[k] += part[c * kParts + off + k];
  }
  block_sum3(out, red);
}

__device__ __forceinline__ void store_parts(double* part, long long chunk, int off, const double v[3]) {
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) part[chunk * kParts + off + k] = v[k];
  }
}

// (L x)_i of the fp32 vertices, in float64
__device__ __forceinline__ void lap_f32(const float* __restrict__ x, const int* __restrict__ row_ptr,
                                        const int* __restrict__ col, int i, double o[3]) {
  const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
  double s[3] = {0.0, 0.0, 0.0};
  for (int e = e0; e < e1; ++e) {
    const long long j = col[e];
#pragma unroll
    for (int k = 0; k < 3; ++k) s[k] += (double)x[3 * j + k];
  }
  const double inv = e1 > e0 ? rcp64((double)(e1 - e0)) : 0.0;
#pragma unroll
  for (int k = 0; k < 3; ++k) o[k] = s[k] * inv - (double)x[3 * (long long)i + k];
}

__global__ void __launch_bounds__(kLapThreads) lap_setup_kernel(
    const float* __restrict__ x, int V, const int* __restrict__ row_ptr, const int* __restrict__ col,
    const int* __restrict__ deg, const long long* __restrict__ cidx, const float* __restrict__ ctgt, long long M,
    double c, LapWs w, float* __restrict__ stats) {
  __shared__ double red[3][kLapThreads];
  const int i = blockIdx.x * kLapThreads + threadIdx.x;
  double bb[3] = {0.0, 0.0, 0.0}, rz[3] = {0.0, 0.0, 0.0}, rr[3] = {0.0, 0.0, 0.0};
  if (i < V) {
    // the vertex's constraints: a segment of the sorted indices
    const long long k0 = lower_bound_idx(cidx, M, i), k1 = lower_bound_idx(cidx, M, (long long)i + 1);
    double su[3] = {0.0, 0.0, 0.0};
    for (long long k = k0; k < k1; ++k) {
#pragma unroll
      for (int a = 0; a < 3; ++a) su[a] += (double)ctgt[3 * k + a];
    }
    const double cnt = (double)(k1 - k0);
    // (L^T L x)_i = sum_{j in N(i)} (L x)_j / deg_j - (L x)_i, and the diagonal of L^T L from L's entries: the
    // neighbours are ascending, so the repeats of a column are adjacent and are summed before squaring
    double lx[3], ltl[3];
    lap_f32(x, row_ptr, col, i, lx);
#pragma unroll
    for (int a = 0; a < 3; ++a) ltl[a] = -lx[a];
    const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
    const double inv_di = e1 > e0 ? rcp64((double)(e1 - e0)) : 0.0;
    double diag = 0.0, lii = -1.0;
    for (int e = e0; e < e1;) {
      const int j = col[e];
      int m = 0;
      for (; e < e1 && col[e] == j; ++e) {
        double lj[3];
        lap_f32(x, row_ptr, col, j, lj);
        const double inv_dj = rcp64((double)deg[j]);
#pragma unroll
        for (int a = 0; a < 3; ++a) ltl[a] += lj[a] * inv_dj;
        ++m;
      }
      if (j == i) {
        lii += (double)m * inv_di;
      } else {
        const double l = (double)m * rcp64((double)deg[j]);   // L_ji: i occurs m times in row j as j does in row i
        diag += l * l;
      }
    }
    diag += lii * lii + c * cnt;
    const double dinv = diag > 0.0 ? rcp64(diag) : 0.0;
    w.inv_deg[i] = inv_di;
    w.dinv[i] = dinv;
    w.cc[i] = c * cnt;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double xi = (double)x[3 * (long long)i + a];
      const double b = ltl[a] + c * su[a];
      const double r = c * (su[a] - cnt * xi);   // b - A x, exactly zero without a constraint
      const double z = dinv * r;
      w.y[a][i] = xi;
      w.r[a][i] = r;
      w.p[a][i] = z;
      bb[a] = b * b;
      rz[a] = r * z;
      rr[a] = r * r;
    }
  }
  block_sum3(bb, red);
  block_sum3(rz, red);
  block_sum3(rr, red);
  store_parts(w.part, blockIdx.x, 0, bb);
  store_parts(w.part, blockIdx.x, 3, rz);
  store_parts(w.part, blockIdx.x, 6, rr);
  if (blockIdx.x == 0 && threadIdx.x == 0)
    stats[7] = (float)(M - (lower_bound_idx(cidx, M, V) - lower_bound_idx(cidx, M, 0)));
}

// Jacobi-preconditioned CG over all iterations; every thread of every block holds the same column state.  The minimum
// of one block per SM lets ptxas keep that state in registers (it spills it otherwise).
__global__ void __launch_bounds__(kLapThreads, 1) lap_pcg_kernel(int V, const int* __restrict__ row_ptr,
                                                                const int* __restrict__ col, LapWs w, double tol,
                                                                int max_iter, float* __restrict__ stats) {
  __shared__ double red[3][kLapThreads];
  cg::grid_group grid = cg::this_grid();
  const long long nc = lap_chunks(V);
  // a column stops when |r|^2 <= tol^2 |b|^2, or when r.r (or, at the start, b.b) is not finite
  const double tol2 = tol * tol;
  double bb[3], rz[3], rr[3], t[3];
  reduce_parts(w.part, nc, 0, bb, red);
  reduce_parts(w.part, nc, 3, rz, red);
  reduce_parts(w.part, nc, 6, rr, red);
  bool active[3];
  int iters[3] = {0, 0, 0};
  bool nonfinite = false;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const bool finite = isfinite(rr[k]) && isfinite(bb[k]);
    if (!finite) nonfinite = true;
    active[k] = finite && !(rr[k] <= tol2 * bb[k]);
  }
  for (int it = 0; it < max_iter && (active[0] || active[1] || active[2]); ++it) {
    // w = L p
    for (long long ch = blockIdx.x; ch < nc; ch += gridDim.x) {
      const long long i = ch * kLapThreads + threadIdx.x;
      if (i < V) {
        const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
        double s[3] = {0.0, 0.0, 0.0};
        for (int e = e0; e < e1; ++e) {
          const int j = col[e];
#pragma unroll
          for (int k = 0; k < 3; ++k) s[k] += w.p[k][j];
        }
        const double inv = w.inv_deg[i];
#pragma unroll
        for (int k = 0; k < 3; ++k) w.w[k][i] = s[k] * inv - w.p[k][i];
      }
    }
    grid.sync();
    // q = A p = L^T w + c cnt p, and p.q
    for (long long ch = blockIdx.x; ch < nc; ch += gridDim.x) {
      const long long i = ch * kLapThreads + threadIdx.x;
      double pq[3] = {0.0, 0.0, 0.0};
      if (i < V) {
        const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
        double s[3] = {0.0, 0.0, 0.0};
        for (int e = e0; e < e1; ++e) {
          const int j = col[e];
          const double inv_dj = w.inv_deg[j];   // j has i as a neighbour: deg_j >= 1
#pragma unroll
          for (int k = 0; k < 3; ++k) s[k] += w.w[k][j] * inv_dj;
        }
        const double cc = w.cc[i];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double pk = w.p[k][i];
          const double q = s[k] - w.w[k][i] + cc * pk;
          w.q[k][i] = q;
          pq[k] = pk * q;
        }
      }
      block_sum3(pq, red);
      store_parts(w.part, ch, 0, pq);
    }
    grid.sync();
    double alpha[3];
    reduce_parts(w.part, nc, 0, t, red);
#pragma unroll
    for (int k = 0; k < 3; ++k) alpha[k] = rz[k] * rcp64(t[k]);
    // y += alpha p, r -= alpha q, z = r / diag; r.z and r.r
    for (long long ch = blockIdx.x; ch < nc; ch += gridDim.x) {
      const long long i = ch * kLapThreads + threadIdx.x;
      double pz[3] = {0.0, 0.0, 0.0}, pr[3] = {0.0, 0.0, 0.0};
      if (i < V) {
        const double dinv = w.dinv[i];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          if (!active[k]) continue;
          w.y[k][i] += alpha[k] * w.p[k][i];
          const double r = w.r[k][i] - alpha[k] * w.q[k][i];
          w.r[k][i] = r;
          pz[k] = r * (dinv * r);
          pr[k] = r * r;
        }
      }
      block_sum3(pz, red);
      block_sum3(pr, red);
      store_parts(w.part, ch, 3, pz);
      store_parts(w.part, ch, 6, pr);
    }
    grid.sync();
    double rz_new[3], rr_new[3], beta[3];
    reduce_parts(w.part, nc, 3, rz_new, red);
    reduce_parts(w.part, nc, 6, rr_new, red);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      beta[k] = 0.0;
      if (!active[k]) continue;
      ++iters[k];
      rr[k] = rr_new[k];
      if (!isfinite(rr[k])) {
        nonfinite = true;
        active[k] = false;
      } else if (rr[k] <= tol2 * bb[k]) {
        active[k] = false;
      } else {
        beta[k] = rz_new[k] * rcp64(rz[k]);
        rz[k] = rz_new[k];
      }
    }
    // p = z + beta p
    for (long long ch = blockIdx.x; ch < nc; ch += gridDim.x) {
      const long long i = ch * kLapThreads + threadIdx.x;
      if (i < V) {
        const double dinv = w.dinv[i];
#pragma unroll
        for (int k = 0; k < 3; ++k)
          if (active[k]) w.p[k][i] = dinv * w.r[k][i] + beta[k] * w.p[k][i];
      }
    }
    grid.sync();
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    bool converged = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      stats[k] = (float)iters[k];
      stats[3 + k] = (float)sqrt64(bb[k] > 0.0 ? rr[k] * rcp64(bb[k]) : rr[k]);
      converged = converged && rr[k] <= tol2 * bb[k];
    }
    stats[6] = nonfinite ? -1.f : (converged ? 1.f : 0.f);
  }
}

// y'_i = (1/deg_i) sum_{j in N(i), j != i} y_j (the reference's L with its diagonal zeroed; 0 at deg_i = 0)
__global__ void __launch_bounds__(kLapThreads) lap_finalize_kernel(int V, const int* __restrict__ row_ptr,
                                                                  const int* __restrict__ col, LapWs w, int smooth,
                                                                  float* __restrict__ out) {
  const int i = blockIdx.x * kLapThreads + threadIdx.x;
  if (i >= V) return;
  double o[3];
  if (smooth) {
    const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
    double s[3] = {0.0, 0.0, 0.0};
    for (int e = e0; e < e1; ++e) {
      const int j = col[e];
      if (j == i) continue;
#pragma unroll
      for (int k = 0; k < 3; ++k) s[k] += w.y[k][j];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) o[k] = s[k] * w.inv_deg[i];
  } else {
#pragma unroll
    for (int k = 0; k < 3; ++k) o[k] = w.y[k][i];
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) out[3 * (long long)i + k] = (float)o[k];
}

int lap_shape(long long V, long long M) {
  if (V < 0 || M < 0) return RECMV_E_SHAPE;
  if (V >= 0x7fffffffLL - kLapThreads) return RECMV_E_RANGE;   // int row pointers and vertex indices
  return RECMV_OK;
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_lap_edit_workspace_bytes(int64_t V, int64_t M, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  const int s = lap_shape(V, M);
  if (s) return s;
  *bytes = lap_ws_bytes(V);
  return RECMV_OK;
}

extern "C" int recmv_lap_edit_solve(const float* verts, int64_t V, const int32_t* row_ptr, const int32_t* col,
                                    const int32_t* deg, const int64_t* cidx, const float* ctgt, int64_t M,
                                    double constrain_weight, double tol, int max_iter, int smooth, int max_blocks,
                                    void* workspace, float* out, float* stats, recmv_stream_t stream) {
  int s = lap_shape(V, M);
  if (s) return s;
  if (max_iter < 1 || !(tol > 0.0) || !(constrain_weight >= 0.0) || max_blocks < 0) return RECMV_E_SHAPE;
  if (!row_ptr || !workspace || !stats || (V > 0 && (!verts || !deg || !out)) || (M > 0 && (!cidx || !ctgt)))
    return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  LapWs w = carve_lap(workspace, V);
  const long long nc = lap_chunks(V);
  const unsigned nb = (unsigned)(nc > 0 ? nc : 1);
  const int Vi = (int)V;
  lap_setup_kernel<<<nb, kLapThreads, 0, st>>>(verts, Vi, row_ptr, col, deg, (const long long*)cidx, ctgt, M,
                                               constrain_weight, w, stats);
  s = launch_status();
  if (s) return s;
  // every block must be co-resident for the grid syncs: at most what the occupancy allows, and no more than the chunks
  int per_sm = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lap_pcg_kernel, kLapThreads, 0);
  if (e != cudaSuccess) return (int)e;
  long long grid = (long long)per_sm * num_sms();
  if (grid > nc) grid = nc;
  if (max_blocks > 0 && grid > max_blocks) grid = max_blocks;
  if (grid < 1) grid = 1;
  void* args[] = {(void*)&Vi, (void*)&row_ptr, (void*)&col, (void*)&w, (void*)&tol, (void*)&max_iter,
                  (void*)&stats};
  e = cudaLaunchCooperativeKernel((const void*)lap_pcg_kernel, dim3((unsigned)grid), dim3(kLapThreads), args, 0, st);
  s = launch_status();
  if (e != cudaSuccess) return (int)e;
  if (s) return s;
  lap_finalize_kernel<<<nb, kLapThreads, 0, st>>>(Vi, row_ptr, col, w, smooth, out);
  return launch_status();
}

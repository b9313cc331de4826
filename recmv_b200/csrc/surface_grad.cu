// Per-ray algebra of the implicit-surface gradient (engineer/networks/OptimNetwork.py:726-879,
// propagateTmpPsGrad; garment variant OptimGarmentNetwork.py:2159-2313): the surface point p* of a ray is defined
// implicitly by  f(p) = 0  and  (D(p) - c) x v = 0;  its sensitivity to the network parameters is the
// least-squares solution of  b dp = rhs  with the 4 x 3 matrix  b = [grad f ; [v]x J]  (J = dD/dp).  Given the
// loss gradient g = dL/dp*, the reference forms  r = g (b^T b)^-1 b^T  (1 x 4) with FastMinv's singularity rule and
// then back-propagates  -r[0]  through the SDF network and  r[1:4] (-[v]x)  through the deformer.  This kernel does
// everything between the two network evaluations in registers: 21 floats in, 8 floats + 1 flag out per ray
// (the reference: ~40 small kernels and a FastMinv call on the legacy stream).
//
// recmv_implicit_grad (DESIGN section 1l) runs the same per-row algebra for all garments of a call, rows of garment g
// at [offsets[g], offsets[g+1]), and reduces per garment the ok count and cam_grad = -sum def_vec (the reference's
// invInfo[1] and `-temp.sum(0)`).  Rows are cut into fixed 1024-row chunks that never straddle two garments; each
// chunk's f64 sums and its count go to the workspace (frame_mean.cuh's block reductions), and one CTA per garment
// combines them in chunk order.  No atomics, and the partition does not depend on the grid, so the reductions are
// bit-identical from run to run and for any launch configuration.
#include "../../include/recmv_b200.h"
#include "../../include/recmv_b200_diag.h"   // recmv_implicit_grad_grid (diagnostics entry, not in the product header)
#include "common.cuh"
#include "frame_mean.cuh"

namespace recmv {
namespace {

// Row i: returns FastMinv's flag; coef = -r0, vec = r[1:4] (-[v]x), r = r[1:4].
__device__ __forceinline__ bool surface_grad_row(const float* __restrict__ gl, const float* __restrict__ gf,
                                                 const float* __restrict__ J, const float* __restrict__ v, long long i,
                                                 float& coef, float vec[3], float r[3]) {
  const float vx = __ldg(v + 3 * i), vy = __ldg(v + 3 * i + 1), vz = __ldg(v + 3 * i + 2);
  float Jm[9], a[9], b0[3], g[3];
#pragma unroll
  for (int e = 0; e < 9; ++e) Jm[e] = __ldg(J + 9 * i + e);
#pragma unroll
  for (int e = 0; e < 3; ++e) { b0[e] = __ldg(gf + 3 * i + e); g[e] = __ldg(gl + 3 * i + e); }
  // a = [v]x J : row 0 = -vz J1 + vy J2, row 1 = vz J0 - vx J2, row 2 = -vy J0 + vx J1
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    a[c] = -vz * Jm[3 + c] + vy * Jm[6 + c];
    a[3 + c] = vz * Jm[c] - vx * Jm[6 + c];
    a[6 + c] = -vy * Jm[c] + vx * Jm[3 + c];
  }
  // btb = b^T b = gf gf^T + a^T a
  float M[9], Mi[9];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c)
      M[3 * r + c] = b0[r] * b0[c] + a[r] * a[c] + a[3 + r] * a[3 + c] + a[6 + r] * a[6 + c];
  const bool good = inv3x3<float>(M, Mi);   // |det| < 1e-4 -> zeros, flag false (Matrix3x3InvKernels.cu:29-60)
  // w = (btb_inv b^T) contracted with g from the left: r = g btb_inv b^T  ->  w = g btb_inv (1 x 3)
  float w[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) w[c] = g[0] * Mi[c] + g[1] * Mi[3 + c] + g[2] * Mi[6 + c];
  const float r0 = w[0] * b0[0] + w[1] * b0[1] + w[2] * b0[2];
#pragma unroll
  for (int k = 0; k < 3; ++k) r[k] = w[0] * a[3 * k] + w[1] * a[3 * k + 1] + w[2] * a[3 * k + 2];
  coef = -r0;
  // temp = r (-[v]x) = -(r x ... ) : (r [v]x)_j = sum_i r_i [v]x_ij  = (r_1 vz - r_2 vy, -r_0 vz + r_2 vx, r_0 vy - r_1 vx)
  vec[0] = -(r[1] * vz - r[2] * vy);
  vec[1] = -(-r[0] * vz + r[2] * vx);
  vec[2] = -(r[0] * vy - r[1] * vx);
  return good;
}

// r [dc]x : the gradient w.r.t. the ray direction (OptimNetwork.py:862-873)
__device__ __forceinline__ void ray_grad_row(const float r[3], float dx, float dy, float dz, float* __restrict__ out) {
  out[0] = r[1] * dz - r[2] * dy;
  out[1] = -r[0] * dz + r[2] * dx;
  out[2] = r[0] * dy - r[1] * dx;
}

__global__ void __launch_bounds__(256) surface_grad_kernel(const float* __restrict__ gl, const float* __restrict__ gf,
                                                           const float* __restrict__ J, const float* __restrict__ v,
                                                           const float* __restrict__ dc, float* __restrict__ sdf_coef,
                                                           float* __restrict__ def_vec, float* __restrict__ ray_grad,
                                                           unsigned char* __restrict__ ok, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float coef, vec[3], r[3];
    const bool good = surface_grad_row(gl, gf, J, v, i, coef, vec, r);
    sdf_coef[i] = coef;
#pragma unroll
    for (int k = 0; k < 3; ++k) def_vec[3 * i + k] = vec[k];
    if (ray_grad) ray_grad_row(r, __ldg(dc + 3 * i), __ldg(dc + 3 * i + 1), __ldg(dc + 3 * i + 2), ray_grad + 3 * i);
    ok[i] = good ? 1 : 0;
  }
}

constexpr int kMaxGarments = 8;    // garments per launch pair; a call with more runs one pair per group

// a[g] by a select chain: a dynamic index into a kernel parameter would copy the parameter to the stack
template <class T>
__device__ __forceinline__ T pick(const T (&a)[kMaxGarments + 1], int g) {
  T v = a[0];
#pragma unroll
  for (int k = 1; k <= kMaxGarments; ++k)
    if (k == g) v = a[k];
  return v;
}

struct GarmentGroup {
  long long row0[kMaxGarments + 1];   // garment g's rows: [row0[g], row0[g+1])
  int chunk0[kMaxGarments + 1];       // its first chunk (within the call); chunk0[G] ends the group
  int g0;                             // index of garment 0 in the call
  int G;
};

struct RowIO {
  const float *gl, *gf, *J, *v, *d, *cam;
  float *sdf_coef, *def_vec, *ray_grad;
  unsigned char* ok;
};

// One chunk per CTA iteration: the rows' outputs, then the chunk's f64 sums of def_vec -> part_sum[3 t + k] and its
// ok count -> part_cnt[t].  The grid only decides which CTA handles a chunk, never the order of a sum.
__global__ void __launch_bounds__(kMeanThreads) implicit_grad_kernel(const GarmentGroup L, const RowIO io,
                                                                     double* __restrict__ part_sum,
                                                                     int* __restrict__ part_cnt) {
  __shared__ double red_d[kMeanThreads / 32];
  __shared__ int red_i[kMeanThreads / 32];
  float cx = 0.f, cy = 0.f, cz = 0.f;
  if (io.ray_grad) { cx = __ldg(io.cam); cy = __ldg(io.cam + 1); cz = __ldg(io.cam + 2); }
  const int chunks = pick(L.chunk0, L.G) - L.chunk0[0];
  for (int c = blockIdx.x; c < chunks; c += gridDim.x) {
    const int t = L.chunk0[0] + c;
    int g = 0;
#pragma unroll
    for (int k = 1; k < kMaxGarments; ++k)
      if (k < L.G && t >= L.chunk0[k]) g = k;
    const long long r0 = pick(L.row0, g) + (long long)(t - pick(L.chunk0, g)) * kChunkRows;
    const long long end = pick(L.row0, g + 1);
    const long long r1 = r0 + kChunkRows < end ? r0 + kChunkRows : end;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    int n = 0;
#pragma unroll
    for (int k = 0; k < kRowsPerThread; ++k) {
      const long long i = r0 + k * kMeanThreads + threadIdx.x;
      if (i < r1) {
        float coef, vec[3], r[3];
        const bool good = surface_grad_row(io.gl, io.gf, io.J, io.v, i, coef, vec, r);
        io.sdf_coef[i] = coef;
#pragma unroll
        for (int a = 0; a < 3; ++a) io.def_vec[3 * i + a] = vec[a];
        if (io.ray_grad) {   // d - c formed here, one f32 rounding per coordinate
          const float dx = __fsub_rn(__ldg(io.d + 3 * i), cx), dy = __fsub_rn(__ldg(io.d + 3 * i + 1), cy);
          const float dz = __fsub_rn(__ldg(io.d + 3 * i + 2), cz);
          ray_grad_row(r, dx, dy, dz, io.ray_grad + 3 * i);
        }
        io.ok[i] = good ? 1 : 0;
        s0 += (double)vec[0];
        s1 += (double)vec[1];
        s2 += (double)vec[2];
        n += good ? 1 : 0;
      }
    }
    s0 = block_sum(s0, red_d);
    s1 = block_sum(s1, red_d);
    s2 = block_sum(s2, red_d);
    n = block_count(n, red_i);
    if (threadIdx.x == 0) {
      part_sum[3 * (size_t)t] = s0;
      part_sum[3 * (size_t)t + 1] = s1;
      part_sum[3 * (size_t)t + 2] = s2;
      part_cnt[t] = n;
    }
  }
}

// One CTA per garment: its chunk partials combined in chunk order (strided by thread, then the block tree).
__global__ void __launch_bounds__(kMeanThreads) implicit_grad_finish_kernel(const GarmentGroup L,
                                                                            const double* __restrict__ part_sum,
                                                                            const int* __restrict__ part_cnt,
                                                                            int* __restrict__ ok_count,
                                                                            float* __restrict__ cam_grad) {
  __shared__ double red_d[kMeanThreads / 32];
  __shared__ int red_i[kMeanThreads / 32];
  const int g = blockIdx.x;
  double s[3] = {0.0, 0.0, 0.0};
  int n = 0;
  const int t1 = pick(L.chunk0, g + 1);
  for (int t = pick(L.chunk0, g) + threadIdx.x; t < t1; t += kMeanThreads) {
#pragma unroll
    for (int a = 0; a < 3; ++a) s[a] += part_sum[3 * (size_t)t + a];
    n += part_cnt[t];
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) s[a] = block_sum(s[a], red_d);
  n = block_count(n, red_i);
  if (threadIdx.x == 0) {
    ok_count[L.g0 + g] = n;
    if (cam_grad)
#pragma unroll
      for (int a = 0; a < 3; ++a) cam_grad[3 * (L.g0 + g) + a] = __double2float_rn(-s[a]);
  }
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

long long chunks_of(long long rows) { return (rows + kChunkRows - 1) / kChunkRows; }

// an upper bound of the call's chunks: every garment adds at most one partial chunk
long long max_chunks(int64_t n, int G) { return n / kChunkRows + G + 1; }

int grad_sizes(int64_t n, int G) {
  if (n < 0 || G < 0) return RECMV_E_SHAPE;
  if (n > 0x7fffffffLL) return RECMV_E_RANGE;
  return RECMV_OK;
}

int implicit_grad(const float* grad_l_p, const float* grad_f_p, const float* jac, const float* rays, const float* d,
                  const float* cam_pos, const int64_t* offsets, int G, float* sdf_coef, float* def_vec,
                  float* ray_grad, uint8_t* ok, int32_t* ok_count, float* cam_grad, void* workspace, int64_t n,
                  int max_ctas, cudaStream_t st) {
  int s = grad_sizes(n, G);
  if (s) return s;
  if (G == 0) return n == 0 ? RECMV_OK : RECMV_E_SHAPE;
  if (!offsets || !ok_count || !workspace) return RECMV_E_NULL;
  if (offsets[0] != 0 || offsets[G] != n) return RECMV_E_SHAPE;
  for (int g = 0; g < G; ++g)
    if (offsets[g + 1] < offsets[g]) return RECMV_E_SHAPE;
  if (n > 0 && (!grad_l_p || !grad_f_p || !jac || !rays || !sdf_coef || !def_vec || !ok)) return RECMV_E_NULL;
  if (ray_grad && (!d || !cam_pos)) return RECMV_E_NULL;
  const RowIO io{grad_l_p, grad_f_p, jac, rays, d, cam_pos, sdf_coef, def_vec, ray_grad, (unsigned char*)ok};
  double* part_sum = (double*)workspace;
  int* part_cnt = (int*)((char*)workspace + align256((size_t)max_chunks(n, G) * 3 * sizeof(double)));
  const int cap = num_sms() * 4;   // the row kernel's residency at 62 registers
  int chunk = 0;
  for (int g0 = 0; g0 < G; g0 += kMaxGarments) {
    GarmentGroup L = {};
    L.g0 = g0;
    L.G = G - g0 < kMaxGarments ? G - g0 : kMaxGarments;
    for (int g = 0; g < L.G; ++g) {
      L.row0[g] = offsets[g0 + g];
      L.chunk0[g] = chunk;
      chunk += (int)chunks_of(offsets[g0 + g + 1] - offsets[g0 + g]);
    }
    L.row0[L.G] = offsets[g0 + L.G];
    L.chunk0[L.G] = chunk;
    const int chunks = L.chunk0[L.G] - L.chunk0[0];
    if (chunks > 0) {
      int grid = chunks < cap ? chunks : cap;
      if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
      implicit_grad_kernel<<<grid, kMeanThreads, 0, st>>>(L, io, part_sum, part_cnt);
      if ((s = launch_status())) return s;
    }
    implicit_grad_finish_kernel<<<L.G, kMeanThreads, 0, st>>>(L, part_sum, part_cnt, ok_count, cam_grad);
    if ((s = launch_status())) return s;
  }
  return RECMV_OK;
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_surface_grad_coeffs(const float* grad_l_p, const float* grad_f_p, const float* jac,
                                         const float* rays, const float* d_minus_c, float* sdf_coef, float* def_vec,
                                         float* ray_grad, uint8_t* ok, int64_t n, recmv_stream_t stream) {
  if (n < 0) return RECMV_E_SHAPE;
  if (n == 0) return RECMV_OK;
  if (!grad_l_p || !grad_f_p || !jac || !rays || !sdf_coef || !def_vec || !ok) return RECMV_E_NULL;
  if (ray_grad && !d_minus_c) return RECMV_E_NULL;
  surface_grad_kernel<<<stride_grid(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(grad_l_p, grad_f_p, jac, rays, d_minus_c,
                                                                               sdf_coef, def_vec, ray_grad, ok, n);
  return launch_status();
}

extern "C" int recmv_implicit_grad_workspace_bytes(int64_t n, int G, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  const int s = grad_sizes(n, G);
  if (s) return s;
  const size_t chunks = (size_t)max_chunks(n, G);
  *bytes = align256(chunks * 3 * sizeof(double)) + align256(chunks * sizeof(int));
  return RECMV_OK;
}

extern "C" int recmv_implicit_grad(const float* grad_l_p, const float* grad_f_p, const float* jac, const float* rays,
                                   const float* d, const float* cam_pos, const int64_t* offsets, int G,
                                   float* sdf_coef, float* def_vec, float* ray_grad, uint8_t* ok, int32_t* ok_count,
                                   float* cam_grad, void* workspace, int64_t n, recmv_stream_t stream) {
  return implicit_grad(grad_l_p, grad_f_p, jac, rays, d, cam_pos, offsets, G, sdf_coef, def_vec, ray_grad, ok, ok_count,
                       cam_grad, workspace, n, 0, (cudaStream_t)stream);
}

extern "C" int recmv_implicit_grad_grid(const float* grad_l_p, const float* grad_f_p, const float* jac,
                                        const float* rays, const float* d, const float* cam_pos, const int64_t* offsets,
                                        int G, float* sdf_coef, float* def_vec, float* ray_grad, uint8_t* ok,
                                        int32_t* ok_count, float* cam_grad, void* workspace, int64_t n, int max_ctas,
                                        recmv_stream_t stream) {
  return implicit_grad(grad_l_p, grad_f_p, jac, rays, d, cam_pos, offsets, G, sdf_coef, def_vec, ray_grad, ok, ok_count,
                       cam_grad, workspace, n, max_ctas, (cudaStream_t)stream);
}

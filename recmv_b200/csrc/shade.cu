// Shading of the rasterized garment meshes (DESIGN section 1d): deterministic per-vertex normals and a hard Phong pass
// over the K = 1 fragments of raster.cu.  Replaces pytorch3d's `Meshes.verts_normals_packed` and the `HardPhongShader`
// that `infer_fl.py` installs behind `maskRender`.
//
// Vertex normals, verts [N,V,3] with one face list [F,3] shared by the N frames:
//   every (face f, corner k) pair contributes cross(v[k+1] - v[k], v[k+2] - v[k]) (indices cyclic) to vertex faces[f][k];
//   n / max(|n|, 1e-6).  The sum runs in increasing (face, corner) order -- no float atomics, so the result is
//   bit-identical from run to run and independent of the SM count.  A face with an index outside [0, V) contributes
//   nothing; a vertex no face references gets 0.
//   1. corner_keys_kernel    one thread per (face, corner) e = 3 f + k: key = its vertex (V for an invalid face), value e
//                            (segments.cuh);
//   2. CUB radix sort        stable, so each vertex's values stay in increasing e order;
//   3. segment_bounds_kernel the [begin, end) range of every vertex in the sorted list (segments.cuh);
//   4. normals_sum_kernel    one thread per (frame, vertex): sum its range in order and normalise.
//
// Hard Phong, one thread per pixel: interpolate world position, vertex normal and vertex colour of the winning face
// with the perspective-corrected barycentrics, then ambient + diffuse + specular of one point light (pytorch3d's
// `phong_shading` with `hard_rgb_blend`: alpha 1, background colour where no face was hit).
#include <math.h>

#include "common.cuh"
#include "segments.cuh"

namespace recmv {
namespace {

constexpr int kNormThreads = 256;
constexpr int kShadeThreads = 256;
constexpr int kShadeParams = 28;   // per-frame constants, layout in include/recmv_b200.h

// |(x, y, z)|^2 in the order the sm_90a compiler contracts the plain x * x + y * y + z * z to, written out so that the
// float32 restatement in tests/shade_f32.py is exact: y * y rounded, then x and z fused.
__device__ __forceinline__ float norm2(float x, float y, float z) {
  return __fmaf_rn(z, z, __fmaf_rn(x, x, __fmul_rn(y, y)));
}

__global__ void __launch_bounds__(kNormThreads) normals_sum_kernel(const float* __restrict__ verts, int V,
                                                                    const long long* __restrict__ faces,
                                                                    const unsigned* __restrict__ vals,
                                                                    const int* __restrict__ beg,
                                                                    const int* __restrict__ end, long long NV,
                                                                    float* __restrict__ out) {
  const long long gid = blockIdx.x * (long long)kNormThreads + threadIdx.x;
  if (gid >= NV) return;
  const long long n = gid / V;
  const int v = (int)(gid - n * V);
  const float* fv = verts + n * V * 3;
  const float px = fv[3 * (long long)v], py = fv[3 * (long long)v + 1], pz = fv[3 * (long long)v + 2];
  float sx = 0.f, sy = 0.f, sz = 0.f;
  const int e0 = beg[v], e1 = end[v];
  for (int i = e0; i < e1; ++i) {
    const unsigned e = vals[i];
    const unsigned f = e / 3u, k = e - 3u * f;
    const long long* fc = faces + 3 * (long long)f;
    const long long b = fc[k == 2u ? 0 : k + 1], c = fc[k == 0u ? 2 : k - 1];
    const float* pb = fv + 3 * b;
    const float* pc = fv + 3 * c;
    const float ux = pb[0] - px, uy = pb[1] - py, uz = pb[2] - pz;
    const float wx = pc[0] - px, wy = pc[1] - py, wz = pc[2] - pz;
    // each product rounded on its own (no contraction), so a face with two coincident corners adds exactly 0
    sx += __fsub_rn(__fmul_rn(uy, wz), __fmul_rn(uz, wy));
    sy += __fsub_rn(__fmul_rn(uz, wx), __fmul_rn(ux, wz));
    sz += __fsub_rn(__fmul_rn(ux, wy), __fmul_rn(uy, wx));
  }
  const float inv = 1.f / fmaxf(sqrtf(norm2(sx, sy, sz)), 1e-6f);
  float* o = out + 3 * gid;
  o[0] = sx * inv; o[1] = sy * inv; o[2] = sz * inv;
}

__device__ __forceinline__ void normalize3(float& x, float& y, float& z) {
  const float inv = 1.f / fmaxf(sqrtf(norm2(x, y, z)), 1e-6f);
  x *= inv; y *= inv; z *= inv;
}

// A correctly rounded a * b + c.  The interpolation uses the PTX instruction rather than __fmaf_rn: the two round alike,
// but the intrinsic leads ptxas to a different schedule than the one the plain, contracted expression compiled to.
__device__ __forceinline__ float fma_rn(float a, float b, float c) {
  float d;
  asm("fma.rn.f32 %0, %1, %2, %3;" : "=f"(d) : "f"(a), "f"(b), "f"(c));
  return d;
}

__global__ void __launch_bounds__(kShadeThreads) shade_phong_kernel(
    const long long* __restrict__ pix_to_face, const float* __restrict__ bary, const float* __restrict__ verts,
    const float* __restrict__ normals, const float* __restrict__ colors, const long long* __restrict__ faces,
    long long F, int V, int N, long long HW, const float* __restrict__ params, float4* __restrict__ out) {
  const long long pix = blockIdx.x * (long long)kShadeThreads + threadIdx.x;
  if (pix >= (long long)N * HW) return;
  const float* prm = params + kShadeParams * (pix / HW);
  const float4 bg = make_float4(__ldg(prm + 25), __ldg(prm + 26), __ldg(prm + 27), 1.f);
  const long long p = pix_to_face[pix];
  if (p < 0 || p >= (long long)N * F) { out[pix] = bg; return; }
  const long long m = p / F, f = p - m * F;
  long long vi[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    vi[k] = __ldg(faces + 3 * f + k);
    if (vi[k] < 0 || vi[k] >= V) { out[pix] = bg; return; }
    vi[k] += m * V;
  }
  const float b[3] = {bary[3 * pix], bary[3 * pix + 1], bary[3 * pix + 2]};
  // Every contraction is written out, in the order the compiler chose for the plain expressions, so that the float32
  // restatement in tests/shade_f32.py is exact; powf is the one operation it does not restate.  The interpolation is
  // a fused chain over the corners from +0: fma(b2, a2, fma(b1, a1, fma(b0, a0, 0))).
  float P[3] = {0.f, 0.f, 0.f}, Nr[3] = {0.f, 0.f, 0.f}, C[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      P[j] = fma_rn(b[k], __ldg(verts + 3 * vi[k] + j), P[j]);
      Nr[j] = fma_rn(b[k], __ldg(normals + 3 * vi[k] + j), Nr[j]);
      C[j] = fma_rn(b[k], colors ? __ldg(colors + 3 * vi[k] + j) : 1.f, C[j]);
    }
  float nx = Nr[0], ny = Nr[1], nz = Nr[2];
  normalize3(nx, ny, nz);
  float lx = __ldg(prm + 3) - P[0], ly = __ldg(prm + 4) - P[1], lz = __ldg(prm + 5) - P[2];
  normalize3(lx, ly, lz);
  float vx = __ldg(prm + 0) - P[0], vy = __ldg(prm + 1) - P[1], vz = __ldg(prm + 2) - P[2];
  normalize3(vx, vy, vz);
  // dot products in norm2's order; R = 2 cos N - L with 2 cos exact and each product fused with -L
  const float cosl = __fmaf_rn(nz, lz, __fmaf_rn(nx, lx, __fmul_rn(ny, ly)));
  const float c2 = 2.f * cosl;
  const float rx = __fmaf_rn(nx, c2, -lx), ry = __fmaf_rn(ny, c2, -ly), rz = __fmaf_rn(nz, c2, -lz);
  const float sa = cosl > 0.f ? fmaxf(__fmaf_rn(vz, rz, __fmaf_rn(vx, rx, __fmul_rn(vy, ry))), 0.f) : 0.f;
  const float spec = powf(sa, __ldg(prm + 24));
  const float dif = fmaxf(cosl, 0.f);
  float rgb[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    // (ambient + diffuse) colour + specular: the ambient product fused into the sum, that sum fused with the colour
    const float ma = __ldg(prm + 15 + j), la = __ldg(prm + 6 + j);
    const float d = __fmul_rn(__fmul_rn(__ldg(prm + 18 + j), __ldg(prm + 9 + j)), dif);
    const float s = __fmul_rn(__fmul_rn(__ldg(prm + 21 + j), __ldg(prm + 12 + j)), spec);
    rgb[j] = __fmaf_rn(__fmaf_rn(ma, la, d), C[j], s);
  }
  out[pix] = make_float4(rgb[0], rgb[1], rgb[2], 1.f);
}

int normals_shape(int V, int64_t F) {
  if (V < 0 || F < 0) return RECMV_E_SHAPE;
  if (3 * F > 0x7fffffffLL || V == 0x7fffffff) return RECMV_E_RANGE;   // int list positions; V is the sentinel key
  return RECMV_OK;
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_vertex_normals_workspace_bytes(int V, int64_t F, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  int s = normals_shape(V, F);
  if (s) return s;
  const long long M = 3 * (long long)F;
  size_t temp = 0;
  s = sort_temp_bytes(M, (unsigned)V, &temp);
  if (s) return s;
  *bytes = layout_bytes(segment_layout, M, V) + temp;
  return RECMV_OK;
}

extern "C" int recmv_vertex_normals(const float* verts, int N, int V, const int64_t* faces, int64_t F, void* workspace,
                                    float* out_normals, recmv_stream_t stream) {
  int s = normals_shape(V, F);
  if (s) return s;
  if (N < 0) return RECMV_E_SHAPE;
  if ((int64_t)N * V > ((int64_t)1 << 38)) return RECMV_E_RANGE;   // grid.x of the per-vertex pass
  if ((long long)N * V == 0) return RECMV_OK;
  if (!verts || !out_normals || !workspace || (F > 0 && !faces)) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  const long long M = 3 * (long long)F;
  const SegmentWs w = carve(workspace, segment_layout, M, V);
  cudaError_t e = cudaMemsetAsync(w.beg, 0, w.ranges_bytes, st);   // beg and end: empty ranges
  if (e != cudaSuccess) return (int)e;
  if (M > 0) {
    const int nb = (int)((M + kSegThreads - 1) / kSegThreads);
    corner_keys_kernel<<<nb, kSegThreads, 0, st>>>((const long long*)faces, M, V, w.keys_in, w.vals_in, nullptr);
    s = launch_status();
    if (s) return s;
    s = sort_pairs(w.temp, w.keys_in, w.keys_out, w.vals_in, w.vals_out, M, (unsigned)V, st);
    if (s) return s;
    segment_bounds_kernel<<<(unsigned)((M + kSegThreads - 1) / kSegThreads), kSegThreads, 0, st>>>(
        w.keys_out, M, (unsigned)V, w.beg, w.end);
    s = launch_status();
    if (s) return s;
  }
  const long long NV = (long long)N * V;
  normals_sum_kernel<<<(unsigned)((NV + kNormThreads - 1) / kNormThreads), kNormThreads, 0, st>>>(
      verts, V, (const long long*)faces, w.vals_out, w.beg, w.end, NV, out_normals);
  return launch_status();
}

extern "C" int recmv_shade_phong(const int64_t* pix_to_face, const float* bary, int N, int H, int W, const float* verts,
                                 const float* normals, const float* colors, int V, const int64_t* faces, int64_t F,
                                 const float* params, float* out_rgba, recmv_stream_t stream) {
  if (N < 0 || H < 0 || W < 0 || V < 0 || F < 0) return RECMV_E_SHAPE;
  if ((int64_t)N * H * W > 0x7fffffffffffLL || (int64_t)N * F > 0x7fffffffffffLL) return RECMV_E_RANGE;
  const long long npix = (long long)N * H * W;
  if (npix == 0) return RECMV_OK;
  if (!pix_to_face || !bary || !params || !out_rgba) return RECMV_E_NULL;
  if (V > 0 && F > 0 && (!verts || !normals || !faces)) return RECMV_E_NULL;
  if (((uintptr_t)out_rgba & 15) != 0) return RECMV_E_DTYPE;   // one float4 per pixel
  const long long blocks = (npix + kShadeThreads - 1) / kShadeThreads;
  if (blocks > 0x7fffffffLL) return RECMV_E_RANGE;
  // with no faces (or no vertices) every pixel is background: F = 0 makes every pix_to_face out of range
  shade_phong_kernel<<<(unsigned)blocks, kShadeThreads, 0, (cudaStream_t)stream>>>(
      (const long long*)pix_to_face, bary, verts, normals, colors, (const long long*)faces, V > 0 ? F : 0, V, N,
      (long long)H * W, params, reinterpret_cast<float4*>(out_rgba));
  return launch_status();
}

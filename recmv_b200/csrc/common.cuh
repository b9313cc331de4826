// Shared helpers for librecmv_b200.so (sm_100a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/recmv_b200.h"

namespace recmv {

extern unsigned long long g_launch_count;  // defined in capi.cu

inline int launch_status() {
  ++g_launch_count;
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) {
    cudaGetLastError();  // clear
    return (int)e;
  }
  return RECMV_OK;
}

inline int num_sms() {
  static int cached[16] = {0};   // per device
  int dev = 0;
  cudaGetDevice(&dev);
  int& n = cached[dev & 15];
  if (n == 0) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 148;
  }
  return n;
}

// grid for a grid-stride kernel: a whole number of waves over the SMs (148 on B200)
inline int stride_grid(int64_t work, int threads, int ctas_per_sm) {
  int64_t need = (work + threads - 1) / threads;
  int64_t cap = (int64_t)num_sms() * ctas_per_sm;
  if (need < 1) need = 1;
  return (int)(need < cap ? need : cap);
}

// Skinning voxel, channels-last [D,H,W,24] fp32, with the reference's normalisation
// nps = 2 (p - c) / e   (model/Deformer.py:342-355)
struct Voxel {
  const float* ws;
  int D, H, W;
  float cx, cy, cz, ext;
};

inline Voxel to_voxel(const recmv_voxel_t* v) {
  Voxel o;
  o.ws = v->ws_cl; o.D = v->D; o.H = v->H; o.W = v->W;
  o.cx = v->center[0]; o.cy = v->center[1]; o.cz = v->center[2]; o.ext = v->extend;
  return o;
}

// ((g+1)*S-1)/2 exactly as GridSamplerMineKernel.cu:210-212 (the double literals there only
// postpone one rounding across an exact halving, so the float result is identical), without
// letting the compiler contract mul+sub into an FMA.
__device__ __forceinline__ float unnormalize(float g, int size) {
  float t = __fmul_rn(__fadd_rn(g, 1.f), (float)size);
  return __fmul_rn(__fsub_rn(t, 1.f), 0.5f);
}
__device__ __forceinline__ double unnormalize(double g, int size) {
  return ((g + 1.0) * (double)size - 1.0) / 2.0;
}

// clip_coordinates_set_grad (GridSamplerMineKernel.cu:42-59)
template <typename T>
__device__ __forceinline__ T clip_grad(T in, int size, T* mult) {
  if (in <= (T)0) { *mult = (T)0; return (T)0; }
  T mx = (T)(size - 1);
  if (in >= mx) { *mult = (T)0; return mx; }
  *mult = (T)1;
  return in;
}

// Trilinear sample of the 24-channel channels-last skinning voxel at normalised point (gx,gy,gz).
// Border-clamped coordinates can only address in-range corners or corners with zero weight, so the
// reference's within_bounds tests reduce to clamping the +1 index.
__device__ __forceinline__ void sample_skin24(const Voxel& v, float px, float py, float pz,
                                              float w[24]) {
  float gx = (px - v.cx) / v.ext * 2.f;
  float gy = (py - v.cy) / v.ext * 2.f;
  float gz = (pz - v.cz) / v.ext * 2.f;
  float ix = fminf(fmaxf(unnormalize(gx, v.W), 0.f), (float)(v.W - 1));
  float iy = fminf(fmaxf(unnormalize(gy, v.H), 0.f), (float)(v.H - 1));
  float iz = fminf(fmaxf(unnormalize(gz, v.D), 0.f), (float)(v.D - 1));
  if (!(ix == ix)) ix = 0.f;  // NaN guard (reference maps non-finite to -100 => zero output)
  if (!(iy == iy)) iy = 0.f;
  if (!(iz == iz)) iz = 0.f;
  int x0 = (int)floorf(ix), y0 = (int)floorf(iy), z0 = (int)floorf(iz);
  float fx = ix - (float)x0, fy = iy - (float)y0, fz = iz - (float)z0;
  int x1 = min(x0 + 1, v.W - 1), y1 = min(y0 + 1, v.H - 1), z1 = min(z0 + 1, v.D - 1);
  float wx[2] = {(float)(x0 + 1) - ix, fx};
  float wy[2] = {(float)(y0 + 1) - iy, fy};
  float wz[2] = {(float)(z0 + 1) - iz, fz};
  int xs[2] = {x0, x1}, ys[2] = {y0, y1}, zs[2] = {z0, z1};
#pragma unroll
  for (int c = 0; c < 24; ++c) w[c] = 0.f;
  // corner order tnw,tne,tsw,tse,bnw,bne,bsw,bse = (z,y,x) with x fastest, as the reference sums
#pragma unroll
  for (int dz = 0; dz < 2; ++dz)
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        float cw = wx[dx] * wy[dy] * wz[dz];
        const float4* p = reinterpret_cast<const float4*>(
            v.ws + (((size_t)zs[dz] * v.H + ys[dy]) * v.W + xs[dx]) * 24);
#pragma unroll
        for (int q = 0; q < 6; ++q) {
          float4 t = __ldg(p + q);
          w[4 * q + 0] = fmaf(t.x, cw, w[4 * q + 0]);
          w[4 * q + 1] = fmaf(t.y, cw, w[4 * q + 1]);
          w[4 * q + 2] = fmaf(t.z, cw, w[4 * q + 2]);
          w[4 * q + 3] = fmaf(t.w, cw, w[4 * q + 3]);
        }
      }
}

// T[0..11] = rows 0..2 of sum_j w_j A_j  (A_j 4x4 row-major, 16 floats per bone)
__device__ __forceinline__ void blend_bones(const float* __restrict__ Af, const float w[24],
                                            float T[12]) {
#pragma unroll
  for (int e = 0; e < 12; ++e) T[e] = 0.f;
#pragma unroll 4
  for (int j = 0; j < 24; ++j) {
    const float4* a = reinterpret_cast<const float4*>(Af + j * 16);
    float4 r0 = __ldg(a), r1 = __ldg(a + 1), r2 = __ldg(a + 2);
    float wj = w[j];
    T[0] = fmaf(wj, r0.x, T[0]); T[1] = fmaf(wj, r0.y, T[1]); T[2] = fmaf(wj, r0.z, T[2]); T[3] = fmaf(wj, r0.w, T[3]);
    T[4] = fmaf(wj, r1.x, T[4]); T[5] = fmaf(wj, r1.y, T[5]); T[6] = fmaf(wj, r1.z, T[6]); T[7] = fmaf(wj, r1.w, T[7]);
    T[8] = fmaf(wj, r2.x, T[8]); T[9] = fmaf(wj, r2.y, T[9]); T[10] = fmaf(wj, r2.z, T[10]); T[11] = fmaf(wj, r2.w, T[11]);
  }
}

// In-register 3x3 inverse with the FastMinv rule (Matrix3x3InvKernels.cu:29-60).
// m row-major 9 floats; returns false (and zeros) when |det| < 1e-4.
template <typename T>
__device__ __forceinline__ bool inv3x3(const T m[9], T inv[9]) {
  T c00 = m[4] * m[8] - m[5] * m[7];
  T c01 = -m[3] * m[8] + m[5] * m[6];
  T c02 = m[3] * m[7] - m[4] * m[6];
  T c10 = -m[1] * m[8] + m[2] * m[7];
  T c11 = m[0] * m[8] - m[2] * m[6];
  T c12 = -m[0] * m[7] + m[1] * m[6];
  T c20 = m[1] * m[5] - m[2] * m[4];
  T c21 = -m[0] * m[5] + m[2] * m[3];
  T c22 = m[0] * m[4] - m[1] * m[3];
  T det = m[0] * c00 + m[1] * c01 + m[2] * c02;
  if (fabs(det) < (T)0.0001) {
#pragma unroll
    for (int i = 0; i < 9; ++i) inv[i] = (T)0;
    return false;
  }
  inv[0] = c00 / det; inv[1] = c10 / det; inv[2] = c20 / det;
  inv[3] = c01 / det; inv[4] = c11 / det; inv[5] = c21 / det;
  inv[6] = c02 / det; inv[7] = c12 / det; inv[8] = c22 / det;
  return true;
}

// Inverse LBS of one observation-space point (SURVEY 8a row A5').
__device__ __forceinline__ bool inverse_lbs_point(const Voxel& v, const float* __restrict__ Af,
                                                  const float* __restrict__ tf, float ox, float oy,
                                                  float oz, float& cx, float& cy, float& cz) {
  float w[24], T[12];
  sample_skin24(v, ox, oy, oz, w);
  blend_bones(Af, w, T);
  float M[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
  float Mi[9];
  bool ok = inv3x3<float>(M, Mi);
  float rx = ox - __ldg(tf + 0) - T[3];
  float ry = oy - __ldg(tf + 1) - T[7];
  float rz = oz - __ldg(tf + 2) - T[11];
  cx = Mi[0] * rx + Mi[1] * ry + Mi[2] * rz;
  cy = Mi[3] * rx + Mi[4] * ry + Mi[5] * rz;
  cz = Mi[6] * rx + Mi[7] * ry + Mi[8] * rz;
  return ok;
}

// LBS forward of one canonical point WITH its Jacobian: x' = T(w(q)) [q;1] + trans and
//   d x'_i / d q_j = T_ij + sum_bones (A_b [q;1])_i * d w_b / d q_j
// (the weights are sampled at q itself, LBSkinner.forward, model/Deformer.py:406-445; d w / d q follows the
// sampler's backward, GridSamplerMineKernel.cu:42-59,330-520: factor size/2 * 2/extend per axis, zero on an axis
// whose coordinate was clamped).  Evaluated corner by corner -- T_c = sum_b ws[corner][b] A_b, Y_c = T_c [q;1] --
// so nothing of size 24 x 3 is ever live in registers.
//
// lbs_blend_jac is the shared core: the weights are sampled at s and the blended transform is applied to a (the
// `[tps, ps]` form of LBSkinner.repose samples at tps and moves ps).  It returns T (rows 0..2 of sum_b w_b A_b) and
// only the weight term Jw_ij = sum_b (A_b [a;1])_i * d w_b / d s_j; lbs_forward_jac is the case s = a.
__device__ __forceinline__ void lbs_blend_jac(const Voxel& v, const float* __restrict__ Af, float sx, float sy,
                                              float sz, float qx, float qy, float qz, float T[12], float J[9]) {
  float gx = (sx - v.cx) / v.ext * 2.f;
  float gy = (sy - v.cy) / v.ext * 2.f;
  float gz = (sz - v.cz) / v.ext * 2.f;
  float mx, my, mz;
  float ix = clip_grad<float>(unnormalize(gx, v.W), v.W, &mx);
  float iy = clip_grad<float>(unnormalize(gy, v.H), v.H, &my);
  float iz = clip_grad<float>(unnormalize(gz, v.D), v.D, &mz);
  if (!(ix == ix)) { ix = 0.f; mx = 0.f; }
  if (!(iy == iy)) { iy = 0.f; my = 0.f; }
  if (!(iz == iz)) { iz = 0.f; mz = 0.f; }
  mx *= (float)v.W / v.ext; my *= (float)v.H / v.ext; mz *= (float)v.D / v.ext;   // d i / d q
  int x0 = (int)floorf(ix), y0 = (int)floorf(iy), z0 = (int)floorf(iz);
  int x1 = min(x0 + 1, v.W - 1), y1 = min(y0 + 1, v.H - 1), z1 = min(z0 + 1, v.D - 1);
  const float wx[2] = {(float)(x0 + 1) - ix, ix - (float)x0};
  const float wy[2] = {(float)(y0 + 1) - iy, iy - (float)y0};
  const float wz[2] = {(float)(z0 + 1) - iz, iz - (float)z0};
  const int xs[2] = {x0, x1}, ys[2] = {y0, y1}, zs[2] = {z0, z1};
#pragma unroll
  for (int e = 0; e < 12; ++e) T[e] = 0.f;
#pragma unroll
  for (int e = 0; e < 9; ++e) J[e] = 0.f;
#pragma unroll 1
  for (int c = 0; c < 8; ++c) {
    const int dx = c & 1, dy = (c >> 1) & 1, dz = c >> 2;
    const float* wsp = v.ws + (((size_t)zs[dz] * v.H + ys[dy]) * v.W + xs[dx]) * 24;
    float Tc[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) Tc[e] = 0.f;
#pragma unroll 4
    for (int b = 0; b < 24; ++b) {
      const float wb = __ldg(wsp + b);
      const float4* a = reinterpret_cast<const float4*>(Af + b * 16);
      const float4 r0 = __ldg(a), r1 = __ldg(a + 1), r2 = __ldg(a + 2);
      Tc[0] = fmaf(wb, r0.x, Tc[0]); Tc[1] = fmaf(wb, r0.y, Tc[1]); Tc[2] = fmaf(wb, r0.z, Tc[2]); Tc[3] = fmaf(wb, r0.w, Tc[3]);
      Tc[4] = fmaf(wb, r1.x, Tc[4]); Tc[5] = fmaf(wb, r1.y, Tc[5]); Tc[6] = fmaf(wb, r1.z, Tc[6]); Tc[7] = fmaf(wb, r1.w, Tc[7]);
      Tc[8] = fmaf(wb, r2.x, Tc[8]); Tc[9] = fmaf(wb, r2.y, Tc[9]); Tc[10] = fmaf(wb, r2.z, Tc[10]); Tc[11] = fmaf(wb, r2.w, Tc[11]);
    }
    const float cw = wx[dx] * wy[dy] * wz[dz];
#pragma unroll
    for (int e = 0; e < 12; ++e) T[e] = fmaf(cw, Tc[e], T[e]);
    const float Y[3] = {Tc[0] * qx + Tc[1] * qy + Tc[2] * qz + Tc[3], Tc[4] * qx + Tc[5] * qy + Tc[6] * qz + Tc[7],
                        Tc[8] * qx + Tc[9] * qy + Tc[10] * qz + Tc[11]};
    const float dcx = (dx ? 1.f : -1.f) * wy[dy] * wz[dz] * mx;
    const float dcy = (dy ? 1.f : -1.f) * wx[dx] * wz[dz] * my;
    const float dcz = (dz ? 1.f : -1.f) * wx[dx] * wy[dy] * mz;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      J[3 * i + 0] = fmaf(Y[i], dcx, J[3 * i + 0]);
      J[3 * i + 1] = fmaf(Y[i], dcy, J[3 * i + 1]);
      J[3 * i + 2] = fmaf(Y[i], dcz, J[3 * i + 2]);
    }
  }
}

__device__ __forceinline__ void lbs_forward_jac(const Voxel& v, const float* __restrict__ Af,
                                                const float* __restrict__ tf, float qx, float qy, float qz,
                                                float out[3], float J[9]) {
  float T[12];
  lbs_blend_jac(v, Af, qx, qy, qz, qx, qy, qz, T, J);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    out[i] = (T[4 * i] * qx + T[4 * i + 1] * qy + T[4 * i + 2] * qz + T[4 * i + 3]) + __ldg(tf + i);
    J[3 * i + 0] += T[4 * i + 0]; J[3 * i + 1] += T[4 * i + 1]; J[3 * i + 2] += T[4 * i + 2];
  }
}

// ------------------------------------------------------------------------------------------
// SDF network geometry (model/network.py:135-141 getTmpSdf)
// ------------------------------------------------------------------------------------------
constexpr int kNumLayers = 9;
constexpr int kPE = 39;     // 3 + 3*2*6
constexpr int kHidden = 512;
constexpr int kSkipOut = 473;  // layer 3 out = 512 - 39
constexpr int kOutDim = 257;   // 1 + 256
__host__ __device__ constexpr int layer_in(int l) { return l == 0 ? kPE : kHidden; }
__host__ __device__ constexpr int layer_out(int l) { return l == 3 ? kSkipOut : (l == 8 ? kOutDim : kHidden); }

// Packed weight blob layout (built by recmv_sdf_pack_weights, sdf_mlp_simt.cu).
//  * fp32 transposed copies [K][Npad32] + padded biases: the FP32_SIMT kernel
//  * fp16 hi/lo "panels" for tcgen05: the K dimension of every layer is cut into 64-wide blocks; a panel
//    is [512 n][64 k] fp16 (128-byte rows = one TMA/UMMA swizzle row).  Panels of all layers are
//    stacked, plane hi first then plane lo, so ONE 2-D tensor map [2*66*512 rows, 64 cols] serves every
//    weight tile.  Layer 4 has 9 panels: 8 for the 473(+39 zero) hidden inputs and 1 for the
//    positional-encoding inputs of the skip connection (its 1/sqrt2 folded into the weights).
constexpr int kNumPanels = 66;
// Exact power-of-two operand scaling of the tensor-core path: activations are stored as fp16(hi)+fp16(lo) of
// 2^6 * a, weights of 2^10 * w, so the `lo` residuals (~2^-12 of the value) stay in fp16's NORMAL range
// (unscaled they are subnormal whenever |value| < 0.125 and carry only ~2^-20 relative precision);
// the epilogue multiplies the fp32 accumulator by 2^-16.  Range: |a| < 1023, |w| < 63.9.
constexpr float kActScale = 64.f;
constexpr float kWgtScale = 1024.f;
constexpr float kAccUnscale = 1.f / (64.f * 1024.f);
__host__ __device__ constexpr int panel_base(int l) {
  return l == 0 ? 0 : (l <= 4 ? 1 + 8 * (l - 1) : 34 + 8 * (l - 5));
}
__host__ __device__ constexpr int num_panels(int l) { return l == 0 ? 1 : (l == 4 ? 9 : 8); }
// softplus(beta=100) evaluated in base 2: u = 100 log2(e) z;  softplus = ln2/100 * log2(1 + 2^u)
constexpr float kSoftplusLog2Scale = 144.26950408889634f;   // 100 * log2(e)
struct PackedLayout {
  size_t w32_off[kNumLayers];   // fp32 [K, Npad32] (transposed) for the SIMT kernel
  size_t b32_off[kNumLayers];   // fp32 [512] bias padded with zeros
  size_t bias_all_off;          // == b32_off[0]; the 9 padded biases are contiguous, stride 512 floats;
                                // a second [9][512] plane holds b * kSoftplusLog2Scale
  size_t f16_off;               // fp16 panels: [2 planes][66 panels][512][64]
  size_t total;
};
PackedLayout packed_layout();

// positional encoding of one point: pe[0..2] = x, then per band k: w*sin(2^k x) (3), w*cos(2^k x) (3)
// (model/Embedder.py:33-37 order), accurate sincosf (fast intrinsics lose >1e-4 at 32x).
__device__ __forceinline__ void positional_encode(float x, float y, float z,
                                                  const float* __restrict__ pw /*12*/, float pe[39]) {
  pe[0] = x; pe[1] = y; pe[2] = z;
  float f = 1.f;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    float sx, cxv, sy, cyv, sz, czv;
    sincosf(x * f, &sx, &cxv);
    sincosf(y * f, &sy, &cyv);
    sincosf(z * f, &sz, &czv);
    float ws = pw[2 * k], wc = pw[2 * k + 1];
    pe[3 + 6 * k + 0] = ws * sx; pe[3 + 6 * k + 1] = ws * sy; pe[3 + 6 * k + 2] = ws * sz;
    pe[3 + 6 * k + 3] = wc * cxv; pe[3 + 6 * k + 4] = wc * cyv; pe[3 + 6 * k + 5] = wc * czv;
    f *= 2.f;
  }
}

// softplus(beta=100, threshold=20) as torch: x*beta > 20 ? x : log1p(exp(beta x))/beta
__device__ __forceinline__ float softplus100(float x) {
  float bx = 100.f * x;
  return bx > 20.f ? x : log1pf(expf(bx)) * 0.01f;
}

}  // namespace recmv

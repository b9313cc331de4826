// The exact-fp32 (CUDA-core) implementation of the fused SDF path, the per-ray first-hit scan, and the C-ABI entry
// points that dispatch between the SIMT and tensor-core kernels.
//
// Fused per tile of 32 points: [ray -> x_obs -> skinning-voxel sample -> inverse LBS ->] positional
// encoding -> 9 linears with softplus(100) -> sdf (+256 features).  Activations live in shared
// memory for the whole network (2 x 32 x 512 fp32 ping-pong); nothing but 4 B/sample (sdf) goes back
// to HBM unless features are requested.  Replaces model/Embedder.py:43-50 + model/network.py:89-119
// (13 PE kernels + 9 cuBLAS SGEMMs + 8 softplus kernels + cat, every [P,512] activation through HBM).
// This mode exists for verification (it is bit-for-bit plain fp32 FMA math); the production path is
// sdf_mlp_tc.cu.
#include "sdf_mlp.cuh"

namespace recmv {

using Sdf = Net<0>;

// ---------------------------------------------------------------------------------------------
// SIMT fused forward
// ---------------------------------------------------------------------------------------------
constexpr int kTileM = 32;
constexpr int kSimtThreads = 256;
constexpr int kLd = 516;  // activation row stride in floats (516 % 32 = 4: the 4 point-groups of a
                          // float4 read hit different banks)

struct SimtWeights {
  const float* w[Sdf::kLayers];
  const float* b[Sdf::kLayers];
};

// out[m][n] = sum_k in[m][k] * Wt[k][n] + b[n]   for m in [ty*8, ty*8+8), n in [tx*8, tx*8+8)
template <bool kSoftplus>
__device__ __forceinline__ void simt_layer(const float* __restrict__ in, float* __restrict__ outp,
                                           const float* __restrict__ Wt, const float* __restrict__ bias,
                                           int K, int npad, int nvalid, int tx, int ty) {
  float acc[8][8];
  int n0 = tx * 8;
  bool active = n0 < npad;
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  if (active) {
    int k = 0;
    for (; k + 4 <= K; k += 4) {
      float4 a[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = *reinterpret_cast<const float4*>(in + (ty * 8 + i) * kLd + k);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const float4* wp = reinterpret_cast<const float4*>(Wt + (size_t)(k + kk) * npad + n0);
        float4 w0 = __ldg(wp), w1 = __ldg(wp + 1);
        float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float av = kk == 0 ? a[i].x : (kk == 1 ? a[i].y : (kk == 2 ? a[i].z : a[i].w));
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av, w[j], acc[i][j]);
        }
      }
    }
    for (; k < K; ++k) {
      const float4* wp = reinterpret_cast<const float4*>(Wt + (size_t)k * npad + n0);
      float4 w0 = __ldg(wp), w1 = __ldg(wp + 1);
      float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float av = in[(ty * 8 + i) * kLd + k];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av, w[j], acc[i][j]);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int n = n0 + j;
      if (n < nvalid) {
        float bv = __ldg(bias + n);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float v = acc[i][j] + bv;
          outp[(ty * 8 + i) * kLd + n] = kSoftplus ? softplus100(v) : v;
        }
      }
    }
  }
}

__global__ void __launch_bounds__(kSimtThreads, 1) sdf_simt_kernel(PointSource src, SimtWeights wts,
                                                                   PeWeights pw,
                                                                   float* __restrict__ out_sdf,
                                                                   float* __restrict__ out_feat,
                                                                   int64_t P) {
  extern __shared__ __align__(16) float smem[];
  float* bufA = smem;                  // [32][516]
  float* bufB = smem + kTileM * kLd;   // [32][516]
  float* pe = bufB + kTileM * kLd;     // [32][40]
  __shared__ unsigned char s_valid[kTileM];
  int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  int64_t num_tiles = (P + kTileM - 1) / kTileM;
  for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int64_t p0 = tile * kTileM;
    if (threadIdx.x < kTileM) {
      int64_t p = p0 + threadIdx.x;
      float e[39];
      bool ok = true;
      if (p < P) {
        float cx, cy, cz;
        ok = fetch_point(src, p, cx, cy, cz);
        positional_encode(cx, cy, cz, pw.w, e);
      } else {
#pragma unroll
        for (int q = 0; q < 39; ++q) e[q] = 0.f;
      }
      s_valid[threadIdx.x] = ok;
#pragma unroll
      for (int q = 0; q < 39; ++q) pe[threadIdx.x * 40 + q] = e[q];
      pe[threadIdx.x * 40 + 39] = 0.f;
    }
    __syncthreads();
    // layer 0: K = 39 straight from the pe buffer (row stride 40) -> copy into bufA rows first
    for (int q = threadIdx.x; q < kTileM * 40; q += kSimtThreads) bufA[(q / 40) * kLd + (q % 40)] = pe[q];
    __syncthreads();
    simt_layer<true>(bufA, bufB, wts.w[0], wts.b[0], Sdf::kPE, 512, 512, tx, ty); __syncthreads();
    simt_layer<true>(bufB, bufA, wts.w[1], wts.b[1], 512, 512, 512, tx, ty); __syncthreads();
    simt_layer<true>(bufA, bufB, wts.w[2], wts.b[2], 512, 512, 512, tx, ty); __syncthreads();
    simt_layer<true>(bufB, bufA, wts.w[3], wts.b[3], 512, 512, Sdf::kSkipOut, tx, ty); __syncthreads();
    // skip: columns 473..511 of the layer-4 input are the positional encoding (1/sqrt2 is in W4)
    for (int q = threadIdx.x; q < kTileM * Sdf::kPE; q += kSimtThreads)
      bufA[(q / Sdf::kPE) * kLd + Sdf::kSkipOut + (q % Sdf::kPE)] = pe[(q / Sdf::kPE) * 40 + (q % Sdf::kPE)];
    __syncthreads();
    simt_layer<true>(bufA, bufB, wts.w[4], wts.b[4], 512, 512, 512, tx, ty); __syncthreads();
    simt_layer<true>(bufB, bufA, wts.w[5], wts.b[5], 512, 512, 512, tx, ty); __syncthreads();
    simt_layer<true>(bufA, bufB, wts.w[6], wts.b[6], 512, 512, 512, tx, ty); __syncthreads();
    simt_layer<true>(bufB, bufA, wts.w[7], wts.b[7], 512, 512, 512, tx, ty); __syncthreads();
    simt_layer<false>(bufA, bufB, wts.w[8], wts.b[8], 512, 264, Sdf::kOutDim, tx, ty); __syncthreads();
    if (threadIdx.x < kTileM && p0 + threadIdx.x < P)
      out_sdf[p0 + threadIdx.x] = s_valid[threadIdx.x] ? bufB[threadIdx.x * kLd] : kInvalidSdf;
    if (out_feat) {
      for (int q = threadIdx.x; q < kTileM * 256; q += kSimtThreads) {
        int m = q >> 8, n = q & 255;
        if (p0 + m < P) out_feat[(p0 + m) * 256 + n] = bufB[m * kLd + 1 + n];
      }
    }
    __syncthreads();
  }
}

int simt_sdf_forward(const PointSource& src, const void* packed, const PeWeights& pw, float* out_sdf,
                     float* out_feat, int64_t P, cudaStream_t st) {
  const PackedBlob blob = carve(const_cast<void*>(packed), blob_layout<0>);
  SimtWeights w;
  for (int l = 0; l < Sdf::kLayers; ++l) {
    w.w[l] = blob.w32[l];
    w.b[l] = blob.bias + l * 512;
  }
  size_t smem = (size_t)(2 * kTileM * kLd + kTileM * 40) * sizeof(float);
  int s = smem_opt_in<sdf_simt_kernel>((int)smem);
  if (s) return s;
  int64_t tiles = (P + kTileM - 1) / kTileM;
  int grid = (int)(tiles < num_sms() ? tiles : num_sms());
  sdf_simt_kernel<<<grid, kSimtThreads, smem, st>>>(src, w, pw, out_sdf, out_feat, P);
  return launch_status();
}

// ---------------------------------------------------------------------------------------------
// per-ray first hit: one warp per ray, coalesced reads of the sdf row
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) first_hit_kernel(const float* __restrict__ sdf, int S,
                                                        float t_near, float dt,
                                                        int32_t* __restrict__ hit_idx,
                                                        float* __restrict__ hit_t, int64_t R) {
  int lane = threadIdx.x & 31;
  int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < R; r += nwarps) {
    const float* row = sdf + r * S;
    int found = -1;
    for (int base = 0; base < S && found < 0; base += 32) {
      int k = base + lane;
      float v = k < S ? row[k] : 1.f;
      unsigned m = __ballot_sync(0xffffffffu, k < S && v <= 0.f);
      if (m) found = base + __ffs(m) - 1;
    }
    if (lane == 0) {
      int hi = found > 0 ? found : -1;
      float t = 0.f;
      if (hi > 0) {
        float s0 = row[hi - 1], s1 = row[hi];
        float t0 = t_near + ((float)(hi - 1) + 0.5f) * dt;
        t = t0 + dt * (s0 / (s0 - s1));
      }
      if (hit_idx) hit_idx[r] = hi;
      if (hit_t) hit_t[r] = t;
    }
  }
}

}  // namespace recmv

using namespace recmv;

static int run_forward(const PointSource& src, const void* packed, const float* pe_w, float* out_sdf,
                       float* out_feat, int64_t P, int mode, cudaStream_t st) {
  const PeWeights pw = pe_weights(pe_w);
  if (mode == RECMV_MLP_FP32_SIMT) return simt_sdf_forward(src, packed, pw, out_sdf, out_feat, P, st);
  const int passes = tc_passes(mode);
  if (!passes) return RECMV_E_DTYPE;
  return tc_sdf_forward(src, packed, pw, out_sdf, out_feat, P, passes, st);
}

extern "C" int recmv_sdf_mlp_fwd(const float* x, const void* packed, const float* pe_w, float* out_sdf,
                                 float* out_feat, int64_t P, int mode, recmv_stream_t stream) {
  if (P < 0) return RECMV_E_SHAPE;
  if (P == 0) return RECMV_OK;
  if (!x || !packed || !pe_w || !out_sdf) return RECMV_E_NULL;
  PointSource src = {};
  src.x = x;
  src.S = 1;
  return run_forward(src, packed, pe_w, out_sdf, out_feat, P, mode, (cudaStream_t)stream);
}

// Same as recmv_sdf_mlp_fwd with the number of points read from DEVICE memory (*count_dev, clamped to `capacity`): the
// consumer of a device-built worklist (coarse-to-fine sweep) launches without a host round trip.
extern "C" int recmv_sdf_mlp_fwd_counted(const float* x, const void* packed, const float* pe_w, float* out_sdf,
                                         float* out_feat, int64_t capacity, const int* count_dev, int mode,
                                         recmv_stream_t stream) {
  if (capacity < 0) return RECMV_E_SHAPE;
  if (capacity == 0) return RECMV_OK;
  if (!x || !packed || !pe_w || !out_sdf || !count_dev) return RECMV_E_NULL;
  const int passes = tc_passes(mode);
  if (!passes) return RECMV_E_UNSUPPORTED;
  PointSource src = {};
  src.x = x;
  src.S = 1;
  return tc_sdf_forward(src, packed, pe_weights(pe_w), out_sdf, out_feat, capacity, passes, (cudaStream_t)stream,
                        count_dev);
}

extern "C" int recmv_sdf_mlp_fwd_grad(const float* x, const void* packed, const float* pe_w, float* out_sdf,
                                      float* out_feat, float* out_grad, int64_t P, int mode,
                                      recmv_stream_t stream) {
  if (P < 0) return RECMV_E_SHAPE;
  if (P == 0) return RECMV_OK;
  if (!x || !packed || !pe_w || !out_sdf || !out_grad) return RECMV_E_NULL;
  const int passes = tc_passes(mode);
  if (!passes) return RECMV_E_UNSUPPORTED;
  return tc_sdf_forward_grad(x, packed, pe_weights(pe_w), out_sdf, out_feat, out_grad, P, passes, (cudaStream_t)stream);
}

extern "C" int recmv_ray_first_hit(const float* sdf, const recmv_raymarch_t* rm, int32_t* hit_idx,
                                   float* hit_t, int64_t R, recmv_stream_t stream) {
  if (R < 0) return RECMV_E_SHAPE;
  if (R == 0) return RECMV_OK;
  if (!sdf || !rm) return RECMV_E_NULL;
  if (rm->samples_per_ray <= 0) return RECMV_E_SHAPE;
  float dt = (rm->t_far - rm->t_near) / (float)rm->samples_per_ray;
  first_hit_kernel<<<stride_grid(R * 32, 256, 8), 256, 0, (cudaStream_t)stream>>>(
      sdf, rm->samples_per_ray, rm->t_near, dt, hit_idx, hit_t, R);
  return launch_status();
}

extern "C" int recmv_render_sdf(const float* ray_dirs, const recmv_raymarch_t* rm, const float* A,
                                const float* trans, const int32_t* frame_of_ray, int64_t rays_per_frame,
                                int num_frames, const recmv_voxel_t* vox, const void* packed,
                                const float* pe_w, float* out_sdf, float* out_xc, int32_t* hit_idx,
                                float* hit_t, int64_t R, int mode, recmv_stream_t stream) {
  if (R < 0) return RECMV_E_SHAPE;
  if (R == 0) return RECMV_OK;
  if (!ray_dirs || !rm || !A || !trans || !vox || !vox->ws_cl || !packed || !pe_w || !out_sdf)
    return RECMV_E_NULL;
  if (rm->samples_per_ray <= 0 || num_frames <= 0 || vox->D <= 0 || vox->H <= 0 || vox->W <= 0)
    return RECMV_E_SHAPE;
  PointSource src = {};
  src.x = nullptr;
  src.ray_dirs = ray_dirs; src.A = A; src.trans = trans; src.frame_of_ray = frame_of_ray;
  src.rays_per_frame = rays_per_frame; src.num_frames = num_frames; src.vox = to_voxel(vox);
  src.cam[0] = rm->cam_pos[0]; src.cam[1] = rm->cam_pos[1]; src.cam[2] = rm->cam_pos[2];
  src.t_near = rm->t_near;
  src.dt = (rm->t_far - rm->t_near) / (float)rm->samples_per_ray;
  src.S = rm->samples_per_ray;
  src.out_xc = out_xc;
  int64_t P = R * (int64_t)rm->samples_per_ray;
  int s = run_forward(src, packed, pe_w, out_sdf, nullptr, P, mode, (cudaStream_t)stream);
  if (s) return s;
  if (hit_idx || hit_t) return recmv_ray_first_hit(out_sdf, rm, hit_idx, hit_t, R, stream);
  return RECMV_OK;
}

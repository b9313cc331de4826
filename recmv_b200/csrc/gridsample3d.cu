// 3-D trilinear / border / align_corners=False grid sampler: forward, backward, double backward.
// Replaces MCAcc/cuda/GridSamplerMineKernel.cu:160-328 (K4), :331-570 (K5), :573-914 (K6).
//
// Differences from the reference that do not change any consumed value:
//  * a channels-last [N,D,H,W,C] input layout is supported next to NCDHW (one 32 B sector per
//    8 channels instead of one per channel) -- the skinning voxel is relaid out once by the host
//    shim and cached;
//  * grad_input is OPTIONAL: the skinning voxel is a frozen buffer, yet the reference allocates and
//    atomically fills a zero volume of its size on every backward (GridSamplerMineKernel.cu:955);
//  * one derivation for all eight corners (sign/weight tables) instead of eight hand-expanded copies.
#include "common.cuh"

namespace recmv {

template <typename T>
struct Cell {
  int x[2], y[2], z[2];  // corner indices (unclamped +1)
  bool inx[2], iny[2], inz[2];
  T wx[2], wy[2], wz[2];
  T mx, my, mz;  // clip multipliers
};

template <typename T>
__device__ __forceinline__ Cell<T> make_cell(T gx, T gy, T gz, int D, int H, int W) {
  Cell<T> c;
  T ix = clip_grad<T>(unnormalize(gx, W), W, &c.mx);
  T iy = clip_grad<T>(unnormalize(gy, H), H, &c.my);
  T iz = clip_grad<T>(unnormalize(gz, D), D, &c.mz);
  // NaN: clip_grad's comparisons are false for NaN -> passes through; the reference's max/min clip
  // maps NaN to 0 in forward; keep that, and give the NaN axis no gradient (mult = 0), as the fused
  // skinning kernels do (common.cuh skin_cell), so both LBSkinner paths agree on such a point.
  if (!(ix == ix)) { ix = (T)0; c.mx = (T)0; }
  if (!(iy == iy)) { iy = (T)0; c.my = (T)0; }
  if (!(iz == iz)) { iz = (T)0; c.mz = (T)0; }
  int x0 = (int)floor(ix), y0 = (int)floor(iy), z0 = (int)floor(iz);
  c.x[0] = x0; c.x[1] = x0 + 1; c.y[0] = y0; c.y[1] = y0 + 1; c.z[0] = z0; c.z[1] = z0 + 1;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    c.inx[i] = c.x[i] >= 0 && c.x[i] < W;
    c.iny[i] = c.y[i] >= 0 && c.y[i] < H;
    c.inz[i] = c.z[i] >= 0 && c.z[i] < D;
  }
  c.wx[0] = (T)(x0 + 1) - ix; c.wx[1] = ix - (T)x0;
  c.wy[0] = (T)(y0 + 1) - iy; c.wy[1] = iy - (T)y0;
  c.wz[0] = (T)(z0 + 1) - iz; c.wz[1] = iz - (T)z0;
  return c;
}

template <int LAYOUT>
__device__ __forceinline__ size_t vox_index(int n, int c, int z, int y, int x, int C, int D, int H, int W) {
  if (LAYOUT == RECMV_LAYOUT_NCDHW)
    return ((((size_t)n * C + c) * D + z) * H + y) * W + x;
  else
    return ((((size_t)n * D + z) * H + y) * W + x) * C + c;
}

template <typename T, int LAYOUT>
__global__ void __launch_bounds__(256) gs3d_fwd_kernel(const T* __restrict__ input,
                                                       const T* __restrict__ grid,
                                                       T* __restrict__ output, int N, int C, int D,
                                                       int H, int W, int64_t P) {
  int64_t total = (int64_t)N * P;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    int n = (int)(idx / P);
    int64_t p = idx - (int64_t)n * P;
    const T* g = grid + idx * 3;
    Cell<T> cl = make_cell<T>(g[0], g[1], g[2], D, H, W);
    for (int c = 0; c < C; ++c) {
      T acc = (T)0;
#pragma unroll
      for (int dz = 0; dz < 2; ++dz)
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
          for (int dx = 0; dx < 2; ++dx)
            if (cl.inx[dx] && cl.iny[dy] && cl.inz[dz]) {
              T w = cl.wx[dx] * cl.wy[dy] * cl.wz[dz];
              acc += input[vox_index<LAYOUT>(n, c, cl.z[dz], cl.y[dy], cl.x[dx], C, D, H, W)] * w;
            }
      output[((size_t)n * C + c) * P + p] = acc;
    }
  }
}

// fp32, channels-last, C % 4 == 0: one 128-bit load per corner and channel quad (the 24-channel skinning voxel:
// 6 loads per corner, 3 fully used sectors), same summation order as the generic kernel.
__global__ void __launch_bounds__(256) gs3d_fwd_cl4_kernel(const float* __restrict__ input, const float* __restrict__ grid,
                                                           float* __restrict__ output, int N, int C, int D, int H,
                                                           int W, int64_t P) {
  const int64_t total = (int64_t)N * P;
  const int Q = C >> 2;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / P);
    const int64_t p = idx - (int64_t)n * P;
    const float* g = grid + idx * 3;
    const Cell<float> cl = make_cell<float>(__ldg(g), __ldg(g + 1), __ldg(g + 2), D, H, W);
    const float4* corner[8];
    float cw[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int dx = k & 1, dy = (k >> 1) & 1, dz = k >> 2;
      const bool in = cl.inx[dx] && cl.iny[dy] && cl.inz[dz];
      cw[k] = in ? cl.wx[dx] * cl.wy[dy] * cl.wz[dz] : 0.f;
      corner[k] = in ? reinterpret_cast<const float4*>(input + ((((size_t)n * D + cl.z[dz]) * H + cl.y[dy]) * W + cl.x[dx]) * C)
                     : nullptr;
    }
    for (int q = 0; q < Q; ++q) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (corner[k]) {
          const float4 t = __ldg(corner[k] + q);
          acc.x += t.x * cw[k]; acc.y += t.y * cw[k]; acc.z += t.z * cw[k]; acc.w += t.w * cw[k];
        }
      float* o = output + ((size_t)n * C + 4 * q) * P + p;
      o[0] = acc.x; o[P] = acc.y; o[2 * P] = acc.z; o[3 * P] = acc.w;
    }
  }
}

template <typename T, int LAYOUT>
__global__ void __launch_bounds__(256) gs3d_bwd_kernel(const T* __restrict__ input,
                                                       const T* __restrict__ grid,
                                                       const T* __restrict__ grad_out,
                                                       T* __restrict__ grad_input /*nullable*/,
                                                       T* __restrict__ grad_grid, int N, int C,
                                                       int D, int H, int W, int64_t P) {
  int64_t total = (int64_t)N * P;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    int n = (int)(idx / P);
    int64_t p = idx - (int64_t)n * P;
    const T* g = grid + idx * 3;
    Cell<T> cl = make_cell<T>(g[0], g[1], g[2], D, H, W);
    T gix = 0, giy = 0, giz = 0;
    for (int c = 0; c < C; ++c) {
      T go = grad_out[((size_t)n * C + c) * P + p];
#pragma unroll
      for (int dz = 0; dz < 2; ++dz)
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
          for (int dx = 0; dx < 2; ++dx)
            if (cl.inx[dx] && cl.iny[dy] && cl.inz[dz]) {
              size_t vi = vox_index<LAYOUT>(n, c, cl.z[dz], cl.y[dy], cl.x[dx], C, D, H, W);
              if (grad_input) atomicAdd(grad_input + vi, cl.wx[dx] * cl.wy[dy] * cl.wz[dz] * go);
              T v = input[vi];
              T sx = dx ? (T)1 : (T)-1, sy = dy ? (T)1 : (T)-1, sz = dz ? (T)1 : (T)-1;
              gix += sx * v * cl.wy[dy] * cl.wz[dz] * go;
              giy += sy * v * cl.wx[dx] * cl.wz[dz] * go;
              giz += sz * v * cl.wx[dx] * cl.wy[dy] * go;
            }
    }
    T* gg = grad_grid + idx * 3;
    gg[0] = cl.mx * (gix * (T)W / (T)2);
    gg[1] = cl.my * (giy * (T)H / (T)2);
    gg[2] = cl.mz * (giz * (T)D / (T)2);
  }
}

template <typename T, int LAYOUT>
__global__ void __launch_bounds__(256) gs3d_bwd2_kernel(
    const T* __restrict__ gg_input /*nullable*/, const T* __restrict__ gg_grid,
    const T* __restrict__ input, const T* __restrict__ grid, const T* __restrict__ grad_out,
    T* __restrict__ g_input /*nullable*/, T* __restrict__ g_grid, T* __restrict__ gg_out, int N,
    int C, int D, int H, int W, int64_t P) {
  int64_t total = (int64_t)N * P;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    int n = (int)(idx / P);
    int64_t p = idx - (int64_t)n * P;
    const T* g = grid + idx * 3;
    Cell<T> cl = make_cell<T>(g[0], g[1], g[2], D, H, W);
    T qx = gg_grid[idx * 3 + 0], qy = gg_grid[idx * 3 + 1], qz = gg_grid[idx * 3 + 2];
    T scx = (T)0.5 * (T)W * cl.mx, scy = (T)0.5 * (T)H * cl.my, scz = (T)0.5 * (T)D * cl.mz;
    // tmp[corner] = sum_a gg_grid_a * scale_a * d_a w(corner)
    T tmp[8];
#pragma unroll
    for (int dz = 0; dz < 2; ++dz)
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          T sx = dx ? (T)1 : (T)-1, sy = dy ? (T)1 : (T)-1, sz = dz ? (T)1 : (T)-1;
          tmp[dz * 4 + dy * 2 + dx] = qx * scx * sx * cl.wy[dy] * cl.wz[dz] +
                                      qy * scy * sy * cl.wx[dx] * cl.wz[dz] +
                                      qz * scz * sz * cl.wx[dx] * cl.wy[dy];
        }
    T gix = 0, giy = 0, giz = 0;
    for (int c = 0; c < C; ++c) {
      T go = grad_out[((size_t)n * C + c) * P + p];
      T ggo = 0;
#pragma unroll
      for (int dz = 0; dz < 2; ++dz)
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
          for (int dx = 0; dx < 2; ++dx)
            if (cl.inx[dx] && cl.iny[dy] && cl.inz[dz]) {
              int k = dz * 4 + dy * 2 + dx;
              size_t vi = vox_index<LAYOUT>(n, c, cl.z[dz], cl.y[dy], cl.x[dx], C, D, H, W);
              T sx = dx ? (T)1 : (T)-1, sy = dy ? (T)1 : (T)-1, sz = dz ? (T)1 : (T)-1;
              if (g_input) atomicAdd(g_input + vi, tmp[k] * go);
              T t = gg_input ? gg_input[vi] : (T)0;
              gix += sx * t * cl.wy[dy] * cl.wz[dz] * go * scx;
              giy += sy * t * cl.wx[dx] * cl.wz[dz] * go * scy;
              giz += sz * t * cl.wx[dx] * cl.wy[dy] * go * scz;
              ggo += t * (cl.wx[dx] * cl.wy[dy] * cl.wz[dz]);
              T v = input[vi];
              gix += v * (qy * scx * scy * sx * sy * cl.wz[dz] + qz * scx * scz * sx * sz * cl.wy[dy]) * go;
              giy += v * (qx * scx * scy * sx * sy * cl.wz[dz] + qz * scy * scz * sy * sz * cl.wx[dx]) * go;
              giz += v * (qx * scx * scz * sx * sz * cl.wy[dy] + qy * scy * scz * sy * sz * cl.wx[dx]) * go;
              ggo += v * tmp[k];
            }
      gg_out[((size_t)n * C + c) * P + p] = ggo;
    }
    T* o = g_grid + idx * 3;
    o[0] = gix; o[1] = giy; o[2] = giz;
  }
}

// [C,D,H,W] -> [D,H,W,C] through a 32x(C<=32) shared tile: coalesced on both sides
__global__ void __launch_bounds__(256) vox_cl_kernel(const float* __restrict__ src,
                                                     float* __restrict__ dst, int C, int64_t S) {
  __shared__ float tile[32][33];
  // block handles 32 spatial positions x up to 32 channels per pass
  for (int64_t s0 = (int64_t)blockIdx.x * 32; s0 < S; s0 += (int64_t)gridDim.x * 32) {
    for (int c0 = 0; c0 < C; c0 += 32) {
      int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 8 rows of 32
      for (int cc = ty; cc < 32; cc += 8) {
        int c = c0 + cc;
        int64_t s = s0 + tx;
        tile[cc][tx] = (c < C && s < S) ? src[(size_t)c * S + s] : 0.f;
      }
      __syncthreads();
      for (int ss = ty; ss < 32; ss += 8) {
        int c = c0 + tx;
        int64_t s = s0 + ss;
        if (c < C && s < S) dst[(size_t)s * C + c] = tile[tx][ss];
      }
      __syncthreads();
    }
  }
}

template <typename T>
static int gs_dispatch_fwd(const void* input, const void* grid, void* output, int N, int C, int D,
                           int H, int W, int64_t P, int layout, cudaStream_t st) {
  int g = stride_grid((int64_t)N * P, 256, 8);
  if (layout == RECMV_LAYOUT_NCDHW)
    gs3d_fwd_kernel<T, RECMV_LAYOUT_NCDHW><<<g, 256, 0, st>>>((const T*)input, (const T*)grid, (T*)output, N, C, D, H, W, P);
  else if (sizeof(T) == 4 && (C & 3) == 0 && ((uintptr_t)input & 15) == 0)
    gs3d_fwd_cl4_kernel<<<g, 256, 0, st>>>((const float*)input, (const float*)grid, (float*)output, N, C, D, H, W, P);
  else
    gs3d_fwd_kernel<T, RECMV_LAYOUT_NDHWC><<<g, 256, 0, st>>>((const T*)input, (const T*)grid, (T*)output, N, C, D, H, W, P);
  return launch_status();
}

template <typename T>
static int gs_dispatch_bwd(const void* input, const void* grid, const void* go, void* gi, void* gg,
                           int N, int C, int D, int H, int W, int64_t P, int layout, cudaStream_t st) {
  int g = stride_grid((int64_t)N * P, 256, 8);
  if (layout == RECMV_LAYOUT_NCDHW)
    gs3d_bwd_kernel<T, RECMV_LAYOUT_NCDHW><<<g, 256, 0, st>>>((const T*)input, (const T*)grid, (const T*)go, (T*)gi, (T*)gg, N, C, D, H, W, P);
  else
    gs3d_bwd_kernel<T, RECMV_LAYOUT_NDHWC><<<g, 256, 0, st>>>((const T*)input, (const T*)grid, (const T*)go, (T*)gi, (T*)gg, N, C, D, H, W, P);
  return launch_status();
}

template <typename T>
static int gs_dispatch_bwd2(const void* ggi, const void* ggg, const void* input, const void* grid,
                            const void* go, void* gi, void* gg, void* ggo, int N, int C, int D,
                            int H, int W, int64_t P, int layout, cudaStream_t st) {
  int g = stride_grid((int64_t)N * P, 256, 8);
  if (layout == RECMV_LAYOUT_NCDHW)
    gs3d_bwd2_kernel<T, RECMV_LAYOUT_NCDHW><<<g, 256, 0, st>>>((const T*)ggi, (const T*)ggg, (const T*)input, (const T*)grid, (const T*)go, (T*)gi, (T*)gg, (T*)ggo, N, C, D, H, W, P);
  else
    gs3d_bwd2_kernel<T, RECMV_LAYOUT_NDHWC><<<g, 256, 0, st>>>((const T*)ggi, (const T*)ggg, (const T*)input, (const T*)grid, (const T*)go, (T*)gi, (T*)gg, (T*)ggo, N, C, D, H, W, P);
  return launch_status();
}

static int gs_check(int N, int C, int D, int H, int W, int64_t P, int dtype, int layout) {
  if (dtype != RECMV_F32 && dtype != RECMV_F64) return RECMV_E_DTYPE;
  if (layout != RECMV_LAYOUT_NCDHW && layout != RECMV_LAYOUT_NDHWC) return RECMV_E_DTYPE;
  if (N <= 0 || C <= 0 || D <= 0 || H <= 0 || W <= 0 || P < 0) return RECMV_E_SHAPE;
  return RECMV_OK;
}

}  // namespace recmv

using namespace recmv;

extern "C" int recmv_gridsample3d_fwd(const void* input, const void* grid, void* output, int N,
                                      int C, int D, int H, int W, int64_t P, int dtype, int layout,
                                      recmv_stream_t stream) {
  int s = gs_check(N, C, D, H, W, P, dtype, layout);
  if (s) return s;
  if (P == 0) return RECMV_OK;
  if (!input || !grid || !output) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  return dtype == RECMV_F32 ? gs_dispatch_fwd<float>(input, grid, output, N, C, D, H, W, P, layout, st)
                            : gs_dispatch_fwd<double>(input, grid, output, N, C, D, H, W, P, layout, st);
}

extern "C" int recmv_gridsample3d_bwd(const void* input, const void* grid, const void* grad_out,
                                      void* grad_input, void* grad_grid, int N, int C, int D, int H,
                                      int W, int64_t P, int dtype, int layout, recmv_stream_t stream) {
  int s = gs_check(N, C, D, H, W, P, dtype, layout);
  if (s) return s;
  if (P == 0) return RECMV_OK;
  if (!input || !grid || !grad_out || !grad_grid) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  return dtype == RECMV_F32
             ? gs_dispatch_bwd<float>(input, grid, grad_out, grad_input, grad_grid, N, C, D, H, W, P, layout, st)
             : gs_dispatch_bwd<double>(input, grid, grad_out, grad_input, grad_grid, N, C, D, H, W, P, layout, st);
}

extern "C" int recmv_gridsample3d_bwd2(const void* gg_input, const void* gg_grid, const void* input,
                                       const void* grid, const void* grad_out, void* g_input,
                                       void* g_grid, void* gg_out, int N, int C, int D, int H, int W,
                                       int64_t P, int dtype, int layout, recmv_stream_t stream) {
  int s = gs_check(N, C, D, H, W, P, dtype, layout);
  if (s) return s;
  if (P == 0) return RECMV_OK;
  if (!gg_grid || !input || !grid || !grad_out || !g_grid || !gg_out) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  return dtype == RECMV_F32
             ? gs_dispatch_bwd2<float>(gg_input, gg_grid, input, grid, grad_out, g_input, g_grid, gg_out, N, C, D, H, W, P, layout, st)
             : gs_dispatch_bwd2<double>(gg_input, gg_grid, input, grid, grad_out, g_input, g_grid, gg_out, N, C, D, H, W, P, layout, st);
}

extern "C" int recmv_voxel_to_channels_last(const float* src, float* dst, int C, int D, int H, int W,
                                            recmv_stream_t stream) {
  if (!src || !dst) return RECMV_E_NULL;
  if (C <= 0 || D <= 0 || H <= 0 || W <= 0) return RECMV_E_SHAPE;
  int64_t S = (int64_t)D * H * W;
  int g = stride_grid(S / 32 + 1, 1, 8);
  vox_cl_kernel<<<g, 256, 0, (cudaStream_t)stream>>>(src, dst, C, S);
  return launch_status();
}

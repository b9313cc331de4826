// Construction of the 24-channel skinning voxel (model/Deformer.py:533-591, utils/LBSWsmpl.py:2-51):
//   lbsw_knn_kernel     k nearest body vertices of every voxel centre + clamped inverse-distance blend
//   lbsw_smooth_kernel  one Jacobi pass of the 6-neighbour stencil + renormalisation over the channels
// This is setup work (once per dataset), not part of a training or render step.  Every rounding step the reference
// takes in fp32 is taken here with the _rn intrinsics, so no FMA contraction changes its order; the kNN distance
// itself is the one place that uses fmaf (see recmv_b200.h).  No atomics: results are bit-identical run to run.
#include <math.h>

#include "common.cuh"

namespace recmv {
namespace {

constexpr int kCh = 24;
constexpr int kKnnThreads = 256;              // 8 warps
constexpr int kMaxVerts = 14336;              // 224 KB of float4 in shared memory
// A warp owns a 4 (x) x 4 (y) x 2 (z) brick of voxels: its lanes' reject thresholds stay close, so the rare
// insertion path is taken by most lanes of a warp at once or by none.
constexpr int kBx = 4, kBy = 4, kBz = 2;

// Voxel centre along one axis, in the reference's fp32 order (Deformer.py:566-571):
//   align_corners: c / (res - 1);  otherwise c / res + (1 / res) / 2;  then * (bmax - bmin) + bmin
__device__ __forceinline__ float voxel_centre(int c, int res, bool ac, float bmin, float bmax) {
  const float r = (float)res;
  float u;
  if (ac) u = __fdiv_rn((float)c, __fsub_rn(r, 1.f));
  else u = __fadd_rn(__fdiv_rn((float)c, r), __fmul_rn(__fdiv_rn(1.f, r), 0.5f));
  return __fadd_rn(__fmul_rn(u, __fsub_rn(bmax, bmin)), bmin);
}

// The fp32 squared distance that orders the candidates.  Written out so that the insertion path, which recomputes it
// for the current k-th neighbour, gets exactly the value the scan compared.
__device__ __forceinline__ float dist2(float px, float py, float pz, float4 v) {
  const float dx = __fsub_rn(px, v.x), dy = __fsub_rn(py, v.y), dz = __fsub_rn(pz, v.z);
  return fmaf(dz, dz, fmaf(dy, dy, __fmul_rn(dx, dx)));
}

// Sorted list of the best candidates seen so far, ascending in (distance, index).  The last k of the KMAX slots hold
// the real entries; the first KMAX - k hold -inf sentinels that never move, so a runtime k needs no dynamic register
// index.  Vertices are scanned in ascending index order, so a newcomer goes after every entry of equal distance: on
// exactly equal distances the lower vertex index wins.
template <int KMAX>
struct TopK {
  float s[KMAX];
  int id[KMAX];
  float thr2;   // squared distance of the k-th entry (+inf until k entries exist): d2 >= thr2 can never enter

  __device__ __forceinline__ void init(int k) {
#pragma unroll
    for (int i = 0; i < KMAX; ++i) {
      s[i] = i < KMAX - k ? -INFINITY : INFINITY;
      id[i] = 0;
    }
    thr2 = INFINITY;
  }

  // candidate j with squared distance d2 < thr2
  __device__ __forceinline__ void offer(float d2, int j, float px, float py, float pz, const float4* sv) {
    const float sn = __fsqrt_rn(d2);
    if (!(sn < s[KMAX - 1])) return;   // equal distance, higher index: the current k-th entry stays
#pragma unroll
    for (int i = KMAX - 1; i >= 1; --i) {
      const bool up = sn < s[i - 1];            // entry i-1 moves to i
      const bool here = !up && sn < s[i];       // the newcomer lands at i
      s[i] = up ? s[i - 1] : (here ? sn : s[i]);
      id[i] = up ? id[i - 1] : (here ? j : id[i]);
    }
    if (sn < s[0]) { s[0] = sn; id[0] = j; }
    thr2 = s[KMAX - 1] == INFINITY ? INFINITY : dist2(px, py, pz, sv[id[KMAX - 1]]);
  }
};

template <int KMAX>
__global__ void __launch_bounds__(kKnnThreads, 2)
lbsw_knn_kernel(const float* __restrict__ verts, const float* __restrict__ vert_ws, int V, float bx0, float by0,
                float bz0, float bx1, float by1, float bz1, int W, int H, int D, int align_corners, int k,
                float* __restrict__ out_cl, int32_t* __restrict__ out_idx) {
  extern __shared__ float4 sv[];
  for (int j = threadIdx.x; j < V; j += blockDim.x)
    sv[j] = make_float4(__ldg(verts + 3 * j), __ldg(verts + 3 * j + 1), __ldg(verts + 3 * j + 2), 0.f);
  __syncthreads();

  const int lane = threadIdx.x & 31;
  const int nbx = (W + kBx - 1) / kBx, nby = (H + kBy - 1) / kBy, nbz = (D + kBz - 1) / kBz;
  const int64_t nbricks = (int64_t)nbx * nby * nbz;
  const int64_t warps = (int64_t)gridDim.x * (kKnnThreads / 32);
  const bool ac = align_corners != 0;
  for (int64_t b = (int64_t)blockIdx.x * (kKnnThreads / 32) + (threadIdx.x >> 5); b < nbricks; b += warps) {
    const int x = (int)(b % nbx) * kBx + (lane & 3);
    const int y = (int)((b / nbx) % nby) * kBy + ((lane >> 2) & 3);
    const int z = (int)(b / ((int64_t)nbx * nby)) * kBz + (lane >> 4);
    if (x >= W || y >= H || z >= D) continue;
    const float px = voxel_centre(x, W, ac, bx0, bx1);
    const float py = voxel_centre(y, H, ac, by0, by1);
    const float pz = voxel_centre(z, D, ac, bz0, bz1);

    TopK<KMAX> t;
    t.init(k);
    int j = 0;
    for (; j + 4 <= V; j += 4) {
      const float d0 = dist2(px, py, pz, sv[j]), d1 = dist2(px, py, pz, sv[j + 1]);
      const float d2 = dist2(px, py, pz, sv[j + 2]), d3 = dist2(px, py, pz, sv[j + 3]);
      if (fminf(fminf(d0, d1), fminf(d2, d3)) < t.thr2) {
        if (d0 < t.thr2) t.offer(d0, j, px, py, pz, sv);
        if (d1 < t.thr2) t.offer(d1, j + 1, px, py, pz, sv);
        if (d2 < t.thr2) t.offer(d2, j + 2, px, py, pz, sv);
        if (d3 < t.thr2) t.offer(d3, j + 3, px, py, pz, sv);
      }
    }
    for (; j < V; ++j) {
      const float d = dist2(px, py, pz, sv[j]);
      if (d < t.thr2) t.offer(d, j, px, py, pz, sv);
    }

    // Deformer.py:579-582: w_i = (1 / clamp(d_i, 1e-4, 1)) / sum_i(...), then sum_i ws[id_i] * w_i, in neighbour order
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < KMAX; ++i) {
      t.s[i] = __frcp_rn(fminf(fmaxf(t.s[i], 1e-4f), 1.f));
      if (i >= KMAX - k) sum = __fadd_rn(sum, t.s[i]);
    }
    float acc[kCh];
#pragma unroll
    for (int c = 0; c < kCh; ++c) acc[c] = 0.f;
    const int64_t n = ((int64_t)z * H + y) * W + x;
#pragma unroll
    for (int i = 0; i < KMAX; ++i) {
      if (i >= KMAX - k) {
        const float w = __fdiv_rn(t.s[i], sum);
        const float* src = vert_ws + (int64_t)t.id[i] * kCh;
#pragma unroll
        for (int c = 0; c < kCh; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(__ldg(src + c), w));
        if (out_idx) out_idx[n * k + (i - (KMAX - k))] = t.id[i];
      }
    }
    float* dst = out_cl + n * kCh;
#pragma unroll
    for (int c = 0; c < kCh; ++c) dst[c] = acc[c];
  }
}

// mean = (z+ + z- + y+ + y- + x+ + x-) / 6.0, then (w - mean) * 0.7 + mean  (Deformer.py:536-540)
__device__ __forceinline__ float stencil(float w, float zp, float zm, float yp, float ym, float xp, float xm) {
  const float sum6 = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(zp, zm), yp), ym), xp), xm);
  const float mean = __fdiv_rn(sum6, 6.f);
  return __fadd_rn(__fmul_rn(__fsub_rn(w, mean), 0.7f), mean);
}

// One pass of smooth_weights (Deformer.py:533-544) over a channels-last [D,H,W,24] buffer, one thread per voxel.
// smooth = 0: no stencil and no renormalisation (what `times = 0` leaves).  out_ncdhw != NULL marks the last pass: it
// applies the zero_below threshold (LBSWsmpl.py:10) and also writes the reference layout [24,D,H,W].
__global__ void __launch_bounds__(256)
lbsw_smooth_kernel(const float* __restrict__ src, float* __restrict__ dst, float* __restrict__ out_ncdhw, int D,
                   int H, int W, int smooth, float zero_below) {
  const int64_t S = (int64_t)D * H * W;
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= S) return;
  const int x = (int)(n % W), y = (int)((n / W) % H), z = (int)(n / ((int64_t)W * H));
  const float4* c4 = reinterpret_cast<const float4*>(src + n * kCh);
  float w[kCh];
#pragma unroll
  for (int q = 0; q < kCh / 4; ++q) {
    const float4 v = __ldg(c4 + q);
    w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w;
  }
  if (smooth) {
    const bool interior = x >= 1 && x <= W - 2 && y >= 1 && y <= H - 2 && z >= 1 && z <= D - 2;
    if (interior) {
      const int64_t sz = (int64_t)H * W * kCh, sy = (int64_t)W * kCh;
      const float4* zp = c4 + sz / 4; const float4* zm = c4 - sz / 4;
      const float4* yp = c4 + sy / 4; const float4* ym = c4 - sy / 4;
      const float4* xp = c4 + kCh / 4; const float4* xm = c4 - kCh / 4;
#pragma unroll
      for (int q = 0; q < kCh / 4; ++q) {
        const float4 a = __ldg(zp + q), b = __ldg(zm + q), c = __ldg(yp + q), d = __ldg(ym + q);
        const float4 e = __ldg(xp + q), f = __ldg(xm + q);
        w[4 * q + 0] = stencil(w[4 * q + 0], a.x, b.x, c.x, d.x, e.x, f.x);
        w[4 * q + 1] = stencil(w[4 * q + 1], a.y, b.y, c.y, d.y, e.y, f.y);
        w[4 * q + 2] = stencil(w[4 * q + 2], a.z, b.z, c.z, d.z, e.z, f.z);
        w[4 * q + 3] = stencil(w[4 * q + 3], a.w, b.w, c.w, d.w, e.w, f.w);
      }
    }
    float sum = 0.f;
#pragma unroll
    for (int c = 0; c < kCh; ++c) sum = __fadd_rn(sum, w[c]);
#pragma unroll
    for (int c = 0; c < kCh; ++c) w[c] = __fdiv_rn(w[c], sum);
  }
  if (out_ncdhw) {
    if (zero_below > 0.f) {
#pragma unroll
      for (int c = 0; c < kCh; ++c) w[c] = w[c] < zero_below ? 0.f : w[c];
    }
#pragma unroll
    for (int c = 0; c < kCh; ++c) out_ncdhw[c * S + n] = w[c];
  }
  float4* d4 = reinterpret_cast<float4*>(dst + n * kCh);
#pragma unroll
  for (int q = 0; q < kCh / 4; ++q) d4[q] = make_float4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]);
}

template <int KMAX>
int knn_launch(const float* verts, const float* vert_ws, int V, const float* bmin, const float* bmax, int W, int H,
               int D, int align_corners, int k, float* out_cl, int32_t* out_idx, cudaStream_t st) {
  const size_t smem = (size_t)V * sizeof(float4);
  cudaError_t e = cudaFuncSetAttribute(lbsw_knn_kernel<KMAX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { cudaGetLastError(); return (int)e; }
  int per_sm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lbsw_knn_kernel<KMAX>, kKnnThreads, smem);
  if (e != cudaSuccess) { cudaGetLastError(); return (int)e; }
  if (per_sm < 1) per_sm = 1;
  const int64_t bricks = (int64_t)((W + kBx - 1) / kBx) * ((H + kBy - 1) / kBy) * ((D + kBz - 1) / kBz);
  const int g = stride_grid(bricks * 32, kKnnThreads, per_sm);
  lbsw_knn_kernel<KMAX><<<g, kKnnThreads, smem, st>>>(verts, vert_ws, V, bmin[0], bmin[1], bmin[2], bmax[0], bmax[1],
                                                      bmax[2], W, H, D, align_corners, k, out_cl, out_idx);
  return launch_status();
}

bool misaligned(const void* p) { return ((uintptr_t)p & 15) != 0; }

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_lbsw_knn_blend(const float* verts, const float* vert_ws, int V, int C, const float bmin[3],
                                    const float bmax[3], int W, int H, int D, int align_corners, int k, float* out_cl,
                                    int32_t* out_idx, recmv_stream_t stream) {
  if (!verts || !vert_ws || !bmin || !bmax || !out_cl) return RECMV_E_NULL;
  if (C != kCh || V <= 0 || W <= 0 || H <= 0 || D <= 0 || k < 1 || k > V) return RECMV_E_SHAPE;
  if (align_corners && (W < 2 || H < 2 || D < 2)) return RECMV_E_SHAPE;   // c / (res - 1) divides by zero
  if (k > 32 || V > kMaxVerts || (int64_t)W * H * D > ((int64_t)1 << 31) / kCh) return RECMV_E_RANGE;
  cudaStream_t st = (cudaStream_t)stream;
  if (k <= 8) return knn_launch<8>(verts, vert_ws, V, bmin, bmax, W, H, D, align_corners, k, out_cl, out_idx, st);
  if (k <= 16) return knn_launch<16>(verts, vert_ws, V, bmin, bmax, W, H, D, align_corners, k, out_cl, out_idx, st);
  return knn_launch<32>(verts, vert_ws, V, bmin, bmax, W, H, D, align_corners, k, out_cl, out_idx, st);
}

extern "C" int recmv_lbsw_smooth(float* buf_a, float* buf_b, int D, int H, int W, int times, float zero_below,
                                 float* out_ncdhw, float* out_cl, recmv_stream_t stream) {
  if (!buf_a || !out_ncdhw || !out_cl || (times >= 2 && !buf_b)) return RECMV_E_NULL;
  if (D <= 0 || H <= 0 || W <= 0 || times < 0) return RECMV_E_SHAPE;
  if (misaligned(buf_a) || misaligned(buf_b) || misaligned(out_cl)) return RECMV_E_SHAPE;
  if (out_cl == buf_a || out_cl == buf_b || buf_a == buf_b) return RECMV_E_SHAPE;
  if ((int64_t)W * H * D > ((int64_t)1 << 31) / kCh) return RECMV_E_RANGE;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t S = (int64_t)D * H * W;
  const int g = (int)((S + 255) / 256);
  if (times == 0) {
    lbsw_smooth_kernel<<<g, 256, 0, st>>>(buf_a, out_cl, out_ncdhw, D, H, W, 0, zero_below);
    return launch_status();
  }
  float* src = buf_a;
  float* spare = buf_b;
  for (int p = 0; p < times; ++p) {
    const bool last = p == times - 1;
    lbsw_smooth_kernel<<<g, 256, 0, st>>>(src, last ? out_cl : spare, last ? out_ncdhw : nullptr, D, H, W, 1,
                                          zero_below);
    int s = launch_status();
    if (s) return s;
    float* t = src; src = spare; spare = t;
  }
  return RECMV_OK;
}

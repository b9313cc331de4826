// Differentiable K-nearest point rasterizer with a fused alpha compositor.  Replaces the pytorch3d PointsRasterizer +
// AlphaCompositor behind the reference's `pcRender` (model/CameraMine.py:347-415, weights 1 - d / r^2).
//
// Input points are already projected: [N,P,3] = (NDC x, NDC y, view z); pixel (row, col) has its centre at NDC
// (1 - (2 col + 1) / W, 1 - (2 row + 1) / H).  A point is skipped (and counted) when z < 0 (or any coordinate is not a
// number; x, y must be finite); it covers a pixel when d = (xf - x)^2 + (yf - y)^2 < r^2.  Each pixel keeps the K
// covering points with the smallest (z, packed index n * P + p), sorted, so equal depths go to the lower index and the
// result does not depend on the order in which a tile meets its points.  Composite with alpha_k = 1 - d_k / r^2:
// T_0 = 1, image[g_k] += f_k alpha_k T_k, T_{k+1} = T_k (1 - alpha_k); g_k = 0 when p < split_size, else 1.
//
// Forward, four launches (no per-bin cap, no point is ever dropped):
//   1. points_setup_kernel   one thread per (frame, point): cull, clip the disc's pixel bbox, write a 32-byte record,
//                            count the point's tiles and add it to the histogram of the 32x8-pixel tiles it touches;
//   2. raster_scan_kernel    (tile_scan.cuh) twice: the per-point tile counts -> each point's contiguous range of
//                            (tile, point) pair slots, and the tile histogram -> per-tile list offsets;
//   3. points_emit_kernel    counting sort: each point appends its packed index to the list of every tile it touches;
//   4. points_tile_kernel    one CTA per tile, one pixel per thread: records stream through shared memory, each pixel
//                            keeps its sorted K-list (64-bit keys z << 32 | index) in shared memory, then composites
//                            in order and writes each image once (and the fragments when asked).
// Backward, two launches over the forward's workspace: the tile kernel in backward mode rebuilds each pixel's list
// bit-identically, turns it into dL/dalpha per entry (one forward and one reverse pass, O(K)), then each thread takes a
// (tile, point) pair and sums its contribution over the pixels of the tile in a fixed order into the pair's slot;
// points_grad_reduce_kernel sums every point's slots in order.  No float atomics: the gradient is bit-identical from
// run to run and on any GPU.
#include <math.h>

#include "common.cuh"
#include "tile_scan.cuh"
#include "workspace.cuh"

namespace recmv {
namespace {

constexpr int kTileW = 32, kTileH = 8;          // one warp per tile row, as in raster.cu
constexpr int kTileThreads = kTileW * kTileH;
constexpr int kSetupThreads = 256;
constexpr int kMaxK = 64;

struct __align__(16) PointRec {
  float x, y, z, f;        // NDC x, y, view z (never -0), feature
  int x0, x1, y0, y1;      // pixel bbox of the disc, clipped to the image (x1 < x0 when culled or off-screen)
};
static_assert(sizeof(PointRec) == 32, "record layout");

// Pixel-centre NDC and the squared distance, each operation rounded on its own: the forward, its fragments and the
// backward's recomputation agree bit for bit.
__device__ __forceinline__ float pixel_ndc(int i, int size) {
  return __fsub_rn(1.f, __fdiv_rn((float)(2 * i + 1), (float)size));
}

__device__ __forceinline__ float dist2(float xf, float yf, float x, float y) {
  const float dx = __fsub_rn(xf, x), dy = __fsub_rn(yf, y);
  return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
}

__device__ __forceinline__ float alpha_of(float d, float r2) { return __fsub_rn(1.f, __fdiv_rn(d, r2)); }

__global__ void __launch_bounds__(kSetupThreads) points_setup_kernel(
    const float* __restrict__ points, const float* __restrict__ features, long long NP, int H, int W, float radius,
    int tiles_x, int tiles_per_frame, long long P, PointRec* __restrict__ recs, int* __restrict__ point_counts,
    int* __restrict__ tile_counts, int* __restrict__ counters) {
  const long long gid = blockIdx.x * (long long)kSetupThreads + threadIdx.x;
  int skipped = 0;
  if (gid < NP) {
    const float x = points[3 * gid], y = points[3 * gid + 1], z = points[3 * gid + 2];
    PointRec r;
    r.x = x; r.y = y; r.z = __fadd_rn(z, 0.f);   // -0 -> +0: the bits of a non-negative z order like the value
    r.f = features ? features[gid] : 1.f;
    r.x0 = 0; r.x1 = -1; r.y0 = 0; r.y1 = -1;
    int ntile = 0;
    const bool keep = z >= 0.f && isfinite(x) && isfinite(y);   // NaN z fails too
    skipped = keep ? 0 : 1;
    if (keep) {
      // column c covers when |c - cx| < r W / 2 with cx = ((1 - x) W - 1) / 2 (rows alike); the 1/100-pixel slack keeps
      // the bbox conservative under rounding -- the tile kernel's exact test decides
      const float cx = 0.5f * ((1.f - x) * (float)W - 1.f), cy = 0.5f * ((1.f - y) * (float)H - 1.f);
      const float rx = 0.5f * radius * (float)W + 0.01f, ry = 0.5f * radius * (float)H + 0.01f;
      const float lx = floorf(cx - rx), hx = ceilf(cx + rx), ly = floorf(cy - ry), hy = ceilf(cy + ry);
      if (hx >= 0.f && lx <= (float)(W - 1) && hy >= 0.f && ly <= (float)(H - 1)) {
        r.x0 = (int)fmaxf(lx, 0.f); r.x1 = (int)fminf(hx, (float)(W - 1));
        r.y0 = (int)fmaxf(ly, 0.f); r.y1 = (int)fminf(hy, (float)(H - 1));
        const int tx0 = r.x0 / kTileW, tx1 = r.x1 / kTileW, ty0 = r.y0 / kTileH, ty1 = r.y1 / kTileH;
        ntile = (tx1 - tx0 + 1) * (ty1 - ty0 + 1);
        int* tc = tile_counts + (gid / P) * tiles_per_frame;
        for (int ty = ty0; ty <= ty1; ++ty)
          for (int tx = tx0; tx <= tx1; ++tx) atomicAdd(tc + ty * tiles_x + tx, 1);
      }
    }
    point_counts[gid] = ntile;
    float4* dst = reinterpret_cast<float4*>(recs + gid);
    const float4* src = reinterpret_cast<const float4*>(&r);
    dst[0] = src[0];
    dst[1] = src[1];
  }
  const unsigned m = __ballot_sync(0xffffffffu, skipped);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(counters + 1, __popc(m));
}

__global__ void __launch_bounds__(kSetupThreads) points_emit_kernel(const PointRec* __restrict__ recs, long long NP,
                                                                    long long P, int tiles_x, int tiles_per_frame,
                                                                    long long* __restrict__ cursor, long long capacity,
                                                                    int* __restrict__ list) {
  const long long gid = blockIdx.x * (long long)kSetupThreads + threadIdx.x;
  if (gid >= NP) return;
  const int4 bb = reinterpret_cast<const int4*>(recs + gid)[1];   // x0, x1, y0, y1
  if (bb.y < bb.x) return;
  long long* cur = cursor + (gid / P) * tiles_per_frame;
  for (int ty = bb.z / kTileH; ty <= bb.w / kTileH; ++ty)
    for (int tx = bb.x / kTileW; tx <= bb.y / kTileW; ++tx) {
      const long long pos = (long long)atomicAdd((unsigned long long*)(cur + ty * tiles_x + tx), 1ull);
      if (pos < capacity) list[pos] = (int)gid;
    }
}

constexpr int kChunk = kTileThreads;   // records per shared-memory chunk: one per thread

struct TileArgs {
  const PointRec* recs;
  const int* list;
  const long long* tile_off;
  const long long* point_off;
  int H, W, tiles_x, tiles_per_frame, K, split, G;
  long long P;
  float r2;
};

// Dynamic shared memory: K * 256 64-bit entries, entry k of pixel t at [k * 256 + t] (conflict-free per warp).  While
// selecting, an entry is the key z_bits << 32 | index; afterwards the backward reuses it as index << 32 | payload.
// Image g of the forward is out_img[g], its cotangent in the backward grad_img[g] (index 1 unused when G = 1).
template <bool kBackward>
__global__ void __launch_bounds__(kTileThreads) points_tile_kernel(TileArgs a, float* __restrict__ out_img0,
                                                                   float* __restrict__ out_img1,
                                                                   long long* __restrict__ out_idx,
                                                                   float* __restrict__ out_zbuf,
                                                                   float* __restrict__ out_dists,
                                                                   const float* __restrict__ grad_img0,
                                                                   const float* __restrict__ grad_img1,
                                                                   float2* __restrict__ pair_grad,
                                                                   int* __restrict__ counters) {
  extern __shared__ unsigned long long slist[];
  __shared__ PointRec srec[kChunk];
  __shared__ int sidx[kChunk];
  __shared__ int scnt[kTileThreads];
  if (!kBackward && counters[3]) return;   // the pair list overflowed: the caller re-runs with a larger one
  const int n = blockIdx.y, tile = blockIdx.x;
  const int tx = tile % a.tiles_x, ty = tile / a.tiles_x;
  const int tid = threadIdx.x;
  const int col = tx * kTileW + (tid % kTileW), row = ty * kTileH + (tid / kTileW);
  const bool inside = col < a.W && row < a.H;
  const float xf = pixel_ndc(col, a.W), yf = pixel_ndc(row, a.H);
  const long long t = (long long)n * a.tiles_per_frame + tile;
  const int beg = (int)a.tile_off[t], end = (int)a.tile_off[t + 1];   // list entries < capacity <= INT32_MAX
  const int K = a.K;
  unsigned long long* my = slist + tid;
  int cnt = 0;
  for (int c0 = beg; c0 < end; c0 += kChunk) {
    const int m_cnt = min(kChunk, end - c0);
    __syncthreads();
    if (tid < m_cnt) {
      const int g = a.list[c0 + tid];
      sidx[tid] = g;
      const float4* src = reinterpret_cast<const float4*>(a.recs + g);
      float4* dst = reinterpret_cast<float4*>(srec + tid);
      dst[0] = __ldg(src);
      dst[1] = __ldg(src + 1);
    }
    __syncthreads();
    // the warp owns one tile row: a ballot over 32 records keeps those whose rows include it
    for (int k0 = 0; k0 < m_cnt; k0 += 32) {
      const int kl = k0 + (tid & 31);
      unsigned m = __ballot_sync(0xffffffffu, kl < m_cnt && srec[kl].y0 <= row && row <= srec[kl].y1);
      while (m) {
        const int k = k0 + __ffs(m) - 1;
        m &= m - 1;
        const PointRec& r = srec[k];
        if (!inside || col < r.x0 || col > r.x1) continue;
        if (!(dist2(xf, yf, r.x, r.y) < a.r2)) continue;
        const unsigned long long key = ((unsigned long long)__float_as_uint(r.z) << 32) | (unsigned)sidx[k];
        int pos;
        if (cnt < K) {
          pos = cnt++;
        } else {
          if (key >= my[(K - 1) * kTileThreads]) continue;
          pos = K - 1;
        }
        while (pos > 0) {   // insertion into the sorted list
          const unsigned long long prev = my[(pos - 1) * kTileThreads];
          if (prev < key) break;
          my[pos * kTileThreads] = prev;
          --pos;
        }
        my[pos * kTileThreads] = key;
      }
    }
  }
  const long long pix = ((long long)n * a.H + row) * a.W + col;
  const long long base = (long long)n * a.P;
  if (!kBackward) {
    const int covered = __syncthreads_count(inside && cnt > 0);
    if (tid == 0 && covered) atomicAdd(counters, covered);
    if (!inside) return;
    float acc0 = 0.f, acc1 = 0.f, T = 1.f;
    for (int k = 0; k < cnt; ++k) {
      const int g = (int)(unsigned)my[k * kTileThreads];
      const float4 q = __ldg(reinterpret_cast<const float4*>(a.recs + g));
      const float d = dist2(xf, yf, q.x, q.y);
      const float al = alpha_of(d, a.r2);
      const float c = __fmul_rn(__fmul_rn(q.w, al), T);
      if ((g - base) < a.split) acc0 = __fadd_rn(acc0, c); else acc1 = __fadd_rn(acc1, c);
      T = __fmul_rn(T, __fsub_rn(1.f, al));
      if (out_idx) out_idx[pix * K + k] = g;
      if (out_zbuf) out_zbuf[pix * K + k] = q.z;
      if (out_dists) out_dists[pix * K + k] = d;
    }
    for (int k = cnt; k < K; ++k) {
      if (out_idx) out_idx[pix * K + k] = -1;
      if (out_zbuf) out_zbuf[pix * K + k] = -1.f;
      if (out_dists) out_dists[pix * K + k] = -1.f;
    }
    out_img0[pix] = acc0;
    if (a.G == 2) out_img1[pix] = acc1;
    return;
  }
  // ---- backward: dL/dalpha of every entry, O(K) ----
  if (inside && cnt > 0) {
    const float G0 = grad_img0[pix], G1 = a.G == 2 ? grad_img1[pix] : 0.f;
    float T = 1.f;
    for (int k = 0; k < cnt; ++k) {   // entry <- index << 32 | T_k
      const unsigned g = (unsigned)my[k * kTileThreads];
      const float4 q = __ldg(reinterpret_cast<const float4*>(a.recs + g));
      my[k * kTileThreads] = ((unsigned long long)g << 32) | __float_as_uint(T);
      T = __fmul_rn(T, __fsub_rn(1.f, alpha_of(dist2(xf, yf, q.x, q.y), a.r2)));
    }
    // dL/dalpha_t = sum_g G_g (f_t [grp_t = g] T_t - S_{t,g} / (1 - alpha_t + 1e-9)), S_{t,g} = sum_{k>t} of group g's
    // f_k alpha_k T_k
    float S0 = 0.f, S1 = 0.f;
    for (int k = cnt - 1; k >= 0; --k) {
      const unsigned long long e = my[k * kTileThreads];
      const unsigned g = (unsigned)(e >> 32);
      const float Tk = __uint_as_float((unsigned)e);
      const float4 q = __ldg(reinterpret_cast<const float4*>(a.recs + g));
      const float al = alpha_of(dist2(xf, yf, q.x, q.y), a.r2);
      const bool first = ((long long)g - base) < a.split;
      const float ft = __fmul_rn(q.w, Tk);
      const float own = __fmul_rn(first ? G0 : G1, ft);
      const float rest = __fadd_rn(__fmul_rn(G0, S0), __fmul_rn(G1, S1));
      const float da = __fsub_rn(own, __fdiv_rn(rest, __fadd_rn(__fsub_rn(1.f, al), 1e-9f)));
      if (first) S0 = __fadd_rn(S0, __fmul_rn(ft, al)); else S1 = __fadd_rn(S1, __fmul_rn(ft, al));
      my[k * kTileThreads] = ((unsigned long long)g << 32) | __float_as_uint(da);
    }
  }
  scnt[tid] = inside ? cnt : 0;
  __syncthreads();
  // ---- each thread one (tile, point) pair: sum over the disc's pixels in this tile, row-major ----
  const float inv_r2x2 = __fdiv_rn(2.f, a.r2);
  for (int c0 = beg; c0 < end; c0 += kTileThreads) {
    if (c0 + tid >= end) break;
    const int g = a.list[c0 + tid];
    const float4 q = __ldg(reinterpret_cast<const float4*>(a.recs + g));
    const int4 bb = __ldg(reinterpret_cast<const int4*>(a.recs + g) + 1);
    const int cx0 = max(bb.x, tx * kTileW), cx1 = min(bb.y, tx * kTileW + kTileW - 1);
    const int ry0 = max(bb.z, ty * kTileH), ry1 = min(bb.w, ty * kTileH + kTileH - 1);
    float gx = 0.f, gy = 0.f;
    for (int rr = ry0; rr <= ry1; ++rr) {
      const float yq = pixel_ndc(rr, a.H);
      for (int cc = cx0; cc <= cx1; ++cc) {
        const float xq = pixel_ndc(cc, a.W);
        if (!(dist2(xq, yq, q.x, q.y) < a.r2)) continue;
        const int lp = (rr - ty * kTileH) * kTileW + (cc - tx * kTileW);
        const int c = scnt[lp];
        for (int k = 0; k < c; ++k) {
          const unsigned long long e = slist[k * kTileThreads + lp];
          if ((int)(e >> 32) != g) continue;
          const float da = __fmul_rn(__uint_as_float((unsigned)e), inv_r2x2);   // dalpha/dx = 2 (xf - x) / r^2
          gx = __fadd_rn(gx, __fmul_rn(da, __fsub_rn(xq, q.x)));
          gy = __fadd_rn(gy, __fmul_rn(da, __fsub_rn(yq, q.y)));
          break;
        }
      }
    }
    const int ptx0 = bb.x / kTileW, ptx1 = bb.y / kTileW, pty0 = bb.z / kTileH;
    pair_grad[a.point_off[g] + (long long)(ty - pty0) * (ptx1 - ptx0 + 1) + (tx - ptx0)] = make_float2(gx, gy);
  }
}

__global__ void __launch_bounds__(kSetupThreads) points_grad_reduce_kernel(const long long* __restrict__ point_off,
                                                                           const float2* __restrict__ pair_grad,
                                                                           long long NP, float* __restrict__ grad) {
  const long long gid = blockIdx.x * (long long)kSetupThreads + threadIdx.x;
  if (gid >= NP) return;
  float sx = 0.f, sy = 0.f;
  for (long long i = point_off[gid], e = point_off[gid + 1]; i < e; ++i) {
    const float2 v = pair_grad[i];
    sx = __fadd_rn(sx, v.x);
    sy = __fadd_rn(sy, v.y);
  }
  grad[3 * gid] = sx;
  grad[3 * gid + 1] = sy;
  grad[3 * gid + 2] = 0.f;
}

struct PointsWs {
  PointRec* recs;
  int* point_counts;
  long long* point_off;   // NP + 1
  int* tile_counts;
  long long* tile_off;    // ntiles + 1
  long long* cursor;
  int* list;
};

PointsWs points_layout(Carve& c, long long NP, long long ntiles, long long capacity) {
  PointsWs w;
  w.recs = c.take<PointRec>(NP);
  w.point_counts = c.take<int>(NP);
  w.point_off = c.take<long long>(NP + 1);
  w.tile_counts = c.take<int>(ntiles);
  w.tile_off = c.take<long long>(ntiles + 1);
  w.cursor = c.take<long long>(ntiles);
  w.list = c.take<int>(capacity);
  return w;
}

int points_dims(int N, int64_t P, int H, int W) {
  if (N < 0 || P < 0 || H <= 0 || W <= 0) return RECMV_E_SHAPE;
  if ((int64_t)N * P > 0x7fffffffLL || (int64_t)N * H * W > 2000000000LL) return RECMV_E_RANGE;
  return RECMV_OK;
}

int check_args(int N, int64_t P, int H, int W, float radius, int K, int64_t split_size, int num_images) {
  if (K < 1 || split_size < 0 || split_size > P) return RECMV_E_SHAPE;
  if (!(radius > 0.f) || !isfinite(radius)) return RECMV_E_SHAPE;
  if (num_images != 1 && num_images != 2) return RECMV_E_SHAPE;
  const int s = points_dims(N, P, H, W);
  if (s) return s;
  if (K > kMaxK) return RECMV_E_RANGE;
  if (N > 65535) return RECMV_E_RANGE;   // frames are the tile pass's grid.y
  return RECMV_OK;
}

template <bool kBackward>
int launch_tile(const TileArgs& a, int N, cudaStream_t st, float* images, long long* idx, float* zbuf, float* dists,
                const float* grad_images, float2* pair_grad, int* counters) {
  const long long NHW = (long long)N * a.H * a.W;   // image planes [G][N][H][W]
  float* img1 = images && a.G == 2 ? images + NHW : nullptr;
  const float* gimg1 = grad_images && a.G == 2 ? grad_images + NHW : nullptr;
  const size_t smem = (size_t)a.K * kTileThreads * sizeof(unsigned long long);
  cudaError_t e = cudaFuncSetAttribute(points_tile_kernel<kBackward>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem);
  if (e != cudaSuccess) return (int)e;
  points_tile_kernel<kBackward><<<dim3(a.tiles_per_frame, N), kTileThreads, smem, st>>>(
      a, images, img1, idx, zbuf, dists, grad_images, gimg1, pair_grad, counters);
  return launch_status();
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_points_raster_workspace_bytes(int N, int64_t P, int H, int W, int64_t capacity, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  if (capacity < 0) return RECMV_E_SHAPE;
  const int s = points_dims(N, P, H, W);
  if (s) return s;
  if (capacity > 0x7fffffffLL) return RECMV_E_RANGE;
  const long long ntiles = (long long)N * ((W + kTileW - 1) / kTileW) * ((H + kTileH - 1) / kTileH);
  *bytes = layout_bytes(points_layout, (long long)N * P, ntiles, capacity);
  return RECMV_OK;
}

extern "C" int recmv_rasterize_points(const float* points, const float* features, int N, int64_t P, int H, int W,
                                      float radius, int K, int64_t split_size, int num_images, void* workspace,
                                      int64_t capacity, float* out_images, int64_t* out_idx, float* out_zbuf,
                                      float* out_dists, int32_t* counters, recmv_stream_t stream) {
  int s = check_args(N, P, H, W, radius, K, split_size, num_images);
  if (s) return s;
  if (capacity < 0) return RECMV_E_SHAPE;
  if (capacity > 0x7fffffffLL) return RECMV_E_RANGE;
  if (!counters) return RECMV_E_NULL;
  if (N > 0 && (!workspace || !out_images)) return RECMV_E_NULL;
  if (N > 0 && P > 0 && !points) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(counters, 0, 4 * sizeof(int32_t), st);
  if (e != cudaSuccess) return (int)e;
  if (N == 0) return RECMV_OK;
  const int tiles_x = (W + kTileW - 1) / kTileW, tiles_y = (H + kTileH - 1) / kTileH;
  const int tiles_per_frame = tiles_x * tiles_y;
  const long long ntiles = (long long)N * tiles_per_frame;
  const long long NP = (long long)N * P;
  const PointsWs w = carve(workspace, points_layout, NP, ntiles, capacity);
  e = cudaMemsetAsync(w.tile_counts, 0, (size_t)ntiles * 4, st);
  if (e != cudaSuccess) return (int)e;
  const int nb = (int)((NP + kSetupThreads - 1) / kSetupThreads);
  if (NP > 0) {
    points_setup_kernel<<<nb, kSetupThreads, 0, st>>>(points, features, NP, H, W, radius, tiles_x, tiles_per_frame, P,
                                                      w.recs, w.point_counts, w.tile_counts, counters);
    s = launch_status();
    if (s) return s;
    // the point-major pair ranges (same total as the tile scan below, which then overwrites counters[2..3] alike)
    raster_scan_kernel<<<1, kScanThreads, 0, st>>>(w.point_counts, (int)NP, w.point_off, nullptr, capacity, counters);
    s = launch_status();
    if (s) return s;
  }
  raster_scan_kernel<<<1, kScanThreads, 0, st>>>(w.tile_counts, (int)ntiles, w.tile_off, w.cursor, capacity, counters);
  s = launch_status();
  if (s) return s;
  if (NP > 0) {
    points_emit_kernel<<<nb, kSetupThreads, 0, st>>>(w.recs, NP, P, tiles_x, tiles_per_frame, w.cursor, capacity, w.list);
    s = launch_status();
    if (s) return s;
  }
  TileArgs a{w.recs, w.list, w.tile_off, w.point_off, H, W, tiles_x, tiles_per_frame, K, (int)split_size, num_images,
             (long long)P, radius * radius};
  return launch_tile<false>(a, N, st, out_images, (long long*)out_idx, out_zbuf, out_dists, nullptr, nullptr, counters);
}

extern "C" int recmv_rasterize_points_backward(int N, int64_t P, int H, int W, float radius, int K, int64_t split_size,
                                               int num_images, const void* workspace, int64_t pairs,
                                               const float* grad_images, float* pair_scratch, float* grad_points,
                                               recmv_stream_t stream) {
  int s = check_args(N, P, H, W, radius, K, split_size, num_images);
  if (s) return s;
  if (pairs < 0) return RECMV_E_SHAPE;
  if (pairs > 0x7fffffffLL) return RECMV_E_RANGE;
  if ((int64_t)N * P == 0) return RECMV_OK;
  if (!workspace || !grad_images || !grad_points || (pairs > 0 && !pair_scratch)) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  const int tiles_x = (W + kTileW - 1) / kTileW, tiles_y = (H + kTileH - 1) / kTileH;
  const int tiles_per_frame = tiles_x * tiles_y;
  const long long ntiles = (long long)N * tiles_per_frame;
  const long long NP = (long long)N * P;
  // the list holds the forward's pairs
  const PointsWs w = carve(const_cast<void*>(workspace), points_layout, NP, ntiles, pairs);
  TileArgs a{w.recs, w.list, w.tile_off, w.point_off, H, W, tiles_x, tiles_per_frame, K, (int)split_size, num_images,
             (long long)P, radius * radius};
  float2* pg = reinterpret_cast<float2*>(pair_scratch);
  s = launch_tile<true>(a, N, st, nullptr, nullptr, nullptr, nullptr, grad_images, pg, nullptr);
  if (s) return s;
  points_grad_reduce_kernel<<<(int)((NP + kSetupThreads - 1) / kSetupThreads), kSetupThreads, 0, st>>>(w.point_off, pg,
                                                                                                        NP, grad_points);
  return launch_status();
}

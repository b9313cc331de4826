// Sparse z-buffer probe: the mesh rasterizer's front depth at the four bilinear taps of a set of query points, sampled
// as the reference's visibility test samples its full-frame zbuf (`z_buff_check` of fl_visible_by_body_zbuff,
// OptimGarmentNetwork.py:1374-1465, and check_zbuf_body, fl_optimizer.py:30-59) -- without rasterizing the frame.
//
// Per query (n, q) with screen point (sx, sy) and normalisation size (w, h) = norm_size[n]:
//   u = 2 sx / w - 1, v = 2 sy / h - 1                       (the reference's own normalisation, each op rounded)
//   ix = ((u + 1) / 2) (W - 1), iy = ((v + 1) / 2) (H - 1)   (ATen's grid_sampler_2d, align_corners=True)
//   taps nw, ne, sw, se at (floor ix + {0,1,0,1}, floor iy + {0,0,1,1}) with ATen's weights; a tap outside the image
//   contributes 0 (zeros padding); a tap's value is the rasterizer's zbuf at that pixel, or fill[n] where the
//   reference's `zbuf == -1.` test fires (background, or a covered pixel of depth exactly -1);
//   out = ((nw v_nw + ne v_ne) + sw v_sw) + se v_se, accumulated with fused multiply-adds as ATen's CUDA kernel is;
//   a non-finite ix or iy gives 0.
//
// The depth at a tap is the tile pass's lexicographic minimum of (zbuf, packed face) over the faces that cover the
// pixel (raster.cu), found by scattering the faces onto the taps instead of gathering faces per pixel:
//   1. zprobe_tap_kernel      one thread per query: its four tap pixels, and the histogram of the 32x8 tiles they fall in;
//   2. raster_scan_kernel     offsets of each tile's taps (tile_scan.cuh);
//   3. zprobe_emit_kernel     one thread per tap: append it to its tile's list;
//   4. zprobe_face_kernel     one thread per (frame, face): the rasterizer's own record (make_face_rec), then for every
//                             tile of its bbox the taps listed there, tested with the rasterizer's shade(); a covering
//                             candidate the tile pass would accept (zbuf < +inf) goes into a 64-bit atomicMin on
//                             (order-preserving bits of zbuf) << 32 | packed face, so the winner does not depend on
//                             the order in which faces arrive;
//   5. zprobe_combine_kernel  one thread per query: the winner's record is rebuilt and shaded at the tap (the tile
//                             pass's output step), then the fill rule and the bilinear sum.
// No pair list, no capacity and no host read: the workspace depends on N, Q and the image size only.
#include <math.h>

#include "common.cuh"
#include "raster_common.cuh"
#include "tile_scan.cuh"
#include "workspace.cuh"

namespace recmv {
namespace {

constexpr int kThreads = 256;
constexpr unsigned long long kNoHit = ~0ull;

struct Taps {
  float w[4];   // ATen's weights nw, ne, sw, se
  int col[4], row[4];
  bool valid;   // false: a non-finite or far-off coordinate, every tap is outside the image
};

// The query's unnormalised sample position and taps, with the reference's rounding at every step.
__device__ __forceinline__ Taps query_taps(const float* __restrict__ pts, long long i, int D,
                                           const float* __restrict__ norm_size, int n, int H, int W) {
  Taps t;
  const float sx = pts[i * D], sy = pts[i * D + 1];
  const float u = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, sx), norm_size[2 * n]), 1.f);
  const float v = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, sy), norm_size[2 * n + 1]), 1.f);
  const float ix = __fmul_rn(__fdiv_rn(__fadd_rn(u, 1.f), 2.f), (float)(W - 1));
  const float iy = __fmul_rn(__fdiv_rn(__fadd_rn(v, 1.f), 2.f), (float)(H - 1));
  // beyond these bounds every tap is outside the image; inside them the integer conversions are exact
  t.valid = ix > -2.f && ix < (float)W + 1.f && iy > -2.f && iy < (float)H + 1.f;   // NaN fails
  if (!t.valid) return t;
  const int x = (int)floorf(ix), y = (int)floorf(iy);
  const float fx0 = (float)x, fx1 = (float)(x + 1), fy0 = (float)y, fy1 = (float)(y + 1);
  t.w[0] = __fmul_rn(__fsub_rn(fx1, ix), __fsub_rn(fy1, iy));
  t.w[1] = __fmul_rn(__fsub_rn(ix, fx0), __fsub_rn(fy1, iy));
  t.w[2] = __fmul_rn(__fsub_rn(fx1, ix), __fsub_rn(iy, fy0));
  t.w[3] = __fmul_rn(__fsub_rn(ix, fx0), __fsub_rn(iy, fy0));
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    t.col[c] = x + (c & 1);
    t.row[c] = y + (c >> 1);
  }
  return t;
}

__device__ __forceinline__ bool in_image(int col, int row, int H, int W) {
  return col >= 0 && col < W && row >= 0 && row < H;
}

__global__ void __launch_bounds__(kThreads) zprobe_tap_kernel(const float* __restrict__ pts, long long NQ, int Q, int D,
                                                              const float* __restrict__ norm_size, int H, int W,
                                                              int tiles_x, int tiles_per_frame,
                                                              int* __restrict__ tap_pix,
                                                              unsigned long long* __restrict__ keys,
                                                              int* __restrict__ tile_counts) {
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= NQ) return;
  const int n = (int)(i / Q);
  const Taps t = query_taps(pts, i, D, norm_size, n, H, W);
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    int p = -1;
    if (t.valid && in_image(t.col[c], t.row[c], H, W)) {
      p = t.row[c] * W + t.col[c];
      atomicAdd(tile_counts + (long long)n * tiles_per_frame + (t.row[c] / kTileH) * tiles_x + t.col[c] / kTileW, 1);
    }
    tap_pix[4 * i + c] = p;
    keys[4 * i + c] = kNoHit;
  }
}

__global__ void __launch_bounds__(kThreads) zprobe_emit_kernel(const int* __restrict__ tap_pix, long long T, int Q, int W,
                                                               int tiles_x, int tiles_per_frame,
                                                               long long* __restrict__ cursor, int* __restrict__ list) {
  const long long k = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (k >= T) return;
  const int p = tap_pix[k];
  if (p < 0) return;
  const int n = (int)(k / (4ll * Q)), col = p % W, row = p / W;
  const long long pos = (long long)atomicAdd(
      (unsigned long long*)(cursor + (long long)n * tiles_per_frame + (row / kTileH) * tiles_x + col / kTileW), 1ull);
  list[pos] = (int)k;
}

__global__ void __launch_bounds__(kThreads) zprobe_face_kernel(
    const float* __restrict__ verts, int V, const long long* __restrict__ faces, int F, int N,
    const float* __restrict__ cameras, int H, int W, float z_clip, float area_eps, int tiles_x, int tiles_per_frame,
    const long long* __restrict__ offsets, const int* __restrict__ list, const int* __restrict__ tap_pix,
    unsigned long long* __restrict__ keys) {
  const long long gid = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (gid >= (long long)N * F) return;
  const int n = (int)(gid / F), f = (int)(gid % F);
  float cam[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) cam[i] = __ldg(cameras + 16 * n + i);
  FaceRec r;
  make_face_rec(verts, faces, cam, V, f, n, H, W, z_clip, area_eps, r);
  if (r.x1 < r.x0) return;
  const long long* off = offsets + (long long)n * tiles_per_frame;
  for (int ty = r.y0 / kTileH; ty <= r.y1 / kTileH; ++ty)
    for (int tx = r.x0 / kTileW; tx <= r.x1 / kTileW; ++tx) {
      const int t = ty * tiles_x + tx;
      const long long end = off[t + 1];
      for (long long j = off[t]; j < end; ++j) {
        const int k = __ldg(list + j);
        const int p = __ldg(tap_pix + k);
        const int col = p % W, row = p / W;
        if (col < r.x0 || col > r.x1 || row < r.y0 || row > r.y1) continue;
        float bp[3], zb;
        if (!shade(r, (float)(col - r.x0), (float)(row - r.y0), bp, zb) || !(zb < INFINITY)) continue;
        // order-preserving bits; -0 and +0 compare equal in the tile pass, so they share a key and the face decides
        unsigned b = __float_as_uint(zb == 0.f ? 0.f : zb);
        b = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
        atomicMin(keys + k, ((unsigned long long)b << 32) | (unsigned)gid);
      }
    }
}

__global__ void __launch_bounds__(kThreads) zprobe_combine_kernel(
    const float* __restrict__ verts, int V, const long long* __restrict__ faces, int F,
    const float* __restrict__ cameras, int H, int W, float z_clip, float area_eps, const float* __restrict__ pts,
    long long NQ, int Q, int D, const float* __restrict__ norm_size, const float* __restrict__ fill,
    const unsigned long long* __restrict__ keys, float* __restrict__ out, float* __restrict__ tap_zbuf,
    long long* __restrict__ tap_face) {
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= NQ) return;
  const int n = (int)(i / Q);
  const Taps t = query_taps(pts, i, D, norm_size, n, H, W);
  const float bg = fill[n];
  float acc = 0.f;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    float zb = -1.f;
    long long face = -1;
    if (t.valid && in_image(t.col[c], t.row[c], H, W)) {
      const unsigned long long key = keys[4 * i + c];
      if (key != kNoHit) {
        const int g = (int)(unsigned)(key & 0xffffffffu);
        float cam[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) cam[j] = __ldg(cameras + 16 * n + j);
        FaceRec r;
        make_face_rec(verts, faces, cam, V, g - n * F, n, H, W, z_clip, area_eps, r);
        float bp[3];
        shade(r, (float)(t.col[c] - r.x0), (float)(t.row[c] - r.y0), bp, zb);
        face = g;
      }
      acc = __fmaf_rn(zb == -1.f ? bg : zb, t.w[c], acc);
    }
    if (tap_zbuf) {
      tap_zbuf[4 * i + c] = zb;
      tap_face[4 * i + c] = face;
    }
  }
  out[i] = acc;
}

struct ProbeWs {
  unsigned long long* keys;
  int* tap_pix;
  int* list;
  int* tile_counts;
  long long* offsets;   // ntiles + 1
  long long* cursor;
  int* counters;        // the scan's 4 counters (unused: the list always fits)
};

ProbeWs probe_layout(Carve& c, long long T, long long ntiles) {
  ProbeWs w;
  w.keys = c.take<unsigned long long>(T);
  w.tap_pix = c.take<int>(T);
  w.list = c.take<int>(T);
  w.tile_counts = c.take<int>(ntiles);
  w.offsets = c.take<long long>(ntiles + 1);
  w.cursor = c.take<long long>(ntiles);
  w.counters = c.take<int>(4);
  return w;
}

int probe_dims(int N, int64_t Q, int H, int W) {
  if (N < 0 || Q < 0 || H <= 0 || W <= 0) return RECMV_E_SHAPE;
  if (4 * (int64_t)N * Q > 0x7fffffffLL || (int64_t)N * H * W > 2000000000LL) return RECMV_E_RANGE;
  return RECMV_OK;
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_zbuf_probe_workspace_bytes(int N, int64_t Q, int H, int W, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  const int s = probe_dims(N, Q, H, W);
  if (s) return s;
  const long long ntiles = (long long)N * ((W + kTileW - 1) / kTileW) * ((H + kTileH - 1) / kTileH);
  *bytes = layout_bytes(probe_layout, 4ll * N * Q, ntiles);
  return RECMV_OK;
}

extern "C" int recmv_zbuf_probe(const float* verts, int V, const int64_t* faces, int64_t F, int N, const float* camera,
                                int H, int W, float z_clip, float area_eps, const float* screen_pts, int64_t Q, int D,
                                const float* norm_size, const float* fill, void* workspace, float* out,
                                float* out_tap_zbuf, int64_t* out_tap_face, recmv_stream_t stream) {
  int s = probe_dims(N, Q, H, W);
  if (s) return s;
  if (V < 0 || F < 0 || D < 2 || (F > 0 && V == 0)) return RECMV_E_SHAPE;
  if ((int64_t)N * F > 0x7fffffffLL) return RECMV_E_RANGE;
  if ((out_tap_zbuf == nullptr) != (out_tap_face == nullptr)) return RECMV_E_NULL;
  const long long NQ = (long long)N * Q;
  if (NQ == 0) return RECMV_OK;
  if (!camera || !screen_pts || !norm_size || !fill || !workspace || !out) return RECMV_E_NULL;
  if (F > 0 && (!faces || !verts)) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  const int tiles_x = (W + kTileW - 1) / kTileW, tiles_y = (H + kTileH - 1) / kTileH;
  const int tiles_per_frame = tiles_x * tiles_y;
  const long long ntiles = (long long)N * tiles_per_frame, T = 4 * NQ, NF = (long long)N * F;
  const ProbeWs w = carve(workspace, probe_layout, T, ntiles);
  cudaError_t e = cudaMemsetAsync(w.tile_counts, 0, (size_t)ntiles * 4, st);
  if (e != cudaSuccess) return (int)e;
  zprobe_tap_kernel<<<(int)((NQ + kThreads - 1) / kThreads), kThreads, 0, st>>>(
      screen_pts, NQ, (int)Q, D, norm_size, H, W, tiles_x, tiles_per_frame, w.tap_pix, w.keys, w.tile_counts);
  if ((s = launch_status())) return s;
  raster_scan_kernel<<<1, kScanThreads, 0, st>>>(w.tile_counts, (int)ntiles, w.offsets, w.cursor, 0x7fffffffffffffffLL,
                                                 w.counters);
  if ((s = launch_status())) return s;
  zprobe_emit_kernel<<<(int)((T + kThreads - 1) / kThreads), kThreads, 0, st>>>(w.tap_pix, T, (int)Q, W, tiles_x,
                                                                                 tiles_per_frame, w.cursor, w.list);
  if ((s = launch_status())) return s;
  if (NF > 0) {
    zprobe_face_kernel<<<(int)((NF + kThreads - 1) / kThreads), kThreads, 0, st>>>(
        verts, V, (const long long*)faces, (int)F, N, camera, H, W, z_clip, area_eps, tiles_x, tiles_per_frame,
        w.offsets, w.list, w.tap_pix, w.keys);
    if ((s = launch_status())) return s;
  }
  zprobe_combine_kernel<<<(int)((NQ + kThreads - 1) / kThreads), kThreads, 0, st>>>(
      verts, V, (const long long*)faces, (int)F, camera, H, W, z_clip, area_eps, screen_pts, NQ, (int)Q, D, norm_size,
      fill, w.keys, out, out_tap_zbuf, (long long*)out_tap_face);
  return launch_status();
}

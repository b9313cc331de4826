// Single-layer mesh rasterizer (faces_per_pixel = 1) in the reference camera's screen space, producing the fragments
// FindSurfacePs reads.  Replaces the pytorch3d MeshRasterizer behind `maskRender` (model/network.py:307-322:
// blur_radius 0, perspective_correct, no barycentric clipping, no back-face culling).
//
// Per frame n with camera {fx, fy, px, py, R (row-major), T}:
//   view   X_v = X R + T                                  (CameraMine.project, :169-173)
//   screen (sx, sy) = (px - fx X_v / Z_v, py - fy Y_v / Z_v); pixel (row, col) has its centre at (sx, sy) = (col, row)
//   a face is skipped (and counted) when a vertex has Z_v <= z_clip or its screen doubled area |A| <= area_eps;
//   it covers a pixel when its three screen barycentrics (edge functions / A) are all >= 0, either winding;
//   b'_i = (b_i / Z_i) / sum_j (b_j / Z_j),  zbuf = sum_i b'_i Z_i;  the smallest zbuf wins, ties to the lower packed
//   face index n * F + f -- so the result does not depend on the order in which a tile meets its faces.
//
// Four launches, no per-bin cap (no face is ever dropped):
//   1. raster_setup_kernel   one thread per (frame, face): project, cull, clip the pixel bbox, write a 96-byte
//                            record (edge coefficients relative to an integer pixel origin, 1/Z, Z, bbox), and add the
//                            face to the histogram of the 32x8-pixel tiles its bbox touches;
//   2. raster_scan_kernel    exclusive scan of the tile histogram -> per-tile offsets + cursors, pair total, overflow;
//   3. raster_emit_kernel    counting sort: each face appends its packed index to the list of every tile it touches;
//   4. raster_tile_kernel    one CTA per tile: stream the tile's records through shared memory, each thread keeps the
//                            best (zbuf, face) of its pixel in registers (each warp, one tile row, tests only the
//                            records whose rows include it), then writes every output element once.
// The pair list is sized by the caller; when it is too small the tile pass writes nothing, counters[3] is set and the
// caller re-runs with counters[2] entries.
#include <math.h>

#include "common.cuh"
#include "tile_scan.cuh"

namespace recmv {
namespace {

constexpr int kTileW = 32, kTileH = 8;          // one warp per tile row: 128-byte rows of every 4-byte output
constexpr int kTileThreads = kTileW * kTileH;
constexpr int kSetupThreads = 256;

// 24 words.  Barycentric i at pixel (col, row) = ka[i] * (col - ox) + kb[i] * (row - oy) + kc[i]; (ox, oy) = (x0, y0)
// is an integer, so col - ox and row - oy are exact and the constants stay the size of the face, not of the image.
struct __align__(16) FaceRec {
  int x0, x1, y0, y1;      // covered pixel-centre bbox, clipped to the image (x1 < x0 when the face is culled)
  float ka[3], kb[3], kc[3];
  float iz[3], z[3];
  float pad[2];
};
static_assert(sizeof(FaceRec) == 96, "record layout");

struct ScreenTri {
  float sx[3], sy[3], z[3];
};

// Every operation is rounded on its own (no contraction), so the setup and the winner's dists pass agree bit for bit.
__device__ __forceinline__ void project_face(const float* __restrict__ verts, const long long* __restrict__ faces,
                                             const float* __restrict__ cam, int V, int f, int n, ScreenTri& t,
                                             bool& bad_index) {
  bad_index = false;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const long long vi = faces[3 * (long long)f + k];
    if (vi < 0 || vi >= V) { bad_index = true; t.sx[k] = t.sy[k] = 0.f; t.z[k] = 0.f; continue; }
    const float* p = verts + ((long long)n * V + vi) * 3;
    const float X = p[0], Y = p[1], Z = p[2];
    float v[3];
#pragma unroll
    for (int j = 0; j < 3; ++j)
      v[j] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(X, cam[4 + j]), __fmul_rn(Y, cam[7 + j])), __fmul_rn(Z, cam[10 + j])),
                       cam[13 + j]);
    t.z[k] = v[2];
    t.sx[k] = __fsub_rn(cam[2], __fdiv_rn(__fmul_rn(cam[0], v[0]), v[2]));
    t.sy[k] = __fsub_rn(cam[3], __fdiv_rn(__fmul_rn(cam[1], v[1]), v[2]));
  }
}

__device__ __forceinline__ float edge_fn(float ax, float ay, float bx, float by, float cx, float cy) {
  // (b - a) x (c - a)
  return __fsub_rn(__fmul_rn(__fsub_rn(bx, ax), __fsub_rn(cy, ay)), __fmul_rn(__fsub_rn(by, ay), __fsub_rn(cx, ax)));
}

// Barycentrics, perspective-corrected barycentrics and zbuf of record r at pixel offset (qx, qy) from its origin.
// Returns false when the pixel is not covered.  The one definition the winner search and the output pass share.
__device__ __forceinline__ bool shade(const FaceRec& r, float qx, float qy, float bp[3], float& zb) {
  float b[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) b[i] = __fadd_rn(__fadd_rn(__fmul_rn(r.ka[i], qx), __fmul_rn(r.kb[i], qy)), r.kc[i]);
  if (!(b[0] >= 0.f && b[1] >= 0.f && b[2] >= 0.f)) return false;
  const float w0 = __fmul_rn(b[0], r.iz[0]), w1 = __fmul_rn(b[1], r.iz[1]), w2 = __fmul_rn(b[2], r.iz[2]);
  const float s = __fadd_rn(__fadd_rn(w0, w1), w2);
  if (!(s > 0.f)) return false;
  bp[0] = __fdiv_rn(w0, s); bp[1] = __fdiv_rn(w1, s); bp[2] = __fdiv_rn(w2, s);
  zb = __fadd_rn(__fadd_rn(__fmul_rn(bp[0], r.z[0]), __fmul_rn(bp[1], r.z[1])), __fmul_rn(bp[2], r.z[2]));
  return true;
}

__device__ __forceinline__ int block_sum(int v, int* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if (lane == 0) red[wid] = v;
  __syncthreads();
  int t = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
  return t;   // valid in thread 0
}

__global__ void __launch_bounds__(kSetupThreads) raster_setup_kernel(
    const float* __restrict__ verts, int V, const long long* __restrict__ faces, int F, int N,
    const float* __restrict__ cameras, int H, int W, float z_clip, float area_eps, int tiles_x, int tiles_per_frame,
    FaceRec* __restrict__ recs, int* __restrict__ tile_counts, int* __restrict__ counters) {
  __shared__ int red[kSetupThreads / 32];
  const long long gid = blockIdx.x * (long long)kSetupThreads + threadIdx.x;
  int skipped = 0;
  if (gid < (long long)N * F) {
    const int n = (int)(gid / F), f = (int)(gid % F);
    float cam[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) cam[i] = __ldg(cameras + 16 * n + i);
    ScreenTri t;
    bool bad;
    project_face(verts, faces, cam, V, f, n, t, bad);
    FaceRec r{};
    r.x1 = -1; r.y1 = -1;
    bool keep = !bad && t.z[0] > z_clip && t.z[1] > z_clip && t.z[2] > z_clip;   // NaN Z fails too
    const float A = keep ? edge_fn(t.sx[0], t.sy[0], t.sx[1], t.sy[1], t.sx[2], t.sy[2]) : 0.f;
    if (keep && !(fabsf(A) > area_eps)) keep = false;                              // degenerate (or NaN) area
    skipped = keep ? 0 : 1;
    if (keep) {
      const float xmin = fminf(fminf(t.sx[0], t.sx[1]), t.sx[2]), xmax = fmaxf(fmaxf(t.sx[0], t.sx[1]), t.sx[2]);
      const float ymin = fminf(fminf(t.sy[0], t.sy[1]), t.sy[2]), ymax = fmaxf(fmaxf(t.sy[0], t.sy[1]), t.sy[2]);
      // pixel centres inside the bbox and the image (culls faces that are off-screen or fall between centres)
      const int x0 = (int)ceilf(fmaxf(xmin, 0.f)), x1 = (int)floorf(fminf(xmax, (float)(W - 1)));
      const int y0 = (int)ceilf(fmaxf(ymin, 0.f)), y1 = (int)floorf(fminf(ymax, (float)(H - 1)));
      if (xmax >= 0.f && ymax >= 0.f && xmin <= (float)(W - 1) && ymin <= (float)(H - 1) && x0 <= x1 && y0 <= y1) {
        r.x0 = x0; r.x1 = x1; r.y0 = y0; r.y1 = y1;
        const float ox = (float)x0, oy = (float)y0;
        float ex[3], ey[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) { ex[k] = __fsub_rn(t.sx[k], ox); ey[k] = __fsub_rn(t.sy[k], oy); }
        const float Ar = edge_fn(ex[0], ey[0], ex[1], ey[1], ex[2], ey[2]);   // same area, origin-relative rounding
        const float inv = __fdiv_rn(1.f, Ar);
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          // b_i(q) = E(v_{i+1}, v_{i+2}, q) / A = (-(dy) qx + (dx) qy + (dy ax - dx ay)) / A
          const int a = (i + 1) % 3, b = (i + 2) % 3;
          const float dx = __fsub_rn(ex[b], ex[a]), dy = __fsub_rn(ey[b], ey[a]);
          r.ka[i] = __fmul_rn(-dy, inv);
          r.kb[i] = __fmul_rn(dx, inv);
          r.kc[i] = __fmul_rn(__fsub_rn(__fmul_rn(dy, ex[a]), __fmul_rn(dx, ey[a])), inv);
          r.z[i] = t.z[i];
          r.iz[i] = __fdiv_rn(1.f, t.z[i]);
        }
        const int tx0 = x0 / kTileW, tx1 = x1 / kTileW, ty0 = y0 / kTileH, ty1 = y1 / kTileH;
        int* tc = tile_counts + (long long)n * tiles_per_frame;
        for (int ty = ty0; ty <= ty1; ++ty)
          for (int tx = tx0; tx <= tx1; ++tx) atomicAdd(tc + ty * tiles_x + tx, 1);
      }
    }
    float4* dst = reinterpret_cast<float4*>(recs + gid);
    const float4* src = reinterpret_cast<const float4*>(&r);
#pragma unroll
    for (int q = 0; q < 6; ++q) dst[q] = src[q];
  }
  const int tot = block_sum(skipped, red);
  if (threadIdx.x == 0 && tot) atomicAdd(counters + 1, tot);
}

__global__ void __launch_bounds__(kSetupThreads) raster_emit_kernel(const FaceRec* __restrict__ recs, long long NF, int F,
                                                                    int tiles_x, int tiles_per_frame,
                                                                    long long* __restrict__ cursor, long long capacity,
                                                                    int* __restrict__ list) {
  const long long gid = blockIdx.x * (long long)kSetupThreads + threadIdx.x;
  if (gid >= NF) return;
  const int4 bb = reinterpret_cast<const int4*>(recs + gid)[0];   // x0, x1, y0, y1
  if (bb.y < bb.x) return;
  const int n = (int)(gid / F);
  long long* cur = cursor + (long long)n * tiles_per_frame;
  for (int ty = bb.z / kTileH; ty <= bb.w / kTileH; ++ty)
    for (int tx = bb.x / kTileW; tx <= bb.y / kTileW; ++tx) {
      const long long pos = (long long)atomicAdd((unsigned long long*)(cur + ty * tiles_x + tx), 1ull);
      if (pos < capacity) list[pos] = (int)gid;
    }
}

constexpr int kChunk = kTileThreads;   // records per shared-memory chunk: one per thread

__global__ void __launch_bounds__(kTileThreads) raster_tile_kernel(
    const FaceRec* __restrict__ recs, const int* __restrict__ list, const long long* __restrict__ offsets, int H, int W,
    int tiles_x, int tiles_per_frame, const float* __restrict__ verts, int V, const long long* __restrict__ faces,
    const float* __restrict__ cameras, int F, long long* __restrict__ out_p2f, float* __restrict__ out_zbuf,
    float* __restrict__ out_bary, float* __restrict__ out_dists, int* __restrict__ counters) {
  __shared__ FaceRec srec[kChunk];
  __shared__ int sidx[kChunk];
  if (counters[3]) return;   // the pair list overflowed: the caller re-runs with a larger one
  const int n = blockIdx.y, tile = blockIdx.x;
  const int tx = tile % tiles_x, ty = tile / tiles_x;
  const int col = tx * kTileW + (threadIdx.x % kTileW), row = ty * kTileH + (threadIdx.x / kTileW);
  const bool inside = col < W && row < H;
  const long long t = (long long)n * tiles_per_frame + tile;
  const long long beg = offsets[t], end = offsets[t + 1];
  float best_z = INFINITY;
  int best_f = 0x7fffffff;
  for (long long c0 = beg; c0 < end; c0 += kChunk) {
    const int cnt = (int)min((long long)kChunk, end - c0);
    __syncthreads();
    if ((int)threadIdx.x < cnt) {
      const int g = list[c0 + threadIdx.x];
      sidx[threadIdx.x] = g;
      const float4* src = reinterpret_cast<const float4*>(recs + g);
      float4* dst = reinterpret_cast<float4*>(srec + threadIdx.x);
#pragma unroll
      for (int q = 0; q < 6; ++q) dst[q] = __ldg(src + q);
    }
    __syncthreads();
    // The warp owns one tile row: a ballot over 32 records at a time keeps those whose rows include it, and only
    // they are tested pixel by pixel (a small face spans one or two of the tile's eight rows).
    for (int k0 = 0; k0 < cnt; k0 += 32) {
      const int kl = k0 + (int)(threadIdx.x & 31);
      unsigned m = __ballot_sync(0xffffffffu, kl < cnt && srec[kl].y0 <= row && row <= srec[kl].y1);
      while (m) {
        const int k = k0 + __ffs(m) - 1;
        m &= m - 1;
        const FaceRec& r = srec[k];
        if (!inside || col < r.x0 || col > r.x1) continue;
        float bp[3], zb;
        if (!shade(r, (float)(col - r.x0), (float)(row - r.y0), bp, zb)) continue;
        const int g = sidx[k];
        if (zb < best_z || (zb == best_z && g < best_f)) { best_z = zb; best_f = g; }
      }
    }
  }
  const bool hit = inside && best_f != 0x7fffffff;
  const int covered = __syncthreads_count(hit);
  if (threadIdx.x == 0 && covered) atomicAdd(counters, covered);
  if (!inside) return;
  const long long pix = ((long long)n * H + row) * W + col;
  if (!hit) {
    out_p2f[pix] = -1;
    out_zbuf[pix] = -1.f;
    out_bary[3 * pix] = -1.f; out_bary[3 * pix + 1] = -1.f; out_bary[3 * pix + 2] = -1.f;
    if (out_dists) out_dists[pix] = -1.f;
    return;
  }
  FaceRec r;
  {
    const float4* src = reinterpret_cast<const float4*>(recs + best_f);
    float4* dst = reinterpret_cast<float4*>(&r);
#pragma unroll
    for (int q = 0; q < 6; ++q) dst[q] = __ldg(src + q);
  }
  float bp[3], zb;
  shade(r, (float)(col - r.x0), (float)(row - r.y0), bp, zb);
  out_p2f[pix] = best_f;
  out_zbuf[pix] = zb;
  out_bary[3 * pix] = bp[0]; out_bary[3 * pix + 1] = bp[1]; out_bary[3 * pix + 2] = bp[2];
  if (out_dists) {
    // signed squared distance to the nearest edge (segment) in the reference camera's NDC, negative inside
    float cam[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) cam[i] = __ldg(cameras + 16 * n + i);
    ScreenTri st;
    bool bad;
    project_face(verts, faces, cam, V, best_f - n * F, n, st, bad);
    float nx[3], ny[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      nx[k] = 1.f - (2.f * st.sx[k] + 1.f) / (float)W;
      ny[k] = 1.f - (2.f * st.sy[k] + 1.f) / (float)H;
    }
    const float qx = 1.f - (2.f * (float)col + 1.f) / (float)W, qy = 1.f - (2.f * (float)row + 1.f) / (float)H;
    float dmin = INFINITY;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float ax = nx[k], ay = ny[k], bx = nx[(k + 1) % 3], by = ny[(k + 1) % 3];
      const float ux = bx - ax, uy = by - ay, wx = qx - ax, wy = qy - ay;
      const float l2 = ux * ux + uy * uy;
      const float s = l2 > 0.f ? fminf(fmaxf((wx * ux + wy * uy) / l2, 0.f), 1.f) : 0.f;
      const float dx = wx - s * ux, dy = wy - s * uy;
      dmin = fminf(dmin, dx * dx + dy * dy);
    }
    out_dists[pix] = -dmin;
  }
}

struct RasterWs {
  FaceRec* recs;
  int* tile_counts;
  long long* offsets;   // ntiles + 1
  long long* cursor;
  int* list;
};

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

RasterWs carve(void* ws, long long NF, long long ntiles) {
  RasterWs w;
  char* p = (char*)ws;
  w.recs = (FaceRec*)p; p += align256((size_t)NF * sizeof(FaceRec));
  w.tile_counts = (int*)p; p += align256((size_t)ntiles * 4);
  w.offsets = (long long*)p; p += align256((size_t)(ntiles + 1) * 8);
  w.cursor = (long long*)p; p += align256((size_t)ntiles * 8);
  w.list = (int*)p;
  return w;
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_raster_workspace_bytes(int N, int64_t F, int H, int W, int64_t capacity, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  if (N < 0 || F < 0 || H <= 0 || W <= 0 || capacity < 0) return RECMV_E_SHAPE;
  if ((int64_t)N * F > 0x7fffffffLL || capacity > 0x7fffffffLL || (int64_t)N * H * W > 2000000000LL) return RECMV_E_RANGE;
  const int64_t tiles = (int64_t)N * ((W + kTileW - 1) / kTileW) * ((H + kTileH - 1) / kTileH);
  *bytes = align256((size_t)N * F * sizeof(FaceRec)) + align256((size_t)tiles * 4) + align256((size_t)(tiles + 1) * 8) +
           align256((size_t)tiles * 8) + align256((size_t)capacity * 4);
  return RECMV_OK;
}

extern "C" int recmv_rasterize_meshes(const float* verts, int V, const int64_t* faces, int64_t F, int N,
                                      const float* camera, int H, int W, float z_clip, float area_eps, void* workspace,
                                      int64_t capacity, int64_t* out_pix_to_face, float* out_zbuf, float* out_bary,
                                      float* out_dists, int32_t* counters, recmv_stream_t stream) {
  if (V < 0 || F < 0 || N < 0 || H <= 0 || W <= 0 || capacity < 0 || (F > 0 && V == 0)) return RECMV_E_SHAPE;
  if ((int64_t)N * F > 0x7fffffffLL || capacity > 0x7fffffffLL || (int64_t)N * H * W > 2000000000LL) return RECMV_E_RANGE;
  if (N > 65535) return RECMV_E_RANGE;   // frames are the tile pass's grid.y
  if (!counters) return RECMV_E_NULL;
  if (N > 0 && (!camera || !workspace || !out_pix_to_face || !out_zbuf || !out_bary)) return RECMV_E_NULL;
  if (N > 0 && F > 0 && (!faces || !verts)) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(counters, 0, 4 * sizeof(int32_t), st);
  if (e != cudaSuccess) return (int)e;
  if (N == 0) return RECMV_OK;
  const int tiles_x = (W + kTileW - 1) / kTileW, tiles_y = (H + kTileH - 1) / kTileH;
  const int tiles_per_frame = tiles_x * tiles_y;
  const long long ntiles = (long long)N * tiles_per_frame;
  const long long NF = (long long)N * F;
  RasterWs w = carve(workspace, NF, ntiles);
  e = cudaMemsetAsync(w.tile_counts, 0, (size_t)ntiles * 4, st);
  if (e != cudaSuccess) return (int)e;
  const int nb = (int)((NF + kSetupThreads - 1) / kSetupThreads);
  if (NF > 0) {
    raster_setup_kernel<<<nb, kSetupThreads, 0, st>>>(verts, V, (const long long*)faces, (int)F, N, camera, H, W, z_clip,
                                                      area_eps, tiles_x, tiles_per_frame, w.recs, w.tile_counts, counters);
    int s = launch_status();
    if (s) return s;
  }
  raster_scan_kernel<<<1, kScanThreads, 0, st>>>(w.tile_counts, (int)ntiles, w.offsets, w.cursor, capacity, counters);
  int s = launch_status();
  if (s) return s;
  if (NF > 0) {
    raster_emit_kernel<<<nb, kSetupThreads, 0, st>>>(w.recs, NF, (int)F, tiles_x, tiles_per_frame, w.cursor, capacity,
                                                     w.list);
    s = launch_status();
    if (s) return s;
  }
  raster_tile_kernel<<<dim3(tiles_per_frame, N), kTileThreads, 0, st>>>(
      w.recs, w.list, w.offsets, H, W, tiles_x, tiles_per_frame, verts, V, (const long long*)faces, camera, (int)F,
      (long long*)out_pix_to_face, out_zbuf, out_bary, out_dists, counters);
  return launch_status();
}

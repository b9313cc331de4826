// The mesh rasterizer's per-face setup and per-pixel test, shared by the tile pass (raster.cu) and the sparse depth
// probe (zbuf_probe.cu) so that both decide coverage and depth with the same instructions (DESIGN section 1b, 1i).
#pragma once
#include <math.h>

namespace recmv {
namespace {

constexpr int kTileW = 32, kTileH = 8;          // one warp per tile row: 128-byte rows of every 4-byte output

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

// The record of face f in frame n (camera row cam[16]).  Returns false when the face is skipped (an index outside
// [0, V), a vertex at Z <= z_clip, or |A| <= area_eps); r.x1 < r.x0 whenever the face covers no pixel centre of the
// image, skipped or not.
__device__ __forceinline__ bool make_face_rec(const float* __restrict__ verts, const long long* __restrict__ faces,
                                              const float* cam, int V, int f, int n, int H, int W, float z_clip,
                                              float area_eps, FaceRec& r) {
  ScreenTri t;
  bool bad;
  project_face(verts, faces, cam, V, f, n, t, bad);
  r = FaceRec{};
  r.x1 = -1; r.y1 = -1;
  bool keep = !bad && t.z[0] > z_clip && t.z[1] > z_clip && t.z[2] > z_clip;   // NaN Z fails too
  const float A = keep ? edge_fn(t.sx[0], t.sy[0], t.sx[1], t.sy[1], t.sx[2], t.sy[2]) : 0.f;
  if (keep && !(fabsf(A) > area_eps)) keep = false;                              // degenerate (or NaN) area
  if (!keep) return false;
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
  }
  return true;
}

}  // namespace
}  // namespace recmv

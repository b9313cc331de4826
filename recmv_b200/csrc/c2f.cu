// Coarse-to-fine sweep helpers (Seg3dLossless, MCAcc/seg3d_lossless.py:233-428).
//  * recmv_interp2x_boundary3d_{fwd,bwd}: the 2x-1 upsampling + "mixed occupancy" flag of the reference's optional
//    extension (MCAcc/cuda/interp2x_boundary3d_kernel.cu:9-242; off by default there, use_cuda_impl=False) -- and,
//    selectable by `order`, the same operation with the rounding of the default path
//    (F.interpolate(trilinear, align_corners=True) on the values and on the 0/1 flags, seg3d_lossless.py:270-281),
//    so the default sweep can use one fused pass and stay bit-identical.
//  * recmv_c2f_todo_mask: 3x3x3 dilation of the flags (smooth_conv3x3 > 0) AND NOT already-evaluated.
// HBM-bound: 4 B read per coarse voxel (L2-resident re-reads), 5 B written per fine voxel.
#include "../../include/recmv_b200.h"
#include "common.cuh"

namespace recmv {
namespace {

// order 0: sequential sum / count as the reference kernel; order 1: ATen's nested x, y, z interpolation with
// lambda in {0, 1/2} (every product by 1/2 is exact, one rounding per addition)
// value and "mixed occupancy" flag of fine voxel (x, y, z) of the 2x-1 upsampling of p [D][H][W]
template <int kOrder>
__device__ __forceinline__ float interp2x_value(const float* __restrict__ p, int D, int H, int W, int x, int y, int z,
                                                float balance, bool* mixed) {
  const int x0 = x >> 1, y0 = y >> 1, z0 = z >> 1;             // (x-1)/2 for odd x, x/2 for even x
  const int ox = x & 1, oy = y & 1, oz = z & 1;                 // odd: second neighbour at +1
  float v[8];
  bool any_in = false, any_out = false;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int dz = (k >> 2) & oz, dy = ((k >> 1) & 1) & oy, dx = (k & 1) & ox;
    v[k] = __ldg(p + ((long long)(z0 + dz) * H + (y0 + dy)) * W + (x0 + dx));
    const bool f = v[k] > balance;
    any_in |= f; any_out |= !f;
  }
  *mixed = any_in && any_out;
  float r;
  if (kOrder == 0) {
    // the reference's summation orders (interp2x_boundary3d_kernel.cu:38-129): left to right over
    //   1 axis odd : the two neighbours;   x,y odd : (y-,x-)(y-,x+)(y+,x-)(y+,x+);
    //   y,z odd    : (z-,y-)(z+,y-)(z-,y+)(z+,y+);   x,z odd : (z-,x-)(z+,x-)(z-,x+)(z+,x+);   all odd : x, y, z nested
    const int n = (1 << ox) << (oy + oz);
    float s;
    if (n == 1) s = v[0];
    else if (n == 2) s = v[0] + (ox ? v[1] : (oy ? v[2] : v[4]));
    else if (n == 8) s = ((((((v[0] + v[1]) + v[2]) + v[3]) + v[4]) + v[5]) + v[6]) + v[7];
    else if (!oz) s = ((v[0] + v[1]) + v[2]) + v[3];
    else if (!ox) s = ((v[0] + v[4]) + v[2]) + v[6];
    else s = ((v[0] + v[4]) + v[1]) + v[5];
    r = n == 1 ? s : (float)((double)s / (double)n);
  } else {
    const float a00 = ox ? 0.5f * v[0] + 0.5f * v[1] : v[0], a01 = ox ? 0.5f * v[2] + 0.5f * v[3] : v[2];
    const float a10 = ox ? 0.5f * v[4] + 0.5f * v[5] : v[4], a11 = ox ? 0.5f * v[6] + 0.5f * v[7] : v[6];
    const float b0 = oy ? 0.5f * a00 + 0.5f * a01 : a00, b1 = oy ? 0.5f * a10 + 0.5f * a11 : a10;
    r = oz ? 0.5f * b0 + 0.5f * b1 : b0;
  }
  return r;
}

template <int kOrder>
__global__ void __launch_bounds__(256) interp2x_fwd_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                           unsigned char* __restrict__ flag, int NC, int D, int H,
                                                           int W, float balance) {
  const int d = 2 * D - 1, h = 2 * H - 1, w = 2 * W - 1;
  const long long total = (long long)NC * d * h * w;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % w), y = (int)((i / w) % h), z = (int)((i / ((long long)w * h)) % d);
    const long long nc = i / ((long long)w * h * d);
    bool mixed;
    out[i] = interp2x_value<kOrder>(in + nc * ((long long)D * H * W), D, H, W, x, y, z, balance, &mixed);
    flag[i] = mixed ? 1 : 0;
  }
}

// gradient of the (order 0 == order 1 up to rounding) linear map: gather of the 27 fine neighbours of 2*(z,y,x)
__global__ void __launch_bounds__(256) interp2x_bwd_kernel(const float* __restrict__ go, float* __restrict__ gi,
                                                           int NC, int D, int H, int W) {
  const int d = 2 * D - 1, h = 2 * H - 1, w = 2 * W - 1;
  const long long total = (long long)NC * D * H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % W), y = (int)((i / W) % H), z = (int)((i / ((long long)W * H)) % D);
    const long long nc = i / ((long long)W * H * D);
    const float* g = go + nc * ((long long)d * h * w);
    // same accumulation order as the reference: centre, 6 axis neighbours (x-, x+, y-, y+, z-, z+) / 2, 12 face
    // diagonals (xy, xz, yz) / 4, 8 corners / 8
    auto at = [&](int dz, int dy, int dx) { return __ldg(g + ((long long)(2 * z + dz) * h + (2 * y + dy)) * w + (2 * x + dx)); };
    const bool xm = x > 0, xp = x < W - 1, ym = y > 0, yp = y < H - 1, zm = z > 0, zp = z < D - 1;
    float a = at(0, 0, 0);
    if (xm) a += at(0, 0, -1) / 2.f;
    if (xp) a += at(0, 0, 1) / 2.f;
    if (ym) a += at(0, -1, 0) / 2.f;
    if (yp) a += at(0, 1, 0) / 2.f;
    if (zm) a += at(-1, 0, 0) / 2.f;
    if (zp) a += at(1, 0, 0) / 2.f;
    if (xm && ym) a += at(0, -1, -1) / 4.f;
    if (xp && ym) a += at(0, -1, 1) / 4.f;
    if (xm && yp) a += at(0, 1, -1) / 4.f;
    if (xp && yp) a += at(0, 1, 1) / 4.f;
    if (xm && zm) a += at(-1, 0, -1) / 4.f;
    if (xp && zm) a += at(-1, 0, 1) / 4.f;
    if (xm && zp) a += at(1, 0, -1) / 4.f;
    if (xp && zp) a += at(1, 0, 1) / 4.f;
    if (ym && zm) a += at(-1, -1, 0) / 4.f;
    if (yp && zm) a += at(-1, 1, 0) / 4.f;
    if (ym && zp) a += at(1, -1, 0) / 4.f;
    if (yp && zp) a += at(1, 1, 0) / 4.f;
    if (xm && ym && zm) a += at(-1, -1, -1) / 8.f;
    if (xp && ym && zm) a += at(-1, -1, 1) / 8.f;
    if (xm && yp && zm) a += at(-1, 1, -1) / 8.f;
    if (xp && yp && zm) a += at(-1, 1, 1) / 8.f;
    if (xm && ym && zp) a += at(1, -1, -1) / 8.f;
    if (xp && ym && zp) a += at(1, -1, 1) / 8.f;
    if (xm && yp && zp) a += at(1, 1, -1) / 8.f;
    if (xp && yp && zp) a += at(1, 1, 1) / 8.f;
    gi[i] = a;
  }
}

// todo = dilate3x3x3(flag) & ~done   (zero padding at the volume border)
__global__ void __launch_bounds__(256) c2f_todo_kernel(const unsigned char* __restrict__ flag,
                                                       const unsigned char* __restrict__ done,
                                                       unsigned char* __restrict__ todo, int D, int H, int W) {
  const long long total = (long long)D * H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    unsigned char r = 0;
    if (!done[i]) {
      const int x = (int)(i % W), y = (int)((i / W) % H), z = (int)(i / ((long long)W * H));
      for (int dz = -1; dz <= 1 && !r; ++dz) {
        const int zz = z + dz;
        if (zz < 0 || zz >= D) continue;
        for (int dy = -1; dy <= 1 && !r; ++dy) {
          const int yy = y + dy;
          if (yy < 0 || yy >= H) continue;
          const unsigned char* row = flag + ((long long)zz * H + yy) * W;
          r = (x > 0 && row[x - 1]) || row[x] || (x < W - 1 && row[x + 1]);
        }
      }
    }
    todo[i] = r;
  }
}

// ---- device worklist of the sweep (Seg3dLossless._forward, MCAcc/seg3d_lossless.py:306-428) ---------------------------
// Voxels to query -> (flat level index, query point) list; the order is irrelevant: the fused SDF kernel evaluates every
// point independently and results are scattered back by index.
struct C2fGeom {
  int D, H, W;          // level lattice
  int sx, sy, sz;       // level step in final-lattice units
  int Wf, Hf, Df;       // final lattice
  float inv_step2[3];   // (1 / res) / 2 per axis (x, y, z)
  float res[3];         // final resolution as float (x, y, z)
  float ext[3], bmin[3];
};

// Query point of level voxel (x, y, z) -> pts[0..3), exactly as batch_eval (:89-100): c = coords / res + (1 / res) / 2;
// p = c * (b_max - b_min) + b_min, every operation rounded separately (no FMA contraction), so the values equal the torch
// path's bit for bit.
__device__ __forceinline__ void c2f_query_point(const C2fGeom& g, int x, int y, int z, float* __restrict__ pts) {
  const float c[3] = {(float)(x * g.sx), (float)(y * g.sy), (float)(z * g.sz)};
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float u = __fadd_rn(__fdiv_rn(c[a], g.res[a]), g.inv_step2[a]);
    pts[a] = __fadd_rn(__fmul_rn(u, g.ext[a]), g.bmin[a]);
  }
}

// ---- one fused pass per level --------------------------------------------------------------------------------------
// mixed[cell] = the 8 corners of coarse cell (cz, cy, cx) straddle the balance value.  The 3x3x3 dilation of the fine
// "mixed stencil" flags (seg3d_lossless.py:283-288) collapses onto this coarse mask EXACTLY: along an axis a fine voxel
// with even coordinate 2a sees the stencils of cells a-1 and a, one with odd coordinate 2a+1 only cell a; every neighbour's
// stencil lies inside one of those cells, and each of those cells' centre voxels IS a neighbour.
__global__ void __launch_bounds__(256) c2f_cell_mixed_kernel(const float* __restrict__ occ, int D, int H, int W, float balance,
                                                             unsigned char* __restrict__ mixed) {
  const int cd = D - 1, chh = H - 1, cw = W - 1;
  const long long total = (long long)cd * chh * cw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % cw), y = (int)((i / cw) % chh), z = (int)(i / ((long long)cw * chh));
    bool any_in = false, any_out = false;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const bool f = __ldg(occ + ((long long)(z + (k >> 2)) * H + (y + ((k >> 1) & 1))) * W + (x + (k & 1))) > balance;
      any_in |= f; any_out |= !f;
    }
    mixed[i] = (any_in && any_out) ? 1 : 0;
  }
}

// upsample + done lattice + todo decision + worklist append (one warp-aggregated atomic per warp), one pass over the
// fine level
template <int kOrder>
__global__ void __launch_bounds__(256) c2f_refine_kernel(const float* __restrict__ occ_c, const unsigned char* __restrict__ done_c,
                                                         const unsigned char* __restrict__ mixed, int D, int H, int W /*coarse*/,
                                                         C2fGeom g /*fine level*/, float balance, float* __restrict__ occ_f,
                                                         unsigned char* __restrict__ done_f, int* __restrict__ idx_out,
                                                         float* __restrict__ pts_out, int* __restrict__ counters, int cap) {
  const long long total = (long long)g.D * g.H * g.W;
  const int lane = threadIdx.x & 31;
  const int cd = D - 1, chh = H - 1, cw = W - 1;
  for (long long i0 = (blockIdx.x * (long long)blockDim.x + threadIdx.x) - lane; i0 < total; i0 += (long long)gridDim.x * blockDim.x) {
    const long long i = i0 + lane;
    bool on = false;
    int x = 0, y = 0, z = 0;
    if (i < total) {
      x = (int)(i % g.W); y = (int)((i / g.W) % g.H); z = (int)(i / ((long long)g.W * g.H));
      bool m_;
      occ_f[i] = interp2x_value<kOrder>(occ_c, D, H, W, x, y, z, balance, &m_);
      const bool coincident = ((x | y | z) & 1) == 0;
      const unsigned char dn = coincident ? done_c[((long long)(z >> 1) * H + (y >> 1)) * W + (x >> 1)] : 0;
      done_f[i] = dn;
      if (!dn) {
        const int xa = x >> 1, ya = y >> 1, za = z >> 1;
        const int x_lo = (x & 1) ? xa : xa - 1, y_lo = (y & 1) ? ya : ya - 1, z_lo = (z & 1) ? za : za - 1;
        for (int cz = max(z_lo, 0); cz <= min(za, cd - 1) && !on; ++cz)
          for (int cy = max(y_lo, 0); cy <= min(ya, chh - 1) && !on; ++cy)
            for (int cx = max(x_lo, 0); cx <= min(xa, cw - 1) && !on; ++cx)
              on = mixed[((long long)cz * chh + cy) * cw + cx] != 0;
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, on);
    if (m == 0u) continue;
    int base = 0;
    if (lane == 0) base = atomicAdd(counters, __popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (!on) continue;
    const int slot = base + __popc(m & ((1u << lane) - 1u));
    if (slot >= cap) { counters[1] = 1; continue; }
    idx_out[slot] = (int)i;
    c2f_query_point(g, x, y, z, pts_out + 3 * (size_t)slot);
  }
}

// conflict round: every conflicting voxel (list from the scatter pass) claims its not-yet-evaluated 3x3x3 neighbours for the
// next worklist; a voxel is claimed once (atomicOr on the byte's word in `claim`, an all-zero mask between rounds: the
// scatter pass of the next round clears the bytes it consumed)
__global__ void __launch_bounds__(256) c2f_mark_kernel(const int* __restrict__ clist, const int* __restrict__ ccount, int ccap,
                                                       const unsigned char* __restrict__ calculated, C2fGeom g,
                                                       unsigned int* __restrict__ claim, int* __restrict__ idx_out,
                                                       float* __restrict__ pts_out, int* __restrict__ counters, int cap) {
  const int n = min(*ccount, ccap);
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < 27 * n; t += gridDim.x * blockDim.x) {
    const int j = clist[t / 27], k = t % 27;
    const int x = j % g.W + (k % 3) - 1, y = (j / g.W) % g.H + ((k / 3) % 3) - 1, z = j / (g.W * g.H) + (k / 9) - 1;
    if (x < 0 || y < 0 || z < 0 || x >= g.W || y >= g.H || z >= g.D) continue;
    if (calculated[((size_t)(z * g.sz) * g.Hf + (size_t)(y * g.sy)) * g.Wf + (size_t)(x * g.sx)]) continue;
    const long long i = ((long long)z * g.H + y) * g.W + x;
    const unsigned bit = 1u << (8 * (int)(i & 3));
    if (atomicOr(claim + (i >> 2), bit) & bit) continue;          // somebody else claimed it
    const int slot = atomicAdd(counters, 1);
    if (slot >= cap) { counters[1] = 1; continue; }
    idx_out[slot] = (int)i;
    c2f_query_point(g, x, y, z, pts_out + 3 * (size_t)slot);
  }
}

// scatter of a worklist's results, list form: conflicts are appended to clist (ccount zeroed by the caller), claim bytes of
// the consumed entries are cleared
__global__ void __launch_bounds__(256) c2f_scatter_list_kernel(const int* __restrict__ idx, const float* __restrict__ vals,
                                                               const int* __restrict__ counters, int cap, C2fGeom g,
                                                               float* __restrict__ occ, unsigned char* __restrict__ done,
                                                               unsigned char* __restrict__ calculated,
                                                               unsigned char* __restrict__ claim, float balance,
                                                               int* __restrict__ clist, int* __restrict__ ccount,
                                                               int* __restrict__ stats /*[0]+=queried [1]=conflicts*/) {
  const int n = min(counters[0], cap);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int j = idx[i];
    const float v = vals[i], it = occ[j];
    occ[j] = v;
    done[j] = 1;
    claim[j] = 0;
    const int x = j % g.W, y = (j / g.W) % g.H, z = j / (g.W * g.H);
    calculated[((size_t)(z * g.sz) * g.Hf + (size_t)(y * g.sy)) * g.Wf + (size_t)(x * g.sx)] = 1;
    if (__fmul_rn(__fsub_rn(it, balance), __fsub_rn(v, balance)) < 0.f) {
      const int slot = atomicAdd(ccount, 1);
      if (slot < cap) clist[slot] = j;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(stats, n);
}

C2fGeom make_geom(const int level[3], const int final_res[3], const float b_min[3], const float b_max[3]) {
  C2fGeom g;
  g.W = level[0]; g.H = level[1]; g.D = level[2];
  g.Wf = final_res[0]; g.Hf = final_res[1]; g.Df = final_res[2];
  g.sx = level[0] > 1 ? (final_res[0] - 1) / (level[0] - 1) : 1;
  g.sy = level[1] > 1 ? (final_res[1] - 1) / (level[1] - 1) : 1;
  g.sz = level[2] > 1 ? (final_res[2] - 1) / (level[2] - 1) : 1;
  for (int a = 0; a < 3; ++a) {
    g.res[a] = (float)final_res[a];
    g.inv_step2[a] = (1.0f / (float)final_res[a]) / 2.f;   // torch: step = 1.0 / res.float(); step / 2
    g.ext[a] = b_max[a] - b_min[a];
    g.bmin[a] = b_min[a];
  }
  return g;
}
}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_interp2x_boundary3d_fwd(const float* input, float* output, uint8_t* is_boundary, int NC, int D,
                                             int H, int W, float balance_value, int order, recmv_stream_t stream) {
  if (NC < 0 || D <= 0 || H <= 0 || W <= 0) return RECMV_E_SHAPE;
  if (order != 0 && order != 1) return RECMV_E_RANGE;
  if (NC == 0) return RECMV_OK;
  if (!input || !output || !is_boundary) return RECMV_E_NULL;
  const int64_t total = (int64_t)NC * (2 * D - 1) * (2 * H - 1) * (2 * W - 1);
  const int g = stride_grid(total, 256, 16);
  if (order == 0) interp2x_fwd_kernel<0><<<g, 256, 0, (cudaStream_t)stream>>>(input, output, is_boundary, NC, D, H, W, balance_value);
  else interp2x_fwd_kernel<1><<<g, 256, 0, (cudaStream_t)stream>>>(input, output, is_boundary, NC, D, H, W, balance_value);
  return launch_status();
}

extern "C" int recmv_interp2x_boundary3d_bwd(const float* grad_output, float* grad_input, int NC, int D, int H, int W,
                                             recmv_stream_t stream) {
  if (NC < 0 || D <= 0 || H <= 0 || W <= 0) return RECMV_E_SHAPE;
  if (NC == 0) return RECMV_OK;
  if (!grad_output || !grad_input) return RECMV_E_NULL;
  interp2x_bwd_kernel<<<stride_grid((int64_t)NC * D * H * W, 256, 16), 256, 0, (cudaStream_t)stream>>>(grad_output, grad_input, NC, D, H, W);
  return launch_status();
}

extern "C" int recmv_c2f_todo_mask(const uint8_t* is_boundary, const uint8_t* done, uint8_t* todo, int D, int H, int W,
                                   recmv_stream_t stream) {
  if (D <= 0 || H <= 0 || W <= 0) return RECMV_E_SHAPE;
  if (!is_boundary || !done || !todo) return RECMV_E_NULL;
  c2f_todo_kernel<<<stride_grid((int64_t)D * H * W, 256, 16), 256, 0, (cudaStream_t)stream>>>(is_boundary, done, todo, D, H, W);
  return launch_status();
}

// ---- the fused level pass + list-driven conflict rounds (what Seg3dLossless._forward_device uses) ---------------------------
// coarse (D, H, W) -> fine level (2D-1, 2H-1, 2W-1): occ_fine / done_fine are written for every voxel, the voxels to query are
// appended to (idx_out, points_out) [counters zeroed by the caller].  mixed_scratch: (D-1)(H-1)(W-1) bytes.
extern "C" int recmv_c2f_refine(const float* occ_coarse, const uint8_t* done_coarse, int D, int H, int W,
                                const int final_res[3], const float b_min[3], const float b_max[3], float balance_value,
                                int order, uint8_t* mixed_scratch, float* occ_fine, uint8_t* done_fine, int32_t* idx_out,
                                float* points_out, int32_t* counters, int capacity, recmv_stream_t stream) {
  if (!occ_coarse || !done_coarse || !final_res || !b_min || !b_max || !mixed_scratch || !occ_fine || !done_fine || !idx_out ||
      !points_out || !counters)
    return RECMV_E_NULL;
  if (D < 2 || H < 2 || W < 2 || capacity <= 0) return RECMV_E_SHAPE;
  if (order != 0 && order != 1) return RECMV_E_RANGE;
  const int level[3] = {2 * W - 1, 2 * H - 1, 2 * D - 1};
  const C2fGeom g = make_geom(level, final_res, b_min, b_max);
  cudaStream_t st = (cudaStream_t)stream;
  c2f_cell_mixed_kernel<<<stride_grid((int64_t)(D - 1) * (H - 1) * (W - 1), 256, 8), 256, 0, st>>>(occ_coarse, D, H, W, balance_value,
                                                                                             mixed_scratch);
  int s = launch_status();
  if (s) return s;
  const int grid = stride_grid((int64_t)g.D * g.H * g.W, 256, 8);
  if (order == 0)
    c2f_refine_kernel<0><<<grid, 256, 0, st>>>(occ_coarse, done_coarse, mixed_scratch, D, H, W, g, balance_value, occ_fine, done_fine,
                                               idx_out, points_out, counters, capacity);
  else
    c2f_refine_kernel<1><<<grid, 256, 0, st>>>(occ_coarse, done_coarse, mixed_scratch, D, H, W, g, balance_value, occ_fine, done_fine,
                                               idx_out, points_out, counters, capacity);
  return launch_status();
}

// scatter of one worklist's values; conflicts -> conflict_list / conflict_count (device int32, zeroed by the caller);
// claim (level-lattice bytes, zero between rounds) entries of the consumed voxels are cleared.  stats[0] += queried.
extern "C" int recmv_c2f_scatter_list(const int32_t* idx, const float* vals, const int32_t* counters, int capacity,
                                      const int level[3], const int final_res[3], float* occ, uint8_t* done,
                                      uint8_t* calculated, uint8_t* claim, float balance_value, int32_t* conflict_list,
                                      int32_t* conflict_count, int32_t* stats, recmv_stream_t stream) {
  if (!idx || !vals || !counters || !level || !final_res || !occ || !done || !calculated || !claim || !conflict_list ||
      !conflict_count || !stats)
    return RECMV_E_NULL;
  if (capacity <= 0) return RECMV_E_SHAPE;
  const float z3[3] = {0.f, 0.f, 0.f};
  const C2fGeom g = make_geom(level, final_res, z3, z3);
  c2f_scatter_list_kernel<<<stride_grid(capacity, 256, 4), 256, 0, (cudaStream_t)stream>>>(
      idx, vals, counters, capacity, g, occ, done, calculated, claim, balance_value, conflict_list, conflict_count, stats);
  return launch_status();
}

// next worklist = the not-yet-evaluated 3x3x3 neighbours of the conflicting voxels, each once (counters zeroed by the caller)
extern "C" int recmv_c2f_mark_conflicts(const int32_t* conflict_list, const int32_t* conflict_count, int list_capacity,
                                        const uint8_t* calculated, const int level[3], const int final_res[3],
                                        const float b_min[3], const float b_max[3], uint8_t* claim, int32_t* idx_out,
                                        float* points_out, int32_t* counters, int capacity, recmv_stream_t stream) {
  if (!conflict_list || !conflict_count || !calculated || !level || !final_res || !b_min || !b_max || !claim || !idx_out ||
      !points_out || !counters)
    return RECMV_E_NULL;
  if (capacity <= 0 || list_capacity <= 0) return RECMV_E_SHAPE;
  if (((uintptr_t)claim & 3) != 0) return RECMV_E_SHAPE;   // claimed through 32-bit atomics
  const C2fGeom g = make_geom(level, final_res, b_min, b_max);
  c2f_mark_kernel<<<num_sms() * 2, 256, 0, (cudaStream_t)stream>>>(conflict_list, conflict_count, list_capacity, calculated, g,
                                                                  (unsigned int*)claim, idx_out, points_out, counters, capacity);
  return launch_status();
}

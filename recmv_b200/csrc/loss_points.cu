// The loss points of `surface_render_loss` (DESIGN section 1k): engineer/networks/OptimGarmentNetwork.py:1103-1167 for
// G garments in one launch sequence, with counter-based draws in place of the reference's CPU `torch.rand` and
// `torch.randn_like`, and the `check` compaction in place of its boolean indexing.
//
// Garment g has M_g surface-solve points P (with check, batch, row, col and ray per point) and V_g MC vertices; its
// input rows are i < C_g = M_g + V_g, row i < M_g being point i and row M_g + v vertex v.  S = 4096 // G.
//   draws      vertex v is kept in lane L (E eikonal, D regulariser) iff u < thr_g, thr_g = fp32(double(S) / V_g),
//              u = (x0 >> 8) 2^-24;
//   points     B_L = cat(P, kept_L vertices); X_E = cat(B_E + 0.01 z, G) with |B_E| // 6 global rows, each coordinate
//              fp32(fp32(u 3.6f) - 1.8f); X_D = cat(B_D, B_D + 0.01 z); a local point is x + fp32(z 0.01f);
//   normals    z0, z1 = sqrt(-2 ln ua) (cos, sin)(2 pi ub) of (x0, x1), z2 the cosine of (x2, x3), in double,
//              ua = ((x >> 8) + 1) 2^-24, ub = (x >> 8) 2^-24, rounded once to f32;
//   counters   row i of lane l (0 E-draw, 1 D-draw, 2 E-local, 3 E-global, 4 D-local) uses Philox4x32-10 counter
//              offset + 5 (C_0 + ... + C_{g-1}) + l C_g + i;
//   compaction the rows of (P, rays, batch, row, col) whose check is true, in order, and their input indices.
//
//   1. lp_count_kernel  one thread per input row: check flag or the two draws, per-block counts of the three;
//   2. lp_scan_kernel   one CTA per (garment, count): exclusive scan, the total -> counts[3 g + k];
//      (the caller reads the 3G counts and sizes the outputs)
//   3. lp_emit_kernel   one thread per input row: its rows of X_E, X_D and the compaction, and global row i.
// No atomics: the output is bit-identical from run to run.
#include "common.cuh"
#include "compact.cuh"
#include "philox.cuh"
#include "workspace.cuh"

namespace recmv {
namespace {

constexpr int kRowThreads = 256;
constexpr int kMaxLists = 8;       // garments per launch sequence; a call with more runs one sequence per group
constexpr unsigned char kKeepE = 1, kKeepD = 2, kCheck = 4;

struct PointLists {
  const float* pts[kMaxLists];
  const float* verts[kMaxLists];
  const unsigned char* check[kMaxLists];
  const long long* batch[kMaxLists];
  const long long* row[kMaxLists];
  const long long* col[kMaxLists];
  const float* rays[kMaxLists];
  float* out_e[kMaxLists];                    // X_E [|B_E| + |B_E| / 6, 3]
  float* out_d[kMaxLists];                    // X_D [2 |B_D|, 3]
  float* out_pts[kMaxLists];                  // the checked rows, [checked, 3] ...
  float* out_rays[kMaxLists];
  long long* out_batch[kMaxLists];
  long long* out_row[kMaxLists];
  long long* out_col[kMaxLists];
  long long* out_index[kMaxLists];            // ... and their input indices
  long long M[kMaxLists];
  long long V[kMaxLists];
  long long nE[kMaxLists];                    // |B_E|, |B_D| (emit only)
  long long nD[kMaxLists];
  float thr[kMaxLists];
  long long row_base[kMaxLists];              // its first flag in the workspace
  unsigned long long ctr_base[kMaxLists];     // offset + 5 (C_0 + ... + C_{g-1})
  int tile_base[kMaxLists + 1];               // its first block (absolute); tile_base[G] ends the group
  int g0;                                     // index of list 0 in the call
  int G;
};

__device__ __forceinline__ int list_of(const PointLists& L, int t) {
  int g = 0;
  while (g + 1 < L.G && t >= L.tile_base[g + 1]) ++g;
  return g;
}

// rank of this thread's predicate among the block's true predicates, in thread order
__device__ __forceinline__ int block_rank(bool p, int* warp_cnt) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, p);
  if (lane == 0) warp_cnt[wid] = __popc(m);
  __syncthreads();
  int r = __popc(m & ((1u << lane) - 1u));
  for (int w = 0; w < wid; ++w) r += warp_cnt[w];
  return r;
}

__device__ __forceinline__ Philox4 draw(unsigned long long ctr, unsigned long long seed) {
  return philox4x32_10((unsigned)ctr, (unsigned)(ctr >> 32), (unsigned)seed, (unsigned)(seed >> 32));
}

__device__ __forceinline__ float unit24(unsigned x) { return (float)(x >> 8) * 0x1p-24f; }

// three N(0,1) samples of one Philox call, each computed in double and rounded once
__device__ __forceinline__ void normals3(const Philox4& x, float* z) {
  const double two_pi = 6.283185307179586;
  const double ua = (double)((x.x[0] >> 8) + 1u) * 0x1p-24, ub = (double)(x.x[1] >> 8) * 0x1p-24;
  const double uc = (double)((x.x[2] >> 8) + 1u) * 0x1p-24, ud = (double)(x.x[3] >> 8) * 0x1p-24;
  const double r0 = sqrt(-2.0 * log(ua)), r1 = sqrt(-2.0 * log(uc));
  z[0] = __double2float_rn(r0 * cos(two_pi * ub));
  z[1] = __double2float_rn(r0 * sin(two_pi * ub));
  z[2] = __double2float_rn(r1 * cos(two_pi * ud));
}

// out[0..3) = p + fp32(z 0.01f), z from counter ctr
__device__ __forceinline__ void local_point(const float* p, unsigned long long ctr, unsigned long long seed, float* out) {
  float z[3];
  normals3(draw(ctr, seed), z);
#pragma unroll
  for (int a = 0; a < 3; ++a) out[a] = __fadd_rn(p[a], __fmul_rn(z[a], 0.01f));
}

__global__ void __launch_bounds__(kRowThreads) lp_count_kernel(const PointLists L, unsigned long long seed,
                                                               unsigned char* __restrict__ flags,
                                                               int* __restrict__ cnt_e, int* __restrict__ cnt_d,
                                                               int* __restrict__ cnt_c) {
  const int t = L.tile_base[0] + blockIdx.x;
  const int g = list_of(L, t);
  const long long i = (long long)(t - L.tile_base[g]) * kRowThreads + threadIdx.x;
  const long long M = L.M[g], C = M + L.V[g];
  unsigned char f = 0;
  if (i < M) {
    f = L.check[g][i] ? kCheck : 0;
  } else if (i < C) {
    const unsigned long long v = (unsigned long long)(i - M);
    const float thr = L.thr[g];
    if (unit24(draw(L.ctr_base[g] + v, seed).x[0]) < thr) f |= kKeepE;
    if (unit24(draw(L.ctr_base[g] + (unsigned long long)C + v, seed).x[0]) < thr) f |= kKeepD;
  }
  if (i < C) flags[L.row_base[g] + i] = f;
  const int ne = __syncthreads_count(f & kKeepE);
  const int nd = __syncthreads_count(f & kKeepD);
  const int nc = __syncthreads_count(f & kCheck);
  if (threadIdx.x == 0) { cnt_e[t] = ne; cnt_d[t] = nd; cnt_c[t] = nc; }
}

// blockIdx.x = list, blockIdx.y = count k (E, D, check): counts_k[tile_base[g] ..) -> exclusive offsets, the total
// -> totals[3 (g0 + g) + k]
__global__ void __launch_bounds__(1024) lp_scan_kernel(const PointLists L, int* __restrict__ counts, int tiles,
                                                       int* __restrict__ totals) {
  const int g = blockIdx.x, k = blockIdx.y;
  scan_block_counts(counts + (size_t)k * tiles + L.tile_base[g], L.tile_base[g + 1] - L.tile_base[g],
                    totals + 3 * (L.g0 + g) + k);
}

__global__ void __launch_bounds__(kRowThreads) lp_emit_kernel(const PointLists L, unsigned long long seed,
                                                              const unsigned char* __restrict__ flags,
                                                              const int* __restrict__ off_e,
                                                              const int* __restrict__ off_d,
                                                              const int* __restrict__ off_c) {
  __shared__ int wc_e[kRowThreads / 32], wc_d[kRowThreads / 32], wc_c[kRowThreads / 32];
  const int t = L.tile_base[0] + blockIdx.x;
  const int g = list_of(L, t);
  const long long i = (long long)(t - L.tile_base[g]) * kRowThreads + threadIdx.x;
  const long long M = L.M[g], C = M + L.V[g];
  const unsigned char f = i < C ? flags[L.row_base[g] + i] : 0;
  const int re = block_rank(f & kKeepE, wc_e);
  const int rd = block_rank(f & kKeepD, wc_d);
  const int rc = block_rank(f & kCheck, wc_c);
  if (i >= C) return;
  const unsigned long long cb = L.ctr_base[g], uC = (unsigned long long)C;
  const long long nE = L.nE[g], nD = L.nD[g];
  float* xe = L.out_e[g];
  float* xd = L.out_d[g];
  float p[3], q[3];
  long long se = -1, sd = -1;            // this row's B_E / B_D row, if any
  if (i < M) {
#pragma unroll
    for (int a = 0; a < 3; ++a) p[a] = __ldg(L.pts[g] + 3 * i + a);
    se = sd = i;
    if (f & kCheck) {
      const long long s = (long long)off_c[t] + rc;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        L.out_pts[g][3 * s + a] = p[a];
        L.out_rays[g][3 * s + a] = __ldg(L.rays[g] + 3 * i + a);
      }
      L.out_batch[g][s] = __ldg(L.batch[g] + i);
      L.out_row[g][s] = __ldg(L.row[g] + i);
      L.out_col[g][s] = __ldg(L.col[g] + i);
      L.out_index[g][s] = i;
    }
  } else if (f & (kKeepE | kKeepD)) {
#pragma unroll
    for (int a = 0; a < 3; ++a) p[a] = __ldg(L.verts[g] + 3 * (i - M) + a);
    if (f & kKeepE) se = M + off_e[t] + re;
    if (f & kKeepD) sd = M + off_d[t] + rd;
  }
  if (se >= 0) {
    local_point(p, cb + 2 * uC + (unsigned long long)se, seed, q);
#pragma unroll
    for (int a = 0; a < 3; ++a) xe[3 * se + a] = q[a];
  }
  if (sd >= 0) {
    local_point(p, cb + 4 * uC + (unsigned long long)sd, seed, q);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      xd[3 * sd + a] = p[a];
      xd[3 * (nD + sd) + a] = q[a];
    }
  }
  if (i < nE / 6) {                      // global row i (|B_E| / 6 <= C / 6 rows: every one has a thread)
    const Philox4 x = draw(cb + 3 * uC + (unsigned long long)i, seed);
#pragma unroll
    for (int a = 0; a < 3; ++a) xe[3 * (nE + i) + a] = __fsub_rn(__fmul_rn(unit24(x.x[a]), 3.6f), 1.8f);
  }
}

long long tiles_of(long long C) { return (C + kRowThreads - 1) / kRowThreads; }

// rows and blocks of the call, or an error for a bad size
int list_sizes(int G, const int64_t* M, const int64_t* V, long long* rows, long long* tiles) {
  if (G < 0) return RECMV_E_SHAPE;
  if (G > 0 && (!M || !V)) return RECMV_E_NULL;
  *rows = 0;
  *tiles = 0;
  for (int g = 0; g < G; ++g) {
    if (M[g] < 0 || V[g] <= 0) return RECMV_E_SHAPE;         // the reference divides by V_g
    if (M[g] > 0x7fffffffLL || V[g] > 0x7fffffffLL - M[g]) return RECMV_E_RANGE;   // counts and ranks are int32
    *rows += M[g] + V[g];
    *tiles += tiles_of(M[g] + V[g]);
  }
  if (*tiles > 0x7fffffffLL) return RECMV_E_RANGE;
  return RECMV_OK;
}

struct Workspace {
  unsigned char* flags;
  int* cnt;                               // [3, tiles]: E, D, check
};

Workspace lp_layout(Carve& c, long long rows, long long tiles) {
  return {c.take<unsigned char>(rows), c.take<int>(3 * tiles)};
}

// fills the per-group fields shared by both passes; returns the next group's tile base
long long group(PointLists& L, int g0, int G, const int64_t* M, const int64_t* V, int S, long long* row_base,
                long long tile_base, unsigned long long* ctr) {
  L.g0 = g0;
  L.G = G - g0 < kMaxLists ? G - g0 : kMaxLists;
  for (int g = 0; g < L.G; ++g) {
    const int a = g0 + g;
    L.M[g] = M[a];
    L.V[g] = V[a];
    L.thr[g] = (float)((double)S / (double)V[a]);
    L.row_base[g] = *row_base;
    L.ctr_base[g] = *ctr;
    L.tile_base[g] = (int)tile_base;
    *row_base += M[a] + V[a];
    *ctr += 5ull * (unsigned long long)(M[a] + V[a]);
    tile_base += tiles_of(M[a] + V[a]);
  }
  L.tile_base[L.G] = (int)tile_base;
  return tile_base;
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_loss_points_workspace_bytes(int G, const int64_t* M, const int64_t* V, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  long long rows, tiles;
  const int s = list_sizes(G, M, V, &rows, &tiles);
  if (s) return s;
  *bytes = layout_bytes(lp_layout, rows, tiles);
  return RECMV_OK;
}

extern "C" int recmv_loss_points_count(int G, const int64_t* M, const int64_t* V, const uint8_t* const* check, int S,
                                       uint64_t seed, uint64_t offset, void* workspace, int32_t* counts,
                                       recmv_stream_t stream) {
  long long rows, tiles;
  int s = list_sizes(G, M, V, &rows, &tiles);
  if (s) return s;
  if (S < 0) return RECMV_E_SHAPE;
  if (G == 0) return RECMV_OK;
  if (!counts || !workspace || !check) return RECMV_E_NULL;
  for (int g = 0; g < G; ++g)
    if (M[g] > 0 && !check[g]) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  const Workspace w = carve(workspace, lp_layout, rows, tiles);
  long long row_base = 0, tile_base = 0;
  unsigned long long ctr = (unsigned long long)offset;
  for (int g0 = 0; g0 < G; g0 += kMaxLists) {
    PointLists L = {};
    const long long t0 = tile_base;
    tile_base = group(L, g0, G, M, V, S, &row_base, tile_base, &ctr);
    for (int g = 0; g < L.G; ++g) L.check[g] = (const unsigned char*)check[g0 + g];
    lp_count_kernel<<<(int)(tile_base - t0), kRowThreads, 0, st>>>(L, (unsigned long long)seed, w.flags, w.cnt,
                                                                    w.cnt + tiles, w.cnt + 2 * tiles);
    if ((s = launch_status())) return s;
    lp_scan_kernel<<<dim3(L.G, 3), 1024, 0, st>>>(L, w.cnt, (int)tiles, counts);
    if ((s = launch_status())) return s;
  }
  return RECMV_OK;
}

extern "C" int recmv_loss_points_emit(int G, const float* const* init_pts, const int64_t* M, const float* const* verts,
                                      const int64_t* V, const int64_t* const* batch, const int64_t* const* row,
                                      const int64_t* const* col, const float* const* rays, const int32_t* counts, int S,
                                      uint64_t seed, uint64_t offset, void* workspace, float* const* out_eikonal,
                                      float* const* out_regular, float* const* out_pts, float* const* out_rays,
                                      int64_t* const* out_batch, int64_t* const* out_row, int64_t* const* out_col,
                                      int64_t* const* out_index, recmv_stream_t stream) {
  long long rows, tiles;
  int s = list_sizes(G, M, V, &rows, &tiles);
  if (s) return s;
  if (S < 0) return RECMV_E_SHAPE;
  if (G == 0) return RECMV_OK;
  if (!counts || !workspace || !init_pts || !verts || !batch || !row || !col || !rays || !out_eikonal ||
      !out_regular || !out_pts || !out_rays || !out_batch || !out_row || !out_col || !out_index)
    return RECMV_E_NULL;
  for (int g = 0; g < G; ++g) {
    if (counts[3 * g] < 0 || counts[3 * g] > V[g] || counts[3 * g + 1] < 0 || counts[3 * g + 1] > V[g] ||
        counts[3 * g + 2] < 0 || counts[3 * g + 2] > M[g])
      return RECMV_E_SHAPE;
    if (!verts[g] || !out_eikonal[g] || !out_regular[g]) return RECMV_E_NULL;
    if (M[g] > 0 && (!init_pts[g] || !batch[g] || !row[g] || !col[g] || !rays[g])) return RECMV_E_NULL;
    if (counts[3 * g + 2] > 0 && (!out_pts[g] || !out_rays[g] || !out_batch[g] || !out_row[g] || !out_col[g] ||
                                  !out_index[g]))
      return RECMV_E_NULL;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const Workspace w = carve(workspace, lp_layout, rows, tiles);
  long long row_base = 0, tile_base = 0;
  unsigned long long ctr = (unsigned long long)offset;
  for (int g0 = 0; g0 < G; g0 += kMaxLists) {
    PointLists L = {};
    const long long t0 = tile_base;
    tile_base = group(L, g0, G, M, V, S, &row_base, tile_base, &ctr);
    for (int g = 0; g < L.G; ++g) {
      const int a = g0 + g;
      L.pts[g] = init_pts[a]; L.verts[g] = verts[a]; L.rays[g] = rays[a];
      L.batch[g] = (const long long*)batch[a]; L.row[g] = (const long long*)row[a]; L.col[g] = (const long long*)col[a];
      L.out_e[g] = out_eikonal[a]; L.out_d[g] = out_regular[a]; L.out_pts[g] = out_pts[a]; L.out_rays[g] = out_rays[a];
      L.out_batch[g] = (long long*)out_batch[a]; L.out_row[g] = (long long*)out_row[a];
      L.out_col[g] = (long long*)out_col[a]; L.out_index[g] = (long long*)out_index[a];
      L.nE[g] = M[a] + counts[3 * a];
      L.nD[g] = M[a] + counts[3 * a + 1];
    }
    lp_emit_kernel<<<(int)(tile_base - t0), kRowThreads, 0, st>>>(L, (unsigned long long)seed, w.flags, w.cnt,
                                                                   w.cnt + tiles, w.cnt + 2 * tiles);
    if ((s = launch_status())) return s;
  }
  return RECMV_OK;
}

// Marching cubes with shared vertices -- deterministic sign-mask / count / scan / emit.
// Replaces MCGpu/CudaKernels.cu:316-521 (d_mc_get_mesh_on_gpu, d_conver_ijkd_to_pindex, d_set_int,
// d_scale_vertices) and the MCGpu singleton (CudaKernels.cu:524-639).
//
// Reference cost per call: memset of 3*N ints (-1), case tables in global memory, two global atomics
// per triangle, output buffers sized to 5 % of the cells with no overflow check, blocking D2H copy.
// Here: ONE read of the grid, then everything works on a 1-bit-per-voxel sign mask (N / 8 bytes, L2 resident):
//   pass 0 (signs): coalesced read of the grid -> ballot -> bit t of word w = (sdf[32 w + t] < iso)        [HBM bound]
//   pass 1 (count): one lane per run of 32 consecutive cells: the eight corner masks of the run are 8 funnel-shifted
//                   words of the sign mask; cells with mixed signs = (OR of the masks) & ~(AND of the masks) -- 98 % of
//                   the runs are done after ~40 instructions for 32 cells; only surface cells index the case tables
//   pass 2 (scan) : exclusive scan of the per-segment (verts, tris) sums (one CTA); totals stay on the device
//   pass 3 (verts): same decode -> warp scan -> owned-edge vertices (v*step+origin) and a packed (first vertex id,
//                   rank of edges 0/3/8) word for ACTIVE cells only (no memset: only written entries are ever read)
//   pass 4 (faces): same decode -> warp scan -> int64 faces, neighbours' vertex ids from the packed words
// Algorithmic bytes = 4 B x N (one read of the grid) + 12 B x V + 24 B x F.
// Output order = the order a sequential sweep of the reference kernel would produce (cells by linear
// index, vertices by first appearance in the cell's triangle list), so results are reproducible and
// comparable index-for-index with the CPU restatement (oracle/mc_oracle.c); against the reference kernel's own
// (atomics-ordered) output they are bit-identical after canonical ordering (tests/golden/mc_ref.npz).
#include "common.cuh"
#include "mc_tables.h"
#include "workspace.cuh"

namespace recmv {

constexpr int kMcThreads = 1024;   // cells per segment (one warp: 32 lanes x 32 consecutive cells)
// Division of a 31-bit index by a runtime constant through a precomputed multiplier (Granlund-Montgomery):
// the per-cell (i,j,k) decomposition otherwise costs two ~20-instruction integer divisions per cell.
struct FastDiv {
  unsigned d, m, s;
  __host__ static FastDiv make(unsigned d) {
    FastDiv f;
    f.d = d;
    unsigned s = 0;
    while ((1ull << s) < d) ++s;
    f.s = s;
    f.m = (unsigned)(((1ull << 32) * ((1ull << s) - d)) / d + 1);
    return f;
  }
  __device__ __forceinline__ unsigned div(unsigned n) const {
    unsigned t = __umulhi(m, n);
    return (t + n) >> s;  // n < 2^31 and t <= n: no overflow
  }
};

struct McTables {
  signed char tri[256][16];
  unsigned char ntri[256];
  unsigned char vinfo[256];  // bits 0-1 rank(edge0), 2-3 rank(edge3), 4-5 rank(edge8) (3 = absent), 6-7 count
  signed char owner[12][4];  // owning voxel offset + axis of every cube edge
};
__constant__ McTables c_mc;
// copy of the triangle table in global memory: the face kernel indexes it with per-thread case numbers, and
// divergent __constant__ reads serialise 32-way (L1-cached global loads do not)
__device__ signed char g_mc_tri[256][16];
// ... and so are the per-case counts and the edge-owner table: the emit / count passes index them with per-lane case
// numbers and edge ids (packed: di | dj << 8 | dk << 16 | axis << 24)
__device__ unsigned char g_mc_ntri[256];
__device__ unsigned char g_mc_vinfo[256];
__device__ unsigned int g_mc_owner[12];

static void build_tables(McTables& t) {
  for (int c = 0; c < 256; ++c) {
    int n = 0;
    while (n < 5 && mc_tri_entry(c, 3 * n) >= 0) ++n;
    t.ntri[c] = (unsigned char)n;
    int rank[3] = {3, 3, 3}, cnt = 0;
    for (int q = 0; q < 3 * n; ++q) {
      int e = mc_tri_entry(c, q);
      int slot = e == 0 ? 0 : (e == 3 ? 1 : (e == 8 ? 2 : -1));
      if (slot >= 0 && rank[slot] == 3) rank[slot] = cnt++;
    }
    t.vinfo[c] = (unsigned char)(rank[0] | (rank[1] << 2) | (rank[2] << 4) | (cnt << 6));
    for (int q = 0; q < 16; ++q) t.tri[c][q] = (signed char)mc_tri_entry(c, q);
  }
  for (int e = 0; e < 12; ++e)
    for (int q = 0; q < 4; ++q) t.owner[e][q] = kMcEdgeOwner[e][q];
}

static int ensure_tables() {
  static int dev_done[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return RECMV_E_RANGE;
  if (!dev_done[dev]) {
    static McTables host;
    build_tables(host);
    cudaError_t e = cudaMemcpyToSymbol(c_mc, &host, sizeof(McTables));
    if (e != cudaSuccess) return (int)e;
    e = cudaMemcpyToSymbol(g_mc_tri, host.tri, sizeof(host.tri));
    if (e != cudaSuccess) return (int)e;
    e = cudaMemcpyToSymbol(g_mc_ntri, host.ntri, sizeof(host.ntri));
    if (e != cudaSuccess) return (int)e;
    e = cudaMemcpyToSymbol(g_mc_vinfo, host.vinfo, sizeof(host.vinfo));
    if (e != cudaSuccess) return (int)e;
    unsigned int owner[12];
    for (int q = 0; q < 12; ++q)
      owner[q] = (unsigned)(host.owner[q][0] & 255) | ((unsigned)(host.owner[q][1] & 255) << 8) |
                 ((unsigned)(host.owner[q][2] & 255) << 16) | ((unsigned)(host.owner[q][3] & 255) << 24);
    e = cudaMemcpyToSymbol(g_mc_owner, owner, sizeof(owner));
    if (e != cudaSuccess) return (int)e;
    dev_done[dev] = 1;
  }
  return RECMV_OK;
}

// CTA-wide exclusive scan of an int2 (x = verts, y = tris); returns exclusive prefix, total in *tot.
__device__ __forceinline__ int2 block_excl_scan(int2 v, int2* tot) {
  __shared__ int2 warp_sums[32];
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int2 inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int ax = __shfl_up_sync(0xffffffffu, inc.x, o);
    int ay = __shfl_up_sync(0xffffffffu, inc.y, o);
    if (lane >= o) { inc.x += ax; inc.y += ay; }
  }
  if (lane == 31) warp_sums[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    int2 w = warp_sums[lane];
    int2 wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int ax = __shfl_up_sync(0xffffffffu, wi.x, o);
      int ay = __shfl_up_sync(0xffffffffu, wi.y, o);
      if (lane >= o) { wi.x += ax; wi.y += ay; }
    }
    warp_sums[lane] = make_int2(wi.x - w.x, wi.y - w.y);  // exclusive
    if (lane == 31) *tot = wi;
  }
  __syncthreads();
  int2 base = warp_sums[wid];
  int2 r = make_int2(base.x + inc.x - v.x, base.y + inc.y - v.y);
  __syncthreads();
  return r;
}

constexpr int kMcWarpBlock = 256;  // 8 warps per CTA in the warp-per-segment passes

// Pass 0: sign mask.  words = ceil(N / 32) + 2 (two zero words of padding so 64-bit windows never run off the end).
__global__ void __launch_bounds__(256) mc_sign_kernel(const float* __restrict__ sdf, unsigned N, float iso,
                                                      unsigned* __restrict__ bits, unsigned nwords) {
  const int lane = threadIdx.x & 31;
  const unsigned warp = (blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5;
  const unsigned nwarps = (gridDim.x * (unsigned)blockDim.x) >> 5;
  // 4 words per warp iteration: four independent coalesced 128-byte loads in flight per lane
  for (unsigned w0 = warp * 4; w0 < nwords; w0 += nwarps * 4) {
    float v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const unsigned idx = (w0 + q) * 32u + lane;
      v[q] = idx < N ? __ldg(sdf + idx) : iso;          // padding: not below the iso value -> bit 0
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const unsigned b = __ballot_sync(0xffffffffu, v[q] < iso);
      if (lane == q && w0 + q < nwords) bits[w0 + q] = b;
    }
  }
}

// The eight corner masks of the 32 cells [b, b + 32): bit t of m[c] = sign of corner c of cell b + t, corners in the
// cube-index bit order of the reference (CudaKernels.cu:316-360): (i,j,k) (i+1,j,k) (i+1,j+1,k) (i,j+1,k), then k+1.
struct RunMasks { unsigned m[8]; unsigned active; };
__device__ __forceinline__ unsigned bit_window(const unsigned* __restrict__ bits, unsigned pos) {
  const unsigned w = pos >> 5;
  return __funnelshift_r(__ldg(bits + w), __ldg(bits + w + 1), pos & 31u);
}
__device__ __forceinline__ RunMasks decode_run(const unsigned* __restrict__ bits, unsigned b, unsigned NZ, unsigned plane) {
  RunMasks r;
  const unsigned off[4] = {0u, plane, plane + NZ, NZ};
  unsigned any = 0u, all = 0xffffffffu;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    r.m[q] = bit_window(bits, b + off[q]);
    r.m[q + 4] = bit_window(bits, b + off[q] + 1u);
    any |= r.m[q] | r.m[q + 4];
    all &= r.m[q] & r.m[q + 4];
  }
  r.active = any & ~all;
  return r;
}
__device__ __forceinline__ int cube_index(const RunMasks& r, int t) {
  int ci = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) ci |= (int)((r.m[c] >> t) & 1u) << c;
  return ci;
}
// (i, j, k) of a flat index and whether it is the base corner of a cell
__device__ __forceinline__ bool cell_coords(unsigned idx, unsigned N, int NX, int NY, int NZ, unsigned plane,
                                            const FastDiv& dplane, const FastDiv& dnz, int& i, int& j, int& k) {
  i = (int)dplane.div(idx);
  const unsigned rem = idx - (unsigned)i * plane;
  j = (int)dnz.div(rem);
  k = (int)(rem - (unsigned)j * (unsigned)NZ);
  return idx < N && i < NX - 1 && j < NY - 1 && k < NZ - 1;
}

// Pass 1: one warp per 1024-cell segment (lane L owns cells seg*1024 + 32 L .. + 31): (verts, tris) of the segment.
__global__ void __launch_bounds__(kMcWarpBlock) mc_count_kernel(const unsigned* __restrict__ bits, int NX, int NY, int NZ,
                                                                int2* __restrict__ block_sums, int nseg,
                                                                FastDiv dplane, FastDiv dnz) {
  const unsigned N = (unsigned)NX * NY * NZ, plane = (unsigned)NY * NZ;
  const int lane = threadIdx.x & 31;
  const int seg = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
  if (seg >= nseg) return;
  const unsigned b = (unsigned)seg * kMcThreads + 32u * lane;
  int acc = 0;  // verts | tris << 16 of this lane
  if (b < N) {
    RunMasks r = decode_run(bits, b, (unsigned)NZ, plane);
    unsigned a = r.active;
    while (a) {
      const int t = __ffs(a) - 1;
      a &= a - 1;
      int i, j, k;
      if (!cell_coords(b + t, N, NX, NY, NZ, plane, dplane, dnz, i, j, k)) continue;
      const int ci = cube_index(r, t);
      acc += (g_mc_vinfo[ci] >> 6) | ((int)g_mc_ntri[ci] << 16);
    }
  }
  const int tot = __reduce_add_sync(0xffffffffu, acc);
  if (lane == 0) block_sums[seg] = make_int2(tot & 0xffff, tot >> 16);
}

// totals[0] = V, totals[1] = F, totals[2] = overflow flag (set by the emit passes), totals[3] = 0.
// One CTA, one pass: every thread owns a contiguous run of ceil(nb / 1024) segment sums (serial), the 1024 run totals
// are scanned once across the CTA, and the run is rewritten as exclusive prefixes.
__global__ void __launch_bounds__(kMcThreads) mc_scan_kernel(int2* __restrict__ block_sums, int nb,
                                                             int* __restrict__ totals) {
  __shared__ int2 tot;
  const int per = (nb + kMcThreads - 1) / kMcThreads;
  const int b0 = threadIdx.x * per, b1 = min(b0 + per, nb);
  int2 mine = make_int2(0, 0);
  for (int b = b0; b < b1; ++b) { const int2 v = block_sums[b]; mine.x += v.x; mine.y += v.y; }
  int2 run = block_excl_scan(mine, &tot);
  for (int b = b0; b < b1; ++b) {
    const int2 v = block_sums[b];
    block_sums[b] = run;
    run.x += v.x; run.y += v.y;
  }
  if (threadIdx.x == 0) { totals[0] = tot.x; totals[1] = tot.y; totals[2] = 0; totals[3] = 0; }
}

// (iso - v1) / (v2 - v1) evaluated like d_fGetOffset (CudaKernels.cu:304-314): float differences,
// double division, rounded to float; 0.5 when the edge is flat.
__device__ __forceinline__ float edge_offset(float v1, float v2, float iso) {
  double d = (double)(v2 - v1);
  if (d == 0.0) return 0.5f;
  return (float)((double)(iso - v1) / d);
}

// warp-wide exclusive scan
__device__ __forceinline__ int warp_excl_scan(int v, int lane, int* total) {
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  *total = __shfl_sync(0xffffffffu, inc, 31);
  return inc - v;
}

// Passes 3 and 4, one warp per segment, same decode as the count pass.  `cap` = capacity (rows) of the output buffer:
// a segment whose rows would not fit sets totals[2] and writes nothing (the host grows the buffer and re-runs).
// Active cells are rare (1-2 %) and clustered: a lane whose 32-cell run lies along the surface would own most of the
// warp's work.  So the warp first COMPACTS its active cells (cell order = lane-major, bit order) into a shared-memory
// list, then walks the list 32 cells per round, one cell per lane: every lane does the same amount of work, and the row
// offsets (segment base + exclusive prefix in cell order) are exactly those of a serial sweep.
template <bool kFaces>
__global__ void __launch_bounds__(kMcWarpBlock) mc_emit_kernel(
    const float* __restrict__ sdf, int NX, int NY, int NZ, float iso,
    const unsigned* __restrict__ bits, const int2* __restrict__ block_offs,
    int* __restrict__ cellinfo, float sx, float sy, float sz, float ox, float oy, float oz,
    float* __restrict__ verts, long long* __restrict__ faces, long long cap, int* __restrict__ totals, int nseg,
    FastDiv dplane, FastDiv dnz) {
  __shared__ unsigned s_list[kMcWarpBlock / 32][kMcThreads];   // (cell within segment) | cube index << 10
  const unsigned N = (unsigned)NX * NY * NZ, plane = (unsigned)NY * NZ;
  const int lane = threadIdx.x & 31;
  const int seg = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
  if (seg >= nseg) return;
  const int2 segoff = block_offs[seg];
  const int seg_end = seg + 1 < nseg ? (kFaces ? block_offs[seg + 1].y : block_offs[seg + 1].x)
                                     : (kFaces ? totals[1] : totals[0]);
  const int seg_begin = kFaces ? segoff.y : segoff.x;
  if (seg_end == seg_begin) return;   // nothing to emit here
  if ((long long)seg_end > cap) { if (lane == 0) totals[2] = 1; return; }
  const unsigned seg_base = (unsigned)seg * kMcThreads;
  const unsigned b = seg_base + 32u * lane;
  RunMasks r;
  r.active = 0u;
  if (b < N) r = decode_run(bits, b, (unsigned)NZ, plane);
  // sweep 1: drop the "cells" on the far faces of the grid, count mine
  int mine = 0;
  {
    unsigned a = r.active;
    while (a) {
      const int t = __ffs(a) - 1;
      a &= a - 1;
      int i, j, k;
      if (!cell_coords(b + t, N, NX, NY, NZ, plane, dplane, dnz, i, j, k)) r.active &= ~(1u << t);
      else ++mine;
    }
  }
  int n_cells;
  int pos = warp_excl_scan(mine, lane, &n_cells);
  // sweep 2: compact (cell, cube index) into the warp's list
  unsigned* list = s_list[threadIdx.x >> 5];
  {
    unsigned a = r.active;
    while (a) {
      const int t = __ffs(a) - 1;
      a &= a - 1;
      list[pos++] = (unsigned)(32 * lane + t) | ((unsigned)cube_index(r, t) << 10);
    }
  }
  __syncwarp();
  int carry = seg_begin;
  for (int base = 0; base < n_cells; base += 32) {
    const bool have = base + lane < n_cells;
    const unsigned rec = have ? list[base + lane] : 0u;
    const int ci = (int)(rec >> 10);
    const int info = kFaces ? 0 : (int)g_mc_vinfo[ci];
    const int cnt = !have ? 0 : (kFaces ? (int)g_mc_ntri[ci] : (info >> 6));
    int round_total;
    const int off = carry + warp_excl_scan(cnt, lane, &round_total);
    carry += round_total;
    if (cnt == 0) continue;
    const unsigned idx = seg_base + (rec & 1023u);
    int i, j, k;
    cell_coords(idx, N, NX, NY, NZ, plane, dplane, dnz, i, j, k);
    if (!kFaces) {
      const int vbase = off;
      cellinfo[idx] = (vbase << 6) | (info & 63);
      const float* p = sdf + idx;
      const float v0 = __ldg(p);
      const float fX = (float)i, fY = (float)j, fZ = (float)k;
      const int r0 = info & 3, r3 = (info >> 2) & 3, r8 = (info >> 4) & 3;
      if (r0 != 3) {  // edge 0: corner 0 -> 1, +x
        const float o_ = edge_offset(v0, __ldg(p + plane), iso);
        float* o = verts + (size_t)(vbase + r0) * 3;
        o[0] = fmaf(fX + o_, sx, ox); o[1] = fmaf(fY, sy, oy); o[2] = fmaf(fZ, sz, oz);
      }
      if (r3 != 3) {  // edge 3: corner 3 (0,1,0) -> 0, -y
        const float o_ = edge_offset(__ldg(p + NZ), v0, iso);
        float* o = verts + (size_t)(vbase + r3) * 3;
        o[0] = fmaf(fX, sx, ox); o[1] = fmaf(fY + (1.f - o_), sy, oy); o[2] = fmaf(fZ, sz, oz);
      }
      if (r8 != 3) {  // edge 8: corner 0 -> 4, +z
        const float o_ = edge_offset(v0, __ldg(p + 1), iso);
        float* o = verts + (size_t)(vbase + r8) * 3;
        o[0] = fmaf(fX, sx, ox); o[1] = fmaf(fY, sy, oy); o[2] = fmaf(fZ + o_, sz, oz);
      }
    } else {
      const long long fbase = off;
      for (int tt = 0; tt < cnt; ++tt) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int e = g_mc_tri[ci][3 * tt + c];
          const unsigned ow = g_mc_owner[e];
          const int oi = i + (int)(ow & 255u), oj = j + (int)((ow >> 8) & 255u), ok = k + (int)((ow >> 16) & 255u);
          const int d = (int)(ow >> 24);
          long long vid = -1;
          if (oi < NX - 1 && oj < NY - 1 && ok < NZ - 1) {
            const int oinfo = cellinfo[((int64_t)oi * NY + oj) * NZ + ok];
            vid = (long long)(oinfo >> 6) + ((oinfo >> (2 * d)) & 3);
          }
          faces[(fbase + tt) * 3 + (2 - c)] = vid;  // reversed winding (CudaKernels.cu:502)
        }
      }
    }
  }
}

struct McScratch {
  unsigned* bits;      // sign mask, nwords words
  unsigned nwords;
  int* cellinfo;
  int2* block_sums;
  int* totals;
  int nb;
};

static McScratch mc_layout(Carve& c, int NX, int NY, int NZ) {
  int64_t N = (int64_t)NX * NY * NZ;
  McScratch s;
  s.nb = (int)((N + kMcThreads - 1) / kMcThreads);
  s.nwords = (unsigned)((N + 31) / 32 + 2);
  s.bits = c.take<unsigned>(s.nwords);
  s.cellinfo = c.take<int>(N);
  s.block_sums = c.take<int2>(s.nb);
  s.totals = c.take<int>(4);
  return s;
}

static int mc_dims(int NX, int NY, int NZ) {
  if (NX <= 0 || NY <= 0 || NZ <= 0) return RECMV_E_SHAPE;
  if ((int64_t)NX * NY * NZ > 2000000000LL) return RECMV_E_RANGE;
  return RECMV_OK;
}

}  // namespace recmv

using namespace recmv;

extern "C" int recmv_mc_scratch_bytes(int NX, int NY, int NZ, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  const int s = mc_dims(NX, NY, NZ);
  if (s) return s;
  *bytes = layout_bytes(mc_layout, NX, NY, NZ);
  return RECMV_OK;
}

namespace {
// passes 0-2: sign mask, per-segment counts, scan (totals stay on the device)
int mc_classify(const float* sdf, int NX, int NY, int NZ, float iso, const McScratch& sc, cudaStream_t st) {
  const unsigned N = (unsigned)((int64_t)NX * NY * NZ);
  mc_sign_kernel<<<stride_grid((int64_t)sc.nwords * 8, 256, 8), 256, 0, st>>>(sdf, N, iso, sc.bits, sc.nwords);
  int s = launch_status();
  if (s) return s;
  const int grid = (sc.nb * 32 + kMcWarpBlock - 1) / kMcWarpBlock;  // one warp per 1024-cell segment
  const FastDiv dplane = FastDiv::make((unsigned)NY * NZ), dnz = FastDiv::make((unsigned)NZ);
  mc_count_kernel<<<grid, kMcWarpBlock, 0, st>>>(sc.bits, NX, NY, NZ, sc.block_sums, sc.nb, dplane, dnz);
  s = launch_status();
  if (s) return s;
  mc_scan_kernel<<<1, kMcThreads, 0, st>>>(sc.block_sums, sc.nb, sc.totals);
  return launch_status();
}

int mc_emit_passes(const float* sdf, int NX, int NY, int NZ, float iso, const McScratch& sc, const float step[3],
                   const float origin[3], float* verts, int64_t cap_v, int64_t* faces, int64_t cap_f, cudaStream_t st) {
  const int grid = (sc.nb * 32 + kMcWarpBlock - 1) / kMcWarpBlock;
  const FastDiv dplane = FastDiv::make((unsigned)NY * NZ), dnz = FastDiv::make((unsigned)NZ);
  mc_emit_kernel<false><<<grid, kMcWarpBlock, 0, st>>>(sdf, NX, NY, NZ, iso, sc.bits, sc.block_sums, sc.cellinfo,
                                                       step[0], step[1], step[2], origin[0], origin[1], origin[2],
                                                       verts, nullptr, cap_v, sc.totals, sc.nb, dplane, dnz);
  int s = launch_status();
  if (s) return s;
  // the faces read the packed vertex words the vertex pass wrote
  mc_emit_kernel<true><<<grid, kMcWarpBlock, 0, st>>>(sdf, NX, NY, NZ, iso, sc.bits, sc.block_sums, sc.cellinfo,
                                                      0.f, 0.f, 0.f, 0.f, 0.f, 0.f, nullptr, (long long*)faces, cap_f,
                                                      sc.totals, sc.nb, dplane, dnz);
  return launch_status();
}
}  // namespace

// One call, no host synchronisation: classify + count + scan + emit into caller-provided buffers of capacity
// (cap_verts, cap_faces) rows.  counts (device, int32[4]) receives {V, F, overflow, 0}: with overflow != 0 at least one of
// the buffers was too small -- rows that did fit are valid, the caller re-runs with buffers of (V, F) rows.
extern "C" int recmv_mc_run(const float* sdf, int NX, int NY, int NZ, float iso, void* scratch, const float step[3],
                            const float origin[3], float* verts, int64_t cap_verts, int64_t* faces, int64_t cap_faces,
                            int32_t* counts, recmv_stream_t stream) {
  if (!step || !origin || !counts || !verts || !faces) return RECMV_E_NULL;
  if (cap_verts < 0 || cap_faces < 0) return RECMV_E_SHAPE;
  if (!sdf || !scratch) return RECMV_E_NULL;
  int s = mc_dims(NX, NY, NZ);
  if (s) return s;
  if ((s = ensure_tables())) return s;
  cudaStream_t st = (cudaStream_t)stream;
  const McScratch sc = carve(scratch, mc_layout, NX, NY, NZ);
  s = mc_classify(sdf, NX, NY, NZ, iso, sc, st);
  if (s) return s;
  const int64_t cv = cap_verts < (1 << 25) ? cap_verts : (1 << 25) - 1;   // packed vertex ids are 26 bit signed-safe
  s = mc_emit_passes(sdf, NX, NY, NZ, iso, sc, step, origin, verts, cv, faces, cap_faces, st);
  if (s) return s;
  cudaError_t e = cudaMemcpyAsync(counts, sc.totals, 4 * sizeof(int32_t), cudaMemcpyDeviceToDevice, st);
  return e == cudaSuccess ? RECMV_OK : (int)e;
}

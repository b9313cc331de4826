// The random sub-sampling of the training rays (DESIGN section 1j): `sample_train_ray`
// (engineer/networks/OptimGarmentNetwork.py:983-1055) for G garments in one launch sequence, from the lists the
// fragment decode returns, with a counter-based Bernoulli draw in place of the reference's CPU `torch.rand`.
//
// Per garment g with input rows i < P_g (batch, row, col, init point) and ground-truth mask [N,H,W]:
//   candidates  rows with mask[b, r, c] > 0 (NaN fails; an index outside the mask is not a candidate), in input
//               order; pnum = their count, known only on the device;
//   selection   pnum <= T: every candidate, no draw.  Otherwise candidate j is kept iff u_j < thr, with
//               thr = fp32(double(T) / double(pnum)) and u_j = (x0 >> 8) 2^-24, x0 the first word of Philox4x32-10
//               under the 64-bit seed with counter offset + base_g + j, base_g = P_0 + ... + P_{g-1};
//   outputs     batch, row, col and the init point copied, and camera 0's view ray (compact.cuh), in candidate order.
//
//   1. tr_count_kernel  one thread per row: the candidate flag, per-block candidate counts;
//   2. tr_scan_kernel   one CTA per garment: exclusive scan of the counts, pnum;
//   3. tr_draw_kernel   one thread per row: candidate index j, the draw, per-block kept counts;
//   4. tr_scan_kernel   the kept counts, and the garment's kept count -> counts[g];
//   5. tr_emit_kernel   one thread per kept row: its slot and outputs.
// No atomics: the output is bit-identical from run to run.
#include "common.cuh"
#include "compact.cuh"
#include "philox.cuh"

namespace recmv {
namespace {

constexpr int kRowThreads = 256;
constexpr int kMaxLists = 8;       // garments per launch sequence; a call with more runs one sequence per group

struct RayLists {
  const long long* batch[kMaxLists];
  const long long* row[kMaxLists];
  const long long* col[kMaxLists];
  const float* pts[kMaxLists];
  const float* mask[kMaxLists];
  long long* out_batch[kMaxLists];
  long long* out_row[kMaxLists];
  long long* out_col[kMaxLists];
  float* out_pts[kMaxLists];
  float* out_rays[kMaxLists];
  long long len[kMaxLists];                   // input rows of list g
  long long row_base[kMaxLists];              // its first flag in the workspace
  unsigned long long ctr_base[kMaxLists];     // offset + the input rows of the earlier lists of the call
  int tile_base[kMaxLists + 1];               // its first block (absolute); tile_base[G] ends the group
  int g0;                                     // index of list 0 in the call
  int G;
};

// the list that absolute block t belongs to (lists without rows own no block)
__device__ __forceinline__ int list_of(const RayLists& L, int t) {
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

__global__ void __launch_bounds__(kRowThreads) tr_count_kernel(const RayLists L, int N, int H, int W,
                                                               unsigned char* __restrict__ flags,
                                                               int* __restrict__ cand_counts) {
  const int t = L.tile_base[0] + blockIdx.x;
  const int g = list_of(L, t);
  const long long i = (long long)(t - L.tile_base[g]) * kRowThreads + threadIdx.x;
  bool cand = false;
  if (i < L.len[g]) {
    const long long b = __ldg(L.batch[g] + i), r = __ldg(L.row[g] + i), c = __ldg(L.col[g] + i);
    if (b >= 0 && b < N && r >= 0 && r < H && c >= 0 && c < W)
      cand = __ldg(L.mask[g] + (b * H + r) * W + c) > 0.f;
    flags[L.row_base[g] + i] = cand;
  }
  const int n = __syncthreads_count(cand);
  if (threadIdx.x == 0) cand_counts[t] = n;
}

// blockIdx.x = list: counts[tile_base[g] ..) -> exclusive offsets, their total -> totals[g0 + g]
__global__ void __launch_bounds__(1024) tr_scan_kernel(const RayLists L, int* __restrict__ counts,
                                                       int* __restrict__ totals) {
  const int g = blockIdx.x;
  scan_block_counts(counts + L.tile_base[g], L.tile_base[g + 1] - L.tile_base[g], totals + L.g0 + g);
}

__global__ void __launch_bounds__(kRowThreads) tr_draw_kernel(const RayLists L, long long target,
                                                              unsigned long long seed,
                                                              unsigned char* __restrict__ flags,
                                                              const int* __restrict__ cand_offs,
                                                              const int* __restrict__ pnum,
                                                              int* __restrict__ keep_counts) {
  __shared__ int warp_cnt[kRowThreads / 32];
  const int t = L.tile_base[0] + blockIdx.x;
  const int g = list_of(L, t);
  const long long i = (long long)(t - L.tile_base[g]) * kRowThreads + threadIdx.x;
  const bool cand = i < L.len[g] && flags[L.row_base[g] + i];
  const int j = cand_offs[t] + block_rank(cand, warp_cnt);
  bool keep = false;
  if (cand) {
    const int pn = pnum[L.g0 + g];
    if ((long long)pn <= target) {
      keep = true;
    } else {
      const float thr = __double2float_rn(__ddiv_rn((double)target, (double)pn));
      const unsigned long long ctr = L.ctr_base[g] + (unsigned long long)j;
      const Philox4 x = philox4x32_10((unsigned)ctr, (unsigned)(ctr >> 32), (unsigned)seed, (unsigned)(seed >> 32));
      keep = (float)(x.x[0] >> 8) * 0x1p-24f < thr;
    }
    flags[L.row_base[g] + i] = keep;
  }
  const int n = __syncthreads_count(keep);
  if (threadIdx.x == 0) keep_counts[t] = n;
}

__global__ void __launch_bounds__(kRowThreads) tr_emit_kernel(const RayLists L, const unsigned char* __restrict__ flags,
                                                              const int* __restrict__ keep_offs,
                                                              const float* __restrict__ cam) {
  __shared__ int warp_cnt[kRowThreads / 32];
  const int t = L.tile_base[0] + blockIdx.x;
  const int g = list_of(L, t);
  const long long i = (long long)(t - L.tile_base[g]) * kRowThreads + threadIdx.x;
  const bool keep = i < L.len[g] && flags[L.row_base[g] + i];
  const int r = block_rank(keep, warp_cnt);
  if (!keep) return;
  const long long slot = keep_offs[t] + r;
  const long long row = __ldg(L.row[g] + i), col = __ldg(L.col[g] + i);
  L.out_batch[g][slot] = __ldg(L.batch[g] + i);
  L.out_row[g][slot] = row;
  L.out_col[g][slot] = col;
#pragma unroll
  for (int a = 0; a < 3; ++a) L.out_pts[g][3 * slot + a] = __ldg(L.pts[g] + 3 * i + a);
  float R[9], ray[3];
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = __ldg(cam + 4 + k);
  view_ray(__ldg(cam), __ldg(cam + 1), __ldg(cam + 2), __ldg(cam + 3), R, (float)col, (float)row, ray);
#pragma unroll
  for (int a = 0; a < 3; ++a) L.out_rays[g][3 * slot + a] = ray[a];
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

long long tiles_of(int64_t P) { return (P + kRowThreads - 1) / kRowThreads; }

// rows and blocks of the call, or an error for a bad length
int list_sizes(int G, const int64_t* lengths, long long* rows, long long* tiles) {
  if (G < 0) return RECMV_E_SHAPE;
  if (G > 0 && !lengths) return RECMV_E_NULL;
  *rows = 0;
  *tiles = 0;
  for (int g = 0; g < G; ++g) {
    if (lengths[g] < 0) return RECMV_E_SHAPE;
    if (lengths[g] > 0x7fffffffLL) return RECMV_E_RANGE;          // counts and ranks are int32
    *rows += lengths[g];
    *tiles += tiles_of(lengths[g]);
  }
  if (*tiles > 0x7fffffffLL) return RECMV_E_RANGE;
  return RECMV_OK;
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_train_rays_workspace_bytes(int G, const int64_t* lengths, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  long long rows, tiles;
  const int s = list_sizes(G, lengths, &rows, &tiles);
  if (s) return s;
  *bytes = align256((size_t)rows) + 2 * align256((size_t)tiles * 4) + align256((size_t)G * 4);
  return RECMV_OK;
}

extern "C" int recmv_train_rays_sample(int G, const int64_t* const* batch, const int64_t* const* row,
                                       const int64_t* const* col, const float* const* init_pts,
                                       const int64_t* lengths, const float* const* masks, int N, int H, int W,
                                       const float* camera, int64_t target, uint64_t seed, uint64_t offset,
                                       void* workspace, int64_t* const* out_batch, int64_t* const* out_row,
                                       int64_t* const* out_col, float* const* out_pts, float* const* out_rays,
                                       int32_t* counts, recmv_stream_t stream) {
  long long rows, tiles;
  int s = list_sizes(G, lengths, &rows, &tiles);
  if (s) return s;
  if (N < 0 || H <= 0 || W <= 0) return RECMV_E_SHAPE;
  if (G == 0) return RECMV_OK;
  if (!counts) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  if (rows == 0) return (int)cudaMemsetAsync(counts, 0, (size_t)G * 4, st);
  if (!batch || !row || !col || !init_pts || !masks || !out_batch || !out_row || !out_col || !out_pts || !out_rays ||
      !camera || !workspace)
    return RECMV_E_NULL;
  for (int g = 0; g < G; ++g)
    if (lengths[g] > 0 && (!batch[g] || !row[g] || !col[g] || !init_pts[g] || !masks[g] || !out_batch[g] ||
                           !out_row[g] || !out_col[g] || !out_pts[g] || !out_rays[g]))
      return RECMV_E_NULL;
  unsigned char* flags = (unsigned char*)workspace;
  int* cand = (int*)((char*)workspace + align256((size_t)rows));
  int* keep = (int*)((char*)cand + align256((size_t)tiles * 4));
  int* pnum = (int*)((char*)keep + align256((size_t)tiles * 4));
  long long row_base = 0, tile_base = 0;
  unsigned long long ctr = (unsigned long long)offset;
  for (int g0 = 0; g0 < G; g0 += kMaxLists) {
    RayLists L = {};
    L.g0 = g0;
    L.G = G - g0 < kMaxLists ? G - g0 : kMaxLists;
    for (int g = 0; g < L.G; ++g) {
      const int a = g0 + g;
      L.batch[g] = (const long long*)batch[a]; L.row[g] = (const long long*)row[a]; L.col[g] = (const long long*)col[a];
      L.pts[g] = init_pts[a]; L.mask[g] = masks[a];
      L.out_batch[g] = (long long*)out_batch[a]; L.out_row[g] = (long long*)out_row[a];
      L.out_col[g] = (long long*)out_col[a]; L.out_pts[g] = out_pts[a]; L.out_rays[g] = out_rays[a];
      L.len[g] = lengths[a];
      L.row_base[g] = row_base;
      L.ctr_base[g] = ctr;
      L.tile_base[g] = (int)tile_base;
      row_base += lengths[a];
      ctr += (unsigned long long)lengths[a];
      tile_base += tiles_of(lengths[a]);
    }
    L.tile_base[L.G] = (int)tile_base;
    const int nb = L.tile_base[L.G] - L.tile_base[0];
    if (nb > 0) {
      tr_count_kernel<<<nb, kRowThreads, 0, st>>>(L, N, H, W, flags, cand);
      if ((s = launch_status())) return s;
    }
    tr_scan_kernel<<<L.G, 1024, 0, st>>>(L, cand, pnum);
    if ((s = launch_status())) return s;
    if (nb > 0) {
      tr_draw_kernel<<<nb, kRowThreads, 0, st>>>(L, (long long)target, (unsigned long long)seed, flags, cand, pnum,
                                                 keep);
      if ((s = launch_status())) return s;
    }
    tr_scan_kernel<<<L.G, 1024, 0, st>>>(L, keep, counts);
    if ((s = launch_status())) return s;
    if (nb > 0) {
      tr_emit_kernel<<<nb, kRowThreads, 0, st>>>(L, flags, keep, camera);
      if ((s = launch_status())) return s;
    }
  }
  return RECMV_OK;
}

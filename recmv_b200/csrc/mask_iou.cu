// The dilation and soft IoU of `mask_loss` (DESIGN section 1m), in place of the reference's
// `F.max_pool2d(gt, 2r+1, 1, r)` and `compute_garment_pc_loss`'s IoU arithmetic
// (engineer/networks/OptimGarmentNetwork.py:621-629, 941-947), for all G garments and N frames of a call.
//
//   g'    = max over the (2r+1)^2 window of gt, out-of-image taps ignored (max_pool2d's -inf padding; a NaN tap wins,
//           as in torch).  Row maxima then column maxima over a 32 x 32 tile with an r-pixel halo in shared memory.
//   I     = sum m g',  U = sum |(m + g') - m g'|: each product and sum in f32 as the reference forms them, the pixel
//           terms accumulated in f64 per 32 x 32 tile (one tile = one frame_mean.cuh chunk), the tile partials then
//           combined in tile order per (g, n).  L_gn = 1 - I / U (U = 0 gives NaN, as 0 / 0 does), loss_g = mean_n L_gn.
//   dm    = -(w_g / N) (g' U - I s (1 - g')) / U^2, s = sign((m + g') - m g') with sign(0) = 0 (torch's abs gradient),
//           in double from the saved g' and (I, U), rounded once.
// No float atomics and a partition fixed by the image shape, so every output is bit-identical from run to run.
#include "common.cuh"
#include "frame_mean.cuh"
#include "workspace.cuh"

namespace recmv {
namespace {

constexpr int kTile = 32;                 // output tile edge: one tile is one kChunkRows chunk
constexpr int kMaxRadius = 32;            // (32 + 2r)^2 + (32 + 2r) 32 floats of shared memory: 48 KB at r = 32
constexpr int kMaxGarments = 8;           // garments per pixel launch; a call with more runs one launch per group
static_assert(kTile * kTile == kChunkRows, "one tile per chunk");
static_assert(((kTile + 2 * kMaxRadius) * (kTile + 2 * kMaxRadius) + (kTile + 2 * kMaxRadius) * kTile) * 4 <= 48 * 1024,
              "the largest halo tile fits the default dynamic shared memory");

struct MaskGroup {
  const float* m[kMaxGarments];           // silhouettes [N,H,W]
  const float* gt[kMaxGarments];          // ground-truth masks [N,H,W]
  float* mgt[kMaxGarments];               // forward: dilated masks out; backward: read
  float* dm[kMaxGarments];                // backward: dL/dm out
};

template <class T>
__device__ __forceinline__ T pick(const T (&a)[kMaxGarments], int g) {
  T v = a[0];
#pragma unroll
  for (int k = 1; k < kMaxGarments; ++k)
    if (g == k) v = a[k];
  return v;
}

// max_pool2d's update: a larger value or a NaN replaces the running maximum.
__device__ __forceinline__ float pool_max(float acc, float v) { return (v > acc || isnan(v)) ? v : acc; }

// One CTA per (tile, frame, garment of the group): g' of the tile, and the tile's (I, U) partial.
__global__ void __launch_bounds__(kMeanThreads) mask_iou_tile_kernel(const MaskGroup P, int g0, int N, int H, int W,
                                                                     int r, int tiles_x, long long tiles,
                                                                     double2* __restrict__ part) {
  extern __shared__ float sm[];
  const int S = kTile + 2 * r;
  float* halo = sm;                       // [S][S] gt, -inf outside the image
  float* rows = sm + S * S;               // [S][kTile] row maxima
  const int g = blockIdx.z, n = blockIdx.y;
  const int ty0 = (int)(blockIdx.x / tiles_x) * kTile, tx0 = (int)(blockIdx.x % tiles_x) * kTile;
  const size_t img = (size_t)n * H * W;
  const float* gt = pick(P.gt, g) + img;
  for (int i = threadIdx.x; i < S * S; i += kMeanThreads) {
    const int y = ty0 - r + i / S, x = tx0 - r + i % S;
    halo[i] = (y >= 0 && y < H && x >= 0 && x < W) ? __ldg(gt + (size_t)y * W + x) : -INFINITY;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < S * kTile; i += kMeanThreads) {
    const float* h = halo + (i / kTile) * S + i % kTile;
    float v = h[0];
    for (int j = 1; j <= 2 * r; ++j) v = pool_max(v, h[j]);
    rows[i] = v;
  }
  __syncthreads();
  const float* m = pick(P.m, g) + img;
  float* mgt = pick(P.mgt, g) + img;
  double I = 0.0, U = 0.0;
#pragma unroll
  for (int k = 0; k < kRowsPerThread; ++k) {
    const int ly = k * (kMeanThreads / kTile) + threadIdx.x / kTile, lx = threadIdx.x % kTile;
    const int y = ty0 + ly, x = tx0 + lx;
    if (y >= H || x >= W) continue;
    const float* c = rows + ly * kTile + lx;
    float v = c[0];
    for (int j = 1; j <= 2 * r; ++j) v = pool_max(v, c[j * kTile]);
    const size_t p = (size_t)y * W + x;
    mgt[p] = v;
    const float mv = __ldg(m + p);
    const float prod = __fmul_rn(mv, v);
    I += (double)prod;
    U += (double)fabsf(__fsub_rn(__fadd_rn(mv, v), prod));
  }
  __shared__ double red[kMeanThreads / 32];
  I = block_sum(I, red);
  U = block_sum(U, red);
  if (threadIdx.x == 0) part[((size_t)(g0 + g) * N + n) * tiles + blockIdx.x] = make_double2(I, U);
}

// One CTA per garment: per frame the tile partials summed in tile order, then L_gn and the mean over the frames.
__global__ void __launch_bounds__(kMeanThreads) mask_iou_finish_kernel(const double2* __restrict__ part, int N,
                                                                       long long tiles, double2* __restrict__ iu,
                                                                       float* __restrict__ loss_gn,
                                                                       float* __restrict__ loss) {
  __shared__ double red[kMeanThreads / 32];
  const int g = blockIdx.x;
  double L = 0.0;
  for (int n = 0; n < N; ++n) {
    const double2* p = part + ((size_t)g * N + n) * tiles;
    double I = 0.0, U = 0.0;
    for (long long c = threadIdx.x; c < tiles; c += kMeanThreads) {
      I += p[c].x;
      U += p[c].y;
    }
    I = block_sum(I, red);
    U = block_sum(U, red);
    if (threadIdx.x == 0) {
      const double l = 1.0 - I / U;
      iu[(size_t)g * N + n] = make_double2(I, U);
      loss_gn[(size_t)g * N + n] = __double2float_rn(l);
      L += l;
    }
  }
  if (threadIdx.x == 0) loss[g] = __double2float_rn(L / (double)N);
}

// One thread per kRowsPerThread pixels (strided by the block), blockIdx.y = frame, blockIdx.z = garment of the group.
__global__ void __launch_bounds__(kMeanThreads) mask_iou_backward_kernel(const MaskGroup P, int g0, int N,
                                                                         long long HW,
                                                                         const double2* __restrict__ iu,
                                                                         const float* __restrict__ grad_loss) {
  const int g = blockIdx.z, n = blockIdx.y;
  const double2 s = iu[(size_t)(g0 + g) * N + n];
  const double I = s.x, U = s.y;
  const double w = (double)__ldg(grad_loss + g0 + g) / (double)N;
  const size_t img = (size_t)n * HW;
  const float* m = pick(P.m, g) + img;
  const float* mgt = pick(P.mgt, g) + img;
  float* dm = pick(P.dm, g) + img;
  const long long p0 = (long long)blockIdx.x * kChunkRows + threadIdx.x;
#pragma unroll
  for (int k = 0; k < kRowsPerThread; ++k) {
    const long long p = p0 + k * kMeanThreads;
    if (p >= HW) break;
    const float mv = __ldg(m + p), gv = __ldg(mgt + p);
    const float u = __fsub_rn(__fadd_rn(mv, gv), __fmul_rn(mv, gv));
    const double sg = u > 0.f ? 1.0 : u < 0.f ? -1.0 : 0.0;
    const double G = (double)gv;
    dm[p] = __double2float_rn(-w * (G * U - I * sg * (1.0 - G)) / (U * U));
  }
}

int mask_iou_sizes(int G, int N, int H, int W, int r, long long* tiles, int* tiles_x) {
  if (G <= 0 || N <= 0 || H <= 0 || W <= 0 || r < 1) return RECMV_E_SHAPE;
  if (r > kMaxRadius || N > 65535) return RECMV_E_RANGE;
  *tiles_x = (W + kTile - 1) / kTile;
  *tiles = (long long)*tiles_x * ((H + kTile - 1) / kTile);
  if (*tiles > 0x7fffffffLL) return RECMV_E_RANGE;
  return RECMV_OK;
}

double2* mask_iou_layout(Carve& c, int G, int N, long long tiles) { return c.take<double2>((size_t)G * N * tiles); }

bool group_ok(const float* const* a, int g0, int n) {
  for (int k = 0; k < n; ++k)
    if (!a[g0 + k]) return false;
  return true;
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_mask_iou_workspace_bytes(int G, int N, int H, int W, int r, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  long long tiles;
  int tiles_x;
  const int s = mask_iou_sizes(G, N, H, W, r, &tiles, &tiles_x);
  if (s) return s;
  *bytes = layout_bytes(mask_iou_layout, G, N, tiles);
  return RECMV_OK;
}

extern "C" int recmv_mask_iou(int G, const float* const* m, const float* const* gt, int N, int H, int W, int r,
                              void* workspace, float* const* mgt, double* iu, float* loss_gn, float* loss,
                              recmv_stream_t stream) {
  long long tiles;
  int tiles_x;
  int s = mask_iou_sizes(G, N, H, W, r, &tiles, &tiles_x);
  if (s) return s;
  if (!m || !gt || !mgt || !workspace || !iu || !loss_gn || !loss) return RECMV_E_NULL;
  if (!group_ok(m, 0, G) || !group_ok(gt, 0, G) || !group_ok(mgt, 0, G)) return RECMV_E_NULL;
  const cudaStream_t st = (cudaStream_t)stream;
  double2* part = carve(workspace, mask_iou_layout, G, N, tiles);
  const int S = kTile + 2 * r;
  const size_t smem = (size_t)(S * S + S * kTile) * sizeof(float);
  for (int g0 = 0; g0 < G; g0 += kMaxGarments) {
    const int n = G - g0 < kMaxGarments ? G - g0 : kMaxGarments;
    MaskGroup P{};
    for (int k = 0; k < n; ++k) {
      P.m[k] = m[g0 + k];
      P.gt[k] = gt[g0 + k];
      P.mgt[k] = mgt[g0 + k];
    }
    mask_iou_tile_kernel<<<dim3((unsigned)tiles, (unsigned)N, (unsigned)n), kMeanThreads, smem, st>>>(
        P, g0, N, H, W, r, tiles_x, tiles, part);
    if ((s = launch_status())) return s;
  }
  mask_iou_finish_kernel<<<G, kMeanThreads, 0, st>>>(part, N, tiles, (double2*)iu, loss_gn, loss);
  return launch_status();
}

extern "C" int recmv_mask_iou_backward(int G, const float* const* m, const float* const* mgt, int N, int H, int W,
                                       const double* iu, const float* grad_loss, float* const* dm,
                                       recmv_stream_t stream) {
  if (G <= 0 || N <= 0 || H <= 0 || W <= 0) return RECMV_E_SHAPE;
  if (N > 65535) return RECMV_E_RANGE;
  if (!m || !mgt || !dm || !iu || !grad_loss) return RECMV_E_NULL;
  if (!group_ok(m, 0, G) || !group_ok(mgt, 0, G) || !group_ok(dm, 0, G)) return RECMV_E_NULL;
  const long long HW = (long long)H * W;
  const long long blocks = (HW + kChunkRows - 1) / kChunkRows;
  if (blocks > 0x7fffffffLL) return RECMV_E_RANGE;
  for (int g0 = 0; g0 < G; g0 += kMaxGarments) {
    const int n = G - g0 < kMaxGarments ? G - g0 : kMaxGarments;
    MaskGroup P{};
    for (int k = 0; k < n; ++k) {
      P.m[k] = m[g0 + k];
      P.mgt[k] = (float*)mgt[g0 + k];
      P.dm[k] = dm[g0 + k];
    }
    mask_iou_backward_kernel<<<dim3((unsigned)blocks, (unsigned)N, (unsigned)n), kMeanThreads, 0,
                               (cudaStream_t)stream>>>(P, g0, N, HW, (const double2*)iu, grad_loss);
    const int s = launch_status();
    if (s) return s;
  }
  return RECMV_OK;
}

// Rasteriser-fragment decode + seed points + view rays in one ordered compaction.
// Replaces utils/FindSurfacePs.py:7-60 (FindSurfacePs: `nonzero`, torch_scatter `scatter(min)`, three gathers, an
// index_select of the mesh, several host syncs) and the ray construction that follows it in the training step
// (model/CameraMine.py:146-167 view_rays, called from OptimGarmentNetwork.py:1046-1050 sample_train_ray), plus the
// ground-truth mask filter of sample_train_ray (:1006-1011).
//
// Per pixel (n, r, c) with K fragments: first k with pix_to_face >= 0 and all three barycentrics > 0; covered pixels are
// emitted in (n, r, c) order -- the order `nonzero` gives the reference -- with
//   finds = pix_to_face % F,   p = sum_i bary_i * verts[faces[finds][i]]   (same summation order as the reference's
//   (V[F] * w[:, :, None]).sum(1): ((w0 v0 + w1 v1) + w2 v2), one rounding per operation)
//   ray   = normalize(-c / fx + px / fx, -r / fy + py / fy, 1) @ R^T        (optional)
// HBM-bound: 8 K + 12 K bytes read per pixel, 64 bytes written per covered pixel.
#include "common.cuh"
#include "compact.cuh"
#include "workspace.cuh"

namespace recmv {
namespace {

constexpr int kFragThreads = 256;

struct FragCamera {
  float fx, fy, px, py;
  float R[9];      // row-major; rays = v @ R^T  ->  out_i = sum_j v_j R[i][j]
  int enabled;
};

__device__ __forceinline__ int first_valid(const long long* __restrict__ p2f, const float* __restrict__ bary, long long pix, int K) {
  for (int k = 0; k < K; ++k) {
    const float* b = bary + (pix * K + k) * 3;
    if (p2f[pix * K + k] >= 0 && b[0] > 0.f && b[1] > 0.f && b[2] > 0.f) return k;
  }
  return -1;
}

__global__ void __launch_bounds__(kFragThreads) frag_count_kernel(const long long* __restrict__ p2f, const float* __restrict__ bary,
                                                                  const float* __restrict__ mask, long long npix, int K,
                                                                  signed char* __restrict__ first, int* __restrict__ block_counts) {
  const long long pix = blockIdx.x * (long long)kFragThreads + threadIdx.x;
  int k = -1;
  if (pix < npix) {
    k = first_valid(p2f, bary, pix, K);
    if (k >= 0 && mask && !(mask[pix] > 0.f)) k = -1;
    first[pix] = (signed char)k;
  }
  const int n = __syncthreads_count(k >= 0);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = n;
}

// exclusive scan of the block counts (one CTA; nb <= a few thousand for a 1024^2 x 4 batch), total -> counters[0]
__global__ void __launch_bounds__(1024) frag_scan_kernel(int* __restrict__ block_counts, int nb, int* __restrict__ counters) {
  scan_block_counts(block_counts, nb, counters);
}

__global__ void __launch_bounds__(kFragThreads) frag_emit_kernel(
    const long long* __restrict__ p2f, const float* __restrict__ bary, const signed char* __restrict__ first,
    const int* __restrict__ block_offs, const float* __restrict__ verts, const long long* __restrict__ faces,
    long long num_faces, long long npix, int H, int W, int K, FragCamera cam, long long* __restrict__ out_batch,
    long long* __restrict__ out_row, long long* __restrict__ out_col, float* __restrict__ out_pts,
    long long* __restrict__ out_finds, float* __restrict__ out_rays) {
  __shared__ int warp_cnt[kFragThreads / 32];
  const long long pix = blockIdx.x * (long long)kFragThreads + threadIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int k = pix < npix ? (int)first[pix] : -1;
  const unsigned m = __ballot_sync(0xffffffffu, k >= 0);
  if (lane == 0) warp_cnt[wid] = __popc(m);
  __syncthreads();
  if (k < 0) return;
  int slot = block_offs[blockIdx.x] + __popc(m & ((1u << lane) - 1u));
  for (int w = 0; w < wid; ++w) slot += warp_cnt[w];
  const int c = (int)(pix % W), r = (int)((pix / W) % H);
  const long long n = pix / ((long long)W * H);
  out_batch[slot] = n; out_row[slot] = r; out_col[slot] = c;
  const long long f = p2f[pix * K + k] % num_faces;
  out_finds[slot] = f;
  const float* b = bary + (pix * K + k) * 3;
  const long long i0 = faces[3 * f], i1 = faces[3 * f + 1], i2 = faces[3 * f + 2];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float t0 = __fmul_rn(verts[3 * i0 + a], b[0]), t1 = __fmul_rn(verts[3 * i1 + a], b[1]), t2 = __fmul_rn(verts[3 * i2 + a], b[2]);
    out_pts[3 * (size_t)slot + a] = __fadd_rn(__fadd_rn(t0, t1), t2);
  }
  if (cam.enabled && out_rays) {
    float ray[3];
    view_ray(cam.fx, cam.fy, cam.px, cam.py, cam.R, (float)c, (float)r, ray);
#pragma unroll
    for (int i = 0; i < 3; ++i) out_rays[3 * (size_t)slot + i] = ray[i];
  }
}

struct FragWs { signed char* first; int* block_counts; };

// The block counts follow the first layers with 4-byte alignment.  No kernel reads the 256 bytes after them and
// nothing records what they were for; they stay so that the size does not change.
FragWs frag_layout(Carve& c, int64_t npix, int64_t nb) {
  const FragWs w{c.take<signed char>(npix), c.take<int>(nb, 4)};
  c.take<char>(256, 4);
  return w;
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" size_t recmv_fragment_decode_scratch_bytes(int64_t npix) {
  return layout_bytes(frag_layout, npix, (npix + kFragThreads - 1) / kFragThreads);
}

// camera: host float[13] = {fx, fy, px, py, R[9] row-major} or NULL (no rays).  counters: device int32[1] <- count.
// Outputs have capacity N*H*W rows; rows [0, count) are valid, in (n, row, col) order.
extern "C" int recmv_fragment_decode(const int64_t* pix_to_face, const float* bary, int N, int H, int W, int K,
                                     const float* verts, const int64_t* faces, int64_t num_faces, const float* mask,
                                     const float* camera, void* scratch, int64_t* out_batch, int64_t* out_row,
                                     int64_t* out_col, float* out_pts, int64_t* out_finds, float* out_rays,
                                     int32_t* counters, recmv_stream_t stream) {
  if (N < 0 || H <= 0 || W <= 0 || K <= 0 || K > 127 || num_faces <= 0) return RECMV_E_SHAPE;
  const int64_t npix = (int64_t)N * H * W;
  if (npix > 2000000000LL) return RECMV_E_RANGE;
  if (!counters) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  if (npix == 0) return (int)cudaMemsetAsync(counters, 0, 4, st);
  if (!pix_to_face || !bary || !verts || !faces || !scratch || !out_batch || !out_row || !out_col || !out_pts || !out_finds)
    return RECMV_E_NULL;
  if (camera && !out_rays) return RECMV_E_NULL;
  const int nb = (int)((npix + kFragThreads - 1) / kFragThreads);
  const FragWs w = carve(scratch, frag_layout, npix, nb);
  FragCamera cam = {};
  if (camera) {
    cam.fx = camera[0]; cam.fy = camera[1]; cam.px = camera[2]; cam.py = camera[3];
    for (int i = 0; i < 9; ++i) cam.R[i] = camera[4 + i];
    cam.enabled = 1;
  }
  frag_count_kernel<<<nb, kFragThreads, 0, st>>>((const long long*)pix_to_face, bary, mask, npix, K, w.first,
                                                 w.block_counts);
  int s = launch_status();
  if (s) return s;
  frag_scan_kernel<<<1, 1024, 0, st>>>(w.block_counts, nb, counters);
  s = launch_status();
  if (s) return s;
  frag_emit_kernel<<<nb, kFragThreads, 0, st>>>((const long long*)pix_to_face, bary, w.first, w.block_counts, verts,
                                                (const long long*)faces, num_faces, npix, H, W, K, cam,
                                                (long long*)out_batch, (long long*)out_row, (long long*)out_col, out_pts,
                                                (long long*)out_finds, out_rays);
  return launch_status();
}

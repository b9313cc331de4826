// The per-frame means of `surface_render_loss`'s photometric terms (DESIGN section 1k), in place of torch_scatter's
// `scatter(e, batch, reduce='mean', dim_size=N).mean()` (engineer/networks/OptimGarmentNetwork.py:1186-1188, 1198-1215),
// with their first-order backward.  The mean itself is frame_mean.cuh's.
//
//   colour  e_i = sum_c |gtCs[b, r, c, ch] - col_i[ch]|, the gather inside the kernel, the channels summed in order
//           0, 1, 2 in f32; backward dcol = -sign(gt - col) g / (N max(1, n_b)), sign(0) = 0.
//   normal  nn = |gtn_i|, valid iff nn > 1e-4, n = gtn / nn when valid (else gtn), d = J^T n - nx, e_i = |d| w_i,
//           mean over the valid rows only, in double; backward to nx, J and gtn (through the normalisation,
//           (I - n n^T) / nn), 0 at |d| = 0; w is a constant.
// Forward: one CTA per 1024-row chunk, then one CTA for the frames; backward: one thread per row.  No atomics.
#include "common.cuh"
#include "frame_mean.cuh"
#include "workspace.cuh"

namespace recmv {
namespace {

struct ColorRow {
  const float* gt;
  const long long* batch;
  const long long* row;
  const long long* col;
  const float* colors;
  int N, H, W;

  // pixel of row i, or -1 when its index lies outside gtCs
  __device__ __forceinline__ long long pixel(long long i) const {
    const long long b = __ldg(batch + i), r = __ldg(row + i), c = __ldg(col + i);
    if (b < 0 || b >= N || r < 0 || r >= H || c < 0 || c >= W) return -1;
    return (b * H + r) * W + c;
  }

  __device__ __forceinline__ void operator()(long long i, double& e, int& b) const {
    const long long p = pixel(i);
    if (p < 0) return;
    float s = fabsf(__fsub_rn(__ldg(gt + 3 * p), __ldg(colors + 3 * i)));
    s = __fadd_rn(s, fabsf(__fsub_rn(__ldg(gt + 3 * p + 1), __ldg(colors + 3 * i + 1))));
    s = __fadd_rn(s, fabsf(__fsub_rn(__ldg(gt + 3 * p + 2), __ldg(colors + 3 * i + 2))));
    e = (double)s;
    b = (int)__ldg(batch + i);
  }
};

// The per-row algebra of the normal term in double: n (normalised when valid), d = J^T n - nx.
struct NormalRow {
  const float* gtn;
  const float* J;
  const float* nx;
  const float* w;
  const long long* batch;
  int N;

  // false when the row is invalid or outside [0, N)
  __device__ __forceinline__ bool load(long long i, double* n, double& nn, double* d) const {
    const long long b = __ldg(batch + i);
    if (b < 0 || b >= N) return false;
#pragma unroll
    for (int a = 0; a < 3; ++a) n[a] = (double)__ldg(gtn + 3 * i + a);
    nn = sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
    if (!(nn > 1e-4)) return false;
#pragma unroll
    for (int a = 0; a < 3; ++a) n[a] /= nn;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      double s = 0.0;
#pragma unroll
      for (int a = 0; a < 3; ++a) s += (double)__ldg(J + 9 * i + 3 * a + c) * n[a];
      d[c] = s - (double)__ldg(nx + 3 * i + c);
    }
    return true;
  }

  __device__ __forceinline__ void operator()(long long i, double& e, int& b) const {
    double n[3], nn, d[3];
    if (!load(i, n, nn, d)) return;
    e = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]) * (double)__ldg(w + i);
    b = (int)__ldg(batch + i);
  }
};

template <class Row>
__global__ void __launch_bounds__(kMeanThreads) frame_partials_kernel(const Row row, long long M, int N,
                                                                      double* __restrict__ part_sum,
                                                                      int* __restrict__ part_cnt) {
  chunk_partials(row, M, N, part_sum, part_cnt);
}

__global__ void __launch_bounds__(kMeanThreads) frame_finish_kernel(const double* __restrict__ part_sum,
                                                                    const int* __restrict__ part_cnt, int chunks, int N,
                                                                    float* __restrict__ loss, int* __restrict__ counts) {
  finish_mean(part_sum, part_cnt, chunks, N, loss, counts);
}

__global__ void __launch_bounds__(kMeanThreads) color_backward_kernel(const ColorRow R, long long M,
                                                                      const int* __restrict__ counts,
                                                                      const float* __restrict__ grad_loss,
                                                                      float* __restrict__ dcol) {
  const long long i = (long long)blockIdx.x * kMeanThreads + threadIdx.x;
  if (i >= M) return;
  const long long p = R.pixel(i);
  const double s = p < 0 ? 0.0 : frame_scale(grad_loss, counts, R.N, (int)__ldg(R.batch + i));
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    float v = 0.f;
    if (p >= 0) {
      const float diff = __fsub_rn(__ldg(R.gt + 3 * p + ch), __ldg(R.colors + 3 * i + ch));
      v = diff > 0.f ? __double2float_rn(-s) : diff < 0.f ? __double2float_rn(s) : 0.f;
    }
    dcol[3 * i + ch] = v;
  }
}

__global__ void __launch_bounds__(kMeanThreads) normal_backward_kernel(const NormalRow R, long long M,
                                                                       const int* __restrict__ counts,
                                                                       const float* __restrict__ grad_loss,
                                                                       float* __restrict__ dgtn, float* __restrict__ dJ,
                                                                       float* __restrict__ dnx) {
  const long long i = (long long)blockIdx.x * kMeanThreads + threadIdx.x;
  if (i >= M) return;
  double n[3], nn = 1.0, d[3], gd[3] = {0.0, 0.0, 0.0};
  const bool ok = R.load(i, n, nn, d);
  if (ok) {
    const double dn = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    if (dn > 0.0) {
      const double s = frame_scale(grad_loss, counts, R.N, (int)__ldg(R.batch + i)) * (double)__ldg(R.w + i) / dn;
#pragma unroll
      for (int c = 0; c < 3; ++c) gd[c] = s * d[c];
    }
  } else {
    n[0] = n[1] = n[2] = 0.0;
  }
  double dn_hat[3], proj = 0.0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    double s = 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      s += (double)__ldg(R.J + 9 * i + 3 * a + c) * gd[c];
      dJ[9 * i + 3 * a + c] = __double2float_rn(n[a] * gd[c]);
    }
    dn_hat[a] = s;
    proj += n[a] * s;
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    dnx[3 * i + a] = __double2float_rn(-gd[a]);
    dgtn[3 * i + a] = ok ? __double2float_rn((dn_hat[a] - n[a] * proj) / nn) : 0.f;
  }
}

long long chunks_of(long long M) { return (M + kChunkRows - 1) / kChunkRows; }

int mean_sizes(int64_t M, int N, long long* chunks) {
  if (M < 0 || N <= 0) return RECMV_E_SHAPE;
  *chunks = chunks_of(M);
  if (*chunks > 0x7fffffffLL) return RECMV_E_RANGE;
  return RECMV_OK;
}

struct MeanWs { double* part_sum; int* part_cnt; };

MeanWs mean_layout(Carve& c, long long chunks, int N) { return {c.take<double>(chunks * N), c.take<int>(chunks * N)}; }

template <class Row>
int frame_mean(const Row& row, int64_t M, int N, void* workspace, float* loss, int32_t* counts, cudaStream_t st) {
  long long chunks;
  int s = mean_sizes(M, N, &chunks);
  if (s) return s;
  if (!loss || !counts || (chunks > 0 && !workspace)) return RECMV_E_NULL;
  const MeanWs w = carve(workspace, mean_layout, chunks, N);
  if (chunks > 0) {
    frame_partials_kernel<<<(unsigned)chunks, kMeanThreads, 0, st>>>(row, (long long)M, N, w.part_sum, w.part_cnt);
    if ((s = launch_status())) return s;
  }
  frame_finish_kernel<<<1, kMeanThreads, 0, st>>>(w.part_sum, w.part_cnt, (int)chunks, N, loss, (int*)counts);
  return launch_status();
}

unsigned row_blocks(int64_t M) { return (unsigned)((M + kMeanThreads - 1) / kMeanThreads); }

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_frame_loss_workspace_bytes(int64_t M, int N, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  long long chunks;
  const int s = mean_sizes(M, N, &chunks);
  if (s) return s;
  *bytes = layout_bytes(mean_layout, chunks, N);
  return RECMV_OK;
}

extern "C" int recmv_color_frame_mean(const float* gt, int N, int H, int W, const int64_t* batch, const int64_t* row,
                                      const int64_t* col, const float* colors, int64_t M, void* workspace, float* loss,
                                      int32_t* counts, recmv_stream_t stream) {
  if (H <= 0 || W <= 0) return RECMV_E_SHAPE;
  if (M > 0 && (!gt || !batch || !row || !col || !colors)) return RECMV_E_NULL;
  const ColorRow R{gt, (const long long*)batch, (const long long*)row, (const long long*)col, colors, N, H, W};
  return frame_mean(R, M, N, workspace, loss, counts, (cudaStream_t)stream);
}

extern "C" int recmv_color_frame_mean_backward(const float* gt, int N, int H, int W, const int64_t* batch,
                                               const int64_t* row, const int64_t* col, const float* colors, int64_t M,
                                               const int32_t* counts, const float* grad_loss, float* dcol,
                                               recmv_stream_t stream) {
  if (M < 0 || N <= 0 || H <= 0 || W <= 0) return RECMV_E_SHAPE;
  if (M == 0) return RECMV_OK;
  if (!gt || !batch || !row || !col || !colors || !counts || !grad_loss || !dcol) return RECMV_E_NULL;
  const ColorRow R{gt, (const long long*)batch, (const long long*)row, (const long long*)col, colors, N, H, W};
  color_backward_kernel<<<row_blocks(M), kMeanThreads, 0, (cudaStream_t)stream>>>(R, (long long)M, (const int*)counts,
                                                                                   grad_loss, dcol);
  return launch_status();
}

extern "C" int recmv_normal_frame_mean(const float* gtn, const float* J, const float* nx, const float* w,
                                       const int64_t* batch, int64_t M, int N, void* workspace, float* loss,
                                       int32_t* counts, recmv_stream_t stream) {
  if (M > 0 && (!gtn || !J || !nx || !w || !batch)) return RECMV_E_NULL;
  const NormalRow R{gtn, J, nx, w, (const long long*)batch, N};
  return frame_mean(R, M, N, workspace, loss, counts, (cudaStream_t)stream);
}

extern "C" int recmv_normal_frame_mean_backward(const float* gtn, const float* J, const float* nx, const float* w,
                                                const int64_t* batch, int64_t M, int N, const int32_t* counts,
                                                const float* grad_loss, float* dgtn, float* dJ, float* dnx,
                                                recmv_stream_t stream) {
  if (M < 0 || N <= 0) return RECMV_E_SHAPE;
  if (M == 0) return RECMV_OK;
  if (!gtn || !J || !nx || !w || !batch || !counts || !grad_loss || !dgtn || !dJ || !dnx) return RECMV_E_NULL;
  const NormalRow R{gtn, J, nx, w, (const long long*)batch, N};
  normal_backward_kernel<<<row_blocks(M), kMeanThreads, 0, (cudaStream_t)stream>>>(
      R, (long long)M, (const int*)counts, grad_loss, dgtn, dJ, dnx);
  return launch_status();
}

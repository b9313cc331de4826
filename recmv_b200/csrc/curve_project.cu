// The projection, visibility mask and compaction of `project_2d_loss` (DESIGN section 1n), in place of
// CameraMine.transform_points_screen, the z-buffer threshold test and the argsort / gather of `utils.fl_proj_loss`
// (engineer/networks/OptimGarmentNetwork.py:1604-1676), for every curve of every garment in one launch.
//
// Rows X [R,3] are the deformed curve points.  Curve k of the call (garment curves in order) owns, in frame n, the S
// rows base_k + n stride_k + s.  Per row, in double and rounded once:
//   view (X, Y, Z) = p R_n + T_n;  ndc = (fx' X/Z + px', fy' Y/Z + py', 1/Z) with pytorch3d's SfM K for (W, H):
//   fx' = fx / (W/2), px' = 1 - 1/W - px / (W/2) (likewise y);  screen = ((W-1)/2 - W ndc_x/2, (H-1)/2 - H ndc_y/2,
//   ndc_z).  visible = fl_masks[n, col_k] != 0 && body[row] < threshold_k.
// One CTA per cloud (k, n) then compacts its visible (x, y) in row order to clouds[(k N + n) S ...] (zeros after),
// counts[k N + n] = how many, slot[row] = the cloud row it went to or -1.  The scan is compact.cuh's.
// Backward: dX[row] = J^T dclouds[slot[row]] (0 for rows without a slot), J the 2 x 3 Jacobian of (x, y); a gather,
// so no atomics.  The cameras are constants.  Bit-identical across runs.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "compact.cuh"
#include "workspace.cuh"

namespace recmv {
namespace {

constexpr int kProjectThreads = 1024;     // scan_block_counts' block size
constexpr int kMaxProjectCurves = 64;

struct CurveTable {
  int base[kMaxProjectCurves], stride[kMaxProjectCurves], col[kMaxProjectCurves];
  float threshold[kMaxProjectCurves];
};

struct ProjectLayout {
  int* flags;                             // [K N][S]: visible flags, scanned in place to cloud positions
};

ProjectLayout project_layout(Carve& c, int K, int N, int S) {
  return ProjectLayout{c.take<int>((size_t)K * N * S)};
}

// view point of p under camera row cam {fx, fy, px, py, R row-major, T}: v_j = sum_k p_k R[k][j] + T_j
__device__ __forceinline__ void view_point(const float* cam, const float* p, double* v) {
  for (int j = 0; j < 3; ++j)
    v[j] = (double)p[0] * cam[4 + j] + (double)p[1] * cam[7 + j] + (double)p[2] * cam[10 + j] + (double)cam[13 + j];
}

__global__ void __launch_bounds__(kProjectThreads) curve_project_kernel(
    const float* __restrict__ X, const float* __restrict__ cams, int N, int W, int H, const CurveTable tab, int S,
    const float* __restrict__ fl_masks, int M, const float* __restrict__ body, ProjectLayout ws,
    float* __restrict__ screen, uint8_t* __restrict__ visible, int* __restrict__ slot, float* __restrict__ clouds,
    int64_t* __restrict__ counts) {
  __shared__ int total;
  const int cloud = blockIdx.x, k = cloud / N, n = cloud % N;
  const long long r0 = tab.base[k] + (long long)n * tab.stride[k];
  const float* cam = cams + 16 * n;
  const double fx = cam[0] / (W / 2.0), fy = cam[1] / (H / 2.0);
  const double px = 1.0 - 1.0 / W - cam[2] / (W / 2.0), py = 1.0 - 1.0 / H - cam[3] / (H / 2.0);
  const bool labelled = fl_masks[(size_t)n * M + tab.col[k]] != 0.f;
  const float thr = tab.threshold[k];
  int* flags = ws.flags + (size_t)cloud * S;
  for (int s = threadIdx.x; s < S; s += kProjectThreads) {
    const long long r = r0 + s;
    double v[3];
    view_point(cam, X + 3 * r, v);
    const double nx = fx * v[0] / v[2] + px, ny = fy * v[1] / v[2] + py;
    screen[3 * r] = (float)((W - 1.0) / 2.0 - W * nx / 2.0);
    screen[3 * r + 1] = (float)((H - 1.0) / 2.0 - H * ny / 2.0);
    screen[3 * r + 2] = (float)(1.0 / v[2]);
    const bool vis = labelled && body[r] < thr;
    visible[r] = vis;
    flags[s] = vis;
  }
  __syncthreads();
  scan_block_counts(flags, S, &total);
  __syncthreads();
  float* out = clouds + (size_t)cloud * S * 2;
  for (int s = threadIdx.x; s < S; s += kProjectThreads) {
    const long long r = r0 + s;
    if (visible[r]) {
      const int j = flags[s];
      out[2 * j] = screen[3 * r];
      out[2 * j + 1] = screen[3 * r + 1];
      slot[r] = cloud * S + j;
    } else {
      slot[r] = -1;
    }
    if (s >= total) out[2 * s] = out[2 * s + 1] = 0.f;
  }
  if (threadIdx.x == 0) counts[cloud] = total;
}

__global__ void curve_project_backward_kernel(const float* __restrict__ X, long long R, const float* __restrict__ cams,
                                              int N, int S, const int* __restrict__ slot,
                                              const float* __restrict__ dclouds, float* __restrict__ dX) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const int j = slot[r];
  if (j < 0) {
    dX[3 * r] = dX[3 * r + 1] = dX[3 * r + 2] = 0.f;
    return;
  }
  const float* cam = cams + 16 * ((j / S) % N);
  double v[3];
  view_point(cam, X + 3 * r, v);
  const double dx = dclouds[2 * (size_t)j], dy = dclouds[2 * (size_t)j + 1];
  // screen x = px - fx X/Z, screen y = py - fy Y/Z in pixels (the NDC round trip cancels)
  const double gv[3] = {-cam[0] * dx / v[2], -cam[1] * dy / v[2],
                        (cam[0] * v[0] * dx + cam[1] * v[1] * dy) / (v[2] * v[2])};
  for (int k = 0; k < 3; ++k)
    dX[3 * r + k] = (float)(cam[4 + 3 * k] * gv[0] + cam[5 + 3 * k] * gv[1] + cam[6 + 3 * k] * gv[2]);
}

int check_extents(int K, int N, int S) {
  if (K <= 0 || N <= 0 || S <= 0) return RECMV_E_SHAPE;
  if (K > kMaxProjectCurves || (long long)K * N * S > 0x7fffffffLL) return RECMV_E_RANGE;
  return RECMV_OK;
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_curve_project_workspace_bytes(int K, int N, int S, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  const int s = check_extents(K, N, S);
  if (s) return s;
  *bytes = layout_bytes(project_layout, K, N, S);
  return RECMV_OK;
}

extern "C" int recmv_curve_project(const float* X, int64_t R, const float* cams, int N, int W, int H,
                                   const int32_t* curves, const float* thresholds, int K, int S,
                                   const float* fl_masks, int M, const float* body, void* workspace, float* screen,
                                   uint8_t* visible, int32_t* slot, float* clouds, int64_t* counts,
                                   recmv_stream_t stream) {
  int s = check_extents(K, N, S);
  if (s) return s;
  if (W <= 0 || H <= 0 || M <= 0 || R <= 0) return RECMV_E_SHAPE;
  if (!X || !cams || !curves || !thresholds || !fl_masks || !body || !workspace || !screen || !visible || !slot ||
      !clouds || !counts)
    return RECMV_E_NULL;
  CurveTable tab{};
  long long rows = 0;
  for (int k = 0; k < K; ++k) {
    const long long base = curves[3 * k], stride = curves[3 * k + 1], col = curves[3 * k + 2];
    if (base < 0 || stride < 0 || col < 0 || col >= M || base + (N - 1) * stride + S > R) return RECMV_E_SHAPE;
    tab.base[k] = (int)base;
    tab.stride[k] = (int)stride;
    tab.col[k] = (int)col;
    tab.threshold[k] = thresholds[k];
    rows += (long long)N * S;
  }
  if (rows != R) return RECMV_E_SHAPE;
  // the K N ranges of S rows must not overlap (with the total equal to R they then cover every row exactly once):
  // two CTAs writing one row's flag and slot would race
  std::vector<long long> starts;
  starts.reserve((size_t)K * N);
  for (int k = 0; k < K; ++k)
    for (int n = 0; n < N; ++n) starts.push_back(tab.base[k] + (long long)n * tab.stride[k]);
  std::sort(starts.begin(), starts.end());
  for (size_t i = 1; i < starts.size(); ++i)
    if (starts[i] < starts[i - 1] + S) return RECMV_E_SHAPE;
  const ProjectLayout ws = carve(workspace, project_layout, K, N, S);
  curve_project_kernel<<<K * N, kProjectThreads, 0, (cudaStream_t)stream>>>(
      X, cams, N, W, H, tab, S, fl_masks, M, body, ws, screen, visible, slot, clouds, counts);
  return launch_status();
}

extern "C" int recmv_curve_project_backward(const float* X, int64_t R, const float* cams, int N, int K, int S,
                                            const int32_t* slot, const float* dclouds, float* dX,
                                            recmv_stream_t stream) {
  int s = check_extents(K, N, S);
  if (s) return s;
  if (R <= 0) return RECMV_E_SHAPE;
  if (R > 0x7fffffffLL * 256) return RECMV_E_RANGE;
  if (!X || !cams || !slot || !dclouds || !dX) return RECMV_E_NULL;
  curve_project_backward_kernel<<<(unsigned)((R + 255) / 256), 256, 0, (cudaStream_t)stream>>>(X, R, cams, N, S, slot,
                                                                                             dclouds, dX);
  return launch_status();
}

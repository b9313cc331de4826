// Surface-point solve of a batch of rays, entirely on the device (SURVEY 8a row A10; utils/FindSurfacePs.py:145-353:
// OptimizeSurfacePs / OptimizeGarmentSurfaceSinlge and the per-garment loop of OptimizeGarmentSurfacePs).
//
// The reference iterates  p <- p - L g / |g|^2  with  L = w1 |f(p)| + w2 |(D(p)-c) x v| / |D(p)-c|,  g = grad_p L
// on the not-yet-converged points, re-evaluating both networks after every step for the acceptance test
// (|f| < dthr and asin(.) 180/pi < athr), with an active-set compaction + several host syncs per iteration.
// Here one ROUND = two forward-mode launches (SDF value + gradient, deformer value + Jacobian; the tensor-core engine)
// and one update kernel; the evaluation at p_k serves BOTH as the acceptance test of step k-1 and as the
// gradient of step k, so `times` steps need times + 1 rounds (reference: 2 times + 1 evaluations), converged
// points are frozen by a flag instead of being compacted away, and nothing ever waits for the host.
#include "../../include/recmv_b200.h"
#include "common.cuh"
#include "workspace.cuh"

namespace recmv {
namespace {

struct SolveCfg {
  float cam[3];
  float dthr, athr_deg, w1, w2;
  int allow_step;
};

__global__ void __launch_bounds__(256) surface_update_kernel(float* __restrict__ ps, const float* __restrict__ rays,
                                                             const float* __restrict__ f, const float* __restrict__ gf,
                                                             const float* __restrict__ d, const float* __restrict__ J,
                                                             unsigned char* __restrict__ done, long long n, SolveCfg c) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (done[i]) continue;
    const float fv = f[i];
    const float dx = d[3 * i] - c.cam[0], dy = d[3 * i + 1] - c.cam[1], dz = d[3 * i + 2] - c.cam[2];
    const float vx = __ldg(rays + 3 * i), vy = __ldg(rays + 3 * i + 1), vz = __ldg(rays + 3 * i + 2);
    const float ux = dy * vz - dz * vy, uy = dz * vx - dx * vz, uz = dx * vy - dy * vx;   // (D - c) x v
    const float nu = sqrtf(ux * ux + uy * uy + uz * uz), nd = sqrtf(dx * dx + dy * dy + dz * dz);
    const float s = nu / nd;                                                             // sin of the angle
    const bool ok = fabsf(fv) < c.dthr && asinf(s) * 180.f / 3.14159265358979323846f < c.athr_deg;
    if (ok) { done[i] = 1; continue; }
    if (!c.allow_step) continue;
    // d s / d (D - c):  (d|u|/dd) / |d| - |u| d / |d|^3,   d|u|/dd = v x u / |u|   (u = d x v)
    float gx = 0.f, gy = 0.f, gz = 0.f;
    if (nu > 0.f) {
      const float inv = 1.f / (nu * nd);
      gx = (vy * uz - vz * uy) * inv; gy = (vz * ux - vx * uz) * inv; gz = (vx * uy - vy * ux) * inv;
    }
    const float k = nu / (nd * nd * nd);
    gx -= k * dx; gy -= k * dy; gz -= k * dz;
    const float sg = fv > 0.f ? 1.f : (fv < 0.f ? -1.f : 0.f);
    const float* Jm = J + 9 * i;
    float g[3];
#pragma unroll
    for (int j = 0; j < 3; ++j)   // J^T (w2 ds/dd) + w1 sign(f) grad f
      g[j] = c.w2 * (Jm[j] * gx + Jm[3 + j] * gy + Jm[6 + j] * gz) + c.w1 * sg * gf[3 * i + j];
    const float loss = c.w1 * fabsf(fv) + c.w2 * s;
    const float t = -loss / (g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
    ps[3 * i] += t * g[0]; ps[3 * i + 1] += t * g[1]; ps[3 * i + 2] += t * g[2];
  }
}

struct SolveWs { float *f, *gf, *d, *J; };   // SDF value and gradient, deformed point and its Jacobian

// Packed with 4-byte alignment.  No kernel reads the 256 bytes after J and nothing records what they were for; they
// stay so that the size does not change.
SolveWs solve_layout(Carve& c, int64_t P) {
  const SolveWs w{c.take<float>(P, 4), c.take<float>(3 * P, 4), c.take<float>(3 * P, 4), c.take<float>(9 * P, 4)};
  c.take<char>(256, 4);
  return w;
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" size_t recmv_surface_solve_workspace(int64_t P) {
  if (P <= 0) return 0;
  return layout_bytes(solve_layout, P);
}

extern "C" int recmv_surface_solve(const float* cam_pos, const float* rays, float* ps, const int64_t* batch_inds,
                                   const void* sdf_packed, const float* sdf_pe_w, const void* tr_packed,
                                   const float* tr_pe_w, const float* conds, int num_frames, const float* A,
                                   const float* trans, const recmv_voxel_t* vox, float dthreshold, float athreshold_deg,
                                   float w1, float w2, int times, int mode, void* workspace, size_t workspace_bytes,
                                   uint8_t* ok, int64_t P, recmv_stream_t stream) {
  if (P < 0 || times < 0 || num_frames <= 0) return RECMV_E_SHAPE;
  if (P == 0) return RECMV_OK;
  if (!cam_pos || !rays || !ps || !sdf_packed || !sdf_pe_w || !tr_packed || !tr_pe_w || !conds || !A || !trans || !vox ||
      !workspace || !ok)
    return RECMV_E_NULL;
  if (workspace_bytes < recmv_surface_solve_workspace(P)) return RECMV_E_SHAPE;
  if (!tc_passes(mode)) return RECMV_E_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const SolveWs w = carve(workspace, solve_layout, P);
  cudaError_t e = cudaMemsetAsync(ok, 0, (size_t)P, st);
  if (e != cudaSuccess) return (int)e;
  SolveCfg c;
  c.cam[0] = cam_pos[0]; c.cam[1] = cam_pos[1]; c.cam[2] = cam_pos[2];
  c.dthr = dthreshold; c.athr_deg = athreshold_deg; c.w1 = w1; c.w2 = w2;
  for (int round = 0; round <= times; ++round) {
    int s = recmv_sdf_mlp_fwd_grad(ps, sdf_packed, sdf_pe_w, w.f, nullptr, w.gf, P, mode, stream);
    if (s) return s;
    s = recmv_deformer_fwd_jac(ps, conds, batch_inds, batch_inds ? 0 : P, num_frames, tr_packed, tr_pe_w, A, trans, vox,
                               nullptr, nullptr, w.d, w.J, P, mode, stream);
    if (s) return s;
    c.allow_step = round < times ? 1 : 0;
    surface_update_kernel<<<stride_grid(P, 256, 4), 256, 0, st>>>(ps, rays, w.f, w.gf, w.d, w.J, ok, P, c);
    s = launch_status();
    if (s) return s;
  }
  return RECMV_OK;
}

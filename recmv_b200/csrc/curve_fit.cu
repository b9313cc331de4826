// The learnable feature curves of `project_2d_loss` and their regulariser (DESIGN section 1n), in place of
// Intersect_Free_Curve.forward and .regularization (engineer/utils/garment_structure.py:109-145).
//
//   v_s    = c + d_s s0_s relu(scale_s) + t_s nx                                     per curve, s = 0 .. S-1
//   e_i    = v_a(i) - v_b(i), i = 0 .. S: (i, i+1) for i < S-1, (S-1, 0), (0, 1)    the closed loop plus one wrap
//   u_i    = e_i / (|e_i| + 1e-6)
//   diff   = sum_{i<S} 1 - (u_i / max(|u_i|, 1e-8)) . (u_{i+1} / max(|u_{i+1}|, 1e-8))   (torch's cosine_similarity)
//   centre = sum_j |mean_s v_sj - c_j|
// One CTA per curve.  Everything is formed in double; v is rounded once to f32, and each curve's diff and centre are
// summed in double in index order and rounded once.  The backward follows torch's rules at the kinks: relu'(0) = 0,
// d|e|/de = 0 at e = 0, sign(0) = 0, and cosine_similarity's eps clamp is not differentiated (torch clamps the norms
// in place under no_grad, so the gradient reaches the norm as if unclamped).  No atomics: bit-identical across runs.
#include "common.cuh"

namespace recmv {
namespace {

constexpr int kCurveThreads = 256;
constexpr int kMaxCurvePoints = 1024;     // the backward's 13 S + 10 doubles of shared memory: 107 KB at S = 1024
constexpr double kNormEps = 1e-6, kCosEps = 1e-8;

struct CurveIn {
  const float *center, *dirs, *init_scale, *nx, *scale, *nx_scale;
};

__device__ __forceinline__ double norm3(const double* a) { return sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]); }

// v [S][3] of curve c in double, into shared memory; the f32 copy to out when out is not NULL.
__device__ void eval_curve(const CurveIn& in, int c, int S, double* v, float* out) {
  const double cx = in.center[3 * c], cy = in.center[3 * c + 1], cz = in.center[3 * c + 2];
  const double nx = in.nx[3 * c], ny = in.nx[3 * c + 1], nz = in.nx[3 * c + 2];
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    const size_t r = (size_t)c * S + s;
    const double sc = in.scale[r];
    const double k = (double)in.init_scale[r] * (sc > 0.0 ? sc : (sc == sc ? 0.0 : sc)), t = in.nx_scale[r];  // relu: NaN stays NaN
    const double p[3] = {cx + (double)in.dirs[3 * r] * k + t * nx, cy + (double)in.dirs[3 * r + 1] * k + t * ny,
                         cz + (double)in.dirs[3 * r + 2] * k + t * nz};
    for (int j = 0; j < 3; ++j) {
      v[3 * s + j] = p[j];
      if (out) out[3 * r + j] = (float)p[j];
    }
  }
}

// e_i (and |e_i|) for i = 0 .. S.
__device__ void edges(const double* v, int S, double* e, double* n) {
  for (int i = threadIdx.x; i <= S; i += blockDim.x) {
    const int a = i < S ? i : 0, b = i < S - 1 ? i + 1 : (i == S - 1 ? 0 : 1);
    for (int j = 0; j < 3; ++j) e[3 * i + j] = v[3 * a + j] - v[3 * b + j];
    n[i] = norm3(e + 3 * i);
  }
}

__global__ void __launch_bounds__(kCurveThreads) curve_fit_kernel(const CurveIn in, int S, float* __restrict__ v_out,
                                                                  float* __restrict__ reg) {
  extern __shared__ double sh[];
  double* v = sh;                     // [S][3]
  double* u = v + 3 * S;              // [S+1][3]
  double* n = u + 3 * (S + 1);        // [S+1]
  double* term = n + (S + 1);         // [S]
  const int c = blockIdx.x;
  eval_curve(in, c, S, v, v_out);
  __syncthreads();
  edges(v, S, u, n);
  __syncthreads();
  for (int i = threadIdx.x; i <= S; i += blockDim.x)
    for (int j = 0; j < 3; ++j) u[3 * i + j] /= n[i] + kNormEps;
  __syncthreads();
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    const double* a = u + 3 * i;
    const double* b = a + 3;
    const double na = fmax(norm3(a), kCosEps), nb = fmax(norm3(b), kCosEps);
    term[i] = 1.0 - ((a[0] / na) * (b[0] / nb) + (a[1] / na) * (b[1] / nb) + (a[2] / na) * (b[2] / nb));
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double diff = 0.0, m[3] = {0.0, 0.0, 0.0};
    for (int i = 0; i < S; ++i) diff += term[i];
    for (int s = 0; s < S; ++s)
      for (int j = 0; j < 3; ++j) m[j] += v[3 * s + j];
    double centre = 0.0;
    for (int j = 0; j < 3; ++j) centre += fabs(m[j] / S - (double)in.center[3 * c + j]);
    reg[2 * c] = (float)diff;
    reg[2 * c + 1] = (float)centre;
  }
}

__global__ void __launch_bounds__(kCurveThreads) curve_fit_backward_kernel(const CurveIn in, int S,
                                                                           const float* __restrict__ dv_up,
                                                                           const float* __restrict__ dreg,
                                                                           float* __restrict__ dscale,
                                                                           float* __restrict__ dnx_scale) {
  extern __shared__ double sh[];
  double* v = sh;                     // [S][3]
  double* e = v + 3 * S;              // [S+1][3] edges, then dL/de
  double* n = e + 3 * (S + 1);        // [S+1]
  double* u = n + (S + 1);            // [S+1][3]
  double* gu = u + 3 * (S + 1);       // [S+1][3] dL/du
  __shared__ double sgn[3];
  const int c = blockIdx.x;
  const double g_diff = dreg[2 * c], g_centre = dreg[2 * c + 1];
  eval_curve(in, c, S, v, nullptr);
  __syncthreads();
  edges(v, S, e, n);
  __syncthreads();
  for (int i = threadIdx.x; i <= S; i += blockDim.x)
    for (int j = 0; j < 3; ++j) u[3 * i + j] = e[3 * i + j] / (n[i] + kNormEps);
  if (threadIdx.x == 0) {
    double m[3] = {0.0, 0.0, 0.0};
    for (int s = 0; s < S; ++s)
      for (int j = 0; j < 3; ++j) m[j] += v[3 * s + j];
    for (int j = 0; j < 3; ++j) {
      const double d = m[j] / S - (double)in.center[3 * c + j];
      sgn[j] = d > 0.0 ? 1.0 : (d < 0.0 ? -1.0 : (d == d ? 0.0 : d));   // torch's sign: NaN stays NaN
    }
  }
  __syncthreads();
  // dL/du_i = dcos_i/da + dcos_{i-1}/db, each cos term with cotangent -g_diff
  for (int i = threadIdx.x; i <= S; i += blockDim.x) {
    double g[3] = {0.0, 0.0, 0.0};
    for (int side = 0; side < 2; ++side) {
      const int k = side == 0 ? i : i - 1;            // term k pairs (u_k, u_{k+1}); u_i is its a (side 0) or b
      if (k < 0 || k >= S) continue;
      const double* a = u + 3 * k;
      const double* b = a + 3;
      const double ra = norm3(a), rb = norm3(b);
      const double na = fmax(ra, kCosEps), nb = fmax(rb, kCosEps);
      const double dot = a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
      const double* self = side == 0 ? a : b;
      const double* other = side == 0 ? b : a;
      const double rs = side == 0 ? ra : rb, ns = side == 0 ? na : nb;
      for (int j = 0; j < 3; ++j) {
        const double us = rs > 0.0 ? self[j] / rs : 0.0;
        g[j] += -g_diff * (other[j] / (na * nb) - dot / (ns * na * nb) * us);
      }
    }
    for (int j = 0; j < 3; ++j) gu[3 * i + j] = g[j];
  }
  __syncthreads();
  // dL/de_i = gu / q - (gu . e) / q^2 * e / |e|, q = |e| + 1e-6; written over e
  for (int i = threadIdx.x; i <= S; i += blockDim.x) {
    const double q = n[i] + kNormEps;
    double* ei = e + 3 * i;
    const double* g = gu + 3 * i;
    const double ge = g[0] * ei[0] + g[1] * ei[1] + g[2] * ei[2];
    double out[3];
    for (int j = 0; j < 3; ++j) out[j] = g[j] / q - (n[i] > 0.0 ? ge / (q * q) * ei[j] / n[i] : 0.0);
    for (int j = 0; j < 3; ++j) ei[j] = out[j];
  }
  __syncthreads();
  const double nx[3] = {in.nx[3 * c], in.nx[3 * c + 1], in.nx[3 * c + 2]};
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    const size_t r = (size_t)c * S + s;
    double acc_d = 0.0, acc_t = 0.0;
    for (int j = 0; j < 3; ++j) {
      double g = e[3 * s + j];                                   // edge s starts at v_s
      if (s >= 1) g -= e[3 * (s - 1) + j];                       // edge s-1 ends at v_s
      if (s == 0) g += e[3 * S + j] - e[3 * (S - 1) + j];        // the wrap edge (0, 1) starts, (S-1, 0) ends here
      if (s == 1) g -= e[3 * S + j];
      g += g_centre * sgn[j] / S;
      if (dv_up) g += (double)dv_up[3 * r + j];
      acc_d += (double)in.dirs[3 * r + j] * g;
      acc_t += nx[j] * g;
    }
    dscale[r] = in.scale[r] > 0.f ? (float)((double)in.init_scale[r] * acc_d) : 0.f;
    dnx_scale[r] = (float)acc_t;
  }
}

int check_curves(int C, int S, const CurveIn& in) {
  if (C <= 0 || S < 2) return RECMV_E_SHAPE;
  if (S > kMaxCurvePoints || C > 65535) return RECMV_E_RANGE;
  if (!in.center || !in.dirs || !in.init_scale || !in.nx || !in.scale || !in.nx_scale) return RECMV_E_NULL;
  return RECMV_OK;
}

size_t fit_shared(int S) { return sizeof(double) * (3 * (size_t)S + 3 * (S + 1) + (S + 1) + S); }
size_t fit_backward_shared(int S) { return sizeof(double) * (3 * (size_t)S + 7 * (S + 1) + 3 * (S + 1)); }

// Opt the kernel into more than the default 48 KB of dynamic shared memory when S needs it.
template <class K>
int allow_shared(K kernel, size_t smem) {
  if (smem <= 48 * 1024) return RECMV_OK;
  return (int)cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_curve_fit(int C, int S, const float* center, const float* dirs, const float* init_scale,
                               const float* nx, const float* scale, const float* nx_scale, float* v, float* reg,
                               recmv_stream_t stream) {
  const CurveIn in{center, dirs, init_scale, nx, scale, nx_scale};
  int s = check_curves(C, S, in);
  if (s) return s;
  if (!v || !reg) return RECMV_E_NULL;
  const size_t smem = fit_shared(S);
  if ((s = allow_shared(curve_fit_kernel, smem))) return s;
  curve_fit_kernel<<<C, kCurveThreads, smem, (cudaStream_t)stream>>>(in, S, v, reg);
  return launch_status();
}

extern "C" int recmv_curve_fit_backward(int C, int S, const float* center, const float* dirs,
                                        const float* init_scale, const float* nx, const float* scale,
                                        const float* nx_scale, const float* dv, const float* dreg, float* dscale,
                                        float* dnx_scale, recmv_stream_t stream) {
  const CurveIn in{center, dirs, init_scale, nx, scale, nx_scale};
  int s = check_curves(C, S, in);
  if (s) return s;
  if (!dreg || !dscale || !dnx_scale) return RECMV_E_NULL;
  const size_t smem = fit_backward_shared(S);
  if ((s = allow_shared(curve_fit_backward_kernel, smem))) return s;
  curve_fit_backward_kernel<<<C, kCurveThreads, smem, (cudaStream_t)stream>>>(in, S, dv, dreg, dscale, dnx_scale);
  return launch_status();
}

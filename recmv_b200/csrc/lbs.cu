// Linear blend skinning on the diffused SMPL skinning voxel: forward warp and inverse warp.
// Replaces model/Deformer.py:406-445 (LBSkinner.forward after the bone matrices are built):
//   GridSamplerMine3dFunction (K4) -> matmul(ps_ws, A) -> matmul(T, [p;1]) -> + trans,
// including the per-frame python loop with a host sync per frame (Deformer.py:438-444).
//
// One thread per point: 8 corners x 24 channels gathered from the channels-last voxel as 48 128-bit
// loads (768 algorithmic bytes per point), 24x12 FMA bone blend with the bone matrices broadcast from
// L1/constant cache, 12 FMA apply; nothing but the 12-byte result goes back to HBM.
#include "common.cuh"

namespace recmv {

__device__ __forceinline__ int frame_of(const int64_t* __restrict__ batch_inds, int64_t p,
                                        int64_t ppf, int nf) {
  int64_t f = batch_inds ? batch_inds[p] : (ppf > 0 ? p / ppf : 0);
  if (f < 0) f = 0;
  if (f >= nf) f = nf - 1;
  return (int)f;
}

__global__ void __launch_bounds__(128) lbs_fwd_kernel(const float* __restrict__ ps,
                                                      const float* __restrict__ tps,
                                                      const float* __restrict__ A,
                                                      const float* __restrict__ trans,
                                                      const int64_t* __restrict__ batch_inds,
                                                      int64_t ppf, int nf, Voxel vox,
                                                      float* __restrict__ out,
                                                      float* __restrict__ weights_out, int64_t P) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < P;
       p += (int64_t)gridDim.x * blockDim.x) {
    float x = ps[3 * p], y = ps[3 * p + 1], z = ps[3 * p + 2];
    float tx = x, ty = y, tz = z;
    if (tps) { tx = tps[3 * p]; ty = tps[3 * p + 1]; tz = tps[3 * p + 2]; }
    float w[24], T[12];
    sample_skin24(vox, tx, ty, tz, w);
    int f = frame_of(batch_inds, p, ppf, nf);
    blend_bones(A + (size_t)f * 24 * 16, w, T);
    const float* t = trans + 3 * f;
    // T [p;1] accumulated in the order of a 4-term dot product, then + trans (Deformer.py:430-431)
    out[3 * p + 0] = (T[0] * x + T[1] * y + T[2] * z + T[3]) + __ldg(t + 0);
    out[3 * p + 1] = (T[4] * x + T[5] * y + T[6] * z + T[7]) + __ldg(t + 1);
    out[3 * p + 2] = (T[8] * x + T[9] * y + T[10] * z + T[11]) + __ldg(t + 2);
    if (weights_out) {
#pragma unroll
      for (int q = 0; q < 6; ++q)
        reinterpret_cast<float4*>(weights_out + p * 24)[q] =
            make_float4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]);
    }
  }
}

__global__ void __launch_bounds__(128) lbs_inverse_kernel(const float* __restrict__ xo,
                                                          const float* __restrict__ A,
                                                          const float* __restrict__ trans,
                                                          const int64_t* __restrict__ batch_inds,
                                                          int64_t ppf, int nf, Voxel vox,
                                                          float* __restrict__ xc,
                                                          uint8_t* __restrict__ valid, int64_t P) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < P;
       p += (int64_t)gridDim.x * blockDim.x) {
    int f = frame_of(batch_inds, p, ppf, nf);
    float cx, cy, cz;
    bool ok = inverse_lbs_point(vox, A + (size_t)f * 24 * 16, trans + 3 * f, xo[3 * p],
                                xo[3 * p + 1], xo[3 * p + 2], cx, cy, cz);
    xc[3 * p] = cx; xc[3 * p + 1] = cy; xc[3 * p + 2] = cz;
    if (valid) valid[p] = ok ? 1 : 0;
  }
}


// Bone matrices A = G . init_pose of the SMPL kinematic chain (model/Deformer.py:372-405): axis-angle -> rotation
// (the un-vendored smpl_pytorch.util.batch_rodrigues, standard HMR quaternion form: angle = |theta + 1e-8|), chain
// G_i = G_parent(i) . [R_i | J_i - J_parent(i)], then A_i = G_i . init_pose_i (or G_i - [0 | G_i J_i] without an init
// pose).  One thread per frame walks the 24 joints (parents precede children); replaces ~150 tiny torch launches
// per call of LBSkinner.forward / .inverse when no autograd graph is needed.
__global__ void __launch_bounds__(64) bone_matrices_kernel(const float* __restrict__ poses, const float* __restrict__ Js,
                                                           const int* __restrict__ parents, const float* __restrict__ init_pose,
                                                           float* __restrict__ G, float* __restrict__ A, int F) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  float* g = G + (size_t)f * 24 * 16;
  for (int i = 0; i < 24; ++i) {
    const float* th = poses + ((size_t)f * 24 + i) * 3;
    const float ax = th[0], ay = th[1], az = th[2];
    const float bx = ax + 1e-8f, by = ay + 1e-8f, bz = az + 1e-8f;
    const float angle = sqrtf(bx * bx + by * by + bz * bz);
    const float half = angle * 0.5f;
    float sn, cs;
    sincosf(half, &sn, &cs);
    float qw = cs, qx = sn * (ax / angle), qy = sn * (ay / angle), qz = sn * (az / angle);
    const float qn = sqrtf(qw * qw + qx * qx + qy * qy + qz * qz);
    qw /= qn; qx /= qn; qy /= qn; qz /= qn;
    const float w2 = qw * qw, x2 = qx * qx, y2 = qy * qy, z2 = qz * qz;
    const float wx = qw * qx, wy = qw * qy, wz = qw * qz, xy = qx * qy, xz = qx * qz, yz = qy * qz;
    float L[16];   // local transform [R | t; 0 0 0 1]
    L[0] = w2 + x2 - y2 - z2; L[1] = 2 * xy - 2 * wz;   L[2] = 2 * wy + 2 * xz;
    L[4] = 2 * wz + 2 * xy;   L[5] = w2 - x2 + y2 - z2; L[6] = 2 * yz - 2 * wx;
    L[8] = 2 * xz - 2 * wy;   L[9] = 2 * wx + 2 * yz;   L[10] = w2 - x2 - y2 + z2;
    const int par = i == 0 ? -1 : parents[i];
    L[3] = Js[3 * i] - (par >= 0 ? Js[3 * par] : 0.f);
    L[7] = Js[3 * i + 1] - (par >= 0 ? Js[3 * par + 1] : 0.f);
    L[11] = Js[3 * i + 2] - (par >= 0 ? Js[3 * par + 2] : 0.f);
    L[12] = 0.f; L[13] = 0.f; L[14] = 0.f; L[15] = 1.f;
    float* gi = g + 16 * i;
    if (par < 0) {
#pragma unroll
      for (int e = 0; e < 16; ++e) gi[e] = L[e];
    } else {
      const float* gp = g + 16 * par;
      float Pm[16];
#pragma unroll
      for (int e = 0; e < 16; ++e) Pm[e] = gp[e];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c)
          gi[4 * r + c] = Pm[4 * r] * L[c] + Pm[4 * r + 1] * L[4 + c] + Pm[4 * r + 2] * L[8 + c] + Pm[4 * r + 3] * L[12 + c];
    }
  }
  if (!A) return;
  for (int i = 0; i < 24; ++i) {
    const float* gi = g + 16 * i;
    float* a = A + ((size_t)f * 24 + i) * 16;
    if (init_pose) {
      const float* ip = init_pose + 16 * i;
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c)
          a[4 * r + c] = gi[4 * r] * ip[c] + gi[4 * r + 1] * ip[4 + c] + gi[4 * r + 2] * ip[8 + c] + gi[4 * r + 3] * ip[12 + c];
    } else {
      const float jx = Js[3 * i], jy = Js[3 * i + 1], jz = Js[3 * i + 2];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        a[4 * r] = gi[4 * r]; a[4 * r + 1] = gi[4 * r + 1]; a[4 * r + 2] = gi[4 * r + 2];
        a[4 * r + 3] = gi[4 * r + 3] - (gi[4 * r] * jx + gi[4 * r + 1] * jy + gi[4 * r + 2] * jz);
      }
    }
  }
}

// quat2mat of utils/utils.py:21-38 applied to the half-angle quaternion of batch_rodrigues, as in bone_matrices_kernel.
// Keeps what the backward needs: the unnormalised quaternion, its norm and the angle terms.
struct Rodrigues {
  float R[9];
  float angle, sn, cs, qn;
  float qw, qx, qy, qz;   // normalised
};

__device__ __forceinline__ void rodrigues(const float* __restrict__ th, Rodrigues& o) {
  const float ax = th[0], ay = th[1], az = th[2];
  const float bx = ax + 1e-8f, by = ay + 1e-8f, bz = az + 1e-8f;
  o.angle = sqrtf(bx * bx + by * by + bz * bz);
  sincosf(o.angle * 0.5f, &o.sn, &o.cs);
  float qw = o.cs, qx = o.sn * (ax / o.angle), qy = o.sn * (ay / o.angle), qz = o.sn * (az / o.angle);
  o.qn = sqrtf(qw * qw + qx * qx + qy * qy + qz * qz);
  qw /= o.qn; qx /= o.qn; qy /= o.qn; qz /= o.qn;
  o.qw = qw; o.qx = qx; o.qy = qy; o.qz = qz;
  const float w2 = qw * qw, x2 = qx * qx, y2 = qy * qy, z2 = qz * qz;
  const float wx = qw * qx, wy = qw * qy, wz = qw * qz, xy = qx * qy, xz = qx * qz, yz = qy * qz;
  o.R[0] = w2 + x2 - y2 - z2; o.R[1] = 2 * xy - 2 * wz;   o.R[2] = 2 * wy + 2 * xz;
  o.R[3] = 2 * wz + 2 * xy;   o.R[4] = w2 - x2 + y2 - z2; o.R[5] = 2 * yz - 2 * wx;
  o.R[6] = 2 * xz - 2 * wy;   o.R[7] = 2 * wx + 2 * yz;   o.R[8] = w2 - x2 - y2 + z2;
}

// VJP of rodrigues: dR (3x3) -> d theta.  quat2mat -> its re-normalisation q / |q| -> q = [cos(a/2), sin(a/2) theta / a]
// with a = |theta + 1e-8| (the HMR form: the 1e-8 enters the norm only).
__device__ __forceinline__ void rodrigues_vjp(const float* __restrict__ th, const Rodrigues& o, const float d[9],
                                              float* __restrict__ dth) {
  const float w = o.qw, x = o.qx, y = o.qy, z = o.qz;
  const float gw = 2.f * (w * (d[0] + d[4] + d[8]) + z * (d[3] - d[1]) + y * (d[2] - d[6]) + x * (d[7] - d[5]));
  const float gx = 2.f * (x * (d[0] - d[4] - d[8]) + y * (d[1] + d[3]) + z * (d[2] + d[6]) + w * (d[7] - d[5]));
  const float gy = 2.f * (y * (d[4] - d[0] - d[8]) + x * (d[1] + d[3]) + w * (d[2] - d[6]) + z * (d[5] + d[7]));
  const float gz = 2.f * (z * (d[8] - d[0] - d[4]) + w * (d[3] - d[1]) + x * (d[2] + d[6]) + y * (d[5] + d[7]));
  // through q / |q|
  const float dot = w * gw + x * gx + y * gy + z * gz;
  const float uw = (gw - w * dot) / o.qn, ux = (gx - x * dot) / o.qn, uy = (gy - y * dot) / o.qn,
              uz = (gz - z * dot) / o.qn;
  const float ax = th[0], ay = th[1], az = th[2];
  const float a = o.angle;
  const float nx = ax / a, ny = ay / a, nz = az / a;
  // q_w = cos(a/2), q_v = sin(a/2) n, n = theta / a
  float da = -0.5f * o.sn * uw + 0.5f * o.cs * (nx * ux + ny * uy + nz * uz);
  const float dnx = o.sn * ux, dny = o.sn * uy, dnz = o.sn * uz;
  da -= (ax * dnx + ay * dny + az * dnz) / (a * a);
  const float bx = ax + 1e-8f, by = ay + 1e-8f, bz = az + 1e-8f;
  dth[0] = dnx / a + da * (bx / a);
  dth[1] = dny / a + da * (by / a);
  dth[2] = dnz / a + da * (bz / a);
}

// Reverse of bone_matrices_kernel for one frame per thread.  dG of every joint (rows 0..2; row 3 of G is constant)
// lives in shared memory, [joint][element][thread] so that the 32 threads of a warp hit 32 banks.  Joints are visited
// from 23 down to 0: parents precede children, so a joint's dG is complete when it is reached.  Each child c of p
// (G_c = G_p L_c) adds dG_c L_c^T to dG_p and gives dR_c = (G_p^T dG_c)[:3,:3]; the root's dR is dG_0[:3,:3].
constexpr int kChainThreads = 32;

__global__ void __launch_bounds__(kChainThreads) bone_matrices_bwd_kernel(
    const float* __restrict__ poses, const float* __restrict__ Js, const int* __restrict__ parents,
    const float* __restrict__ init_pose, const float* __restrict__ G, const float* __restrict__ dG_in,
    const float* __restrict__ dA, float* __restrict__ dposes, int F) {
  __shared__ float sdG[24 * 12][kChainThreads];
  const int t = threadIdx.x;
  const int f = blockIdx.x * kChainThreads + t;
  if (f >= F) return;   // every shared column belongs to one thread: no barrier is needed
  const float* g = G + (size_t)f * 24 * 16;
  // seed: dG (rows 0..2) + the contribution of A_i = G_i . init_pose_i  (or G_i - [0 | G_i J_i])
  for (int i = 0; i < 24; ++i) {
    float acc[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) acc[e] = dG_in ? dG_in[((size_t)f * 24 + i) * 16 + e] : 0.f;
    if (dA) {
      const float* da = dA + ((size_t)f * 24 + i) * 16;
      if (init_pose) {
        const float* ip = init_pose + 16 * i;
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c)
            acc[4 * r + c] += da[4 * r] * ip[4 * c] + da[4 * r + 1] * ip[4 * c + 1] + da[4 * r + 2] * ip[4 * c + 2] +
                              da[4 * r + 3] * ip[4 * c + 3];
      } else {
        const float jx = Js[3 * i], jy = Js[3 * i + 1], jz = Js[3 * i + 2];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const float d3 = da[4 * r + 3];
          acc[4 * r + 0] += da[4 * r + 0] - d3 * jx;
          acc[4 * r + 1] += da[4 * r + 1] - d3 * jy;
          acc[4 * r + 2] += da[4 * r + 2] - d3 * jz;
          acc[4 * r + 3] += d3;
        }
      }
    }
#pragma unroll
    for (int e = 0; e < 12; ++e) sdG[12 * i + e][t] = acc[e];
  }
  for (int i = 23; i >= 0; --i) {
    Rodrigues q;
    const float* th = poses + ((size_t)f * 24 + i) * 3;
    rodrigues(th, q);
    float d[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) d[e] = sdG[12 * i + e][t];
    float dR[9];
    const int par = i == 0 ? -1 : parents[i];
    if (par < 0) {
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) dR[3 * r + c] = d[4 * r + c];
    } else {
      const float* gp = g + 16 * par;
      float Pm[12];
#pragma unroll
      for (int e = 0; e < 12; ++e) Pm[e] = gp[e];
      // dR = (G_p^T dG_c)[:3,:3]  (row 3 of dG_c is zero)
#pragma unroll
      for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int m = 0; m < 3; ++m)
          dR[3 * k + m] = Pm[k] * d[m] + Pm[4 + k] * d[4 + m] + Pm[8 + k] * d[8 + m];
      // dG_p += dG_c L_c^T,  L_c = [R | J_c - J_p; 0 0 0 1]
      const float t0 = Js[3 * i] - Js[3 * par], t1 = Js[3 * i + 1] - Js[3 * par + 1], t2 = Js[3 * i + 2] - Js[3 * par + 2];
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const float d0 = d[4 * r], d1 = d[4 * r + 1], d2 = d[4 * r + 2], d3 = d[4 * r + 3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
          sdG[12 * par + 4 * r + k][t] += d0 * q.R[3 * k] + d1 * q.R[3 * k + 1] + d2 * q.R[3 * k + 2] +
                                          d3 * (k == 0 ? t0 : (k == 1 ? t1 : t2));
        sdG[12 * par + 4 * r + 3][t] += d3;
      }
    }
    rodrigues_vjp(th, q, dR, dposes + ((size_t)f * 24 + i) * 3);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Skinning backward.  out_p = T_f(w(s_p)) [a_p;1] + trans_f with T_f = sum_j w_j A_{f,j}, s = tps (or ps), a = ps.
// Kernel 1, one CTA per fixed chunk of kBwdChunk points, one thread per point: dps / dtps per point, then the chunk's
// contributions to dA_f[j][r][c] = sum_p w_j g_r [a;1]_c and dtrans_f = sum_p g.  The frames present in the chunk get
// slots in order of first appearance; thread e of the CTA owns entry e of every slot record and walks the chunk's
// points in order, flushing its running sum into the record whenever the frame changes.  Kernel 2 sums, for each
// frame, the records of all chunks in chunk order (a fixed split over 32 thread rows, then those 32 partials in
// order).  Every sum therefore has one order that depends on P, the frames and nothing else: no atomics, and no
// dependence on the SM count.
constexpr int kBwdChunk = 256;
constexpr int kRecEntries = 291;   // 24 x 3 x 4 of dA (rows 0..2) + 3 of dtrans
constexpr int kRecStride = 292;

__host__ __device__ inline int64_t lbs_bwd_slots(int nf) { return nf < kBwdChunk ? nf : kBwdChunk; }

struct LbsBwdWorkspace {
  float* rec;          // [chunks][slots][kRecStride]
  int* slot_frame;     // [chunks][slots]
  int* nslots;         // [chunks]
};

__host__ inline size_t lbs_bwd_layout(int64_t P, int nf, size_t* off_frame, size_t* off_n) {
  const int64_t chunks = (P + kBwdChunk - 1) / kBwdChunk;
  const int64_t slots = lbs_bwd_slots(nf);
  size_t rec = (size_t)chunks * slots * kRecStride * sizeof(float);
  size_t fr = (size_t)chunks * slots * sizeof(int);
  *off_frame = rec;
  *off_n = (rec + fr + 15) & ~(size_t)15;
  return *off_n + (size_t)chunks * sizeof(int);
}

__global__ void __launch_bounds__(kBwdChunk) lbs_bwd_chunk_kernel(
    const float* __restrict__ ps, const float* __restrict__ tps, const float* __restrict__ A,
    const int64_t* __restrict__ batch_inds, int64_t ppf, int nf, Voxel vox,
    const float* __restrict__ grad_out, float* __restrict__ dps, float* __restrict__ dtps, LbsBwdWorkspace ws,
    int slots, int reduce, int64_t P) {
  __shared__ float s_w[kBwdChunk * 25];        // weights, padded row of 25 (conflict-free both ways)
  __shared__ float s_ga[kBwdChunk * 8];        // g0 g1 g2 | a0 a1 a2 1
  __shared__ int s_frame[kBwdChunk];
  __shared__ int s_slot[kBwdChunk];
  __shared__ unsigned char s_opens[kBwdChunk];
  __shared__ int s_warp_first[kBwdChunk / 32];
  const int t = threadIdx.x;
  const int64_t chunk = blockIdx.x;
  const int64_t p = chunk * kBwdChunk + t;
  const int n = (int)min((int64_t)kBwdChunk, P - chunk * kBwdChunk);
  int f = 0;
  if (t < n) {
    const float ax = ps[3 * p], ay = ps[3 * p + 1], az = ps[3 * p + 2];
    float sx = ax, sy = ay, sz = az;
    if (tps) { sx = tps[3 * p]; sy = tps[3 * p + 1]; sz = tps[3 * p + 2]; }
    const float g0 = grad_out[3 * p], g1 = grad_out[3 * p + 1], g2 = grad_out[3 * p + 2];
    f = frame_of(batch_inds, p, ppf, nf);
    const float* Af = A + (size_t)f * 24 * 16;
    const bool want_jac = tps ? (dtps != nullptr) : (dps != nullptr);
    float T[12];
    if (want_jac) {
      float J[9];
      lbs_blend_jac(vox, Af, sx, sy, sz, ax, ay, az, T, J);
      if (tps) {
#pragma unroll
        for (int j = 0; j < 3; ++j) dtps[3 * p + j] = J[j] * g0 + J[3 + j] * g1 + J[6 + j] * g2;
      } else {
#pragma unroll
        for (int i = 0; i < 3; ++i) {   // J + T[:3,:3], as lbs_forward_jac
          J[3 * i + 0] += T[4 * i + 0]; J[3 * i + 1] += T[4 * i + 1]; J[3 * i + 2] += T[4 * i + 2];
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) dps[3 * p + j] = J[j] * g0 + J[3 + j] * g1 + J[6 + j] * g2;
      }
    }
    // with tps, dps = T[:3,:3]^T g (the weights do not depend on ps), T blended from the sampled weights whichever
    // other outputs are requested, so that dropping one output changes no bit of another
    const bool split_dps = tps && dps;
    if (reduce || split_dps) {
      float w[24];
      sample_skin24(vox, sx, sy, sz, w);
      if (split_dps) {
        blend_bones(Af, w, T);
#pragma unroll
        for (int j = 0; j < 3; ++j) dps[3 * p + j] = T[j] * g0 + T[4 + j] * g1 + T[8 + j] * g2;
      }
      if (reduce) {
#pragma unroll
        for (int j = 0; j < 24; ++j) s_w[t * 25 + j] = w[j];
      }
    }
    float* ga = s_ga + t * 8;
    ga[0] = g0; ga[1] = g1; ga[2] = g2; ga[3] = ax; ga[4] = ay; ga[5] = az; ga[6] = 1.f;
  }
  if (!reduce) return;
  s_frame[t] = t < n ? f : -1;
  __syncthreads();
  // slots: the first point of each frame in the chunk opens a slot, numbered in order of appearance
  int first = t;
  if (t < n) {
    for (int j = 0; j < t; ++j)
      if (s_frame[j] == f) { first = j; break; }
  }
  const bool opens = t < n && first == t;
  s_opens[t] = opens ? 1 : 0;
  const unsigned ball = __ballot_sync(0xffffffffu, opens);
  if ((t & 31) == 0) s_warp_first[t >> 5] = __popc(ball);
  __syncthreads();
  if (t == 0) {
    int run = 0;
    for (int k = 0; k < kBwdChunk / 32; ++k) { const int c = s_warp_first[k]; s_warp_first[k] = run; run += c; }
    ws.nslots[chunk] = run;
  }
  __syncthreads();
  if (opens) {
    const int my_slot = s_warp_first[t >> 5] + __popc(ball & ((1u << (t & 31)) - 1u));
    s_slot[t] = my_slot;
    ws.slot_frame[chunk * slots + my_slot] = f;
  }
  __syncthreads();
  if (t < n && !opens) s_slot[t] = s_slot[first];
  __syncthreads();
  // thread e owns entry e of every record of this chunk; a run that starts at the point opening its slot stores,
  // later runs of the same frame add
  float* rec = ws.rec + (size_t)chunk * slots * kRecStride;
  for (int e = t; e < kRecEntries; e += kBwdChunk) {
    const bool is_dA = e < 288;
    const int j = is_dA ? e / 12 : 0, r = is_dA ? (e >> 2) % 3 : e - 288, c = is_dA ? (e & 3) : 3;
    float acc = 0.f;
    int start = 0;
    for (int i = 0; i < n; ++i) {
      if (s_slot[i] != s_slot[start]) {
        float* d = rec + (size_t)s_slot[start] * kRecStride + e;
        *d = s_opens[start] ? acc : *d + acc;
        acc = 0.f; start = i;
      }
      const float* ga = s_ga + i * 8;
      if (is_dA) acc = fmaf(s_w[i * 25 + j], ga[r] * ga[3 + c], acc);
      else acc += ga[r];
    }
    if (n > 0) {
      float* d = rec + (size_t)s_slot[start] * kRecStride + e;
      *d = s_opens[start] ? acc : *d + acc;
    }
  }
}

__global__ void __launch_bounds__(1024) lbs_bwd_reduce_kernel(LbsBwdWorkspace ws, int slots, int64_t chunks,
                                                               float* __restrict__ dA, float* __restrict__ dtrans) {
  __shared__ float part[32][33];
  const int f = blockIdx.x;
  const int x = threadIdx.x, y = threadIdx.y;
  const int e = blockIdx.y * 32 + x;
  const int64_t c0 = chunks * y / 32, c1 = chunks * (y + 1) / 32;
  float acc = 0.f;
  if (e < kRecEntries) {
    for (int64_t c = c0; c < c1; ++c) {
      const int ns = ws.nslots[c];
      const int* fr = ws.slot_frame + c * slots;
      for (int s = 0; s < ns; ++s)
        if (fr[s] == f) acc += ws.rec[((size_t)c * slots + s) * kRecStride + e];
    }
  }
  part[y][x] = acc;
  __syncthreads();
  if (y == 0 && e < kRecEntries) {
    float s = 0.f;
    for (int k = 0; k < 32; ++k) s += part[k][x];
    if (e < 288) {
      if (dA) dA[((size_t)f * 24 + e / 12) * 16 + (e % 12)] = s;
    } else if (dtrans) {
      dtrans[(size_t)f * 3 + (e - 288)] = s;
    }
  }
  if (y == 1 && blockIdx.y == 0 && dA && x < 24) {   // row 3 of every dA_f[j] is zero
    float* d = dA + ((size_t)f * 24 + x) * 16 + 12;
    d[0] = 0.f; d[1] = 0.f; d[2] = 0.f; d[3] = 0.f;
  }
}

static int lbs_check(const recmv_voxel_t* vox, int nf, int64_t P) {
  if (!vox || !vox->ws_cl) return RECMV_E_NULL;
  if (vox->D <= 0 || vox->H <= 0 || vox->W <= 0 || nf <= 0 || P < 0) return RECMV_E_SHAPE;
  if (((uintptr_t)vox->ws_cl & 15) != 0) return RECMV_E_SHAPE;  // float4 gathers
  return RECMV_OK;
}

}  // namespace recmv

using namespace recmv;

extern "C" int recmv_lbs_fwd(const float* ps, const float* tps, const float* A, const float* trans,
                             const int64_t* batch_inds, int64_t points_per_frame, int num_frames,
                             const recmv_voxel_t* vox, float* out, float* weights_out, int64_t P,
                             recmv_stream_t stream) {
  int s = lbs_check(vox, num_frames, P);
  if (s) return s;
  if (P == 0) return RECMV_OK;
  if (!ps || !A || !trans || !out) return RECMV_E_NULL;
  int g = stride_grid(P, 128, 8);
  lbs_fwd_kernel<<<g, 128, 0, (cudaStream_t)stream>>>(ps, tps, A, trans, batch_inds, points_per_frame,
                                                      num_frames, to_voxel(vox), out, weights_out, P);
  return launch_status();
}

extern "C" int recmv_lbs_inverse(const float* x_obs, const float* A, const float* trans,
                                 const int64_t* batch_inds, int64_t points_per_frame, int num_frames,
                                 const recmv_voxel_t* vox, float* x_can, uint8_t* valid, int64_t P,
                                 recmv_stream_t stream) {
  int s = lbs_check(vox, num_frames, P);
  if (s) return s;
  if (P == 0) return RECMV_OK;
  if (!x_obs || !A || !trans || !x_can) return RECMV_E_NULL;
  int g = stride_grid(P, 128, 8);
  lbs_inverse_kernel<<<g, 128, 0, (cudaStream_t)stream>>>(x_obs, A, trans, batch_inds, points_per_frame,
                                                          num_frames, to_voxel(vox), x_can, valid, P);
  return launch_status();
}

extern "C" int recmv_bone_matrices(const float* poses, const float* Js, const int* parents, const float* init_pose,
                                   float* G, float* A, int num_frames, recmv_stream_t stream) {
  if (num_frames < 0) return RECMV_E_SHAPE;
  if (num_frames == 0) return RECMV_OK;
  if (!poses || !Js || !parents || !G) return RECMV_E_NULL;
  bone_matrices_kernel<<<(num_frames + 63) / 64, 64, 0, (cudaStream_t)stream>>>(poses, Js, parents, init_pose, G, A,
                                                                                num_frames);
  return launch_status();
}

extern "C" int recmv_bone_matrices_backward(const float* poses, const float* Js, const int* parents,
                                            const float* init_pose, const float* G, const float* dG, const float* dA,
                                            float* dposes, int num_frames, recmv_stream_t stream) {
  if (num_frames < 0) return RECMV_E_SHAPE;
  if (num_frames == 0) return RECMV_OK;
  if (!poses || !Js || !parents || !G || !dposes) return RECMV_E_NULL;
  bone_matrices_bwd_kernel<<<(num_frames + kChainThreads - 1) / kChainThreads, kChainThreads, 0,
                             (cudaStream_t)stream>>>(poses, Js, parents, init_pose, G, dG, dA, dposes, num_frames);
  return launch_status();
}

extern "C" int recmv_lbs_backward_workspace_bytes(int64_t P, int num_frames, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  if (P < 0 || num_frames <= 0) return RECMV_E_SHAPE;
  size_t a, b;
  *bytes = lbs_bwd_layout(P, num_frames, &a, &b);
  return RECMV_OK;
}

extern "C" int recmv_lbs_backward(const float* ps, const float* tps, const float* A, const float* trans,
                                  const int64_t* batch_inds, int64_t points_per_frame, int num_frames,
                                  const recmv_voxel_t* vox, const float* grad_out, float* dps, float* dtps, float* dA,
                                  float* dtrans, void* workspace, int64_t P, recmv_stream_t stream) {
  (void)trans;   // the gradients do not depend on the translation
  int s = lbs_check(vox, num_frames, P);
  if (s) return s;
  if (!tps) dtps = nullptr;
  const int reduce = (dA || dtrans) ? 1 : 0;
  const int64_t chunks = (P + kBwdChunk - 1) / kBwdChunk;
  if (chunks > 0x7fffffff) return RECMV_E_RANGE;
  if (P > 0 && (dps || dtps || reduce) && (!ps || !A || !grad_out)) return RECMV_E_NULL;
  if (reduce && P > 0 && !workspace) return RECMV_E_NULL;
  if (((uintptr_t)workspace & 15) != 0) return RECMV_E_SHAPE;
  size_t off_frame, off_n;
  lbs_bwd_layout(P, num_frames, &off_frame, &off_n);
  LbsBwdWorkspace ws;
  ws.rec = (float*)workspace;
  ws.slot_frame = (int*)((char*)workspace + off_frame);
  ws.nslots = (int*)((char*)workspace + off_n);
  const int slots = (int)lbs_bwd_slots(num_frames);
  cudaStream_t st = (cudaStream_t)stream;
  if (P > 0 && (dps || dtps || reduce)) {
    lbs_bwd_chunk_kernel<<<(unsigned)chunks, kBwdChunk, 0, st>>>(ps, tps, A, batch_inds, points_per_frame,
                                                                  num_frames, to_voxel(vox), grad_out, dps, dtps, ws,
                                                                  slots, reduce, P);
    s = launch_status();
    if (s) return s;
  }
  if (reduce) {
    lbs_bwd_reduce_kernel<<<dim3((unsigned)num_frames, (kRecEntries + 31) / 32), dim3(32, 32), 0, st>>>(
        ws, slots, chunks, dA, dtrans);
    s = launch_status();
  }
  return s;
}

// Internal interface shared by the SIMT and tensor-core implementations of the fused MLP paths: the geometry and the
// packed weight blob of each network the engine runs.
#pragma once
#include "common.cuh"
#include "workspace.cuh"

namespace recmv {

// Where a tile's canonical points come from.
//   x != nullptr : canonical points [P,3] read from memory (ImplicitNetwork.forward)
//   x == nullptr : render mode -- point p = ray r * S + k, x_obs = cam + t_k dir_r, inverse LBS
struct PointSource {
  const float* x;
  // render mode
  const float* ray_dirs;
  const float* A;
  const float* trans;
  const int32_t* frame_of_ray;
  int64_t rays_per_frame;
  int num_frames;
  Voxel vox;
  float cam[3];
  float t_near, dt;  // t_k = t_near + (k + 0.5) * dt
  int S;
  float* out_xc;  // optional [P,3]
};

// 12 annealing weights, passed by value to kernels
struct PeWeights {
  float w[12];
};

// the annealing weights of the first `bands` frequency bands (two per band), zero beyond
inline PeWeights pe_weights(const float* pe_w, int bands = 6) {
  PeWeights pw;
  for (int i = 0; i < 12; ++i) pw.w[i] = i < 2 * bands ? pe_w[i] : 0.f;
  return pw;
}

// Geometry of the networks the tensor-core engine runs, read by its kernel and by the host code that packs and
// launches them.  The K dimension of every layer is cut into 64-wide blocks; a weight panel is [512 n][64 k] fp16
// (128-byte rows = one TMA swizzle row).  The panels of all layers are stacked, plane hi first then plane lo, so ONE
// 2-D tensor map [2 kPanels 512 rows, 64 columns] serves every weight box.
//   in(l), out(l): the widths of layer l;  nkb(l): its K blocks = panels, the first at panel pbase(l);
//   kb_at(l, i): the i-th K block (64 inputs) of layer l's input, 8 = the positional-encoding block;
//   ntiles(l, last): 128-wide output tiles of layer l (warpgroup g owns tiles 2 g and 2 g + 1; `last` =
//   TcParams::last_tiles);  kInFreeLayer: the layer after whose MMAs the tile input may be refilled;
//   src_col(l, pi, kk): the weight column behind input kk of panel pi of layer l (-1: zero padding);
//   wscale(l): factor folded into layer l's weights at pack time.
template <int kNet> struct Net;
// SDF network (model/network.py:135-141): PE block -> 512 x3 -> 473 -> [skip: +PE block] 512 x4 -> 257.  Layer 4 has 9
// panels: 8 for the 473 (+39 zero) hidden inputs and 1 for the positional-encoding inputs of the skip connection (its
// 1/sqrt2 folded into the weights).  The SIMT kernel also reads fp32 transposed copies [in(l)][npad32(l)].
template <> struct Net<0> {
  static constexpr int kLayers = 9, kPanels = 66, kInFreeLayer = 4;
  static constexpr int kPE = 39;        // 3 + 3*2*6
  static constexpr int kSkipOut = 473;  // layer 3 out = 512 - 39
  static constexpr int kOutDim = 257;   // 1 + 256
  __host__ __device__ static constexpr int in(int l) { return l == 0 ? kPE : 512; }
  __host__ __device__ static constexpr int out(int l) { return l == 3 ? kSkipOut : (l == 8 ? kOutDim : 512); }
  __host__ __device__ static constexpr int nkb(int l) { return l == 0 ? 1 : (l == 4 ? 9 : 8); }
  __host__ __device__ static constexpr int pbase(int l) { return l == 0 ? 0 : (l <= 4 ? 1 + 8 * (l - 1) : 34 + 8 * (l - 5)); }
  __host__ __device__ static constexpr int kb_at(int l, int i) { return l == 0 ? 8 : (l == 4 ? (i == 0 ? 8 : i - 1) : i); }
  __host__ __device__ static constexpr int ntiles(int l, int last) { return l == 8 ? last : 4; }
  __host__ __device__ static constexpr int src_col(int l, int pi, int kk) {
    return l == 0 ? (kk < kPE ? kk : -1)
                  : l == 4 ? (pi < 8 ? (pi * 64 + kk < kSkipOut ? pi * 64 + kk : -1) : (kk < kPE ? kSkipOut + kk : -1))
                           : pi * 64 + kk;
  }
  __host__ __device__ static constexpr float wscale(int l) { return l == 4 ? 0.70710678118654752440f : 1.f; }
  static constexpr int npad32(int l) { return l == 8 ? 264 : 512; }
};
// The ReLU networks: [input row of kIn columns, zero-padded to kInKb K blocks] -> 512 x4 (ReLU) -> 3.  The input row is
// written into the activation buffer itself, so every K block is an activation block.
template <int kIn, int kInKb> struct ReluNet {
  static constexpr int kLayers = 5, kPanels = kInKb + 32, kInFreeLayer = 4;
  __host__ __device__ static constexpr int in(int l) { return l == 0 ? kIn : 512; }
  __host__ __device__ static constexpr int out(int l) { return l == 4 ? 3 : 512; }
  __host__ __device__ static constexpr int nkb(int l) { return l == 0 ? kInKb : 8; }
  __host__ __device__ static constexpr int pbase(int l) { return l == 0 ? 0 : kInKb + 8 * (l - 1); }
  __host__ __device__ static constexpr int kb_at(int, int i) { return i; }
  __host__ __device__ static constexpr int ntiles(int l, int) { return l == 4 ? 1 : 4; }
  __host__ __device__ static constexpr int src_col(int l, int pi, int kk) { return pi * 64 + kk < in(l) ? pi * 64 + kk : -1; }
  __host__ __device__ static constexpr float wscale(int) { return 1.f; }
};
// MLPTranslator (model/Deformer.py:141-206): [PE(39) | cond(128) | 0 x25] = 3 K blocks
template <> struct Net<1> : ReluNet<167, 3> {};
// RenderingNetwork_view_norm, mode 'idr' (model/RenderNet.py:59-96): [p 3 | PE4(v) 27 | n 3 | feat 256 | 0 x31] = 5 K
// blocks, then tanh
template <> struct Net<2> : ReluNet<289, 5> {};

// The packed weight blob of network kNet (recmv_*_pack_weights), every part 1 KiB-aligned:
//   bias:   [kLayers][512] fp32 padded with zeros; the SDF adds a second such plane of b * kSoftplusLog2Scale
//   w32[l]: SDF only, the SIMT kernel's fp32 [in(l)][npad32(l)] transposed copy of layer l
//   panels: [2 planes][kPanels][512][64] fp16, hi and lo of 1024 w
struct PackedBlob {
  float* bias;
  float* w32[Net<0>::kLayers];
  __half* panels;
};
template <int kNet>
PackedBlob blob_layout(Carve& c) {
  using N = Net<kNet>;
  PackedBlob b = {};
  b.bias = c.take<float>((kNet == 0 ? 2 : 1) * N::kLayers * 512, 1024);
  if constexpr (kNet == 0)
    for (int l = 0; l < N::kLayers; ++l) b.w32[l] = c.take<float>((size_t)N::in(l) * N::npad32(l), 1024);
  b.panels = c.take<__half>((size_t)2 * N::kPanels * 512 * 64, 1024);
  return b;
}

// Canonical point of global sample index p; returns false when the inverse warp is singular.
__device__ __forceinline__ bool fetch_point(const PointSource& src, int64_t p, float& cx, float& cy,
                                            float& cz) {
  if (src.x) {
    cx = __ldg(src.x + 3 * p); cy = __ldg(src.x + 3 * p + 1); cz = __ldg(src.x + 3 * p + 2);
    return true;
  }
  int64_t r = p / src.S;
  int k = (int)(p - r * src.S);
  float t = src.t_near + ((float)k + 0.5f) * src.dt;
  float dx = __ldg(src.ray_dirs + 3 * r), dy = __ldg(src.ray_dirs + 3 * r + 1), dz = __ldg(src.ray_dirs + 3 * r + 2);
  float ox = src.cam[0] + t * dx, oy = src.cam[1] + t * dy, oz = src.cam[2] + t * dz;
  int64_t f = src.frame_of_ray ? (int64_t)__ldg(src.frame_of_ray + r)
                               : (src.rays_per_frame > 0 ? r / src.rays_per_frame : 0);
  if (f < 0) f = 0;
  if (f >= src.num_frames) f = src.num_frames - 1;
  bool ok = inverse_lbs_point(src.vox, src.A + (size_t)f * 384, src.trans + 3 * f, ox, oy, oz, cx, cy, cz);
  if (src.out_xc) { src.out_xc[3 * p] = cx; src.out_xc[3 * p + 1] = cy; src.out_xc[3 * p + 2] = cz; }
  return ok;
}

constexpr float kInvalidSdf = 1e10f;

// implemented in sdf_mlp_simt.cu / sdf_mlp_tc.cu
int simt_sdf_forward(const PointSource& src, const void* packed, const PeWeights& pw, float* out_sdf,
                     float* out_feat, int64_t P, cudaStream_t st);
int tc_sdf_forward(const PointSource& src, const void* packed, const PeWeights& pw, float* out_sdf,
                   float* out_feat, int64_t P, int passes, cudaStream_t st, const int* P_dev = nullptr);

// the per-device status record (mapped pinned host memory) the tensor-core kernels report into: bounded-wait
// time-outs (code 1) and fp16 operand-range violations (code 2); see recmv_check_async_errors
int device_status_record(void** out);

// value + input gradient in one forward-mode launch (tensor-core path only)
int tc_sdf_forward_grad(const float* x, const void* packed, const PeWeights& pw, float* out_sdf, float* out_feat,
                        float* out_grad, int64_t P, int passes, cudaStream_t st);

}  // namespace recmv

/* recmv_b200.h -- C ABI of the B200-native REC-MV hot path (librecmv_b200.so).
 *
 * Every entry point takes raw DEVICE pointers (unless a parameter says "host"), plain sizes and a
 * cudaStream_t passed as void*.  No torch types.  Return value: 0 = ok, negative = argument error
 * (RECMV_E_*), positive = cudaError_t raised by the launch.  All kernels run on the caller's stream
 * and no entry point waits for the work it queued (marching cubes copies its case tables to the
 * device once, on its first call per device).  Nothing here allocates result storage:
 * results of data-dependent size go into caller buffers of a given capacity, and the counts and an
 * overflow flag are written to device memory (re-run with larger buffers when the flag is set).
 *
 * Each block cites the reference interface (path:line under /root/reference) it replaces.
 */
#ifndef RECMV_B200_H_
#define RECMV_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* recmv_stream_t; /* cudaStream_t */

#if defined(__GNUC__)
#define RECMV_API __attribute__((visibility("default")))
#else
#define RECMV_API
#endif

enum {
  RECMV_OK = 0,
  RECMV_E_NULL = -1,      /* required pointer is NULL            */
  RECMV_E_DTYPE = -2,     /* dtype / layout / mode flag unknown  */
  RECMV_E_SHAPE = -3,     /* non-positive or inconsistent extent */
  RECMV_E_RANGE = -4,     /* size exceeds an implementation limit (e.g. > 2^26 MC vertices) */
  RECMV_E_UNSUPPORTED = -5,
  RECMV_E_DEVICE = -6     /* a tensor-core launch aborted on a bounded mbarrier wait (see recmv_check_async_errors) */
};

enum { RECMV_F32 = 0, RECMV_F64 = 1 };
enum { RECMV_LAYOUT_NCDHW = 0, RECMV_LAYOUT_NDHWC = 1 };

/* SDF-MLP arithmetic.  All modes accumulate in fp32.
 *   FP32_SIMT : fp32 FMA on CUDA cores (exact-fp32 verification mode, slow)
 *   TC_F16X3  : tcgen05 kind::f16, operands split a = hi + lo (fp16 each), 3 MMAs per product
 *               (hi*hi + lo*hi + hi*lo) -> ~2^-21 relative per product; meets the 1e-4 parity bar
 *   TC_F16X1  : tcgen05 kind::f16 single pass (11-bit operands, like the TF32 the reference ran
 *               with on Ampere); ~1e-3, NOT parity grade                                          */
enum { RECMV_MLP_FP32_SIMT = 0, RECMV_MLP_TC_F16X3 = 1, RECMV_MLP_TC_F16X1 = 2 };

RECMV_API int recmv_version(void);
RECMV_API const char* recmv_error_string(int status);
/* number of kernels this library has launched since load (bench.py's gpu_launches) */
RECMV_API int64_t recmv_launch_count(void);

/* ---- A6: FastMinv.Fast3x3Minv / Fast3x3Minv_backward --------------------------------------
 * replaces FastMinv/M3x3Inv.cpp:12-59 (pybind) + Matrix3x3InvKernels.cu:21-142.
 * ms/invs/grads/outs: [n,3,3] contiguous; ok: [n] bytes (1 = invertible, |det| >= 1e-4).        */
RECMV_API int recmv_minv3x3_fwd(const void* ms, void* invs, uint8_t* ok, int64_t n, int dtype,
                      recmv_stream_t stream);
RECMV_API int recmv_minv3x3_bwd(const void* grads, const void* invs, void* outs, int64_t n, int dtype,
                      recmv_stream_t stream);

/* ---- K4-K6: GridSamplerMine.forward / backward / dbackward --------------------------------
 * replaces MCAcc/cuda/GridSamplerMine.cpp:75-103 + GridSamplerMineKernel.cu:160-1022.
 * trilinear, border padding, align_corners=False.  input [N,C,D,H,W] (layout NCDHW) or
 * [N,D,H,W,C] (NDHWC, the coalesced internal layout); grid [N,P,3] (x->W, y->H, z->D);
 * output / grad_out / gg_out [N,C,P].
 * bwd : grad_input may be NULL (skipped -- the skinning voxel is a frozen buffer); otherwise it
 *       must be zero-filled by the caller and has the layout of `input`.
 * bwd2: cotangents gg_input (layout of input, may be NULL = zeros) and gg_grid [N,P,3];
 *       outputs g_input (may be NULL; else zero-filled), g_grid [N,P,3], gg_out [N,C,P].         */
RECMV_API int recmv_gridsample3d_fwd(const void* input, const void* grid, void* output, int N, int C, int D,
                           int H, int W, int64_t P, int dtype, int layout, recmv_stream_t stream);
RECMV_API int recmv_gridsample3d_bwd(const void* input, const void* grid, const void* grad_out,
                           void* grad_input, void* grad_grid, int N, int C, int D, int H, int W,
                           int64_t P, int dtype, int layout, recmv_stream_t stream);
RECMV_API int recmv_gridsample3d_bwd2(const void* gg_input, const void* gg_grid, const void* input,
                            const void* grid, const void* grad_out, void* g_input, void* g_grid,
                            void* gg_out, int N, int C, int D, int H, int W, int64_t P, int dtype,
                            int layout, recmv_stream_t stream);
/* [C,D,H,W] -> [D,H,W,C] copy (private cache of LBSkinner.ws) */
RECMV_API int recmv_voxel_to_channels_last(const float* src, float* dst, int C, int D, int H, int W,
                                 recmv_stream_t stream);

/* ---- skinning-voxel construction: compute_lbswField / smooth_weights ------------------------
 * replaces model/Deformer.py:533-591 and utils/LBSWsmpl.py:2-51.  Setup work (once per body), not per step.
 * knn_blend: voxel centre (x,y,z) of cell (i_W,i_H,i_D) is c/res + (1/res)/2 (align_corners = 0) or c/(res-1)
 *   (align_corners != 0, every extent >= 2), times (bmax - bmin) plus bmin, all in fp32 as the reference rounds.
 *   verts [V,3] f32 (V <= 14336, staged in shared memory), vert_ws [V,C] f32 with C == 24, bmin / bmax host [3].
 *   The k nearest vertices (1 <= k <= 32, k <= V) by fp32 distance sqrt(fma(dz,dz,fma(dy,dy,dx*dx))); on
 *   exactly equal distances the LOWER vertex index wins (torch.topk leaves that case undefined).  Each distance is
 *   clamped to [1e-4, 1] and inverted, the inverses are normalised, and the 24 weights are blended in neighbour
 *   order (nearest first).  out_cl [D,H,W,24] f32, voxel (z H + y) W + x; out_idx [D*H*W, k] int32 (nearest
 *   first) or NULL.  No atomics: bit-identical from run to run.
 * smooth: `times` Jacobi passes of the 6-neighbour stencil on channels-last buffers: interior voxels get
 *   mean = (z+ + z- + y+ + y- + x+ + x-) / 6 (summed in that order, true division), w' = (w - mean) * 0.7 + mean;
 *   boundary voxels (and every voxel of a grid with an extent below 3) keep their values; then every voxel is
 *   divided by its sequential channel sum.  No FMA contraction.  times == 0 leaves the values as they are
 *   (the reference's loop does not run).  Afterwards, if zero_below > 0, values below it become 0 with no
 *   renormalisation (LBSWsmpl.py:10).  buf_a holds the input [D,H,W,24] and is overwritten; buf_b is scratch of
 *   the same size (may be NULL when times <= 1).  Outputs: out_ncdhw [24,D,H,W] (the reference's `ws`) and
 *   out_cl [D,H,W,24], bit-identical to recmv_voxel_to_channels_last(out_ncdhw).  buf_a, buf_b, out_cl must be
 *   distinct and 16-byte aligned.                                                                             */
RECMV_API int recmv_lbsw_knn_blend(const float* verts, const float* vert_ws, int V, int C, const float bmin[3] /*host*/,
                                   const float bmax[3] /*host*/, int W, int H, int D, int align_corners, int k,
                                   float* out_cl, int32_t* out_idx, recmv_stream_t stream);
RECMV_API int recmv_lbsw_smooth(float* buf_a, float* buf_b, int D, int H, int W, int times, float zero_below,
                                float* out_ncdhw, float* out_cl, recmv_stream_t stream);

/* ---- A12: MCGpu.mc_gpu --------------------------------------------------------------------
 * replaces MCGpu/MCGpu.cpp:20-56 + CudaKernels.cu:316-521.  sdf [NX,NY,NZ] f32, z fastest.
 * Deterministic: vertices and faces come out in the order a sequential sweep of the reference
 * kernel (cell index ascending) would create them; faces int64 with the reference's reversed
 * winding; vertices referenced on the far boundary planes get index -1 exactly as the reference.
 * recmv_mc_run is one call with NO host synchronisation (the reference blocks on a cudaMemcpy
 * between its two kernels, MCGpu/CudaKernels.cu:628): classify + count + scan + emit of
 * verts [V,3] = v*step+origin and faces [F,3] into caller-provided buffers of capacity cap_verts /
 * cap_faces rows, with scratch of recmv_mc_scratch_bytes.  counts (DEVICE, int32[4]) receives
 * {V, F, overflow, 0}; overflow != 0 = a buffer was too small: rows that fit are valid, re-run with
 * V / F rows.  Rows beyond V / F are left untouched.  V >= 2^25 exceeds the packed vertex ids:
 * overflow is then set whatever the capacity.                                                    */
RECMV_API int recmv_mc_scratch_bytes(int NX, int NY, int NZ, size_t* bytes /*host*/);
RECMV_API int recmv_mc_run(const float* sdf, int NX, int NY, int NZ, float iso, void* scratch,
                 const float step[3] /*host*/, const float origin[3] /*host*/, float* verts, int64_t cap_verts,
                 int64_t* faces, int64_t cap_faces, int32_t* counts /*device*/, recmv_stream_t stream);

/* ---- A5 / A5': LBSkinner.forward and the inverse warp ----------------------------------------
 * replaces model/Deformer.py:359-445 (+342-355, GridSamplerMine3dFunction at :421).
 * ws_cl: skinning voxel channels-last [D,H,W,24] f32; A [F,24,4,4] row-major bone matrices
 * (G*init_pose, computed on the host side); trans [F,3] (already + extra_trans);
 * batch_inds [P] int64 or NULL (then frame = point / points_per_frame).
 * fwd: out = (sum_j w_j(tp) A_j) [p;1] + trans;  tps may be NULL (= ps).
 *      weights_out [P,24] optional (NULL to skip).
 * inverse: x_c = M^-1 (x_obs - trans - t), [M|t] = sum_j w_j(x_obs) A_j ; valid=0 and x_c=0 when
 *      |det M| < 1e-4 (FastMinv rule, Matrix3x3InvKernels.cu:40).                                */
typedef struct {
  const float* ws_cl;
  int D, H, W;
  float center[3];
  float extend; /* nps = 2 (p - center) / extend   (Deformer.py:342-355) */
} recmv_voxel_t;

RECMV_API int recmv_lbs_fwd(const float* ps, const float* tps, const float* A, const float* trans,
                  const int64_t* batch_inds, int64_t points_per_frame, int num_frames,
                  const recmv_voxel_t* vox /*host*/, float* out, float* weights_out, int64_t P,
                  recmv_stream_t stream);
RECMV_API int recmv_lbs_inverse(const float* x_obs, const float* A, const float* trans,
                      const int64_t* batch_inds, int64_t points_per_frame, int num_frames,
                      const recmv_voxel_t* vox /*host*/, float* x_can, uint8_t* valid, int64_t P,
                      recmv_stream_t stream);

/* Bone matrices of the SMPL kinematic chain: replaces the 24-joint python loop of model/Deformer.py:372-405 (and
 * posedSkeleton, :305-326) when no autograd graph is needed.  poses [F,24,3] axis-angle, Js [24,3], parents [24] int32
 * (device), init_pose [24,4,4] or NULL (Deformer.py:397-404).  G [F,24,4,4] = chained joint transforms (always
 * written; G[:,:,:3,3] is the posed skeleton), A [F,24,4,4] = G . init_pose (may be NULL).                       */
RECMV_API int recmv_bone_matrices(const float* poses, const float* Js, const int* parents, const float* init_pose,
                        float* G, float* A, int num_frames, recmv_stream_t stream);

/* VJP of recmv_bone_matrices (the autograd path of LBSkinner.bone_matrices / posedSkeleton when poses require grad).
 * G [F,24,4,4] is what recmv_bone_matrices wrote for these poses.  dG [F,24,4,4] (cotangent of G, e.g. of the posed
 * skeleton) and dA [F,24,4,4] (cotangent of A) may each be NULL; row 3 of either is ignored.  init_pose as in the
 * forward.  Writes dposes [F,24,3].  One thread per frame, no atomics: deterministic.                              */
RECMV_API int recmv_bone_matrices_backward(const float* poses, const float* Js, const int* parents,
                                           const float* init_pose, const float* G, const float* dG, const float* dA,
                                           float* dposes, int num_frames, recmv_stream_t stream);

/* Backward of recmv_lbs_fwd for the training step (pose / translation / point gradients).  Same inputs as the
 * forward (trans is accepted for symmetry and may be NULL: no gradient depends on it) plus grad_out [P,3].  Outputs,
 * each may be NULL:
 *   dps    [P,3]       = J^T g (J = d out / d ps, weights resampled at ps) when tps is NULL, else T[:3,:3]^T g
 *   dtps   [P,3]       the weight term, only when tps is given (ignored otherwise)
 *   dA     [F,24,4,4]  dA_f[j][r][c] = sum over the points of frame f of w_j g_r [ps;1]_c; row 3 is zero
 *   dtrans [F,3]       sum over the points of frame f of g
 * Frames as in the forward (batch_inds, unsorted allowed, or points_per_frame; clamped to [0, F)).  dA / dtrans are
 * reduced over fixed chunks of 256 points and then over the chunks in order, so they are bit-identical from run to run
 * and on any GPU.  workspace: recmv_lbs_backward_workspace_bytes(P, F) bytes, 16-byte aligned, needed when dA or
 * dtrans is requested (it may be NULL when P == 0); it carries nothing between calls.                              */
RECMV_API int recmv_lbs_backward_workspace_bytes(int64_t P, int num_frames, size_t* bytes /*host*/);
RECMV_API int recmv_lbs_backward(const float* ps, const float* tps, const float* A, const float* trans,
                                 const int64_t* batch_inds, int64_t points_per_frame, int num_frames,
                                 const recmv_voxel_t* vox /*host*/, const float* grad_out, float* dps, float* dtps,
                                 float* dA, float* dtrans, void* workspace, int64_t P, recmv_stream_t stream);

/* VJP of the point outputs of recmv_lbs_backward (the train-phase Jacobians of utils.compute_Jacobian, differentiated
 * again by the loss).  V(ps, tps, A, g) = (dps, dtps) of recmv_lbs_backward: dps = (T3 + Jw)^T g when tps is NULL
 * (s = ps), else dps = T3^T g and dtps = Jw^T g, with T3 = sum_b w_b(s) A_b[:3,:3] and Jw = sum_b (A_b [ps;1]) (x)
 * grad w_b(s).  Cotangents: cot_ps u [P,3] of dps and cot_tps v [P,3] of dtps (tps form only; v' = u when tps is
 * NULL).  At least one is needed; a missing one is zero.  Outputs, each may be NULL, and dropping one changes no bit
 * of another:
 *   d_grad_out [P,3]       = T3 u + Jw v'
 *   dps        [P,3]       = sum_b (grad w_b . v') A_b3^T g, plus dtps's term when tps is NULL
 *   dtps       [P,3]       = sum_b (g^T A_b3 u) grad w_b + sum_b (g . A_b [ps;1]) H_b v'   (H_b: Hessian of w_b; a
 *                            clamped axis contributes zero, as to the first derivative)
 *   dA         [F,24,4,4]  dA_f[b] rows 0..2 = sum over the points of frame f of g (w_b [u;0] + (grad w_b . v') [ps;1])^T;
 *                          row 3 is zero
 * Frames, the workspace (recmv_lbs_backward_workspace_bytes, needed for dA) and the deterministic chunked reduce are
 * those of recmv_lbs_backward.  cot_tps or dtps without tps is rejected.                                           */
RECMV_API int recmv_lbs_vjp_backward(const float* ps, const float* tps, const float* A, const int64_t* batch_inds,
                                     int64_t points_per_frame, int num_frames, const recmv_voxel_t* vox /*host*/,
                                     const float* grad_out, const float* cot_ps, const float* cot_tps,
                                     float* d_grad_out, float* dps, float* dtps, float* dA, void* workspace, int64_t P,
                                     recmv_stream_t stream);

/* ---- A1+A2: Embedder + ImplicitNetwork.forward -------------------------------------------------
 * replaces model/Embedder.py:43-50 + model/network.py:89-119 (+ utils/utils.py:40-46 weights).
 * Network shape is the reference's getTmpSdf: PE(6) 39 -> 512 x3 -> 473 (+39 skip)/sqrt2 -> 512 x4
 * -> 257, softplus(beta=100, threshold 20) on layers 0..7.
 * pack: W_l [out_l, in_l] row-major fp32 EFFECTIVE weights (weight-norm already applied by the host
 * shim), concatenated l = 0..8; b likewise.  `packed` (recmv_sdf_packed_bytes() bytes) holds the
 * fp32 copy used by FP32_SIMT and the padded fp16 hi/lo K-major planes the TMA descriptors read.  */
RECMV_API size_t recmv_sdf_packed_bytes(void);
RECMV_API int recmv_sdf_pack_weights(const float* W_all, const float* b_all, void* packed,
                           recmv_stream_t stream);
/* x [P,3] canonical points; pe_w [12] host (annealing weights); out_sdf [P]; out_feat [P,256] or
 * NULL.                                                                                           */
RECMV_API int recmv_sdf_mlp_fwd(const float* x, const void* packed, const float* pe_w /*host*/,
                      float* out_sdf, float* out_feat, int64_t P, int mode, recmv_stream_t stream);
/* the same with the point count read from DEVICE memory: *count_dev points (clamped to `capacity`, for which the launch
 * is sized) -- consumer of device-built worklists (recmv_c2f_refine, recmv_c2f_mark_conflicts).  TC modes only.  */
RECMV_API int recmv_sdf_mlp_fwd_counted(const float* x, const void* packed, const float* pe_w /*host*/, float* out_sdf,
                              float* out_feat, int64_t capacity, const int* count_dev, int mode,
                              recmv_stream_t stream);

/* ---- A2/A3 training path: what `loss.backward()` (train.py:325) runs through model/network.py:89-119 ---------
 * (and through Deformer.py:171-206 / RenderNet.py:59-96 -- the entry points below are generic over the layer list).
 *
 * recmv_pe_forward: positional encoding rows (model/Embedder.py:43-50 with the annealing weights pe_w [2*bands] host)
 *   written as a saved layer input: out[p*ld + e], e < 3 + 6*bands; out2 (optional) gets the same row.
 *
 * recmv_pe_backward: dx [P,3] (+)= (d PE / d x)^T (g + g2): g [P][ldg] cotangent of the 3 + 6*bands encoding
 *   (model/Embedder.py:43-50 order), g2 optional second cotangent of the same encoding, pe_w [2*bands] host.       */
RECMV_API int recmv_pe_forward(const float* x, const float* pe_w /*host*/, int bands, float* out, int64_t ld, float* out2,
                     int64_t ld2, int64_t P, recmv_stream_t stream);
RECMV_API int recmv_pe_backward(const float* x, const float* g, int64_t ldg, const float* g2, int64_t ldg2,
                      const float* pe_w /*host*/, int bands, float* dx, int accumulate, int64_t P,
                      recmv_stream_t stream);

/* Layer GEMMs (3 fp16 MMAs per product, fp32 accumulation): operands as fp16 hi / lo PLANES in HBM, fed by TMA
 * (csrc/gemm3_tma.cu) -- every tensor a later GEMM consumes is written in consumable form by its producer, the main
 * loop converts nothing.
 *  recmv_split_planes      : fp32 [R][C] (row stride ld) -> planes hi = fp16(s v), lo = fp16(s v - hi), s = scale * (*scale_dev
 *                            if given); transpose != 0 writes [C][R].  ldp = plane row stride in elements (multiple of 8, plane
 *                            base 16-byte aligned).  Weights: scale 1024 ([out][in] for the forward, transposed for
 *                            backward-data); the loss cotangent: scale 64 with scale_dev = the call's dyn scale.
 *  recmv_pe_forward_planes : recmv_pe_forward + the planes (scale 64) of the same rows.
 *  recmv_mlp_layer_planes  : one layer.  mode 4 / 5 / 6 = forward with none / softplus(100) / ReLU:
 *                              Y = act(scale * (A . B^T) + bias);
 *                            mode 0 / 1 / 2 = backward-data with none / softplus' / ReLU':
 *                              Y = scale * (A . B^T) * act'(saved_input); columns >= split -> Y2 without the derivative.
 *                            A planes [M][lda_p] hold 64 (x dyn if a_has_dyn) * value, B planes [N][ldb_p] 1024 * weight; K
 *                            columns of each are used.  Y fp32 [M][ldy] (+ Y2); y_hi / y_lo (optional) receive the planes
 *                            of Y's columns < split, scaled 64 (x dyn if planes_with_dyn) -- the next GEMM's A operand.      */
RECMV_API int recmv_split_planes(const float* in, int64_t ld, int64_t R, int C, float scale, const float* scale_dev /*device*/,
                       int transpose, void* hi, void* lo, int64_t ldp, recmv_stream_t stream);
RECMV_API int recmv_pe_forward_planes(const float* x, const float* pe_w /*host*/, int bands, float* out, int64_t ld,
                            void* out_hi, void* out_lo, int64_t ldp, int64_t P, recmv_stream_t stream);
RECMV_API int recmv_mlp_layer_planes(const void* a_hi, const void* a_lo, int64_t lda_p, const void* b_hi, const void* b_lo,
                           int64_t ldb_p, int64_t M, int N, int K, int mode, const float* bias, const float* saved_input,
                           int64_t lds, float scale, const float* dyn_scale /*device*/, int a_has_dyn, int split, float* Y,
                           int64_t ldy, float* Y2, int64_t ldy2, void* y_hi, void* y_lo, int64_t ldyp, int planes_with_dyn,
                           recmv_stream_t stream);

/* Weight gradient from the same planes, no transposed copies (wgmma reads the row-major planes as MN-major operands):
 *   dW [out_dim][in_dim] = scale * G^T X,  g planes [P][ldg_p] = 64 * dyn * g (columns < out_dim), x planes [P][ldx_p] = 64 * x.
 * The sample range is split over the SMs, partial tiles are summed in a fixed order (deterministic).  db [out_dim] (optional)
 * = sum_p g[p][:] = the bias gradient, from one more product of the G tiles with a tile of ones in the same launch.  workspace:
 * device fp32, recmv_mlp_wgrad_workspace_floats() elements, reusable across calls on one stream.
 *   recmv_colsum: out[c] = sum_r g[r][c] (the bias gradient from the fp32 cotangent); partial = scratch of 128 * cols floats. */
RECMV_API size_t recmv_mlp_wgrad_workspace_floats(void);
RECMV_API int recmv_mlp_wgrad_planes(const void* g_hi, const void* g_lo, int64_t ldg_p, const void* x_hi, const void* x_lo,
                                     int64_t ldx_p, int64_t P, int out_dim, int in_dim, float scale,
                                     const float* dyn_scale /*device*/, float* workspace, float* dW, float* db /*or NULL*/,
                                     recmv_stream_t stream);
RECMV_API int recmv_colsum(const float* g, int64_t ld, int64_t rows, int cols, float* partial, float* out,
                           recmv_stream_t stream);
/* (f4) element-wise steps of the second-order pass between two plane GEMMs (recmv_b200/second_order.py), each one launch that
 * also writes the next GEMM's A planes (scaled plane_scale [x *scale_dev]):
 *   softplus_tangent: u = s tz (fp32 + planes), inj = 100 (1 - s) h tz,  s = 1 - exp(-100 a)  (softplus_100' from the saved
 *                     output a; h = first-order cotangent at the same pre-activation)
 *   add_split:        y += addend (in place), planes of y                                                                   */
RECMV_API int recmv_softplus_tangent_planes(const float* tz, int64_t ldt, const float* a, int64_t lda, const float* h,
                                            int64_t ldh, int64_t rows, int cols, float plane_scale, float* u, int64_t ldu,
                                            void* u_hi, void* u_lo, int64_t ldp, float* inj, int64_t ldi,
                                            recmv_stream_t stream);
RECMV_API int recmv_add_split_planes(float* y, int64_t ldy, const float* addend, int64_t lda, int64_t rows, int cols,
                                     float scale, const float* scale_dev, void* y_hi, void* y_lo, int64_t ldp,
                                     recmv_stream_t stream);

/* ---- A3: sdf and its input gradient (ImplicitNetwork.gradient, model/network.py:121-133; the
 * autograd.grad(sdf, p) of utils/FindSurfacePs.py:176 and OptimGarmentNetwork.py:1171,3192) --------------
 * One forward-mode launch of the tensor-core kernel: every point occupies four tile rows (value and the three
 * directional derivatives), no activations are stored and no transposed weights are needed.
 * out_grad [P,3] = d sdf / d x.  TC modes only (RECMV_E_UNSUPPORTED otherwise).                            */
RECMV_API int recmv_sdf_mlp_fwd_grad(const float* x, const void* packed, const float* pe_w /*host*/,
                           float* out_sdf, float* out_feat, float* out_grad, int64_t P, int mode,
                           recmv_stream_t stream);

/* ---- A4 + A5: MLPTranslator.forward followed by LBSkinner.forward (CompositeDeformer) in ONE launch ------
 * replaces model/Deformer.py:171-206 (PE ++ cond[batch] -> 512 x4 ReLU -> 3, p + offset) and :406-445.
 * Same tensor-core engine as the SDF network (3 input K blocks, 4 hidden layers, 32-wide tail tile).
 * pack: W_l [out,in] row-major fp32, l = 0..4 concatenated (167->512, 512->512 x3, 512->3); b likewise.
 * conds [F,128]; batch_inds [P] i64 or NULL (frame = p / points_per_frame); pe_w [12] host.
 * Outputs (each may be NULL): out_translated = p + offset, out_offset, out_posed = LBS(p + offset) (needs
 * A [F,24,4,4], trans [F,3] (+extra_trans) and the channels-last voxel).  TC modes only.                   */
RECMV_API size_t recmv_translator_packed_bytes(void);
RECMV_API int recmv_translator_pack_weights(const float* W_all, const float* b_all, void* packed,
                                  recmv_stream_t stream);
RECMV_API int recmv_deformer_fwd(const float* ps, const float* conds, const int64_t* batch_inds,
                       int64_t points_per_frame, int num_frames, const void* packed,
                       const float* pe_w /*host*/, const float* A, const float* trans,
                       const recmv_voxel_t* vox /*host, may be NULL*/, float* out_translated,
                       float* out_offset, float* out_posed, int64_t P, int mode, recmv_stream_t stream);

/* Forward-mode variant of recmv_deformer_fwd (A7, utils/utils.py:133-156 compute_Jacobian without autograd): every
 * point travels as 4 tile rows (value + 3 tangents); out_jac [P,9] row-major, J[i][j] = d out_i / d p_j where
 * `out` is out_posed when the skeleton/voxel are given, else out_translated.  The skinning weights' own
 * dependence on the point (d w / d q, sampler backward semantics incl. zero gradient on clamped axes) is included. */
RECMV_API int recmv_deformer_fwd_jac(const float* ps, const float* conds, const int64_t* batch_inds,
                           int64_t points_per_frame, int num_frames, const void* packed,
                           const float* pe_w /*host*/, const float* A, const float* trans,
                           const recmv_voxel_t* vox /*host, may be NULL*/, float* out_translated,
                           float* out_offset, float* out_posed, float* out_jac, int64_t P, int mode,
                           recmv_stream_t stream);

/* ---- A8: RenderingNetwork_view_norm.forward, mode 'idr' (model/RenderNet.py:59-96) in one launch -----------------
 * cat[points 3 | PE4(view_dirs) 27 | normals 3 | feature_vectors 256] = 289 -> 512 x4 ReLU -> 3 -> tanh.
 * pack: effective (weight-norm materialised) W_l [out,in] row-major fp32 concatenated, l = 0..4; b likewise.
 * pe_w [8] host = annealing weights of the 4-band view-direction encoding.  All tensors [P,*] row-major fp32.
 * TC modes only.                                                                                              */
RECMV_API size_t recmv_rendernet_packed_bytes(void);
RECMV_API int recmv_rendernet_pack_weights(const float* W_all, const float* b_all, void* packed,
                                 recmv_stream_t stream);
RECMV_API int recmv_rendernet_fwd(const float* points, const float* normals, const float* view_dirs,
                        const float* feats, const void* packed, const float* pe_w /*host*/, float* out_rgb,
                        int64_t P, int mode, recmv_stream_t stream);

/* ---- coarse-to-fine sweep helpers (A11, MCAcc/seg3d_lossless.py:233-428) -------------------------------------------
 * interp2x_boundary3d: replaces MCAcc/cuda/interp2x_boundary3d.cpp:18-35 (forward(input, balance) -> [output,
 * is_boundary]; backward(grad_output) -> grad_input).  input [NC,D,H,W] f32 -> output [NC,2D-1,2H-1,2W-1] f32 and
 * is_boundary (1 byte per voxel: the contributing coarse voxels are not all on one side of balance_value).
 * order 0 = the rounding of the reference extension (sequential sum / count), order 1 = the rounding of
 * F.interpolate(mode='trilinear', align_corners=True), the reference's default path (seg3d_lossless.py:270-281).
 * recmv_c2f_todo_mask: todo = (3x3x3 dilation of is_boundary) & ~done  (seg3d_lossless.py:297-303).                */
RECMV_API int recmv_interp2x_boundary3d_fwd(const float* input, float* output, uint8_t* is_boundary, int NC,
                                  int D, int H, int W, float balance_value, int order,
                                  recmv_stream_t stream);
RECMV_API int recmv_interp2x_boundary3d_bwd(const float* grad_output, float* grad_input, int NC, int D, int H,
                                  int W, recmv_stream_t stream);
RECMV_API int recmv_c2f_todo_mask(const uint8_t* is_boundary, const uint8_t* done, uint8_t* todo, int D, int H,
                        int W, recmv_stream_t stream);

/* ---- A9 + (f3): FindSurfacePs + view_rays + the mask filter of sample_train_ray ------------------------------------
 * replaces utils/FindSurfacePs.py:7-60 (nonzero / torch_scatter scatter(min) / gathers), model/CameraMine.py:146-167
 * (view_rays) and the `gt_mask > 0` selection of OptimGarmentNetwork.py:1006-1011, in three launches and one ordered
 * compaction.  pix_to_face [N,H,W,K] int64, bary [N,H,W,K,3] f32 (pytorch3d Fragments), verts [V,3], faces [F,3] int64,
 * mask [N,H,W] f32 or NULL, camera = host float[13] {fx, fy, px, py, R row-major} or NULL.
 * Outputs have capacity N*H*W rows and are filled in (n, row, col) order -- the order of the reference's `nonzero`:
 * out_batch/out_row/out_col/out_finds int64, out_pts [.,3] (barycentric seed point on the canonical mesh), out_rays [.,3]
 * (only with a camera).  counters (device int32[1]) <- number of rows.  scratch: recmv_fragment_decode_scratch_bytes.   */
RECMV_API size_t recmv_fragment_decode_scratch_bytes(int64_t npix);
RECMV_API int recmv_fragment_decode(const int64_t* pix_to_face, const float* bary, int N, int H, int W, int K,
                          const float* verts, const int64_t* faces, int64_t num_faces, const float* mask,
                          const float* camera /*host[13]*/, void* scratch, int64_t* out_batch, int64_t* out_row,
                          int64_t* out_col, float* out_pts, int64_t* out_finds, float* out_rays, int32_t* counters,
                          recmv_stream_t stream);

/* ---- mesh rasterizer: the fragments recmv_fragment_decode reads ---------------------------------------------------
 * replaces the pytorch3d MeshRasterizer of `maskRender` (model/network.py:307-322; faces_per_pixel 1, blur 0,
 * perspective-correct, unclipped barycentrics, no culling of back faces).  verts [N,V,3] f32, faces [F,3] int64 shared by
 * the N frames, camera = DEVICE float[N][16] {fx, fy, px, py, R[9] row-major, T[3]}: view X R + T, screen
 * (px - fx X/Z, py - fy Y/Z), pixel (row, col) centred at (col, row).  A face is skipped when a vertex has Z <= z_clip or
 * its doubled screen area |A| <= area_eps; it covers a pixel whose three barycentrics are >= 0; the smallest
 * perspective-correct zbuf wins, ties to the lower packed index n*F + f (deterministic).  Outputs in the Fragments layout
 * with K = 1: out_pix_to_face [N,H,W] int64 (packed), out_zbuf [N,H,W], out_bary [N,H,W,3] (perspective-corrected),
 * out_dists [N,H,W] (NULL = not computed: signed squared NDC distance to the nearest edge); background = -1 in all.
 * workspace: recmv_raster_workspace_bytes(N, F, H, W, capacity); capacity = (tile, face) pair-list entries.
 * counters (DEVICE int32[4]) <- {covered pixels, skipped faces, pairs, overflow}.  No host synchronisation: when
 * pairs > capacity, overflow = 1 and NO output is written -- re-run with capacity >= pairs.                           */
RECMV_API int recmv_raster_workspace_bytes(int N, int64_t F, int H, int W, int64_t capacity, size_t* bytes);
RECMV_API int recmv_rasterize_meshes(const float* verts, int V, const int64_t* faces, int64_t F, int N,
                          const float* camera /*device[N][16]*/, int H, int W, float z_clip, float area_eps,
                          void* workspace, int64_t capacity, int64_t* out_pix_to_face, float* out_zbuf, float* out_bary,
                          float* out_dists, int32_t* counters /*device*/, recmv_stream_t stream);

/* ---- sparse z-buffer probe: the visibility test of fl_visible_by_body_zbuff / check_zbuf_body (DESIGN section 1i) --
 * the value the reference's `grid_sample(zbuf filled, uv, align_corners=True)` returns at a set of query points, with
 * zbuf the recmv_rasterize_meshes zbuf of the same verts, faces, camera, H, W, z_clip, area_eps -- without rasterizing
 * the frame.  screen_pts [N,Q,D] f32 (D >= 2; x, y read), norm_size DEVICE float[N][2] = (w, h), fill DEVICE float[N].
 * u = 2 sx / w - 1, v = 2 sy / h - 1, ix = ((u + 1) / 2) (W - 1), iy = ((v + 1) / 2) (H - 1); ATen's bilinear taps nw,
 * ne, sw, se and weights, zeros padding; a tap's value is the rasterizer's zbuf there, or fill[n] where that zbuf is
 * -1 (background); out [N,Q] = the weighted taps accumulated in that order with fused multiply-adds; 0 when ix or iy
 * is not finite.  out_tap_zbuf [N,Q,4] f32 / out_tap_face [N,Q,4] int64 (both NULL or both set): the rasterizer's
 * (zbuf, packed face) at each tap, (-1, -1) on background and outside the image.  A face with an index outside [0, V)
 * is skipped.  Five launches, no host synchronisation, deterministic.  workspace: recmv_zbuf_probe_workspace_bytes.  */
RECMV_API int recmv_zbuf_probe_workspace_bytes(int N, int64_t Q, int H, int W, size_t* bytes);
RECMV_API int recmv_zbuf_probe(const float* verts, int V, const int64_t* faces, int64_t F, int N,
                          const float* camera /*device[N][16]*/, int H, int W, float z_clip, float area_eps,
                          const float* screen_pts, int64_t Q, int D, const float* norm_size, const float* fill,
                          void* workspace, float* out, float* out_tap_zbuf, int64_t* out_tap_face,
                          recmv_stream_t stream);

/* ---- point rasterizer + alpha compositor: the silhouettes of `pcRender` ------------------------------------------
 * replaces pytorch3d's PointsRasterizer + AlphaCompositor (model/CameraMine.py:347-415, weights 1 - d / r^2).
 * points [N,P,3] f32 already projected: (NDC x, NDC y, view z); pixel (row, col) has its centre at NDC
 * (1 - (2 col + 1) / W, 1 - (2 row + 1) / H).  A point with z < 0 is skipped; it covers a pixel when d < radius^2
 * (strict, d = squared NDC distance).  Each pixel keeps the K (1..64; more is RECMV_E_RANGE) covering points with the
 * smallest z, ties to the lower packed index n*P + p (deterministic), and composites them in order:
 * T_0 = 1, image[g] += f alpha T, T *= 1 - alpha, alpha = 1 - d / radius^2, g = 0 when p < split_size, else 1.
 * features [N,P] f32 (NULL = all ones).  num_images G = 1 or 2 (image 1 only gets points p >= split_size).
 * out_images [G,N,H,W].  Fragments (each NULL = not written): out_idx [N,H,W,K] int64 packed, out_zbuf, out_dists
 * [N,H,W,K], padded with -1.  workspace: recmv_points_raster_workspace_bytes(N, P, H, W, capacity), capacity =
 * (tile, point) pair entries.  counters (DEVICE int32[4]) <- {covered pixels, skipped points, pairs, overflow}.  No host
 * synchronisation: when pairs > capacity, overflow = 1 and NO output is written -- re-run with capacity >= pairs.
 * The backward reads the forward's workspace unchanged (same arguments, pairs = counters[2]): grad_images [G,N,H,W],
 * pair_scratch 2 * pairs floats, grad_points [N,P,3] (z component 0: the selection is piecewise constant).  It is
 * summed in a fixed order without float atomics, so it is bit-identical from run to run and on any GPU.           */
RECMV_API int recmv_points_raster_workspace_bytes(int N, int64_t P, int H, int W, int64_t capacity, size_t* bytes);
RECMV_API int recmv_rasterize_points(const float* points, const float* features, int N, int64_t P, int H, int W,
                          float radius, int K, int64_t split_size, int num_images, void* workspace, int64_t capacity,
                          float* out_images, int64_t* out_idx, float* out_zbuf, float* out_dists,
                          int32_t* counters /*device*/, recmv_stream_t stream);
RECMV_API int recmv_rasterize_points_backward(int N, int64_t P, int H, int W, float radius, int K, int64_t split_size,
                          int num_images, const void* workspace, int64_t pairs, const float* grad_images,
                          float* pair_scratch, float* grad_points, recmv_stream_t stream);

/* ---- vertex normals + hard Phong shading: the images of `maskRender` with a HardPhongShader ----------------------
 * replaces pytorch3d's `Meshes.verts_normals_packed` and `HardPhongShader` (infer_fl.py:167; DESIGN section 1d).
 * Normals: verts [N,V,3] f32, faces [F,3] int64 shared by the N frames -> out_normals [N,V,3].  Every (face, corner k)
 * adds cross(v[k+1] - v[k], v[k+2] - v[k]) to its vertex, summed in increasing (face, corner) order without float
 * atomics (bit-identical from run to run and on any GPU), then n / max(|n|, 1e-6).  A face with an index outside
 * [0, V) adds nothing; an unreferenced vertex gets 0.  workspace: recmv_vertex_normals_workspace_bytes(V, F).
 * No host synchronisation.
 * Phong: pix_to_face [N,H,W] int64 packed m*F + f and bary [N,H,W,3] (perspective-corrected) from
 * recmv_rasterize_meshes; verts, normals [N,V,3]; colors [N,V,3] or NULL (= 1); params DEVICE float[N][28] per frame
 * {camera centre[3], light location[3], light ambient[3], light diffuse[3], light specular[3], material ambient[3],
 * material diffuse[3], material specular[3], shininess, background[3]}.  out_rgba [N,H,W,4], 16-byte aligned:
 * rgb = (ambient + diffuse) * colour + specular, alpha 1; background where pix_to_face is outside [0, N*F) or the face
 * has an index outside [0, V).                                                                                      */
RECMV_API int recmv_vertex_normals_workspace_bytes(int V, int64_t F, size_t* bytes);
RECMV_API int recmv_vertex_normals(const float* verts, int N, int V, const int64_t* faces, int64_t F, void* workspace,
                          float* out_normals, recmv_stream_t stream);
RECMV_API int recmv_shade_phong(const int64_t* pix_to_face, const float* bary, int N, int H, int W, const float* verts,
                          const float* normals, const float* colors, int V, const int64_t* faces, int64_t F,
                          const float* params /*device[N][28]*/, float* out_rgba, recmv_stream_t stream);

/* ---- area-weighted surface sampling: the fans of `curve_aware_loss` (DESIGN section 1h) ---------------------------
 * replaces trimesh's `sample_surface` (OptimGarmentNetwork.py:808-809,832-833) with a pinned stream.  verts [M,V,3]
 * f32, faces [F,3] int64 shared by the M meshes -> out [M,S,3] f32.  Sample s of mesh m depends only on (seed, offset,
 * m, s): Philox4x32-10 with key {seed low word, seed high word} and counter {low, high word of offset + m*S + s
 * (mod 2^64), 0, 0} gives x0..x3; u = ((x0 << 21) | (x1 >> 11)) 2^-53, a = x2 2^-32, b = x3 2^-32, and (a, b) ->
 * (1 - a, 1 - b) when a + b > 1.  Areas in fp64 from the fp32 corners, e1 = v1 - v0, e2 = v2 - v0, c = e1 x e2,
 * area = 0.5 sqrt((cx^2 + cy^2) + cz^2); a face with an index outside [0, V) or a non-finite area counts 0.  C[f]
 * fp64 inclusive, summed sequentially inside each 256-face chunk, the chunk totals summed sequentially, C = chunk prefix
 * + local (np.cumsum for F <= 256).  Face = first f with C[f] >= u C[F-1] (face 0 when the total is 0); point =
 * (a e1 + b e2) + v0 in fp64, rounded once to f32; NaN when the face has an invalid index.  Every fp64 operation is
 * rounded on its own (no FMA).  Three launches, no atomics (bit-identical from run to run and on any GPU), no host
 * synchronisation.  F = 0 with M*S > 0 is RECMV_E_SHAPE.  workspace: recmv_surface_sample_workspace_bytes(M, F).     */
RECMV_API int recmv_surface_sample_workspace_bytes(int M, int64_t F, size_t* bytes);
RECMV_API int recmv_surface_sample(const float* verts, int M, int V, const int64_t* faces, int64_t F, int64_t S,
                          uint64_t seed, uint64_t offset, void* workspace, float* out, recmv_stream_t stream);

/* ---- training-ray sub-sampling: sample_train_ray's mask selection, random draw and view rays -----------------------
 * replaces engineer/networks/OptimGarmentNetwork.py:983-1055 after `find_surface_ps` (DESIGN section 1j).
 * G lists (garments); the pointer arguments ending in [G] are HOST arrays of G device pointers.  List g has
 * lengths[g] (host) rows: batch / row / col int64 [P_g] and init_pts f32 [P_g,3], against masks[g] f32 [N,H,W].
 * Candidates are the rows with mask[b, r, c] > 0 (NaN fails; an index outside the mask is not a candidate), in input
 * order; pnum_g is their count.  pnum_g <= target keeps every candidate; otherwise candidate j is kept iff u_j < thr,
 * thr = (float)((double)target / (double)pnum_g), u_j = (x0 >> 8) * 2^-24 with x0 the first word of Philox4x32-10 under
 * key (seed lo, seed hi) at counter (lo, hi, 0, 0) of offset + P_0 + ... + P_{g-1} + j.  Kept rows go, in candidate
 * order, to the capacity outputs out_* [P_g] / [P_g,3]: batch, row, col and init point copied bit for bit, and the view
 * ray of camera 0 (camera: DEVICE f32 >= 13 = {fx, fy, px, py, R row-major}, raster.camera_rows' layout) by the formula
 * of recmv_fragment_decode.  counts: DEVICE int32[G] <- kept rows per list.  Five launches per 8 lists, no atomics
 * (bit-identical from run to run), no host synchronisation.  P_g > 2^31 - 1 is RECMV_E_RANGE.
 * workspace: recmv_train_rays_workspace_bytes(G, lengths).                                                            */
RECMV_API int recmv_train_rays_workspace_bytes(int G, const int64_t* lengths, size_t* bytes);
RECMV_API int recmv_train_rays_sample(int G, const int64_t* const* batch, const int64_t* const* row,
                             const int64_t* const* col, const float* const* init_pts, const int64_t* lengths,
                             const float* const* masks, int N, int H, int W, const float* camera, int64_t target,
                             uint64_t seed, uint64_t offset, void* workspace, int64_t* const* out_batch,
                             int64_t* const* out_row, int64_t* const* out_col, float* const* out_pts,
                             float* const* out_rays, int32_t* counts, recmv_stream_t stream);

/* ---- surface-render loss points: surface_render_loss's eikonal / regulariser samples and the `check` compaction -----
 * replaces engineer/networks/OptimGarmentNetwork.py:1103-1167's CPU draws and boolean indexing (DESIGN section 1k).
 * G garments; the pointer arguments ending in [G] are HOST arrays of G device pointers; M[g] (surface-solve points)
 * and V[g] (MC vertices, >= 1) are host int64.  Garment g: init_pts f32 [M_g,3], verts f32 [V_g,3], check uint8 [M_g],
 * batch / row / col int64 [M_g], rays f32 [M_g,3].  S = 4096 // G; thr_g = (float)((double)S / (double)V_g).
 * Counter of row i of lane l (0 E-draw, 1 D-draw, 2 E-local, 3 E-global, 4 D-local) of garment g:
 * offset + 5 (C_0 + ... + C_{g-1}) + l C_g + i, C_g = M_g + V_g; Philox4x32-10 under key (seed lo, seed hi) at counter
 * (lo, hi, 0, 0).  Vertex v is kept in lane E / D iff (x0 >> 8) 2^-24 < thr_g (E-draw / D-draw row v).
 * recmv_loss_points_count: DEVICE counts int32[3G] <- (kept E, kept D, checked) per garment; two launches per 8
 * garments, no host synchronisation.  The caller reads the counts and passes them (HOST int32[3G]) to
 * recmv_loss_points_emit, which writes, with B_L = cat(init_pts, kept_L vertices in index order):
 *   out_eikonal[g] f32 [|B_E| + |B_E| / 6, 3] = cat(B_E + 0.01 z (E-local row), global rows fp32(fp32(u 3.6f) - 1.8f)
 *                  with u = (x_k >> 8) 2^-24, k = coordinate (E-global row));
 *   out_regular[g] f32 [2 |B_D|, 3] = cat(B_D, B_D + 0.01 z (D-local row));
 *   out_pts / out_rays [checked, 3], out_batch / out_row / out_col / out_index int64 [checked]: the rows whose check is
 *   non-zero, in order, copied bit for bit, and their input indices.
 * z = (r0 cos 2 pi ub, r0 sin 2 pi ub, r1 cos 2 pi ud) in double, r = sqrt(-2 ln ((x >> 8) + 1) 2^-24) of x0 / x2,
 * ub / ud = (x >> 8) 2^-24 of x1 / x3, rounded to f32; a local point is x + fp32(z 0.01f).  The workspace
 * (recmv_loss_points_workspace_bytes(G, M, V)) carries the draws from count to emit.  No atomics (bit-identical from
 * run to run).  V_g = 0 is RECMV_E_SHAPE; C_g > 2^31 - 1 is RECMV_E_RANGE.                                           */
RECMV_API int recmv_loss_points_workspace_bytes(int G, const int64_t* M, const int64_t* V, size_t* bytes);
RECMV_API int recmv_loss_points_count(int G, const int64_t* M, const int64_t* V, const uint8_t* const* check, int S,
                             uint64_t seed, uint64_t offset, void* workspace, int32_t* counts, recmv_stream_t stream);
RECMV_API int recmv_loss_points_emit(int G, const float* const* init_pts, const int64_t* M, const float* const* verts,
                            const int64_t* V, const int64_t* const* batch, const int64_t* const* row,
                            const int64_t* const* col, const float* const* rays, const int32_t* counts, int S,
                            uint64_t seed, uint64_t offset, void* workspace, float* const* out_eikonal,
                            float* const* out_regular, float* const* out_pts, float* const* out_rays,
                            int64_t* const* out_batch, int64_t* const* out_row, int64_t* const* out_col,
                            int64_t* const* out_index, recmv_stream_t stream);

/* ---- per-frame means of the photometric terms: torch_scatter's scatter(e, batch, reduce='mean', dim_size=N).mean() --
 * L = (1/N) sum_b [sum_{i in b} e_i / max(1, n_b)] (an empty frame gives 0; a row whose frame lies outside [0, N) is
 * not counted), with f64 partials over fixed 1024-row chunks combined in chunk order: no float atomics, bit-identical
 * from run to run (DESIGN section 1k).  loss: DEVICE f32[1]; counts: DEVICE int32[N] <- n_b, kept for the backward;
 * grad_loss: DEVICE f32[1].  workspace: recmv_frame_loss_workspace_bytes(M, N).  N <= 0 is RECMV_E_SHAPE.
 * colour: e_i = sum_ch |gt[b, r, c, ch] - colors[i, ch]| (f32, channels in order), gt f32 [N,H,W,3]; an index outside
 *   gt is not counted.  Backward dcolors [M,3] = -sign(gt - colors) g / (N max(1, n_b)), sign(0) = 0.
 * normal: gtn [M,3], J [M,3,3] (row a = grad of D_a), nx [M,3], w [M] f32; nn = |gtn| (double), valid iff nn > 1e-4,
 *   n = gtn / nn, d = J^T n - nx, e_i = |d| w_i over the valid rows.  Backward to gtn, J and nx (w is constant; 0 at
 *   |d| = 0 and for invalid rows).                                                                                   */
RECMV_API int recmv_frame_loss_workspace_bytes(int64_t M, int N, size_t* bytes);
RECMV_API int recmv_color_frame_mean(const float* gt, int N, int H, int W, const int64_t* batch, const int64_t* row,
                            const int64_t* col, const float* colors, int64_t M, void* workspace, float* loss,
                            int32_t* counts, recmv_stream_t stream);
RECMV_API int recmv_color_frame_mean_backward(const float* gt, int N, int H, int W, const int64_t* batch,
                                     const int64_t* row, const int64_t* col, const float* colors, int64_t M,
                                     const int32_t* counts, const float* grad_loss, float* dcolors,
                                     recmv_stream_t stream);
RECMV_API int recmv_normal_frame_mean(const float* gtn, const float* J, const float* nx, const float* w,
                             const int64_t* batch, int64_t M, int N, void* workspace, float* loss, int32_t* counts,
                             recmv_stream_t stream);
RECMV_API int recmv_normal_frame_mean_backward(const float* gtn, const float* J, const float* nx, const float* w,
                                      const int64_t* batch, int64_t M, int N, const int32_t* counts,
                                      const float* grad_loss, float* dgtn, float* dJ, float* dnx,
                                      recmv_stream_t stream);

/* ---- mask_loss's ground-truth dilation and soft silhouette IoU, all garments and frames in one call --------------
 * m[g], gt[g]: DEVICE f32 [N,H,W] per garment (silhouette, ground-truth mask); r: radius, 1..32 (r < 1 is
 * RECMV_E_SHAPE, r > 32 RECMV_E_RANGE).  Forward writes mgt[g] f32 [N,H,W] = max_pool2d(gt[g], 2r+1, stride 1,
 * padding r) bit for bit (out-of-image taps ignored, a NaN tap wins); iu f64 [G,N,2] = (I, U) with I = sum m g',
 * U = sum |(m + g') - m g'| (each pixel term formed in f32, summed in f64 over fixed 32 x 32 tiles, the tiles combined
 * in order); loss_gn f32 [G,N] = 1 - I / U (NaN when U = 0); loss f32 [G] = mean_n loss_gn.  No float atomics:
 * bit-identical from run to run (DESIGN section 1m).  workspace: recmv_mask_iou_workspace_bytes(G, N, H, W, r).
 * Backward: grad_loss DEVICE f32 [G], dm[g] f32 [N,H,W] = -(grad_loss[g] / N) (g' U - I s (1 - g')) / U^2 with
 * s = sign((m + g') - m g'), sign(0) = 0, in double from the forward's mgt and iu, rounded once.  The host arrays m,
 * gt, mgt and dm hold G device pointers.  N > 65535 is RECMV_E_RANGE.  No host synchronisation.                    */
RECMV_API int recmv_mask_iou_workspace_bytes(int G, int N, int H, int W, int r, size_t* bytes);
RECMV_API int recmv_mask_iou(int G, const float* const* m, const float* const* gt, int N, int H, int W, int r,
                    void* workspace, float* const* mgt, double* iu, float* loss_gn, float* loss,
                    recmv_stream_t stream);
RECMV_API int recmv_mask_iou_backward(int G, const float* const* m, const float* const* mgt, int N, int H, int W,
                             const double* iu, const float* grad_loss, float* const* dm, recmv_stream_t stream);

/* ---- nearest neighbour (K = 1 knn_points): the feature-curve chamfer loss and template registration --------------
 * replaces pytorch3d's KNN extension behind `knn_points` / `chamfer_distance` (DESIGN section 1e).
 * p1 [N,P1,D] queries, p2 [N,P2,D] candidates, f32, D = 2 or 3; lengths1 / lengths2 DEVICE int64[N] or NULL (= P1, P2),
 * clamped to [0, P] on the device.  d = (dx*dx + dy*dy) [+ dz*dz], dx = x1 - x2, each operation rounded in fp32 in
 * that order (no FMA); the smallest d wins, on equal d the lower index.  out_dists [N,P1] f32, out_idx [N,P1] int64;
 * rows i >= lengths1[n], and every row of a cloud with lengths2[n] == 0, get dists 0 and idx -1.  Non-finite
 * coordinates never give an index outside [-1, lengths2).  The result does not depend on the launch shape or the SM
 * count.  workspace: recmv_knn_workspace_bytes(N, P1, P2) (serves both the forward and the backward).
 * Backward from grad_dists [N,P1]: grad_p1 [N,P1,D] = 2 g (p1_i - p2_idx_i); grad_p2 [N,P2,D] (NULL = not computed) =
 * -sum over the queries i with idx_i = j of grad_p1_i, in increasing i.  Entries with idx outside [0, P2) add nothing.
 * No float atomics: bit-identical from run to run and on any GPU.  No host synchronisation.                        */
RECMV_API int recmv_knn_workspace_bytes(int N, int64_t P1, int64_t P2, size_t* bytes);
RECMV_API int recmv_knn_nearest(const float* p1, const float* p2, const int64_t* lengths1, const int64_t* lengths2,
                          int N, int64_t P1, int64_t P2, int D, void* workspace, float* out_dists, int64_t* out_idx,
                          recmv_stream_t stream);
RECMV_API int recmv_knn_nearest_backward(const float* p1, const float* p2, const int64_t* idx, const float* grad_dists,
                          int N, int64_t P1, int64_t P2, int D, void* workspace, float* grad_p1, float* grad_p2,
                          recmv_stream_t stream);

/* ---- template registration: the inner step of NRICP_Optimizer_AdamW (DESIGN section 1f) ---------------------------
 * replaces the per-iteration torch graph of nricp_optimizer.py:382-423 (Local_Affine warp, edge stiffness, pytorch3d's
 * uniform mesh_laplacian_smoothing, autograd and AdamW(amsgrad=True)).
 * Adjacency: faces [F,3] int64 over V vertices (a face with an index outside [0, V) is skipped).  E = the unique
 * sorted pairs of the 3F face sides; row_ptr [V+1] int32 and col [6F] int32 are the symmetric CSR of E (both
 * directions of every edge, so a self edge (a, a) appears twice in row a), neighbours ascending within a row; only
 * col[0, row_ptr[V]) is used, the rest is -1.  deg [V] int32 = row length; boundary [V] u8 = 1 where one of the
 * vertex's sides occurs exactly once among the 3F sides.  No host synchronisation.
 * workspace: recmv_mesh_adjacency_workspace_bytes(V, F).
 * Warp: X [V,3,4] f32 = [A | b] per vertex, x [V,3] source points -> out_v = A x + b; out_n = inv(A)^T n and out_ok
 * (|det A| >= 1e-4, else n' = 0) when not NULL (they need normals [V,3]).
 * Step, one AdamW-AMSGrad iteration in two launches, in place on X and its moments exp_avg / exp_avg_sq /
 * max_exp_avg_sq [V,3,4] (prm->step == 1 starts them from zero and does not read them): with c_i = target_v[corr_idx
 * [i]], m_i = target_n[corr_idx[i]] (corr_idx [V] int64, an index outside [0, T) gates the vertex out) and
 * w_i = !boundary_i & ok_i & (cos(m_i, n'_i) > threshold), loss = sqrt(S) + lw / V sum_i |Lv_i| with
 * S = sum_i w_i |v_i - c_i|^2 + sw sum_{(i,j) in E} ||(X_i - X_j) diag(1,1,1,gamma)||^2 and Lv_i = mean_{j in N(i)} v_j
 * - v_i (-v_i when deg_i = 0).  stats DEVICE float[8] = {data sum, sw * stiffness sum, Laplacian term, loss, gate
 * count, S, 0, 0} of the state before the update.  Every reduction runs in a fixed order that depends on V alone: the
 * results are bit-identical from run to run and on any GPU.  No float atomics, no host synchronisation.
 * workspace: recmv_nricp_workspace_bytes(V).                                                                        */
typedef struct {
  float stiffness_weight, laplacian_weight, gamma, threshold;
  float lr, beta1, beta2, eps, weight_decay;   /* torch.optim.AdamW: 1e-4, 0.9, 0.999, 1e-8, 1e-2 in the reference */
  int step;                                    /* 1-based step count since the moments were last reset */
} recmv_nricp_params_t;

RECMV_API int recmv_mesh_adjacency_workspace_bytes(int64_t V, int64_t F, size_t* bytes);
RECMV_API int recmv_mesh_adjacency(const int64_t* faces, int64_t F, int64_t V, void* workspace, int32_t* row_ptr,
                          int32_t* col, int32_t* deg, uint8_t* boundary, recmv_stream_t stream);
RECMV_API int recmv_nricp_warp(const float* X, const float* x, const float* normals, int64_t V, float* out_v,
                          float* out_n, uint8_t* out_ok, recmv_stream_t stream);
RECMV_API int recmv_nricp_workspace_bytes(int64_t V, size_t* bytes);
RECMV_API int recmv_nricp_step(const float* x, const float* normals, const float* target_v, const float* target_n,
                          int64_t T, const int64_t* corr_idx, const int32_t* row_ptr, const int32_t* col,
                          const uint8_t* boundary, int64_t V, const recmv_nricp_params_t* prm /*host*/, float* X,
                          float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq, void* workspace,
                          float* stats /*device[8]*/, recmv_stream_t stream);

/* ---- template fitting: the Laplacian-editing solve of Laplacian_Optimizer (DESIGN section 1g) ----------------------
 * replaces the dense inv(L^T W L) L^T W t of lap_deform_optimizer.py:144-183.  verts [V,3] f32 = x; (row_ptr, col, deg)
 * = recmv_mesh_adjacency of the template's faces; L = D^-1 Adj - I (-I on a row with deg 0).  Constraints: cidx [M]
 * int64 SORTED ascending (duplicates allowed, each its own row of P; an index outside [0, V) is skipped) with targets
 * ctgt [M,3] f32 in the same order.  Solves A y = b, A = L^T L + c P^T P, b = L^T L x + c P^T u (c = constrain_weight
 * >= 0), for the three columns independently by Jacobi-preconditioned CG in float64 from y0 = x: a column stops when
 * |r| <= tol |b|, when r.r is not finite, or after max_iter iterations.  A component with no constraint keeps y = x
 * exactly.  smooth != 0 then stores y'_i = (1/deg_i) sum_{j in N(i), j != i} y_j (0 at deg_i = 0), else y; out [V,3]
 * f32.  stats DEVICE float[8] = {iterations of x, y, z; |r| / |b| of x, y, z (|r| where |b| = 0); 1 = every column
 * met tol, 0 = one stopped at max_iter, -1 = one had a non-finite residual; constraints skipped}.  Three launches, the
 * second cooperative; max_blocks = 0 runs every co-resident block, > 0 caps the grid (the result does not depend on
 * it).  Reductions run in a fixed order over 256-vertex chunks: bit-identical from run to run and for any grid.  No
 * atomics, no host synchronisation.  workspace: recmv_lap_edit_workspace_bytes(V, M).                            */
RECMV_API int recmv_lap_edit_workspace_bytes(int64_t V, int64_t M, size_t* bytes);
RECMV_API int recmv_lap_edit_solve(const float* verts, int64_t V, const int32_t* row_ptr, const int32_t* col,
                          const int32_t* deg, const int64_t* cidx, const float* ctgt, int64_t M, double constrain_weight,
                          double tol, int max_iter, int smooth, int max_blocks, void* workspace, float* out,
                          float* stats /*device[8]*/, recmv_stream_t stream);

/* ---- A11 / (f2): the sweep of one pyramid level as a DEVICE WORKLIST (SURVEY 8b `recmv_c2f_sweep`) -----------------
 * replaces the coordinate-list bookkeeping of MCAcc/seg3d_lossless.py:306-428 (nonzero / unique / index scatter, a
 * host sync per step).  level / final_res are (W, H, D) = (x, y, z) lattice sizes (host).  A worklist is idx_out[i]
 * (flat level index) and points_out[i] (the query point of batch_eval, :89-100, bit-identical arithmetic), in no
 * particular order; counters (device int32[2] = {count, overflow}, zeroed by the caller) is advanced atomically and
 * overflow is set when more than `capacity` voxels are appended.
 *  recmv_c2f_refine       : coarse level (D,H,W) -> fine level (2D-1,2H-1,2W-1) in one full-grid pass: upsampled values
 *                           (order as recmv_interp2x_boundary3d_fwd), the level's done lattice (done_fine[2z,2y,2x] =
 *                           done_coarse[z,y,x], 0 elsewhere), and the worklist of the voxels to query: not done and in
 *                           the 3x3x3 dilation of the mixed-stencil flags, evaluated exactly from a coarse "mixed cell"
 *                           mask (mixed_scratch, (D-1)(H-1)(W-1) bytes).
 *  recmv_sdf_mlp_fwd_counted (above): evaluates points_out[0 .. *counters) without the host knowing the count.
 *  recmv_c2f_scatter_list : occ[idx] = vals, done[idx] = 1, calculated[final-lattice position] = 1, claim[idx] = 0; a
 *                           sign flip against the interpolated value appends idx to conflict_list / conflict_count
 *                           (device int32, zeroed by the caller); stats[0] (device int32) += queried.
 *  recmv_c2f_mark_conflicts: next worklist = the 3x3x3 neighbours of the conflicting voxels not yet evaluated at any
 *                           level (calculated[z*sz, y*sy, x*sx] == 0, :392-420), each claimed once through `claim`
 *                           (level-lattice bytes, 4-byte aligned, all zero between rounds).                            */
RECMV_API int recmv_c2f_refine(const float* occ_coarse, const uint8_t* done_coarse, int D, int H, int W,
                     const int final_res[3] /*host*/, const float b_min[3] /*host*/, const float b_max[3] /*host*/,
                     float balance_value, int order, uint8_t* mixed_scratch, float* occ_fine, uint8_t* done_fine,
                     int32_t* idx_out, float* points_out, int32_t* counters, int capacity, recmv_stream_t stream);
RECMV_API int recmv_c2f_scatter_list(const int32_t* idx, const float* vals, const int32_t* counters, int capacity,
                           const int level[3] /*host*/, const int final_res[3] /*host*/, float* occ, uint8_t* done,
                           uint8_t* calculated, uint8_t* claim, float balance_value, int32_t* conflict_list,
                           int32_t* conflict_count, int32_t* stats, recmv_stream_t stream);
RECMV_API int recmv_c2f_mark_conflicts(const int32_t* conflict_list, const int32_t* conflict_count, int list_capacity,
                             const uint8_t* calculated, const int level[3] /*host*/, const int final_res[3] /*host*/,
                             const float b_min[3] /*host*/, const float b_max[3] /*host*/, uint8_t* claim,
                             int32_t* idx_out, float* points_out, int32_t* counters, int capacity,
                             recmv_stream_t stream);

/* ---- A10: surface-point solve of a batch of rays on the device (utils/FindSurfacePs.py:145-353) -------------------
 * ps [P,3]: in = seeds (FindSurfacePs), out = solution; ok [P] = converged (|f| < dthreshold and the angle between
 * D(p) - cam and the ray < athreshold_deg).  Networks: packed SDF weights, packed translator weights + conds
 * [F,128] + skeleton (A [F,24,4,4], trans [F,3]) + channels-last voxel, i.e. the CompositeDeformer
 * [MLPTranslator, LBSkinner]; batch_inds [P] i64 (or NULL: one frame).  `times` steps = times + 1 rounds of two
 * forward-mode launches + one update kernel; no host synchronisation.  workspace: recmv_surface_solve_workspace(P)
 * bytes of device memory.  TC modes only.                                                                            */
RECMV_API size_t recmv_surface_solve_workspace(int64_t P);
RECMV_API int recmv_surface_solve(const float* cam_pos /*host[3]*/, const float* rays, float* ps,
                        const int64_t* batch_inds, const void* sdf_packed, const float* sdf_pe_w /*host[12]*/,
                        const void* tr_packed, const float* tr_pe_w /*host[12]*/, const float* conds,
                        int num_frames, const float* A, const float* trans, const recmv_voxel_t* vox /*host*/,
                        float dthreshold, float athreshold_deg, float w1, float w2, int times, int mode,
                        void* workspace, size_t workspace_bytes, uint8_t* ok, int64_t P, recmv_stream_t stream);

/* ---- implicit-surface gradient, per-ray algebra (SURVEY 8f rank 1; engineer/networks/OptimNetwork.py:788-851) -------
 * b = [grad_f_p ; [v]x J] (4x3), r = grad_l_p (b^T b)^-1 b^T with FastMinv's |det| < 1e-4 rule (ok = 0, zeros).
 * Outputs: sdf_coef [n] = -r[0] (the cotangent the reference feeds to autograd.grad(sdf(p), params, .)),
 * def_vec [n,3] = r[1:4] (-[v]x) (the cotangent for autograd.grad(D(p), params, .)), optional ray_grad [n,3] =
 * r[1:4] [d - c]x (needs d_minus_c [n,3]).  All inputs [n,3] except jac [n,3,3] (row i = gradient of D_i), fp32.   */
RECMV_API int recmv_surface_grad_coeffs(const float* grad_l_p, const float* grad_f_p, const float* jac,
                              const float* rays, const float* d_minus_c /*may be NULL*/, float* sdf_coef,
                              float* def_vec, float* ray_grad /*may be NULL*/, uint8_t* ok, int64_t n,
                              recmv_stream_t stream);

/* ---- implicit-surface gradient of every garment of a call (DESIGN section 1l; OptimGarmentNetwork.py:2159-2313) ----
 * The per-row algebra of recmv_surface_grad_coeffs (bit-identical per row) over n rows, garment g's rows at
 * [offsets[g], offsets[g+1]) (offsets: HOST int64[G+1], offsets[0] = 0, non-decreasing, offsets[G] = n).
 * Per row: sdf_coef [n] = -r0, def_vec [n,3] = r[1:4] (-[v]x), ok [n]; ray_grad [n,3] = r[1:4] [d - c]x when not NULL
 * (needs d [n,3] and cam_pos = c, DEVICE f32[3]; d - c is formed in the kernel).
 * Per garment: ok_count int32[G] = its ok rows; cam_grad [G,3] = -sum of its def_vec rows (may be NULL); a garment
 * without rows gives 0 and 0.  The sums are f64 partials over fixed 1024-row chunks combined in chunk order, the
 * counts block counts combined in block order: no atomics, bit-identical from run to run and for any grid.
 * Two launches per 8 garments, no host synchronisation.  workspace: recmv_implicit_grad_workspace_bytes(n, G) bytes
 * of device memory.  n > 2^31 - 1 is RECMV_E_RANGE.                                                                  */
RECMV_API int recmv_implicit_grad_workspace_bytes(int64_t n, int G, size_t* bytes);
RECMV_API int recmv_implicit_grad(const float* grad_l_p, const float* grad_f_p, const float* jac, const float* rays,
                        const float* d /*may be NULL*/, const float* cam_pos /*[3] or NULL*/,
                        const int64_t* offsets /*host, G+1*/, int G, float* sdf_coef, float* def_vec,
                        float* ray_grad /*NULL unless wanted*/, uint8_t* ok, int32_t* ok_count /*[G]*/,
                        float* cam_grad /*[G,3] or NULL*/, void* workspace, int64_t n, recmv_stream_t stream);

/* Calibration knob of the tensor-core modes.  The tensor core accumulates in fp32 with truncation: each of the K/16
 * MMAs that adds into the full-size accumulator loses on average ~2^-24 of it, a systematic bias towards zero.  The
 * epilogue therefore scales a layer's raw accumulators by (1 + gain_per_kblock * K/64); the default gain is
 * 4 * 2^-24 (measured optimum against the reference's fp32 results, tools/calibrate_acc_gain.py; 0 disables).      */
RECMV_API int recmv_tc_set_acc_gain(int mode, float gain_per_kblock);

/* Non-blocking health check of the tensor-core path on the current device: every mbarrier wait in the kernel is
 * bounded; a wait that times out records {code, barrier tag, block} in mapped host memory and later launches
 * are refused with RECMV_E_DEVICE.  info may be NULL; clear != 0 resets the record.                        */
RECMV_API int recmv_check_async_errors(int* info /*host [3]*/, int clear);

/* ---- (f4) deformation regulariser: 3x3 SVD of the translator Jacobians ---------------------------------------------
 * replaces `_, s, _ = torch.svd(Jacobs.cpu())` and its autograd backward (engineer/networks/OptimGarmentNetwork.py:1148:
 * device -> host copy, LAPACK, host -> device copy on every training step).  J [N,3,3] f32 row-major = U diag(S) V^T,
 * S [N,3] descending (torch.svd's convention); U, V [N,3,3] may be NULL.  One-sided Jacobi in registers, one matrix per
 * thread.  recmv_svd3x3_backward_s: dJ = U diag(dS) V^T -- the VJP of S alone (what a loss on the singular values needs). */
RECMV_API int recmv_svd3x3(const float* J, int64_t N, float* U, float* S, float* V, recmv_stream_t stream);
RECMV_API int recmv_svd3x3_backward_s(const float* U, const float* V, const float* dS, int64_t N, float* dJ,
                                      recmv_stream_t stream);

/* Diagnostics (tcgen05 bring-up trace entry, issue-rate microbenchmark) are NOT part of this ABI: include/recmv_b200_diag.h,
 * librecmv_b200_diag.so (tools/ only).                                                                                  */

/* ---- the fused render path (BASELINE north star) -------------------------------------------------
 * One launch: ray r, sample k -> x_obs = cam_pos + t_k dir_r, t_k = t_near + (k+1/2)(t_far-t_near)/S
 * -> inverse LBS (frame = frame_of_ray[r] or r / rays_per_frame) -> PE -> SDF MLP -> sdf [R,S].
 * Per ray also: hit_idx[r] = first k with sdf_k <= 0 (-1 if none or if sample 0 is already inside),
 * hit_t[r] = depth of the linear zero crossing between samples k-1 and k.
 * out_xc [R,S,3] optional (NULL).  Samples whose inverse warp is singular get sdf = +1e10 (never hit).*/
typedef struct {
  float cam_pos[3];
  float t_near, t_far;
  int samples_per_ray;
} recmv_raymarch_t;

RECMV_API int recmv_render_sdf(const float* ray_dirs /*[R,3]*/, const recmv_raymarch_t* rm /*host*/,
                     const float* A, const float* trans, const int32_t* frame_of_ray,
                     int64_t rays_per_frame, int num_frames, const recmv_voxel_t* vox /*host*/,
                     const void* packed, const float* pe_w /*host*/, float* out_sdf, float* out_xc,
                     int32_t* hit_idx, float* hit_t, int64_t R, int mode, recmv_stream_t stream);
/* second pass of the same launch sequence: per-ray first-hit scan over out_sdf (exposed for tests) */
RECMV_API int recmv_ray_first_hit(const float* sdf /*[R,S]*/, const recmv_raymarch_t* rm /*host*/,
                        int32_t* hit_idx, float* hit_t, int64_t R, recmv_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* RECMV_B200_H_ */

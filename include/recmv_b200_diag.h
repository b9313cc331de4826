/* recmv_b200_diag.h -- diagnostics of the tensor-core engine, kept OUT of the product ABI (include/recmv_b200.h).
 *
 *   recmv_sdf_mlp_tc_debug is exported by librecmv_b200.so (it launches the product kernel with its raw-accumulator
 *                          hook enabled) but is declared only here: no reference interface maps to it.
 * Used by tools/tc_bringup.py and tools/tc_stall_profile.py.
 *   recmv_implicit_grad_grid runs recmv_implicit_grad on a capped grid; tests/test_gpu_propagate.py checks with it
 *                          that the per-garment reductions do not depend on the launch configuration.
 */
#ifndef RECMV_B200_DIAG_H_
#define RECMV_B200_DIAG_H_
#include "recmv_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* Same computation as recmv_sdf_mlp_fwd in a TC mode (passes = 1 or 3), plus status_host[4] = {code, barrier tag,
 * block, 0} of the kernel's bounded mbarrier waits (code 0 = no wait timed out) and, when dbg_out != NULL, the raw
 * fp32 accumulator (before bias) of layer dbg_layer for the first 64 points, [64][512].                        */
RECMV_API int recmv_sdf_mlp_tc_debug(const float* x, const void* packed, const float* pe_w /*host*/,
                           float* out_sdf, float* out_feat, int64_t P, int passes, int dbg_layer,
                           float* dbg_out, int* status_host /*host*/, recmv_stream_t stream);

/* Exported ONLY by a library built with -DRECMV_TC_STALL_PROF=1 (tools/tc_stall_profile.py builds one in a temporary
 * directory; librecmv_b200.so does not have it).  counters[0..7] (host) = SM cycles summed over the CTAs of every
 * tensor-core launch since the last reset: consumer waits on FULL, consumer wgmma.wait_group, consumer epilogue,
 * consumer named barriers, consumer wait for the tile input, consumer tile loop total (thread 0 of each MMA warpgroup),
 * producer waits on EMPTY, producer tile loop total (the producer lane of each ring).  n >= 8; reset != 0 clears them.
 * Synchronises the device.                                                                                      */
RECMV_API int recmv_tc_stall_profile(unsigned long long* counters /*host*/, int n, int reset);

/* recmv_implicit_grad with its row kernel's grid capped at max_ctas CTAs (max_ctas <= 0: the product's grid).  The
 * results do not depend on the grid; the tests check that with this entry.                                       */
RECMV_API int recmv_implicit_grad_grid(const float* grad_l_p, const float* grad_f_p, const float* jac,
                                       const float* rays, const float* d, const float* cam_pos,
                                       const int64_t* offsets /*host, G+1*/, int G, float* sdf_coef, float* def_vec,
                                       float* ray_grad, uint8_t* ok, int32_t* ok_count, float* cam_grad,
                                       void* workspace, int64_t n, int max_ctas, recmv_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif  /* RECMV_B200_DIAG_H_ */

// sm_90a primitives used by the tensor-core kernels: mbarrier (with bounded waits), TMA tile loads, wgmma (warpgroup
// MMA with shared-memory operands and register accumulators), shared-memory matrix descriptors.
// Encodings follow the PTX ISA (wgmma matrix descriptor: start address, leading / stride byte offsets, swizzle mode).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace recmv {
namespace tc {

// ------------------------------------------------------------------------------------------------
// error reporting from device code: first failing wait wins; later waits return immediately
// ------------------------------------------------------------------------------------------------
struct DevStatus {
  int code;      // 0 ok, else which wait timed out
  int detail;    // role / barrier tag
  int block;
  int pad;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

// ---- mbarrier ------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy smem writes -> visible to the async proxy (TMA / tensor core operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_local(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}

// Bounded wait.  `abort_flag` is a CTA-shared int: once any wait in the CTA has timed out all later
// waits fall through immediately, so a protocol bug ends the kernel in milliseconds with a status
// instead of hanging the GPU.
__device__ __forceinline__ bool mbar_wait(uint32_t bar, uint32_t parity, volatile int* abort_flag,
                                          DevStatus* status, int tag) {
  if (mbar_try_wait(bar, parity)) return true;
  long long t0 = clock64();
  while (true) {
    if (mbar_try_wait(bar, parity)) return true;
    if (*abort_flag) return false;
    if (clock64() - t0 > 400000000LL) {  // ~0.2 s at 2 GHz
      *abort_flag = 1;
      // status lives in mapped pinned host memory: plain system-visible stores (first writer wins is not
      // needed -- any timed-out wait is a valid report)
      volatile DevStatus* vs = status;
      vs->detail = tag;
      vs->block = blockIdx.x;
      __threadfence_system();
      vs->code = 1;
      __threadfence_system();
      return false;
    }
  }
}

// named barrier over `count` threads (a multiple of 32), id 1..15 (0 is __syncthreads)
__device__ __forceinline__ void named_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ---- TMA ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
// 2-D tile load into this CTA's shared memory; completion bytes on a local mbarrier
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const void* tmap, uint32_t bar, int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx_local(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}

// ---- wgmma -------------------------------------------------------------------------------------------
// A warpgroup (4 consecutive warps, the first a multiple of 4) issues D[64 x N] (+)= A[64 x 16] . B[N x 16]^T with both
// operands in shared memory; D lives in registers.  Fragment of thread t (warp w = t / 32 of the group, lane l):
// register 4 j + 2 h + e holds row 16 w + l / 4 + 8 h, column 8 j + 2 (l % 4) + e.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across a wait
template <int R> __device__ __forceinline__ void wg_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// M 64, N 128, K 16, fp16 inputs, fp32 accumulators.  scale_d = 0: D = A.B (the old contents are ignored).
// TA / TB = 1: the operand is MN-major in shared memory (transposed), 0: K-major.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "
      "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}
// M 64, N 16, K 16 (the bias-gradient product with a tile of ones)
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}

// ---- descriptors ------------------------------------------------------------------------------------
// K-major, 128-byte swizzle: rows of 128 B (64 fp16 along K), 8-row groups 1024 B apart (SBO), atoms 1024-B aligned
// (base offset 0).  bits: [0,14) addr>>4, [16,30) LBO>>4 (unused for swizzled K-major; 1), [32,46) SBO>>4,
// [62,64) swizzle mode (1 = 128 B).  One K = 16 step inside the 64-wide atom advances the start address by 32 B.
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// K-major, 64-byte swizzle: rows of 64 B (32 fp16 along K), 8-row groups 512 B apart (SBO), atoms 512-B aligned;
// [62,64) = 2 (64 B).  One K = 16 step inside the 32-wide atom advances the start address by 32 B.
__device__ __forceinline__ uint64_t smem_desc_sw64(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(512 >> 4) << 32) | ((uint64_t)2 << 62);
}
// MN-major, 128-byte swizzle: canonical layout ((8,8,m),(8,k)):((1,8,LBO),(64,SBO)) in fp16 elements -- a [8 k-rows]
// [64 mn] atom of 1024 B, atoms stacked along k every SBO = 1024 B and along mn every LBO (8192 B here: two TMA boxes of
// {64 columns, 64 rows}).  One K = 16 step advances the start address by 16 rows = 2048 B.
__device__ __forceinline__ uint64_t smem_desc_sw128_mn(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)(8192 >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) |
         ((uint64_t)1 << 62);
}

// byte offset of the 16-byte chunk `chunk` (0..7) of row `row` inside a [rows x 128 B] SW128 tile
__device__ __forceinline__ uint32_t sw128_offset(int row, int chunk) {
  return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4));
}
// byte offset of element `col` (0..63) of row `row` inside a [rows x 128 B] SW128 tile
__device__ __forceinline__ uint32_t sw128_elem(int row, int col) {
  return sw128_offset(row, col >> 3) + (uint32_t)((col & 7) * 2);
}

// Gain that undoes the tensor core's truncating fp32 accumulation after `kblocks` 64-wide K blocks of 3-pass MMAs into
// one accumulator (the layer GEMMs of gemm3_tma.cu): the signed projection <ours, fp64> / <fp64, fp64> - 1 of
// a GEMM's output is ~ -(3.23 n - 1.5) 2^-24 after n K blocks (the first MMA overwrites the accumulator and loses
// nothing; later ones drop a fraction of an ulp of a growing sum).
__host__ __device__ __forceinline__ float acc_trunc_gain(int kblocks) {
  return 1.f + (3.23f * (float)kblocks - 1.5f) * 5.9604645e-8f;
}

// fp32 -> fp16 hi/lo split.  cvt.rn.f16x2.f32 packs two conversions into one ALU-pipe instruction; the scalar
// __float2half_rn path compiles to F2F on the quarter-rate XU pipe.
// .satfinite: an operand beyond fp16's range saturates to +-65504 instead of becoming inf (hi = inf would make
// lo = v - inf = -inf and the MMA NaN); the writers below additionally raise the overflow status (range_check).
__device__ __forceinline__ uint32_t pack_f16x2(float lo_elem, float hi_elem) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));
  return r;
}
// Operand range of the tensor-core path: scaled activations (2^6 a) and weights (2^10 w) must stay below fp16's
// 65504, i.e. |a| < 1023.5, |w| < 63.97.  The reference's fp32 has no such limit, so a violation is REPORTED
// (status code 2 in the mapped record -> recmv_check_async_errors / RECMV_E_DEVICE), never silent.
constexpr int kStatusTimeout = 1, kStatusRange = 2;
__device__ __forceinline__ void report_range(DevStatus* status, int tag) {
  volatile DevStatus* vs = status;
  if (vs->code == 0) {
    vs->detail = tag;
    vs->block = blockIdx.x;
    __threadfence_system();
    vs->code = kStatusRange;
  }
}
__device__ __forceinline__ void range_check8(const float v[8], DevStatus* status, int tag) {
  const float m = fmaxf(fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3]))),
                        fmaxf(fmaxf(fabsf(v[4]), fabsf(v[5])), fmaxf(fabsf(v[6]), fabsf(v[7]))));
  if (!(m < 65504.f)) report_range(status, tag);   // also catches NaN
}
__device__ __forceinline__ void range_check2(float a, float b, DevStatus* status, int tag) {
  if (!(fmaxf(fabsf(a), fabsf(b)) < 65504.f)) report_range(status, tag);
}
__device__ __forceinline__ void split8(const float v[8], uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    h[i] = pack_f16x2(v[2 * i], v[2 * i + 1]);
    const float2 back = __half22float2(*reinterpret_cast<const __half2*>(&h[i]));
    l[i] = pack_f16x2(v[2 * i] - back.x, v[2 * i + 1] - back.y);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}
// two adjacent values -> packed fp16 hi pair and lo pair
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  hi = pack_f16x2(a, b);
  const float2 back = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  lo = pack_f16x2(a - back.x, b - back.y);
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint4 v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

// ---- host: tensor maps ------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// the driver's cuTensorMapEncodeTiled, looked up once
inline int tensor_map_encoder(EncodeTiledFn* out) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    cudaDriverEntryPointQueryResult q;
    void* p = nullptr;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || !p) return e != cudaSuccess ? (int)e : (int)cudaErrorNotSupported;
    fn = (EncodeTiledFn)p;
  }
  *out = fn;
  return 0;
}

// The fp16 weight panels: 2-D tensor [rows, 64] fp16 (128-byte rows), box [32 x box_rows] (half a row: inputs 0..31
// or 32..63 of a panel), 64-byte swizzle -- the layout smem_desc_sw64 describes.
inline int make_panel_tmap(CUtensorMap* out, const void* base, uint64_t rows, uint32_t box_rows) {
  EncodeTiledFn fn = nullptr;
  int s = tensor_map_encoder(&fn);
  if (s) return s;
  cuuint64_t dims[2] = {64, rows};
  cuuint64_t strides[1] = {128};
  cuuint32_t box[2] = {32, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)cudaErrorInvalidValue;
}

}  // namespace tc
}  // namespace recmv

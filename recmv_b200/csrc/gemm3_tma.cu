// Training-path layer GEMMs: forward layers and backward-data with BOTH operands already split into fp16 hi / lo planes in
// HBM and fed by TMA -- no conversion in the main loop.  Every fp32 value a product reads is a = hi + lo of two fp16
// values, and a product is 3 MMAs (hi*hi + lo*hi + hi*lo) with fp32 accumulation.
//
// Every tensor a later GEMM consumes is WRITTEN in consumable form by the kernel that produces it:
//   * a layer's output  Y  -> fp32 [P][ld] (activation derivative, weight gradient) AND two fp16 planes [P][ldp]
//     hi = fp16(64 y), lo = fp16(64 y - hi)  (K-major rows: exactly what the next layer's A operand is);
//   * a cotangent       G  -> fp32 AND planes of 64 * dyn * g  (dyn = the call's power-of-two gradient scale, device scalar);
//   * weights           W  -> planes of 1024 w, once per step: [out][in] for the forward, [in][out] for backward-data
//     (recmv_split_planes, optionally transposing).
// Main loop: a TMA warp streams [128 rows x 64 k] SW128 boxes of the four planes through a 3-stage ring (complete_tx on
// the stage's mbarrier; out-of-range rows / columns are zero-filled by TMA, so ragged M, N, K need no masking); two
// consumer warpgroups (one per 64-row half of the 128 x 128 tile) issue 12 wgmma m64n128k16 per K block (lo*hi, hi*lo,
// hi*hi) into register accumulators and release a stage once the MMAs that read it have completed.  PERSISTENT: a CTA
// walks tiles blockIdx.x, + gridDim.x, ...; the TMA warp runs up to three K blocks ahead, so the next tile's loads overlap
// the epilogue (bias / activation or activation derivative, fp32 store, hi / lo split and plane store).
#include "sdf_mlp.cuh"
#include "tc_common.cuh"

namespace recmv {
using namespace tc;

namespace {

constexpr int kBM = 128, kBN = 128, kBK = 64;
constexpr int kStages = 3;
constexpr uint32_t kPlane = 16384;                 // one [128 rows][64 fp16] tile
constexpr uint32_t kStageBytes = 4 * kPlane;       // A hi | A lo | B hi | B lo
constexpr int kMmaWarps = 8;                       // two consumer warpgroups
constexpr int kThreads = 32 * (kMmaWarps + 1);     // + warp 8: TMA producer
constexpr uint32_t kOffBar = kStages * kStageBytes;
constexpr int kBarFull = 0, kBarEmpty = kStages;
constexpr int kNumBars = 2 * kStages;
constexpr uint32_t kOffMisc = kOffBar + kNumBars * 8;
constexpr uint32_t kSmemBytes = kOffMisc + 64 + 1024 /* alignment slack */;

enum { TEPI_BWD_NONE = 0, TEPI_BWD_SOFTPLUS100 = 1, TEPI_BWD_RELU = 2, TEPI_FWD_NONE = 4, TEPI_FWD_SOFTPLUS100 = 5,
       TEPI_FWD_RELU = 6 };

struct GtParams {
  float* D; long long ldd;                 // fp32 output, columns n < split
  float* D2; long long ldd2;               // fp32 output, columns n >= split (no activation derivative), may be NULL
  __half* DH; __half* DL; long long ldp;   // optional planes of the < split columns: split(plane_scale * value)
  const float* E; long long lde;           // saved layer input (backward-data activation derivative)
  const float* bias;                       // forward
  const float* dyn_scale;                  // backward-data: device scalar in the A planes' scale
  float unscale;                           // d_scale / (a_scale * b_scale), before dyn
  float plane_scale;                       // 64 (x dyn for cotangents)
  int M, N, K, split, tiles_m, tiles_n, epi, dyn_in_planes;
  DevStatus* status;
};

__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float lg2_approx(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
// softplus(beta = 100, threshold 20) in the inference engine's form (sdf_mlp_tc.cu softplus100_scaled): two MUFU ops;
// absolute error <= ~2e-9 on activations of scale 0.05 (lg2.approx: 2^-22 absolute near 1)
__device__ __forceinline__ float softplus100_fast(float z) {
  constexpr float kUThr = 20.f * 1.4426950408889634f;
  const float u = z * kSoftplusLog2Scale;
  const float y = lg2_approx(1.f + ex2_approx(fminf(u, kUThr))) * 0.0069314718055994531f;
  return u > kUThr ? z : y;
}

}  // namespace

// One 64-wide K block of the 3-pass product (K-major operands) into a warpgroup's [64 x 128] accumulator: A rows
// 64 g .. 64 g + 63 of the stage.  Correction products first (they are 2^-11 of the result: added while the K block's
// contribution is still small they cost no accumulator precision), then hi*hi.
__device__ __forceinline__ void mma_kblock3_k(float (&acc)[64], uint32_t st, int g, bool first) {
  const uint64_t a_hi = smem_desc_sw128(st + (uint32_t)g * 8192u), a_lo = smem_desc_sw128(st + kPlane + (uint32_t)g * 8192u);
  const uint64_t b_hi = smem_desc_sw128(st + 2 * kPlane), b_lo = smem_desc_sw128(st + 3 * kPlane);
  wg_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) wgmma_n128<0, 0>(acc, a_lo + 2 * k, b_hi + 2 * k, (first && k == 0) ? 0u : 1u);
#pragma unroll
  for (int k = 0; k < 4; ++k) wgmma_n128<0, 0>(acc, a_hi + 2 * k, b_lo + 2 * k, 1u);
#pragma unroll
  for (int k = 0; k < 4; ++k) wgmma_n128<0, 0>(acc, a_hi + 2 * k, b_hi + 2 * k, 1u);
  wg_commit();
}

__global__ void __launch_bounds__(kThreads, 1)
gemm3_tma_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                 const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo, const GtParams prm) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t bar0 = base + kOffBar;
  volatile int* abort_flag = reinterpret_cast<volatile int*>(gbase + kOffMisc + 4);
  auto BAR = [&](int i) { return bar0 + 8u * (uint32_t)i; };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_tiles = prm.tiles_m * prm.tiles_n;
  const int nkb = (prm.K + kBK - 1) / kBK;

  if (threadIdx.x == 0) {
    *abort_flag = 0;
    for (int s = 0; s < kStages; ++s) { mbar_init(BAR(kBarFull + s), 1); mbar_init(BAR(kBarEmpty + s), 2); }
    fence_mbar_init();
    prefetch_tmap(&tm_a_hi); prefetch_tmap(&tm_a_lo); prefetch_tmap(&tm_b_hi); prefetch_tmap(&tm_b_lo);
  }
  __syncthreads();

  if (warp == kMmaWarps) {
    // =========================================== TMA producer =======================================================
    if (lane == 0) {
      long long kbg = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int tm = tile / prm.tiles_n, tn = tile - tm * prm.tiles_n;
        for (int kb = 0; kb < nkb; ++kb, ++kbg) {
          const int s = (int)(kbg % kStages);
          const uint32_t par = (uint32_t)((kbg / kStages) & 1);
          mbar_wait(BAR(kBarEmpty + s), par ^ 1u, abort_flag, prm.status, 3000 + s);
          const uint32_t st = base + (uint32_t)s * kStageBytes;
          mbar_expect_tx_local(BAR(kBarFull + s), kStageBytes);
          tma_load_2d(st, &tm_a_hi, BAR(kBarFull + s), kb * kBK, tm * kBM);
          tma_load_2d(st + kPlane, &tm_a_lo, BAR(kBarFull + s), kb * kBK, tm * kBM);
          tma_load_2d(st + 2 * kPlane, &tm_b_hi, BAR(kBarFull + s), kb * kBK, tn * kBN);
          tma_load_2d(st + 3 * kPlane, &tm_b_lo, BAR(kBarFull + s), kb * kBK, tn * kBN);
        }
      }
    }
  } else {
    // =========================================== MMA warpgroups + epilogue ==========================================
    const int g = warp >> 2, wq = warp & 3;
    const bool signaller = (threadIdx.x & 127) == 0;
    const float dyn = prm.dyn_scale ? __ldg(prm.dyn_scale) : 1.f;
    // truncating-accumulation compensation (acc_trunc_gain, tc_common.cuh)
    const float unscale = prm.unscale / dyn * acc_trunc_gain(nkb);
    const float pscale = prm.plane_scale * (prm.dyn_in_planes ? dyn : 1.f);
    const bool fwd = prm.epi >= TEPI_FWD_NONE;
    const bool d_pair = (prm.ldd & 1) == 0 && (reinterpret_cast<uintptr_t>(prm.D) & 7) == 0;
    const bool p_pair = prm.DH != nullptr && (prm.ldp & 1) == 0 && (reinterpret_cast<uintptr_t>(prm.DH) & 3) == 0 &&
                        (reinterpret_cast<uintptr_t>(prm.DL) & 3) == 0;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    long long kbg = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int tm = tile / prm.tiles_n, tn = tile - tm * prm.tiles_n;
      int pending = -1;
      for (int kb = 0; kb < nkb; ++kb, ++kbg) {
        const int s = (int)(kbg % kStages);
        mbar_wait(BAR(kBarFull + s), (uint32_t)((kbg / kStages) & 1), abort_flag, prm.status, 3100 + s);
        mma_kblock3_k(acc, base + (uint32_t)s * kStageBytes, g, kb == 0);
        wg_wait<1>();
        if (pending >= 0 && signaller) mbar_arrive_local(BAR(kBarEmpty + pending));
        pending = s;
      }
      wg_wait<0>();
      wg_fence_regs(acc);
      if (signaller) mbar_arrive_local(BAR(kBarEmpty + pending));
      // ---- epilogue: thread owns rows r0, r0 + 8 and column pairs 8 j + 2 (lane % 4) of the warpgroup's 64 x 128 block
      const int n_base = tn * kBN + 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = tm * kBM + 64 * g + 16 * wq + (lane >> 2) + 8 * h;
        if (m >= prm.M) continue;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int n = n_base + 8 * j;
          if (n >= prm.N) continue;
          float o[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float v = acc[4 * j + 2 * h + e] * unscale;
            const int nn = n + e;
            if (nn < prm.N) {
              if (fwd) {
                if (prm.bias) v += __ldg(prm.bias + nn);
                if (prm.epi == TEPI_FWD_SOFTPLUS100) v = softplus100_fast(v);
                else if (prm.epi == TEPI_FWD_RELU) v = fmaxf(v, 0.f);
              } else if (prm.epi != TEPI_BWD_NONE && nn < prm.split) {
                const float a = __ldg(prm.E + (long long)m * prm.lde + nn);
                v = prm.epi == TEPI_BWD_SOFTPLUS100 ? v * (1.f - ex2_approx(-kSoftplusLog2Scale * a)) : (a > 0.f ? v : 0.f);
              }
            }
            o[e] = v;
          }
          const bool both = n + 1 < prm.N && n + 1 < prm.split;
          if (both && d_pair) {
            *reinterpret_cast<float2*>(prm.D + (long long)m * prm.ldd + n) = make_float2(o[0], o[1]);
          } else {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int nn = n + e;
              if (nn >= prm.N) continue;
              if (nn < prm.split) prm.D[(long long)m * prm.ldd + nn] = o[e];
              else if (prm.D2) prm.D2[(long long)m * prm.ldd2 + (nn - prm.split)] = o[e];
            }
          }
          if (prm.DH && n < prm.split) {   // the same values as the next GEMM's A operand: fp16 hi / lo of plane_scale * value
            const float v0 = o[0] * pscale, v1 = (n + 1 < prm.split) ? o[1] * pscale : 0.f;
            range_check2(v0, v1, prm.status, 3500);
            uint32_t hi, lo;
            split2(v0, v1, hi, lo);
            if (both && p_pair) {
              *reinterpret_cast<uint32_t*>(prm.DH + (long long)m * prm.ldp + n) = hi;
              *reinterpret_cast<uint32_t*>(prm.DL + (long long)m * prm.ldp + n) = lo;
            } else {
              prm.DH[(long long)m * prm.ldp + n] = reinterpret_cast<const __half*>(&hi)[0];
              prm.DL[(long long)m * prm.ldp + n] = reinterpret_cast<const __half*>(&lo)[0];
              if (n + 1 < prm.split) {
                prm.DH[(long long)m * prm.ldp + n + 1] = reinterpret_cast<const __half*>(&hi)[1];
                prm.DL[(long long)m * prm.ldp + n + 1] = reinterpret_cast<const __half*>(&lo)[1];
              }
            }
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Weight gradient on the SAME planes:  dW[m][n] = sum_p G[p][m] X[p][n]  (m = output row, n = input column, p = sample).
// Both operands are the row-major planes the layer GEMMs already wrote ([P][ld], the reduction index p is the ROW), i.e.
// they are MN-major for this product.  wgmma reads MN-major fp16 operands natively (the transpose immediates; canonical
// SW128 layout ((8,8,m),(8,k)):((1,8,LBO),(64,SBO)) in fp16 elements: a [8 k-rows][64 mn] swizzle atom of 1024 B, atoms
// stacked along k every SBO = 1024 B and along mn every LBO), and that layout is exactly what TMA writes for a
// {64 columns, 64 rows} SW128 box: a 128-wide operand tile is two such boxes 8192 B apart (LBO), one MMA (K = 16 samples)
// advances the start address by 16 rows = 2048 B.  So the weight gradient needs NO transposed copy of anything.
// Work split: the output is at most 4 x 4 tiles, so the sample range is split over CTAs (grid = tiles x splits, one wave);
// inside a CTA the accumulation runs in chunks of 32 K blocks, each chunk's accumulator added into fp32 registers (a
// 10^5-sample reduction in one truncating accumulator would be cut short, DESIGN.md 5b); partial tiles go to a workspace and
// are summed in split order by a second launch (deterministic).
struct WgParams {
  float* ws;                 // [splits][tiles_m * 128][tiles_n * 128] raw partial sums (accumulator units, gain applied)
  float* ws_db;              // [splits][tiles_m * 128] raw partial row sums of A (the bias gradient), or NULL
  long long nkb;             // ceil(P / 64)
  int M, N, tiles_m, tiles_n, splits, chunk_kb;
  DevStatus* status;
};

// Bias gradient for free: db[m] = sum_p G[p][m] is one more product of the A tile, with a [16 x 64] tile of ones as a K-major B
// operand (2 KB of shared memory, written once per CTA): 8 extra N = 16 MMAs per K block, spread over the CTAs of a tile row.
constexpr uint32_t kOffOnes = (kOffMisc + 64 + 1023u) & ~1023u;
constexpr uint32_t kSmemBytesWg = kOffOnes + 2048 + 1024 /* alignment slack */;

__global__ void __launch_bounds__(kThreads, 1)
gemm3_wgrad_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                   const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo, const WgParams prm) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t bar0 = base + kOffBar;
  volatile int* abort_flag = reinterpret_cast<volatile int*>(gbase + kOffMisc + 4);
  auto BAR = [&](int i) { return bar0 + 8u * (uint32_t)i; };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x / prm.splits, split = blockIdx.x - tile * prm.splits;
  const int tm = tile / prm.tiles_n, tn = tile - tm * prm.tiles_n;
  const long long kb0 = prm.nkb * split / prm.splits, kb1 = prm.nkb * (split + 1) / prm.splits;

  // every CTA of a tile row does the bias-gradient product for the K blocks kb with kb % tiles_n == tn (spreading the extra
  // MMAs over the row's CTAs)
  const bool with_db = prm.ws_db != nullptr;
  auto db_blocks = [&](long long c0, long long c1) {   // number of K blocks of [c0, c1) this CTA owns for the bias gradient
    const long long first = c0 + ((tn - c0 % prm.tiles_n) + prm.tiles_n) % prm.tiles_n;
    return first < c1 ? (c1 - first + prm.tiles_n - 1) / prm.tiles_n : 0LL;
  };
  if (threadIdx.x == 0) {
    *abort_flag = 0;
    for (int s = 0; s < kStages; ++s) { mbar_init(BAR(kBarFull + s), 1); mbar_init(BAR(kBarEmpty + s), 2); }
    fence_mbar_init();
    prefetch_tmap(&tm_a_hi); prefetch_tmap(&tm_a_lo); prefetch_tmap(&tm_b_hi); prefetch_tmap(&tm_b_lo);
  }
  if (threadIdx.x < 128) {    // the ones tile: 128 x 16 bytes of fp16 1.0 (layout-free: all equal)
    *reinterpret_cast<uint4*>(gbase + kOffOnes + 16 * threadIdx.x) = make_uint4(0x3C003C00u, 0x3C003C00u, 0x3C003C00u, 0x3C003C00u);
    fence_proxy_async();
  }
  __syncthreads();

  if (warp == kMmaWarps) {
    if (lane == 0) {
      long long kbg = 0;
      for (long long kb = kb0; kb < kb1; ++kb, ++kbg) {
        const int s = (int)(kbg % kStages);
        mbar_wait(BAR(kBarEmpty + s), (uint32_t)(((kbg / kStages) & 1) ^ 1), abort_flag, prm.status, 3800 + s);
        const uint32_t st = base + (uint32_t)s * kStageBytes;
        mbar_expect_tx_local(BAR(kBarFull + s), kStageBytes);
        const int row = (int)(kb * kBK);
#pragma unroll
        for (int h = 0; h < 2; ++h) {   // the two 64-wide halves of each 128-wide operand tile
          tma_load_2d(st + h * 8192u, &tm_a_hi, BAR(kBarFull + s), tm * kBM + 64 * h, row);
          tma_load_2d(st + kPlane + h * 8192u, &tm_a_lo, BAR(kBarFull + s), tm * kBM + 64 * h, row);
          tma_load_2d(st + 2 * kPlane + h * 8192u, &tm_b_hi, BAR(kBarFull + s), tn * kBN + 64 * h, row);
          tma_load_2d(st + 3 * kPlane + h * 8192u, &tm_b_lo, BAR(kBarFull + s), tn * kBN + 64 * h, row);
        }
      }
    }
  } else {
    const int g = warp >> 2, wq = warp & 3;     // warpgroup g: output rows 64 g .. 64 g + 63 of the tile (A half g)
    const bool signaller = (threadIdx.x & 127) == 0;
    const uint64_t ones = smem_desc_sw128(base + kOffOnes);
    float acc[64], sum[64], dbacc[8];
    float dbsum[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 64; ++j) { acc[j] = 0.f; sum[j] = 0.f; }
#pragma unroll
    for (int j = 0; j < 8; ++j) dbacc[j] = 0.f;
    long long kbg = 0;
    for (long long c0 = kb0; c0 < kb1; c0 += prm.chunk_kb) {
      const long long c1 = c0 + prm.chunk_kb < kb1 ? c0 + prm.chunk_kb : kb1;
      bool db_started = false;
      int pending = -1;
      for (long long kb = c0; kb < c1; ++kb, ++kbg) {
        const int s = (int)(kbg % kStages);
        mbar_wait(BAR(kBarFull + s), (uint32_t)((kbg / kStages) & 1), abort_flag, prm.status, 3950 + s);
        const uint32_t st = base + (uint32_t)s * kStageBytes;
        const uint64_t a_hi = smem_desc_sw128_mn(st + (uint32_t)g * 8192u), a_lo = smem_desc_sw128_mn(st + kPlane + (uint32_t)g * 8192u);
        const uint64_t b_hi = smem_desc_sw128_mn(st + 2 * kPlane), b_lo = smem_desc_sw128_mn(st + 3 * kPlane);
        wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_n128<1, 1>(acc, a_lo + 128 * k, b_hi + 128 * k, (kb == c0 && k == 0) ? 0u : 1u);
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_n128<1, 1>(acc, a_hi + 128 * k, b_lo + 128 * k, 1u);
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_n128<1, 1>(acc, a_hi + 128 * k, b_hi + 128 * k, 1u);
        if (with_db && kb % prm.tiles_n == tn) {
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_n16<1, 0>(dbacc, a_lo + 128 * k, ones + 2 * k, (!db_started && k == 0) ? 0u : 1u);
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_n16<1, 0>(dbacc, a_hi + 128 * k, ones + 2 * k, 1u);
          db_started = true;
        }
        wg_commit();
        wg_wait<1>();
        if (pending >= 0 && signaller) mbar_arrive_local(BAR(kBarEmpty + pending));
        pending = s;
      }
      wg_wait<0>();
      wg_fence_regs(acc);
      wg_fence_regs(dbacc);
      if (signaller) mbar_arrive_local(BAR(kBarEmpty + pending));
      const float gain = acc_trunc_gain((int)(c1 - c0));
#pragma unroll
      for (int j = 0; j < 64; ++j) sum[j] = fmaf(acc[j], gain, sum[j]);
      if (db_started) {
        // every column of the ones product is the row sum: registers 0 / 2 hold rows r0 / r0 + 8
        const float gdb = acc_trunc_gain((int)db_blocks(c0, c1));
        dbsum[0] = fmaf(dbacc[0], gdb, dbsum[0]);
        dbsum[1] = fmaf(dbacc[2], gdb, dbsum[1]);
      }
    }
    const long long ldw = (long long)prm.tiles_n * kBN;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = 64 * g + 16 * wq + (lane >> 2) + 8 * h;
      float* d = prm.ws + ((long long)split * prm.tiles_m * kBM + tm * kBM + row) * ldw + tn * kBN + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < 16; ++j) *reinterpret_cast<float2*>(d + 8 * j) = make_float2(sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1]);
      if (with_db && (lane & 3) == 0)
        prm.ws_db[((long long)split * prm.tiles_n + tn) * prm.tiles_m * kBM + tm * kBM + row] = dbsum[h];
    }
  }
}

namespace {

// dW[m][n] = unscale * sum over splits (in split order) of the partial tiles
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float* __restrict__ ws, int splits, long long split_stride,
                                                           long long ldw, int M, int N, float scale,
                                                           const float* __restrict__ dyn_scale, float* __restrict__ dW,
                                                           long long ldd) {
  const float s = scale / (dyn_scale ? __ldg(dyn_scale) : 1.f);
  const long long total = (long long)M * N;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int m = (int)(i / N), n = (int)(i - (long long)m * N);
    float a = 0.f;
    for (int k = 0; k < splits; ++k) a += ws[k * split_stride + m * ldw + n];
    dW[m * ldd + n] = a * s;
  }
}

// db[m] = (1 / (64 dyn)) * sum over splits of the partial row sums
__global__ void __launch_bounds__(256) wgrad_reduce_db_kernel(const float* __restrict__ ws_db, int splits, long long split_stride,
                                                              int M, const float* __restrict__ dyn_scale, float* __restrict__ db) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float a = 0.f;
  for (int k = 0; k < splits; ++k) a += ws_db[k * split_stride + m];
  db[m] = a / (64.f * (dyn_scale ? __ldg(dyn_scale) : 1.f));
}

// column sums of an fp32 matrix (bias gradient), two deterministic stages: partial[rs][c] over row slab rs, then the slabs
constexpr int kCsSlabs = 128;
__global__ void __launch_bounds__(256) colsum_partial_kernel(const float* __restrict__ g, long long ld, long long R, int C,
                                                             float* __restrict__ partial) {
  __shared__ float sh[8][33];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31), ry = threadIdx.x >> 5;
  const long long r0 = R * blockIdx.y / kCsSlabs, r1 = R * (blockIdx.y + 1) / kCsSlabs;
  float a = 0.f;
  if (c < C)
    for (long long r = r0 + ry; r < r1; r += 8) a += __ldg(g + r * ld + c);
  sh[ry][threadIdx.x & 31] = a;
  __syncthreads();
  if (ry == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += sh[k][threadIdx.x & 31];
    partial[(long long)blockIdx.y * C + c] = t;
  }
}
__global__ void __launch_bounds__(256) colsum_final_kernel(const float* __restrict__ partial, int C, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float t = 0.f;
  for (int k = 0; k < kCsSlabs; ++k) t += partial[(long long)k * C + c];
  out[c] = t;
}

}  // namespace

namespace {

// fp32 [R][C] (row stride ld) -> fp16 hi / lo planes of scale * value: out[r][c] (transpose == 0, row stride ldp) or
// out[c][r] (transpose != 0).  scale_dev: optional device scalar multiplied into scale.
__global__ void __launch_bounds__(256) split_planes_kernel(const float* __restrict__ in, long long ld, long long R, int C,
                                                           float scale, const float* __restrict__ scale_dev, int transpose,
                                                           __half* __restrict__ hi, __half* __restrict__ lo, long long ldp,
                                                           DevStatus* status) {
  const float s = scale * (scale_dev ? __ldg(scale_dev) : 1.f);
  const long long total = R * (long long)C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C;
    const int c = (int)(i - r * C);
    float v = __ldg(in + r * ld + c) * s;
    if (!(fabsf(v) < 65504.f)) { report_range(status, 3600); v = fminf(fmaxf(v, -65504.f), 65504.f); }
    const __half h = __float2half_rn(v);
    const long long o = transpose ? (long long)c * ldp + r : r * ldp + c;
    hi[o] = h;
    lo[o] = __float2half_rn(v - __half2float(h));
  }
}

// Second-order helpers (recmv_b200/second_order.py): the element-wise step between two layer GEMMs of the tangent pass and of
// the downward pass, each ONE launch that also writes the next GEMM's operand planes.
//   softplus_tangent: tz = raw tangent of z_l, a = softplus_100(z_l) (saved), h = first-order cotangent at z_l
//       u   = s tz                 (tangent of a_{l+1};  s = softplus' = 1 - exp(-100 a))      -> fp32 + planes
//       inj = 100 (1 - s) h tz     (softplus'' u_{l+1} tz: what the second differentiation adds to the cotangent of z_l)
//   add_split: y += addend, planes of y
__global__ void __launch_bounds__(256) softplus_tangent_kernel(const float* __restrict__ tz, long long ldt, const float* __restrict__ a,
                                                               long long lda, const float* __restrict__ h, long long ldh,
                                                               long long R, int C, float plane_scale, float* __restrict__ u,
                                                               long long ldu, __half* __restrict__ uh, __half* __restrict__ ul,
                                                               long long ldp, float* __restrict__ inj, long long ldi,
                                                               DevStatus* status) {
  const long long total = R * (long long)C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C;
    const int c = (int)(i - r * C);
    const float t = __ldg(tz + r * ldt + c);
    const float em = expm1f(-100.f * __ldg(a + r * lda + c));      // -s, accurate where s is small
    const float uv = -em * t;
    u[r * ldu + c] = uv;
    inj[r * ldi + c] = 100.f * (1.f + em) * __ldg(h + r * ldh + c) * t;
    float v = uv * plane_scale;
    if (!(fabsf(v) < 65504.f)) { report_range(status, 3700); v = fminf(fmaxf(v, -65504.f), 65504.f); }
    const __half hh = __float2half_rn(v);
    uh[r * ldp + c] = hh;
    ul[r * ldp + c] = __float2half_rn(v - __half2float(hh));
  }
}

__global__ void __launch_bounds__(256) add_split_kernel(float* __restrict__ y, long long ldy, const float* __restrict__ addend,
                                                        long long lda, long long R, int C, float scale,
                                                        const float* __restrict__ scale_dev, __half* __restrict__ yh,
                                                        __half* __restrict__ yl, long long ldp, DevStatus* status) {
  const float s = scale * (scale_dev ? __ldg(scale_dev) : 1.f);
  const long long total = R * (long long)C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C;
    const int c = (int)(i - r * C);
    const float o = y[r * ldy + c] + __ldg(addend + r * lda + c);
    y[r * ldy + c] = o;
    float v = o * s;
    if (!(fabsf(v) < 65504.f)) { report_range(status, 3710); v = fminf(fmaxf(v, -65504.f), 65504.f); }
    const __half hh = __float2half_rn(v);
    yh[r * ldp + c] = hh;
    yl[r * ldp + c] = __float2half_rn(v - __half2float(hh));
  }
}

// d PE / d x applied to a cotangent: dx_j = g[j] + sum_k f_k (w_sin_k cos(f_k x_j) g[3+6k+j] - w_cos_k sin(f_k x_j) g[3+6k+3+j])
// (model/Embedder.py:43-50 order; `bands` = 6 for points, 4 for view directions).  g2: optional second cotangent of the
// same encoding (the SDF network's skip connection), added before the contraction.
__global__ void __launch_bounds__(256) pe_backward_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                          long long ldg, const float* __restrict__ g2, long long ldg2,
                                                          PeWeights pw, int bands, float* __restrict__ dx, long long P,
                                                          int accumulate) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= 3 * P) return;
  const long long p = i / 3;
  const int j = (int)(i - 3 * p);
  const float* gp = g + p * ldg;
  const float* gq = g2 ? g2 + p * ldg2 : nullptr;
  auto G = [&](int e) { return gp[e] + (gq ? gq[e] : 0.f); };
  const float xj = x[i];
  float acc = G(j);
  float f = 1.f;
  for (int k = 0; k < bands; ++k) {
    float sn, cs;
    sincosf(xj * f, &sn, &cs);
    acc += f * (pw.w[2 * k] * cs * G(3 + 6 * k + j) - pw.w[2 * k + 1] * sn * G(3 + 6 * k + 3 + j));
    f *= 2.f;
  }
  dx[i] = accumulate ? dx[i] + acc : acc;
}
// positional encoding written as a saved layer input: out[p * ld + e], e < 3 + 6 * bands (model/Embedder.py:43-50);
// out2 (optional) receives the same row (the SDF network's skip input)
__global__ void __launch_bounds__(256) pe_forward_kernel(const float* __restrict__ x, PeWeights pw, int bands,
                                                         float* __restrict__ out, long long ld, float* __restrict__ out2,
                                                         long long ld2, long long P) {
  const long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (p >= P) return;
  float pe[39];
  positional_encode(x[3 * p], x[3 * p + 1], x[3 * p + 2], pw.w, pe);
  const int n = 3 + 6 * bands;
  for (int e = 0; e < n; ++e) {
    out[p * ld + e] = pe[e];
    if (out2) out2[p * ld2 + e] = pe[e];
  }
}

// positional encoding as a saved layer input AND as operand planes.  One thread per (point, column): consecutive threads write
// consecutive columns (the one-thread-per-point form wrote 39-element rows at a 2 KB stride from every lane: 139 us for 131 k
// points under ncu).  Same arithmetic as positional_encode (common.cuh): w * sin / cos (2^k x), accurate sincosf.
__global__ void __launch_bounds__(256) pe_forward_planes_kernel(const float* __restrict__ x, PeWeights pw, int bands,
                                                                float* __restrict__ out, long long ld, __half* __restrict__ oh,
                                                                __half* __restrict__ ol, long long ldp, long long P) {
  const int n = 3 + 6 * bands;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long p = i / 40;
  const int e = (int)(i - p * 40);
  if (p >= P || e >= n) return;
  float val;
  if (e < 3) {
    val = x[3 * p + e];
  } else {
    const int k = (e - 3) / 6, r = (e - 3) - 6 * k, c = r % 3;
    float s, co;
    sincosf(x[3 * p + c] * (float)(1 << k), &s, &co);
    val = r < 3 ? pw.w[2 * k] * s : pw.w[2 * k + 1] * co;
  }
  if (out) out[p * ld + e] = val;
  const float v = val * kActScale;
  const __half h = __float2half_rn(v);
  oh[p * ldp + e] = h;
  ol[p * ldp + e] = __float2half_rn(v - __half2float(h));
}

int make_plane_tmap(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t row_pitch_elems,
                    uint32_t box_rows = 128) {
  EncodeTiledFn fn = nullptr;
  int s = tensor_map_encoder(&fn);
  if (s) return s;
  if (((uintptr_t)base & 15) != 0 || (row_pitch_elems & 7) != 0) return RECMV_E_SHAPE;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {row_pitch_elems * 2};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)cudaErrorInvalidValue;
}

}  // namespace
}  // namespace recmv

using namespace recmv;

// fp32 [R][C] -> fp16 hi / lo planes of scale (* *scale_dev) * value, optionally transposed ([C][R]); ldp = row stride of the
// planes in elements (multiple of 8).  Weights: scale 1024; activations 64; cotangents 64 with scale_dev = the dyn scale.
extern "C" int recmv_split_planes(const float* in, int64_t ld, int64_t R, int C, float scale, const float* scale_dev,
                                  int transpose, void* hi, void* lo, int64_t ldp, recmv_stream_t stream) {
  if (R < 0 || C <= 0) return RECMV_E_SHAPE;
  if (R == 0) return RECMV_OK;
  if (!in || !hi || !lo) return RECMV_E_NULL;
  void* sd = nullptr;
  int s0 = device_status_record(&sd);
  if (s0) return s0;
  split_planes_kernel<<<stride_grid(R * (int64_t)C, 256, 8), 256, 0, (cudaStream_t)stream>>>(
      in, ld, R, C, scale, scale_dev, transpose, (__half*)hi, (__half*)lo, ldp, (DevStatus*)sd);
  return launch_status();
}

extern "C" int recmv_softplus_tangent_planes(const float* tz, int64_t ldt, const float* a, int64_t lda, const float* h,
                                            int64_t ldh, int64_t rows, int cols, float plane_scale, float* u, int64_t ldu,
                                            void* u_hi, void* u_lo, int64_t ldp, float* inj, int64_t ldi,
                                            recmv_stream_t stream) {
  if (rows < 0 || cols <= 0) return RECMV_E_SHAPE;
  if (rows == 0) return RECMV_OK;
  if (!tz || !a || !h || !u || !u_hi || !u_lo || !inj) return RECMV_E_NULL;
  void* sd = nullptr;
  int s0 = device_status_record(&sd);
  if (s0) return s0;
  softplus_tangent_kernel<<<stride_grid(rows * (int64_t)cols, 256, 8), 256, 0, (cudaStream_t)stream>>>(
      tz, ldt, a, lda, h, ldh, rows, cols, plane_scale, u, ldu, (__half*)u_hi, (__half*)u_lo, ldp, inj, ldi, (DevStatus*)sd);
  return launch_status();
}

extern "C" int recmv_add_split_planes(float* y, int64_t ldy, const float* addend, int64_t lda, int64_t rows, int cols,
                                      float scale, const float* scale_dev, void* y_hi, void* y_lo, int64_t ldp,
                                      recmv_stream_t stream) {
  if (rows < 0 || cols <= 0) return RECMV_E_SHAPE;
  if (rows == 0) return RECMV_OK;
  if (!y || !addend || !y_hi || !y_lo) return RECMV_E_NULL;
  void* sd = nullptr;
  int s0 = device_status_record(&sd);
  if (s0) return s0;
  add_split_kernel<<<stride_grid(rows * (int64_t)cols, 256, 8), 256, 0, (cudaStream_t)stream>>>(
      y, ldy, addend, lda, rows, cols, scale, scale_dev, (__half*)y_hi, (__half*)y_lo, ldp, (DevStatus*)sd);
  return launch_status();
}

extern "C" int recmv_pe_forward(const float* x, const float* pe_w, int bands, float* out, int64_t ld, float* out2,
                                int64_t ld2, int64_t P, recmv_stream_t stream) {
  if (P < 0 || bands < 0 || bands > 6) return RECMV_E_SHAPE;
  if (P == 0) return RECMV_OK;
  if (!x || !pe_w || !out) return RECMV_E_NULL;
  const PeWeights pw = pe_weights(pe_w, bands);
  pe_forward_kernel<<<(unsigned)((P + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, pw, bands, out, ld, out2, ld2, P);
  return launch_status();
}

extern "C" int recmv_pe_backward(const float* x, const float* g, int64_t ldg, const float* g2, int64_t ldg2,
                                 const float* pe_w, int bands, float* dx, int accumulate, int64_t P,
                                 recmv_stream_t stream) {
  if (P < 0 || bands < 0 || bands > 6) return RECMV_E_SHAPE;
  if (P == 0) return RECMV_OK;
  if (!x || !g || !pe_w || !dx) return RECMV_E_NULL;
  const PeWeights pw = pe_weights(pe_w, bands);
  const long long n = 3 * P;
  pe_backward_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, g, ldg, g2, ldg2, pw, bands, dx, P,
                                                                                   accumulate);
  return launch_status();
}

extern "C" int recmv_pe_forward_planes(const float* x, const float* pe_w, int bands, float* out, int64_t ld, void* out_hi,
                                       void* out_lo, int64_t ldp, int64_t P, recmv_stream_t stream) {
  if (P < 0 || bands < 0 || bands > 6) return RECMV_E_SHAPE;
  if (P == 0) return RECMV_OK;
  if (!x || !pe_w || !out_hi || !out_lo) return RECMV_E_NULL;
  const PeWeights pw = pe_weights(pe_w, bands);
  pe_forward_planes_kernel<<<(unsigned)((P * 40 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, pw, bands, out, ld, (__half*)out_hi,
                                                                                          (__half*)out_lo, ldp, P);
  return launch_status();
}

// One layer GEMM with TMA-fed operand planes.
//   forward       (mode 4/5/6 = none / softplus100 / ReLU):  Y = act(pre_scale * (A . B^T) + bias)
//   backward-data (mode 0/1/2 = none / softplus100' / ReLU'): Y = (A . B^T) * out_scale * act'(saved_input), columns >= split
//                 to Y2 without the derivative
// A planes [M][lda_p] (K columns used, scaled 64 [x dyn when a_has_dyn]), B planes [N][ldb_p] (scaled 1024).
// Outputs: Y fp32 [M][ldy]; optional planes of the < split columns, scaled 64 (x dyn when planes_with_dyn).
extern "C" int recmv_mlp_layer_planes(const void* a_hi, const void* a_lo, int64_t lda_p, const void* b_hi, const void* b_lo,
                                      int64_t ldb_p, int64_t M, int N, int K, int mode, const float* bias,
                                      const float* saved_input, int64_t lds, float scale, const float* dyn_scale,
                                      int a_has_dyn, int split, float* Y, int64_t ldy, float* Y2, int64_t ldy2, void* y_hi,
                                      void* y_lo, int64_t ldyp, int planes_with_dyn, recmv_stream_t stream) {
  if (M < 0 || N <= 0 || K <= 0) return RECMV_E_SHAPE;
  if (M == 0) return RECMV_OK;
  if (!a_hi || !a_lo || !b_hi || !b_lo || !Y) return RECMV_E_NULL;
  if (!(mode == 0 || mode == 1 || mode == 2 || mode == 4 || mode == 5 || mode == 6)) return RECMV_E_DTYPE;
  if ((mode == 1 || mode == 2) && !saved_input) return RECMV_E_NULL;
  if ((y_hi == nullptr) != (y_lo == nullptr)) return RECMV_E_NULL;
  if (M > (int64_t)1 << 30) return RECMV_E_RANGE;
  CUtensorMap ta_h, ta_l, tb_h, tb_l;
  int s = make_plane_tmap(&ta_h, a_hi, (uint64_t)K, (uint64_t)M, (uint64_t)lda_p);
  if (!s) s = make_plane_tmap(&ta_l, a_lo, (uint64_t)K, (uint64_t)M, (uint64_t)lda_p);
  if (!s) s = make_plane_tmap(&tb_h, b_hi, (uint64_t)K, (uint64_t)N, (uint64_t)ldb_p);
  if (!s) s = make_plane_tmap(&tb_l, b_lo, (uint64_t)K, (uint64_t)N, (uint64_t)ldb_p);
  if (!s) s = smem_opt_in<gemm3_tma_kernel>((int)kSmemBytes);
  if (s) return s;
  void* sd = nullptr;
  int s0 = device_status_record(&sd);
  if (s0) return s0;
  if (((DevStatus*)sd)->code != 0) return RECMV_E_DEVICE;
  GtParams prm = {};
  prm.D = Y; prm.ldd = ldy; prm.D2 = Y2; prm.ldd2 = ldy2;
  prm.DH = (__half*)y_hi; prm.DL = (__half*)y_lo; prm.ldp = ldyp;
  prm.E = saved_input; prm.lde = lds; prm.bias = bias;
  prm.dyn_scale = a_has_dyn ? dyn_scale : nullptr;
  prm.unscale = scale / (kActScale * kWgtScale);
  prm.plane_scale = kActScale;
  prm.dyn_in_planes = 0;
  if (planes_with_dyn) {
    // cotangent planes carry the dyn scale; when the A planes do not (never the case in backward-data) it would have to be
    // multiplied in separately
    if (!a_has_dyn || !dyn_scale) return RECMV_E_UNSUPPORTED;
    prm.dyn_in_planes = 1;
  }
  prm.M = (int)M; prm.N = N; prm.K = K;
  prm.split = (split > 0 && split < N) ? split : N;
  prm.tiles_m = (int)((M + kBM - 1) / kBM); prm.tiles_n = (N + kBN - 1) / kBN;
  prm.epi = mode; prm.status = (DevStatus*)sd;
  const int total = prm.tiles_m * prm.tiles_n;
  const int grid = total < num_sms() ? total : num_sms();
  gemm3_tma_kernel<<<grid, kThreads, kSmemBytes, (cudaStream_t)stream>>>(ta_h, ta_l, tb_h, tb_l, prm);
  return launch_status();
}

// dW [out_dim][in_dim] (row stride in_dim) = scale * G^T X from the planes the layer GEMMs wrote: g planes [P][ldg_p] hold
// 64 * dyn * g (columns < out_dim), x planes [P][ldx_p] hold 64 * x (columns < in_dim).  workspace: fp32, at least
// recmv_mlp_wgrad_workspace_floats() elements, reused across calls on one stream.
extern "C" size_t recmv_mlp_wgrad_workspace_floats(void) {
  int dev = 0;
  cudaGetDevice(&dev);
  return (size_t)(num_sms() + 16) * (kBM * kBN + kBM);   // tiles x splits <= SMs partial tiles + as many partial row sums
}

extern "C" int recmv_mlp_wgrad_planes(const void* g_hi, const void* g_lo, int64_t ldg_p, const void* x_hi, const void* x_lo,
                                      int64_t ldx_p, int64_t P, int out_dim, int in_dim, float scale, const float* dyn_scale,
                                      float* workspace, float* dW, float* db, recmv_stream_t stream) {
  if (P < 0 || out_dim <= 0 || in_dim <= 0) return RECMV_E_SHAPE;
  if (!g_hi || !g_lo || !x_hi || !x_lo || !workspace || !dW) return RECMV_E_NULL;
  if (P > (int64_t)1 << 30) return RECMV_E_RANGE;
  cudaStream_t st = (cudaStream_t)stream;
  if (P == 0) {
    cudaError_t e0 = cudaMemsetAsync(dW, 0, sizeof(float) * (size_t)out_dim * in_dim, st);
    if (e0 == cudaSuccess && db) e0 = cudaMemsetAsync(db, 0, sizeof(float) * (size_t)out_dim, st);
    return (int)e0;
  }
  CUtensorMap ta_h, ta_l, tb_h, tb_l;
  int s = make_plane_tmap(&ta_h, g_hi, (uint64_t)out_dim, (uint64_t)P, (uint64_t)ldg_p, 64);
  if (!s) s = make_plane_tmap(&ta_l, g_lo, (uint64_t)out_dim, (uint64_t)P, (uint64_t)ldg_p, 64);
  if (!s) s = make_plane_tmap(&tb_h, x_hi, (uint64_t)in_dim, (uint64_t)P, (uint64_t)ldx_p, 64);
  if (!s) s = make_plane_tmap(&tb_l, x_lo, (uint64_t)in_dim, (uint64_t)P, (uint64_t)ldx_p, 64);
  if (s) return s;
  void* sd = nullptr;
  s = device_status_record(&sd);
  if (!s) s = smem_opt_in<gemm3_wgrad_kernel>((int)kSmemBytesWg);
  if (s) return s;
  WgParams prm = {};
  prm.ws = workspace;
  prm.nkb = (P + kBK - 1) / kBK;
  prm.M = out_dim; prm.N = in_dim;
  prm.tiles_m = (out_dim + kBM - 1) / kBM; prm.tiles_n = (in_dim + kBN - 1) / kBN;
  const int tiles = prm.tiles_m * prm.tiles_n;
  int splits = num_sms() / tiles;
  if (splits < 1) splits = 1;
  if ((long long)splits > prm.nkb) splits = (int)prm.nkb;
  prm.splits = splits;
  prm.chunk_kb = 32;
  prm.status = (DevStatus*)sd;
  const long long db_stride = (long long)prm.tiles_m * kBM;
  prm.ws_db = db ? workspace + (size_t)splits * prm.tiles_m * kBM * prm.tiles_n * kBN : nullptr;
  gemm3_wgrad_kernel<<<tiles * splits, kThreads, kSmemBytesWg, st>>>(ta_h, ta_l, tb_h, tb_l, prm);
  s = launch_status();
  if (s) return s;
  const long long ldw = (long long)prm.tiles_n * kBN, split_stride = (long long)prm.tiles_m * kBM * ldw;
  wgrad_reduce_kernel<<<stride_grid((int64_t)out_dim * in_dim, 256, 4), 256, 0, st>>>(
      workspace, splits, split_stride, ldw, out_dim, in_dim, scale / (64.f * 64.f), dyn_scale, dW, in_dim);
  s = launch_status();
  if (s || !db) return s;
  wgrad_reduce_db_kernel<<<(out_dim + 255) / 256, 256, 0, st>>>(prm.ws_db, splits * prm.tiles_n, db_stride, out_dim, dyn_scale, db);
  return launch_status();
}

// out[c] = sum_r g[r][c], c < cols (bias gradient); partial: fp32 scratch of 128 * cols elements
extern "C" int recmv_colsum(const float* g, int64_t ld, int64_t rows, int cols, float* partial, float* out,
                            recmv_stream_t stream) {
  if (rows < 0 || cols <= 0) return RECMV_E_SHAPE;
  if (!g || !partial || !out) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  colsum_partial_kernel<<<dim3((unsigned)((cols + 31) / 32), kCsSlabs), 256, 0, st>>>(g, ld, rows, cols, partial);
  int s = launch_status();
  if (s) return s;
  colsum_final_kernel<<<(cols + 255) / 256, 256, 0, st>>>(partial, cols, out);
  return launch_status();
}

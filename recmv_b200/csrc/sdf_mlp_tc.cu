// Tensor-core implementation of the fused MLP paths (sm_90a: wgmma, TMA, mbarrier).  ONE persistent kernel: for every
// tile of 64 rows it runs  [ray -> x_obs -> skinning-voxel sample -> inverse LBS ->] positional encoding -> 9 linears
// (+softplus) -> sdf / 256 features  with every activation kept on-chip.  Replaces model/Embedder.py:43-50 +
// model/network.py:89-119 (and, in render mode, the Deformer.py:406-445 gather/blend and a FastMinv inverse) for the
// forward path.
//
// Mapping to the hardware (H100, sm_90a):
//  * tensor cores: wgmma.mma_async m64n128k16 (fp16 inputs, fp32 accumulators in registers).  Two consumer warpgroups
//    each own half of a layer's 512 outputs (two 128-column accumulators, 128 registers per thread).  fp32 parity mode
//    (passes = 3): operands are split a = hi + lo in fp16 and every product is 3 MMAs (hi*hi + lo*hi + hi*lo).
//  * weights: fp16 hi/lo panels streamed by TMA from L2, one ring per warpgroup of 5 slots x 8 KB, each slot one
//    [128 outputs x 32 inputs] half of a [128 x 64] weight box (64-byte swizzle), signalled with mbarrier complete_tx; a
//    warpgroup releases a slot as soon as the wgmma commit group that last reads it has retired.
//  * activations: 64 x 512 fp16 hi + lo (128 KB) in shared memory in the K-major SW128 layout, rewritten IN PLACE by
//    the epilogue of the warpgroups once both have finished the layer's MMAs (two named barriers per layer).
//  * warp roles (12 warps): 0-7 the two MMA / epilogue warpgroups; 8, 9 TMA producers (ring of warpgroup 0, 1);
//    10-11 prologue for the NEXT tile (point fetch / inverse LBS / PE, or the input rows of the translator / colour
//    networks).
//  * the same engine runs three networks (Net<0> SDF, Net<1> translator + LBS, Net<2> colour) and a forward-mode
//    (value + tangents, 4 rows per point) variant of the first two.
// Every mbarrier wait is bounded: a protocol bug surfaces as a status code, not a hung GPU.
#include <type_traits>

#include "sdf_mlp.cuh"
#include "tc_common.cuh"
#include "../../include/recmv_b200_diag.h"   // recmv_sdf_mlp_tc_debug (diagnostics entry, not in the product header)

namespace recmv {
using namespace tc;

namespace {

constexpr int kMmaWarps = 8;                      // two warpgroups
constexpr int kProducerWarp = kMmaWarps;          // warps 8, 9: TMA producer of the weight ring of warpgroup 0, 1
constexpr int kPrologueWarp = kProducerWarp + 2;  // warps 10, 11: one thread per tile row
constexpr int kPrologueWarps = 2;
constexpr int kThreads = 32 * (kPrologueWarp + kPrologueWarps);   // 12 warps = three whole warpgroups
constexpr int kRowsPerCta = 64;
// Per-thread register budgets after setmaxnreg.  The launch gives every thread 65536 / 384 = 168 registers and the CTA
// owns exactly that pool, so setmaxnreg.inc can only hand the MMA warpgroups what the third warpgroup (producers +
// prologue) gave back with setmaxnreg.dec; a larger request would wait forever.
constexpr int kLaunchRegs = 168, kMmaRegs = 200, kAuxRegs = 104;
static_assert(kLaunchRegs * kThreads <= 65536, "one CTA per SM at the launch bound");
static_assert(2 * kMmaRegs + kAuxRegs <= 3 * kLaunchRegs && kMmaRegs % 8 == 0 && kAuxRegs % 8 == 0,
              "setmaxnreg: the two MMA warpgroups get what the third one releases");
#ifndef RECMV_TC_TWO_SWEEPS
#define RECMV_TC_TWO_SWEEPS 1   // last layer, parity mode: correction MMAs first, hi*hi MMAs in a second sweep
#endif
constexpr bool kTwoSweeps = RECMV_TC_TWO_SWEEPS != 0;
#ifndef RECMV_TC_STALL_PROF
#define RECMV_TC_STALL_PROF 0   // diagnostics build only (tools/tc_stall_profile.py): per-CTA clock64() stall counters
#endif
constexpr bool kStallProf = RECMV_TC_STALL_PROF != 0;
// Stall counters of the diagnostics build, in SM cycles summed over CTAs.  Consumer counters are taken by thread 0 of
// each MMA warpgroup, producer counters by the producer lane; what a warpgroup does outside them is issuing MMAs.
enum StallCounter {
  kStFull,           // consumer: waits on a FULL barrier (weights not there yet)
  kStWgWait,         // consumer: wgmma.wait_group (tensor pipe still busy with this warpgroup's groups)
  kStEpilogue,       // consumer: softplus / store epilogue of every layer
  kStNamedBar,       // consumer: the two named barriers per hidden layer
  kStPeReady,        // consumer: wait for the prologue's tile input
  kStConsumerTotal,  // consumer: the whole tile loop
  kStEmpty,          // producer: waits on an EMPTY barrier (ring full)
  kStProducerTotal,  // producer: the whole tile loop
  kStCounters
};
// One weight ring per warpgroup.  A slot holds a [128 outputs x 32 inputs] half of a weight box (64-byte swizzle), so a
// box = two consecutive slots; 5 slots let a warpgroup keep two half-boxes in flight beyond the three its MMAs may hold.
constexpr int kSlots = 5;                         // per ring
constexpr uint32_t kSlotBytes = 8192;             // [128 outputs][32 inputs] fp16
// shared memory map (offsets from a 1024-aligned base)
constexpr uint32_t kOffAHi = 0;
constexpr uint32_t kOffALo = 65536;
constexpr uint32_t kOffPeHi = 131072;
constexpr uint32_t kOffPeLo = 139264;
constexpr uint32_t kOffW = 147456;                         // ring g at kOffW + g * kSlots * kSlotBytes
constexpr uint32_t kOffBar = kOffW + 2 * kSlots * kSlotBytes;  // 229376
// barrier indices (8 bytes each)
constexpr int kBarFull = 0;      // [2][5] weight slot filled (1 arming arrival + tx bytes)
constexpr int kBarEmpty = 10;    // [2][5] slot consumed (one arrival by the ring's warpgroup)
constexpr int kBarPeReady = 20;  //       tile input written by the prologue warps (one arrival per warp)
constexpr int kBarPeFree = 21;   //       the MMAs of layer kInFreeLayer are done with the tile input (one arrival per warpgroup)
constexpr int kNumBars = 22;
constexpr int kBarConsumers = 1; // named barrier of the 256 MMA threads
constexpr uint32_t kOffMisc = kOffBar + kNumBars * 8;  // abort flag, valid flags
// SDF forward: warpgroup 1's share of each row's sdf sum, [64] fp32.  One buffer is enough: warpgroup 0 reads it before
// the next tile's layer-0 named barriers, and warpgroup 1 writes it again only in the next tile's layer 7.
constexpr uint32_t kOffSdfPart = kOffMisc + 16 + 128;
constexpr uint32_t kOffProf = kOffSdfPart + 64 * 4;    // diagnostics build: [4 roles][kStCounters] u64
constexpr uint32_t kSmemBytes = kOffProf + (kStallProf ? 4 * kStCounters * 8 : 0) + 1024 /*alignment slack*/;
static_assert(kSmemBytes <= 227 * 1024, "shared memory: within the per-block opt-in");
#if RECMV_TC_STALL_PROF
__device__ unsigned long long g_tc_stall[kStCounters];   // read and cleared by recmv_tc_stall_profile
#endif

struct TcParams {
  PointSource src;
  PeWeights pw;
  const float* bias;  // [9][512] padded
  float* out_sdf;
  float* out_feat;
  long long P;
  const int* P_dev;   // optional: actual point count in device memory (<= P)
  int passes;
  float acc_gain_kb;  // relative accumulator gain per 64-wide K block of a layer (4 accumulating MMAs)
  DevStatus* status;
  // diagnostics: raw accumulator (before bias) of layer dbg_layer for tile 0 -> dbg_out [64][512]
  int dbg_layer;
  float* dbg_out;
  // forward-mode (JVP) variant: out_grad [P,3] = d sdf / d x; each point occupies 4 adjacent tile rows
  float* out_grad;
  // deformer network (kNet == 1): MLPTranslator 167 -> 512 x4 -> 3 (ReLU) followed by LBS forward
  const float* conds;            // [F,128]
  const long long* batch_inds;   // [P] or NULL (frame = p / points_per_frame)
  long long points_per_frame;
  int num_frames;
  const float* bones;            // A [F,24,4,4] (NULL: translator only)
  const float* trans;            // [F,3]
  Voxel vox;
  float* out_translated;         // [P,3]  p + delta
  float* out_offset;             // [P,3]  delta (MLPTranslator.offset), optional
  float* out_posed;              // [P,3]  LBS(p + delta), optional
  float* out_jac;                // [P,9]  forward-mode variant: d out / d p (row i = gradient of output i)
  // colour network (kNet == 2): cat[p, PE4(view), n, feat] = 289 -> 512 x4 (ReLU) -> 3 -> tanh; src.x = points
  const float* normals;          // [P,3]
  const float* view_dirs;        // [P,3]
  const float* feats;            // [P,256]
  float* out_rgb;                // [P,3]
  // SDF network: 128-wide output tiles of the last layer, 3 with features.  Without them: 0 for the plain forward in
  // parity mode (its sdf comes from layer 7's epilogue either way), otherwise 1 (tile 0 holds the sdf).
  int last_tiles;
  // SDF network: layer 8's weight row n = 0 (the sdf column) in the hi plane of the panels, [8 panels][512 n][64 k]
  // apart; the lo plane lies kPanels * 512 * 64 halves further
  const __half* sdf_w;
};

// softplus(beta=100, threshold=20) * kActScale straight from the raw accumulator, in base 2:
//   u = acc * (2^-16 * 100 log2 e) + b * 100 log2 e  (the bias plane is pre-multiplied at pack time)
//   u <= 20 log2 e : ln2/100 * log2(1 + 2^u)     else : z = u / (100 log2 e)        (torch's threshold branch)
// ex2/lg2 .ftz skip the denormal range fix-ups of __expf/__logf.
__device__ __forceinline__ float ex2_ftz(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float lg2_ftz(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float softplus100_scaled(float acc, float bias_u, float kU1 /* acc unscale * 100 log2 e */) {
  constexpr float kUThr = 20.f * 1.4426950408889634f;
  constexpr float kC1 = 0.0069314718055994531f * kActScale;    // ln2 / 100
  constexpr float kC2 = kActScale / kSoftplusLog2Scale;
  const float u = fmaf(acc, kU1, bias_u);
  const float y = lg2_ftz(1.f + ex2_ftz(fminf(u, kUThr))) * kC1;
  return u > kUThr ? u * kC2 : y;
}

// value row: softplus100(z); tangent row: z_tangent * sigmoid(100 z_value)  (d softplus / dz; torch's
// threshold branch z > 0.2 has derivative 1, which sigmoid(20+) equals to 2e-9)
__device__ __forceinline__ float act_jvp(float z_own, float z_val, bool is_value) {
  const float t = 100.f * z_val;
  const float e = __expf(-fabsf(t));
  const float inv = __fdividef(1.f, 1.f + e);
  const float sp = t > 20.f ? z_val : (fmaxf(t, 0.f) + __logf(1.f + e)) * 0.01f;
  const float sig = t >= 0.f ? inv : e * inv;
  return is_value ? sp : z_own * sig;
}

// tangent row j of the forward-mode variants: d PE / d x_j  (x -> e_j ; w sin(f x_c) -> w f cos(f x_c) [c == j] ;
// w cos(f x_c) -> -w f sin(f x_c) [c == j])
__device__ __forceinline__ void positional_encode_tangent(float cx, float cy, float cz, int j, const float* pw, float* pe) {
  const float xj = j == 0 ? cx : (j == 1 ? cy : cz);
#pragma unroll
  for (int e = 0; e < 39; ++e) pe[e] = 0.f;
  pe[j] = 1.f;
  float f = 1.f;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    float sn, cs;
    sincosf(xj * f, &sn, &cs);
    pe[3 + 6 * k + j] = pw[2 * k] * f * cs;
    pe[3 + 6 * k + 3 + j] = -pw[2 * k + 1] * f * sn;
    f *= 2.f;
  }
}

// The MMAs of one weight box (one 64-wide K block x one 128-wide output tile x one weight plane) into accumulator `acc`.
// The box arrives as two ring slots, b0 = inputs 0..31 and b1 = inputs 32..63 (K steps 0, 1 and 2, 3), and its MMAs
// form two commit groups: the first is the last to read b0, the second reads b1 only, so b0 is released one group
// before b1.  Straight-line code with a fixed accumulator: wgmma.fence ... commit holds no branch, which lets ptxas keep
// the MMAs in flight instead of serialising them.  Per accumulator element the order of the products is
//   box_mmas:        a . w            K steps 0..3        (tc1; parity mode: the w_lo box and every two-sweep box)
//   box_mmas_hi_lo:  a_hi . w_hi      K steps 0..3, then a_lo . w_hi K steps 0..3      (parity mode, the w_hi box)
// Parity mode, last layer (two sweeps): sweep 0 plane 0: a_lo . w_hi;  plane 1: a_hi . w_lo;  sweep 1: a_hi . w_hi (the
// tensor core accumulates with truncation, so every MMA added to a LARGE accumulator costs ~1 ulp of it; the correction
// products are 2^-11 of the result and issued first, while the accumulator is still tiny.)
// scale0 = 0: the first MMA overwrites the accumulator.
__device__ __forceinline__ void box_mmas(float (&acc)[64], uint64_t a, uint64_t b0, uint64_t b1, uint32_t scale0) {
  wg_fence();
  wgmma_n128<0, 0>(acc, a, b0, scale0);
  wgmma_n128<0, 0>(acc, a + 2, b0 + 2, 1u);
  wg_commit();
  wgmma_n128<0, 0>(acc, a + 4, b1, 1u);
  wgmma_n128<0, 0>(acc, a + 6, b1 + 2, 1u);
  wg_commit();
}
__device__ __forceinline__ void box_mmas_hi_lo(float (&acc)[64], uint64_t a_hi, uint64_t a_lo, uint64_t b0, uint64_t b1,
                                               uint32_t scale0) {
  wg_fence();
  wgmma_n128<0, 0>(acc, a_hi, b0, scale0);
  wgmma_n128<0, 0>(acc, a_hi + 2, b0 + 2, 1u);
  wgmma_n128<0, 0>(acc, a_hi + 4, b1, 1u);
  wgmma_n128<0, 0>(acc, a_hi + 6, b1 + 2, 1u);
  wgmma_n128<0, 0>(acc, a_lo, b0, 1u);
  wgmma_n128<0, 0>(acc, a_lo + 2, b0 + 2, 1u);
  wg_commit();
  wgmma_n128<0, 0>(acc, a_lo + 4, b1, 1u);
  wgmma_n128<0, 0>(acc, a_lo + 6, b1 + 2, 1u);
  wg_commit();
}

// output tiles of a layer with T tiles that warpgroup g owns (tiles 2 g, 2 g + 1): 0, 1 or 2
__device__ __forceinline__ int own_tiles(int T, int g) { return min(max(T - 2 * g, 0), 2); }

}  // namespace

// kPasses: 3 = parity mode (hi * hi + lo * hi + hi * lo), 1 = hi * hi only (TcParams::passes must agree)
template <bool kJvp, int kNet, int kPasses>
__global__ void __launch_bounds__(kThreads, 1)
sdf_tc_kernel(const __grid_constant__ CUtensorMap tmap, const TcParams prm) {
  using NetT = Net<kNet>;
  constexpr int kNumLayers = NetT::kLayers;
  constexpr bool kSdfFwd = !kJvp && kNet == 0;   // the SDF network's plain forward
  // parity mode: the sdf column is folded into layer 7's epilogue (tc1 keeps it on the tensor cores: DESIGN.md section 5)
  constexpr bool kFoldSdf = kSdfFwd && kPasses == 3;
  static_assert(!kJvp || kNet == 0 || kNet == 1, "the forward-mode variant exists for the SDF network and the deformer");
  static_assert(kPasses == 1 || kPasses == 3, "precision mode");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t bar0 = base + kOffBar;
  volatile int* abort_flag = reinterpret_cast<volatile int*>(gbase + kOffMisc + 4);
  volatile unsigned char* valid = reinterpret_cast<volatile unsigned char*>(gbase + kOffMisc + 16);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kPtsPerTile = kJvp ? kRowsPerCta / 4 : kRowsPerCta;  // JVP: rows = 4 per point (value, d/dx, d/dy, d/dz)
  // number of points: by value, or -- device worklists (coarse-to-fine sweep) -- read from device memory, bounded by
  // the capacity prm.P the grid was sized for
  const long long Ptot = prm.P_dev ? (long long)min((long long)max(__ldg(prm.P_dev), 0), prm.P) : prm.P;
  const long long num_tiles = (Ptot + kPtsPerTile - 1) / kPtsPerTile;
  const long long n_iter = (long long)blockIdx.x < num_tiles ? (num_tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
  auto tile_of = [&](long long it) { return (long long)blockIdx.x + it * gridDim.x; };
  auto BAR = [&](int i) { return bar0 + 8u * (uint32_t)i; };
  // slot s of the weight ring of warpgroup g, its full / empty barriers
  auto SLOT = [&](int g, int s) { return base + kOffW + (uint32_t)(g * kSlots + s) * kSlotBytes; };
  auto FULL = [&](int g, int s) { return BAR(kBarFull + g * kSlots + s); };
  auto EMPTY = [&](int g, int s) { return BAR(kBarEmpty + g * kSlots + s); };
  // diagnostics build: the stall counters of role r (0, 1: MMA warpgroup g; 2, 3: producer of ring g), kept by one
  // thread each in shared memory and added to g_tc_stall when its loop ends
  auto stall_begin = [&](bool mine, int r) -> unsigned long long* {
    unsigned long long* c = reinterpret_cast<unsigned long long*>(gbase + kOffProf) + r * kStCounters;
    if (kStallProf && mine)
      for (int k = 0; k < kStCounters; ++k) c[k] = 0;
    return c;
  };
  auto stall_now = [&]() -> long long { return kStallProf ? clock64() : 0; };
  auto stall_add = [&](unsigned long long* c, bool mine, int k, long long t0) {
    if (kStallProf && mine) c[k] += (unsigned long long)(clock64() - t0);
  };
  auto stall_end = [&](unsigned long long* c, bool mine) {
#if RECMV_TC_STALL_PROF
    if (mine)
      for (int k = 0; k < kStCounters; ++k) atomicAdd(&g_tc_stall[k], c[k]);
#endif
    (void)c; (void)mine;
  };

  if (threadIdx.x == 0) {
    *abort_flag = 0;
    for (int s = 0; s < 2 * kSlots; ++s) { mbar_init(BAR(kBarFull + s), 1); mbar_init(BAR(kBarEmpty + s), 1); }
    mbar_init(BAR(kBarPeReady), kPrologueWarps);
    mbar_init(BAR(kBarPeFree), 2);
    fence_mbar_init();
  }
  if (warp >= kProducerWarp && warp < kPrologueWarp && lane == 0) prefetch_tmap(&tmap);
  __syncthreads();

  if (warp < kMmaWarps) {
    // the two MMA warpgroups take the registers the third one released (two accumulators + the epilogue)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kMmaRegs));
    // ================================ MMA warpgroups + epilogue =========================================
    const int g = warp >> 2, wq = warp & 3;
    const bool signaller = (threadIdx.x & 127) == 0;
    const int c = lane & 3;                        // column pair of the fragment
    const int comp = kJvp ? ((lane >> 2) & 3) : 0; // JVP: 0 = value row, 1..3 = tangent rows (same for both fragment rows)
    const bool is_value = comp == 0;
    float acc[2][64];   // output tiles 2 g and 2 g + 1
#pragma unroll
    for (int i = 0; i < 64; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    // this warpgroup's ring: next slot to consume, parity of its pass, and the slot its in-flight MMAs still read
    int slot = 0, held = -1, s0 = 0, s1 = 0;
    uint32_t phase = 0;
    // wait for the next box (two slots) and return its B descriptors
    unsigned long long* stall = stall_begin(signaller, g);
    auto acquire = [&](uint64_t& b0, uint64_t& b1) {
      const long long t0 = stall_now();
      s0 = slot;
      mbar_wait(FULL(g, slot), phase, abort_flag, prm.status, 230 + g * kSlots + slot);
      if (++slot == kSlots) { slot = 0; phase ^= 1u; }
      s1 = slot;
      mbar_wait(FULL(g, slot), phase, abort_flag, prm.status, 230 + g * kSlots + slot);
      if (++slot == kSlots) { slot = 0; phase ^= 1u; }
      stall_add(stall, signaller, kStFull, t0);
      b0 = smem_desc_sw64(SLOT(g, s0));
      b1 = smem_desc_sw64(SLOT(g, s1));
    };
    // once the box's first commit group has retired: release its first half and the previous box's second half (whose
    // group retired before it); the second half stays held until the next box's first group has retired
    auto retire = [&]() {
      const long long t0 = stall_now();
      wg_wait<1>();
      stall_add(stall, signaller, kStWgWait, t0);
      if (signaller) {
        if (held >= 0) mbar_arrive_local(EMPTY(g, held));
        mbar_arrive_local(EMPTY(g, s0));
      }
      held = s1;
    };
    const long long t_loop = stall_now();
    for (long long it = 0; it < n_iter; ++it) {
      const long long tile = tile_of(it);
      for (int l = 0; l < kNumLayers; ++l) {
        if (l == 0) {
          const long long t0 = stall_now();
          mbar_wait(BAR(kBarPeReady), (uint32_t)(it & 1), abort_flag, prm.status, 220);
          stall_add(stall, signaller, kStPeReady, t0);
        }
        const int nkb = NetT::nkb(l), T = NetT::ntiles(l, prm.last_tiles), nt_own = own_tiles(T, g);
        if (kFoldSdf && T == 0) continue;   // the last layer without features: the producers stream nothing for it
        const bool hidden = l < kNumLayers - 1;
        const bool two_sweeps = kTwoSweeps && kPasses == 3 && l == kNumLayers - 1;
        // the layer's first MMA overwrites the accumulators; zeroing them here tells the compiler that the previous
        // layer's values are dead once its epilogue has read them
#pragma unroll
        for (int i = 0; i < 64; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
        for (int sweep = 0; sweep < (two_sweeps ? 2 : 1); ++sweep) {
          for (int i = 0; i < nkb; ++i) {
            const int kbi = NetT::kb_at(l, i);
            const bool is_pe = kbi == 8;
            const uint64_t a_hi = smem_desc_sw128(is_pe ? base + kOffPeHi : base + kOffAHi + kbi * 8192);
            const uint64_t a_lo = smem_desc_sw128(is_pe ? base + kOffPeLo : base + kOffALo + kbi * 8192);
            const uint32_t scale0 = (sweep == 0 && i == 0) ? 0u : 1u;   // the layer's first MMA overwrites
#pragma unroll
            for (int t = 0; t < 2; ++t) {
              if (t >= nt_own) continue;   // warpgroup-uniform: a tile this warpgroup does not own in this layer
              uint64_t b0, b1;
              if (kPasses == 1) {
                acquire(b0, b1);
                box_mmas(acc[t], a_hi, b0, b1, scale0);
                retire();
              } else if (!two_sweeps) {
                acquire(b0, b1);                                   // w_hi
                box_mmas_hi_lo(acc[t], a_hi, a_lo, b0, b1, scale0);
                retire();
                acquire(b0, b1);                                   // w_lo
                box_mmas(acc[t], a_hi, b0, b1, 1u);
                retire();
              } else if (sweep == 0) {
                acquire(b0, b1);                                   // w_hi: a_lo . w_hi
                box_mmas(acc[t], a_lo, b0, b1, scale0);
                retire();
                acquire(b0, b1);                                   // w_lo: a_hi . w_lo
                box_mmas(acc[t], a_hi, b0, b1, 1u);
                retire();
              } else {
                acquire(b0, b1);                                   // w_hi: a_hi . w_hi
                box_mmas(acc[t], a_hi, b0, b1, 1u);
                retire();
              }
            }
          }
        }
        long long t_ep = stall_now();
        wg_wait<0>();
        wg_fence_regs(acc[0]);
        wg_fence_regs(acc[1]);
        stall_add(stall, signaller, kStWgWait, t_ep);
        if (held >= 0 && signaller) mbar_arrive_local(EMPTY(g, held));
        held = -1;
        if (l == NetT::kInFreeLayer && signaller) mbar_arrive_local(BAR(kBarPeFree));   // prologue may refill its block

        const float* bias = prm.bias + l * 512;
        // 2^-16 x (1 + compensation of the tensor core's truncating accumulation: every one of the K/16 hi*hi MMAs that
        // adds into the full-size fp32 accumulator drops on average ~2^-24 of it; recmv_tc_set_acc_gain)
        const float acc_unscale = kAccUnscale * (1.f + prm.acc_gain_kb * (float)nkb);
        const float acc_u1 = acc_unscale * kSoftplusLog2Scale;
        if (hidden) {
          t_ep = stall_now();
          named_sync(kBarConsumers, 256);   // both warpgroups are done reading the layer input: overwrite it in place
          stall_add(stall, signaller, kStNamedBar, t_ep);
          t_ep = stall_now();
          const float* bsel = kSdfFwd ? bias + kNumLayers * 512 : bias;   // SDF: the b * 100 log2 e plane
          // SDF forward, layer 7: the sdf column of layer 8, sum_k v_k w_k over this thread's columns per fragment row
          float sdf_part[2] = {0.f, 0.f};
          // The loop body holds no per-element branch: an operand beyond fp16's range is reported once per layer (same tag),
          // the diagnostics dump branches once per column group, and the activation stores are plain C++ stores (no asm
          // memory clobber), so ptxas can overlap the bias loads and MUFU chains of neighbouring elements.  The epilogue
          // runs with two warps per scheduler and is latency-bound.  A pass either writes the activation planes (the next
          // layer's input) or, kFold, sums the sdf column into sdf_part; the choice is made once per layer.  Both in one
          // pass would hold the weight pairs and row sums next to the stores' operands, and that spills in the SDF
          // kernels at 200 registers.  The fold pass dumps before its loop, which then has no branch at all: ptxas can
          // issue the weight loads of later column groups early (DESIGN.md section 9 has the measurement).
          auto epilogue = [&](auto fold) {
            constexpr bool kFold = decltype(fold)::value;
            bool out_of_range = false;
            if (kFold && prm.dbg_out && prm.dbg_layer == l && tile == 0) {
#pragma unroll
              for (int t = 0; t < 2; ++t)
#pragma unroll
                for (int i = 0; i < 64; ++i)
                  prm.dbg_out[(16 * wq + (lane >> 2) + 8 * ((i >> 1) & 1)) * 512 + (2 * g + t) * 128 + 8 * (i >> 2) +
                              2 * c + (i & 1)] = acc[t][i] * kAccUnscale;
            }
#pragma unroll
            for (int t = 0; t < 2; ++t) {
              const int f_base = (2 * g + t) * 128 + 2 * c;
              // column pair j outer, fragment row h inner: each bias pair is used as soon as it is loaded (the other order
              // keeps a tile's 16 bias pairs live next to the 128 accumulator registers)
#pragma unroll
              for (int j = 0; j < 16; ++j) {
                const int f = f_base + 8 * j;
                if (!kFold && prm.dbg_out && prm.dbg_layer == l && tile == 0) {
#pragma unroll
                  for (int i = 0; i < 4; ++i)
                    prm.dbg_out[(16 * wq + (lane >> 2) + 8 * (i >> 1)) * 512 + f + (i & 1)] = acc[t][4 * j + i] * kAccUnscale;
                }
                float2 w = make_float2(0.f, 0.f);   // layer 8's weights of columns f, f + 1 into the sdf: hi + lo
                if (kFold) {
                  const __half* wp = prm.sdf_w + (f >> 6) * (512 * 64) + (f & 63);
                  const float2 w_hi = __half22float2(__ldg(reinterpret_cast<const __half2*>(wp)));
                  const float2 w_lo = __half22float2(__ldg(reinterpret_cast<const __half2*>(wp + NetT::kPanels * 512 * 64)));
                  w = make_float2(w_hi.x + w_lo.x, w_hi.y + w_lo.y);
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const int row = 16 * wq + (lane >> 2) + 8 * h;
                  const float r0 = acc[t][4 * j + 2 * h];
                  const float r1 = acc[t][4 * j + 2 * h + 1];
                  const float2 bb = __ldg(reinterpret_cast<const float2*>(bsel + f));
                  float v0, v1;
                  if (kSdfFwd) {
                    v0 = softplus100_scaled(r0, bb.x, acc_u1);
                    v1 = softplus100_scaled(r1, bb.y, acc_u1);
                  } else if (!kJvp) {
                    v0 = fmaxf(fmaf(r0, acc_unscale, bb.x), 0.f) * kActScale;   // ReLU (deformer, colour)
                    v1 = fmaxf(fmaf(r1, acc_unscale, bb.y), 0.f) * kActScale;
                  } else {
                    const float z0 = is_value ? fmaf(r0, acc_unscale, bb.x) : r0 * acc_unscale;   // tangents: no bias
                    const float z1 = is_value ? fmaf(r1, acc_unscale, bb.y) : r1 * acc_unscale;
                    const float zv0 = __shfl_sync(0xffffffffu, z0, lane & ~12);   // the point's value row
                    const float zv1 = __shfl_sync(0xffffffffu, z1, lane & ~12);
                    v0 = (kNet == 0 ? act_jvp(z0, zv0, is_value) : (zv0 > 0.f ? z0 : 0.f)) * kActScale;
                    v1 = (kNet == 0 ? act_jvp(z1, zv1, is_value) : (zv1 > 0.f ? z1 : 0.f)) * kActScale;
                  }
                  if (kFold) {
                    sdf_part[h] = fmaf(v0, w.x, sdf_part[h]);
                    sdf_part[h] = fmaf(v1, w.y, sdf_part[h]);
                  } else {
                    out_of_range |= !(fmaxf(fabsf(v0), fabsf(v1)) < 65504.f);
                    uint32_t hi, lo;
                    split2(v0, v1, hi, lo);
                    const uint32_t off = (uint32_t)(f >> 6) * 8192u + sw128_elem(row, f & 63);
                    *reinterpret_cast<uint32_t*>(gbase + kOffAHi + off) = hi;
                    if (kPasses == 3) *reinterpret_cast<uint32_t*>(gbase + kOffALo + off) = lo;
                  }
                }
              }
            }
            if (out_of_range) report_range(prm.status, 1000 + l);
          };
          const bool fold = kFoldSdf && l == kNumLayers - 2;
          // layer 7 of the SDF forward writes its output only for the features of layer 8
          if (!fold || prm.last_tiles > 0) epilogue(std::false_type{});
          if constexpr (kFoldSdf) {   // the fold pass is instantiated in these kernels only
            if (fold) epilogue(std::true_type{});
          }
          if (kFoldSdf && fold) {
            // the row sums over the quad's four column pairs, then warpgroup 1 hands its share to warpgroup 0
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              sdf_part[h] += __shfl_xor_sync(0xffffffffu, sdf_part[h], 1);
              sdf_part[h] += __shfl_xor_sync(0xffffffffu, sdf_part[h], 2);
              if (g == 1 && c == 0)
                reinterpret_cast<float*>(gbase + kOffSdfPart)[16 * wq + (lane >> 2) + 8 * h] = sdf_part[h];
            }
          }
          fence_proxy_async();
          stall_add(stall, signaller, kStEpilogue, t_ep);
          t_ep = stall_now();
          named_sync(kBarConsumers, 256);   // the next layer's input (SDF, layer 7: warpgroup 1's sdf sums) is complete
          stall_add(stall, signaller, kStNamedBar, t_ep);
          if (kFoldSdf && fold && g == 0 && c == 0) {
            // sdf = (s0 + s1) 2^-16 + b8[0]: both scales of the operands undone, the last layer's bias added
            const float b8 = __ldg(prm.bias + (kNumLayers - 1) * 512);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = 16 * wq + (lane >> 2) + 8 * h;
              const long long p = tile * kPtsPerTile + row;
              const float s1 = reinterpret_cast<const float*>(gbase + kOffSdfPart)[row];
              if (p < Ptot)
                prm.out_sdf[p] = valid[(it & 1) * 64 + row] != 0 ? fmaf(sdf_part[h] + s1, kAccUnscale, b8) : kInvalidSdf;
            }
          }
          continue;
        }
        // ---- last layer ----
        t_ep = stall_now();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = 16 * wq + (lane >> 2) + 8 * h;
          const long long p = kJvp ? tile * kPtsPerTile + (row >> 2) : tile * kPtsPerTile + row;
          if (kNet == 0) {
            const bool ok = valid[(it & 1) * 64 + row] != 0;
#pragma unroll
            for (int t = 0; t < 2; ++t) {
              if (2 * g + t >= T || p >= Ptot) continue;
#pragma unroll
              for (int j = 0; j < 16; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const int f = (2 * g + t) * 128 + 8 * j + 2 * c + e;
                  const float r = acc[t][4 * j + 2 * h + e];
                  if (prm.dbg_out && prm.dbg_layer == l && tile == 0) prm.dbg_out[row * 512 + f] = r * kAccUnscale;
                  // column 0 = sdf (kFoldSdf: stored from layer 7's epilogue), columns 1..256 = features
                  if (kJvp && !is_value) {
                    if (f == 0) prm.out_grad[p * 3 + (comp - 1)] = r * acc_unscale;
                  } else if (f == 0) {
                    if (!kFoldSdf) prm.out_sdf[p] = ok ? fmaf(r, acc_unscale, __ldg(bias)) : kInvalidSdf;
                  } else if (f <= 256 && prm.out_feat) {
                    prm.out_feat[p * 256 + (f - 1)] = fmaf(r, acc_unscale, __ldg(bias + f));
                  }
                }
              }
            }
          } else if (kNet == 2) {
            // colour network: columns 0..2 -> tanh
            if (g == 0 && p < Ptot) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int f0 = 2 * c + e, f1 = 8 + 2 * c + e;
                (void)f1;
                if (f0 < 3) prm.out_rgb[3 * p + f0] = tanhf(fmaf(acc[0][2 * h + e], acc_unscale, __ldg(bias + f0)));
              }
            }
          } else if (g == 0) {
            // deformer: columns 0..2 = offset; out = p + offset, then LBS forward.  Columns 0, 1 live in lane 4 r, column 2
            // in lane 4 r + 1 of the fragment row: gather them (warp-uniform shuffles)
            const float own0 = acc[0][2 * h] * acc_unscale, own1 = acc[0][2 * h + 1] * acc_unscale;
            const float v[3] = {__shfl_sync(0xffffffffu, own0, lane & ~3), __shfl_sync(0xffffffffu, own1, lane & ~3),
                                __shfl_sync(0xffffffffu, own0, (lane & ~3) + 1)};
            if (kJvp) {
              // rows 4i..4i+3 = (value, d/dx, d/dy, d/dz) in lanes 16 i' + 4 k; offset and d offset_c / d p_j
              float dv[3], dt[9];
#pragma unroll
              for (int cc = 0; cc < 3; ++cc) {
                dv[cc] = v[cc] + __ldg(bias + cc);
#pragma unroll
                for (int j = 0; j < 3; ++j) dt[3 * cc + j] = __shfl_sync(0xffffffffu, v[cc], (lane & 16) + 4 * (1 + j));
              }
              if (is_value && c == 0 && p < Ptot) {
                const float x = __ldg(prm.src.x + 3 * p), y = __ldg(prm.src.x + 3 * p + 1), z = __ldg(prm.src.x + 3 * p + 2);
                const float tx = x + dv[0], ty = y + dv[1], tz = z + dv[2];
                dt[0] += 1.f; dt[4] += 1.f; dt[8] += 1.f;   // d (p + offset) / d p
                if (prm.out_translated) { prm.out_translated[3 * p] = tx; prm.out_translated[3 * p + 1] = ty; prm.out_translated[3 * p + 2] = tz; }
                if (prm.out_offset) { prm.out_offset[3 * p] = dv[0]; prm.out_offset[3 * p + 1] = dv[1]; prm.out_offset[3 * p + 2] = dv[2]; }
                if (prm.out_posed) {
                  long long fr = prm.batch_inds ? prm.batch_inds[p] : (prm.points_per_frame > 0 ? p / prm.points_per_frame : 0);
                  fr = fr < 0 ? 0 : (fr >= prm.num_frames ? prm.num_frames - 1 : fr);
                  float o[3], Jl[9];
                  lbs_forward_jac(prm.vox, prm.bones + (size_t)fr * 384, prm.trans + 3 * fr, tx, ty, tz, o, Jl);
#pragma unroll
                  for (int i = 0; i < 3; ++i) {
                    prm.out_posed[3 * p + i] = o[i];
#pragma unroll
                    for (int j = 0; j < 3; ++j)
                      prm.out_jac[9 * p + 3 * i + j] = Jl[3 * i] * dt[j] + Jl[3 * i + 1] * dt[3 + j] + Jl[3 * i + 2] * dt[6 + j];
                  }
                } else {
#pragma unroll
                  for (int e = 0; e < 9; ++e) prm.out_jac[9 * p + e] = dt[e];
                }
              }
            } else if (c == 0 && p < Ptot) {
              const float dx = v[0] + __ldg(bias + 0), dy = v[1] + __ldg(bias + 1), dz = v[2] + __ldg(bias + 2);
              const float x = __ldg(prm.src.x + 3 * p), y = __ldg(prm.src.x + 3 * p + 1), z = __ldg(prm.src.x + 3 * p + 2);
              const float tx = x + dx, ty = y + dy, tz = z + dz;
              if (prm.out_translated) { prm.out_translated[3 * p] = tx; prm.out_translated[3 * p + 1] = ty; prm.out_translated[3 * p + 2] = tz; }
              if (prm.out_offset) { prm.out_offset[3 * p] = dx; prm.out_offset[3 * p + 1] = dy; prm.out_offset[3 * p + 2] = dz; }
              if (prm.out_posed) {
                long long fr = prm.batch_inds ? prm.batch_inds[p] : (prm.points_per_frame > 0 ? p / prm.points_per_frame : 0);
                fr = fr < 0 ? 0 : (fr >= prm.num_frames ? prm.num_frames - 1 : fr);
                float w[24], Tm[12];
                sample_skin24(prm.vox, tx, ty, tz, w);
                blend_bones(prm.bones + (size_t)fr * 384, w, Tm);
                const float* tr = prm.trans + 3 * fr;
                prm.out_posed[3 * p + 0] = (Tm[0] * tx + Tm[1] * ty + Tm[2] * tz + Tm[3]) + __ldg(tr + 0);
                prm.out_posed[3 * p + 1] = (Tm[4] * tx + Tm[5] * ty + Tm[6] * tz + Tm[7]) + __ldg(tr + 1);
                prm.out_posed[3 * p + 2] = (Tm[8] * tx + Tm[9] * ty + Tm[10] * tz + Tm[11]) + __ldg(tr + 2);
              }
            }
          }
        }
        stall_add(stall, signaller, kStEpilogue, t_ep);
      }
    }
    stall_add(stall, signaller, kStConsumerTotal, t_loop);
    stall_end(stall, signaller);
  } else {
    // producers and prologue: one setmaxnreg for the whole warpgroup (.aligned), before it splits into roles
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kAuxRegs));
    if (warp < kPrologueWarp) {
      // ====== TMA producers: warp 8 + g streams the weight boxes of warpgroup g, in the order that warpgroup consumes them ======
      const int g = warp - kProducerWarp;
      if (lane == 0) {
        unsigned long long* stall = stall_begin(true, 2 + g);
        const long long t_loop = stall_now();
        int slot = 0;
        uint32_t phase = 0;   // parity of the ring's current pass
        for (long long it = 0; it < n_iter; ++it) {
          for (int l = 0; l < kNumLayers; ++l) {
            const int nkb = NetT::nkb(l), nt_own = own_tiles(NetT::ntiles(l, prm.last_tiles), g);
            // last layer, parity mode: sweep 0 streams (w_hi, w_lo) for the correction MMAs, sweep 1 streams w_hi again
            const int nsweep = (kTwoSweeps && kPasses == 3 && l == kNumLayers - 1) ? 2 : 1;
            for (int sweep = 0; sweep < nsweep; ++sweep) {
              const int nplanes = (kPasses == 3 && sweep == 0) ? 2 : 1;
              for (int i = 0; i < nkb; ++i) {
                const int kbi = NetT::kb_at(l, i);
                const int panel = NetT::pbase(l) + (kbi == 8 ? nkb - 1 : kbi);   // the PE block is the layer's last panel
                for (int t = 0; t < nt_own; ++t) {
                  for (int plane = 0; plane < nplanes; ++plane) {
                    for (int half = 0; half < 2; ++half) {
                      const long long t0 = stall_now();
                      mbar_wait(EMPTY(g, slot), phase ^ 1u, abort_flag, prm.status, 100 + g * kSlots + slot);
                      stall_add(stall, true, kStEmpty, t0);
                      mbar_expect_tx_local(FULL(g, slot), kSlotBytes);
                      tma_load_2d(SLOT(g, slot), &tmap, FULL(g, slot), 32 * half,
                                  (plane * NetT::kPanels + panel) * 512 + (2 * g + t) * 128);
                      if (++slot == kSlots) { slot = 0; phase ^= 1u; }
                    }
                  }
                }
              }
            }
          }
        }
        stall_add(stall, true, kStProducerTotal, t_loop);
        stall_end(stall, true);
      }
    } else {
      // ================================ prologue for the next tile ========================
      const int row = (warp - kPrologueWarp) * 32 + lane;
      for (long long it = 0; it < n_iter; ++it) {
        const long long tile = tile_of(it);
        const long long p = kJvp ? tile * kPtsPerTile + (row >> 2) : tile * kPtsPerTile + row;
        bool ok = true;
        if (kNet == 2) {
          // colour-network input row, 8 columns at a time straight into the activation buffer (K blocks 0..4)
          float head[40];   // [p 3 | PE4(v) 27 | n 3 | feat 0..6]
#pragma unroll
          for (int e = 0; e < 40; ++e) head[e] = 0.f;
          const bool live = p < Ptot;
          const float* ft = prm.feats + (size_t)(live ? p : 0) * 256;
          if (live) {
            float pe[39];
            positional_encode(__ldg(prm.view_dirs + 3 * p), __ldg(prm.view_dirs + 3 * p + 1), __ldg(prm.view_dirs + 3 * p + 2),
                              prm.pw.w, pe);   // the first 27 entries of a 6-band encoding are the 4-band encoding
#pragma unroll
            for (int e = 0; e < 3; ++e) { head[e] = __ldg(prm.src.x + 3 * p + e); head[30 + e] = __ldg(prm.normals + 3 * p + e); }
#pragma unroll
            for (int e = 0; e < 27; ++e) head[3 + e] = pe[e];
#pragma unroll
            for (int e = 0; e < 7; ++e) head[33 + e] = __ldg(ft + e);
          }
          if (it > 0) mbar_wait(BAR(kBarPeFree), (uint32_t)((it - 1) & 1), abort_flag, prm.status, 400);
#pragma unroll 1
          for (int chunk = 0; chunk < 40; ++chunk) {
            float v[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const int col = 8 * chunk + e;              // feature j sits in column 33 + j
              v[e] = (live && col >= 40 && col < 289) ? __ldg(ft + (col - 33)) : 0.f;
            }
            if (chunk < 5) {
#pragma unroll
              for (int c5 = 0; c5 < 5; ++c5)
                if (chunk == c5) {
#pragma unroll
                  for (int e = 0; e < 8; ++e) v[e] = head[8 * c5 + e];
                }
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] *= kActScale;
            range_check8(v, prm.status, 1100);
            uint4 hi, lo;
            split8(v, hi, lo);
            const uint32_t off = (uint32_t)(chunk >> 3) * 8192u + sw128_offset(row, chunk & 7);
            st_shared_v4(base + kOffAHi + off, hi);
            if (kPasses == 3) st_shared_v4(base + kOffALo + off, lo);
          }
        } else if (kNet == 1) {
          // deformer input row: [PE(p) (39) | cond[frame] (128) | 0 (25)] = three 64-wide K blocks written into the
          // activation buffer itself (free again once the previous tile's last layer has been issued and done)
          // (written 8 columns at a time; only the 40-wide head [PE | first cond value] lives in registers)
          float head[40];
#pragma unroll
          for (int e = 0; e < 40; ++e) head[e] = 0.f;
          const bool live = p < Ptot;
          const bool value_row = !kJvp || (row & 3) == 0;
          const float* cond = prm.conds;
          if (live) {
            const float x = __ldg(prm.src.x + 3 * p), y = __ldg(prm.src.x + 3 * p + 1), z = __ldg(prm.src.x + 3 * p + 2);
            if (value_row) {
              positional_encode(x, y, z, prm.pw.w, head);
              long long f = prm.batch_inds ? prm.batch_inds[p] : (prm.points_per_frame > 0 ? p / prm.points_per_frame : 0);
              f = f < 0 ? 0 : (f >= prm.num_frames ? prm.num_frames - 1 : f);
              cond = prm.conds + (size_t)f * 128;
              head[39] = __ldg(cond);
            } else {
              positional_encode_tangent(x, y, z, (row & 3) - 1, prm.pw.w, head);   // the condition does not depend on p
            }
#pragma unroll
            for (int e = 0; e < 40; ++e) head[e] *= kActScale;
          }
          if (it > 0) mbar_wait(BAR(kBarPeFree), (uint32_t)((it - 1) & 1), abort_flag, prm.status, 400);
#pragma unroll
          for (int chunk = 0; chunk < 5; ++chunk) {          // columns 0..39
            range_check8(head + 8 * chunk, prm.status, 1101);
            uint4 hi, lo;
            split8(head + 8 * chunk, hi, lo);
            const uint32_t off = sw128_offset(row, chunk);
            st_shared_v4(base + kOffAHi + off, hi);
            if (kPasses == 3) st_shared_v4(base + kOffALo + off, lo);
          }
#pragma unroll 1
          for (int chunk = 5; chunk < 24; ++chunk) {         // columns 40..191: cond[1..127] then zeros
            float v[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const int ci = 8 * chunk + e - 39;             // index into the condition vector
              v[e] = (live && value_row && ci < 128) ? __ldg(cond + ci) * kActScale : 0.f;
            }
            range_check8(v, prm.status, 1102);
            uint4 hi, lo;
            split8(v, hi, lo);
            const uint32_t off = (uint32_t)(chunk >> 3) * 8192u + sw128_offset(row, chunk & 7);
            st_shared_v4(base + kOffAHi + off, hi);
            if (kPasses == 3) st_shared_v4(base + kOffALo + off, lo);
          }
        } else {
          float pe[40];
          if (p < Ptot) {
            float cx, cy, cz;
            ok = fetch_point(prm.src, p, cx, cy, cz);
            if (!kJvp || (row & 3) == 0) {
              positional_encode(cx, cy, cz, prm.pw.w, pe);
            } else {
              positional_encode_tangent(cx, cy, cz, (row & 3) - 1, prm.pw.w, pe);
            }
#pragma unroll
            for (int e = 0; e < 39; ++e) pe[e] *= kActScale;
          } else {
#pragma unroll
            for (int e = 0; e < 39; ++e) pe[e] = 0.f;
          }
          pe[39] = 0.f;
          if (it > 0) mbar_wait(BAR(kBarPeFree), (uint32_t)((it - 1) & 1), abort_flag, prm.status, 400);
          const uint4 zero = make_uint4(0, 0, 0, 0);
#pragma unroll
          for (int chunk = 0; chunk < 8; ++chunk) {
            uint4 hi = zero, lo = zero;
            if (chunk < 5) { range_check8(pe + 8 * chunk, prm.status, 1103); split8(pe + 8 * chunk, hi, lo); }
            const uint32_t off = sw128_offset(row, chunk);
            st_shared_v4(base + kOffPeHi + off, hi);
            st_shared_v4(base + kOffPeLo + off, lo);
          }
        }
        valid[(it & 1) * 64 + row] = ok ? 1 : 0;
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) mbar_arrive_local(BAR(kBarPeReady));
      }
    }
  }
}

namespace {
// one mapped, pinned status record per device
DevStatus* g_status_host[16] = {nullptr};
// relative compensation of the accumulation bias per 64-wide K block (= 4 accumulating hi*hi MMAs x 2^-24), per
// precision mode {3 passes, 1 pass}; calibrated against the reference's fp32 results (tools/calibrate_acc_gain.py)
float g_acc_gain_kb[2] = {4.f * 5.9604645e-8f, 4.f * 5.9604645e-8f};

int tc_status_record(int dev, DevStatus** out) {
  DevStatus*& h = g_status_host[dev & 15];
  if (!h) {
    cudaError_t e = cudaHostAlloc((void**)&h, sizeof(DevStatus), cudaHostAllocMapped);
    if (e != cudaSuccess) return (int)e;
    h->code = 0; h->detail = 0; h->block = 0; h->pad = 0;
  }
  *out = h;
  return 0;
}
}  // namespace

int device_status_record(void** out) {
  int dev = 0;
  cudaGetDevice(&dev);
  DevStatus* sd = nullptr;
  int s = tc_status_record(dev, &sd);
  *out = sd;
  return s;
}

namespace {
// Packs layer l of network kNet into its blob: the fp16 hi / lo panels of 1024 w (zero padding; a weight beyond fp16's
// range is reported -- tag 1201 SDF, 1200 translator / colour -- and saturated), the zero-padded bias and, for the SDF,
// the fp32 transposed copy and the bias plane b * kSoftplusLog2Scale.
template <int kNet>
__global__ void __launch_bounds__(256) pack_layer_kernel(const float* __restrict__ W /*[out,in]*/, const float* __restrict__ b,
                                                         int l, PackedBlob blob, DevStatus* status) {
  using N = Net<kNet>;
  const int out = N::out(l), in = N::in(l);
  const float scale = N::wscale(l);
  const int64_t total = (int64_t)N::nkb(l) * 512 * 64;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int pi = (int)(i / (512 * 64)), n = (int)((i / 64) % 512), kk = (int)(i % 64);
    const int k = N::src_col(l, pi, kk);
    float v = (n < out && k >= 0) ? W[(size_t)n * in + k] * scale * kWgtScale : 0.f;
    if (!(fabsf(v) < 65504.f)) {   // |w| >= 63.97: outside the tensor-core operand range
      report_range(status, kNet == 0 ? 1201 : 1200);
      v = fminf(fmaxf(v, -65504.f), 65504.f);
    }
    const __half h = __float2half_rn(v);
    const size_t o = ((size_t)(N::pbase(l) + pi) * 512 + n) * 64 + kk;
    blob.panels[o] = h;
    blob.panels[(size_t)N::kPanels * 512 * 64 + o] = __float2half_rn(v - __half2float(h));
  }
  if constexpr (kNet == 0) {
    const int npad = N::npad32(l);
    const int64_t total32 = (int64_t)in * npad;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total32; i += (int64_t)gridDim.x * blockDim.x) {
      const int k = (int)(i / npad), n = (int)(i - (int64_t)k * npad);
      blob.w32[l][i] = n < out ? W[(size_t)n * in + k] * scale : 0.f;
    }
  }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 512; i += gridDim.x * blockDim.x) {
    blob.bias[l * 512 + i] = i < out ? b[i] : 0.f;
    if (kNet == 0) blob.bias[(N::kLayers + l) * 512 + i] = i < out ? b[i] * kSoftplusLog2Scale : 0.f;
  }
}

// W_all / b_all: every layer's [out, in] weights / [out] bias, concatenated; one launch per layer
template <int kNet>
int pack_weights(const float* W_all, const float* b_all, void* packed, recmv_stream_t stream) {
  if (!W_all || !b_all || !packed) return RECMV_E_NULL;
  if (((uintptr_t)packed & 1023) != 0) return RECMV_E_SHAPE;
  void* sd = nullptr;
  int s = device_status_record(&sd);
  if (s) return s;
  using N = Net<kNet>;
  const PackedBlob blob = carve(packed, blob_layout<kNet>);
  for (int l = 0; l < N::kLayers; ++l) {
    pack_layer_kernel<kNet><<<stride_grid((int64_t)N::nkb(l) * 512 * 64, 256, 4), 256, 0, (cudaStream_t)stream>>>(
        W_all, b_all, l, blob, (DevStatus*)sd);
    s = launch_status();
    if (s) return s;
    W_all += (size_t)N::in(l) * N::out(l);
    b_all += N::out(l);
  }
  return RECMV_OK;
}

// per device and network: the tensor map of the panels it was last launched with
struct TmapCacheEntry {
  const void* base = nullptr;
  CUtensorMap map;
};
TmapCacheEntry g_tmap[16][3];

// Launches network kNet (kJvp: its forward-mode variant) on P points with the weights of blob `packed`; prm holds the
// network's own fields.  status_host != nullptr (diagnostics): waits for the launch, then reports and clears the
// device status record.
template <bool kJvp, int kNet>
int tc_launch(const void* packed, TcParams prm, int passes, int64_t P, cudaStream_t st, int* status_host = nullptr) {
  int dev = 0;
  cudaGetDevice(&dev);
  const PackedBlob blob = carve(const_cast<void*>(packed), blob_layout<kNet>);
  TmapCacheEntry& tm = g_tmap[dev & 15][kNet];
  if (tm.base != blob.panels) {
    int s = make_panel_tmap(&tm.map, blob.panels, (uint64_t)2 * Net<kNet>::kPanels * 512, 128);
    if (s) return s;
    tm.base = blob.panels;
  }
  int s = passes == 3 ? smem_opt_in<sdf_tc_kernel<kJvp, kNet, 3>>((int)kSmemBytes)
                      : smem_opt_in<sdf_tc_kernel<kJvp, kNet, 1>>((int)kSmemBytes);
  if (s) return s;
  // Device status record in MAPPED pinned host memory: a bounded wait that times out writes it there, the
  // host sees it without a synchronisation and refuses further work (recmv_check_async_errors()).
  DevStatus* sd = nullptr;
  s = tc_status_record(dev, &sd);
  if (s) return s;
  if (sd->code != 0) return RECMV_E_DEVICE;  // a previous launch on this device aborted
  prm.bias = blob.bias;
  if (kNet == 0) prm.sdf_w = blob.panels + (size_t)Net<0>::pbase(Net<0>::kLayers - 1) * 512 * 64;
  prm.P = P;
  prm.passes = passes;
  prm.acc_gain_kb = g_acc_gain_kb[passes == 3 ? 0 : 1];
  prm.status = sd;
  // persistent kernel: one CTA per SM (at most one per tile); the forward-mode variant holds 4 rows per point
  constexpr int kPtsPerTile = kJvp ? kRowsPerCta / 4 : kRowsPerCta;
  const int64_t tiles = (P + kPtsPerTile - 1) / kPtsPerTile;
  const int grid = (int)(tiles < num_sms() ? tiles : num_sms());
  if (passes == 3)
    sdf_tc_kernel<kJvp, kNet, 3><<<grid, kThreads, kSmemBytes, st>>>(tm.map, prm);
  else
    sdf_tc_kernel<kJvp, kNet, 1><<<grid, kThreads, kSmemBytes, st>>>(tm.map, prm);
  s = launch_status();
  if (s || !status_host) return s;
  cudaError_t e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return (int)e;
  status_host[0] = sd->code; status_host[1] = sd->detail; status_host[2] = sd->block; status_host[3] = 0;
  sd->code = 0; sd->detail = 0; sd->block = 0;
  return RECMV_OK;
}
}  // namespace

// SDF network.  In parity mode layer 7's epilogue computes the sdf and the last layer runs only when someone reads the
// features; in tc1 the last layer's tile 0 computes it.
int tc_sdf_forward(const PointSource& src, const void* packed, const PeWeights& pw, float* out_sdf,
                   float* out_feat, int64_t P, int passes, cudaStream_t st, const int* P_dev) {
  TcParams prm = {};
  prm.src = src; prm.pw = pw; prm.out_sdf = out_sdf; prm.out_feat = out_feat; prm.P_dev = P_dev; prm.dbg_layer = -1;
  prm.last_tiles = out_feat ? 3 : (passes == 3 ? 0 : 1);
  return tc_launch<false, 0>(packed, prm, passes, P, st);
}

int tc_sdf_forward_grad(const float* x, const void* packed, const PeWeights& pw, float* out_sdf, float* out_feat,
                        float* out_grad, int64_t P, int passes, cudaStream_t st) {
  TcParams prm = {};
  prm.src.x = x; prm.src.S = 1; prm.pw = pw; prm.out_sdf = out_sdf; prm.out_feat = out_feat; prm.dbg_layer = -1;
  prm.out_grad = out_grad;
  prm.last_tiles = out_feat ? 3 : 1;
  return tc_launch<true, 0>(packed, prm, passes, P, st);
}

}  // namespace recmv

using namespace recmv;

extern "C" size_t recmv_sdf_packed_bytes(void) { return layout_bytes(blob_layout<0>); }
extern "C" size_t recmv_translator_packed_bytes(void) { return layout_bytes(blob_layout<1>); }
extern "C" size_t recmv_rendernet_packed_bytes(void) { return layout_bytes(blob_layout<2>); }

extern "C" int recmv_sdf_pack_weights(const float* W_all, const float* b_all, void* packed, recmv_stream_t stream) {
  return pack_weights<0>(W_all, b_all, packed, stream);
}
extern "C" int recmv_translator_pack_weights(const float* W_all, const float* b_all, void* packed,
                                             recmv_stream_t stream) {
  return pack_weights<1>(W_all, b_all, packed, stream);
}
extern "C" int recmv_rendernet_pack_weights(const float* W_all, const float* b_all, void* packed,
                                            recmv_stream_t stream) {
  return pack_weights<2>(W_all, b_all, packed, stream);
}

// ---------------------------------------------------------------------------------------------------------
// Deformer network: MLPTranslator (model/Deformer.py:141-206) + LBSkinner.forward (Deformer.py:406-445)
// ---------------------------------------------------------------------------------------------------------
static int deformer_launch(const float* ps, const float* conds, const int64_t* batch_inds, int64_t points_per_frame,
                           int num_frames, const void* packed, const float* pe_w, const float* A, const float* trans,
                           const recmv_voxel_t* vox, float* out_translated, float* out_offset, float* out_posed,
                           float* out_jac, int64_t P, int mode, recmv_stream_t stream) {
  if (P < 0 || num_frames <= 0) return RECMV_E_SHAPE;
  if (P == 0) return RECMV_OK;
  if (!ps || !conds || !packed || !pe_w) return RECMV_E_NULL;
  if (out_posed && (!A || !trans || !vox || !vox->ws_cl)) return RECMV_E_NULL;
  const int passes = tc_passes(mode);
  if (!passes) return RECMV_E_UNSUPPORTED;
  TcParams prm = {};
  prm.src.x = ps; prm.src.S = 1; prm.pw = pe_weights(pe_w); prm.dbg_layer = -1;
  prm.conds = conds; prm.batch_inds = (const long long*)batch_inds; prm.points_per_frame = points_per_frame;
  prm.num_frames = num_frames; prm.bones = A; prm.trans = trans;
  if (vox) prm.vox = to_voxel(vox);
  prm.out_translated = out_translated; prm.out_offset = out_offset; prm.out_posed = out_posed; prm.out_jac = out_jac;
  if (out_jac) return tc_launch<true, 1>(packed, prm, passes, P, (cudaStream_t)stream);
  return tc_launch<false, 1>(packed, prm, passes, P, (cudaStream_t)stream);
}

extern "C" int recmv_deformer_fwd_jac(const float* ps, const float* conds, const int64_t* batch_inds,
                                      int64_t points_per_frame, int num_frames, const void* packed, const float* pe_w,
                                      const float* A, const float* trans, const recmv_voxel_t* vox, float* out_translated,
                                      float* out_offset, float* out_posed, float* out_jac, int64_t P, int mode,
                                      recmv_stream_t stream) {
  if (!out_jac) return RECMV_E_NULL;
  return deformer_launch(ps, conds, batch_inds, points_per_frame, num_frames, packed, pe_w, A, trans, vox, out_translated,
                         out_offset, out_posed, out_jac, P, mode, stream);
}

extern "C" int recmv_deformer_fwd(const float* ps, const float* conds, const int64_t* batch_inds,
                                  int64_t points_per_frame, int num_frames, const void* packed, const float* pe_w,
                                  const float* A, const float* trans, const recmv_voxel_t* vox, float* out_translated,
                                  float* out_offset, float* out_posed, int64_t P, int mode, recmv_stream_t stream) {
  return deformer_launch(ps, conds, batch_inds, points_per_frame, num_frames, packed, pe_w, A, trans, vox, out_translated,
                         out_offset, out_posed, nullptr, P, mode, stream);
}

// ---------------------------------------------------------------------------------------------------------
// Colour network: RenderingNetwork_view_norm, mode 'idr' (model/RenderNet.py:59-96)
// ---------------------------------------------------------------------------------------------------------
extern "C" int recmv_rendernet_fwd(const float* points, const float* normals, const float* view_dirs,
                                   const float* feats, const void* packed, const float* pe_w, float* out_rgb,
                                   int64_t P, int mode, recmv_stream_t stream) {
  if (P < 0) return RECMV_E_SHAPE;
  if (P == 0) return RECMV_OK;
  if (!points || !normals || !view_dirs || !feats || !packed || !pe_w || !out_rgb) return RECMV_E_NULL;
  const int passes = tc_passes(mode);
  if (!passes) return RECMV_E_UNSUPPORTED;
  TcParams prm = {};
  prm.src.x = points; prm.src.S = 1; prm.pw = pe_weights(pe_w, 4); prm.dbg_layer = -1;
  prm.normals = normals; prm.view_dirs = view_dirs; prm.feats = feats; prm.out_rgb = out_rgb;
  return tc_launch<false, 2>(packed, prm, passes, P, (cudaStream_t)stream);
}

// Diagnostics / calibration: relative gain per 64-wide K block applied to the raw accumulators of a precision mode
// (RECMV_MLP_TC_F16X3 or RECMV_MLP_TC_F16X1) to compensate the tensor core's truncating accumulation.
extern "C" int recmv_tc_set_acc_gain(int mode, float gain_per_kblock) {
  const int passes = tc_passes(mode);
  if (!passes) return RECMV_E_DTYPE;
  if (!(fabsf(gain_per_kblock) < 1e-4f)) return RECMV_E_RANGE;
  g_acc_gain_kb[passes == 3 ? 0 : 1] = gain_per_kblock;
  return RECMV_OK;
}

// Reports (without synchronising) whether any tensor-core launch on the current device has aborted on a bounded
// wait since the last check: 0 = none, RECMV_E_DEVICE otherwise; info[3] = {code, barrier tag, block}.
extern "C" int recmv_check_async_errors(int* info, int clear) {
  int dev = 0;
  cudaGetDevice(&dev);
  DevStatus* h = g_status_host[dev & 15];
  if (!h || h->code == 0) {
    if (info) { info[0] = 0; info[1] = 0; info[2] = 0; }
    return RECMV_OK;
  }
  if (info) { info[0] = h->code; info[1] = h->detail; info[2] = h->block; }
  if (clear) { h->code = 0; h->detail = 0; h->block = 0; }
  return RECMV_E_DEVICE;
}

// Diagnostics entry (see include/recmv_b200_diag.h): runs the tensor-core path on canonical points and returns
// the device status record (which bounded wait timed out, if any) plus the raw accumulator of one layer.
extern "C" int recmv_sdf_mlp_tc_debug(const float* x, const void* packed, const float* pe_w, float* out_sdf,
                                      float* out_feat, int64_t P, int passes, int dbg_layer, float* dbg_out,
                                      int* status_host, recmv_stream_t stream) {
  if (P <= 0) return RECMV_E_SHAPE;
  if (!x || !packed || !pe_w || !out_sdf || !status_host) return RECMV_E_NULL;
  if (passes != 1 && passes != 3) return RECMV_E_DTYPE;
  TcParams prm = {};
  prm.src.x = x; prm.src.S = 1; prm.pw = pe_weights(pe_w); prm.out_sdf = out_sdf; prm.out_feat = out_feat;
  prm.dbg_layer = dbg_layer; prm.dbg_out = dbg_out;
  prm.last_tiles = (out_feat || (dbg_out && dbg_layer == Net<0>::kLayers - 1)) ? 3 : (passes == 3 ? 0 : 1);
  return tc_launch<false, 0>(packed, prm, passes, P, (cudaStream_t)stream, status_host);
}

#if RECMV_TC_STALL_PROF
// Diagnostics build only (see include/recmv_b200_diag.h): the stall counters summed over every launch since the last
// reset, in the order of StallCounter.  Synchronises the device.
extern "C" int recmv_tc_stall_profile(unsigned long long* counters, int n, int reset) {
  if (!counters) return RECMV_E_NULL;
  if (n < kStCounters) return RECMV_E_SHAPE;
  cudaError_t e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpyFromSymbol(counters, g_tc_stall, sizeof(unsigned long long) * kStCounters);
  if (e == cudaSuccess && reset) {
    const unsigned long long zero[kStCounters] = {};
    e = cudaMemcpyToSymbol(g_tc_stall, zero, sizeof(zero));
  }
  return e == cudaSuccess ? RECMV_OK : (int)e;
}
#endif

// Area-weighted surface sampling of M meshes with one face list (DESIGN section 1h): trimesh's `sample_surface` with a
// counter-based stream, so every sample is a pure function of (seed, offset, mesh, sample) and a float64 NumPy
// restatement (oracle/sample_oracle.py) reproduces each output bit.  Replaces the per-step `trimesh.sample` of
// `curve_aware_loss` (engineer/networks/OptimGarmentNetwork.py:787-839).
//
//   1. area_scan_kernel    one block per (256-face chunk, mesh): fp64 face areas (0 for an out-of-range index or a
//                          non-finite area), then a sequential inclusive sum inside the chunk -> local[m][f], and the
//                          chunk total -> tot[m][c];
//   2. chunk_scan_kernel   one block per mesh, its first thread: tot[m][c] becomes the exclusive sequential prefix of
//                          the chunk totals;
//   3. sample_kernel       one thread per sample: Philox4x32-10, a binary search over C[f] = tot[m][f / 256] + local[m][f]
//                          (the first f with C[f] >= u C[F-1]), the folded parallelogram point, one fp32 store.
// Every fp64 operation is rounded explicitly (no FMA contraction) so the oracle can match it.  No atomics: the output
// is bit-identical from run to run and on any SM count.
#include <math.h>

#include "common.cuh"
#include "philox.cuh"

namespace recmv {
namespace {

constexpr int kChunk = 256;          // faces per chunk of the pinned cumulative-sum order
constexpr int kSampleThreads = 256;

struct Tri {
  double v0x, v0y, v0z, e1x, e1y, e1z, e2x, e2y, e2z;
};

// edges e1 = v1 - v0, e2 = v2 - v0 in fp64 from the fp32 corners; false for an index outside [0, V)
__device__ __forceinline__ bool load_tri(const float* __restrict__ vm, int V, const long long* __restrict__ faces,
                                         long long f, Tri& t) {
  const long long a = __ldg(faces + 3 * f), b = __ldg(faces + 3 * f + 1), c = __ldg(faces + 3 * f + 2);
  if (a < 0 || a >= V || b < 0 || b >= V || c < 0 || c >= V) return false;
  const float* pa = vm + 3 * a;
  const float* pb = vm + 3 * b;
  const float* pc = vm + 3 * c;
  t.v0x = (double)__ldg(pa); t.v0y = (double)__ldg(pa + 1); t.v0z = (double)__ldg(pa + 2);
  t.e1x = __dsub_rn((double)__ldg(pb), t.v0x);
  t.e1y = __dsub_rn((double)__ldg(pb + 1), t.v0y);
  t.e1z = __dsub_rn((double)__ldg(pb + 2), t.v0z);
  t.e2x = __dsub_rn((double)__ldg(pc), t.v0x);
  t.e2y = __dsub_rn((double)__ldg(pc + 1), t.v0y);
  t.e2z = __dsub_rn((double)__ldg(pc + 2), t.v0z);
  return true;
}

__global__ void __launch_bounds__(kChunk) area_scan_kernel(const float* __restrict__ verts, int V,
                                                          const long long* __restrict__ faces, long long F,
                                                          long long nchunks, double* __restrict__ local,
                                                          double* __restrict__ tot) {
  __shared__ double area[kChunk];
  const long long c = blockIdx.x;
  const int m = blockIdx.y;
  const long long f = c * kChunk + threadIdx.x;
  double A = 0.0;
  Tri t;
  if (f < F && load_tri(verts + (long long)m * V * 3, V, faces, f, t)) {
    const double cx = __dsub_rn(__dmul_rn(t.e1y, t.e2z), __dmul_rn(t.e1z, t.e2y));
    const double cy = __dsub_rn(__dmul_rn(t.e1z, t.e2x), __dmul_rn(t.e1x, t.e2z));
    const double cz = __dsub_rn(__dmul_rn(t.e1x, t.e2y), __dmul_rn(t.e1y, t.e2x));
    const double ss = __dadd_rn(__dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy)), __dmul_rn(cz, cz));
    A = __dmul_rn(0.5, __dsqrt_rn(ss));
    if (!isfinite(A)) A = 0.0;
  }
  area[threadIdx.x] = A;
  __syncthreads();
  if (threadIdx.x == 0) {
    const int n = (int)min((long long)kChunk, F - c * kChunk);
    double* out = local + (long long)m * F + c * kChunk;
    double s = 0.0;
    for (int i = 0; i < n; ++i) {
      s = __dadd_rn(s, area[i]);
      out[i] = s;
    }
    tot[(long long)m * nchunks + c] = s;
  }
}

__global__ void chunk_scan_kernel(double* __restrict__ tot, long long nchunks) {
  if (threadIdx.x != 0) return;
  double* t = tot + (long long)blockIdx.x * nchunks;
  double run = 0.0;
  for (long long c = 0; c < nchunks; ++c) {
    const double x = t[c];
    t[c] = run;
    run = __dadd_rn(run, x);
  }
}

__device__ __forceinline__ double cum(const double* __restrict__ loc, const double* __restrict__ pre, long long f) {
  return __dadd_rn(__ldg(pre + f / kChunk), __ldg(loc + f));
}

__global__ void __launch_bounds__(kSampleThreads) sample_kernel(const float* __restrict__ verts, int V,
                                                               const long long* __restrict__ faces, long long F,
                                                               long long nchunks, const double* __restrict__ local,
                                                               const double* __restrict__ pre, long long S,
                                                               long long total, unsigned long long seed,
                                                               unsigned long long offset, float* __restrict__ out) {
  const long long g = blockIdx.x * (long long)kSampleThreads + threadIdx.x;
  if (g >= total) return;
  const long long m = g / S;
  const unsigned long long ctr = offset + (unsigned long long)g;   // offset + m S + s, modulo 2^64
  const Philox4 r = philox4x32_10((unsigned)ctr, (unsigned)(ctr >> 32), (unsigned)seed, (unsigned)(seed >> 32));
  const double u = (double)(((unsigned long long)r.x[0] << 21) | (r.x[1] >> 11)) * 0x1p-53;
  double a = (double)r.x[2] * 0x1p-32, b = (double)r.x[3] * 0x1p-32;
  if (__dadd_rn(a, b) > 1.0) { a = __dsub_rn(1.0, a); b = __dsub_rn(1.0, b); }
  const double* loc = local + m * F;
  const double* pr = pre + m * nchunks;
  const double x = __dmul_rn(u, cum(loc, pr, F - 1));
  long long lo = 0, hi = F - 1;   // first f with C[f] >= x; C[F-1] >= x always holds
  while (lo < hi) {
    const long long mid = lo + ((hi - lo) >> 1);
    if (cum(loc, pr, mid) >= x) hi = mid; else lo = mid + 1;
  }
  Tri t;
  float* o = out + 3 * g;
  if (!load_tri(verts + m * V * 3, V, faces, lo, t)) {
    o[0] = o[1] = o[2] = __int_as_float(0x7fc00000);
    return;
  }
  o[0] = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn(a, t.e1x), __dmul_rn(b, t.e2x)), t.v0x));
  o[1] = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn(a, t.e1y), __dmul_rn(b, t.e2y)), t.v0y));
  o[2] = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn(a, t.e1z), __dmul_rn(b, t.e2z)), t.v0z));
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

int sample_shape(int M, int V, int64_t F) {
  if (M < 0 || V < 0 || F < 0) return RECMV_E_SHAPE;
  if (M > 65535) return RECMV_E_RANGE;                               // grid.y of the area pass
  if (F > ((int64_t)1 << 40) || (int64_t)M * F > ((int64_t)1 << 40)) return RECMV_E_RANGE;
  return RECMV_OK;
}

long long num_chunks(int64_t F) { return (F + kChunk - 1) / kChunk; }

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_surface_sample_workspace_bytes(int M, int64_t F, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  const int s = sample_shape(M, 0, F);
  if (s) return s;
  *bytes = align256((size_t)M * F * 8) + align256((size_t)M * num_chunks(F) * 8);
  return RECMV_OK;
}

extern "C" int recmv_surface_sample(const float* verts, int M, int V, const int64_t* faces, int64_t F, int64_t S,
                                    uint64_t seed, uint64_t offset, void* workspace, float* out,
                                    recmv_stream_t stream) {
  int s = sample_shape(M, V, F);
  if (s) return s;
  if (S < 0) return RECMV_E_SHAPE;
  const long long total = (long long)M * S;
  if (S > 0 && M > 0 && total / M != S) return RECMV_E_RANGE;
  if (total == 0) return RECMV_OK;
  if (F == 0) return RECMV_E_SHAPE;                                  // nothing to sample from
  const long long blocks = (total + kSampleThreads - 1) / kSampleThreads;
  if (blocks > 0x7fffffffLL || num_chunks(F) > 0x7fffffffLL) return RECMV_E_RANGE;
  if (!faces || !workspace || !out || (V > 0 && !verts)) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  const long long nch = num_chunks(F);
  double* local = (double*)workspace;
  double* tot = (double*)((char*)workspace + align256((size_t)M * F * 8));
  area_scan_kernel<<<dim3((unsigned)nch, (unsigned)M), kChunk, 0, st>>>(verts, V, (const long long*)faces, F, nch,
                                                                        local, tot);
  s = launch_status();
  if (s) return s;
  chunk_scan_kernel<<<(unsigned)M, 32, 0, st>>>(tot, nch);
  s = launch_status();
  if (s) return s;
  sample_kernel<<<(unsigned)blocks, kSampleThreads, 0, st>>>(verts, V, (const long long*)faces, F, nch, local, tot, S,
                                                             total, (unsigned long long)seed,
                                                             (unsigned long long)offset, out);
  return launch_status();
}

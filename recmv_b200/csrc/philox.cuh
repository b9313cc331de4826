// Random123's Philox4x32 with 10 rounds, the counter-based stream of the device samplers (surface_sample.cu,
// train_rays.cu).  oracle/sample_oracle.py restates it in NumPy.
#pragma once

namespace recmv {
namespace {

struct Philox4 {
  unsigned x[4];
};

// counter {c0, c1, 0, 0}, key {k0, k1}
__device__ __forceinline__ Philox4 philox4x32_10(unsigned c0, unsigned c1, unsigned k0, unsigned k1) {
  unsigned x0 = c0, x1 = c1, x2 = 0u, x3 = 0u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const unsigned lo0 = 0xD2511F53u * x0, hi0 = __umulhi(0xD2511F53u, x0);
    const unsigned lo1 = 0xCD9E8D57u * x2, hi1 = __umulhi(0xCD9E8D57u, x2);
    const unsigned y0 = hi1 ^ x1 ^ k0, y2 = hi0 ^ x3 ^ k1;
    x0 = y0; x1 = lo1; x2 = y2; x3 = lo0;
  }
  return Philox4{{x0, x1, x2, x3}};
}

}  // namespace
}  // namespace recmv

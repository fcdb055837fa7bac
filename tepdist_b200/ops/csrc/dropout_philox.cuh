// Dropout mask generation on the device: Philox4x32-10, bit-identical to the host reference DropoutKeep
// (csrc/runtime/slice_philox.cc), which states the mask's definition (DESIGN.md "Dropout").  Key = the seed, counter =
// (column group, row, step, site); an element is kept iff its byte of the call's 16 is >= thr, and kept values are scaled
// by 256 / (256 - thr).
#pragma once
#include <stdint.h>

namespace dropout {

__device__ __forceinline__ uint4 philox(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, unsigned long long seed) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

// byte b (0..15, little-endian within the four words) of a call's output
__device__ __forceinline__ uint32_t byte_of(const uint4& r, int b) {
  const uint32_t w = (b >> 2) == 0 ? r.x : (b >> 2) == 1 ? r.y : (b >> 2) == 2 ? r.z : r.w;
  return (w >> (8 * (b & 3))) & 0xffu;
}

}  // namespace dropout

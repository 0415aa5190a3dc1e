// Element-wise dropout at p = 0.5 (nn.Dropout(0.5) of the attention head, network/utils.py:359-360) without a stored
// mask: the keep bit of element i of an NHWC map (i = pixel * C + channel, the dense index whatever the row pitch) is
// bit i % 128 of Philox4x32-10(counter = {i / 128 (64 bit), pass, 0}, key = seed). One generator call covers 128
// consecutive elements, so the forward (BatchNorm apply) and the backward passes regenerate exactly the same bits from
// the 64-bit seed alone. `pass` separates the scale passes of one step.
#pragma once
#include <cstdint>

namespace b200seg {

struct DropKey {
  const unsigned long long* seed;   // device pointer (the step's seed, rewritten before every graph replay); nullptr = off
  int pass;
};

__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    const uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}

// Keep bits of the 8 elements i0 .. i0 + 7 (i0 a multiple of 8) in bits 0 .. 7.
__device__ __forceinline__ uint32_t dropout_keep8(unsigned long long seed, int pass, long long i0) {
  const unsigned long long blk = (unsigned long long)i0 >> 7;
  const uint4 r = philox4x32_10(make_uint4((uint32_t)blk, (uint32_t)(blk >> 32), (uint32_t)pass, 0u),
                                make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  const int word = (int)(i0 >> 5) & 3;
  const uint32_t w = word == 0 ? r.x : (word == 1 ? r.y : (word == 2 ? r.z : r.w));
  return (w >> ((int)i0 & 31)) & 0xFFu;
}

// v[j] <- keep ? 2 v[j] : 0 for the 8 elements starting at i0.
__device__ __forceinline__ void dropout_apply8(float (&v)[8], unsigned long long seed, int pass, long long i0) {
  const uint32_t keep = dropout_keep8(seed, pass, i0);
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = (keep >> j) & 1u ? 2.f * v[j] : 0.f;
}

}  // namespace b200seg

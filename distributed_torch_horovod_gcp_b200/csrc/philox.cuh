// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11): a counter-based
// generator, so every dropout mask here is a pure function of (key, counter) and any thread can draw any part
// of it in any order.  Shared by the LSTM inter-layer dropout (lstm_rec_sm90.cu), the dropout inside flash
// attention (attn_sm90.cu) and the fused dropout + residual add (elementwise.cu).  It is a header of its own
// (included by sm90_common.cuh) because elementwise.cu does not include sm90_common.cuh.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * ctr.x, hi0 = __umulhi(0xD2511F53u, ctr.x);
    const uint32_t lo1 = 0xCD9E8D57u * ctr.z, hi1 = __umulhi(0xCD9E8D57u, ctr.z);
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += 0x9E3779B9u;
    key.y += 0xBB67AE85u;
  }
  return ctr;
}

// Keep threshold of a 16-bit uniform draw for dropout probability p: an element is kept when its 16 bits are
// below t = round((1 - p) 2^16), so the keep probability is exactly t / 2^16 (p has a resolution of 2^-16)
// and the scale of a kept element is its exact reciprocal 2^16 / t (0 when t = 0: everything is dropped).
inline uint32_t dropout_thr16(double p) {
  const double t = (1.0 - p) * 65536.0 + 0.5;
  return t <= 0.0 ? 0u : (t >= 65536.0 ? 65536u : (uint32_t)t);
}
inline float dropout_scale16(uint32_t thr) { return thr ? (float)(65536.0 / (double)thr) : 0.f; }

}  // namespace

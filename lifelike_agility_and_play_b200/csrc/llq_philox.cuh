// Philox4x32-10 of the policy kernels' sampling noise (same generator as the engine's reset streams, csrc/llq_math.cuh):
// llq_policy.cu keys the Gaussian action noise and llq_policy_hier.cu the Gumbel code noise with it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

static __device__ __forceinline__ uint4 philox4x32(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; r++) {
    const uint32_t h0 = __umulhi(0xD2511F53u, c.x), l0 = 0xD2511F53u * c.x;
    const uint32_t h1 = __umulhi(0xCD9E8D57u, c.z), l1 = 0xCD9E8D57u * c.z;
    c = make_uint4(h1 ^ c.y ^ k.x, l1, h0 ^ c.w ^ k.y, l0);
    k.x += 0x9E3779B9u; k.y += 0xBB67AE85u;
  }
  return c;
}

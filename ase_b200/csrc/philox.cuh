// Counter-based generator of the device rollout and the device resets: Philox4x32-10 (Salmon et al. 2011) and its fp32 uniform / normal
// mappings.  Element (row, group) of draw number `rng[1]` of stream `sid` is a pure function of (rng[0] = seed, sid, rng[1], row, group);
// the addressing is documented in include/ase_b200.h and restated in oracle/philox_oracle.py.
#pragma once
#include "common.cuh"

namespace ase {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u; k.y += 0xBB67AE85u;
  }
  return c;
}
// (0, 1]: from 2^23 up, code + 0.5 rounds to an even integer, and the top code 0xFFFFFF rounds to 2^24, i.e. 1.0.  Box-Muller input only
// (-2 log(1) = 0 is a valid radius).
__device__ __forceinline__ float u01(uint32_t x) { return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f); }
// (0, 1) like torch.rand: u01 capped at the largest float below 1, so `u < p` holds for p = 1 and a target never reaches the top of its range.
__device__ __forceinline__ float u01_open(uint32_t x) { return fminf(u01(x), 0x1.fffffep-1f); }
// 4 standard normals of draw `call`, stream `sid`, element group (row, grp)
__device__ __forceinline__ float4 philox_normal4(const uint64_t* rng, uint32_t sid, uint32_t row, uint32_t grp) {
  const uint64_t seed = rng[0], call = rng[1];
  const uint4 r = philox4x32_10(make_uint4(row, grp, (uint32_t)call, (uint32_t)(call >> 32)), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32) ^ (sid * 0x9E3779B1u)));
  const float a = sqrtf(-2.0f * logf(u01(r.x))), b = sqrtf(-2.0f * logf(u01(r.z)));
  float s0, c0, s1, c1;
  sincospif(2.0f * u01(r.y), &s0, &c0); sincospif(2.0f * u01(r.w), &s1, &c1);
  return make_float4(a * c0, a * s0, b * c1, b * s1);
}
__device__ __forceinline__ uint4 philox_u4(const uint64_t* rng, uint32_t sid, uint32_t row, uint32_t grp) {
  const uint64_t seed = rng[0], call = rng[1];
  return philox4x32_10(make_uint4(row, grp, (uint32_t)call, (uint32_t)(call >> 32)), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32) ^ (sid * 0x9E3779B1u)));
}

}  // namespace ase

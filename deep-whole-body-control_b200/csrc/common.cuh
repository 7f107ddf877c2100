// Shared device helpers for libdwbc (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dwbc.h"

// every kernel launch of the library passes through one of these (host-side launch counter,
// read back with dwbc_launch_count(); bench.py reports it as gpu_launches)
extern unsigned long long dwbc_launch_counter;
#define DWBC_LAUNCH_CHECK()                                   \
  do {                                                        \
    ++dwbc_launch_counter;                                    \
    cudaError_t e__ = cudaGetLastError();                     \
    if (e__ != cudaSuccess) return DWBC_ERR_LAUNCH;           \
  } while (0)

namespace dwbc {

constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL, v, o));
  return v;
}

// 128-bit streaming accesses: inputs read once bypass L1 allocation, outputs are write-once.
__device__ __forceinline__ float4 ldg_stream(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void stg_stream(float4* p, float4 v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

// Philox4x32-10 (Salmon et al. 2011), counter = (c0,c1,c2,c3), key = (k0,k1).
__device__ __forceinline__ void philox_round(uint32_t& c0, uint32_t& c1, uint32_t& c2, uint32_t& c3, uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
  uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
  uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
  uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
  c0 = n0; c1 = n1; c2 = n2; c3 = n3;
}
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  uint32_t c0 = ctr.x, c1 = ctr.y, c2 = ctr.z, c3 = ctr.w, k0 = key.x, k1 = key.y;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    philox_round(c0, c1, c2, c3, k0, k1);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}
// uniform in [0,1) with a 24-bit mantissa, like torch.rand(float32)
__device__ __forceinline__ float u01(uint32_t x) { return (float)(x >> 8) * 5.9604644775390625e-08f; }

// Fixed-order sums across blocks: every block writes its partials to a slot of its own, then calls this.  It returns true, in every
// thread, in the block that arrives last (counted on `ticket`, which that block returns to zero for the next launch); that block sees
// every partial and adds them up in slot order, so the result does not depend on which block ran when.
__device__ __forceinline__ bool last_block(unsigned* ticket) {
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    last = atomicAdd(ticket, 1u) == gridDim.x * gridDim.y * gridDim.z - 1;
    if (last) *ticket = 0u;
  }
  __syncthreads();
  if (last) __threadfence();
  return last;
}

}  // namespace dwbc

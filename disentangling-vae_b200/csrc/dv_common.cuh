// Shared helpers for the disvae_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "disvae_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "disvae_b200 kernels are written for sm_90a (Hopper H100) only"
#endif

namespace dv {

constexpr int kWarp = 32;
constexpr int kLoCh = 32;          // channels of every "lo" tensor (encoders.py:43, decoders.py:43)
constexpr int kTaps = 16;          // 4x4 kernel
constexpr int kNumSMs = 132;       // H100 SXM

extern thread_local int g_last_cuda_error;
extern long long g_launches;

inline int check_launch() {
  cudaError_t e = cudaGetLastError();
  __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
  if (e != cudaSuccess) { g_last_cuda_error = (int)e; return DV_ERR_CUDA; }
  return DV_OK;
}
inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// Opt a kernel in to `bytes` of dynamic shared memory, once per process (*done caches the success).
template <typename Kernel>
inline int set_max_dynamic_smem(Kernel kernel, int bytes, bool* done) {
  if (*done) return DV_OK;
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess) {
    g_last_cuda_error = (int)cudaGetLastError();
    return DV_ERR_CUDA;
  }
  *done = true;
  return DV_OK;
}

// First 1024-byte aligned address at or after p (TMA destinations with the 128-byte swizzle need it).
__device__ __forceinline__ uint8_t* align1024(uint8_t* p) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~uintptr_t(1023));
}

__device__ __forceinline__ float4 ldg4(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float apply_act(float v, int act, float slope) {
  if (act == DV_ACT_RELU) return fmaxf(v, 0.f);
  if (act == DV_ACT_SIGMOID) return 1.f / (1.f + expf(-v));
  if (act == DV_ACT_LEAKY) return v > 0.f ? v : v * slope;
  return v;
}

// Philox4x32-10 (Salmon et al. 2011) -- counter-based RNG for on-device eps / permutations.
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0; key.y += W1;
  }
  return ctr;
}
__device__ __forceinline__ float u32_to_unit_open(uint32_t x) {   // (0,1]
  return (float)(x >> 8) * (1.0f / 16777216.0f) + (1.0f / 33554432.0f);
}

}  // namespace dv

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

// True when p is not a multiple of `a` bytes (a power of two).  NULL passes: optional operands are checked for
// presence elsewhere.
inline bool misaligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0; }

// A workspace cut into consecutive segments of sizes[s] bytes, each starting on a 256-byte boundary: the offsets into
// off[] -> the total bytes.
inline size_t align_up(size_t b) { return (b + 255) & ~size_t(255); }
template <int kSegs>
inline size_t carve_workspace(const size_t (&sizes)[kSegs], size_t (&off)[kSegs]) {
  size_t total = 0;
  for (int s = 0; s < kSegs; ++s) {
    off[s] = total;
    total += align_up(sizes[s]);
  }
  return total;
}

// First 1024-byte aligned address at or after p (TMA destinations with the 128-byte swizzle need it).
__device__ __forceinline__ uint8_t* align1024(uint8_t* p) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~uintptr_t(1023));
}

__device__ __forceinline__ float4 ldg4(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}

// The fixed-order sums behind the "bit-identical run to run" results: over a warp by the butterfly (xor 16, 8, 4, 2,
// 1), over a block of kWarps warps by the warps' sums added in order 0 .. kWarps - 1 (red: kWarps shared slots).
// Every thread ends with the same bits.
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <int kWarps, typename T>
__device__ T block_sum(T v, T* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & (kWarp - 1)) == 0) red[threadIdx.x / kWarp] = v;
  __syncthreads();
  T s = 0;
  for (int w = 0; w < kWarps; ++w) s += red[w];
  return s;
}

// The classes of scored factor k: n_classes[k] clamped to [0, S].
__device__ __forceinline__ int class_count(const int* n_classes, int k, int S) { return min(max(n_classes[k], 0), S); }

// disentanglement_lib's 20-bin histogram discretisation of an fp32 column, np.digitize(x, np.histogram(x, 20)[1][:-1]).
constexpr int kHistBins = 20;

// Every thread's partial min `lo` and max `hi` of the column -> edge[0 .. 20] (shared) for the whole block: the column's
// range (lo - 0.5, hi + 0.5 in fp32 when equal, as np.histogram widens it), then np.linspace(lo, hi, 21) in fp32 without
// contraction: step = (hi - lo) / 20, edge_j = j * step + lo, the last edge hi.  wlo, whi: kWarps shared slots each.
// Ends with a barrier.
template <int kWarps>
__device__ void histogram_edges(float lo, float hi, float* wlo, float* whi, float* edge) {
  const int t = threadIdx.x;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((t & (kWarp - 1)) == 0) {
    wlo[t / kWarp] = lo;
    whi[t / kWarp] = hi;
  }
  __syncthreads();
  if (t == 0) {
    lo = wlo[0];
    hi = whi[0];
    for (int w = 1; w < kWarps; ++w) {
      lo = fminf(lo, wlo[w]);
      hi = fmaxf(hi, whi[w]);
    }
    if (lo == hi) {
      lo = __fsub_rn(lo, 0.5f);
      hi = __fadd_rn(hi, 0.5f);
    }
    const float step = __fdiv_rn(__fsub_rn(hi, lo), (float)kHistBins);
    for (int j = 0; j < kHistBins; ++j) edge[j] = __fadd_rn(__fmul_rn((float)j, step), lo);
    edge[kHistBins] = hi;
  }
  __syncthreads();
}

// np.digitize(v, edge[:-1]) - 1: the number of edge_0 .. edge_19 at or below v, less one (0 .. 19).  edge_0 = lo unless
// the range overflows fp32, so every value of the column has at least one.
__device__ __forceinline__ int histogram_bin(const float* edge, float v) {
  int b = 0;
#pragma unroll
  for (int j = 0; j < kHistBins; ++j) b += edge[j] <= v ? 1 : 0;
  return max(b, 1) - 1;
}

// Sorting fp32 columns in shared memory (DCI's training columns, IRS's latents): order_key maps a float to an unsigned
// key whose order is the float's (-0 just below +0), key_value maps it back, and bitonic_sort_pairs sorts P (a power of
// two) (key, position) pairs ascending on (key, position) with kThreads threads, so equal values keep their order.
// Padding pairs take the key 0xffffffff.  Called after a barrier; ends with one.
inline int pow2_at_least(int n) {
  int p = 1;
  while (p < n) p <<= 1;
  return p;
}

__device__ __forceinline__ unsigned order_key(float v) {
  const unsigned u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

template <int kThreads>
__device__ void bitonic_sort_pairs(unsigned* key, unsigned short* idx, int P) {
  const int t = threadIdx.x;
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = t; i < P; i += kThreads) {
        const int o = i ^ j;
        if (o > i) {
          const unsigned ka = key[i], kb = key[o];
          const unsigned short ia = idx[i], ib = idx[o];
          const bool greater = ka > kb || (ka == kb && ia > ib);
          if (greater == ((i & k) == 0)) {
            key[i] = kb; key[o] = ka;
            idx[i] = ib; idx[o] = ia;
          }
        }
      }
      __syncthreads();
    }
  }
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

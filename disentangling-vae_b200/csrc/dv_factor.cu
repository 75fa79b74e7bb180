// FactorVAE pieces: per-dimension batch permutation, TC estimate from the discriminator logits,
// two-class cross entropy.  Reference: disvae/models/losses.py:483-508 (_permute_dims),
// :265 (tc_loss), :291-295 (d_tc_loss).
#include <climits>
#include <algorithm>
#include "dv_common.cuh"

namespace dv {

constexpr int kPermMaxB = 4096;          // one CTA sorts this many keys in shared memory (32 KB)

// Rows [row0, row0 + nrows) of the permuted matrix are written to out[0, nrows): out[i][d] = z[pi_d(row0 + i)][d].

// perms given: pi_d = perms[d]
__global__ void permute_given_kernel(const float* __restrict__ z, const long long* __restrict__ perms,
                                     float* __restrict__ out, int B, int D, int row0, int nrows) {
  const long long n = (long long)nrows * D;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / D), d = (int)(i % D);
    const long long src = perms[(long long)d * B + row0 + b];
    out[i] = z[src * D + d];
  }
}

// Sort key of row b of dimension d: the Philox draw in the high half, the row index in the low half.  The keys of one
// dimension are unique, so every correct sort orders them the same way: pi_d = the index column of the sorted keys.
__device__ __forceinline__ unsigned long long perm_key(unsigned long long off, int b, unsigned long long seed) {
  const unsigned long long c = off + (unsigned long long)b;
  const uint4 r = philox4x32_10(make_uint4((uint32_t)c, (uint32_t)(c >> 32), 0x5eedu, 0u),
                                make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  return ((unsigned long long)r.x << 32) | (unsigned long long)(uint32_t)b;
}

// Ascending bitonic sort of keys[0, npow2) in shared memory by the whole CTA (npow2 a power of two).
__device__ __forceinline__ void bitonic_sort_smem(unsigned long long* keys, int npow2) {
  for (int size = 2; size <= npow2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = threadIdx.x; t < (npow2 >> 1); t += blockDim.x) {
        const int lo = 2 * t - (t & (stride - 1));
        const int hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const unsigned long long a = keys[lo], b2 = keys[hi];
        if ((a > b2) == up) { keys[lo] = b2; keys[hi] = a; }
      }
      __syncthreads();
    }
  }
}

// perms generated on device, B <= kPermMaxB: block d sorts its B keys in shared memory and gathers the window.
__global__ void __launch_bounds__(512)
permute_philox_kernel(const float* __restrict__ z, unsigned long long seed, const unsigned long long* __restrict__ offset_dev,
                      float* __restrict__ out, int B, int D, int npow2, int row0, int nrows) {
  extern __shared__ unsigned long long keys[];
  const int d = blockIdx.x;
  const unsigned long long off = *offset_dev + (unsigned long long)d * (unsigned long long)B;
  for (int b = threadIdx.x; b < npow2; b += blockDim.x) keys[b] = b < B ? perm_key(off, b, seed) : ~0ull;
  __syncthreads();
  bitonic_sort_smem(keys, npow2);
  for (int i = threadIdx.x; i < nrows; i += blockDim.x) {
    const int src = (int)(keys[row0 + i] & 0xffffffffull);
    out[(long long)i * D + d] = z[(long long)src * D + d];
  }
}

// perms generated on device, B > kPermMaxB: the keys of each dimension are sorted in a [D][B] workspace buffer.
// Tile pass: block (t, d) sorts keys [t*kPermMaxB, (t+1)*kPermMaxB) of dimension d in shared memory; the padding keys
// of a partial last tile (~0, larger than any real key) sort to its end and are not written.
__global__ void __launch_bounds__(512)
permute_tile_sort_kernel(unsigned long long seed, const unsigned long long* __restrict__ offset_dev,
                         unsigned long long* __restrict__ sorted, int B, int D) {
  __shared__ unsigned long long keys[kPermMaxB];
  const int base = blockIdx.x * kPermMaxB;
  for (int d = blockIdx.y; d < D; d += gridDim.y) {
    const unsigned long long off = *offset_dev + (unsigned long long)d * (unsigned long long)B;
    for (int j = threadIdx.x; j < kPermMaxB; j += blockDim.x) keys[j] = base + j < B ? perm_key(off, base + j, seed) : ~0ull;
    __syncthreads();
    bitonic_sort_smem(keys, kPermMaxB);
    unsigned long long* dst = sorted + (long long)d * B + base;
    for (int j = threadIdx.x; j < kPermMaxB && base + j < B; j += blockDim.x) dst[j] = keys[j];
    __syncthreads();                                   // keys[] is refilled for the next dimension
  }
}

// Merge pass: the sorted runs [2k*w, (2k+1)*w) and [(2k+1)*w, (2k+2)*w) of every dimension become one sorted run of
// 2w.  A key's place in the merged run is its place in its own run plus the number of keys of the partner run below
// it (a binary search; the keys are unique, so no tie rule is needed).  Every key is written once: no atomics.
__global__ void __launch_bounds__(256)
permute_merge_kernel(const unsigned long long* __restrict__ src, unsigned long long* __restrict__ dst, int B, int D, int w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  const int run = i / w, pair0 = (run & ~1) * w;
  const int p0 = (run & 1) ? pair0 : (int)min((long long)pair0 + w, (long long)B);
  const int p1 = (run & 1) ? pair0 + w : (int)min((long long)pair0 + 2ll * w, (long long)B);
  for (int d = blockIdx.y; d < D; d += gridDim.y) {
    const unsigned long long* s = src + (long long)d * B;
    const unsigned long long k = s[i];
    int lo = p0, hi = p1;                              // ends as p0 + (keys of the partner run below k)
    while (lo < hi) {
      const int mid = (int)(((unsigned)lo + (unsigned)hi) >> 1);   // no int overflow for runs near INT_MAX
      if (s[mid] < k) lo = mid + 1; else hi = mid;
    }
    dst[(long long)d * B + pair0 + (i - run * w) + (lo - p0)] = k;
  }
}

// Gather of the window from the fully sorted keys.
__global__ void permute_sorted_gather_kernel(const float* __restrict__ z, const unsigned long long* __restrict__ sorted,
                                             float* __restrict__ out, int B, int D, int row0, int nrows) {
  const long long n = (long long)nrows * D;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / D), d = (int)(i % D);
    const long long src = (long long)(sorted[(long long)d * B + row0 + b] & 0xffffffffull);
    out[i] = z[src * D + d];
  }
}
// In place over the fully sorted keys of one dimension: key i becomes its row index as int64 (keys and idx alias).
__global__ void sorted_index_column_kernel(unsigned long long* keys, int n) {
  long long* idx = reinterpret_cast<long long*>(keys);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    idx[i] = (long long)(keys[i] & 0xffffffffull);
}
__global__ void advance_offset2_kernel(unsigned long long* offset_dev, unsigned long long by) { *offset_dev += by; }

__global__ void __launch_bounds__(256) factor_tc_fwd_kernel(const float* __restrict__ d_z, int h, float* __restrict__ tc) {
  __shared__ float red[8];
  float s = 0.f;
  for (int b = threadIdx.x; b < h; b += blockDim.x) s += d_z[2 * b] - d_z[2 * b + 1];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) { float t = 0.f; for (int w = 0; w < 8; ++w) t += red[w]; tc[0] = t / (float)h; }
}
__global__ void factor_tc_bwd_kernel(const float* __restrict__ upstream, int h, float* __restrict__ g) {
  const float u = upstream[0] / (float)h;
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < h; b += gridDim.x * blockDim.x) { g[2 * b] = u; g[2 * b + 1] = -u; }
}

__device__ __forceinline__ float nll2(float x0, float x1, int target) {
  const float m = fmaxf(x0, x1);
  const float lse = m + logf(expf(x0 - m) + expf(x1 - m));
  return lse - (target == 0 ? x0 : x1);
}
__global__ void __launch_bounds__(256)
factor_ce_fwd_kernel(const float* __restrict__ d_z, const float* __restrict__ d_perm, int h, float* __restrict__ out) {
  __shared__ float red[2][8];
  float s0 = 0.f, s1 = 0.f;
  for (int b = threadIdx.x; b < h; b += blockDim.x) {
    s0 += nll2(d_z[2 * b], d_z[2 * b + 1], 0);
    s1 += nll2(d_perm[2 * b], d_perm[2 * b + 1], 1);
  }
  s0 = warp_sum(s0); s1 = warp_sum(s1);
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = s0; red[1][threadIdx.x >> 5] = s1; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t0 = 0.f, t1 = 0.f;
    for (int w = 0; w < 8; ++w) { t0 += red[0][w]; t1 += red[1][w]; }
    out[0] = 0.5f * (t0 / (float)h + t1 / (float)h);
  }
}
__global__ void factor_ce_bwd_kernel(const float* __restrict__ d_z, const float* __restrict__ d_perm,
                                     const float* __restrict__ upstream, int h, float* __restrict__ g_z, float* __restrict__ g_p) {
  const float u = upstream[0] * 0.5f / (float)h;
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < h; b += gridDim.x * blockDim.x) {
    {
      const float x0 = d_z[2 * b], x1 = d_z[2 * b + 1], m = fmaxf(x0, x1);
      const float e0 = expf(x0 - m), e1 = expf(x1 - m), inv = 1.f / (e0 + e1);
      if (g_z) { g_z[2 * b] = u * (e0 * inv - 1.f); g_z[2 * b + 1] = u * (e1 * inv); }
    }
    {
      const float x0 = d_perm[2 * b], x1 = d_perm[2 * b + 1], m = fmaxf(x0, x1);
      const float e0 = expf(x0 - m), e1 = expf(x1 - m), inv = 1.f / (e0 + e1);
      if (g_p) { g_p[2 * b] = u * (e0 * inv); g_p[2 * b + 1] = u * (e1 * inv - 1.f); }
    }
  }
}

}  // namespace dv

using namespace dv;

extern "C" {

int dv_permute_dims(const float* z, const long long* perms, unsigned long long seed, unsigned long long* offset_dev,
                    float* out, int B, int D, void* stream) {
  if (!z || !out) return DV_ERR_BAD_ARG;
  if (B <= 0 || D <= 0) return DV_ERR_BAD_SHAPE;
  cudaStream_t st = as_stream(stream);
  if (perms) {
    const long long n = (long long)B * D;
    int grid = (int)((n + 255) / 256); if (grid > 4 * kNumSMs) grid = 4 * kNumSMs;
    permute_given_kernel<<<grid, 256, 0, st>>>(z, perms, out, B, D, 0, B);
    return check_launch();
  }
  if (!offset_dev) return DV_ERR_BAD_ARG;
  if (B > kPermMaxB) return DV_ERR_BAD_SHAPE;
  int npow2 = 2; while (npow2 < B) npow2 <<= 1;
  permute_philox_kernel<<<D, 512, npow2 * sizeof(unsigned long long), st>>>(z, seed, offset_dev, out, B, D, npow2, 0, B);
  int rc = check_launch();
  if (rc != DV_OK) return rc;
  advance_offset2_kernel<<<1, 1, 0, st>>>(offset_dev, (unsigned long long)B * D);
  return check_launch();
}

size_t dv_permute_dims_workspace_bytes(int B, int D) {
  if (B <= kPermMaxB || D <= 0) return 0;
  return 2 * (size_t)B * (size_t)D * sizeof(unsigned long long);
}

int dv_permute_dims_rows(const float* z, const long long* perms, unsigned long long seed, unsigned long long* offset_dev,
                         float* out, int B, int D, int row0, int nrows, void* workspace, void* stream) {
  if (B < 1 || D < 1 || row0 < 0 || nrows < 1 || row0 > B - nrows || (long long)B * D > INT_MAX) return DV_ERR_BAD_SHAPE;
  if (!z || !out) return DV_ERR_BAD_ARG;
  cudaStream_t st = as_stream(stream);
  const long long n = (long long)nrows * D;
  const int gather_grid = (int)std::min<long long>((n + 255) / 256, 4 * kNumSMs);
  if (perms) {
    permute_given_kernel<<<gather_grid, 256, 0, st>>>(z, perms, out, B, D, row0, nrows);
    return check_launch();
  }
  if (!offset_dev) return DV_ERR_BAD_ARG;
  int rc;
  if (B <= kPermMaxB) {
    int npow2 = 2; while (npow2 < B) npow2 <<= 1;
    permute_philox_kernel<<<D, 512, npow2 * sizeof(unsigned long long), st>>>(z, seed, offset_dev, out, B, D, npow2,
                                                                             row0, nrows);
    rc = check_launch();
  } else {
    if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 7)) return DV_ERR_BAD_ARG;
    unsigned long long* buf[2] = {static_cast<unsigned long long*>(workspace),
                                  static_cast<unsigned long long*>(workspace) + (size_t)B * D};
    const int dims = std::min(D, 65535);
    permute_tile_sort_kernel<<<dim3((B + kPermMaxB - 1) / kPermMaxB, dims), 512, 0, st>>>(seed, offset_dev, buf[0], B, D);
    rc = check_launch();
    int cur = 0;
    for (long long w = kPermMaxB; w < B && rc == DV_OK; w *= 2, cur ^= 1) {
      permute_merge_kernel<<<dim3((B + 255) / 256, dims), 256, 0, st>>>(buf[cur], buf[cur ^ 1], B, D, (int)w);
      rc = check_launch();
    }
    if (rc == DV_OK) {
      permute_sorted_gather_kernel<<<gather_grid, 256, 0, st>>>(z, buf[cur], out, B, D, row0, nrows);
      rc = check_launch();
    }
  }
  if (rc != DV_OK) return rc;
  advance_offset2_kernel<<<1, 1, 0, st>>>(offset_dev, (unsigned long long)B * D);
  return check_launch();
}

size_t dv_index_permutation_workspace_bytes(int N) {
  return N > kPermMaxB ? (size_t)N * sizeof(unsigned long long) : 0;
}

int dv_index_permutation(int N, unsigned long long seed, unsigned long long* offset_dev, long long* out_idx,
                         void* workspace, void* stream) {
  if (N < 1) return DV_ERR_BAD_SHAPE;
  if (!offset_dev || !out_idx || (reinterpret_cast<uintptr_t>(out_idx) & 7)) return DV_ERR_BAD_ARG;
  int passes = 0;
  for (long long w = kPermMaxB; w < N; w *= 2) ++passes;
  if (passes > 0 && (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 7))) return DV_ERR_BAD_ARG;
  // The key buffers ping-pong between out_idx (N x 8 bytes, like the keys) and the workspace; the tile pass writes to
  // the one that makes the last merge pass land in out_idx, where the index column is then extracted in place.
  unsigned long long* out_keys = reinterpret_cast<unsigned long long*>(out_idx);
  unsigned long long* ws = static_cast<unsigned long long*>(workspace);
  unsigned long long* buf[2] = {(passes & 1) ? ws : out_keys, (passes & 1) ? out_keys : ws};
  cudaStream_t st = as_stream(stream);
  permute_tile_sort_kernel<<<dim3((N + kPermMaxB - 1) / kPermMaxB, 1), 512, 0, st>>>(seed, offset_dev, buf[0], N, 1);
  int rc = check_launch();
  int cur = 0;
  for (long long w = kPermMaxB; w < N && rc == DV_OK; w *= 2, cur ^= 1) {
    permute_merge_kernel<<<dim3((N + 255) / 256, 1), 256, 0, st>>>(buf[cur], buf[cur ^ 1], N, 1, (int)w);
    rc = check_launch();
  }
  if (rc != DV_OK) return rc;
  sorted_index_column_kernel<<<(int)std::min<long long>((N + 255) / 256, 8 * kNumSMs), 256, 0, st>>>(out_keys, N);
  rc = check_launch();
  if (rc != DV_OK) return rc;
  advance_offset2_kernel<<<1, 1, 0, st>>>(offset_dev, (unsigned long long)N);
  return check_launch();
}

int dv_factor_tc_fwd(const float* d_z, int h, float* tc, void* stream) {
  if (!d_z || !tc) return DV_ERR_BAD_ARG;
  if (h <= 0) return DV_ERR_BAD_SHAPE;
  factor_tc_fwd_kernel<<<1, 256, 0, as_stream(stream)>>>(d_z, h, tc);
  return check_launch();
}
int dv_factor_tc_bwd(const float* upstream, int h, float* g_d_z, void* stream) {
  if (!upstream || !g_d_z) return DV_ERR_BAD_ARG;
  if (h <= 0) return DV_ERR_BAD_SHAPE;
  factor_tc_bwd_kernel<<<(h + 255) / 256, 256, 0, as_stream(stream)>>>(upstream, h, g_d_z);
  return check_launch();
}
int dv_factor_ce_fwd(const float* d_z, const float* d_perm, int h, float* out, void* stream) {
  if (!d_z || !d_perm || !out) return DV_ERR_BAD_ARG;
  if (h <= 0) return DV_ERR_BAD_SHAPE;
  factor_ce_fwd_kernel<<<1, 256, 0, as_stream(stream)>>>(d_z, d_perm, h, out);
  return check_launch();
}
int dv_factor_ce_bwd(const float* d_z, const float* d_perm, const float* upstream, int h, float* g_d_z, float* g_d_perm, void* stream) {
  if (!d_z || !d_perm || !upstream) return DV_ERR_BAD_ARG;
  if (h <= 0) return DV_ERR_BAD_SHAPE;
  factor_ce_bwd_kernel<<<(h + 255) / 256, 256, 0, as_stream(stream)>>>(d_z, d_perm, upstream, h, g_d_z, g_d_perm);
  return check_launch();
}

}  // extern "C"

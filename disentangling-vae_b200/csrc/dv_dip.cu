// DIP-VAE covariance penalty (Kumar et al. 2018, "Variational Inference of Disentangled Latent Concepts from Unlabeled
// Observations", eq. 6 for DIP-VAE-I and the second form of section 3 for DIP-VAE-II).  The reference has no DIP-VAE;
// the entry points are declared in include/disvae_b200.h.
//
//   c_b   = (mu_b - m1) - r,  m1 = s + mean_b(mu_b - s) with s = mu_0 (row 0),  r = mean_b(mu_b - m1)
//           Near s the differences are exact in fp32, so the offset of a column never enters a rounded sum (a plain
//           fp32 mean of 2048 values near 100 is off by 1e-5..1e-4).  But when row 0 is an outlier every mu_b - s is
//           rounded at the outlier's scale and m1 is off by about that much; the second pass takes the differences
//           from m1, which is within a few ulps of the batch's spread of the true mean, so c_b is within a few u |c_b|
//           plus the mean's rounding of the spread, wherever the column sits and whichever row comes first.
//   C     = (1/B) sum_b c_b c_b^T            (+ diag(mean_b exp(logvar_b)) for DIP-VAE-II)
//   od    = sum_{i != j} C_ij^2,   dd = sum_i (C_ii - 1)^2
//   d/dmu_b     = (2/B) G c_b,  G_ij = 2 g_od C_ij (i != j),  G_ii = 2 g_dd (C_ii - 1)
//   d/dlogvar_bi = G_ii exp(logvar_bi) / B   (DIP-VAE-II)
//
// Forward: two launches.  dip_mean_kernel takes m1 and r (one CTA per column, two passes) and zeroes the counters;
// dip_cov_kernel runs one CTA per (32x32 tile of C, chunk of the batch), writes the tile's partial sum over its chunk
// and the last CTA of a tile (counter) sums the chunks in chunk order; the last tile (second counter) sums the tiles'
// (od, dd) in tile order.  Backward: one launch, one CTA per 32 rows x 32 columns of the mu gradient.  Every sum has a
// fixed order and no floating-point atomics: results are bit-identical run to run, and C is exactly symmetric (the
// (i, j) and (j, i) entries are the same products fmaf(a, b) == fmaf(b, a) summed in the same order).
#include "dv_common.cuh"

namespace dv {
namespace {

constexpr int kDipTile = 32;
constexpr int kDipTileElems = kDipTile * kDipTile;
constexpr int kDipThreads = 256;                   // 32 rows x 8 threads, 4 columns each (stride 8)
constexpr int kDipTargetCtas = 2 * kNumSMs;        // the batch is split until the covariance pass has about this many CTAs
constexpr int kDipMinChunk = 64;                   // ... or its chunks have this many rows
constexpr int kDipMaxB = 65535 * kDipTile;         // the backward's grid y is ceil(B / 32)

size_t round4(size_t n) { return (n + 3) & ~size_t(3); }

// Workspace layout (floats, each piece a multiple of 16 bytes): counters [ntiles + 1] (unsigned), m1 [D] (shifted
// column means), r [D] (column means of mu - m1), v [D] (column means of exp(logvar), DIP-VAE-II), C [D][D], chunk
// partials [nchunks][ntiles][32 * 32], tile (od, dd) [ntiles][2].
struct DipPlan {
  int tps, ntiles, chunk, nchunks;
  size_t m, r, v, c, part, red, total;
};

DipPlan dip_plan(int B, int D) {
  DipPlan p;
  p.tps = (D + kDipTile - 1) / kDipTile;
  p.ntiles = p.tps * p.tps;
  int want = kDipTargetCtas / p.ntiles;
  const int by_rows = (B + kDipMinChunk - 1) / kDipMinChunk;     // a chunk of fewer rows costs more to reduce than to sum
  if (want > by_rows) want = by_rows;
  if (want < 1) want = 1;
  const int rows = (B + want - 1) / want;
  p.chunk = (rows + kDipTile - 1) / kDipTile * kDipTile;
  p.nchunks = (B + p.chunk - 1) / p.chunk;
  p.m = round4((size_t)p.ntiles + 1);
  p.r = p.m + round4(D);
  p.v = p.r + round4(D);
  p.c = p.v + round4(D);
  p.part = p.c + round4((size_t)D * D);
  p.red = p.part + (size_t)p.nchunks * p.ntiles * kDipTileElems;
  p.total = p.red + round4(2 * (size_t)p.ntiles);
  return p;
}

// Sum over the CTA of two values in a fixed order; valid in thread 0.
__device__ __forceinline__ float2 dip_block_sum2(float a, float b, float2* red /* [8] */) {
  a = warp_sum(a);
  b = warp_sum(b);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = make_float2(a, b);
  __syncthreads();
  float2 t = make_float2(0.f, 0.f);
  if (warp == 0) {
    const float2 x = lane < kDipThreads / 32 ? red[lane] : make_float2(0.f, 0.f);
    t = make_float2(warp_sum(x.x), warp_sum(x.y));
  }
  return t;
}

// One CTA per column d: m1[d] = mu[0][d] + mean_b(mu[b][d] - mu[0][d]), r[d] = mean_b(mu[b][d] - m1[d]),
// v[d] = mean_b exp(logvar[b][d]) (DIP-VAE-II).
__global__ void __launch_bounds__(kDipThreads)
dip_mean_kernel(const float* __restrict__ mu, const float* __restrict__ logvar, int ld, int rs, int B, int dip_type,
                float* __restrict__ m, float* __restrict__ r, float* __restrict__ v, unsigned* __restrict__ cnt,
                int ncnt) {
  __shared__ float2 wred[kDipThreads / 32];
  __shared__ float m1_s;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ncnt; i += gridDim.x * blockDim.x) cnt[i] = 0u;
  const int d = blockIdx.x;
  const float s = mu[(long long)d * ld];
  float t = 0.f, e = 0.f;
#pragma unroll 4
  for (int b = threadIdx.x; b < B; b += kDipThreads) {
    const long long o = (long long)b * rs + (long long)d * ld;
    t += mu[o] - s;
    if (dip_type == DV_DIP_II) e += expf(logvar[o]);
  }
  const float2 sum = dip_block_sum2(t, e, wred);
  if (threadIdx.x == 0) m1_s = s + sum.x / (float)B;
  __syncthreads();
  const float m1 = m1_s;
  float t2 = 0.f;
#pragma unroll 4
  for (int b = threadIdx.x; b < B; b += kDipThreads) t2 += mu[(long long)b * rs + (long long)d * ld] - m1;
  const float2 sum2 = dip_block_sum2(t2, 0.f, wred);
  if (threadIdx.x == 0) {
    m[d] = m1;
    r[d] = sum2.x / (float)B;
    v[d] = sum.y / (float)B;
  }
}

__global__ void __launch_bounds__(kDipThreads)
dip_cov_kernel(const float* __restrict__ mu, int ld, int rs, int B, int D, int dip_type, int tps, int chunk,
               const float* __restrict__ m, const float* __restrict__ r, const float* __restrict__ v,
               float* __restrict__ C, float* __restrict__ part, float* __restrict__ red, unsigned* __restrict__ cnt,
               float* __restrict__ terms) {
  __shared__ float sa[kDipTile][kDipTile + 1], sb[kDipTile][kDipTile + 1];
  __shared__ float shift[2][kDipTile], rmean[2][kDipTile];
  __shared__ float2 wred[kDipThreads / 32];
  __shared__ bool is_last;
  const int tile = blockIdx.x, ntiles = gridDim.x, nchunks = gridDim.y;
  const int i0 = (tile / tps) * kDipTile, j0 = (tile % tps) * kDipTile;
  const int t = threadIdx.x, ty = t >> 3, tx = t & 7;
  if (t < 2 * kDipTile) {
    const int side = t >> 5, col = (side ? j0 : i0) + (t & 31);
    shift[side][t & 31] = col < D ? m[col] : 0.f;
    rmean[side][t & 31] = col < D ? r[col] : 0.f;
  }
  __syncthreads();

  // (1) partial sums over this CTA's chunk of rows: acc[q] = sum_b c_b[i0 + ty] * c_b[j0 + tx + 8q]
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const int b_begin = blockIdx.y * chunk, b_end = min(B, b_begin + chunk);
  for (int b0 = b_begin; b0 < b_end; b0 += kDipTile) {
#pragma unroll
    for (int k = 0; k < kDipTileElems / kDipThreads; ++k) {
      const int e = t + kDipThreads * k, row = e >> 5, col = e & 31, b = b0 + row;
      float xa = 0.f, xb = 0.f;
      if (b < b_end) {
        const long long o = (long long)b * rs;
        if (i0 + col < D) xa = (mu[o + (long long)(i0 + col) * ld] - shift[0][col]) - rmean[0][col];
        if (j0 + col < D) xb = (mu[o + (long long)(j0 + col) * ld] - shift[1][col]) - rmean[1][col];
      }
      sa[row][col] = xa;
      sb[row][col] = xb;
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < kDipTile; ++k) {
      const float a = sa[k][ty];
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[q] = fmaf(a, sb[k][tx + 8 * q], acc[q]);
    }
    __syncthreads();
  }
  float* pt = part + ((size_t)blockIdx.y * ntiles + tile) * kDipTileElems + ty * kDipTile + tx;
#pragma unroll
  for (int q = 0; q < 4; ++q) pt[8 * q] = acc[q];

  // (2) the last CTA of this tile sums the chunks in chunk order -> C, and the tile's (od, dd)
  __threadfence();
  __syncthreads();
  if (t == 0) is_last = atomicAdd(&cnt[tile], 1u) == (unsigned)(nchunks - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  float od = 0.f, dd = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = i0 + ty, j = j0 + tx + 8 * q;
    const float* src = part + (size_t)tile * kDipTileElems + ty * kDipTile + tx + 8 * q;
    float s = 0.f;
#pragma unroll 8
    for (int p = 0; p < nchunks; ++p) s += __ldcg(src + (size_t)p * ntiles * kDipTileElems);
    if (i < D && j < D) {
      float c = s / (float)B;
      if (i == j) {
        if (dip_type == DV_DIP_II) c += v[i];
        dd += (c - 1.f) * (c - 1.f);
      } else {
        od += c * c;
      }
      C[(size_t)i * D + j] = c;
    }
  }
  const float2 tsum = dip_block_sum2(od, dd, wred);
  if (t == 0) {
    red[2 * tile] = tsum.x;
    red[2 * tile + 1] = tsum.y;
  }

  // (3) the last tile sums the tiles' (od, dd) in tile order
  __threadfence();
  __syncthreads();
  if (t == 0) is_last = atomicAdd(&cnt[ntiles], 1u) == (unsigned)(ntiles - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  od = dd = 0.f;
  for (int k = t; k < ntiles; k += kDipThreads) {
    od += __ldcg(red + 2 * k);
    dd += __ldcg(red + 2 * k + 1);
  }
  const float2 all = dip_block_sum2(od, dd, wred);
  if (t == 0) {
    terms[0] = all.x;
    terms[1] = all.y;
  }
}

__global__ void __launch_bounds__(kDipThreads)
dip_bwd_kernel(const float* __restrict__ mu, const float* __restrict__ logvar, int ld, int rs, int B, int D, int dip_type,
               const float* __restrict__ m, const float* __restrict__ r, const float* __restrict__ C,
               const float* __restrict__ g_terms, float* __restrict__ g_mu, float* __restrict__ g_logvar) {
  __shared__ float sc[kDipTile][kDipTile + 1];     // centred mu [b][j]
  __shared__ float sg[kDipTile][kDipTile + 1];     // G [j][i]
  const int i0 = blockIdx.x * kDipTile, b0 = blockIdx.y * kDipTile;
  const int t = threadIdx.x, ty = t >> 3, tx = t & 7;
  const float god2 = 2.f * g_terms[0], gdd2 = 2.f * g_terms[1];
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int j0 = 0; j0 < D; j0 += kDipTile) {
#pragma unroll
    for (int k = 0; k < kDipTileElems / kDipThreads; ++k) {
      const int e = t + kDipThreads * k, row = e >> 5, col = e & 31;
      const int b = b0 + row, j = j0 + col;
      float x = 0.f;
      if (b < B && j < D) x = (mu[(long long)b * rs + (long long)j * ld] - m[j]) - r[j];
      sc[row][col] = x;
      const int jj = j0 + row, ii = i0 + col;
      float g = 0.f;
      if (jj < D && ii < D) {
        const float c = C[(size_t)jj * D + ii];
        g = jj == ii ? gdd2 * (c - 1.f) : god2 * c;
      }
      sg[row][col] = g;
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < kDipTile; ++k) {
      const float x = sc[ty][k];
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[q] = fmaf(x, sg[k][tx + 8 * q], acc[q]);
    }
    __syncthreads();
  }
  const int b = b0 + ty;
  if (b >= B) return;
  const float scale = 2.f / (float)B;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = i0 + tx + 8 * q;
    if (i >= D) continue;
    const size_t o = (size_t)b * D + i;
    if (g_mu) g_mu[o] = acc[q] * scale;
    if (g_logvar) {
      float g = 0.f;
      if (dip_type == DV_DIP_II) {
        const float gii = gdd2 * (C[(size_t)i * D + i] - 1.f);
        g = gii * expf(logvar[(long long)b * rs + (long long)i * ld]) / (float)B;
      }
      g_logvar[o] = g;
    }
  }
}

bool bad_dims(int B, int D) { return B < 1 || B > kDipMaxB || D < 1 || D > 1024; }

int dip_check(const float* mu, const float* logvar, int ld, int rs, int B, int D, int dip_type, const void* ws) {
  if (bad_dims(B, D) || ld < 1 || rs < 1 || (dip_type != DV_DIP_I && dip_type != DV_DIP_II)) return DV_ERR_BAD_SHAPE;
  if (!mu || !logvar || !ws) return DV_ERR_BAD_ARG;
  if (misaligned(mu, 4) || misaligned(logvar, 4) || misaligned(ws, 16)) return DV_ERR_BAD_ARG;
  return DV_OK;
}

}  // namespace
}  // namespace dv

using namespace dv;

extern "C" {

size_t dv_dip_workspace_bytes(int B, int D) {
  if (bad_dims(B, D)) return 0;
  return dip_plan(B, D).total * sizeof(float);
}

int dv_dip_fwd(const float* mu, const float* logvar, int ld, int row_stride, int B, int D, int dip_type,
               float* terms_out, void* workspace, void* stream) {
  int rc = dip_check(mu, logvar, ld, row_stride, B, D, dip_type, workspace);
  if (rc != DV_OK) return rc;
  if (!terms_out || misaligned(terms_out, 4)) return DV_ERR_BAD_ARG;
  const DipPlan p = dip_plan(B, D);
  float* ws = reinterpret_cast<float*>(workspace);
  unsigned* cnt = reinterpret_cast<unsigned*>(ws);
  dip_mean_kernel<<<D, kDipThreads, 0, as_stream(stream)>>>(mu, logvar, ld, row_stride, B, dip_type, ws + p.m, ws + p.r,
                                                            ws + p.v, cnt, p.ntiles + 1);
  rc = check_launch();
  if (rc != DV_OK) return rc;
  dip_cov_kernel<<<dim3(p.ntiles, p.nchunks), kDipThreads, 0, as_stream(stream)>>>(
      mu, ld, row_stride, B, D, dip_type, p.tps, p.chunk, ws + p.m, ws + p.r, ws + p.v, ws + p.c, ws + p.part,
      ws + p.red, cnt, terms_out);
  return check_launch();
}

int dv_dip_bwd(const float* mu, const float* logvar, int ld, int row_stride, int B, int D, int dip_type,
               const float* g_terms, float* g_mu, float* g_logvar, const void* workspace, void* stream) {
  int rc = dip_check(mu, logvar, ld, row_stride, B, D, dip_type, workspace);
  if (rc != DV_OK) return rc;
  if (!g_terms || misaligned(g_terms, 4) || misaligned(g_mu, 4) || misaligned(g_logvar, 4)) return DV_ERR_BAD_ARG;
  if (!g_mu && !g_logvar) return DV_OK;
  const DipPlan p = dip_plan(B, D);
  const float* ws = reinterpret_cast<const float*>(workspace);
  dip_bwd_kernel<<<dim3((D + kDipTile - 1) / kDipTile, (B + kDipTile - 1) / kDipTile), kDipThreads, 0,
                   as_stream(stream)>>>(mu, logvar, ld, row_stride, B, D, dip_type, ws + p.m, ws + p.r, ws + p.c,
                                        g_terms, g_mu, g_logvar);
  return check_launch();
}

}  // extern "C"

// Unsupervised Disentanglement Ranking (Duan et al., ICLR 2020; disentanglement_lib's udr.py, compute_udr_sklearn):
// for K models encoding the same n points, every model's per-latent KL, its standardised (Lasso) or rank (Spearman)
// features, the similarity matrix R_ij of every ordered pair and the pair's relative-strength score.  The reference has
// no such score; the entry points and their rules are declared in include/disvae_b200.h.
//
// dv_udr_fit (three launches, no host synchronisation):
//   column  one CTA per (model, latent): the KL mean over the points in fp64, the informative mask, then the column's
//           features into Z [K D][n] fp64 -- (x - mean) / std, or in Spearman mode the average ranks of the fp32
//           values (a bitonic sort of (value, row) keys in shared memory) standardised the same way; 0 when the latent
//           is not informative.
//   gram    P = Z Z^T / n over all K D columns: 64 x 64 tiles of the upper triangle, each output one fp64 accumulator
//           over the points in order, mirrored below the diagonal.
//   pair    one CTA per ordered pair (i, j): Lasso -- one warp per target latent b of j runs cyclic coordinate descent
//           on G_i (block (i, i) of P) and the column b of C_ij (block (i, j)) to a duality gap of 1e-12 of the
//           target's y^T y / n; Spearman -- |P| of block (i, j).  Then the filter and the pair score.
// Every sum has a fixed order and there are no floating-point atomics, so results are bit-identical run to run.
#include <float.h>
#include <math_constants.h>

#include "dv_common.cuh"

namespace dv {
namespace {

constexpr int kUdrMaxD = 128;                 // latents of a model (the Lasso warp keeps 4 coordinates per lane)
constexpr int kUdrMaxCols = 4096;             // K * D: P is at most 4096^2 fp64 = 128 MiB
constexpr int kUdrMaxN = 16384;               // points: the Spearman sort keys fill 128 KiB of shared memory
constexpr int kUdrMaxSweeps = 10000;          // coordinate-descent sweeps of one Lasso fit
constexpr double kUdrGapTol = 1e-12;          // duality gap relative to y^T y / n
constexpr int kColThreads = 512;
constexpr int kColWarps = kColThreads / kWarp;
constexpr int kTile = 64;                     // gram tile (outputs), 4 x 4 per thread
constexpr int kTileK = 16;                    // points per staged slice
constexpr int kGramThreads = 256;
constexpr int kPairThreads = 256;
constexpr int kPairWarps = kPairThreads / kWarp;

struct UdrWs {
  double* z;    // [K D][n] features
  double* p;    // [K D][K D] = Z Z^T / n
};

size_t udr_layout(int K, int n, int D, char* base, UdrWs* w) {
  const size_t M = (size_t)K * D;
  const size_t sizes[2] = {M * n * 8, M * M * 8};
  size_t off[2];
  const size_t total = carve_workspace(sizes, off);
  if (w) {
    w->z = reinterpret_cast<double*>(base + off[0]);
    w->p = reinterpret_cast<double*>(base + off[1]);
  }
  return total;
}

// An order-preserving integer key of an fp32 value (-0 taken as +0).
__device__ __forceinline__ unsigned int f32_key(float v) {
  const unsigned int u = __float_as_uint(v == 0.f ? 0.f : v);
  return (u >> 31) ? ~u : (u | 0x80000000u);
}

// First index in keys[0, len) whose upper 32 bits are >= hi (keys sorted ascending).
__device__ __forceinline__ int lower_bound_hi(const unsigned long long* keys, int len, unsigned long long hi) {
  int a = 0, b = len;
  while (a < b) {
    const int h = (a + b) >> 1;
    if ((keys[h] >> 32) < hi) a = h + 1; else b = h;
  }
  return a;
}

// Mean and standard deviation (ddof 0, 0 -> 1) of z[0, n), each a fixed-order fp64 sum; z <- (z - mean) / std.
__device__ void standardise_column(double* z, int n, double* red) {
  const int t = threadIdx.x;
  double s = 0.0;
  for (int i = t; i < n; i += kColThreads) s += z[i];
  const double mean = block_sum<kColWarps>(s, red) / n;
  s = 0.0;
  for (int i = t; i < n; i += kColThreads) {
    const double e = __dsub_rn(z[i], mean);
    s = __dadd_rn(s, __dmul_rn(e, e));
  }
  double sd = sqrt(block_sum<kColWarps>(s, red) / n);
  if (sd == 0.0) sd = 1.0;                                     // StandardScaler's rule for a constant feature
  for (int i = t; i < n; i += kColThreads) z[i] = __ddiv_rn(__dsub_rn(z[i], mean), sd);
}

__global__ void __launch_bounds__(kColThreads)
udr_column_kernel(const float* __restrict__ mu, const float* __restrict__ logvar, int n, int D, int spearman,
                  double kl_threshold, double* __restrict__ kl_out, UdrWs w) {
  extern __shared__ unsigned long long key[];                  // [pow2 >= n] (Spearman only)
  __shared__ double red[kColWarps];
  const int t = threadIdx.x, col = blockIdx.x, k = col / D, d = col % D;
  const float* m = mu + (long long)k * n * D + d;
  const float* lv = logvar + (long long)k * n * D + d;
  double s = 0.0;
  for (int i = t; i < n; i += kColThreads) {
    const double u = (double)m[(long long)i * D], v = (double)lv[(long long)i * D];
    // 0.5 (mu^2 + exp(logvar) - logvar - 1), added left to right
    s = __dadd_rn(s, __dmul_rn(0.5, __dsub_rn(__dsub_rn(__dadd_rn(__dmul_rn(u, u), exp(v)), v), 1.0)));
  }
  const double kl = block_sum<kColWarps>(s, red) / n;
  if (t == 0) kl_out[col] = kl;
  double* z = w.z + (long long)col * n;
  if (!(kl > kl_threshold)) {                                  // not informative: the feature is 0
    for (int i = t; i < n; i += kColThreads) z[i] = 0.0;
    return;
  }
  if (!spearman) {
    for (int i = t; i < n; i += kColThreads) z[i] = (double)m[(long long)i * D];
  } else {
    int P2 = 1;
    while (P2 < n) P2 <<= 1;
    for (int i = t; i < P2; i += kColThreads)
      key[i] = i < n ? ((unsigned long long)f32_key(m[(long long)i * D]) << 32) | (unsigned)i : ~0ull;
    __syncthreads();
    for (int kk = 2; kk <= P2; kk <<= 1) {
      for (int j = kk >> 1; j > 0; j >>= 1) {
        for (int i = t; i < P2; i += kColThreads) {
          const int o = i ^ j;
          if (o > i) {
            const unsigned long long a = key[i], b = key[o];
            if ((a > b) == ((i & kk) == 0)) {
              key[i] = b;
              key[o] = a;
            }
          }
        }
        __syncthreads();
      }
    }
    // the average rank (1-based) of a run of equal values at sorted places [lo, hi) is (lo + hi + 1) / 2
    for (int p = t; p < n; p += kColThreads) {
      const unsigned long long v = key[p] >> 32;
      const int lo = lower_bound_hi(key, n, v), hi = lower_bound_hi(key, n, v + 1);
      z[(unsigned)(key[p] & 0xffffffffu)] = 0.5 * (double)(lo + hi + 1);
    }
  }
  __syncthreads();
  standardise_column(z, n, red);
}

// P[a][b] = sum_i Z[a][i] Z[b][i] / n for the tiles on or above the diagonal; each output is one accumulator over the
// points in order, written to (a, b) and (b, a).
__global__ void __launch_bounds__(kGramThreads)
udr_gram_kernel(int M, int n, UdrWs w) {
  __shared__ double sa[kTileK][kTile + 1], sb[kTileK][kTile + 1];
  // blockIdx.x enumerates the upper-triangular tile pairs (ta <= tb) row by row
  const int T = (M + kTile - 1) / kTile;
  int ta = 0, rem = blockIdx.x;
  while (rem >= T - ta) {
    rem -= T - ta;
    ++ta;
  }
  const int tb = ta + rem;
  const int t = threadIdx.x, tx = t % 16, ty = t / 16;
  const int a0 = ta * kTile, b0 = tb * kTile;
  double acc[4][4] = {};
  for (int k0 = 0; k0 < n; k0 += kTileK) {
    for (int e = t; e < kTile * kTileK; e += kGramThreads) {
      const int r = e / kTileK, c = e % kTileK, kk = k0 + c;
      sa[c][r] = (a0 + r < M && kk < n) ? w.z[(long long)(a0 + r) * n + kk] : 0.0;
      sb[c][r] = (b0 + r < M && kk < n) ? w.z[(long long)(b0 + r) * n + kk] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < kTileK; ++c) {
      double x[4], y[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        x[q] = sa[c][ty + 16 * q];
        y[q] = sb[c][tx + 16 * q];
      }
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int r = 0; r < 4; ++r) acc[q][r] = fma(x[q], y[r], acc[q][r]);
    }
    __syncthreads();
  }
  const double dn = (double)n;
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int a = a0 + ty + 16 * q, b = b0 + tx + 16 * r;
      if (a < M && b < M && a <= b) {
        const double v = __ddiv_rn(acc[q][r], dn);
        w.p[(long long)a * M + b] = v;
        w.p[(long long)b * M + a] = v;
      }
    }
}

__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One Lasso fit on a warp: min_w 1/2 (q - 2 c^T w + w^T G w) + alpha |w|_1 with G = P[g0 + a][g0 + b] and
// c = P[g0 + a][cb] (a, b < D), by cyclic coordinate descent keeping g = c - G w; after every sweep g is recomputed
// from w and the duality gap taken.  Lane l keeps coordinates l, l + 32, l + 64, l + 96.  -> sweeps, -1 at the cap.
__device__ int lasso_warp(const double* __restrict__ P, long long M, long long g0, long long cb, int D, double q,
                          double alpha, double (&w)[4]) {
  const int lane = threadIdx.x & (kWarp - 1);
  double c[4], g[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int a = lane + kWarp * r;
    w[r] = 0.0;
    c[r] = a < D ? P[(g0 + a) * M + cb] : 0.0;
    g[r] = c[r];
  }
  if (q == 0.0) return 0;                                      // y = 0: w = 0 is the minimiser
  const double tol = kUdrGapTol * q;
  for (int sweeps = 0;; ++sweeps) {
    // the gap of the current w, from g = c - G w recomputed in a fixed order
    if (sweeps > 0) {
#pragma unroll
      for (int r = 0; r < 4; ++r) g[r] = c[r];
#pragma unroll
      for (int rr = 0; rr < 4; ++rr)
        for (int l = 0; l < kWarp; ++l) {
          const int b = rr * kWarp + l;
          if (b >= D) break;
          const double wb = __shfl_sync(0xffffffffu, w[rr], l);
          if (wb == 0.0) continue;
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const int a = lane + kWarp * r;
            if (a < D) g[r] = fma(-P[(g0 + a) * M + g0 + b], wb, g[r]);
          }
        }
    }
    double cw = 0.0, wg = 0.0, l1 = 0.0, gmax = 0.0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      cw = fma(c[r], w[r], cw);
      wg = fma(w[r], g[r], wg);
      l1 += fabs(w[r]);
      if (lane + kWarp * r < D) gmax = fmax(gmax, fabs(g[r]));
    }
    cw = warp_sum(cw);
    wg = warp_sum(wg);
    l1 = warp_sum(l1);
    gmax = warp_max_d(gmax);
    const double r2 = q - cw - wg, ry = q - cw;               // |y - Xw|^2 / n and (y - Xw)^T y / n
    double gap, cst = 1.0;
    if (gmax > alpha) {
      cst = alpha / gmax;
      gap = 0.5 * r2 * (1.0 + cst * cst);
    } else {
      gap = r2;
    }
    gap += alpha * l1 - cst * ry;
    if (gap <= tol) return sweeps;
    if (sweeps == kUdrMaxSweeps) return -1;
    // one sweep over the coordinates in order
#pragma unroll
    for (int r = 0; r < 4; ++r)
      for (int l = 0; l < kWarp; ++l) {
        const int a = r * kWarp + l;
        if (a >= D) break;
        const double gaa = P[(g0 + a) * M + g0 + a];
        if (gaa == 0.0) continue;                              // an all-zero input: its coefficient stays 0
        const double wa = __shfl_sync(0xffffffffu, w[r], l), ga = __shfl_sync(0xffffffffu, g[r], l);
        const double rho = fma(gaa, wa, ga);
        const double mag = fabs(rho) - alpha;
        const double wn = mag > 0.0 ? copysign(mag, rho) / gaa : 0.0;
        const double delta = wn - wa;
        if (lane == l) w[r] = wn;
        if (delta == 0.0) continue;
#pragma unroll
        for (int rr = 0; rr < 4; ++rr) {
          const int b = lane + kWarp * rr;
          if (b < D) g[rr] = fma(-P[(g0 + a) * M + g0 + b], delta, g[rr]);
        }
      }
  }
}

__global__ void __launch_bounds__(kPairThreads)
udr_pair_kernel(int K, int D, int spearman, double alpha, double kl_threshold, const double* __restrict__ kl,
                double* __restrict__ raw, double* __restrict__ pair, int* __restrict__ iters, UdrWs w) {
  __shared__ int sweeps[kUdrMaxD];
  __shared__ double rx[kUdrMaxD], ry[kUdrMaxD];
  const int t = threadIdx.x, lane = t & (kWarp - 1), warp = t / kWarp;
  const int i = blockIdx.x / K, j = blockIdx.x % K;
  const long long M = (long long)K * D;
  double* R = raw + (long long)blockIdx.x * D * D;             // R[a][b]: a latent of i, b latent of j
  if (i == j) {
    for (int e = t; e < D * D; e += kPairThreads) R[e] = CUDART_NAN;
    if (t == 0) {
      pair[blockIdx.x] = CUDART_NAN;
      iters[blockIdx.x] = 0;
    }
    return;
  }
  const double* P = w.p;
  const long long gi = (long long)i * D, gj = (long long)j * D;
  if (spearman) {
    for (int e = t; e < D * D; e += kPairThreads) R[e] = fabs(P[(gi + e / D) * M + gj + e % D]);
  } else {
    for (int b = warp; b < D; b += kPairWarps) {
      double wv[4];
      const int s = lasso_warp(P, M, gi, gj + b, D, P[(gj + b) * M + gj + b], alpha, wv);
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int a = lane + kWarp * r;
        if (a < D) R[(long long)a * D + b] = fabs(wv[r]);
      }
      if (lane == 0) sweeps[b] = s;
    }
  }
  __syncthreads();
  // the pair score over the informative rows (i) and columns (j): per column and per row max^2 / sum, 0 for 0 / 0
  if (t < D) {
    const bool col_in = kl[gj + t] > kl_threshold, row_in = kl[gi + t] > kl_threshold;
    double mx = 0.0, s = 0.0;
    if (col_in)
      for (int a = 0; a < D; ++a)
        if (kl[gi + a] > kl_threshold) {
          const double v = R[(long long)a * D + t];
          mx = fmax(mx, v);
          s += v;
        }
    rx[t] = col_in && s > 0.0 ? __ddiv_rn(mx * mx, s) : 0.0;
    mx = 0.0;
    s = 0.0;
    if (row_in)
      for (int b = 0; b < D; ++b)
        if (kl[gj + b] > kl_threshold) {
          const double v = R[(long long)t * D + b];
          mx = fmax(mx, v);
          s += v;
        }
    ry[t] = row_in && s > 0.0 ? __ddiv_rn(mx * mx, s) : 0.0;
  }
  __syncthreads();
  if (t == 0) {
    int di = 0, dj = 0, it = 0;
    double sx = 0.0, sy = 0.0;
    for (int a = 0; a < D; ++a) {
      if (kl[gj + a] > kl_threshold) {
        ++dj;
        sx += rx[a];
      }
      if (kl[gi + a] > kl_threshold) {
        ++di;
        sy += ry[a];
      }
      if (!spearman) it = (it < 0 || sweeps[a] < 0) ? -1 : max(it, sweeps[a]);
    }
    pair[blockIdx.x] = (di == 0 || dj == 0) ? 0.0 : 0.5 * (sx / dj + sy / di);
    iters[blockIdx.x] = it;
  }
}

bool udr_shape_ok(int K, int n, int D) {
  return K >= 2 && D >= 1 && D <= kUdrMaxD && (long long)K * D <= kUdrMaxCols && n >= 2 && n <= kUdrMaxN;
}

}  // namespace
}  // namespace dv

using namespace dv;

extern "C" {

size_t dv_udr_workspace_bytes(int K, int n, int D) {
  if (!udr_shape_ok(K, n, D)) return 0;
  return udr_layout(K, n, D, nullptr, nullptr);
}

int dv_udr_fit(const float* mu, const float* logvar, int K, int n, int D, int mode, double alpha, double kl_threshold,
               double* raw, double* pair, double* kl, int* iters, void* workspace, size_t workspace_bytes,
               void* stream) {
  if (!udr_shape_ok(K, n, D)) return DV_ERR_BAD_SHAPE;
  if (!mu || !logvar || !raw || !pair || !kl || !iters) return DV_ERR_BAD_ARG;
  if (mode != DV_UDR_LASSO && mode != DV_UDR_SPEARMAN) return DV_ERR_BAD_ARG;
  if (!(alpha > 0.0 && alpha <= DBL_MAX) || !(kl_threshold >= 0.0 && kl_threshold <= DBL_MAX)) return DV_ERR_BAD_ARG;
  if (misaligned(mu, 4) || misaligned(logvar, 4) || misaligned(raw, 8) || misaligned(pair, 8) || misaligned(kl, 8) ||
      misaligned(iters, 4) || misaligned(workspace, 8))
    return DV_ERR_BAD_ARG;
  if (!workspace || workspace_bytes < udr_layout(K, n, D, nullptr, nullptr)) return DV_ERR_WORKSPACE;
  UdrWs w;
  udr_layout(K, n, D, static_cast<char*>(workspace), &w);
  const int spearman = mode == DV_UDR_SPEARMAN;
  int smem = 0;
  if (spearman) {
    smem = 8;
    while (smem < 8 * n) smem <<= 1;
    static bool attr = false;
    int rc = set_max_dynamic_smem(udr_column_kernel, 8 * kUdrMaxN, &attr);
    if (rc != DV_OK) return rc;
  }
  cudaStream_t s = as_stream(stream);
  const int M = K * D, T = (M + kTile - 1) / kTile;
  int rc;
  udr_column_kernel<<<M, kColThreads, smem, s>>>(mu, logvar, n, D, spearman, kl_threshold, kl, w);
  if ((rc = check_launch()) != DV_OK) return rc;
  udr_gram_kernel<<<T * (T + 1) / 2, kGramThreads, 0, s>>>(M, n, w);
  if ((rc = check_launch()) != DV_OK) return rc;
  udr_pair_kernel<<<K * K, kPairThreads, 0, s>>>(K, D, spearman, alpha, kl_threshold, kl, raw, pair, iters, w);
  return check_launch();
}

}  // extern "C"

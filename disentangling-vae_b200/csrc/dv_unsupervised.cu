// The unsupervised scores of disentanglement_lib's unsupervised_metrics.py (Locatello et al. 2019, section 5.1) on the
// mean and the sampled representation of n drawn points: the fp64 covariance of each, the eigenvalues of its
// correlation matrix R and of S = diag(c)^1/2 C diag(c)^1/2 (c = diag(C)), and the histogram mutual information of every
// pair of latents.  The reference has no such score; the entry point and its rules are declared in
// include/disvae_b200.h.
//
// dv_unsupervised_fit (six launches, no host synchronisation):
//   gather    one thread per (point, latent): the mean code and z = fmaf(expf(0.5f * logvar), eps, mu), both fp32, into
//             the workspace column by column ([2][D][n]); the row list 0 .. n - 1 for the mutual information.
//   column    one CTA per (representation, latent): the column mean in fp64 (a fixed-order sum), the 20 histogram edges
//             and bins (histogram_edges / histogram_bin, dv_discrete_mutual_info's), and the column's classes: each
//             row's bin renumbered over the occupied bins only.
//   cov       one CTA per (representation, i <= j): sum_k (x_ik - m_i)(x_jk - m_j) / (n - 1) in fp64, a fixed-order
//             sum over the points, written to (i, j) and (j, i).
//   eig       four CTAs, one per matrix (R and S of each representation): the matrix in fp64 shared memory, parallel
//             cyclic Jacobi in round-robin order (D/2 disjoint rotations per round, D - 1 rounds per sweep) until the
//             off-diagonal Frobenius norm is at most 1e-15 of the Frobenius norm; the diagonal sorted ascending.
//   mi x 2    dv_discrete_mutual_info once per representation, the classes of every latent as its K = D factors.
// Every sum has a fixed order and there are no floating-point atomics, so results are bit-identical run to run.
#include <float.h>
#include <math_constants.h>

#include "dv_common.cuh"

namespace dv {
namespace {

constexpr int kUnsMaxD = 128;                 // the Jacobi matrix, D (D + 1) fp64, fills 129 KiB of shared memory
constexpr int kUnsMaxN = 32768;               // dv_discrete_mutual_info keeps the bins in shared memory as bytes
constexpr int kUnsMaxSweeps = 50;
constexpr double kUnsOffTol2 = 1e-30;         // (off-diagonal norm / norm)^2 at convergence
constexpr int kGatherThreads = 256;
constexpr int kColThreads = 512;
constexpr int kColWarps = kColThreads / kWarp;
constexpr int kCovThreads = 256;
constexpr int kCovWarps = kCovThreads / kWarp;
constexpr int kEigThreads = 1024;
constexpr int kEigWarps = kEigThreads / kWarp;

struct UnsWs {
  float* codes;      // [2][D][n] the mean and the sampled codes, column by column
  double* mean;      // [2][D]
  int* cls;          // [2][D][n] classes (occupied bins renumbered 0 .. ncls - 1)
  int* ncls;         // [2][D]
  long long* rows;   // [n] 0 .. n - 1
};

size_t uns_layout(int n, int D, char* base, UnsWs* w) {
  const size_t cells = (size_t)2 * D * n;
  const size_t sizes[5] = {cells * 4, (size_t)2 * D * 8, cells * 4, (size_t)2 * D * 4, (size_t)n * 8};
  size_t off[5];
  const size_t total = carve_workspace(sizes, off);
  if (w) {
    w->codes = reinterpret_cast<float*>(base + off[0]);
    w->mean = reinterpret_cast<double*>(base + off[1]);
    w->cls = reinterpret_cast<int*>(base + off[2]);
    w->ncls = reinterpret_cast<int*>(base + off[3]);
    w->rows = reinterpret_cast<long long*>(base + off[4]);
  }
  return total;
}

__global__ void __launch_bounds__(kGatherThreads)
uns_gather_kernel(const float* __restrict__ mu, const float* __restrict__ logvar, int ld, int rs,
                  const long long* __restrict__ rows, int n, int D, const float* __restrict__ eps,
                  float* __restrict__ sampled, UnsWs w) {
  const long long e = (long long)blockIdx.x * kGatherThreads + threadIdx.x;
  if (e >= (long long)n * D) return;
  const int i = (int)(e % n), d = (int)(e / n);
  const long long at = rows[i] * (long long)rs + (long long)d * ld;
  const float m = mu[at];
  const float z = fmaf(expf(0.5f * logvar[at]), eps[(long long)i * D + d], m);
  w.codes[e] = m;
  w.codes[(long long)n * D + e] = z;
  if (sampled) sampled[(long long)i * D + d] = z;
  if (d == 0) w.rows[i] = i;
}

__global__ void __launch_bounds__(kColThreads)
uns_column_kernel(int n, UnsWs w) {
  __shared__ double red[kColWarps];
  __shared__ float wlo[kColWarps], whi[kColWarps];
  __shared__ float edge[kHistBins + 1];
  __shared__ int bcnt[kHistBins], renum[kHistBins];
  const int t = threadIdx.x, col = blockIdx.x;
  const float* x = w.codes + (long long)col * n;
  double s = 0.0;
  float lo = CUDART_INF_F, hi = -CUDART_INF_F;
  for (int i = t; i < n; i += kColThreads) {
    const float v = x[i];
    s += (double)v;
    lo = fminf(lo, v);
    hi = fmaxf(hi, v);
  }
  const double mean = block_sum<kColWarps>(s, red) / n;
  if (t < kHistBins) bcnt[t] = 0;
  histogram_edges<kColWarps>(lo, hi, wlo, whi, edge);
  for (int i = t; i < n; i += kColThreads) atomicAdd(&bcnt[histogram_bin(edge, x[i])], 1);
  __syncthreads();
  if (t == 0) {
    int o = 0;
    for (int j = 0; j < kHistBins; ++j) {
      renum[j] = o;
      o += bcnt[j] > 0 ? 1 : 0;
    }
    w.ncls[col] = o;
    w.mean[col] = mean;
  }
  __syncthreads();
  int* cls = w.cls + (long long)col * n;
  for (int i = t; i < n; i += kColThreads) cls[i] = renum[histogram_bin(edge, x[i])];
}

__global__ void __launch_bounds__(kCovThreads)
uns_cov_kernel(int n, int D, double* __restrict__ cov, UnsWs w) {
  __shared__ double red[kCovWarps];
  const int r = blockIdx.y;
  int i = 0, rem = blockIdx.x;                                 // blockIdx.x enumerates i <= j row by row
  while (rem >= D - i) {
    rem -= D - i;
    ++i;
  }
  const int j = i + rem;
  const float* xi = w.codes + ((long long)r * D + i) * n;
  const float* xj = w.codes + ((long long)r * D + j) * n;
  const double mi = w.mean[r * D + i], mj = w.mean[r * D + j];
  double s = 0.0;
  for (int k = threadIdx.x; k < n; k += kCovThreads) s += ((double)xi[k] - mi) * ((double)xj[k] - mj);
  s = block_sum<kCovWarps>(s, red) / (n - 1);
  if (threadIdx.x == 0) {
    double* c = cov + (long long)r * D * D;
    c[(long long)i * D + j] = s;
    c[(long long)j * D + i] = s;
  }
}

// One symmetric eigenproblem per CTA: blockIdx.x = 2 representation + matrix (0: R, 1: S).
__global__ void __launch_bounds__(kEigThreads, 1)
uns_eig_kernel(int D, const double* __restrict__ cov, double* __restrict__ eig, int* __restrict__ sweeps_out) {
  extern __shared__ double A[];                                // [D][D + 1]
  __shared__ double red[kEigWarps];
  __shared__ double rc[kUnsMaxD / 2], rs[kUnsMaxD / 2], dp[kUnsMaxD / 2], dq[kUnsMaxD / 2];
  __shared__ int rp[kUnsMaxD / 2], rq[kUnsMaxD / 2], ract[kUnsMaxD / 2];
  const int t = threadIdx.x, L = D + 1, r = blockIdx.x >> 1, which = blockIdx.x & 1;
  const double* C = cov + (long long)r * D * D;
  for (int e = t; e < D * D; e += kEigThreads) {
    const int a = min(e / D, e % D), b = max(e / D, e % D);
    const double ca = C[a * D + a], cb = C[b * D + b], cab = C[a * D + b];
    double v;
    if (which == 0)                                            // R; a constant latent a unit row and column
      v = a == b ? 1.0 : (ca == 0.0 || cb == 0.0 ? 0.0 : cab / (sqrt(ca) * sqrt(cb)));
    else
      v = sqrt(ca) * cab * sqrt(cb);
    A[(e / D) * L + e % D] = v;
  }
  __syncthreads();
  const int m = D + (D & 1), P = m / 2;                        // an odd D plays a dummy index D, never rotated
  int sweeps = 0;
  for (;; ++sweeps) {
    double off = 0.0, all = 0.0;
    for (int e = t; e < D * D; e += kEigThreads) {
      const double v = A[(e / D) * L + e % D];
      all += v * v;
      if (e / D != e % D) off += v * v;
    }
    off = block_sum<kEigWarps>(off, red);
    all = block_sum<kEigWarps>(all, red);
    if (off <= kUnsOffTol2 * all) break;
    if (sweeps == kUnsMaxSweeps) {
      sweeps = -1;
      break;
    }
    for (int round = 0; round < m - 1; ++round) {
      if (t < P) {                                             // the circle method: m - 1 fixed, the others rotate
        int p = t == 0 ? round : (round + t) % (m - 1), q = t == 0 ? m - 1 : (round - t + m - 1) % (m - 1);
        if (p > q) {
          const int x = p;
          p = q;
          q = x;
        }
        rp[t] = p;
        rq[t] = q;
        int act = 0;
        if (q < D) {
          const double apq = A[p * L + q];
          if (apq != 0.0) {
            // the symmetric Schur rotation that zeroes (p, q) (Golub & Van Loan, 8.5.2)
            const double app = A[p * L + p], aqq = A[q * L + q];
            const double theta = (aqq - app) / (2.0 * apq);
            const double tn = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(1.0 + theta * theta));
            const double c = 1.0 / sqrt(tn * tn + 1.0);
            rc[t] = c;
            rs[t] = tn * c;
            dp[t] = app - tn * apq;
            dq[t] = aqq + tn * apq;
            act = 1;
          }
        }
        ract[t] = act;
      }
      __syncthreads();
      for (int e = t; e < P * D; e += kEigThreads) {           // rows p, q <- J^T A
        const int k = e / D, j = e % D;
        if (!ract[k] || rs[k] == 0.0) continue;
        const double c = rc[k], s = rs[k];
        double* ap = A + rp[k] * L + j;
        double* aq = A + rq[k] * L + j;
        const double x = *ap, y = *aq;
        *ap = c * x - s * y;
        *aq = s * x + c * y;
      }
      __syncthreads();
      for (int e = t; e < P * D; e += kEigThreads) {           // columns p, q <- (J^T A) J
        const int k = e / D, i = e % D;
        if (!ract[k] || rs[k] == 0.0) continue;
        const double c = rc[k], s = rs[k];
        double* ap = A + i * L + rp[k];
        double* aq = A + i * L + rq[k];
        const double x = *ap, y = *aq;
        *ap = c * x - s * y;
        *aq = s * x + c * y;
      }
      __syncthreads();
      if (t < P && ract[t]) {                                  // the rotated 2 x 2 block exactly
        const int p = rp[t], q = rq[t];
        A[p * L + q] = 0.0;
        A[q * L + p] = 0.0;
        A[p * L + p] = dp[t];
        A[q * L + q] = dq[t];
      }
      __syncthreads();
    }
  }
  if (t < D) {                                                 // ascending, ties in index order
    const double v = A[t * L + t];
    int rank = 0;
    for (int j = 0; j < D; ++j) {
      const double u = A[j * L + j];
      rank += (u < v || (u == v && j < t)) ? 1 : 0;
    }
    eig[(long long)blockIdx.x * D + rank] = v;
  }
  if (t == 0) sweeps_out[blockIdx.x] = sweeps;
}

bool uns_shape_ok(int n, int D) { return D >= 2 && D <= kUnsMaxD && n >= 2 && n <= kUnsMaxN; }

}  // namespace
}  // namespace dv

using namespace dv;

extern "C" {

size_t dv_unsupervised_workspace_bytes(int n, int D) {
  if (!uns_shape_ok(n, D)) return 0;
  return uns_layout(n, D, nullptr, nullptr);
}

int dv_unsupervised_fit(const float* mu, const float* logvar, int ld, int row_stride, int N, int D,
                        const long long* rows, int n, const float* eps, double* cov, double* eig, int* sweeps,
                        double* mi, float* edges, float* sampled, void* workspace, size_t workspace_bytes,
                        void* stream) {
  if (N < 1 || !uns_shape_ok(n, D) || ld < 1 || row_stride < 1) return DV_ERR_BAD_SHAPE;
  if (!mu || !logvar || !rows || !eps || !cov || !eig || !sweeps || !mi) return DV_ERR_BAD_ARG;
  if (misaligned(mu, 4) || misaligned(logvar, 4) || misaligned(rows, 8) || misaligned(eps, 4) || misaligned(cov, 8) ||
      misaligned(eig, 8) || misaligned(sweeps, 4) || misaligned(mi, 8) || misaligned(edges, 4) ||
      misaligned(sampled, 4) || misaligned(workspace, 8))
    return DV_ERR_BAD_ARG;
  if (!workspace || workspace_bytes < uns_layout(n, D, nullptr, nullptr)) return DV_ERR_WORKSPACE;
  UnsWs w;
  uns_layout(n, D, static_cast<char*>(workspace), &w);
  static bool attr = false;
  int rc = set_max_dynamic_smem(uns_eig_kernel, kUnsMaxD * (kUnsMaxD + 1) * 8, &attr);
  if (rc != DV_OK) return rc;
  cudaStream_t s = as_stream(stream);
  const long long cells = (long long)n * D;
  uns_gather_kernel<<<(unsigned)((cells + kGatherThreads - 1) / kGatherThreads), kGatherThreads, 0, s>>>(
      mu, logvar, ld, row_stride, rows, n, D, eps, sampled, w);
  if ((rc = check_launch()) != DV_OK) return rc;
  uns_column_kernel<<<2 * D, kColThreads, 0, s>>>(n, w);
  if ((rc = check_launch()) != DV_OK) return rc;
  uns_cov_kernel<<<dim3(D * (D + 1) / 2, 2), kCovThreads, 0, s>>>(n, D, cov, w);
  if ((rc = check_launch()) != DV_OK) return rc;
  uns_eig_kernel<<<4, kEigThreads, D * (D + 1) * 8, s>>>(D, cov, eig, sweeps);
  if ((rc = check_launch()) != DV_OK) return rc;
  for (int r = 0; r < 2; ++r) {
    rc = dv_discrete_mutual_info(w.codes + (long long)r * cells, n, 1, n, D, w.rows, n, w.cls + (long long)r * cells,
                                 w.ncls + r * D, D, kHistBins, mi + (long long)r * D * D,
                                 edges ? edges + (long long)r * D * (kHistBins + 1) : nullptr, stream);
    if (rc != DV_OK) return rc;
  }
  return DV_OK;
}

}  // extern "C"

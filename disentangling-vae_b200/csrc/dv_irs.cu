// IRS, the interventional robustness score (Suter et al. 2019; disentanglement_lib's irs.py): how far each latent moves
// while one factor's bin is held fixed, against how far it moves over all drawn rows.  The reference has no such score;
// the entry point and its rules are declared in include/disvae_b200.h.
//
// Plan (3 launches, no host synchronisation):
//   columns  one CTA per latent: gathers the latent's drawn values (mu read in place through ld and row_stride), takes
//            their fp64 mean and largest deviation from it, and sorts the column once (bitonic sort in shared memory on
//            (value, row), dv_common.cuh's, as DCI's prep does).
//   bins     one CTA per scored factor: the factor's min and max over the drawn rows, numpy's 20 fp64 histogram edges,
//            every row's bin (one byte) and every bin's row count (integer shared-memory atomics).
//   groups   one CTA per (latent, factor): stably partitions the latent's sorted values by the factor's bins in shared
//            memory, so every group arrives sorted; one warp per bin takes the group's fp64 mean, then walks inward
//            from both ends of the group for the two order statistics of |x - mean| (|x - c| is convex in x, so the
//            largest remaining one is always at an end); thread 0 adds the bins in order into the IRS matrix.
// Every sum has a fixed order and there are no floating-point atomics, so results are bit-identical run to run.
#include <math.h>
#include <math_constants.h>

#include "dv_common.cuh"

namespace dv {
namespace {

constexpr int kIrsMaxD = 1024;
constexpr int kIrsMaxRows = 32768;         // row positions are sorted as uint16
constexpr int kIrsThreads = 1024;
constexpr int kIrsWarps = kIrsThreads / kWarp;
constexpr int kIrsBins = kHistBins;        // disentanglement_lib's make_discretizer: 20 bins
constexpr unsigned kIrsNoBin = 0xffu;

struct IrsWs {
  float* sval;              // [D][n] drawn values, sorted per latent
  unsigned short* spos;     // [D][n] their row positions
  uint8_t* bin;             // [K][n] the bin of every drawn row, per factor
};

// Offsets of the workspace segments from `base` (NULL for the size only) -> total bytes.
size_t irs_layout(int D, int n, int K, char* base, IrsWs* w) {
  const size_t sizes[3] = {(size_t)D * n * 4, (size_t)D * n * 2, (size_t)K * n};
  size_t off[3];
  const size_t total = carve_workspace(sizes, off);
  if (w) {
    w->sval = reinterpret_cast<float*>(base + off[0]);
    w->spos = reinterpret_cast<unsigned short*>(base + off[1]);
    w->bin = reinterpret_cast<uint8_t*>(base + off[2]);
  }
  return total;
}

__global__ void __launch_bounds__(kIrsThreads, 1)
irs_column_kernel(const float* __restrict__ mu, int ld, int rs, const long long* __restrict__ rows, int n, int P,
                  IrsWs w, double* __restrict__ max_deviation, int* __restrict__ active) {
  extern __shared__ __align__(16) uint8_t smem[];
  unsigned* key = reinterpret_cast<unsigned*>(smem);
  unsigned short* idx = reinterpret_cast<unsigned short*>(key + P);
  __shared__ double red[kIrsWarps];
  const int t = threadIdx.x, d = blockIdx.x;
  const long long col = (long long)d * ld;
  double s = 0.0;
  for (int i = t; i < P; i += kIrsThreads) {
    if (i < n) {
      const float v = mu[rows[i] * (long long)rs + col];
      s += (double)v;
      key[i] = order_key(v);
      idx[i] = (unsigned short)i;
    } else {
      key[i] = 0xffffffffu;                                    // padding sorts after every row
      idx[i] = 0xffffu;
    }
  }
  const double mean = block_sum<kIrsWarps>(s, red) / (double)n;
  double dev = 0.0;
  for (int i = t; i < n; i += kIrsThreads) dev = fmax(dev, fabs((double)key_value(key[i]) - mean));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dev = fmax(dev, __shfl_xor_sync(0xffffffffu, dev, o));
  __syncthreads();                                             // every thread has read block_sum's slots
  if ((t & (kWarp - 1)) == 0) red[t / kWarp] = dev;
  __syncthreads();
  if (t == 0) {
    double m = red[0];
    for (int v = 1; v < kIrsWarps; ++v) m = fmax(m, red[v]);
    max_deviation[d] = m;
    active[d] = m > 0.0 ? 1 : 0;                               // not all equal (the fp64 mean of equal values is them)
  }
  bitonic_sort_pairs<kIrsThreads>(key, idx, P);
  for (int i = t; i < n; i += kIrsThreads) {
    w.sval[(long long)d * n + i] = key_value(key[i]);
    w.spos[(long long)d * n + i] = idx[i];
  }
}

__global__ void __launch_bounds__(kIrsThreads)
irs_bin_kernel(const int* __restrict__ values, int n, IrsWs w, int* __restrict__ group_count,
               double* __restrict__ edges) {
  __shared__ int wlo[kIrsWarps], whi[kIrsWarps], cnt[kIrsBins];
  __shared__ double edge[kIrsBins + 1];
  const int t = threadIdx.x, k = blockIdx.x;
  const int* v = values + (long long)k * n;
  int lo = 0x7fffffff, hi = (int)0x80000000;
  for (int i = t; i < n; i += kIrsThreads) {
    lo = min(lo, v[i]);
    hi = max(hi, v[i]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((t & (kWarp - 1)) == 0) {
    wlo[t / kWarp] = lo;
    whi[t / kWarp] = hi;
  }
  if (t < kIrsBins) cnt[t] = 0;
  __syncthreads();
  if (t == 0) {                                                // np.histogram's edges of an int64 array, in fp64
    for (int u = 1; u < kIrsWarps; ++u) {
      lo = min(lo, wlo[u]);
      hi = max(hi, whi[u]);
    }
    double a = (double)lo, b = (double)hi;
    if (lo == hi) {
      a = __dsub_rn(a, 0.5);
      b = __dadd_rn(b, 0.5);
    }
    const double step = __ddiv_rn(__dsub_rn(b, a), (double)kIrsBins);
    for (int j = 0; j < kIrsBins; ++j) edge[j] = __dadd_rn(__dmul_rn((double)j, step), a);
    edge[kIrsBins] = b;
  }
  __syncthreads();
  for (int i = t; i < n; i += kIrsThreads) {
    const double x = (double)v[i];
    int b = 0;
#pragma unroll
    for (int j = 0; j < kIrsBins; ++j) b += edge[j] <= x ? 1 : 0;
    b = max(b, 1) - 1;                                         // edge_0 is the minimum: every row has one
    w.bin[(long long)k * n + i] = (uint8_t)b;
    atomicAdd(&cnt[b], 1);
  }
  __syncthreads();
  if (t < kIrsBins) group_count[k * kIrsBins + t] = cnt[t];
  if (t <= kIrsBins) edges[k * (kIrsBins + 1) + t] = edge[t];
}

struct IrsGroupArgs {
  int n, D, K;
  double q;                   // (diff_quantile * 100) / 100, numpy's quantile
  const double* max_deviation;
  const int* active;
  const int* group_count;
  double* irs_matrix;
  double* group_deviation;
};

__global__ void __launch_bounds__(kIrsThreads, 1)
irs_group_kernel(IrsGroupArgs a, IrsWs w) {
  extern __shared__ __align__(16) uint8_t smem[];
  float* part = reinterpret_cast<float*>(smem);               // [n]: the latent's sorted values, grouped by bin
  __shared__ int start[kIrsBins], count[kIrsBins], next[kIrsBins];
  __shared__ int wcnt[kIrsWarps][kIrsBins];
  __shared__ double dev[kIrsBins];
  const int t = threadIdx.x, lane = t & (kWarp - 1), warp = t / kWarp;
  const int d = blockIdx.x / a.K, k = blockIdx.x % a.K;
  const int n = a.n;
  if (t == 0) {
    int s = 0;
    for (int b = 0; b < kIrsBins; ++b) {
      count[b] = a.group_count[k * kIrsBins + b];
      start[b] = next[b] = s;
      s += count[b];
    }
  }
  // ---- stable partition: chunk by chunk, each row's place among the earlier rows of its bin (lanes of the same bin
  // by __match_any_sync, then the warps in order, then the earlier chunks)
  const float* sv = w.sval + (long long)d * n;
  const unsigned short* sp = w.spos + (long long)d * n;
  const uint8_t* bins = w.bin + (long long)k * n;
  const unsigned lt = (1u << lane) - 1u;
  for (int base = 0; base < n; base += kIrsThreads) {
    for (int i = t; i < kIrsWarps * kIrsBins; i += kIrsThreads) (&wcnt[0][0])[i] = 0;
    __syncthreads();
    const int i = base + t;
    unsigned b = kIrsNoBin;
    float v = 0.f;
    if (i < n) {
      v = sv[i];
      b = bins[sp[i]];
    }
    const unsigned same = __match_any_sync(0xffffffffu, b);
    if (b != kIrsNoBin && (same & lt) == 0u) wcnt[warp][b] = __popc(same);
    __syncthreads();
    if (t < kIrsBins) {
      int s = next[t];
      for (int u = 0; u < kIrsWarps; ++u) {
        const int c = wcnt[u][t];
        wcnt[u][t] = s;
        s += c;
      }
      next[t] = s;
    }
    __syncthreads();
    if (b != kIrsNoBin) part[wcnt[warp][b] + __popc(same & lt)] = v;
    __syncthreads();
  }
  // ---- one warp per bin: the fp64 group mean, then the quantile of |x - mean| by numpy's linear rule
  if (warp < kIrsBins) {
    const int m = count[warp];
    const float* g = part + start[warp];
    double r = CUDART_NAN;
    if (m > 0) {
      double s = 0.0;
      for (int j = lane; j < m; j += kWarp) s += (double)g[j];
      const double c = warp_sum(s) / (double)m;
      if (lane == 0) {
        const double h = __dmul_rn((double)(m - 1), a.q);
        const double fl = floor(h);
        const int lo = (int)fl, hi = min(lo + 1, m - 1);
        const double frac = __dsub_rn(h, fl);
        const int rank_hi = m - 1 - hi, rank_lo = m - 1 - lo; // places in descending order of |x - c|
        double x_lo = 0.0, x_hi = 0.0;
        int l = 0, u = m - 1;
        for (int step = 0; step <= rank_lo; ++step) {
          const double dl = fabs(__dsub_rn((double)g[l], c)), du = fabs(__dsub_rn((double)g[u], c));
          double x;
          if (dl >= du) {
            x = dl;
            ++l;
          } else {
            x = du;
            --u;
          }
          if (step == rank_hi) x_hi = x;
          if (step == rank_lo) x_lo = x;
        }
        const double diff = __dsub_rn(x_hi, x_lo);
        r = frac < 0.5 ? __dadd_rn(x_lo, __dmul_rn(diff, frac)) : __dsub_rn(x_hi, __dmul_rn(diff, __dsub_rn(1.0, frac)));
      }
    }
    if (lane == 0) {
      dev[warp] = r;
      a.group_deviation[((long long)k * kIrsBins + warp) * a.D + d] = r;
    }
  }
  __syncthreads();
  if (t == 0) {
    double s = 0.0;
    int groups = 0;
    for (int b = 0; b < kIrsBins; ++b) {
      if (count[b] == 0) continue;
      s += dev[b];
      ++groups;
    }
    const double cum = s / (double)groups;
    a.irs_matrix[(long long)d * a.K + k] = a.active[d] ? 1.0 - cum / a.max_deviation[d] : CUDART_NAN;
  }
}

bool irs_shape_ok(int D, int n, int K) {
  return D >= 1 && D <= kIrsMaxD && n >= 1 && n <= kIrsMaxRows && K >= 1 && (long long)K * n <= 0x7fffffffLL &&
         (long long)K * D <= 0x7fffffffLL && (long long)K * kIrsBins * D <= 0x7fffffffLL;
}

}  // namespace
}  // namespace dv

using namespace dv;

extern "C" {

size_t dv_irs_workspace_bytes(int D, int n, int K) {
  if (!irs_shape_ok(D, n, K)) return 0;
  return irs_layout(D, n, K, nullptr, nullptr);
}

int dv_irs_fit(const float* mu, int ld, int row_stride, int N, int D, const long long* rows, int n, const int* values,
               int K, double diff_quantile, double* max_deviation, int* active, double* irs_matrix,
               double* group_deviation, int* group_count, double* edges, void* workspace, size_t workspace_bytes,
               void* stream) {
  if (N < 1 || !irs_shape_ok(D, n, K) || ld < 1 || row_stride < 1 || !(diff_quantile >= 0.0 && diff_quantile <= 1.0))
    return DV_ERR_BAD_SHAPE;
  if (!mu || !rows || !values || !max_deviation || !active || !irs_matrix || !group_deviation || !group_count ||
      !edges)
    return DV_ERR_BAD_ARG;
  if (misaligned(mu, 4) || misaligned(rows, 8) || misaligned(values, 4) || misaligned(max_deviation, 8) ||
      misaligned(active, 4) || misaligned(irs_matrix, 8) || misaligned(group_deviation, 8) ||
      misaligned(group_count, 4) || misaligned(edges, 8) || misaligned(workspace, 8))
    return DV_ERR_BAD_ARG;
  if (!workspace || workspace_bytes < irs_layout(D, n, K, nullptr, nullptr)) return DV_ERR_WORKSPACE;
  IrsWs w;
  irs_layout(D, n, K, static_cast<char*>(workspace), &w);
  const int P = pow2_at_least(n);
  static bool col_attr = false, group_attr = false;
  int rc = set_max_dynamic_smem(irs_column_kernel, kIrsMaxRows * 6, &col_attr);
  if (rc != DV_OK) return rc;
  if ((rc = set_max_dynamic_smem(irs_group_kernel, kIrsMaxRows * 4, &group_attr)) != DV_OK) return rc;
  cudaStream_t s = as_stream(stream);
  irs_column_kernel<<<D, kIrsThreads, (size_t)P * 6, s>>>(mu, ld, row_stride, rows, n, P, w, max_deviation, active);
  if ((rc = check_launch()) != DV_OK) return rc;
  irs_bin_kernel<<<K, kIrsThreads, 0, s>>>(values, n, w, group_count, edges);
  if ((rc = check_launch()) != DV_OK) return rc;
  const IrsGroupArgs a{n, D, K, (diff_quantile * 100.0) / 100.0, max_deviation, active, group_count, irs_matrix,
                       group_deviation};
  irs_group_kernel<<<D * K, kIrsThreads, (size_t)n * 4, s>>>(a, w);
  return check_launch();
}

}  // extern "C"

// DCI disentanglement score (Eastwood & Williams 2018; disentanglement_lib's dci.py): for every scored factor the
// gradient-boosted trees of sklearn's GradientBoostingClassifier() at its defaults, grown on the GPU, with their
// feature importances and the predictions on the training and test rows.  The reference has no such score; the entry
// points and the rules of the fit are declared in include/disvae_b200.h.
//
// Plan (4 + 2 * stages launches, no host synchronisation):
//   prep      one CTA per latent: gathers the latent's training and test values (mu read in place through ld and
//             row_stride) and sorts the training column once (bitonic sort in shared memory on (value, row), so equal
//             values keep their row order).
//   init      one CTA per (factor, column): the prior raw score of the column on every row; clears the importance sums.
//   per stage
//     residual  one thread per (factor, training row): the log-loss residuals of every column of the factor from the
//               stage's starting scores, in fp64 and rounded to int64 fixed point at 2^-40 for the split proxy.
//     tree      one CTA per (factor, column): grows the column's depth-3 tree level by level.  At each level one pass
//               over the rows adds up every node's count, sum of residuals, sum of p (1 - p) and sum of fixed-point
//               residuals, and a second its sum of squared deviations from the mean; then each warp scans the presorted columns of its latents (latents warp,
//               warp + 16, ...), 32 rows at a time, keeping every open node's running count and exact fixed-point sum
//               across the chunks, and evaluates the friedman_mse proxy at every gap between consecutive values of a
//               node.  The node's best split (largest proxy, the lowest latent and then the lowest threshold on an
//               exact tie) routes its rows.  The CTA then sets the leaf values, adds its importance contributions to
//               the (factor, column) sums and updates the training and test scores (product and sum rounded apart).
//   importance one CTA per factor: the mean over the factor's trees of more than one node, normalised to sum 1.
//   predict    one thread per (factor, row): argmax over the columns, or the sign for two classes.
// Every sum has a fixed order and there are no floating-point atomics, so results are bit-identical run to run.
#include <math.h>
#include <math_constants.h>

#include "dv_common.cuh"

namespace dv {
namespace {

constexpr int kDciMaxD = 1024;
constexpr int kDciMaxClasses = 256;
constexpr int kDciMaxTrain = 32768;        // row indices are sorted as uint16, the node of a row is a uint8
constexpr int kDciSortThreads = 1024;
constexpr int kDciTreeThreads = 512;
constexpr int kDciTreeWarps = kDciTreeThreads / kWarp;
constexpr int kDciThreads = 256;
constexpr int kDciDepth = 3;
constexpr int kDciNodes = 15;              // heap order: the children of node h are 2h + 1 and 2h + 2
constexpr int kDciLevelMax = 8;            // nodes at the deepest level
constexpr int kDciSplitMax = 4;            // nodes that can split at one level
constexpr int kDciLeaf = -1, kDciAbsent = -2;
constexpr double kDciFix = 1099511627776.0;              // 2^40
constexpr double kDciUnfix = 1.0 / 1099511627776.0;
constexpr double kDciFeatureThreshold = 1e-7;            // sklearn's FEATURE_THRESHOLD
constexpr double kDciLearningRate = 0.1;
constexpr double kDciEps32 = 1.1920928955078125e-07;     // the clip of the prior probabilities
constexpr double kDciDblEps = 2.220446049250313e-16;     // DBL_EPSILON

struct DciWs {
  float* xt;        // [D][n] training values, training order
  float* xe;        // [D][m] test values
  float* sval;      // [D][n] training values, sorted per latent
  int* sidx;        // [D][n] their training rows
  double* raw;      // [K][S][n + m] raw scores
  double* r;        // [K][S][n] residuals
  long long* q;     // [K][S][n] residuals in fixed point
  double* acc;      // [K][S][D] importance sums
  double* cnt;      // [K][S] trees of more than one node
};

// Offsets of the workspace segments from `base` (NULL for the size only) -> total bytes.
size_t dci_layout(int D, int n, int m, int K, int S, char* base, DciWs* w) {
  const size_t KS = (size_t)K * S;
  const size_t sizes[9] = {(size_t)D * n * 4, (size_t)D * m * 4, (size_t)D * n * 4, (size_t)D * n * 4,
                           KS * ((size_t)n + m) * 8, KS * n * 8, KS * n * 8, KS * D * 8, KS * 8};
  size_t off[9];
  const size_t total = carve_workspace(sizes, off);
  if (w) {
    w->xt = reinterpret_cast<float*>(base + off[0]);
    w->xe = reinterpret_cast<float*>(base + off[1]);
    w->sval = reinterpret_cast<float*>(base + off[2]);
    w->sidx = reinterpret_cast<int*>(base + off[3]);
    w->raw = reinterpret_cast<double*>(base + off[4]);
    w->r = reinterpret_cast<double*>(base + off[5]);
    w->q = reinterpret_cast<long long*>(base + off[6]);
    w->acc = reinterpret_cast<double*>(base + off[7]);
    w->cnt = reinterpret_cast<double*>(base + off[8]);
  }
  return total;
}

__device__ __forceinline__ int dci_columns(int nc) { return nc > 2 ? nc : (nc == 2 ? 1 : 0); }

__global__ void __launch_bounds__(kDciSortThreads, 1)
dci_prep_kernel(const float* __restrict__ mu, int ld, int rs, const long long* __restrict__ train_rows, int n,
                const long long* __restrict__ test_rows, int m, int P, DciWs w) {
  extern __shared__ __align__(16) uint8_t smem[];
  unsigned* key = reinterpret_cast<unsigned*>(smem);
  unsigned short* idx = reinterpret_cast<unsigned short*>(key + P);
  const int t = threadIdx.x, d = blockIdx.x;
  const long long col = (long long)d * ld;
  for (int i = t; i < P; i += kDciSortThreads) {
    if (i < n) {
      const float v = mu[train_rows[i] * (long long)rs + col];
      w.xt[(long long)d * n + i] = v;
      key[i] = order_key(v);
      idx[i] = (unsigned short)i;
    } else {
      key[i] = 0xffffffffu;                                    // padding sorts after every row
      idx[i] = 0xffffu;
    }
  }
  for (int j = t; j < m; j += kDciSortThreads) w.xe[(long long)d * m + j] = mu[test_rows[j] * (long long)rs + col];
  __syncthreads();
  bitonic_sort_pairs<kDciSortThreads>(key, idx, P);
  for (int i = t; i < n; i += kDciSortThreads) {
    w.sval[(long long)d * n + i] = key_value(key[i]);
    w.sidx[(long long)d * n + i] = idx[i];
  }
}

__device__ __forceinline__ double dci_prior(const int* counts, int k, int S, int c, int n) {
  return fmin(fmax((double)counts[(long long)k * S + c] / (double)n, kDciEps32), 1.0 - kDciEps32);
}

__global__ void __launch_bounds__(kDciThreads)
dci_init_kernel(const int* __restrict__ n_classes, const int* __restrict__ counts, int S, int D, int n, int m,
                DciWs w) {
  const int t = threadIdx.x, k = blockIdx.x / S, c = blockIdx.x % S;
  const long long ks = (long long)k * S + c;
  for (int d = t; d < D; d += kDciThreads) w.acc[ks * D + d] = 0.0;
  if (t == 0) w.cnt[ks] = 0.0;
  const int nc = class_count(n_classes, k, S);
  if (c >= dci_columns(nc)) return;
  double v;
  if (nc == 2) {
    const double p = dci_prior(counts, k, S, 1, n);
    v = log(p / (1.0 - p));
  } else {                                                     // log(p_c / gmean(p))
    double s = 0.0;
    for (int j = 0; j < nc; ++j) s += log(dci_prior(counts, k, S, j, n));
    v = log(dci_prior(counts, k, S, c, n) / exp(s / nc));
  }
  double* raw = w.raw + ks * ((long long)n + m);
  for (int i = t; i < n + m; i += kDciThreads) raw[i] = v;
}

__global__ void __launch_bounds__(kDciThreads)
dci_residual_kernel(const int* __restrict__ train_cls, const int* __restrict__ n_classes, int K, int S, int n, int m,
                    DciWs w) {
  const long long g = (long long)blockIdx.x * kDciThreads + threadIdx.x;
  if (g >= (long long)K * n) return;
  const int k = (int)(g / n), i = (int)(g % n);
  const int nc = class_count(n_classes, k, S);
  if (nc < 2) return;
  const int y = train_cls[g];
  const long long N2 = (long long)n + m;
  const double* raw = w.raw + (long long)k * S * N2 + i;
  double* r = w.r + (long long)k * S * n + i;
  long long* q = w.q + (long long)k * S * n + i;
  if (nc == 2) {                                               // r = t - sigmoid(z), in sklearn's stable form
    const double z = raw[0], tt = y == 1 ? 1.0 : 0.0;
    const double e = exp(-fabs(z));
    const double grad = z < 0.0 ? ((1.0 - tt) * e - tt) / (1.0 + e) : ((1.0 - tt) - tt * e) / (1.0 + e);
    r[0] = -grad;
    q[0] = __double2ll_rn(-grad * kDciFix);
    return;
  }
  double mx = raw[0];
  for (int c = 1; c < nc; ++c) mx = fmax(mx, raw[c * N2]);
  double s = 0.0;
  for (int c = 0; c < nc; ++c) s += exp(raw[c * N2] - mx);
  for (int c = 0; c < nc; ++c) {
    const double v = (c == y ? 1.0 : 0.0) - exp(raw[c * N2] - mx) / s;
    r[(long long)c * n] = v;
    q[(long long)c * n] = __double2ll_rn(v * kDciFix);
  }
}

struct DciTreeArgs {
  const int* train_cls;
  const int* n_classes;
  int K, S, D, n, m, stage, stages;
  int* tree_feature;
  double* tree_threshold;
  double* tree_value;
};

__global__ void __launch_bounds__(kDciTreeThreads, 1)
dci_tree_kernel(DciTreeArgs a, DciWs w) {
  extern __shared__ __align__(16) uint8_t node[];             // [n]: heap index of every training row's node
  __shared__ int feat[kDciNodes];
  __shared__ double thr[kDciNodes], val[kDciNodes], imp[kDciNodes], size[kDciNodes];
  __shared__ double wred[kDciTreeWarps][4 * kDciLevelMax];
  __shared__ long long wq[kDciTreeWarps][kDciLevelMax];
  __shared__ double stat[4 * kDciLevelMax];           // per node: count, sum r, sum (r - mean)^2, sum p (1 - p)
  __shared__ double mean[kDciLevelMax];
  __shared__ long long qtot[kDciLevelMax];
  __shared__ int open[kDciSplitMax];
  __shared__ double bproxy[kDciTreeWarps][kDciSplitMax];
  __shared__ int bfeat[kDciTreeWarps][kDciSplitMax];
  __shared__ float ba[kDciTreeWarps][kDciSplitMax], bb[kDciTreeWarps][kDciSplitMax];

  const int t = threadIdx.x, lane = t & (kWarp - 1), warp = t / kWarp;
  const int k = blockIdx.x / a.S, c = blockIdx.x % a.S;
  const int n = a.n, m = a.m, D = a.D;
  const long long ks = (long long)k * a.S + c;
  const long long tree0 = (ks * a.stages + a.stage) * kDciNodes;
  const int nc = class_count(a.n_classes, k, a.S);
  if (t < kDciNodes) {
    feat[t] = kDciAbsent;
    thr[t] = CUDART_NAN;
    val[t] = CUDART_NAN;
  }
  if (c >= dci_columns(nc)) {                                  // no such column: an absent tree
    if (t < kDciNodes) {
      if (a.tree_feature) a.tree_feature[tree0 + t] = kDciAbsent;
      if (a.tree_threshold) a.tree_threshold[tree0 + t] = CUDART_NAN;
      if (a.tree_value) a.tree_value[tree0 + t] = CUDART_NAN;
    }
    return;
  }
  const double* rr = w.r + ks * n;
  const long long* qq = w.q + ks * n;
  const int* cls = a.train_cls + (long long)k * n;
  const int pos = nc > 2 ? c : 1;                              // the class whose indicator is the target
  for (int i = t; i < n; i += kDciTreeThreads) node[i] = 0;
  __syncthreads();

  for (int depth = 0; depth <= kDciDepth; ++depth) {
    const int first = (1 << depth) - 1, width = 1 << depth;
    // ---- every node's count, sum r, sum p (1 - p) and sum of fixed-point r, then its mean and sum (r - mean)^2
    // (the centred form, so a node of equal residuals has an impurity of about 0): thread, warp, then CTA order;
    // four nodes per pass over the rows
    for (int pass = 0; pass < 2; ++pass) {
      for (int g0 = 0; g0 < width; g0 += kDciSplitMax) {
        double acc[kDciSplitMax][3];
        long long accq[kDciSplitMax];
#pragma unroll
        for (int j = 0; j < kDciSplitMax; ++j) {
          acc[j][0] = acc[j][1] = acc[j][2] = 0.0;
          accq[j] = 0;
        }
        for (int i = t; i < n; i += kDciTreeThreads) {
          const int j = (int)node[i] - first - g0;
          if (j < 0 || j >= kDciSplitMax || j + g0 >= width) continue;
          const double r = rr[i];
          if (pass == 0) {
            const double p = (cls[i] == pos ? 1.0 : 0.0) - r;
            const double h = __dmul_rn(p, 1.0 - p);
            const long long qv = qq[i];
#pragma unroll
            for (int s = 0; s < kDciSplitMax; ++s) {
              if (s == j) {
                acc[s][0] += 1.0;
                acc[s][1] += r;
                acc[s][2] += h;
                accq[s] += qv;
              }
            }
          } else {
            const double e = r - mean[g0 + j];
#pragma unroll
            for (int s = 0; s < kDciSplitMax; ++s)
              if (s == j) acc[s][0] = __dadd_rn(acc[s][0], __dmul_rn(e, e));
          }
        }
#pragma unroll
        for (int s = 0; s < kDciSplitMax; ++s) {
#pragma unroll
          for (int u = 0; u < 3; ++u) acc[s][u] = warp_sum(acc[s][u]);
          accq[s] = warp_sum(accq[s]);
        }
        if (lane == 0) {
#pragma unroll
          for (int s = 0; s < kDciSplitMax; ++s) {
            if (pass == 0) {
              wred[warp][4 * (g0 + s)] = acc[s][0];
              wred[warp][4 * (g0 + s) + 1] = acc[s][1];
              wred[warp][4 * (g0 + s) + 3] = acc[s][2];
              wq[warp][g0 + s] = accq[s];
            } else {
              wred[warp][4 * (g0 + s) + 2] = acc[s][0];
            }
          }
        }
      }
      __syncthreads();
      if (pass == 0) {
        if (t < 4 * kDciLevelMax) {
          if (t % 4 != 2) {
            double s = 0.0;
            for (int v = 0; v < kDciTreeWarps; ++v) s += wred[v][t];
            stat[t] = s;
          }
        } else if (t < 5 * kDciLevelMax) {
          long long s = 0;
          for (int v = 0; v < kDciTreeWarps; ++v) s += wq[v][t - 4 * kDciLevelMax];
          qtot[t - 4 * kDciLevelMax] = s;
        }
        __syncthreads();
        if (t < kDciLevelMax) mean[t] = stat[4 * t] > 0.0 ? stat[4 * t + 1] / stat[4 * t] : 0.0;
      } else if (t < kDciLevelMax) {
        double s = 0.0;
        for (int v = 0; v < kDciTreeWarps; ++v) s += wred[v][4 * t + 2];
        stat[4 * t + 2] = s;
      }
      __syncthreads();
    }
    // ---- which nodes of this level exist, which are leaves, which may split
    if (t == 0) {
      for (int j = 0; j < kDciSplitMax; ++j) open[j] = 0;
      for (int j = 0; j < width; ++j) {
        const int h = first + j;
        if (h > 0 && feat[(h - 1) / 2] < 0) continue;          // the parent is a leaf: no such node
        const double cn = stat[4 * j], s = stat[4 * j + 1];
        size[h] = cn;
        imp[h] = stat[4 * j + 2] / cn;
        if (depth < kDciDepth && cn >= 2.0 && imp[h] > kDciDblEps) {
          open[j] = 1;
        } else {
          feat[h] = kDciLeaf;
          const double num = nc > 2 ? s * ((double)(nc - 1) / (double)nc) : s;
          const double den = stat[4 * j + 3];
          val[h] = fabs(den) < 1e-150 ? 0.0 : num / den;
        }
      }
    }
    __syncthreads();
    if (depth == kDciDepth) break;
    int any = 0;
#pragma unroll
    for (int j = 0; j < kDciSplitMax; ++j) any |= open[j];
    if (!any) break;

    // ---- split search: each warp scans the sorted columns of its latents, 32 rows at a time
    double wbest[kDciSplitMax];
    int wfeat[kDciSplitMax];
    float wa[kDciSplitMax], wb[kDciSplitMax];
#pragma unroll
    for (int j = 0; j < kDciSplitMax; ++j) {
      wbest[j] = -CUDART_INF;
      wfeat[j] = -1;
      wa[j] = wb[j] = 0.f;
    }
    const unsigned lt = (1u << lane) - 1u;
    for (int d = warp; d < D; d += kDciTreeWarps) {
      const float* sv = w.sval + (long long)d * n;
      const int* si = w.sidx + (long long)d * n;
      int cnt[kDciSplitMax];
      long long sum[kDciSplitMax];
      float last[kDciSplitMax];
      double lbest[kDciSplitMax];
      int lpos[kDciSplitMax];
      float la[kDciSplitMax], lb[kDciSplitMax];
#pragma unroll
      for (int j = 0; j < kDciSplitMax; ++j) {
        cnt[j] = 0;
        sum[j] = 0;
        last[j] = 0.f;
        lbest[j] = -CUDART_INF;
        lpos[j] = 0x7fffffff;
        la[j] = lb[j] = 0.f;
      }
      for (int base = 0; base < n; base += kWarp) {
        const int i = base + lane;
        int j_in = -1;
        float v = 0.f;
        long long qv = 0;
        if (i < n) {
          const int row = si[i];
          const int j = (int)node[row] - first;
          if (j >= 0 && j < kDciSplitMax && j < width && open[j]) {
            j_in = j;
            v = sv[i];
            qv = qq[row];
          }
        }
#pragma unroll
        for (int j = 0; j < kDciSplitMax; ++j) {
          if (j >= width || !open[j]) continue;                 // warp-uniform
          const bool in = j_in == j;
          const unsigned mask = __ballot_sync(0xffffffffu, in);
          if (mask == 0u) continue;
          long long x = in ? qv : 0;
#pragma unroll
          for (int o = 1; o < kWarp; o <<= 1) {
            const long long y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
          }
          const unsigned before = mask & lt;
          const int prev = before ? 31 - __clz(before) : lane;
          const float vprev = __shfl_sync(0xffffffffu, v, prev);
          if (in && (before || cnt[j] > 0)) {
            const float xa = before ? vprev : last[j];
            if ((double)v > __dadd_rn((double)xa, kDciFeatureThreshold)) {
              const long long ql = sum[j] + x - qv;             // the node's rows before this one
              const int nl = cnt[j] + __popc(before);
              const double nld = (double)nl, nrd = size[first + j] - nld;
              const double sl = __dmul_rn(__ll2double_rn(ql), kDciUnfix);
              const double sr = __dmul_rn(__ll2double_rn(qtot[j] - ql), kDciUnfix);
              const double diff = __dsub_rn(__dmul_rn(nrd, sl), __dmul_rn(nld, sr));
              const double proxy = __ddiv_rn(__dmul_rn(diff, diff), __dmul_rn(nld, nrd));
              if (proxy > lbest[j]) {
                lbest[j] = proxy;
                lpos[j] = i;
                la[j] = xa;
                lb[j] = v;
              }
            }
          }
          cnt[j] += __popc(mask);
          sum[j] += __shfl_sync(0xffffffffu, x, 31);
          last[j] = __shfl_sync(0xffffffffu, v, 31 - __clz(mask));
        }
      }
      // the latent's best per node over the warp (the lowest position on a tie), then against the warp's earlier
      // latents (strictly better only, so the lowest latent keeps a tie)
#pragma unroll
      for (int j = 0; j < kDciSplitMax; ++j) {
        double p = lbest[j];
        int ps = lpos[j];
        float xa = la[j], xb = lb[j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const double p2 = __shfl_xor_sync(0xffffffffu, p, o);
          const int ps2 = __shfl_xor_sync(0xffffffffu, ps, o);
          const float a2 = __shfl_xor_sync(0xffffffffu, xa, o), b2 = __shfl_xor_sync(0xffffffffu, xb, o);
          if (p2 > p || (p2 == p && ps2 < ps)) {
            p = p2;
            ps = ps2;
            xa = a2;
            xb = b2;
          }
        }
        if (p > wbest[j]) {
          wbest[j] = p;
          wfeat[j] = d;
          wa[j] = xa;
          wb[j] = xb;
        }
      }
    }
    if (lane == 0) {
#pragma unroll
      for (int j = 0; j < kDciSplitMax; ++j) {
        bproxy[warp][j] = wbest[j];
        bfeat[warp][j] = wfeat[j];
        ba[warp][j] = wa[j];
        bb[warp][j] = wb[j];
      }
    }
    __syncthreads();
    if (t == 0) {
      for (int j = 0; j < width && j < kDciSplitMax; ++j) {
        if (!open[j]) continue;
        const int h = first + j;
        double best = -CUDART_INF;
        int bw = -1;
        for (int v = 0; v < kDciTreeWarps; ++v) {
          if (bfeat[v][j] < 0) continue;                         // a warp's found split has a finite proxy
          if (bw < 0 || bproxy[v][j] > best || (bproxy[v][j] == best && bfeat[v][j] < bfeat[bw][j])) {
            best = bproxy[v][j];
            bw = v;
          }
        }
        if (bw < 0) {                                          // no gap anywhere: a leaf
          feat[h] = kDciLeaf;
          const double s = stat[4 * j + 1];
          const double num = nc > 2 ? s * ((double)(nc - 1) / (double)nc) : s;
          const double den = stat[4 * j + 3];
          val[h] = fabs(den) < 1e-150 ? 0.0 : num / den;
        } else {
          const double xa = (double)ba[bw][j], xb = (double)bb[bw][j];
          const double mid = __dadd_rn(xa * 0.5, xb * 0.5);
          feat[h] = bfeat[bw][j];
          thr[h] = mid == xb ? xa : mid;
        }
      }
    }
    __syncthreads();
    // ---- route the rows of the split nodes
    for (int i = t; i < n; i += kDciTreeThreads) {
      const int h = node[i];
      if (h < first || h >= first + width) continue;
      const int f = feat[h];
      if (f < 0) continue;
      node[i] = (uint8_t)((double)w.xt[(long long)f * n + i] <= thr[h] ? 2 * h + 1 : 2 * h + 2);
    }
    __syncthreads();
  }

  // ---- importance contributions, the tree, and the scores
  if (t == 0) {
    double* acc = w.acc + ks * D;
    for (int h = 0; h < 7; ++h) {
      if (feat[h] < 0) continue;
      const int l = 2 * h + 1, r = 2 * h + 2;
      const double v = __dsub_rn(__dsub_rn(__dmul_rn(size[h], imp[h]), __dmul_rn(size[l], imp[l])),
                                 __dmul_rn(size[r], imp[r]));
      acc[feat[h]] += v / (double)n;
    }
    if (feat[0] >= 0) w.cnt[ks] += 1.0;
  }
  if (t < kDciNodes) {
    if (a.tree_feature) a.tree_feature[tree0 + t] = feat[t];
    if (a.tree_threshold) a.tree_threshold[tree0 + t] = thr[t];
    if (a.tree_value) a.tree_value[tree0 + t] = val[t];
  }
  double* raw = w.raw + ks * ((long long)n + m);
  for (int i = t; i < n; i += kDciTreeThreads)
    raw[i] = __dadd_rn(raw[i], __dmul_rn(kDciLearningRate, val[node[i]]));
  for (int j = t; j < m; j += kDciTreeThreads) {
    int h = 0;
    while (feat[h] >= 0) h = (double)w.xe[(long long)feat[h] * m + j] <= thr[h] ? 2 * h + 1 : 2 * h + 2;
    raw[n + j] = __dadd_rn(raw[n + j], __dmul_rn(kDciLearningRate, val[h]));
  }
}

__global__ void __launch_bounds__(kDciThreads)
dci_importance_kernel(const int* __restrict__ n_classes, int K, int S, int D, DciWs w, double* __restrict__ out) {
  __shared__ double mean[kDciMaxD];
  __shared__ double norm;
  const int t = threadIdx.x, k = blockIdx.x;
  const int cols = dci_columns(class_count(n_classes, k, S));
  double trees = 0.0;
  for (int c = 0; c < cols; ++c) trees += w.cnt[(long long)k * S + c];
  for (int d = t; d < D; d += kDciThreads) {
    double s = 0.0;
    for (int c = 0; c < cols; ++c) s += w.acc[((long long)k * S + c) * D + d];
    mean[d] = trees > 0.0 ? s / trees : 0.0;
  }
  __syncthreads();
  if (t == 0) {
    double s = 0.0;
    for (int d = 0; d < D; ++d) s += mean[d];
    norm = s;
  }
  __syncthreads();
  for (int d = t; d < D; d += kDciThreads) out[(long long)d * K + k] = norm != 0.0 ? fabs(mean[d] / norm) : 0.0;
}

__global__ void __launch_bounds__(kDciThreads)
dci_predict_kernel(const int* __restrict__ n_classes, int K, int S, int n, int m, DciWs w, int* __restrict__ pred) {
  const long long N2 = (long long)n + m;
  const long long g = (long long)blockIdx.x * kDciThreads + threadIdx.x;
  if (g >= (long long)K * N2) return;
  const int k = (int)(g / N2);
  const long long i = g % N2;
  const int nc = class_count(n_classes, k, S);
  const double* raw = w.raw + (long long)k * S * N2 + i;
  int best = 0;
  if (nc == 2) {
    best = raw[0] >= 0.0 ? 1 : 0;
  } else if (nc > 2) {
    double b = raw[0];
    for (int c = 1; c < nc; ++c) {
      const double v = raw[c * N2];
      if (v > b) { b = v; best = c; }
    }
  }
  pred[g] = best;
}

bool dci_shape_ok(int D, int n, int m, int K, int S) {
  return D >= 1 && D <= kDciMaxD && n >= 1 && n <= kDciMaxTrain && m >= 1 && K >= 1 && S >= 1 &&
         S <= kDciMaxClasses && (long long)n + m <= 0x7fffffffLL && (long long)K * ((long long)n + m) <= 0x7fffffffLL &&
         (long long)K * S <= 0x7fffffffLL;
}

unsigned blocks_of(long long threads) { return (unsigned)((threads + kDciThreads - 1) / kDciThreads); }

}  // namespace
}  // namespace dv

using namespace dv;

extern "C" {

size_t dv_dci_workspace_bytes(int D, int num_train, int num_test, int K, int class_stride) {
  if (!dci_shape_ok(D, num_train, num_test, K, class_stride)) return 0;
  return dci_layout(D, num_train, num_test, K, class_stride, nullptr, nullptr);
}

int dv_dci_fit(const float* mu, int ld, int row_stride, int N, int D, const long long* train_rows, int num_train,
               const long long* test_rows, int num_test, const int* train_cls, const int* n_classes,
               const int* counts, int K, int class_stride, int stages, double* importance, int* pred,
               int* tree_feature, double* tree_threshold, double* tree_value, void* workspace,
               size_t workspace_bytes, void* stream) {
  if (N < 1 || !dci_shape_ok(D, num_train, num_test, K, class_stride) || stages < 0 || ld < 1 || row_stride < 1 ||
      (long long)K * class_stride * stages * kDciNodes > 0x7fffffffLL)
    return DV_ERR_BAD_SHAPE;
  if (!mu || !train_rows || !test_rows || !train_cls || !n_classes || !counts || !importance || !pred)
    return DV_ERR_BAD_ARG;
  if (misaligned(mu, 4) || misaligned(train_rows, 8) || misaligned(test_rows, 8) || misaligned(train_cls, 4) ||
      misaligned(n_classes, 4) || misaligned(counts, 4) || misaligned(importance, 8) || misaligned(pred, 4) ||
      misaligned(tree_feature, 4) || misaligned(tree_threshold, 8) || misaligned(tree_value, 8) ||
      misaligned(workspace, 8))
    return DV_ERR_BAD_ARG;
  const int S = class_stride, n = num_train, m = num_test;
  if (!workspace || workspace_bytes < dci_layout(D, n, m, K, S, nullptr, nullptr)) return DV_ERR_WORKSPACE;
  DciWs w;
  dci_layout(D, n, m, K, S, static_cast<char*>(workspace), &w);
  const int P = pow2_at_least(n);
  const size_t sort_smem = (size_t)P * (sizeof(unsigned) + sizeof(unsigned short));
  static bool attr = false;
  int rc = set_max_dynamic_smem(dci_prep_kernel, (int)((size_t)kDciMaxTrain * 6), &attr);
  if (rc != DV_OK) return rc;
  cudaStream_t s = as_stream(stream);
  dci_prep_kernel<<<D, kDciSortThreads, sort_smem, s>>>(mu, ld, row_stride, train_rows, n, test_rows, m, P, w);
  if ((rc = check_launch()) != DV_OK) return rc;
  dci_init_kernel<<<K * S, kDciThreads, 0, s>>>(n_classes, counts, S, D, n, m, w);
  if ((rc = check_launch()) != DV_OK) return rc;
  DciTreeArgs a{train_cls, n_classes, K, S, D, n, m, 0, stages, tree_feature, tree_threshold, tree_value};
  for (int st = 0; st < stages; ++st) {
    dci_residual_kernel<<<blocks_of((long long)K * n), kDciThreads, 0, s>>>(train_cls, n_classes, K, S, n, m, w);
    if ((rc = check_launch()) != DV_OK) return rc;
    a.stage = st;
    dci_tree_kernel<<<K * S, kDciTreeThreads, n, s>>>(a, w);
    if ((rc = check_launch()) != DV_OK) return rc;
  }
  dci_importance_kernel<<<K, kDciThreads, 0, s>>>(n_classes, K, S, D, w, importance);
  if ((rc = check_launch()) != DV_OK) return rc;
  dci_predict_kernel<<<blocks_of((long long)K * (n + m)), kDciThreads, 0, s>>>(n_classes, K, S, n, m, w, pred);
  return check_launch();
}

}  // extern "C"

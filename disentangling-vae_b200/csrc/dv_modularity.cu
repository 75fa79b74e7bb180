// Modularity and explicitness (Ridgeway & Zemel 2018; disentanglement_lib's modularity_explicitness.py): the
// histogram mutual information between every latent and every scored factor, and for every factor the exact fit of
// sklearn's LogisticRegression() on the standardised latents with the ROC AUC of each class column.  The reference has
// no such score; the entry points and their rules are declared in include/disvae_b200.h.
//
// dv_discrete_mutual_info (one launch, one CTA per latent): gathers the latent's training column (mu read in place
// through ld and row_stride), takes its min and max, builds numpy's 20 histogram edges in fp32 without contraction,
// bins every row into shared memory, then for each factor counts the (class, bin) cells in integer shared memory and
// adds sklearn's mutual_info_score terms in a fixed order (bins of a class, then the classes).
//
// dv_explicitness_fit (three launches, no host synchronisation):
//   standardise  one CTA per latent: the training mean and standard deviation (ddof 0) in fp64, each a fixed-order
//                sum, and the standardised training and test features, fp64 [rows][D], into the workspace.
//   fit          one CTA per factor: logistic_fit_cta (dv_logistic.cuh) on the factor's labels with its own slice of
//                the workspace, then the class probabilities of every training and test row.
//   auc          one CTA per (factor, column, set): the column's positives are staged in shared memory in tiles of
//                4096, each tile sorted; every other row of the set finds its place in the tile by binary search, and
//                the CTA adds the pairs with the positive above it and the pairs tied with it in int64.
// Every sum has a fixed order and there are no floating-point atomics, so results are bit-identical run to run.
#include <float.h>

#include "dv_logistic.cuh"

namespace dv {
namespace {

constexpr int kMiThreads = 512;
constexpr int kMiWarps = kMiThreads / kWarp;
constexpr int kMiBins = kHistBins;            // disentanglement_lib's num_bins
constexpr int kMiMaxD = 1024;
constexpr int kModMaxD = kFitMaxD;            // dv_explicitness_fit's latents
constexpr int kModMaxClasses = 256;
constexpr int kModMaxTrain = 32768;           // the training bins sit in shared memory as bytes
constexpr int kStdThreads = 512;
constexpr int kStdWarps = kStdThreads / kWarp;
constexpr int kAucThreads = 512;
constexpr int kAucWarps = kAucThreads / kWarp;
constexpr int kAucTile = 4096;                // positives sorted in shared memory at a time

// ---- mutual information --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kMiThreads)
discrete_mi_kernel(const float* __restrict__ mu, int ld, int rs, const long long* __restrict__ train_rows, int n,
                   const int* __restrict__ train_cls, const int* __restrict__ n_classes, int K, int S,
                   double* __restrict__ mi, float* __restrict__ edges_out) {
  extern __shared__ uint8_t bin[];                             // [n]
  __shared__ int cnt[kModMaxClasses * kMiBins];
  __shared__ int bcnt[kMiBins];
  __shared__ double part[kModMaxClasses];
  __shared__ float wlo[kMiWarps], whi[kMiWarps];
  __shared__ float edge[kMiBins + 1];
  __shared__ int occupied;
  const int t = threadIdx.x, d = blockIdx.x;
  const long long col = (long long)d * ld;

  float lo = CUDART_INF_F, hi = -CUDART_INF_F;
  for (int i = t; i < n; i += kMiThreads) {
    const float v = mu[train_rows[i] * (long long)rs + col];
    lo = fminf(lo, v);
    hi = fmaxf(hi, v);
  }
  if (t < kMiBins) bcnt[t] = 0;
  histogram_edges<kMiWarps>(lo, hi, wlo, whi, edge);
  if (edges_out && t <= kMiBins) edges_out[(long long)d * (kMiBins + 1) + t] = edge[t];
  for (int i = t; i < n; i += kMiThreads) {
    const int b = histogram_bin(edge, mu[train_rows[i] * (long long)rs + col]);
    bin[i] = (uint8_t)b;
    atomicAdd(&bcnt[b], 1);
  }
  __syncthreads();
  if (t == 0) {
    int o = 0;
    for (int j = 0; j < kMiBins; ++j) o += bcnt[j] > 0 ? 1 : 0;
    occupied = o;
  }
  const double dn = (double)n, ln = log(dn);
  for (int k = 0; k < K; ++k) {
    const int nc = class_count(n_classes, k, S);
    for (int j = t; j < nc * kMiBins; j += kMiThreads) cnt[j] = 0;
    __syncthreads();
    const int* cls = train_cls + (long long)k * n;
    for (int i = t; i < n; i += kMiThreads) atomicAdd(&cnt[cls[i] * kMiBins + bin[i]], 1);
    __syncthreads();
    // sklearn's terms c/n (log c - log n) + c/n (-log(a b) + log n + log n) over the non-zero cells, each rounded as
    // numpy rounds it (no contraction); |term| < DBL_EPSILON counts 0
    for (int c = t; c < nc; c += kMiThreads) {
      const int* row = cnt + c * kMiBins;
      long long a = 0;
      for (int j = 0; j < kMiBins; ++j) a += row[j];
      double s = 0.0;
      for (int j = 0; j < kMiBins; ++j) {
        if (row[j] == 0) continue;
        const double cv = (double)row[j];
        const double cn = __ddiv_rn(cv, dn);
        const double outer = (double)(a * (long long)bcnt[j]);
        const double lo_ = __dadd_rn(__dadd_rn(-log(outer), ln), ln);
        double term = __dadd_rn(__dmul_rn(cn, __dsub_rn(log(cv), ln)), __dmul_rn(cn, lo_));
        if (fabs(term) < DBL_EPSILON) term = 0.0;
        s = __dadd_rn(s, term);
      }
      part[c] = s;
    }
    __syncthreads();
    if (t == 0) {
      double s = 0.0;
      if (nc > 1 && occupied > 1)
        for (int c = 0; c < nc; ++c) s = __dadd_rn(s, part[c]);
      mi[(long long)d * K + k] = s > 0.0 ? s : 0.0;
    }
    __syncthreads();
  }
}

// ---- explicitness ------------------------------------------------------------------------------------------------
struct ModWs {
  double* feat;     // [n + m][D] standardised features, training rows first
  double* fit;      // [K][fit_stride] solver workspaces
  double* proba;    // [K][S][n + m] probabilities (when the caller does not ask for them)
  size_t fit_stride;
};

// Offsets of the workspace segments from `base` (NULL for the size only) -> total bytes.
size_t mod_layout(int D, int n, int m, int K, int S, char* base, ModWs* w) {
  const size_t rows = (size_t)n + m;
  const size_t fit_bytes = align_up(fit_workspace_doubles(n, D, S) * sizeof(double));
  const size_t sizes[3] = {rows * D * 8, (size_t)K * fit_bytes, (size_t)K * S * rows * 8};
  size_t off[3];
  const size_t total = carve_workspace(sizes, off);
  if (w) {
    w->feat = reinterpret_cast<double*>(base + off[0]);
    w->fit = reinterpret_cast<double*>(base + off[1]);
    w->proba = reinterpret_cast<double*>(base + off[2]);
    w->fit_stride = fit_bytes / sizeof(double);
  }
  return total;
}

__global__ void __launch_bounds__(kStdThreads)
standardise_kernel(const float* __restrict__ mu, int ld, int rs, int D, const long long* __restrict__ train_rows,
                   int n, const long long* __restrict__ test_rows, int m, double* __restrict__ mean_out,
                   double* __restrict__ std_out, ModWs w) {
  __shared__ double red[kStdWarps];
  const int t = threadIdx.x, d = blockIdx.x;
  const long long col = (long long)d * ld;
  double s = 0.0;
  for (int i = t; i < n; i += kStdThreads) s += (double)mu[train_rows[i] * (long long)rs + col];
  const double mean = block_sum<kStdWarps>(s, red) / n;
  s = 0.0;
  for (int i = t; i < n; i += kStdThreads) {
    const double e = __dsub_rn((double)mu[train_rows[i] * (long long)rs + col], mean);
    s = __dadd_rn(s, __dmul_rn(e, e));
  }
  double sd = sqrt(block_sum<kStdWarps>(s, red) / n);
  if (sd == 0.0) sd = 1.0;                                     // StandardScaler's rule for a constant feature
  if (t == 0) {
    mean_out[d] = mean;
    std_out[d] = sd;
  }
  for (int i = t; i < n + m; i += kStdThreads) {
    const long long row = i < n ? train_rows[i] : test_rows[i - n];
    w.feat[(long long)i * D + d] = __ddiv_rn(__dsub_rn((double)mu[row * (long long)rs + col], mean), sd);
  }
}

__global__ void __launch_bounds__(kFitThreads, 1)
explicitness_fit_kernel(int D, int n, int m, const int* __restrict__ train_cls, const int* __restrict__ n_classes,
                        int S, double* __restrict__ coef, int* __restrict__ iters, double* __restrict__ proba,
                        ModWs w) {
  const int t = threadIdx.x, k = blockIdx.x;
  const int nc = class_count(n_classes, k, S);
  const int Dp = D + 1;
  const long long rows = (long long)n + m;
  double* ck = coef + (long long)k * S * Dp;
  logistic_fit_cta(w.feat, D, n, train_cls + (long long)k * n, nc, nc > 2, 1.0, S, ck, iters + k,
                   w.fit + k * w.fit_stride);

  // probabilities: softmax of the decisions (classes added in order) for nc > 2; p_1 = 1 / (1 + exp(-z)) and
  // p_0 = 1 - p_1 for nc = 2 (sklearn's predict_proba); NaN for nc < 2 and beyond the factor's columns
  double* pk = (proba ? proba : w.proba) + (long long)k * S * rows;
  const int cols = nc > 2 ? nc : (nc == 2 ? 2 : 0);
  for (long long j = t; j < (long long)(S - cols) * rows; j += kFitThreads) pk[cols * rows + j] = CUDART_NAN;
  if (cols == 0) return;
  for (long long i = t; i < rows; i += kFitThreads) {
    const double* xi = w.feat + i * D;
    if (nc == 2) {
      double z = ck[D];
      for (int d = 0; d < D; ++d) z = fma(ck[d], xi[d], z);
      const double p1 = __ddiv_rn(1.0, __dadd_rn(1.0, exp(-z)));
      pk[i] = __dsub_rn(1.0, p1);
      pk[rows + i] = p1;
      continue;
    }
    double mx = -CUDART_INF;
    for (int c = 0; c < nc; ++c) {
      const double* wc = ck + (long long)c * Dp;
      double z = wc[D];
      for (int d = 0; d < D; ++d) z = fma(wc[d], xi[d], z);
      pk[c * rows + i] = z;
      mx = fmax(mx, z);
    }
    double se = 0.0;
    for (int c = 0; c < nc; ++c) se = __dadd_rn(se, exp(__dsub_rn(pk[c * rows + i], mx)));
    for (int c = 0; c < nc; ++c) pk[c * rows + i] = __ddiv_rn(exp(__dsub_rn(pk[c * rows + i], mx)), se);
  }
}

// An order-preserving integer key of a probability (-0 taken as +0).
__device__ __forceinline__ unsigned long long prob_key(double v) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(v == 0.0 ? 0.0 : v);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

__global__ void __launch_bounds__(kAucThreads)
auc_kernel(int n, int m, int K, const int* __restrict__ train_cls, const int* __restrict__ test_cls,
           const int* __restrict__ n_classes, int S, const double* __restrict__ proba, double* __restrict__ auc,
           ModWs w) {
  __shared__ unsigned long long key[kAucTile];
  __shared__ long long red[kAucWarps];
  __shared__ int wcount[kAucWarps];
  const int t = threadIdx.x, lane = t & (kWarp - 1), warp = t / kWarp;
  const int set = blockIdx.x & 1, c = (blockIdx.x >> 1) % S, k = (blockIdx.x >> 1) / S;
  const int nc = class_count(n_classes, k, S);
  const int cols = nc > 2 ? nc : (nc == 2 ? 2 : 0);
  double* out = auc + ((long long)set * K + k) * S + c;
  if (c >= cols) {
    if (t == 0) *out = CUDART_NAN;
    return;
  }
  const long long rows = (long long)n + m;
  const int len = set == 0 ? n : m;
  const int* lab = set == 0 ? train_cls + (long long)k * n : test_cls + (long long)k * m;
  const double* p = (proba ? proba : w.proba) + ((long long)k * S + c) * rows + (set == 0 ? 0 : n);

  long long np_ = 0;
  for (int i = t; i < len; i += kAucThreads) np_ += lab[i] == c ? 1 : 0;
  const long long n_pos = block_sum<kAucWarps>(np_, red), n_neg = (long long)len - n_pos;
  __syncthreads();
  if (n_pos == 0 || n_neg == 0) {
    if (t == 0) *out = CUDART_NAN;
    return;
  }
  const unsigned lt = (1u << lane) - 1u;
  long long gt = 0, eq = 0;
  for (long long first = 0; first < n_pos; first += kAucTile) {
    const int tn = (int)min((long long)kAucTile, n_pos - first);
    // stage the positives of ranks [first, first + tn), ranks in row order
    long long base = 0;
    for (int s0 = 0; s0 < len; s0 += kAucThreads) {
      const int i = s0 + t;
      const bool in = i < len && lab[i] == c;
      const unsigned mask = __ballot_sync(0xffffffffu, in);
      if (lane == 0) wcount[warp] = __popc(mask);
      __syncthreads();
      long long rank = base + __popc(mask & lt);
      int total = 0;
      for (int v = 0; v < kAucWarps; ++v) {
        if (v < warp) rank += wcount[v];
        total += wcount[v];
      }
      if (in && rank >= first && rank < first + tn) key[rank - first] = prob_key(p[i]);
      base += total;
      __syncthreads();
    }
    int P2 = 1;
    while (P2 < tn) P2 <<= 1;
    for (int i = tn + t; i < P2; i += kAucThreads) key[i] = ~0ull;
    __syncthreads();
    for (int kk = 2; kk <= P2; kk <<= 1) {
      for (int j = kk >> 1; j > 0; j >>= 1) {
        for (int i = t; i < P2; i += kAucThreads) {
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
    // every negative: the staged positives above it and those equal to it
    for (int i = t; i < len; i += kAucThreads) {
      if (lab[i] == c) continue;
      const unsigned long long q = prob_key(p[i]);
      int a = 0, b = tn;                                       // lower bound: first key >= q
      while (a < b) {
        const int h = (a + b) >> 1;
        if (key[h] < q) a = h + 1; else b = h;
      }
      int u = a, e = tn;                                       // upper bound: first key > q
      while (u < e) {
        const int h = (u + e) >> 1;
        if (key[h] <= q) u = h + 1; else e = h;
      }
      gt += tn - u;
      eq += u - a;
    }
    __syncthreads();
  }
  gt = block_sum<kAucWarps>(gt, red);
  __syncthreads();
  eq = block_sum<kAucWarps>(eq, red);
  __syncthreads();
  if (t == 0) *out = (double)(2 * gt + eq) / (2.0 * (double)n_pos * (double)n_neg);
}

bool mod_shape_ok(int D, int n, int m, int K, int S) {
  return D >= 1 && D <= kModMaxD && n >= 1 && n <= kModMaxTrain && m >= 1 && K >= 1 && S >= 1 &&
         S <= kModMaxClasses && (long long)n + m <= 0x7fffffffLL && (long long)K * ((long long)n + m) <= 0x7fffffffLL &&
         (long long)K * S * 2 <= 0x7fffffffLL;
}

}  // namespace
}  // namespace dv

using namespace dv;

extern "C" {

int dv_discrete_mutual_info(const float* mu, int ld, int row_stride, int N, int D, const long long* train_rows,
                            int num_train, const int* train_cls, const int* n_classes, int K, int class_stride,
                            double* mi, float* edges, void* stream) {
  if (N < 1 || D < 1 || D > kMiMaxD || num_train < 1 || num_train > kModMaxTrain || K < 1 || class_stride < 1 ||
      class_stride > kModMaxClasses || ld < 1 || row_stride < 1 || (long long)K * num_train > 0x7fffffffLL)
    return DV_ERR_BAD_SHAPE;
  if (!mu || !train_rows || !train_cls || !n_classes || !mi) return DV_ERR_BAD_ARG;
  if (misaligned(mu, 4) || misaligned(train_rows, 8) || misaligned(train_cls, 4) || misaligned(n_classes, 4) ||
      misaligned(mi, 8) || misaligned(edges, 4))
    return DV_ERR_BAD_ARG;
  static bool attr = false;
  int rc = set_max_dynamic_smem(discrete_mi_kernel, kModMaxTrain, &attr);
  if (rc != DV_OK) return rc;
  discrete_mi_kernel<<<D, kMiThreads, num_train, as_stream(stream)>>>(mu, ld, row_stride, train_rows, num_train,
                                                                      train_cls, n_classes, K, class_stride, mi, edges);
  return check_launch();
}

size_t dv_explicitness_workspace_bytes(int D, int num_train, int num_test, int K, int class_stride) {
  if (!mod_shape_ok(D, num_train, num_test, K, class_stride)) return 0;
  return mod_layout(D, num_train, num_test, K, class_stride, nullptr, nullptr);
}

int dv_explicitness_fit(const float* mu, int ld, int row_stride, int N, int D, const long long* train_rows,
                        int num_train, const long long* test_rows, int num_test, const int* train_cls,
                        const int* test_cls, const int* n_classes, int K, int class_stride, double* coef,
                        double* auc, int* iters, double* mean, double* std, double* proba, void* workspace,
                        size_t workspace_bytes, void* stream) {
  if (N < 1 || !mod_shape_ok(D, num_train, num_test, K, class_stride) || ld < 1 || row_stride < 1)
    return DV_ERR_BAD_SHAPE;
  if (!mu || !train_rows || !test_rows || !train_cls || !test_cls || !n_classes || !coef || !auc || !iters || !mean ||
      !std)
    return DV_ERR_BAD_ARG;
  if (misaligned(mu, 4) || misaligned(train_rows, 8) || misaligned(test_rows, 8) || misaligned(train_cls, 4) ||
      misaligned(test_cls, 4) || misaligned(n_classes, 4) || misaligned(coef, 8) || misaligned(auc, 8) ||
      misaligned(iters, 4) || misaligned(mean, 8) || misaligned(std, 8) || misaligned(proba, 8) ||
      misaligned(workspace, 8))
    return DV_ERR_BAD_ARG;
  const int S = class_stride, n = num_train, m = num_test;
  if (!workspace || workspace_bytes < mod_layout(D, n, m, K, S, nullptr, nullptr)) return DV_ERR_WORKSPACE;
  ModWs w;
  mod_layout(D, n, m, K, S, static_cast<char*>(workspace), &w);
  cudaStream_t s = as_stream(stream);
  int rc;
  standardise_kernel<<<D, kStdThreads, 0, s>>>(mu, ld, row_stride, D, train_rows, n, test_rows, m, mean, std, w);
  if ((rc = check_launch()) != DV_OK) return rc;
  explicitness_fit_kernel<<<K, kFitThreads, 0, s>>>(D, n, m, train_cls, n_classes, S, coef, iters, proba, w);
  if ((rc = check_launch()) != DV_OK) return rc;
  auc_kernel<<<K * S * 2, kAucThreads, 0, s>>>(n, m, K, train_cls, test_cls, n_classes, S, proba, auc, w);
  return check_launch();
}

}  // extern "C"

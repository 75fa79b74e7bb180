// Downstream-task logistic regression (Locatello et al. 2019, section 6; disentanglement_lib's downstream_task.py with
// LogisticRegressionCV(Cs=10, cv=KFold(5))): for every scored factor, the cross-validated choice of C among the
// caller's grid, the refit at that C on every training row, and the predicted class of every training and test row.
// The reference has no such score; the entry points and their rules are declared in include/disvae_b200.h.
//
// dv_downstream_logistic_cv (two launches, no host synchronisation):
//   folds   one fit per (factor, fold, C), each the exact minimiser by logistic_fit_cta (dv_logistic.cuh) over the
//           classes present in the fold's training part: the CTA gathers those rows from mu in fp64, compacts the
//           present classes to 0 .. p-1 (order kept), fits, and counts the held-out rows it predicts right.
//   refit   one fit per factor: the fold accuracies of each C added in fold order, the first maximum chosen, the fit
//           on every training row at that C, and the predictions of every training and test row.
// Both launches run a fixed grid of fit slots, each with its own workspace, that walk the fits in a static order
// (slot s takes fits s, s + slots, ...).  Fits are independent, so the slot count changes no result, and the workspace
// is bounded by the slots, not by the number of fits.  Every sum has a fixed order and there are no floating-point
// atomics, so results are bit-identical run to run.
#include <float.h>

#include "dv_logistic.cuh"

namespace dv {
namespace {

constexpr int kDsFolds = 5;                   // KFold(n_splits=5)
constexpr int kDsMaxCs = 32;                  // the grid travels in the kernels' parameters
constexpr int kDsMinTrain = kDsFolds;         // every fold holds a row
constexpr int kDsMaxTrain = 32768;
constexpr int kDsMaxClasses = 256;
constexpr int kDsMaxNewton = 300;             // fits at C = 1e4 on unstandardised means take more steps than C = 1
constexpr int kDsMaxCG = 500;
constexpr size_t kDsBudget = size_t(8) << 30; // workspace bytes the slots may take, at least one slot

struct CsArg {
  double v[kDsMaxCs];
};

struct DsWs {
  char* base;
  size_t slot_bytes;                          // per slot: solver workspace, gathered rows, labels, model rows
  size_t fit_off, x_off, y_off, coef_off;
};

__device__ __forceinline__ double* slot_ptr(const DsWs& w, int s, size_t off) {
  return reinterpret_cast<double*>(w.base + (size_t)s * w.slot_bytes + off);
}

// The layout of one slot for n training rows (the refit's, the most a fold fit needs).
DsWs ds_slot_layout(int D, int n, int S) {
  DsWs w;
  const size_t sizes[4] = {fit_workspace_doubles(n, D, S) * sizeof(double), (size_t)n * D * sizeof(double),
                           (size_t)n * sizeof(int), (size_t)S * (D + 1) * sizeof(double)};
  size_t off[4];
  w.base = nullptr;
  w.slot_bytes = carve_workspace(sizes, off);
  w.fit_off = off[0];
  w.x_off = off[1];
  w.y_off = off[2];
  w.coef_off = off[3];
  return w;
}

// Slots: one per SM at most, no more than there are fold fits, and within kDsBudget (at least one).
int ds_slots(const DsWs& w, int K, int nC) {
  const long long fits = (long long)K * kDsFolds * nC;
  long long s = (long long)(kDsBudget / w.slot_bytes);
  s = s < 1 ? 1 : s;
  s = s < kNumSMs ? s : kNumSMs;
  return (int)(s < fits ? s : fits);
}

// Fold f of n rows under KFold: [*s0, *s1), the first n % 5 folds one row longer.
__device__ __forceinline__ void fold_bounds(int n, int f, int* s0, int* s1) {
  const int q = n / kDsFolds, r = n % kDsFolds;
  *s0 = f * q + min(f, r);
  *s1 = *s0 + q + (f < r ? 1 : 0);
}

// argmax_r W_r x + b_r over R model rows (the lowest r on a tie), or 1 when w.x + b > 0 (binary, R = 1); 0 for R = 0.
// x is row `row` of mu in fp64; the decisions are added as dv_logistic_fit adds them.
__device__ __forceinline__ int predict_row(const float* __restrict__ mu, long long rs, int ld, long long row,
                                           const double* __restrict__ coef, int D, int R, bool multi) {
  const int Dp = D + 1;
  int best_r = 0;
  double best = 0.0;
  for (int r = 0; r < R; ++r) {
    const double* w = coef + (long long)r * Dp;
    double s = w[D];
    for (int d = 0; d < D; ++d) s = fma(w[d], (double)mu[row * rs + (long long)d * ld], s);
    if (r == 0 || s > best) { best = s; best_r = r; }
  }
  return multi ? best_r : (R == 1 && best > 0.0 ? 1 : 0);
}

__global__ void __launch_bounds__(kFitThreads, 1)
ds_fold_kernel(const float* __restrict__ mu, int ld, int rs, int D, const long long* __restrict__ train_rows, int n,
               const int* __restrict__ train_cls, const int* __restrict__ n_classes, int K, int S, CsArg cs, int nC,
               double* __restrict__ fold_acc, int* __restrict__ iters, double* __restrict__ fold_coef,
               int* __restrict__ fold_pred, DsWs w) {
  __shared__ int present[kDsMaxClasses];      // flags, then the compact index of each present class (-1 absent)
  __shared__ int inv[kDsMaxClasses];          // compact index -> class
  __shared__ int npres;
  __shared__ int red[kFitWarps];
  const int t = threadIdx.x, Dp = D + 1;
  const int fits = K * kDsFolds * nC;
  double* fit_ws = slot_ptr(w, blockIdx.x, w.fit_off);
  double* x = slot_ptr(w, blockIdx.x, w.x_off);
  int* y = reinterpret_cast<int*>(slot_ptr(w, blockIdx.x, w.y_off));
  double* scratch = slot_ptr(w, blockIdx.x, w.coef_off);
  for (int j = blockIdx.x; j < fits; j += gridDim.x) {
    const int k = j / (kDsFolds * nC), f = (j / nC) % kDsFolds, c = j % nC;
    const int nc = class_count(n_classes, k, S);
    const int* cls = train_cls + (long long)k * n;
    int s0, s1;
    fold_bounds(n, f, &s0, &s1);
    const int m = n - (s1 - s0);
    for (int v = t; v < S; v += kFitThreads) present[v] = 0;
    __syncthreads();
    for (int i = t; i < m; i += kFitThreads) present[cls[i < s0 ? i : i + (s1 - s0)]] = 1;   // flags: no order
    __syncthreads();
    if (t == 0) {
      int p = 0;
      for (int v = 0; v < S; ++v) {
        if (present[v]) inv[p] = v;
        present[v] = present[v] ? p++ : -1;
      }
      npres = p;
    }
    __syncthreads();
    const int p = npres;
    for (long long e = t; e < (long long)m * D; e += kFitThreads) {
      const int i = (int)(e / D), d = (int)(e % D);
      x[e] = (double)mu[train_rows[i < s0 ? i : i + (s1 - s0)] * (long long)rs + (long long)d * ld];
    }
    for (int i = t; i < m; i += kFitThreads) y[i] = present[cls[i < s0 ? i : i + (s1 - s0)]];
    __syncthreads();
    // a fold missing classes fits the limit of its objective: the fit over the classes it has, still multinomial
    // when the factor has more than two classes
    const bool multi = nc > 2;
    const int R = p < 2 ? 0 : (multi ? p : 1);
    logistic_fit_cta<kDsMaxNewton, kDsMaxCG>(x, D, m, y, p, multi, cs.v[c], S, scratch,
                                             iters + (long long)k * (kDsFolds * nC + 1) + f * nC + c, fit_ws);
    if (fold_coef) {
      double* out = fold_coef + (long long)j * S * Dp;
      for (int o = t; o < S * Dp; o += kFitThreads) {
        const int v = o / Dp, r = multi ? present[v] : v;
        out[o] = r >= 0 && r < R ? scratch[r * Dp + o % Dp] : CUDART_NAN;
      }
    }
    int right = 0;
    for (int i = s0 + t; i < s1; i += kFitThreads) {
      const int r = predict_row(mu, rs, ld, train_rows[i], scratch, D, R, multi);
      const int v = R == 0 ? inv[0] : (multi ? inv[r] : r);
      right += v == cls[i] ? 1 : 0;
      if (fold_pred) fold_pred[((long long)k * nC + c) * n + i] = v;
    }
    right = block_sum<kFitWarps>(right, red);
    if (t == 0) fold_acc[j] = (double)right / (double)(s1 - s0);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kFitThreads, 1)
ds_refit_kernel(const float* __restrict__ mu, int ld, int rs, int D, const long long* __restrict__ train_rows, int n,
                const long long* __restrict__ test_rows, int m, const int* __restrict__ train_cls,
                const int* __restrict__ n_classes, int K, int S, CsArg cs, int nC,
                const double* __restrict__ fold_acc, int* __restrict__ chosen, double* __restrict__ coef,
                int* __restrict__ pred, int* __restrict__ iters, DsWs w) {
  __shared__ int sel;
  const int t = threadIdx.x, Dp = D + 1;
  double* fit_ws = slot_ptr(w, blockIdx.x, w.fit_off);
  double* x = slot_ptr(w, blockIdx.x, w.x_off);
  for (int k = blockIdx.x; k < K; k += gridDim.x) {
    const int nc = class_count(n_classes, k, S);
    if (t == 0) {
      // numpy's scores.sum(axis=0) over the folds, then the first maximum (the smallest C on a tie)
      const double* a = fold_acc + (long long)k * kDsFolds * nC;
      int best = 0;
      double best_v = 0.0;
      for (int c = 0; c < nC; ++c) {
        double s = a[c];
        for (int f = 1; f < kDsFolds; ++f) s = __dadd_rn(s, a[f * nC + c]);
        if (c == 0 || s > best_v) { best_v = s; best = c; }
      }
      sel = best;
      chosen[k] = best;
    }
    for (long long e = t; e < (long long)n * D; e += kFitThreads) {
      const int i = (int)(e / D), d = (int)(e % D);
      x[e] = (double)mu[train_rows[i] * (long long)rs + (long long)d * ld];
    }
    __syncthreads();
    const bool multi = nc > 2;
    const int R = nc < 2 ? 0 : (multi ? nc : 1);
    double* ck = coef + (long long)k * S * Dp;
    logistic_fit_cta<kDsMaxNewton, kDsMaxCG>(x, D, n, train_cls + (long long)k * n, nc, multi, cs.v[sel], S, ck,
                                             iters + (long long)k * (kDsFolds * nC + 1) + kDsFolds * nC, fit_ws);
    int* pk = pred + (long long)k * (n + m);
    for (int i = t; i < n + m; i += kFitThreads)
      pk[i] = predict_row(mu, rs, ld, i < n ? train_rows[i] : test_rows[i - n], ck, D, R, multi);
    __syncthreads();
  }
}

bool ds_shape_ok(int D, int n, int K, int S, int nC) {
  return D >= 1 && D <= kFitMaxD && n >= kDsMinTrain && n <= kDsMaxTrain && K >= 1 && S >= 1 && S <= kDsMaxClasses &&
         nC >= 1 && nC <= kDsMaxCs && (long long)K * kDsFolds * nC <= 0x7fffffffLL;
}

}  // namespace
}  // namespace dv

using namespace dv;

extern "C" {

size_t dv_downstream_workspace_bytes(int D, int num_train, int K, int class_stride, int nC) {
  if (!ds_shape_ok(D, num_train, K, class_stride, nC)) return 0;
  const DsWs w = ds_slot_layout(D, num_train, class_stride);
  return (size_t)ds_slots(w, K, nC) * w.slot_bytes;
}

int dv_downstream_logistic_cv(const float* mu, int ld, int row_stride, int N, int D, const long long* train_rows,
                              int num_train, const long long* test_rows, int num_test, const int* train_cls,
                              const int* n_classes, int K, int class_stride, const double* Cs, int nC,
                              double* fold_acc, int* chosen, double* coef, int* pred, int* iters, double* fold_coef,
                              int* fold_pred, void* workspace, size_t workspace_bytes, void* stream) {
  if (N < 1 || !ds_shape_ok(D, num_train, K, class_stride, nC) || num_test < 1 || ld < 1 || row_stride < 1 ||
      (long long)num_train + num_test > 0x7fffffffLL)
    return DV_ERR_BAD_SHAPE;
  if (!mu || !train_rows || !test_rows || !train_cls || !n_classes || !Cs || !fold_acc || !chosen || !coef || !pred ||
      !iters)
    return DV_ERR_BAD_ARG;
  if (misaligned(mu, 4) || misaligned(train_rows, 8) || misaligned(test_rows, 8) || misaligned(train_cls, 4) ||
      misaligned(n_classes, 4) || misaligned(fold_acc, 8) || misaligned(chosen, 4) || misaligned(coef, 8) ||
      misaligned(pred, 4) || misaligned(iters, 4) || misaligned(fold_coef, 8) || misaligned(fold_pred, 4) ||
      misaligned(workspace, 8))
    return DV_ERR_BAD_ARG;
  CsArg cs;
  for (int c = 0; c < kDsMaxCs; ++c) {
    cs.v[c] = c < nC ? Cs[c] : 1.0;
    if (!(cs.v[c] > 0.0 && cs.v[c] <= DBL_MAX)) return DV_ERR_BAD_ARG;    // NaN, 0, negative or infinite
  }
  DsWs w = ds_slot_layout(D, num_train, class_stride);
  const int slots = ds_slots(w, K, nC);
  if (!workspace || workspace_bytes < (size_t)slots * w.slot_bytes) return DV_ERR_WORKSPACE;
  w.base = static_cast<char*>(workspace);
  cudaStream_t s = as_stream(stream);
  int rc;
  ds_fold_kernel<<<slots, kFitThreads, 0, s>>>(mu, ld, row_stride, D, train_rows, num_train, train_cls, n_classes, K,
                                               class_stride, cs, nC, fold_acc, iters, fold_coef, fold_pred, w);
  if ((rc = check_launch()) != DV_OK) return rc;
  ds_refit_kernel<<<slots < K ? slots : K, kFitThreads, 0, s>>>(mu, ld, row_stride, D, train_rows, num_train,
                                                                test_rows, num_test, train_cls, n_classes, K,
                                                                class_stride, cs, nC, fold_acc, chosen, coef, pred,
                                                                iters, w);
  return check_launch();
}

}  // extern "C"

// SAP score (Separated Attribute Predictability, Kumar et al. 2018, section 3): for every (latent d, scored factor
// k) the exact fit of LinearSVC(C, class_weight="balanced") on the 1-D training column mu[train_rows][d] against
// factor k's labels, then the accuracy of that classifier on the test rows.  The reference has no such score; the
// entry point is declared in include/disvae_b200.h.
//
// Each binary problem (one-vs-rest per class when there are more than two classes, one problem for two) is
//   min over z = (w, b):  f(z) = 1/2 (w^2 + b^2) + sum_i C_i max(0, m_i)^2,   m_i = 1 - s_i (w x_i + b),
// the objective liblinear minimises for the squared hinge with the intercept as a regularised feature of scale 1.
// f is strictly convex and piecewise quadratic, so semismooth Newton on the generalised Hessian
//   H = I + 2 sum_{m_i > 0} C_i (x_i, 1)(x_i, 1)^T
// with an Armijo backtracking line search reaches the exact minimiser once the active set is settled (a few steps).
// Convergence is |grad f|_inf <= kSapTol * (|w| + |b| + 2 sum_{m_i > 0} C_i m_i (|x_i| + 1)), the scale of the two
// parts of the gradient; every sum is fp64.
//
// One CTA per (latent, factor).  It stages the latent's training column (fp32) and the factor's training labels
// (uint8) in shared memory; its warps take the binary problems in turn (warp w: problems w, w + 16, ...), each lane
// summing rows lane, lane + 32, ... in order and a butterfly over the warp adding the partials (every lane ends with
// the same bits, so the solver's control flow is warp-uniform).  The CTA then scores the test rows against the fitted
// lines and adds the correct predictions in a fixed integer tree.  No floating-point atomics: results are bit-identical run to run.
#include <math.h>
#include <math_constants.h>

#include "dv_common.cuh"

namespace dv {
namespace {

constexpr int kSapThreads = 512;
constexpr int kSapWarps = kSapThreads / kWarp;
constexpr int kSapMaxD = 1024;
constexpr int kSapMaxClasses = 256;        // labels are staged as uint8
constexpr int kSapMaxTrain = 32768;        // 5 bytes a row of shared memory
constexpr int kSapMaxIter = 64;            // Newton steps per problem
constexpr int kSapMaxHalvings = 40;        // line-search halvings per step
constexpr double kSapTol = 1e-10;
constexpr double kSapArmijo = 1e-4;

// shared memory: class weights, fitted lines, the per-warp counts, then the column and the labels
constexpr int kSapFixedSmem = kSapMaxClasses * 8 + kSapMaxClasses * 16 + kSapWarps * 4;

size_t sap_smem_bytes(int num_train) { return (size_t)kSapFixedSmem + (size_t)num_train * 5; }

struct SapEval {
  double f, gw, gb, hww, hwb, hbb, scale;
};

// f, gradient, generalised Hessian and the stationarity scale at (w, b), summed by one warp over the staged rows.
__device__ __forceinline__ SapEval sap_eval(const float* x, const uint8_t* lab, int n, double w, double b, int pos,
                                            bool binary, double C, const double* cw, int lane) {
  const double cpos = binary ? 0.0 : C * cw[pos];
  double f = 0.0, gx = 0.0, g1 = 0.0, hxx = 0.0, hx = 0.0, h1 = 0.0, sc = 0.0;
  for (int i = lane; i < n; i += kWarp) {
    const double xi = (double)x[i];
    const int y = lab[i];
    const double s = y == pos ? 1.0 : -1.0;
    const double ci = binary ? C * cw[y] : (y == pos ? cpos : C);
    const double m = 1.0 - s * (w * xi + b);
    if (m > 0.0) {
      const double cm = ci * m;
      f = fma(cm, m, f);
      gx = fma(cm * s, xi, gx);
      g1 += cm * s;
      hxx = fma(ci * xi, xi, hxx);
      hx = fma(ci, xi, hx);
      h1 += ci;
      sc = fma(cm, fabs(xi) + 1.0, sc);
    }
  }
  SapEval e;
  e.f = 0.5 * (w * w + b * b) + warp_sum(f);
  e.gw = w - 2.0 * warp_sum(gx);
  e.gb = b - 2.0 * warp_sum(g1);
  e.hww = 1.0 + 2.0 * warp_sum(hxx);
  e.hwb = 2.0 * warp_sum(hx);
  e.hbb = 1.0 + 2.0 * warp_sum(h1);
  e.scale = fabs(w) + fabs(b) + 2.0 * warp_sum(sc);
  return e;
}

__device__ __forceinline__ bool sap_stationary(const SapEval& e) {
  return fmax(fabs(e.gw), fabs(e.gb)) <= kSapTol * e.scale;
}

// One binary problem by one warp -> (w, b) and the Newton steps taken (-1 if not converged).
__device__ __forceinline__ int sap_solve(const float* x, const uint8_t* lab, int n, int pos, bool binary, double C,
                                         const double* cw, int lane, double* w_out, double* b_out) {
  double w = 0.0, b = 0.0;
  SapEval e = sap_eval(x, lab, n, w, b, pos, binary, C, cw, lane);
  for (int it = 0; it <= kSapMaxIter; ++it) {
    if (sap_stationary(e)) {
      *w_out = w;
      *b_out = b;
      return it;
    }
    if (it == kSapMaxIter) break;
    const double det = e.hww * e.hbb - e.hwb * e.hwb;      // H is positive definite: det >= 1
    const double pw = -(e.hbb * e.gw - e.hwb * e.gb) / det;
    const double pb = -(e.hww * e.gb - e.hwb * e.gw) / det;
    const double slope = e.gw * pw + e.gb * pb;               // < 0
    double t = 1.0;
    bool moved = false;
    for (int h = 0; h <= kSapMaxHalvings; ++h, t *= 0.5) {
      const double wt = w + t * pw, bt = b + t * pb;
      const SapEval et = sap_eval(x, lab, n, wt, bt, pos, binary, C, cw, lane);
      // sufficient decrease, or a change of f below its rounding (where only the gradient test can decide)
      if (et.f - e.f <= kSapArmijo * t * slope + 1e-15 * fabs(e.f)) {
        w = wt;
        b = bt;
        e = et;
        moved = true;
        break;
      }
    }
    if (!moved) break;
  }
  *w_out = w;
  *b_out = b;
  return -1;
}

__global__ void __launch_bounds__(kSapThreads, 1)
sap_kernel(const float* __restrict__ mu, int ld, int rs, int D, const long long* __restrict__ train_rows, int n_train,
           const long long* __restrict__ test_rows, int n_test, const int* __restrict__ train_cls,
           const int* __restrict__ test_cls, const int* __restrict__ n_classes, const int* __restrict__ counts, int K,
           int cs, double C, float* __restrict__ score, double* __restrict__ coef, int* __restrict__ iters) {
  extern __shared__ __align__(16) uint8_t smem[];
  double* cw = reinterpret_cast<double*>(smem);
  double* line = cw + kSapMaxClasses;                         // [class][2]
  int* wcount = reinterpret_cast<int*>(line + 2 * kSapMaxClasses);
  float* x = reinterpret_cast<float*>(wcount + kSapWarps);
  uint8_t* lab = reinterpret_cast<uint8_t*>(x + n_train);
  const int t = threadIdx.x, lane = t & (kWarp - 1), warp = t / kWarp;
  const int cell = blockIdx.x, d = cell / K, k = cell % K;
  const int nc = class_count(n_classes, k, cs);
  const long long col = (long long)d * ld;

  for (int i = t; i < n_train; i += kSapThreads) {
    x[i] = mu[train_rows[i] * (long long)rs + col];
    lab[i] = (uint8_t)train_cls[(long long)k * n_train + i];
  }
  for (int c = t; c < nc; c += kSapThreads)
    cw[c] = (double)n_train / ((double)nc * (double)counts[(long long)k * cs + c]);
  __syncthreads();

  // problems: one per class (one-vs-rest) above two classes, one (positive class 1) for two, none for one
  const bool binary = nc == 2;
  const int np = nc > 2 ? nc : (binary ? 1 : 0);
  const long long slot0 = (long long)cell * cs;
  for (int p = warp; p < np; p += kSapWarps) {
    double w, b;
    const int n_it = sap_solve(x, lab, n_train, binary ? 1 : p, binary, C, cw, lane, &w, &b);
    if (lane == 0) {
      line[2 * p] = w;
      line[2 * p + 1] = b;
      if (coef) { coef[2 * (slot0 + p)] = w; coef[2 * (slot0 + p) + 1] = b; }
      if (iters) iters[slot0 + p] = n_it;
    }
  }
  for (int p = np + t; p < cs; p += kSapThreads) {
    if (coef) { coef[2 * (slot0 + p)] = CUDART_NAN; coef[2 * (slot0 + p) + 1] = CUDART_NAN; }
    if (iters) iters[slot0 + p] = 0;
  }
  __syncthreads();

  // predictions: argmax over the classes of w x + b (lowest class on a tie), or the sign for two classes; the
  // products and sums are rounded separately (no fma), as a plain fp64 restatement computes them
  int correct = 0;
  for (int j = t; j < n_test; j += kSapThreads) {
    const double xj = (double)mu[test_rows[j] * (long long)rs + col];
    int pred = 0;
    if (binary) {
      pred = __dadd_rn(__dmul_rn(line[0], xj), line[1]) > 0.0 ? 1 : 0;
    } else if (nc > 2) {
      double best = __dadd_rn(__dmul_rn(line[0], xj), line[1]);
      for (int c = 1; c < nc; ++c) {
        const double v = __dadd_rn(__dmul_rn(line[2 * c], xj), line[2 * c + 1]);
        if (v > best) { best = v; pred = c; }
      }
    }
    correct += pred == test_cls[(long long)k * n_test + j];
  }
  correct = warp_sum(correct);
  if (lane == 0) wcount[warp] = correct;
  __syncthreads();
  if (t == 0) {
    int total = 0;
    for (int w = 0; w < kSapWarps; ++w) total += wcount[w];
    score[cell] = (float)((double)total / (double)n_test);
  }
}

}  // namespace
}  // namespace dv

using namespace dv;

extern "C" {

int dv_sap_score_matrix(const float* mu, int ld, int row_stride, int N, int D, const long long* train_rows,
                        int num_train, const long long* test_rows, int num_test, const int* train_cls,
                        const int* test_cls, const int* n_classes, const int* counts, int K, int class_stride,
                        double C, float* score, double* coef, int* iters, void* stream) {
  if (N < 1 || D < 1 || D > kSapMaxD || num_train < 1 || num_train > kSapMaxTrain || num_test < 1 || K < 1 ||
      class_stride < 1 || class_stride > kSapMaxClasses || (long long)D * K > 0x7fffffffLL || ld < 1 ||
      row_stride < 1)
    return DV_ERR_BAD_SHAPE;
  if (!mu || !train_rows || !test_rows || !train_cls || !test_cls || !n_classes || !counts || !score)
    return DV_ERR_BAD_ARG;
  if (!(C > 0.0) || !isfinite(C)) return DV_ERR_BAD_ARG;
  if (misaligned(mu, 4) || misaligned(train_rows, 8) || misaligned(test_rows, 8) || misaligned(train_cls, 4) ||
      misaligned(test_cls, 4) || misaligned(n_classes, 4) || misaligned(counts, 4) || misaligned(score, 4) ||
      misaligned(coef, 8) || misaligned(iters, 4))
    return DV_ERR_BAD_ARG;
  static bool attr = false;
  const int rc = set_max_dynamic_smem(sap_kernel, (int)sap_smem_bytes(kSapMaxTrain), &attr);
  if (rc != DV_OK) return rc;
  sap_kernel<<<D * K, kSapThreads, sap_smem_bytes(num_train), as_stream(stream)>>>(
      mu, ld, row_stride, D, train_rows, num_train, test_rows, num_test, train_cls, test_cls, n_classes, counts, K,
      class_stride, C, score, coef, iters);
  return check_launch();
}

}  // extern "C"

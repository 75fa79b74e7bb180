// beta-VAE score (Higgins et al. 2017, section 3): the point features and the logistic-regression fit.  The reference
// has no such score; the entry points are declared in include/disvae_b200.h.
//
// dv_pair_abs_diff_mean: x[v][d] = (sum_l |mu[a_vl][d] - mu[b_vl][d]|) / L, one thread per (v, d), the L terms added
// in ascending l in fp64 (an in-order fp64 sum gives the same bits).
//
// dv_logistic_fit: the exact minimiser of what sklearn's LogisticRegression(C=1) minimises on the first num_train
// rows of x, then the predicted class of every row.  With R parameter rows theta = (W [R][D], b [R]):
//   nc > 2 (multinomial, R = nc):  f = 1/2 |W|^2 + sum_i (logsumexp_r z_ir - z_{i,y_i}),         z_ir = W_r x_i + b_r
//   nc = 2 (binary, R = 1):        f = 1/2 |w|^2 + sum_i (logsumexp(0, z_i) - [y_i = 1] z_i)
// (the binary loss is the multinomial one with class 0's logit pinned at 0).  Both are solved the same way, in fp64:
//   - The features are centred on their training mean m, an exact change of variables because b is unpenalised
//     (b = b' - W m afterwards); it keeps features far from zero from coupling the intercept to the weights.
//   - Truncated Newton: preconditioned conjugate gradient on Hessian-vector products H v = v_W + sum_i q_i(v) x~_i^T
//     (q_ir = p_ir (u_ir - sum_s p_is u_is), u_i = V x~_i; p(1-p) u for binary), with the Hessian's diagonal as the
//     preconditioner, stopped at |r| <= min(0.5, sqrt(|g| / |g_0|)) |g|; then an Armijo backtracking line search,
//     except that a full step promising a decrease below 1e-12 |f| (beneath f's rounding) is taken whole.
//   - For nc > 2 f is flat along "add a constant to every b_r", so every gradient, product and preconditioned
//     residual has its b part projected onto sum_r b_r = 0, and the solution is reported with sum_r b_r = 0.
//   - Converged when max_j |g_j| <= 1e-10 * max_j s_j, s_j = [j a weight] |theta_j| + sum_i |q_ir x~_id|: the scale of
//     the gradient's parts, as dv_sap.cu measures it.  At most 100 Newton steps; otherwise iters = -1.
// One CTA does the whole fit.  Row sums over the training rows go through fixed row segments and a fixed-order sum
// of the segments; block sums add the warps in order.  No floating-point atomics: results are bit-identical run to
// run.  Vectors and per-row values live in the caller's workspace.  The solver itself is in dv_logistic.cuh, which
// dv_explicitness_fit (dv_modularity.cu) shares.
#include "dv_logistic.cuh"

namespace dv {
namespace {

constexpr int kFitMaxClasses = 32;            // dv_logistic_fit's K
constexpr int kPairThreads = 256;

__global__ void __launch_bounds__(kPairThreads)
pair_abs_diff_mean_kernel(const float* __restrict__ mu, int ld, int rs, int D, const long long* __restrict__ rows_a,
                          const long long* __restrict__ rows_b, int V, int L, double* __restrict__ x) {
  const long long j = (long long)blockIdx.x * kPairThreads + threadIdx.x;
  if (j >= (long long)V * D) return;
  const int v = (int)(j / D), d = (int)(j % D);
  const long long* ra = rows_a + (long long)v * L;
  const long long* rb = rows_b + (long long)v * L;
  const long long col = (long long)d * ld;
  double s = 0.0;
  for (int l = 0; l < L; ++l) {
    const double a = (double)mu[ra[l] * (long long)rs + col];
    const double b = (double)mu[rb[l] * (long long)rs + col];
    s = __dadd_rn(s, fabs(__dsub_rn(a, b)));
  }
  x[j] = __ddiv_rn(s, (double)L);
}

__global__ void __launch_bounds__(kFitThreads, 1)
logistic_fit_kernel(const double* __restrict__ x, int D, int num_train, int num_eval, const int* __restrict__ labels,
                    const int* __restrict__ n_classes, int K, double* __restrict__ coef, int* __restrict__ pred,
                    int* __restrict__ iters, double* __restrict__ ws) {
  const int t = threadIdx.x;
  const int nc = min(max(n_classes[0], 1), K);
  const int R = nc > 2 ? nc : (nc == 2 ? 1 : 0);
  const bool multi = nc > 2;
  const int Dp = D + 1;
  const int rows = num_train + num_eval;
  logistic_fit_cta(x, D, num_train, labels, nc, multi, 1.0, K, coef, iters, ws);

  // predictions: argmax_r W_r x + b_r (lowest r on a tie), or class 1 when w x + b > 0; 0 for nc = 1
  for (int i = t; i < rows; i += kFitThreads) {
    const double* xi = x + (long long)i * D;
    int best_r = 0;
    double best = 0.0;
    for (int r = 0; r < R; ++r) {
      const double* w = coef + (long long)r * Dp;
      double s = w[D];
      for (int d = 0; d < D; ++d) s = fma(w[d], xi[d], s);
      if (r == 0 || s > best) { best = s; best_r = r; }
    }
    pred[i] = multi ? best_r : (best > 0.0 ? 1 : 0);
  }
}

bool fit_shape_ok(int num_train, int D, int K) {
  return num_train >= 1 && D >= 1 && D <= kFitMaxD && K >= 1 && K <= kFitMaxClasses;
}

}  // namespace
}  // namespace dv

using namespace dv;

extern "C" {

int dv_pair_abs_diff_mean(const float* mu, int ld, int row_stride, int N, int D, const long long* rows_a,
                          const long long* rows_b, int V, int L, double* x, void* stream) {
  if (N < 1 || D < 1 || V < 1 || L < 1 || (long long)V * D > 0x7fffffffLL || ld < 1 || row_stride < 1)
    return DV_ERR_BAD_SHAPE;
  if (!mu || !rows_a || !rows_b || !x) return DV_ERR_BAD_ARG;
  if (misaligned(mu, 4) || misaligned(rows_a, 8) || misaligned(rows_b, 8) || misaligned(x, 8)) return DV_ERR_BAD_ARG;
  const long long total = (long long)V * D;
  pair_abs_diff_mean_kernel<<<(unsigned)((total + kPairThreads - 1) / kPairThreads), kPairThreads, 0,
                              as_stream(stream)>>>(mu, ld, row_stride, D, rows_a, rows_b, V, L, x);
  return check_launch();
}

size_t dv_logistic_fit_workspace_bytes(int num_train, int D, int K) {
  if (!fit_shape_ok(num_train, D, K)) return 0;
  return fit_workspace_doubles(num_train, D, K) * sizeof(double);
}

int dv_logistic_fit(const double* x, int D, int num_train, int num_eval, const int* labels, const int* n_classes,
                    int K, double* coef, int* pred, int* iters, void* workspace, size_t workspace_bytes,
                    void* stream) {
  if (!fit_shape_ok(num_train, D, K) || num_eval < 0 || (long long)num_train + num_eval > 0x7fffffffLL ||
      ((long long)num_train + num_eval) * D > 0x7fffffffLL)
    return DV_ERR_BAD_SHAPE;
  if (!x || !labels || !n_classes || !coef || !pred || !iters) return DV_ERR_BAD_ARG;
  if (misaligned(x, 8) || misaligned(labels, 4) || misaligned(n_classes, 4) || misaligned(coef, 8) ||
      misaligned(pred, 4) || misaligned(iters, 4) || misaligned(workspace, 8))
    return DV_ERR_BAD_ARG;
  if (!workspace || workspace_bytes < fit_workspace_doubles(num_train, D, K) * sizeof(double))
    return DV_ERR_WORKSPACE;
  logistic_fit_kernel<<<1, kFitThreads, 0, as_stream(stream)>>>(x, D, num_train, num_eval, labels, n_classes, K, coef,
                                                                pred, iters, static_cast<double*>(workspace));
  return check_launch();
}

}  // extern "C"

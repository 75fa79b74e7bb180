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
// run.  Vectors and per-row values live in the caller's workspace.
#include <math.h>
#include <math_constants.h>

#include "dv_common.cuh"

namespace dv {
namespace {

constexpr int kFitThreads = 512;
constexpr int kFitWarps = kFitThreads / kWarp;
constexpr int kFitMaxD = 128;
constexpr int kFitMaxClasses = 32;
constexpr int kFitMaxNewton = 100;
constexpr int kFitMaxCG = 250;              // conjugate-gradient steps per Newton step
constexpr int kFitMaxHalvings = 40;
constexpr double kFitTol = 1e-10;
constexpr double kFitArmijo = 1e-4;
constexpr double kFitFlat = 1e-12;          // a full step's promised decrease f cannot resolve, relative to |f|
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

// ---- the fit -------------------------------------------------------------------------------------------------------
struct Fit {
  const double* x;      // [rows][D], the first n are the training rows
  const int* y;         // [n] class indices
  int n, D, Dp, R, O;   // Dp = D + 1, O = R * Dp parameters, parameter (r, d) at r * Dp + d (d = D: the intercept)
  bool multi;
  double* mean;         // [D]
  double *theta, *grad, *scale, *dir, *res, *zv, *pv, *hp, *trial, *diag;   // [O] each
  double *P, *Q, *U;    // [n][R]
  double* part;         // 2 * max(kFitThreads, O)
  int part_stride;
  double* red;          // shared: kFitWarps
};

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Sum (or max) over the block; every thread gets the same bits.
__device__ double block_sum(double v, double* red) {
  v = warp_sum_d(v);
  __syncthreads();
  if ((threadIdx.x & (kWarp - 1)) == 0) red[threadIdx.x / kWarp] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < kFitWarps; ++w) s += red[w];
  return s;
}
__device__ double block_max(double v, double* red) {
  v = warp_max_d(v);
  __syncthreads();
  if ((threadIdx.x & (kWarp - 1)) == 0) red[threadIdx.x / kWarp] = v;
  __syncthreads();
  double s = red[0];
  for (int w = 1; w < kFitWarps; ++w) s = fmax(s, red[w]);
  return s;
}

__device__ double dot(const Fit& F, const double* a, const double* b) {
  double s = 0.0;
  for (int o = threadIdx.x; o < F.O; o += kFitThreads) s = fma(a[o], b[o], s);
  return block_sum(s, F.red);
}

__device__ __forceinline__ double xc(const Fit& F, int i, int d) {
  return d < F.D ? F.x[(long long)i * F.D + d] - F.mean[d] : 1.0;
}

// out0[o] = sum_i w(i, r) x~_id (squared when `square`), out1[o] = sum_i |w(i, r) x~_id| (when given), o = (r, d),
// with w = W[i * R + r].  The rows are cut into S fixed segments, each summed in order by one thread, and the segments
// added in order.
__device__ void colsum(const Fit& F, const double* W, bool square, double* out0, double* out1) {
  const int O = F.O, n = F.n;
  const int S = O >= kFitThreads ? 1 : min(kFitThreads / O, n);
  const int items = S * O;
  for (int j = threadIdx.x; j < items; j += kFitThreads) {
    const int o = j % O, s = j / O, r = o / F.Dp, d = o % F.Dp;
    const int i0 = (int)((long long)s * n / S), i1 = (int)((long long)(s + 1) * n / S);
    double a0 = 0.0, a1 = 0.0;
    for (int i = i0; i < i1; ++i) {
      const double w = W[(long long)i * F.R + r], v = xc(F, i, d);
      const double t = square ? w * (v * v) : w * v;
      a0 += t;
      a1 += fabs(t);
    }
    F.part[j] = a0;
    F.part[F.part_stride + j] = a1;
  }
  __syncthreads();
  for (int o = threadIdx.x; o < O; o += kFitThreads) {
    double s0 = 0.0, s1 = 0.0;
    for (int s = 0; s < S; ++s) {
      s0 += F.part[s * O + o];
      s1 += F.part[F.part_stride + s * O + o];
    }
    out0[o] = s0;
    if (out1) out1[o] = s1;
  }
  __syncthreads();
}

// U[i][r] = V_r . x~_i (the intercept's entry times 1).
__device__ void rows_dot(const Fit& F, const double* V) {
  const long long items = (long long)F.n * F.R;
  for (long long j = threadIdx.x; j < items; j += kFitThreads) {
    const int i = (int)(j / F.R), r = (int)(j % F.R);
    const double* v = V + (long long)r * F.Dp;
    double s = v[F.D];
    for (int d = 0; d < F.D; ++d) s = fma(v[d], xc(F, i, d), s);
    F.U[j] = s;
  }
  __syncthreads();
}

// Subtract the mean of the intercept entries (nc > 2 only).
__device__ void project(const Fit& F, double* v) {
  __syncthreads();
  if (!F.multi) return;
  double m = 0.0;
  for (int r = 0; r < F.R; ++r) m += v[r * F.Dp + F.D];
  m /= F.R;
  __syncthreads();
  for (int r = threadIdx.x; r < F.R; r += kFitThreads) v[r * F.Dp + F.D] -= m;
  __syncthreads();
}

// f at V, the probabilities into P and the gradient weights p - onehot into Q.
__device__ double objective(const Fit& F, const double* V) {
  rows_dot(F, V);
  double acc = 0.0;
  for (int i = threadIdx.x; i < F.n; i += kFitThreads) {
    const int y = F.y[i];
    const double* u = F.U + (long long)i * F.R;
    double* p = F.P + (long long)i * F.R;
    double* q = F.Q + (long long)i * F.R;
    if (!F.multi) {
      const double z = u[0];
      const double lse = fmax(z, 0.0) + log1p(exp(-fabs(z)));
      const double e = exp(-fabs(z));
      const double pr = z >= 0.0 ? 1.0 / (1.0 + e) : e / (1.0 + e);
      acc += lse - (y == 1 ? z : 0.0);
      p[0] = pr;
      q[0] = pr - (y == 1 ? 1.0 : 0.0);
    } else {
      double mx = u[0];
      for (int r = 1; r < F.R; ++r) mx = fmax(mx, u[r]);
      double se = 0.0;
      for (int r = 0; r < F.R; ++r) se += exp(u[r] - mx);
      acc += mx + log(se) - u[y];
      for (int r = 0; r < F.R; ++r) {
        const double pr = exp(u[r] - mx) / se;
        p[r] = pr;
        q[r] = pr - (r == y ? 1.0 : 0.0);
      }
    }
  }
  double reg = 0.0;
  for (int o = threadIdx.x; o < F.O; o += kFitThreads)
    if (o % F.Dp != F.D) reg = fma(V[o], V[o], reg);
  return 0.5 * block_sum(reg, F.red) + block_sum(acc, F.red);
}

// grad and scale at theta, from the Q of the last `objective(theta)`.
__device__ void gradient(const Fit& F) {
  colsum(F, F.Q, false, F.grad, F.scale);
  for (int o = threadIdx.x; o < F.O; o += kFitThreads)
    if (o % F.Dp != F.D) {
      F.grad[o] += F.theta[o];
      F.scale[o] += fabs(F.theta[o]);
    }
  project(F, F.grad);
}

// hp = H v at the P of the last accepted point.
__device__ void hess_vec(const Fit& F, const double* v, double* hp) {
  rows_dot(F, v);
  for (int i = threadIdx.x; i < F.n; i += kFitThreads) {
    const double* u = F.U + (long long)i * F.R;
    const double* p = F.P + (long long)i * F.R;
    double* q = F.Q + (long long)i * F.R;
    if (!F.multi) {
      q[0] = p[0] * (1.0 - p[0]) * u[0];
    } else {
      double a = 0.0;
      for (int r = 0; r < F.R; ++r) a = fma(p[r], u[r], a);
      for (int r = 0; r < F.R; ++r) q[r] = p[r] * (u[r] - a);
    }
  }
  __syncthreads();
  colsum(F, F.Q, false, hp, nullptr);
  for (int o = threadIdx.x; o < F.O; o += kFitThreads)
    if (o % F.Dp != F.D) hp[o] += v[o];
  project(F, hp);
}

// diag = the Hessian's diagonal at P (1 where it is not positive).
__device__ void hess_diag(const Fit& F) {
  const long long items = (long long)F.n * F.R;
  for (long long j = threadIdx.x; j < items; j += kFitThreads) F.Q[j] = F.P[j] * (1.0 - F.P[j]);
  __syncthreads();
  colsum(F, F.Q, true, F.diag, nullptr);
  for (int o = threadIdx.x; o < F.O; o += kFitThreads) {
    const double h = F.diag[o] + (o % F.Dp != F.D ? 1.0 : 0.0);
    F.diag[o] = h > 0.0 ? h : 1.0;
  }
  __syncthreads();
}

// zv = diag^-1 res, projected; returns res . zv
__device__ double precondition(const Fit& F) {
  for (int o = threadIdx.x; o < F.O; o += kFitThreads) F.zv[o] = F.res[o] / F.diag[o];
  project(F, F.zv);
  return dot(F, F.res, F.zv);
}

// dir ~= -H^-1 grad by preconditioned conjugate gradient.
__device__ void newton_direction(const Fit& F, double gnorm, double gnorm0) {
  const double eta = fmin(0.5, sqrt(gnorm / gnorm0));
  for (int o = threadIdx.x; o < F.O; o += kFitThreads) {
    F.dir[o] = 0.0;
    F.res[o] = -F.grad[o];
  }
  __syncthreads();
  double rz = precondition(F);
  for (int o = threadIdx.x; o < F.O; o += kFitThreads) F.pv[o] = F.zv[o];
  __syncthreads();
  for (int j = 0; j < kFitMaxCG; ++j) {
    if (sqrt(dot(F, F.res, F.res)) <= eta * gnorm) break;
    hess_vec(F, F.pv, F.hp);
    const double php = dot(F, F.pv, F.hp);
    if (!(php > 0.0)) {
      if (j == 0)
        for (int o = threadIdx.x; o < F.O; o += kFitThreads) F.dir[o] = F.pv[o];
      __syncthreads();
      break;
    }
    const double alpha = rz / php;
    for (int o = threadIdx.x; o < F.O; o += kFitThreads) {
      F.dir[o] = fma(alpha, F.pv[o], F.dir[o]);
      F.res[o] = fma(-alpha, F.hp[o], F.res[o]);
    }
    __syncthreads();
    const double rz_new = precondition(F);
    const double beta = rz_new / rz;
    rz = rz_new;
    for (int o = threadIdx.x; o < F.O; o += kFitThreads) F.pv[o] = fma(beta, F.pv[o], F.zv[o]);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kFitThreads, 1)
logistic_fit_kernel(const double* __restrict__ x, int D, int num_train, int num_eval, const int* __restrict__ labels,
                    const int* __restrict__ n_classes, int K, double* __restrict__ coef, int* __restrict__ pred,
                    int* __restrict__ iters, double* __restrict__ ws) {
  __shared__ double red[kFitWarps];
  const int t = threadIdx.x;
  const int nc = min(max(n_classes[0], 1), K);
  const int R = nc > 2 ? nc : (nc == 2 ? 1 : 0);
  const int Dp = D + 1;
  const int rows = num_train + num_eval;
  for (int o = t; o < K * Dp; o += kFitThreads) coef[o] = CUDART_NAN;
  if (R == 0) {
    for (int i = t; i < rows; i += kFitThreads) pred[i] = 0;
    if (t == 0) *iters = 0;
    return;
  }
  __syncthreads();

  __shared__ Fit F;                             // the layout, read from shared memory rather than held in registers
  if (t == 0) {
    F.x = x;
    F.y = labels;
    F.n = num_train;
    F.D = D;
    F.Dp = Dp;
    F.R = R;
    F.O = R * Dp;
    F.multi = nc > 2;
    const int OK = K * Dp;                        // vectors are laid out for the largest R, so the layout is fixed
    F.part_stride = max(kFitThreads, OK);
    F.mean = ws;
    double* v = ws + D;
    F.theta = v;
    F.grad = v + OK;
    F.scale = v + 2 * OK;
    F.dir = v + 3 * OK;
    F.res = v + 4 * OK;
    F.zv = v + 5 * OK;
    F.pv = v + 6 * OK;
    F.hp = v + 7 * OK;
    F.trial = v + 8 * OK;
    F.diag = v + 9 * OK;
    v += 10 * OK;
    F.P = v;
    F.Q = v + (long long)num_train * K;
    F.U = v + 2LL * num_train * K;
    F.part = v + 3LL * num_train * K;
    F.red = red;
  }
  __syncthreads();

  // training means: each d's rows added in order, by segments as in colsum
  {
    const int S = D >= kFitThreads ? 1 : min(kFitThreads / D, num_train);
    for (int j = t; j < S * D; j += kFitThreads) {
      const int d = j % D, s = j / D;
      const int i0 = (int)((long long)s * num_train / S), i1 = (int)((long long)(s + 1) * num_train / S);
      double a = 0.0;
      for (int i = i0; i < i1; ++i) a += x[(long long)i * D + d];
      F.part[j] = a;
    }
    __syncthreads();
    for (int d = t; d < D; d += kFitThreads) {
      double a = 0.0;
      for (int s = 0; s < S; ++s) a += F.part[s * D + d];
      F.mean[d] = a / num_train;
    }
    for (int o = t; o < F.O; o += kFitThreads) F.theta[o] = 0.0;
    __syncthreads();
  }

  double f = objective(F, F.theta);
  gradient(F);
  const double gnorm0 = sqrt(dot(F, F.grad, F.grad));
  int steps = -1;
  for (int it = 0; it <= kFitMaxNewton; ++it) {
    double gmax = 0.0, smax = 0.0;
    for (int o = t; o < F.O; o += kFitThreads) {
      gmax = fmax(gmax, fabs(F.grad[o]));
      smax = fmax(smax, F.scale[o]);
    }
    gmax = block_max(gmax, red);
    smax = block_max(smax, red);
    if (gmax <= kFitTol * smax) {
      steps = it;
      break;
    }
    if (it == kFitMaxNewton) break;
    hess_diag(F);
    newton_direction(F, sqrt(dot(F, F.grad, F.grad)), gnorm0);
    const double slope = dot(F, F.grad, F.dir);
    if (!(slope < 0.0)) break;
    // A full step that promises less than kFitFlat |f| of decrease is below what f's rounding can rank: f's noise
    // would reject it and admit a needlessly short step instead, and the fit would stall just short of the gradient
    // test (as on separable data with large margins).  Such a step is taken whole, and the gradient test decides.
    const bool flat = -slope <= kFitFlat * fabs(f);
    bool moved = false;
    double step = 1.0;
    for (int h = 0; h <= kFitMaxHalvings; ++h, step *= 0.5) {
      for (int o = t; o < F.O; o += kFitThreads) F.trial[o] = fma(step, F.dir[o], F.theta[o]);
      __syncthreads();
      const double ft = objective(F, F.trial);
      // sufficient decrease, or a change of f below its rounding (where only the gradient test can decide)
      if (flat || ft - f <= kFitArmijo * step * slope + 1e-15 * fabs(f)) {
        for (int o = t; o < F.O; o += kFitThreads) F.theta[o] = F.trial[o];
        __syncthreads();
        f = ft;
        moved = true;
        break;
      }
    }
    if (!moved) break;
    gradient(F);
  }

  // back to uncentred features: b_r = b'_r - W_r . m, then sum_r b_r = 0 for nc > 2
  for (int r = t; r < R; r += kFitThreads) {
    const double* w = F.theta + (long long)r * Dp;
    double s = 0.0;
    for (int d = 0; d < D; ++d) s = fma(w[d], F.mean[d], s);
    F.trial[r] = w[D] - s;
  }
  __syncthreads();
  double bmean = 0.0;
  if (F.multi) {
    for (int r = 0; r < R; ++r) bmean += F.trial[r];
    bmean /= R;
  }
  for (int o = t; o < F.O; o += kFitThreads) {
    const int r = o / Dp, d = o % Dp;
    coef[o] = d < D ? F.theta[o] : F.trial[r] - bmean;
  }
  __syncthreads();

  // predictions: argmax_r W_r x + b_r (lowest r on a tie), or class 1 when w x + b > 0
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
    pred[i] = F.multi ? best_r : (best > 0.0 ? 1 : 0);
  }
  if (t == 0) *iters = steps;
}

bool misaligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0; }

size_t fit_workspace_doubles(int num_train, int D, int K) {
  const size_t OK = (size_t)K * (D + 1);
  return (size_t)D + 10 * OK + 3 * (size_t)num_train * K + 2 * (OK > (size_t)kFitThreads ? OK : kFitThreads);
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

// The fp64 logistic-regression solver shared by dv_logistic_fit (dv_beta_vae_score.cu) and dv_explicitness_fit
// (dv_modularity.cu) at C = 1, and by dv_downstream_logistic_cv (dv_downstream.cu) at every C of its grid: the exact
// minimiser of sklearn's LogisticRegression(C) objective C sum_i loss_i + 1/2 |W|^2, one CTA of kFitThreads threads per
// fit.  The objective, the method and the rules of the solve are described at the top of dv_beta_vae_score.cu and in
// include/disvae_b200.h.  C multiplies each row sum once, so at C = 1 every operation rounds as it did without it.
#pragma once

#include <math.h>
#include <math_constants.h>

#include "dv_common.cuh"

namespace dv {
namespace {

constexpr int kFitThreads = 512;
constexpr int kFitWarps = kFitThreads / kWarp;
constexpr int kFitMaxD = 128;
constexpr int kFitMaxNewton = 100;
constexpr int kFitMaxCG = 250;              // conjugate-gradient steps per Newton step
constexpr int kFitMaxHalvings = 40;
constexpr double kFitTol = 1e-10;
constexpr double kFitArmijo = 1e-4;
constexpr double kFitFlat = 1e-12;          // a full step's promised decrease f cannot resolve, relative to |f|

// ---- the fit -------------------------------------------------------------------------------------------------------
struct Fit {
  const double* x;      // [rows][D], the first n are the training rows
  const int* y;         // [n] class indices
  int n, D, Dp, R, O;   // Dp = D + 1, O = R * Dp parameters, parameter (r, d) at r * Dp + d (d = D: the intercept)
  bool multi;
  double C;             // the weight of the loss against 1/2 |W|^2
  double* mean;         // [D]
  double *theta, *grad, *scale, *dir, *res, *zv, *pv, *hp, *trial, *diag;   // [O] each
  double *P, *Q, *U;    // [n][R]
  double* part;         // 2 * max(kFitThreads, O)
  int part_stride;
  double* red;          // shared: kFitWarps
};

__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Max over the block; every thread gets the same bits.
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
  return block_sum<kFitWarps>(s, F.red);
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

// Subtract the mean of the intercept entries (multinomial fits only).
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
  return 0.5 * block_sum<kFitWarps>(reg, F.red) + F.C * block_sum<kFitWarps>(acc, F.red);
}

// grad and scale at theta, from the Q of the last `objective(theta)`.
__device__ void gradient(const Fit& F) {
  colsum(F, F.Q, false, F.grad, F.scale);
  for (int o = threadIdx.x; o < F.O; o += kFitThreads) {
    F.grad[o] *= F.C;
    F.scale[o] *= F.C;
    if (o % F.Dp != F.D) {
      F.grad[o] += F.theta[o];
      F.scale[o] += fabs(F.theta[o]);
    }
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
  for (int o = threadIdx.x; o < F.O; o += kFitThreads) {
    hp[o] *= F.C;
    if (o % F.Dp != F.D) hp[o] += v[o];
  }
  project(F, hp);
}

// diag = the Hessian's diagonal at P (1 where it is not positive).
__device__ void hess_diag(const Fit& F) {
  const long long items = (long long)F.n * F.R;
  for (long long j = threadIdx.x; j < items; j += kFitThreads) F.Q[j] = F.P[j] * (1.0 - F.P[j]);
  __syncthreads();
  colsum(F, F.Q, true, F.diag, nullptr);
  for (int o = threadIdx.x; o < F.O; o += kFitThreads) {
    const double h = F.C * F.diag[o] + (o % F.Dp != F.D ? 1.0 : 0.0);
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

// dir ~= -H^-1 grad by preconditioned conjugate gradient, at most kMaxCG steps.
template <int kMaxCG>
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
  for (int j = 0; j < kMaxCG; ++j) {
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

// One fit by the whole CTA: the minimiser of C sum_i loss_i + 1/2 |W|^2 for the nc classes of `labels` [num_train]
// on the first num_train rows of x [rows][D], multinomial over R = nc model rows when `multi`, else one binary model
// (nc = 2, R = 1), into coef [K][D + 1] (row r = (W_r, b_r) for the uncentred features, NaN beyond the R rows; R = 0
// for nc < 2) and *iters (Newton steps, -1 if kMaxNewton did not converge, 0 for nc < 2).  The existing fits call it
// with C = 1 and multi = nc > 2.  ws holds fit_workspace_doubles(num_train, D, K) doubles.  Every thread of the CTA
// calls it with the same arguments; it ends with the coefficients visible to the whole CTA.
template <int kMaxNewton = kFitMaxNewton, int kMaxCG = kFitMaxCG>
__device__ void logistic_fit_cta(const double* __restrict__ x, int D, int num_train, const int* __restrict__ labels,
                                 int nc, bool multi, double C, int K, double* __restrict__ coef,
                                 int* __restrict__ iters, double* __restrict__ ws) {
  __shared__ double red[kFitWarps];
  const int t = threadIdx.x;
  const int R = nc < 2 ? 0 : (multi ? nc : 1);
  const int Dp = D + 1;
  for (int o = t; o < K * Dp; o += kFitThreads) coef[o] = CUDART_NAN;
  if (R == 0) {
    if (t == 0) *iters = 0;
    __syncthreads();
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
    F.multi = multi;
    F.C = C;
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
  for (int it = 0; it <= kMaxNewton; ++it) {
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
    if (it == kMaxNewton) break;
    hess_diag(F);
    newton_direction<kMaxCG>(F, sqrt(dot(F, F.grad, F.grad)), gnorm0);
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

  // back to uncentred features: b_r = b'_r - W_r . m, then sum_r b_r = 0 for a multinomial fit
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
  if (t == 0) *iters = steps;
}

size_t fit_workspace_doubles(int num_train, int D, int K) {
  const size_t OK = (size_t)K * (D + 1);
  return (size_t)D + 10 * OK + 3 * (size_t)num_train * K + 2 * (OK > (size_t)kFitThreads ? OK : kFitThreads);
}

}  // namespace
}  // namespace dv

// FactorVAE disentanglement score (Kim & Mnih 2018, section 4): per-group unbiased variances of gathered rows of the
// encoder means, and for the votes the argmin of those variances over the global ones.  The reference has no such
// score; the entry point is declared in include/disvae_b200.h.
//
//   group g = rows[g][0 .. L-1],  s = mu[rows[g][0]][d] (the group's first row)
//   r       = mean_l (mu[rows[g][l]][d] - s)
//   var[d]  = sum_l ((mu[rows[g][l]][d] - s) - r)^2 / (L - 1)
//   vote    = argmin over d with global_var[d] >= min_var and var[d] / global_var[d] not NaN of that ratio, lowest d
//             on a tie, -1 if no dim qualifies
//
// The two-pass form around s keeps a column far from zero (means near 100, spread 0.01) at full precision: the
// differences from s are exact in fp32 near s.  Since s is a row of the group, |s - mean| is at most about sqrt(L)
// times the group's spread, so the shift costs at most that factor in the rounding of r and of the squares.
//
// One CTA per (group, slice of dims).  Its 256 threads are `lanes` row lanes x `dt` dim lanes (dt a power of two, at
// most 32, the dims fastest so a warp reads whole runs of a row); row lane j sums rows j, j + lanes, ... in order and a
// fixed tree over the lanes adds the partials.  When votes are asked for, the CTA walks every dim of its group (the
// variances stay in shared memory for the argmin); otherwise the dims are spread over gridDim.y.  dt shrinks until the
// grid has about 2 CTAs per SM, so the one long group of the global estimate still spreads over the GPU.  Every sum has
// a fixed order and there are no floating-point atomics: results are bit-identical run to run.
#include "dv_common.cuh"

namespace dv {
namespace {

constexpr int kFsThreads = 256;
constexpr int kFsMaxD = 1024;

struct FsPlan {
  int dt, slices;
};

FsPlan fs_plan(int D, int V, bool votes) {
  int dt = 1;
  while (dt < D && dt < kWarp) dt <<= 1;
  while (dt > 1 && (long long)V * ((D + dt - 1) / dt) < 2LL * kNumSMs) dt >>= 1;
  FsPlan p;
  p.dt = dt;
  p.slices = votes ? 1 : (D + dt - 1) / dt;
  return p;
}

// Fixed-order tree over the row lanes of red[lanes][dt]; the total lands in red[0][dim lane].
__device__ __forceinline__ void fs_lane_tree(float* red, int lane, int dl, int dt, int lanes) {
  for (int h = lanes >> 1; h > 0; h >>= 1) {
    __syncthreads();
    if (lane < h) red[lane * dt + dl] += red[(lane + h) * dt + dl];
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kFsThreads)
fs_group_var_kernel(const float* __restrict__ mu, int ld, int rs, int D, const long long* __restrict__ rows, int L,
                    int dt, const float* __restrict__ global_var, float min_var, float* __restrict__ var_out,
                    int* __restrict__ argmin_out) {
  __shared__ float red[kFsThreads];
  __shared__ float sv[kFsMaxD];
  __shared__ float bval[kFsThreads / kWarp];
  __shared__ int bidx[kFsThreads / kWarp];
  const int t = threadIdx.x, lanes = kFsThreads / dt, lane = t / dt, dl = t % dt;
  const long long g = blockIdx.x;
  const long long* grow = rows + g * L;
  const long long r0 = grow[0] * (long long)rs;

  for (int d0 = blockIdx.y * dt; d0 < D; d0 += gridDim.y * dt) {
    const int d = d0 + dl;
    const bool on = d < D;
    const long long col = (long long)(on ? d : 0) * ld;
    const float s = mu[r0 + col];
    float acc = 0.f;
#pragma unroll 4
    for (int l = lane; l < L; l += lanes) acc += mu[grow[l] * (long long)rs + col] - s;
    red[t] = acc;
    fs_lane_tree(red, lane, dl, dt, lanes);
    const float r = red[dl] / (float)L;
    __syncthreads();                                  // every lane has read red[dl] before it is overwritten
    acc = 0.f;
#pragma unroll 4
    for (int l = lane; l < L; l += lanes) {
      const float c = (mu[grow[l] * (long long)rs + col] - s) - r;
      acc = fmaf(c, c, acc);
    }
    red[t] = acc;
    fs_lane_tree(red, lane, dl, dt, lanes);
    if (lane == 0 && on) {
      const float v = red[dl] / (float)(L - 1);
      if (var_out) var_out[g * D + d] = v;
      if (argmin_out) sv[d] = v;
    }
    __syncthreads();
  }
  if (!argmin_out) return;

  // argmin of var / global_var over the active dims; (value, index) order, so the lowest index wins a tie.  A NaN
  // ratio (a NaN variance, or inf / inf) does not qualify, as a NaN global variance does not: kept, it would compare
  // false against everything and drop the true minimum wherever it met it in the butterfly.
  float best = 0.f;
  int bi = -1;
  for (int d = t; d < D; d += kFsThreads) {
    const float gv = global_var[d];
    if (!(gv >= min_var)) continue;
    const float q = sv[d] / gv;
    if (isnan(q)) continue;
    if (bi < 0 || q < best) { best = q; bi = d; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (oi >= 0 && (bi < 0 || ob < best || (ob == best && oi < bi))) { best = ob; bi = oi; }
  }
  if ((t & 31) == 0) { bval[t >> 5] = best; bidx[t >> 5] = bi; }
  __syncthreads();
  if (t == 0) {
    best = bval[0];
    bi = bidx[0];
    for (int w = 1; w < kFsThreads / kWarp; ++w) {
      const int oi = bidx[w];
      const float ob = bval[w];
      if (oi >= 0 && (bi < 0 || ob < best || (ob == best && oi < bi))) { best = ob; bi = oi; }
    }
    argmin_out[g] = bi;
  }
}

}  // namespace
}  // namespace dv

using namespace dv;

extern "C" {

int dv_group_variance(const float* mu, int ld, int row_stride, int N, int D, const long long* rows, int V, int L,
                      const float* global_var, float min_var, float* var_out, int* argmin_out, void* stream) {
  if (L < 2 || V < 1 || N < 1 || D < 1 || D > kFsMaxD || ld < 1 || row_stride < 1) return DV_ERR_BAD_SHAPE;
  if (!mu || !rows || (!var_out && !argmin_out) || (argmin_out && !global_var)) return DV_ERR_BAD_ARG;
  if (misaligned(mu, 4) || misaligned(rows, 8) || misaligned(global_var, 4) || misaligned(var_out, 4) ||
      misaligned(argmin_out, 4))
    return DV_ERR_BAD_ARG;
  const FsPlan p = fs_plan(D, V, argmin_out != nullptr);
  fs_group_var_kernel<<<dim3(V, p.slices), kFsThreads, 0, as_stream(stream)>>>(
      mu, ld, row_stride, D, rows, L, p.dt, global_var, min_var, var_out, argmin_out);
  return check_launch();
}

}  // extern "C"

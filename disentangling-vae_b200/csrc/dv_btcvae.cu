// beta-TCVAE log-density decomposition: the B x B (x D) pairwise Gaussian log-density "matrix"
// of the reference and its three logsumexp reductions, evaluated without materialising anything
// larger than O(B*D).
//
// Reference: disvae/models/losses.py:523-544 (_get_log_pz_qz_prodzi_qzCx), :369-373 (mi/tc/dw_kl),
//            disvae/utils/math.py:8-51 (matrix_log_density_gaussian), :54-73 (importance weights).
//
//   m[i,j,d] = -0.5*(log 2pi + lv[j,d]) - 0.5*(z[i,d]-mu[j,d])^2 * exp(-lv[j,d])
//   lw[i,j]  = log W[i,j]  (MSS; column-structured, trap T3)     or 0 (is_mss = False, trap T4)
//   log_qz[i]       = LSE_j ( sum_d m[i,j,d] + D*lw[i,j] )        (trap T2: D-fold weight)
//   log_prod_qzi[i] = sum_d LSE_j ( m[i,j,d] + lw[i,j] )
//
// Two forward paths (both without anything larger than O(B*D) in memory), one backward:
//   * btcvae_fwd4_kernel  -- D <= 16, the whole batch: ONE launch, clusters of 4 CTAs (columns split over the cluster,
//     partial logsumexp states merged through distributed shared memory).  BASELINE configs[1] runs here.
//   * btcvae_prep_kernel + btcvae_fwd2_kernel + btcvae_finalize_kernel -- any D, any row window [row0, row0+nrows) of
//     the batch (z = 64 of configs[4]; the global-batch estimator over an all-gathered batch, SURVEY.md 8f-1):
//     (row group x column range) tiles with per-tile reference exponents, merged in a fixed order.
//   * btcvae_bwd_kernel   -- rows role (g_z) and columns role (g_mu, g_logvar), same row-window semantics.
// All exponent arithmetic is done in the log2 domain (c and hiv pre-multiplied by log2 e) so that each (i,j,d) costs
// one MUFU.EX2 and no extra multiply; cross-lane merges are warp shuffles; every reduction has a fixed order.
#include <cooperative_groups.h>
#include "dv_common.cuh"

namespace dv {

constexpr float kLog2Pi = 1.8378770664093453f;
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
constexpr int kRows = 4;          // rows per warp (and per block)
constexpr int kJL = 8;            // column lanes per warp
constexpr int kBtWarps = 8;
constexpr int kWsHeader = 16;     // floats before the float4 array (keeps it 64-byte aligned)

struct LogW { float ln, ls, lm; int mss; int B; };   // log2 of 1/N, strat, 1/M
__device__ __forceinline__ float logw2(const LogW& w, int i, int j) {
  if (!w.mss) return 0.f;
  if (j == 0) return (i == w.B - 2) ? w.ls : w.ln;
  return (j == 1) ? w.ls : w.lm;
}

// A row's own Gaussian terms of one latent dim (natural-log units), added to the row's sums.
__device__ __forceinline__ void add_row_gauss(float zz, float m, float lv, float& lq, float& lp) {
  const float t = zz - m;
  lq += -0.5f * (kLog2Pi + lv) - 0.5f * (t * t * expf(-lv));   // log N(z; mu, lv)   (math.py:48-51)
  lp += -0.5f * kLog2Pi - 0.5f * (zz * zz);                      // log N(z; 0, 1)     (losses.py:531-532)
}

// rowstats is a structure of arrays [4 + D][B]: log_pz, log_qz, log_prod_qzi, log_q_zCx, P[d]
// (natural-log units).  pj[d][b] = { c*log2e, hiv*log2e, mu, z } of batch row b.
__global__ void btcvae_prep_kernel(const float* __restrict__ z, const float* __restrict__ mu, const float* __restrict__ logvar,
                                   int ld, int row_stride, int B, int D, float4* __restrict__ pj, float* __restrict__ rowstats) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= B) return;
  float lq = 0.f, lp = 0.f;
  for (int d = lane; d < D; d += 32) {
    const float m = mu[(long long)row * row_stride + (long long)d * ld];
    const float lv = logvar[(long long)row * row_stride + (long long)d * ld];
    const float zz = z[(long long)row * D + d];
    const float cc = -0.5f * (kLog2Pi + lv);
    const float iv = expf(-lv);
    pj[(long long)d * B + row] = make_float4(cc * kLog2e, 0.5f * iv * kLog2e, m, zz);
    add_row_gauss(zz, m, lv, lq, lp);
  }
  lq = warp_sum(lq); lp = warp_sum(lp);
  if (lane == 0) { rowstats[row] = lp; rowstats[3LL * B + row] = lq; }
}

// merge of (max, sum) logsumexp states, log2 domain
__device__ __forceinline__ void lse_merge2(float& m, float& s, float m2, float s2) {
  if (s2 == 0.f) return;                                        // empty / fully underflowed state: identity
  if (s == 0.f) { m = m2; s = s2; return; }
  const float nm = fmaxf(m, m2);
  if (nm == -INFINITY) { s = 0.f; return; }
  s = s * exp2f(m - nm) + s2 * exp2f(m2 - nm);
  m = nm;
}

// ------------------------------------------------------------------------------------------
// Forward for any D and any row window: (row-group x column-range) tiling.
// A block owns 32 rows (8 warps x 4 rows; the 8 lanes of a row split the columns) and ONE column range
// of kJT columns whose parameters are staged once in shared memory (10 KB at D=10, kJT=64), so every
// row of the block reads them from shared memory with conflict-free 128-bit loads instead of from L2.
// A block emits partial logsumexp states (max, sum) per (row, dim) for its column range;
// btcvae_finalize_kernel merges the ranges in a fixed order, forms the row statistics and the three
// means.  Grid: (nrows/32) x (B/kJT).
// ------------------------------------------------------------------------------------------
// JT = columns per block: 64 (8 per lane), or 16 (2 per lane) when (rows/32) x (B/64) blocks would leave most SMs idle
// (B = 256: 32 blocks -> 128).
constexpr int kJTBig = 64, kJTSmall = 16;
constexpr int kRG = 32;            // rows per block

// Single sweep: instead of a max pass, every (row, dim) of a block uses the reference exponent
//   ref = max( upper bound of the block's columns - 60,  the diagonal term if column i is in the block )
// (log2 units).  The bound max_j (c_j + w_j) >= every term, so exp2(term - ref) <= 2^60 never overflows;
// the diagonal term (always part of the sum) keeps the row's total from underflowing; a block whose terms
// all underflow against its own bound contributes (ref, 0), which the merge treats as the identity -- such
// terms are < 2^-66 of the block bound and, unless row i is an outlier, far below the diagonal term.  When every term
// of a (row, dim) underflows, diagonal included, btcvae_finalize_kernel redoes it exactly.
// One MUFU.EX2, ~8 FP32 ops per (i,j,d).
template <int DC, bool EXACT, int kJT>
__global__ void __launch_bounds__(kBtWarps * 32)
btcvae_fwd2_kernel(int B, int D, int row0, int nrows, LogW lw, const float4* __restrict__ pj, float2* __restrict__ part) {
  constexpr int kJPL = kJT / kJL;    // columns per lane
  __shared__ float4 sp[DC][kJT];
  __shared__ float sbound[DC];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = lane >> 3, jl = lane & 7;
  const int i_raw = row0 + blockIdx.x * kRG + warp * kRows + r;       // rows [row0, row0 + nrows) of the global batch
  const int row_end = row0 + nrows;
  const int i = min(i_raw, row_end - 1);
  const int js = blockIdx.y;
  const int j0 = js * kJT;
  const float Df = (float)D;
  const float w_col0_max = lw.mss ? fmaxf(lw.ln, lw.ls) : 0.f;
  float sa[kJPL], wj[kJPL];
#pragma unroll
  for (int t = 0; t < kJPL; ++t) { sa[t] = 0.f; wj[t] = logw2(lw, i, j0 + jl + kJL * t); }

  for (int d0 = 0; d0 < D; d0 += DC) {
    const int nd = EXACT ? DC : min(DC, D - d0);
    if (d0 > 0) __syncthreads();                              // previous chunk fully consumed
    for (int e = threadIdx.x; e < nd * kJT; e += blockDim.x) {
      const int k = e / kJT, jj = e % kJT;
      const int j = min(j0 + jj, B - 1);
      sp[k][jj] = __ldg(pj + (long long)(d0 + k) * B + j);
    }
    __syncthreads();
    // per-dimension upper bound over this block's columns: 8 lanes scan 8 columns each
    {                                                          // all threads take part (full-mask shuffles)
      const int kk = threadIdx.x >> 3, l = threadIdx.x & 7;
      const int k = min(kk, nd - 1);
      float bmax = -INFINITY;
#pragma unroll
      for (int t = 0; t < kJPL; ++t) {
        const int j = j0 + l + kJL * t;
        if (j < B) {
          const float w = !lw.mss ? 0.f : (j == 0 ? w_col0_max : (j == 1 ? lw.ls : lw.lm));
          bmax = fmaxf(bmax, sp[k][l + kJL * t].x + w);
        }
      }
#pragma unroll
      for (int o = 1; o < 8; o <<= 1) bmax = fmaxf(bmax, __shfl_xor_sync(0xffffffffu, bmax, o));
      if (l == 0 && kk < nd) sbound[kk] = bmax;
    }
    __syncthreads();
    float zc[DC], ref[DC], sx[DC];
    const bool diag_here = (i >= j0 && i < j0 + kJT);
#pragma unroll
    for (int k = 0; k < DC; ++k) {
      sx[k] = 0.f;
      if (EXACT || k < nd) {
        zc[k] = __ldg(&pj[(long long)(d0 + k) * B + i].w);
        float rf = sbound[k] - 60.f;
        if (diag_here) {
          const float4 p = sp[k][i - j0];
          const float tt = zc[k] - p.z;
          rf = fmaxf(rf, p.x - p.y * (tt * tt) + logw2(lw, i, i));
        }
        ref[k] = rf;
      } else { zc[k] = 0.f; ref[k] = 0.f; }
    }
#pragma unroll
    for (int t = 0; t < kJPL; ++t) {
      if (j0 + jl + kJL * t < B) {
#pragma unroll
        for (int k = 0; k < DC; ++k) {
          if (EXACT || k < nd) {
            const float4 p = sp[k][jl + kJL * t];
            const float tt = zc[k] - p.z;
            const float m = p.x - p.y * (tt * tt);
            sa[t] += m;
            sx[k] += exp2f(m + (wj[t] - ref[k]));
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < DC; ++k) {
#pragma unroll
      for (int o = 1; o < kJL; o <<= 1) sx[k] += __shfl_xor_sync(0xffffffffu, sx[k], o);
      if (jl == 0 && i_raw < row_end && (EXACT || k < nd))
        part[((long long)js * (D + 1) + d0 + k) * B + i] = make_float2(ref[k], sx[k]);
    }
  }
  // log_qz partial: logsumexp over this block's columns of (sum_d m + D*lw)
  float am = -INFINITY, as = 0.f;
#pragma unroll
  for (int t = 0; t < kJPL; ++t) {
    if (j0 + jl + kJL * t < B) {
      const float a = sa[t] + Df * wj[t];
      const float nm = fmaxf(am, a);
      as = as * exp2f(am - nm) + exp2f(a - nm);
      am = nm;
    }
  }
#pragma unroll
  for (int o = 1; o < kJL; o <<= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, am, o), s2 = __shfl_xor_sync(0xffffffffu, as, o);
    lse_merge2(am, as, m2, s2);
  }
  if (jl == 0 && i_raw < row_end) part[((long long)js * (D + 1) + D) * B + i] = make_float2(am, as);
}

// Exact two-pass logsumexp_j (m[i,j,d] + lw[i,j]) in log2 units, from the column parameters pjd = pj[d][.].
__device__ __forceinline__ float exact_lse2(int B, int i, const float4* __restrict__ pjd, LogW lw) {
  const float zi = pjd[i].w;
  auto term = [&](int j) {
    const float4 p = pjd[j];
    const float t = zi - p.z;
    return p.x - p.y * (t * t) + logw2(lw, i, j);
  };
  float mx = -INFINITY;
  for (int j = 0; j < B; ++j) mx = fmaxf(mx, term(j));
  float s = 0.f;
  for (int j = 0; j < B; ++j) s += exp2f(term(j) - mx);
  return mx + log2f(s);
}

// merge the column ranges in a fixed order: 16 lanes per row (lane l owns dims l, l+16, ... and lane
// D%16.. the log_qz slot), rowstats rows 1, 2, 4.. written per row; the last block forms the three means.
// A (row, dim) whose terms all lie far below its blocks' reference exponents (an outlier sample) has lost them to
// exp2f's underflow, the diagonal one included; a merged value more than 90 log2 units below the largest block
// reference (or no value at all) is redone exactly from pj.  Terms flushed against a reference are < 2^-126 of it,
// so a merged value above that bar has lost at most B * 2^-36 of itself.
__global__ void __launch_bounds__(256)
btcvae_finalize_kernel(int B, int D, int row0, int nrows, int JS, LogW lw, const float4* __restrict__ pj,
                       const float2* __restrict__ part, float* __restrict__ rowstats, float* __restrict__ terms,
                       unsigned* __restrict__ counter) {
  __shared__ bool is_last;
  const int gl = threadIdx.x & 15;
  const int i = row0 + blockIdx.x * 16 + (threadIdx.x >> 4);
  const int row_end = row0 + nrows;
  float lprod = 0.f;
  if (i < row_end) {
    for (int d = gl; d <= D; d += 16) {
      float2 st = part[(long long)d * B + i];
      float m = st.x, s = st.y, mref = st.x;
      for (int js = 1; js < JS; ++js) {
        st = part[((long long)js * (D + 1) + d) * B + i];
        mref = fmaxf(mref, st.x);
        lse_merge2(m, s, st.x, st.y);
      }
      float v2 = m + log2f(s);
      if (d < D && !(v2 > mref - 90.f)) v2 = exact_lse2(B, i, pj + (long long)d * B, lw);
      const float v = v2 * kLn2;
      if (d < D) { rowstats[(long long)(4 + d) * B + i] = v; lprod += v; }
      else rowstats[1LL * B + i] = v;                         // log_qz
    }
  }
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) lprod += __shfl_xor_sync(0xffffffffu, lprod, o);
  if (i < row_end && gl == 0) rowstats[2LL * B + i] = lprod;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  __shared__ float red[3][8];
  float mi = 0.f, tc = 0.f, dw = 0.f;
  for (int r = row0 + threadIdx.x; r < row_end; r += blockDim.x) {     // means over THIS window's rows
    const float lpz = rowstats[r], lqz = rowstats[1LL * B + r], lp = rowstats[2LL * B + r], lqc = rowstats[3LL * B + r];
    mi += lqc - lqz; tc += lqz - lp; dw += lp - lpz;
  }
  mi = warp_sum(mi); tc = warp_sum(tc); dw = warp_sum(dw);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { red[0][warp] = mi; red[1][warp] = tc; red[2][warp] = dw; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b2 = 0.f, c = 0.f;
    for (int w = 0; w < 8; ++w) { a += red[0][w]; b2 += red[1][w]; c += red[2][w]; }
    terms[0] = a / (float)nrows; terms[1] = b2 / (float)nrows; terms[2] = c / (float)nrows;
    *counter = 0u;
  }
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// ------------------------------------------------------------------------------------------
// Forward for D <= 16 over the whole batch: ONE launch, thread-block CLUSTERS of 4.
//   * a cluster of 4 CTAs owns R rows; CTA c of the cluster stages only ITS QUARTER of the columns (40 KB at
//     (1024,10)) and sweeps those columns for all R rows; the four partial logsumexp states of every (row, dim) are
//     merged through distributed shared memory after one cluster barrier -- no global-memory round trip, no second
//     launch, nothing but the O(B*D) outputs touches HBM;
//   * register blocking over ROWS: a lane owns columns and applies each loaded column to RPT rows whose z_d and
//     running sums it keeps in registers, so one LDS.128 serves RPT evaluations.  An LDS.128 costs four shared-memory
//     cycles whatever the addresses, so broadcasting one column ACROSS lanes would save nothing; lanes read
//     consecutive columns instead, and the odd float4 pitch (DC + 1) keeps those reads conflict free where an even
//     pitch gives 2-way conflicts;
//   * the reference exponent is per CTA and per dimension (r_cd = max over the CTA's columns of c_jd + w_j, an
//     upper bound of every term it sums, so no ex2 and no sum can overflow), folded with the column weight into the
//     staged constant (t = z - mu; arg = x'' - hiv*t*t; a += arg; s_d += ex2(arg)); partial sums of different CTAs
//     are brought to the common exponent max_c r_cd in the merge.  log q(z): online logsumexp with one ex2 per column.
//   * for an outlier sample (its best term > 60 nats below the column bound) ex2 flushes the terms against that bound
//     to zero, so rows whose merged sum (nearly) underflows are redone exactly (two passes straight from global memory)
//     by the finalising warp.
// Rows of a cluster are finalised by its 4 CTAs round-robin (one warp per row: lanes = latent dims); the block's
// contribution to the three means goes to `blockpart`, the last block adds them in block order (deterministic).
// Clusters of 4 CTAs, rows spread over at most 32 of them (B = 1024: 32 rows per cluster).  32 is an estimate of how
// many 4-CTA clusters a 132-SM H100 holds at once (not measured); more clusters only run as a second wave.
// ------------------------------------------------------------------------------------------
constexpr int kF4Threads = 512;
constexpr int kF4Warps = kF4Threads / 32;
constexpr int kF4Clus = 4;
constexpr int kF4MaxClusters = 32;   // the rows are spread over at most this many clusters
constexpr int kF4MaxTasks = 32;      // (row group of 4) x (column split) pairs per CTA
constexpr int kF4MaxRows = 128;      // rows per cluster
constexpr int kF4MaxSmem = 200 * 1024;   // dynamic shared memory opt-in (column stage)

__device__ __forceinline__ void atomic_max_float(float* addr, float v) {   // shared memory; works for mixed signs
  if (v >= 0.f) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
  else atomicMin(reinterpret_cast<unsigned*>(addr), __float_as_uint(v));
}

// RPT = rows per thread (register blocking over rows: one LDS.128 of a column's parameters serves RPT evaluations)
template <int DC, bool EXACT, int RPT>
__global__ void __launch_bounds__(kF4Threads, 1)
btcvae_fwd4_kernel(const float* __restrict__ z, const float* __restrict__ mu, const float* __restrict__ logvar, int ld,
                   int row_stride, int B, int D_rt, LogW lw, int R, int S, int NC, float4* __restrict__ pj_out,
                   float* __restrict__ rowstats, float* __restrict__ terms, float* __restrict__ blockpart,
                   unsigned* __restrict__ counter) {
  extern __shared__ float4 sp[];                               // [NC][DC+1]: {x'', hiv*log2e, mu, z} of this CTA's columns
  constexpr int DP = DC + 1;                                   // odd pitch: lanes over consecutive columns are conflict free
  __shared__ float s_ref[DC];                                  // r_cd (log2 units); -inf if the CTA owns no column
  __shared__ float s_rsum;                                     // sum_d r_cd
  __shared__ float s_tsx[kF4MaxTasks * kRows][DC];             // per (task, row) partial sums
  __shared__ float2 s_tq[kF4MaxTasks * kRows];
  __shared__ float s_sx[kF4MaxRows][DC];                       // per row: this CTA's sum_j ex2(arg)  (read by the peers)
  __shared__ float2 s_q[kF4MaxRows];                           // per row: this CTA's log q(z) state, relative to s_rsum
  __shared__ float s_means[kF4MaxRows / kF4Clus][3];
  __shared__ bool is_last;
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int D = EXACT ? DC : D_rt;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int crank = (int)cluster.block_rank();
  const int clus = blockIdx.x / kF4Clus;
  const int c0 = crank * NC;
  const int ncols = max(0, min(B, c0 + NC) - c0);

  // ---- phase 1: this CTA's columns -> shared memory with the weight and the reference exponent folded in ----
  // thread = (latent dim k, every CPT-th column): its running max is ONE register, the block-wide r_cd one shared-memory
  // atomic per thread; the (cheap, L1/L2-resident) inputs are then read a second time to store x'' = c + w - r_cd.
  {
    if (tid < DC) s_ref[tid] = -INFINITY;
    __syncthreads();
    const int CPT = kF4Threads / D;
    const bool worker = tid < CPT * D;
    const int k = tid % D, jl0 = tid / D;
    const float col0_extra = lw.mss ? fmaxf(lw.ls - lw.ln, 0.f) : 0.f;    // column 0: the larger of its two weights
    if (worker) {
      float bm = -INFINITY;
      for (int jl = jl0; jl < ncols; jl += CPT) {
        const int j = c0 + jl;
        const float lv = logvar[(long long)j * row_stride + (long long)k * ld];
        const float w = !lw.mss ? 0.f : (j == 0 ? lw.ln + col0_extra : (j == 1 ? lw.ls : lw.lm));
        bm = fmaxf(bm, -0.5f * (kLog2Pi + lv) * kLog2e + w);
      }
      if (bm > -INFINITY) atomic_max_float(&s_ref[k], bm);
    }
    __syncthreads();
    if (worker) {
      const float ref = s_ref[k];
      for (int jl = jl0; jl < ncols; jl += CPT) {
        const int j = c0 + jl;
        const long long off = (long long)j * row_stride + (long long)k * ld;
        const float m = mu[off], lv = logvar[off], zz = z[(long long)j * D + k];
        const float cc = -0.5f * (kLog2Pi + lv) * kLog2e;
        const float hiv = 0.5f * expf(-lv) * kLog2e;
        const float w = !lw.mss ? 0.f : (j == 0 ? lw.ln : (j == 1 ? lw.ls : lw.lm));
        sp[jl * DP + k] = make_float4(cc + w - ref, hiv, m, zz);
        if (clus == 0) pj_out[(long long)k * B + j] = make_float4(cc, hiv, m, zz);   // the backward pass reads [D][B]
      }
    }
    if (tid == 0) {
      float rs = 0.f;
      for (int kk = 0; kk < D; ++kk) rs += s_ref[kk];
      s_rsum = rs;
    }
    __syncthreads();
  }

  // ---- phase 2: tasks = (group of RPT rows) x (column split); lanes = columns, RPT rows in registers ----
  {
    const int G = (R + RPT - 1) / RPT;
    const int ntasks = G * S;
    const int CS = (((NC + S - 1) / S) + 31) / 32 * 32;
    for (int task = warp; task < ntasks; task += kF4Warps) {
      const int g = task / S, s = task - g * S;
      float zc[RPT][DC], sx[RPT][DC], am[RPT], as[RPT], dw0[RPT];
#pragma unroll
      for (int r = 0; r < RPT; ++r) {
        const int i = min(clus * R + g * RPT + r, B - 1);      // rows past the end recompute row B-1 (never finalised)
        dw0[r] = (lw.mss && i == B - 2) ? (lw.ls - lw.ln) : 0.f;
        am[r] = -INFINITY; as[r] = 0.f;
#pragma unroll
        for (int k = 0; k < DC; ++k) {
          sx[r][k] = 0.f;
          zc[r][k] = (EXACT || k < D) ? __ldg(z + (long long)i * D + k) : 0.f;
        }
      }
      const int jend = min(ncols, (s + 1) * CS);
      int jl = s * CS + lane;
      bool first = (c0 + jl == 0);                             // the only (row-dependent) weight: row B-2, column 0
      for (; jl < jend; jl += 32) {
        const float4* pr = sp + jl * DP;
        float a[RPT];
#pragma unroll
        for (int r = 0; r < RPT; ++r) a[r] = 0.f;
#pragma unroll
        for (int k = 0; k < DC; ++k) {
          if (EXACT || k < D) {
            const float4 p = pr[k];
#pragma unroll
            for (int r = 0; r < RPT; ++r) {
              const float tt = zc[r][k] - p.z;
              float arg = fmaf(-p.y, tt * tt, p.x);
              if (first) arg += dw0[r];
              a[r] += arg;
              sx[r][k] += ex2_approx(arg);
            }
          }
        }
#pragma unroll
        for (int r = 0; r < RPT; ++r) {
          const float d = a[r] - am[r];
          const float e = ex2_approx(-fabsf(d));
          const bool up = d > 0.f;
          as[r] = up ? fmaf(as[r], e, 1.f) : as[r] + e;
          am[r] = up ? a[r] : am[r];
        }
        first = false;
      }
#pragma unroll
      for (int r = 0; r < RPT; ++r) {
#pragma unroll
        for (int k = 0; k < DC; ++k) sx[r][k] = warp_sum(sx[r][k]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float m2 = __shfl_xor_sync(0xffffffffu, am[r], o), s2 = __shfl_xor_sync(0xffffffffu, as[r], o);
          lse_merge2(am[r], as[r], m2, s2);
        }
        if (lane == 0) {
#pragma unroll
          for (int k = 0; k < DC; ++k) s_tsx[task * RPT + r][k] = sx[r][k];
          s_tq[task * RPT + r] = make_float2(am[r], as[r]);
        }
      }
    }
    __syncthreads();
    // merge the column splits of every row in a fixed order -> this CTA's partial state
    for (int e = tid; e < R * (DC + 1); e += kF4Threads) {
      const int rr = e / (DC + 1), k = e - rr * (DC + 1);
      const int g = rr / RPT, r2 = rr - g * RPT;
      if (k < DC) {
        float a = 0.f;
        for (int s = 0; s < S; ++s) a += s_tsx[(g * S + s) * RPT + r2][k];
        s_sx[rr][k] = a;
      } else {
        float m = -INFINITY, a = 0.f;
        for (int s = 0; s < S; ++s) { const float2 q = s_tq[(g * S + s) * RPT + r2]; lse_merge2(m, a, q.x, q.y); }
        s_q[rr] = make_float2(m, a);
      }
    }
  }
  cluster.sync();                                              // every CTA's s_sx / s_q / s_ref / s_rsum are final

  // ---- phase 4: cluster rows round-robin over the 4 CTAs; one warp per row, lanes = latent dims ----
  for (int slot = warp; slot * kF4Clus + crank < R; slot += kF4Warps) {
    const int rr = slot * kF4Clus + crank;
    const int i = clus * R + rr;
    if (i >= B) { if (lane == 0) { s_means[slot][0] = 0.f; s_means[slot][1] = 0.f; s_means[slot][2] = 0.f; } continue; }
    float P2 = 0.f;
    bool bad = false;
    if (lane < D) {
      float rc[kF4Clus], sc[kF4Clus], Rm = -INFINITY;
#pragma unroll
      for (int c = 0; c < kF4Clus; ++c) {
        sc[c] = *cluster.map_shared_rank(&s_sx[rr][lane], c);
        rc[c] = *cluster.map_shared_rank(&s_ref[lane], c);
        if (sc[c] > 0.f) Rm = fmaxf(Rm, rc[c]);
      }
      float tot = 0.f;
#pragma unroll
      for (int c = 0; c < kF4Clus; ++c)
        if (sc[c] > 0.f) tot += sc[c] * exp2f(rc[c] - Rm);
      // ex2 flushes terms below 2^-126 of a CTA's reference: a total under ~2^-90 could have lost a visible share
      bad = !(tot > 1e-27f && tot < INFINITY);
      P2 = Rm + log2f(tot);
    }
    float lqz2 = 0.f;
    if (lane == 31) {
      float m = -INFINITY, a = 0.f;
#pragma unroll
      for (int c = 0; c < kF4Clus; ++c) {
        const float2 q = *cluster.map_shared_rank(&s_q[rr], c);
        const float rs = *cluster.map_shared_rank(&s_rsum, c);
        if (q.y > 0.f) lse_merge2(m, a, q.x + rs, q.y);
      }
      lqz2 = m + log2f(a);
    }
    const unsigned badmask = __ballot_sync(0xffffffffu, bad);
    if (badmask) {                                             // rare: exact two-pass logsumexp from global memory
      for (int k = 0; k < D; ++k) {
        if (!((badmask >> k) & 1u)) continue;
        const float zk = z[(long long)i * D + k];
        auto term = [&](int j) {                               // m[i,j,k] + lw[i,j], log2 units
          const long long off = (long long)j * row_stride + (long long)k * ld;
          const float tt = zk - mu[off], lv = logvar[off];
          return (-0.5f * (kLog2Pi + lv) - 0.5f * (tt * tt) * expf(-lv)) * kLog2e + logw2(lw, i, j);
        };
        float mx = -INFINITY;
        for (int j = lane; j < B; j += 32) mx = fmaxf(mx, term(j));
        mx = warp_max(mx);
        float sm = 0.f;
        for (int j = lane; j < B; j += 32) sm += exp2f(term(j) - mx);
        sm = warp_sum(sm);
        if (lane == k) P2 = mx + log2f(sm);
      }
    }
    float lq = 0.f, lp = 0.f;
    for (int d = lane; d < D; d += 32) {
      const long long off = (long long)i * row_stride + (long long)d * ld;
      add_row_gauss(z[(long long)i * D + d], mu[off], logvar[off], lq, lp);
    }
    lq = warp_sum(lq); lp = warp_sum(lp);
    const float Pn = (lane < D) ? P2 * kLn2 : 0.f;
    if (lane < D) rowstats[(long long)(4 + lane) * B + i] = Pn;
    const float lprod = warp_sum(Pn);
    const float lqz = __shfl_sync(0xffffffffu, lqz2, 31) * kLn2;
    if (lane == 0) {
      rowstats[i] = lp; rowstats[1LL * B + i] = lqz; rowstats[2LL * B + i] = lprod; rowstats[3LL * B + i] = lq;
      s_means[slot][0] = lq - lqz; s_means[slot][1] = lqz - lprod; s_means[slot][2] = lprod - lp;
    }
  }
  __syncthreads();
  if (tid == 0) {
    float a = 0.f, b = 0.f, c = 0.f;
    for (int slot = 0; slot * kF4Clus + crank < R; ++slot) { a += s_means[slot][0]; b += s_means[slot][1]; c += s_means[slot][2]; }
    blockpart[4 * blockIdx.x + 0] = a; blockpart[4 * blockIdx.x + 1] = b; blockpart[4 * blockIdx.x + 2] = c;
    __threadfence();
    is_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  }
  cluster.sync();                                              // no CTA leaves while a peer may still read its shared memory
  if (!is_last || warp != 0) return;
  __threadfence();
  float a = 0.f, b = 0.f, c = 0.f;
  for (int g = lane; g < (int)gridDim.x; g += 32) {             // lane-strided, then a fixed shuffle tree
    a += __ldcg(blockpart + 4 * g); b += __ldcg(blockpart + 4 * g + 1); c += __ldcg(blockpart + 4 * g + 2);
  }
  a = warp_sum(a); b = warp_sum(b); c = warp_sum(c);
  if (lane == 0) {
    terms[0] = a / (float)B; terms[1] = b / (float)B; terms[2] = c / (float)B;
    *counter = 0u;
  }
}

// ---- backward ---------------------------------------------------------------------
// G[i,j,d] = cq * S[i,j] + cp * T[i,j,d],  S = exp(A[i,j] - log_qz[i]),  T = exp(M[i,j,d] - P[i,d])
// role 0 (rows):    g_z[i,d]  = sum_j G * (-(z_i - mu_j) * iv_j)            + direct terms
// role 1 (columns): g_mu[j,d] = sum_i G * ( (z_i - mu_j) * iv_j)            + direct terms
//                   g_lv[j,d] = sum_i G * (-0.5 + 0.5 (z_i - mu_j)^2 iv_j)  + direct terms
// The thread owns a "line" (i for role 0, j for role 1) and sweeps the other index.
// Row window [row0, row0 + nrows) of the global batch (the whole batch, or one rank's rows when the estimator runs
// over an all-gathered batch): role 0 lines are the window's rows and sweep all B columns (g_z is [nrows, D]);
// role 1 lines are ALL B columns and sweep the window's rows (g_mu / g_lv are [B, D] partial sums, to be
// reduce-scattered over the ranks); the diagonal terms belong to the rank that owns the row.
template <int ROLE, int DC, bool FUSE, bool EXACT>
__device__ __forceinline__ void btcvae_bwd_body(int B, int D, int row0, int nrows, const LogW& lw, const float* __restrict__ ws,
                                                const float* __restrict__ rowstats, float cq, float cp, float cqc, float cpz,
                                                float* __restrict__ g_z, float* __restrict__ g_mu, float* __restrict__ g_lv,
                                                int block) {
  __shared__ float sm_a[kBtWarps][kRows][DC];
  __shared__ float sm_b[kBtWarps][kRows][DC];
  const float4* __restrict__ pj = reinterpret_cast<const float4*>(ws + kWsHeader);
  const float* __restrict__ lqz = rowstats + 1LL * B;
  const float* __restrict__ P = rowstats + 4LL * B;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = lane >> 3, ol = lane & 7;
  const int row_end = row0 + nrows;
  const int line = (ROLE == 0) ? min(row0 + block * kRows + r, row_end - 1) : min(block * kRows + r, B - 1);
  const int sweep0 = (ROLE == 0) ? 0 : row0, sweep1 = (ROLE == 0) ? B : row_end;
  const int slice = ((sweep1 - sweep0 + kBtWarps - 1) / kBtWarps + kJL - 1) / kJL * kJL;
  const int o_begin = sweep0 + warp * slice, o_end = min(sweep1, o_begin + slice);
  const float Df = (float)D;
  const float own_lqz2 = (ROLE == 0) ? lqz[line] * kLog2e : 0.f;

  for (int d0 = 0; d0 < D; d0 += DC) {
    const int nd = EXACT ? DC : min(DC, D - d0);
    float4 own[DC];                // role 0: {., ., ., z_i} + P_i*log2e in .x ; role 1: {c, hiv, mu, .} of column j
    float acc_a[DC], acc_b[DC];
#pragma unroll
    for (int k = 0; k < DC; ++k) {
      acc_a[k] = 0.f; acc_b[k] = 0.f;
      if (EXACT || k < nd) {
        own[k] = __ldg(pj + (long long)(d0 + k) * B + line);
        if (ROLE == 0) own[k].x = P[(long long)(d0 + k) * B + line] * kLog2e;
      } else own[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int o = o_begin + ol; o < o_end; o += kJL) {
      const int i = (ROLE == 0) ? line : o;
      const int j = (ROLE == 0) ? o : line;
      const float w = logw2(lw, i, j);
      float mk[DC], tk[DC], hk[DC], pk[DC];
      float sa = 0.f;
#pragma unroll
      for (int k = 0; k < DC; ++k) {
        if (EXACT || k < nd) {
          const float4 q = __ldg(pj + (long long)(d0 + k) * B + o);
          float t, h, cc;
          if (ROLE == 0) { t = own[k].w - q.z; h = q.y; cc = q.x; pk[k] = own[k].x; }
          else           { t = q.w - own[k].z; h = own[k].y; cc = own[k].x; pk[k] = P[(long long)(d0 + k) * B + o] * kLog2e; }
          tk[k] = t; hk[k] = h;
          mk[k] = cc - h * (t * t);
          sa += mk[k];
        } else { mk[k] = 0.f; tk[k] = 0.f; hk[k] = 0.f; pk[k] = 0.f; }
      }
      if (!FUSE) {                 // A[i,j] needs ALL dims, not only this chunk
        sa = 0.f;
        for (int d = 0; d < D; ++d) {
          const float4 pi = __ldg(pj + (long long)d * B + i), pjv = __ldg(pj + (long long)d * B + j);
          const float t = pi.w - pjv.z;
          sa += pjv.x - pjv.y * (t * t);
        }
      }
      const float lq2 = (ROLE == 0) ? own_lqz2 : lqz[i] * kLog2e;
      const float gS = cq * exp2f(sa + Df * w - lq2);
#pragma unroll
      for (int k = 0; k < DC; ++k) {
        if (EXACT || k < nd) {
          const float T = exp2f(mk[k] + (w - pk[k]));
          const float G = gS + cp * T;
          // hk is 0.5*iv*log2e: (z-mu)*iv = 2*hk*t/log2e ; 0.5 (z-mu)^2 iv = hk t^2 / log2e
          const float tiv = (2.f * kLn2) * hk[k] * tk[k];
          if (ROLE == 0) acc_a[k] -= G * tiv;
          else { acc_a[k] += G * tiv; acc_b[k] += G * (kLn2 * hk[k] * (tk[k] * tk[k]) - 0.5f); }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < DC; ++k) {
#pragma unroll
      for (int o = 1; o < kJL; o <<= 1) {
        acc_a[k] += __shfl_xor_sync(0xffffffffu, acc_a[k], o);
        if (ROLE == 1) acc_b[k] += __shfl_xor_sync(0xffffffffu, acc_b[k], o);
      }
      if (ol == 0) { sm_a[warp][r][k] = acc_a[k]; if (ROLE == 1) sm_b[warp][r][k] = acc_b[k]; }
    }
    __syncthreads();
    if (warp == 0) {
      for (int e = lane; e < kRows * DC; e += 32) {
        const int rr = e / DC, k = e % DC;
        const int ln = (ROLE == 0 ? row0 : 0) + block * kRows + rr;
        if (k < nd && ln < (ROLE == 0 ? row_end : B)) {
          float a = 0.f, b = 0.f;
          for (int w2 = 0; w2 < kBtWarps; ++w2) { a += sm_a[w2][rr][k]; if (ROLE == 1) b += sm_b[w2][rr][k]; }
          const float4 q = __ldg(pj + (long long)(d0 + k) * B + ln);
          const float t = q.w - q.z;
          const float tiv = (2.f * kLn2) * q.y * t;              // (z-mu) iv  of the diagonal pair
          if (ROLE == 0) {
            // d log_q_zCx / dz = -(z-mu) iv ; d log_pz / dz = -z
            if (g_z) g_z[(long long)(ln - row0) * D + d0 + k] = a - cqc * tiv - cpz * q.w;
          } else {
            const float own = (ln >= row0 && ln < row_end) ? cqc : 0.f;   // the diagonal pair lives with its row
            if (g_mu) g_mu[(long long)ln * D + d0 + k] = a + own * tiv;
            if (g_lv) g_lv[(long long)ln * D + d0 + k] = b + own * (kLn2 * q.y * (t * t) - 0.5f);
          }
        }
      }
    }
    __syncthreads();
  }
}

template <int DC, bool FUSE, bool EXACT>
__global__ void __launch_bounds__(kBtWarps * 32)
btcvae_bwd_kernel(int B, int D, int row0, int nrows, LogW lw, const float* __restrict__ ws, const float* __restrict__ rowstats,
                  const float* __restrict__ g_terms, float* __restrict__ g_z, float* __restrict__ g_mu, float* __restrict__ g_lv) {
  const float invB = 1.f / (float)nrows;       // the three terms are means over the window's rows
  const float g_mi = g_terms[0], g_tc = g_terms[1], g_dw = g_terms[2];
  const float cq = (g_tc - g_mi) * invB;       // d loss / d log_qz[i]
  const float cp = (g_dw - g_tc) * invB;       // d loss / d log_prod_qzi[i]
  const float cqc = g_mi * invB;               // d loss / d log_q_zCx[i]
  const float cpz = -g_dw * invB;              // d loss / d log_pz[i]
  const int nblk = (nrows + kRows - 1) / kRows;
  if ((int)blockIdx.x < nblk)
    btcvae_bwd_body<0, DC, FUSE, EXACT>(B, D, row0, nrows, lw, ws, rowstats, cq, cp, cqc, cpz, g_z, g_mu, g_lv, blockIdx.x);
  else
    btcvae_bwd_body<1, DC, FUSE, EXACT>(B, D, row0, nrows, lw, ws, rowstats, cq, cp, cqc, cpz, g_z, g_mu, g_lv, blockIdx.x - nblk);
}

static LogW make_logw(int B, long long n_data, int is_mss) {
  LogW w; w.mss = is_mss; w.B = B;
  const double N = (double)n_data, M = (double)(B - 1);
  // math.py:66-73: the weights are stored in an fp32 tensor, then .log() in fp32
  w.ln = logf((float)(1.0 / N)) * kLog2e;
  w.ls = logf((float)((N - M) / (N * M))) * kLog2e;
  w.lm = logf((float)(1.0 / M)) * kLog2e;
  return w;
}

#define DV_BT_DISPATCH(D, CALL)                                   \
  do {                                                            \
    if ((D) == 10)      { CALL(10, true, true); }                 \
    else if ((D) == 16) { CALL(16, true, true); }                 \
    else if ((D) == 8)  { CALL(8, true, true); }                  \
    else if ((D) <= 4)  { CALL(4, true, false); }                 \
    else if ((D) < 8)   { CALL(8, true, false); }                 \
    else if ((D) < 16)  { CALL(16, true, false); }                \
    else if ((D) % 16 == 0) { CALL(16, false, true); }            \
    else                { CALL(16, false, false); }               \
  } while (0)

}  // namespace dv

using namespace dv;

extern "C" {

// blocks of the 64-column tiling: (rows/32) x (B/64); below one block per SM the 16-column tiling is used.  The choice
// for a row window never needs more workspace than the choice for the whole batch (fewer rows -> small tiles only if
// the whole-batch rule picked them too, or B is small enough that dv_btcvae_workspace_bytes reserved them).
static bool fwd2_small_tiles(int B, int nrows) {
  return (long long)((nrows + kRG - 1) / kRG) * ((B + kJTBig - 1) / kJTBig) < kNumSMs && B <= 1024;
}
// header | float4 pj[D][B] | float2 part[ceil(B/JT)][D+1][B]
// The cluster path keeps its per-CTA partial means (4 floats per CTA) where `part` goes; at tiny B * D that is more
// than `part` itself.
static long long btcvae_part_offset_floats(int B, int D) { return kWsHeader + 4LL * B * D; }
size_t dv_btcvae_workspace_bytes(int B, int D) {
  const long long JS = (B + kJTSmall - 1) / kJTSmall;          // room for either column tile width when B is small
  const long long JS_big = (B + kJTBig - 1) / kJTBig;
  const long long js = fwd2_small_tiles(B, B) ? JS : JS_big;
  const long long part = std::max(2LL * js * (D + 1) * B, 4LL * kF4Clus * kF4MaxClusters);
  return (size_t)(btcvae_part_offset_floats(B, D) + part) * sizeof(float);
}

int dv_btcvae_fwd(const float* z, const float* mu, const float* logvar, int ld, int row_stride, int B, int D,
                  long long n_data, int is_mss, float* rowstats, float* terms, void* workspace, void* stream) {
  return dv_btcvae_fwd_rows(z, mu, logvar, ld, row_stride, B, D, 0, B, n_data, is_mss, rowstats, terms, workspace, stream);
}

int dv_btcvae_fwd_rows(const float* z, const float* mu, const float* logvar, int ld, int row_stride, int B, int D,
                       int row0, int nrows, long long n_data, int is_mss, float* rowstats, float* terms, void* workspace,
                       void* stream) {
  if (!z || !mu || !logvar || !rowstats || !terms || !workspace) return DV_ERR_BAD_ARG;
  if (B < 2 || D < 1 || n_data < 1) return DV_ERR_BAD_SHAPE;
  if (row0 < 0 || nrows < 1 || row0 + nrows > B) return DV_ERR_BAD_SHAPE;
  const bool whole = (row0 == 0 && nrows == B);
  if ((uintptr_t)workspace & 15) return DV_ERR_BAD_ARG;
  float* ws = reinterpret_cast<float*>(workspace);
  cudaStream_t st = as_stream(stream);
  const LogW lw = make_logw(B, n_data, is_mss);
  {
    // single-launch cluster path (D <= 16): columns split over the 4 CTAs of a cluster, rows over the clusters
    const int dc = D == 10 ? 10 : 16;
    // kF4MaxClusters: estimated 4-CTA cluster capacity of a 132-SM H100 (see above)
    int R = ((B + kF4MaxClusters - 1) / kF4MaxClusters + kRows - 1) / kRows * kRows;
    const int NC = ((B + kF4Clus - 1) / kF4Clus + kJL - 1) / kJL * kJL;
    const size_t smem = (size_t)NC * (dc + 1) * sizeof(float4);
    const int rpt = (dc == 10) ? 4 : 2;                        // rows per thread (register budget)
    const int G = R / rpt;
    int S = G >= kF4Warps ? 1 : kF4Warps / G;
    if (S > NC / 32) S = NC / 32;
    if (S < 1) S = 1;
    if (whole && D <= 16 && smem <= kF4MaxSmem && R <= kF4MaxRows && G * S <= kF4MaxTasks) {
      const int nclus = (B + R - 1) / R;
      float4* pj = reinterpret_cast<float4*>(ws + kWsHeader);
      float* blockpart = ws + btcvae_part_offset_floats(B, D);
      unsigned* counter = reinterpret_cast<unsigned*>(ws);
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(nclus * kF4Clus); cfg.blockDim = dim3(kF4Threads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = kF4Clus; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
      cfg.attrs = attr; cfg.numAttrs = 1;
      auto launch = [&](auto kernel, bool* smem_set) -> int {
        const int rc = set_max_dynamic_smem(kernel, kF4MaxSmem, smem_set);
        if (rc != DV_OK) return rc;
        const cudaError_t err = cudaLaunchKernelEx(&cfg, kernel, z, mu, logvar, ld, row_stride, B, D, lw, R, S, NC, pj,
                                                   rowstats, terms, blockpart, counter);
        if (err != cudaSuccess) { g_last_cuda_error = (int)err; cudaGetLastError(); return DV_ERR_CUDA; }
        return check_launch();
      };
      static bool smem_set_10, smem_set_16, smem_set_16_any;
      if (D == 10) return launch(btcvae_fwd4_kernel<10, true, 4>, &smem_set_10);
      if (D == 16) return launch(btcvae_fwd4_kernel<16, true, 2>, &smem_set_16);
      return launch(btcvae_fwd4_kernel<16, false, 2>, &smem_set_16_any);
    }
  }
  btcvae_prep_kernel<<<(B + 3) / 4, 128, 0, st>>>(z, mu, logvar, ld, row_stride, B, D,
                                                  reinterpret_cast<float4*>(ws + kWsHeader), rowstats);
  int rc = check_launch();
  if (rc != DV_OK) return rc;
  // small tiles only where the whole-batch rule reserved workspace for them
  const bool small = fwd2_small_tiles(B, nrows) && fwd2_small_tiles(B, B);
  const int JT = small ? kJTSmall : kJTBig;
  const int JS = (B + JT - 1) / JT;
  float2* part = reinterpret_cast<float2*>(ws + btcvae_part_offset_floats(B, D));
  const float4* pjc = reinterpret_cast<const float4*>(ws + kWsHeader);
  dim3 grid((nrows + kRG - 1) / kRG, JS);
#define DV_FWD2(DC, EXACT)                                                                                         \
  do {                                                                                                             \
    if (small) btcvae_fwd2_kernel<DC, EXACT, kJTSmall><<<grid, kBtWarps * 32, 0, st>>>(B, D, row0, nrows, lw, pjc, part); \
    else       btcvae_fwd2_kernel<DC, EXACT, kJTBig><<<grid, kBtWarps * 32, 0, st>>>(B, D, row0, nrows, lw, pjc, part);   \
  } while (0)
  if (D == 10)          DV_FWD2(10, true);
  else if (D % 16 == 0) DV_FWD2(16, true);
  else if (D <= 8)      DV_FWD2(8, false);
  else                  DV_FWD2(16, false);
#undef DV_FWD2
  rc = check_launch();
  if (rc != DV_OK) return rc;
  btcvae_finalize_kernel<<<(nrows + 15) / 16, 256, 0, st>>>(B, D, row0, nrows, JS, lw, pjc, part, rowstats, terms,
                                                            reinterpret_cast<unsigned*>(ws));
  return check_launch();
}

int dv_btcvae_bwd(int B, int D, long long n_data, int is_mss, const float* rowstats, const void* workspace,
                  const float* g_terms, float* g_z, float* g_mu, float* g_logvar, void* stream) {
  return dv_btcvae_bwd_rows(B, D, 0, B, n_data, is_mss, rowstats, workspace, g_terms, g_z, g_mu, g_logvar, stream);
}

int dv_btcvae_bwd_rows(int B, int D, int row0, int nrows, long long n_data, int is_mss, const float* rowstats,
                       const void* workspace, const float* g_terms, float* g_z, float* g_mu, float* g_logvar, void* stream) {
  if (!rowstats || !g_terms || !workspace) return DV_ERR_BAD_ARG;
  if (B < 2 || D < 1) return DV_ERR_BAD_SHAPE;
  if (row0 < 0 || nrows < 1 || row0 + nrows > B) return DV_ERR_BAD_SHAPE;
  const float* ws = reinterpret_cast<const float*>(workspace);
  cudaStream_t st = as_stream(stream);
  const LogW lw = make_logw(B, n_data, is_mss);
  const int grid = (nrows + kRows - 1) / kRows + (B + kRows - 1) / kRows;
#define DV_BWD_CALL(DC, FUSE, EXACT) \
  btcvae_bwd_kernel<DC, FUSE, EXACT><<<grid, kBtWarps * 32, 0, st>>>(B, D, row0, nrows, lw, ws, rowstats, g_terms, g_z, g_mu, g_logvar)
  DV_BT_DISPATCH(D, DV_BWD_CALL);
#undef DV_BWD_CALL
  return check_launch();
}

}  // extern "C"

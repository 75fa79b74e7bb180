// Fully-connected layers: one tiled FP32 GEMM with fused bias / activation / activation-gradient
// epilogues.  Replaces nn.Linear + ReLU / LeakyReLU in disvae/models/encoders.py:81-86,
// disvae/models/decoders.py:71-73, disvae/models/discriminator.py:63-68 and their backward.
//
//   C[m][n] = sum_r A(m, r) * Bm(r, n)         (r = reduction index)
//   A(m, r)  = A[m * a_sm + r * a_sr]
//   Bm(r, n) = Bp[r * b_sr + n * b_sn]
// fwd  : A = x[M,K]  (a_sm=K, a_sr=1), Bm = w[N,K]^T (b_sr=1, b_sn=K), R = K
// dgrad: A = g[M,N]  (a_sm=N, a_sr=1), Bm = w[N,K]   (b_sr=K, b_sn=1), R = N, output [M,K]
// wgrad: A = g[M,N]^T(a_sm=1, a_sr=N), Bm = x[M,K]   (b_sr=K, b_sn=1), R = M, output [N,K]
#include "dv_common.cuh"

namespace dv {

constexpr int BM = 64, BN = 64, BK = 16;

struct GemmEpilogue {
  const float* bias;       // per output column (may be null)
  const float* mask_src;   // same shape as C: C *= act'(mask_src)   (may be null)
  int act;                 // forward activation, or the activation whose gradient masks
  float slope;
};

// A_R_CONTIG: A's reduction index is contiguous (a_sr == 1); else A's m index is contiguous.
// B_R_CONTIG: B's reduction index is contiguous (b_sr == 1); else B's n index is contiguous.
// The next K tile is fetched into registers while the current one is consumed from shared memory
// (these GEMMs are small: without the prefetch every k-step exposes a full L2/HBM round trip).
// blockIdx.z selects a split of the reduction range (split-K); partial results go to C + z*Mo*No.
template <bool A_R_CONTIG, bool B_R_CONTIG>
__global__ void __launch_bounds__(256)
gemm_kernel(const float* __restrict__ A, const float* __restrict__ Bp, float* __restrict__ C,
            int Mo, int No, int R, long long a_sm, long long a_sr, long long b_sr, long long b_sn,
            GemmEpilogue ep, int r_per_split) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;              // 16 x 16 threads, 4 x 4 outputs each
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int r_begin = blockIdx.z * r_per_split;
  const int r_end = min(R, r_begin + r_per_split);
  C += (long long)blockIdx.z * Mo * No;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  float ra[4], rb[4];
  auto fetch = [&](int r0) {
    if (A_R_CONTIG) {
      const int m = tid >> 2, rq = (tid & 3) * 4;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int gm = m0 + m, gr = r0 + rq + e;
        ra[e] = (gm < Mo && gr < r_end) ? __ldg(A + gm * a_sm + gr * a_sr) : 0.f;
      }
    } else {
      const int r = tid >> 4, mq = (tid & 15) * 4;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int gm = m0 + mq + e, gr = r0 + r;
        ra[e] = (gm < Mo && gr < r_end) ? __ldg(A + gm * a_sm + gr * a_sr) : 0.f;
      }
    }
    if (B_R_CONTIG) {
      const int n = tid >> 2, rq = (tid & 3) * 4;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int gn = n0 + n, gr = r0 + rq + e;
        rb[e] = (gn < No && gr < r_end) ? __ldg(Bp + gr * b_sr + gn * b_sn) : 0.f;
      }
    } else {
      const int r = tid >> 4, nq = (tid & 15) * 4;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int gn = n0 + nq + e, gr = r0 + r;
        rb[e] = (gn < No && gr < r_end) ? __ldg(Bp + gr * b_sr + gn * b_sn) : 0.f;
      }
    }
  };
  auto stash = [&]() {
    if (A_R_CONTIG) { const int m = tid >> 2, rq = (tid & 3) * 4;
#pragma unroll
      for (int e = 0; e < 4; ++e) As[rq + e][m] = ra[e];
    } else { const int r = tid >> 4, mq = (tid & 15) * 4;
#pragma unroll
      for (int e = 0; e < 4; ++e) As[r][mq + e] = ra[e];
    }
    if (B_R_CONTIG) { const int n = tid >> 2, rq = (tid & 3) * 4;
#pragma unroll
      for (int e = 0; e < 4; ++e) Bs[rq + e][n] = rb[e];
    } else { const int r = tid >> 4, nq = (tid & 15) * 4;
#pragma unroll
      for (int e = 0; e < 4; ++e) Bs[r][nq + e] = rb[e];
    }
  };

  fetch(r_begin);
  for (int r0 = r_begin; r0 < r_end; r0 += BK) {
    stash();
    __syncthreads();
    if (r0 + BK < r_end) fetch(r0 + BK);               // in flight while this tile is consumed
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty * 4 + i;
    if (gm >= Mo) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn >= No) continue;
      float v = acc[i][j];
      const long long idx = (long long)gm * No + gn;
      if (ep.mask_src) {
        const float y = ep.mask_src[idx];
        if (ep.act == DV_ACT_RELU) v = y > 0.f ? v : 0.f;
        else if (ep.act == DV_ACT_LEAKY) v = y > 0.f ? v : v * ep.slope;
      } else {
        if (ep.bias) v += ep.bias[gn];
        v = apply_act(v, ep.act, ep.slope);
      }
      C[idx] = v;
    }
  }
}

// fixed-order sum of split-K partials
__global__ void splitk_reduce_kernel(const float* __restrict__ part, float* __restrict__ out, long long n, int S) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int z = 0; z < S; ++z) s += part[(long long)z * n + i];
    out[i] = s;
  }
}

// out[n] = sum_m g[m][n]  (bias gradient): block = 32 columns x 32 row-slices (4 independent partial sums each),
// combined in a fixed order.
__global__ void __launch_bounds__(1024) colsum_kernel(const float* __restrict__ g, float* __restrict__ out, int M, int N) {
  __shared__ float red[32][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = blockIdx.x * 32 + lane;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  if (n < N) {
    int m = warp;
    for (; m + 96 < M; m += 128) {
      s0 += g[(long long)m * N + n];
      s1 += g[(long long)(m + 32) * N + n];
      s2 += g[(long long)(m + 64) * N + n];
      s3 += g[(long long)(m + 96) * N + n];
    }
    for (; m < M; m += 32) s0 += g[(long long)m * N + n];
  }
  red[warp][lane] = (s0 + s1) + (s2 + s3);
  __syncthreads();
  if (warp == 0 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 32; ++w) t += red[w][lane];
    out[n] = t;
  }
}

static int wgrad_splits(int M, int N, int K) {
  const int tiles = ((K + BN - 1) / BN) * ((N + BM - 1) / BM);
  if (tiles >= 120) return 1;
  int S = (2 * kNumSMs + tiles - 1) / tiles;
  const int maxS = (M + 4 * BK - 1) / (4 * BK);         // at least 4 k-steps per split
  if (S > maxS) S = maxS;
  if (S > 32) S = 32;
  return S < 1 ? 1 : S;
}

}  // namespace dv

namespace dv { namespace ltc {
bool nt_ok(int R);
size_t packed_floats(int N, int K);
int pack_multi(int n, const float* const* w, float* const* packed, const int* N, const int* K, cudaStream_t st);
int fwd_packed(const float* x, const float* packed, const float* bias, float* y, int M, int N, int K, int act, float slope,
               cudaStream_t st);
int dgrad_packed(const float* g, const float* packed, const float* mask_src, float* dx, int M, int N, int K, int act, float slope,
                 cudaStream_t st);
bool wgrad_ok(int M, int N, int K);
size_t wgrad_workspace_bytes(int M, int N, int K);
int wgrad(const float* g, const float* x, float* dw, float* dbias, float* ws, int M, int N, int K, int* nsplit, cudaStream_t st);
} }

using namespace dv;

// The tensor-core GEMMs read their activation operand and the packed weight planes through TMA, which takes 16-byte
// aligned global addresses only (the tensor-core paths refuse others with `misaligned`); the CUDA-core GEMM reads
// single floats.

// act of an input gradient: the activation whose derivative masks it
static bool dgrad_act_ok(int act) { return act == DV_ACT_NONE || act == DV_ACT_RELU || act == DV_ACT_LEAKY; }

extern "C" {

// The tensor-core path packs w into the workspace (the layout of dv_linear_pack_multi) and runs on those planes.
size_t dv_linear_fwd_workspace_bytes(int M, int N, int K) {
  if (M <= 0 || N <= 0 || K <= 0 || !ltc::nt_ok(K)) return 0;
  return ltc::packed_floats(N, K) * sizeof(float);
}
size_t dv_linear_dgrad_workspace_bytes(int M, int N, int K) {
  if (M <= 0 || N <= 0 || K <= 0 || !ltc::nt_ok(N)) return 0;
  return ltc::packed_floats(N, K) * sizeof(float);
}

int dv_linear_fwd(const float* x, const float* w, const float* bias, float* y, int M, int N, int K,
                  int act, float slope, void* workspace, void* stream) {
  if (!x || !w || !y) return DV_ERR_BAD_ARG;
  if (M <= 0 || N <= 0 || K <= 0) return DV_ERR_BAD_SHAPE;
  if (act < DV_ACT_NONE || act > DV_ACT_LEAKY) return DV_ERR_BAD_ARG;
  if (ltc::nt_ok(K)) {
    if (!workspace) return DV_ERR_WORKSPACE;
    if (misaligned(x, 16) || misaligned(workspace, 16)) return DV_ERR_BAD_ARG;
    float* packed = reinterpret_cast<float*>(workspace);
    const int rc = ltc::pack_multi(1, &w, &packed, &N, &K, as_stream(stream));
    if (rc != DV_OK) return rc;
    return ltc::fwd_packed(x, packed, bias, y, M, N, K, act, slope, as_stream(stream));
  }
  GemmEpilogue ep{bias, nullptr, act, slope};
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
  gemm_kernel<true, true><<<grid, 256, 0, as_stream(stream)>>>(x, w, y, M, N, K, K, 1, 1, K, ep, K);
  return check_launch();
}

int dv_linear_dgrad(const float* g, const float* w, const float* mask_src, float* dx, int M, int N, int K,
                    int act, float slope, void* workspace, void* stream) {
  if (!g || !w || !dx) return DV_ERR_BAD_ARG;
  if (M <= 0 || N <= 0 || K <= 0) return DV_ERR_BAD_SHAPE;
  if (!dgrad_act_ok(act)) return DV_ERR_BAD_ARG;
  if (ltc::nt_ok(N)) {
    if (!workspace) return DV_ERR_WORKSPACE;
    if (misaligned(g, 16) || misaligned(workspace, 16)) return DV_ERR_BAD_ARG;
    float* packed = reinterpret_cast<float*>(workspace);
    const int rc = ltc::pack_multi(1, &w, &packed, &N, &K, as_stream(stream));
    if (rc != DV_OK) return rc;
    return ltc::dgrad_packed(g, packed, mask_src, dx, M, N, K, act, slope, as_stream(stream));
  }
  GemmEpilogue ep{nullptr, mask_src, mask_src ? act : DV_ACT_NONE, slope};
  dim3 grid((K + BN - 1) / BN, (M + BM - 1) / BM);
  gemm_kernel<true, false><<<grid, 256, 0, as_stream(stream)>>>(g, w, dx, M, K, N, N, 1, K, 1, ep, N);
  return check_launch();
}

size_t dv_linear_packed_floats(int N, int K) {
  if (N <= 0 || K <= 0) return 0;
  return ltc::packed_floats(N, K);
}

int dv_linear_pack_multi(int n, const void* const* w, void* const* packed, const int* N, const int* K, void* stream) {
  if (n < 1 || !w || !packed || !N || !K) return DV_ERR_BAD_ARG;
  for (int i = 0; i < n; ++i)
    if (!w[i] || !packed[i] || N[i] <= 0 || K[i] <= 0 || misaligned(packed[i], 16)) return DV_ERR_BAD_ARG;
  return ltc::pack_multi(n, reinterpret_cast<const float* const*>(w), reinterpret_cast<float* const*>(packed), N, K,
                         as_stream(stream));
}

int dv_linear_fwd_packed(const float* x, const float* w, const float* packed, const float* bias, float* y, int M, int N, int K,
                         int act, float slope, void* stream) {
  if (!x || !w || !y) return DV_ERR_BAD_ARG;
  if (M <= 0 || N <= 0 || K <= 0) return DV_ERR_BAD_SHAPE;
  if (act < DV_ACT_NONE || act > DV_ACT_LEAKY) return DV_ERR_BAD_ARG;
  if (ltc::nt_ok(K)) {
    if (!packed) return DV_ERR_WORKSPACE;
    if (misaligned(x, 16) || misaligned(packed, 16)) return DV_ERR_BAD_ARG;
    return ltc::fwd_packed(x, packed, bias, y, M, N, K, act, slope, as_stream(stream));
  }
  return dv_linear_fwd(x, w, bias, y, M, N, K, act, slope, nullptr, stream);       // CUDA-core path: reads w itself
}

int dv_linear_dgrad_packed(const float* g, const float* w, const float* packed, const float* mask_src, float* dx, int M, int N,
                           int K, int act, float slope, void* stream) {
  if (!g || !w || !dx) return DV_ERR_BAD_ARG;
  if (M <= 0 || N <= 0 || K <= 0) return DV_ERR_BAD_SHAPE;
  if (!dgrad_act_ok(act)) return DV_ERR_BAD_ARG;
  if (ltc::nt_ok(N)) {
    if (!packed) return DV_ERR_WORKSPACE;
    if (misaligned(g, 16) || misaligned(packed, 16)) return DV_ERR_BAD_ARG;
    return ltc::dgrad_packed(g, packed, mask_src, dx, M, N, K, act, slope, as_stream(stream));
  }
  return dv_linear_dgrad(g, w, mask_src, dx, M, N, K, act, slope, nullptr, stream);
}

size_t dv_linear_wgrad_workspace_bytes(int M, int N, int K) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if (ltc::wgrad_ok(M, N, K)) return ltc::wgrad_workspace_bytes(M, N, K);
  const int S = wgrad_splits(M, N, K);
  return S > 1 ? (size_t)S * N * K * sizeof(float) : 0;
}

int dv_linear_wgrad(const float* g, const float* x, float* dw, float* dbias, int M, int N, int K, void* workspace,
                    void* stream) {
  if (!g || !x || !dw) return DV_ERR_BAD_ARG;
  if (M <= 0 || N <= 0 || K <= 0) return DV_ERR_BAD_SHAPE;
  cudaStream_t st = as_stream(stream);
  if (ltc::wgrad_ok(M, N, K)) {
    if (ltc::wgrad_workspace_bytes(M, N, K) > 0 && !workspace) return DV_ERR_WORKSPACE;
    if (misaligned(g, 16) || misaligned(x, 16)) return DV_ERR_BAD_ARG;
    int S = 1;
    int rc = ltc::wgrad(g, x, dw, dbias, reinterpret_cast<float*>(workspace), M, N, K, &S, st);
    if (rc != DV_OK) return rc;
    if (S > 1) {                                               // fixed-order reduction of the split-K partials (dW, then dbias)
      const float* part = reinterpret_cast<const float*>(workspace);
      const long long n = (long long)N * K;
      int gr = (int)((n + 255) / 256); if (gr > 4 * kNumSMs) gr = 4 * kNumSMs;
      splitk_reduce_kernel<<<gr, 256, 0, st>>>(part, dw, n, S);
      rc = check_launch();
      if (rc != DV_OK) return rc;
      if (dbias) {
        splitk_reduce_kernel<<<(N + 255) / 256, 256, 0, st>>>(part + (size_t)S * n, dbias, N, S);
        rc = check_launch();
      }
    }
    return rc;
  }
  const int S = wgrad_splits(M, N, K);
  if (S > 1 && !workspace) return DV_ERR_WORKSPACE;
  GemmEpilogue ep{nullptr, nullptr, DV_ACT_NONE, 0.f};
  const int per = ((M + S - 1) / S + BK - 1) / BK * BK;
  dim3 grid((K + BN - 1) / BN, (N + BM - 1) / BM, S);
  float* target = S > 1 ? reinterpret_cast<float*>(workspace) : dw;
  gemm_kernel<false, false><<<grid, 256, 0, st>>>(g, x, target, N, K, M, 1, N, K, 1, ep, per);
  int rc = check_launch();
  if (rc != DV_OK) return rc;
  if (S > 1) {
    const long long n = (long long)N * K;
    int gr = (int)((n + 255) / 256); if (gr > 4 * kNumSMs) gr = 4 * kNumSMs;
    splitk_reduce_kernel<<<gr, 256, 0, st>>>(target, dw, n, S);
    rc = check_launch();
    if (rc != DV_OK) return rc;
  }
  if (!dbias) return rc;
  colsum_kernel<<<(N + 31) / 32, 1024, 0, st>>>(g, dbias, M, N);
  return check_launch();
}

}  // extern "C"

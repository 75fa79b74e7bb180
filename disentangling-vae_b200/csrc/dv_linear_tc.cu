// Tensor-core GEMMs for the fully connected layers (encoder/decoder MLPs and the FactorVAE discriminator):
//     C[M, Nout] = epilogue( A[M, R] . Bw[Nout, R]^T )          (both operands K-major = R contiguous)
// used for the forward pass (A = activations, Bw = weight [N, K], bias + ReLU/LeakyReLU epilogue) and for the
// input gradient (A = upstream gradient [M, N], Bw = weight transposed [K, N], activation-gradient mask epilogue),
// and the weight gradient dW = G^T . X further down.  Replaces nn.Linear + activation
// (disvae/models/encoders.py:81-86, decoders.py:71-73, discriminator.py:63-68) and their autograd backward.
//
// Error-compensated 3xTF32 like the convolutions (dv_ptx.cuh): the weight is split once by a pack kernel into tf32
// hi and residual lo planes (plus the transposed copy for dgrad); the activation fragments are split in registers.
//   CTA tile 128 x 64, grid = ceil(M/128) x ceil(Nout/64); 4-stage TMA ring of {A raw 16 KB, B hi 8 KB, B lo 8 KB};
//   warps 0-7 (4 x 2, 32 x 32 each) issue mma.sync m16n8k8 and run the epilogue, warp 8 is the TMA producer.
//   Row / column / K tails are handled by TMA out-of-bounds zero fill and guarded stores.
#include "dv_common.cuh"
#include "dv_ptx.cuh"

namespace dv {
namespace ltc {

using namespace ptx;

constexpr int kBM = 128, kBN = 64, kBK = 32;
constexpr int kConsumers = 8;
constexpr int kThreads = (kConsumers + 1) * 32;
constexpr int kStages = 4;
constexpr int kATile = kBM * 128;                 // 16 KB raw activation tile
constexpr int kBTile = kBN * 128;                 // 8 KB per weight plane tile
constexpr int kStageBytes = kATile + 2 * kBTile;  // 32 KB

struct Barriers {
  uint64_t full[kStages], empty[kStages];
};
constexpr int kSmemBytes = kStages * kStageBytes + 1024 + 256;
static_assert(sizeof(Barriers) <= 256, "barriers");

struct Epilogue {
  const float* bias;       // [Nout] or null
  const float* mask_src;   // [M, Nout] post-activation output of the previous layer, or null
  int act;                 // DV_ACT_* (forward activation, or which activation's gradient masks)
  float slope;
};


__global__ void __launch_bounds__(kThreads, 1)
linear_nt_mma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_bhi,
                     const __grid_constant__ CUtensorMap tmap_blo, float* __restrict__ C, int M, int Nout, int R,
                     Epilogue ep) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  Barriers* bars = reinterpret_cast<Barriers*>(smem + kStages * kStageBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * kBN;
  const int nkb = (R + kBK - 1) / kBK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&bars->full[s], 1); mbar_init(&bars->empty[s], kConsumers); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kConsumers) {
    if (lane != 0) return;
    prefetch_tmap(&tmap_a); prefetch_tmap(&tmap_bhi); prefetch_tmap(&tmap_blo);
    for (int kb = 0; kb < nkb; ++kb) {
      const int stage = kb % kStages;
      mbar_wait(&bars->empty[stage], ((kb / kStages) & 1u) ^ 1u);
      uint8_t* st = smem + stage * kStageBytes;
      mbar_arrive_expect_tx(&bars->full[stage], kStageBytes);
      tma_load_2d(st, &tmap_a, &bars->full[stage], kb * kBK, m0);
      tma_load_2d(st + kATile, &tmap_bhi, &bars->full[stage], kb * kBK, n0);
      tma_load_2d(st + kATile + kBTile, &tmap_blo, &bars->full[stage], kb * kBK, n0);
    }
    return;
  }

  const int gq = lane >> 2, t = lane & 3;
  const int wm = warp & 3, wn = warp >> 2;                   // rows [32 wm, 32 wm + 32), columns [32 wn, 32 wn + 32)
  float tot[2][4][4] = {}, corr[2][4][4] = {};
  for (int kb = 0; kb < nkb; ++kb) {
    const int stage = kb % kStages;
    mbar_wait(&bars->full[stage], (kb / kStages) & 1u);
    const uint32_t a_base = smem_u32(smem + stage * kStageBytes);
    const uint32_t bh_base = a_base + kATile, bl_base = bh_base + kBTile;
    float mn[2][4][4] = {};                                  // hi*hi of this K block, added to tot in fp32 below
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      uint32_t ah[2][4], al[2][4], bh[4][2], bl[4][2];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int r = wm * 32 + mt * 16 + gq;
        split_tf32(lds32(a_base + swz128(r, 8 * ks + t)), ah[mt][0], al[mt][0]);
        split_tf32(lds32(a_base + swz128(r + 8, 8 * ks + t)), ah[mt][1], al[mt][1]);
        split_tf32(lds32(a_base + swz128(r, 8 * ks + t + 4)), ah[mt][2], al[mt][2]);
        split_tf32(lds32(a_base + swz128(r + 8, 8 * ks + t + 4)), ah[mt][3], al[mt][3]);
      }
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int n = wn * 32 + nt * 8 + gq;
        bh[nt][0] = lds32(bh_base + swz128(n, 8 * ks + t));
        bh[nt][1] = lds32(bh_base + swz128(n, 8 * ks + t + 4));
        bl[nt][0] = lds32(bl_base + swz128(n, 8 * ks + t));
        bl[nt][1] = lds32(bl_base + swz128(n, 8 * ks + t + 4));
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) mma_3xtf32(mn[mt][nt], corr[mt][nt], ah[mt], al[mt], bh[nt], bl[nt]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars->empty[stage]);
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) tot[mt][nt][e] += mn[mt][nt][e];
  }

#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + wm * 32 + mt * 16 + gq + 8 * h;
      if (m >= M) continue;
      float* crow = C + (long long)m * Nout;
      const float* mrow = ep.mask_src ? ep.mask_src + (long long)m * Nout : nullptr;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int n = n0 + wn * 32 + nt * 8 + 2 * t + e;
          if (n >= Nout) continue;
          float v = tot[mt][nt][2 * h + e] + corr[mt][nt][2 * h + e];
          if (mrow) {
            const float y = mrow[n];
            if (ep.act == DV_ACT_RELU) v = y > 0.f ? v : 0.f;
            else if (ep.act == DV_ACT_LEAKY) v = y > 0.f ? v : v * ep.slope;
          } else {
            if (ep.bias) v += ep.bias[n];
            v = apply_act(v, ep.act, ep.slope);
          }
          crow[n] = v;
        }
    }
}

// ------------------------------------------------------------------------------------------
// weight gradient:  dW[n][k] = sum_m G[m][n] * X[m][k]   (reduction over the batch rows)
// Both operands come from TMA as [128 batch rows][32 features] tiles (128-byte swizzle), read transposed by the fragment
// loads: A = G^T (M = 32 output rows n), B = X (N = 64 columns k, warp w owns columns [8w, 8w+8)).  K slot t of an MMA
// holds batch row 8ks + 2t and slot t + 4 row 8ks + 2t + 1, which keeps the transposed loads free of bank conflicts.
// A CTA owns one 32 x 64 block of dW and one slice of the batch (deterministic split-K: partials to the workspace,
// reduced in a fixed order).  Warp 0 also sums the columns of G (bias gradient).
// ------------------------------------------------------------------------------------------
constexpr int kWgStages = 3;
constexpr int kWgStageBytes = 3 * kATile;              // G, X columns [0,32), X columns [32,64)
struct WgBarriers {
  uint64_t full[kWgStages], empty[kWgStages];
};
constexpr int kWgSmemBytes = kWgStages * kWgStageBytes + 1024 + 256;
static_assert(sizeof(WgBarriers) <= 256, "barriers");
static_assert(kWgSmemBytes <= 232448, "smem");

struct WgGeom {
  int M, N, K;
  int m_tiles, tiles_per_split;
};

__global__ void __launch_bounds__(kThreads, 1)
linear_wgrad_mma_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_g,
                        float* __restrict__ out_base, long long split_stride, float* __restrict__ dbias_base,
                        long long dbias_stride, WgGeom g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  WgBarriers* bars = reinterpret_cast<WgBarriers*>(smem + kWgStages * kWgStageBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ng = blockIdx.x, kg = blockIdx.y, sp = blockIdx.z;
  const int t_begin = sp * g.tiles_per_split;
  const int t_end = min(g.m_tiles, t_begin + g.tiles_per_split);

  if (threadIdx.x == 0) {
    for (int s = 0; s < kWgStages; ++s) { mbar_init(&bars->full[s], 1); mbar_init(&bars->empty[s], kConsumers); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kConsumers) {
    if (lane != 0) return;
    prefetch_tmap(&tmap_x); prefetch_tmap(&tmap_g);
    for (int tile = t_begin, i = 0; tile < t_end; ++tile, ++i) {
      const int stage = i % kWgStages, m0 = tile * 128;
      mbar_wait(&bars->empty[stage], ((i / kWgStages) & 1u) ^ 1u);
      uint8_t* st = smem + stage * kWgStageBytes;
      mbar_arrive_expect_tx(&bars->full[stage], kWgStageBytes);
      tma_load_2d(st, &tmap_g, &bars->full[stage], ng * 32, m0);
      tma_load_2d(st + kATile, &tmap_x, &bars->full[stage], kg * 64, m0);        // columns past K: zero fill
      tma_load_2d(st + 2 * kATile, &tmap_x, &bars->full[stage], kg * 64 + 32, m0);
    }
    return;
  }

  const int gq = lane >> 2, t = lane & 3;
  const bool want_bias = dbias_base != nullptr && kg == 0 && warp == 0;   // (every k block sees the same G tiles)
  float tot[2][4] = {};                                      // [n block][fragment]
  float bsum[2][2] = {};                                     // G column sums of n = 16 mt + gq + 8 h
  for (int tile = t_begin, i = 0; tile < t_end; ++tile, ++i) {
    const int stage = i % kWgStages;
    mbar_wait(&bars->full[stage], (i / kWgStages) & 1u);
    const uint32_t g_base = smem_u32(smem + stage * kWgStageBytes);
    const uint32_t x_base = g_base + kATile + (warp >> 2) * kATile;
    const int xc = (warp & 3) * 8 + gq;                      // this lane's X column inside its 32-column tile
    float mn[2][4] = {}, cr[2][4] = {};
#pragma unroll 4
    for (int ks = 0; ks < 16; ++ks) {
      const int r0 = 8 * ks + 2 * t, r1 = r0 + 1;
      uint32_t ah[2][4], al[2][4], bh[2], bl[2];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int n = mt * 16 + gq;
        uint32_t a[4];
        a[0] = lds32(g_base + swz128(r0, n));
        a[1] = lds32(g_base + swz128(r0, n + 8));
        a[2] = lds32(g_base + swz128(r1, n));
        a[3] = lds32(g_base + swz128(r1, n + 8));
        if (want_bias) {
          bsum[mt][0] += __uint_as_float(a[0]) + __uint_as_float(a[2]);
          bsum[mt][1] += __uint_as_float(a[1]) + __uint_as_float(a[3]);
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) split_tf32(a[e], ah[mt][e], al[mt][e]);
      }
      split_tf32(lds32(x_base + swz128(r0, xc)), bh[0], bl[0]);
      split_tf32(lds32(x_base + swz128(r1, xc)), bh[1], bl[1]);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) mma_3xtf32(mn[mt], cr[mt], ah[mt], al[mt], bh, bl);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars->empty[stage]);
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int e = 0; e < 4; ++e) tot[mt][e] += mn[mt][e] + cr[mt][e];
  }

  float* out = out_base + (long long)sp * split_stride;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = ng * 32 + mt * 16 + gq + 8 * h;
      if (n >= g.N) continue;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int k = kg * 64 + warp * 8 + 2 * t + e;
        if (k < g.K) out[(long long)n * g.K + k] = tot[mt][2 * h + e];
      }
    }
  if (want_bias) {                                           // fixed order: the four lanes of a row group, then store
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float s = bsum[mt][h];
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        const int n = ng * 32 + mt * 16 + gq + 8 * h;
        if (t == 0 && n < g.N) dbias_base[(long long)sp * dbias_stride + n] = s;
      }
  }
}

// Weight packing: every weight matrix of a network node (encoder MLP, decoder MLP, the 6-layer discriminator) in
// ONE launch, both layouts at once -- packed[i] = [fwd hi | fwd lo | transposed hi | transposed lo] with pitches
// round4(K) / round4(N) (TMA row pitches are multiples of 16 bytes); the transposed copy is what the input-gradient
// GEMM reads.
constexpr int kPackMax = 8;
struct PackTable {
  const float* w[kPackMax];
  float* dst[kPackMax];
  int N[kPackMax], K[kPackMax], tiles_k[kPackMax], tile0[kPackMax + 1];
  int n;
};
__global__ void linear_pack_multi_kernel(PackTable t) {
  __shared__ float tile[32][33];
  int m = 0;
  while (m + 1 < t.n && (int)blockIdx.x >= t.tile0[m + 1]) ++m;
  const int local = blockIdx.x - t.tile0[m];
  const int N = t.N[m], K = t.K[m];
  const int Kp = (K + 3) & ~3, Np = (N + 3) & ~3;
  const int k0 = (local % t.tiles_k[m]) * 32, n0 = (local / t.tiles_k[m]) * 32;
  const float* __restrict__ w = t.w[m];
  float* f_hi = t.dst[m];
  float* f_lo = f_hi + (size_t)N * Kp;
  float* t_hi = f_lo + (size_t)N * Kp;
  float* t_lo = t_hi + (size_t)K * Np;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;     // 32 x 8
  for (int r = ty; r < 32; r += 8) {
    const int n = n0 + r, k = k0 + tx;
    const float v = (n < N && k < K) ? w[(long long)n * K + k] : 0.f;
    tile[r][tx] = v;
    if (n < N && k < Kp) {
      const float hi = tf32_round(v);
      f_hi[(long long)n * Kp + k] = hi;
      f_lo[(long long)n * Kp + k] = tf32_round(v - hi);
    }
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int k = k0 + r, n = n0 + tx;
    if (k < K && n < Np) {
      const float v = tile[tx][r];
      const float hi = tf32_round(v);
      t_hi[(long long)k * Np + n] = hi;
      t_lo[(long long)k * Np + n] = tf32_round(v - hi);
    }
  }
}

// row-major [rows][cols] fp32 with a row pitch of `pitch` floats; box = {32 cols, box_rows}, 128-byte swizzle
static bool make_2d(CUtensorMap* m, const float* base, long long rows, long long cols, long long pitch, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)pitch * 4};
  cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstr, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static inline int round4(int v) { return (v + 3) & ~3; }

// C[M,Nout] = epi(A[M,R] . B[Nout,R]^T);  b_hi/b_lo are packed planes with row pitch round4(R)
static int launch_nt(const float* A, long long a_pitch, const float* b_hi, const float* b_lo, float* C, int M, int Nout, int R,
                     Epilogue ep, cudaStream_t st) {
  CUtensorMap ta, tbh, tbl;
  if (!make_2d(&ta, A, M, R, a_pitch, kBM)) return DV_ERR_CUDA;
  if (!make_2d(&tbh, b_hi, Nout, R, round4(R), kBN)) return DV_ERR_CUDA;
  if (!make_2d(&tbl, b_lo, Nout, R, round4(R), kBN)) return DV_ERR_CUDA;
  static bool attr = false;
  const int rc = set_max_dynamic_smem(linear_nt_mma_kernel, kSmemBytes, &attr);
  if (rc != DV_OK) return rc;
  dim3 grid((M + kBM - 1) / kBM, (Nout + kBN - 1) / kBN);
  linear_nt_mma_kernel<<<grid, kThreads, kSmemBytes, st>>>(ta, tbh, tbl, C, M, Nout, R, ep);
  return check_launch();
}

// the NT GEMM reads its activation rows through TMA: they need a 16-byte pitch, R % 4 == 0 (R = K forward, N dgrad)
bool nt_ok(int R) { return R % 4 == 0 && R >= 32; }

size_t packed_floats(int N, int K) { return (size_t)2 * N * round4(K) + (size_t)2 * K * round4(N); }

int pack_multi(int n, const float* const* w, float* const* packed, const int* N, const int* K, cudaStream_t st) {
  for (int base = 0; base < n; base += kPackMax) {
    PackTable t;
    t.n = n - base < kPackMax ? n - base : kPackMax;
    int tiles = 0;
    for (int i = 0; i < t.n; ++i) {
      t.w[i] = w[base + i]; t.dst[i] = packed[base + i]; t.N[i] = N[base + i]; t.K[i] = K[base + i];
      t.tiles_k[i] = (round4(K[base + i]) + 31) / 32;
      t.tile0[i] = tiles;
      tiles += t.tiles_k[i] * ((round4(N[base + i]) + 31) / 32);
    }
    t.tile0[t.n] = tiles;
    linear_pack_multi_kernel<<<tiles, 256, 0, st>>>(t);
    int rc = check_launch();
    if (rc != DV_OK) return rc;
  }
  return DV_OK;
}

// forward and input-gradient GEMMs on planes written by pack_multi
int fwd_packed(const float* x, const float* packed, const float* bias, float* y, int M, int N, int K, int act, float slope,
               cudaStream_t st) {
  const float* hi = packed;
  const float* lo = packed + (size_t)N * round4(K);
  Epilogue ep{bias, nullptr, act, slope};
  return launch_nt(x, K, hi, lo, y, M, N, K, ep, st);
}
int dgrad_packed(const float* g, const float* packed, const float* mask_src, float* dx, int M, int N, int K, int act, float slope,
                 cudaStream_t st) {
  const float* hi = packed + (size_t)2 * N * round4(K);
  const float* lo = hi + (size_t)K * round4(N);
  Epilogue ep{nullptr, mask_src, mask_src ? act : DV_ACT_NONE, slope};
  return launch_nt(g, N, hi, lo, dx, M, K, N, ep, st);
}

static void wgrad_plan(int M, int N, int K, int* S, int* tiles_per_split) {
  const int m_tiles = (M + 127) / 128;
  const int base = ((N + 31) / 32) * ((K + 63) / 64);
  int want = (kNumSMs + base - 1) / base;
  if (want > m_tiles) want = m_tiles;
  if (want < 1) want = 1;
  const int per = (m_tiles + want - 1) / want;
  *tiles_per_split = per;
  *S = (m_tiles + per - 1) / per;                             // no empty split
}
bool wgrad_ok(int M, int N, int K) { return N % 4 == 0 && K % 4 == 0 && K >= 32 && M >= 32; }
size_t wgrad_workspace_bytes(int M, int N, int K) {
  int S, per;
  wgrad_plan(M, N, K, &S, &per);
  return S > 1 ? ((size_t)S * N * K + (size_t)S * N) * sizeof(float) : 0;     // dW partials, then dbias partials
}
// returns the number of splits written (1: dw is final) through *nsplit
// dbias != NULL: the column sums of g come out of the same kernel (partials at ws + S*N*K when S > 1)
int wgrad(const float* g, const float* x, float* dw, float* dbias, float* ws, int M, int N, int K, int* nsplit, cudaStream_t st) {
  int S, per;
  wgrad_plan(M, N, K, &S, &per);
  CUtensorMap tx, tg;
  if (!make_2d(&tx, x, M, K, K, 128)) return DV_ERR_CUDA;
  if (!make_2d(&tg, g, M, N, N, 128)) return DV_ERR_CUDA;
  static bool attr = false;
  const int rc = set_max_dynamic_smem(linear_wgrad_mma_kernel, kWgSmemBytes, &attr);
  if (rc != DV_OK) return rc;
  WgGeom geo{M, N, K, (M + 127) / 128, per};
  dim3 grid((N + 31) / 32, (K + 63) / 64, S);
  float* dbias_base = !dbias ? nullptr : (S > 1 ? ws + (size_t)S * N * K : dbias);
  linear_wgrad_mma_kernel<<<grid, kThreads, kWgSmemBytes, st>>>(tx, tg, S > 1 ? ws : dw, (long long)N * K, dbias_base, (long long)N, geo);
  *nsplit = S;
  return check_launch();
}

}  // namespace ltc
}  // namespace dv

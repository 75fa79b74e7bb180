// Tensor-core implicit-GEMM convolutions for the 32-channel Burgess layers (sm_90a): down, up (halo-resident) and wgrad.
//
// Common scheme (details above each kernel):
//   * The operand that comes from the ACTIVATIONS is fetched by TMA tiled loads straight from the NHWC tensor -- for the
//     down kernel one load per tap with box {32 c, W cols, TR rows, TB images}, element strides {1,2,2,1} and start
//     coordinate (0, kw-1, 2*i0-1+kh, b0): the stride-2 gather and the zero padding (out-of-bounds fill) are done by the
//     TMA unit, nothing is im2col'ed in memory.  Every tile lands with the 128-byte swizzle, so the fragment loads of the
//     MMAs below are free of bank conflicts.
//   * fp32 parity on tf32 tensor cores: error-compensated 3xTF32 (dv_ptx.cuh).  The operands are split into hi/lo planes
//     in registers right after their fragment loads; the packed weights already hold both planes.
//   * warp roles (288 threads, 1 CTA/SM, persistent over tiles): warps 0-7 load fragments, run the MMAs and the
//     epilogue; warp 8 is the TMA producer.  mbarrier rings between them: raw-full (TMA transaction count) and
//     raw-empty (one arrival per consumer warp that reads the slot).  Warps 0-3 and 4-7 are two warpgroups of 64 MMA
//     rows issuing wgmma with A from registers and B from shared memory: the resident packed weights (down, up), or the
//     lo tile transposed and split once per tile by the consumer warps (wgrad).
#include "dv_common.cuh"
#include "dv_ptx.cuh"

namespace dv {
namespace tc {

using namespace ptx;

constexpr int kATile = 128 * 128;            // bytes: 128 pixel rows x 32 fp32
constexpr int kBTap = 64 * 128;              // bytes: (32 hi + 32 lo) rows x 32 fp32
constexpr int kBBytes = kTaps * kBTap;       // 131072
constexpr int kConsumers = 8;                // MMA / epilogue warps
constexpr int kThreads = (kConsumers + 1) * 32;
constexpr int kSmemMax = 232448;             // 227 KB per block on sm_90

__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumers * 32) : "memory"); }

// The two consumer warpgroups of the up kernel take their epilogues in turn, so that while one drains its
// accumulators and stores, the other has MMAs queued on the tensor cores.  Named barrier 2 passes the turn from
// warpgroup 0 to warpgroup 1, barrier 3 from 1 to 0; the passing warpgroup arrives, the other waits (128 + 128
// threads).  Every pass is followed by a wait of the passer before its next pass, so a barrier never collects two
// passes of one warpgroup.  Start-up: warpgroup 0 passes once in the middle of its first output phase and warpgroup 1
// waits for that before its first MMA, then passes straight back: warpgroup 1 runs half a phase behind.
// Warpgroup 0 takes the last pass with one more wait before it exits.
__device__ __forceinline__ void epilogue_turn_wait(int wg) { named_bar_sync(3 - wg, kConsumers * 32); }
__device__ __forceinline__ void epilogue_turn_pass(int wg) { named_bar_arrive(2 + wg, kConsumers * 32); }

// The ReLU-backward mask of output pixel p for this thread's channels (8 nt + 2 t + e) as a bit word: mask_bits[p]
// when given, else [mask > 0] of the float mask, else all ones (also for a pixel past the end).  Called ahead of the
// MMAs whose outputs it masks (down: before the tile's taps, up: before the phase's products), so the loads run under them.
__device__ __forceinline__ uint32_t mask_word(const uint32_t* __restrict__ mask_bits, const float* __restrict__ mask,
                                              long long p, bool valid, int t) {
  if (!valid || (!mask_bits && !mask)) return 0xffffffffu;
  if (mask_bits) return __ldg(mask_bits + p);
  uint32_t mb = 0u;
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const int c = nt * 8 + 2 * t;
    const float2 m2 = __ldg(reinterpret_cast<const float2*>(mask + p * 32 + c));
    mb |= (m2.x > 0.f ? 1u : 0u) << c | (m2.y > 0.f ? 1u : 0u) << (c + 1);
  }
  return mb;
}

// Once a product's commit groups are complete: its hi*hi is added to the fp32 total.  tot[4 nt + e] (like every
// accumulator here) is element e of n-tile nt in the m16n8 accumulator layout.
__device__ __forceinline__ void fold_tap(float (&tot)[16], float (&acc)[16]) {
  fence_regs(acc);
#pragma unroll
  for (int i = 0; i < 16; ++i) tot[i] += acc[i];
}

// 3xTF32 of one (activation tile, weight tap) product, K = 32 channels, on the warpgroup's tensor cores.
// A: rows p0 and p1 (this thread's MMA rows g and g + 8) of a swizzled [pixel][32 ch] tile at a_base, AND-ed with
// keep0 / keep1 (0 zeroes a row), split into hi and lo planes in registers.  B: the packed tap at tap_base,
// [32 hi | 32 lo rows][32 K].  Per k8: acc = A_hi.W_hi (overwritten by the first slice), corr += A_hi.W_lo + A_lo.W_hi
// (overwritten first when corr_accumulate == 0): the summation of the mma.sync kernels, where the correction products
// run across taps and hi*hi is folded into an fp32 total per tap.  (One m64n64k8 against [W_hi | W_lo] would issue the
// same work, but its 32 accumulators per thread, double-buffered, do not fit the 168 registers a 288-thread wgmma kernel
// gets: ptxas allocates whole warpgroups.)
// Every k8 slice is its own commit group, and the previous product (accumulating into acc_prev) is still in flight:
// before slice ks is loaded into ah/al[4 ks, 4 ks + 4), wait_group 3 completes slice ks of the previous product (the
// last reader of those registers), and before the last slice it completes the whole previous product, which is then
// folded.  So one register set of A fragments serves both products, and the fold runs beside this product's MMAs.
__device__ __forceinline__ void product(float (&acc)[16], float (&acc_prev)[16], float (&corr)[16], float (&tot)[16],
                                        uint32_t (&ah)[16], uint32_t (&al)[16], uint32_t a_base, int p0, int p1,
                                        uint32_t keep0, uint32_t keep1, int t, uint32_t tap_base, int corr_accumulate) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    wgmma_wait<3>();
    if (ks == 3) fold_tap(tot, acc_prev);
    split_tf32(lds32(a_base + swz128(p0, 8 * ks + t)) & keep0, ah[4 * ks + 0], al[4 * ks + 0]);
    split_tf32(lds32(a_base + swz128(p1, 8 * ks + t)) & keep1, ah[4 * ks + 1], al[4 * ks + 1]);
    split_tf32(lds32(a_base + swz128(p0, 8 * ks + t + 4)) & keep0, ah[4 * ks + 2], al[4 * ks + 2]);
    split_tf32(lds32(a_base + swz128(p1, 8 * ks + t + 4)) & keep1, ah[4 * ks + 3], al[4 * ks + 3]);
    fence_regs(acc);
    fence_regs(corr);
    wgmma_fence();
    const uint64_t w_hi = wgmma_desc_k128(tap_base + 32 * ks), w_lo = wgmma_desc_k128(tap_base + 32 * 128 + 32 * ks);
    wgmma_m64n32k8_rs(acc, ah + 4 * ks, w_hi, ks);
    wgmma_m64n32k8_rs(corr, ah + 4 * ks, w_lo, ks | corr_accumulate);
    wgmma_m64n32k8_rs(corr, al + 4 * ks, w_hi, 1);
    wgmma_commit();
  }
}

// ------------------------------------------------------------------------------------------
// down: lo[p][cl] = act(sum_{tap,c} hi(2i-1+kh, 2j-1+kw)[c] * w[cl][c][tap] + bias) * mask
//   M = 128 lo pixels per tile (warp w: rows [16w, 16w+16)), N = 32, K = 16 taps x 32 channels.
//   smem: weights (hi|lo, 128 KB) resident + a 5-stage ring of 16 KB tap tiles.
// ------------------------------------------------------------------------------------------
struct DownGeom {
  int B, H, W;          // lo geometry
  int rows_per_tile;    // 128 / W image-rows of lo per tile
  int num_tiles;
  long long total_px;
};
constexpr int kDownStages = 5;
struct DownBarriers {
  uint64_t raw_full[kDownStages], raw_empty[kDownStages];
  uint64_t b_full;
  float bias[32];
  float csum[kConsumers][32];
};
constexpr int kDownSmem = kBBytes + kDownStages * kATile + 1024 + 2048;
static_assert(sizeof(DownBarriers) <= 2048, "barrier block too large");
static_assert(kDownSmem <= kSmemMax, "smem");

__global__ void __launch_bounds__(kThreads, 1)
conv_down32_mma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const float* __restrict__ bias, const float* __restrict__ mask, float* __restrict__ lo,
                       DownGeom g, int act, float* __restrict__ colsum_part,
                       const uint32_t* __restrict__ mask_bits, uint32_t* __restrict__ bits_out) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* Bs = smem;
  uint8_t* Raw = smem + kBBytes;
  DownBarriers* bars = reinterpret_cast<DownBarriers*>(Raw + kDownStages * kATile);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kDownStages; ++s) { mbar_init(&bars->raw_full[s], 1); mbar_init(&bars->raw_empty[s], kConsumers); }
    mbar_init(&bars->b_full, 1);
    fence_mbar_init();
  }
  if (threadIdx.x < 32) bars->bias[threadIdx.x] = bias ? bias[threadIdx.x] : 0.f;
  __syncthreads();

  if (warp == kConsumers) {
    if (lane != 0) return;
    prefetch_tmap(&tmap_a); prefetch_tmap(&tmap_b);
    mbar_arrive_expect_tx(&bars->b_full, kBBytes);
    for (int tap = 0; tap < kTaps; ++tap) tma_load_2d(Bs + tap * kBTap, &tmap_b, &bars->b_full, 0, tap * 64);
    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
      const int r0 = tile * g.rows_per_tile;
      const int b0 = r0 / g.H, i0 = r0 % g.H;
      if (tile + (int)gridDim.x < g.num_tiles) {
        // the four taps (kh,kw) in {1,2}^2 touch every hi pixel of a tile exactly once: pull the NEXT tile into L2
        const int rn = (tile + gridDim.x) * g.rows_per_tile;
        const int bn = rn / g.H, in_ = rn % g.H;
        for (int t4 = 0; t4 < 4; ++t4) tma_prefetch_4d(&tmap_a, 0, (t4 & 1), 2 * in_ + (t4 >> 1), bn);
      }
      for (int tap = 0; tap < kTaps; ++tap) {
        const int kh = tap >> 2, kw = tap & 3;
        mbar_wait(&bars->raw_empty[stage], phase ^ 1);
        mbar_arrive_expect_tx(&bars->raw_full[stage], kATile);
        tma_load_4d(Raw + stage * kATile, &tmap_a, &bars->raw_full[stage], 0, kw - 1, 2 * i0 - 1 + kh, b0);
        if (++stage == kDownStages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  const int gq = lane >> 2, t = lane & 3;
  const int r0 = warp * 16 + gq;                             // this thread's tile rows: r0 and r0 + 8
  const uint32_t bs = smem_u32(Bs), raw0 = smem_u32(Raw);
  float csum[4][2] = {};                                     // channel sums of the stored output (colsum_part)
  mbar_wait(&bars->b_full, 0);
  int stage = 0; uint32_t phase = 0;
  uint32_t ah[16], al[16];
  // tap `tap` of the ring's current tile into acc while the previous tap (acc_prev) completes; the stage is free again
  // once its fragments are in registers
  auto tap_product = [&](float (&acc)[16], float (&acc_prev)[16], float (&corr)[16], float (&tot)[16], int tap) {
    mbar_wait(&bars->raw_full[stage], phase);
    product(acc, acc_prev, corr, tot, ah, al, raw0 + stage * kATile, r0, r0 + 8, ~0u, ~0u, t, bs + tap * kBTap, tap);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars->raw_empty[stage]);
    if (++stage == kDownStages) { stage = 0; phase ^= 1; }
  };
  for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
    // the ReLU-backward mask of this thread's two rows, one word per pixel (bit c = channel c), requested before the
    // tile's 16 taps so that its latency hides under them
    long long p[2];
    bool valid[2];
    uint32_t mb[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      p[h] = (long long)tile * 128 + r0 + 8 * h;
      valid[h] = p[h] < g.total_px;
      mb[h] = mask_word(mask_bits, mask, p[h], valid[h], t);
    }
    float tot[16] = {}, corr[16], acc[2][16];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[1][i] = 0.f;           // folded while tap 0 runs
#pragma unroll 1
    for (int tap = 0; tap < kTaps; tap += 2) {
      tap_product(acc[0], acc[1], corr, tot, tap);
      tap_product(acc[1], acc[0], corr, tot, tap + 1);
    }
    wgmma_wait<0>();
    fold_tap(tot, acc[1]);
    fence_regs(corr);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint32_t ob = 0u;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int c = nt * 8 + 2 * t;
        float v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float x = (tot[4 * nt + 2 * h + e] + corr[4 * nt + 2 * h + e]) + bars->bias[c + e];
          if (act == DV_ACT_RELU) x = fmaxf(x, 0.f);
          v[e] = ((mb[h] >> (c + e)) & 1u) ? x : 0.f;
        }
        if (valid[h]) *reinterpret_cast<float2*>(lo + p[h] * 32 + c) = make_float2(v[0], v[1]);
        else v[0] = v[1] = 0.f;
        ob |= (v[0] > 0.f ? 1u : 0u) << c | (v[1] > 0.f ? 1u : 0u) << (c + 1);
        csum[nt][0] += v[0]; csum[nt][1] += v[1];
      }
      ob |= __shfl_xor_sync(0xffffffffu, ob, 1);
      ob |= __shfl_xor_sync(0xffffffffu, ob, 2);
      if (bits_out && valid[h] && t == 0) bits_out[p[h]] = ob;  // [x > 0] of the stored pixel: the next backward pass's mask
    }
  }
  if (colsum_part) {                                         // fixed-order reduction: lanes of a quad column, then warps
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float s = csum[nt][e];
        s += __shfl_xor_sync(0xffffffffu, s, 4);
        s += __shfl_xor_sync(0xffffffffu, s, 8);
        s += __shfl_xor_sync(0xffffffffu, s, 16);
        if (gq == 0) bars->csum[warp][nt * 8 + 2 * t + e] = s;
      }
    consumers_sync();
    if (warp == 0) {
      float s = 0.f;
      for (int w = 0; w < kConsumers; ++w) s += bars->csum[w][lane];
      colsum_part[blockIdx.x * 32 + lane] = s;
    }
  }
}

// ------------------------------------------------------------------------------------------
// wgrad: dw[cl][c][tap] = sum_p lo[p][cl] * hi(2i-1+kh, 2j-1+kw)[c]   (reduction over PIXELS)
//   Per 128-pixel tile one GEMM per pair of taps: M = 64 (2 taps x 32 hi channels), N = 32 lo channels, K = 128 pixels
//   in 16 k8 slices.  Each warpgroup owns 8 taps: warpgroup wg runs the tap pairs (4j + 2wg, 4j + 2wg + 1), j = 0..3,
//   and inside a pair warps 0-1 hold the first tap (channels 0-15 / 16-31), warps 2-3 the second.
//   A (registers): the tap tiles, read transposed out of the swizzled [pixel][channel] TMA tile and split hi/lo.  K slot
//   t of a slice holds pixel 8ks + 2t and slot t + 4 pixel 8ks + 2t + 1: with the 128-byte swizzle the transposed loads
//   then hit 32 distinct banks.
//   B (shared memory): tf32 wgmma reads shared operands K-major only and the lo tile lands [pixel][channel], so once per
//   tile the consumer warps transpose it: warp w reads pixels [16w, 16w + 16) of channel `lane`, splits them and writes
//   the hi and the lo plane, each [32 channels][128 pixels] as four K-blocks of 32 pixels (4 KB, 128-byte rows, 128-byte
//   swizzle: what wgmma_desc_k128 describes), in the K-slot order of A.  The channel sums of lo (bias gradient) come
//   from the same registers.
//   Per (tile, tap pair): acc = A_hi.B_hi and corr = A_hi.B_lo + A_lo.B_hi accumulate over the 16 slices in the tensor
//   core, one commit group per slice, four slices of A fragments in flight; acc + corr is then added to the fp32
//   running totals, which live in shared memory, lane-interleaved (conflict-free).
//   Split-K over CTAs; the partials are reduced in a fixed order by conv_wgrad_reduce_kernel.
//   smem: 7-slot ring of 16 KB tap tiles (112 KB) + raw lo tile (16 KB) + hi/lo planes (32 KB) + barriers (2 KB) +
//   totals (64 KB) + 1 KB alignment slack = 227 KB.
// ------------------------------------------------------------------------------------------
constexpr int kWtSlots = 7;
constexpr int kWtPlane = 32 * 128 * 4;                 // bytes: one plane, [32 channels][128 pixels]
struct WtBarriers {
  uint64_t raw_full[kWtSlots], raw_empty[kWtSlots];
  uint64_t l_full, l_empty;
  float lsum[kConsumers][32];
};
constexpr int kWtTotFloats = 4 * 16 * 32;              // per consumer warp: [tap pair][16 accumulator values][lane]
constexpr int kWtSmem = kWtSlots * kATile + kATile + 2 * kWtPlane + 2048 + kConsumers * kWtTotFloats * 4 + 1024;
static_assert(sizeof(WtBarriers) <= 2048, "barrier block too large");
static_assert(kWtSmem <= kSmemMax, "smem");

struct WtGeom {
  int B, H, W, rows_per_tile, num_tiles, tiles_per_cta;
};

__global__ void __launch_bounds__(kThreads, 1)
conv_wgrad32_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_hi, const __grid_constant__ CUtensorMap tmap_lo,
                          float* __restrict__ ws, WtGeom g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* Raw = smem;                                       // [slot][128 px][32 ch]
  uint8_t* Ls = smem + kWtSlots * kATile;                    // [128 px][32 ch]
  uint8_t* Planes = Ls + kATile;                             // [hi / lo][K-block][32 ch][32 px]
  WtBarriers* bars = reinterpret_cast<WtBarriers*>(Planes + 2 * kWtPlane);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* tot = reinterpret_cast<float*>(Planes + 2 * kWtPlane + 2048) + warp * kWtTotFloats + lane;   // tot[k * 32]
  const int t_begin = blockIdx.x * g.tiles_per_cta;
  const int t_end = min(g.num_tiles, t_begin + g.tiles_per_cta);

  if (threadIdx.x == 0) {
    for (int s = 0; s < kWtSlots; ++s) { mbar_init(&bars->raw_full[s], 1); mbar_init(&bars->raw_empty[s], 2); }
    mbar_init(&bars->l_full, 1); mbar_init(&bars->l_empty, kConsumers);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kConsumers) {
    if (lane != 0) return;
    prefetch_tmap(&tmap_hi); prefetch_tmap(&tmap_lo);
    int slot = 0; uint32_t phase = 0, tseq = 0;
    for (int tile = t_begin; tile < t_end; ++tile, ++tseq) {
      const int r0 = tile * g.rows_per_tile;
      const int b0 = r0 / g.H, i0 = r0 % g.H;
      if (tile + 1 < t_end) {                                // pull the next tile's hi rows (and lo tile) into L2
        const int rn = (tile + 1) * g.rows_per_tile;
        const int bn = rn / g.H, in_ = rn % g.H;
        for (int t4 = 0; t4 < 4; ++t4) tma_prefetch_4d(&tmap_hi, 0, (t4 & 1), 2 * in_ + (t4 >> 1), bn);
        tma_prefetch_4d(&tmap_lo, 0, 0, in_, bn);
      }
      mbar_wait(&bars->l_empty, (tseq & 1u) ^ 1u);
      mbar_arrive_expect_tx(&bars->l_full, kATile);
      tma_load_4d(Ls, &tmap_lo, &bars->l_full, 0, 0, i0, b0);
      for (int tap = 0; tap < kTaps; ++tap) {                // the order the two warpgroups consume them in
        const int kh = tap >> 2, kw = tap & 3;
        mbar_wait(&bars->raw_empty[slot], phase ^ 1);
        mbar_arrive_expect_tx(&bars->raw_full[slot], kATile);
        tma_load_4d(Raw + slot * kATile, &tmap_hi, &bars->raw_full[slot], 0, kw - 1, 2 * i0 - 1 + kh, b0);
        if (++slot == kWtSlots) { slot = 0; phase ^= 1; }
      }
    }
    return;
  }

  const int gq = lane >> 2, t = lane & 3, wg = warp >> 2, wq = warp & 3;
  const uint32_t raw0 = smem_u32(Raw), l_base = smem_u32(Ls), planes = smem_u32(Planes);
  // A fragment {A[g][t], A[g+8][t], A[g][t+4], A[g+8][t+4]} of slice ks = the tap tile at (pixel 8ks + 2t, c),
  // (8ks + 2t, c + 8), (8ks + 2t + 1, c), (8ks + 2t + 1, c + 8): 1024 ks bytes past these offsets
  const int c0 = (wq & 1) * 16 + gq;
  const uint32_t a_off[4] = {swz128(2 * t, c0), swz128(2 * t, c0 + 8), swz128(2 * t + 1, c0), swz128(2 * t + 1, c0 + 8)};
  for (int k = 0; k < 64; ++k) tot[k * 32] = 0.f;          // k = tap pair * 16 + accumulator index
  float lsum = 0.f;                                          // lo channel `lane` over this warp's 16 rows of every tile
  uint32_t tseq = 0;
  for (int tile = t_begin; tile < t_end; ++tile, ++tseq) {
    mbar_wait(&bars->l_full, tseq & 1u);
    consumers_sync();                                        // every warp's MMAs of the previous tile have read the planes
    {
      uint32_t v[16];
#pragma unroll
      for (int r = 0; r < 16; ++r) v[r] = lds32(l_base + swz128(warp * 16 + r, lane));
#pragma unroll
      for (int r = 0; r < 16; ++r) lsum += __uint_as_float(v[r]);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->l_empty);            // the raw tile is in registers
      // slice ks = 2 warp + h, pixels 8ks + 2q + par -> K columns 8 (ks & 3) + 4 par + q of K-block ks >> 2: one 16-byte
      // chunk of row `lane` per (h, par)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int par = 0; par < 2; ++par) {
          const int ks = 2 * warp + h;
          uint32_t ph[4], pl[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) split_tf32(v[8 * h + 2 * q + par], ph[q], pl[q]);
          const uint32_t dst = planes + (ks >> 2) * 4096 + swz128(lane, 8 * (ks & 3) + 4 * par);
          sts128(dst, ph);
          sts128(dst + kWtPlane, pl);
        }
    }
    fence_proxy_async();
    consumers_sync();
#pragma unroll 1
    for (int j = 0; j < 4; ++j) {
      const uint32_t n = tseq * kTaps + 4 * j + 2 * wg + (wq >> 1);      // this warp's tap tile in the producer's sequence
      const uint32_t slot = n % kWtSlots;
      mbar_wait(&bars->raw_full[slot], (n / kWtSlots) & 1u);
      const uint32_t a_base = raw0 + slot * kATile;
      float acc[16], corr[16];
      uint32_t ah[16], al[16];
#pragma unroll 1
      for (int kb = 0; kb < 4; ++kb) {
#pragma unroll
        for (int k4 = 0; k4 < 4; ++k4) {
          const int ks = 4 * kb + k4;
          wgmma_wait<3>();                                   // slice ks - 4, the last reader of these A registers
#pragma unroll
          for (int e = 0; e < 4; ++e) split_tf32(lds32(a_base + 1024 * ks + a_off[e]), ah[4 * k4 + e], al[4 * k4 + e]);
          fence_regs(acc);
          fence_regs(corr);
          wgmma_fence();
          const uint64_t b_hi = wgmma_desc_k128(planes + kb * 4096 + 32 * k4), b_lo = wgmma_desc_k128(planes + kWtPlane + kb * 4096 + 32 * k4);
          wgmma_m64n32k8_rs(acc, ah + 4 * k4, b_hi, ks);
          wgmma_m64n32k8_rs(corr, ah + 4 * k4, b_lo, ks);
          wgmma_m64n32k8_rs(corr, al + 4 * k4, b_hi, 1);
          wgmma_commit();
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->raw_empty[slot]);    // the tap tile is in registers
      wgmma_wait<0>();
      fence_regs(acc);
      fence_regs(corr);
#pragma unroll
      for (int i = 0; i < 16; ++i) tot[(j * 16 + i) * 32] += acc[i] + corr[i];
    }
  }

  // accumulator i = 4 nt + 2 h + e of tap pair j: tap 4j + 2wg + (wq >> 1), c = c0 + 8 h, cl = 8 nt + 2 t + e
  float* out = ws + (long long)blockIdx.x * (kTaps * 32 + 1) * kLoCh;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int tap = 4 * j + 2 * wg + (wq >> 1);
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        *reinterpret_cast<float2*>(out + (tap * 32 + c0 + 8 * h) * kLoCh + nt * 8 + 2 * t) =
            make_float2(tot[(j * 16 + 4 * nt + 2 * h) * 32], tot[(j * 16 + 4 * nt + 2 * h + 1) * 32]);
  }
  bars->lsum[warp][lane] = lsum;                             // bias gradient: channel sums of lo, fixed order
  consumers_sync();
  if (warp == 0) {
    float s = 0.f;
    for (int w = 0; w < kConsumers; ++w) s += bars->lsum[w][lane];
    out[(kTaps * 32) * kLoCh + lane] = s;
  }
}

// ==========================================================================================
// up, halo-resident ("one load per input pixel"), CH == 32:
// The nine shifted operand tiles of the up convolution overlap almost completely, so instead of
// nine TMA loads per 128 positions ONE tile with a row halo [TB images][(TR+2) rows][W cols][32 ch] is
// loaded per tile (box start row i0-1: the rows above / below the image are TMA out-of-bounds fill).
// The 128 MMA rows enumerate the TB*TR*W valid lo pixels, so the operand of shift (di,dj) is the resident
// pixel (row + di, col + dj) (a column shift that leaves the image row yields zero).  Shift (di,dj) feeds the
// output phase (ph,pw) through tap (ph+1-2di, pw+1-2dj) when that tap exists: four accumulators of N = 32 per
// row, one per phase, weights 128 KB resident.  (The image-boundary layer, CH in {1,3}, is not a tensor-core
// problem: dv_conv_img.cu.)
// ==========================================================================================
constexpr int kHaloStageBytes = 26 * 1024;      // 208 pixel rows: the largest box of the supported geometries is 192 px
constexpr int kHaloStages = 3;
struct HaloGeom {
  int B, H, W, TR, TB, tiles_per_img, num_tiles, valid_rows, box_px, box_bytes;
};
struct HaloBarriers {
  uint64_t raw_full[kHaloStages], raw_empty[kHaloStages];
  uint64_t b_full;
  float bias[32];
};
constexpr int kHaloSmem = kBBytes + kHaloStages * kHaloStageBytes + 1024 + 1024;
static_assert(sizeof(HaloBarriers) <= 1024, "barrier block too large");
static_assert(kHaloSmem <= kSmemMax, "smem");

__global__ void __launch_bounds__(kThreads, 1)
conv_up_halo_mma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                        const float* __restrict__ bias, const float* __restrict__ mask, float* __restrict__ hi_out,
                        HaloGeom g, int act, const uint32_t* __restrict__ mask_bits, uint32_t* __restrict__ bits_out) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* Bs = smem;
  uint8_t* Raw = smem + kBBytes;
  HaloBarriers* bars = reinterpret_cast<HaloBarriers*>(Raw + kHaloStages * kHaloStageBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kHaloStages; ++s) { mbar_init(&bars->raw_full[s], 1); mbar_init(&bars->raw_empty[s], kConsumers); }
    mbar_init(&bars->b_full, 1);
    fence_mbar_init();
  }
  if (threadIdx.x < 32) bars->bias[threadIdx.x] = bias ? bias[threadIdx.x] : 0.f;
  __syncthreads();

  if (warp == kConsumers) {
    if (lane != 0) return;
    prefetch_tmap(&tmap_a); prefetch_tmap(&tmap_b);
    mbar_arrive_expect_tx(&bars->b_full, kBBytes);
    for (int tap = 0; tap < kTaps; ++tap) tma_load_2d(Bs + tap * kBTap, &tmap_b, &bars->b_full, 0, tap * 64);
    uint32_t t_seq = 0;
    for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x, ++t_seq) {
      const int stage = t_seq % kHaloStages;
      int b0, i0;
      if (g.TB > 1) { b0 = tile * g.TB; i0 = 0; } else { b0 = tile / g.tiles_per_img; i0 = (tile % g.tiles_per_img) * g.TR; }
      mbar_wait(&bars->raw_empty[stage], ((t_seq / kHaloStages) & 1u) ^ 1u);
      mbar_arrive_expect_tx(&bars->raw_full[stage], g.box_bytes);
      tma_load_4d(Raw + stage * kHaloStageBytes, &tmap_a, &bars->raw_full[stage], 0, 0, i0 - 1, b0);
    }
    return;
  }

  const int gq = lane >> 2, t = lane & 3;
  const int HH = 2 * g.H, WW = 2 * g.W;
  const uint32_t bs = smem_u32(Bs), raw0 = smem_u32(Raw);
  // the two MMA rows of this thread (r = 16*warp + gq + 8h): centre pixel inside the resident box [TB][TR+2][W]
  int rj[2], src0[2];
  bool row_ok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = warp * 16 + gq + 8 * h;
    const int rt = row / g.W, rtb = rt / g.TR;
    rj[h] = row - rt * g.W;
    src0[h] = min((rtb * (g.TR + 2) + (rt - rtb * g.TR) + 1) * g.W + rj[h], g.box_px - 1);
    row_ok[h] = row < g.valid_rows;
  }
  uint32_t ah[16], al[16];
  mbar_wait(&bars->b_full, 0);
  const int wg = warp >> 2;
  if (wg == 1) { epilogue_turn_wait(1); epilogue_turn_pass(1); }
  bool lead = wg == 0;                                       // warpgroup 0 before its start-up pass
  uint32_t t_seq = 0;
  for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x, ++t_seq) {
    const int stage = t_seq % kHaloStages;
    const uint32_t a_base = raw0 + stage * kHaloStageBytes;
    mbar_wait(&bars->raw_full[stage], (t_seq / kHaloStages) & 1u);
    int b0, i0;
    if (g.TB > 1) { b0 = tile * g.TB; i0 = 0; } else { b0 = tile / g.tiles_per_img; i0 = (tile % g.tiles_per_img) * g.TR; }
    // one output phase (ph, pw) at a time: its four (shift, tap) products, shift (di, dj) = (ph - 1 + (q >> 1),
    // pw - 1 + (q & 1)) through tap (3 - ph - 2 (q >> 1), 3 - pw - 2 (q & 1)); hi*hi added to the fp32 total after
    // every product, the correction products in their own total.
#pragma unroll 1
    for (int pidx = 0; pidx < 4; ++pidx) {
      const int ph = pidx >> 1, pw = pidx & 1;
      // output pixel of this thread's row h in this phase (valid: inside the batch and the tile's rows)
      auto out_pixel = [&](int h, bool& valid) -> long long {
        const int r = warp * 16 + gq + 8 * h, tr = r / g.W;
        const int tb = tr / g.TR, rr = tr - tb * g.TR;
        const int b = b0 + tb, i = i0 + rr, j = r - tr * g.W;
        valid = r < g.valid_rows && b < g.B && i < g.H;
        return valid ? ((long long)(b * HH + 2 * i + ph) * WW + 2 * j + pw) : 0;
      };
      uint32_t mb[2];                                        // requested before the phase's products, used after them
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        bool valid;
        const long long opix = out_pixel(h, valid);
        mb[h] = mask_word(mask_bits, mask, opix, valid, t);
      }
      float tot[16] = {}, corr[16], acc[2][16];
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[1][i] = 0.f;         // folded while product 0 runs
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int di = ph - 1 + (q >> 1), dj = pw - 1 + (q & 1);
        const uint32_t b_base = bs + ((3 - ph - 2 * (q >> 1)) * 4 + 3 - pw - 2 * (q & 1)) * kBTap;
        int p[2];
        uint32_t keep[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const bool ok = row_ok[h] && (unsigned)(rj[h] + dj) < (unsigned)g.W;
          p[h] = ok ? src0[h] + di * g.W + dj : src0[h];
          keep[h] = ok ? 0xffffffffu : 0u;
        }
        product(acc[q & 1], acc[(q + 1) & 1], corr, tot, ah, al, a_base, p[0], p[1], keep[0], keep[1], t, b_base, q);
        if (q == 1 && lead) { epilogue_turn_pass(0); lead = false; }
      }
      epilogue_turn_wait(wg);
      wgmma_wait<0>();
      fold_tap(tot, acc[1]);
      fence_regs(corr);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        bool valid;
        const long long opix = out_pixel(h, valid);
        uint32_t ob = 0u;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int c = nt * 8 + 2 * t;
          float v[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float x = (tot[4 * nt + 2 * h + e] + corr[4 * nt + 2 * h + e]) + bars->bias[c + e];
            if (act == DV_ACT_RELU) x = fmaxf(x, 0.f);
            v[e] = ((mb[h] >> (c + e)) & 1u) ? x : 0.f;
          }
          if (valid) *reinterpret_cast<float2*>(hi_out + opix * 32 + c) = make_float2(v[0], v[1]);
          ob |= (v[0] > 0.f ? 1u : 0u) << c | (v[1] > 0.f ? 1u : 0u) << (c + 1);
        }
        ob |= __shfl_xor_sync(0xffffffffu, ob, 1);
        ob |= __shfl_xor_sync(0xffffffffu, ob, 2);
        if (bits_out && valid && t == 0) bits_out[opix] = ob;  // [x > 0] of the stored pixel
      }
      epilogue_turn_pass(wg);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars->raw_empty[stage]);
  }
  if (wg == 0) epilogue_turn_wait(0);
}

// ---- weight packing ----------------------------------------------------------------------
// Every conv layer of a network node in ONE launch (blockIdx.y = layer), w[cl][c][tap] ->
//   CH == 32:     down section Wd[tap][row][c] at wp,  row < 32: hi (nearest tf32) of w[row][c][tap], row >= 32: lo;
//                 up section   Wu[tap][row][cl] at wp + 16*64*32,  row < 32: hi of w[cl][row][tap], row >= 32: lo
//   CH in {1,3}:  the fp32 layout [tap*CH + c][cl] of the dv_conv_img.cu kernels, twice (down section, up section)
constexpr int kPackMultiMax = 8;
struct ConvPackTable {
  const float* w[kPackMultiMax];
  float* wp[kPackMultiMax];
  int CH[kPackMultiMax];
};
__global__ void conv_pack_multi_kernel(ConvPackTable tab) {
  const float* __restrict__ w = tab.w[blockIdx.y];
  float* __restrict__ wp = tab.wp[blockIdx.y];
  const int CH = tab.CH[blockIdx.y];
  const int n = kLoCh * CH * kTaps;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += gridDim.x * blockDim.x) {
    const int tap = idx % kTaps, c = (idx / kTaps) % CH, cl = idx / (kTaps * CH);
    const float v = w[idx];
    if (CH != 32) {
      wp[(tap * CH + c) * kLoCh + cl] = v;
      wp[n + (tap * CH + c) * kLoCh + cl] = v;
      continue;
    }
    float* wd = wp;
    float* wu = wp + kTaps * 64 * 32;
    const float hi = tf32_round(v);
    const float lo = tf32_round(v - hi);
    wd[(tap * 64 + cl) * 32 + c] = hi;
    wd[(tap * 64 + 32 + cl) * 32 + c] = lo;
    wu[(tap * 64 + c) * 32 + cl] = hi;
    wu[(tap * 64 + 32 + c) * 32 + cl] = lo;
  }
}

// ---- host side ---------------------------------------------------------------------------
// NHWC activation [B][HH][WW][32] fp32; box = {32, bw, bh, bb} traversed with element strides {1, sw, sh, 1}, 128-byte swizzle
static bool make_act_tmap(CUtensorMap* m, const float* base, int B, int HH, int WW, int bw, int bh, int bb, int stride) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t gdim[4] = {32, (cuuint64_t)WW, (cuuint64_t)HH, (cuuint64_t)B};
  cuuint64_t gstr[3] = {128, (cuuint64_t)WW * 128, (cuuint64_t)HH * WW * 128};
  cuuint32_t box[4] = {32, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bb};
  cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base), gdim, gstr, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// packed weights [16*64 rows][32] fp32, box = one tap (64 rows)
static bool make_w_tmap(CUtensorMap* m, const float* base) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t gdim[2] = {32, (cuuint64_t)kTaps * 64};
  cuuint64_t gstr[1] = {128};
  cuuint32_t box[2] = {32, 64};
  cuuint32_t estr[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstr, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

int pack_multi(int n, const float* const* w, float* const* wp, const int* CH, cudaStream_t st) {
  for (int base = 0; base < n; base += kPackMultiMax) {
    ConvPackTable tab = {};
    const int m = n - base < kPackMultiMax ? n - base : kPackMultiMax;
    for (int i = 0; i < m; ++i) { tab.w[i] = w[base + i]; tab.wp[i] = wp[base + i]; tab.CH[i] = CH[base + i]; }
    conv_pack_multi_kernel<<<dim3(16, m), 256, 0, st>>>(tab);
    const int rc = check_launch();
    if (rc != DV_OK) return rc;
  }
  return DV_OK;
}

// lo[B,H,W,32] = act(down(hi[B,2H,2W,32]) + bias) * [mask > 0]
// colsum_part != NULL: the kernel also leaves per-CTA channel sums of `lo` in colsum_part[grid][32] and sets
// *nparts = grid.
int conv_down32_tc(const float* hi, const float* wd_packed, const float* bias, const float* mask, float* lo,
                   int B, int H, int W, int act, cudaStream_t st, float* colsum_part, int* nparts,
                   const uint32_t* mask_bits, uint32_t* bits_out) {
  if (nparts) *nparts = 0;
  if (W > 128 || 128 % W != 0) return DV_ERR_BAD_SHAPE;
  DownGeom g = {};
  g.B = B; g.H = H; g.W = W;
  g.rows_per_tile = 128 / W;
  const int TR = g.rows_per_tile < H ? g.rows_per_tile : H;
  if (H % TR != 0 || g.rows_per_tile % TR != 0) return DV_ERR_BAD_SHAPE;
  const int TB = g.rows_per_tile / TR;
  g.total_px = (long long)B * H * W;
  g.num_tiles = (int)((g.total_px + 127) / 128);
  CUtensorMap ta, tb;
  if (!make_act_tmap(&ta, hi, B, 2 * H, 2 * W, 2 * W, 2 * TR, TB, 2)) return DV_ERR_CUDA;
  if (!make_w_tmap(&tb, wd_packed)) return DV_ERR_CUDA;
  static bool attr = false;
  const int rc = set_max_dynamic_smem(conv_down32_mma_kernel, kDownSmem, &attr);
  if (rc != DV_OK) return rc;
  const int grid = g.num_tiles < kNumSMs ? g.num_tiles : kNumSMs;
  conv_down32_mma_kernel<<<grid, kThreads, kDownSmem, st>>>(ta, tb, bias, mask, lo, g, act, colsum_part, mask_bits, bits_out);
  if (nparts && colsum_part) *nparts = grid;
  return check_launch();
}

// CTAs of conv_wgrad32_wgmma_kernel, one split-K partial each: at most one per SM, no empty CTA
int wgrad_splits(int B, int H, int W) {
  const int num_tiles = (int)(((long long)B * H * W + 127) / 128);
  const int grid = num_tiles < kNumSMs ? num_tiles : kNumSMs;
  const int tiles_per_cta = (num_tiles + grid - 1) / grid;
  return (num_tiles + tiles_per_cta - 1) / tiles_per_cta;
}

// partial sums of dw (and of lo, last row) per CTA into ws[wgrad_splits(B, H, W)][16*32+1][32]
int conv_wgrad32_tc(const float* lo, const float* hi, float* ws, int B, int H, int W, cudaStream_t st) {
  if (W > 128 || 128 % W != 0) return DV_ERR_BAD_SHAPE;
  WtGeom g = {};
  g.B = B; g.H = H; g.W = W;
  g.rows_per_tile = 128 / W;
  const int TR = g.rows_per_tile < H ? g.rows_per_tile : H;
  if (H % TR != 0 || g.rows_per_tile % TR != 0) return DV_ERR_BAD_SHAPE;
  const int TB = g.rows_per_tile / TR;
  g.num_tiles = (int)(((long long)B * H * W + 127) / 128);
  const int grid = wgrad_splits(B, H, W);
  g.tiles_per_cta = (g.num_tiles + grid - 1) / grid;
  CUtensorMap thi, tlo;
  if (!make_act_tmap(&thi, hi, B, 2 * H, 2 * W, 2 * W, 2 * TR, TB, 2)) return DV_ERR_CUDA;
  if (!make_act_tmap(&tlo, lo, B, H, W, W, TR, TB, 1)) return DV_ERR_CUDA;
  static bool attr = false;
  const int rc = set_max_dynamic_smem(conv_wgrad32_wgmma_kernel, kWtSmem, &attr);
  if (rc != DV_OK) return rc;
  conv_wgrad32_wgmma_kernel<<<grid, kThreads, kWtSmem, st>>>(thi, tlo, ws, g);
  return check_launch();
}

// hi[B,2H,2W,32] = act(up(lo[B,H,W,32]) + bias) * [mask > 0]
int conv_up_halo(const float* lo, const float* wu, const float* bias, const float* mask, float* hi,
                 int B, int H, int W, int act, cudaStream_t st, const uint32_t* mask_bits, uint32_t* bits_out) {
  HaloGeom g = {};
  g.B = B; g.H = H; g.W = W;
  if (W > 32 || 128 % W != 0) return DV_ERR_BAD_SHAPE;
  // 128 MMA rows = 128 / W image rows of W pixels: whole rows of one image (TB = 1) or whole small images (TB > 1)
  const int rpt = 128 / W;
  if (rpt >= H) {
    g.TR = H;
    g.TB = rpt / H < 1 ? 1 : rpt / H;
    while (g.TB > 1 && g.TB * (H + 2) * W * 128 > kHaloStageBytes) --g.TB;
    g.tiles_per_img = 1;
    g.num_tiles = (B + g.TB - 1) / g.TB;
  } else {
    g.TR = rpt; g.TB = 1;
    g.tiles_per_img = (H + rpt - 1) / rpt;
    g.num_tiles = B * g.tiles_per_img;
  }
  g.valid_rows = g.TB * g.TR * W;
  g.box_px = g.TB * (g.TR + 2) * W;
  g.box_bytes = g.box_px * 128;
  if (g.box_bytes > kHaloStageBytes) return DV_ERR_BAD_SHAPE;
  CUtensorMap ta, tb;
  if (!make_act_tmap(&ta, lo, g.B, g.H, g.W, g.W, g.TR + 2, g.TB, 1)) return DV_ERR_CUDA;
  if (!make_w_tmap(&tb, wu)) return DV_ERR_CUDA;
  static bool attr = false;
  const int rc = set_max_dynamic_smem(conv_up_halo_mma_kernel, kHaloSmem, &attr);
  if (rc != DV_OK) return rc;
  const int grid = g.num_tiles < kNumSMs ? g.num_tiles : kNumSMs;
  conv_up_halo_mma_kernel<<<grid, kThreads, kHaloSmem, st>>>(ta, tb, bias, mask, hi, g, act, mask_bits, bits_out);
  return check_launch();
}

}  // namespace tc
}  // namespace dv

// Image-boundary layers of the Burgess networks on the CUDA cores: the first Conv2d of the encoder and the last
// ConvTranspose2d of the decoder (encoders.py:54-55,72; decoders.py:58-59,82), whose "hi" side is the image itself
// (CH = 1 or 3 channels, NCHW) and whose "lo" side is the 32-channel NHWC activation.
//
// With K = 16*CH these layers have ~1/30 of the arithmetic intensity of the 32->32 layers: 2*512*CH FLOP per lo
// pixel against 128 B (lo) + 16*CH B (hi) of compulsory traffic, i.e. they are pure HBM streaming problems (151 MB per
// launch at B = 1024, 1x64x64) whose whole arithmetic (1.07 GFLOP) is small next to that traffic.  Tensor-core
// variants would pay for operand staging they cannot amortise (im2col gather, hi/lo splitting, three tensor passes);
// these kernels do exact fp32 FMAs from shared-memory tiles with register blocking instead:
//
//   down  (Conv2d fwd, ConvTranspose2d dgrad): thread = 8 (4) consecutive output pixels x 8 output channels; the image
//         tile (with halo and zero padding) in shared memory, one 18-value input row segment per kernel row, two LDS.128
//         of weights per tap for 64 FMAs; bias / ReLU / ReLU-mask (prefetched as bits) epilogue, a lane quartet stores
//         64 contiguous bytes; optional channel sums of the stored tile (the previous ConvTranspose2d's bias gradient).
//   up    (ConvTranspose2d fwd, NCHW + sigmoid): thread = a block of PY x 2 lo positions -> (2PY) x 4 output pixels per
//         channel; the 32-channel lo tile (16-byte chunks XOR-swizzled by the column: conflict-free LDS.128 for a
//         2-pixel lane stride) with a 1-pixel halo in shared memory; per 4-channel chunk (PY+2) x 4 neighbour float4
//         serve 2*PY*16*4*CH FMAs; float4 row stores.
//   All tiles arrive by cp.async (every copy of a tile in flight at once).
//   wgrad (both weight gradients + the lo-side bias gradient): a "stream" of 16 threads owns the whole 32 x 16*CH
//         output (thread = 4 lo channels x 8 taps x CH) in registers and walks over pixels (1 LDS.128 + 4*CH LDS.64 per
//         32*CH FMAs); 16 streams per CTA, persistent CTAs, one ordered cross-stream reduction at the end, partials in
//         the layout conv_wgrad_reduce_kernel already consumes (deterministic).
//
// Geometry handled here: square images of 32 or 64 pixels (lo W = H in {16, 32}), CH in {1, 3} -- every image-boundary
// layer the shape check of dv_conv.cu accepts.
#include "dv_common.cuh"

namespace dv {
namespace img {

constexpr int kThreads = 256;
constexpr int kLoPitch = 36;                 // floats per lo pixel in shared memory (32 + 4: 16-byte groups rotate)

// Tiles are brought in with cp.async (global -> shared without a register round trip): a thread issues ALL its copies
// back to back, so the whole tile is in flight at once.  (A plain "load, then store" loop kept ONE load per thread in
// flight: 16-38 dependent round trips to HBM per tile, 4x the time of everything else in these kernels.)
// src-size 0 = zero fill (padding / halo outside the image); the source pointer is then any valid address.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  const int sz = valid ? 4 : 0;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// hi tile: rows 2*i0-1 .. 2*i0+2*TR of image b, columns -1 .. 2W (in-tile column = x + 1), zero outside the image
template <int CH, int W, int TR>
__device__ __forceinline__ void load_hi_tile(float* __restrict__ s_hi, const float* __restrict__ hi, int b, int i0, int H) {
  constexpr int IN_ROWS = 2 * TR + 2, COLS = 2 * W + 2, PITCH = 2 * W + 4;
  const int HH = 2 * H, WW = 2 * W;
#pragma unroll 4
  for (int e = threadIdx.x; e < CH * IN_ROWS * COLS; e += kThreads) {
    const int xx = e % COLS, rr = (e / COLS) % IN_ROWS, c = e / (COLS * IN_ROWS);
    const int iy = 2 * i0 - 1 + rr, ix = xx - 1;
    const bool ok = (unsigned)iy < (unsigned)HH && (unsigned)ix < (unsigned)WW;
    cp_async4(s_hi + (c * IN_ROWS + rr) * PITCH + xx, ok ? hi + ((long long)(b * CH + c) * HH + iy) * WW + ix : hi, ok);
  }
}

// ------------------------------------------------------------------------------------------------------------
// down: thread = PXG consecutive output pixels of a row x 8 output channels {4cg..4cg+3, 16+4cg..16+4cg+3}
// (4 threads cover the 32 channels of a pixel group; 256 threads = one 16-row tile).  Per input row kh the thread
// fetches the 2*PXG+2 input values its pixels share (broadcast among the 4 channel threads) and per tap two LDS.128
// of weights feed 8*PXG FMAs -- ~1 shared-memory instruction per 14 FMAs.  (The first mapping, 2 pixels x 32
// channels per thread, needed one LDS.128 per 8 FMAs and was bound by the LSU queue.)  A lane quartet writes 64 contiguous bytes per store instruction (whole sectors).
// ------------------------------------------------------------------------------------------------------------
template <int CH, int W>
__global__ void __launch_bounds__(kThreads, 2)
img_down_kernel(const float* __restrict__ hi, const float* __restrict__ wd, const float* __restrict__ bias,
                const float* __restrict__ mask, float* __restrict__ lo, int B, int H, int act,
                float* __restrict__ colsum_part, const uint32_t* __restrict__ mask_bits, uint32_t* __restrict__ bits_out) {
  constexpr int TR = 16;                       // output rows per tile
  constexpr int PXG = (TR * W) / 64;           // pixels per thread: 8 (W = 32), 4 (W = 16)
  constexpr int CB = W / PXG;                  // pixel groups per row (4)
  constexpr int NX = 2 * PXG + 2;              // input values per input row and pixel group
  constexpr int IN_ROWS = 2 * TR + 2, PITCH = 2 * W + 4;
  __shared__ __align__(16) float s_w[kTaps * CH * kLoCh];
  __shared__ __align__(16) float s_hi[CH * IN_ROWS * PITCH];
  __shared__ __align__(16) float s_bias[kLoCh];
  __shared__ float s_cs[kThreads / 32][kLoCh];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < kTaps * CH * kLoCh; i += kThreads) s_w[i] = wd[i];
  if (tid < kLoCh) s_bias[tid] = bias ? bias[tid] : 0.f;
  const int cg = tid & 3, pg = tid >> 2;       // channel group, pixel group (0..63)
  const int r_thr = pg / CB, c0 = (pg % CB) * PXG;
  const int tiles_per_img = H / TR;
  const int num_tiles = B * tiles_per_img;
  float csum[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) csum[k] = 0.f;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int b = tile / tiles_per_img, i0 = (tile % tiles_per_img) * TR;
    __syncthreads();                                           // previous tile fully consumed (and weights staged)
    load_hi_tile<CH, W, TR>(s_hi, hi, b, i0, H);
    const long long p0 = ((long long)b * H + i0 + r_thr) * W + c0;          // first pixel of the group
    // ReLU-backward mask of this thread's 8 channels x PXG pixels as bits, requested BEFORE the FMAs
    uint32_t mb_lo = 0xffffffffu, mb_hi = 0xffffffffu;                      // bit (4*i + e): pixel i, channels 4cg+e / 16+4cg+e
    if (mask_bits) {                                           // the mask already as one word per pixel (bit c = channel c)
      mb_lo = 0u; mb_hi = 0u;
#pragma unroll
      for (int i = 0; i < PXG; ++i) {
        const uint32_t mw = __ldg(mask_bits + p0 + i);
        mb_lo |= ((mw >> (4 * cg)) & 15u) << (4 * i);
        mb_hi |= ((mw >> (16 + 4 * cg)) & 15u) << (4 * i);
      }
    } else if (mask) {
      mb_lo = 0u; mb_hi = 0u;
#pragma unroll
      for (int i = 0; i < PXG; ++i) {
        const float* mk = mask + (p0 + i) * kLoCh + 4 * cg;
        const float4 a = ldg4(mk), d = ldg4(mk + 16);
        mb_lo |= ((a.x > 0.f ? 1u : 0u) | (a.y > 0.f ? 2u : 0u) | (a.z > 0.f ? 4u : 0u) | (a.w > 0.f ? 8u : 0u)) << (4 * i);
        mb_hi |= ((d.x > 0.f ? 1u : 0u) | (d.y > 0.f ? 2u : 0u) | (d.z > 0.f ? 4u : 0u) | (d.w > 0.f ? 8u : 0u)) << (4 * i);
      }
    }
    cp_async_wait_all();
    __syncthreads();
    float acc[PXG][8];
#pragma unroll
    for (int i = 0; i < PXG; ++i)
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[i][k] = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
#pragma unroll
      for (int kh = 0; kh < 4; ++kh) {
        float x[NX];
        const float* row = s_hi + (c * IN_ROWS + 2 * r_thr + kh) * PITCH + 2 * c0;    // in-tile column of input col 2*c0 - 1
#pragma unroll
        for (int v = 0; v < NX / 2; ++v) {
          const float2 t2 = *reinterpret_cast<const float2*>(row + 2 * v);
          x[2 * v] = t2.x; x[2 * v + 1] = t2.y;
        }
#pragma unroll
        for (int kw = 0; kw < 4; ++kw) {
          const float* wp = s_w + ((kh * 4 + kw) * CH + c) * kLoCh + 4 * cg;
          const float4 wa = *reinterpret_cast<const float4*>(wp), wb = *reinterpret_cast<const float4*>(wp + 16);
#pragma unroll
          for (int i = 0; i < PXG; ++i) {
            const float xv = x[2 * i + kw];
            acc[i][0] = fmaf(xv, wa.x, acc[i][0]); acc[i][1] = fmaf(xv, wa.y, acc[i][1]);
            acc[i][2] = fmaf(xv, wa.z, acc[i][2]); acc[i][3] = fmaf(xv, wa.w, acc[i][3]);
            acc[i][4] = fmaf(xv, wb.x, acc[i][4]); acc[i][5] = fmaf(xv, wb.y, acc[i][5]);
            acc[i][6] = fmaf(xv, wb.z, acc[i][6]); acc[i][7] = fmaf(xv, wb.w, acc[i][7]);
          }
        }
      }
    }
    const float4 ba = *reinterpret_cast<const float4*>(s_bias + 4 * cg), bb = *reinterpret_cast<const float4*>(s_bias + 16 + 4 * cg);
    const float bv[8] = {ba.x, ba.y, ba.z, ba.w, bb.x, bb.y, bb.z, bb.w};
#pragma unroll
    for (int i = 0; i < PXG; ++i) {
      float v[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        float t = acc[i][k] + bv[k];
        if (act == DV_ACT_RELU) t = fmaxf(t, 0.f);
        const uint32_t bit = ((k < 4 ? mb_lo : mb_hi) >> (4 * i + (k & 3))) & 1u;
        v[k] = bit ? t : 0.f;
        csum[k] += v[k];
      }
      float* dst = lo + (p0 + i) * kLoCh + 4 * cg;
      *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(dst + 16) = make_float4(v[4], v[5], v[6], v[7]);
      if (bits_out) {                                          // [x > 0] of the stored pixel: the lane quartet holds its 32 channels
        uint32_t ob = 0u;
#pragma unroll
        for (int k = 0; k < 8; ++k) ob |= (v[k] > 0.f ? 1u : 0u) << ((k < 4 ? 0 : 16) + 4 * cg + (k & 3));
        ob |= __shfl_xor_sync(0xffffffffu, ob, 1);
        ob |= __shfl_xor_sync(0xffffffffu, ob, 2);
        if (cg == 0) bits_out[p0 + i] = ob;
      }
    }
  }
  if (colsum_part) {
    // lanes with the same channel group (lane & 3) hold partial sums of the same 8 channels: fold them (xor 4, 8, 16)
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float t = csum[k];
      t += __shfl_xor_sync(0xffffffffu, t, 4); t += __shfl_xor_sync(0xffffffffu, t, 8); t += __shfl_xor_sync(0xffffffffu, t, 16);
      if (lane < 4) s_cs[warp][(k < 4 ? 0 : 16) + 4 * lane + (k & 3)] = t;
    }
    __syncthreads();
    if (warp == 0) {
      float t = 0.f;
#pragma unroll
      for (int w2 = 0; w2 < kThreads / 32; ++w2) t += s_cs[w2][lane];
      colsum_part[blockIdx.x * kLoCh + lane] = t;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// wgrad:  ws[block][k][cl], k = tap*CH + c (k == 16*CH: the lo-side bias gradient)
// ------------------------------------------------------------------------------------------------------------
template <int CH, int W>
__global__ void __launch_bounds__(kThreads, (CH == 1) ? 2 : 1)
img_wgrad_kernel(const float* __restrict__ lo, const float* __restrict__ hi, float* __restrict__ ws, int B, int H) {
  constexpr int TR = (W == 32) ? 16 : 16;
  constexpr int IN_ROWS = 2 * TR + 2, PITCH = 2 * W + 4;
  constexpr int NPX = TR * W;                                  // lo pixels per tile
  constexpr int NSTREAM = kThreads / 16;
  extern __shared__ __align__(16) float smem[];
  float* s_lo = smem;                                          // [NPX][kLoPitch]
  float* s_hi = smem + NPX * kLoPitch;                         // [CH][IN_ROWS][PITCH]
  const int tid = threadIdx.x;
  const int stream = tid >> 4, st = tid & 15;
  const int cl4 = st & 7, half = st >> 3;                      // 4 lo channels x taps of rows {2*half, 2*half+1}
  float acc[CH][8][4];
  float bsum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int c = 0; c < CH; ++c)
#pragma unroll
    for (int t = 0; t < 8; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[c][t][e] = 0.f;
  const int tiles_per_img = H / TR;
  const int num_tiles = B * tiles_per_img;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int b = tile / tiles_per_img, i0 = (tile % tiles_per_img) * TR;
    __syncthreads();
    load_hi_tile<CH, W, TR>(s_hi, hi, b, i0, H);
    {
      const float4* src = reinterpret_cast<const float4*>(lo + ((long long)b * H + i0) * W * kLoCh);
#pragma unroll 4
      for (int e = tid; e < NPX * 8; e += kThreads) {
        const int px = e >> 3, j = e & 7;
        cp_async16(s_lo + px * kLoPitch + 4 * j, src + e, true);
      }
    }
    cp_async_wait_all();
    __syncthreads();
#pragma unroll 2
    for (int px = stream; px < NPX; px += NSTREAM) {
      const int r = px / W, cc = px % W;
      const float4 l4 = *reinterpret_cast<const float4*>(s_lo + px * kLoPitch + 4 * cl4);
      if (half == 0) { bsum[0] += l4.x; bsum[1] += l4.y; bsum[2] += l4.z; bsum[3] += l4.w; }
#pragma unroll
      for (int c = 0; c < CH; ++c) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const float* row = s_hi + (c * IN_ROWS + 2 * r + 2 * half + rr) * PITCH + 2 * cc;
          const float2 a = *reinterpret_cast<const float2*>(row), d = *reinterpret_cast<const float2*>(row + 2);
          const float xv[4] = {a.x, a.y, d.x, d.y};
#pragma unroll
          for (int kw = 0; kw < 4; ++kw) {
            acc[c][rr * 4 + kw][0] = fmaf(xv[kw], l4.x, acc[c][rr * 4 + kw][0]);
            acc[c][rr * 4 + kw][1] = fmaf(xv[kw], l4.y, acc[c][rr * 4 + kw][1]);
            acc[c][rr * 4 + kw][2] = fmaf(xv[kw], l4.z, acc[c][rr * 4 + kw][2]);
            acc[c][rr * 4 + kw][3] = fmaf(xv[kw], l4.w, acc[c][rr * 4 + kw][3]);
          }
        }
      }
    }
  }
  // ordered reduction over the 16 streams through shared memory (the tiles are free now)
  __syncthreads();
  constexpr int K = kTaps * CH;
  float* red = smem;                                           // [NSTREAM][(K + 1) * 32]
  {
    float* mine = red + stream * (K + 1) * kLoCh;
#pragma unroll
    for (int c = 0; c < CH; ++c)
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const int tap = (2 * half + (t >> 2)) * 4 + (t & 3);
#pragma unroll
        for (int e = 0; e < 4; ++e) mine[(tap * CH + c) * kLoCh + 4 * cl4 + e] = acc[c][t][e];
      }
    if (half == 0) {
#pragma unroll
      for (int e = 0; e < 4; ++e) mine[K * kLoCh + 4 * cl4 + e] = bsum[e];
    }
  }
  __syncthreads();
  float* out = ws + (long long)blockIdx.x * (K + 1) * kLoCh;
  for (int idx = tid; idx < (K + 1) * kLoCh; idx += kThreads) {
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < NSTREAM; ++q) s += red[q * (K + 1) * kLoCh + idx];
    out[idx] = s;
  }
}

// ------------------------------------------------------------------------------------------------------------
// up: hi[b][c][2m+py][2n+px] = bias[c] + sum_{cl} sum_{(dm, kh) valid for py} sum_{(dn, kw) valid for px}
//                                        lo[b][m+dm][n+dn][cl] * w[cl][c][kh][kw]
//     py = 0: (dm, kh) in {(0,1), (-1,3)};  py = 1: (dm, kh) in {(+1,0), (0,2)}   (same for px / dn / kw)
// weights wu[(tap*CH + c)*32 + cl] (the "up" section of conv_pack_multi_kernel for CH < 32)
// ------------------------------------------------------------------------------------------------------------
template <int CH, int W>
__global__ void __launch_bounds__(128, 2)
img_up_kernel(const float* __restrict__ lo, const float* __restrict__ wu, const float* __restrict__ bias,
              float* __restrict__ hi, int B, int H, int act) {
  constexpr int NT = 128;
  constexpr int PY = 2;                                        // lo rows per thread
  constexpr int TCOLS = W / 2;                                 // thread columns (2 lo positions each)
  constexpr int TROWS = NT / TCOLS;                            // thread rows
  constexpr int TR = TROWS * PY;                               // lo rows per tile: 16 (W = 32), 32 -> capped below (W = 16)
  constexpr int SW = W + 2;                                    // tile width incl. halo
  extern __shared__ __align__(16) float smem[];
  // [(TR + 2)][SW][32]; the 16-byte chunk j of the pixel in tile column xx sits at chunk j ^ ((xx >> 1) & 7): a thread
  // reads columns 2*tn .. 2*tn+3, so the 8 lanes of a quarter-warp hit 8 different 16-byte bank groups (pitch padding
  // cannot do that for a 2-pixel lane stride)
  float* s_lo = smem;
  float* s_w = smem + (TR + 2) * SW * kLoCh;                   // [16*CH][32]
  const int tid = threadIdx.x;
  for (int i = tid; i < kTaps * CH * kLoCh; i += NT) s_w[i] = wu[i];
  const int tn = tid % TCOLS, tm = tid / TCOLS;
  const int tiles_per_img = (H + TR - 1) / TR;
  const int num_tiles = B * tiles_per_img;
  const int HH = 2 * H, WW = 2 * W;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int b = tile / tiles_per_img, m0 = (tile % tiles_per_img) * TR;
    __syncthreads();
    // lo rows m0-1 .. m0+TR, columns -1 .. W (zero outside the image)
#pragma unroll 4
    for (int e = tid; e < (TR + 2) * SW * 8; e += NT) {
      const int j = e & 7, xx = (e >> 3) % SW, rr = (e >> 3) / SW;
      const int m = m0 - 1 + rr, n = xx - 1;
      const bool ok = (unsigned)m < (unsigned)H && (unsigned)n < (unsigned)W;
      cp_async16(s_lo + (rr * SW + xx) * kLoCh + 4 * (j ^ ((xx >> 1) & 7)),
                 ok ? lo + (((long long)b * H + m) * W + n) * kLoCh + 4 * j : lo, ok);
    }
    cp_async_wait_all();
    __syncthreads();
    if (m0 + PY * tm < H) {
      float out[CH][2 * PY][4];
#pragma unroll
      for (int c = 0; c < CH; ++c)
#pragma unroll
        for (int y = 0; y < 2 * PY; ++y)
#pragma unroll
          for (int x = 0; x < 4; ++x) out[c][y][x] = 0.f;
      // neighbourhood rows PY*tm .. PY*tm + PY + 1 (tile rows; +1 halo offset folded in), columns 2*tn .. 2*tn + 3
      const float* base = s_lo + ((PY * tm) * SW + 2 * tn) * kLoCh;
#pragma unroll 1
      for (int j = 0; j < 8; ++j) {                            // 4-channel chunk of the lo side
        float4 nb[PY + 2][4];
#pragma unroll
        for (int rr = 0; rr < PY + 2; ++rr)
#pragma unroll
          for (int xx = 0; xx < 4; ++xx)
            nb[rr][xx] = *reinterpret_cast<const float4*>(base + (rr * SW + xx) * kLoCh + 4 * (j ^ ((tn + (xx >> 1)) & 7)));
#pragma unroll
        for (int c = 0; c < CH; ++c) {
#pragma unroll
          for (int tap = 0; tap < kTaps; ++tap) {
            const int kh = tap >> 2, kw = tap & 3;
            const float4 w4 = *reinterpret_cast<const float4*>(s_w + (tap * CH + c) * kLoCh + 4 * j);
            // kh -> (py, dm): kh=1:(0,0) kh=3:(0,-1) kh=0:(1,+1) kh=2:(1,0); tile row of lo row m is (m - m0 + 1)
            const int py = (kh & 1) ? 0 : 1, dm = (kh == 1 || kh == 2) ? 0 : ((kh == 3) ? -1 : 1);
            const int px = (kw & 1) ? 0 : 1, dn = (kw == 1 || kw == 2) ? 0 : ((kw == 3) ? -1 : 1);
#pragma unroll
            for (int a = 0; a < PY; ++a)
#pragma unroll
              for (int d = 0; d < 2; ++d) {
                const float4 v = nb[a + 1 + dm][d + 1 + dn];
                float o = out[c][2 * a + py][2 * d + px];
                o = fmaf(v.x, w4.x, o); o = fmaf(v.y, w4.y, o); o = fmaf(v.z, w4.z, o); o = fmaf(v.w, w4.w, o);
                out[c][2 * a + py][2 * d + px] = o;
              }
          }
        }
      }
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const float bv = bias ? __ldg(bias + c) : 0.f;
#pragma unroll
        for (int y = 0; y < 2 * PY; ++y) {
          const int oy = 2 * (m0 + PY * tm) + y;
          if (oy < HH) {
            float v[4];
#pragma unroll
            for (int x = 0; x < 4; ++x) v[x] = apply_act(out[c][y][x] + bv, act, 0.f);
            *reinterpret_cast<float4*>(hi + ((long long)(b * CH + c) * HH + oy) * WW + 4 * tn) = make_float4(v[0], v[1], v[2], v[3]);
          }
        }
      }
    }
  }
}

template <int W> constexpr int up_tile_rows() { return (128 / (W / 2)) * 2; }
template <int CH, int W> constexpr size_t up_smem() {
  return (size_t)((up_tile_rows<W>() + 2) * (W + 2) * kLoCh + kTaps * CH * kLoCh) * sizeof(float);
}
template <int CH, int W> constexpr size_t wgrad_smem() {
  constexpr size_t tiles = (size_t)16 * W * kLoPitch + (size_t)CH * 34 * (2 * W + 4);
  constexpr size_t red = (size_t)(kThreads / 16) * (kTaps * CH + 1) * kLoCh;
  return (tiles > red ? tiles : red) * sizeof(float);
}

template <typename K>
static bool set_smem(K kernel, size_t bytes) {
  return bytes <= 48 * 1024 || cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) == cudaSuccess;
}

int conv_down(const float* hi, const float* wd, const float* bias, const float* mask, const uint32_t* mask_bits, float* lo,
              uint32_t* bits_out, int B, int H, int W, int CH,
              int act, cudaStream_t st, float* colsum_part, int* nparts, int max_parts) {
  const int tiles = B * (H / 16);
  int grid = tiles < 2 * kNumSMs ? tiles : 2 * kNumSMs;
  if (colsum_part && grid > max_parts) grid = max_parts;
#define DV_IMG_DOWN(CHV, WV) \
  img_down_kernel<CHV, WV><<<grid, kThreads, 0, st>>>(hi, wd, bias, mask, lo, B, H, act, colsum_part, mask_bits, bits_out)
  if (CH == 1 && W == 32) DV_IMG_DOWN(1, 32);
  else if (CH == 3 && W == 32) DV_IMG_DOWN(3, 32);
  else if (CH == 1 && W == 16) DV_IMG_DOWN(1, 16);
  else DV_IMG_DOWN(3, 16);
#undef DV_IMG_DOWN
  *nparts = colsum_part ? grid : 0;
  return check_launch();
}

// CTAs of img_wgrad_kernel<CH, W>, one split-K partial each: persistent, as many as fit on the SMs (2 per SM for CH = 1)
int wgrad_splits(int B, int H, int CH) {
  const int tiles = B * (H / 16);
  const int per_sm = (CH == 1) ? 2 : 1;
  return tiles < per_sm * kNumSMs ? tiles : per_sm * kNumSMs;
}

int conv_wgrad(const float* lo, const float* hi, float* ws, int B, int H, int W, int CH, cudaStream_t st) {
  const int grid = wgrad_splits(B, H, CH);
#define DV_IMG_WG(CHV, WV)                                                                     \
  do {                                                                                         \
    if (!set_smem(img_wgrad_kernel<CHV, WV>, wgrad_smem<CHV, WV>())) return DV_ERR_CUDA;       \
    img_wgrad_kernel<CHV, WV><<<grid, kThreads, wgrad_smem<CHV, WV>(), st>>>(lo, hi, ws, B, H); \
  } while (0)
  if (CH == 1 && W == 32) DV_IMG_WG(1, 32);
  else if (CH == 3 && W == 32) DV_IMG_WG(3, 32);
  else if (CH == 1 && W == 16) DV_IMG_WG(1, 16);
  else DV_IMG_WG(3, 16);
#undef DV_IMG_WG
  return check_launch();
}

int conv_up(const float* lo, const float* wu, const float* bias, float* hi, int B, int H, int W, int CH, int act, cudaStream_t st) {
#define DV_IMG_UP(CHV, WV)                                                                     \
  do {                                                                                         \
    const int tiles = B * ((H + up_tile_rows<WV>() - 1) / up_tile_rows<WV>());                \
    const int grid = tiles < 2 * kNumSMs ? tiles : 2 * kNumSMs;                                \
    if (!set_smem(img_up_kernel<CHV, WV>, up_smem<CHV, WV>())) return DV_ERR_CUDA;             \
    img_up_kernel<CHV, WV><<<grid, 128, up_smem<CHV, WV>(), st>>>(lo, wu, bias, hi, B, H, act); \
  } while (0)
  if (CH == 1 && W == 32) DV_IMG_UP(1, 32);
  else if (CH == 3 && W == 32) DV_IMG_UP(3, 32);
  else if (CH == 1 && W == 16) DV_IMG_UP(1, 16);
  else DV_IMG_UP(3, 16);
#undef DV_IMG_UP
  return check_launch();
}

}  // namespace img
}  // namespace dv

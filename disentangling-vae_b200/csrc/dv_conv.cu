// Convolution entry points (dv_conv_down / dv_conv_up / dv_conv_wgrad / packs) of the Burgess 4x4/stride-2/pad-1 layers:
// the dispatch to the tensor-core kernels (dv_conv_tc.cu, 32-channel layers) and to the exact-fp32 image-boundary kernels
// (dv_conv_img.cu, CH in {1,3}), the split-K / channel-sum reductions they share, and the generic FP32 CUDA-core kernels
// below -- the fallback for every geometry the specialised kernels do not take (and the A/B reference: DV_CONV_IMPL=ffma).
//
// Every layer links lo[B,H,W,32] and hi[B,2H,2W,CH] through w[32][CH][4][4]
// (see include/disvae_b200.h).  Thread mapping is "lane = channel": the 32 lanes of a warp
// own the 32 channels of the output pixel line (one coalesced 128-byte store per pixel),
// activations of the other side are read as warp-broadcast 128-bit loads, weights sit in
// shared memory in a [k][channel] layout (conflict-free).  No block-level barrier inside
// the main loops.  The *_small variants handle the CH in {1,3} image-boundary layers (NCHW).
//
// Reference call sites replaced: disvae/models/encoders.py:73-77 (Conv2d+ReLU),
// disvae/models/decoders.py:77-82 (ConvTranspose2d+ReLU/sigmoid) and their autograd
// backward (disvae/training.py:157).
#include <stdlib.h>
#include <string.h>
#include "dv_common.cuh"

namespace dv {

// ------------------------------------------------------------------------------------
// weight packing: w[cl][c][tap] -> down section Wd[tap*CH + c][cl]
//                               -> up section   CH==32: Wu[tap][cl][c] ; CH<32: Wu[tap][c][cl]
// ------------------------------------------------------------------------------------
__global__ void conv_pack_kernel(const float* __restrict__ w, float* __restrict__ wp, int CH) {
  const int n = kLoCh * CH * kTaps;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += gridDim.x * blockDim.x) {
    const int tap = idx % kTaps;
    const int c = (idx / kTaps) % CH;
    const int cl = idx / (kTaps * CH);
    const float v = w[idx];
    wp[(tap * CH + c) * kLoCh + cl] = v;
    if (CH == 32) wp[n + (tap * kLoCh + cl) * CH + c] = v;
    else          wp[n + (tap * CH + c) * kLoCh + cl] = v;
  }
}

__device__ __forceinline__ void stage_weights(float* smem, const float* __restrict__ src, int n_floats) {
  for (int i = threadIdx.x * 4; i < n_floats; i += blockDim.x * 4)
    *reinterpret_cast<float4*>(smem + i) = ldg4(src + i);
  __syncthreads();
}

// ------------------------------------------------------------------------------------
// down, CH == 32 (NHWC hi).  One warp = 16 consecutive lo pixels x 32 lo channels.
// ------------------------------------------------------------------------------------
constexpr int kDownPxPerWarp = 16;
constexpr int kDownWarps = 8;

__global__ void __launch_bounds__(kDownWarps * 32)
conv_down32_kernel(const float* __restrict__ hi, const float* __restrict__ wp, const float* __restrict__ bias,
                   const float* __restrict__ mask, float* __restrict__ lo, int B, int H, int W, int act) {
  extern __shared__ __align__(16) float Ws[];          // [tap*32 + c][cl]
  stage_weights(Ws, wp, kTaps * 32 * kLoCh);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int HH = 2 * H, WW = 2 * W;
  const long long total = (long long)B * H * W;
  const long long n_groups = (total + kDownPxPerWarp - 1) / kDownPxPerWarp;
  const float bv = bias ? bias[lane] : 0.f;

  for (long long g = (long long)blockIdx.x * kDownWarps + warp; g < n_groups; g += (long long)gridDim.x * kDownWarps) {
    const long long p0 = g * kDownPxPerWarp;
    int base[kDownPxPerWarp];      // hi pixel index of (2i-1, 2j-1); only used where valid
    int ij[kDownPxPerWarp];        // (2i-1) << 16 | ((2j-1) & 0xffff); -32768 marks "no pixel"
#pragma unroll
    for (int q = 0; q < kDownPxPerWarp; ++q) {
      const long long p = p0 + q;
      if (p < total) {
        const int j = (int)(p % W), i = (int)((p / W) % H), b = (int)(p / ((long long)W * H));
        base[q] = (b * HH + 2 * i - 1) * WW + 2 * j - 1;
        ij[q] = (2 * i - 1) * 65536 + ((2 * j - 1) & 0xffff);
      } else { base[q] = 0; ij[q] = -30000 * 65536 + 30000; }
    }
    float acc[kDownPxPerWarp];
#pragma unroll
    for (int q = 0; q < kDownPxPerWarp; ++q) acc[q] = 0.f;

    for (int tap = 0; tap < kTaps; ++tap) {
      const int kh = tap >> 2, kw = tap & 3;
      const float* wrow = Ws + tap * 32 * kLoCh + lane;
      unsigned valid = 0;
#pragma unroll
      for (int q = 0; q < kDownPxPerWarp; ++q) {
        const int ih = (ij[q] >> 16) + kh, iw = (int)(short)(ij[q] & 0xffff) + kw;
        if ((unsigned)ih < (unsigned)HH && (unsigned)iw < (unsigned)WW) valid |= 1u << q;
      }
      const int tap_off = kh * WW + kw;
#pragma unroll 2
      for (int c4 = 0; c4 < 8; ++c4) {
        const float w0 = wrow[(c4 * 4 + 0) * kLoCh], w1 = wrow[(c4 * 4 + 1) * kLoCh];
        const float w2 = wrow[(c4 * 4 + 2) * kLoCh], w3 = wrow[(c4 * 4 + 3) * kLoCh];
#pragma unroll
        for (int q = 0; q < kDownPxPerWarp; ++q) {
          if (valid & (1u << q)) {
            const float4 v = ldg4(hi + (long long)(base[q] + tap_off) * 32 + c4 * 4);
            acc[q] = fmaf(v.x, w0, acc[q]); acc[q] = fmaf(v.y, w1, acc[q]);
            acc[q] = fmaf(v.z, w2, acc[q]); acc[q] = fmaf(v.w, w3, acc[q]);
          }
        }
      }
    }
#pragma unroll
    for (int q = 0; q < kDownPxPerWarp; ++q) {
      const long long p = p0 + q;
      if (p < total) {
        float v = acc[q] + bv;
        if (act == DV_ACT_RELU) v = fmaxf(v, 0.f);
        if (mask) v = (mask[p * kLoCh + lane] > 0.f) ? v : 0.f;
        lo[p * kLoCh + lane] = v;
      }
    }
  }
}

// ------------------------------------------------------------------------------------
// down, CH in {1,3} (NCHW hi): conv1 forward, convT3 input-gradient.
// ------------------------------------------------------------------------------------
template <int CH>
__global__ void __launch_bounds__(kDownWarps * 32)
conv_down_small_kernel(const float* __restrict__ hi, const float* __restrict__ wp, const float* __restrict__ bias,
                       const float* __restrict__ mask, float* __restrict__ lo, int B, int H, int W, int act) {
  __shared__ __align__(16) float Ws[kTaps * CH * kLoCh];
  for (int i = threadIdx.x; i < kTaps * CH * kLoCh; i += blockDim.x) Ws[i] = wp[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int HH = 2 * H, WW = 2 * W;
  const int plane = HH * WW;
  const long long total = (long long)B * H * W;
  const long long n_groups = (total + kDownPxPerWarp - 1) / kDownPxPerWarp;
  const float bv = bias ? bias[lane] : 0.f;

  for (long long g = (long long)blockIdx.x * kDownWarps + warp; g < n_groups; g += (long long)gridDim.x * kDownWarps) {
    const long long p0 = g * kDownPxPerWarp;
    long long base[kDownPxPerWarp];
    int ij[kDownPxPerWarp];
#pragma unroll
    for (int q = 0; q < kDownPxPerWarp; ++q) {
      const long long p = p0 + q;
      if (p < total) {
        const int j = (int)(p % W), i = (int)((p / W) % H), b = (int)(p / ((long long)W * H));
        base[q] = ((long long)b * CH * HH + 2 * i - 1) * WW + 2 * j - 1;
        ij[q] = (2 * i - 1) * 65536 + ((2 * j - 1) & 0xffff);
      } else { base[q] = 0; ij[q] = -30000 * 65536 + 30000; }
    }
    float acc[kDownPxPerWarp];
#pragma unroll
    for (int q = 0; q < kDownPxPerWarp; ++q) acc[q] = 0.f;
    for (int tap = 0; tap < kTaps; ++tap) {
      const int kh = tap >> 2, kw = tap & 3;
      unsigned valid = 0;
#pragma unroll
      for (int q = 0; q < kDownPxPerWarp; ++q) {
        const int ih = (ij[q] >> 16) + kh, iw = (int)(short)(ij[q] & 0xffff) + kw;
        if ((unsigned)ih < (unsigned)HH && (unsigned)iw < (unsigned)WW) valid |= 1u << q;
      }
      const int tap_off = kh * WW + kw;
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const float wv = Ws[(tap * CH + c) * kLoCh + lane];
#pragma unroll
        for (int q = 0; q < kDownPxPerWarp; ++q) {
          if (valid & (1u << q)) acc[q] = fmaf(__ldg(hi + base[q] + tap_off + (long long)c * plane), wv, acc[q]);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < kDownPxPerWarp; ++q) {
      const long long p = p0 + q;
      if (p < total) {
        float v = acc[q] + bv;
        if (act == DV_ACT_RELU) v = fmaxf(v, 0.f);
        if (mask) v = (mask[p * kLoCh + lane] > 0.f) ? v : 0.f;
        lo[p * kLoCh + lane] = v;
      }
    }
  }
}

// ------------------------------------------------------------------------------------
// up, CH == 32 (NHWC hi).  One warp = 4 consecutive lo positions of a row -> 2x8 hi pixels.
// hi(2i+ph, 2j+pw) = sum over taps with kh = ph+1-2*di, kw = pw+1-2*dj of lo(i+di, j+dj).
// ------------------------------------------------------------------------------------
constexpr int kUpPos = 4;
constexpr int kUpWarps = 8;

__global__ void __launch_bounds__(kUpWarps * 32)
conv_up32_kernel(const float* __restrict__ lo, const float* __restrict__ wp_up, const float* __restrict__ bias,
                 const float* __restrict__ mask, float* __restrict__ hi, int B, int H, int W, int act) {
  extern __shared__ __align__(16) float Ws[];          // [tap][cl][c]
  stage_weights(Ws, wp_up, kTaps * kLoCh * 32);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int HH = 2 * H, WW = 2 * W;
  const int wgroups = W / kUpPos;
  const long long n_units = (long long)B * H * wgroups;
  const float bv = bias ? bias[lane] : 0.f;

  for (long long u = (long long)blockIdx.x * kUpWarps + warp; u < n_units; u += (long long)gridDim.x * kUpWarps) {
    const int j0 = (int)(u % wgroups) * kUpPos;
    const int i = (int)((u / wgroups) % H);
    const int b = (int)(u / ((long long)wgroups * H));
    float acc[2][2][kUpPos];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int c = 0; c < 2; ++c)
#pragma unroll
        for (int n = 0; n < kUpPos; ++n) acc[a][c][n] = 0.f;

#pragma unroll
    for (int di = -1; di <= 1; ++di) {
      const int ih = i + di;
      if ((unsigned)ih >= (unsigned)H) continue;               // warp-uniform
      const float* lrow = lo + ((long long)(b * H + ih) * W) * kLoCh;
#pragma unroll 2
      for (int cl4 = 0; cl4 < 8; ++cl4) {
        float4 lv[kUpPos + 2];
#pragma unroll
        for (int t = 0; t < kUpPos + 2; ++t) {
          const int jj = j0 - 1 + t;
          lv[t] = ((unsigned)jj < (unsigned)W) ? ldg4(lrow + (long long)jj * kLoCh + cl4 * 4)
                                               : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int ph = 0; ph < 2; ++ph) {
          const int kh = ph + 1 - 2 * di;
          if (kh < 0 || kh > 3) continue;                      // compile-time after unrolling
#pragma unroll
          for (int kw = 0; kw < 4; ++kw) {
            const int pw = (kw + 1) & 1;
            const int dj = (pw + 1 - kw) / 2;
            const float* wp = Ws + ((kh * 4 + kw) * kLoCh + cl4 * 4) * 32 + lane;
            const float w0 = wp[0], w1 = wp[32], w2 = wp[64], w3 = wp[96];
#pragma unroll
            for (int n = 0; n < kUpPos; ++n) {
              const float4 v = lv[n + dj + 1];
              float a = acc[ph][pw][n];
              a = fmaf(v.x, w0, a); a = fmaf(v.y, w1, a); a = fmaf(v.z, w2, a); a = fmaf(v.w, w3, a);
              acc[ph][pw][n] = a;
            }
          }
        }
      }
    }
#pragma unroll
    for (int ph = 0; ph < 2; ++ph)
#pragma unroll
      for (int pw = 0; pw < 2; ++pw)
#pragma unroll
        for (int n = 0; n < kUpPos; ++n) {
          const long long idx = ((long long)(b * HH + 2 * i + ph) * WW + 2 * (j0 + n) + pw) * 32 + lane;
          float v = acc[ph][pw][n] + bv;
          if (act == DV_ACT_RELU) v = fmaxf(v, 0.f);
          else if (act == DV_ACT_SIGMOID) v = 1.f / (1.f + expf(-v));
          if (mask) v = (mask[idx] > 0.f) ? v : 0.f;
          hi[idx] = v;
        }
  }
}

// ------------------------------------------------------------------------------------
// up, CH in {1,3} (NCHW hi): convT3 forward (sigmoid).  One thread = one lo position ->
// 2x2 hi pixels x CH channels; weights broadcast from shared memory as [tap][c][cl].
// ------------------------------------------------------------------------------------
template <int CH>
__global__ void __launch_bounds__(256)
conv_up_small_kernel(const float* __restrict__ lo, const float* __restrict__ wp_up, const float* __restrict__ bias,
                     const float* __restrict__ mask, float* __restrict__ hi, int B, int H, int W, int act) {
  __shared__ __align__(16) float Ws[kTaps * CH * kLoCh];
  for (int i = threadIdx.x; i < kTaps * CH * kLoCh; i += blockDim.x) Ws[i] = wp_up[i];
  __syncthreads();
  const int HH = 2 * H, WW = 2 * W;
  const long long total = (long long)B * H * W;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(p % W), i = (int)((p / W) % H), b = (int)(p / ((long long)W * H));
    float acc[2][2][CH];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int c2 = 0; c2 < 2; ++c2)
#pragma unroll
        for (int c = 0; c < CH; ++c) acc[a][c2][c] = 0.f;
#pragma unroll 1
    for (int cl4 = 0; cl4 < 8; ++cl4) {
      float4 lv[3][3];
#pragma unroll
      for (int di = -1; di <= 1; ++di)
#pragma unroll
        for (int dj = -1; dj <= 1; ++dj) {
          const int ih = i + di, jw = j + dj;
          lv[di + 1][dj + 1] = ((unsigned)ih < (unsigned)H && (unsigned)jw < (unsigned)W)
              ? ldg4(lo + ((long long)(b * H + ih) * W + jw) * kLoCh + cl4 * 4)
              : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
      for (int di = -1; di <= 1; ++di)
#pragma unroll
        for (int ph = 0; ph < 2; ++ph) {
          const int kh = ph + 1 - 2 * di;
          if (kh < 0 || kh > 3) continue;
#pragma unroll
          for (int kw = 0; kw < 4; ++kw) {
            const int pw = (kw + 1) & 1;
            const int dj = (pw + 1 - kw) / 2;
            const float4 v = lv[di + 1][dj + 1];
#pragma unroll
            for (int c = 0; c < CH; ++c) {
              const float4 w4 = *reinterpret_cast<const float4*>(Ws + ((kh * 4 + kw) * CH + c) * kLoCh + cl4 * 4);
              float a = acc[ph][pw][c];
              a = fmaf(v.x, w4.x, a); a = fmaf(v.y, w4.y, a); a = fmaf(v.z, w4.z, a); a = fmaf(v.w, w4.w, a);
              acc[ph][pw][c] = a;
            }
          }
        }
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const float bv = bias ? bias[c] : 0.f;
#pragma unroll
      for (int ph = 0; ph < 2; ++ph) {
        const long long idx = (((long long)b * CH + c) * HH + 2 * i + ph) * WW + 2 * j;
        float v0 = acc[ph][0][c] + bv, v1 = acc[ph][1][c] + bv;
        if (act == DV_ACT_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
        else if (act == DV_ACT_SIGMOID) { v0 = 1.f / (1.f + expf(-v0)); v1 = 1.f / (1.f + expf(-v1)); }
        if (mask) { v0 = (mask[idx] > 0.f) ? v0 : 0.f; v1 = (mask[idx + 1] > 0.f) ? v1 : 0.f; }
        *reinterpret_cast<float2*>(hi + idx) = make_float2(v0, v1);
      }
    }
  }
}

// ------------------------------------------------------------------------------------
// wgrad.  dw[cl][c][tap] = sum_p lo[p][cl] * hi(2i-1+kh, 2j-1+kw)[c].  lane = cl.
// Split-K over CTAs (pixel chunks), partials ws[split][16*CH + 1][32] (last row = sum of lo),
// then a fixed-order reduction -> deterministic.
// CH == 32: warp w owns taps {2w, 2w+1} (64 accumulators), all warps walk the same pixels.
// ------------------------------------------------------------------------------------
constexpr int kWgWarps = 8;

__global__ void __launch_bounds__(kWgWarps * 32)
conv_wgrad32_kernel(const float* __restrict__ lo, const float* __restrict__ hi, float* __restrict__ ws,
                    int B, int H, int W, long long chunk) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int HH = 2 * H, WW = 2 * W;
  const long long total = (long long)B * H * W;
  const long long p_begin = (long long)blockIdx.x * chunk;
  const long long p_end = min(total, p_begin + chunk);
  float acc[2][32];
#pragma unroll
  for (int t = 0; t < 2; ++t)
#pragma unroll
    for (int c = 0; c < 32; ++c) acc[t][c] = 0.f;
  float lsum = 0.f;
  const int kh0 = (2 * warp) >> 2, kw0 = (2 * warp) & 3;      // taps 2w and 2w+1 share kh; kw0 in {0,2}

  int j = (int)(p_begin % W), i = (int)((p_begin / W) % H), b = (int)(p_begin / ((long long)W * H));
  for (long long p = p_begin; p < p_end; ++p) {
    const float l = __ldg(lo + p * kLoCh + lane);
    lsum += l;
    const int ih = 2 * i - 1 + kh0;
    if ((unsigned)ih < (unsigned)HH) {
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        const int iw = 2 * j - 1 + kw0 + t;
        if ((unsigned)iw < (unsigned)WW) {
          const float* hp = hi + ((long long)(b * HH + ih) * WW + iw) * 32;
#pragma unroll
          for (int c4 = 0; c4 < 8; ++c4) {
            const float4 v = ldg4(hp + c4 * 4);
            acc[t][c4 * 4 + 0] = fmaf(l, v.x, acc[t][c4 * 4 + 0]);
            acc[t][c4 * 4 + 1] = fmaf(l, v.y, acc[t][c4 * 4 + 1]);
            acc[t][c4 * 4 + 2] = fmaf(l, v.z, acc[t][c4 * 4 + 2]);
            acc[t][c4 * 4 + 3] = fmaf(l, v.w, acc[t][c4 * 4 + 3]);
          }
        }
      }
    }
    if (++j == W) { j = 0; if (++i == H) { i = 0; ++b; } }
  }
  float* out = ws + (long long)blockIdx.x * (kTaps * 32 + 1) * kLoCh;
#pragma unroll
  for (int t = 0; t < 2; ++t)
#pragma unroll
    for (int c = 0; c < 32; ++c) out[((2 * warp + t) * 32 + c) * kLoCh + lane] = acc[t][c];
  if (warp == 0) out[(kTaps * 32) * kLoCh + lane] = lsum;
}

// CH in {1,3}: every warp keeps all 16*CH accumulators, warps split the pixels of the chunk.
template <int CH>
__global__ void __launch_bounds__(kWgWarps * 32)
conv_wgrad_small_kernel(const float* __restrict__ lo, const float* __restrict__ hi, float* __restrict__ ws,
                        int B, int H, int W, long long chunk) {
  constexpr int K = kTaps * CH;
  __shared__ float red[(K + 1) * kLoCh];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int HH = 2 * H, WW = 2 * W;
  const long long plane = (long long)HH * WW;
  const long long total = (long long)B * H * W;
  const long long p_begin = (long long)blockIdx.x * chunk;
  const long long p_end = min(total, p_begin + chunk);
  float acc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k] = 0.f;
  float lsum = 0.f;
  for (long long p = p_begin + warp; p < p_end; p += kWgWarps) {
    const int j = (int)(p % W), i = (int)((p / W) % H), b = (int)(p / ((long long)W * H));
    const float l = __ldg(lo + p * kLoCh + lane);
    lsum += l;
    const float* hb = hi + (long long)b * CH * plane;
#pragma unroll
    for (int kh = 0; kh < 4; ++kh) {
      const int ih = 2 * i - 1 + kh;
      if ((unsigned)ih >= (unsigned)HH) continue;
#pragma unroll
      for (int kw = 0; kw < 4; ++kw) {
        const int iw = 2 * j - 1 + kw;
        if ((unsigned)iw >= (unsigned)WW) continue;
#pragma unroll
        for (int c = 0; c < CH; ++c)
          acc[(kh * 4 + kw) * CH + c] = fmaf(l, __ldg(hb + c * plane + (long long)ih * WW + iw), acc[(kh * 4 + kw) * CH + c]);
      }
    }
  }
  // fixed-order cross-warp reduction
  for (int w = 0; w < kWgWarps; ++w) {
    if (warp == w) {
#pragma unroll
      for (int k = 0; k < K; ++k) red[k * kLoCh + lane] = (w == 0 ? 0.f : red[k * kLoCh + lane]) + acc[k];
      red[K * kLoCh + lane] = (w == 0 ? 0.f : red[K * kLoCh + lane]) + lsum;
    }
    __syncthreads();
  }
  float* out = ws + (long long)blockIdx.x * (K + 1) * kLoCh;
  for (int idx = threadIdx.x; idx < (K + 1) * kLoCh; idx += blockDim.x) out[idx] = red[idx];
}

// dw[cl][c][tap] = sum_s ws[s][tap*CH + c][cl] ; dbias[cl] = sum_s ws[s][16*CH][cl]
// block = 32 outputs x 8 split groups: group j sums splits j, j+8, ... (coalesced over the outputs), the eight group
// sums are combined in a fixed order -> deterministic for a given nsplit.
__global__ void __launch_bounds__(256)
conv_wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw, float* __restrict__ dbias, int CH, int nsplit) {
  __shared__ float part[8][33];
  const int K = kTaps * CH;
  const int n = (K + 1) * kLoCh;
  const int o = threadIdx.x & 31, grp = threadIdx.x >> 5;
  const int idx = blockIdx.x * 32 + o;
  float s = 0.f;
  if (idx < n)
    for (int sp = grp; sp < nsplit; sp += 8) s += ws[(long long)sp * n + idx];
  part[grp][o] = s;
  __syncthreads();
  if (grp != 0 || idx >= n) return;
  s = ((part[0][o] + part[1][o]) + (part[2][o] + part[3][o])) + ((part[4][o] + part[5][o]) + (part[6][o] + part[7][o]));
  const int cl = idx % kLoCh, k = idx / kLoCh;
  if (k == K) { if (dbias) dbias[cl] = s; }
  else {
    const int tap = k / CH, c = k % CH;
    dw[(cl * CH + c) * kTaps + tap] = s;
  }
}

// ------------------------------------------------------------------------------------
// channel sums (bias gradients of the transposed-conv layers), two deterministic stages.
// ------------------------------------------------------------------------------------
constexpr int kCsBlocks = 296;
__global__ void __launch_bounds__(256)
channel_sum_nhwc_kernel(const float* __restrict__ x, float* __restrict__ partial, long long rows, int C) {
  // C <= 32; lane = channel, warps stride over rows
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float s = 0.f;
  if (lane < C)
    for (long long r = (long long)blockIdx.x * 8 + warp; r < rows; r += (long long)gridDim.x * 8) s += x[r * C + lane];
  red[warp][lane] = s;
  __syncthreads();
  if (warp == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][lane];
    partial[blockIdx.x * 32 + lane] = t;
  }
}
__global__ void __launch_bounds__(256)
channel_sum_nchw_kernel(const float* __restrict__ x, float* __restrict__ partial, int B, int C, int hw) {
  // block (b-strided) x channel: partial[blockIdx.x][c]
  __shared__ float red[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int c = 0; c < C; ++c) {
    float s = 0.f;
    for (int b = blockIdx.x; b < B; b += gridDim.x) {
      const float* px = x + ((long long)b * C + c) * hw;
      for (int e = threadIdx.x; e < hw; e += blockDim.x) s += px[e];
    }
    s = warp_sum(s);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int w = 0; w < 8; ++w) t += red[w];
      partial[blockIdx.x * 32 + c] = t;
    }
    __syncthreads();
  }
}
// 32 channels x 32 slices of the per-block partials, combined in a fixed order
__global__ void __launch_bounds__(1024)
channel_sum_final_kernel(const float* __restrict__ partial, float* __restrict__ out, int nblocks, int C) {
  __shared__ float red[32][33];
  const int c = threadIdx.x & 31, w = threadIdx.x >> 5;
  float s = 0.f;
  if (c < C)
    for (int b = w; b < nblocks; b += 32) s += partial[b * 32 + c];
  red[w][c] = s;
  __syncthreads();
  if (w == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) t += red[k][c];
    out[c] = t;
  }
}

__global__ void flat_transpose_kernel(const float* __restrict__ src, float* __restrict__ dst, long long n, int C, int S, int to_nhwc) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
    const int per = C * S;
    const long long b = idx / per;
    const int r = (int)(idx % per);
    if (to_nhwc) { const int s = r / C, c = r % C; dst[idx] = src[b * per + c * S + s]; }     // dst[b][s][c]
    else         { const int c = r / S, s = r % S; dst[idx] = src[b * per + s * C + c]; }     // dst[b][c][s]
  }
}

__global__ void act_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ g,
                               long long n, int act, float slope) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float yv = y[i], d = dy[i];
    float r;
    if (act == DV_ACT_SIGMOID) r = d * ((1.f - yv) * yv);      // aten sigmoid_backward: grad * (1 - y) * y
    else if (act == DV_ACT_RELU) r = yv > 0.f ? d : 0.f;
    else if (act == DV_ACT_LEAKY) r = yv > 0.f ? d : d * slope;
    else r = d;
    g[i] = r;
  }
}

static int grid_for(long long work_items, int per_block, int max_blocks) {
  long long g = (work_items + per_block - 1) / per_block;
  if (g < 1) g = 1;
  if (g > max_blocks) g = max_blocks;
  return (int)g;
}

static bool shape_ok(int B, int H, int W, int CH) {
  if (B <= 0 || H <= 0 || W <= 0) return false;
  if (CH != 1 && CH != 3 && CH != 32) return false;
  if (W % 4 != 0 || W > 4096 || H > 4096) return false;
  if ((long long)B * 4 * H * W * (CH > 32 ? CH : 32) >= (1LL << 31)) return false;   // int pixel indices
  return true;
}

static int wgrad_nsplit(int B, int H, int W, long long* chunk) {
  const long long total = (long long)B * H * W;
  long long ns = (total + 63) / 64;
  if (ns > 2 * kNumSMs) ns = 2 * kNumSMs;
  if (ns < 1) ns = 1;
  *chunk = (total + ns - 1) / ns;
  return (int)((total + *chunk - 1) / *chunk);
}

}  // namespace dv

namespace dv {
namespace tc {        // dv_conv_tc.cu: tensor-core kernels of the 32-channel layers
int pack_tc(const float* w, float* wd, float* wu, float* wf, cudaStream_t st);
int pack_multi(int n, const float* const* w, float* const* wp, const int* CH, cudaStream_t st);
int conv_down32_tc(const float* hi, const float* wd_packed, const float* bias, const float* mask, float* lo,
                   int B, int H, int W, int act, cudaStream_t st, float* colsum_part, int* nparts,
                   const uint32_t* mask_bits, uint32_t* bits_out);
int conv_up_halo(const float* lo, const float* wu, const float* bias, const float* mask, float* hi,
                 int B, int H, int W, int act, cudaStream_t st, const uint32_t* mask_bits, uint32_t* bits_out);
int conv_wgrad32_tc(const float* lo, const float* hi, float* ws, int B, int H, int W, int* nsplit, cudaStream_t st);
}  // namespace tc
namespace img {       // dv_conv_img.cu: exact-fp32 CUDA-core kernels for the image-boundary layers (CH in {1,3})
bool shape_ok(int B, int H, int W, int CH);
int conv_down(const float* hi, const float* wd, const float* bias, const float* mask, const uint32_t* mask_bits, float* lo,
              uint32_t* bits_out, int B, int H, int W, int CH, int act, cudaStream_t st, float* colsum_part, int* nparts,
              int max_parts);
int conv_wgrad(const float* lo, const float* hi, float* ws, int B, int H, int W, int CH, int max_split, int* nsplit, cudaStream_t st);
int conv_up(const float* lo, const float* wu, const float* bias, float* hi, int B, int H, int W, int CH, int act, cudaStream_t st);
}  // namespace img

// packed-weight sections for CH == 32 (floats): [0,16K) ffma down, [16K,32K) ffma up,
// [32K,64K) tensor-core down (hi|lo), [64K,96K) tensor-core up (hi|lo)
constexpr int kPackFfma = 2 * kLoCh * 32 * kTaps;
constexpr int kPackTcSection = kTaps * 64 * 32;

// DV_CONV_IMPL=ffma forces the CUDA-core kernels for the 32-channel layers (A/B testing)
// DV_TC_DISABLE=down,up,wgrad switches individual tensor-core kernels off.
// DV_IMG=0 switches the dv_conv_img.cu kernels off (the image-boundary layers then run on the CUDA-core fallbacks).
static bool use_img() {
  static const int v = env_switch("DV_IMG", 1);
  return v == 1;
}
static bool use_tc(const char* which = nullptr) {
  static const int v = [] { const char* e = getenv("DV_CONV_IMPL"); return (e && e[0] == 'f') ? 0 : 1; }();
  static const char* const dis = getenv("DV_TC_DISABLE");
  if (v != 1) return false;
  return !(which && dis && strstr(dis, which));
}
}  // namespace dv

using namespace dv;

extern "C" {

// CH in {1,3}: [0, 512*CH) down layout, [512*CH, 1024*CH) up layout (shared by dv_conv_img.cu and the CUDA-core kernels)
size_t dv_conv_packed_floats(int CH) {
  return CH == 32 ? (size_t)kPackFfma + 2 * kPackTcSection
                  : (size_t)2 * kLoCh * CH * kTaps;
}

int dv_conv_pack_weights(const float* w, float* w_packed, int CH, void* stream) {
  if (!w || !w_packed) return DV_ERR_BAD_ARG;
  if (CH != 1 && CH != 3 && CH != 32) return DV_ERR_BAD_SHAPE;
  const int n = kLoCh * CH * kTaps;
  if (CH == 32)                                     // ONE launch: both tensor-core operand layouts + the two CUDA-core layouts
    return tc::pack_tc(w, w_packed + kPackFfma, w_packed + kPackFfma + kPackTcSection, w_packed, as_stream(stream));
  conv_pack_kernel<<<(n + 255) / 256, 256, 0, as_stream(stream)>>>(w, w_packed, CH);
  return check_launch();
}

int dv_conv_pack_multi(int n, const void* const* w, void* const* w_packed, const int* CH, void* stream) {
  if (n < 1 || !w || !w_packed || !CH) return DV_ERR_BAD_ARG;
  for (int i = 0; i < n; ++i) {
    if (!w[i] || !w_packed[i]) return DV_ERR_BAD_ARG;
    if (CH[i] != 1 && CH[i] != 3 && CH[i] != 32) return DV_ERR_BAD_SHAPE;
  }
  static_assert(kPackFfma == 2 * kLoCh * 32 * kTaps && kPackTcSection == kTaps * 64 * 32, "layout shared with conv_pack_multi_kernel");
  return tc::pack_multi(n, reinterpret_cast<const float* const*>(w), reinterpret_cast<float* const*>(w_packed), CH, as_stream(stream));
}

// [x > 0] of a 32-channel NHWC tensor as one word per pixel, for the kernels that do not produce it in their epilogue
__global__ void relu_bits_kernel(const float* __restrict__ x, uint32_t* __restrict__ bits, long long npx) {
  const long long p = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (p >= npx) return;
  const uint32_t b = __ballot_sync(0xffffffffu, x[p * 32 + (threadIdx.x & 31)] > 0.f);
  if ((threadIdx.x & 31) == 0) bits[p] = b;
}
static int relu_bits(const float* x, uint32_t* bits, long long npx, cudaStream_t st) {
  relu_bits_kernel<<<(unsigned)((npx + 7) / 8), 256, 0, st>>>(x, bits, npx);
  return check_launch();
}

static int conv_down_impl(const float* hi, const float* w_packed, const float* bias, const float* mask, float* lo,
                          int B, int H, int W, int CH, int act, cudaStream_t st, float* colsum_part, int* nparts,
                          const uint32_t* mask_bits, uint32_t* bits_out, bool* bits_done) {
  *nparts = 0;
  *bits_done = true;
  const long long groups = ((long long)B * H * W + kDownPxPerWarp - 1) / kDownPxPerWarp;
  if (CH == 32 && use_tc("down"))
    return tc::conv_down32_tc(hi, w_packed + kPackFfma, bias, mask, lo, B, H, W, act, st, colsum_part, nparts, mask_bits, bits_out);
  if (CH != 32 && use_img() && img::shape_ok(B, H, W, CH))
    return img::conv_down(hi, w_packed, bias, mask, mask_bits, lo, bits_out, B, H, W, CH, act, st, colsum_part, nparts, kCsBlocks);
  *bits_done = false;                               // the CUDA-core fallbacks below read the float mask and write no bits
  if (CH == 32) {
    const int smem = kTaps * 32 * kLoCh * sizeof(float);
    static bool attr_set = false;
    if (!attr_set) {
      if (cudaFuncSetAttribute(conv_down32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
        return DV_ERR_CUDA;
      attr_set = true;
    }
    const int grid = grid_for(groups, kDownWarps, 2 * kNumSMs);
    conv_down32_kernel<<<grid, kDownWarps * 32, smem, st>>>(hi, w_packed, bias, mask, lo, B, H, W, act);
  } else {
    const int grid = grid_for(groups, kDownWarps, 8 * kNumSMs);
    if (CH == 1) conv_down_small_kernel<1><<<grid, kDownWarps * 32, 0, st>>>(hi, w_packed, bias, mask, lo, B, H, W, act);
    else         conv_down_small_kernel<3><<<grid, kDownWarps * 32, 0, st>>>(hi, w_packed, bias, mask, lo, B, H, W, act);
  }
  return check_launch();
}

int dv_conv_down(const float* hi, const float* w_packed, const float* bias, const float* mask, float* lo,
                 int B, int H, int W, int CH, int hi_nchw, int act, float* colsum_out, void* colsum_workspace,
                 const unsigned* mask_bits, unsigned* relu_bits_out, void* stream) {
  if (!hi || !w_packed || !lo) return DV_ERR_BAD_ARG;
  if (mask_bits && !mask) return DV_ERR_BAD_ARG;               // the words accelerate the float mask, they do not replace it
  if (!shape_ok(B, H, W, CH)) return DV_ERR_BAD_SHAPE;
  if (act != DV_ACT_NONE && act != DV_ACT_RELU) return DV_ERR_BAD_ARG;
  if ((CH == 32) == (hi_nchw != 0)) return DV_ERR_BAD_SHAPE;   // CH==32 <=> NHWC
  if (colsum_out && !colsum_workspace) return DV_ERR_WORKSPACE;
  cudaStream_t st = as_stream(stream);
  float* part = colsum_out ? reinterpret_cast<float*>(colsum_workspace) : nullptr;
  static const int fuse = env_switch("DV_FUSE_COLSUM", 1);
  int nparts = 0;
  bool bits_done = true;
  int rc = conv_down_impl(hi, w_packed, bias, mask, lo, B, H, W, CH, act, st, fuse ? part : nullptr, &nparts, mask_bits,
                          relu_bits_out, &bits_done);
  if (rc == DV_OK && relu_bits_out && !bits_done) rc = relu_bits(lo, relu_bits_out, (long long)B * H * W, st);
  if (rc != DV_OK || !colsum_out) return rc;
  if (nparts == 0) {                                           // this variant does not sum in its epilogue: one more pass over lo
    const long long rows = (long long)B * H * W;
    nparts = grid_for(rows, 8, kCsBlocks);
    channel_sum_nhwc_kernel<<<nparts, 256, 0, st>>>(lo, part, rows, kLoCh);
    rc = check_launch();
    if (rc != DV_OK) return rc;
  }
  channel_sum_final_kernel<<<1, 1024, 0, st>>>(part, colsum_out, nparts, kLoCh);
  return check_launch();
}

int dv_conv_up(const float* lo, const float* w_packed, const float* bias, const float* mask, float* hi,
               int B, int H, int W, int CH, int hi_nchw, int act, const unsigned* mask_bits, unsigned* relu_bits_out,
               void* stream) {
  if (!lo || !w_packed || !hi) return DV_ERR_BAD_ARG;
  if (mask_bits && !mask) return DV_ERR_BAD_ARG;
  if ((mask_bits || relu_bits_out) && CH != 32) return DV_ERR_BAD_ARG;   // one word per pixel = 32 NHWC channels
  if (!shape_ok(B, H, W, CH)) return DV_ERR_BAD_SHAPE;
  if (act != DV_ACT_NONE && act != DV_ACT_RELU && act != DV_ACT_SIGMOID) return DV_ERR_BAD_ARG;
  if ((CH == 32) == (hi_nchw != 0)) return DV_ERR_BAD_SHAPE;
  const float* wu = w_packed + kLoCh * CH * kTaps;
  if (CH != 32 && !mask && use_img() && img::shape_ok(B, H, W, CH))
    return img::conv_up(lo, wu, bias, hi, B, H, W, CH, act, as_stream(stream));
  if (CH == 32 && use_tc("halo") && act != DV_ACT_SIGMOID && W <= 32 && 128 % W == 0)
    return tc::conv_up_halo(lo, w_packed + kPackFfma + kPackTcSection, bias, mask, hi, B, H, W, act, as_stream(stream),
                            mask_bits, relu_bits_out);
  if (CH == 32) {
    const int smem = kTaps * 32 * kLoCh * sizeof(float);
    static bool attr_set = false;
    if (!attr_set) {
      if (cudaFuncSetAttribute(conv_up32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
        return DV_ERR_CUDA;
      attr_set = true;
    }
    const long long units = (long long)B * H * (W / kUpPos);
    const int grid = grid_for(units, kUpWarps, 2 * kNumSMs);
    conv_up32_kernel<<<grid, kUpWarps * 32, smem, as_stream(stream)>>>(lo, wu, bias, mask, hi, B, H, W, act);
    if (relu_bits_out) {                                        // (this fallback writes no bits in its epilogue)
      const int rc = check_launch();
      if (rc != DV_OK) return rc;
      return relu_bits(hi, relu_bits_out, (long long)B * 4 * H * W, as_stream(stream));
    }
  } else {
    const int grid = grid_for((long long)B * H * W, 256, 16 * kNumSMs);
    if (CH == 1) conv_up_small_kernel<1><<<grid, 256, 0, as_stream(stream)>>>(lo, wu, bias, mask, hi, B, H, W, act);
    else         conv_up_small_kernel<3><<<grid, 256, 0, as_stream(stream)>>>(lo, wu, bias, mask, hi, B, H, W, act);
  }
  return check_launch();
}

size_t dv_conv_wgrad_workspace_bytes(int B, int H, int W, int CH) {
  long long chunk;
  int ns = wgrad_nsplit(B, H, W, &chunk);
  if (ns < kNumSMs) ns = kNumSMs;                    // the tensor-core path uses at most one CTA per SM
  return (size_t)ns * (kTaps * CH + 1) * kLoCh * sizeof(float);
}

int dv_conv_wgrad(const float* lo, const float* hi, float* dw, float* dbias_lo, void* workspace,
                  size_t workspace_bytes, int B, int H, int W, int CH, int hi_nchw, void* stream) {
  if (!lo || !hi || !dw || !workspace) return DV_ERR_BAD_ARG;
  if (!shape_ok(B, H, W, CH)) return DV_ERR_BAD_SHAPE;
  if ((CH == 32) == (hi_nchw != 0)) return DV_ERR_BAD_SHAPE;
  if (workspace_bytes < dv_conv_wgrad_workspace_bytes(B, H, W, CH)) return DV_ERR_WORKSPACE;
  long long chunk;
  const int ns = wgrad_nsplit(B, H, W, &chunk);
  float* ws = reinterpret_cast<float*>(workspace);
  cudaStream_t st = as_stream(stream);
  if (CH != 32 && use_img() && img::shape_ok(B, H, W, CH)) {
    int nsplit_img = 0;
    const int max_split = (int)(dv_conv_wgrad_workspace_bytes(B, H, W, CH) / ((size_t)(kTaps * CH + 1) * kLoCh * sizeof(float)));
    int rc = img::conv_wgrad(lo, hi, ws, B, H, W, CH, max_split, &nsplit_img, st);
    if (rc != DV_OK) return rc;
    const int n = (kTaps * CH + 1) * kLoCh;
    conv_wgrad_reduce_kernel<<<(n + 31) / 32, 256, 0, st>>>(ws, dw, dbias_lo, CH, nsplit_img);
    return check_launch();
  }
  if (CH == 32 && use_tc("wgrad")) {
    int nsplit_tc = 0;
    int rc = tc::conv_wgrad32_tc(lo, hi, ws, B, H, W, &nsplit_tc, st);
    if (rc != DV_OK) return rc;
    const int n = (kTaps * CH + 1) * kLoCh;
    conv_wgrad_reduce_kernel<<<(n + 31) / 32, 256, 0, st>>>(ws, dw, dbias_lo, CH, nsplit_tc);
    return check_launch();
  }
  if (CH == 32)      conv_wgrad32_kernel<<<ns, kWgWarps * 32, 0, st>>>(lo, hi, ws, B, H, W, chunk);
  else if (CH == 3)  conv_wgrad_small_kernel<3><<<ns, kWgWarps * 32, 0, st>>>(lo, hi, ws, B, H, W, chunk);
  else               conv_wgrad_small_kernel<1><<<ns, kWgWarps * 32, 0, st>>>(lo, hi, ws, B, H, W, chunk);
  int rc = check_launch();
  if (rc != DV_OK) return rc;
  const int n = (kTaps * CH + 1) * kLoCh;
  conv_wgrad_reduce_kernel<<<(n + 31) / 32, 256, 0, st>>>(ws, dw, dbias_lo, CH, ns);
  return check_launch();
}

size_t dv_channel_sum_workspace_bytes(void) { return (size_t)kCsBlocks * 32 * sizeof(float); }

int dv_channel_sum(const float* x, float* out, long long rows, int C, int nchw, int hw, void* workspace, void* stream) {
  if (!x || !out || !workspace) return DV_ERR_BAD_ARG;
  if (C < 1 || C > 32 || rows <= 0) return DV_ERR_BAD_SHAPE;
  float* partial = reinterpret_cast<float*>(workspace);
  cudaStream_t st = as_stream(stream);
  int nb;
  if (nchw) {
    if (hw <= 0) return DV_ERR_BAD_SHAPE;
    nb = (int)(rows < kCsBlocks ? rows : kCsBlocks);
    channel_sum_nchw_kernel<<<nb, 256, 0, st>>>(x, partial, (int)rows, C, hw);
  } else {
    nb = grid_for(rows, 8, kCsBlocks);
    channel_sum_nhwc_kernel<<<nb, 256, 0, st>>>(x, partial, rows, C);
  }
  int rc = check_launch();
  if (rc != DV_OK) return rc;
  channel_sum_final_kernel<<<1, 1024, 0, st>>>(partial, out, nb, C);
  return check_launch();
}

int dv_flat_transpose(const float* src, float* dst, int B, int C, int S, int to_nhwc, void* stream) {
  if (!src || !dst) return DV_ERR_BAD_ARG;
  if (B <= 0 || C <= 0 || S <= 0) return DV_ERR_BAD_SHAPE;
  const long long n = (long long)B * C * S;
  flat_transpose_kernel<<<grid_for(n, 256, 8 * kNumSMs), 256, 0, as_stream(stream)>>>(src, dst, n, C, S, to_nhwc);
  return check_launch();
}

int dv_act_bwd(const float* dy, const float* y, float* g, long long n, int act, float slope, void* stream) {
  if (!dy || !y || !g) return DV_ERR_BAD_ARG;
  if (n <= 0) return DV_ERR_BAD_SHAPE;
  act_bwd_kernel<<<grid_for(n, 256, 16 * kNumSMs), 256, 0, as_stream(stream)>>>(dy, y, g, n, act, slope);
  return check_launch();
}

}  // extern "C"

// Convolution entry points (dv_conv_down / dv_conv_up / dv_conv_wgrad / packs) of the Burgess 4x4/stride-2/pad-1 layers.
// Each entry point checks the shape contract (include/disvae_b200.h) and then has one kernel per geometry: the
// 32-channel layers run on the tensor-core kernels of dv_conv_tc.cu, the image-boundary layers (CH in {1,3}) on the
// exact-fp32 kernels of dv_conv_img.cu.  This file also holds the split-K / channel-sum reductions they share and the
// small layout and activation-gradient kernels of the conv/linear seam.
//
// Every layer links lo[B,H,W,32] and hi[B,2H,2W,CH] through w[32][CH][4][4]
// (see include/disvae_b200.h).
//
// Reference call sites replaced: disvae/models/encoders.py:73-77 (Conv2d+ReLU),
// disvae/models/decoders.py:77-82 (ConvTranspose2d+ReLU/sigmoid) and their autograd
// backward (disvae/training.py:157).
#include <climits>
#include "dv_common.cuh"

namespace dv {

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
    if (act == DV_ACT_SIGMOID) r = (d * (1.f - yv)) * yv;      // aten sigmoid_backward: grad * (1 - y) * y, left to right
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

// The shape contract of the conv entry points: exactly the layers of the Burgess encoder and decoder on 32x32 and
// 64x64 images (vae.py:28), lo square.  CH in {1,3}: lo 16 or 32, hi NCHW;  CH == 32: lo 4, 8 or 16, hi NHWC.
static bool conv_shape_ok(int B, int H, int W, int CH, int hi_nchw) {
  if (B <= 0 || H != W) return false;
  if ((long long)B * 4 * H * W * kLoCh >= (1LL << 31)) return false;   // int pixel indices
  if (CH == 32) return !hi_nchw && (H == 4 || H == 8 || H == 16);
  if (CH == 1 || CH == 3) return hi_nchw && (H == 16 || H == 32);
  return false;
}

// The alignment contract of the conv entry points (include/disvae_b200.h): the tensor-core kernels read activations
// and packed weights through TMA, the image kernels move activations, masks and workspaces as 16-byte vectors; bias,
// weight-gradient, channel-sum and bit-word operands are read or written as single words.  The entry points refuse
// other addresses with `misaligned` (dv_common.cuh).
}  // namespace dv

namespace dv {
namespace tc {        // dv_conv_tc.cu: tensor-core kernels of the 32-channel layers
int pack_multi(int n, const float* const* w, float* const* wp, const int* CH, cudaStream_t st);
int conv_down32_tc(const float* hi, const float* wd_packed, const float* bias, const float* mask, float* lo,
                   int B, int H, int W, int act, cudaStream_t st, float* colsum_part, int* nparts,
                   const uint32_t* mask_bits, uint32_t* bits_out);
int conv_up_halo(const float* lo, const float* wu, const float* bias, const float* mask, float* hi,
                 int B, int H, int W, int act, cudaStream_t st, const uint32_t* mask_bits, uint32_t* bits_out);
int wgrad_splits(int B, int H, int W);
int conv_wgrad32_tc(const float* lo, const float* hi, float* ws, int B, int H, int W, cudaStream_t st);
}  // namespace tc
namespace img {       // dv_conv_img.cu: exact-fp32 CUDA-core kernels for the image-boundary layers (CH in {1,3})
int conv_down(const float* hi, const float* wd, const float* bias, const float* mask, const uint32_t* mask_bits, float* lo,
              uint32_t* bits_out, int B, int H, int W, int CH, int act, cudaStream_t st, float* colsum_part, int* nparts,
              int max_parts);
int wgrad_splits(int B, int H, int CH);
int conv_wgrad(const float* lo, const float* hi, float* ws, int B, int H, int W, int CH, cudaStream_t st);
int conv_up(const float* lo, const float* wu, const float* bias, float* hi, int B, int H, int W, int CH, int act, cudaStream_t st);
}  // namespace img

// packed-weight sections for CH == 32 (floats): [0, 32K) tensor-core down (hi|lo), [32K, 64K) tensor-core up (hi|lo)
constexpr int kPackTcSection = kTaps * 64 * 32;

// split-K partials of dv_conv_wgrad: one per CTA of the kernel that runs
static int wgrad_splits(int B, int H, int W, int CH) {
  return CH == 32 ? tc::wgrad_splits(B, H, W) : img::wgrad_splits(B, H, CH);
}
}  // namespace dv

using namespace dv;

extern "C" {

// CH in {1,3}: [0, 512*CH) down layout, [512*CH, 1024*CH) up layout of the dv_conv_img.cu kernels
size_t dv_conv_packed_floats(int CH) {
  return CH == 32 ? (size_t)2 * kPackTcSection : (size_t)2 * kLoCh * CH * kTaps;
}

int dv_conv_pack_weights(const float* w, float* w_packed, int CH, void* stream) {
  if (!w || !w_packed) return DV_ERR_BAD_ARG;
  if (CH != 1 && CH != 3 && CH != 32) return DV_ERR_BAD_SHAPE;
  return tc::pack_multi(1, &w, &w_packed, &CH, as_stream(stream));
}

int dv_conv_pack_multi(int n, const void* const* w, void* const* w_packed, const int* CH, void* stream) {
  if (n < 1 || !w || !w_packed || !CH) return DV_ERR_BAD_ARG;
  for (int i = 0; i < n; ++i) {
    if (!w[i] || !w_packed[i]) return DV_ERR_BAD_ARG;
    if (CH[i] != 1 && CH[i] != 3 && CH[i] != 32) return DV_ERR_BAD_SHAPE;
  }
  return tc::pack_multi(n, reinterpret_cast<const float* const*>(w), reinterpret_cast<float* const*>(w_packed), CH, as_stream(stream));
}

int dv_conv_down(const float* hi, const float* w_packed, const float* bias, const float* mask, float* lo,
                 int B, int H, int W, int CH, int hi_nchw, int act, float* colsum_out, void* colsum_workspace,
                 const unsigned* mask_bits, unsigned* relu_bits_out, void* stream) {
  if (!hi || !w_packed || !lo) return DV_ERR_BAD_ARG;
  if (mask_bits && !mask) return DV_ERR_BAD_ARG;               // the words accelerate the float mask, they do not replace it
  if (!conv_shape_ok(B, H, W, CH, hi_nchw)) return DV_ERR_BAD_SHAPE;
  if (act != DV_ACT_NONE && act != DV_ACT_RELU) return DV_ERR_BAD_ARG;
  if (misaligned(hi, 16) || misaligned(w_packed, 16) || misaligned(mask, 16) || misaligned(lo, 16) ||
      misaligned(colsum_workspace, 16) || misaligned(bias, 4) || misaligned(colsum_out, 4) ||
      misaligned(mask_bits, 4) || misaligned(relu_bits_out, 4))
    return DV_ERR_BAD_ARG;
  if (colsum_out && !colsum_workspace) return DV_ERR_WORKSPACE;
  cudaStream_t st = as_stream(stream);
  float* part = colsum_out ? reinterpret_cast<float*>(colsum_workspace) : nullptr;
  int nparts = 0;
  const int rc = CH == 32
      ? tc::conv_down32_tc(hi, w_packed, bias, mask, lo, B, H, W, act, st, part, &nparts, mask_bits, relu_bits_out)
      : img::conv_down(hi, w_packed, bias, mask, mask_bits, lo, relu_bits_out, B, H, W, CH, act, st, part, &nparts, kCsBlocks);
  if (rc != DV_OK || !colsum_out) return rc;
  channel_sum_final_kernel<<<1, 1024, 0, st>>>(part, colsum_out, nparts, kLoCh);
  return check_launch();
}

int dv_conv_up(const float* lo, const float* w_packed, const float* bias, const float* mask, float* hi,
               int B, int H, int W, int CH, int hi_nchw, int act, const unsigned* mask_bits, unsigned* relu_bits_out,
               void* stream) {
  if (!lo || !w_packed || !hi) return DV_ERR_BAD_ARG;
  if (mask_bits && !mask) return DV_ERR_BAD_ARG;
  if (!conv_shape_ok(B, H, W, CH, hi_nchw)) return DV_ERR_BAD_SHAPE;
  if (act != DV_ACT_NONE && act != DV_ACT_RELU && act != DV_ACT_SIGMOID) return DV_ERR_BAD_ARG;
  if (act == DV_ACT_SIGMOID && CH == 32) return DV_ERR_BAD_ARG;          // sigmoid only follows the image layer
  if ((mask || relu_bits_out) && CH != 32) return DV_ERR_BAD_ARG;        // mask epilogues of the 32-channel kernel only
  if (misaligned(lo, 16) || misaligned(w_packed, 16) || misaligned(mask, 16) || misaligned(hi, 16) ||
      misaligned(bias, 4) || misaligned(mask_bits, 4) || misaligned(relu_bits_out, 4))
    return DV_ERR_BAD_ARG;
  if (CH == 32)
    return tc::conv_up_halo(lo, w_packed + kPackTcSection, bias, mask, hi, B, H, W, act, as_stream(stream), mask_bits,
                            relu_bits_out);
  return img::conv_up(lo, w_packed + kLoCh * CH * kTaps, bias, hi, B, H, W, CH, act, as_stream(stream));
}

size_t dv_conv_wgrad_workspace_bytes(int B, int H, int W, int CH) {
  if (!conv_shape_ok(B, H, W, CH, CH != 32)) return 0;
  return (size_t)wgrad_splits(B, H, W, CH) * (kTaps * CH + 1) * kLoCh * sizeof(float);
}

int dv_conv_wgrad(const float* lo, const float* hi, float* dw, float* dbias_lo, void* workspace,
                  size_t workspace_bytes, int B, int H, int W, int CH, int hi_nchw, void* stream) {
  if (!lo || !hi || !dw || !workspace) return DV_ERR_BAD_ARG;
  if (!conv_shape_ok(B, H, W, CH, hi_nchw)) return DV_ERR_BAD_SHAPE;
  if (misaligned(lo, 16) || misaligned(hi, 16) || misaligned(workspace, 16) || misaligned(dw, 4) ||
      misaligned(dbias_lo, 4))
    return DV_ERR_BAD_ARG;
  if (workspace_bytes < dv_conv_wgrad_workspace_bytes(B, H, W, CH)) return DV_ERR_WORKSPACE;
  float* ws = reinterpret_cast<float*>(workspace);
  cudaStream_t st = as_stream(stream);
  const int rc = CH == 32 ? tc::conv_wgrad32_tc(lo, hi, ws, B, H, W, st) : img::conv_wgrad(lo, hi, ws, B, H, W, CH, st);
  if (rc != DV_OK) return rc;
  const int n = (kTaps * CH + 1) * kLoCh;
  conv_wgrad_reduce_kernel<<<(n + 31) / 32, 256, 0, st>>>(ws, dw, dbias_lo, CH, wgrad_splits(B, H, W, CH));
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
    if (hw <= 0 || rows > INT_MAX) return DV_ERR_BAD_SHAPE;   // the kernel counts images in int
    nb =(int)(rows < kCsBlocks ? rows : kCsBlocks);
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
  if (B <= 0 || C <= 0 || S <= 0 || (long long)C * S > INT_MAX) return DV_ERR_BAD_SHAPE;   // C * S indexes in int
  const long long n = (long long)B * C * S;
  flat_transpose_kernel<<<grid_for(n, 256, 8 * kNumSMs), 256, 0, as_stream(stream)>>>(src, dst, n, C, S, to_nhwc);
  return check_launch();
}

int dv_act_bwd(const float* dy, const float* y, float* g, long long n, int act, float slope, void* stream) {
  if (!dy || !y || !g) return DV_ERR_BAD_ARG;
  if (n <= 0) return DV_ERR_BAD_SHAPE;
  if (act != DV_ACT_NONE && act != DV_ACT_RELU && act != DV_ACT_SIGMOID && act != DV_ACT_LEAKY) return DV_ERR_BAD_ARG;
  act_bwd_kernel<<<grid_for(n, 256, 16 * kNumSMs), 256, 0, as_stream(stream)>>>(dy, y, g, n, act, slope);
  return check_launch();
}

}  // extern "C"

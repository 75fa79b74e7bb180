// Small fused "glue" kernels that replace chains of tiny framework launches on the training step
// (VERDICT r1 #8 "launch and glue diet") and the uint8 input path (SURVEY.md 8f-3).
//
//   dv_u8_to_f32          uint8 image batch -> fp32 / 255  (torchvision ToTensor semantics, utils/datasets.py:182,247,
//                         364-367: `img.float().div(255)`), so a host batch travels over PCIe as bytes (4x less H2D)
//   dv_gather_u8_to_f32   the same conversion of rows picked by an index list from a device-resident uint8 dataset:
//                         one training batch per launch (disvae.data.DeviceLoader)
//   dv_loss_combine_*     loss = sum_i ca[i]*a[i] + sum_j cb[j]*b[j] for two short device vectors (the fused loss kernel's
//                         (rec, kl, ...) and the beta-TCVAE (mi, tc, dw_kl)): losses.py:151, 199-200, 381-382 as ONE
//                         launch forward and ONE backward instead of ~10 scalar mul/add/select kernels and their
//                         zero-filled gradient buffers
//   dv_loss_combine_sched_*  the same with the annealing coefficient computed on the device from the loss's step counter
//   dv_betab_loss_*       beta-VAE_B's rec + gamma*|kl - C(step)| (losses.py:199-200) with its autograd gradient
//   dv_loss_record        the device loss log: a recording step's scalars into a ring row (also done by the two above)
//   dv_act_bwd_chansum    ConvTranspose2d output layer backward prologue: g = dy * act'(y) (decoders.py:82 sigmoid) fused
//                         with the per-channel sum of g (that layer's bias gradient) -- one pass instead of two
#include <algorithm>
#include <climits>
#include "dv_common.cuh"

namespace dv {

// torchvision ToTensor's byte -> float: true division, like Tensor.div(255) (not a multiply by 1/255)
__device__ __forceinline__ float u8_to_unit(uint32_t b) { return (float)b / 255.0f; }
__device__ __forceinline__ float4 u8x4_to_unit(uint32_t w) {
  return make_float4(u8_to_unit(w & 0xffu), u8_to_unit((w >> 8) & 0xffu), u8_to_unit((w >> 16) & 0xffu),
                     u8_to_unit(w >> 24));
}

__global__ void u8_to_f32_kernel(const uint8_t* __restrict__ src, float* __restrict__ dst, long long n) {
  const long long n16 = n >> 4;
  const uint4* s4 = reinterpret_cast<const uint4*>(src);
  float4* d4 = reinterpret_cast<float4*>(dst);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = s4[i];
    d4[4 * i + 0] = u8x4_to_unit(v.x);
    d4[4 * i + 1] = u8x4_to_unit(v.y);
    d4[4 * i + 2] = u8x4_to_unit(v.z);
    d4[4 * i + 3] = u8x4_to_unit(v.w);
  }
  for (long long i = (n16 << 4) + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = u8_to_unit(src[i]);
}

// dst row i = src row idx[i] / 255; one thread per 16-byte chunk of a destination row (row_bytes a multiple of 16).
__global__ void __launch_bounds__(256)
gather_u8_to_f32_kernel(const uint8_t* __restrict__ src, const long long* __restrict__ idx, int nrows, int chunks,
                        float* __restrict__ dst) {
  const long long n = (long long)nrows * chunks;
  float4* d4 = reinterpret_cast<float4*>(dst);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / chunks, c = i - row * chunks;
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(src) + idx[row] * chunks + c);
    d4[4 * i + 0] = u8x4_to_unit(v.x);
    d4[4 * i + 1] = u8x4_to_unit(v.y);
    d4[4 * i + 2] = u8x4_to_unit(v.z);
    d4[4 * i + 3] = u8x4_to_unit(v.w);
  }
}

struct Coefs { float a[8]; float b[8]; };

// The arithmetic both combine kernels share, spelled out (an fma chain per vector, then one add) so that the host-
// coefficient and the scheduled kernel round identically.
__device__ __forceinline__ float combine_value(const float* a, int na, const float* b, int nb, const Coefs& c) {
  float s = 0.f;
  for (int i = 0; i < na; ++i) s = __fmaf_rn(c.a[i], a[i], s);  // fixed order: rec first, like rec + (...) in the reference
  float t = 0.f;
  for (int j = 0; j < nb; ++j) t = __fmaf_rn(c.b[j], b[j], t);
  return __fadd_rn(s, t);
}

__global__ void loss_combine_fwd_kernel(const float* __restrict__ a, int na, const float* __restrict__ b, int nb, Coefs c,
                                        float* __restrict__ loss) {
  if (threadIdx.x != 0) return;
  loss[0] = combine_value(a, na, b, nb, c);
}

// ---- annealed coefficients from a device step counter (dv_loss_combine_sched_*, dv_betab_loss_*, dv_loss_record) ----
// linear_annealing(init, fin, step, steps_anneal) of losses.py in double, in Python's operation order:
// min(init + (fin - init) * step / steps_anneal, fin), or fin outside training and when steps_anneal == 0.
__device__ __forceinline__ double anneal_value(double init, double fin, long long step, long long steps_anneal,
                                               int is_train) {
  if (!is_train || steps_anneal == 0) return fin;
  const double x = __dadd_rn(init, __ddiv_rn(__dmul_rn(__dsub_rn(fin, init), (double)step), (double)steps_anneal));
  return fin < x ? fin : x;                                     // Python's min(x, fin) keeps x unless fin < x
}

// Thread 0: the step this launch computes for -- on a training step the counter is advanced first.
__device__ __forceinline__ long long take_step(long long* step, int is_train) {
  if (!is_train) return 0;
  const long long s = *step + 1;
  *step = s;
  return s;
}

// Whole block: when `step` records (step % every == 1, losses.py's rule), concatenate the sources into ring row
// ((step - 1) / every) % cap.  A NULL source (length 1) is `self_value`, the scalar the calling kernel just computed.
__device__ void log_record(const dv_loss_log& L, long long step, float self_value) {
  if (step % L.every != 1) return;
  float* row = L.ring + ((step - 1) / L.every % L.cap) * (long long)L.ncols;
  int off = 0;
  for (int k = 0; k < L.nsrc; ++k) {
    const float* src = L.src[k];
    for (int i = threadIdx.x; i < L.len[k]; i += blockDim.x) row[off + i] = src ? src[i] : self_value;
    off += L.len[k];
  }
}

struct Sched {
  double base[16];              // coefficient k: base[k], times the annealing value when bit k of `mask` is set
  unsigned mask;
  double init, fin;
  long long steps_anneal;
  int is_train;
};

__global__ void loss_combine_sched_fwd_kernel(const float* __restrict__ a, int na, const float* __restrict__ b, int nb,
                                              Sched sc, long long* __restrict__ step, float* __restrict__ loss,
                                              float* __restrict__ coefs, dv_loss_log log) {
  long long s = 0;
  float value = 0.f;
  if (threadIdx.x == 0) {
    s = take_step(step, sc.is_train);
    const double v = anneal_value(sc.init, sc.fin, s, sc.steps_anneal, sc.is_train);
    Coefs c = {};
    for (int k = 0; k < na + nb; ++k) {
      // (float)(anneal * base): what ctypes made of the Python product anneal_reg * coefficient
      const float ck = __double2float_rn((sc.mask >> k) & 1u ? __dmul_rn(v, sc.base[k]) : sc.base[k]);
      if (k < na) c.a[k] = ck; else c.b[k - na] = ck;
      coefs[k] = ck;
    }
    value = combine_value(a, na, b, nb, c);
    loss[0] = value;
  }
  if (!log.ring || !sc.is_train) return;
  s = __shfl_sync(0xffffffffu, s, 0);
  value = __shfl_sync(0xffffffffu, value, 0);
  log_record(log, s, value);
}

__global__ void loss_combine_sched_bwd_kernel(const float* __restrict__ g, const float* __restrict__ coefs, int na,
                                              int na_total, int nb, float* __restrict__ g_a, float* __restrict__ g_b) {
  const float gv = g[0];
  for (int i = threadIdx.x; i < na_total; i += blockDim.x) g_a[i] = i < na ? gv * coefs[i] : 0.f;
  if (g_b)
    for (int j = threadIdx.x; j < nb; j += blockDim.x) g_b[j] = gv * coefs[na + j];
}

struct BetaB { double gamma, c_init, c_fin; long long steps_anneal; int is_train; };

// rec + gamma * |kl - C| with torch's rounding: kl - C and gamma * |.| in float, then the add (losses.py:199-200)
__global__ void betab_loss_fwd_kernel(const float* __restrict__ rec_kl, BetaB p, long long* __restrict__ step,
                                      float* __restrict__ loss, float* __restrict__ consts, dv_loss_log log) {
  long long s = 0;
  float value = 0.f;
  if (threadIdx.x == 0) {
    s = take_step(step, p.is_train);
    const float C = __double2float_rn(anneal_value(p.c_init, p.c_fin, s, p.steps_anneal, p.is_train));
    const float gm = __double2float_rn(p.gamma);
    value = __fadd_rn(rec_kl[0], __fmul_rn(gm, fabsf(__fsub_rn(rec_kl[1], C))));
    loss[0] = value;
    consts[0] = C;
    consts[1] = gm;
  }
  if (!log.ring || !p.is_train) return;
  s = __shfl_sync(0xffffffffu, s, 0);
  value = __shfl_sync(0xffffffffu, value, 0);
  log_record(log, s, value);
}

// The gradient autograd gives the same expression: d rec = g, d kl = (g * gamma) * sgn(kl - C) with sgn(0) = 0, each
// landing in a zero-filled [n] buffer (hence the + 0: -0 becomes +0 as it does there); zeros past the two.
__global__ void betab_loss_bwd_kernel(const float* __restrict__ g, const float* __restrict__ rec_kl,
                                      const float* __restrict__ consts, int n, float* __restrict__ g_out) {
  const float gv = g[0];
  const float d = __fsub_rn(rec_kl[1], consts[0]);
  const float sg = (float)((d > 0.f) - (d < 0.f));
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    g_out[i] = i == 0 ? __fadd_rn(0.f, gv) : i == 1 ? __fadd_rn(0.f, __fmul_rn(__fmul_rn(gv, consts[1]), sg)) : 0.f;
}

__global__ void loss_record_kernel(const long long* __restrict__ step, dv_loss_log log) {
  log_record(log, *step, 0.f);
}

// g_a has na_total entries (the producing node's full output, e.g. 2 + latent_dim): zeros beyond the na weighted ones
__global__ void loss_combine_bwd_kernel(const float* __restrict__ g, int na, int na_total, int nb, Coefs c,
                                        float* __restrict__ g_a, float* __restrict__ g_b) {
  const float gv = g[0];
  for (int i = threadIdx.x; i < na_total; i += blockDim.x) g_a[i] = i < na ? gv * c.a[i] : 0.f;
  if (g_b)
    for (int j = threadIdx.x; j < nb; j += blockDim.x) g_b[j] = gv * c.b[j];
}

// one block walks whole (image, channel) planes: plane p = b*C + c; per-channel partial sums -> partial[block][32]
__global__ void __launch_bounds__(256)
act_bwd_chansum_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ g, int planes, int C,
                       int hw, int act, float slope, float* __restrict__ partial) {
  __shared__ float red[8][4];
  float cs[4] = {0.f, 0.f, 0.f, 0.f};
  const int hw4 = hw >> 2;
  for (int p = blockIdx.x; p < planes; p += gridDim.x) {
    const int c = p % C;
    const float4* dy4 = reinterpret_cast<const float4*>(dy + (long long)p * hw);
    const float4* y4 = reinterpret_cast<const float4*>(y + (long long)p * hw);
    float4* g4 = reinterpret_cast<float4*>(g + (long long)p * hw);
    float s = 0.f;
    for (int i = threadIdx.x; i < hw4; i += blockDim.x) {
      const float4 d = dy4[i], yv = y4[i];
      float4 r;
      if (act == DV_ACT_SIGMOID) {                             // aten sigmoid_backward: grad * (1 - y) * y, left to right
        r.x = (d.x * (1.f - yv.x)) * yv.x; r.y = (d.y * (1.f - yv.y)) * yv.y;
        r.z = (d.z * (1.f - yv.z)) * yv.z; r.w = (d.w * (1.f - yv.w)) * yv.w;
      } else if (act == DV_ACT_RELU) {
        r.x = yv.x > 0.f ? d.x : 0.f; r.y = yv.y > 0.f ? d.y : 0.f; r.z = yv.z > 0.f ? d.z : 0.f; r.w = yv.w > 0.f ? d.w : 0.f;
      } else if (act == DV_ACT_LEAKY) {
        r.x = yv.x > 0.f ? d.x : d.x * slope; r.y = yv.y > 0.f ? d.y : d.y * slope;
        r.z = yv.z > 0.f ? d.z : d.z * slope; r.w = yv.w > 0.f ? d.w : d.w * slope;
      } else r = d;
      g4[i] = r;
      s += (r.x + r.y) + (r.z + r.w);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) if (k == c) cs[k] += s;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float v = warp_sum(cs[k]);
    if (lane == 0) red[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = 0.f;
    if (threadIdx.x < 4)
      for (int w = 0; w < 8; ++w) t += red[w][threadIdx.x];
    partial[blockIdx.x * 32 + threadIdx.x] = t;                // channel_sum_final_kernel layout: [block][32]
  }
}

__global__ void __launch_bounds__(1024)
chansum_final32_kernel(const float* __restrict__ partial, float* __restrict__ out, int nblocks, int C) {
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

}  // namespace dv

using namespace dv;

extern "C" {

int dv_u8_to_f32(const unsigned char* src, float* dst, long long n, void* stream) {
  if (!src || !dst) return DV_ERR_BAD_ARG;
  if (n <= 0) return DV_ERR_BAD_SHAPE;
  if (((uintptr_t)src & 15) || ((uintptr_t)dst & 15)) return DV_ERR_BAD_ARG;
  long long blocks = ((n >> 4) + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > 8 * kNumSMs) blocks = 8 * kNumSMs;
  u8_to_f32_kernel<<<(int)blocks, 256, 0, as_stream(stream)>>>(src, dst, n);
  return check_launch();
}

int dv_gather_u8_to_f32(const unsigned char* src, const long long* idx, int nrows, int row_bytes, float* dst,
                        void* stream) {
  if (!src || !idx || !dst) return DV_ERR_BAD_ARG;
  if (nrows < 1 || row_bytes < 16 || (row_bytes & 15)) return DV_ERR_BAD_SHAPE;
  if (((uintptr_t)src & 15) || ((uintptr_t)dst & 15) || ((uintptr_t)idx & 7)) return DV_ERR_BAD_ARG;
  const int chunks = row_bytes >> 4;
  const long long blocks = std::min<long long>(((long long)nrows * chunks + 255) / 256, 8 * kNumSMs);
  gather_u8_to_f32_kernel<<<(int)blocks, 256, 0, as_stream(stream)>>>(src, idx, nrows, chunks, dst);
  return check_launch();
}

int dv_loss_combine_fwd(const float* a, const float* coef_a, int na, const float* b, const float* coef_b, int nb, float* loss,
                        void* stream) {
  if (!a || !coef_a || !loss || na < 1 || na > 8 || nb < 0 || nb > 8 || (nb > 0 && (!b || !coef_b))) return DV_ERR_BAD_ARG;
  Coefs c = {};
  for (int i = 0; i < na; ++i) c.a[i] = coef_a[i];             // HOST arrays: the coefficients travel by value
  for (int j = 0; j < nb; ++j) c.b[j] = coef_b[j];
  loss_combine_fwd_kernel<<<1, 32, 0, as_stream(stream)>>>(a, na, b, nb, c, loss);
  return check_launch();
}

int dv_loss_combine_bwd(const float* g, const float* coef_a, int na, int na_total, const float* coef_b, int nb, float* g_a,
                        float* g_b, void* stream) {
  if (!g || !coef_a || !g_a || na < 1 || na > 8 || na_total < na || nb < 0 || nb > 8 || (nb > 0 && !coef_b)) return DV_ERR_BAD_ARG;
  Coefs c = {};
  for (int i = 0; i < na; ++i) c.a[i] = coef_a[i];
  for (int j = 0; j < nb; ++j) c.b[j] = coef_b[j];
  loss_combine_bwd_kernel<<<1, 128, 0, as_stream(stream)>>>(g, na, na_total, nb, c, g_a, g_b);
  return check_launch();
}

}  // extern "C"

// A caller's log description -> the kernel argument (ring == NULL: no record).  self_ok: a NULL source of length 1 may
// stand for the launch's own result.
static int log_arg(const dv_loss_log* log, bool self_ok, dv_loss_log* out) {
  *out = dv_loss_log{};
  if (!log) return DV_OK;
  if (!log->ring || log->cap < 1 || log->every < 1 || log->nsrc < 1 || log->nsrc > DV_LOSS_LOG_MAX_SRC) return DV_ERR_BAD_ARG;
  int total = 0;
  for (int k = 0; k < log->nsrc; ++k) {
    if (log->len[k] < 0 || (!log->src[k] && !(self_ok && log->len[k] == 1))) return DV_ERR_BAD_ARG;
    total += log->len[k];
  }
  if (total != log->ncols) return DV_ERR_BAD_SHAPE;
  *out = *log;
  return DV_OK;
}

extern "C" {

int dv_loss_combine_sched_fwd(const float* a, int na, const float* b, int nb, const double* base, unsigned sched_mask,
                              double init, double fin, long long steps_anneal, int is_train, long long* step, float* loss,
                              float* coefs, const dv_loss_log* log, void* stream) {
  if (!a || !base || !loss || !coefs || na < 1 || na > 8 || nb < 0 || nb > 8 || (nb > 0 && !b)) return DV_ERR_BAD_ARG;
  if (steps_anneal < 0 || (is_train && !step) || (sched_mask >> (na + nb)) != 0) return DV_ERR_BAD_ARG;
  Sched sc = {};
  for (int k = 0; k < na + nb; ++k) sc.base[k] = base[k];       // HOST array: travels by value
  sc.mask = sched_mask;
  sc.init = init;
  sc.fin = fin;
  sc.steps_anneal = steps_anneal;
  sc.is_train = is_train ? 1 : 0;
  dv_loss_log L;
  const int rc = log_arg(is_train ? log : nullptr, true, &L);
  if (rc != DV_OK) return rc;
  loss_combine_sched_fwd_kernel<<<1, 32, 0, as_stream(stream)>>>(a, na, b, nb, sc, step, loss, coefs, L);
  return check_launch();
}

int dv_loss_combine_sched_bwd(const float* g, const float* coefs, int na, int na_total, int nb, float* g_a, float* g_b,
                              void* stream) {
  if (!g || !coefs || !g_a || na < 1 || na > 8 || na_total < na || nb < 0 || nb > 8) return DV_ERR_BAD_ARG;
  loss_combine_sched_bwd_kernel<<<1, 128, 0, as_stream(stream)>>>(g, coefs, na, na_total, nb, g_a, nb > 0 ? g_b : nullptr);
  return check_launch();
}

int dv_betab_loss_fwd(const float* rec_kl, double gamma, double c_init, double c_fin, long long steps_anneal, int is_train,
                      long long* step, float* loss, float* consts, const dv_loss_log* log, void* stream) {
  if (!rec_kl || !loss || !consts || steps_anneal < 0 || (is_train && !step)) return DV_ERR_BAD_ARG;
  const BetaB p = {gamma, c_init, c_fin, steps_anneal, is_train ? 1 : 0};
  dv_loss_log L;
  const int rc = log_arg(is_train ? log : nullptr, true, &L);
  if (rc != DV_OK) return rc;
  betab_loss_fwd_kernel<<<1, 32, 0, as_stream(stream)>>>(rec_kl, p, step, loss, consts, L);
  return check_launch();
}

int dv_betab_loss_bwd(const float* g, const float* rec_kl, const float* consts, int n, float* g_rec_kl, void* stream) {
  if (!g || !rec_kl || !consts || !g_rec_kl || n < 2) return DV_ERR_BAD_ARG;
  betab_loss_bwd_kernel<<<1, 128, 0, as_stream(stream)>>>(g, rec_kl, consts, n, g_rec_kl);
  return check_launch();
}

int dv_loss_record(const long long* step, const dv_loss_log* log, void* stream) {
  if (!step || !log) return DV_ERR_BAD_ARG;
  dv_loss_log L;
  const int rc = log_arg(log, false, &L);
  if (rc != DV_OK) return rc;
  loss_record_kernel<<<1, 32, 0, as_stream(stream)>>>(step, L);
  return check_launch();
}

int dv_act_bwd_chansum(const float* dy, const float* y, float* g, int B, int C, int hw, int act, float slope, float* chansum,
                       void* workspace, void* stream) {
  if (!dy || !y || !g || !chansum || !workspace) return DV_ERR_BAD_ARG;
  if (B < 1 || C < 1 || C > 4 || hw < 4 || (hw & 3) || (long long)B * C > INT_MAX) return DV_ERR_BAD_SHAPE;
  if (act != DV_ACT_NONE && act != DV_ACT_RELU && act != DV_ACT_SIGMOID && act != DV_ACT_LEAKY) return DV_ERR_BAD_ARG;
  // dy, y and g move as float4; the partial rows and the sums as single words
  if (((uintptr_t)dy & 15) || ((uintptr_t)y & 15) || ((uintptr_t)g & 15) || ((uintptr_t)chansum & 3) ||
      ((uintptr_t)workspace & 3))
    return DV_ERR_BAD_ARG;
  const int planes = B * C;
  const int grid = planes < 296 ? planes : 296;                // <= dv_channel_sum_workspace_bytes() / 128 partial rows
  float* partial = reinterpret_cast<float*>(workspace);
  cudaStream_t st = as_stream(stream);
  act_bwd_chansum_kernel<<<grid, 256, 0, st>>>(dy, y, g, planes, C, hw, act, slope, partial);
  int rc = check_launch();
  if (rc != DV_OK) return rc;
  chansum_final32_kernel<<<1, 1024, 0, st>>>(partial, chansum, grid, C);
  return check_launch();
}

}  // extern "C"

/*
 * disvae_b200.h -- C ABI of libdisvae_b200.so: hand-written sm_90a kernels for the
 * disvae training hot path (BASELINE.json:north_star, SURVEY.md section 8).
 *
 * The reference (YannDubs/disentangling-vae) is pure Python on PyTorch and has NO
 * native/FFI layer; every arithmetic op it runs is an ATen call.  Each entry point
 * below therefore cites the reference *call site* (file:line relative to the
 * reference checkout) whose ATen work it replaces.  The Python binding a maintainer
 * adds is a ctypes stub -- see INTEGRATION.md.
 *
 * Conventions
 *  - plain C: raw DEVICE pointers + explicit sizes; no torch types; fp32 everywhere.
 *  - the caller owns and allocates every buffer including workspaces
 *    (dv_*_workspace_bytes() say how much); the callee never allocates, frees or retains.
 *  - every call is asynchronous on `stream` (a cudaStream_t passed as void*), re-entrant
 *    across streams, CUDA-graph capturable (no host sync, no allocation, no host RNG).
 *  - return value: DV_OK (0) or a negative DvStatus.  Nothing throws.
 *  - activations between conv layers are NHWC ("pixel-major": 32 channels = one 128-byte
 *    line per pixel).  Images at the model boundary (input x, reconstruction) are NCHW,
 *    as the reference's callers expect (utils/visualize.py:219-222).
 *  - "lo"/"hi": every Burgess conv layer (k=4, s=2, p=1) links a low-resolution tensor
 *    lo[B,H,W,32] and a high-resolution tensor hi[B,2H,2W,CH], CH in {1,3,32}, through a
 *    weight w[32][CH][4][4].  That is the memory layout of BOTH nn.Conv2d.weight
 *    [Cout=32,Cin=CH,4,4] and nn.ConvTranspose2d.weight [Cin=32,Cout=CH,4,4]
 *    (SURVEY.md trap T14), so three kernels cover all conv work:
 *       down : hi -> lo   (Conv2d forward;           ConvTranspose2d input-gradient)
 *       up   : lo -> hi   (ConvTranspose2d forward;  Conv2d input-gradient)
 *       wgrad: lo x hi -> dw (both weight-gradients)
 */
#ifndef DISVAE_B200_H
#define DISVAE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum DvStatus {
  DV_OK = 0,
  DV_ERR_BAD_SHAPE = -1,     /* unsupported size / channel count */
  DV_ERR_BAD_ARG = -2,       /* null pointer, bad enum */
  DV_ERR_WORKSPACE = -3,     /* workspace too small */
  DV_ERR_CUDA = -4,          /* a CUDA runtime call failed; see dv_last_cuda_error() */
  DV_ERR_ARCH = -5           /* device is not sm_90 */
} DvStatus;

enum { DV_ACT_NONE = 0, DV_ACT_RELU = 1, DV_ACT_SIGMOID = 2, DV_ACT_LEAKY = 3 };
enum { DV_DIST_BERNOULLI = 0, DV_DIST_GAUSSIAN = 1, DV_DIST_LAPLACE = 2 };

/* ---- library probes ------------------------------------------------------------- */
int dv_version(void);                 /* 10000*major + 100*minor + patch */
int dv_built_arch(void);              /* 90 == compiled for sm_90a */
const char* dv_status_string(int status);
int dv_last_cuda_error(void);         /* cudaError_t of the last failing call on this thread */
int dv_device_check(void);            /* DV_OK if the current device is compute capability 9.0 */
/* how many kernels this library has launched in this process (for bench.py "gpu_launches") */
long long dv_launch_count(void);

/* ---- convolutions ---------------------------------------------------------------
 * Replaces: nn.Conv2d forward  (disvae/models/encoders.py:73-77)   -> dv_conv_down
 *           nn.ConvTranspose2d forward (disvae/models/decoders.py:77-82) -> dv_conv_up
 *           their autograd backward (disvae/training.py:157, aten::convolution_backward)
 *           -> dv_conv_up / dv_conv_down (input grads), dv_conv_wgrad (+ bias grads).
 * w is the torch weight tensor itself, [32][CH][4][4] contiguous; w_packed is produced by
 * dv_conv_pack_weights (layout private to the library).  B images, lo is H x W.
 * hi_nchw != 0: hi is [B,CH,2H,2W];  hi_nchw == 0: hi is [B,2H,2W,CH].
 * Shapes: the layers of the Burgess encoder and decoder on 32x32 and 64x64 images (vae.py:28).
 * dv_conv_down, dv_conv_up and dv_conv_wgrad return DV_ERR_BAD_SHAPE for anything else:
 *     CH       lo geometry (H == W)   layout of hi
 *     1 or 3   16 or 32               NCHW (hi_nchw != 0)
 *     32       4, 8 or 16             NHWC (hi_nchw == 0)
 * mask (optional, same shape/layout as the OUTPUT): out *= (mask > 0) -- the ReLU backward
 * of the layer that produced `mask`, fused into this epilogue.
 * Alignment (one rule for every layer): activations (hi, lo), mask, w_packed and the workspaces must be 16-byte
 * aligned; bias, dw, dbias_lo, colsum_out and the bit words (mask_bits, relu_bits_out) 4-byte aligned.  Otherwise
 * dv_conv_down, dv_conv_up and dv_conv_wgrad return DV_ERR_BAD_ARG before launching anything.
 */
size_t dv_conv_packed_floats(int CH);                         /* size of w_packed in floats */
int dv_conv_pack_weights(const float* w, float* w_packed, int CH, void* stream);
/* the same for n layers in ONE launch: w[i], w_packed[i] (dv_conv_packed_floats(CH[i]) floats each) and CH are HOST
 * arrays of device pointers / channel counts (the conv layers of an encoder or decoder node, whose weights only
 * change in the optimizer step). */
int dv_conv_pack_multi(int n, const void* const* w, void* const* w_packed, const int* CH, void* stream);
/* lo = act(down(hi) + bias) * [mask>0];  bias may be NULL.  act in {NONE, RELU}.
 * colsum_out (optional, [32]): sum of the stored `lo` over all pixels, accumulated in the kernel's
 * epilogue.  In the backward pass `lo` is the gradient reaching the previous ConvTranspose2d's
 * output, so this IS that layer's bias gradient (no extra pass over the tensor).
 * colsum_workspace: dv_channel_sum_workspace_bytes() bytes, required with colsum_out.
 * ReLU masks as bits (both optional, 32-channel NHWC outputs only, one 32-bit word per OUTPUT pixel, bit c =
 * channel c):  relu_bits_out receives [out > 0] of the stored tensor from the same epilogue -- kept by the
 * caller, it is the mask of the backward pass through the ReLU that follows this layer;  mask_bits is that
 * word form of `mask` (which must be passed as well): the backward epilogue then reads 4 bytes per pixel instead
 * of 128 (autograd's threshold_backward, fused and compressed). */
int dv_conv_down(const float* hi, const float* w_packed, const float* bias, const float* mask,
                 float* lo, int B, int H, int W, int CH, int hi_nchw, int act, float* colsum_out,
                 void* colsum_workspace, const unsigned* mask_bits, unsigned* relu_bits_out, void* stream);
/* hi = act(up(lo) + bias) * [mask>0];  bias[CH] may be NULL.  act in {NONE, RELU, SIGMOID}; SIGMOID for
 * CH in {1,3} only (DV_ERR_BAD_ARG otherwise).  mask, mask_bits and relu_bits_out as above, CH == 32 only
 * (DV_ERR_BAD_ARG otherwise). */
int dv_conv_up(const float* lo, const float* w_packed, const float* bias, const float* mask,
               float* hi, int B, int H, int W, int CH, int hi_nchw, int act, const unsigned* mask_bits,
               unsigned* relu_bits_out, void* stream);
/* dw[32][CH][4][4] = sum_pixels lo (x) patch(hi);  dbias_lo[32] (optional) = sum_pixels lo.
 * Deterministic split-K: partials go to `workspace`, reduced in a fixed order.  The workspace query returns 0
 * for a shape outside the table above. */
size_t dv_conv_wgrad_workspace_bytes(int B, int H, int W, int CH);
int dv_conv_wgrad(const float* lo, const float* hi, float* dw, float* dbias_lo, void* workspace,
                  size_t workspace_bytes, int B, int H, int W, int CH, int hi_nchw, void* stream);
/* out[C] = sum over all pixels of x; x is [rows, C] pixel-major (nchw == 0) or
 * [B, C, HW] (nchw != 0, rows = B, hw given).  Bias gradients of the ConvTranspose2d layers.
 * DV_ERR_BAD_SHAPE: C < 1, C > 32, rows < 1, or (nchw != 0) hw < 1 or rows > INT_MAX. */
size_t dv_channel_sum_workspace_bytes(void);
int dv_channel_sum(const float* x, float* out, long long rows, int C, int nchw, int hw,
                   void* workspace, void* stream);
/* [B,32,4,4] <-> [B,4,4,32] re-ordering at the conv/linear seam (encoders.py:80, decoders.py:74): [B][C][S] ->
 * [B][S][C] (to_nhwc != 0) or back.  DV_ERR_BAD_SHAPE: B, C or S < 1, or C * S > INT_MAX. */
int dv_flat_transpose(const float* src, float* dst, int B, int C, int S, int to_nhwc, void* stream);
/* g = dy * act'(y) for y = act(.) over n elements, as autograd computes it from the activation's output y:
 *   SIGMOID  aten sigmoid_backward, (dy * (1 - y)) * y in that order (decoders.py:82)
 *   RELU     dy where y > 0, else +0 (aten threshold_backward(dy, y, 0), except at y = NaN: 0 here, dy there;
 *            every ReLU mask of this library is [y > 0])
 *   LEAKY    dy where y > 0, else dy * slope (aten leaky_relu_backward with self_is_result)
 *   NONE     dy
 * DV_ERR_BAD_ARG: a NULL pointer or act outside these four.  DV_ERR_BAD_SHAPE: n < 1. */
int dv_act_bwd(const float* dy, const float* y, float* g, long long n, int act, float slope, void* stream);

/* ---- fully connected -------------------------------------------------------------
 * Replaces nn.Linear + activation: encoders.py:81-86, decoders.py:71-73, discriminator.py:63-68.
 * x[M,K], w[N,K] (torch layout), y[M,N].  slope is the LeakyReLU negative slope.
 */
/* The shape selects the kernel.  A reduction length (K forward, N input gradient) that is a multiple of 4 and at
 * least 32 runs on the tensor cores (mma.sync tf32, 3xTF32); the call then packs w into `workspace`
 * (dv_linear_packed_floats(N, K) floats, the layout of dv_linear_pack_multi) and reads the activation operand (x
 * forward, g input gradient) through TMA: both must be 16-byte aligned, or the call returns DV_ERR_BAD_ARG before
 * launching anything (DV_ERR_WORKSPACE when workspace is NULL).  Other shapes run on the CUDA cores (FFMA): the query
 * returns 0 for them, workspace may be NULL and 4-byte aligned operands are enough. */
size_t dv_linear_fwd_workspace_bytes(int M, int N, int K);
size_t dv_linear_dgrad_workspace_bytes(int M, int N, int K);
int dv_linear_fwd(const float* x, const float* w, const float* bias, float* y, int M, int N, int K,
                  int act, float slope, void* workspace, void* stream);
/* dx[M,K] = (g[M,N] . w[N,K]) * act'(mask_src[M,K]); mask_src is the POST-activation output
 * of the previous layer (NULL: no mask); act in {NONE, RELU, LEAKY}, anything else (with or without a mask) is
 * DV_ERR_BAD_ARG. */
int dv_linear_dgrad(const float* g, const float* w, const float* mask_src, float* dx, int M, int N,
                    int K, int act, float slope, void* workspace, void* stream);
/* dw[N,K] = g^T . x ; dbias[N] = column sums of g (may be NULL).  Small N*K problems are split over
 * the batch (deterministic split-K); workspace may be NULL when the query returns 0.  N % 4 == 0, K % 4 == 0, K >= 32
 * and M >= 32 run on the tensor cores, which read g and x through TMA: both must be 16-byte aligned there
 * (DV_ERR_BAD_ARG otherwise, before any launch). */
size_t dv_linear_wgrad_workspace_bytes(int M, int N, int K);
int dv_linear_wgrad(const float* g, const float* x, float* dw, float* dbias, int M, int N, int K,
                    void* workspace, void* stream);
/* Pre-packed weights: dv_linear_pack_multi splits n weight matrices (w[i]: [N[i], K[i]], HOST arrays of device
 * pointers / sizes) into the tensor-core hi/lo operand planes of BOTH directions in one launch, into caller-owned
 * buffers of dv_linear_packed_floats(N, K) floats (16-byte aligned); dv_linear_fwd_packed / dv_linear_dgrad_packed are
 * dv_linear_fwd / dv_linear_dgrad on those planes (w is still passed: shapes that run on the CUDA cores read it), with
 * the same refusals: on a tensor-core shape, NULL packed is DV_ERR_WORKSPACE, and packed or the activation operand
 * not 16-byte aligned is DV_ERR_BAD_ARG.
 * One pack launch per network node per step instead of one per layer per direction. */
size_t dv_linear_packed_floats(int N, int K);
int dv_linear_pack_multi(int n, const void* const* w, void* const* packed, const int* N, const int* K, void* stream);
int dv_linear_fwd_packed(const float* x, const float* w, const float* packed, const float* bias, float* y,
                         int M, int N, int K, int act, float slope, void* stream);
int dv_linear_dgrad_packed(const float* g, const float* w, const float* packed, const float* mask_src, float* dx,
                           int M, int N, int K, int act, float slope, void* stream);

/* ---- reparameterised sampling ------------------------------------------------------
 * Replaces VAE.reparameterize (disvae/models/vae.py:65-68): z = mu + exp(0.5*logvar)*eps.
 * mu/logvar are read with an element stride (`ld`), rows are `row_stride` apart, so the
 * interleaved encoder output (encoders.py:86-87) can be consumed in place.
 * eps_in != NULL: use the caller's noise (parity tests).  eps_in == NULL: Philox4x32-10 +
 * Box-Muller on the device, keyed by (seed, *offset_dev + element index); the kernel then
 * advances *offset_dev by B*D (graph-replay safe).  eps_out (optional) receives the noise.
 */
int dv_reparam_fwd(const float* mu, const float* logvar, int ld, int row_stride, const float* eps_in,
                   unsigned long long seed, unsigned long long* offset_dev, float* z, float* eps_out,
                   int B, int D, void* stream);
/* g_mu = g_z ; g_logvar = g_z * eps * 0.5 * exp(0.5*logvar)  (contiguous [B,D] outputs) */
int dv_reparam_bwd(const float* g_z, const float* logvar, int ld, int row_stride, const float* eps,
                   float* g_mu, float* g_logvar, int B, int D, void* stream);

/* ---- fused reconstruction loss + analytic KL ---------------------------------------
 * Replaces _reconstruction_loss (losses.py:394-449) and _kl_normal_loss (losses.py:452-480)
 * in ONE launch.  out[0] = reconstruction loss (sum / B, all three distributions, traps
 * T8/T9), out[1] = total KL, out[2+d] = per-dimension KL (the kl_loss_<d> log entries).
 * recon/data: n_img_elems = C*H*W per image, any layout (same for both).
 */
/* workspace: zero on first use (the kernel leaves its counter at zero). */
size_t dv_vae_loss_workspace_bytes(int B, long long n_img_elems);
int dv_vae_loss_fwd(const float* recon, const float* data, long long n_img_elems, int B, int dist,
                    const float* mu, const float* logvar, int ld, int row_stride, int D,
                    float* out, void* workspace, void* stream);
/* upstream = device float[2]: d loss / d out[0], d loss / d out[1].  g_recon like recon;
 * g_mu, g_logvar contiguous [B,D].  Any output pointer may be NULL. */
int dv_vae_loss_bwd(const float* recon, const float* data, long long n_img_elems, int B, int dist,
                    const float* mu, const float* logvar, int ld, int row_stride, int D,
                    const float* fwd_out, const float* upstream, float* g_recon, float* g_mu,
                    float* g_logvar, void* stream);

/* ---- beta-TCVAE log-density decomposition --------------------------------------------
 * Replaces _get_log_pz_qz_prodzi_qzCx (losses.py:523-544) + matrix_log_density_gaussian /
 * log_importance_weight_matrix (disvae/utils/math.py:8-73) + the three means at
 * losses.py:369-373.  Nothing B x B (x D) is ever materialised; the importance-weight
 * matrix is evaluated analytically from its column structure (trap T3), D-fold in log_qz
 * (trap T2).  is_mss == 0 reproduces the reference's is_mss=False branch (trap T4).
 * rowstats is a structure of arrays [4 + D][B]: rows log_pz, log_qz, log_prod_qzi, log_q_zCx,
 * then the per-dimension logsumexp P[d][i] (kept for the backward).  terms[3] = mi, tc, dw_kl.
 * `workspace` must be 16-byte aligned and its first 64 bytes zero on first use (the kernel
 * leaves them zero); it holds the per-column parameters the backward re-reads, so pass the
 * SAME workspace (untouched) and rowstats to dv_btcvae_bwd.
 */
size_t dv_btcvae_workspace_bytes(int B, int D);
int dv_btcvae_fwd(const float* z, const float* mu, const float* logvar, int ld, int row_stride,
                  int B, int D, long long n_data, int is_mss, float* rowstats, float* terms,
                  void* workspace, void* stream);
/* g_terms = device float[3] (d loss / d mi, tc, dw_kl); outputs contiguous [B,D] (any may be NULL). */
int dv_btcvae_bwd(int B, int D, long long n_data, int is_mss, const float* rowstats,
                  const void* workspace, const float* g_terms, float* g_z, float* g_mu,
                  float* g_logvar, void* stream);
/* Row-window form (SURVEY.md 8f-1: the estimator over a batch all-gathered from several GPUs, each rank
 * evaluating its own rows of the B x B matrix -- losses.py:523-544 semantics of the GLOBAL batch).
 * z / mu / logvar hold all B rows; only rows [row0, row0 + nrows) are evaluated: their rowstats entries are
 * written (global row index), terms = means over the window.  Backward: g_z is [nrows, D] (the window's rows);
 * g_mu / g_logvar are [B, D] PARTIAL sums over the window's rows for every column -- summing them over the
 * windows of all ranks (reduce-scatter) gives the gradient of the mean-over-ranks loss.
 * dv_btcvae_fwd / dv_btcvae_bwd are the (0, B) window. */
int dv_btcvae_fwd_rows(const float* z, const float* mu, const float* logvar, int ld, int row_stride,
                       int B, int D, int row0, int nrows, long long n_data, int is_mss, float* rowstats,
                       float* terms, void* workspace, void* stream);
int dv_btcvae_bwd_rows(int B, int D, int row0, int nrows, long long n_data, int is_mss,
                       const float* rowstats, const void* workspace, const float* g_terms, float* g_z,
                       float* g_mu, float* g_logvar, void* stream);

/* ---- DIP-VAE covariance penalty ----------------------------------------------------------------
 * The reference has no DIP-VAE: these implement Kumar et al. 2018 ("Variational Inference of Disentangled Latent
 * Concepts from Unlabeled Observations"), the regulariser of eq. 6 (DIP-VAE-I) and of the second form in section 3
 * (DIP-VAE-II), on the batch of encoder outputs mu / logvar [B, D] (element (b, d) at b*row_stride + d*ld, as for
 * dv_vae_loss_fwd: the interleaved encoder output is read in place):
 *   Cov_mu = (1/B) sum_b c_b c_b^T   (biased; c_b = (mu_b - m1) - mean_b(mu_b - m1), m1 = mu_0 + mean_b(mu_b - mu_0):
 *            centred on an accurate mean, whatever the offset of a column and whichever row comes first)
 *   C = Cov_mu (DV_DIP_I)  or  Cov_mu + diag(mean_b exp(logvar_b)) (DV_DIP_II)
 *   terms_out[0] = od = sum_{i != j} C_ij^2,   terms_out[1] = dd = sum_i (C_ii - 1)^2   (unweighted)
 * The weights lambda_od, lambda_d and the annealing are applied by the caller (dv_loss_combine_sched_fwd).
 * workspace: dv_dip_workspace_bytes(B, D) bytes, 16-byte aligned, contents irrelevant on entry; the forward leaves the
 * column means and C in it for dv_dip_bwd, so pass the SAME workspace untouched.  Deterministic (fixed-order
 * reductions, no floating-point atomics).  logvar is read only by DV_DIP_II but must be a valid pointer for both.
 * DV_ERR_BAD_SHAPE: B < 1, B > 65535 * 32 = 2097120 (the backward runs one CTA row per 32 rows of the batch), D < 1,
 * D > 1024, ld < 1, row_stride < 1, or dip_type not DV_DIP_I / DV_DIP_II.
 * DV_ERR_BAD_ARG: a NULL required pointer, or mu / logvar / terms / gradients not 4-byte or workspace not 16-byte aligned.
 * Backward: g_terms = device float[2], the upstream gradient of (od, dd) (the lambdas and the annealing included);
 *   g_mu[b] = (2/B) G c_b with G_ij = 2 g_terms[0] C_ij (i != j), G_ii = 2 g_terms[1] (C_ii - 1);
 *   g_logvar[b][i] = G_ii exp(logvar[b][i]) / B for DV_DIP_II, 0 for DV_DIP_I.
 *   Outputs contiguous [B, D]; either may be NULL (both NULL: nothing is launched). */
enum { DV_DIP_I = 1, DV_DIP_II = 2 };
size_t dv_dip_workspace_bytes(int B, int D);      /* 0 for an unsupported B or D */
int dv_dip_fwd(const float* mu, const float* logvar, int ld, int row_stride, int B, int D, int dip_type,
               float* terms_out, void* workspace, void* stream);
int dv_dip_bwd(const float* mu, const float* logvar, int ld, int row_stride, int B, int D, int dip_type,
               const float* g_terms, float* g_mu, float* g_logvar, const void* workspace, void* stream);

/* ---- input pipeline and step glue (SURVEY.md 8f-3, VERDICT r1 #8) -----------------------------
 * dv_u8_to_f32: dst[i] = src[i] / 255 (true division) -- torchvision ToTensor on the device, so host batches can be
 * uploaded as bytes (training.py:150; utils/datasets.py:182,247,364-367).  Both pointers 16-byte aligned.
 */
int dv_u8_to_f32(const unsigned char* src, float* dst, long long n, void* stream);
/* Device-resident dataset (disvae.data.DeviceLoader): replaces the per-item ToTensor of the reference's datasets
 * (utils/datasets.py:182,206-210) and the collate of its DataLoader for one batch.  src is the dataset as uint8
 * [N, row_bytes] on the device; dst row i = src row idx[i] / 255 (true division, bit-identical to dv_u8_to_f32 and to
 * ToTensor), dst is fp32 [nrows, row_bytes].  idx: int64 device array of nrows entries in [0, N) (not checked: the
 * kernel does not know N), repeats allowed.  One launch, 16-byte loads.
 * DV_ERR_BAD_SHAPE: nrows < 1 or row_bytes not a positive multiple of 16 (every Burgess geometry is: 1024, 3072,
 * 4096 or 12288 bytes).  DV_ERR_BAD_ARG: a NULL pointer, src or dst not 16-byte aligned, idx not 8-byte aligned. */
int dv_gather_u8_to_f32(const unsigned char* src, const long long* idx, int nrows, int row_bytes, float* dst,
                        void* stream);
/* loss[0] = sum_{i<na} coef_a[i]*a[i] + sum_{j<nb} coef_b[j]*b[j]; a, b device vectors, coef_* HOST arrays (<= 8 each,
 * passed to the kernel by value).  The scalar combinations of losses.py:151 (rec + anneal*beta*kl), :199-200 is not
 * covered (|kl - C|: dv_betab_loss_fwd below), :381-382 (rec + alpha*mi + beta*tc + anneal*gamma*dw_kl).  The training
 * path uses the scheduled form below.  Backward: g_a[0..na_total) (zeros past
 * na), g_b[0..nb) from the upstream scalar g[0]. */
int dv_loss_combine_fwd(const float* a, const float* coef_a, int na, const float* b, const float* coef_b, int nb,
                        float* loss, void* stream);
int dv_loss_combine_bwd(const float* g, const float* coef_a, int na, int na_total, const float* coef_b, int nb,
                        float* g_a, float* g_b, void* stream);

/* ---- annealed loss combinations and the device loss log (graph-capturable training steps) ----------
 * Each loss owns an int64 device step counter (`step`).  On a training step (is_train != 0) the forward kernels first
 * advance it by one, then anneal with the new value -- so a captured CUDA graph sees the step of every replay.
 * The annealing value is linear_annealing (losses.py:511-518) in double, in Python's operation order:
 *   A(step) = min(init + (fin - init) * step / steps_anneal, fin),  A = fin when steps_anneal == 0 or !is_train,
 * and a coefficient is (float)(A * base), which is what ctypes made of the host product: bit-identical to the
 * host-coefficient entry points above given the same step.
 *
 * Device loss log: on a training step whose counter value s satisfies s % every == 1 (the reference's record rule,
 * losses.py:105-114), a kernel writes the concatenation of its sources into row ((s - 1) / every) % cap of ring
 * [cap][ncols] (fp32, device).  The host reads rows back later; no host synchronisation inside the step.
 * src[k] is a device pointer to len[k] floats; in the forward entry points a NULL src[k] of length 1 stands for the
 * loss that launch computes.  sum(len) must equal ncols.  log == NULL (or !is_train): nothing is recorded. */
#define DV_LOSS_LOG_MAX_SRC 8
typedef struct dv_loss_log {
  float* ring;
  int cap, ncols, every, nsrc;
  const float* src[DV_LOSS_LOG_MAX_SRC];
  int len[DV_LOSS_LOG_MAX_SRC];
} dv_loss_log;
/* loss[0] = sum_{i<na} c[i]*a[i] + sum_{j<nb} c[na+j]*b[j] with c[k] = (float)(A * base[k]) if bit k of sched_mask is set,
 * else (float)base[k]; base is a HOST array of na + nb doubles (na, nb <= 8).  coefs[na + nb] (device) receives the c[k]
 * used; the backward reads them: g_a[0..na_total) (zeros past na), g_b[0..nb) from the upstream scalar g[0]. */
int dv_loss_combine_sched_fwd(const float* a, int na, const float* b, int nb, const double* base, unsigned sched_mask,
                              double init, double fin, long long steps_anneal, int is_train, long long* step, float* loss,
                              float* coefs, const dv_loss_log* log, void* stream);
int dv_loss_combine_sched_bwd(const float* g, const float* coefs, int na, int na_total, int nb, float* g_a, float* g_b,
                              void* stream);
/* beta-VAE_B (losses.py:199-200): loss = rec + gamma * |kl - C| with rec = rec_kl[0], kl = rec_kl[1] (the output of
 * dv_vae_loss_fwd) and C = (float)A(step) for (init, fin) = (c_init, c_fin); rounded like the torch expression (kl - C
 * and gamma * |.| in float, gamma = (float)gamma).  consts[2] (device) receives (C, gamma).  Backward: g_rec_kl[0] = g,
 * g_rec_kl[1] = (g * gamma) * sign(kl - C) with sign(0) = 0 -- torch's abs backward -- and zeros up to n. */
int dv_betab_loss_fwd(const float* rec_kl, double gamma, double c_init, double c_fin, long long steps_anneal, int is_train,
                      long long* step, float* loss, float* consts, const dv_loss_log* log, void* stream);
int dv_betab_loss_bwd(const float* g, const float* rec_kl, const float* consts, int n, float* g_rec_kl, void* stream);
/* The log alone (no NULL sources), predicated on the counter as it stands: for scalars computed after the loss
 * combination (FactorVAE's discriminator loss). */
int dv_loss_record(const long long* step, const dv_loss_log* log, void* stream);
/* g = dy * act'(y) over an NCHW tensor [B, C <= 4, hw] fused with chansum[c] = sum_{b,hw} g (the bias gradient of the
 * ConvTranspose2d that produced y; decoders.py:82).  g is bit-identical to dv_act_bwd's (same act codes and rounding).
 * workspace: dv_channel_sum_workspace_bytes().
 * DV_ERR_BAD_SHAPE: B < 1, C < 1, C > 4, hw < 4, hw % 4 != 0 or B * C > INT_MAX.
 * DV_ERR_BAD_ARG: a NULL pointer, act outside {NONE, RELU, SIGMOID, LEAKY}, dy, y or g not 16-byte aligned (they move
 * as float4), chansum or workspace not 4-byte aligned; nothing is launched then. */
int dv_act_bwd_chansum(const float* dy, const float* y, float* g, int B, int C, int hw, int act, float slope,
                       float* chansum, void* workspace, void* stream);

/* ---- disentanglement metrics: marginal-entropy estimator (SURVEY.md 8f-4) ---------------------
 * Replaces Evaluator._estimate_latent_entropies (disvae/evaluate.py:233-297), the inner loop of the MIG / AAM metrics
 * (:119-161, :299-317): for S samples zs[D][S] (row d = samples of latent dimension d) and the N posteriors
 * mean/logvar[n][d] (element (n,d) at n*row_stride + d*ld),
 *   H[d] = -(1/S) sum_s ( -log N + logsumexp_n log N(zs[d][s]; mean[n][d], exp(logvar[n][d])) ).
 * logq_out (optional, [D][S]) receives the per-sample log q(z).  Deterministic (fixed merge order).
 */
size_t dv_latent_entropy_workspace_bytes(int N, int D, int S);
int dv_latent_entropy(const float* zs, const float* mean, const float* logvar, int ld, int row_stride,
                      int N, int D, int S, float* H, float* logq_out, void* workspace, void* stream);

/* ---- disentanglement metrics: FactorVAE score (Kim & Mnih 2018, section 4) ----------------------
 * V groups of L gathered rows of mu [N, D] (element (n, d) at n*row_stride + d*ld, as dv_latent_entropy reads it; the
 * interleaved q_zCx [N, D, 2] buffer is read in place).  rows: int64 [V][L], every entry in [0, N) (not checked: the
 * caller builds them), repeats allowed.
 *   var_out[g][d] = unbiased variance (ddof 1) of mu[rows[g][l]][d] over l, in the centred two-pass form around
 *                   the group's first row (optional, [V][D])
 *   argmin_out[g] = the d minimising var[g][d] / global_var[d] over the dims that qualify: global_var[d] >= min_var
 *                   and the ratio (fp32, IEEE division) not NaN.  The lowest d wins a tie; -1 if no dim qualifies
 *                   (optional, [V]; needs global_var [D]).  A NaN variance (inf or NaN among the group's rows) thus
 *                   never takes or blocks a vote; an infinite ratio qualifies and orders above every finite one.
 * One launch, no workspace.  Deterministic (fixed-order reductions, no floating-point atomics), graph-capturable.
 * DV_ERR_BAD_SHAPE: L < 2, V < 1, N < 1, D < 1, D > 1024, ld < 1 or row_stride < 1.
 * DV_ERR_BAD_ARG: mu or rows NULL, both outputs NULL, argmin_out without global_var, or a pointer misaligned (rows
 * 8 bytes, the others 4). */
int dv_group_variance(const float* mu, int ld, int row_stride, int N, int D, const long long* rows, int V, int L,
                      const float* global_var, float min_var, float* var_out, int* argmin_out, void* stream);

/* ---- disentanglement metrics: SAP score (Kumar et al. 2018, section 3) --------------------------
 * For every latent d and factor k (k < K): the exact fit of LinearSVC(C, class_weight="balanced") -- squared hinge, L2,
 * the intercept a regularised feature of scale 1 -- on the 1-D training column x_i = mu[train_rows[i]][d] (element
 * (n, d) at n*row_stride + d*ld, so the interleaved q_zCx buffer is read in place), then its accuracy on the test rows.
 *   train_cls  int32 [K][num_train]: the class index (0 .. n_classes[k]-1, classes in ascending value) of each row
 *   test_cls   int32 [K][num_test]: the class index of each test row, or -1 for a value absent from the training rows
 *   n_classes  int32 [K] (1 .. class_stride), counts int32 [K][class_stride]: training rows of each class (> 0)
 * Class weights cw_c = num_train / (n_classes * counts_c).  More than two classes: one-vs-rest, class c's problem with
 * C_i = C*cw_c on its rows and plain C on the others (liblinear's convention); two classes: one problem, positive
 * class 1, C_i = C*cw_{y_i}; one class: no fit.  Each problem minimises
 *   1/2 (w^2 + b^2) + sum_i C_i max(0, 1 - s_i (w x_i + b))^2
 * in fp64 by semismooth Newton (at most 64 steps) to |gradient| <= 1e-10 of its scale.  A test row is predicted as
 * the argmax over classes of w_c x + b_c (lowest c on a tie), class 1 if w x + b > 0 for two classes, else class 0.
 *   score [D][K] fp32: the share of the test rows predicted as their class
 *   coef  fp64 [D][K][class_stride][2] (optional): (w, b) of problem p (the class for one-vs-rest, 0 for two
 *         classes); NaN beyond the factor's problems
 *   iters int32 [D][K][class_stride] (optional): Newton steps of problem p, -1 if it did not converge; 0 beyond
 * Rows are in [0, N) and labels within their ranges (not checked: the caller builds them).  One launch of D*K CTAs, no
 * workspace.  Deterministic (fixed-order reductions, no floating-point atomics), graph-capturable.
 * DV_ERR_BAD_SHAPE: N < 1, D < 1, D > 1024, num_train < 1, num_train > 32768, num_test < 1, K < 1, class_stride < 1,
 * class_stride > 256, ld < 1 or row_stride < 1.
 * DV_ERR_BAD_ARG: a required pointer NULL, C not finite and positive, or a pointer misaligned (rows and coef 8 bytes,
 * the others 4). */
int dv_sap_score_matrix(const float* mu, int ld, int row_stride, int N, int D, const long long* train_rows,
                        int num_train, const long long* test_rows, int num_test, const int* train_cls,
                        const int* test_cls, const int* n_classes, const int* counts, int K, int class_stride,
                        double C, float* score, double* coef, int* iters, void* stream);

/* ---- disentanglement metrics: beta-VAE score (Higgins et al. 2017, section 3) -------------------
 * dv_pair_abs_diff_mean: x[v][d] = (sum_{l < L} |mu[rows_a[v][l]][d] - mu[rows_b[v][l]][d]|) / L in fp64, the
 * differences of the fp32 values taken in fp64 and added in ascending l (an in-order fp64 sum gives the same bits).
 * mu is read as dv_group_variance reads it (element (n, d) at n*row_stride + d*ld; q_zCx in place).  rows_a, rows_b:
 * int64 [V][L], every entry in [0, N) (not checked).  x: fp64 [V][D].  One launch, no workspace, deterministic,
 * graph-capturable.
 * DV_ERR_BAD_SHAPE: N < 1, D < 1, V < 1, L < 1, V*D > INT_MAX, ld < 1 or row_stride < 1.
 * DV_ERR_BAD_ARG: a NULL pointer, or one misaligned (mu 4 bytes, the others 8). */
int dv_pair_abs_diff_mean(const float* mu, int ld, int row_stride, int N, int D, const long long* rows_a,
                          const long long* rows_b, int V, int L, double* x, void* stream);

/* dv_logistic_fit: the exact minimiser of sklearn's LogisticRegression(C=1) objective (L2 on the weights, unpenalised
 * intercept) on the first num_train rows of x (fp64 [num_train + num_eval][D]) and their class indices labels (int32
 * [num_train], 0 .. nc-1), with nc = *n_classes read from device memory (1 .. K; clamped to that range).
 *   nc > 2: multinomial, 1/2 |W|_F^2 + sum_i -log softmax(W x_i + b)_{y_i} over nc rows of (W, b), reported with
 *           sum_c b_c = 0;
 *   nc = 2: one binary model, 1/2 |w|^2 + sum_i log(1 + exp(-s_i (w.x_i + b))), s_i = +1 for class 1;
 *   nc = 1: no fit.
 * Solved in fp64 by truncated Newton (diagonally preconditioned conjugate gradient on Hessian-vector products over
 * features centred on their training mean, Armijo line search; a full step whose promised decrease is below 1e-12 |f|,
 * which f's rounding cannot rank, is taken whole), to max |gradient| <= 1e-10 of the largest scale of
 * the gradient's parts (|weight| + sum_i |q_i x_i|).
 *   coef  fp64 [K][D + 1]: row c = (W_c, b_c) for c < nc (nc > 2) or row 0 = (w, b) (nc = 2); NaN elsewhere
 *   pred  int32 [num_train + num_eval]: argmax_c W_c x + b_c, the lowest c on a tie; class 1 if w.x + b > 0 for nc = 2;
 *         0 for nc = 1
 *   iters int32 [1]: Newton steps taken, -1 if 100 did not converge (or the line search failed); 0 for nc = 1
 * workspace: dv_logistic_fit_workspace_bytes(num_train, D, K) bytes, 8-byte aligned, contents irrelevant.  One launch
 * of one CTA.  Deterministic (fixed-order reductions, no floating-point atomics), graph-capturable.
 * DV_ERR_BAD_SHAPE: num_train < 1, num_eval < 0, D < 1, D > 128, K < 1, K > 32, or (num_train + num_eval)*D > INT_MAX.
 * DV_ERR_BAD_ARG: a NULL pointer, or one misaligned (x, coef and workspace 8 bytes, the others 4).
 * DV_ERR_WORKSPACE: workspace NULL or smaller than the query. */
size_t dv_logistic_fit_workspace_bytes(int num_train, int D, int K);   /* 0 for an unsupported shape */
int dv_logistic_fit(const double* x, int D, int num_train, int num_eval, const int* labels, const int* n_classes,
                    int K, double* coef, int* pred, int* iters, void* workspace, size_t workspace_bytes,
                    void* stream);

/* ---- FactorVAE pieces ---------------------------------------------------------------------
 * dv_permute_dims replaces _permute_dims (losses.py:483-508): out[b][d] = z[perm[d][b]][d].
 * perms != NULL: int64 [D][B] (the reference's CPU randperm stream, trap T7).  perms == NULL:
 * per-dimension Philox-keyed random permutation generated on the device (B <= 4096; larger B through
 * dv_permute_dims_rows).
 */
int dv_permute_dims(const float* z, const long long* perms, unsigned long long seed,
                    unsigned long long* offset_dev, float* out, int B, int D, void* stream);
/* Row-window form of _permute_dims (losses.py:483-508) at any B, for the FactorVAE permutation of a half-batch
 * all-gathered from several GPUs (SURVEY.md 8e): z holds all B rows, only rows [row0, row0 + nrows) of the permuted
 * matrix are written, out[i][d] = z[pi_d(row0 + i)][d] for 0 <= i < nrows (out is [nrows][D]).
 * perms != NULL: pi_d = perms[d] (int64 [D][B]).  perms == NULL: pi_d is the order that sorts the keys
 * (philox4x32_10(*offset_dev + d*B + b, seed).x << 32) | b ascending -- the permutation dv_permute_dims draws --
 * and *offset_dev advances by B*D whatever the window, so the windows of one call on every rank agree.
 * Device permutations with B > 4096 sort through `workspace` (dv_permute_dims_workspace_bytes, 8-byte aligned,
 * contents irrelevant); below that it may be NULL.  Deterministic, host-synchronisation free, graph-capturable.
 * DV_ERR_BAD_SHAPE: B < 1, D < 1, row0 < 0, nrows < 1, row0 + nrows > B or B*D > INT_MAX. */
size_t dv_permute_dims_workspace_bytes(int B, int D);   /* 0 when B <= 4096 */
int dv_permute_dims_rows(const float* z, const long long* perms, unsigned long long seed,
                         unsigned long long* offset_dev, float* out, int B, int D, int row0, int nrows,
                         void* workspace, void* stream);
/* Epoch order of a device-resident dataset: replaces the RandomSampler of the reference's DataLoader
 * (utils/datasets.py:67-71, `shuffle=True`).  out_idx (int64 [N], 8-byte aligned) receives the Philox-keyed permutation
 * of [0, N) that dv_permute_dims_rows draws for one dimension (D = 1): the order that sorts the keys
 * (philox4x32_10(*offset_dev + i, seed).x << 32) | i ascending.  *offset_dev advances by N.  N up to INT_MAX.
 * workspace: dv_index_permutation_workspace_bytes(N) bytes, 8-byte aligned, contents irrelevant (NULL allowed when
 * that is 0, N <= 4096).  Deterministic, host-synchronisation free, graph-capturable.
 * DV_ERR_BAD_SHAPE: N < 1.  DV_ERR_BAD_ARG: a NULL or misaligned pointer. */
size_t dv_index_permutation_workspace_bytes(int N);
int dv_index_permutation(int N, unsigned long long seed, unsigned long long* offset_dev, long long* out_idx,
                         void* workspace, void* stream);
/* tc[0] = mean(d_z[:,0] - d_z[:,1])  (losses.py:265) */
int dv_factor_tc_fwd(const float* d_z, int h, float* tc, void* stream);
int dv_factor_tc_bwd(const float* upstream, int h, float* g_d_z, void* stream);
/* out[0] = 0.5*(CE(d_z, 0) + CE(d_perm, 1))  (losses.py:293-295) */
int dv_factor_ce_fwd(const float* d_z, const float* d_perm, int h, float* out, void* stream);
int dv_factor_ce_bwd(const float* d_z, const float* d_perm, const float* upstream, int h,
                     float* g_d_z, float* g_d_perm, void* stream);

/* ---- optimiser (SURVEY.md 8f-2) -------------------------------------------------------
 * torch.optim.Adam semantics (main.py:208, losses.py:238): eps outside the sqrt, no weight
 * decay, bias correction from *step_dev (float, incremented by the kernel).  Operates on one
 * flat fp32 buffer so a whole model is one launch.  betas are doubles: 1-beta and the bias corrections are
 * evaluated in fp64 like torch's Python-side arithmetic.  grad_scale multiplies the gradient
 * (1/world_size after a sum-allreduce). */
int dv_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                 float* step_dev, long long n, float lr, double beta1, double beta2, float eps,
                 float grad_scale, void* stream);

/* Multi-tensor form: `count` (<= dv_adam_multi_max_tensors()) parameter tensors updated by ONE launch.
 * The arrays are HOST arrays of device pointers / element counts; they are copied into kernel-parameter
 * space, nothing is retained.  Same arithmetic and step counter semantics as dv_adam_step. */
int dv_adam_multi_max_tensors(void);
int dv_adam_multi(int count, float* const* params, const float* const* grads, float* const* exp_avg,
                  float* const* exp_avg_sq, const long long* numel, float* step_dev, float lr, double beta1,
                  double beta2, float eps, float grad_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DISVAE_B200_H */

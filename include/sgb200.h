/*
 * sgb200.h -- C ABI of libsgb200.so: the H100 (sm_90a) hot path behind SuperGradients' YOLO-NAS / ResNet
 * training and inference modules.
 *
 * The reference (Deci-AI/super-gradients) has no FFI: every kernel on this path is reached through
 * torch.nn / torchvision calls inside Python nn.Modules.  Each entry point below therefore cites the reference
 * call site (file:line under src/super_gradients/) whose arithmetic it replaces; INTEGRATION.md shows the ctypes
 * binding a maintainer would add on the reference side.
 *
 * Conventions
 *   - plain pointers + sizes only; all pointers are DEVICE pointers unless a name ends in _host;
 *   - activations are NHWC bf16 (uint16_t storage) with an explicit channel pitch and channel offset, so a tensor
 *     may be a channel slice of a wider NHWC buffer (concat-free CSP layers);
 *   - functions never allocate, never synchronise; they enqueue on `stream` (a cudaStream_t passed as void*);
 *   - return 0 on success, a negative SGB_E_* code on error (no exceptions cross the boundary).
 */
#ifndef SGB200_H_
#define SGB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SGB_OK 0
#define SGB_E_INVALID (-1)     /* bad shape / argument */
#define SGB_E_UNSUPPORTED (-2) /* valid but not implemented for this configuration */
#define SGB_E_CUDA (-3)        /* a CUDA runtime / driver call failed (see sgb_last_error) */
#define SGB_E_ARCH (-4)        /* device is not sm_90 */

#define SGB_ACT_NONE 0
#define SGB_ACT_RELU 1
#define SGB_ACT_SILU 2

typedef uint16_t sgb_bf16; /* raw bfloat16 bits */

/* Convolution problem, cuDNN-style names.  Weights are KRSC (out-ch, kh, kw, in-ch) bf16 for fprop/wgrad and
 * CRSK for dgrad (sgb_weight_prepare makes both from the fp32 OIHW master copy). */
typedef struct SgbConvDesc {
  int32_t N, H, W, C; /* input batch, height, width, channels (C % 8 == 0) */
  int32_t K, R, S;    /* output channels, filter height / width */
  int32_t P, Q;       /* output height / width */
  int32_t stride, pad;
  int32_t x_pitch, x_off; /* channel pitch / offset of the buffer holding the input  (elements) */
  int32_t y_pitch, y_off; /* channel pitch / offset of the buffer holding the output (elements) */
  int32_t up2;            /* 1: ConvTranspose2d(k=2,s=2) mode -- see sgb_convt2x2_* */
  /* 0, or the first of the K channels (fprop: output channels; dgrad: dy channels; wgrad: dy rows) whose eight off-centre
   * filter taps are known to be zero (fprop, dgrad) or not wanted (wgrad: those dw entries are left as they are) -- the folded
   * QARepVGG filter [K3 ; centre(alpha*K1 + I)].  The kernels skip that work; the results are the same.  Needs R = S = 3,
   * stride 1, pad 1, 0 < centre_from < K and centre_from % 16 == 0, else SGB_E_INVALID. */
  int32_t centre_from;
} SgbConvDesc;

/* Fused epilogue of the forward implicit GEMM.  All pointers may be NULL. */
typedef struct SgbEpilogue {
  const float* scale;       /* [K]  y = acc*scale + shift   (inference: folded BN) */
  const float* shift;       /* [K]  also used as plain bias when scale == NULL */
  const sgb_bf16* residual; /* same geometry as y; added before the activation */
  double* stats;            /* [stats_repl][2][K] running sums of y and y*y over all pixels (train-mode BN) */
  int32_t stats_repl;       /* number of replicas of the stats buffer (power of two, >= 1) */
  int32_t act;              /* SGB_ACT_* */
  int32_t out_f32;          /* 1: y is float32 (parity tests of the accumulators); 0: bf16 */
} SgbEpilogue;

const char* sgb_last_error(void);
int sgb_version(void);
/* 0 if the current device is sm_90 and the library was built for it. */
int sgb_check_device(void);
/* Number of wgmma/TMA convolution launches issued by this process so far (evidence that the Hopper-native path,
 * not the generic mma.sync kernel, served a call). */
int64_t sgb_sm100_launches(void);
/* Number of those launches served by the halo-tile kernel of 3x3 / stride-1 convolutions (conv3x3_halo_kernel). */
int64_t sgb_conv_halo_launches(void);
/* Test-only: on != 0 sends every later 3x3 / stride-1 convolution to the im2col wgmma kernel instead of the halo-tile kernel,
 * so tests and timing tools can compare the two engines on one shape.  Not a user option. */
void sgb_conv_force_im2col(int on);
/* Number of wgmma/TMA launches served by the halo-tile weight-gradient kernel of 3x3 / stride-1 convolutions
 * (wgrad3x3_halo_kernel). */
int64_t sgb_conv_wgrad_halo_launches(void);
/* Test-only: on != 0 sends every later 3x3 / stride-1 weight gradient to the per-tap wgmma kernel (wgrad_wgmma_kernel) instead
 * of the halo-tile kernel, so tests and timing tools can compare the two engines on one shape.  Not a user option. */
void sgb_conv_wgrad_force_im2col(int on);

/* ---- convolution family (rows C1-C5, C8, C10 of SURVEY.md section 8a) --------------------------------------
 * replaces nn.Conv2d forward in modules/qarepvgg_block.py:184-204, modules/conv_bn_act_block.py:92-93,
 * training/models/classification_models/resnet.py:53-84, dfl_heads.py:65-66, and their autograd backward
 * (training/sg_trainer/sg_trainer.py:622). */
int sgb_conv_fprop(const SgbConvDesc* d, const sgb_bf16* x, const sgb_bf16* w_krsc, void* y, const SgbEpilogue* ep,
                   void* stream);
/* dx = conv_transpose(dy, w).  accumulate != 0: dx += result (dx is read-modify-written). */
int sgb_conv_dgrad(const SgbConvDesc* d, const sgb_bf16* dy, const sgb_bf16* w_crsk, sgb_bf16* dx, int accumulate,
                   void* stream);
/* dw_krsc (fp32, KRSC) += dy^T * im2col(x).  Split-K partial sums are reduced with fp32 atomics: the caller
 * zeroes dw_krsc.  */
int sgb_conv_wgrad(const SgbConvDesc* d, const sgb_bf16* x, const sgb_bf16* dy, float* dw_krsc, void* stream);
/* fp32 OIHW master weights -> bf16 KRSC (+ optional CRSK), zero-padding C up to c_pad. `scale` (may be NULL) is
 * a single device float multiplied into every weight; add_identity adds 1 to the centre tap of channel k==c. */
int sgb_weight_prepare(const float* w_oihw, int K, int C, int R, int S, int c_pad, sgb_bf16* w_krsc, sgb_bf16* w_crsk,
                       const float* scale, int add_identity, void* stream);
/* fp32 KRSC (c_pad channels) gradient -> fp32 OIHW gradient; accumulate != 0 adds into g_oihw. */
int sgb_wgrad_to_oihw(const float* dw_krsc, int K, int C, int R, int S, int c_pad, float* g_oihw, int accumulate,
                      void* stream);
/* Batched forms of the two calls above for a whole network: the item tables live in DEVICE memory, `start` is the
 * exclusive prefix sum of the per-item element counts (KRSC + CRSK elements / OIHW elements) and `total` their sum.
 * One launch replaces the per-layer weight casts of a step (reference: the fp32 -> bf16 autocast copies implied by
 * training/sg_trainer/sg_trainer.py:622-644) and the per-layer gradient layout changes. */
typedef struct SgbWeightItem {
  const float* w;     /* fp32 OIHW */
  const float* scale; /* device scalar or NULL */
  sgb_bf16* krsc;
  sgb_bf16* crsk;     /* or NULL */
  int32_t K, C, R, S, c_pad, add_identity;
  /* Destination inside a WIDER filter (the folded QARepVGG filter [K3 ; centre(alpha*K1 + I)] with 2K output channels):
   * kp > 0: the CRSK rows have kp entries and this filter's K outputs start at column koff (only k < K is written);
   * etaps > 0: the (1 x 1) source is the tap `etap` of an etaps-tap destination filter (KRSC row = etaps * c_pad entries,
   * CRSK row index = c * etaps + etap); krsc already points at this filter's first destination row.  The destination's
   * other entries are never written: allocate it zeroed. */
  int32_t kp, koff, etaps, etap;
  int64_t start;
} SgbWeightItem;
typedef struct SgbWgradItem {
  const float* dw; /* fp32 KRSC with c_pad channels */
  float* g;        /* fp32 OIHW */
  int32_t K, C, R, S, c_pad, accumulate;
  int64_t start;
} SgbWgradItem;
int sgb_weight_prepare_batch(const SgbWeightItem* items_dev, int n_items, int64_t total, void* stream);
typedef struct SgbAlphaItem {
  const float* dw1;   /* fp32 KRSC [K][1][1][c_pad]: gradient of the FOLDED 1x1 filter (alpha * K1 + I) */
  const float* w1;    /* fp32 OIHW [K][C][1][1]: branch_1x1.weight */
  const float* alpha; /* fp32 [1] */
  const float* dab;   /* fp32 [K]: gradient of (alpha * b1), or NULL */
  const float* bias1; /* fp32 [K]: branch_1x1.bias, or NULL */
  float* g_w1;        /* += alpha * dw1 */
  float* g_bias;      /* += alpha * dab (NULL: skipped) */
  float* g_alpha;     /* += <dw1, w1> + <dab, bias1> */
  int32_t K, C, c_pad, pad_;
} SgbAlphaItem;
/* QARepVGG `alpha` chain rule for every block of a step in ONE launch (one CTA per block, fixed-order reduction): replaces
 * mul / sum / add / addcmul_ launches per block (modules/qarepvgg_block.py:196-198: x_1x1 = alpha * branch_1x1(inputs)). */
int sgb_qarep_alpha_finish_batch(const SgbAlphaItem* items_dev, int n_items, void* stream);
int sgb_wgrad_to_oihw_batch(const SgbWgradItem* items_dev, int n_items, int64_t total, void* stream);
/* ConvTranspose2d(kernel=2, stride=2) (modules/sampling.py:72-73): desc describes the EQUIVALENT 2x2/s2 convolution
 * from the upsampled tensor (N,H,W,C) to the small tensor (N,P,Q,K); w is [K_small][2][2][C_up] bf16. */
int sgb_convt2x2_fprop(const SgbConvDesc* d, const sgb_bf16* x_small, const sgb_bf16* w_up, const float* bias,
                       sgb_bf16* y_up, void* stream);

/* ---- layout ---------------------------------------------------------------------------------------------- */
/* fp32 NCHW -> bf16 NHWC; channels [C, c_out) of the destination are written as zeros (c_out % 8 == 0). */
int sgb_nchw_f32_to_nhwc_bf16(const float* x, int N, int C, int H, int W, sgb_bf16* y, int y_pitch, int y_off, int c_out,
                              void* stream);
/* Patch gather for a first-layer R x R / stride / pad convolution over a FEW input channels (C * R * R <= c_out, e.g. the
 * YOLO-NAS stem: 3 channels, 3 x 3, stride 2): fp32 NCHW image -> bf16 NHWC [N, P, Q, c_out] with channel (r * R + s) * C + c
 * of output pixel (p, q) = x[n, c, p * stride - pad + r, q * stride - pad + s] (0 outside the image; channels >= C * R * R zero).
 * The stem convolution then is a 1 x 1 GEMM over this tensor: its input is fetched once instead of once per tap, and the
 * QARepVGG 1 x 1 branch (which samples exactly the centre tap) shares the GEMM (training/models/.../yolo_stages.py:61-63,
 * modules/qarepvgg_block.py:184-204). */
int sgb_stem_patches_f32(const float* x, int N, int C, int H, int W, int R, int stride, int pad, sgb_bf16* y, int P, int Q, int c_out,
                         void* stream);
int sgb_nhwc_bf16_to_nchw_f32(const sgb_bf16* x, int N, int C, int H, int W, int x_pitch, int x_off, float* y,
                              void* stream);

/* ---- BatchNorm (train) + residual + activation (row C9; nn.BatchNorm2d semantics, momentum / eps overridden by
 * customizable_detector.py:97-104) -------------------------------------------------------------------------- */
typedef struct SgbBnDesc {
  int64_t M;                     /* pixels = N*H*W */
  int32_t C;                     /* channels */
  int32_t x_pitch, x_off;        /* pre-BN tensor */
  int32_t y_pitch, y_off;        /* output tensor */
  int32_t r_pitch, r_off;        /* residual tensor (if any) */
  float eps, momentum;
  int32_t act;
  int32_t stats_repl;
  int32_t dy_pitch, dy_off;      /* backward passes: layout of dy when it is a channel slice of a wider buffer (a concat's
                                    gradient); dy_pitch == 0: dy is laid out like y */
  /* drop-path (stochastic depth, training/utils/regularization_utils.py:4-15): y = act(bn(x) * sample_scale[n] + residual) with
   * n = pixel / hw; sample_scale holds 0 or 1/keep_prob per image.  NULL: no drop-path. */
  int64_t hw;
  const float* sample_scale;
  /* backward passes of two layers that share one GEMM (functional._DualConvBnAct: the two 1x1 convolutions of a CSP layer run as one
   * GEMM with concatenated output channels): channels [dy2_split, C) of dy come from a second tensor.  dy2 == NULL: one source. */
  int32_t dy2_split, dy2_pitch, dy2_off, dy2_reserved;
  const void* dy2;
  /* cross-rank statistics (torch.nn.SyncBatchNorm under data parallelism), two-pass entry points only: `count` is a device pointer to
   * the element count of the layer over all ranks, read by the forward and backward apply passes in place of M (means, variance,
   * unbiased running variance).  `param_scale` multiplies the dgamma / dbeta the backward apply pass accumulates from all-reduced
   * sums: 1 / (ranks in the group), so that the data-parallel average of the per-rank gradients equals the average of torch's
   * per-rank SyncBatchNorm gradients.  count == NULL: local statistics, param_scale unused. */
  const double* count;
  float param_scale;
  int32_t count_reserved;
} SgbBnDesc;
/* Reduces stats -> mean / rstd (saved for backward), updates running stats, writes y = act(bn(x) + residual). */
int sgb_bn_act_fwd(const SgbBnDesc* d, const sgb_bf16* x, const double* stats, const float* gamma, const float* beta,
                   float* running_mean, float* running_var, const sgb_bf16* residual, sgb_bf16* y, float* save_mean,
                   float* save_rstd, void* stream);
/* Inference-mode BN (running stats) + residual + activation. */
int sgb_bn_act_infer(const SgbBnDesc* d, const sgb_bf16* x, const float* gamma, const float* beta,
                     const float* running_mean, const float* running_var, const sgb_bf16* residual, sgb_bf16* y,
                     void* stream);
/* Backward, pass 1: sums[0][c] = sum dz, sums[1][c] = sum dz * xhat with dz = dy * act'(pre-activation).
 * y (the forward output) is only needed when a residual was added; pass NULL otherwise and the activation mask is
 * recomputed from x, gamma, beta (one tensor read less). */
int sgb_bn_act_bwd_reduce(const SgbBnDesc* d, const sgb_bf16* dy, const sgb_bf16* x, const sgb_bf16* y, const float* gamma,
                          const float* beta, const float* save_mean, const float* save_rstd, double* sums, void* stream);
/* Backward, pass 2: dx (pre-BN grad), dresidual (= dz, optional), dgamma / dbeta (+=). */
int sgb_bn_act_bwd_apply(const SgbBnDesc* d, const sgb_bf16* dy, const sgb_bf16* x, const sgb_bf16* y,
                         const float* gamma, const float* beta, const float* save_mean, const float* save_rstd,
                         const double* sums, sgb_bf16* dx, sgb_bf16* dresidual, float* dgamma, float* dbeta, void* stream);
/* Per-channel sums of an NHWC bf16 tensor (used where the producer is not one of our GEMMs). */
int sgb_channel_stats(const sgb_bf16* x, int64_t M, int C, int pitch, int off, double* stats, void* stream);

/* ---- QARepVGG train-mode branch algebra (modules/qarepvgg_block.py:184-204) ---------------------------------
 * y3 = conv3x3(x) (raw), u = conv1x1_{alpha*K1 + I}(x) (raw, identity folded into the 1x1 weights).
 * z = s3*(y3 - mu3) + beta3 + u + alpha*b1 ;  out = act(post_bn(z)).
 * moments: [stats_repl][5][C] doubles = sum y3, y3^2, u, u^2, y3*u (produced by sgb_qarep_moments).         */
typedef struct SgbQarepDesc {
  int64_t M;
  int32_t C;
  int32_t pitch3, off3, pitchu, offu, pitcho, offo;
  float eps3, eps_post, momentum;
  int32_t act;
  int32_t use_post_bn;
  int32_t pitchd, offd; /* backward passes: layout of dout when it is a channel slice; pitchd == 0: laid out like out */
  /* forward passes: out = act(...) + (*res_alpha) * res -- the learnable shortcut of a YOLO-NAS bottleneck
   * (training/models/detection_models/yolo_nas/yolo_stages.py:61-63) fused into its second block.  res == NULL: none. */
  int32_t pitchr, offr;
  const void* res;
  const float* res_alpha;
  /* cross-rank statistics, exactly as SgbBnDesc.count / param_scale: the forward apply pass takes the all-reduced moments and the
   * global count, the backward apply pass the all-reduced sums; both BatchNorms of the block follow from them. */
  const double* count;
  float param_scale;
  int32_t count_reserved;
} SgbQarepDesc;
int sgb_qarep_moments(const SgbQarepDesc* d, const sgb_bf16* y3, const sgb_bf16* u, double* moments, void* stream);
/* coef out: [9][C] floats = mu3, rstd3, mu_u, rstd_z, a3 (coefficient of y3), au (of u), c0 (constant),
 * mean(zhat*y3hat), s3 = gamma3*rstd3 */
int sgb_qarep_fwd(const SgbQarepDesc* d, const sgb_bf16* y3, const sgb_bf16* u, const double* moments,
                  const float* gamma3, const float* beta3, const float* bias1_alpha, const float* gamma_p,
                  const float* beta_p, float* rm3, float* rv3, float* rm_p, float* rv_p, sgb_bf16* out, float* coef,
                  void* stream);
/* sgb_qarep_moments + sgb_qarep_fwd as ONE cooperative launch (moments, grid-wide barrier, apply); `moments` must be zero on entry. */
int sgb_qarep_fwd_fused(const SgbQarepDesc* d, const sgb_bf16* y3, const sgb_bf16* u, double* moments, const float* gamma3,
                        const float* beta3, const float* bias1_alpha, const float* gamma_p, const float* beta_p, float* rm3, float* rv3,
                        float* rm_p, float* rv_p, sgb_bf16* out, float* coef, void* stream);
/* pass 1: sums [3][C] = sum dzp, sum dzp*zhat, sum dzp*y3hat, dzp = dout*act'(pre).  `out` is unused (may be NULL):
 * the activation mask is recomputed from y3, u and the saved coefficients. */
int sgb_qarep_bwd_reduce(const SgbQarepDesc* d, const sgb_bf16* dout, const sgb_bf16* out, const sgb_bf16* y3,
                         const sgb_bf16* u, const float* coef, double* sums, void* stream);
/* pass 2: dy3, du (bf16), param grads (+=): dgamma3, dbeta3, dbias1a (grad of alpha*b1), dgamma_p, dbeta_p. */
int sgb_qarep_bwd_apply(const SgbQarepDesc* d, const sgb_bf16* dout, const sgb_bf16* out, const sgb_bf16* y3,
                        const sgb_bf16* u, const float* coef, const double* sums, const float* gamma3,
                        const float* gamma_p, sgb_bf16* dy3, sgb_bf16* du, float* dgamma3, float* dbeta3,
                        float* dbias1a, float* dgamma_p, float* dbeta_p, void* stream);
/* The two backward passes above as ONE cooperative launch (reduction, grid-wide barrier, apply): one launch less per layer and, for
 * operands that fit L2, one HBM read of them instead of two.  `sums` must be zero on entry, as for the two-pass form. */
int sgb_bn_act_bwd_fused(const SgbBnDesc* d, const sgb_bf16* dy, const sgb_bf16* x, const sgb_bf16* y, const float* gamma,
                         const float* beta, const float* save_mean, const float* save_rstd, double* sums, sgb_bf16* dx,
                         sgb_bf16* dresidual, float* dgamma, float* dbeta, void* stream);
/* Per-channel sums of x + sgb_bn_act_fwd as ONE cooperative launch, for convolutions whose epilogue produced no statistics (more than
 * 96 output channels); `stats` ([stats_repl][2][C]) must be zero on entry.  Same reference lines as sgb_bn_act_fwd. */
int sgb_bn_act_fwd_fused(const SgbBnDesc* d, const sgb_bf16* x, double* stats, const float* gamma, const float* beta,
                         float* running_mean, float* running_var, const sgb_bf16* residual, sgb_bf16* y, float* save_mean,
                         float* save_rstd, void* stream);
int sgb_qarep_bwd_fused(const SgbQarepDesc* d, const sgb_bf16* dout, const sgb_bf16* y3, const sgb_bf16* u, const float* coef,
                        double* sums, const float* gamma3, const float* gamma_p, sgb_bf16* dy3, sgb_bf16* du, float* dgamma3,
                        float* dbeta3, float* dbias1a, float* dgamma_p, float* dbeta_p, void* stream);

/* The passes above for the train-mode QARepVGG stem on patches (functional._QARepVGGStem), with y3 / u never stored: each pass
 * recomputes [y3 | u] = xp @ w^T from the 32-channel patch tensor xp ([M][32] bf16, dense) and the resident filter w ([2C][32] bf16)
 * exactly as sgb_conv_fprop would have stored them, then does what the pass of the same name above does with them.  C = 32, 48 or 64;
 * the layouts of out / dout / dy3 / du are those of the desc (y3 / u fields: dy3 / du).  Forward: sgb_stem_qarep_moments (moments zero
 * on entry), then sgb_stem_qarep_fwd; backward: sgb_stem_qarep_bwd_reduce (sums zero on entry), then sgb_stem_qarep_bwd_apply.
 * sgb_stem_gemm writes [y3 | u] itself ([M][2C]), for tests.  sgb_stem_recompute_launches counts the launches of all five. */
int sgb_stem_gemm(const SgbQarepDesc* d, const sgb_bf16* xp, const sgb_bf16* w, sgb_bf16* y, void* stream);
int sgb_stem_qarep_moments(const SgbQarepDesc* d, const sgb_bf16* xp, const sgb_bf16* w, double* moments, void* stream);
int sgb_stem_qarep_fwd(const SgbQarepDesc* d, const sgb_bf16* xp, const sgb_bf16* w, const double* moments, const float* gamma3,
                       const float* beta3, const float* bias1_alpha, const float* gamma_p, const float* beta_p, float* rm3, float* rv3,
                       float* rm_p, float* rv_p, sgb_bf16* out, float* coef, void* stream);
int sgb_stem_qarep_bwd_reduce(const SgbQarepDesc* d, const sgb_bf16* dout, const sgb_bf16* xp, const sgb_bf16* w, const float* coef,
                              double* sums, void* stream);
int sgb_stem_qarep_bwd_apply(const SgbQarepDesc* d, const sgb_bf16* dout, const sgb_bf16* xp, const sgb_bf16* w, const float* coef,
                             const double* sums, const float* gamma3, const float* gamma_p, sgb_bf16* dy3, sgb_bf16* du, float* dgamma3,
                             float* dbeta3, float* dbias1a, float* dgamma_p, float* dbeta_p, void* stream);
int64_t sgb_stem_recompute_launches(void);


/* ---- pooling / elementwise (rows C6, C7, C8) --------------------------------------------------------------- */
/* stride-`stride` max-pool k x k, pad k/2 (csp_darknet53.py:135-157 SPP; resnet.py maxpool 3/2/1). idx (int8,
 * optional) records the arg-max tap for the backward pass. */
int sgb_maxpool_fwd(const sgb_bf16* x, int N, int H, int W, int C, int x_pitch, int x_off, int k, int stride, int pad,
                    sgb_bf16* y, int P, int Q, int y_pitch, int y_off, uint8_t* idx, void* stream);
int sgb_maxpool_bwd(const sgb_bf16* dy, int N, int H, int W, int C, int k, int stride, int pad, int P, int Q,
                    int dy_pitch, int dy_off, const uint8_t* idx, float* dx_f32, void* stream);
/* The same gradient written as bf16 by a gather (every input pixel sums the dy of the <= ceil(k/stride)^2 windows whose arg-max is that
 * pixel): no zeroed fp32 tensor, no atomics, no conversion pass.  Meant for stride >= 2 (ResNet's 3 x 3 / 2 after the stem). */
int sgb_maxpool_bwd_bf16(const sgb_bf16* dy, int N, int H, int W, int C, int k, int stride, int pad, int P, int Q,
                         int dy_pitch, int dy_off, const uint8_t* idx, sgb_bf16* dx, int dx_pitch, void* stream);
/* y[slice] = a*x1 + b*x2 (x2 optional) over NHWC bf16 slices: concat copies, residual adds, grad accumulation */
int sgb_axpby(const sgb_bf16* x1, int p1, int o1, float a, const sgb_bf16* x2, int p2, int o2, float b, sgb_bf16* y,
              int py, int oy, int64_t M, int C, void* stream);
/* y = (*a_dev)*x1 + x2 with the scalar read on the device (learnable residual weight, yolo_stages.py:61-63) and
 * out[c] += sum_pixels a*b (fp64), used for d(alpha). */
int sgb_scale_add(const sgb_bf16* x1, int p1, int o1, const float* a_dev, const sgb_bf16* x2, int p2, int o2, sgb_bf16* y,
                  int py, int oy, int64_t M, int C, void* stream);
/* y = (*a_dev)*x1 + x2 (x2 optional) and out_dot[c] += sum_pixels x1*xd (fp64) in one pass over x1: backward of the learnable-alpha
 * shortcut (alpha * dy for the shortcut input, sum(dy * x) for alpha).  y may alias x2 (in-place accumulation). */
int sgb_scale_add_dot(const sgb_bf16* x1, int p1, int o1, const float* a_dev, const sgb_bf16* x2, int p2, int o2, const sgb_bf16* xd, int pd,
                      int od, sgb_bf16* y, int py, int oy, int64_t M, int C, double* out_dot, void* stream);
int sgb_channel_dot(const sgb_bf16* a, int pa, int oa, const sgb_bf16* b, int pb, int ob, int64_t M, int C, double* out,
                    void* stream);
int sgb_f32_to_bf16(const float* x, sgb_bf16* y, int64_t n, void* stream);
/* global average pool NHWC bf16 -> [N, C] bf16 and its backward */
int sgb_avgpool_fwd(const sgb_bf16* x, int N, int HW, int C, sgb_bf16* y, void* stream);
int sgb_avgpool_bwd(const sgb_bf16* dy, int N, int HW, int C, sgb_bf16* dx, void* stream);

/* ---- DFL head decode (row L0: dfl_heads.py:199-245, bbox_utils.py:9-29) --------------------------------------
 * per level: reg [N, HW, reg_pitch] bf16 (4*(reg_max+1) logits), cls [N, HW, cls_pitch] bf16 -> writes rows
 * [anchor_base, anchor_base + HW) of pred_bboxes [N, L, 4] f32 (xyxy, pixels), pred_scores [N, L, ncls] f32
 * (sigmoid), and optionally the raw fp32 copies cls_logits [N, L, ncls], reg_distri [N, L, 4*(reg_max+1)]. */
int sgb_dfl_decode(const sgb_bf16* reg, int reg_pitch, const sgb_bf16* cls, int cls_pitch, int N, int Hf, int Wf,
                   int L, int anchor_base, int ncls, int reg_max, float stride, float cell_offset, float* pred_bboxes,
                   float* pred_scores, float* cls_logits, float* reg_distri, void* stream);

/* Keypoint decode of one level (row L8: pose_estimation_models/yolo_nas_pose/yolo_nas_pose_ndfl_heads.py:186-199):
 * pose [N, HW, pose_pitch] bf16 (channel 2j = x offset, 2j+1 = y offset of joint j), logit [N, HW, logit_pitch] bf16 (joint j
 * at channel logit_off + j) -> rows [anchor_base, anchor_base + HW) of pose_coords [N, L, J, 2] f32
 * = (offset * offset_multiplier + grid centre - (compensate ? cell_offset : 0)) * stride, pose_scores [N, L, J] f32
 * (sigmoid) and optionally the raw pose_logits [N, L, J].  Boxes and the person score of the same head go through
 * sgb_dfl_decode with ncls = 1 (channel 0 of the class head). */
int sgb_pose_keypoint_decode(const sgb_bf16* pose, int pose_pitch, const sgb_bf16* logit, int logit_pitch, int logit_off, int N,
                             int Hf, int Wf, int L, int anchor_base, int J, float stride, float cell_offset,
                             float offset_multiplier, int compensate_grid_cell_offset, float* pose_coords, float* pose_scores,
                             float* pose_logits, void* stream);

/* ---- PPYoloE / YOLO-NAS loss (rows L1-L6: training/losses/ppyolo_loss.py) ----------------------------------- */
typedef struct SgbLossDesc {
  int32_t B, L, ncls, reg_max; /* batch, anchors, classes, DFL bins - 1 */
  int32_t n_max;               /* padded number of GT boxes per image */
  int32_t topk;                /* TAL top-k (13) */
  float alpha, beta;           /* TAL exponents (1, 6) */
  float w_cls, w_iou, w_dfl;   /* 1.0, 2.5, 0.5 */
  int32_t iou_type;            /* 0 = GIoU (PPYoloELoss), 1 = CIoU (YoloNASPoseLoss) */
} SgbLossDesc;
/* Task-aligned assigner (ppyolo_loss.py:454-561). gt_boxes [B, n_max, 4] xyxy pixels, gt_labels [B, n_max] int32,
 * gt_valid [B, n_max] uint8.  Outputs: assigned_label [B, L] int32 (ncls = background), assigned_box [B, L, 4],
 * assigned_score [B, L] f32 (the single non-zero entry of the reference's one-hot * metric row). */
int sgb_tal_assign(const SgbLossDesc* d, const float* cls_logits, const float* reg_distri, const float* anchor_points,
                   const float* stride_tensor, const float* gt_boxes, const int32_t* gt_labels, const uint8_t* gt_valid,
                   int32_t* assigned_label, float* assigned_box, float* assigned_score, double* sums, void* workspace,
                   int64_t workspace_bytes, void* stream);
int64_t sgb_tal_workspace_bytes(const SgbLossDesc* d);
/* ATSS assigner (ppyolo_loss.py:301-434 the way PPYoloELoss calls it, :810-820: topk = d->topk (9) per pyramid level,
 * force_gt_matching = False, scores = IoU(gt, predicted box)).  anchors [L, 4] xyxy pixels (the head's anchor boxes);
 * level_sizes: HOST array [n_levels <= 8] (num_anchors_list; sums to L, each >= topk <= 16).  d->alpha / beta are unused.
 * Outputs exactly as sgb_tal_assign, including sum(assigned_score) added into sums[3].  Equal centre distances are ordered
 * by anchor index. */
int sgb_atss_assign(const SgbLossDesc* d, const float* reg_distri, const float* anchors, const float* anchor_points,
                    const float* stride_tensor, const int32_t* level_sizes, int32_t n_levels, const float* gt_boxes,
                    const int32_t* gt_labels, const uint8_t* gt_valid, int32_t* assigned_label, float* assigned_box,
                    float* assigned_score, double* sums, void* workspace, int64_t workspace_bytes, void* stream);
int64_t sgb_atss_workspace_bytes(const SgbLossDesc* d);
/* Varifocal + GIoU/CIoU + DFL loss, forward and backward in one launch (ppyolo_loss.py:944-1084).
 * sums [4] doubles: sgb_tal_assign has already added sum(assigned_score) into sums[3] (the normaliser, clipped at 1);
 * this call adds {cls_sum, iou_sum, dfl_sum} into sums[0..2] and writes the FINAL gradients of
 * grad_scale * (w_cls*cls + w_iou*iou + w_dfl*dfl) / normaliser  w.r.t. the logits (grad_cls / grad_reg may be NULL). */
int sgb_dfl_iou_loss_fwd_bwd(const SgbLossDesc* d, const float* cls_logits, const float* reg_distri,
                             const float* anchor_points, const float* stride_tensor, const int32_t* assigned_label,
                             const float* assigned_box, const float* assigned_score, double* sums, float grad_scale,
                             float* grad_cls, float* grad_reg, void* stream);
/* Focal classification term (PPYoloELoss use_varifocal_loss=False: ppyolo_loss.py:1069-1077; alpha = 0.25 behind the ATSS
 * assigner, <= 0 (no alpha_t) behind the task-aligned one, :820 / :832).  Call AFTER sgb_dfl_iou_loss_fwd_bwd and before
 * sgb_loss_finalize: replaces sums[0] by the focal sum and grad_cls by the focal term's final gradient. */
int sgb_focal_cls_fwd_bwd(const SgbLossDesc* d, const float* cls_logits, const int32_t* assigned_label,
                          const float* assigned_score, double* sums, float grad_scale, float alpha, float* grad_cls,
                          void* stream);
/* loss_out [4] = {cls, iou, dfl, total} (weighted, normalised) -- the reference's log_losses. */
int sgb_loss_finalize(const SgbLossDesc* d, const double* sums, float* loss_out, void* stream);
/* d(raw fp32 logits [N, L, gC]) -> bf16 NHWC head-output gradient of one level (rows anchor_base..+HW). */
int sgb_head_grad_scatter(const float* grad, int gC, int N, int HW, int L, int anchor_base, sgb_bf16* dy, int pitch,
                          void* stream);

/* ---- YoloNASPoseLoss (row L7: training/losses/yolo_nas_pose_loss.py:45-682) --------------------------------- */
typedef struct SgbPoseLossDesc {
  int32_t B, L, J, reg_max;                         /* batch, anchors, joints, DFL bins - 1 */
  int32_t n_max;                                    /* padded number of GT instances per image */
  int32_t topk;                                     /* assigner top-k (13) */
  float alpha, beta;                                /* assigner exponents (1, 6) */
  float w_cls, w_iou, w_dfl, w_pose_cls, w_pose_reg; /* 1.0, 2.5, 0.5, 1.0, 1.0 */
  int32_t iou_type;                                 /* 0 = GIoU, 1 = CIoU (default) */
  int32_t cls_type;                                 /* person classification: 0 = focal (default), 1 = BCE */
  int32_t pose_cls_type;                            /* joint visibility: 0 = BCE (default), 1 = focal */
  int32_t multiply_by_oks;                          /* assigner_multiply_by_pose_oks */
  int32_t rescale_with_score;                       /* rescale_pose_loss_with_assigned_score */
} SgbPoseLossDesc;
int64_t sgb_pose_tal_workspace_bytes(const SgbPoseLossDesc* d);
/* YoloNASPoseTaskAlignedAssigner (:77-244).  cls_logits [B, L] (one class), reg_distri [B, L, 4*(reg_max+1)], pose_coords
 * [B, L, J, 2] decoded pixels, anchor_points [L, 2], stride_tensor [L]; gt_boxes [B, n_max, 4] xyxy pixels, gt_poses
 * [B, n_max, J, 3] (x, y, visibility), gt_crowd / gt_valid [B, n_max] uint8, sigmas [J].  Outputs: assigned_gt [B, L]
 * int32 = index of the assigned NON-CROWD instance or -1, assigned_score [B, L] f32 (0 for background and crowd).
 * Adds sum(assigned_score) into sums[3] and the number of positive anchors into sums[6] (sums: 8 doubles, zeroed by the
 * caller). */
int sgb_pose_tal_assign(const SgbPoseLossDesc* d, const float* cls_logits, const float* reg_distri, const float* pose_coords,
                        const float* anchor_points, const float* stride_tensor, const float* gt_boxes, const float* gt_poses,
                        const uint8_t* gt_crowd, const uint8_t* gt_valid, const float* sigmas, int32_t* assigned_gt,
                        float* assigned_score, double* sums, void* workspace, int64_t workspace_bytes, void* stream);
/* YoloNASPoseLoss.forward (:404-494) after the assignment, forward and backward in one launch: adds {cls, iou, dfl} into
 * sums[0..2] and {pose_cls, pose_reg} into sums[4..5], and writes the FINAL gradients of grad_scale * total loss w.r.t.
 * cls_logits [B, L], reg_distri, pose_coords [B, L, J, 2] and pose_logits [B, L, J] (any grad pointer may be NULL). */
int sgb_pose_loss_fwd_bwd(const SgbPoseLossDesc* d, const float* cls_logits, const float* reg_distri, const float* pose_coords,
                          const float* pose_logits, const float* anchor_points, const float* stride_tensor,
                          const float* gt_boxes, const float* gt_poses, const float* sigmas, const int32_t* assigned_gt,
                          const float* assigned_score, double* sums, float grad_scale, float* grad_cls, float* grad_reg,
                          float* grad_pose, float* grad_pose_logits, void* stream);
/* loss_out [6] = {cls, iou, dfl, pose_cls, pose_reg, total} (weighted, normalised) -- the reference's log_losses. */
int sgb_pose_loss_finalize(const SgbPoseLossDesc* d, const double* sums, float* loss_out, void* stream);

/* ---- batched NMS (rows N1-N5: pp_yolo_e/post_prediction_callback.py:42-98 + torchvision.ops.batched_nms) ---- */
typedef struct SgbNmsDesc {
  int32_t B, L, ncls;
  float score_thr;
  double iou_thr; /* compared in double, as torchvision's CPU kernel does */
  int32_t top_k, max_out;
  int32_t multi_label;    /* 1: every (anchor, class) above threshold is a candidate; 0: arg-max class only */
  int32_t class_agnostic; /* 1: torchvision.ops.nms ; 0: batched_nms (coordinate-offset trick) */
  int32_t thr_inclusive;  /* 1: score >= thr (pose callback / single-label), 0: score > thr (multi-label) */
} SgbNmsDesc;
int64_t sgb_nms_workspace_bytes(const SgbNmsDesc* d);
/* boxes [B, L, 4] f32 xyxy, scores [B, L, ncls] f32. out [B, max_out, 6] f32 rows (x1,y1,x2,y2,conf,label) in the
 * reference's order, out_idx [B, max_out] int32 = flat candidate index anchor*ncls + class, out_count [B] int32. */
int sgb_batched_nms(const SgbNmsDesc* d, const float* boxes, const float* scores, float* out, int32_t* out_idx,
                    int32_t* out_count, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- sliding-window detection (sliding_window_detection_forward_wrapper.py:107-166: tiles, per-image merge NMS) ---- */
/* canvas: bf16 NHWC [B, H, W, pitch] (pitch a multiple of 8), tiles: int32 [T, 3] rows (image, y0, x0) in host (validated here)
 * and device memory.  out: bf16 NHWC [T, tile, tile, pitch] = canvas[image, y0:y0+tile, x0:x0+tile], zero outside the canvas.
 * One launch. */
int sgb_sliding_window_gather(const sgb_bf16* canvas, int32_t B, int32_t H, int32_t W, int32_t pitch, const int32_t* tiles_host,
                              const int32_t* tiles, int32_t T, int32_t tile, sgb_bf16* out, void* stream);
/* image_tiles_host [B + 1]: image b owns tiles [image_tiles[b], image_tiles[b + 1]), ascending from 0 to T.  cap = P * the largest
 * tile count of an image.  0 when the arguments are malformed. */
int64_t sgb_sliding_window_merge_workspace_bytes(int32_t B, const int32_t* image_tiles_host, int32_t T, int32_t P, int32_t ncls);
/* rows [T, P, 6] f32 / counts [T] int32: the per-tile NMS result in tile pixels (sgb_batched_nms with max_out P), tiles [T, 3] as
 * above (device), image_tiles [B + 1] (host and device).  Per image: rows + (x0, y0, x0, y0) in fp32, concatenated in (tile, row)
 * order, then torchvision's CPU batched_nms(boxes, score, label, iou_thr): the coordinate trick iff 4 n <= 4000, else per-class
 * NMS.  out [B, cap, 6] f32 rows in (score desc, position asc) order, out_count [B]; a count outside [0, P] or a label outside
 * [0, ncls) (or not integral) makes out_count[b] -1 / -2.  No host synchronisation; workspace linear in B * cap. */
int sgb_sliding_window_merge(const float* rows, const int32_t* counts, const int32_t* tiles, const int32_t* image_tiles_host,
                             const int32_t* image_tiles, int32_t B, int32_t T, int32_t P, int32_t ncls, double iou_thr, float* out,
                             int32_t* out_count, void* workspace, int64_t workspace_bytes, void* stream);
/* kernels launched by one sgb_sliding_window_merge call with these dimensions */
int32_t sgb_sliding_window_merge_launches(int32_t B, const int32_t* image_tiles_host, int32_t T, int32_t P);

/* ---- DetectionMetrics matching (SURVEY section 8(f) N4: training/utils/detection_utils.py:1120-1290, IoUMatching :880-1005) ---- */
#define SGB_MATCH_MAX_THRESHOLDS 32
typedef struct SgbMatchDesc {
  int32_t B;                     /* images of the batch */
  int32_t max_preds;             /* row pitch of the prediction tensor (the NMS kernel's max_out) */
  int32_t max_targets;           /* row pitch of the padded target tensor (>= 1) */
  int32_t max_crowd;             /* row pitch of the padded crowd-target tensor (0: none) */
  int32_t n_thresholds;          /* IoU thresholds, ascending, <= SGB_MATCH_MAX_THRESHOLDS */
  int32_t top_k;                 /* predictions kept per class and image (DetectionMetrics top_k_predictions) */
  int32_t denormalize_targets;   /* targets are normalised (cx, cy, w, h): scale by width / height */
  float height, width;           /* image size the predictions are clipped to */
} SgbMatchDesc;
/* preds [B, max_preds, 6] f32 rows (x1, y1, x2, y2, score, class) as sgb_batched_nms writes them, pred_count [B];
 * targets [B, max_targets, 5] f32 rows (class, cx, cy, w, h), target_count [B]; crowd likewise (NULL when max_crowd == 0);
 * thresholds [n_thresholds] f32.  matched / ignore [B, max_preds, n_thresholds] uint8 (rows >= pred_count[b] are zeroed) =
 * compute_img_detection_matching's preds_matched / preds_to_ignore for every image, bit-exact.  One CTA per image, one warp
 * per threshold. */
int sgb_detection_matching(const SgbMatchDesc* d, const float* preds, const int32_t* pred_count, const float* targets,
                           const int32_t* target_count, const float* crowd, const int32_t* crowd_count, const float* thresholds,
                           uint8_t* matched, uint8_t* ignore, void* stream);

/* ---- DetectionMetricsDistanceBased matching (training/utils/detection_utils.py:1196-1290 with DistanceMatching :1008-1118,
 * EuclideanDistance / ManhattanDistance :1293-1340, get_top_k_idx_per_cls :1342-1359; metric: training/metrics/detection_metrics.py:295-374) ----
 * The buffers, layouts and outputs of sgb_detection_matching, with the distance between box centres as the pair score: a
 * prediction matches the nearest free same-class target (lowest index on equal distances) when distance < threshold (strict), and
 * is ignored at threshold j when its nearest same-class crowd target is nearer than thresholds[j].  Euclidean: sqrt(dx*dx + dy*dy)
 * with single-rounded products, add and sqrt; Manhattan: |dx| + |dy|.  thresholds [n_thresholds] f32 pixel distances, in any
 * order, live in HOST memory (they are checked here and travel in the launch parameters).  An unknown metric, a non-finite or
 * negative threshold, more than SGB_MATCH_MAX_THRESHOLDS thresholds or an image over the 200 KB shared-memory bound is refused
 * with SGB_E_INVALID. */
#define SGB_DISTANCE_EUCLIDEAN 0
#define SGB_DISTANCE_MANHATTAN 1
int sgb_detection_distance_matching(const SgbMatchDesc* d, int32_t metric, const float* preds, const int32_t* pred_count,
                                    const float* targets, const int32_t* target_count, const float* crowd,
                                    const int32_t* crowd_count, const float* thresholds, uint8_t* matched, uint8_t* ignore,
                                    void* stream);

/* ---- PoseEstimationMetrics matching (training/metrics/pose_estimation_metrics.py:237-314, pose_estimation_utils.py:35-263) ---- */
/* poses [B, max_preds, n_joints, 3] f32 (x, y, joint score; only x, y are read), scores [B, max_preds] f32, pred_count [B] (rows
 * in any order; the top_k by score are used); gt_joints [B, max_targets, n_joints, 3] f32 (x, y, visibility), gt_boxes
 * [B, max_targets, 4] f32 XYWH, gt_areas [B, max_targets] f32, gt_flags [B, max_targets] u8 (1: is_crowd, 2: box given, 4: area
 * given; missing ones are derived from the visible joints), gt_count [B]; sigmas [n_joints] f32; thresholds [n_thresholds] f32.
 * With K = min(top_k, max_preds): matched / ignore [B, K, n_thresholds] u8 and used_scores [B, K] f32 in score order (rows past
 * used_count[b] are zero), used_count [B], n_targets [B] (targets neither crowd nor fully invisible) =
 * compute_img_keypoint_matching's preds_matched / preds_to_ignore / preds_scores / num_targets.  oks_out (NULL: not written)
 * [B, K, max_targets] f32 receives the OKS of every used prediction against every target.  One CTA per image, one warp per
 * threshold; an image's working set must fit in 200 KB of shared memory (pose_match.cu states the formula). */
int sgb_pose_keypoint_matching(const float* poses, const float* scores, const int32_t* pred_count, const float* gt_joints,
                               const float* gt_boxes, const float* gt_areas, const uint8_t* gt_flags, const int32_t* gt_count,
                               const float* sigmas, const float* thresholds, int32_t B, int32_t max_preds, int32_t max_targets,
                               int32_t n_joints, int32_t n_thresholds, int32_t top_k, uint8_t* matched, uint8_t* ignore,
                               float* used_scores, int32_t* used_count, int32_t* n_targets, float* oks_out, void* stream);

/* ---- fused predict() pre-processing (SURVEY section 8(f) N3: training/processing/processing.py:205-590, pipelines.py:192-216) ---- */
typedef struct SgbPreprocDesc {
  int32_t src_h, src_w, src_c; /* uint8 H x W x C source image (C <= 4) */
  int32_t src_pitch;           /* bytes per source row */
  int32_t dst_h, dst_w;        /* size after the rescale step (== src_h, src_w: no resize) */
  int32_t out_h, out_w;        /* padded canvas = the model's input size */
  int32_t pad_top, pad_left;   /* where the resized image sits on the canvas */
  int32_t out_pitch;           /* channel pitch (elements) of the bf16 NHWC output slot; channels >= src_c are written as 0 */
  int32_t reverse_channels;    /* ReverseImageChannels: output channel c reads source channel src_c - 1 - c */
  int32_t normalize;           /* NormalizeImage: (v - mean[c]) / std[c] after the standardisation */
  float pad_value;             /* Detection*Padding pad_value, in uint8 units (114) */
  double max_value;            /* StandardizeImage: v / max_value; <= 0 skips it */
  float mean[4], std[4];
} SgbPreprocDesc;
/* src: device uint8 image; out: device bf16 [out_h, out_w, out_pitch] (one image slot of an NHWC batch).  Bit-exact with
 * cv2.resize(INTER_LINEAR) + numpy padding / scaling of the reference pipeline followed by a round-to-nearest bf16 store. */
int sgb_preprocess_u8(const SgbPreprocDesc* d, const uint8_t* src, sgb_bf16* out, void* stream);

/* ---- ImageNet predict() pre-processing of a whole batch (processing.py:614-680 Resize + CenterCrop, transforms/utils.py:28-42
 *      PIL.Image.resize(BILINEAR), processing.py:1142-1151 default_imagenet_processing_params) ---- */
/* Per-image table: int64 [batch][SGB_RS_FIELDS] rows of (byte offset of the image's first row in src, source h, w, bytes per source
 * row, size after Resize (resized_h, resized_w; == h, w: no resize), CenterCrop window origin (crop_top, crop_left)). */
#define SGB_RS_OFFSET 0
#define SGB_RS_H 1
#define SGB_RS_W 2
#define SGB_RS_PITCH 3
#define SGB_RS_RESIZED_H 4
#define SGB_RS_RESIZED_W 5
#define SGB_RS_CROP_TOP 6
#define SGB_RS_CROP_LEFT 7
#define SGB_RS_FIELDS 8
/* table_host: the table in host memory (validated here, sizes the launch); table: the same table in device memory.  src: device
 * uint8 buffer of src_bytes holding every H x W x channels image (channels == 3); out: device bf16 [batch, out_h, out_w, out_pitch]
 * (out_pitch >= channels, a multiple of 8; channels >= `channels` are written as 0).  reverse_channels: output channel c reads
 * source channel channels - 1 - c (ReverseImageChannels); max_value > 0: v / max_value (StandardizeImage); mean_host / std_host
 * (NULL: none): (v - mean[c]) / std[c] (NormalizeImage).  ONE launch for the batch: Pillow's antialiased bilinear resize evaluated
 * only inside each crop window [crop_top, crop_top + out_h) x [crop_left, crop_left + out_w), then the standardisation and a
 * round-to-nearest bf16 store, bit-exact with the reference pipeline.  A CTA stages the horizontally resized source rows of one
 * output-row tile in shared memory; a batch whose rows cannot fit in 200 KB (a downscale factor of ~150 at a 224 crop) is
 * refused with SGB_E_INVALID.  batch == 0 is a no-op. */
int sgb_resample_crop_u8(const int64_t* table_host, const int64_t* table, const uint8_t* src, int64_t src_bytes, int32_t batch,
                         int32_t channels, int32_t out_h, int32_t out_w, int32_t out_pitch, int32_t reverse_channels,
                         double max_value, const float* mean_host, const float* std_host, sgb_bf16* out, void* stream);

/* ---- detection train augmentation (training/transforms/transforms.py:603-690 DetectionRandomAffine, :693-809 DetectionMixup,
 *      :945-977 DetectionPaddedRescale, :980-1009 DetectionHorizontalFlip, :1150-1229 DetectionRGB2BGR / DetectionHSV,
 *      :490-511 DetectionStandardize; random_affine :1464-1534, augment_hsv :1623-1634, utils.py:203-226) ---- */
/* Per-image table: int64 [batch][SGB_AUG_FIELDS]; the six affine coefficients are float64 values stored bit for bit in their slots.
 *   source image: byte offset in src, h, w (dense rows of w * 3 bytes)
 *   affine: flag, output size (the image size after the affine; == h, w when the flag is 0), forward 2 x 3 matrix M (row major),
 *           border value
 *   channel swap flag (DetectionRGB2BGR), HSV flag and int gains dh / ds / dv, bgr_channels packed as c0 | c1 << 2 | c2 << 4,
 *   horizontal flip flag
 *   mixup: flag, partner byte offset / h / w, partner flip flag, first resize size, canvas size (target_dim), border value,
 *          second resize size (jit_factor), crop offsets x / y
 *   padded rescale: resized size (int(h * r), int(w * r)) of the affine-size image inside the out_h x out_w canvas
 *   mosaic (transforms.py:513-599 DetectionMosaic, get_mosaic_coordinate detection_utils.py:738-768): flag, canvas size
 *          (2 * input_dim; the image size the affine, or the chain when the affine is off, receives), centre xc / yc, border
 *          value, then SGB_AUG_MOS_TILES tiles of SGB_AUG_MOS_TILE_FIELDS from SGB_AUG_MOS_TILE (top-left, top-right,
 *          bottom-left, bottom-right, tile 0 being the sample's own image): byte offset in src, source h / w, resized size
 *          (int(h0 * scale), int(w0 * scale)), placement rectangle [x1, x2) x [y1, y2) on the canvas and the resized tile's
 *          pixel (sx, sy) that lands on (x1, y1).  Each rectangle lies in its quadrant of (xc, yc).  With the flag set, the
 *          source image fields (offset, h, w) repeat tile 0 and the affine reads the canvas instead of the source image. */
#define SGB_AUG_OFFSET 0
#define SGB_AUG_H 1
#define SGB_AUG_W 2
#define SGB_AUG_AFFINE 3
#define SGB_AUG_AFF_H 4
#define SGB_AUG_AFF_W 5
#define SGB_AUG_M 6 /* 6 slots */
#define SGB_AUG_AFF_BORDER 12
#define SGB_AUG_SWAP 13
#define SGB_AUG_HSV 14
#define SGB_AUG_DH 15
#define SGB_AUG_DS 16
#define SGB_AUG_DV 17
#define SGB_AUG_BGR 18
#define SGB_AUG_FLIP 19
#define SGB_AUG_MIX 20
#define SGB_AUG_MIX_OFFSET 21
#define SGB_AUG_MIX_H 22
#define SGB_AUG_MIX_W 23
#define SGB_AUG_MIX_FLIP 24
#define SGB_AUG_MIX_R1_H 25
#define SGB_AUG_MIX_R1_W 26
#define SGB_AUG_MIX_CANVAS_H 27
#define SGB_AUG_MIX_CANVAS_W 28
#define SGB_AUG_MIX_BORDER 29
#define SGB_AUG_MIX_R2_H 30
#define SGB_AUG_MIX_R2_W 31
#define SGB_AUG_MIX_X 32
#define SGB_AUG_MIX_Y 33
#define SGB_AUG_RS_H 34
#define SGB_AUG_RS_W 35
#define SGB_AUG_MOS 36
#define SGB_AUG_MOS_CANVAS_H 37
#define SGB_AUG_MOS_CANVAS_W 38
#define SGB_AUG_MOS_XC 39
#define SGB_AUG_MOS_YC 40
#define SGB_AUG_MOS_BORDER 41
#define SGB_AUG_MOS_TILE 42
#define SGB_AUG_MOS_TILES 4
/* fields of one mosaic tile, relative to SGB_AUG_MOS_TILE + i * SGB_AUG_MOS_TILE_FIELDS */
#define SGB_AUG_T_OFFSET 0
#define SGB_AUG_T_H 1
#define SGB_AUG_T_W 2
#define SGB_AUG_T_RH 3
#define SGB_AUG_T_RW 4
#define SGB_AUG_T_X1 5
#define SGB_AUG_T_Y1 6
#define SGB_AUG_T_X2 7
#define SGB_AUG_T_Y2 8
#define SGB_AUG_T_SX 9
#define SGB_AUG_T_SY 10
#define SGB_AUG_MOS_TILE_FIELDS 11
#define SGB_AUG_FIELDS 86
/* table_host: the table in host memory (validated here); table: the same table in device memory.  src: device uint8 buffer of
 * src_bytes holding every source, mosaic-tile and mixup-partner image (channels == 3).  out: device bf16 [batch, out_h, out_w,
 * out_pitch] (out_pitch >= 3, a multiple of 8; channels >= 3 written as 0).  ONE launch for the batch.  Per output pixel: [mosaic:
 * each source pixel read below is a canvas pixel, i.e. the cv2.resize (INTER_LINEAR) of the one tile whose rectangle holds it,
 * else the mosaic border value; the affine's border value applies only outside the canvas] -> cv2.warpAffine
 * (INTER_LINEAR, BORDER_CONSTANT, fixed point) -> channel swap -> augment_hsv (cv2 BGR2HSV / HSV2BGR; hsv_simd_block: the pixel
 * count of one vector block of cv2's HSV2BGR, whose columns below w - w % block truncate and whose tail rounds) -> horizontal flip
 * -> mixup with the partner's canvas, each cv2.resize on the way recomputed -> bottom-right placement, resized (INTER_LINEAR)
 * when the rescale size differs from the affine size, onto pad_value -> v / max_value -> round-to-nearest bf16.  Bit-exact with
 * the reference's cv2 / numpy chain.  A table naming bytes outside src, a degenerate or non-finite matrix, a matrix mapping
 * the output outside +-2^20 source pixels, or a bad size or flag is refused with SGB_E_INVALID; so is a mosaic whose tile lies
 * outside src, whose resized size is not in [1, 32768), whose rectangle leaves its quadrant of the canvas or reads outside the
 * resized tile, whose centre lies outside the canvas or whose border value is not in [0, 255].  batch == 0 is a no-op. */
int sgb_detection_augment(const int64_t* table_host, const int64_t* table, const uint8_t* src, int64_t src_bytes, int32_t batch,
                          int32_t channels, int32_t out_h, int32_t out_w, int32_t out_pitch, int32_t pad_value, double max_value,
                          int32_t hsv_simd_block, sgb_bf16* out, void* stream);

/* ---- ImageNet train augmentation (recipes/dataset_params/imagenet_resnet50_dataset_params.yaml train chain:
 *      datasets/datasets_utils.py:316-354 RandomResizedCropAndInterpolation, RandomHorizontalFlip, datasets/auto_augment.py:271-447
 *      RandAugment, ToTensor, Normalize; datasets/mixup.py:104-313 CollateMixup, batch mode) ---- */
/* Per-image table: int64 [batch][SGB_IN_FIELDS].
 *   crop window: byte offset in src, h, w (dense rows of w * 3 bytes: only the window RandomResizedCrop chose), filter (0 bilinear,
 *   1 bicubic), horizontal flip flag, byte offset in the workspace of the window's horizontally resized rows (h * size * 3 bytes)
 *   then SGB_IN_OPS RandAugment ops in order, SGB_IN_OP_FIELDS each from SGB_IN_OP: the op code, then its arguments:
 *     AFFINE: Pillow's inverse 2 x 3 matrix as six float64 values stored bit for bit (ShearX / Y, TranslateXRel / YRel, Rotate)
 *     POSTERIZE: bits kept in [0, 8); SOLARIZE: threshold in [0, 256]; SOLARIZE_ADD: the addend in [0, 255]
 *     BRIGHTNESS, CONTRAST, COLOR, SHARPNESS: the enhance factor as a float64 value stored bit for bit
 *     NONE, INVERT, AUTOCONTRAST, EQUALIZE: none */
#define SGB_IN_OFFSET 0
#define SGB_IN_H 1
#define SGB_IN_W 2
#define SGB_IN_FILTER 3
#define SGB_IN_FLIP 4
#define SGB_IN_WS_OFFSET 5
#define SGB_IN_OP 6
#define SGB_IN_OP_FIELDS 7
#define SGB_IN_OPS 2
#define SGB_IN_FIELDS 20
#define SGB_IN_OP_NONE 0
#define SGB_IN_OP_AFFINE 1
#define SGB_IN_OP_INVERT 2
#define SGB_IN_OP_POSTERIZE 3
#define SGB_IN_OP_SOLARIZE 4
#define SGB_IN_OP_SOLARIZE_ADD 5
#define SGB_IN_OP_BRIGHTNESS 6
#define SGB_IN_OP_CONTRAST 7
#define SGB_IN_OP_AUTOCONTRAST 8
#define SGB_IN_OP_EQUALIZE 9
#define SGB_IN_OP_COLOR 10
#define SGB_IN_OP_SHARPNESS 11
/* table_host: the table in host memory (validated here); table: the same table in device memory.  src: device uint8 buffer of
 * src_bytes holding every crop window.  workspace: caller-owned device uint8 buffer of workspace_bytes receiving each window's
 * horizontal resize pass.  out: device bf16 [batch, size, size, out_pitch] (out_pitch >= 3, a multiple of 8; channels >= 3 written
 * as 0).  fill_host[3]: RandAugment's fill colour (img_mean in uint8); mean_host[3] / std_host[3]: Normalize.  mix_mode 0: no mix,
 * 1: mixup with lam / one_minus_lam (float32 values of lam and 1 - lam), 2: cutmix of the box box_host[4] = (yl, yh, xl, xh);
 * image i mixes with image batch - 1 - i.  ONE launch for the batch (batch even): a thread-block cluster of two CTAs holds the
 * pair (i, batch - 1 - i), each CTA its image in shared memory: Pillow's 8-bit crop resize -> flip -> the two RandAugment ops ->
 * ToTensor / Normalize in float32 -> the mix, reading the partner's pixels from its CTA's shared memory -> round-to-nearest
 * bf16.  Bit-exact with the reference's PIL chain and CollateMixup.  Bytes outside src or the workspace, an unknown op or filter,
 * a bad argument, size, flag, mix mode or box, or an odd batch is refused with SGB_E_INVALID.  batch == 0 is a no-op. */
int sgb_imagenet_augment(const int64_t* table_host, const int64_t* table, const uint8_t* src, int64_t src_bytes, uint8_t* workspace,
                         int64_t workspace_bytes, int32_t batch, int32_t size, int32_t out_pitch, const int32_t* fill_host,
                         const float* mean_host, const float* std_host, int32_t mix_mode, float lam, float one_minus_lam,
                         const int32_t* box_host, sgb_bf16* out, void* stream);

/* ---- CIFAR-10 augmentation (recipes/dataset_params/cifar10_dataset_params.yaml:9-23 train chain, torchvision 0.26's: RandomCrop(32,
 *      padding=4) (F.pad with fill 0, then get_params's two torch.randint draws), RandomHorizontalFlip (torch.rand(1) < 0.5),
 *      ToTensor (float32 / 255), Normalize (tensor.sub_(mean).div_(std)); cifar10_dataset_params.yaml:37-49 validation chain:
 *      Resize(32), the identity on the 32 x 32 images of datasets/classification_datasets/cifar.py:14-45, ToTensor, Normalize) ---- */
/* Per-sample table: int32 [batch][SGB_CF_FIELDS]: the source image's index in src, the crop's top and left corner in the
 * 40 x 40 zero-padded image (each in [0, 8]; the validation chain is top = left = 4), the horizontal flip flag (0 or 1). */
#define SGB_CF_SOURCE 0
#define SGB_CF_TOP 1
#define SGB_CF_LEFT 2
#define SGB_CF_FLIP 3
#define SGB_CF_FIELDS 4
#define SGB_CF_SIZE 32
#define SGB_CF_PAD 4
/* table_host: the table in host memory (validated here); table: the same table in device memory.  src: device uint8
 * [src_images][32][32][3] RGB (a batch's packed images, or a whole resident data set indexed by the table).  out: device bf16
 * [batch, 32, 32, out_pitch] (16-byte aligned, out_pitch >= 3 and a multiple of 8; channels >= 3 written as 0).  mean_host[3] /
 * std_host[3]: Normalize.  ONE launch for the batch: per output pixel, the zero-padded crop -> flip -> ToTensor / Normalize in
 * float32 with IEEE division in torchvision's order -> round-to-nearest-even bf16.  Bit-exact with torchvision's chain rounded to
 * bf16.  batch < 1, a source index outside [0, src_images), a crop corner outside [0, 8], a flip flag other than 0 / 1, a bad
 * pitch, a misaligned out or a non-finite mean / std (or a zero std) is refused with SGB_E_INVALID. */
int sgb_cifar_augment(const int32_t* table_host, const int32_t* table, const uint8_t* src, int64_t src_images, int32_t batch,
                      int32_t out_pitch, const float* mean_host, const float* std_host, sgb_bf16* out, void* stream);

/* ---- pose train augmentation (training/transforms/keypoints/*.py of the YOLO-NAS-POSE recipes: KeypointsRandomHorizontalFlip,
 *      KeypointsBrightnessContrast, KeypointsReverseImageChannels, KeypointsHSV, KeypointsRandomRotate90,
 *      KeypointsRandomAffineTransform, KeypointsMosaic, KeypointsLongestMaxSize, KeypointsPadIfNeeded, KeypointsImageStandardize) ---- */
/* Per-sample table: int64 [batch][SGB_POSE_FIELDS].  Three uint8 values (pad colours) are packed as v0 | v1 << 8 | v2 << 16.
 *   NSUB: 1, or 4 for a mosaic; CANVAS_H / W: the mosaic canvas (or the single tile's size); MOSAIC_PAD: the mosaic pad colour
 *   RS_H / W: the LongestMaxSize size of the canvas (== the canvas size when it is not resized)
 *   PAD_TOP / PAD_LEFT: the resized canvas' position in the out_size x out_size output; PAD_VALUE: the pad colour
 *   then NSUB sub-sample records of SGB_POSE_SUB_FIELDS from SGB_POSE_SUB (top-left, top-right, bottom-left, bottom-right):
 *     source byte offset in src, h, w (dense rows of w * 3 bytes); flip flag; brightness-contrast flag, the three float32 channel
 *     means, the float32 contrast and brightness gains (float32 bits); channel reversal flag; HSV flag and gains dh / ds / dv;
 *     np.rot90 count k in [0, 3]; affine flag, forward 2 x 3 matrix (float64 bits), cv2 interpolation flag in [0, 4], border
 *     colour; the byte offset of the tile's rotated image in the workspace; the tile's position y / x in the canvas; its size
 *     rh / rw after rot90 (the affine keeps the size) */
#define SGB_POSE_NSUB 0
#define SGB_POSE_CANVAS_H 1
#define SGB_POSE_CANVAS_W 2
#define SGB_POSE_MOSAIC_PAD 3
#define SGB_POSE_RS_H 4
#define SGB_POSE_RS_W 5
#define SGB_POSE_PAD_TOP 6
#define SGB_POSE_PAD_LEFT 7
#define SGB_POSE_PAD_VALUE 8
#define SGB_POSE_SUB 16
#define SGB_POSE_SUB_FIELDS 32
#define SGB_POSE_FIELDS 144
#define SGB_POSE_S_OFFSET 0
#define SGB_POSE_S_H 1
#define SGB_POSE_S_W 2
#define SGB_POSE_S_FLIP 3
#define SGB_POSE_S_BC 4
#define SGB_POSE_S_MEAN 5 /* 3 slots */
#define SGB_POSE_S_CONTRAST 8
#define SGB_POSE_S_BRIGHTNESS 9
#define SGB_POSE_S_REVERSE 10
#define SGB_POSE_S_HSV 11
#define SGB_POSE_S_DH 12
#define SGB_POSE_S_DS 13
#define SGB_POSE_S_DV 14
#define SGB_POSE_S_ROT 15
#define SGB_POSE_S_AFFINE 16
#define SGB_POSE_S_M 17 /* 6 slots */
#define SGB_POSE_S_MODE 23
#define SGB_POSE_S_BORDER 24
#define SGB_POSE_S_WS_OFFSET 25
#define SGB_POSE_S_Y 26
#define SGB_POSE_S_X 27
#define SGB_POSE_S_RH 28
#define SGB_POSE_S_RW 29
/* table_host: the table in host memory (validated here); table: the same table in device memory.  src: device uint8 buffer of
 * src_bytes holding every sub-sample's source image (H x W x 3).  workspace: caller-owned device uint8 buffer of workspace_bytes
 * receiving every tile's rotated image at its WS_OFFSET.  out: device bf16 [batch, out_size, out_size, out_pitch] (out_pitch >= 3,
 * a multiple of 8; channels >= 3 written as 0).  TWO launches for the batch, whatever its size: (1) per tile pixel, flip ->
 * brightness-contrast -> channel reversal -> augment_hsv (hsv_simd_block as in sgb_detection_augment) -> np.rot90 into the
 * workspace; (2) per output pixel, pad -> cv2.resize INTER_LINEAR of the canvas -> mosaic placement -> cv2.warpAffine
 * (BORDER_CONSTANT, fixed point, INTER_NEAREST / LINEAR / CUBIC / AREA / LANCZOS4) -> v / max_value -> round-to-nearest bf16.
 * Bit-exact with the reference's cv2 / numpy chain.  Bytes outside src or the workspace, a degenerate or non-finite matrix, a
 * matrix mapping the tile outside +-2^20 pixels, a tile outside the canvas, or a bad size, count, mode or flag is refused with
 * SGB_E_INVALID.  batch == 0 is a no-op. */
int sgb_pose_augment(const int64_t* table_host, const int64_t* table, const uint8_t* src, int64_t src_bytes, uint8_t* workspace,
                     int64_t workspace_bytes, int32_t batch, int32_t out_size, int32_t out_pitch, double max_value, int32_t hsv_simd_block,
                     sgb_bf16* out, void* stream);

/* ---- row-wise classification decode (training/metrics/classification_metrics.py:40-78 Accuracy / Top5, utils.py accuracy(),
 *      pipelines.py:516-531 torch.max(softmax(logits), 1)) ---- */
/* logits [N, C] (row stride row_stride >= C elements; bf16 when logits_bf16, else f32).  One warp per row, one pass over the row.
 * Ranking is (value desc, index asc) with NaN above every number: the top-1 index is the first maximum (torch.argmax), and the
 * target is in the top k when fewer than k elements rank above it.  The target is target[N] (int64) or the argmax of the soft-label
 * row soft_target[N, C] (row stride target_stride, bf16 when target_bf16, else f32); exactly one of the two when counters are given.
 * counters[4] (int64, accumulated): top-1 correct, top-k correct (1 <= k <= C), rows, rows whose target is outside [0, C).
 * label[N] int32 / confidence[N] f32 (each optional): the top-1 index and 1 / sum_j exp(x_j - max), the maximum of
 * softmax(logits).  N == 0 is a no-op. */
int sgb_classify_rows(const void* logits, int64_t N, int32_t C, int64_t row_stride, int32_t logits_bf16, const int64_t* target,
                      const void* soft_target, int64_t target_stride, int32_t target_bf16, int32_t k, int64_t* counters,
                      int32_t* label, float* confidence, void* stream);

/* ---- optimizer over the flat parameter buffer (sg_trainer.py:634-644) --------------------------------------- */
/* Hyper-parameters live in DEVICE memory (so a CUDA-graph-captured step follows the host-side LR schedule).  hp is ONE device
 * float32 row in the layout of csrc/optim_math.cuh, grad_scale included:
 *   sgd   SGD_*     torch.optim.SGD
 *   adamw ADAMW_*   torch.optim.AdamW */
int sgb_sgd_step(float* p, const float* g, float* mom, int64_t n, const float* hp, void* stream);
int sgb_adamw_step(float* p, const float* g, float* m, float* v, int64_t n, const float* hp, void* stream);
/* The other optimizers of the reference's registry (common/object_names.py:143-152), one launch per weight-decay range.  hp is ONE
 * device float32 row in the layout of csrc/optim_math.cuh (ADAM_*, RMS_*, RTF_*, LION_*), grad_scale included; every element is
 * computed op for op as the reference's single-tensor CPU step, each op rounded to float32 on its own (FMA exactly where torch's CPU
 * kernels fuse: add with alpha, addcmul, lerp).  n == 0 is a no-op; a NULL required pointer is refused with SGB_E_INVALID.
 *   adam        torch.optim.Adam, L2-coupled decay g + wd * p (training/params.py:90; torch/optim/adam.py _single_tensor_adam)
 *   rmsprop     torch.optim.RMSprop: momentum_buffer only with momentum > 0, grad_avg only when centered, else NULL
 *               (training/params.py:92; torch/optim/rmsprop.py _single_tensor_rmsprop)
 *   rmsprop_tf  RMSpropTF: eps inside the sqrt, TF update order, decoupled_decay, lr_in_momentum
 *               (training/utils/optimizers/rmsprop_tf.py:89-153)
 *   lion        Lion: p *= 1 - lr * wd; p -= lr * sign(b1 * m + (1 - b1) * g); m = b2 * m + (1 - b2) * g  (lion.py:57-79) */
int sgb_adam_step(float* p, const float* g, float* m, float* v, int64_t n, const float* hp, void* stream);
int sgb_rmsprop_step(float* p, const float* g, float* square_avg, float* momentum_buffer, float* grad_avg, int64_t n, const float* hp, void* stream);
int sgb_rmsprop_tf_step(float* p, const float* g, float* square_avg, float* momentum_buffer, float* grad_avg, int64_t n, const float* hp, void* stream);
int sgb_lion_step(float* p, const float* g, float* m, int64_t n, const float* hp, void* stream);
/* Lamb (training/utils/optimizers/lamb.py:123-216) over EVERY live parameter at once: chunks is a device int64 [nchunk][4] table
 * {start, len, first chunk of its tensor, chunks of its tensor} (a chunk lies inside one parameter tensor); hp is two LAMB_* rows,
 * row 0 for elements before n_decay, row 1 after; partials is device float64 [3 * nchunk].
 *   sgb_lamb_grad_sqnorm  (1 launch)  partials[c] = sum over chunk c of (g * grad_scale)^2
 *   sgb_lamb_step         (2 launches) clip = max(||g|| / max_grad_norm, 1) over all chunks; m / v update with grad_averaging and
 *                         bias_correction; update = m^ / (sqrt(v) / sqrt(bc2) + eps) + wd * p into `update`; per tensor
 *                         trust = ||p|| / ||update|| with the reference's zero-norm branches and trust_clip (1 where the row does
 *                         not adapt); p -= lr * trust * update.
 * Every sum is float64 in a fixed order with no atomics: two runs of one step are bit-identical.  No host synchronisation. */
int sgb_lamb_grad_sqnorm(const float* g, const int64_t* chunks, int32_t nchunk, const float* hp, double* partials, void* stream);
int sgb_lamb_step(float* p, const float* g, float* m, float* v, float* update, int64_t n_decay, const int64_t* chunks, int32_t nchunk,
                  const float* hp, double* partials, void* stream);
/* clip_grad_norm (sg_trainer.py:634-636; the value is refused when <= 0, :1416-1417): torch.nn.utils.clip_grad_norm_ with norm
 * type 2 over every live gradient, run once per optimisation step after the all-reduce and before the optimizer.  The gradients
 * are not rewritten: the coefficient is folded into the optimizer's grad_scale, column gs_col of both hp rows (hp is the
 * optimizer's device table of two hp_len-wide rows: SGD_GS / ADAMW_GS / ADAM_GS / RMS_GS / RTF_GS / LION_GS / LAMB_GS of
 * csrc/optim_math.cuh).  chunks / nchunk: the chunk table of sgb_lamb_step; partials: device float64 [nchunk].
 *   launch 1  partials[c] = sum over chunk c of (g * hp[gs_col])^2                       (the kernel of sgb_lamb_grad_sqnorm)
 *   launch 2  one CTA: total = (float)sqrt(sum of partials, float64, fixed order);
 *             coef = min(reciprocal(total + 1e-6) * max_norm, 1) in float32 (torch's op order; NaN stays NaN, inf gives 0);
 *             norm_coef[0] = total, norm_coef[1] = coef; hp[gs_col] *= coef; hp[hp_len + gs_col] *= coef.
 * No host synchronisation and no branch on the norm on the host: capturable.  max_norm <= 0 or gs_col outside [0, hp_len) is
 * refused with SGB_E_INVALID. */
int sgb_clip_grad_norm(const float* g, const int64_t* chunks, int32_t nchunk, float* hp, int32_t hp_len, int32_t gs_col, float max_norm, double* partials,
                       float* norm_coef, void* stream);
/* ema = ema * (*decay) + (1 - *decay) * p   (training/utils/ema.py:126-142) */
int sgb_ema_update(float* ema, const float* p, int64_t n, const float* decay, void* stream);

/* ---- best-snapshot average (training/utils/weight_averaging_utils.py:89-95, sg_trainer.py:732-739) ----------------------- */
#define SGB_AVG_MAX_SLOTS 64
/* slots: DEVICE array of k device pointers, each to n float32 values (snapshot slots 0 .. k-1, in slot order).  out[i] is the
 * reference's running mean  a <- s_0[i];  for m = 1 .. k-1: a <- (a * m + s_m[i]) / (m + 1),  every multiply, add and divide
 * rounded to float32 on its own (no FMA contraction), so the result is bit-identical to the reference's torch loop on the CPU,
 * Inf and subnormals included; NaN stays NaN.  One pass: k * n * 4 bytes read, n * 4 written.  k outside [1, SGB_AVG_MAX_SLOTS],
 * n < 0 or a NULL pointer is refused with SGB_E_INVALID; n == 0 is a no-op.  out may not alias a slot. */
int sgb_average_snapshots(const float* const* slots, int32_t k, int64_t n, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SGB200_H_ */

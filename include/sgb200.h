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
/* Hyper-parameters live in DEVICE memory (so a CUDA-graph-captured step follows the host-side LR schedule):
 *   sgd   hp[5] = {lr, momentum, weight_decay, grad_scale, nesterov}
 *   adamw hp[8] = {lr, beta1, beta2, eps, weight_decay, 1-beta1^t, 1-beta2^t, grad_scale}   (torch.optim semantics) */
int sgb_sgd_step(float* p, const float* g, float* mom, int64_t n, const float* hp, void* stream);
int sgb_adamw_step(float* p, const float* g, float* m, float* v, int64_t n, const float* hp, void* stream);
/* ema = ema * (*decay) + (1 - *decay) * p   (training/utils/ema.py:126-142) */
int sgb_ema_update(float* ema, const float* p, int64_t n, const float* decay, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SGB200_H_ */

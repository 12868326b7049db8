// The hyper-parameter rows of all seven flat-buffer optimizers, and the per-element arithmetic of Adam, RMSprop, RMSpropTF, Lion
// and Lamb and of clip_grad_norm's coefficient, host+device: the CUDA kernels in optim.cu run it per element, and the CPU suite
// compiles this header with g++ (-ffp-contract=off) behind serial drivers (tests/host_kernels/optim_host.cpp, clip_host.cpp).
// SGD and AdamW keep their arithmetic in their kernels in optim.cu, written with plain operators that nvcc contracts into FMAs.
//
// Each function restates, op for op, the reference's single-tensor CPU step in float32 (torch.optim.Adam / RMSprop, and the
// RMSpropTF, Lion and Lamb classes of training/utils/optimizers/).  torch's CPU kernels round as follows, and so does this header:
//   x.add(y, alpha=a)          fma(y, a, x)
//   x.addcmul(y, z, value=a)   fma(a * y, z, x)
//   x.addcdiv(y, z, value=a)   x + (a * y) / z             (no fused op)
//   x.lerp(y, w)               |w| < 0.5 ? fma(w, y - x, x) : fma(w - 1, y - x, y)
//   x * s, x / s (s a Python float)   one float32 multiply / divide by (float)s
// nvcc would contract a separate multiply and add into an FMA, so the device side spells every op with its round-to-nearest
// intrinsic; the host side relies on -ffp-contract=off.  Every scalar the host derives from the hyper-parameters (bias
// corrections, step sizes, 1 - beta) is computed there in double and rounded to float32 once, as torch does with Python floats.
#pragma once
#include <math.h>
#include <stdint.h>

#ifndef SGB_HD
#ifdef __CUDACC__
#define SGB_HD __host__ __device__ __forceinline__
#else
#define SGB_HD static inline
#endif
#endif

namespace sgb_optim {

// ---- hyper-parameter rows (float32, one row per weight-decay group; row 1 is the zero-decay group)
// sgd:        torch.optim.SGD; nesterov is 0 or 1
enum { SGD_LR, SGD_MOMENTUM, SGD_WD, SGD_GS, SGD_NESTEROV, SGD_HP };
// adamw:      torch.optim.AdamW; bc1 = 1 - beta1^t, bc2 = 1 - beta2^t
enum { ADAMW_LR, ADAMW_B1, ADAMW_B2, ADAMW_EPS, ADAMW_WD, ADAMW_BC1, ADAMW_BC2, ADAMW_GS, ADAMW_HP };
// adam:       torch.optim.Adam, L2-coupled decay
enum { ADAM_WD, ADAM_W1, ADAM_B2, ADAM_1MB2, ADAM_NEG_STEP, ADAM_BC2_SQRT, ADAM_EPS, ADAM_GS, ADAM_HP };
// rmsprop:    torch.optim.RMSprop (zero-initialised square_avg, eps outside the sqrt)
enum { RMS_WD, RMS_ALPHA, RMS_1MA, RMS_EPS, RMS_MOMENTUM, RMS_NEG_LR, RMS_CENTERED, RMS_GS, RMS_HP };
// rmsprop_tf: RMSpropTF (square_avg initialised to ones, eps inside the sqrt); flags: 1 centered, 2 decoupled_decay, 4 lr_in_momentum
enum { RTF_WD, RTF_1MA, RTF_EPS, RTF_MOMENTUM, RTF_LR, RTF_NEG_LR, RTF_FLAGS, RTF_GS, RTF_HP };
// lion:       decay = 1 - lr * weight_decay
enum { LION_DECAY, LION_B1, LION_1MB1, LION_NEG_LR, LION_B2, LION_1MB2, LION_GS, LION_HP };
// lamb:       beta3 = 1 - beta1 with grad_averaging, else 1; bc1 / bc2_sqrt = 1 without bias_correction; adapt = weight_decay != 0
//             or always_adapt
enum { LAMB_B1, LAMB_BETA3, LAMB_B2, LAMB_1MB2, LAMB_BC2_SQRT, LAMB_BC1, LAMB_EPS, LAMB_WD, LAMB_NEG_LR, LAMB_GS, LAMB_MAX_NORM,
       LAMB_ADAPT, LAMB_TRUST_CLIP, LAMB_HP };

// ---- float32 ops, each rounded on its own
SGB_HD float mul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
SGB_HD float add(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
SGB_HD float sub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
SGB_HD float div(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
SGB_HD float fma_(float a, float b, float c) {
#ifdef __CUDA_ARCH__
  return __fmaf_rn(a, b, c);
#else
  return fmaf(a, b, c);
#endif
}
SGB_HD float sqrt_(float a) {
#ifdef __CUDA_ARCH__
  return __fsqrt_rn(a);
#else
  return sqrtf(a);
#endif
}
// torch's lerp(x, y, w)
SGB_HD float lerp(float x, float y, float w) {
  const float d = sub(y, x);
  return fabsf(w) < 0.5f ? fma_(w, d, x) : fma_(sub(w, 1.f), d, y);
}

// ---- Adam (torch/optim/adam.py _single_tensor_adam, amsgrad=False)
SGB_HD void adam(float& p, float g, float& m, float& v, const float* hp) {
  float gr = mul(g, hp[ADAM_GS]);
  if (hp[ADAM_WD] != 0.f) gr = fma_(p, hp[ADAM_WD], gr);                 // grad = grad.add(param, alpha=weight_decay)
  m = lerp(m, gr, hp[ADAM_W1]);                                           // exp_avg.lerp_(grad, 1 - beta1)
  v = fma_(mul(hp[ADAM_1MB2], gr), gr, mul(v, hp[ADAM_B2]));              // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
  const float denom = add(div(sqrt_(v), hp[ADAM_BC2_SQRT]), hp[ADAM_EPS]);  // (exp_avg_sq.sqrt() / bias_correction2_sqrt).add_(eps)
  p = add(p, div(mul(hp[ADAM_NEG_STEP], m), denom));                      // param.addcdiv_(exp_avg, denom, value=-step_size)
}

// ---- RMSprop (torch/optim/rmsprop.py _single_tensor_rmsprop); buf / ga are read only with momentum > 0 / centered
SGB_HD void rmsprop(float& p, float g, float& sa, float* buf, float* ga, const float* hp) {
  float gr = mul(g, hp[RMS_GS]);
  if (hp[RMS_WD] != 0.f) gr = fma_(p, hp[RMS_WD], gr);
  sa = fma_(mul(hp[RMS_1MA], gr), gr, mul(sa, hp[RMS_ALPHA]));  // square_avg.mul_(alpha).addcmul_(grad, grad, value=1 - alpha)
  float avg;
  if (hp[RMS_CENTERED] != 0.f) {
    *ga = lerp(*ga, gr, hp[RMS_1MA]);       // grad_avg.lerp_(grad, 1 - alpha)
    avg = sqrt_(fma_(-*ga, *ga, sa));       // square_avg.addcmul(grad_avg, grad_avg, value=-1).sqrt_()
  } else {
    avg = sqrt_(sa);
  }
  avg = add(avg, hp[RMS_EPS]);
  if (hp[RMS_MOMENTUM] > 0.f) {
    *buf = add(mul(*buf, hp[RMS_MOMENTUM]), div(gr, avg));  // buf.mul_(momentum).addcdiv_(grad, avg)
    p = fma_(*buf, hp[RMS_NEG_LR], p);                      // param.add_(buf, alpha=-lr)
  } else {
    p = add(p, div(mul(hp[RMS_NEG_LR], gr), avg));  // param.addcdiv_(grad, avg, value=-lr)
  }
}

// ---- RMSpropTF (training/utils/optimizers/rmsprop_tf.py:89-153); buf / ga are read only with momentum > 0 / centered
SGB_HD void rmsprop_tf(float& p, float g, float& sa, float* buf, float* ga, const float* hp) {
  const int flags = (int)hp[RTF_FLAGS];
  const float wd = hp[RTF_WD], oma = hp[RTF_1MA];
  float gr = mul(g, hp[RTF_GS]);
  if (wd != 0.f) {
    if (flags & 2) p = fma_(p, -wd, p);  // p.data.add_(-weight_decay, p.data)
    else gr = fma_(p, wd, gr);           // grad = grad.add(weight_decay, p.data)
  }
  sa = fma_(sub(mul(gr, gr), sa), oma, sa);  // square_avg.add_(1 - alpha, grad.pow(2) - square_avg)
  float avg;
  if (flags & 1) {
    *ga = fma_(sub(gr, *ga), oma, *ga);                     // grad_avg.add_(1 - alpha, grad - grad_avg)
    avg = sqrt_(add(fma_(-*ga, *ga, sa), hp[RTF_EPS]));     // square_avg.addcmul(-1, grad_avg, grad_avg).add(eps).sqrt_()
  } else {
    avg = sqrt_(add(sa, hp[RTF_EPS]));  // square_avg.add(eps).sqrt_()
  }
  if (hp[RTF_MOMENTUM] > 0.f) {
    if (flags & 4) {
      *buf = add(mul(*buf, hp[RTF_MOMENTUM]), div(mul(hp[RTF_LR], gr), avg));  // buf.mul_(momentum).addcdiv_(lr, grad, avg)
      p = sub(p, *buf);                                                        // p.data.add_(-buf)
    } else {
      *buf = add(mul(*buf, hp[RTF_MOMENTUM]), div(gr, avg));  // buf.mul_(momentum).addcdiv_(grad, avg)
      p = fma_(*buf, hp[RTF_NEG_LR], p);                      // p.data.add_(-lr, buf)
    }
  } else {
    p = add(p, div(mul(hp[RTF_NEG_LR], gr), avg));  // p.data.addcdiv_(-lr, grad, avg)
  }
}

// ---- Lion (training/utils/optimizers/lion.py:57-79); sign(0) = 0
SGB_HD void lion(float& p, float g, float& m, const float* hp) {
  p = mul(p, hp[LION_DECAY]);  // p.data.mul_(1 - lr * weight_decay)
  const float gr = mul(g, hp[LION_GS]);
  const float u = add(mul(m, hp[LION_B1]), mul(gr, hp[LION_1MB1]));  // exp_avg * beta1 + grad * (1 - beta1)
  const float s = u > 0.f ? 1.f : (u < 0.f ? -1.f : u);              // torch.sign (NaN stays NaN)
  p = fma_(s, hp[LION_NEG_LR], p);                                   // p.add_(torch.sign(update), alpha=-lr)
  m = fma_(gr, hp[LION_1MB2], mul(m, hp[LION_B2]));                  // exp_avg.mul_(beta2).add_(grad, alpha=1 - beta2)
}

// ---- Lamb (training/utils/optimizers/lamb.py:135-214)
// the global clip divisor from the sum of squares of every live (scaled) gradient: where(norm > max_grad_norm, norm / max, 1)
SGB_HD float lamb_clip(double grad_sqsum, const float* hp) {
  const float norm = sqrt_((float)grad_sqsum), mx = hp[LAMB_MAX_NORM];
  return norm > mx ? div(norm, mx) : 1.f;
}
// m / v update and the un-adapted update (weight decay included); returns the update
SGB_HD float lamb_update(float p, float g, float& m, float& v, float clip, const float* hp) {
  const float gr = div(mul(g, hp[LAMB_GS]), clip);                        // p.grad.div_(clip_global_grad_norm)
  m = fma_(gr, hp[LAMB_BETA3], mul(m, hp[LAMB_B1]));                       // exp_avg.mul_(beta1).add_(grad, alpha=beta3)
  v = fma_(mul(hp[LAMB_1MB2], gr), gr, mul(v, hp[LAMB_B2]));               // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
  const float denom = add(div(sqrt_(v), hp[LAMB_BC2_SQRT]), hp[LAMB_EPS]);  // (exp_avg_sq.sqrt() / math.sqrt(bc2)).add_(eps)
  float u = div(div(m, hp[LAMB_BC1]), denom);                              // (exp_avg / bias_correction1).div_(denom)
  if (hp[LAMB_WD] != 0.f) u = fma_(p, hp[LAMB_WD], u);                      // update.add_(p, alpha=weight_decay)
  return u;
}
// the per-tensor trust ratio from sum(p^2) and sum(update^2) over that tensor (1 when the group does not adapt)
SGB_HD float lamb_trust(double p_sqsum, double u_sqsum, const float* hp) {
  if (hp[LAMB_ADAPT] == 0.f) return 1.f;
  const float w = sqrt_((float)p_sqsum), u = sqrt_((float)u_sqsum);
  float t = w > 0.f ? (u > 0.f ? div(w, u) : 1.f) : 1.f;
  if (hp[LAMB_TRUST_CLIP] != 0.f && t > 1.f) t = 1.f;  // torch.minimum(trust_ratio, 1) (NaN stays NaN)
  return t;
}
// update.mul_(trust_ratio); p.add_(update, alpha=-lr)
SGB_HD float lamb_apply(float p, float u, float trust, const float* hp) { return fma_(mul(u, trust), hp[LAMB_NEG_LR], p); }

// ---- clip_grad_norm (sg_trainer.py:634-636: torch.nn.utils.clip_grad_norm_, norm type 2)
// total = ||g||_2 from the float64 sum of squares, rounded to float32 once, as torch's float32 norm returns it.  torch adds the
// squares in float32: a sum beyond float32's range is an infinite norm there (so coef 0), and here too.
SGB_HD float clip_total_norm(double grad_sqsum) {
  const float s = (float)grad_sqsum;
  return isinf(s) ? s : (float)sqrt(grad_sqsum);
}
// clip_coef = max_norm / (total_norm + 1e-6), which torch's Tensor.__rtruediv__ evaluates as reciprocal(total + 1e-6) * max_norm;
// clamp(max=1.0) keeps NaN (a NaN gradient) and gives 0 for an infinite norm, as torch does
SGB_HD float clip_coef(float total, float max_norm) {
  const float c = mul(div(1.f, add(total, 1e-6f)), max_norm);
  return c > 1.f ? 1.f : c;
}
// g.mul_(clip_coef) folded into the optimizer's grad_scale: column gs_col of both weight-decay rows of an hp_len-wide table
SGB_HD void clip_scale_rows(float* hp, int hp_len, int gs_col, float coef) {
  hp[gs_col] = mul(hp[gs_col], coef);
  hp[hp_len + gs_col] = mul(hp[hp_len + gs_col], coef);
}

}  // namespace sgb_optim

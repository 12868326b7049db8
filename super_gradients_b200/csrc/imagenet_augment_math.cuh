// Arithmetic of the ImageNet train augmentation (the ResNet-50 recipe's chain), host+device: the CUDA kernel in imagenet_augment.cu
// calls these functions and the CPU suite compiles this header with g++ to check them, bit for bit, against the installed Pillow.
//
// Reference chain (recipes/dataset_params/imagenet_resnet50_dataset_params.yaml): RandomResizedCropAndInterpolation(224, random)
// (datasets/datasets_utils.py:316-354: PIL crop, then Image.resize BILINEAR or BICUBIC; the resize is resample_math.cuh) ->
// RandomHorizontalFlip -> RandAugment rand-m7-mstd0.5 (datasets/auto_augment.py:271-447: two ops from Pillow's Image.transform,
// ImageOps and ImageEnhance) -> ToTensor -> Normalize -> CollateMixup batch mode (datasets/mixup.py:272-293).
//
// The Pillow C code each op runs, as the installed Pillow computes it:
//   Image.transform(AFFINE, BILINEAR, fillcolor): the output pixel (x, y) maps to (a0 (x + .5) + a1 (y + .5) + a2, a3 (x + .5) +
//     a4 (y + .5) + a5) in double; a point outside [0, w) x [0, h) keeps the fill colour; otherwise bilinear weights from the
//     point minus .5, edge-clamped taps (a missing row below repeats the row), and the double result truncated to uint8.
//   Image.blend(im1, im2, alpha) (every ImageEnhance op): alpha is a C float; out = (uint8)(im1 + alpha (im2 - im1)) in float,
//     clipped to [0, 255] when alpha is outside [0, 1].
//   convert("L"): (19595 r + 38470 g + 7471 b + 0x8000) >> 16.
//   ImageFilter.SMOOTH (Sharpness): 3x3 kernel (1 1 1 / 1 5 1 / 1 1 1) / 13 in float with offset .5, the border rows and columns
//     copied.
//   ImageOps LUTs (Invert, Posterize, Solarize, SolarizeAdd's point()), AutoContrast / Equalize from per-channel histograms and
//     Contrast's mean of the L image: Python integer or double arithmetic, restated below.
// The float and double arithmetic goes through explicitly rounded intrinsics on the device, as in resample_math.cuh: nvcc contracts
// a * b + c into an FMA by default, g++ does not.
#pragma once
#include <math.h>
#include <stdint.h>

#include "resample_math.cuh"
#include "sgb200.h"

namespace sgb_in {

using sgb_rs::dadd;
using sgb_rs::dmul;
using sgb_rs::ddiv;

SGB_HD float fadd(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
SGB_HD float fmul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
SGB_HD float fdiv(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

SGB_HD double arg_f64(const int64_t* args, int i) {
  union {
    int64_t i;
    double d;
  } u;
  u.i = args[i];
  return u.d;
}

// Image.blend(im1, im2, alpha) of one channel value
SGB_HD uint8_t blend(int in1, int in2, float alpha) {
  const float v = fadd((float)in1, fmul(alpha, (float)(in2 - in1)));
  if (alpha >= 0.f && alpha <= 1.f) return (uint8_t)v;
  if (v <= 0.f) return 0;
  if (v >= 255.f) return 255;
  return (uint8_t)v;
}

SGB_HD int rgb_to_l(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

// value v after a point-wise op (SGB_IN_OP_INVERT .. SGB_IN_OP_CONTRAST); `mean`: Contrast's grey level
SGB_HD uint8_t lut_value(int op, const int64_t* args, int mean, int v) {
  switch (op) {
    case SGB_IN_OP_INVERT:
      return (uint8_t)(255 - v);
    case SGB_IN_OP_POSTERIZE:  // bits in [0, 8): v & ~(2^(8 - bits) - 1)
      return (uint8_t)(v & ~((1 << (8 - (int)args[0])) - 1));
    case SGB_IN_OP_SOLARIZE:
      return (uint8_t)(v < args[0] ? v : 255 - v);
    case SGB_IN_OP_SOLARIZE_ADD: {
      const int s = v + (int)args[0];
      return (uint8_t)(v < 128 ? (s > 255 ? 255 : s) : v);
    }
    case SGB_IN_OP_BRIGHTNESS:
      return blend(0, v, (float)arg_f64(args, 0));
    case SGB_IN_OP_CONTRAST:
      return blend(mean, v, (float)arg_f64(args, 0));
    default:
      return (uint8_t)v;
  }
}

// ImageEnhance.Contrast's grey level: int(sum / count + 0.5) of the L image
SGB_HD int contrast_mean(int64_t sum, int64_t count) { return (int)dadd(ddiv((double)sum, (double)count), 0.5); }

// ImageOps.autocontrast (cutoff 0) of one channel's histogram
SGB_HD void autocontrast_lut(const int32_t* h, uint8_t* lut) {
  int lo = 0, hi = 255;
  while (lo < 255 && !h[lo]) ++lo;
  while (hi > 0 && !h[hi]) --hi;
  if (hi <= lo) {
    for (int i = 0; i < 256; ++i) lut[i] = (uint8_t)i;
    return;
  }
  const double scale = ddiv(255.0, (double)(hi - lo));
  const double offset = dmul((double)-lo, scale);
  for (int i = 0; i < 256; ++i) {
    const int v = (int)dadd(dmul((double)i, scale), offset);
    lut[i] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
  }
}

// ImageOps.equalize of one channel's histogram (point() clips the table to [0, 255])
SGB_HD void equalize_lut(const int32_t* h, uint8_t* lut) {
  int64_t total = 0;
  int used = 0, last = 0;
  for (int i = 0; i < 256; ++i)
    if (h[i]) total += h[i], ++used, last = h[i];
  const int64_t step = used <= 1 ? 0 : (total - last) / 255;
  if (step == 0) {
    for (int i = 0; i < 256; ++i) lut[i] = (uint8_t)i;
    return;
  }
  int64_t n = step / 2;
  for (int i = 0; i < 256; ++i) {
    const int64_t v = n / step;
    lut[i] = (uint8_t)(v > 255 ? 255 : v);
    n += h[i];
  }
}

// Image.transform(AFFINE, BILINEAR) of one channel plane (S x S, dense) at output pixel (x, y); m: Pillow's inverse matrix
SGB_HD uint8_t affine_sample(const uint8_t* plane, int S, const double* m, int fill, int x, int y) {
  const double xo = dadd((double)x, 0.5), yo = dadd((double)y, 0.5);
  double xin = dadd(dadd(dmul(m[0], xo), dmul(m[1], yo)), m[2]);
  double yin = dadd(dadd(dmul(m[3], xo), dmul(m[4], yo)), m[5]);
  if (xin < 0.0 || xin >= (double)S || yin < 0.0 || yin >= (double)S) return (uint8_t)fill;
  xin = dadd(xin, -0.5);
  yin = dadd(yin, -0.5);
  const int xi = xin < 0.0 ? (int)floor(xin) : (int)xin;
  const int yi = yin < 0.0 ? (int)floor(yin) : (int)yin;
  const double dx = dadd(xin, -(double)xi), dy = dadd(yin, -(double)yi);
  const int x0 = xi < 0 ? 0 : (xi < S ? xi : S - 1);
  const int x1 = xi + 1 < 0 ? 0 : (xi + 1 < S ? xi + 1 : S - 1);
  const int y0 = yi < 0 ? 0 : (yi < S ? yi : S - 1);
  const uint8_t* r0 = plane + (int64_t)y0 * S;
  const double v1 = dadd((double)r0[x0], dmul((double)(r0[x1] - r0[x0]), dx));
  double v2 = v1;
  if (yi + 1 >= 0 && yi + 1 < S) {
    const uint8_t* r1 = plane + (int64_t)(yi + 1) * S;
    v2 = dadd((double)r1[x0], dmul((double)(r1[x1] - r1[x0]), dx));
  }
  return (uint8_t)dadd(v1, dmul(dadd(v2, -v1), dy));
}

// ImageFilter.SMOOTH of one channel plane at (x, y): the border keeps its value
SGB_HD uint8_t smooth(const uint8_t* plane, int S, int x, int y) {
  const uint8_t* r = plane + (int64_t)y * S;
  if (x == 0 || y == 0 || x == S - 1 || y == S - 1) return r[x];
  const float k1 = fdiv(1.f, 13.f), k5 = fdiv(5.f, 13.f);
  float s = 0.5f;
  const uint8_t* rows[3] = {r + S, r, r - S};  // Pillow sums the row below first
  for (int i = 0; i < 3; ++i) {
    const uint8_t* q = rows[i];
    const float kc = i == 1 ? k5 : k1;
    s = fadd(s, fadd(fadd(fmul((float)q[x - 1], k1), fmul((float)q[x], kc)), fmul((float)q[x + 1], k1)));
  }
  if (s <= 0.f) return 0;
  if (s >= 255.f) return 255;
  return (uint8_t)s;
}

// ToTensor + Normalize of one channel value
SGB_HD float normalize(int u, float mean, float std) { return fdiv(fadd(fdiv((float)u, 255.f), -mean), std); }

// CollateMixup batch mode: mixed = x_i * lam + x_j * (1 - lam), added to a zero output
SGB_HD float mix(float xi, float xj, float lam, float one_minus_lam) { return fadd(0.f, fadd(fmul(xi, lam), fmul(xj, one_minus_lam))); }

}  // namespace sgb_in

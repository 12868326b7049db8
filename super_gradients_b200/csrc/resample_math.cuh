// Arithmetic of the ImageNet predict() pre-processing (row (f)-N3, classification chain), host+device like preprocess_math.cuh:
// the CUDA kernel in resample.cu calls these functions and the CPU suite compiles this header with g++ to check it, bit for bit,
// against Pillow and the reference's pipeline.
//
// Reference chain (src/super_gradients/training/processing/processing.py:1142-1151): Resize(256) (:614-644, through
// _rescale_image_with_pil = PIL.Image.resize(..., BILINEAR), transforms/utils.py:28-42) -> CenterCrop(224) (:647-680) ->
// StandardizeImage -> NormalizeImage -> ImagePermute.
//
// Pillow's 8-bit resample (libImaging/Resample.c) is integer arithmetic on coefficients computed in double.  Per axis, for output
// index xx of an in -> out resize:
//   scale = in / out;  fs = max(scale, 1);  support = fs;  ss = 1 / fs;  center = (xx + 0.5) * scale
//   xmin = max((int)(center - support + 0.5), 0);  n = min((int)(center + support + 0.5), in) - xmin
//   w[x] = tri((x + xmin - center + 0.5) * ss), tri(t) = max(0, 1 - |t|);  w[x] /= sum(w)   (double)
//   k[x] = (int)(0.5 + w[x] * 2^22)   (22-bit fixed point; the weights are never negative)
// The horizontal pass runs first and stores uint8: clip8((2^21 + sum src * k) >> 22); the vertical pass runs on that uint8
// intermediate with the same rounding.  An axis whose size does not change gets the one-tap weight 2^22, which reproduces
// Pillow's skipped pass exactly ((v << 22) + 2^21) >> 22 == v).
//
// The double arithmetic goes through explicitly rounded intrinsics on the device: nvcc contracts a * b + c into an FMA by default,
// g++ does not, and one contracted rounding moves a coefficient by one fixed-point unit.
#pragma once
#include <math.h>
#include <stdint.h>

#include "sgb200.h"

#ifndef SGB_HD
#ifdef __CUDACC__
#define SGB_HD __host__ __device__ __forceinline__
#else
#define SGB_HD static inline
#endif
#endif

namespace sgb_rs {

constexpr int kPrecisionBits = 22;

SGB_HD double dadd(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
SGB_HD double dmul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
SGB_HD double ddiv(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}

struct Axis {
  double scale, support, ss;
};

SGB_HD Axis axis(int in, int out) {
  Axis a;
  a.scale = ddiv((double)in, (double)out);
  const double fs = a.scale < 1.0 ? 1.0 : a.scale;
  a.support = fs;  // the bilinear filter's support is 1
  a.ss = ddiv(1.0, fs);
  return a;
}

// most taps any output index of an in -> out resize can have (Pillow's ksize)
SGB_HD int max_taps(int in, int out) { return (int)ceil(axis(in, out).support) * 2 + 1; }

// first source index and tap count of output index xx
SGB_HD void bounds(const Axis& a, int xx, int in, int& xmin, int& n) {
  const double center = dmul((double)xx + 0.5, a.scale);
  xmin = (int)dadd(dadd(center, -a.support), 0.5);
  if (xmin < 0) xmin = 0;
  int xmax = (int)dadd(dadd(center, a.support), 0.5);
  if (xmax > in) xmax = in;
  n = xmax - xmin;
}

SGB_HD double tri_weight(const Axis& a, int x, int xmin, double center) {
  double t = dmul(dadd(dadd((double)(x + xmin), -center), 0.5), a.ss);
  if (t < 0.0) t = -t;
  return t < 1.0 ? dadd(1.0, -t) : 0.0;
}

// fixed-point weights of output index xx into k[0..n); returns n, and the first source index in xmin
SGB_HD int coeffs(const Axis& a, int xx, int in, int32_t* k, int& xmin) {
  int n;
  bounds(a, xx, in, xmin, n);
  const double center = dmul((double)xx + 0.5, a.scale);
  double ww = 0.0;
  for (int x = 0; x < n; ++x) ww = dadd(ww, tri_weight(a, x, xmin, center));
  for (int x = 0; x < n; ++x) {
    double w = tri_weight(a, x, xmin, center);
    if (ww != 0.0) w = ddiv(w, ww);
    k[x] = (int32_t)dadd(0.5, dmul(w, (double)(1 << kPrecisionBits)));
  }
  return n;
}

SGB_HD uint8_t clip8(int32_t acc) {
  const int32_t v = acc >> kPrecisionBits;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// source rows the vertical pass of output rows [y0, y1] (resized-image coordinates) reads: [first, first + count)
SGB_HD void row_span(int in_h, int out_h, int y0, int y1, int& first, int& count) {
  const Axis a = axis(in_h, out_h);
  int m0, n0, m1, n1;
  bounds(a, y0, in_h, m0, n0);
  bounds(a, y1, in_h, m1, n1);  // both ends are non-decreasing in the output index
  first = m0;
  count = m1 + n1 - m0;
}

}  // namespace sgb_rs

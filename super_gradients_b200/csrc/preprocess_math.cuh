// Arithmetic of the fused predict() pre-processing (row (f)-N3), host+device like pose_loss_math.cuh: the CUDA kernel in
// preprocess.cu calls sample_pixel() per output element and the CPU suite compiles this header with g++ to check it, bit for
// bit, against OpenCV and the reference's numpy pipeline.
//
// Reference chain (src/super_gradients/training/processing/processing.py): [ReverseImageChannels :232-257] ->
// DetectionLongestMaxSizeRescale / DetectionRescale (:516-590; cv2.resize(..., INTER_LINEAR) on uint8 via
// transforms/utils.py:17-25) -> Detection{Center,BottomRight}Padding (:383-440, _pad_image utils.py:109-150) ->
// StandardizeImage (:260-295: (image / max_value).astype(float32)) -> [NormalizeImage :298-330] -> ImagePermute.
//
// cv2.resize INTER_LINEAR on 8-bit images is fixed point (OpenCV 4.x modules/imgproc/src/resize.cpp): per axis
//   f = (float)((d + 0.5) * (src / dst) - 0.5);  s = floor(f);  f -= s;          (x only: s < 0 -> s = 0, f = 0;  s >= src-1 -> s = src-1, f = 0)
//   coefficients c0 = round_half_even((1 - f) * 2048), c1 = round_half_even(f * 2048)  (shorts)
//   horizontal: D = S[s] * a0 + S[s + 1] * a1 (int);  vertical (rows clipped to [0, src-1]):
//   out = (((b0 * (D0 >> 4)) >> 16) + ((b1 * (D1 >> 4)) >> 16) + 2) >> 2
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

namespace sgb_prep {

struct Coef {
  int s;       // first source index
  int c0, c1;  // 11-bit fixed-point weights of s and s + 1
};

SGB_HD Coef resize_coef(int d, int dst, int src, bool clamp) {
  const double scale = (double)src / (double)dst;
  float f = (float)(((double)d + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f -= (float)s;
  if (clamp) {
    if (s < 0) {
      s = 0;
      f = 0.f;
    }
    if (s >= src - 1) {
      s = src - 1;
      f = 0.f;
    }
  }
  Coef c;
  c.s = s;
  c.c0 = (int)rintf((1.f - f) * 2048.f);
  c.c1 = (int)rintf(f * 2048.f);
  return c;
}

// channel c of pixel (y, x) of the dst_h x dst_w INTER_LINEAR resize of an H x W x C uint8 image (row pitch in bytes)
SGB_HD int resized_u8(const uint8_t* img, int H, int W, int C, int pitch, int dst_h, int dst_w, int y, int x, int c) {
  if (dst_h == H && dst_w == W) return img[(int64_t)y * pitch + x * C + c];
  const Coef cx = resize_coef(x, dst_w, W, true), cy = resize_coef(y, dst_h, H, false);
  const int x0 = cx.s, x1 = cx.s + 1 < W ? cx.s + 1 : W - 1;  // c1 == 0 whenever s + 1 would leave the row
  int y0 = cy.s < 0 ? 0 : (cy.s > H - 1 ? H - 1 : cy.s);
  int y1 = cy.s + 1 < 0 ? 0 : (cy.s + 1 > H - 1 ? H - 1 : cy.s + 1);
  const uint8_t* r0 = img + (int64_t)y0 * pitch;
  const uint8_t* r1 = img + (int64_t)y1 * pitch;
  const int d0 = (int)r0[x0 * C + c] * cx.c0 + (int)r0[x1 * C + c] * cx.c1;
  const int d1 = (int)r1[x0 * C + c] * cx.c0 + (int)r1[x1 * C + c] * cx.c1;
  return (((cy.c0 * (d0 >> 4)) >> 16) + ((cy.c1 * (d1 >> 4)) >> 16) + 2) >> 2;
}

// StandardizeImage (max_value > 0) then NormalizeImage (normalize != 0) of one value of output channel c, in fp32
SGB_HD float standardize(float v, double max_value, int normalize, float mean, float std) {
  if (max_value > 0.0) v = (float)((double)v / max_value);  // numpy divides the uint8 image by a Python float (float64), then casts
  if (normalize) v = (v - mean) / std;                      // float32 arrays in the reference
  return v;
}

// value of output channel c at canvas position (oy, ox): resize -> pad -> [reverse] -> standardize -> [normalize], in fp32
SGB_HD float sample_pixel(const SgbPreprocDesc& d, const uint8_t* src, int oy, int ox, int c) {
  const int sc = d.reverse_channels ? d.src_c - 1 - c : c;
  const int y = oy - d.pad_top, x = ox - d.pad_left;
  float v;
  if (y >= 0 && y < d.dst_h && x >= 0 && x < d.dst_w) v = (float)resized_u8(src, d.src_h, d.src_w, d.src_c, d.src_pitch, d.dst_h, d.dst_w, y, x, sc);
  else v = d.pad_value;
  return standardize(v, d.max_value, d.normalize, d.mean[c], d.std[c]);
}

}  // namespace sgb_prep

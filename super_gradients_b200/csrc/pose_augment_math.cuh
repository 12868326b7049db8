// Arithmetic of the pose train augmentation (pose_augment.cu), host+device like augment_math.cuh: the kernels call
// point_pixel() / out_pixel() and the CPU suite compiles this header with g++ to check it, bit for bit, against cv2 4.x and the
// reference's numpy chain (transforms/keypoints/*.py: KeypointsRandomHorizontalFlip, KeypointsBrightnessContrast,
// KeypointsReverseImageChannels, KeypointsHSV, KeypointsRandomRotate90, KeypointsRandomAffineTransform, KeypointsMosaic,
// KeypointsLongestMaxSize, KeypointsPadIfNeeded).
//
// Pass 1 (point_pixel): per sub-sample (the sample itself, or one of the four mosaic tiles), the pointwise steps on the source
//   image, written rotated into a uint8 workspace: flip -> brightness-contrast -> channel reversal -> augment_hsv -> np.rot90.
// Pass 2 (out_pixel): per output pixel, pad -> LongestMaxSize resize (INTER_LINEAR) -> mosaic canvas -> cv2.warpAffine of the
//   tile's workspace image (any of cv2's five interpolation flags) -> the value KeypointsImageStandardize divides.
//
// KeypointsBrightnessContrast: numpy evaluates (x - m) * c + m * b in float32 (c and b are Python floats, cast to float32), clips to
//   [0, 255] and truncates.  The channel means m are np.mean(float32 image, axis=(0, 1)), a sequential float32 sum whose value
//   depends on the pixel order, so the host computes them with the reference's expression and they travel as float32 bits.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "augment_math.cuh"
#include "preprocess_math.cuh"
#include "sgb200.h"

namespace sgb_pose {

#ifdef __CUDA_ARCH__
SGB_HD float fadd(float a, float b) { return __fadd_rn(a, b); }
#else
SGB_HD float fadd(float a, float b) { return a + b; }
#endif

SGB_HD float bits_f32(int64_t v) {
  const uint32_t u = (uint32_t)v;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

SGB_HD int unpack(int64_t packed, int c) { return (int)((packed >> (8 * c)) & 255); }

// uint8 pixel (y, x) of sub-sample s (SGB_POSE_SUB_* fields) after flip -> brightness-contrast -> reversal -> HSV -> rot90
SGB_HD void point_pixel(const uint8_t* src, const int64_t* s, int block, int y, int x, int p[3]) {
  const int H = (int)s[SGB_POSE_S_H], W = (int)s[SGB_POSE_S_W];
  int sy, sx;  // np.rot90(image, k)[y, x]
  switch ((int)s[SGB_POSE_S_ROT]) {
    case 1: sy = x, sx = W - 1 - y; break;
    case 2: sy = H - 1 - y, sx = W - 1 - x; break;
    case 3: sy = H - 1 - x, sx = y; break;
    default: sy = y, sx = x; break;
  }
  const int cx = s[SGB_POSE_S_FLIP] ? W - 1 - sx : sx;
  const uint8_t* q = src + s[SGB_POSE_S_OFFSET] + ((int64_t)sy * W + cx) * 3;
  for (int c = 0; c < 3; ++c) p[c] = q[c];
  if (s[SGB_POSE_S_BC]) {
    const float cg = bits_f32(s[SGB_POSE_S_CONTRAST]), bg = bits_f32(s[SGB_POSE_S_BRIGHTNESS]);
    for (int c = 0; c < 3; ++c) {
      const float m = bits_f32(s[SGB_POSE_S_MEAN + c]);
      float v = fadd(sgb_aug::fmul(sgb_aug::fsub((float)p[c], m), cg), sgb_aug::fmul(m, bg));
      v = v < 0.f ? 0.f : (v > 255.f ? 255.f : v);
      p[c] = (int)v;
    }
  }
  if (s[SGB_POSE_S_REVERSE]) {
    const int t = p[0];
    p[0] = p[2], p[2] = t;
  }
  if (s[SGB_POSE_S_HSV]) {
    const int bgr[3] = {0, 1, 2};
    sgb_aug::augment_hsv(p, (int)s[SGB_POSE_S_DH], (int)s[SGB_POSE_S_DS], (int)s[SGB_POSE_S_DV], bgr, sx, W, block);
  }
}

SGB_HD sgb_aug::Inverse sub_inverse(const int64_t* s) {
  double m[6];
  for (int i = 0; i < 6; ++i) {
    const int64_t bits = s[SGB_POSE_S_M + i];
    memcpy(&m[i], &bits, 8);
  }
  return sgb_aug::invert(m);
}

// uint8 pixel (y, x) of the mosaic canvas (or of the single tile): the warped tile covering it, else the mosaic pad value
SGB_HD void canvas_pixel(const uint8_t* ws, const int64_t* t, const sgb_aug::Inverse* inv, const sgb_aug::RemapTabs& tabs, int y, int x, int p[3]) {
  const int n = (int)t[SGB_POSE_NSUB];
  for (int i = 0; i < n; ++i) {
    const int64_t* s = t + SGB_POSE_SUB + i * SGB_POSE_SUB_FIELDS;
    const int yy = y - (int)s[SGB_POSE_S_Y], xx = x - (int)s[SGB_POSE_S_X], rh = (int)s[SGB_POSE_S_RH], rw = (int)s[SGB_POSE_S_RW];
    if (yy < 0 || yy >= rh || xx < 0 || xx >= rw) continue;
    const uint8_t* img = ws + s[SGB_POSE_S_WS_OFFSET];
    if (s[SGB_POSE_S_AFFINE]) {
      const int border[3] = {unpack(s[SGB_POSE_S_BORDER], 0), unpack(s[SGB_POSE_S_BORDER], 1), unpack(s[SGB_POSE_S_BORDER], 2)};
      sgb_aug::warp_pixel_mode(img, rh, rw, inv[i], (int)s[SGB_POSE_S_MODE], border, tabs, yy, xx, p);
    } else {
      for (int c = 0; c < 3; ++c) p[c] = img[((int64_t)yy * rw + xx) * 3 + c];
    }
    return;
  }
  for (int c = 0; c < 3; ++c) p[c] = unpack(t[SGB_POSE_MOSAIC_PAD], c);
}

// uint8 pixel (oy, ox) of the padded output: the canvas resized to (RS_H, RS_W) at (PAD_TOP, PAD_LEFT) on the pad value
SGB_HD void out_pixel(const uint8_t* ws, const int64_t* t, const sgb_aug::Inverse* inv, const sgb_aug::RemapTabs& tabs, int oy, int ox, int p[3]) {
  const int y = oy - (int)t[SGB_POSE_PAD_TOP], x = ox - (int)t[SGB_POSE_PAD_LEFT];
  const int rh = (int)t[SGB_POSE_RS_H], rw = (int)t[SGB_POSE_RS_W], ch = (int)t[SGB_POSE_CANVAS_H], cw = (int)t[SGB_POSE_CANVAS_W];
  if (y < 0 || y >= rh || x < 0 || x >= rw) {
    for (int c = 0; c < 3; ++c) p[c] = unpack(t[SGB_POSE_PAD_VALUE], c);
    return;
  }
  if (rh == ch && rw == cw) {
    canvas_pixel(ws, t, inv, tabs, y, x, p);
    return;
  }
  const sgb_prep::Taps k = sgb_prep::resize_taps(ch, cw, rh, rw, y, x);
  int q[4][3];
  canvas_pixel(ws, t, inv, tabs, k.y0, k.x0, q[0]);
  canvas_pixel(ws, t, inv, tabs, k.y0, k.x1, q[1]);
  canvas_pixel(ws, t, inv, tabs, k.y1, k.x0, q[2]);
  canvas_pixel(ws, t, inv, tabs, k.y1, k.x1, q[3]);
  for (int c = 0; c < 3; ++c) p[c] = sgb_prep::resize_combine(k, q[0][c], q[1][c], q[2][c], q[3][c]);
}

// host only (a CUDA translation unit compiles these for the host side)
// cv2's interpolateCubic / interpolateLanczos4 (imgwarp.cpp) in float, as initInterTab1D calls them
inline void interpolate_cubic(float x, float* c) {
  const float A = -0.75f;
  c[0] = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A;
  c[1] = ((A + 2) * x - (A + 3)) * x * x + 1;
  c[2] = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1;
  c[3] = 1.f - c[0] - c[1] - c[2];
}

inline void interpolate_lanczos4(float x, float* c) {
  const double s45 = 0.70710678118654752440084436210485, pi = 3.1415926535897932384626433832795;
  const double cs[8][2] = {{1, 0}, {-s45, -s45}, {0, 1}, {s45, -s45}, {-1, 0}, {s45, s45}, {0, -1}, {-s45, s45}};
  float sum = 0;
  const double y0 = -(x + 3) * pi * 0.25, s0 = sin(y0), c0 = cos(y0);
  for (int i = 0; i < 8; ++i) {
    const float y0_ = (x + 3 - i);
    if (fabsf(y0_) >= 1e-6f) {
      const double y = -y0_ * pi * 0.25;
      c[i] = (float)((cs[i][0] * s0 + cs[i][1] * c0) / (y * y));
    } else {
      c[i] = 1e30f;
    }
    sum += c[i];
  }
  sum = 1.f / sum;
  for (int i = 0; i < 8; ++i) c[i] *= sum;
}

// initInterTab2D's fixed-point table of one method (ksize 4: cubic, 8: Lanczos4): [32 * 32 phases][ksize * ksize], each phase's
// rounded products corrected to sum to 2^15 on the largest (or smallest) of the taps [ksize/2, ksize/2 + 2)^2
inline void remap_table(int ksize, int16_t* itab) {
  float tab[32 * 8];
  for (int i = 0; i < 32; ++i) {
    if (ksize == 4) interpolate_cubic(i * (1.f / 32), tab + i * 4);
    else interpolate_lanczos4(i * (1.f / 32), tab + i * 8);
  }
  for (int i = 0; i < 32; ++i)
    for (int j = 0; j < 32; ++j, itab += ksize * ksize) {
      int isum = 0;
      for (int k1 = 0; k1 < ksize; ++k1) {
        const float vy = tab[i * ksize + k1];
        for (int k2 = 0; k2 < ksize; ++k2) {
          const float v = vy * tab[j * ksize + k2];
          long r = lrintf(v * 32768.f);
          r = r < -32768 ? -32768 : (r > 32767 ? 32767 : r);
          isum += itab[k1 * ksize + k2] = (int16_t)r;
        }
      }
      if (isum != 32768) {
        const int diff = isum - 32768, k2h = ksize / 2;
        int Mk1 = k2h, Mk2 = k2h, mk1 = k2h, mk2 = k2h;
        for (int k1 = k2h; k1 < k2h + 2; ++k1)
          for (int k2 = k2h; k2 < k2h + 2; ++k2) {
            if (itab[k1 * ksize + k2] < itab[mk1 * ksize + mk2]) mk1 = k1, mk2 = k2;
            else if (itab[k1 * ksize + k2] > itab[Mk1 * ksize + Mk2]) Mk1 = k1, Mk2 = k2;
          }
        if (diff < 0) itab[Mk1 * ksize + Mk2] = (int16_t)(itab[Mk1 * ksize + Mk2] - diff);
        else itab[mk1 * ksize + mk2] = (int16_t)(itab[mk1 * ksize + mk2] - diff);
      }
    }
}

}  // namespace sgb_pose

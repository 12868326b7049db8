// Arithmetic of the detection train augmentation (augment.cu), host+device like preprocess_math.cuh: the kernel calls
// augment_pixel() per output pixel and the CPU suite compiles this header with g++ to check it, bit for bit, against cv2 4.x and
// the reference's numpy chain (transforms.py DetectionMosaic :536-588, random_affine :1464-1534, augment_hsv :1623-1634,
// DetectionMixup :729-797, _rescale_and_pad_to_size utils.py:203-226).
//
// cv2.warpAffine, uint8, INTER_LINEAR, BORDER_CONSTANT (imgproc/src/imgwarp.cpp): M is inverted in double, then per output row
//   X0 = rint((A12 * y + b1) * 1024) + 16, per column adelta = rint(A11 * x * 1024), X = (X0 + adelta) >> 5 (Y likewise);
//   source pixel (X >> 5, Y >> 5), sub-pixel (X & 31, Y & 31); weights (32 - fx | fx) x (32 - fy | fy) x 32 sum to 32768 exactly;
//   taps outside the image read the border value; out = (sum + 2^14) >> 15.
// cv2.cvtColor BGR2HSV (8-bit, hsv_shift 12): integer tables sdiv / hdiv, identical on the vector and the scalar path.
// cv2.cvtColor HSV2BGR (8-bit): float32 h * (6 / 180), s / 255, v / 255, tab2 = v * fma(-s, f, 1), tab3 = v * fma(-s, 1 - f, 1),
//   times 255, then TRUNCATED on the vector path and rounded half-even on the scalar tail of each row.  Which path a pixel takes
//   depends only on its column: x < w - w % block is vectorised (block = 32 pixels in the x86 builds of cv2 4.x).
#pragma once
#include <math.h>
#include <stdint.h>

#include "preprocess_math.cuh"
#include "sgb200.h"

namespace sgb_aug {

#ifdef __CUDA_ARCH__
SGB_HD double dmul(double a, double b) { return __dmul_rn(a, b); }
SGB_HD double dadd(double a, double b) { return __dadd_rn(a, b); }
SGB_HD float fmul(float a, float b) { return __fmul_rn(a, b); }
SGB_HD float fsub(float a, float b) { return __fsub_rn(a, b); }
#else
SGB_HD double dmul(double a, double b) { return a * b; }
SGB_HD double dadd(double a, double b) { return a + b; }
SGB_HD float fmul(float a, float b) { return a * b; }
SGB_HD float fsub(float a, float b) { return a - b; }
#endif

struct Inverse {
  double a11, a12, b1, a21, a22, b2;
};

// cv2's inversion of the forward matrix m[6] (row major); det == 0 is refused by the caller
SGB_HD Inverse invert(const double* m) {
  double D = dadd(dmul(m[0], m[4]), -dmul(m[1], m[3]));
  D = 1.0 / D;
  Inverse r;
  r.a11 = dmul(m[4], D);
  r.a22 = dmul(m[0], D);
  r.a12 = dmul(m[1], -D);
  r.a21 = dmul(m[3], -D);
  r.b1 = dadd(-dmul(r.a11, m[2]), -dmul(r.a12, m[5]));
  r.b2 = dadd(-dmul(r.a21, m[2]), -dmul(r.a22, m[5]));
  return r;
}

// fixed-point source coordinate (<< 5) of output pixel (y, x)
SGB_HD void warp_coord(const Inverse& a, int y, int x, int& X, int& Y) {
  const int X0 = (int)rint(dmul(dadd(dmul(a.a12, (double)y), a.b1), 1024.0)) + 16;
  const int Y0 = (int)rint(dmul(dadd(dmul(a.a22, (double)y), a.b2), 1024.0)) + 16;
  X = (X0 + (int)rint(dmul(dmul(a.a11, (double)x), 1024.0))) >> 5;
  Y = (Y0 + (int)rint(dmul(dmul(a.a21, (double)x), 1024.0))) >> 5;
}

// cv2's INTER_REMAP_COEF_BITS = 15 coefficient tables of INTER_CUBIC (4 x 4 taps) and INTER_LANCZOS4 (8 x 8 taps) per sub-pixel
// phase (fy * 32 + fx), row-major taps: the fixed-point `itab` of initInterTab2D (imgwarp.cpp).  Filled once on the host.
struct RemapTabs {
  const int16_t* cubic;    // [1024][16]
  const int16_t* lanczos;  // [1024][64]
};

// DetectionMosaic's canvas pixel (y, x) of table row t (its tiles in src) into q[3].  The tiles do not overlap and tile i lies in
// quadrant i of (xc, yc), so only that tile can hold the pixel.  Inside its rectangle the value is cv2.resize (INTER_LINEAR) of the
// tile's source to (rh, rw) at the pixel shifted by the placement; outside, the mosaic border value.
SGB_HD void mosaic_pixel(const uint8_t* src, const int64_t* t, int y, int x, int q[3]) {
  const int i = (y >= (int)t[SGB_AUG_MOS_YC] ? 2 : 0) + (x >= (int)t[SGB_AUG_MOS_XC] ? 1 : 0);
  const int64_t* k = t + SGB_AUG_MOS_TILE + i * SGB_AUG_MOS_TILE_FIELDS;
  if (y < (int)k[SGB_AUG_T_Y1] || y >= (int)k[SGB_AUG_T_Y2] || x < (int)k[SGB_AUG_T_X1] || x >= (int)k[SGB_AUG_T_X2]) {
    q[0] = q[1] = q[2] = (int)t[SGB_AUG_MOS_BORDER];
    return;
  }
  const int H = (int)k[SGB_AUG_T_H], W = (int)k[SGB_AUG_T_W], rh = (int)k[SGB_AUG_T_RH], rw = (int)k[SGB_AUG_T_RW];
  const int ry = y - (int)k[SGB_AUG_T_Y1] + (int)k[SGB_AUG_T_SY], rx = x - (int)k[SGB_AUG_T_X1] + (int)k[SGB_AUG_T_SX];
  const uint8_t* img = src + k[SGB_AUG_T_OFFSET];
  if (rh == H && rw == W) {
    for (int c = 0; c < 3; ++c) q[c] = img[((int64_t)ry * W + rx) * 3 + c];
    return;
  }
  const sgb_prep::Taps r = sgb_prep::resize_taps(H, W, rh, rw, ry, rx);
  const uint8_t* r0 = img + (int64_t)r.y0 * W * 3;
  const uint8_t* r1 = img + (int64_t)r.y1 * W * 3;
  for (int c = 0; c < 3; ++c) q[c] = sgb_prep::resize_combine(r, r0[r.x0 * 3 + c], r0[r.x1 * 3 + c], r1[r.x0 * 3 + c], r1[r.x1 * 3 + c]);
}

// cv2.warpAffine INTER_LINEAR pixel (y, x) of the mosaic canvas (MOS_CANVAS_H x MOS_CANVAS_W) into p[3]: warp_pixel's four taps,
// each a mosaic_pixel, the taps outside the canvas reading border
SGB_HD void warp_mosaic_pixel(const uint8_t* src, const int64_t* t, const Inverse& a, int border, int y, int x, int p[3]) {
  const int H = (int)t[SGB_AUG_MOS_CANVAS_H], W = (int)t[SGB_AUG_MOS_CANVAS_W];
  int X, Y;
  warp_coord(a, y, x, X, Y);
  const int fx = X & 31, fy = Y & 31, sx = X >> 5, sy = Y >> 5;
  const int w[4] = {(32 - fy) * (32 - fx) * 32, (32 - fy) * fx * 32, fy * (32 - fx) * 32, fy * fx * 32};
  int acc[3] = {0, 0, 0};
  for (int k = 0; k < 4; ++k) {
    const int ty = sy + (k >> 1), tx = sx + (k & 1);
    int q[3] = {border, border, border};
    if (ty >= 0 && ty < H && tx >= 0 && tx < W) mosaic_pixel(src, t, ty, tx, q);
    for (int c = 0; c < 3; ++c) acc[c] += q[c] * w[k];
  }
  for (int c = 0; c < 3; ++c) {
    const int v = (acc[c] + (1 << 14)) >> 15;
    p[c] = v < 0 ? 0 : (v > 255 ? 255 : v);
  }
}

// cv2.warpAffine pixel (y, x) of an H x W x 3 image (dense rows) into p[3], BORDER_CONSTANT with border[3].  mode: cv2's
// interpolation flag, 0 INTER_NEAREST, 1 INTER_LINEAR, 2 INTER_CUBIC, 3 INTER_AREA (warpAffine runs it as INTER_LINEAR),
// 4 INTER_LANCZOS4.  Nearest rounds the coordinate (+ 2^9, >> 10) and reads one pixel or the border; the others take the 1/32
// sub-pixel phase and sum ksize x ksize taps from (X >> 5) - (ksize / 2 - 1), reading the border outside the image, as
// (sum + 2^14) >> 15 saturated to uint8.  tabs is only read by modes 2 and 4.
SGB_HD void warp_pixel_mode(const uint8_t* img, int H, int W, const Inverse& a, int mode, const int border[3], const RemapTabs& tabs, int y, int x,
                            int p[3]) {
  if (mode == 0) {
    const int X0 = (int)rint(dmul(dadd(dmul(a.a12, (double)y), a.b1), 1024.0)) + 512;
    const int Y0 = (int)rint(dmul(dadd(dmul(a.a22, (double)y), a.b2), 1024.0)) + 512;
    const int sx = (X0 + (int)rint(dmul(dmul(a.a11, (double)x), 1024.0))) >> 10;
    const int sy = (Y0 + (int)rint(dmul(dmul(a.a21, (double)x), 1024.0))) >> 10;
    const bool in = sy >= 0 && sy < H && sx >= 0 && sx < W;
    for (int c = 0; c < 3; ++c) p[c] = in ? (int)img[((int64_t)sy * W + sx) * 3 + c] : border[c];
    return;
  }
  int X, Y;
  warp_coord(a, y, x, X, Y);
  const int fx = X & 31, fy = Y & 31;
  int acc[3] = {0, 0, 0};
  if (mode == 2 || mode == 4) {
    const int k = mode == 2 ? 4 : 8;
    const int sx = (X >> 5) - (k / 2 - 1), sy = (Y >> 5) - (k / 2 - 1);
    const int16_t* w = (mode == 2 ? tabs.cubic + (fy * 32 + fx) * 16 : tabs.lanczos + (fy * 32 + fx) * 64);
    for (int i = 0; i < k; ++i) {
      const int ty = sy + i;
      const bool row_in = ty >= 0 && ty < H;
      const uint8_t* row = img + (int64_t)(row_in ? ty : 0) * W * 3;
      for (int j = 0; j < k; ++j) {
        const int tx = sx + j, wk = w[i * k + j];
        const bool in = row_in && tx >= 0 && tx < W;
        const uint8_t* s = row + (in ? tx : 0) * 3;
        for (int c = 0; c < 3; ++c) acc[c] += (in ? (int)s[c] : border[c]) * wk;
      }
    }
  } else {
    const int sx = X >> 5, sy = Y >> 5;
    const int w[4] = {(32 - fy) * (32 - fx) * 32, (32 - fy) * fx * 32, fy * (32 - fx) * 32, fy * fx * 32};
    for (int k = 0; k < 4; ++k) {
      const int ty = sy + (k >> 1), tx = sx + (k & 1);
      const bool in = ty >= 0 && ty < H && tx >= 0 && tx < W;
      const uint8_t* s = img + ((int64_t)(in ? ty : 0) * W + (in ? tx : 0)) * 3;
      for (int c = 0; c < 3; ++c) acc[c] += (in ? (int)s[c] : border[c]) * w[k];
    }
  }
  for (int c = 0; c < 3; ++c) {
    const int v = (acc[c] + (1 << 14)) >> 15;
    p[c] = v < 0 ? 0 : (v > 255 ? 255 : v);
  }
}

// cv2.warpAffine INTER_LINEAR pixel (y, x) of an H x W x 3 image (dense rows) into p[3], one border value for every channel
SGB_HD void warp_pixel(const uint8_t* img, int H, int W, const Inverse& a, int border, int y, int x, int p[3]) {
  const int b[3] = {border, border, border};
  warp_pixel_mode(img, H, W, a, 1, b, RemapTabs{nullptr, nullptr}, y, x, p);
}

SGB_HD int sdiv(int i) { return i == 0 ? 0 : (int)rint((double)(255 << 12) / (double)i); }
SGB_HD int hdiv180(int i) { return i == 0 ? 0 : (int)rint((double)(180 << 12) / (6.0 * (double)i)); }

// cv2 COLOR_BGR2HSV of one 8-bit pixel (hue in [0, 180))
SGB_HD void bgr2hsv(int b, int g, int r, int& h, int& s, int& v) {
  v = b > g ? b : g;
  v = v > r ? v : r;
  int vmin = b < g ? b : g;
  vmin = vmin < r ? vmin : r;
  const int diff = v - vmin;
  const int vr = v == r ? -1 : 0, vg = v == g ? -1 : 0;
  s = (diff * sdiv(v) + (1 << 11)) >> 12;
  h = (vr & (g - b)) + (~vr & ((vg & (b - r + 2 * diff)) + ((~vg) & (r - g + 4 * diff))));
  h = (h * hdiv180(diff) + (1 << 11)) >> 12;
  h += h < 0 ? 180 : 0;
}

// cv2 COLOR_HSV2BGR of one 8-bit pixel; vec: the pixel lies in a vectorised block of its row (truncation instead of rounding)
SGB_HD void hsv2bgr(int hi, int si, int vi, bool vec, int& b, int& g, int& r) {
  float h = fmul((float)hi, 6.f / 180.f);
  const float s = fmul((float)si, 1.f / 255.f), v = fmul((float)vi, 1.f / 255.f);
  int sector = (int)h;
  h = fsub(h, (float)sector);
  sector %= 6;
  float tab[4];
  tab[0] = v;
  tab[1] = fmul(v, fsub(1.f, s));
  tab[2] = fmul(v, fmaf(-s, h, 1.f));
  tab[3] = fmul(v, fmaf(-s, fsub(1.f, h), 1.f));
  const int sel[6][3] = {{1, 3, 0}, {1, 0, 2}, {3, 0, 1}, {0, 2, 1}, {0, 1, 3}, {2, 1, 0}};
  int o[3];
  for (int c = 0; c < 3; ++c) {
    const float x = fmul(tab[sel[sector][c]], 255.f);
    const int q = vec ? (int)x : (int)rintf(x);
    o[c] = q < 0 ? 0 : (q > 255 ? 255 : q);
  }
  b = o[0], g = o[1], r = o[2];
}

SGB_HD int clip255(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// augment_hsv on one pixel p[3] at column x of a row of w pixels (bgr: channel indices of B, G, R)
SGB_HD void augment_hsv(int p[3], int dh, int ds, int dv, const int bgr[3], int x, int w, int block) {
  int h, s, v;
  bgr2hsv(p[bgr[0]], p[bgr[1]], p[bgr[2]], h, s, v);
  h = (h + dh) % 180;
  h += h < 0 ? 180 : 0;
  s = clip255(s + ds);
  v = clip255(v + dv);
  int b, g, r;
  hsv2bgr(h, s, v, x < w - w % block, b, g, r);
  p[bgr[0]] = b, p[bgr[1]] = g, p[bgr[2]] = r;
}

// partner image after the optional flip and the first resize, pasted on its border-value canvas: channel c at (y, x)
SGB_HD int mix_canvas1(const uint8_t* mix, const int64_t* t, int y, int x, int c) {
  if (y >= (int)t[SGB_AUG_MIX_R1_H] || x >= (int)t[SGB_AUG_MIX_R1_W]) return (int)t[SGB_AUG_MIX_BORDER];
  const int H = (int)t[SGB_AUG_MIX_H], W = (int)t[SGB_AUG_MIX_W], rh = (int)t[SGB_AUG_MIX_R1_H], rw = (int)t[SGB_AUG_MIX_R1_W];
  const bool flip = t[SGB_AUG_MIX_FLIP] != 0;
  if (rh == H && rw == W) return mix[((int64_t)y * W + (flip ? W - 1 - x : x)) * 3 + c];
  const sgb_prep::Taps k = sgb_prep::resize_taps(H, W, rh, rw, y, x);
  const int x0 = flip ? W - 1 - k.x0 : k.x0, x1 = flip ? W - 1 - k.x1 : k.x1;
  const uint8_t* r0 = mix + (int64_t)k.y0 * W * 3;
  const uint8_t* r1 = mix + (int64_t)k.y1 * W * 3;
  return sgb_prep::resize_combine(k, r0[x0 * 3 + c], r0[x1 * 3 + c], r1[x0 * 3 + c], r1[x1 * 3 + c]);
}

// the mixup partner's cropped canvas at (y, x) of the sample: second resize (jit_factor) of canvas1, on zeros, shifted by the crop
SGB_HD int mix_value(const uint8_t* mix, const int64_t* t, int y, int x, int c) {
  const int py = y + (int)t[SGB_AUG_MIX_Y], px = x + (int)t[SGB_AUG_MIX_X];
  const int rh = (int)t[SGB_AUG_MIX_R2_H], rw = (int)t[SGB_AUG_MIX_R2_W], ch = (int)t[SGB_AUG_MIX_CANVAS_H], cw = (int)t[SGB_AUG_MIX_CANVAS_W];
  if (py >= rh || px >= rw) return 0;
  if (rh == ch && rw == cw) return mix_canvas1(mix, t, py, px, c);
  const sgb_prep::Taps k = sgb_prep::resize_taps(ch, cw, rh, rw, py, px);
  return sgb_prep::resize_combine(k, mix_canvas1(mix, t, k.y0, k.x0, c), mix_canvas1(mix, t, k.y0, k.x1, c), mix_canvas1(mix, t, k.y1, k.x0, c),
                                  mix_canvas1(mix, t, k.y1, k.x1, c));
}

// uint8 pixel (y, x) of the sample after [mosaic] -> affine -> swap -> HSV -> flip -> mixup (the image DetectionPaddedRescale
// receives).  With the mosaic, the affine (or, without it, the chain) reads the canvas instead of the sample's image.  kMosaic ==
// false compiles the mosaic out: the kernel instance for batches without a mosaic sample.
template <bool kMosaic>
SGB_HD void chain_pixel(const uint8_t* src, const int64_t* t, const Inverse& a, int block, int y, int x, int p[3]) {
  const int H = (int)t[SGB_AUG_H], W = (int)t[SGB_AUG_W], aw = (int)t[SGB_AUG_AFF_W];
  const uint8_t* img = src + t[SGB_AUG_OFFSET];
  const int xs = t[SGB_AUG_FLIP] ? aw - 1 - x : x;
  if (kMosaic && t[SGB_AUG_MOS]) {
    if (t[SGB_AUG_AFFINE]) warp_mosaic_pixel(src, t, a, (int)t[SGB_AUG_AFF_BORDER], y, xs, p);
    else mosaic_pixel(src, t, y, xs, p);
  } else if (t[SGB_AUG_AFFINE]) {
    warp_pixel(img, H, W, a, (int)t[SGB_AUG_AFF_BORDER], y, xs, p);
  } else {
    for (int c = 0; c < 3; ++c) p[c] = img[((int64_t)y * W + xs) * 3 + c];
  }
  if (t[SGB_AUG_SWAP]) {
    const int q = p[0];
    p[0] = p[2], p[2] = q;
  }
  if (t[SGB_AUG_HSV]) {
    const int packed = (int)t[SGB_AUG_BGR];
    const int bgr[3] = {packed & 3, (packed >> 2) & 3, (packed >> 4) & 3};
    augment_hsv(p, (int)t[SGB_AUG_DH], (int)t[SGB_AUG_DS], (int)t[SGB_AUG_DV], bgr, xs, aw, block);
  }
  if (t[SGB_AUG_MIX]) {
    const uint8_t* mix = src + t[SGB_AUG_MIX_OFFSET];
    for (int c = 0; c < 3; ++c) p[c] = (p[c] + mix_value(mix, t, y, x, c)) >> 1;
  }
}

// uint8 pixel (oy, ox) of the out_h x out_w padded-rescale canvas: the chain image resized to (RS_H, RS_W) at the top left
// (kMosaic as for chain_pixel; augment_pixel<true> serves every table row)
template <bool kMosaic = true>
SGB_HD void augment_pixel(const uint8_t* src, const int64_t* t, const Inverse& a, int block, int pad_value, int oy, int ox, int p[3]) {
  const int rh = (int)t[SGB_AUG_RS_H], rw = (int)t[SGB_AUG_RS_W], ah = (int)t[SGB_AUG_AFF_H], aw = (int)t[SGB_AUG_AFF_W];
  if (oy >= rh || ox >= rw) {
    p[0] = p[1] = p[2] = pad_value;
    return;
  }
  if (rh == ah && rw == aw) {
    chain_pixel<kMosaic>(src, t, a, block, oy, ox, p);
    return;
  }
  const sgb_prep::Taps k = sgb_prep::resize_taps(ah, aw, rh, rw, oy, ox);
  int q[4][3];
  chain_pixel<kMosaic>(src, t, a, block, k.y0, k.x0, q[0]);
  chain_pixel<kMosaic>(src, t, a, block, k.y0, k.x1, q[1]);
  chain_pixel<kMosaic>(src, t, a, block, k.y1, k.x0, q[2]);
  chain_pixel<kMosaic>(src, t, a, block, k.y1, k.x1, q[3]);
  for (int c = 0; c < 3; ++c) p[c] = sgb_prep::resize_combine(k, q[0][c], q[1][c], q[2][c], q[3][c]);
}

SGB_HD Inverse table_inverse(const int64_t* t) {
  double m[6];
  for (int i = 0; i < 6; ++i) {
    const int64_t bits = t[SGB_AUG_M + i];
    m[i] = *(const double*)&bits;
  }
  return invert(m);
}

}  // namespace sgb_aug

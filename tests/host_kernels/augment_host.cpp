// Serial host drivers around super_gradients_b200/csrc/augment_math.cuh (compiled with g++ by tests/augment_cases.py): the same
// per-pixel functions the CUDA kernel calls, so the CPU suite checks the kernel's arithmetic against cv2 without a GPU.
#include <stdint.h>

#include "augment_math.cuh"

extern "C" {

// cv2.warpAffine(img, m, (ow, oh), INTER_LINEAR, BORDER_CONSTANT, border) of an H x W x 3 image into out[oh][ow][3]
void warp_affine_host(const uint8_t* img, int H, int W, const double* m, int border, int oh, int ow, uint8_t* out) {
  const sgb_aug::Inverse a = sgb_aug::invert(m);
  for (int y = 0; y < oh; ++y)
    for (int x = 0; x < ow; ++x) {
      int p[3];
      sgb_aug::warp_pixel(img, H, W, a, border, y, x, p);
      for (int c = 0; c < 3; ++c) out[((int64_t)y * ow + x) * 3 + c] = (uint8_t)p[c];
    }
}

// BGR2HSV of n pixels
void bgr2hsv_host(const uint8_t* bgr, int64_t n, uint8_t* hsv) {
  for (int64_t i = 0; i < n; ++i) {
    int h, s, v;
    sgb_aug::bgr2hsv(bgr[3 * i], bgr[3 * i + 1], bgr[3 * i + 2], h, s, v);
    hsv[3 * i] = (uint8_t)h, hsv[3 * i + 1] = (uint8_t)s, hsv[3 * i + 2] = (uint8_t)v;
  }
}

// HSV2BGR of n pixels on the vector (vec = 1) or the scalar path
void hsv2bgr_host(const uint8_t* hsv, int64_t n, int vec, uint8_t* bgr) {
  for (int64_t i = 0; i < n; ++i) {
    int b, g, r;
    sgb_aug::hsv2bgr(hsv[3 * i], hsv[3 * i + 1], hsv[3 * i + 2], vec != 0, b, g, r);
    bgr[3 * i] = (uint8_t)b, bgr[3 * i + 1] = (uint8_t)g, bgr[3 * i + 2] = (uint8_t)r;
  }
}

// the kernel's uint8 canvas (before the standardisation) of every image of the batch: out[batch][out_h][out_w][3]
void augment_host(const int64_t* table, const uint8_t* src, int batch, int out_h, int out_w, int pad_value, int block, uint8_t* out) {
  for (int b = 0; b < batch; ++b) {
    const int64_t* t = table + (int64_t)b * SGB_AUG_FIELDS;
    const sgb_aug::Inverse a = sgb_aug::table_inverse(t);
    for (int y = 0; y < out_h; ++y)
      for (int x = 0; x < out_w; ++x) {
        int p[3];
        sgb_aug::augment_pixel(src, t, a, block, pad_value, y, x, p);
        for (int c = 0; c < 3; ++c) out[(((int64_t)b * out_h + y) * out_w + x) * 3 + c] = (uint8_t)p[c];
      }
  }
}
}

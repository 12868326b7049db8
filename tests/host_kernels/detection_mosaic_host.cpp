// Serial host driver around super_gradients_b200/csrc/augment_math.cuh (compiled with g++ by tests/mosaic_cases.py): the mosaic
// canvas exactly as the augmentation kernel reads it, so the CPU suite checks it against the reference's DetectionMosaic image.
#include <stdint.h>

#include "augment_math.cuh"

extern "C" {

// the MOS_CANVAS_H x MOS_CANVAS_W x 3 mosaic canvas of one table row t (its tiles in src) into out
void mosaic_canvas_host(const int64_t* t, const uint8_t* src, uint8_t* out) {
  const int H = (int)t[SGB_AUG_MOS_CANVAS_H], W = (int)t[SGB_AUG_MOS_CANVAS_W];
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      int p[3];
      sgb_aug::mosaic_pixel(src, t, y, x, p);
      for (int c = 0; c < 3; ++c) out[((int64_t)y * W + x) * 3 + c] = (uint8_t)p[c];
    }
}
}

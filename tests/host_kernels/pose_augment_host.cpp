// Serial host drivers around super_gradients_b200/csrc/pose_augment_math.cuh (compiled with g++ by tests/pose_augment_cases.py):
// the same per-pixel functions the two CUDA kernels call, so the CPU suite checks their arithmetic against cv2 without a GPU.
#include <stdint.h>

#include <vector>

#include "pose_augment_math.cuh"

namespace {
struct Tabs {
  std::vector<int16_t> cubic, lanczos;
  Tabs() : cubic(1024 * 16), lanczos(1024 * 64) {
    sgb_pose::remap_table(4, cubic.data());
    sgb_pose::remap_table(8, lanczos.data());
  }
  sgb_aug::RemapTabs view() const { return sgb_aug::RemapTabs{cubic.data(), lanczos.data()}; }
};
const Tabs& tabs() {
  static Tabs t;
  return t;
}
}  // namespace

extern "C" {

// cv2.warpAffine(img, m, (ow, oh), flags=mode, BORDER_CONSTANT, border[3]) of an H x W x 3 image into out[oh][ow][3]
void warp_affine_mode_host(const uint8_t* img, int H, int W, const double* m, int mode, const int* border, int oh, int ow, uint8_t* out) {
  const sgb_aug::Inverse a = sgb_aug::invert(m);
  const sgb_aug::RemapTabs t = tabs().view();
  for (int y = 0; y < oh; ++y)
    for (int x = 0; x < ow; ++x) {
      int p[3];
      sgb_aug::warp_pixel_mode(img, H, W, a, mode, border, t, y, x, p);
      for (int c = 0; c < 3; ++c) out[((int64_t)y * ow + x) * 3 + c] = (uint8_t)p[c];
    }
}

// both passes of the kernel for every sample of the batch: the workspace, then out[batch][size][size][3] before the standardisation
void pose_augment_host(const int64_t* table, const uint8_t* src, uint8_t* ws, int batch, int size, int block, uint8_t* out) {
  const sgb_aug::RemapTabs t = tabs().view();
  for (int b = 0; b < batch; ++b) {
    const int64_t* r = table + (int64_t)b * SGB_POSE_FIELDS;
    sgb_aug::Inverse inv[4];
    for (int i = 0; i < r[SGB_POSE_NSUB]; ++i) {
      const int64_t* s = r + SGB_POSE_SUB + i * SGB_POSE_SUB_FIELDS;
      if (s[SGB_POSE_S_AFFINE]) inv[i] = sgb_pose::sub_inverse(s);
      for (int y = 0; y < s[SGB_POSE_S_RH]; ++y)
        for (int x = 0; x < s[SGB_POSE_S_RW]; ++x) {
          int p[3];
          sgb_pose::point_pixel(src, s, block, y, x, p);
          uint8_t* o = ws + s[SGB_POSE_S_WS_OFFSET] + (y * s[SGB_POSE_S_RW] + x) * 3;
          for (int c = 0; c < 3; ++c) o[c] = (uint8_t)p[c];
        }
    }
    for (int y = 0; y < size; ++y)
      for (int x = 0; x < size; ++x) {
        int p[3];
        sgb_pose::out_pixel(ws, r, inv, t, y, x, p);
        for (int c = 0; c < 3; ++c) out[(((int64_t)b * size + y) * size + x) * 3 + c] = (uint8_t)p[c];
      }
  }
}
}

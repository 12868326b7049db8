// Serial host drivers around super_gradients_b200/csrc/imagenet_augment_math.cuh and resample_math.cuh (compiled with g++ by
// tests/imagenet_augment_cases.py): the same per-value functions the CUDA kernel calls, so the CPU suite checks the kernel's
// arithmetic against Pillow without a GPU.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "imagenet_augment_math.cuh"

namespace {

// Pillow's resize of an h x w x 3 image to oh x ow: horizontal pass to uint8, then vertical
void resize(const uint8_t* src, int h, int w, int oh, int ow, int filter, uint8_t* out) {
  std::vector<uint8_t> mid((size_t)h * ow * 3);
  std::vector<int32_t> k(sgb_rs::max_taps(w, ow, filter) + sgb_rs::max_taps(h, oh, filter));
  const sgb_rs::Axis ax = sgb_rs::axis(w, ow, filter), ay = sgb_rs::axis(h, oh, filter);
  for (int col = 0; col < ow; ++col) {
    int xmin;
    const int n = sgb_rs::coeffs(ax, col, w, k.data(), xmin);
    for (int r = 0; r < h; ++r)
      for (int c = 0; c < 3; ++c) {
        int32_t acc = 1 << (sgb_rs::kPrecisionBits - 1);
        for (int t = 0; t < n; ++t) acc += (int32_t)src[((int64_t)r * w + xmin + t) * 3 + c] * k[t];
        mid[((size_t)r * ow + col) * 3 + c] = sgb_rs::clip8(acc);
      }
  }
  for (int row = 0; row < oh; ++row) {
    int ymin;
    const int n = sgb_rs::coeffs(ay, row, h, k.data(), ymin);
    for (int col = 0; col < ow; ++col)
      for (int c = 0; c < 3; ++c) {
        int32_t acc = 1 << (sgb_rs::kPrecisionBits - 1);
        for (int t = 0; t < n; ++t) acc += (int32_t)mid[((size_t)(ymin + t) * ow + col) * 3 + c] * k[t];
        out[((size_t)row * ow + col) * 3 + c] = sgb_rs::clip8(acc);
      }
  }
}

// one RandAugment op on the planar image p[3][S * S], in place
void apply_op(uint8_t* p, int S, const int64_t* op, const int32_t* fill) {
  const int code = (int)op[0];
  const int64_t* args = op + 1;
  const int n = S * S;
  std::vector<uint8_t> copy(p, p + 3 * (size_t)n);
  switch (code) {
    case SGB_IN_OP_NONE:
      return;
    case SGB_IN_OP_AFFINE: {
      double m[6];
      for (int i = 0; i < 6; ++i) m[i] = sgb_in::arg_f64(args, i);
      for (int c = 0; c < 3; ++c)
        for (int y = 0; y < S; ++y)
          for (int x = 0; x < S; ++x) p[c * n + y * S + x] = sgb_in::affine_sample(copy.data() + c * n, S, m, fill[c], x, y);
      return;
    }
    case SGB_IN_OP_AUTOCONTRAST:
    case SGB_IN_OP_EQUALIZE:
      for (int c = 0; c < 3; ++c) {
        int32_t h[256] = {0};
        uint8_t lut[256];
        for (int i = 0; i < n; ++i) ++h[p[c * n + i]];
        if (code == SGB_IN_OP_AUTOCONTRAST)
          sgb_in::autocontrast_lut(h, lut);
        else
          sgb_in::equalize_lut(h, lut);
        for (int i = 0; i < n; ++i) p[c * n + i] = lut[p[c * n + i]];
      }
      return;
    case SGB_IN_OP_COLOR: {
      const float a = (float)sgb_in::arg_f64(args, 0);
      for (int i = 0; i < n; ++i) {
        const int l = sgb_in::rgb_to_l(copy[i], copy[n + i], copy[2 * n + i]);
        for (int c = 0; c < 3; ++c) p[c * n + i] = sgb_in::blend(l, copy[c * n + i], a);
      }
      return;
    }
    case SGB_IN_OP_SHARPNESS: {
      const float a = (float)sgb_in::arg_f64(args, 0);
      for (int c = 0; c < 3; ++c)
        for (int y = 0; y < S; ++y)
          for (int x = 0; x < S; ++x) p[c * n + y * S + x] = sgb_in::blend(sgb_in::smooth(copy.data() + c * n, S, x, y), copy[c * n + y * S + x], a);
      return;
    }
    default: {
      int mean = 0;
      if (code == SGB_IN_OP_CONTRAST) {
        int64_t sum = 0;
        for (int i = 0; i < n; ++i) sum += sgb_in::rgb_to_l(p[i], p[n + i], p[2 * n + i]);
        mean = sgb_in::contrast_mean(sum, n);
      }
      for (int i = 0; i < 3 * n; ++i) p[i] = sgb_in::lut_value(code, args, mean, p[i]);
    }
  }
}

void to_planes(const uint8_t* hwc, int n, uint8_t* p) {
  for (int i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) p[c * n + i] = hwc[i * 3 + c];
}

void to_hwc(const uint8_t* p, int n, uint8_t* hwc) {
  for (int i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) hwc[i * 3 + c] = p[c * n + i];
}

}  // namespace

extern "C" {

// Image.resize((ow, oh), BILINEAR (filter 0) or BICUBIC (1)) of an h x w x 3 image
void resize_host(const uint8_t* src, int h, int w, int oh, int ow, int filter, uint8_t* out) { resize(src, h, w, oh, ow, filter, out); }

// one op (code, six arguments) on an S x S x 3 image, in place
void op_host(uint8_t* img, int S, const int64_t* op, const int32_t* fill) {
  std::vector<uint8_t> p(3 * (size_t)S * S);
  to_planes(img, S * S, p.data());
  apply_op(p.data(), S, op, fill);
  to_hwc(p.data(), S * S, img);
}

// the kernel's uint8 image (before ToTensor) of every table row: out[batch][S][S][3]
void augment_host(const int64_t* table, const uint8_t* src, int batch, int S, const int32_t* fill, uint8_t* out) {
  const int n = S * S;
  std::vector<uint8_t> hwc(3 * (size_t)n), p(3 * (size_t)n);
  for (int b = 0; b < batch; ++b) {
    const int64_t* t = table + (int64_t)b * SGB_IN_FIELDS;
    resize(src + t[SGB_IN_OFFSET], (int)t[SGB_IN_H], (int)t[SGB_IN_W], S, S, (int)t[SGB_IN_FILTER], hwc.data());
    to_planes(hwc.data(), n, p.data());
    if (t[SGB_IN_FLIP])
      for (int c = 0; c < 3; ++c)
        for (int y = 0; y < S; ++y)
          for (int x = 0; x < S / 2; ++x) {
            uint8_t* r = p.data() + c * n + y * S;
            const uint8_t v = r[x];
            r[x] = r[S - 1 - x], r[S - 1 - x] = v;
          }
    for (int k = 0; k < SGB_IN_OPS; ++k) apply_op(p.data(), S, t + SGB_IN_OP + k * SGB_IN_OP_FIELDS, fill);
    to_hwc(p.data(), n, out + (size_t)b * n * 3);
  }
}
}

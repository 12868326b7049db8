// Serial host driver around super_gradients_b200/csrc/cifar_augment_math.cuh (compiled with g++ by tests/cifar_augment_cases.py):
// the same per-pixel functions the CUDA kernel calls, so the CPU suite checks the kernel's arithmetic against torchvision without
// a GPU.
#include <stdint.h>

#include "cifar_augment_math.cuh"

extern "C" {

// every table row's float32 model input before rounding, f32[batch][3][32][32] (NCHW, as torchvision's chain returns it), and its
// bf16 rounding, bf16[batch][3][32][32]
void augment_host(const int32_t* table, const uint8_t* src, int batch, const float* mean, const float* std, float* f32, uint16_t* bf16) {
  const int n = SGB_CF_SIZE * SGB_CF_SIZE;
  for (int b = 0; b < batch; ++b) {
    const int32_t* t = table + (int64_t)b * SGB_CF_FIELDS;
    const uint8_t* img = src + (int64_t)t[SGB_CF_SOURCE] * n * 3;
    for (int i = 0; i < n; ++i) {
      const int s = sgb_cf::source_pixel(i / SGB_CF_SIZE, i % SGB_CF_SIZE, t[SGB_CF_TOP], t[SGB_CF_LEFT], t[SGB_CF_FLIP]);
      for (int c = 0; c < 3; ++c) {
        const float v = sgb_in::normalize(s < 0 ? 0 : img[s * 3 + c], mean[c], std[c]);
        f32[((int64_t)b * 3 + c) * n + i] = v;
        bf16[((int64_t)b * 3 + c) * n + i] = sgb_cf::bf16_bits(v);
      }
    }
  }
}

// the bf16 bits of n float32 values
void bf16_host(const float* in, int n, uint16_t* out) {
  for (int i = 0; i < n; ++i) out[i] = sgb_cf::bf16_bits(in[i]);
}
}

// Arithmetic of the CIFAR-10 augmentation (the cifar10_resnet recipe's train and validation chains), host+device: the CUDA kernel
// in cifar_augment.cu calls these functions and the CPU suite compiles this header with g++ to check them, bit for bit, against
// torchvision's chain.
//
// Reference chains (recipes/dataset_params/cifar10_dataset_params.yaml:9-23 and 37-49): RandomCrop(32, padding=4) (F.pad with
// fill 0 to 40 x 40, then the 32 x 32 crop at (top, left)) -> RandomHorizontalFlip -> ToTensor (float32(u) / 255) -> Normalize
// (tensor.sub_(mean).div_(std) in float32); validation: Resize(32), the identity on a 32 x 32 image, then ToTensor / Normalize.
// ToTensor / Normalize is the ImageNet chain's sgb_in::normalize (the padding reads 0).  The model input is that float32 value
// rounded to bf16 as tensor.to(torch.bfloat16) rounds it (nearest, ties to even).
#pragma once
#include <stdint.h>
#include <string.h>
#ifdef __CUDACC__
#include <cuda_bf16.h>
#endif

#include "imagenet_augment_math.cuh"

namespace sgb_cf {

// the pixel index (row * 32 + column) of the source image that output pixel (y, x) shows, or -1 where it shows the zero padding
SGB_HD int source_pixel(int y, int x, int top, int left, int flip) {
  const int r = y + top - SGB_CF_PAD;
  const int c = (flip ? SGB_CF_SIZE - 1 - x : x) + left - SGB_CF_PAD;
  return r < 0 || r >= SGB_CF_SIZE || c < 0 || c >= SGB_CF_SIZE ? -1 : r * SGB_CF_SIZE + c;
}

// the bits of v rounded to bf16, nearest with ties to even (a NaN becomes the canonical quiet NaN)
SGB_HD uint16_t bf16_bits(float v) {
#ifdef __CUDA_ARCH__
  return __bfloat16_as_ushort(__float2bfloat16_rn(v));
#else
  uint32_t u;
  memcpy(&u, &v, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return 0x7fc0;
  return (uint16_t)((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);
#endif
}

}  // namespace sgb_cf

// CIFAR-10 augmentation of a whole batch in ONE launch: uint8 32 x 32 x 3 sources -> zero-padded random crop -> flip -> ToTensor /
// Normalize -> bf16 NHWC batch (channels >= 3 zero).  The arithmetic is in cifar_augment_math.cuh (shared with the CPU test build).
//
// One thread makes one output pixel: it reads the three bytes its crop and flip select (or none, in the padding) and writes the
// pixel's whole channel pitch with 16-byte stores.  The sources are either the batch's own packed images or a resident data set
// the table indexes; the kernel does not tell them apart.
#include "cifar_augment_math.cuh"
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kPixels = SGB_CF_SIZE * SGB_CF_SIZE;

struct Params {
  int out_pitch;
  float mean[3], std[3];
};

__global__ void __launch_bounds__(kThreads) cifar_augment_kernel(const Params p, const int4* __restrict__ table, const uint8_t* __restrict__ src,
                                                                 int batch, bf16* __restrict__ out) {
  const int64_t g = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (g >= (int64_t)batch * kPixels) return;
  const int b = (int)(g / kPixels), i = (int)(g - (int64_t)b * kPixels);
  const int4 t = table[b];  // source, top, left, flip
  const int s = sgb_cf::source_pixel(i / SGB_CF_SIZE, i % SGB_CF_SIZE, t.y, t.z, t.w);
  const uint8_t* px = s < 0 ? nullptr : src + ((int64_t)t.x * kPixels + s) * 3;
  uint16_t v[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = sgb_cf::bf16_bits(sgb_in::normalize(s < 0 ? 0 : px[c], p.mean[c], p.std[c]));
  bf16* o = out + g * p.out_pitch;
  for (int c0 = 0; c0 < p.out_pitch; c0 += 8) {
    __align__(16) uint16_t pack[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) pack[j] = c0 + j < 3 ? v[c0 + j] : 0;
    *(uint4*)(o + c0) = *(const uint4*)pack;
  }
}

}  // namespace

extern "C" int sgb_cifar_augment(const int32_t* table_host, const int32_t* table, const uint8_t* src, int64_t src_images, int32_t batch,
                                 int32_t out_pitch, const float* mean_host, const float* std_host, sgb_bf16* out, void* stream) {
  SGB_REQUIRE(table_host && table && src && out && mean_host && std_host, "null pointer");
  SGB_REQUIRE(batch >= 1 && batch <= (1 << 24), "batch must be in [1, 2^24]");
  SGB_REQUIRE(src_images >= 1, "src must hold at least one image");
  SGB_REQUIRE(out_pitch >= 3 && out_pitch % 8 == 0, "output channel pitch must be >= 3 and a multiple of 8");
  SGB_REQUIRE((uintptr_t)out % 16 == 0 && (uintptr_t)table % 16 == 0, "out and table must be 16-byte aligned");
  Params p = {};
  p.out_pitch = out_pitch;
  for (int c = 0; c < 3; ++c) {
    SGB_REQUIRE(std::isfinite(mean_host[c]) && std::isfinite(std_host[c]) && std_host[c] != 0.f, "bad mean or std");
    p.mean[c] = mean_host[c], p.std[c] = std_host[c];
  }
  for (int b = 0; b < batch; ++b) {
    const int32_t* t = table_host + (int64_t)b * SGB_CF_FIELDS;
    SGB_REQUIRE(t[SGB_CF_SOURCE] >= 0 && t[SGB_CF_SOURCE] < src_images, "a source index lies outside src");
    SGB_REQUIRE(t[SGB_CF_TOP] >= 0 && t[SGB_CF_TOP] <= 2 * SGB_CF_PAD && t[SGB_CF_LEFT] >= 0 && t[SGB_CF_LEFT] <= 2 * SGB_CF_PAD,
                "crop corners must lie in [0, 8]");
    SGB_REQUIRE(t[SGB_CF_FLIP] == 0 || t[SGB_CF_FLIP] == 1, "flip must be 0 or 1");
  }
  const int64_t threads = (int64_t)batch * kPixels;
  cifar_augment_kernel<<<(unsigned)((threads + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(p, (const int4*)table, src, batch, (bf16*)out);
  SGB_LAUNCH_CHECK("cifar_augment_kernel");
  return SGB_OK;
}

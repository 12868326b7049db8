// Fused predict() pre-processing (row (f)-N3): uint8 HWC image -> INTER_LINEAR resize (OpenCV's fixed-point arithmetic) -> constant
// padding -> optional channel reversal -> /max_value -> optional mean / std -> bf16 NHWC slot of the batch tensor (channels padded
// with zeros to the slot's pitch), one launch per image instead of five numpy / cv2 passes on the host.  HBM-bound and tiny:
// a 640 x 640 x 16 bf16 slot is 13 MB written, the source image is read through L1 / L2 (4 taps per sample).
// The arithmetic is in preprocess_math.cuh (shared with the CPU test build).
#include "common.cuh"
#include "preprocess_math.cuh"

namespace {

__global__ void preprocess_u8_kernel(const SgbPreprocDesc d, const uint8_t* __restrict__ src, bf16* __restrict__ out) {
  const int64_t total = (int64_t)d.out_h * d.out_w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int oy = (int)(i / d.out_w), ox = (int)(i - (int64_t)oy * d.out_w);
    bf16* o = out + i * d.out_pitch;
    for (int c = 0; c < d.out_pitch; ++c)
      o[c] = __float2bfloat16_rn(c < d.src_c ? sgb_prep::sample_pixel(d, src, oy, ox, c) : 0.f);
  }
}

}  // namespace

extern "C" int sgb_preprocess_u8(const SgbPreprocDesc* d, const uint8_t* src, sgb_bf16* out, void* stream) {
  SGB_REQUIRE(d && src && out, "null pointer");
  SGB_REQUIRE(d->src_h > 0 && d->src_w > 0 && d->src_c > 0 && d->src_c <= 4, "source must be H x W x (1..4) uint8");
  SGB_REQUIRE(d->src_pitch >= d->src_w * d->src_c, "source row pitch");
  SGB_REQUIRE(d->dst_h > 0 && d->dst_w > 0 && d->out_h > 0 && d->out_w > 0, "bad target shape");
  SGB_REQUIRE(d->pad_top >= 0 && d->pad_left >= 0 && d->pad_top + d->dst_h <= d->out_h && d->pad_left + d->dst_w <= d->out_w,
              "the resized image must fit the padded canvas");
  SGB_REQUIRE(d->out_pitch >= d->src_c, "output channel pitch");
  const int64_t total = (int64_t)d->out_h * d->out_w;
  const int grid = (int)((total + 255) / 256 > 132 * 8 ? 132 * 8 : (total + 255) / 256);
  preprocess_u8_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(*d, src, (bf16*)out);
  SGB_LAUNCH_CHECK("preprocess_u8_kernel");
  return SGB_OK;
}

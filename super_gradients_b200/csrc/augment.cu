// Detection train augmentation of a whole batch in ONE launch: uint8 HWC source (mosaic tile and mixup partner) images of any
// sizes -> mosaic -> affine -> channel swap -> HSV -> flip -> mixup -> padded rescale -> /max_value -> bf16 NHWC batch (channels
// >= 3 zero).  The arithmetic is in augment_math.cuh (shared with the CPU test build).  One thread per output pixel recomputes every cv2 step the
// pixel depends on, so no uint8 intermediate image is written; the per-image draws travel in the int64 table.
#include "augment_math.cuh"
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr double kMaxCoord = 1048576.0;  // 2^20: fixed-point source coordinates (<< 10) stay inside int32

// kMosaic: the batch holds a mosaic sample.  The launch picks the instance, so a batch without one runs the mosaic-free code and
// stages only the fields before the mosaic's.
template <bool kMosaic>
__global__ void __launch_bounds__(kThreads) augment_kernel(const int64_t* __restrict__ table, const uint8_t* __restrict__ src,
                                                           bf16* __restrict__ out, int out_h, int out_w, int out_pitch, int pad_value,
                                                           double max_value, int block) {
  constexpr int kFields = kMosaic ? SGB_AUG_FIELDS : SGB_AUG_MOS;
  __shared__ int64_t t[kFields];
  for (int i = threadIdx.x; i < kFields; i += blockDim.x) t[i] = table[(int64_t)blockIdx.y * SGB_AUG_FIELDS + i];
  __syncthreads();
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= out_h * out_w) return;
  const int oy = pix / out_w, ox = pix - oy * out_w;
  const sgb_aug::Inverse a = sgb_aug::table_inverse(t);
  int p[3];
  sgb_aug::augment_pixel<kMosaic>(src, t, a, block, pad_value, oy, ox, p);
  bf16* o = out + ((int64_t)blockIdx.y * out_h * out_w + pix) * out_pitch;
  for (int c0 = 0; c0 < out_pitch; c0 += 8) {
    __align__(16) bf16 pack[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = c0 + j;
      pack[j] = __float2bfloat16_rn(c < 3 ? sgb_prep::standardize((float)p[c], max_value, 0, 0.f, 1.f) : 0.f);
    }
    *(uint4*)(o + c0) = *(const uint4*)pack;
  }
}

bool flag(int64_t v) { return v == 0 || v == 1; }

bool image_in(int64_t off, int64_t h, int64_t w, int64_t src_bytes) {
  return h > 0 && w > 0 && h < 32768 && w < 32768 && off >= 0 && off <= src_bytes && h * w * 3 <= src_bytes - off;
}

}  // namespace

extern "C" int sgb_detection_augment(const int64_t* table_host, const int64_t* table, const uint8_t* src, int64_t src_bytes, int32_t batch,
                                     int32_t channels, int32_t out_h, int32_t out_w, int32_t out_pitch, int32_t pad_value, double max_value,
                                     int32_t hsv_simd_block, sgb_bf16* out, void* stream) {
  if (batch == 0) return SGB_OK;
  SGB_REQUIRE(table_host && table && src && out, "null pointer");
  SGB_REQUIRE(batch > 0 && batch <= 65535, "batch must be in [0, 65535]");
  SGB_REQUIRE(channels == 3, "images must be H x W x 3 uint8");
  SGB_REQUIRE(out_h > 0 && out_w > 0 && out_h < 32768 && out_w < 32768, "bad output size");
  SGB_REQUIRE(out_pitch >= channels && out_pitch % 8 == 0, "output channel pitch must be >= channels and a multiple of 8");
  SGB_REQUIRE(pad_value >= 0 && pad_value <= 255 && max_value > 0.0 && hsv_simd_block > 0, "bad pad value, max value or HSV block");
  bool mosaic = false;
  for (int b = 0; b < batch; ++b) {
    const int64_t* t = table_host + (int64_t)b * SGB_AUG_FIELDS;
    SGB_REQUIRE(image_in(t[SGB_AUG_OFFSET], t[SGB_AUG_H], t[SGB_AUG_W], src_bytes), "bad source image shape, or the image lies outside the buffer");
    SGB_REQUIRE(flag(t[SGB_AUG_AFFINE]) && flag(t[SGB_AUG_SWAP]) && flag(t[SGB_AUG_HSV]) && flag(t[SGB_AUG_FLIP]) && flag(t[SGB_AUG_MIX]) && flag(t[SGB_AUG_MOS]),
                "flags must be 0 or 1");
    int64_t in_h = t[SGB_AUG_H], in_w = t[SGB_AUG_W];  // the image the affine (or the chain) reads
    if (t[SGB_AUG_MOS]) {
      mosaic = true;
      in_h = t[SGB_AUG_MOS_CANVAS_H], in_w = t[SGB_AUG_MOS_CANVAS_W];
      const int64_t xc = t[SGB_AUG_MOS_XC], yc = t[SGB_AUG_MOS_YC];
      SGB_REQUIRE(in_h > 0 && in_w > 0 && in_h < 32768 && in_w < 32768, "bad mosaic canvas size");
      SGB_REQUIRE(xc >= 0 && xc <= in_w && yc >= 0 && yc <= in_h, "the mosaic centre lies outside the canvas");
      SGB_REQUIRE(t[SGB_AUG_MOS_BORDER] >= 0 && t[SGB_AUG_MOS_BORDER] <= 255, "bad mosaic border value");
      for (int i = 0; i < SGB_AUG_MOS_TILES; ++i) {
        const int64_t* k = t + SGB_AUG_MOS_TILE + i * SGB_AUG_MOS_TILE_FIELDS;
        SGB_REQUIRE(image_in(k[SGB_AUG_T_OFFSET], k[SGB_AUG_T_H], k[SGB_AUG_T_W], src_bytes), "bad mosaic tile shape, or the tile lies outside the buffer");
        const int64_t rh = k[SGB_AUG_T_RH], rw = k[SGB_AUG_T_RW];
        SGB_REQUIRE(rh > 0 && rw > 0 && rh < 32768 && rw < 32768, "bad resized mosaic tile size");
        const int64_t x1 = k[SGB_AUG_T_X1], y1 = k[SGB_AUG_T_Y1], x2 = k[SGB_AUG_T_X2], y2 = k[SGB_AUG_T_Y2];
        const bool right = i & 1, bottom = i & 2;  // tile i's quadrant: the only place the kernel looks for it
        SGB_REQUIRE(x1 <= x2 && y1 <= y2 && x1 >= (right ? xc : 0) && x2 <= (right ? in_w : xc) && y1 >= (bottom ? yc : 0) && y2 <= (bottom ? in_h : yc),
                    "a mosaic tile's rectangle leaves its quadrant of the canvas");
        const int64_t sx = k[SGB_AUG_T_SX], sy = k[SGB_AUG_T_SY];
        SGB_REQUIRE(sx >= 0 && sy >= 0 && sx <= rw - (x2 - x1) && sy <= rh - (y2 - y1), "a mosaic tile's rectangle reads outside the resized tile");
      }
    }
    const int64_t ah = t[SGB_AUG_AFF_H], aw = t[SGB_AUG_AFF_W];
    SGB_REQUIRE(ah > 0 && aw > 0 && ah < 32768 && aw < 32768, "bad affine output size");
    if (t[SGB_AUG_AFFINE]) {
      SGB_REQUIRE(t[SGB_AUG_AFF_BORDER] >= 0 && t[SGB_AUG_AFF_BORDER] <= 255, "bad affine border value");
      double m[6];
      for (int i = 0; i < 6; ++i) m[i] = *(const double*)&t[SGB_AUG_M + i];
      const double det = m[0] * m[4] - m[1] * m[3];
      SGB_REQUIRE(std::isfinite(det) && det != 0.0 && std::isfinite(m[2]) && std::isfinite(m[5]), "degenerate or non-finite affine matrix");
      const sgb_aug::Inverse a = sgb_aug::invert(m);
      for (int k = 0; k < 4; ++k) {  // the map is affine: its extremes over the output are at the corners
        const double y = (k & 1) ? (double)(ah - 1) : 0.0, x = (k & 2) ? (double)(aw - 1) : 0.0;
        const double sx = a.a11 * x + a.a12 * y + a.b1, sy = a.a21 * x + a.a22 * y + a.b2;
        SGB_REQUIRE(std::isfinite(sx) && std::isfinite(sy) && fabs(sx) < kMaxCoord && fabs(sy) < kMaxCoord, "the affine matrix maps the output too far outside the image");
      }
    } else {
      SGB_REQUIRE(ah == in_h && aw == in_w, "without the affine the image keeps its size");
    }
    if (t[SGB_AUG_HSV]) {
      const int64_t bgr = t[SGB_AUG_BGR], c0 = bgr & 3, c1 = (bgr >> 2) & 3, c2 = (bgr >> 4) & 3;
      SGB_REQUIRE(bgr >= 0 && bgr < 64 && c0 < 3 && c1 < 3 && c2 < 3 && c0 != c1 && c1 != c2 && c0 != c2, "bgr_channels must be a permutation of (0, 1, 2)");
      SGB_REQUIRE(t[SGB_AUG_DH] > -32768 && t[SGB_AUG_DH] < 32768 && t[SGB_AUG_DS] > -32768 && t[SGB_AUG_DS] < 32768 && t[SGB_AUG_DV] > -32768 && t[SGB_AUG_DV] < 32768,
                  "HSV gains must fit int16");
    }
    if (t[SGB_AUG_MIX]) {
      SGB_REQUIRE(image_in(t[SGB_AUG_MIX_OFFSET], t[SGB_AUG_MIX_H], t[SGB_AUG_MIX_W], src_bytes), "bad mixup image shape, or the image lies outside the buffer");
      SGB_REQUIRE(flag(t[SGB_AUG_MIX_FLIP]) && t[SGB_AUG_MIX_BORDER] >= 0 && t[SGB_AUG_MIX_BORDER] <= 255, "bad mixup flip flag or border value");
      const int64_t ch = t[SGB_AUG_MIX_CANVAS_H], cw = t[SGB_AUG_MIX_CANVAS_W];
      SGB_REQUIRE(ch > 0 && cw > 0 && ch < 32768 && cw < 32768, "bad mixup canvas size");
      SGB_REQUIRE(t[SGB_AUG_MIX_R1_H] > 0 && t[SGB_AUG_MIX_R1_W] > 0 && t[SGB_AUG_MIX_R1_H] <= ch && t[SGB_AUG_MIX_R1_W] <= cw, "the first mixup resize must fit the canvas");
      SGB_REQUIRE(t[SGB_AUG_MIX_R2_H] > 0 && t[SGB_AUG_MIX_R2_W] > 0 && t[SGB_AUG_MIX_R2_H] < 32768 && t[SGB_AUG_MIX_R2_W] < 32768, "bad second mixup resize size");
      SGB_REQUIRE(t[SGB_AUG_MIX_X] >= 0 && t[SGB_AUG_MIX_Y] >= 0 && t[SGB_AUG_MIX_X] < 32768 && t[SGB_AUG_MIX_Y] < 32768, "bad mixup crop offset");
    }
    SGB_REQUIRE(t[SGB_AUG_RS_H] > 0 && t[SGB_AUG_RS_W] > 0 && t[SGB_AUG_RS_H] <= out_h && t[SGB_AUG_RS_W] <= out_w, "the rescaled image must fit the output");
  }
  const dim3 grid((out_h * out_w + kThreads - 1) / kThreads, batch);
  if (mosaic)
    augment_kernel<true><<<grid, kThreads, 0, (cudaStream_t)stream>>>(table, src, (bf16*)out, out_h, out_w, out_pitch, pad_value, max_value, hsv_simd_block);
  else
    augment_kernel<false><<<grid, kThreads, 0, (cudaStream_t)stream>>>(table, src, (bf16*)out, out_h, out_w, out_pitch, pad_value, max_value, hsv_simd_block);
  SGB_LAUNCH_CHECK("augment_kernel");
  return SGB_OK;
}

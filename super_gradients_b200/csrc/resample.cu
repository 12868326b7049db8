// ImageNet predict() pre-processing of a whole batch (row (f)-N3): uint8 HWC images of any sizes -> Pillow's antialiased
// bilinear resize, evaluated only inside the center-crop window -> optional channel reversal -> /max_value -> optional mean / std
// -> bf16 NHWC batch (channels >= C zero), in ONE launch.  The arithmetic is in resample_math.cuh (shared with the CPU test build)
// and preprocess_math.cuh (standardisation).
//
// Grid (row tiles, images).  A CTA computes the fixed-point coefficients of its crop columns and of its TH output rows, runs the
// horizontal pass over the source rows those TH rows read (uint8, in shared memory, only the crop columns), then the vertical pass,
// and writes 8 channels per 16-byte store.  The host picks the largest TH <= 16 whose staged rows fit kSmemCap over the batch.
#include "common.cuh"
#include "preprocess_math.cuh"
#include "resample_math.cuh"

namespace {

constexpr int kMaxTile = 16;
constexpr int kSmemCap = 200 * 1024;
constexpr int kThreads = 256;

struct Params {
  int C, out_h, out_w, out_pitch, reverse, normalize;
  double max_value;
  float mean[4], std[4];
};

__host__ __device__ inline size_t layout_bytes(int out_w, int C, int tile, int kx, int ky, int rows) {
  // int32: horizontal weights [out_w][kx], first / count [out_w] x 2, vertical weights [tile][ky], first / count [tile] x 2; then uint8 rows
  return (size_t)4 * ((size_t)out_w * (kx + 2) + (size_t)tile * (ky + 2)) + (size_t)rows * out_w * C;
}

__global__ void __launch_bounds__(kThreads) resample_crop_kernel(const Params d, const int64_t* __restrict__ table,
                                                                 const uint8_t* __restrict__ src, bf16* __restrict__ out, int tile,
                                                                 int kx, int ky) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int64_t* t = table + (int64_t)blockIdx.y * SGB_RS_FIELDS;
  const int64_t offset = t[SGB_RS_OFFSET];
  const int h = (int)t[SGB_RS_H], w = (int)t[SGB_RS_W], pitch = (int)t[SGB_RS_PITCH], rh = (int)t[SGB_RS_RESIZED_H], rw = (int)t[SGB_RS_RESIZED_W];
  const int top = (int)t[SGB_RS_CROP_TOP], left = (int)t[SGB_RS_CROP_LEFT];
  const int C = d.C, W = d.out_w;
  const int oy0 = blockIdx.x * tile;
  if (oy0 >= d.out_h) return;
  const int nt = min(tile, d.out_h - oy0);
  int32_t* hk = (int32_t*)smem;
  int32_t* hmin = hk + W * kx;
  int32_t* hn = hmin + W;
  int32_t* vk = hn + W;
  int32_t* vmin = vk + tile * ky;
  int32_t* vn = vmin + tile;
  uint8_t* stage = (uint8_t*)(vn + tile);

  const sgb_rs::Axis ax = sgb_rs::axis(w, rw), ay = sgb_rs::axis(h, rh);
  for (int col = threadIdx.x; col < W; col += blockDim.x) {
    int xmin;
    hn[col] = sgb_rs::coeffs(ax, left + col, w, hk + col * kx, xmin);
    hmin[col] = xmin;
  }
  for (int r = threadIdx.x; r < nt; r += blockDim.x) {
    int ymin;
    vn[r] = sgb_rs::coeffs(ay, top + oy0 + r, h, vk + r * ky, ymin);
    vmin[r] = ymin;
  }
  __syncthreads();
  const int r0 = vmin[0], rows = vmin[nt - 1] + vn[nt - 1] - r0;
  const uint8_t* img = src + offset;
  const int row_elems = W * C;
  for (int i = threadIdx.x; i < rows * row_elems; i += blockDim.x) {
    const int r = i / row_elems, e = i - r * row_elems, col = e / C, c = e - col * C;
    const uint8_t* s = img + (int64_t)(r0 + r) * pitch + hmin[col] * C + c;
    const int32_t* k = hk + col * kx;
    int32_t acc = 1 << (sgb_rs::kPrecisionBits - 1);
    for (int t = 0; t < hn[col]; ++t) acc += (int32_t)s[t * C] * k[t];
    stage[i] = sgb_rs::clip8(acc);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nt * W; i += blockDim.x) {
    const int r = i / W, col = i - r * W;
    float v[4];
    for (int c = 0; c < C; ++c) {
      const uint8_t* s = stage + (int64_t)(vmin[r] - r0) * row_elems + col * C + c;
      const int32_t* k = vk + r * ky;
      int32_t acc = 1 << (sgb_rs::kPrecisionBits - 1);
      for (int t = 0; t < vn[r]; ++t) acc += (int32_t)s[t * row_elems] * k[t];
      v[c] = (float)sgb_rs::clip8(acc);
    }
    bf16* o = out + (((int64_t)blockIdx.y * d.out_h + oy0 + r) * W + col) * d.out_pitch;
    for (int c0 = 0; c0 < d.out_pitch; c0 += 8) {
      __align__(16) bf16 pack[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = c0 + j;
        pack[j] = __float2bfloat16_rn(c < C ? sgb_prep::standardize(v[d.reverse ? C - 1 - c : c], d.max_value, d.normalize, d.mean[c], d.std[c]) : 0.f);
      }
      *(uint4*)(o + c0) = *(const uint4*)pack;
    }
  }
}

}  // namespace

extern "C" int sgb_resample_crop_u8(const int64_t* table_host, const int64_t* table, const uint8_t* src, int64_t src_bytes, int32_t batch,
                                    int32_t channels, int32_t out_h, int32_t out_w, int32_t out_pitch, int32_t reverse_channels,
                                    double max_value, const float* mean_host, const float* std_host, sgb_bf16* out, void* stream) {
  if (batch == 0) return SGB_OK;
  SGB_REQUIRE(table_host && table && src && out, "null pointer");
  SGB_REQUIRE(batch > 0 && batch <= 65535, "batch must be in [0, 65535]");
  SGB_REQUIRE(channels == 3, "images must be H x W x 3 uint8");
  SGB_REQUIRE(out_h > 0 && out_w > 0, "bad crop size");
  SGB_REQUIRE(out_pitch >= channels && out_pitch % 8 == 0, "output channel pitch must be >= channels and a multiple of 8");
  SGB_REQUIRE((mean_host == nullptr) == (std_host == nullptr), "mean and std go together");
  Params p = {};
  p.C = channels, p.out_h = out_h, p.out_w = out_w, p.out_pitch = out_pitch, p.reverse = reverse_channels ? 1 : 0, p.max_value = max_value;
  p.normalize = mean_host != nullptr;
  for (int c = 0; c < channels; ++c) {
    p.mean[c] = mean_host ? mean_host[c] : 0.f;
    p.std[c] = std_host ? std_host[c] : 1.f;
  }
  int kx = 1, ky = 1;
  for (int b = 0; b < batch; ++b) {
    const int64_t* t = table_host + (int64_t)b * SGB_RS_FIELDS;
    const int64_t off = t[SGB_RS_OFFSET], h = t[SGB_RS_H], w = t[SGB_RS_W], pitch = t[SGB_RS_PITCH], rh = t[SGB_RS_RESIZED_H], rw = t[SGB_RS_RESIZED_W];
    const int64_t top = t[SGB_RS_CROP_TOP], left = t[SGB_RS_CROP_LEFT];
    SGB_REQUIRE(h > 0 && w > 0 && h < (1 << 24) && w < (1 << 24) && pitch >= w * channels && pitch < (1 << 30), "bad source image shape / pitch");
    SGB_REQUIRE(off >= 0 && off + (h - 1) * pitch + w * channels <= src_bytes, "source image outside the buffer");
    SGB_REQUIRE(rh > 0 && rw > 0 && rh < (1 << 24) && rw < (1 << 24), "bad resized shape");
    SGB_REQUIRE(top >= 0 && left >= 0 && top + out_h <= rh && left + out_w <= rw, "the crop window must lie inside the resized image");
    kx = max(kx, sgb_rs::max_taps((int)w, (int)rw));
    ky = max(ky, sgb_rs::max_taps((int)h, (int)rh));
  }
  int tile = 0;
  size_t bytes = 0;
  for (int th = kMaxTile; th >= 1 && tile == 0; th /= 2) {
    int rows = 0;
    for (int b = 0; b < batch; ++b) {
      const int64_t* t = table_host + (int64_t)b * SGB_RS_FIELDS;
      const int h = (int)t[SGB_RS_H], rh = (int)t[SGB_RS_RESIZED_H], top = (int)t[SGB_RS_CROP_TOP];
      for (int y0 = 0; y0 < out_h; y0 += th) {
        int first, count;
        sgb_rs::row_span(h, rh, top + y0, top + min(y0 + th, out_h) - 1, first, count);
        rows = max(rows, count);
      }
    }
    const size_t need = layout_bytes(out_w, channels, th, kx, ky, rows);
    if (need <= (size_t)kSmemCap) tile = th, bytes = need;
  }
  SGB_REQUIRE(tile > 0, "the source rows of one output row do not fit in shared memory (downscale factor too large)");
  if (bytes > 48 * 1024) {
    if (int rc = sgb_cuda_check(cudaFuncSetAttribute(resample_crop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes), "cudaFuncSetAttribute"))
      return rc;
  }
  const dim3 grid((out_h + tile - 1) / tile, batch);
  resample_crop_kernel<<<grid, kThreads, bytes, (cudaStream_t)stream>>>(p, table, src, (bf16*)out, tile, kx, ky);
  SGB_LAUNCH_CHECK("resample_crop_kernel");
  return SGB_OK;
}

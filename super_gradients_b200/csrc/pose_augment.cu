// Pose train augmentation of a whole batch in TWO launches, whatever its size: (1) the pointwise steps of every tile (flip,
// brightness-contrast, channel reversal, HSV) written rotated (np.rot90) into a caller-owned uint8 workspace, one thread per tile
// pixel; (2) one thread per output pixel recomputing pad -> LongestMaxSize resize -> mosaic placement -> cv2.warpAffine of the
// tile it falls in, then /max_value -> bf16 NHWC (channels >= 3 zero).  Splitting the pointwise steps out means the warp's up to
// 64 taps (Lanczos4) under the resize's 4 read uint8 pixels instead of recomputing the HSV round trip per tap.  The arithmetic is
// in pose_augment_math.cuh (shared with the CPU test build).
#include <mutex>

#include "common.cuh"
#include "pose_augment_math.cuh"

namespace {

constexpr int kThreads = 256;
constexpr double kMaxCoord = 1048576.0;  // 2^20: fixed-point source coordinates (<< 10) stay inside int32

__device__ int16_t g_cubic[1024 * 16];
__device__ int16_t g_lanczos[1024 * 64];

__global__ void __launch_bounds__(kThreads) pose_point_kernel(const int64_t* __restrict__ table, const uint8_t* __restrict__ src,
                                                              uint8_t* __restrict__ ws, int block) {
  __shared__ int64_t s[SGB_POSE_SUB_FIELDS];
  __shared__ int64_t nsub;
  const int b = blockIdx.y >> 2, sub = blockIdx.y & 3;
  const int64_t* t = table + (int64_t)b * SGB_POSE_FIELDS;
  for (int i = threadIdx.x; i < SGB_POSE_SUB_FIELDS; i += blockDim.x) s[i] = t[SGB_POSE_SUB + sub * SGB_POSE_SUB_FIELDS + i];
  if (threadIdx.x == 0) nsub = t[SGB_POSE_NSUB];
  __syncthreads();
  if (sub >= nsub) return;
  const int rw = (int)s[SGB_POSE_S_RW];
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (int)s[SGB_POSE_S_RH] * rw) return;
  const int y = pix / rw, x = pix - y * rw;
  int p[3];
  sgb_pose::point_pixel(src, s, block, y, x, p);
  uint8_t* o = ws + s[SGB_POSE_S_WS_OFFSET] + (int64_t)pix * 3;
  o[0] = (uint8_t)p[0], o[1] = (uint8_t)p[1], o[2] = (uint8_t)p[2];
}

__global__ void __launch_bounds__(kThreads) pose_out_kernel(const int64_t* __restrict__ table, const uint8_t* __restrict__ ws, bf16* __restrict__ out,
                                                            int size, int out_pitch, double max_value) {
  __shared__ int64_t t[SGB_POSE_FIELDS];
  __shared__ sgb_aug::Inverse inv[4];
  for (int i = threadIdx.x; i < SGB_POSE_FIELDS; i += blockDim.x) t[i] = table[(int64_t)blockIdx.y * SGB_POSE_FIELDS + i];
  __syncthreads();
  if (threadIdx.x < t[SGB_POSE_NSUB] && t[SGB_POSE_SUB + threadIdx.x * SGB_POSE_SUB_FIELDS + SGB_POSE_S_AFFINE])
    inv[threadIdx.x] = sgb_pose::sub_inverse(t + SGB_POSE_SUB + threadIdx.x * SGB_POSE_SUB_FIELDS);
  __syncthreads();
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= size * size) return;
  const int oy = pix / size, ox = pix - oy * size;
  const sgb_aug::RemapTabs tabs{g_cubic, g_lanczos};
  int p[3];
  sgb_pose::out_pixel(ws, t, inv, tabs, oy, ox, p);
  bf16* o = out + ((int64_t)blockIdx.y * size * size + pix) * out_pitch;
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

// the cubic and Lanczos4 tables, copied once per device (they are constants of cv2, not of the batch)
cudaError_t ensure_tables() {
  static std::mutex mu;
  static bool done[256] = {};
  static int16_t cubic[1024 * 16], lanczos[1024 * 64];
  static bool built = false;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(mu);
  if (!built) {
    sgb_pose::remap_table(4, cubic);
    sgb_pose::remap_table(8, lanczos);
    built = true;
  }
  if (dev < 0 || dev >= 256 || done[dev]) return cudaSuccess;
  if ((e = cudaMemcpyToSymbol(g_cubic, cubic, sizeof(cubic))) != cudaSuccess) return e;
  if ((e = cudaMemcpyToSymbol(g_lanczos, lanczos, sizeof(lanczos))) != cudaSuccess) return e;
  done[dev] = true;
  return cudaSuccess;
}

bool flag(int64_t v) { return v == 0 || v == 1; }
bool dim_ok(int64_t v) { return v > 0 && v < 32768; }
bool bytes_in(int64_t off, int64_t h, int64_t w, int64_t total) { return dim_ok(h) && dim_ok(w) && off >= 0 && off <= total && h * w * 3 <= total - off; }
bool packed_ok(int64_t v) { return v >= 0 && v < (1 << 24); }

}  // namespace

extern "C" int sgb_pose_augment(const int64_t* table_host, const int64_t* table, const uint8_t* src, int64_t src_bytes, uint8_t* workspace,
                                int64_t workspace_bytes, int32_t batch, int32_t out_size, int32_t out_pitch, double max_value, int32_t hsv_simd_block,
                                sgb_bf16* out, void* stream) {
  if (batch == 0) return SGB_OK;
  SGB_REQUIRE(table_host && table && src && workspace && out, "null pointer");
  SGB_REQUIRE(batch > 0 && batch <= 16383, "batch must be in [0, 16383]");
  SGB_REQUIRE(out_size > 0 && out_size < 32768, "bad output size");
  SGB_REQUIRE(out_pitch >= 3 && out_pitch % 8 == 0, "output channel pitch must be >= 3 and a multiple of 8");
  SGB_REQUIRE(max_value > 0.0 && std::isfinite(max_value) && hsv_simd_block > 0, "bad max value or HSV block");
  int64_t max_pix = 1;
  for (int b = 0; b < batch; ++b) {
    const int64_t* t = table_host + (int64_t)b * SGB_POSE_FIELDS;
    const int64_t n = t[SGB_POSE_NSUB], ch = t[SGB_POSE_CANVAS_H], cw = t[SGB_POSE_CANVAS_W];
    SGB_REQUIRE(n == 1 || n == 4, "a sample has 1 tile, or 4 for a mosaic");
    SGB_REQUIRE(dim_ok(ch) && dim_ok(cw) && dim_ok(t[SGB_POSE_RS_H]) && dim_ok(t[SGB_POSE_RS_W]), "bad canvas or resize size");
    SGB_REQUIRE(t[SGB_POSE_PAD_TOP] >= 0 && t[SGB_POSE_PAD_LEFT] >= 0 && t[SGB_POSE_PAD_TOP] + t[SGB_POSE_RS_H] <= out_size &&
                    t[SGB_POSE_PAD_LEFT] + t[SGB_POSE_RS_W] <= out_size,
                "the resized canvas must fit the output");
    SGB_REQUIRE(packed_ok(t[SGB_POSE_MOSAIC_PAD]) && packed_ok(t[SGB_POSE_PAD_VALUE]), "bad pad colour");
    for (int i = 0; i < n; ++i) {
      const int64_t* s = t + SGB_POSE_SUB + i * SGB_POSE_SUB_FIELDS;
      const int64_t H = s[SGB_POSE_S_H], W = s[SGB_POSE_S_W], rh = s[SGB_POSE_S_RH], rw = s[SGB_POSE_S_RW], k = s[SGB_POSE_S_ROT];
      SGB_REQUIRE(bytes_in(s[SGB_POSE_S_OFFSET], H, W, src_bytes), "bad source image shape, or the image lies outside the buffer");
      SGB_REQUIRE(k >= 0 && k <= 3 && rh == (k & 1 ? W : H) && rw == (k & 1 ? H : W), "rot90 count must be in [0, 3] and the tile size its result");
      SGB_REQUIRE(bytes_in(s[SGB_POSE_S_WS_OFFSET], rh, rw, workspace_bytes), "the tile lies outside the workspace");
      SGB_REQUIRE(s[SGB_POSE_S_Y] >= 0 && s[SGB_POSE_S_X] >= 0 && s[SGB_POSE_S_Y] + rh <= ch && s[SGB_POSE_S_X] + rw <= cw, "the tile must lie inside the canvas");
      SGB_REQUIRE(flag(s[SGB_POSE_S_FLIP]) && flag(s[SGB_POSE_S_BC]) && flag(s[SGB_POSE_S_REVERSE]) && flag(s[SGB_POSE_S_HSV]) && flag(s[SGB_POSE_S_AFFINE]),
                  "flags must be 0 or 1");
      if (s[SGB_POSE_S_BC]) {
        for (int j = 0; j < 5; ++j) {
          const int64_t v = s[SGB_POSE_S_MEAN + j];
          SGB_REQUIRE(v >= 0 && v <= 0xffffffffLL && std::isfinite(sgb_pose::bits_f32(v)), "brightness-contrast values must be finite float32 bits");
        }
      }
      if (s[SGB_POSE_S_HSV]) {
        SGB_REQUIRE(s[SGB_POSE_S_DH] > -32768 && s[SGB_POSE_S_DH] < 32768 && s[SGB_POSE_S_DS] > -32768 && s[SGB_POSE_S_DS] < 32768 && s[SGB_POSE_S_DV] > -32768 &&
                        s[SGB_POSE_S_DV] < 32768,
                    "HSV gains must fit int16");
      }
      if (s[SGB_POSE_S_AFFINE]) {
        SGB_REQUIRE(s[SGB_POSE_S_MODE] >= 0 && s[SGB_POSE_S_MODE] <= 4, "interpolation mode must be in [0, 4]");
        SGB_REQUIRE(packed_ok(s[SGB_POSE_S_BORDER]), "bad affine border colour");
        double m[6];
        for (int j = 0; j < 6; ++j) memcpy(&m[j], &s[SGB_POSE_S_M + j], 8);
        const double det = m[0] * m[4] - m[1] * m[3];
        SGB_REQUIRE(std::isfinite(det) && det != 0.0 && std::isfinite(m[2]) && std::isfinite(m[5]), "degenerate or non-finite affine matrix");
        const sgb_aug::Inverse a = sgb_aug::invert(m);
        for (int c = 0; c < 4; ++c) {  // the map is affine: its extremes over the tile are at the corners
          const double y = (c & 1) ? (double)(rh - 1) : 0.0, x = (c & 2) ? (double)(rw - 1) : 0.0;
          const double sx = a.a11 * x + a.a12 * y + a.b1, sy = a.a21 * x + a.a22 * y + a.b2;
          SGB_REQUIRE(std::isfinite(sx) && std::isfinite(sy) && fabs(sx) < kMaxCoord && fabs(sy) < kMaxCoord, "the affine matrix maps the tile too far outside the image");
        }
      }
      max_pix = rh * rw > max_pix ? rh * rw : max_pix;
    }
  }
  SGB_REQUIRE((max_pix + kThreads - 1) / kThreads < 2147483647LL, "tile too large");
  const cudaError_t e = ensure_tables();
  SGB_REQUIRE(e == cudaSuccess, "copying the interpolation tables to the device failed");
  const dim3 grid1((unsigned)((max_pix + kThreads - 1) / kThreads), batch * 4);
  pose_point_kernel<<<grid1, kThreads, 0, (cudaStream_t)stream>>>(table, src, workspace, hsv_simd_block);
  SGB_LAUNCH_CHECK("pose_point_kernel");
  const dim3 grid2((unsigned)(((int64_t)out_size * out_size + kThreads - 1) / kThreads), batch);
  pose_out_kernel<<<grid2, kThreads, 0, (cudaStream_t)stream>>>(table, workspace, (bf16*)out, out_size, out_pitch, max_value);
  SGB_LAUNCH_CHECK("pose_out_kernel");
  return SGB_OK;
}

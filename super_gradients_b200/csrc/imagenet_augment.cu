// ImageNet train augmentation of a whole batch in ONE launch: uint8 crop windows of any sizes -> Pillow's 8-bit resize (bilinear or
// bicubic) -> flip -> two RandAugment ops -> ToTensor / Normalize -> CollateMixup (batch mode) -> bf16 NHWC batch (channels >= 3
// zero).  The arithmetic is in imagenet_augment_math.cuh and resample_math.cuh (shared with the CPU test build).
//
// One CTA owns one image and keeps it in shared memory as three uint8 planes plus one scratch plane (4 * 224 * 224 bytes = 196 KB
// at the recipe's size), so every RandAugment op, its histograms and its reductions run on chip.  The mix needs the partner image
// B - 1 - i: the CTAs of images i and B - 1 - i form a thread-block cluster of two, and after both have finished their uint8 planes
// each reads its partner's through distributed shared memory.  That keeps the whole chain in one launch with no fp32 workspace.
//
// Resize.  The horizontal pass writes the window's rows at the output width to a global workspace (h * S * 3 bytes, the uint8
// intermediate Pillow keeps), with its coefficients staged in the whole shared memory, which is still free then (column tiles
// when a very wide window needs more).  The vertical pass writes the planes; its coefficients sit in the scratch plane (row tiles).
#include <cooperative_groups.h>

#include "common.cuh"
#include "imagenet_augment_math.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 512;
constexpr int kSmemCap = 227 * 1024;  // H100's opt-in shared memory per block
constexpr int kMaxDim = 32768;        // window sides below this; coordinates and offsets stay in int32

struct Params {
  int S, out_pitch, mix;
  int fill[3];
  float mean[3], std[3];
  float lam, one_minus_lam;
  int box[4];  // yl, yh, xl, xh
};

// the three planes, then the scratch plane at a 16-byte boundary
__host__ __device__ inline size_t scratch_offset(int S) { return ((size_t)3 * S * S + 15) & ~(size_t)15; }
__host__ __device__ inline size_t planes_bytes(int S) { return (scratch_offset(S) + (size_t)S * S + 15) & ~(size_t)15; }
__host__ __device__ inline size_t smem_bytes(int S) { return planes_bytes(S) + 3 * 256 * 4 + 3 * 256 + 16; }

__device__ void resize(const Params& p, const int64_t* t, const uint8_t* __restrict__ src, uint8_t* ws, uint8_t* smem, uint8_t* planes) {
  const int S = p.S, n = S * S;
  const int h = (int)t[SGB_IN_H], w = (int)t[SGB_IN_W], filter = (int)t[SGB_IN_FILTER], flip = (int)t[SGB_IN_FLIP];
  const uint8_t* img = src + t[SGB_IN_OFFSET];
  uint8_t* mid = ws + t[SGB_IN_WS_OFFSET];
  {  // horizontal: [h][w][3] -> [h][S][3] in the workspace
    const sgb_rs::Axis ax = sgb_rs::axis(w, S, filter);
    const int kx = sgb_rs::max_taps(w, S, filter);
    const int cols = min(S, (int)(smem_bytes(S) / (4 * (size_t)(kx + 2))));
    int32_t* k = (int32_t*)smem;
    int32_t* xmin = k + cols * kx;
    int32_t* taps = xmin + cols;
    for (int c0 = 0; c0 < S; c0 += cols) {
      const int nc = min(cols, S - c0);
      for (int c = threadIdx.x; c < nc; c += blockDim.x) {
        int m;
        taps[c] = sgb_rs::coeffs(ax, c0 + c, w, k + c * kx, m);
        xmin[c] = m;
      }
      __syncthreads();
      const int row = nc * 3;
      for (int i = threadIdx.x; i < h * row; i += blockDim.x) {
        const int r = i / row, e = i - r * row, c = e / 3, ch = e - c * 3;
        const uint8_t* s = img + ((int64_t)r * w + xmin[c]) * 3 + ch;
        const int32_t* kc = k + c * kx;
        int32_t acc = 1 << (sgb_rs::kPrecisionBits - 1);
        for (int j = 0; j < taps[c]; ++j) acc += (int32_t)s[j * 3] * kc[j];
        mid[((int64_t)r * S + c0 + c) * 3 + ch] = sgb_rs::clip8(acc);
      }
      __syncthreads();  // the workspace rows are visible to the block, and the coefficients may be overwritten
    }
  }
  {  // vertical: [h][S][3] -> planes[3][S][S], flipped as it is written
    const sgb_rs::Axis ay = sgb_rs::axis(h, S, filter);
    const int ky = sgb_rs::max_taps(h, S, filter);
    const int rows = min(S, (int)((size_t)n / (4 * (size_t)(ky + 2))));
    int32_t* k = (int32_t*)(planes + scratch_offset(S));
    int32_t* ymin = k + rows * ky;
    int32_t* taps = ymin + rows;
    for (int r0 = 0; r0 < S; r0 += rows) {
      const int nr = min(rows, S - r0);
      for (int r = threadIdx.x; r < nr; r += blockDim.x) {
        int m;
        taps[r] = sgb_rs::coeffs(ay, r0 + r, h, k + r * ky, m);
        ymin[r] = m;
      }
      __syncthreads();
      const int row = S * 3;
      for (int i = threadIdx.x; i < nr * row; i += blockDim.x) {
        const int r = i / row, e = i - r * row, c = e / 3, ch = e - c * 3;
        const uint8_t* s = mid + ((int64_t)ymin[r] * S + c) * 3 + ch;
        const int32_t* kr = k + r * ky;
        int32_t acc = 1 << (sgb_rs::kPrecisionBits - 1);
        for (int j = 0; j < taps[r]; ++j) acc += (int32_t)s[(int64_t)j * row] * kr[j];
        planes[ch * n + (r0 + r) * S + (flip ? S - 1 - c : c)] = sgb_rs::clip8(acc);
      }
      __syncthreads();
    }
  }
}

__device__ void apply_op(const Params& p, const int64_t* op, uint8_t* planes, int32_t* hist, uint8_t* lut, unsigned long long* sum) {
  const int S = p.S, n = S * S, code = (int)op[0];
  const int64_t* args = op + 1;
  uint8_t* scratch = planes + scratch_offset(S);
  switch (code) {
    case SGB_IN_OP_NONE:
      return;
    case SGB_IN_OP_AFFINE: {
      double m[6];
      for (int i = 0; i < 6; ++i) m[i] = sgb_in::arg_f64(args, i);
      for (int c = 0; c < 3; ++c) {
        for (int i = threadIdx.x; i < n; i += blockDim.x) scratch[i] = planes[c * n + i];
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += blockDim.x) planes[c * n + i] = sgb_in::affine_sample(scratch, S, m, p.fill[c], i % S, i / S);
        __syncthreads();
      }
      return;
    }
    case SGB_IN_OP_AUTOCONTRAST:
    case SGB_IN_OP_EQUALIZE:
      for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) hist[i] = 0;
      __syncthreads();
      for (int i = threadIdx.x; i < 3 * n; i += blockDim.x) atomicAdd(&hist[(i / n) * 256 + planes[i]], 1);
      __syncthreads();
      if (threadIdx.x < 3) {
        if (code == SGB_IN_OP_AUTOCONTRAST)
          sgb_in::autocontrast_lut(hist + threadIdx.x * 256, lut + threadIdx.x * 256);
        else
          sgb_in::equalize_lut(hist + threadIdx.x * 256, lut + threadIdx.x * 256);
      }
      __syncthreads();
      for (int i = threadIdx.x; i < 3 * n; i += blockDim.x) planes[i] = lut[(i / n) * 256 + planes[i]];
      __syncthreads();
      return;
    case SGB_IN_OP_COLOR: {
      const float a = (float)sgb_in::arg_f64(args, 0);
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int l = sgb_in::rgb_to_l(planes[i], planes[n + i], planes[2 * n + i]);
        for (int c = 0; c < 3; ++c) planes[c * n + i] = sgb_in::blend(l, planes[c * n + i], a);
      }
      __syncthreads();
      return;
    }
    case SGB_IN_OP_SHARPNESS: {
      const float a = (float)sgb_in::arg_f64(args, 0);
      for (int c = 0; c < 3; ++c) {
        for (int i = threadIdx.x; i < n; i += blockDim.x) scratch[i] = planes[c * n + i];
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += blockDim.x) planes[c * n + i] = sgb_in::blend(sgb_in::smooth(scratch, S, i % S, i / S), scratch[i], a);
        __syncthreads();
      }
      return;
    }
    default: {  // point-wise ops; Contrast first reduces the L image to its mean
      int mean = 0;
      if (code == SGB_IN_OP_CONTRAST) {
        if (threadIdx.x == 0) *sum = 0;
        __syncthreads();
        unsigned int part = 0;
        for (int i = threadIdx.x; i < n; i += blockDim.x) part += sgb_in::rgb_to_l(planes[i], planes[n + i], planes[2 * n + i]);
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
        if ((threadIdx.x & 31) == 0) atomicAdd(sum, (unsigned long long)part);
        __syncthreads();
        mean = sgb_in::contrast_mean((int64_t)*sum, n);
      }
      for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = sgb_in::lut_value(code, args, mean, i);
      __syncthreads();
      for (int i = threadIdx.x; i < 3 * n; i += blockDim.x) planes[i] = lut[planes[i]];
      __syncthreads();
    }
  }
}

__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kThreads, 1)
    imagenet_augment_kernel(const Params p, const int64_t* __restrict__ table, const uint8_t* __restrict__ src, uint8_t* ws, int batch,
                            bf16* __restrict__ out) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ int64_t t[SGB_IN_FIELDS];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank(), pair = blockIdx.x >> 1;
  const int b = rank == 0 ? pair : batch - 1 - pair;
  const int S = p.S, n = S * S;
  uint8_t* planes = smem;
  int32_t* hist = (int32_t*)(smem + planes_bytes(S));
  uint8_t* lut = (uint8_t*)(hist + 3 * 256);
  unsigned long long* sum = (unsigned long long*)(lut + 3 * 256);
  for (int i = threadIdx.x; i < SGB_IN_FIELDS; i += blockDim.x) t[i] = table[(int64_t)b * SGB_IN_FIELDS + i];
  __syncthreads();

  resize(p, t, src, ws, smem, planes);
  for (int k = 0; k < SGB_IN_OPS; ++k) apply_op(p, t + SGB_IN_OP + k * SGB_IN_OP_FIELDS, planes, hist, lut, sum);

  cluster.sync();  // both images of the pair are final
  const uint8_t* partner = cluster.map_shared_rank(planes, rank ^ 1);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int y = i / S, x = i - y * S;
    const bool take = p.mix == 2 && y >= p.box[0] && y < p.box[1] && x >= p.box[2] && x < p.box[3];
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float xi = sgb_in::normalize(planes[c * n + i], p.mean[c], p.std[c]);
      if (p.mix == 1)
        v[c] = sgb_in::mix(xi, sgb_in::normalize(partner[c * n + i], p.mean[c], p.std[c]), p.lam, p.one_minus_lam);
      else
        v[c] = sgb_in::fadd(0.f, take ? sgb_in::normalize(partner[c * n + i], p.mean[c], p.std[c]) : xi);
    }
    bf16* o = out + ((int64_t)b * n + i) * p.out_pitch;
    for (int c0 = 0; c0 < p.out_pitch; c0 += 8) {
      __align__(16) bf16 pack[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) pack[j] = __float2bfloat16_rn(c0 + j < 3 ? v[c0 + j] : 0.f);
      *(uint4*)(o + c0) = *(const uint4*)pack;
    }
  }
  cluster.sync();  // the partner has read this CTA's planes
}

bool in_buffer(int64_t off, int64_t bytes, int64_t size) { return off >= 0 && off <= size && bytes <= size - off; }

}  // namespace

extern "C" int sgb_imagenet_augment(const int64_t* table_host, const int64_t* table, const uint8_t* src, int64_t src_bytes, uint8_t* workspace,
                                    int64_t workspace_bytes, int32_t batch, int32_t size, int32_t out_pitch, const int32_t* fill_host,
                                    const float* mean_host, const float* std_host, int32_t mix_mode, float lam, float one_minus_lam,
                                    const int32_t* box_host, sgb_bf16* out, void* stream) {
  if (batch == 0) return SGB_OK;
  SGB_REQUIRE(table_host && table && src && workspace && out && fill_host && mean_host && std_host && box_host, "null pointer");
  SGB_REQUIRE(batch > 0 && batch <= 65536 && batch % 2 == 0, "batch must be even and in [0, 65536]");
  SGB_REQUIRE(size > 0 && smem_bytes(size) <= (size_t)kSmemCap, "the output size does not fit one image per CTA in shared memory");
  SGB_REQUIRE(out_pitch >= 3 && out_pitch % 8 == 0, "output channel pitch must be >= 3 and a multiple of 8");
  SGB_REQUIRE(mix_mode >= 0 && mix_mode <= 2, "mix_mode must be 0 (none), 1 (mixup) or 2 (cutmix)");
  SGB_REQUIRE(std::isfinite(lam) && std::isfinite(one_minus_lam), "non-finite mixup weights");
  Params p = {};
  p.S = size, p.out_pitch = out_pitch, p.mix = mix_mode, p.lam = lam, p.one_minus_lam = one_minus_lam;
  for (int c = 0; c < 3; ++c) {
    SGB_REQUIRE(fill_host[c] >= 0 && fill_host[c] <= 255, "fill colour must be uint8");
    SGB_REQUIRE(std::isfinite(mean_host[c]) && std::isfinite(std_host[c]) && std_host[c] != 0.f, "bad mean or std");
    p.fill[c] = fill_host[c], p.mean[c] = mean_host[c], p.std[c] = std_host[c];
  }
  for (int i = 0; i < 4; ++i) p.box[i] = box_host[i];
  SGB_REQUIRE(p.box[0] >= 0 && p.box[0] <= p.box[1] && p.box[1] <= size && p.box[2] >= 0 && p.box[2] <= p.box[3] && p.box[3] <= size,
              "the cutmix box must lie inside the image");
  for (int b = 0; b < batch; ++b) {
    const int64_t* t = table_host + (int64_t)b * SGB_IN_FIELDS;
    const int64_t h = t[SGB_IN_H], w = t[SGB_IN_W];
    SGB_REQUIRE(h > 0 && w > 0 && h < kMaxDim && w < kMaxDim && in_buffer(t[SGB_IN_OFFSET], h * w * 3, src_bytes), "bad crop window shape, or the window lies outside the buffer");
    SGB_REQUIRE(in_buffer(t[SGB_IN_WS_OFFSET], h * size * 3, workspace_bytes), "the window's resize rows lie outside the workspace");
    SGB_REQUIRE((t[SGB_IN_FILTER] == 0 || t[SGB_IN_FILTER] == 1) && (t[SGB_IN_FLIP] == 0 || t[SGB_IN_FLIP] == 1), "filter and flip must be 0 or 1");
    const int filter = (int)t[SGB_IN_FILTER];
    SGB_REQUIRE((size_t)4 * (sgb_rs::max_taps((int)w, size, filter) + 2) <= smem_bytes(size) && (size_t)4 * (sgb_rs::max_taps((int)h, size, filter) + 2) <= (size_t)size * size,
                "the window is too large to resize to this output size (one output column's or row's coefficients do not fit in shared memory)");
    for (int k = 0; k < SGB_IN_OPS; ++k) {
      const int64_t* op = t + SGB_IN_OP + k * SGB_IN_OP_FIELDS;
      const int64_t code = op[0];
      SGB_REQUIRE(code >= SGB_IN_OP_NONE && code <= SGB_IN_OP_SHARPNESS, "unknown RandAugment op");
      if (code == SGB_IN_OP_AFFINE) {
        for (int i = 0; i < 6; ++i) {
          const double m = sgb_in::arg_f64(op + 1, i);
          SGB_REQUIRE(std::isfinite(m) && fabs(m) < 1048576.0, "affine coefficients must be finite and below 2^20");
        }
      } else if (code == SGB_IN_OP_POSTERIZE) {
        SGB_REQUIRE(op[1] >= 0 && op[1] < 8, "posterize keeps 0 to 7 bits");
      } else if (code == SGB_IN_OP_SOLARIZE) {
        SGB_REQUIRE(op[1] >= 0 && op[1] <= 256, "solarize threshold must be in [0, 256]");
      } else if (code == SGB_IN_OP_SOLARIZE_ADD) {
        SGB_REQUIRE(op[1] >= 0 && op[1] <= 255, "solarize addend must be in [0, 255]");
      } else if (code == SGB_IN_OP_BRIGHTNESS || code == SGB_IN_OP_CONTRAST || code == SGB_IN_OP_COLOR || code == SGB_IN_OP_SHARPNESS) {
        const double f = sgb_in::arg_f64(op + 1, 0);
        SGB_REQUIRE(std::isfinite(f) && fabs(f) < 1e30, "enhance factor must be finite");
      }
    }
  }
  const size_t bytes = smem_bytes(size);
  if (int rc = sgb_cuda_check(cudaFuncSetAttribute(imagenet_augment_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes), "cudaFuncSetAttribute"))
    return rc;
  imagenet_augment_kernel<<<batch, kThreads, bytes, (cudaStream_t)stream>>>(p, table, src, workspace, batch, (bf16*)out);
  SGB_LAUNCH_CHECK("imagenet_augment_kernel");
  return SGB_OK;
}

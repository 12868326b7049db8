// Memory-bound companions of the convolution GEMMs: weight layout/cast, NCHW<->NHWC, train/infer BatchNorm with
// fused residual + activation (forward and both backward passes), the QARepVGG branch algebra, pooling and axpby.
// All tensors are NHWC bf16 with channel pitch/offset; every kernel moves 16-byte vectors (8 channels) per thread with
// consecutive threads on consecutive channel vectors (coalesced), per-channel reductions go registers -> shared
// atomics -> one fp64 global atomic per channel per CTA.
#include "common.cuh"
#include "stream_ring.cuh"

namespace {

constexpr int TPB = 256;

struct V8 {
  float v[8];
};
__device__ __forceinline__ V8 ld8(const bf16* p) {
  uint4 r = *reinterpret_cast<const uint4*>(p);
  V8 o;
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f = __bfloat1622float2(h[i]);
    o.v[2 * i] = f.x;
    o.v[2 * i + 1] = f.y;
  }
  return o;
}
__device__ __forceinline__ V8 unpack8(const uint4& r) {
  V8 o;
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f = __bfloat1622float2(h[i]);
    o.v[2 * i] = f.x;
    o.v[2 * i + 1] = f.y;
  }
  return o;
}
__device__ __forceinline__ void st8(bf16* p, const V8& a) {
  uint4 r;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(a.v[2 * i], a.v[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = r;
}

inline int grid_for(int64_t work, int per_cta = TPB, int max_ctas = 132 * 8) {
  int64_t g = (work + per_cta - 1) / per_cta;
  if (g > max_ctas) g = max_ctas;
  if (g < 1) g = 1;
  return (int)g;
}

// ---------------------------------------------------------------------------------------------- weights / layout
// element i of the concatenated [K][R][S][cp] (KRSC) ++ [C][R][S][Kp] (CRSK) bf16 copies of one fp32 OIHW filter
__device__ __forceinline__ void weight_prepare_elem(const float* __restrict__ w, int K, int C, int R, int S, int cp, bf16* krsc,
                                                    bf16* crsk, float sc, int add_identity, int64_t i64, int kp = 0, int koff = 0, int etaps = 0,
                                                    int etap = 0) {
  // one filter has far fewer than 2^31 elements: 32-bit unsigned index arithmetic (a 64-bit division costs ~10x a 32-bit one)
  const uint32_t Kp = (uint32_t)((K + 7) / 8) * 8, uC = (uint32_t)C, uR = (uint32_t)R, uS = (uint32_t)S, ucp = (uint32_t)cp;
  const uint32_t n1 = (uint32_t)K * uR * uS * ucp;
  const uint32_t i = (uint32_t)i64;
  if (i < n1) {
    const uint32_t c = i % ucp;
    uint32_t t = i / ucp;
    uint32_t s = 0, r = 0;
    if (uR * uS != 1) {
      s = t % uS; t /= uS;
      r = t % uR; t /= uR;
    }
    const uint32_t k = t;
    float v = 0.f;
    if (c < uC) {
      v = w[((k * uC + c) * uR + r) * uS + s] * sc;
      if (add_identity && k == c && r == uR / 2 && s == uS / 2) v += 1.f;
    }
    // destination inside a wider filter: the 1 x 1 source is one tap of an etaps-tap filter
    krsc[etaps > 0 ? (k * (uint32_t)etaps + (uint32_t)etap) * ucp + c : i] = __float2bfloat16_rn(v);
  } else {
    const uint32_t j = i - n1;
    const uint32_t k = j % Kp;
    uint32_t t = j / Kp;
    uint32_t s = 0, r = 0;
    if (uR * uS != 1) {
      s = t % uS; t /= uS;
      r = t % uR; t /= uR;
    }
    const uint32_t c = t;
    float v = 0.f;
    if (k < (uint32_t)K) {
      v = w[((k * uC + c) * uR + r) * uS + s] * sc;
      if (add_identity && k == c && r == uR / 2 && s == uS / 2) v += 1.f;
    }
    if (kp > 0 || etaps > 0) {
      const uint32_t row = etaps > 0 ? c * (uint32_t)etaps + (uint32_t)etap : (c * uR + r) * uS + s;
      if (k < (uint32_t)K) crsk[(size_t)row * (uint32_t)(kp > 0 ? kp : (int)Kp) + (uint32_t)koff + k] = __float2bfloat16_rn(v);
    } else {
      crsk[j] = __float2bfloat16_rn(v);
    }
  }
}

__global__ void weight_prepare_kernel(const float* __restrict__ w, int K, int C, int R, int S, int cp, bf16* krsc,
                                      bf16* crsk, const float* scale, int add_identity) {
  const int Kp = ((K + 7) / 8) * 8;
  const float sc = scale ? *scale : 1.f;
  const int64_t n1 = (int64_t)K * R * S * cp;
  const int64_t n2 = crsk ? (int64_t)C * R * S * Kp : 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n1 + n2; i += (int64_t)gridDim.x * blockDim.x)
    weight_prepare_elem(w, K, C, R, S, cp, krsc, crsk, sc, add_identity, i);
}

// Elements i and i + 1 (i even) of the same index space: they share (k, r, s) in the KRSC part and (c, r, s) in the CRSK part (c_pad
// and Kp are multiples of 8), so the index arithmetic is done once and the two bf16 values leave as one 32-bit store.
__device__ __forceinline__ void weight_prepare_pair(const float* __restrict__ w, int K, int C, int R, int S, int cp, bf16* krsc, bf16* crsk, float sc,
                                                    int add_identity, int64_t i64, int kp, int koff, int etaps, int etap) {
  const uint32_t Kp = (uint32_t)((K + 7) / 8) * 8, uC = (uint32_t)C, uR = (uint32_t)R, uS = (uint32_t)S, ucp = (uint32_t)cp;
  const uint32_t n1 = (uint32_t)K * uR * uS * ucp;
  const uint32_t i = (uint32_t)i64;
  const uint32_t rs = uR * uS;
  if (i < n1) {
    const uint32_t c = i % ucp;
    uint32_t t = i / ucp;
    uint32_t s = 0, r = 0;
    if (rs != 1) {
      s = t % uS; t /= uS;
      r = t % uR; t /= uR;
    }
    const uint32_t k = t;
    const float* src = w + ((k * uC + c) * uR + r) * uS + s;  // element (k, c, r, s); (k, c + 1, r, s) is rs floats further
    float v0 = 0.f, v1 = 0.f;
    const bool centre = add_identity && r == uR / 2 && s == uS / 2;
    if (c < uC) v0 = src[0] * sc + ((centre && k == c) ? 1.f : 0.f);
    if (c + 1 < uC) v1 = src[rs] * sc + ((centre && k == c + 1) ? 1.f : 0.f);
    const uint32_t dst = etaps > 0 ? (k * (uint32_t)etaps + (uint32_t)etap) * ucp + c : i;
    *reinterpret_cast<__nv_bfloat162*>(krsc + dst) = __floats2bfloat162_rn(v0, v1);
  } else {
    const uint32_t j = i - n1;
    const uint32_t k = j % Kp;
    uint32_t t = j / Kp;
    uint32_t s = 0, r = 0;
    if (rs != 1) {
      s = t % uS; t /= uS;
      r = t % uR; t /= uR;
    }
    const uint32_t c = t;
    const float* src = w + ((k * uC + c) * uR + r) * uS + s;  // (k + 1, c, r, s) is C * rs floats further
    const bool ok0 = k < (uint32_t)K, ok1 = k + 1 < (uint32_t)K;
    const bool centre = add_identity && r == uR / 2 && s == uS / 2;
    const float v0 = ok0 ? src[0] * sc + ((centre && k == c) ? 1.f : 0.f) : 0.f;
    const float v1 = ok1 ? src[uC * rs] * sc + ((centre && k + 1 == c) ? 1.f : 0.f) : 0.f;
    if (kp > 0 || etaps > 0) {
      const uint32_t row = etaps > 0 ? c * (uint32_t)etaps + (uint32_t)etap : (c * uR + r) * uS + s;
      bf16* d = crsk + (size_t)row * (uint32_t)(kp > 0 ? kp : (int)Kp) + (uint32_t)koff + k;
      if (ok1) *reinterpret_cast<__nv_bfloat162*>(d) = __floats2bfloat162_rn(v0, v1);  // koff and k are even: 4-byte aligned
      else if (ok0) d[0] = __float2bfloat16_rn(v0);
    } else {
      *reinterpret_cast<__nv_bfloat162*>(crsk + j) = __floats2bfloat162_rn(v0, v1);
    }
  }
}

// element i of the fp32 OIHW gradient gathered from the fp32 KRSC accumulation buffer
__device__ __forceinline__ void wgrad_to_oihw_elem(const float* __restrict__ dw, int C, int R, int S, int cp, float* g,
                                                   int accumulate, int64_t i64) {
  const uint32_t i = (uint32_t)i64, uC = (uint32_t)C, uR = (uint32_t)R, uS = (uint32_t)S;
  uint32_t t = i, s = 0, r = 0;
  if (uR * uS != 1) {
    s = t % uS; t /= uS;
    r = t % uR; t /= uR;
  }
  const uint32_t c = t % uC, k = t / uC;
  const float v = dw[(((size_t)k * uR + r) * uS + s) * (uint32_t)cp + c];
  g[i] = accumulate ? g[i] + v : v;
}

__global__ void wgrad_to_oihw_kernel(const float* __restrict__ dw, int K, int C, int R, int S, int cp, float* g,
                                     int accumulate) {
  const int64_t n = (int64_t)K * C * R * S;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    wgrad_to_oihw_elem(dw, C, R, S, cp, g, accumulate, i);
}

// Batched forms: ONE launch serves every convolution of the network.  The items live in device memory; `start` is the
// exclusive prefix sum of the per-item element counts, so a thread finds its item with a binary search.
template <class Item>
__device__ __forceinline__ int find_item(const Item* items, int n, int64_t i) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (items[mid].start <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// A CTA walks chunks of BATCH_CHUNK consecutive elements; one search per chunk (thread 0, broadcast through shared memory) finds
// the item of the chunk's first element, and a thread re-searches only when its element lies past that item's end (a chunk
// straddling two filters).  The first version searched per element (8 dependent loads for ~200 items): 295 us for 19 M weights.
constexpr int BATCH_CHUNK = 2048;
// UNIT: elements per call of fn (1, or 2 when every item starts at an even offset and has an even length): fn(it, local) gets the
// offset of its first element inside the item.
template <int UNIT = 1, class Item, class Fn>
__device__ __forceinline__ void batch_walk(const Item* __restrict__ items, int n, int64_t total, Fn&& fn) {
  __shared__ int s_first;
  for (int64_t c0 = (int64_t)blockIdx.x * BATCH_CHUNK; c0 < total; c0 += (int64_t)gridDim.x * BATCH_CHUNK) {
    __syncthreads();
    if (threadIdx.x == 0) s_first = find_item(items, n, c0);
    __syncthreads();
    int idx = s_first;
    Item it = items[idx];
    int64_t end = idx + 1 < n ? items[idx + 1].start : total;
    for (int64_t i = c0 + (int64_t)threadIdx.x * UNIT; i < c0 + BATCH_CHUNK && i < total; i += (int64_t)blockDim.x * UNIT) {
      while (i >= end) {  // next filter (filters are much longer than a chunk is wide, so this runs at most a few times)
        ++idx;
        it = items[idx];
        end = idx + 1 < n ? items[idx + 1].start : total;
      }
      fn(it, i - it.start);
    }
  }
}

__global__ void __launch_bounds__(TPB) weight_prepare_batch_kernel(const SgbWeightItem* __restrict__ items, int n, int64_t total) {
  // every filter's index space has an even number of elements starting at an even offset: the walk runs over PAIRS (half the index
  // arithmetic, 32-bit stores)
  batch_walk<2>(items, n, total, [](const SgbWeightItem& it, int64_t local) {
    weight_prepare_pair(it.w, it.K, it.C, it.R, it.S, it.c_pad, (bf16*)it.krsc, (bf16*)it.crsk, it.scale ? *it.scale : 1.f, it.add_identity, local, it.kp,
                        it.koff, it.etaps, it.etap);
  });
}

__global__ void __launch_bounds__(TPB) wgrad_to_oihw_batch_kernel(const SgbWgradItem* __restrict__ items, int n, int64_t total) {
  batch_walk(items, n, total, [](const SgbWgradItem& it, int64_t local) { wgrad_to_oihw_elem(it.dw, it.C, it.R, it.S, it.c_pad, it.g, it.accumulate, local); });
}

__global__ void __launch_bounds__(256) qarep_alpha_finish_kernel(const SgbAlphaItem* __restrict__ items) {
  const SgbAlphaItem it = items[blockIdx.x];
  const float alpha = *it.alpha;
  float acc = 0.f;
  const int total = it.K * it.C;
  for (int i = threadIdx.x; i < total; i += blockDim.x) {
    const int k = i / it.C, c = i - k * it.C;
    const float g = it.dw1[(int64_t)k * it.c_pad + c];
    acc = fmaf(g, it.w1[i], acc);
    it.g_w1[i] += alpha * g;
  }
  if (it.dab) {
    for (int k = threadIdx.x; k < it.K; k += blockDim.x) {
      const float g = it.dab[k];
      if (it.bias1) acc = fmaf(g, it.bias1[k], acc);
      if (it.g_bias) it.g_bias[k] += alpha * g;
    }
  }
  __shared__ float red[256];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {  // fixed order: reproducible
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0 && it.g_alpha) *it.g_alpha += red[0];
}

__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, int N, int C, int H, int W, bf16* y, int pitch,
                                    int off, int cpad) {
  // one thread per (n, h, w, cvec) writes 8 channels; reads are strided by H*W but coalesced across w.
  const int64_t hw = (int64_t)H * W;
  const int cv = cpad / 8;
  const int64_t total = (int64_t)N * cv * hw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t pixel = i % hw;
    int64_t t = i / hw;
    int v = t % cv;
    int n = t / cv;
    V8 o;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      int c = v * 8 + e;
      o.v[e] = c < C ? x[((int64_t)n * C + c) * hw + pixel] : 0.f;
    }
    st8(y + ((int64_t)n * hw + pixel) * pitch + off + v * 8, o);
  }
}

// Patch gather.  One CTA = one output row segment (STEM_QT output pixels of one (image, output row)): the R input rows x C channels
// that feed it are staged in shared memory with coalesced fp32 reads (each input row segment is read once per output row that uses
// it: R / stride times in total), then every thread assembles 8-channel vectors from shared memory and stores them so that a warp
// writes contiguous 16-byte pieces.  (The first version gathered straight from global memory with 4-byte scattered reads: 0.9 TB/s.)
constexpr int STEM_QT = 128;
__global__ void __launch_bounds__(256) stem_patches_kernel(const float* __restrict__ x, int N, int C, int H, int W, int R, int stride, int pad,
                                                           bf16* __restrict__ y, int P, int Q, int cout) {
  extern __shared__ float srow[];  // [C][R][span]
  const int qtiles = (Q + STEM_QT - 1) / STEM_QT;
  const int qt = blockIdx.x % qtiles;
  const int p = (blockIdx.x / qtiles) % P;
  const int n = blockIdx.x / (qtiles * P);
  const int q0 = qt * STEM_QT, nq = min(STEM_QT, Q - q0);
  const int w0 = q0 * stride - pad, span = (STEM_QT - 1) * stride + R;
  const int64_t hw = (int64_t)H * W;
  for (int cr = 0; cr < C * R; ++cr) {  // one staged row per (channel, filter row): no per-element div / mod
    const int r = cr % R, c = cr / R;
    const int h = p * stride - pad + r;
    const bool hin = h >= 0 && h < H;
    const float* src = x + ((int64_t)n * C + c) * hw + (int64_t)(hin ? h : 0) * W;
    for (int j = threadIdx.x; j < span; j += blockDim.x) {
      const int w = w0 + j;
      srow[cr * span + j] = (hin && w >= 0 && w < W) ? src[w] : 0.f;
    }
  }
  // patch channel -> offset of its tap inside the staged rows, computed once per CTA (the div / mod chain per element made the
  // 7 x 7 ResNet stem gather, 160 patch channels, several times slower than its 1 GB of stores)
  int* tab = reinterpret_cast<int*>(srow + (C * R * span + 3) / 4 * 4);  // 16-byte aligned (read as int4)
  const int taps = C * R * R;
  for (int ch = threadIdx.x; ch < cout; ch += blockDim.x) {
    const int c = ch % C, rs = ch / C, r = rs / R, s2 = rs - r * R;
    tab[ch] = ch < taps ? (c * R + r) * span + s2 : -1;
  }
  __syncthreads();
  const int cv = cout / 8;
  bf16* yrow = y + (((int64_t)n * P + p) * Q + q0) * cout;
  for (int i = threadIdx.x; i < nq * cv; i += blockDim.x) {
    const int v = i % cv, q = i / cv;
    const int4 t0 = *reinterpret_cast<const int4*>(tab + v * 8), t1 = *reinterpret_cast<const int4*>(tab + v * 8 + 4);
    const int off[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
    const float* base = srow + q * stride;
    V8 o;
#pragma unroll
    for (int e = 0; e < 8; ++e) o.v[e] = off[e] >= 0 ? base[off[e]] : 0.f;
    st8(yrow + (int64_t)q * cout + v * 8, o);
  }
}

// The YOLO-NAS stem shape (3 channels, 3 x 3, stride 2, pad 1, 32 patch channels) with every index a compile-time constant: no
// integer division anywhere, one CTA per (image, output row), the 3 x 3 input rows staged with coalesced fp32 reads, each thread
// assembles whole 64-byte pixels (4 vectors) from shared memory.  The generic kernel above spent its time in div / mod chains
// (480 us for 32 x 3 x 640 x 640; the data is 157 MB in + 210 MB out = 56 us at the HBM peak).
__global__ void __launch_bounds__(256) stem_patches_c3r3s2_kernel(const float* __restrict__ x, int H, int W, bf16* __restrict__ y, int P, int Q) {
  extern __shared__ float srow[];  // [9 = (c, r)][span], span = 2 * Q + 1 (input columns -1 .. 2Q - 1)
  const int p = blockIdx.x % P, n = blockIdx.x / P;
  const int span = 2 * Q + 1;
  const int64_t hw = (int64_t)H * W;
#pragma unroll
  for (int cr = 0; cr < 9; ++cr) {
    const int c = cr / 3, r = cr % 3;
    const int h = 2 * p - 1 + r;
    const bool hin = h >= 0 && h < H;
    const float* src = x + ((int64_t)n * 3 + c) * hw + (int64_t)(hin ? h : 0) * W - 1;
    for (int j = threadIdx.x; j < span; j += 256) srow[cr * span + j] = (hin && j >= 1 && j <= W) ? src[j] : 0.f;
  }
  __syncthreads();
  bf16* yrow = y + ((int64_t)n * P + p) * Q * 32;
  // thread -> (pixel q, vector v): consecutive threads write consecutive 16-byte pieces
  for (int i = threadIdx.x; i < Q * 4; i += 256) {
    const int v = i & 3, q = i >> 2;
    V8 o;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      // patch channel ch = (r * 3 + s) * 3 + c for ch < 27; v is runtime (0..3), so select among the four constant patterns
      float val = 0.f;
#pragma unroll
      for (int vv = 0; vv < 4; ++vv) {
        const int ch = vv * 8 + e;
        if (ch < 27 && v == vv) {
          const int c = ch % 3, rs = ch / 3, r = rs / 3, s2 = rs % 3;
          val = srow[(c * 3 + r) * span + 2 * q + s2];
        }
      }
      o.v[e] = val;
    }
    st8(yrow + (int64_t)q * 32 + v * 8, o);
  }
}

__global__ void nhwc_to_nchw_kernel(const bf16* __restrict__ x, int N, int C, int H, int W, int pitch, int off,
                                    float* y) {
  const int64_t hw = (int64_t)H * W;
  const int64_t total = (int64_t)N * C * hw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t pixel = i % hw;
    int64_t t = i / hw;
    int c = t % C;
    int n = t / C;
    y[i] = __bfloat162float(x[((int64_t)n * hw + pixel) * pitch + off + c]);
  }
}

// ---------------------------------------------------------------------------------------------- channel reductions
// Generic per-channel reduction skeleton.  F::NACC sums per channel over F::NIN input tensors; F::base(j, c0) / F::pitch(j) locate
// input j; F::eval(raw[NIN], acc[NACC][8]) accumulates the contribution of 8 consecutive channels of one pixel.  The inputs stream
// through the per-thread shared-memory ring of stream_ring.cuh (64 KB per CTA, two or three CTAs per SM).
template <class F>
constexpr int red_unroll() {
  return F::NIN >= 3 ? 1 : 2;
}
template <class F>
constexpr int red_depth() {
  return 16 / (red_unroll<F>() * F::NIN);  // <= 64 KB of ring per 256-thread CTA: two or three CTAs per SM
}
template <class F>
__global__ void __launch_bounds__(TPB) chan_reduce_kernel(F f, int64_t M, int C, double* out, int out_stride) {
  constexpr int NACC = F::NACC, NIN = F::NIN, D = red_depth<F>();
  extern __shared__ __align__(16) unsigned char smem_red[];
  float* sred = reinterpret_cast<float*>(smem_red + sgb_ring::bytes<NIN, red_unroll<F>(), D, TPB>());  // [TPB][NACC*8]
  const uint32_t my_ring = smem_u32(smem_red) + (uint32_t)threadIdx.x * 16u;
  const int cvs = C / 8;
  const int cvb = cvs < TPB ? cvs : TPB;  // channel vectors per CTA pass
  const int lanes = TPB / cvb;
  const int t = threadIdx.x;
  const int pl = t / cvb, cvi = t % cvb;
  const int64_t pix_per_cta = (M + gridDim.x - 1) / gridDim.x;
  const int64_t p0 = blockIdx.x * pix_per_cta;
  int64_t p1 = p0 + pix_per_cta;
  if (p1 > M) p1 = M;
  for (int cv0 = 0; cv0 < cvs; cv0 += cvb) {
    const int cv = cv0 + cvi;
    float acc[NACC][8];
#pragma unroll
    for (int a = 0; a < NACC; ++a)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[a][e] = 0.f;
    if (pl < lanes && cv < cvs) {
      const int64_t first = p0 + pl;
      const int64_t mine = first < p1 ? (p1 - first + lanes - 1) / lanes : 0;
      const bf16* ptr[NIN];
      int64_t kstep[NIN];
#pragma unroll
      for (int j = 0; j < NIN; ++j) {
        const bf16* b = f.base(j, cv * 8);
        kstep[j] = (int64_t)lanes * f.pitch(j);
        ptr[j] = b ? b + first * f.pitch(j) : nullptr;
      }
      sgb_ring::walk<NIN, red_unroll<F>(), D, TPB>(my_ring, ptr, kstep, mine, [&](int64_t q, const uint4(&raw)[NIN]) {
        if constexpr (F::WRITES) f.evalw(first + q * lanes, cv * 8, raw, acc);  // a pass that also writes an output tensor
        else f.eval(raw, acc);
      });
    }
    // every thread parks its NACC*8 partial sums at [pl][cvi][a][e]; output j = (cvi, a, e) sums over pl (no atomics)
    __syncthreads();
    if (pl < lanes) {
#pragma unroll
      for (int a = 0; a < NACC; ++a)
#pragma unroll
        for (int e = 0; e < 8; ++e) sred[(pl * cvb + cvi) * (NACC * 8 + 1) + a * 8 + e] = acc[a][e];  // +1: conflict-free
    }
    __syncthreads();
    const int nout = cvb * NACC * 8;
    for (int j = t; j < nout; j += TPB) {
      float sum = 0.f;
      const int ci = j / (NACC * 8), a = (j / 8) % NACC, e = j % 8;
      for (int q = 0; q < lanes; ++q) sum += sred[(q * cvb + ci) * (NACC * 8 + 1) + a * 8 + e];
      const int c = (cv0 + ci) * 8 + e;
      if (c < C) atomicAdd(&out[(int64_t)a * out_stride + c], (double)sum);
    }
  }
}

template <class F>
int launch_chan_reduce(F f, int64_t M, int C, double* out, int out_stride, cudaStream_t st) {
  int cvs = C / 8;
  int cvb = cvs < TPB ? cvs : TPB;
  size_t smem = sgb_ring::bytes<F::NIN, red_unroll<F>(), red_depth<F>(), TPB>() + (size_t)(F::NACC * 8 + 1) * TPB * sizeof(float);
  static int per_sm = 0;
  if (per_sm == 0) {
    cudaFuncSetAttribute(chan_reduce_kernel<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, chan_reduce_kernel<F>, TPB, smem) != cudaSuccess || n < 1) n = 1;
    per_sm = n;
  }
  int64_t want = (M + 255) / 256;  // >= 256 pixels per CTA
  int64_t cap = (int64_t)132 * per_sm;
  if (cap > sgb_chan_grid_cap()) cap = sgb_chan_grid_cap();
  int grid = (int)(want < 1 ? 1 : (want > cap ? cap : want));
  (void)cvb;
  chan_reduce_kernel<F><<<grid, TPB, smem, st>>>(f, M, C, out, out_stride);
  SGB_LAUNCH_CHECK("chan_reduce_kernel");
  return SGB_OK;
}

struct StatsF {
  static constexpr int NACC = 2, NIN = 1;
  static constexpr bool WRITES = false;
  const bf16* x;
  int pitch_, off;
  __device__ const bf16* base(int, int c0) const { return x + off + c0; }
  __device__ int pitch(int) const { return pitch_; }
  __device__ void eval(const uint4 (&raw)[1], float (&acc)[2][8]) const {
    V8 a = unpack8(raw[0]);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      acc[0][e] += a.v[e];
      acc[1][e] += a.v[e] * a.v[e];
    }
  }
};

struct QarepMomF {
  static constexpr int NACC = 5, NIN = 2;
  static constexpr bool WRITES = false;
  const bf16 *y3, *u;
  int p3, o3, pu, ou;
  __device__ const bf16* base(int j, int c0) const { return j == 0 ? y3 + o3 + c0 : u + ou + c0; }
  __device__ int pitch(int j) const { return j == 0 ? p3 : pu; }
  __device__ void eval(const uint4 (&raw)[2], float (&acc)[5][8]) const {
    V8 a = unpack8(raw[0]), b = unpack8(raw[1]);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      acc[0][e] += a.v[e];
      acc[1][e] += a.v[e] * a.v[e];
      acc[2][e] += b.v[e];
      acc[3][e] += b.v[e] * b.v[e];
      acc[4][e] += a.v[e] * b.v[e];
    }
  }
};

// ---------------------------------------------------------------------------------------------- pooling etc.
__global__ void maxpool_fwd_kernel(const bf16* __restrict__ x, int N, int H, int W, int C, int xp, int xo, int k,
                                   int stride, int pad, bf16* y, int P, int Q, int yp, int yo, uint8_t* idx) {
  const int cvs = C / 8;
  const int64_t total = (int64_t)N * P * Q * cvs;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int cv = i % cvs;
    int64_t t = i / cvs;
    int q = t % Q; t /= Q;
    int p = t % P;
    int n = t / P;
    // torch's selection (aten max_pool2d): the first maximum in row-major order, the last NaN if there is one, and the first in-bounds
    // tap of a window that holds nothing above -inf.  Every recorded tap is therefore inside the image, which the backward kernels rely on.
    const int r0 = max(0, pad - p * stride), s0 = max(0, pad - q * stride);
    float best[8];
    int bi[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; bi[e] = r0 * k + s0; }
    for (int r = 0; r < k; ++r) {
      int h = p * stride - pad + r;
      if ((unsigned)h >= (unsigned)H) continue;
      for (int s = 0; s < k; ++s) {
        int w = q * stride - pad + s;
        if ((unsigned)w >= (unsigned)W) continue;
        V8 a = ld8(x + (((int64_t)n * H + h) * W + w) * xp + xo + cv * 8);
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (a.v[e] > best[e] || a.v[e] != a.v[e]) { best[e] = a.v[e]; bi[e] = r * k + s; }
      }
    }
    V8 o;
#pragma unroll
    for (int e = 0; e < 8; ++e) o.v[e] = best[e];
    int64_t opix = ((int64_t)n * P + p) * Q + q;
    st8(y + opix * yp + yo + cv * 8, o);
    if (idx) {
      uint2 pk;
      pk.x = bi[0] | (bi[1] << 8) | (bi[2] << 16) | (bi[3] << 24);
      pk.y = bi[4] | (bi[5] << 8) | (bi[6] << 16) | (bi[7] << 24);
      *reinterpret_cast<uint2*>(idx + opix * C + cv * 8) = pk;
    }
  }
}

// Stride-1 max-pool (the SPP pools, k = 5 / 9 / 13 over 20 x 20 maps) as two separable passes through shared memory: one CTA owns
// the H x W plane of one image and one 8-channel vector.  Pass 1: per (row, output column) the maximum over the window's columns and
// the FIRST column offset that attains it; pass 2: per output pixel the first window row whose row-maximum is the window maximum.
// Both passes take a NaN over anything and a later NaN over an earlier one, and start from the first in-bounds column / row.  The
// composition is the same element as the direct scan's (row-major order: the first maximum, else the last NaN, else the first
// in-bounds tap), which the backward routes to, at 2k instead of k^2 comparisons per output and with the plane read from HBM once
// (the direct kernel ran at 73 GB/s).
__global__ void __launch_bounds__(256) maxpool_s1_smem_kernel(const bf16* __restrict__ x, int H, int W, int C, int xp, int xo, int k, int pad, bf16* y,
                                                              int P, int Q, int yp, int yo, uint8_t* idx) {
  extern __shared__ __align__(16) unsigned char smem_mp[];
  uint4* plane = reinterpret_cast<uint4*>(smem_mp);                     // [H][W] 8 x bf16
  float* rmax = reinterpret_cast<float*>(plane + (size_t)H * W);        // [H][Q][8]
  uint8_t* rarg = reinterpret_cast<uint8_t*>(rmax + (size_t)H * Q * 8);  // [H][Q][8]
  const int cvs = C / 8, n = blockIdx.x / cvs, cv = blockIdx.x % cvs;
  const bf16* xin = x + (int64_t)n * H * W * xp + xo + cv * 8;
  for (int i = threadIdx.x; i < H * W; i += blockDim.x) plane[i] = *reinterpret_cast<const uint4*>(xin + (int64_t)i * xp);
  __syncthreads();
  for (int i = threadIdx.x; i < H * Q; i += blockDim.x) {
    const int h = i / Q, q = i - h * Q;
    const int s0 = max(0, pad - q);
    float best[8];
    int bi[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; bi[e] = s0; }
    for (int s2 = 0; s2 < k; ++s2) {
      const int w = q - pad + s2;
      if ((unsigned)w >= (unsigned)W) continue;
      const uint4 r = plane[h * W + w];
      const uint32_t ww[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float lo = __uint_as_float(ww[e] << 16), hi = __uint_as_float(ww[e] & 0xffff0000u);
        if (lo > best[2 * e] || lo != lo) { best[2 * e] = lo; bi[2 * e] = s2; }
        if (hi > best[2 * e + 1] || hi != hi) { best[2 * e + 1] = hi; bi[2 * e + 1] = s2; }
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      rmax[(size_t)i * 8 + e] = best[e];
      rarg[(size_t)i * 8 + e] = (uint8_t)bi[e];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < P * Q; i += blockDim.x) {
    const int p = i / Q, q = i - p * Q;
    const int r0 = max(0, pad - p);
    const size_t o0 = ((size_t)(p - pad + r0) * Q + q) * 8;
    float best[8];
    int bi[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; bi[e] = r0 * k + rarg[o0 + e]; }
    for (int r = 0; r < k; ++r) {
      const int h = p - pad + r;
      if ((unsigned)h >= (unsigned)H) continue;
      const size_t o = ((size_t)h * Q + q) * 8;
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (rmax[o + e] > best[e] || rmax[o + e] != rmax[o + e]) { best[e] = rmax[o + e]; bi[e] = r * k + rarg[o + e]; }
    }
    V8 ov;
#pragma unroll
    for (int e = 0; e < 8; ++e) ov.v[e] = best[e];
    const int64_t opix = ((int64_t)n * P + p) * Q + q;
    st8(y + opix * yp + yo + cv * 8, ov);
    if (idx) {
      uint2 pk;
      pk.x = bi[0] | (bi[1] << 8) | (bi[2] << 16) | (bi[3] << 24);
      pk.y = bi[4] | (bi[5] << 8) | (bi[6] << 16) | (bi[7] << 24);
      *reinterpret_cast<uint2*>(idx + opix * C + cv * 8) = pk;
    }
  }
}

// Both backward kernels take the recorded tap as it is: the forward kernels only record taps inside the image (see above).
__global__ void maxpool_bwd_kernel(const bf16* __restrict__ dy, int N, int H, int W, int C, int k, int stride, int pad,
                                   int P, int Q, int dyp, int dyo, const uint8_t* idx, float* dx) {
  const int64_t total = (int64_t)N * P * Q * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int c = i % C;
    int64_t opix = i / C;
    int64_t t = opix;
    int q = t % Q; t /= Q;
    int p = t % P;
    int n = t / P;
    int b = idx[opix * C + c];
    int r = b / k, s = b - r * k;
    int h = p * stride - pad + r, w = q * stride - pad + s;
    float g = __bfloat162float(dy[opix * dyp + dyo + c]);
    atomicAdd(dx + (((int64_t)n * H + h) * W + w) * C + c, g);
  }
}

// Strided max-pool backward as a GATHER: an input pixel lies in at most ceil(k / stride)^2 windows (4 for ResNet's 3 x 3 / stride 2);
// it sums the dy of those whose recorded arg-max tap points at it and writes bf16 once.  The scatter form above needs a zeroed fp32
// tensor, fp32 atomics and a conversion pass afterwards (0.75 ms of a ResNet-50 step at batch 256: 822 MB memset + 416 us + copy).
__global__ void __launch_bounds__(256) maxpool_bwd_gather_kernel(const bf16* __restrict__ dy, int N, int H, int W, int C, int k, int stride, int pad, int P,
                                                                 int Q, int dyp, int dyo, const uint8_t* __restrict__ idx, bf16* __restrict__ dx, int dxp) {
  const int cvs = C / 8;
  const int64_t total = (int64_t)N * H * W * cvs;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    // 32-bit index math (the host checked N * H * W < 2^31): 64-bit div / mod chains cost more than the loads here
    const unsigned pixi = (unsigned)i / (unsigned)cvs;
    const int cv = (int)((unsigned)i - pixi * (unsigned)cvs);
    const unsigned rowi = pixi / (unsigned)W;
    const int w = (int)(pixi - rowi * (unsigned)W);
    const int n = (int)(rowi / (unsigned)H);
    const int h = (int)(rowi - (unsigned)n * (unsigned)H);
    // windows p with p * stride - pad <= h <= p * stride - pad + k - 1
    int p_lo = (h + pad - k + 1 + stride - 1);
    p_lo = p_lo > 0 ? p_lo / stride : 0;
    int p_hi = (h + pad) / stride;
    if (p_hi > P - 1) p_hi = P - 1;
    int q_lo = (w + pad - k + 1 + stride - 1);
    q_lo = q_lo > 0 ? q_lo / stride : 0;
    int q_hi = (w + pad) / stride;
    if (q_hi > Q - 1) q_hi = Q - 1;
    V8 acc;
#pragma unroll
    for (int e = 0; e < 8; ++e) acc.v[e] = 0.f;
    for (int p = p_lo; p <= p_hi; ++p) {
      const int r = h - (p * stride - pad);
      for (int q = q_lo; q <= q_hi; ++q) {
        const int tap = r * k + (w - (q * stride - pad));
        const int64_t opix = ((int64_t)n * P + p) * Q + q;
        const uint2 sel = *reinterpret_cast<const uint2*>(idx + opix * C + cv * 8);
        const V8 g = ld8(dy + opix * dyp + dyo + cv * 8);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const unsigned b = ((e < 4 ? sel.x : sel.y) >> (8 * (e & 3))) & 0xffu;
          if ((int)b == tap) acc.v[e] += g.v[e];
        }
      }
    }
    st8(dx + (((int64_t)n * H + h) * W + w) * dxp + cv * 8, acc);
  }
}

__global__ void axpby_kernel(const bf16* __restrict__ x1, int p1, int o1, float a, const bf16* __restrict__ x2, int p2,
                             int o2, float b, bf16* y, int py, int oy, int64_t M, int C) {
  const int cvs = C / 8;
  const int64_t total = M * cvs;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int cv = i % cvs;
    int64_t pix = i / cvs;
    V8 u = ld8(x1 + pix * p1 + o1 + cv * 8);
    if (x2) {
      V8 v = ld8(x2 + pix * p2 + o2 + cv * 8);
#pragma unroll
      for (int e = 0; e < 8; ++e) u.v[e] = a * u.v[e] + b * v.v[e];
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) u.v[e] = a * u.v[e];
    }
    st8(y + pix * py + oy + cv * 8, u);
  }
}

__global__ void scale_add_kernel(const bf16* __restrict__ x1, int p1, int o1, const float* a_dev,
                                 const bf16* __restrict__ x2, int p2, int o2, bf16* y, int py, int oy, int64_t M, int C) {
  const float a = *a_dev;
  const int cvs = C / 8;
  const int64_t total = M * cvs;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int cv = i % cvs;
    int64_t pix = i / cvs;
    V8 u = ld8(x1 + pix * p1 + o1 + cv * 8);
    if (x2) {
      V8 v = ld8(x2 + pix * p2 + o2 + cv * 8);
#pragma unroll
      for (int e = 0; e < 8; ++e) u.v[e] = a * u.v[e] + v.v[e];
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) u.v[e] = a * u.v[e];
    }
    st8(y + pix * py + oy + cv * 8, u);
  }
}

struct DotF {
  static constexpr int NACC = 1, NIN = 2;
  static constexpr bool WRITES = false;
  const bf16 *a, *b;
  int pa, oa, pb, ob;
  __device__ const bf16* base(int j, int c0) const { return j == 0 ? a + oa + c0 : b + ob + c0; }
  __device__ int pitch(int j) const { return j == 0 ? pa : pb; }
  __device__ void eval(const uint4 (&raw)[2], float (&acc)[1][8]) const {
    V8 u = unpack8(raw[0]), v = unpack8(raw[1]);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[0][e] += u.v[e] * v.v[e];
  }
};

// y = a * x1 (+ x2) and out[c] += sum over pixels of x1 * xd in ONE pass: the backward of the learnable-alpha shortcut
// (yolo_stages.py:61-63) needs alpha * dy for the shortcut's input and sum(dy * x) for alpha; separately that was a scale pass and
// a dot pass, each reading dy.
struct ScaleAddDotF {
  static constexpr int NACC = 1, NIN = 3;
  static constexpr bool WRITES = true;
  const bf16 *x1, *xd, *x2;  // x2 may be null
  int p1, o1, pd, od, p2, o2;
  const float* a_dev;
  bf16* y;
  int py, oy;
  __device__ const bf16* base(int j, int c0) const { return j == 0 ? x1 + o1 + c0 : (j == 1 ? xd + od + c0 : (x2 ? x2 + o2 + c0 : nullptr)); }
  __device__ int pitch(int j) const { return j == 0 ? p1 : (j == 1 ? pd : p2); }
  __device__ void evalw(int64_t pix, int c0, const uint4 (&raw)[3], float (&acc)[1][8]) const {
    const float a = __ldg(a_dev);
    V8 u = unpack8(raw[0]);
    const V8 v = unpack8(raw[1]);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[0][e] = fmaf(u.v[e], v.v[e], acc[0][e]);
    if (x2) {
      const V8 w = unpack8(raw[2]);
#pragma unroll
      for (int e = 0; e < 8; ++e) u.v[e] = a * u.v[e] + w.v[e];
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) u.v[e] = a * u.v[e];
    }
    st8(y + pix * py + oy + c0, u);
  }
  __device__ void eval(const uint4 (&)[3], float (&)[1][8]) const {}
};

__global__ void f32_to_bf16_kernel(const float* __restrict__ x, bf16* y, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = __float2bfloat16_rn(x[i]);
}

__global__ void avgpool_fwd_kernel(const bf16* __restrict__ x, int N, int HW, int C, bf16* y) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  int c = i % C, n = i / C;
  float s = 0.f;
  for (int p = 0; p < HW; ++p) s += __bfloat162float(x[((int64_t)n * HW + p) * C + c]);
  y[i] = __float2bfloat16_rn(s / (float)HW);
}
__global__ void avgpool_bwd_kernel(const bf16* __restrict__ dy, int N, int HW, int C, bf16* dx) {
  const int64_t total = (int64_t)N * HW * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int c = i % C;
    int n = i / ((int64_t)HW * C);
    dx[i] = __float2bfloat16_rn(__bfloat162float(dy[n * C + c]) / (float)HW);
  }
}

}  // namespace

// ================================================================================================== C ABI
extern "C" int sgb_weight_prepare(const float* w, int K, int C, int R, int S, int c_pad, sgb_bf16* krsc,
                                  sgb_bf16* crsk, const float* scale, int add_identity, void* stream) {
  SGB_REQUIRE(w && krsc, "null pointer");
  SGB_REQUIRE(c_pad >= C && c_pad % 8 == 0, "c_pad must be >= C and a multiple of 8");
  SGB_REQUIRE(!crsk || c_pad == C, "CRSK copy requires unpadded C");
  int64_t n = (int64_t)K * R * S * c_pad + (crsk ? (int64_t)C * R * S * (((K + 7) / 8) * 8) : 0);
  weight_prepare_kernel<<<grid_for(n), TPB, 0, (cudaStream_t)stream>>>(w, K, C, R, S, c_pad, (bf16*)krsc, (bf16*)crsk,
                                                                       scale, add_identity);
  SGB_LAUNCH_CHECK("weight_prepare_kernel");
  return SGB_OK;
}

extern "C" int sgb_wgrad_to_oihw(const float* dw, int K, int C, int R, int S, int c_pad, float* g, int accumulate,
                                 void* stream) {
  SGB_REQUIRE(dw && g, "null pointer");
  wgrad_to_oihw_kernel<<<grid_for((int64_t)K * C * R * S), TPB, 0, (cudaStream_t)stream>>>(dw, K, C, R, S, c_pad, g,
                                                                                         accumulate);
  SGB_LAUNCH_CHECK("wgrad_to_oihw_kernel");
  return SGB_OK;
}

extern "C" int sgb_weight_prepare_batch(const SgbWeightItem* items_dev, int n_items, int64_t total, void* stream) {
  SGB_REQUIRE(items_dev && n_items > 0 && total > 0, "bad args");
  weight_prepare_batch_kernel<<<grid_for(total, BATCH_CHUNK), TPB, 0, (cudaStream_t)stream>>>(items_dev, n_items, total);
  SGB_LAUNCH_CHECK("weight_prepare_batch_kernel");
  return SGB_OK;
}

extern "C" int sgb_wgrad_to_oihw_batch(const SgbWgradItem* items_dev, int n_items, int64_t total, void* stream) {
  SGB_REQUIRE(items_dev && n_items > 0 && total > 0, "bad args");
  wgrad_to_oihw_batch_kernel<<<grid_for(total, BATCH_CHUNK), TPB, 0, (cudaStream_t)stream>>>(items_dev, n_items, total);
  SGB_LAUNCH_CHECK("wgrad_to_oihw_batch_kernel");
  return SGB_OK;
}

extern "C" int sgb_qarep_alpha_finish_batch(const SgbAlphaItem* items_dev, int n_items, void* stream) {
  SGB_REQUIRE(items_dev && n_items > 0, "bad args");
  qarep_alpha_finish_kernel<<<n_items, 256, 0, (cudaStream_t)stream>>>(items_dev);
  SGB_LAUNCH_CHECK("qarep_alpha_finish_kernel");
  return SGB_OK;
}

extern "C" int sgb_nchw_f32_to_nhwc_bf16(const float* x, int N, int C, int H, int W, sgb_bf16* y, int y_pitch,
                                         int y_off, int c_out, void* stream) {
  SGB_REQUIRE(x && y, "null pointer");
  SGB_REQUIRE(y_pitch % 8 == 0 && y_off % 8 == 0, "pitch/offset multiples of 8");
  SGB_REQUIRE(c_out >= C && c_out % 8 == 0, "c_out must be >= C and a multiple of 8");
  int cpad = c_out;  // channels [C, c_out) are written as zeros
  SGB_REQUIRE(y_pitch >= y_off + cpad, "slice exceeds pitch");
  nchw_to_nhwc_kernel<<<grid_for((int64_t)N * H * W * (cpad / 8)), TPB, 0, (cudaStream_t)stream>>>(x, N, C, H, W, (bf16*)y, y_pitch, y_off, cpad);
  SGB_LAUNCH_CHECK("nchw_to_nhwc_kernel");
  return SGB_OK;
}

extern "C" int sgb_stem_patches_f32(const float* x, int N, int C, int H, int W, int R, int stride, int pad, sgb_bf16* y, int P, int Q,
                                    int c_out, void* stream) {
  SGB_REQUIRE(x && y && N > 0 && C > 0 && R > 0 && stride > 0 && pad >= 0, "bad args");
  SGB_REQUIRE(c_out % 8 == 0 && c_out >= C * R * R, "c_out must be a multiple of 8 and hold C * R * R patch entries");
  SGB_REQUIRE(P == (H + 2 * pad - R) / stride + 1 && Q == (W + 2 * pad - R) / stride + 1, "P/Q inconsistent");
  if (C == 3 && R == 3 && stride == 2 && pad == 1 && c_out == 32 && H % 2 == 0 && W % 2 == 0 && (size_t)9 * (2 * Q + 1) * sizeof(float) <= 48 * 1024) {
    stem_patches_c3r3s2_kernel<<<N * P, 256, (size_t)9 * (2 * Q + 1) * sizeof(float), (cudaStream_t)stream>>>(x, H, W, (bf16*)y, P, Q);
    SGB_LAUNCH_CHECK("stem_patches_c3r3s2_kernel");
    return SGB_OK;
  }
  const size_t smem = ((size_t)C * R * ((STEM_QT - 1) * stride + R) + 3) / 4 * 4 * sizeof(float) + (size_t)c_out * sizeof(int);  // staged rows (16-byte multiple) + tap table
  SGB_REQUIRE(smem <= 48 * 1024, "patch rows do not fit shared memory");
  const int64_t ctas = (int64_t)N * P * ((Q + STEM_QT - 1) / STEM_QT);
  SGB_REQUIRE(ctas < (1ll << 31), "too many tiles");
  stem_patches_kernel<<<(int)ctas, 256, smem, (cudaStream_t)stream>>>(x, N, C, H, W, R, stride, pad, (bf16*)y, P, Q, c_out);
  SGB_LAUNCH_CHECK("stem_patches_kernel");
  return SGB_OK;
}

extern "C" int sgb_nhwc_bf16_to_nchw_f32(const sgb_bf16* x, int N, int C, int H, int W, int x_pitch, int x_off,
                                         float* y, void* stream) {
  SGB_REQUIRE(x && y, "null pointer");
  nhwc_to_nchw_kernel<<<grid_for((int64_t)N * C * H * W), TPB, 0, (cudaStream_t)stream>>>((const bf16*)x, N, C, H, W, x_pitch, x_off, y);
  SGB_LAUNCH_CHECK("nhwc_to_nchw_kernel");
  return SGB_OK;
}

extern "C" int sgb_channel_stats(const sgb_bf16* x, int64_t M, int C, int pitch, int off, double* stats,
                                 void* stream) {
  SGB_REQUIRE(x && stats && M > 0 && C > 0 && C % 8 == 0 && pitch % 8 == 0 && off % 8 == 0, "bad args");
  StatsF f{(const bf16*)x, pitch, off};
  return launch_chan_reduce(f, M, C, stats, C, (cudaStream_t)stream);
}

extern "C" int sgb_qarep_moments(const SgbQarepDesc* d, const sgb_bf16* y3, const sgb_bf16* u, double* moments,
                                 void* stream) {
  SGB_REQUIRE(d && d->M > 0 && d->C > 0 && d->C % 8 == 0 && y3 && u && moments, "bad args");
  SGB_REQUIRE(d->pitch3 % 8 == 0 && d->off3 % 8 == 0 && d->pitchu % 8 == 0 && d->offu % 8 == 0, "pitch/offset multiples of 8");
  QarepMomF f{(const bf16*)y3, (const bf16*)u, d->pitch3, d->off3, d->pitchu, d->offu};
  return launch_chan_reduce(f, d->M, d->C, moments, d->C, (cudaStream_t)stream);
}

extern "C" int sgb_maxpool_fwd(const sgb_bf16* x, int N, int H, int W, int C, int x_pitch, int x_off, int k,
                               int stride, int pad, sgb_bf16* y, int P, int Q, int y_pitch, int y_off, uint8_t* idx,
                               void* stream) {
  SGB_REQUIRE(x && y && C % 8 == 0 && x_pitch % 8 == 0 && x_off % 8 == 0 && y_pitch % 8 == 0 && y_off % 8 == 0,
              "bad args");
  SGB_REQUIRE(k * k <= 255, "kernel too large for uint8 arg-max");
  SGB_REQUIRE(P == (H + 2 * pad - k) / stride + 1 && Q == (W + 2 * pad - k) / stride + 1, "P/Q inconsistent");
  const size_t smem = (size_t)H * W * 16 + (size_t)H * Q * 8 * (sizeof(float) + 1);
  if (stride == 1 && smem <= 96 * 1024 && (int64_t)N * (C / 8) <= 1 << 20) {  // the SPP pools: separable pass through shared memory
    static bool attr = false;
    if (!attr) {
      cudaFuncSetAttribute(maxpool_s1_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
      attr = true;
    }
    maxpool_s1_smem_kernel<<<N * (C / 8), 256, smem, (cudaStream_t)stream>>>((const bf16*)x, H, W, C, x_pitch, x_off, k, pad, (bf16*)y, P, Q, y_pitch, y_off, idx);
    SGB_LAUNCH_CHECK("maxpool_s1_smem_kernel");
    return SGB_OK;
  }
  maxpool_fwd_kernel<<<grid_for((int64_t)N * P * Q * (C / 8)), TPB, 0, (cudaStream_t)stream>>>((const bf16*)x, N, H, W, C, x_pitch, x_off, k, stride, pad, (bf16*)y, P, Q, y_pitch, y_off, idx);
  SGB_LAUNCH_CHECK("maxpool_fwd_kernel");
  return SGB_OK;
}

extern "C" int sgb_maxpool_bwd(const sgb_bf16* dy, int N, int H, int W, int C, int k, int stride, int pad, int P,
                               int Q, int dy_pitch, int dy_off, const uint8_t* idx, float* dx_f32, void* stream) {
  SGB_REQUIRE(dy && idx && dx_f32, "null pointer");
  maxpool_bwd_kernel<<<grid_for((int64_t)N * P * Q * C), TPB, 0, (cudaStream_t)stream>>>((const bf16*)dy, N, H, W, C, k, stride, pad, P, Q, dy_pitch, dy_off, idx, dx_f32);
  SGB_LAUNCH_CHECK("maxpool_bwd_kernel");
  return SGB_OK;
}

extern "C" int sgb_maxpool_bwd_bf16(const sgb_bf16* dy, int N, int H, int W, int C, int k, int stride, int pad, int P, int Q, int dy_pitch,
                                    int dy_off, const uint8_t* idx, sgb_bf16* dx, int dx_pitch, void* stream) {
  SGB_REQUIRE(dy && idx && dx, "null pointer");
  SGB_REQUIRE(C % 8 == 0 && dy_pitch % 8 == 0 && dy_off % 8 == 0 && dx_pitch % 8 == 0 && dx_pitch >= C, "channels / pitches must be multiples of 8");
  SGB_REQUIRE(stride >= 1 && k >= 1 && k * k <= 255, "bad window");
  SGB_REQUIRE((int64_t)N * H * W * (C / 8) < (1ll << 32) && (int64_t)N * H * W < (1ll << 31), "tensor too large for the 32-bit index math");
  maxpool_bwd_gather_kernel<<<grid_for((int64_t)N * H * W * (C / 8), TPB * 2), 256, 0, (cudaStream_t)stream>>>((const bf16*)dy, N, H, W, C, k, stride, pad,
             P, Q, dy_pitch, dy_off, idx, (bf16*)dx, dx_pitch);
  SGB_LAUNCH_CHECK("maxpool_bwd_gather_kernel");
  return SGB_OK;
}

extern "C" int sgb_axpby(const sgb_bf16* x1, int p1, int o1, float a, const sgb_bf16* x2, int p2, int o2, float b,
                         sgb_bf16* y, int py, int oy, int64_t M, int C, void* stream) {
  SGB_REQUIRE(x1 && y && C % 8 == 0 && p1 % 8 == 0 && o1 % 8 == 0 && py % 8 == 0 && oy % 8 == 0, "bad args");
  SGB_REQUIRE(!x2 || (p2 % 8 == 0 && o2 % 8 == 0), "bad args (x2)");
  axpby_kernel<<<grid_for(M * (C / 8), TPB * 4), TPB, 0, (cudaStream_t)stream>>>((const bf16*)x1, p1, o1, a, (const bf16*)x2, p2, o2, b, (bf16*)y, py, oy, M, C);
  SGB_LAUNCH_CHECK("axpby_kernel");
  return SGB_OK;
}

extern "C" int sgb_scale_add(const sgb_bf16* x1, int p1, int o1, const float* a_dev, const sgb_bf16* x2, int p2, int o2,
                             sgb_bf16* y, int py, int oy, int64_t M, int C, void* stream) {
  SGB_REQUIRE(x1 && y && a_dev && C % 8 == 0 && p1 % 8 == 0 && o1 % 8 == 0 && py % 8 == 0 && oy % 8 == 0, "bad args");
  SGB_REQUIRE(!x2 || (p2 % 8 == 0 && o2 % 8 == 0), "bad args (x2)");
  scale_add_kernel<<<grid_for(M * (C / 8), TPB * 4), TPB, 0, (cudaStream_t)stream>>>((const bf16*)x1, p1, o1, a_dev, (const bf16*)x2, p2, o2, (bf16*)y, py, oy, M, C);
  SGB_LAUNCH_CHECK("scale_add_kernel");
  return SGB_OK;
}

extern "C" int sgb_channel_dot(const sgb_bf16* a, int pa, int oa, const sgb_bf16* b, int pb, int ob, int64_t M, int C,
                               double* out, void* stream) {
  SGB_REQUIRE(a && b && out && C % 8 == 0 && pa % 8 == 0 && oa % 8 == 0 && pb % 8 == 0 && ob % 8 == 0, "bad args");
  DotF f{(const bf16*)a, (const bf16*)b, pa, oa, pb, ob};
  return launch_chan_reduce(f, M, C, out, C, (cudaStream_t)stream);
}

extern "C" int sgb_scale_add_dot(const sgb_bf16* x1, int p1, int o1, const float* a_dev, const sgb_bf16* x2, int p2, int o2, const sgb_bf16* xd,
                                 int pd, int od, sgb_bf16* y, int py, int oy, int64_t M, int C, double* out_dot, void* stream) {
  SGB_REQUIRE(x1 && xd && y && a_dev && out_dot && M > 0 && C > 0 && C % 8 == 0, "bad args");
  SGB_REQUIRE(p1 % 8 == 0 && o1 % 8 == 0 && pd % 8 == 0 && od % 8 == 0 && py % 8 == 0 && oy % 8 == 0 && (!x2 || (p2 % 8 == 0 && o2 % 8 == 0)), "pitch/offset multiples of 8");
  ScaleAddDotF f{(const bf16*)x1, (const bf16*)xd, (const bf16*)x2, p1, o1, pd, od, p2, o2, a_dev, (bf16*)y, py, oy};
  return launch_chan_reduce(f, M, C, out_dot, C, (cudaStream_t)stream);
}

extern "C" int sgb_f32_to_bf16(const float* x, sgb_bf16* y, int64_t n, void* stream) {
  SGB_REQUIRE(x && y, "null pointer");
  f32_to_bf16_kernel<<<grid_for(n, TPB * 4), TPB, 0, (cudaStream_t)stream>>>(x, (bf16*)y, n);
  SGB_LAUNCH_CHECK("f32_to_bf16_kernel");
  return SGB_OK;
}

extern "C" int sgb_avgpool_fwd(const sgb_bf16* x, int N, int HW, int C, sgb_bf16* y, void* stream) {
  SGB_REQUIRE(x && y, "null pointer");
  avgpool_fwd_kernel<<<ceil_div((int64_t)N * C, TPB), TPB, 0, (cudaStream_t)stream>>>((const bf16*)x, N, HW, C,
                                                                                      (bf16*)y);
  SGB_LAUNCH_CHECK("avgpool_fwd_kernel");
  return SGB_OK;
}
extern "C" int sgb_avgpool_bwd(const sgb_bf16* dy, int N, int HW, int C, sgb_bf16* dx, void* stream) {
  SGB_REQUIRE(dy && dx, "null pointer");
  avgpool_bwd_kernel<<<grid_for((int64_t)N * HW * C), TPB, 0, (cudaStream_t)stream>>>((const bf16*)dy, N, HW, C,
                                                                                     (bf16*)dx);
  SGB_LAUNCH_CHECK("avgpool_bwd_kernel");
  return SGB_OK;
}

// Train / inference BatchNorm (+ residual + activation) and the QARepVGG branch algebra: forward apply, backward
// reduction and backward apply passes over NHWC bf16 tensors.
//
// All kernels share one thread mapping: a thread owns ONE 8-channel vector (16 bytes) and walks over pixels, so the
// per-channel coefficients (scale / shift / means / ...) are loaded from shared memory into registers ONCE per thread
// and the inner loop is pure 16-byte loads, FMAs and 16-byte stores; consecutive threads hold consecutive channel
// vectors of the same pixel (coalesced).  Per-channel coefficients are derived in every CTA's prologue from the fp64
// sums produced by the GEMM epilogues / reduction passes (block 0 also writes the side effects: saved statistics,
// running statistics, parameter gradients).
//
// Reference: nn.BatchNorm2d as used by modules/conv_bn_act_block.py:92-93, modules/qarepvgg_block.py:190-204,
// training/models/classification_models/resnet.py:53-84 and its autograd backward.
#include "common.cuh"
#include "stream_ring.cuh"

#include <cooperative_groups.h>

namespace {

constexpr int TPB = 256;

struct V8 {
  float v[8];
};
__device__ __forceinline__ void st8(bf16* p, const V8& a) {
  uint4 r;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(a.v[2 * i], a.v[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = r;
}

// Op interface:
//   static constexpr int NCOEF, NACC;           (NACC == 0: pure map)
//   static constexpr int NIN, UNROLL, DEPTH;    16-byte input vectors per pixel / pixels per ring slot / ring slots per thread
//   __device__ void prologue(float* sc) const;  all threads of the CTA; fills sc[NCOEF][C]
//   __device__ const bf16* base(int j, int c0) const;  address of input j at pixel 0, channel c0 (nullptr: input absent)
//   __device__ int pitch(int j, int c0) const;         its pixel pitch in elements (may depend on the channel: two-source dy)
//   __device__ void finish(int64_t pix, int c0, const uint4 (&raw)[NIN], const float (&r)[NCOEF][8], float (&acc)[NACC or 1][8]) const;
//   double* out; int out_stride;                (only when NACC > 0)
//
// Memory pipeline.  These passes are pure HBM streams, and with the per-channel coefficients in registers (up to 12 x 8 floats) a
// thread has no registers left to keep many loads in flight: at 170-190 registers one 256-thread CTA is resident per SM, and with
// 2-4 pixels x 3 vectors of plain loads per thread that is 24-49 KB in flight per SM -- the passes ran at 1.5-3 TB/s.  Every thread
// now owns a private ring of DEPTH slots in shared memory that it fills with cp.async (16 bytes, L1 bypassed) DEPTH iterations
// ahead and reads back itself: no barrier is involved (a thread only ever reads what it copied), the bytes in flight per SM are
// DEPTH x UNROLL x NIN x 4 KB (96-128 KB) whatever the register count, and channel slices of wider buffers cost nothing extra
// because every thread still forms its own addresses.  One CTA per SM (the ring is the SM's shared memory), grid <= SM count x
// resident CTAs, each CTA walks one contiguous range of pixels.
__device__ __forceinline__ V8 unpack8(const uint4& r) {
  const uint32_t w[4] = {r.x, r.y, r.z, r.w};
  V8 o;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    o.v[2 * i] = __uint_as_float(w[i] << 16);
    o.v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
  return o;
}
// Element count the statistics are taken over: the layer's pixels on every rank (SgbBnDesc / SgbQarepDesc .count, written by the
// all-reduce that also summed the statistics) or the local M; and the factor on the parameter gradients an apply pass accumulates.
template <class D>
__device__ __forceinline__ double stat_count(const D& d) {
  return d.count ? *d.count : (double)d.M;
}
template <class D>
__device__ __forceinline__ double param_scale(const D& d) {
  return d.count ? (double)d.param_scale : 1.0;
}

template <class Op>
constexpr size_t chan_ring_bytes() {
  return sgb_ring::bytes<Op::NIN, Op::UNROLL, Op::DEPTH, TPB>();
}
template <class Op>
size_t chan_smem_bytes(int C) {
  return chan_ring_bytes<Op>() + ((size_t)Op::NCOEF * C + (size_t)(Op::NACC * 8 + 1) * TPB) * sizeof(float);
}

template <class Op>
__device__ __forceinline__ void chan_body(const Op& op, const int64_t M, const int C, float* sc, const uint32_t ring) {
  constexpr int NCOEF = Op::NCOEF, NACC = Op::NACC, NIN = Op::NIN, U = Op::UNROLL, D = Op::DEPTH;
  // sc: [NCOEF][C] (+ [NACC][cvb*8] reduction scratch)
  op.prologue(sc);
  __syncthreads();
  const int cvs = C / 8;
  const int cvb = cvs < TPB ? cvs : TPB;
  const int lanes = TPB / cvb;
  const int t = threadIdx.x, pl = t / cvb, cvi = t % cvb;
  const int64_t per = (M + gridDim.x - 1) / gridDim.x;
  const int64_t p0 = blockIdx.x * per;
  const int64_t p1 = (p0 + per < M) ? p0 + per : M;
  float* sred = sc + NCOEF * C;  // [TPB][NACC * 8]: every thread's partial sums, tree-summed without atomics
  const uint32_t my_ring = ring + (uint32_t)t * 16u;  // slot (d, k, j) of this thread: + ((d * U + k) * NIN + j) * TPB * 16
  for (int cv0 = 0; cv0 < cvs; cv0 += cvb) {
    const int cv = cv0 + cvi;
    const bool active = pl < lanes && cv < cvs;
    float acc[NACC > 0 ? NACC : 1][8];
#pragma unroll
    for (int a = 0; a < (NACC > 0 ? NACC : 1); ++a)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[a][e] = 0.f;
    if (active) {
      float r[NCOEF > 0 ? NCOEF : 1][8];
#pragma unroll
      for (int k = 0; k < NCOEF; ++k)
#pragma unroll
        for (int e = 0; e < 8; ++e) r[k][e] = sc[k * C + cv * 8 + e];
      const int c0 = cv * 8;
      const int64_t first = p0 + pl;
      const int64_t mine = first < p1 ? (p1 - first + lanes - 1) / lanes : 0;  // pixels first, first + lanes, ... of this thread
      const bf16* ptr[NIN];  // this thread's pixel `first` of every input
      int64_t kstep[NIN];    // elements between two consecutive pixels of this thread
#pragma unroll
      for (int j = 0; j < NIN; ++j) {
        const bf16* b = op.base(j, c0);
        kstep[j] = (int64_t)lanes * op.pitch(j, c0);
        ptr[j] = b ? b + first * op.pitch(j, c0) : nullptr;
      }
      sgb_ring::walk<NIN, U, D, TPB>(my_ring, ptr, kstep, mine, [&](int64_t q, const uint4(&raw)[NIN]) { op.finish(first + q * lanes, c0, raw, r, acc); });
    }
    if constexpr (NACC > 0) {
      // thread t = pl * cvb + cvi stores its NACC*8 sums at [pl][cvi][a][e]; output j = (cvi, a, e) then sums over pl
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
        if (c < C) atomicAdd(&op.out[(int64_t)a * op.out_stride + c], (double)sum);
      }
    }
  }
}

// dynamic shared memory: [ring][coefficients + reduction scratch]
template <class Op>
__global__ void __launch_bounds__(TPB) chan_kernel(const Op op, const int64_t M, const int C) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  chan_body(op, M, C, reinterpret_cast<float*>(smem_raw + chan_ring_bytes<Op>()), smem_u32(smem_raw));
}

// A reduction pass and the apply pass that consumes its sums as ONE cooperative launch: grid-wide barrier in between.  Saves a
// launch (ramp-up, tail) per pair and, for the layers whose operands fit the 126 MB L2 (every 80 x 80 and smaller map of YOLO-NAS-S
// at batch 32), the apply pass's re-read of the same tensors hits L2 instead of HBM.  The sums are fp64 global atomics in both forms.
template <class OpA, class OpB>
constexpr size_t chan_ring_bytes2() {
  return chan_ring_bytes<OpA>() > chan_ring_bytes<OpB>() ? chan_ring_bytes<OpA>() : chan_ring_bytes<OpB>();
}
template <class OpA, class OpB>
__global__ void __launch_bounds__(TPB) chan_fused_kernel(const OpA a, const OpB b, const int64_t M, const int C) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* sc = reinterpret_cast<float*>(smem_raw + chan_ring_bytes2<OpA, OpB>());
  chan_body(a, M, C, sc, smem_u32(smem_raw));
  __threadfence();
  cooperative_groups::this_grid().sync();
  chan_body(b, M, C, sc, smem_u32(smem_raw));
}

static int sgb_sm_count() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return sms;
}

template <class OpA, class OpB>
int launch_chan_fused(const OpA& a, const OpB& b, int64_t M, int C, cudaStream_t st, const char* what) {
  auto tail = [&](int ncoef, int nacc) { return ((size_t)ncoef * C + (size_t)(nacc * 8 + 1) * TPB) * sizeof(float); };
  const size_t ta = tail(OpA::NCOEF, OpA::NACC), tb = tail(OpB::NCOEF, OpB::NACC);
  const size_t smem = chan_ring_bytes2<OpA, OpB>() + (ta > tb ? ta : tb);
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(chan_fused_kernel<OpA, OpB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    attr = true;
  }
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, chan_fused_kernel<OpA, OpB>, TPB, smem) != cudaSuccess || per_sm < 1)
    return sgb_cuda_check(cudaErrorCooperativeLaunchTooLarge, what);
  int64_t want = (M + 255) / 256;
  int64_t cap = (int64_t)sgb_sm_count() * per_sm;
  if (cap > sgb_chan_grid_cap()) cap = sgb_chan_grid_cap();
  const int grid = (int)(want < 1 ? 1 : (want > cap ? cap : want));
  int64_t Mv = M;
  int Cv = C;
  void* args[] = {(void*)&a, (void*)&b, (void*)&Mv, (void*)&Cv};
  return sgb_cuda_check(cudaLaunchCooperativeKernel((const void*)chan_fused_kernel<OpA, OpB>, dim3(grid), dim3(TPB), args, smem, st), what);
}

template <class Op>
int launch_chan(const Op& op, int64_t M, int C, cudaStream_t st, const char* what) {
  const size_t smem = chan_smem_bytes<Op>(C);
  static int per_sm = 0;  // resident CTAs per SM of this instantiation at its largest shared-memory footprint seen so far
  static size_t attr_smem = 0;
  if (per_sm == 0 || smem > attr_smem) {
    cudaFuncSetAttribute(chan_kernel<Op>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, chan_kernel<Op>, TPB, smem) != cudaSuccess || n < 1) n = 1;
    per_sm = n;
    attr_smem = smem;
  }
  int64_t want = (M + 255) / 256;
  int64_t cap = (int64_t)sgb_sm_count() * per_sm;
  if (cap > sgb_chan_grid_cap()) cap = sgb_chan_grid_cap();
  const int grid = (int)(want < 1 ? 1 : (want > cap ? cap : want));
  chan_kernel<Op><<<grid, TPB, smem, st>>>(op, M, C);
  return sgb_cuda_check(cudaGetLastError(), what);
}

// ============================================================================================== BatchNorm forward
// Per-channel sum / sum of squares of the stored bf16 values as a pass of the same skeleton: first half of sgb_bn_act_fwd_fused, for
// the layers whose GEMM epilogue has no register-held statistics (more than 96 output channels) -- all of them small enough at
// YOLO-NAS sizes for the apply pass's re-read to hit L2.
struct BnStatsOp {
  static constexpr int NCOEF = 0, NACC = 2;
  SgbBnDesc d;
  const bf16* x;
  double* out;
  int out_stride;
  __device__ void prologue(float*) const {}
  static constexpr int NIN = 1, UNROLL = 4, DEPTH = 4;
  __device__ const bf16* base(int, int c0) const { return x + d.x_off + c0; }
  __device__ int pitch(int, int) const { return d.x_pitch; }
  __device__ void finish(int64_t, int, const uint4 (&raw)[1], const float (&)[1][8], float (&acc)[2][8]) const {
    const V8 a = unpack8(raw[0]);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      acc[0][e] += a.v[e];
      acc[1][e] = fmaf(a.v[e], a.v[e], acc[1][e]);
    }
  }
};

struct BnFwdOp {
  static constexpr int NCOEF = 2, NACC = 0;
  SgbBnDesc d;
  const bf16 *x, *res;
  bf16* y;
  const double* stats;
  const float *gamma, *beta;
  float *rmean, *rvar, *save_mean, *save_rstd;
  double* out = nullptr;
  int out_stride = 0;
  __device__ void prologue(float* sc) const {
    const int C = d.C;
    const double M = stat_count(d);
    for (int c = threadIdx.x; c < C; c += TPB) {
      double s1 = 0, s2 = 0;
      for (int r = 0; r < d.stats_repl; ++r) {  // L2 reads: in the fused launch other CTAs produced the sums just before the grid barrier
        s1 += __ldcg(stats + (int64_t)r * 2 * C + c);
        s2 += __ldcg(stats + (int64_t)r * 2 * C + C + c);
      }
      const double mean = s1 / M;
      double var = s2 / M - mean * mean;
      if (var < 0) var = 0;
      const float rstd = (float)(1.0 / sqrt(var + (double)d.eps));
      const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
      sc[c] = g * rstd;
      sc[C + c] = b - (float)mean * g * rstd;
      if (blockIdx.x == 0) {
        save_mean[c] = (float)mean;
        save_rstd[c] = rstd;
        if (rmean) {
          const double unb = M > 1.0 ? var * M / (M - 1.0) : var;
          rmean[c] = (1.f - d.momentum) * rmean[c] + d.momentum * (float)mean;
          rvar[c] = (1.f - d.momentum) * rvar[c] + d.momentum * (float)unb;
        }
      }
    }
  }
  static constexpr int NIN = 2, UNROLL = 2, DEPTH = 4;  // 64 KB ring: two CTAs per SM
  __device__ const bf16* base(int j, int c0) const { return j == 0 ? x + d.x_off + c0 : (res ? res + d.r_off + c0 : nullptr); }
  __device__ int pitch(int j, int) const { return j == 0 ? d.x_pitch : d.r_pitch; }
  __device__ void finish(int64_t pix, int c0, const uint4 (&raw)[2], const float (&r)[2][8], float (&)[1][8]) const {
    V8 a = unpack8(raw[0]);
    struct {
      V8 rr;
    } in;
    if (res) in.rr = unpack8(raw[1]);
    if (d.sample_scale) {  // drop-path: the normalised branch of image n is scaled by 0 or 1 / keep_prob before the residual joins
      const float ss = d.sample_scale[pix / d.hw];
#pragma unroll
      for (int e = 0; e < 8; ++e) a.v[e] = apply_act(fmaf(a.v[e], r[0][e], r[1][e]) * ss + (res ? in.rr.v[e] : 0.f), d.act);
    } else if (res) {
#pragma unroll
      for (int e = 0; e < 8; ++e) a.v[e] = apply_act(fmaf(a.v[e], r[0][e], r[1][e]) + in.rr.v[e], d.act);
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) a.v[e] = apply_act(fmaf(a.v[e], r[0][e], r[1][e]), d.act);
    }
    st8(y + pix * d.y_pitch + d.y_off + c0, a);
  }
};

struct BnInferOp {
  static constexpr int NCOEF = 2, NACC = 0;
  SgbBnDesc d;
  const bf16 *x, *res;
  bf16* y;
  const float *gamma, *beta, *rmean, *rvar;
  double* out = nullptr;
  int out_stride = 0;
  __device__ void prologue(float* sc) const {
    const int C = d.C;
    for (int c = threadIdx.x; c < C; c += TPB) {
      const float rstd = rsqrtf(rvar[c] + d.eps);
      const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
      sc[c] = g * rstd;
      sc[C + c] = b - rmean[c] * g * rstd;
    }
  }
  static constexpr int NIN = 2, UNROLL = 2, DEPTH = 4;  // 64 KB ring: two CTAs per SM
  __device__ const bf16* base(int j, int c0) const { return j == 0 ? x + d.x_off + c0 : (res ? res + d.r_off + c0 : nullptr); }
  __device__ int pitch(int j, int) const { return j == 0 ? d.x_pitch : d.r_pitch; }
  __device__ void finish(int64_t pix, int c0, const uint4 (&raw)[2], const float (&r)[2][8], float (&)[1][8]) const {
    V8 a = unpack8(raw[0]);
    struct {
      V8 rr;
    } in;
    if (res) in.rr = unpack8(raw[1]);
    if (res) {
#pragma unroll
      for (int e = 0; e < 8; ++e) a.v[e] = apply_act(fmaf(a.v[e], r[0][e], r[1][e]) + in.rr.v[e], d.act);
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) a.v[e] = apply_act(fmaf(a.v[e], r[0][e], r[1][e]), d.act);
    }
    st8(y + pix * d.y_pitch + d.y_off + c0, a);
  }
};

// ============================================================================================== BatchNorm backward
// coefficient rows: 0 mean, 1 rstd, 2 scale (= gamma * rstd), 3 shift (= beta - mean * scale)
struct BnBwdRedOp {
  static constexpr int NCOEF = 4, NACC = 2;
  SgbBnDesc d;
  const bf16 *dy, *x, *y;  // y == nullptr: activation mask recomputed from x (no residual)
  const float *mean, *rstd, *gamma, *beta;
  double* out;
  int out_stride;
  __device__ void prologue(float* sc) const {
    const int C = d.C;
    for (int c = threadIdx.x; c < C; c += TPB) {
      const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
      sc[c] = mean[c];
      sc[C + c] = rstd[c];
      sc[2 * C + c] = g * rstd[c];
      sc[3 * C + c] = b - mean[c] * g * rstd[c];
    }
  }
  static constexpr int NIN = 3, UNROLL = 2, DEPTH = 5;
  __device__ const bf16* base(int j, int c0) const {
    if (j == 0) {
      if (d.dy2 && c0 >= d.dy2_split) return reinterpret_cast<const bf16*>(d.dy2) + d.dy2_off + (c0 - d.dy2_split);
      return dy + (d.dy_pitch ? d.dy_off : d.y_off) + c0;
    }
    if (j == 1) return x + d.x_off + c0;
    return y ? y + d.y_off + c0 : nullptr;
  }
  __device__ int pitch(int j, int c0) const {
    if (j == 0) return (d.dy2 && c0 >= d.dy2_split) ? d.dy2_pitch : (d.dy_pitch ? d.dy_pitch : d.y_pitch);
    return j == 1 ? d.x_pitch : d.y_pitch;
  }
  __device__ void finish(int64_t pix, int, const uint4 (&raw)[3], const float (&r)[4][8], float (&acc)[2][8]) const {
    const V8 g = unpack8(raw[0]), xv = unpack8(raw[1]);
    V8 yv;
    if (y) yv = unpack8(raw[2]);
    const float ss = d.sample_scale ? d.sample_scale[pix / d.hw] : 1.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float dz = g.v[e];
      if (d.act == SGB_ACT_RELU) {
        const float pre = y ? yv.v[e] : fmaf(xv.v[e], r[2][e], r[3][e]);  // same FMA as the forward pass
        dz = pre > 0.f ? dz : 0.f;
      }
      dz *= ss;  // gradient reaching the normalised branch (drop-path)
      acc[0][e] += dz;
      acc[1][e] = fmaf(dz, (xv.v[e] - r[0][e]) * r[1][e], acc[1][e]);
    }
  }
};

// coefficient rows: 0 mean, 1 rstd, 2 scale, 3 shift, 4 m0 (mean dz), 5 m1 (mean dz*xhat)
struct BnBwdApplyOp {
  static constexpr int NCOEF = 6, NACC = 0;
  SgbBnDesc d;
  const bf16 *dy, *x, *y;
  const float *gamma, *beta, *mean, *rstd;
  const double* sums;
  bf16 *dx, *dres;
  float *dgamma, *dbeta;
  double* out = nullptr;
  int out_stride = 0;
  __device__ void prologue(float* sc) const {
    const int C = d.C;
    const double M = stat_count(d), ps = param_scale(d);
    for (int c = threadIdx.x; c < C; c += TPB) {
      const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
      sc[c] = mean[c];
      sc[C + c] = rstd[c];
      sc[2 * C + c] = g * rstd[c];
      sc[3 * C + c] = b - mean[c] * g * rstd[c];
      const double S0 = __ldcg(sums + c), S1 = __ldcg(sums + C + c);  // L2 reads: in the fused launch other CTAs just wrote them
      sc[4 * C + c] = (float)(S0 / M);
      sc[5 * C + c] = (float)(S1 / M);
      if (blockIdx.x == 0) {
        if (dgamma) dgamma[c] += (float)(S1 * ps);
        if (dbeta) dbeta[c] += (float)(S0 * ps);
      }
    }
  }
  static constexpr int NIN = 3, UNROLL = 2, DEPTH = 5;
  __device__ const bf16* base(int j, int c0) const {
    if (j == 0) {
      if (d.dy2 && c0 >= d.dy2_split) return reinterpret_cast<const bf16*>(d.dy2) + d.dy2_off + (c0 - d.dy2_split);
      return dy + (d.dy_pitch ? d.dy_off : d.y_off) + c0;
    }
    if (j == 1) return x + d.x_off + c0;
    return y ? y + d.y_off + c0 : nullptr;
  }
  __device__ int pitch(int j, int c0) const {
    if (j == 0) return (d.dy2 && c0 >= d.dy2_split) ? d.dy2_pitch : (d.dy_pitch ? d.dy_pitch : d.y_pitch);
    return j == 1 ? d.x_pitch : d.y_pitch;
  }
  __device__ void finish(int64_t pix, int c0, const uint4 (&raw)[3], const float (&r)[6][8], float (&)[1][8]) const {
    const V8 g = unpack8(raw[0]), xv = unpack8(raw[1]);
    V8 yv;
    if (y) yv = unpack8(raw[2]);
    const float ss = d.sample_scale ? d.sample_scale[pix / d.hw] : 1.f;
    V8 o, dr;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float dz = g.v[e];
      if (d.act == SGB_ACT_RELU) {
        const float pre = y ? yv.v[e] : fmaf(xv.v[e], r[2][e], r[3][e]);
        dz = pre > 0.f ? dz : 0.f;
      }
      dr.v[e] = dz;  // the residual sees the unscaled gradient
      dz *= ss;
      const float xh = (xv.v[e] - r[0][e]) * r[1][e];
      o.v[e] = r[2][e] * (dz - r[4][e] - xh * r[5][e]);
    }
    st8(dx + pix * d.x_pitch + d.x_off + c0, o);
    if (dres) st8(dres + pix * d.r_pitch + d.r_off + c0, dr);
  }
};

// ============================================================================================== QARepVGG algebra
// y3 = conv3x3(x) (raw), u = conv1x1_{alpha*K1 + I}(x) (raw);  z = s3*(y3 - mu3) + beta3 + u + alpha*b1;
// out = act(post_bn(z)) = act(a3*y3 + au*u + c0).  See include/sgb200.h for the coefficient / moment layout.
// the five moments of (y3, u) as a pass of the same skeleton: first half of the fused forward launch (sgb_qarep_fwd_fused)
struct QarepMomOp {
  static constexpr int NCOEF = 0, NACC = 5;
  SgbQarepDesc d;
  const bf16 *y3, *u;
  double* out;
  int out_stride;
  __device__ void prologue(float*) const {}
  static constexpr int NIN = 2, UNROLL = 2, DEPTH = 4;
  __device__ const bf16* base(int j, int c0) const { return j == 0 ? y3 + d.off3 + c0 : u + d.offu + c0; }
  __device__ int pitch(int j, int) const { return j == 0 ? d.pitch3 : d.pitchu; }
  __device__ void finish(int64_t, int, const uint4 (&raw)[2], const float (&)[1][8], float (&acc)[5][8]) const {
    const V8 a = unpack8(raw[0]), b = unpack8(raw[1]);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      acc[0][e] += a.v[e];
      acc[1][e] = fmaf(a.v[e], a.v[e], acc[1][e]);
      acc[2][e] += b.v[e];
      acc[3][e] = fmaf(b.v[e], b.v[e], acc[3][e]);
      acc[4][e] = fmaf(a.v[e], b.v[e], acc[4][e]);
    }
  }
};

// RES: out = act(a3*y3 + au*u + c0) + (*res_alpha) * res -- a YOLO-NAS bottleneck's learnable shortcut (yolo_stages.py:61-63 of the
// reference: alpha * x + cv2(cv1(x))) fused into its second block's apply pass instead of a scale_add pass of its own.
template <bool RES>
struct QarepFwdOpT {
  static constexpr int NCOEF = 3, NACC = 0;
  SgbQarepDesc d;
  const bf16 *y3, *u;
  bf16* outp;
  const double* mom;
  const float *gamma3, *beta3, *ab, *gamma_p, *beta_p;
  float *rm3, *rv3, *rmp, *rvp, *coef;
  double* out = nullptr;
  int out_stride = 0;
  __device__ void prologue(float* sc) const {
    const int C = d.C;
    const double M = stat_count(d);
    for (int c = threadIdx.x; c < C; c += TPB) {
      // L2 reads: in the fused launch other CTAs produced the sums just before the grid barrier
      const double S3 = __ldcg(mom + c), S33 = __ldcg(mom + C + c), Su = __ldcg(mom + 2 * C + c), Suu = __ldcg(mom + 3 * C + c), S3u = __ldcg(mom + 4 * C + c);
      const double mu3 = S3 / M;
      double var3 = S33 / M - mu3 * mu3;
      if (var3 < 0) var3 = 0;
      const double muu = Su / M;
      double varu = Suu / M - muu * muu;
      if (varu < 0) varu = 0;
      const double cov = S3u / M - mu3 * muu;
      const double rstd3 = 1.0 / sqrt(var3 + (double)d.eps3);
      const double g3 = gamma3[c], b3 = beta3[c], abc = ab ? ab[c] : 0.0;
      const double s3 = g3 * rstd3;
      const double muz = b3 + muu + abc;
      double varz = s3 * s3 * var3 + varu + 2.0 * s3 * cov;
      if (varz < 0) varz = 0;
      double a3, au, c0, rstdz = 1.0, czy = 0.0;
      if (d.use_post_bn) {
        rstdz = 1.0 / sqrt(varz + (double)d.eps_post);
        const double gp = gamma_p[c], bp = beta_p[c];
        a3 = gp * rstdz * s3;
        au = gp * rstdz;
        c0 = gp * rstdz * (-s3 * mu3 - muu) + bp;
        czy = (s3 * var3 + cov) * rstdz * rstd3;
      } else {
        a3 = s3;
        au = 1.0;
        c0 = b3 + abc - s3 * mu3;
      }
      sc[c] = (float)a3;
      sc[C + c] = (float)au;
      sc[2 * C + c] = (float)c0;
      if (blockIdx.x == 0) {
        coef[c] = (float)mu3;
        coef[C + c] = (float)rstd3;
        coef[2 * C + c] = (float)muu;
        coef[3 * C + c] = (float)rstdz;
        coef[4 * C + c] = (float)a3;
        coef[5 * C + c] = (float)au;
        coef[6 * C + c] = (float)c0;
        coef[7 * C + c] = (float)czy;
        coef[8 * C + c] = (float)s3;
        const double unb = M > 1.0 ? M / (M - 1.0) : 1.0;
        if (rm3) {
          rm3[c] = (1.f - d.momentum) * rm3[c] + d.momentum * (float)mu3;
          rv3[c] = (1.f - d.momentum) * rv3[c] + d.momentum * (float)(var3 * unb);
        }
        if (d.use_post_bn && rmp) {
          rmp[c] = (1.f - d.momentum) * rmp[c] + d.momentum * (float)muz;
          rvp[c] = (1.f - d.momentum) * rvp[c] + d.momentum * (float)(varz * unb);
        }
      }
    }
  }
  static constexpr int NIN = RES ? 3 : 2, UNROLL = 2, DEPTH = RES ? 3 : 4;  // 64 KB ring (72 KB with the shortcut): two CTAs per SM
  __device__ const bf16* base(int j, int c0) const {
    if (j == 0) return y3 + d.off3 + c0;
    if (j == 1) return u + d.offu + c0;
    return reinterpret_cast<const bf16*>(d.res) + d.offr + c0;
  }
  __device__ int pitch(int j, int) const { return j == 0 ? d.pitch3 : (j == 1 ? d.pitchu : d.pitchr); }
  __device__ void finish(int64_t pix, int c0, const uint4 (&raw)[NIN], const float (&r)[3][8], float (&)[1][8]) const {
    V8 a = unpack8(raw[0]);
    const V8 b = unpack8(raw[1]);
#pragma unroll
    for (int e = 0; e < 8; ++e) a.v[e] = apply_act(fmaf(r[0][e], a.v[e], fmaf(r[1][e], b.v[e], r[2][e])), d.act);
    if constexpr (RES) {
      // the block's own output is rounded to bf16 first, exactly as when it was stored and re-read by a separate scale_add pass:
      // the fused form is bit-identical to the two-pass form
      const V8 x = unpack8(raw[NIN - 1]);
      const float al = __ldg(d.res_alpha);
#pragma unroll
      for (int e = 0; e < 8; ++e) a.v[e] = fmaf(al, x.v[e], __bfloat162float(__float2bfloat16_rn(a.v[e])));
    }
    st8(outp + pix * d.pitcho + d.offo + c0, a);
  }
};
using QarepFwdOp = QarepFwdOpT<false>;
using QarepFwdResOp = QarepFwdOpT<true>;

// coefficient rows: 0 mu3, 1 rstd3, 2 mu_u, 3 rstd_z, 4 a3, 5 au, 6 c0, 7 s3
struct QarepBwdRedOp {
  static constexpr int NCOEF = 8, NACC = 3;
  SgbQarepDesc d;
  const bf16 *dout, *y3, *u;
  const float* coef;  // [9][C] written by the forward
  double* out;
  int out_stride;
  __device__ void prologue(float* sc) const {
    const int C = d.C;
    for (int c = threadIdx.x; c < C; c += TPB) {
      sc[c] = coef[c];
      sc[C + c] = coef[C + c];
      sc[2 * C + c] = coef[2 * C + c];
      sc[3 * C + c] = coef[3 * C + c];
      sc[4 * C + c] = coef[4 * C + c];
      sc[5 * C + c] = coef[5 * C + c];
      sc[6 * C + c] = coef[6 * C + c];
      sc[7 * C + c] = coef[8 * C + c];
    }
  }
  static constexpr int NIN = 3, UNROLL = 2, DEPTH = 5;
  __device__ const bf16* base(int j, int c0) const {
    if (j == 0) return dout + (d.pitchd ? d.offd : d.offo) + c0;
    return j == 1 ? y3 + d.off3 + c0 : u + d.offu + c0;
  }
  __device__ int pitch(int j, int) const { return j == 0 ? (d.pitchd ? d.pitchd : d.pitcho) : (j == 1 ? d.pitch3 : d.pitchu); }
  __device__ void finish(int64_t, int, const uint4 (&raw)[3], const float (&r)[8][8], float (&acc)[3][8]) const {
    const V8 g = unpack8(raw[0]), a = unpack8(raw[1]), b = unpack8(raw[2]);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float dz = g.v[e];
      if (d.act == SGB_ACT_RELU) dz = fmaf(r[4][e], a.v[e], fmaf(r[5][e], b.v[e], r[6][e])) > 0.f ? dz : 0.f;
      const float y3c = a.v[e] - r[0][e];
      acc[0][e] += dz;
      if (d.use_post_bn) acc[1][e] = fmaf(dz, (fmaf(r[7][e], y3c, b.v[e] - r[2][e])) * r[3][e], acc[1][e]);
      acc[2][e] = fmaf(dz, y3c * r[1][e], acc[2][e]);
    }
  }
};

// coefficient rows: 0 mu3, 1 rstd3, 2 mu_u, 3 rstd_z, 4 a3, 5 au, 6 c0, 7 s3, 8 g (= gamma_p*rstd_z or 1), 9 m0, 10 m1, 11 q
struct QarepBwdApplyOp {
  static constexpr int NCOEF = 12, NACC = 0;
  SgbQarepDesc d;
  const bf16 *dout, *y3, *u;
  const float* coef;
  const double* sums;
  const float *gamma3, *gamma_p;
  bf16 *dy3, *du;
  float *dgamma3, *dbeta3, *dab, *dgamma_p, *dbeta_p;
  double* out = nullptr;
  int out_stride = 0;
  __device__ void prologue(float* sc) const {
    const int C = d.C;
    const double M = stat_count(d), ps = param_scale(d);
    for (int c = threadIdx.x; c < C; c += TPB) {
      const float rstdz = coef[3 * C + c], czy = coef[7 * C + c];
      const double T0 = __ldcg(sums + c), T1 = __ldcg(sums + C + c), T2 = __ldcg(sums + 2 * C + c);  // L2 reads (fused launch)
      const float m0 = (float)(T0 / M), m2 = (float)(T2 / M);
      float m1 = (float)(T1 / M), g, q;
      if (d.use_post_bn) {
        g = gamma_p[c] * rstdz;
        q = g * (m2 - m1 * czy);
      } else {
        g = 1.f;
        q = m2;
        m1 = 0.f;
      }
      sc[c] = coef[c];
      sc[C + c] = coef[C + c];
      sc[2 * C + c] = coef[2 * C + c];
      sc[3 * C + c] = rstdz;
      sc[4 * C + c] = coef[4 * C + c];
      sc[5 * C + c] = coef[5 * C + c];
      sc[6 * C + c] = coef[6 * C + c];
      sc[7 * C + c] = coef[8 * C + c];
      sc[8 * C + c] = g;
      sc[9 * C + c] = m0;
      sc[10 * C + c] = m1;
      sc[11 * C + c] = q;
      if (blockIdx.x == 0) {
        if (d.use_post_bn) {
          if (dgamma_p) dgamma_p[c] += (float)(T1 * ps);
          if (dbeta_p) dbeta_p[c] += (float)(T0 * ps);
          if (dgamma3) dgamma3[c] += (float)(M * (double)q * ps);
          // dbeta3 and d(alpha*b1) are exactly zero: post_bn removes any per-channel constant.
        } else {
          if (dgamma3) dgamma3[c] += (float)(T2 * ps);
          if (dbeta3) dbeta3[c] += (float)(T0 * ps);
          if (dab) dab[c] += (float)(T0 * ps);
        }
      }
    }
  }
  static constexpr int NIN = 3, UNROLL = 2, DEPTH = 5;
  __device__ const bf16* base(int j, int c0) const {
    if (j == 0) return dout + (d.pitchd ? d.offd : d.offo) + c0;
    return j == 1 ? y3 + d.off3 + c0 : u + d.offu + c0;
  }
  __device__ int pitch(int j, int) const { return j == 0 ? (d.pitchd ? d.pitchd : d.pitcho) : (j == 1 ? d.pitch3 : d.pitchu); }
  __device__ void finish(int64_t pix, int c0, const uint4 (&raw)[3], const float (&r)[12][8], float (&)[1][8]) const {
    const V8 g = unpack8(raw[0]), a = unpack8(raw[1]), b = unpack8(raw[2]);
    V8 o3, ou;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float dzp = g.v[e];
      if (d.act == SGB_ACT_RELU) dzp = fmaf(r[4][e], a.v[e], fmaf(r[5][e], b.v[e], r[6][e])) > 0.f ? dzp : 0.f;
      const float y3c = a.v[e] - r[0][e];
      const float y3h = y3c * r[1][e];
      float dz;
      if (d.use_post_bn) {
        const float zh = fmaf(r[7][e], y3c, b.v[e] - r[2][e]) * r[3][e];
        dz = r[8][e] * (dzp - r[9][e] - zh * r[10][e]);
        o3.v[e] = r[7][e] * (dz - y3h * r[11][e]);
      } else {
        dz = dzp;
        o3.v[e] = r[7][e] * (dz - r[9][e] - y3h * r[11][e]);
      }
      ou.v[e] = dz;
    }
    st8(dy3 + pix * d.pitch3 + d.off3 + c0, o3);
    st8(du + pix * d.pitchu + d.offu + c0, ou);
  }
};

int check_bn(const SgbBnDesc* d) {
  SGB_REQUIRE(d && d->M > 0 && d->C > 0, "bad desc");
  SGB_REQUIRE(d->C % 8 == 0, "C must be a multiple of 8");
  SGB_REQUIRE(d->x_pitch % 8 == 0 && d->x_off % 8 == 0 && d->y_pitch % 8 == 0 && d->y_off % 8 == 0,
              "pitch/offset multiples of 8");
  SGB_REQUIRE(d->C <= 4096, "C too large for the shared-memory coefficient cache");
  SGB_REQUIRE(!d->sample_scale || (d->hw > 0 && d->M % d->hw == 0), "drop-path: hw must divide M");
  SGB_REQUIRE(d->dy_pitch % 8 == 0 && d->dy_off % 8 == 0 && (d->dy_pitch == 0 || d->dy_pitch >= d->dy_off + (d->dy2 ? d->dy2_split : d->C)), "dy slice layout");
  SGB_REQUIRE(!d->dy2 || (d->dy2_split > 0 && d->dy2_split < d->C && d->dy2_split % 8 == 0 && d->dy2_pitch % 8 == 0 && d->dy2_off % 8 == 0 &&
                          d->dy2_pitch >= d->dy2_off + d->C - d->dy2_split && ((uintptr_t)d->dy2 & 15) == 0),
              "second dy source layout");
  SGB_REQUIRE(!d->count || (((uintptr_t)d->count & 7) == 0 && d->param_scale > 0.f && d->param_scale <= 1.f), "cross-rank count / param_scale");
  return SGB_OK;
}
int check_qarep(const SgbQarepDesc* d) {
  SGB_REQUIRE(d && d->M > 0 && d->C > 0 && d->C % 8 == 0 && d->C <= 2048, "bad desc");
  SGB_REQUIRE(d->pitch3 % 8 == 0 && d->off3 % 8 == 0 && d->pitchu % 8 == 0 && d->offu % 8 == 0 &&
                  d->pitcho % 8 == 0 && d->offo % 8 == 0 && d->pitchd % 8 == 0 && d->offd % 8 == 0,
              "pitch/offset multiples of 8");
  SGB_REQUIRE(d->pitchd == 0 || d->pitchd >= d->offd + d->C, "dout slice layout");
  SGB_REQUIRE(!d->res || (d->res_alpha && d->pitchr % 8 == 0 && d->offr % 8 == 0 && d->pitchr >= d->offr + d->C && ((uintptr_t)d->res & 15) == 0),
              "shortcut tensor layout");
  SGB_REQUIRE(!d->count || (((uintptr_t)d->count & 7) == 0 && d->param_scale > 0.f && d->param_scale <= 1.f), "cross-rank count / param_scale");
  return SGB_OK;
}

}  // namespace

extern "C" int sgb_bn_act_fwd(const SgbBnDesc* d, const sgb_bf16* x, const double* stats, const float* gamma,
                              const float* beta, float* running_mean, float* running_var, const sgb_bf16* residual,
                              sgb_bf16* y, float* save_mean, float* save_rstd, void* stream) {
  if (int rc = check_bn(d)) return rc;
  SGB_REQUIRE(x && stats && y && save_mean && save_rstd, "null pointer");
  SGB_REQUIRE(d->stats_repl >= 1, "stats_repl");
  BnFwdOp op{*d, (const bf16*)x, (const bf16*)residual, (bf16*)y, stats, gamma, beta, running_mean, running_var, save_mean, save_rstd};
  return launch_chan(op, d->M, d->C, (cudaStream_t)stream, "bn_act_fwd");
}

// sgb_channel-statistics + sgb_bn_act_fwd as ONE cooperative launch (sums, grid-wide barrier, apply): `stats` ([stats_repl][2][C]) must be
// zero on entry; the sums land in replica 0.
extern "C" int sgb_bn_act_fwd_fused(const SgbBnDesc* d, const sgb_bf16* x, double* stats, const float* gamma, const float* beta,
                                    float* running_mean, float* running_var, const sgb_bf16* residual, sgb_bf16* y, float* save_mean,
                                    float* save_rstd, void* stream) {
  if (int rc = check_bn(d)) return rc;
  SGB_REQUIRE(!d->count, "cross-rank statistics need the two-pass entry points (a collective between the passes)");
  SGB_REQUIRE(x && stats && y && save_mean && save_rstd, "null pointer");
  SGB_REQUIRE(d->stats_repl >= 1, "stats_repl");
  BnStatsOp so{*d, (const bf16*)x, stats, d->C};
  BnFwdOp op{*d, (const bf16*)x, (const bf16*)residual, (bf16*)y, stats, gamma, beta, running_mean, running_var, save_mean, save_rstd};
  return launch_chan_fused(so, op, d->M, d->C, (cudaStream_t)stream, "bn_act_fwd_fused");
}

extern "C" int sgb_bn_act_infer(const SgbBnDesc* d, const sgb_bf16* x, const float* gamma, const float* beta,
                                const float* running_mean, const float* running_var, const sgb_bf16* residual,
                                sgb_bf16* y, void* stream) {
  if (int rc = check_bn(d)) return rc;
  SGB_REQUIRE(x && y && running_mean && running_var, "null pointer");
  BnInferOp op{*d, (const bf16*)x, (const bf16*)residual, (bf16*)y, gamma, beta, running_mean, running_var};
  return launch_chan(op, d->M, d->C, (cudaStream_t)stream, "bn_act_infer");
}

extern "C" int sgb_bn_act_bwd_reduce(const SgbBnDesc* d, const sgb_bf16* dy, const sgb_bf16* x, const sgb_bf16* y,
                                     const float* gamma, const float* beta, const float* save_mean,
                                     const float* save_rstd, double* sums, void* stream) {
  if (int rc = check_bn(d)) return rc;
  SGB_REQUIRE(dy && x && save_mean && save_rstd && sums, "null pointer");
  SGB_REQUIRE(!d->sample_scale || y, "drop-path backward needs the forward output (the mask cannot be recomputed from x alone)");
  BnBwdRedOp op{*d, (const bf16*)dy, (const bf16*)x, (const bf16*)y, save_mean, save_rstd, gamma, beta, sums, d->C};
  return launch_chan(op, d->M, d->C, (cudaStream_t)stream, "bn_act_bwd_reduce");
}

extern "C" int sgb_bn_act_bwd_apply(const SgbBnDesc* d, const sgb_bf16* dy, const sgb_bf16* x, const sgb_bf16* y,
                                    const float* gamma, const float* beta, const float* save_mean,
                                    const float* save_rstd, const double* sums, sgb_bf16* dx, sgb_bf16* dresidual,
                                    float* dgamma, float* dbeta, void* stream) {
  if (int rc = check_bn(d)) return rc;
  SGB_REQUIRE(dy && x && save_mean && save_rstd && sums && dx, "null pointer");
  SGB_REQUIRE(!d->sample_scale || y, "drop-path backward needs the forward output (the mask cannot be recomputed from x alone)");
  BnBwdApplyOp op{*d, (const bf16*)dy, (const bf16*)x, (const bf16*)y, gamma, beta, save_mean, save_rstd, sums, (bf16*)dx, (bf16*)dresidual, dgamma, dbeta};
  return launch_chan(op, d->M, d->C, (cudaStream_t)stream, "bn_act_bwd_apply");
}

extern "C" int sgb_bn_act_bwd_fused(const SgbBnDesc* d, const sgb_bf16* dy, const sgb_bf16* x, const sgb_bf16* y, const float* gamma,
                                    const float* beta, const float* save_mean, const float* save_rstd, double* sums, sgb_bf16* dx,
                                    sgb_bf16* dresidual, float* dgamma, float* dbeta, void* stream) {
  if (int rc = check_bn(d)) return rc;
  SGB_REQUIRE(!d->count, "cross-rank statistics need the two-pass entry points (a collective between the passes)");
  SGB_REQUIRE(dy && x && save_mean && save_rstd && sums && dx, "null pointer");
  SGB_REQUIRE(!d->sample_scale || y, "drop-path backward needs the forward output (the mask cannot be recomputed from x alone)");
  BnBwdRedOp ra{*d, (const bf16*)dy, (const bf16*)x, (const bf16*)y, save_mean, save_rstd, gamma, beta, sums, d->C};
  BnBwdApplyOp ap{*d, (const bf16*)dy, (const bf16*)x, (const bf16*)y, gamma, beta, save_mean, save_rstd, sums, (bf16*)dx, (bf16*)dresidual, dgamma, dbeta};
  return launch_chan_fused(ra, ap, d->M, d->C, (cudaStream_t)stream, "bn_act_bwd_fused");
}

extern "C" int sgb_qarep_fwd(const SgbQarepDesc* d, const sgb_bf16* y3, const sgb_bf16* u, const double* moments,
                             const float* gamma3, const float* beta3, const float* bias1_alpha, const float* gamma_p,
                             const float* beta_p, float* rm3, float* rv3, float* rm_p, float* rv_p, sgb_bf16* out,
                             float* coef, void* stream) {
  if (int rc = check_qarep(d)) return rc;
  SGB_REQUIRE(y3 && u && moments && gamma3 && beta3 && out && coef, "null pointer");
  SGB_REQUIRE(!d->use_post_bn || (gamma_p && beta_p), "post_bn parameters missing");
  if (d->res) {
    QarepFwdResOp op{*d, (const bf16*)y3, (const bf16*)u, (bf16*)out, moments, gamma3, beta3, bias1_alpha, gamma_p, beta_p, rm3, rv3, rm_p, rv_p, coef};
    return launch_chan(op, d->M, d->C, (cudaStream_t)stream, "qarep_fwd (shortcut)");
  }
  QarepFwdOp op{*d, (const bf16*)y3, (const bf16*)u, (bf16*)out, moments, gamma3, beta3, bias1_alpha, gamma_p, beta_p, rm3, rv3, rm_p, rv_p, coef};
  return launch_chan(op, d->M, d->C, (cudaStream_t)stream, "qarep_fwd");
}

extern "C" int sgb_qarep_fwd_fused(const SgbQarepDesc* d, const sgb_bf16* y3, const sgb_bf16* u, double* moments, const float* gamma3,
                                   const float* beta3, const float* bias1_alpha, const float* gamma_p, const float* beta_p, float* rm3, float* rv3,
                                   float* rm_p, float* rv_p, sgb_bf16* out, float* coef, void* stream) {
  if (int rc = check_qarep(d)) return rc;
  SGB_REQUIRE(!d->count, "cross-rank statistics need the two-pass entry points (a collective between the passes)");
  SGB_REQUIRE(y3 && u && moments && gamma3 && beta3 && out && coef, "null pointer");
  SGB_REQUIRE(!d->use_post_bn || (gamma_p && beta_p), "post_bn parameters missing");
  QarepMomOp mo{*d, (const bf16*)y3, (const bf16*)u, moments, d->C};
  if (d->res) {
    QarepFwdResOp op{*d, (const bf16*)y3, (const bf16*)u, (bf16*)out, moments, gamma3, beta3, bias1_alpha, gamma_p, beta_p, rm3, rv3, rm_p, rv_p, coef};
    return launch_chan_fused(mo, op, d->M, d->C, (cudaStream_t)stream, "qarep_fwd_fused (shortcut)");
  }
  QarepFwdOp op{*d, (const bf16*)y3, (const bf16*)u, (bf16*)out, moments, gamma3, beta3, bias1_alpha, gamma_p, beta_p, rm3, rv3, rm_p, rv_p, coef};
  return launch_chan_fused(mo, op, d->M, d->C, (cudaStream_t)stream, "qarep_fwd_fused");
}

extern "C" int sgb_qarep_bwd_reduce(const SgbQarepDesc* d, const sgb_bf16* dout, const sgb_bf16* out,
                                    const sgb_bf16* y3, const sgb_bf16* u, const float* coef, double* sums,
                                    void* stream) {
  (void)out;
  if (int rc = check_qarep(d)) return rc;
  SGB_REQUIRE(dout && y3 && u && coef && sums, "null pointer");
  QarepBwdRedOp op{*d, (const bf16*)dout, (const bf16*)y3, (const bf16*)u, coef, sums, d->C};
  return launch_chan(op, d->M, d->C, (cudaStream_t)stream, "qarep_bwd_reduce");
}

extern "C" int sgb_qarep_bwd_apply(const SgbQarepDesc* d, const sgb_bf16* dout, const sgb_bf16* out,
                                   const sgb_bf16* y3, const sgb_bf16* u, const float* coef, const double* sums,
                                   const float* gamma3, const float* gamma_p, sgb_bf16* dy3, sgb_bf16* du,
                                   float* dgamma3, float* dbeta3, float* dbias1a, float* dgamma_p, float* dbeta_p,
                                   void* stream) {
  (void)out;
  if (int rc = check_qarep(d)) return rc;
  SGB_REQUIRE(dout && y3 && u && coef && sums && gamma3 && dy3 && du, "null pointer");
  SGB_REQUIRE(!d->use_post_bn || gamma_p, "gamma_p missing");
  QarepBwdApplyOp op{*d, (const bf16*)dout, (const bf16*)y3, (const bf16*)u, coef, sums, gamma3, gamma_p, (bf16*)dy3, (bf16*)du, dgamma3, dbeta3, dbias1a, dgamma_p, dbeta_p};
  return launch_chan(op, d->M, d->C, (cudaStream_t)stream, "qarep_bwd_apply");
}

extern "C" int sgb_qarep_bwd_fused(const SgbQarepDesc* d, const sgb_bf16* dout, const sgb_bf16* y3, const sgb_bf16* u, const float* coef,
                                   double* sums, const float* gamma3, const float* gamma_p, sgb_bf16* dy3, sgb_bf16* du, float* dgamma3,
                                   float* dbeta3, float* dbias1a, float* dgamma_p, float* dbeta_p, void* stream) {
  if (int rc = check_qarep(d)) return rc;
  SGB_REQUIRE(!d->count, "cross-rank statistics need the two-pass entry points (a collective between the passes)");
  SGB_REQUIRE(dout && y3 && u && coef && sums && gamma3 && dy3 && du, "null pointer");
  SGB_REQUIRE(!d->use_post_bn || gamma_p, "gamma_p missing");
  QarepBwdRedOp ra{*d, (const bf16*)dout, (const bf16*)y3, (const bf16*)u, coef, sums, d->C};
  QarepBwdApplyOp ap{*d, (const bf16*)dout, (const bf16*)y3, (const bf16*)u, coef, sums, gamma3, gamma_p, (bf16*)dy3, (bf16*)du, dgamma3, dbeta3, dbias1a, dgamma_p, dbeta_p};
  return launch_chan_fused(ra, ap, d->M, d->C, (cudaStream_t)stream, "qarep_bwd_fused");
}

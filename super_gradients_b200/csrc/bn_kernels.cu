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
#include "sm100_host.h"
#include "sm100_ptx.cuh"
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

// Grid of chan_fused_kernel<OpA, OpB> over M pixels of C channels (its dynamic shared memory in *smem), or a negative error code.  The
// grid fixes which pixels every fp32 partial sum covers: the stem kernels that recompute the operands use it to sum in the same order.
template <class OpA, class OpB>
int chan_fused_grid(int64_t M, int C, size_t* smem, const char* what) {
  auto tail = [&](int ncoef, int nacc) { return ((size_t)ncoef * C + (size_t)(nacc * 8 + 1) * TPB) * sizeof(float); };
  const size_t ta = tail(OpA::NCOEF, OpA::NACC), tb = tail(OpB::NCOEF, OpB::NACC);
  *smem = chan_ring_bytes2<OpA, OpB>() + (ta > tb ? ta : tb);
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(chan_fused_kernel<OpA, OpB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    attr = true;
  }
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, chan_fused_kernel<OpA, OpB>, TPB, *smem) != cudaSuccess || per_sm < 1)
    return sgb_cuda_check(cudaErrorCooperativeLaunchTooLarge, what);
  int64_t want = (M + 255) / 256;
  int64_t cap = (int64_t)sgb_sm_count() * per_sm;
  if (cap > sgb_chan_grid_cap()) cap = sgb_chan_grid_cap();
  return (int)(want < 1 ? 1 : (want > cap ? cap : want));
}

template <class OpA, class OpB>
int launch_chan_fused(const OpA& a, const OpB& b, int64_t M, int C, cudaStream_t st, const char* what) {
  size_t smem = 0;
  const int grid = chan_fused_grid<OpA, OpB>(M, C, &smem, what);
  if (grid < 0) return grid;
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
// The per-element arithmetic of the passes below, shared with the stem kernels that recompute y3 / u (stem_qarep_kernel): r(k) is
// coefficient row k of the element's channel, acc[a] its running sum a.
__device__ __forceinline__ void qarep_mom(float y3, float u, float* acc) {
  acc[0] += y3;
  acc[1] = fmaf(y3, y3, acc[1]);
  acc[2] += u;
  acc[3] = fmaf(u, u, acc[3]);
  acc[4] = fmaf(y3, u, acc[4]);
}
// out = act(a3 * y3 + au * u + c0) (coefficient rows 0 a3, 1 au, 2 c0)
template <class R>
__device__ __forceinline__ float qarep_out(float y3, float u, R r, int act) {
  return apply_act(fmaf(r(0), y3, fmaf(r(1), u, r(2))), act);
}
// T0 += dzp, T1 += dzp * zhat, T2 += dzp * y3hat (QarepBwdRedOp's coefficient rows)
template <class R>
__device__ __forceinline__ void qarep_bwd_sums(const SgbQarepDesc& d, float g, float y3, float u, R r, float* acc) {
  float dz = g;
  if (d.act == SGB_ACT_RELU) dz = fmaf(r(4), y3, fmaf(r(5), u, r(6))) > 0.f ? dz : 0.f;
  const float y3c = y3 - r(0);
  acc[0] += dz;
  if (d.use_post_bn) acc[1] = fmaf(dz, (fmaf(r(7), y3c, u - r(2))) * r(3), acc[1]);
  acc[2] = fmaf(dz, y3c * r(1), acc[2]);
}
// dy3, du of one element (QarepBwdApplyOp's coefficient rows)
template <class R>
__device__ __forceinline__ void qarep_bwd_grads(const SgbQarepDesc& d, float g, float y3, float u, R r, float& o3, float& ou) {
  float dzp = g;
  if (d.act == SGB_ACT_RELU) dzp = fmaf(r(4), y3, fmaf(r(5), u, r(6))) > 0.f ? dzp : 0.f;
  const float y3c = y3 - r(0);
  const float y3h = y3c * r(1);
  float dz;
  if (d.use_post_bn) {
    const float zh = fmaf(r(7), y3c, u - r(2)) * r(3);
    dz = r(8) * (dzp - r(9) - zh * r(10));
    o3 = r(7) * (dz - y3h * r(11));
  } else {
    dz = dzp;
    o3 = r(7) * (dz - r(9) - y3h * r(11));
  }
  ou = dz;
}

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
      float s[5] = {acc[0][e], acc[1][e], acc[2][e], acc[3][e], acc[4][e]};
      qarep_mom(a.v[e], b.v[e], s);
#pragma unroll
      for (int k = 0; k < 5; ++k) acc[k][e] = s[k];
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
    for (int e = 0; e < 8; ++e) a.v[e] = qarep_out(a.v[e], b.v[e], [&](int k) { return r[k][e]; }, d.act);
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
      float s[3] = {acc[0][e], acc[1][e], acc[2][e]};
      qarep_bwd_sums(d, g.v[e], a.v[e], b.v[e], [&](int k) { return r[k][e]; }, s);
#pragma unroll
      for (int k = 0; k < 3; ++k) acc[k][e] = s[k];
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
    for (int e = 0; e < 8; ++e) qarep_bwd_grads(d, g.v[e], a.v[e], b.v[e], [&](int k) { return r[k][e]; }, o3.v[e], ou.v[e]);
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

// ============================================================================================== QARepVGG stem on patches
// The train-mode stem (functional._QARepVGGStem) is ONE 1 x 1 GEMM over 32 gathered patch channels: [y3 | u] = xp @ W^T with
// W = [K3 ; centre(K1)] ([2K][32] bf16).  Storing [y3 | u] costs 2K bf16 per pixel written once and read by four passes; recomputing
// it costs two k16 wgmma steps per 128-pixel chunk against a filter that stays in shared memory.  So every pass of the block
// recomputes y3 / u from xp instead of reading them, and computes exactly what the stored-operand pass computes:
//   - the GEMM is conv_wgmma_kernel's for that shape (the same two k16 steps in the same order, fp32 accumulators rounded to bf16), so
//     the recomputed values are bit-equal to the stored ones;
//   - the values then go through shared memory to chan_body's thread mapping (a thread owns one 8-channel vector, its coefficients in
//     registers, and every lanes-th pixel of the CTA's range) and the Ops' own per-element code;
//   - the reductions (STEM_MOM, STEM_BRED) split the pixels into the same contiguous ranges as the fused chan launch they replace
//     (chan_fused_grid) and sum in its order -- per thread in pixel order, then over the lanes in order, one fp64 atomic per channel
//     and range -- so the sums, and with them the coefficients, the output and the gradients, are those of the stored-operand path.
//     STEM_GEMM   [y3 | u] written out (a test's view of what the other modes recompute)
//     STEM_MOM    the five moments of QarepMomOp                    (forward, phase 1)
//     STEM_FWD    out = act(a3 y3 + au u + c0), QarepFwdOp's prologue (forward, phase 2)
//     STEM_BRED   T0..T2 of QarepBwdRedOp from dout                  (backward, phase 1)
//     STEM_BAPPLY dy3 | du of QarepBwdApplyOp, its prologue's parameter gradients (backward, phase 2)
// CTA of three warpgroups, persistent over ranges of pixels walked in 128-pixel chunks: warpgroup 0 is the TMA producer (the filter
// once, then per chunk the xp rows and, backward, the dout rows into a ring of stages); warpgroups 1-2 run the wgmma over 64 rows each,
// park the rounded tile in shared memory, and then process it in chan_body's mapping.
enum StemMode { STEM_GEMM, STEM_MOM, STEM_FWD, STEM_BRED, STEM_BAPPLY };
constexpr int STEM_THREADS = 384, STEM_BM = 128, STEM_KP = 32, STEM_STAGES = 6;

struct StemGemmOp {  // STEM_GEMM: [y3 | u] to y ([M][2K] bf16)
  static constexpr int NCOEF = 0, NACC = 0;
  bf16* y;
  double* out = nullptr;
  int out_stride = 0;
  __device__ void prologue(float*) const {}
};

template <int KOUT, int MODE, class Op>
struct StemLayout {
  static constexpr int BN = 2 * KOUT;
  static constexpr int YP = BN + 8;  // row pitch of the parked tile (elements): 16-byte rows, conflict-free fragment stores
  static constexpr bool DOUT = MODE == STEM_BRED || MODE == STEM_BAPPLY;
  static constexpr int NACC = Op::NACC;
  static constexpr uint32_t A_BYTES = STEM_BM * STEM_KP * 2;  // 128 rows x 64 bytes, 64B swizzle
  static constexpr uint32_t G_BYTES = DOUT ? STEM_BM * KOUT * 2 : 0;
  static constexpr uint32_t STAGE = (A_BYTES + G_BYTES + 1023u) & ~1023u;
  static constexpr uint32_t W_BYTES = (BN * STEM_KP * 2 + 1023u) & ~1023u;
  static constexpr uint32_t Y_BYTES = STEM_BM * YP * 2;
  static constexpr uint32_t CTRL = 8u * (2 * STEM_STAGES + 1);
  static size_t smem() {
    return 1024 + W_BYTES + STEM_STAGES * STAGE + Y_BYTES + CTRL + ((size_t)Op::NCOEF * KOUT + (size_t)(NACC * 8 + 1) * TPB) * sizeof(float);
  }
};

__device__ __forceinline__ void stem_consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Pixels [b * per, min((b + 1) * per, M)) form range b, b = 0 .. nranges - 1; CTAs take ranges blockIdx.x, + gridDim.x, ...
template <int KOUT, int MODE, class Op>
__global__ void __launch_bounds__(STEM_THREADS, 1)
stem_qarep_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_g,
                  const Op op, const SgbQarepDesc d, const int64_t M, const int64_t per, const int nranges) {
  using Lay = StemLayout<KOUT, MODE, Op>;
  constexpr int BN = Lay::BN, YP = Lay::YP, NACC = Lay::NACC, NCOEF = Op::NCOEF, JB = KOUT / 8;
  constexpr int CVB = KOUT / 8, LANES = TPB / CVB;  // chan_body's mapping for C = KOUT: one channel-vector pass
  extern __shared__ __align__(16) unsigned char smem_raw[];  // the 64B-swizzled operands want 1024-byte alignment: rounded up here
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t s_w = base, s_stage0 = base + Lay::W_BYTES, s_y = s_stage0 + STEM_STAGES * Lay::STAGE, ctrl = s_y + Lay::Y_BYTES;
  auto full_bar = [&](int s) { return ctrl + 8u * s; };
  auto empty_bar = [&](int s) { return ctrl + 8u * (STEM_STAGES + s); };
  const uint32_t w_bar = ctrl + 8u * 2 * STEM_STAGES;
  auto gen = [&](uint32_t a) { return smem_raw + (a - smem_u32(smem_raw)); };
  bf16* ytile = reinterpret_cast<bf16*>(gen(s_y));                  // [128][YP]: y3 in columns [0, K), u in [K, 2K)
  float* sc = reinterpret_cast<float*>(gen(ctrl + Lay::CTRL));      // [NCOEF][KOUT] coefficients
  float* sred = sc + NCOEF * KOUT;                                   // [TPB][NACC * 8 + 1]: chan_body's reduction scratch

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STEM_STAGES; ++s) {
      sm100::mbar_init(full_bar(s), 1);
      sm100::mbar_init(empty_bar(s), 8);  // one arrival per consumer warp
    }
    sm100::mbar_init(w_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  if (threadIdx.x < TPB) op.prologue(sc);  // the Op's prologue strides its channels by TPB (block 0: the side effects, once)
  __syncthreads();

  if (warp == 0) {
    if (sm100::elect_one()) {
      sm100::mbar_expect_tx(w_bar, BN * STEM_KP * 2);
      sm100::tma_load_2d(s_w, &map_w, w_bar, 0, 0);
      int stg = 0;
      uint32_t par = 1;  // the first pass through the ring is free
      for (int b = blockIdx.x; b < nranges; b += gridDim.x) {
        const int64_t p0 = (int64_t)b * per, p1 = p0 + per < M ? p0 + per : M;
        for (int64_t s0 = p0; s0 < p1; s0 += STEM_BM) {
          sm100::mbar_wait(empty_bar(stg), par);
          const uint32_t sa = s_stage0 + stg * Lay::STAGE;
          sm100::mbar_expect_tx(full_bar(stg), Lay::A_BYTES + Lay::G_BYTES);  // rows past M are zero-filled and still counted
          sm100::tma_load_2d(sa, &map_x, full_bar(stg), 0, (int)s0);
          if constexpr (Lay::DOUT) sm100::tma_load_2d(sa + Lay::A_BYTES, &map_g, full_bar(stg), 0, (int)s0);
          if (++stg == STEM_STAGES) {
            stg = 0;
            par ^= 1;
          }
        }
      }
    }
  } else if (warp >= 4) {
    const int wg = (warp >> 2) - 1, wq = warp & 3;
    const int rl0 = wg * 64 + wq * 16 + (lane >> 2);  // fragment rows rl0, rl0 + 8 of this thread
    const int t = threadIdx.x - 128, pl = t / CVB, cvi = t % CVB, c0 = cvi * 8;
    const bool active = pl < LANES;
    float r[NCOEF > 0 ? NCOEF : 1][8];  // chan_body: the thread's coefficients, in registers for the whole kernel
#pragma unroll
    for (int k = 0; k < NCOEF; ++k)
#pragma unroll
      for (int e = 0; e < 8; ++e) r[k][e] = sc[k * KOUT + c0 + e];
    float acc[BN / 2];
    float sums[NACC > 0 ? NACC : 1][8];
    sm100::mbar_wait(w_bar, 0);
    int stg = 0;
    uint32_t par = 0;
    for (int b = blockIdx.x; b < nranges; b += gridDim.x) {
      const int64_t p0 = (int64_t)b * per, p1 = p0 + per < M ? p0 + per : M;
#pragma unroll
      for (int a = 0; a < (NACC > 0 ? NACC : 1); ++a)
#pragma unroll
        for (int e = 0; e < 8; ++e) sums[a][e] = 0.f;
      for (int64_t s0 = p0; s0 < p1; s0 += STEM_BM) {
        const int rows = (int)(p1 - s0 < STEM_BM ? p1 - s0 : STEM_BM);
        sm100::mbar_wait(full_bar(stg), par);
        const uint32_t sa = s_stage0 + stg * Lay::STAGE;
        // conv_wgmma_kernel's k-sequence for a 32-channel 1 x 1 GEMM: one 64B-swizzled stage, two k16 steps, the first overwriting D
        sm100::wgmma_fence();
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const uint64_t da = sm100::smem_desc(sa + (uint32_t)wg * 64u * 64u + 32u * j, 64, 16u, 512u);
          const uint64_t db = sm100::smem_desc(s_w + 32u * j, 64, 16u, 512u);
          sm100::mma_kk<BN>(acc, da, db, j);
        }
        sm100::wgmma_commit();
        sm100::wgmma_wait<0>();
        sm100::fence_regs(acc);
        // park the tile as conv_wgmma_kernel stores it: bf16 pairs rounded to nearest
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < 2 * JB; ++j)
            *reinterpret_cast<__nv_bfloat162*>(ytile + (rl0 + 8 * h) * YP + 8 * j + 2 * (lane & 3)) =
                __floats2bfloat162_rn(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        stem_consumer_sync();
        if (active) {
          const bf16* g_tile = reinterpret_cast<const bf16*>(gen(sa + Lay::A_BYTES));  // [128][KOUT] dout rows
          const int off = (int)((s0 - p0) % LANES);
          for (int rl = (pl - off + LANES) % LANES; rl < rows; rl += LANES) {  // pixels p0 + pl, + LANES, ... in order
            const int64_t m = s0 + rl;
            const V8 a = unpack8(*reinterpret_cast<const uint4*>(ytile + rl * YP + c0));
            const V8 bu = unpack8(*reinterpret_cast<const uint4*>(ytile + rl * YP + KOUT + c0));
            if constexpr (MODE == STEM_GEMM) {
              *reinterpret_cast<uint4*>(op.y + m * BN + c0) = *reinterpret_cast<const uint4*>(ytile + rl * YP + c0);
              *reinterpret_cast<uint4*>(op.y + m * BN + KOUT + c0) = *reinterpret_cast<const uint4*>(ytile + rl * YP + KOUT + c0);
            } else if constexpr (MODE == STEM_MOM) {
#pragma unroll
              for (int e = 0; e < 8; ++e) {
                float s[5] = {sums[0][e], sums[1][e], sums[2][e], sums[3][e], sums[4][e]};
                qarep_mom(a.v[e], bu.v[e], s);
#pragma unroll
                for (int k = 0; k < 5; ++k) sums[k][e] = s[k];
              }
            } else if constexpr (MODE == STEM_FWD) {
              V8 o;
#pragma unroll
              for (int e = 0; e < 8; ++e) o.v[e] = qarep_out(a.v[e], bu.v[e], [&](int k) { return r[k][e]; }, d.act);
              st8(op.outp + m * d.pitcho + d.offo + c0, o);
            } else {
              const V8 g = unpack8(*reinterpret_cast<const uint4*>(g_tile + rl * KOUT + c0));
              if constexpr (MODE == STEM_BRED) {
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                  float s[3] = {sums[0][e], sums[1][e], sums[2][e]};
                  qarep_bwd_sums(d, g.v[e], a.v[e], bu.v[e], [&](int k) { return r[k][e]; }, s);
#pragma unroll
                  for (int k = 0; k < 3; ++k) sums[k][e] = s[k];
                }
              } else {
                V8 o3, ou;
#pragma unroll
                for (int e = 0; e < 8; ++e) qarep_bwd_grads(d, g.v[e], a.v[e], bu.v[e], [&](int k) { return r[k][e]; }, o3.v[e], ou.v[e]);
                st8(op.dy3 + m * d.pitch3 + d.off3 + c0, o3);
                st8(op.du + m * d.pitchu + d.offu + c0, ou);
              }
            }
          }
        }
        stem_consumer_sync();  // the parked tile and the stage's dout rows are consumed
        if (lane == 0) sm100::mbar_arrive(empty_bar(stg));
        if (++stg == STEM_STAGES) {
          stg = 0;
          par ^= 1;
        }
      }
      if constexpr (NACC > 0) {
        // chan_body's combine: thread (pl, cvi) parks its sums, output (ci, a, e) adds them over pl in order, one fp64 atomic per range
        if (active) {
#pragma unroll
          for (int a = 0; a < NACC; ++a)
#pragma unroll
            for (int e = 0; e < 8; ++e) sred[(pl * CVB + cvi) * (NACC * 8 + 1) + a * 8 + e] = sums[a][e];
        }
        stem_consumer_sync();
        for (int j = t; j < CVB * NACC * 8; j += TPB) {
          float sum = 0.f;
          const int ci = j / (NACC * 8), a = (j / 8) % NACC, e = j % 8;
          for (int q = 0; q < LANES; ++q) sum += sred[(q * CVB + ci) * (NACC * 8 + 1) + a * 8 + e];
          atomicAdd(&op.out[(int64_t)a * op.out_stride + ci * 8 + e], (double)sum);
        }
        stem_consumer_sync();
      }
    }
  }
}

long long g_stem_launches = 0;

// xp: [M][32] bf16 patches (dense), w: [2K][32] bf16, dout: [M] rows of K bf16 at pitch `gpitch` (backward modes only).  nranges:
// the reductions' pixel ranges (the grid of the fused chan launch they replace); the other modes take one 128-pixel chunk per range.
template <int KOUT, int MODE, class Op>
int launch_stem_k(const Op& op, const SgbQarepDesc& d, const void* xp, const void* w, const void* dout, int gpitch, int nranges, cudaStream_t st) {
  using Lay = StemLayout<KOUT, MODE, Op>;
  if (int rc = sm100::init_driver()) return rc;
  const size_t smem = Lay::smem();
  static bool attr = false;
  if (!attr) {
    if (int rc = sgb_cuda_check(cudaFuncSetAttribute(stem_qarep_kernel<KOUT, MODE, Op>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "stem_qarep_kernel"))
      return rc;
    attr = true;
  }
  alignas(64) CUtensorMap map_x, map_w, map_g;
  const cuuint64_t x_dims[2] = {STEM_KP, (cuuint64_t)d.M}, w_dims[2] = {STEM_KP, 2 * KOUT}, g_dims[2] = {KOUT, (cuuint64_t)d.M};
  const cuuint64_t row_bytes[1] = {STEM_KP * 2}, g_row_bytes[1] = {(cuuint64_t)gpitch * 2};
  const cuuint32_t x_box[2] = {STEM_KP, STEM_BM}, w_box[2] = {STEM_KP, 2 * KOUT}, g_box[2] = {KOUT, STEM_BM};
  if (int rc = sm100::encode_tiled(&map_x, xp, 2, x_dims, row_bytes, x_box, CU_TENSOR_MAP_SWIZZLE_64B, "stem patches")) return rc;
  if (int rc = sm100::encode_tiled(&map_w, w, 2, w_dims, row_bytes, w_box, CU_TENSOR_MAP_SWIZZLE_64B, "stem filter")) return rc;
  map_g = map_x;
  if (Lay::DOUT)
    if (int rc = sm100::encode_tiled(&map_g, dout, 2, g_dims, g_row_bytes, g_box, CU_TENSOR_MAP_SWIZZLE_NONE, "stem dout")) return rc;
  const int64_t per = nranges > 0 ? (d.M + nranges - 1) / nranges : STEM_BM;
  const int64_t ranges = (d.M + per - 1) / per;
  const int grid = (int)(ranges < sgb_sm_count() ? ranges : sgb_sm_count());
  stem_qarep_kernel<KOUT, MODE, Op><<<grid, STEM_THREADS, smem, st>>>(map_x, map_w, map_g, op, d, d.M, per, (int)ranges);
  ++g_stem_launches;
  return sgb_cuda_check(cudaGetLastError(), "stem_qarep_kernel");
}

// The stem widths of the YOLO-NAS and YOLO-NAS-POSE recipes: 32, 48 and 64 output channels.
template <int MODE, class Op>
int launch_stem(const Op& op, const SgbQarepDesc& d, const void* xp, const void* w, const void* dout, int gpitch, int nranges, cudaStream_t st) {
  switch (d.C) {
    case 32: return launch_stem_k<32, MODE>(op, d, xp, w, dout, gpitch, nranges, st);
    case 48: return launch_stem_k<48, MODE>(op, d, xp, w, dout, gpitch, nranges, st);
    case 64: return launch_stem_k<64, MODE>(op, d, xp, w, dout, gpitch, nranges, st);
  }
  sgb_set_error("stem_qarep: %d output channels (32, 48 or 64 are served)", d.C);
  return SGB_E_UNSUPPORTED;
}

int check_stem(const SgbQarepDesc* d, const void* xp, const void* w) {
  SGB_REQUIRE(d && xp && w, "null pointer");
  SGB_REQUIRE(d->C == 32 || d->C == 48 || d->C == 64, "stem_qarep: 32, 48 or 64 output channels");
  SGB_REQUIRE(d->M > 0 && d->M < (1ll << 31) - STEM_BM, "stem_qarep: pixel count");
  SGB_REQUIRE((((uintptr_t)xp | (uintptr_t)w) & 15) == 0, "stem_qarep: xp / w must be 16-byte aligned");
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

// ---------------------------------------------------------------------------------------------- QARepVGG stem on patches
extern "C" int64_t sgb_stem_recompute_launches(void) { return (int64_t)g_stem_launches; }

extern "C" int sgb_stem_gemm(const SgbQarepDesc* d, const sgb_bf16* xp, const sgb_bf16* w, sgb_bf16* y, void* stream) {
  if (int rc = check_stem(d, xp, w)) return rc;
  SGB_REQUIRE(y && ((uintptr_t)y & 15) == 0, "null or misaligned y");
  StemGemmOp op{(bf16*)y};
  return launch_stem<STEM_GEMM>(op, *d, xp, w, nullptr, 0, 0, (cudaStream_t)stream);
}

extern "C" int sgb_stem_qarep_moments(const SgbQarepDesc* d, const sgb_bf16* xp, const sgb_bf16* w, double* moments, void* stream) {
  if (int rc = check_stem(d, xp, w)) return rc;
  SGB_REQUIRE(moments, "null pointer");
  QarepMomOp op{*d, nullptr, nullptr, moments, d->C};
  size_t smem = 0;  // the moments half of sgb_qarep_fwd_fused: its pixel ranges, its summation order
  const int nranges = chan_fused_grid<QarepMomOp, QarepFwdOp>(d->M, d->C, &smem, "stem_qarep_moments");
  if (nranges < 0) return nranges;
  return launch_stem<STEM_MOM>(op, *d, xp, w, nullptr, 0, nranges, (cudaStream_t)stream);
}

extern "C" int sgb_stem_qarep_fwd(const SgbQarepDesc* d, const sgb_bf16* xp, const sgb_bf16* w, const double* moments, const float* gamma3,
                                  const float* beta3, const float* bias1_alpha, const float* gamma_p, const float* beta_p, float* rm3, float* rv3,
                                  float* rm_p, float* rv_p, sgb_bf16* out, float* coef, void* stream) {
  if (int rc = check_qarep(d)) return rc;
  if (int rc = check_stem(d, xp, w)) return rc;
  SGB_REQUIRE(!d->res, "stem_qarep_fwd: no shortcut");
  SGB_REQUIRE(moments && gamma3 && beta3 && out && coef && ((uintptr_t)out & 15) == 0 && d->pitcho % 8 == 0, "null or misaligned pointer");
  SGB_REQUIRE(!d->use_post_bn || (gamma_p && beta_p), "post_bn parameters missing");
  QarepFwdOp op{*d, nullptr, nullptr, (bf16*)out, moments, gamma3, beta3, bias1_alpha, gamma_p, beta_p, rm3, rv3, rm_p, rv_p, coef};
  return launch_stem<STEM_FWD>(op, *d, xp, w, nullptr, 0, 0, (cudaStream_t)stream);
}

extern "C" int sgb_stem_qarep_bwd_reduce(const SgbQarepDesc* d, const sgb_bf16* dout, const sgb_bf16* xp, const sgb_bf16* w, const float* coef,
                                         double* sums, void* stream) {
  if (int rc = check_qarep(d)) return rc;
  if (int rc = check_stem(d, xp, w)) return rc;
  SGB_REQUIRE(dout && coef && sums && ((uintptr_t)dout & 15) == 0, "null or misaligned pointer");
  QarepBwdRedOp op{*d, nullptr, nullptr, nullptr, coef, sums, d->C};
  size_t smem = 0;  // the reduction half of sgb_qarep_bwd_fused: its pixel ranges, its summation order
  const int nranges = chan_fused_grid<QarepBwdRedOp, QarepBwdApplyOp>(d->M, d->C, &smem, "stem_qarep_bwd_reduce");
  if (nranges < 0) return nranges;
  return launch_stem<STEM_BRED>(op, *d, xp, w, (const bf16*)dout + (d->pitchd ? d->offd : d->offo), d->pitchd ? d->pitchd : d->pitcho, nranges,
                                (cudaStream_t)stream);
}

extern "C" int sgb_stem_qarep_bwd_apply(const SgbQarepDesc* d, const sgb_bf16* dout, const sgb_bf16* xp, const sgb_bf16* w, const float* coef,
                                        const double* sums, const float* gamma3, const float* gamma_p, sgb_bf16* dy3, sgb_bf16* du, float* dgamma3,
                                        float* dbeta3, float* dbias1a, float* dgamma_p, float* dbeta_p, void* stream) {
  if (int rc = check_qarep(d)) return rc;
  if (int rc = check_stem(d, xp, w)) return rc;
  SGB_REQUIRE(dout && coef && sums && gamma3 && dy3 && du && ((uintptr_t)dout & 15) == 0 && (((uintptr_t)dy3 | (uintptr_t)du) & 15) == 0,
              "null or misaligned pointer");
  SGB_REQUIRE(!d->use_post_bn || gamma_p, "gamma_p missing");
  QarepBwdApplyOp op{*d, nullptr, nullptr, nullptr, coef, sums, gamma3, gamma_p, (bf16*)dy3, (bf16*)du, dgamma3, dbeta3, dbias1a, dgamma_p, dbeta_p};
  return launch_stem<STEM_BAPPLY>(op, *d, xp, w, (const bf16*)dout + (d->pitchd ? d->offd : d->offo), d->pitchd ? d->pitchd : d->pitcho, 0,
                                  (cudaStream_t)stream);
}

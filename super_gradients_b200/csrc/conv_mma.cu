// Generic implicit-GEMM convolution kernels (fprop / dgrad / wgrad) for NHWC bf16 tensors, fp32 accumulation.
//
// This is the shape-agnostic path of libsgb200: any filter size, stride, padding, channel pitch/offset, plus the
// ConvTranspose2d(2,2) scatter store.  It runs on the legacy warp-level tensor-core path (mma.sync m16n8k16) fed
// by a 4-stage cp.async gather pipeline, and serves the shapes the tcgen05/TMA kernels (conv_sm100.cu) do not
// take (3-channel stems, 7x7, strided dgrad, ragged channel counts).  One kernel covers fprop and dgrad: dgrad of
// a stride-s convolution is decomposed into s*s output-parity classes, each an exact (zero-waste) stride-1 gather.
//
// Reference arithmetic being replaced: nn.Conv2d forward/backward as called from
//   src/super_gradients/modules/qarepvgg_block.py:184-204, modules/conv_bn_act_block.py:92-93,
//   training/models/classification_models/resnet.py:26-84 (see include/sgb200.h).
#include "common.cuh"
#include "conv_sm100.h"

namespace {

constexpr int BM = 128;
constexpr int BK = 32;
constexpr int STAGES = 4;
constexpr int THREADS = 256;

struct GatherClass {
  int M;               // GEMM rows in this class
  int Hc, Wc;          // row index m -> (n, j, i) over an Hc x Wc grid
  int nr, ns;          // taps visited
  int Kg;              // nr * ns * Cg
  int hb_add, wb_add;  // gathered row/col base: hb = j * row_mul + hb_add
  int r0, s0;          // first filter tap (B-operand offset)
  int oh_add, ow_add;  // output pixel = (j * o_mul + oh_add, i * o_mul + ow_add)
};

struct IGemmParams {
  const bf16* A;
  const bf16* B;
  void* Y;
  GatherClass cls[4];
  int Ngemm, Cg;
  int row_mul, tap_sgn;
  int inH, inW, in_pitch, in_off;
  int b_pitch, rstep, S_filt;
  int outH, outW, o_mul, out_pitch, out_off;
  int up2_cout;
  const float* scale;
  const float* shift;
  const bf16* residual;
  double* stats;
  int stats_repl;
  int act;
  int out_f32;
};

__device__ __forceinline__ int swz4(int row, int chunk) { return chunk ^ ((row >> 1) & 3); }

template <int BN, int WARPS_M, int WARPS_N>
__global__ void __launch_bounds__(THREADS) igemm_conv_kernel(const __grid_constant__ IGemmParams p) {
  constexpr int WTM = BM / WARPS_M, WTN = BN / WARPS_N;
  constexpr int MT = WTM / 16, NT = WTN / 8;
  static_assert(WARPS_M * WARPS_N * 32 == THREADS, "warp layout");
  static_assert(NT % 2 == 0, "NT must be even");
  constexpr int A_STAGE = BM * BK;  // elements
  constexpr int B_STAGE = BN * BK;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  bf16* As = reinterpret_cast<bf16*>(smem_raw);
  bf16* Bs = As + STAGES * A_STAGE;

  const GatherClass& gc = p.cls[blockIdx.z];
  const int m0 = blockIdx.x * BM;
  if (m0 >= gc.M) return;
  const int n0 = blockIdx.y * BN;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp / WARPS_N, wn = warp % WARPS_N;

  // ---- per-thread gather bookkeeping: 2 A rows x 1 chunk, and up to 2 B rows x 1 chunk
  const int a_chunk = tid & 3;
  int a_hb[2], a_wb[2];
  long long a_img[2];
  bool a_ok[2];
  const int hw = gc.Hc * gc.Wc;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    int m = m0 + (tid >> 2) + i * 64;
    a_ok[i] = m < gc.M;
    int mm = a_ok[i] ? m : 0;
    int n = mm / hw;
    int rem = mm - n * hw;
    int j = rem / gc.Wc;
    int ii = rem - j * gc.Wc;
    a_hb[i] = j * p.row_mul + gc.hb_add;
    a_wb[i] = ii * p.row_mul + gc.wb_add;
    a_img[i] = (long long)n * p.inH * p.inW;
  }
  constexpr int B_ITERS = (BN * 4 + THREADS - 1) / THREADS;

  const int KT = (gc.Kg + BK - 1) / BK;

  auto load_tile = [&](int kt, int stage) {
    const int k = kt * BK + a_chunk * 8;
    const bool kok = k < gc.Kg;
    int t = 0, ch = 0, ir = 0, is = 0;
    if (kok) {
      t = k / p.Cg;
      ch = k - t * p.Cg;
      ir = t / gc.ns;
      is = t - ir * gc.ns;
    }
    bf16* as = As + stage * A_STAGE;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      int row = (tid >> 2) + i * 64;
      int h = a_hb[i] + p.tap_sgn * ir;
      int w = a_wb[i] + p.tap_sgn * is;
      bool ok = kok && a_ok[i] && (unsigned)h < (unsigned)p.inH && (unsigned)w < (unsigned)p.inW;
      const bf16* src = p.A;
      if (ok) src = p.A + ((a_img[i] + (long long)h * p.inW + w) * p.in_pitch + p.in_off + ch);
      cp_async16(smem_u32(as + row * BK + swz4(row, a_chunk) * 8), src, ok);
    }
    bf16* bs = Bs + stage * B_STAGE;
    const long long boff = (long long)((gc.r0 + ir * p.rstep) * p.S_filt + gc.s0 + is * p.rstep) * p.Cg + ch;
#pragma unroll
    for (int i = 0; i < B_ITERS; ++i) {
      int idx = tid + i * THREADS;
      if (BN * 4 % THREADS != 0 && idx >= BN * 4) break;
      int row = idx >> 2;  // chunk == a_chunk because THREADS % 4 == 0
      int nn = n0 + row;
      bool ok = kok && nn < p.Ngemm;
      const bf16* src = ok ? p.B + (long long)nn * p.b_pitch + boff : p.B;
      cp_async16(smem_u32(bs + row * BK + swz4(row, a_chunk) * 8), src, ok);
    }
  };

  float acc[MT][NT][4];
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < KT) load_tile(s, s);
    cp_async_commit();
  }

  for (int kt = 0; kt < KT; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();
    {
      int nk = kt + STAGES - 1;
      if (nk < KT) load_tile(nk, nk % STAGES);
      cp_async_commit();
    }
    const bf16* as = As + (kt % STAGES) * A_STAGE;
    const bf16* bs = Bs + (kt % STAGES) * B_STAGE;
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) {
      uint32_t af[MT][4];
      uint32_t bfr[NT][2];
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        int row = wm * WTM + mt * 16 + (lane & 15);
        int chunk = kk * 2 + (lane >> 4);
        ldmatrix_x4(af[mt][0], af[mt][1], af[mt][2], af[mt][3], smem_u32(as + row * BK + swz4(row, chunk) * 8));
      }
#pragma unroll
      for (int np = 0; np < NT / 2; ++np) {
        int row = wn * WTN + np * 16 + (lane & 7) + ((lane >> 4) << 3);
        int chunk = kk * 2 + ((lane >> 3) & 1);
        ldmatrix_x4(bfr[2 * np][0], bfr[2 * np][1], bfr[2 * np + 1][0], bfr[2 * np + 1][1],
                    smem_u32(bs + row * BK + swz4(row, chunk) * 8));
      }
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) mma_bf16_16816(acc[mt][nt], af[mt], bfr[nt][0], bfr[nt][1]);
    }
  }
  cp_async_wait<0>();
  __syncthreads();

  // ---- epilogue
  float* sstat = reinterpret_cast<float*>(smem_raw);  // [WARPS_M][2][BN]
  const bool do_stats = p.stats != nullptr;
  if (do_stats) {
    for (int i = tid; i < WARPS_M * 2 * BN; i += THREADS) sstat[i] = 0.f;  // one slot per warp row
    __syncthreads();
  }
  float cs1[NT][2], cs2[NT][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) cs1[nt][0] = cs1[nt][1] = cs2[nt][0] = cs2[nt][1] = 0.f;

#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      int m = m0 + wm * WTM + mt * 16 + (lane >> 2) + half * 8;
      if (m >= gc.M) continue;
      int n = m / hw;
      int rem = m - n * hw;
      int j = rem / gc.Wc;
      int ii = rem - j * gc.Wc;
      int oh = j * p.o_mul + gc.oh_add, ow = ii * p.o_mul + gc.ow_add;
      long long obase = (((long long)n * p.outH + oh) * p.outW + ow) * p.out_pitch + p.out_off;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        int col = n0 + wn * WTN + nt * 8 + 2 * (lane & 3);
        if (col >= p.Ngemm) continue;
        float v[2] = {acc[mt][nt][half * 2 + 0], acc[mt][nt][half * 2 + 1]};
        bool two = (col + 1) < p.Ngemm;
        long long o0 = obase + col;
        int pc = col;  // parameter (scale/shift) channel
        if (p.up2_cout > 0) {
          int q4 = col / p.up2_cout;
          pc = col - q4 * p.up2_cout;
          o0 = (((long long)n * p.outH + oh + (q4 >> 1)) * p.outW + ow + (q4 & 1)) * p.out_pitch + p.out_off + pc;
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          if (e == 1 && !two) break;
          float x = v[e];
          if (p.scale) x *= p.scale[pc + e];
          if (p.shift) x += p.shift[pc + e];
          if (p.residual) x += __bfloat162float(p.residual[o0 + e]);
          x = apply_act(x, p.act);
          if (!p.out_f32) x = bf16_round(x);
          v[e] = x;
          cs1[nt][e] += x;
          cs2[nt][e] += x * x;
        }
        if (p.out_f32) {
          float* y = reinterpret_cast<float*>(p.Y);
          y[o0] = v[0];
          if (two) y[o0 + 1] = v[1];
        } else {
          bf16* y = reinterpret_cast<bf16*>(p.Y);
          if (two && ((o0 & 1) == 0)) {
            *reinterpret_cast<__nv_bfloat162*>(y + o0) = __floats2bfloat162_rn(v[0], v[1]);
          } else {
            y[o0] = __float2bfloat16_rn(v[0]);
            if (two) y[o0 + 1] = __float2bfloat16_rn(v[1]);
          }
        }
      }
    }
  }
  if (do_stats) {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float a = cs1[nt][e], b = cs2[nt][e];
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          a += __shfl_xor_sync(0xffffffffu, a, o);
          b += __shfl_xor_sync(0xffffffffu, b, o);
        }
        if (lane < 4) {
          int c = wn * WTN + nt * 8 + 2 * lane + e;
          sstat[wm * 2 * BN + c] = a;  // (wm, column) is owned by exactly one lane of one warp
          sstat[wm * 2 * BN + BN + c] = b;
        }
      }
    __syncthreads();
    int rep = (blockIdx.x + blockIdx.z) & (p.stats_repl - 1);
    double* st = p.stats + (long long)rep * 2 * p.Ngemm;
    for (int c = tid; c < BN; c += THREADS) {
      int col = n0 + c;
      if (col < p.Ngemm) {
        float v1 = sstat[c], v2 = sstat[BN + c];
#pragma unroll
        for (int q = 1; q < WARPS_M; ++q) {  // fixed order
          v1 += sstat[q * 2 * BN + c];
          v2 += sstat[q * 2 * BN + BN + c];
        }
        atomicAdd(&st[col], (double)v1);
        atomicAdd(&st[p.Ngemm + col], (double)v2);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// wgrad: D[ko][(r,s,c)] += sum_pixels dy[pix][ko] * x[pix @ tap][c]      (split-K over pixels, fp32 atomics)
struct WgradParams {
  const bf16* X;
  const bf16* DY;
  float* DW;
  int N, H, W, C, K, R, S, P, Q, stride, pad;
  int x_pitch, x_off, y_pitch, y_off;
  int npix;          // N*P*Q
  int slices_per_z;  // BK-pixel slices handled by one blockIdx.z
  int ncols;         // R*S*C
};

template <int CPR>
__device__ __forceinline__ int swzT(int row, int chunk) {
  return CPR == 4 ? (chunk ^ ((row >> 1) & 3)) : (chunk ^ (row & 7));
}

template <int BMW, int WARPS_M, int WARPS_N>
__global__ void __launch_bounds__(THREADS) wgrad_kernel(const __grid_constant__ WgradParams p) {
  constexpr int BNW = 64;
  constexpr int WTM = BMW / WARPS_M, WTN = BNW / WARPS_N;
  constexpr int MT = WTM / 16, NT = WTN / 8;
  static_assert(NT % 2 == 0, "NT even");
  constexpr int A_CPR = BMW / 8, B_CPR = BNW / 8;
  constexpr int A_STAGE = BK * BMW, B_STAGE = BK * BNW;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  bf16* As = reinterpret_cast<bf16*>(smem_raw);
  bf16* Bs = As + STAGES * A_STAGE;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp / WARPS_N, wn = warp % WARPS_N;
  const int mo0 = blockIdx.y * BMW;  // out-channel tile
  const int n0 = blockIdx.x * BNW;   // (r,s,c) column tile
  const int slice0 = blockIdx.z * p.slices_per_z;
  const int total_slices = (p.npix + BK - 1) / BK;
  int nslices = total_slices - slice0;
  if (nslices > p.slices_per_z) nslices = p.slices_per_z;
  if (nslices <= 0) return;

  // B gather: one chunk per thread, fixed column
  const int b_row = tid >> 3, b_chunk = tid & 7;
  const int b_col = n0 + b_chunk * 8;
  const bool b_colok = b_col < p.ncols;
  int b_r = 0, b_s = 0, b_c = 0;
  if (b_colok) {
    int tap = b_col / p.C;
    b_c = b_col - tap * p.C;
    b_r = tap / p.S;
    b_s = tap - b_r * p.S;
  }
  constexpr int A_ITERS = (BK * A_CPR + THREADS - 1) / THREADS;
  const int pq = p.P * p.Q;

  auto load_tile = [&](int sl, int stage) {
    const int pix0 = (slice0 + sl) * BK;
    bf16* as = As + stage * A_STAGE;
#pragma unroll
    for (int i = 0; i < A_ITERS; ++i) {
      int idx = tid + i * THREADS;
      if ((BK * A_CPR) % THREADS != 0 && idx >= BK * A_CPR) break;
      int row = idx / A_CPR, chunk = idx % A_CPR;
      int pix = pix0 + row;
      int ko = mo0 + chunk * 8;
      bool ok = pix < p.npix && ko < p.K;
      const bf16* src = ok ? p.DY + ((long long)pix * p.y_pitch + p.y_off + ko) : p.DY;
      cp_async16(smem_u32(as + row * BMW + swzT<A_CPR>(row, chunk) * 8), src, ok);
    }
    bf16* bs = Bs + stage * B_STAGE;
    {
      int pix = pix0 + b_row;
      bool ok = b_colok && pix < p.npix;
      const bf16* src = p.X;
      if (ok) {
        int n = pix / pq;
        int rem = pix - n * pq;
        int pp = rem / p.Q;
        int qq = rem - pp * p.Q;
        int h = pp * p.stride - p.pad + b_r, w = qq * p.stride - p.pad + b_s;
        ok = (unsigned)h < (unsigned)p.H && (unsigned)w < (unsigned)p.W;
        if (ok) src = p.X + ((((long long)n * p.H + h) * p.W + w) * p.x_pitch + p.x_off + b_c);
      }
      cp_async16(smem_u32(bs + b_row * BNW + swzT<B_CPR>(b_row, b_chunk) * 8), src, ok);
    }
  };

  float acc[MT][NT][4];
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < nslices) load_tile(s, s);
    cp_async_commit();
  }
  for (int kt = 0; kt < nslices; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();
    {
      int nk = kt + STAGES - 1;
      if (nk < nslices) load_tile(nk, nk % STAGES);
      cp_async_commit();
    }
    const bf16* as = As + (kt % STAGES) * A_STAGE;
    const bf16* bs = Bs + (kt % STAGES) * B_STAGE;
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) {
      uint32_t af[MT][4];
      uint32_t bfr[NT][2];
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        int krow = kk * 16 + (lane & 7) + ((lane >> 4) << 3);
        int chunk = ((wm * WTM + mt * 16) >> 3) + ((lane >> 3) & 1);
        ldmatrix_x4_trans(af[mt][0], af[mt][1], af[mt][2], af[mt][3],
                          smem_u32(as + krow * BMW + swzT<A_CPR>(krow, chunk) * 8));
      }
#pragma unroll
      for (int np = 0; np < NT / 2; ++np) {
        int krow = kk * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
        int chunk = ((wn * WTN + np * 16) >> 3) + (lane >> 4);
        ldmatrix_x4_trans(bfr[2 * np][0], bfr[2 * np][1], bfr[2 * np + 1][0], bfr[2 * np + 1][1],
                          smem_u32(bs + krow * BNW + swzT<B_CPR>(krow, chunk) * 8));
      }
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) mma_bf16_16816(acc[mt][nt], af[mt], bfr[nt][0], bfr[nt][1]);
    }
  }
  cp_async_wait<0>();

#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      int ko = mo0 + wm * WTM + mt * 16 + (lane >> 2) + half * 8;
      if (ko >= p.K) continue;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        int col = n0 + wn * WTN + nt * 8 + 2 * (lane & 3);
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (col + e < p.ncols) atomicAdd(p.DW + (long long)ko * p.ncols + col + e, acc[mt][nt][half * 2 + e]);
      }
    }
}

template <int BN, int WM, int WN>
int launch_igemm(const IGemmParams& p, int ncls, int maxM, cudaStream_t st) {
  size_t smem = (size_t)STAGES * (BM * BK + BN * BK) * sizeof(bf16);
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(igemm_conv_kernel<BN, WM, WN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr_set = true;
  }
  dim3 grid(ceil_div(maxM, BM), ceil_div(p.Ngemm, BN), ncls);
  igemm_conv_kernel<BN, WM, WN><<<grid, THREADS, smem, st>>>(p);
  SGB_LAUNCH_CHECK("igemm_conv_kernel");
  return SGB_OK;
}

int dispatch_igemm(const IGemmParams& p, int ncls, int maxM, cudaStream_t st) {
  int n = p.Ngemm;
  auto waste = [&](int bn) { return ceil_div(n, bn) * bn - n; };
  int best = 128, bw = waste(128);
  if (waste(64) < bw) { best = 64; bw = waste(64); }
  if (waste(32) < bw) { best = 32; bw = waste(32); }
  if (best == 128) return launch_igemm<128, 2, 4>(p, ncls, maxM, st);
  if (best == 64) return launch_igemm<64, 4, 2>(p, ncls, maxM, st);
  return launch_igemm<32, 4, 2>(p, ncls, maxM, st);
}

int check_desc(const SgbConvDesc* d) {
  SGB_REQUIRE(d != nullptr, "desc is null");
  SGB_REQUIRE(d->N > 0 && d->H > 0 && d->W > 0 && d->C > 0 && d->K > 0 && d->R > 0 && d->S > 0, "positive dims");
  SGB_REQUIRE(d->stride >= 1 && d->pad >= 0, "stride/pad");
  SGB_REQUIRE(d->P == (d->H + 2 * d->pad - d->R) / d->stride + 1, "P inconsistent");
  SGB_REQUIRE(d->Q == (d->W + 2 * d->pad - d->S) / d->stride + 1, "Q inconsistent");
  SGB_REQUIRE(d->C % 8 == 0, "C must be a multiple of 8 (pad the channels)");
  SGB_REQUIRE(d->x_pitch % 8 == 0 && d->x_off % 8 == 0, "x pitch/offset must be multiples of 8");
  SGB_REQUIRE(d->x_pitch >= d->x_off + d->C, "x slice exceeds pitch");
  SGB_REQUIRE(d->y_pitch >= d->y_off + d->K, "y slice exceeds pitch");
  SGB_REQUIRE(d->centre_from == 0 || (d->R == 3 && d->S == 3 && d->stride == 1 && d->pad == 1 && d->centre_from > 0 &&
                                      d->centre_from < d->K && d->centre_from % 16 == 0),
              "centre_from needs a 3x3 / stride-1 / pad-1 convolution and 0 < centre_from < K, a multiple of 16");
  return SGB_OK;
}

}  // namespace

extern "C" int sgb_conv_fprop(const SgbConvDesc* d, const sgb_bf16* x, const sgb_bf16* w, void* y,
                              const SgbEpilogue* ep, void* stream) {
  if (int rc = check_desc(d)) return rc;
  SGB_REQUIRE(x && w && y, "null pointer");
  if (!(ep && ep->out_f32)) {
    sm100::Problem q{};
    q.a = x + d->x_off; q.N = d->N; q.H = d->H; q.W = d->W; q.C = d->C; q.a_pitch = d->x_pitch;
    q.b = w; q.b_rows = d->K; q.b_cols = d->R * d->S * d->C; q.b_cols_per_tap = d->C;
    q.R = d->R; q.S = d->S; q.stride = d->stride; q.pad = d->pad; q.P = d->P; q.Q = d->Q; q.flip = 0;
    q.y = y; q.y_pitch = d->y_pitch; q.y_off = d->y_off;
    q.centre_from = d->centre_from;
    if (ep) {
      q.scale = ep->scale; q.shift = ep->shift; q.residual = ep->residual; q.stats = ep->stats;
      q.stats_repl = ep->stats_repl > 0 ? ep->stats_repl : 1; q.act = ep->act;
    } else {
      q.stats_repl = 1;
    }
    if (d->pad == d->R / 2 && sm100::supported(q)) return sm100::launch(q, (cudaStream_t)stream);
    // 2 x 2 / stride 2 / no padding over a dense tensor (the backward of ConvTranspose2d(2, 2), modules/sampling.py:72-73): the
    // patches do not overlap, so the tensor viewed as an image [N * H/2][2][W/2][2C] -- row pair, row parity, column pair, (column
    // parity, channel) -- turns the layer into a 2-tap (rows 0 and 1), stride-1 valid convolution with 2C channels per tap whose
    // B columns are the filter's own (dh, dw, c) order: the im2col tcgen05 kernel serves it through its explicit tap table.
    if (d->R == 2 && d->S == 2 && d->stride == 2 && d->pad == 0 && d->x_pitch == d->C && d->x_off == 0 && d->H % 2 == 0 &&
        d->W % 2 == 0 && d->P == d->H / 2 && d->Q == d->W / 2 && (2 * d->C) % 16 == 0 && d->K % 8 == 0 && d->y_pitch % 8 == 0 && d->y_off % 8 == 0 &&
        (long long)d->N * (d->H / 2) < (1ll << 31)) {
      q.N = d->N * (d->H / 2); q.H = 2; q.W = d->W / 2; q.C = 2 * d->C; q.a_pitch = 2 * d->C;
      q.b_cols_per_tap = 2 * d->C;
      q.centre_from = 0;  // a 2 x 2 filter: check_desc refused a non-zero field
      q.R = 1; q.S = 1; q.stride = 1; q.pad = 0; q.P = 1; q.Q = d->W / 2;
      q.ntaps = 2;
      q.tap_dh[0] = 0; q.tap_dw[0] = 0; q.tap_b[0] = 0;
      q.tap_dh[1] = 1; q.tap_dw[1] = 0; q.tap_b[1] = 1;
      if (sm100::supported(q)) return sm100::launch(q, (cudaStream_t)stream);
      return SGB_E_UNSUPPORTED;
    }
  }
  IGemmParams p{};
  p.A = reinterpret_cast<const bf16*>(x);
  p.B = reinterpret_cast<const bf16*>(w);
  p.Y = y;
  GatherClass& g = p.cls[0];
  g.M = d->N * d->P * d->Q;
  g.Hc = d->P;
  g.Wc = d->Q;
  g.nr = d->R;
  g.ns = d->S;
  g.Kg = d->R * d->S * d->C;
  g.hb_add = -d->pad;
  g.wb_add = -d->pad;
  g.r0 = g.s0 = 0;
  g.oh_add = g.ow_add = 0;
  p.Ngemm = d->K;
  p.Cg = d->C;
  p.row_mul = d->stride;
  p.tap_sgn = 1;
  p.inH = d->H;
  p.inW = d->W;
  p.in_pitch = d->x_pitch;
  p.in_off = d->x_off;
  p.b_pitch = d->R * d->S * d->C;
  p.rstep = 1;
  p.S_filt = d->S;
  p.outH = d->P;
  p.outW = d->Q;
  p.o_mul = 1;
  p.out_pitch = d->y_pitch;
  p.out_off = d->y_off;
  p.up2_cout = 0;
  if (ep) {
    p.scale = ep->scale;
    p.shift = ep->shift;
    p.residual = reinterpret_cast<const bf16*>(ep->residual);
    p.stats = ep->stats;
    p.stats_repl = ep->stats_repl > 0 ? ep->stats_repl : 1;
    SGB_REQUIRE((p.stats_repl & (p.stats_repl - 1)) == 0, "stats_repl must be a power of two");
    p.act = ep->act;
    p.out_f32 = ep->out_f32;
  } else {
    p.stats_repl = 1;
  }
  return dispatch_igemm(p, 1, g.M, (cudaStream_t)stream);
}

extern "C" int sgb_convt2x2_fprop(const SgbConvDesc* d, const sgb_bf16* x_small, const sgb_bf16* w_up,
                                  const float* bias, sgb_bf16* y_up, void* stream) {
  // d: equivalent conv (N,H,W,C)=upsampled -> (N,P,Q,K)=small with R=S=2, stride 2, pad 0
  if (int rc = check_desc(d)) return rc;
  SGB_REQUIRE(d->R == 2 && d->S == 2 && d->stride == 2 && d->pad == 0, "convt2x2 needs R=S=2, stride 2, pad 0");
  SGB_REQUIRE(d->K % 8 == 0 && d->y_pitch % 8 == 0 && d->y_off % 8 == 0, "small-side channels must be multiples of 8");
  if (d->K % 16 == 0 && d->C % 16 == 0) {
    // tcgen05 path: the transposed convolution is four 1x1 GEMMs, one per output parity (dh, dw), each writing the output pixels
    // (2h + dh, 2w + dw) through the strided-row epilogue the stride-2 input gradients use.  w_up rows are ordered (dh, dw, co).
    bool all_ok = true;
    for (int cls = 0; cls < 4 && all_ok; ++cls) {
      sm100::Problem q{};
      q.a = x_small + d->y_off; q.N = d->N; q.H = d->P; q.W = d->Q; q.C = d->K; q.a_pitch = d->y_pitch;
      q.b = w_up + (size_t)cls * d->C * d->K; q.b_rows = d->C; q.b_cols = d->K; q.b_cols_per_tap = d->K;
      q.R = 1; q.S = 1; q.stride = 1; q.pad = 0; q.P = d->P; q.Q = d->Q; q.flip = 0;
      q.y = y_up; q.y_pitch = d->x_pitch; q.y_off = d->x_off;
      q.shift = bias;
      q.stats_repl = 1;
      q.out_mode = 1; q.o_mul = 2; q.oh_add = cls >> 1; q.ow_add = cls & 1; q.outH = d->H; q.outW = d->W;
      q.ntaps = 1; q.tap_dh[0] = 0; q.tap_dw[0] = 0; q.tap_b[0] = 0;
      if (!sm100::supported(q)) { all_ok = false; break; }  // identical for the four classes: fails before any launch
      if (int rc = sm100::launch(q, (cudaStream_t)stream)) return rc;
    }
    if (all_ok) return SGB_OK;
  }
  IGemmParams p{};
  p.A = reinterpret_cast<const bf16*>(x_small);
  p.B = reinterpret_cast<const bf16*>(w_up);
  p.Y = y_up;
  GatherClass& g = p.cls[0];
  g.M = d->N * d->P * d->Q;
  g.Hc = d->P;
  g.Wc = d->Q;
  g.nr = g.ns = 1;
  g.Kg = d->K;
  p.Ngemm = 4 * d->C;
  p.Cg = d->K;
  p.row_mul = 1;
  p.tap_sgn = 1;
  p.inH = d->P;
  p.inW = d->Q;
  p.in_pitch = d->y_pitch;
  p.in_off = d->y_off;
  p.b_pitch = d->K;
  p.rstep = 1;
  p.S_filt = 1;
  p.outH = d->H;
  p.outW = d->W;
  p.o_mul = 2;
  p.out_pitch = d->x_pitch;
  p.out_off = d->x_off;
  p.up2_cout = d->C;
  p.shift = bias;
  p.stats_repl = 1;
  return dispatch_igemm(p, 1, g.M, (cudaStream_t)stream);
}

extern "C" int sgb_conv_dgrad(const SgbConvDesc* d, const sgb_bf16* dy, const sgb_bf16* w_crsk, sgb_bf16* dx,
                              int accumulate, void* stream) {
  if (int rc = check_desc(d)) return rc;
  SGB_REQUIRE(dy && w_crsk && dx, "null pointer");
  SGB_REQUIRE(d->K % 8 == 0 || d->y_pitch - d->y_off >= ((d->K + 7) / 8) * 8, "dy channels must be padded to 8");
  SGB_REQUIRE(d->y_pitch % 8 == 0 && d->y_off % 8 == 0, "dy pitch/offset must be multiples of 8");
  const int s = d->stride;
  SGB_REQUIRE(s == 1 || s == 2, "dgrad supports stride 1 or 2");
  const int Kp = ((d->K + 7) / 8) * 8;  // channels gathered per tap (w_crsk rows are padded with zeros to Kp)
  if (s == 1 && d->pad == d->R / 2 && d->K % 16 == 0) {
    // dgrad of a stride-1 "same" convolution == convolution of dy with the spatially flipped CRSK filter
    sm100::Problem q{};
    q.a = dy + d->y_off; q.N = d->N; q.H = d->P; q.W = d->Q; q.C = d->K; q.a_pitch = d->y_pitch;
    q.b = w_crsk; q.b_rows = d->C; q.b_cols = d->R * d->S * Kp; q.b_cols_per_tap = Kp;
    q.R = d->R; q.S = d->S; q.stride = 1; q.pad = d->R - 1 - d->pad; q.P = d->H; q.Q = d->W; q.flip = 1;
    q.y = dx; q.y_pitch = d->x_pitch; q.y_off = d->x_off;
    q.residual = accumulate ? dx : nullptr;
    q.stats_repl = 1;
    q.centre_from = d->centre_from;
    if (sm100::supported(q)) return sm100::launch(q, (cudaStream_t)stream);
  }
  if (s == 2 && d->K % 16 == 0 && d->R == 3 && d->S == 3 && d->pad == 1 && d->C % 8 == 0 && d->H % 2 == 0 &&
      d->W % 2 == 0 && d->H == 2 * d->P && d->W == 2 * d->Q) {
    // stride-2 dgrad = 4 output-parity classes, each an exact stride-1 gather of dy with a subset of the taps
    bool all_ok = true;
    for (int cls = 0; cls < 4 && all_ok; ++cls) {
      const int ph = cls >> 1, pw = cls & 1;
      sm100::Problem q{};
      q.a = dy + d->y_off; q.N = d->N; q.H = d->P; q.W = d->Q; q.C = d->K; q.a_pitch = d->y_pitch;
      q.b = w_crsk; q.b_rows = d->C; q.b_cols = d->R * d->S * Kp; q.b_cols_per_tap = Kp;
      q.R = d->R; q.S = d->S; q.stride = 1; q.pad = 0; q.P = d->P; q.Q = d->Q; q.flip = 0;
      q.y = dx; q.y_pitch = d->x_pitch; q.y_off = d->x_off;
      q.residual = accumulate ? dx : nullptr;
      q.stats_repl = 1;
      q.out_mode = 1; q.o_mul = 2; q.oh_add = ph; q.ow_add = pw; q.outH = d->H; q.outW = d->W;
      // taps r with (h + pad - r) even, h = 2j + ph:  ho = j + (ph + pad - r) / 2
      int nt = 0;
      for (int r = 0; r < d->R; ++r) {
        if (((ph + d->pad - r) & 1) != 0) continue;
        for (int sx = 0; sx < d->S; ++sx) {
          if (((pw + d->pad - sx) & 1) != 0) continue;
          q.tap_dh[nt] = (ph + d->pad - r) / 2;
          q.tap_dw[nt] = (pw + d->pad - sx) / 2;
          q.tap_b[nt] = r * d->S + sx;
          ++nt;
        }
      }
      q.ntaps = nt;
      if (!sm100::supported(q)) { all_ok = false; break; }  // identical for the 4 classes: fails before any launch
      if (int rc = sm100::launch(q, (cudaStream_t)stream)) return rc;
    }
    if (all_ok) return SGB_OK;
  }
  if (s == 2 && d->K % 16 == 0 && d->R == 1 && d->S == 1 && d->pad == 0 && d->C % 8 == 0 && d->H == 2 * d->P &&
      d->W == 2 * d->Q) {
    // 1x1 stride-2 dgrad: only the even/even input pixels receive a gradient.  With accumulate the other three parity
    // classes are untouched; otherwise they are zero-filled first.
    sm100::Problem q{};
    q.a = dy + d->y_off; q.N = d->N; q.H = d->P; q.W = d->Q; q.C = d->K; q.a_pitch = d->y_pitch;
    q.b = w_crsk; q.b_rows = d->C; q.b_cols = Kp; q.b_cols_per_tap = Kp;
    q.R = 1; q.S = 1; q.stride = 1; q.pad = 0; q.P = d->P; q.Q = d->Q; q.flip = 0;
    q.y = dx; q.y_pitch = d->x_pitch; q.y_off = d->x_off;
    q.residual = accumulate ? dx : nullptr;
    q.stats_repl = 1;
    q.out_mode = 1; q.o_mul = 2; q.oh_add = 0; q.ow_add = 0; q.outH = d->H; q.outW = d->W;
    q.ntaps = 1; q.tap_dh[0] = 0; q.tap_dw[0] = 0; q.tap_b[0] = 0;
    if (sm100::supported(q)) {
      if (!accumulate) {
        if (d->x_pitch == d->C && d->x_off == 0) {
          cudaMemsetAsync(dx, 0, (size_t)d->N * d->H * d->W * d->C * sizeof(sgb_bf16), (cudaStream_t)stream);
          return sm100::launch(q, (cudaStream_t)stream);
        }
      } else {
        return sm100::launch(q, (cudaStream_t)stream);
      }
    }
  }
  IGemmParams p{};
  p.A = reinterpret_cast<const bf16*>(dy);
  p.B = reinterpret_cast<const bf16*>(w_crsk);
  p.Y = dx;
  p.Ngemm = d->C;
  p.Cg = Kp;
  p.row_mul = 1;
  p.tap_sgn = -1;
  p.inH = d->P;
  p.inW = d->Q;
  p.in_pitch = d->y_pitch;
  p.in_off = d->y_off;
  p.b_pitch = d->R * d->S * Kp;
  p.rstep = s;
  p.S_filt = d->S;
  p.outH = d->H;
  p.outW = d->W;
  p.o_mul = s;
  p.out_pitch = d->x_pitch;
  p.out_off = d->x_off;
  p.stats_repl = 1;
  if (accumulate) p.residual = reinterpret_cast<const bf16*>(dx);
  int ncls = 0, maxM = 0;
  for (int ph = 0; ph < s; ++ph)
    for (int pw = 0; pw < s; ++pw) {
      GatherClass& g = p.cls[ncls++];
      g.Hc = (d->H - ph + s - 1) / s;
      g.Wc = (d->W - pw + s - 1) / s;
      g.M = d->N * g.Hc * g.Wc;
      g.r0 = (ph + d->pad) % s;
      g.s0 = (pw + d->pad) % s;
      g.nr = g.r0 < d->R ? (d->R - g.r0 + s - 1) / s : 0;
      g.ns = g.s0 < d->S ? (d->S - g.s0 + s - 1) / s : 0;
      g.Kg = g.nr * g.ns * Kp;
      if (g.ns == 0) g.ns = 1;  // avoid div by zero; Kg == 0 so nothing is gathered
      g.hb_add = (ph + d->pad - g.r0) / s;
      g.wb_add = (pw + d->pad - g.s0) / s;
      g.oh_add = ph;
      g.ow_add = pw;
      if (g.M > maxM) maxM = g.M;
    }
  return dispatch_igemm(p, ncls, maxM, (cudaStream_t)stream);
}

extern "C" int sgb_conv_wgrad(const SgbConvDesc* d, const sgb_bf16* x, const sgb_bf16* dy, float* dw, void* stream) {
  if (int rc = check_desc(d)) return rc;
  SGB_REQUIRE(x && dy && dw, "null pointer");
  SGB_REQUIRE(d->y_pitch % 8 == 0 && d->y_off % 8 == 0, "dy pitch/offset must be multiples of 8");
  SGB_REQUIRE(d->K % 8 == 0 || d->y_pitch - d->y_off >= ((d->K + 7) / 8) * 8, "dy channels must be padded to 8");
  {
    sm100::WgradProblem q{};
    q.x = x + d->x_off; q.dy = dy + d->y_off;
    q.N = d->N; q.H = d->H; q.W = d->W; q.C = d->C; q.x_pitch = d->x_pitch;
    q.K = d->K; q.y_pitch = d->y_pitch;
    q.R = d->R; q.S = d->S; q.stride = d->stride; q.pad = d->pad; q.P = d->P; q.Q = d->Q;
    q.dw = dw;
    q.centre_from = d->centre_from;
    if (sm100::wgrad_supported(q)) return sm100::wgrad_launch(q, (cudaStream_t)stream);
    // 2 x 2 / stride 2 / no padding over a dense x: the same re-description as in sgb_conv_fprop -- a (2 x 1)-tap stride-1 valid
    // convolution over the image [N * H/2][2][W/2][2C]; dW rows [K][dh][(dw, c)] are the KRSC rows of the 2 x 2 filter.
    if (d->R == 2 && d->S == 2 && d->stride == 2 && d->pad == 0 && d->x_pitch == d->C && d->x_off == 0 && d->H % 2 == 0 &&
        d->W % 2 == 0 && d->P == d->H / 2 && d->Q == d->W / 2 && (2 * d->C) % 16 == 0 && d->K % 8 == 0 && (long long)d->N * (d->H / 2) < (1ll << 31)) {
      q.N = d->N * (d->H / 2); q.H = 2; q.W = d->W / 2; q.C = 2 * d->C; q.x_pitch = 2 * d->C;
      q.R = 2; q.S = 1; q.stride = 1; q.pad = 0; q.P = 1; q.Q = d->W / 2;
      return sm100::wgrad_launch(q, (cudaStream_t)stream);
    }
  }
  WgradParams p{};
  p.X = reinterpret_cast<const bf16*>(x);
  p.DY = reinterpret_cast<const bf16*>(dy);
  p.DW = dw;
  p.N = d->N; p.H = d->H; p.W = d->W; p.C = d->C; p.K = d->K; p.R = d->R; p.S = d->S; p.P = d->P; p.Q = d->Q;
  p.stride = d->stride; p.pad = d->pad;
  p.x_pitch = d->x_pitch; p.x_off = d->x_off; p.y_pitch = d->y_pitch; p.y_off = d->y_off;
  p.npix = d->N * d->P * d->Q;
  p.ncols = d->R * d->S * d->C;
  int bmw = d->K <= 32 ? 32 : (d->K <= 64 ? 64 : 128);
  if (d->K > 64 && d->K <= 96) bmw = 32;  // 3 x 32 wastes nothing
  int mt = ceil_div(d->K, bmw), nt = ceil_div(p.ncols, 64);
  int total_slices = ceil_div(p.npix, BK);
  int target = 132 * 4;
  int splits = target / (mt * nt);
  if (splits < 1) splits = 1;
  if (splits > total_slices) splits = total_slices;
  int min_slices = 8;  // keep each CTA's K loop long enough to amortise the atomics
  if (total_slices / splits < min_slices) splits = total_slices / min_slices > 0 ? total_slices / min_slices : 1;
  p.slices_per_z = ceil_div(total_slices, splits);
  splits = ceil_div(total_slices, p.slices_per_z);
  dim3 grid(nt, mt, splits);
  cudaStream_t st = (cudaStream_t)stream;
  size_t smem = (size_t)STAGES * (BK * bmw + BK * 64) * sizeof(bf16);
  if (bmw == 128) {
    wgrad_kernel<128, 4, 2><<<grid, THREADS, smem, st>>>(p);
  } else if (bmw == 64) {
    wgrad_kernel<64, 2, 4><<<grid, THREADS, smem, st>>>(p);
  } else {
    wgrad_kernel<32, 2, 4><<<grid, THREADS, smem, st>>>(p);
  }
  SGB_LAUNCH_CHECK("wgrad_kernel");
  return SGB_OK;
}

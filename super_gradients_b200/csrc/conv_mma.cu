// Generic implicit-GEMM convolution kernels (fprop / dgrad / wgrad) for NHWC bf16 tensors, fp32 accumulation.
//
// This is the shape-agnostic engine of libsgb200: any filter size, stride, padding, channel pitch/offset, plus the
// ConvTranspose2d(2,2) scatter store.  It runs on the warp-level tensor-core path (mma.sync m16n8k16) fed by a 4-stage
// cp.async gather pipeline, and serves the calls the wgmma / TMA kernels of conv_sm100.cu decline (conv.cu routes them):
// 3-channel stems that are not padded to 16 channels, 7x7, ragged channel counts, fp32 outputs, and the strided dgrads other
// than 3x3 and 1x1 stride 2.  One kernel covers fprop and dgrad: dgrad of a stride-s convolution is decomposed into s*s
// output-parity classes, each an exact (zero-waste) stride-1 gather.
//
// Reference arithmetic being replaced: nn.Conv2d forward/backward as called from
//   src/super_gradients/modules/qarepvgg_block.py:184-204, modules/conv_bn_act_block.py:92-93,
//   training/models/classification_models/resnet.py:26-84 (see include/sgb200.h).
#include "common.cuh"
#include "conv_mma.h"

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
  int centre_from;   // 0, or (3x3) the first row whose off-centre entries are left as they are
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
          if (col + e < p.ncols && (p.centre_from == 0 || ko < p.centre_from || (col + e) / p.C == 4))
            atomicAdd(p.DW + (long long)ko * p.ncols + col + e, acc[mt][nt][half * 2 + e]);
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

// A gather of `A` (inH x inW pixels per image, Cg channels per tap at offset in_off of in_pitch) against filter rows of b_pitch
// elements into Ngemm channels of the outH x outW image Y (at out_pitch, out_off): unit strides, taps ascending, no epilogue.
IGemmParams igemm_params(const sgb_bf16* A, int inH, int inW, int in_pitch, int in_off, int Cg, const sgb_bf16* B, int b_pitch,
                         int Ngemm, void* Y, int outH, int outW, int out_pitch, int out_off) {
  IGemmParams p{};
  p.A = reinterpret_cast<const bf16*>(A);
  p.B = reinterpret_cast<const bf16*>(B);
  p.Y = Y;
  p.Ngemm = Ngemm;
  p.Cg = Cg;
  p.row_mul = 1;
  p.tap_sgn = 1;
  p.inH = inH;
  p.inW = inW;
  p.in_pitch = in_pitch;
  p.in_off = in_off;
  p.b_pitch = b_pitch;
  p.rstep = 1;
  p.S_filt = 1;
  p.outH = outH;
  p.outW = outW;
  p.o_mul = 1;
  p.out_pitch = out_pitch;
  p.out_off = out_off;
  p.stats_repl = 1;
  return p;
}
}  // namespace

namespace igemm {

int conv_fprop(const SgbConvDesc& d, const sgb_bf16* x, const sgb_bf16* w, void* y, const SgbEpilogue* ep, cudaStream_t st) {
  IGemmParams p = igemm_params(x, d.H, d.W, d.x_pitch, d.x_off, d.C, w, d.R * d.S * d.C, d.K, y, d.P, d.Q, d.y_pitch, d.y_off);
  p.cls[0] = {d.N * d.P * d.Q, d.P, d.Q, d.R, d.S, d.R * d.S * d.C, -d.pad, -d.pad};
  p.row_mul = d.stride;
  p.S_filt = d.S;
  if (ep) {
    p.scale = ep->scale;
    p.shift = ep->shift;
    p.residual = reinterpret_cast<const bf16*>(ep->residual);
    p.stats = ep->stats;
    p.stats_repl = ep->stats_repl > 0 ? ep->stats_repl : 1;
    SGB_REQUIRE((p.stats_repl & (p.stats_repl - 1)) == 0, "stats_repl must be a power of two");
    p.act = ep->act;
    p.out_f32 = ep->out_f32;
  }
  return dispatch_igemm(p, 1, p.cls[0].M, st);
}

// The transposed convolution as one 1x1 GEMM of 4C columns ordered (dh, dw, co), scattered to the 2 x 2 output pixels.
int convt2x2_fprop(const SgbConvDesc& d, const sgb_bf16* x_small, const sgb_bf16* w_up, const float* bias, sgb_bf16* y_up,
                   cudaStream_t st) {
  IGemmParams p = igemm_params(x_small, d.P, d.Q, d.y_pitch, d.y_off, d.K, w_up, d.K, 4 * d.C, y_up, d.H, d.W, d.x_pitch, d.x_off);
  p.cls[0] = {d.N * d.P * d.Q, d.P, d.Q, 1, 1, d.K};
  p.o_mul = 2;
  p.up2_cout = d.C;
  p.shift = bias;
  return dispatch_igemm(p, 1, p.cls[0].M, st);
}

int conv_dgrad(const SgbConvDesc& d, const sgb_bf16* dy, const sgb_bf16* w_crsk, sgb_bf16* dx, int accumulate, cudaStream_t st) {
  const int s = d.stride;
  const int Kp = ((d.K + 7) / 8) * 8;  // channels gathered per tap (w_crsk rows are padded with zeros to Kp)
  IGemmParams p = igemm_params(dy, d.P, d.Q, d.y_pitch, d.y_off, Kp, w_crsk, d.R * d.S * Kp, d.C, dx, d.H, d.W, d.x_pitch, d.x_off);
  p.tap_sgn = -1;
  p.rstep = s;
  p.S_filt = d.S;
  p.o_mul = s;
  if (accumulate) p.residual = reinterpret_cast<const bf16*>(dx);
  int ncls = 0, maxM = 0;
  for (int ph = 0; ph < s; ++ph)
    for (int pw = 0; pw < s; ++pw) {
      GatherClass& g = p.cls[ncls++];
      g.Hc = (d.H - ph + s - 1) / s;
      g.Wc = (d.W - pw + s - 1) / s;
      g.M = d.N * g.Hc * g.Wc;
      g.r0 = (ph + d.pad) % s;
      g.s0 = (pw + d.pad) % s;
      g.nr = g.r0 < d.R ? (d.R - g.r0 + s - 1) / s : 0;
      g.ns = g.s0 < d.S ? (d.S - g.s0 + s - 1) / s : 0;
      g.Kg = g.nr * g.ns * Kp;
      if (g.ns == 0) g.ns = 1;  // avoid div by zero; Kg == 0 so nothing is gathered
      g.hb_add = (ph + d.pad - g.r0) / s;
      g.wb_add = (pw + d.pad - g.s0) / s;
      g.oh_add = ph;
      g.ow_add = pw;
      if (g.M > maxM) maxM = g.M;
    }
  return dispatch_igemm(p, ncls, maxM, st);
}

int conv_wgrad(const SgbConvDesc& d, const sgb_bf16* x, const sgb_bf16* dy, float* dw, cudaStream_t st) {
  WgradParams p{};
  p.X = reinterpret_cast<const bf16*>(x);
  p.DY = reinterpret_cast<const bf16*>(dy);
  p.DW = dw;
  p.N = d.N; p.H = d.H; p.W = d.W; p.C = d.C; p.K = d.K; p.R = d.R; p.S = d.S; p.P = d.P; p.Q = d.Q;
  p.stride = d.stride; p.pad = d.pad;
  p.x_pitch = d.x_pitch; p.x_off = d.x_off; p.y_pitch = d.y_pitch; p.y_off = d.y_off;
  p.npix = d.N * d.P * d.Q;
  p.ncols = d.R * d.S * d.C;
  p.centre_from = d.centre_from;  // check_desc: only with a 3x3 filter, whose centre tap is tap 4
  int bmw = d.K <= 32 ? 32 : (d.K <= 64 ? 64 : 128);
  if (d.K > 64 && d.K <= 96) bmw = 32;  // 3 x 32 wastes nothing
  int mt = ceil_div(d.K, bmw), nt = ceil_div(p.ncols, 64);
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

}  // namespace igemm

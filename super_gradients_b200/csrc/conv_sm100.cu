// Hopper-native implicit-GEMM convolution: wgmma (M = 64 per warpgroup, fp32 accumulators in registers), the A operand
// streamed by TMA *im2col* descriptors straight from the NHWC activation tensor, the B operand (KRSC / CRSK filters) by
// tiled TMA, an mbarrier ring of shared-memory stages, persistent CTAs of three warpgroups:
//     warpgroup 0     TMA producer (one elected lane)
//     warpgroups 1-2  wgmma over 64 rows each of the 128-pixel tile, then the epilogue straight from the accumulator
//                     registers: (scale, shift, residual, activation) -> bf16 -> global, plus the per-channel sum /
//                     sum-of-squares needed by train-mode BatchNorm, combined across warps in a fixed order
// The producer runs up to `stages` k-iterations ahead, so the loads of tile i+1 overlap the epilogue of tile i.
//
// Serves every 1x1 and 3x3 convolution with C % 16 == 0 (fprop; stride-1 dgrad over the flipped CRSK filter; stride-2 dgrad as
// s^2 output-parity classes through the explicit tap table) and their weight gradients (wgrad_wgmma_kernel, MN-major
// operands; wgrad3x3_halo_kernel for the 3x3 stride-1 ones).  conv_fprop / conv_dgrad / conv_wgrad / convt2x2_fprop at the end of
// the file re-describe each C-ABI call as these GEMMs, or decline it: 3-channel stems that are not padded to 16 channels, 7x7,
// ragged channel counts and fp32 outputs stay on the mma.sync kernels of conv_mma.cu.
//
// Reference arithmetic replaced: nn.Conv2d forward / input-gradient / weight-gradient as used by
// modules/qarepvgg_block.py:184-204, modules/conv_bn_act_block.py:92-93,
// training/models/classification_models/resnet.py:53-84.
#include <cuda.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include "conv_sm100.h"
#include "sm100_host.h"
#include "sm100_ptx.cuh"

namespace sm100 {

constexpr int BLOCK_M = 128;
constexpr int NUM_THREADS = 384;
constexpr int CONSUMER_THREADS = 256;
constexpr int MAX_STAGES = 8;

struct Params {
  int M;            // output pixels (GEMM rows)
  int N;            // output channels (GEMM cols)
  int C;            // channels per tap of the gathered tensor
  int KC;           // channels per TMA box (16 / 32 / 64)
  int n_tiles;      // N tiles of BN columns
  int stages;
  int P, Q;         // output spatial size (rows -> (n, p, q))
  int stride, pad;  // traversal stride, lower padding of the gather
  int b_cols_per_tap;
  int ntaps;                  // taps visited (R*S for fprop / stride-1 dgrad; a subset for a stride-2 dgrad parity class)
  signed char tap_dh[9], tap_dw[9], tap_b[9];  // im2col offsets of each tap and its column block in the B matrix
  // output row m -> address.  out_mode 0: rows are consecutive NHWC pixels.  out_mode 1: row m = (n, j, i) over a
  // (P x Q) grid is written to pixel (n, j*o_mul + oh_add, i*o_mul + ow_add) of an (outH x outW) image.
  int out_mode, o_mul, oh_add, ow_add, outH, outW;
  int halo_tw, halo_thw;  // conv3x3_halo_kernel: 8 x 8 output tiles per image row band / per image
  long long y_pitch;  // elements
  int y_off;
  bf16* y;
  const float* scale;
  const float* shift;
  const bf16* residual;
  double* stats;
  int stats_repl;
  int act;
  // folded QARepVGG filters (Problem::centre_from): output columns >= centre_n (fprop) / gathered channels >= centre_c (dgrad)
  // meet only zeros on the eight off-centre taps (tap 4 of 9 is the centre); 0: off
  int centre_n, centre_c;
};

// The k-steps per off-centre tap on N tile nt when a folded filter's zero taps are skipped (of `steps` per tap, each over
// step_ch gathered channels; the centre tap runs all of them): none for a tile wholly at or past centre_n, those below centre_c.
// A tile that straddles centre_n runs every tap: issuing its off-centre taps as wgmmas of half the tile's width measured slower
// than the full width in the halo kernel.  Each product skipped is one by an exact zero, so skipping changes no sum.
template <int BN>
__device__ __forceinline__ int off_centre_steps(const Params& p, int nt, int steps, int step_ch) {
  if (p.centre_n > 0 && nt * BN >= p.centre_n) return 0;
  if (p.centre_c > 0) return (p.centre_c + step_ch - 1) / step_ch;
  return steps;
}
constexpr int CENTRE_TAP = 4;

__device__ __forceinline__ long long out_row(const Params& p, long long m) {
  if (p.out_mode == 0) return m;
  const int pq = p.P * p.Q;
  const int n = (int)(m / pq);
  const int rem = (int)(m - (long long)n * pq);
  const int j = rem / p.Q, i = rem - j * p.Q;
  return ((long long)n * p.outH + j * p.o_mul + p.oh_add) * p.outW + i * p.o_mul + p.ow_add;
}

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(CONSUMER_THREADS) : "memory"); }
// Both consumer warpgroups (WARPS = 8), or consumer warpgroup wg alone (WARPS = 4, named barrier 2 + wg).
template <int WARPS>
__device__ __forceinline__ void group_sync(int wg) {
  if (WARPS == 8)
    consumer_sync();
  else
    asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
}

// Shared-memory layout after the stages: full / empty barriers, then (statistics only) the per-warp column partials of the
// current tile [8 warps][2][BN] and the CTA's per-channel totals [2][N].
constexpr uint32_t CTRL_BAR_BYTES = 16u * MAX_STAGES;

// Epilogue of one tile straight from the accumulator registers of a consumer warp (warpgroup wg, 16-row slice wq): the thread
// holds two rows, at output pixels orow[0] / orow[1] (row_ok false: the row lies past the output), and the column pairs
// 8 j + 2 (lane % 4) of N tile nt.  (scale, shift, residual, activation) -> bf16 -> global, plus the per-channel sum /
// sum-of-squares of the stored values, combined in a fixed order across the WARPS warps that share the tile (8: both consumer
// warpgroups; 4: warpgroup wg alone, with its own s_part / s_stats) into s_stats.
template <int BN, int WARPS = 8>
__device__ __forceinline__ void tile_epilogue(const Params& p, const float (&acc)[BN / 2], const long long (&orow)[2],
                                              const bool (&row_ok)[2], int nt, int wg, int wq, int lane, float* s_part,
                                              float* s_stats) {
  const int n0 = nt * BN;
  const int ncols = min(BN, p.N - n0);
  bf16* yrow[2];
  const bf16* rrow[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    yrow[h] = p.y + orow[h] * p.y_pitch + p.y_off + n0;
    rrow[h] = p.residual ? p.residual + orow[h] * p.y_pitch + p.y_off + n0 : nullptr;
  }
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = 8 * j + 2 * (lane & 3);
    const bool col_ok = col < ncols;  // N % 8 == 0: both columns of the pair are valid or neither
    float sum0 = 0.f, sum1 = 0.f, sq0 = 0.f, sq1 = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      const bool ok = row_ok[h] && col_ok;
      if (p.scale && col_ok) {
        v0 *= p.scale[n0 + col];
        v1 *= p.scale[n0 + col + 1];
      }
      if (p.shift && col_ok) {
        v0 += p.shift[n0 + col];
        v1 += p.shift[n0 + col + 1];
      }
      if (rrow[h] && ok) {
        const uint32_t rr = *reinterpret_cast<const uint32_t*>(rrow[h] + col);
        v0 += __uint_as_float(rr << 16);
        v1 += __uint_as_float(rr & 0xffff0000u);
      }
      if (p.act != SGB_ACT_NONE) {
        v0 = apply_act(v0, p.act);
        v1 = apply_act(v1, p.act);
      }
      __nv_bfloat162 hh = __floats2bfloat162_rn(v0, v1);
      const uint32_t pk = *reinterpret_cast<uint32_t*>(&hh);
      if (ok) {
        *reinterpret_cast<uint32_t*>(yrow[h] + col) = pk;
        const float lo = __uint_as_float(pk << 16), hi = __uint_as_float(pk & 0xffff0000u);
        sum0 += lo;
        sum1 += hi;
        sq0 = fmaf(lo, lo, sq0);
        sq1 = fmaf(hi, hi, sq1);
      }
    }
    if (p.stats) {
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        sum0 += __shfl_xor_sync(0xffffffffu, sum0, o);
        sum1 += __shfl_xor_sync(0xffffffffu, sum1, o);
        sq0 += __shfl_xor_sync(0xffffffffu, sq0, o);
        sq1 += __shfl_xor_sync(0xffffffffu, sq1, o);
      }
      if (lane < 4) {
        float* part = s_part + (WARPS == 8 ? wg * 4 + wq : wq) * 2 * BN;
        part[col] = sum0;
        part[col + 1] = sum1;
        part[BN + col] = sq0;
        part[BN + col + 1] = sq1;
      }
    }
  }
  if (p.stats) {
    // the eight warps' partials of this tile, summed in a fixed order (bit-reproducible statistics)
    group_sync<WARPS>(wg);
    for (int i = threadIdx.x - 128 - (WARPS == 8 ? 0 : 128 * wg); i < 2 * BN; i += WARPS * 32) {
      const int which = i / BN, c = i - which * BN;
      if (c < ncols) {
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) v += s_part[w * 2 * BN + i];
        s_stats[which * p.N + n0 + c] += v;
      }
    }
    group_sync<WARPS>(wg);
  }
}

// The CTA's per-channel totals -> the fp64 statistics buffer (after a __syncthreads).
__device__ __forceinline__ void flush_stats(const Params& p, const float* s_stats) {
  if (p.stats) {
    double* st = p.stats + (long long)(blockIdx.x & (p.stats_repl - 1)) * 2 * p.N;
    for (int i = threadIdx.x; i < 2 * p.N; i += NUM_THREADS) {
      const float v = s_stats[i];
      if (v != 0.f) atomicAdd(&st[i], (double)v);
    }
  }
}

// ------------------------------------------------------------------------------------------------ the kernel
// SKIP: a folded QARepVGG filter (Params::centre_n / centre_c): the off-centre taps run off_centre_steps chunks.
template <int BN, bool SKIP>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const Params p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_bytes = BLOCK_M * p.KC * 2, b_bytes = BN * p.KC * 2;
  const uint32_t stage_bytes = a_bytes + ((b_bytes + 1023u) & ~1023u);
  const uint32_t ctrl = smem_base + p.stages * stage_bytes;
  auto full_bar = [&](int s) { return ctrl + 8u * s; };
  auto empty_bar = [&](int s) { return ctrl + 8u * (MAX_STAGES + s); };
  float* s_part = reinterpret_cast<float*>(smem_raw + (ctrl + CTRL_BAR_BYTES - smem_u32(smem_raw)));
  float* s_stats = s_part + 8 * 2 * BN;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int total_tiles = m_tiles * p.n_tiles;
  const int chunks = (p.C + p.KC - 1) / p.KC;  // a last chunk reaching past C is zero-filled by TMA (out-of-bounds channels)

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);  // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  if (p.stats)
    for (int i = threadIdx.x; i < 2 * p.N; i += NUM_THREADS) s_stats[i] = 0.f;
  __syncthreads();

  if (warp == 0) {
    // ===================================================================================== TMA producer
    if (elect_one()) {
      int stg = 0;
      uint32_t par = 1;  // parity awaited on the empty barriers: the first pass through the ring is free
      const int pq = p.P * p.Q;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int mt = tile / p.n_tiles, nt = tile - mt * p.n_tiles;
        const int m0 = mt * BLOCK_M;
        const int n_img = m0 / pq;
        const int rem = m0 - n_img * pq;
        const int p0 = rem / p.Q, q0 = rem - p0 * p.Q;
        const int w0 = q0 * p.stride - p.pad, h0 = p0 * p.stride - p.pad;
        const int off = SKIP ? off_centre_steps<BN>(p, nt, chunks, p.KC) : chunks;
        for (int tap = 0; tap < p.ntaps; ++tap) {
          const int r = p.tap_dh[tap], s = p.tap_dw[tap];
          const int btap = p.tap_b[tap];
          const int n_ck = tap == CENTRE_TAP ? chunks : off;
          for (int ck = 0; ck < n_ck; ++ck) {
            mbar_wait(empty_bar(stg), par);
            const uint32_t sa = smem_base + stg * stage_bytes, sb = sa + a_bytes;
            mbar_expect_tx(full_bar(stg), a_bytes + b_bytes);
            tma_load_im2col_4d(sa, &map_a, full_bar(stg), ck * p.KC, w0, h0, n_img, (uint16_t)s, (uint16_t)r);
            tma_load_2d(sb, &map_b, full_bar(stg), btap * p.b_cols_per_tap + ck * p.KC, nt * BN);
            if (++stg == p.stages) {
              stg = 0;
              par ^= 1;
            }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================================================================================== MMA + epilogue
    const int wg = (warp >> 2) - 1;  // rows [64 * wg, 64 * wg + 64) of the tile
    const int wq = warp & 3;         // 16-row slice of the warpgroup's 64 rows
    const int row_bytes = p.KC * 2;
    const uint32_t sbo = 8u * (uint32_t)row_bytes;
    const int ksteps = p.KC / 16;
    float acc[BN / 2];
    int stg = 0;
    uint32_t par = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int mt = tile / p.n_tiles, nt = tile - mt * p.n_tiles;
      // the producer's k-sequence: taps in order, `chunks` k-iterations on the centre tap, fewer on the others when skipping
      const int k_iters = SKIP ? 8 * off_centre_steps<BN>(p, nt, chunks, p.KC) + chunks : p.ntaps * chunks;
      int prev = -1;
      for (int k = 0; k < k_iters; ++k) {
        mbar_wait(full_bar(stg), par);
        const uint32_t sa = smem_base + stg * stage_bytes, sb = sa + a_bytes;
        const uint32_t sa_wg = sa + (uint32_t)wg * 64u * (uint32_t)row_bytes;
        wgmma_fence();
        for (int j = 0; j < ksteps; ++j) {
          // advance 16 bf16 (32 bytes) along K inside the swizzle atom
          const uint64_t da = smem_desc(sa_wg + 32u * j, row_bytes, 16u, sbo), db = smem_desc(sb + 32u * j, row_bytes, 16u, sbo);
          mma_kk<BN>(acc, da, db, (k | j) != 0);
        }
        wgmma_commit();
        if (prev >= 0) {
          wgmma_wait<1>();  // the previous stage's MMAs are complete: its shared memory may be refilled
          __syncwarp();
          if (lane == 0) mbar_arrive(empty_bar(prev));
        }
        prev = stg;
        if (++stg == p.stages) {
          stg = 0;
          par ^= 1;
        }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      __syncwarp();
      if (lane == 0 && prev >= 0) mbar_arrive(empty_bar(prev));

      // ---- epilogue: thread holds rows r_lo, r_lo + 8 of the tile
      const long long m_lo = (long long)mt * BLOCK_M + wg * 64 + wq * 16 + (lane >> 2);
      long long orow[2];
      bool row_ok[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long m = m_lo + 8 * h;
        row_ok[h] = m < p.M;
        orow[h] = out_row(p, row_ok[h] ? m : 0);
      }
      tile_epilogue<BN>(p, acc, orow, row_ok, nt, wg, wq, lane, s_part, s_stats);
    }
  }
  __syncthreads();
  flush_stats(p, s_stats);
}

// ------------------------------------------------------------------------------------------------ halo-tile kernel
// 3x3 / stride 1 / pad 1 convolutions, out_mode 0, no tap table: fprop and the stride-1 dgrad over the flipped CRSK filter.
// A tile is 8 x 8 output pixels of one image (M = 64, one 8-pixel output row per wgmma 8-row core-matrix group), and the two
// consumer warpgroups take alternate tiles of the CTA's sequence, each with its own accumulators, so one warpgroup's epilogue
// overlaps the other's MMAs.  The producer loads a tile's 10 x 10-pixel input halo once, as one tiled TMA box {8 channels, 10, 10}
// per 8-channel group, into the no-swizzle K-major layout [channel group][10 x 10 pixels][8 channels]: the A operand of tap
// (dh, dw) is the same buffer with its start moved by (dh * 10 + dw) * 16 bytes (SBO = one 10-pixel row, LBO = one channel
// group).  Image borders and the padding are TMA's out-of-bounds zero fill; pixels past the image are computed and masked in
// the epilogue.  Each CTA serves one N tile and keeps its 9 x C x BN filter slice resident in shared memory (16 channels per
// box, 32-byte swizzle), loaded once before its first tile; the halo buffers form the mbarrier ring.
// The k16 steps run tap-major, channels ascending, and the epilogue is conv_wgmma_kernel's, so every output equals that kernel's
// bit for bit, except that its zero-filled steps past C (C = 48 / 96) can turn a -0 into +0.
constexpr int HALO_W = 10, HALO_H = 10, HALO_TILE = 8;
constexpr uint32_t HALO_CG_BYTES = 1664;  // one channel group of the halo: 10 x 10 x 16 bytes, padded to the TMA's 128-byte alignment
constexpr uint32_t HALO_CTRL_BYTES = CTRL_BAR_BYTES + 16;  // + the filter barrier
constexpr int HALO_MAX_STAGES = 6;

// N tiles up to 48 wide are held to 80 registers so that two CTAs can share an SM.  SKIP: a folded QARepVGG filter
// (Params::centre_n / centre_c): the off-centre taps run off_centre_steps k16 steps.
template <int BN, bool SKIP>
__global__ void __launch_bounds__(NUM_THREADS, BN <= 48 ? 2 : 1)
conv3x3_halo_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const Params p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int ksteps = p.C / 16;
  constexpr uint32_t b_box = BN * 32;  // 16 channels of BN filter rows
  const uint32_t b_bytes = 9u * ksteps * b_box;
  const uint32_t a_stage = ((uint32_t)(p.C / 8) * HALO_CG_BYTES + 1023u) & ~1023u;
  const uint32_t sb = smem_base, sa0 = smem_base + ((b_bytes + 1023u) & ~1023u);
  const uint32_t ctrl = sa0 + p.stages * a_stage;
  auto full_bar = [&](int s) { return ctrl + 8u * s; };
  auto empty_bar = [&](int s) { return ctrl + 8u * (MAX_STAGES + s); };
  const uint32_t b_bar = ctrl + CTRL_BAR_BYTES;
  float* s_part = reinterpret_cast<float*>(smem_raw + (ctrl + HALO_CTRL_BYTES - smem_u32(smem_raw)));  // [2 wg][4 warps][2][BN]
  float* s_stats = s_part + 8 * 2 * BN;                                                                  // [2 wg][2][N]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tiles = p.M;  // here: the number of 8 x 8 tiles
  const int nt = blockIdx.x % p.n_tiles;
  const int mt_step = gridDim.x / p.n_tiles;
  const int mt0 = blockIdx.x / p.n_tiles;
  // k16 steps of each off-centre tap (the centre tap runs ksteps)
  const int off = SKIP ? off_centre_steps<BN>(p, nt, ksteps, 16) : ksteps;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 4);  // one arrival per warp of the consuming warpgroup
    }
    mbar_init(b_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  if (p.stats)
    for (int i = threadIdx.x; i < 4 * p.N; i += NUM_THREADS) s_stats[i] = 0.f;
  __syncthreads();

  if (warp == 0) {
    // ===================================================================================== TMA producer
    if (elect_one()) {
      // the filter boxes the MMAs read (B tap 4 is the centre, flipped or not); the others stay unloaded
      mbar_expect_tx(b_bar, (uint32_t)(8 * off + ksteps) * b_box);
      for (int bt = 0; bt < 9; ++bt)
        for (int ks = 0; ks < (bt == CENTRE_TAP ? ksteps : off); ++ks)
          tma_load_2d(sb + (uint32_t)(bt * ksteps + ks) * b_box, &map_b, b_bar, bt * p.b_cols_per_tap + 16 * ks, nt * BN);
      const uint32_t a_tx = (uint32_t)(p.C / 8) * (HALO_H * HALO_W * 16);
      int stg = 0;
      uint32_t par = 1;  // the first pass through the ring is free
      for (int mt = mt0; mt < m_tiles; mt += mt_step) {
        const int n_img = mt / p.halo_thw;
        const int rem = mt - n_img * p.halo_thw;
        const int th = rem / p.halo_tw, tw = rem - th * p.halo_tw;
        mbar_wait(empty_bar(stg), par);
        const uint32_t sa = sa0 + stg * a_stage;
        mbar_expect_tx(full_bar(stg), a_tx);
        for (int cg = 0; cg < p.C / 8; ++cg)
          tma_load_tiled_4d(sa + (uint32_t)cg * HALO_CG_BYTES, &map_a, full_bar(stg), 8 * cg, tw * HALO_TILE - 1, th * HALO_TILE - 1,
                            n_img);
        if (++stg == p.stages) {
          stg = 0;
          par ^= 1;
        }
      }
    }
  } else if (warp >= 4) {
    // ===================================================================================== MMA + epilogue
    const int wg = (warp >> 2) - 1;  // takes tiles wg, wg + 2, wg + 4, ... of the CTA's sequence
    const int wq = warp & 3;
    float acc[BN / 2];
    mbar_wait(b_bar, 0);
    for (int j = wg, mt = mt0 + wg * mt_step; mt < m_tiles; j += 2, mt += 2 * mt_step) {
      const int stg = j % p.stages;
      mbar_wait(full_bar(stg), (uint32_t)(j / p.stages) & 1u);
      const uint32_t sa = sa0 + stg * a_stage;
      wgmma_fence();
      // one flat loop over (tap, 16-channel step): a nested loop makes ptxas fence the accumulators at every tap.  Taps in order,
      // ksteps steps on the centre tap and `off` on the others (none: the loop starts at the centre).
      int t = off > 0 ? 0 : CENTRE_TAP;
      uint32_t sa_t = sa + (uint32_t)((t / 3) * HALO_W + t % 3) * 16u, sb_t = sb + (uint32_t)(p.tap_b[t] * ksteps) * b_box;
      for (int k = 0, ks = 0, nk = 8 * off + ksteps; k < nk; ++k) {
        const uint64_t da = smem_desc_noswizzle(sa_t + (uint32_t)(2 * ks) * HALO_CG_BYTES, HALO_CG_BYTES, HALO_W * 16);
        const uint64_t db = smem_desc(sb_t + (uint32_t)ks * b_box, 32, 16u, 256u);
        mma_kk<BN>(acc, da, db, k != 0);
        if (++ks == (t == CENTRE_TAP ? ksteps : off) && ++t < 9) {
          ks = 0;
          sa_t = sa + (uint32_t)((t / 3) * HALO_W + t % 3) * 16u;
          sb_t = sb + (uint32_t)(p.tap_b[t] * ksteps) * b_box;
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(stg));

      // ---- epilogue: thread holds output rows 2 wq and 2 wq + 1 of the tile, column lane / 4
      const int n_img = mt / p.halo_thw;
      const int rem = mt - n_img * p.halo_thw;
      const int th = rem / p.halo_tw, tw = rem - th * p.halo_tw;
      const int ow = tw * HALO_TILE + (lane >> 2);
      long long orow[2];
      bool row_ok[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int oh = th * HALO_TILE + 2 * wq + h;
        row_ok[h] = oh < p.P && ow < p.Q;
        orow[h] = row_ok[h] ? ((long long)n_img * p.P + oh) * p.Q + ow : 0;
      }
      tile_epilogue<BN, 4>(p, acc, orow, row_ok, nt, wg, wq, lane, s_part + wg * 4 * 2 * BN, s_stats + wg * 2 * p.N);
    }
  }
  __syncthreads();
  if (p.stats) {  // the two warpgroups' totals, in a fixed order
    for (int i = threadIdx.x; i < 2 * p.N; i += NUM_THREADS) s_stats[i] += s_stats[2 * p.N + i];
    __syncthreads();
  }
  flush_stats(p, s_stats);
}

// ------------------------------------------------------------------------------------------------ wgrad kernel
// dW[ko][(r,s,c)] += sum_pix dy[pix][ko] * x[pix @ (r,s)][c]       (fp32 reductions over pixel splits)
// GEMM view: M = out-channels (64 per consumer warpgroup), N = NB in-channels of one tap, K = pixels.  Both operands are
// "MN-major": a TMA box of [WPIX pixels][channels] IS the canonical MN-major swizzled layout (each K index is one swizzled
// row), so dy and the im2col'd x stream straight from NHWC memory with no transpose.
// One CTA = (one or two 64-row blocks of out-channels) x (one tap) x (NB in-channels) x (pixel range).  A tap takes the 64-row
// blocks that cover K, or -- off the centre of a folded QARepVGG filter (centre_from) -- those that cover centre_from.  They are
// paired into CTAs of 128 rows, one block per consumer warpgroup; an odd last block is a CTA of its own whose two warpgroups take
// the even / odd pipeline stages and both add their partial sums into dW, so a layer of K <= 64 no longer pays for 128 rows.
struct WParams {
  int K, C;            // out / in channels
  int R, S, stride, pad, P, Q;
  int npix;            // N*P*Q
  int CB;              // in-channels per im2col box (16 / 32 / 64)
  int n_ctiles;
  int rb_all, rb_off;  // 64-row blocks of the centre tap / of each other tap (== rb_all without centre_from)
  int items;           // row items (CTAs per in-channel tile and pixel range) summed over the taps
  int pix_per_cta;     // multiple of WPIX
  int stages;
  int cpad;            // channel count of the KRSC output rows (x channels incl. padding)
  int centre_from;     // 0, or the first row whose off-centre entries are not written (a row block may reach past it)
  float* dw;
  int halo_tw, halo_thw, tiles, tiles_per_cta;  // wgrad3x3_halo_kernel: 8 x 8 tiles per image row band / per image / in all
};
constexpr int WPIX = 64;  // pixels (GEMM K) per pipeline stage

__host__ __device__ __forceinline__ int wgrad_row_blocks(const WParams& p, int tap) {
  return p.R * p.S == 9 && tap != CENTRE_TAP ? p.rb_off : p.rb_all;
}

// dW rows tap `tap` writes: all K, or below centre_from off the centre of a folded filter
__device__ __forceinline__ int wgrad_rows(const WParams& p, int tap) {
  return p.centre_from > 0 && p.R * p.S == 9 && tap != CENTRE_TAP ? p.centre_from : p.K;
}

template <int NB>
__global__ void __launch_bounds__(NUM_THREADS, 1)
wgrad_wgmma_kernel(const __grid_constant__ CUtensorMap map_dy, const __grid_constant__ CUtensorMap map_x, const WParams p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_bytes = 2 * WPIX * 128;                       // two 64-channel blocks of dy
  const uint32_t b_box = WPIX * p.CB * 2;                        // one im2col box
  const int boxes = NB / p.CB;
  const uint32_t stage_bytes = a_bytes + (uint32_t)boxes * b_box;  // multiples of 1024 by construction
  const uint32_t ctrl = smem_base + p.stages * stage_bytes;
  auto full_bar = [&](int s) { return ctrl + 8u * s; };
  auto empty_bar = [&](int s) { return ctrl + 8u * (MAX_STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // decode the CTA's work item: pixel range, then tap, in-channel tile and row item (fastest)
  int w = blockIdx.x;
  const int split = w / (p.items * p.n_ctiles);
  w -= split * p.items * p.n_ctiles;
  int tap = 0, tap_items = (wgrad_row_blocks(p, 0) + 1) / 2;
  while (w >= tap_items * p.n_ctiles) {
    w -= tap_items * p.n_ctiles;
    tap_items = (wgrad_row_blocks(p, ++tap) + 1) / 2;
  }
  const int ctile = w / tap_items, item = w - ctile * tap_items;
  const bool shared_rows = 2 * item + 1 == wgrad_row_blocks(p, tap);  // one row block for both warpgroups
  const int row0 = 128 * item;
  const int pix0 = split * p.pix_per_cta;
  const int pix1 = min(pix0 + p.pix_per_cta, p.npix);
  const int n_iters = (pix1 - pix0 + WPIX - 1) / WPIX;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), shared_rows ? 4 : 8);  // one arrival per warp that reads the stage
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (n_iters > 0) {
    if (warp == 0) {
      if (elect_one()) {
        const int pq = p.P * p.Q;
        const int r = tap / p.S, s = tap - r * p.S;
        int stg = 0;
        uint32_t par = 1;
        for (int it = 0; it < n_iters; ++it) {
          mbar_wait(empty_bar(stg), par);
          const uint32_t sa = smem_base + stg * stage_bytes, sb = sa + a_bytes;
          mbar_expect_tx(full_bar(stg), (shared_rows ? a_bytes / 2 : a_bytes) + (uint32_t)boxes * b_box);
          const int pix = pix0 + it * WPIX;
          tma_load_2d(sa, &map_dy, full_bar(stg), row0, pix);
          if (!shared_rows) tma_load_2d(sa + WPIX * 128, &map_dy, full_bar(stg), row0 + 64, pix);
          const int n_img = pix / pq;
          const int rem = pix - n_img * pq;
          const int p0 = rem / p.Q, q0 = rem - p0 * p.Q;
          const int w0 = q0 * p.stride - p.pad, h0 = p0 * p.stride - p.pad;
          for (int bx = 0; bx < boxes; ++bx)
            tma_load_im2col_4d(sb + (uint32_t)bx * b_box, &map_x, full_bar(stg), ctile * NB + bx * p.CB, w0, h0, n_img, (uint16_t)s,
                               (uint16_t)r);
          if (++stg == p.stages) {
            stg = 0;
            par ^= 1;
          }
        }
      }
    } else if (warp >= 4) {
      const int wg = (warp >> 2) - 1, wq = warp & 3;
      const int b_row_bytes = p.CB * 2;
      float acc[NB / 2];
      // own row block: every stage; shared row block: stages wg, wg + 2, ...
      const int it0 = shared_rows ? wg : 0, it_step = shared_rows ? 2 : 1;
      const uint32_t a_off = shared_rows ? 0u : (uint32_t)wg * (WPIX * 128);
      int stg = it0, prev = -1;
      uint32_t par = 0;
      for (int it = it0; it < n_iters; it += it_step) {
        mbar_wait(full_bar(stg), par);
        const uint32_t sa = smem_base + stg * stage_bytes + a_off, sb = smem_base + stg * stage_bytes + a_bytes;
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < WPIX / 16; ++j) {
          // A: one 64-channel atom of 128-byte pixel rows; B: the boxes are consecutive MN atoms (LBO = box size)
          const uint64_t da = smem_desc(sa + (uint32_t)j * 16u * 128u, 128, WPIX * 128, 8 * 128);
          const uint64_t db = smem_desc(sb + (uint32_t)j * 16u * (uint32_t)b_row_bytes, b_row_bytes, b_box, 8u * (uint32_t)b_row_bytes);
          mma_mn<NB>(acc, da, db, (it != it0 || j != 0) ? 1u : 0u);
        }
        wgmma_commit();
        if (prev >= 0) {
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(empty_bar(prev));
        }
        prev = stg;
        if ((stg += it_step) >= p.stages) {  // it_step <= 2 <= stages
          stg -= p.stages;
          par ^= 1;
        }
      }
      if (prev < 0) return;  // a shared row block with a single stage: nothing for warpgroup 1
      wgmma_wait<0>();
      fence_regs(acc);
      const int row_len = p.R * p.S * p.cpad;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ko = row0 + (shared_rows ? 0 : wg * 64) + wq * 16 + (lane >> 2) + 8 * h;
        if (ko < wgrad_rows(p, tap)) {
          float* drow = p.dw + (long long)ko * row_len + tap * p.cpad + ctile * NB + 2 * (lane & 3);
#pragma unroll
          for (int j = 0; j < NB / 8; ++j)
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(drow + 8 * j), "f"(acc[4 * j + 2 * h]), "f"(acc[4 * j + 2 * h + 1])
                         : "memory");
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ halo-tile wgrad kernel
// Weight gradient of a 3x3 / stride 1 / pad 1 convolution over 8 x 8 output tiles, loading each tile's dy block and input halo
// once for all nine taps (wgrad_wgmma_kernel streams dy and an im2col view of x once per tap).  One CTA = one 64-row block rb of
// out-channels x NB in-channels (in-channel tile ctile) x a range of tiles; GEMM M = the 64 rows, N = NB, K = the tile's 64 pixels.
// Per stage the producer loads
//   A: dy of the tile, one tiled TMA box {64 channels, 8, 8, 1} with 128-byte swizzle: 64 pixel rows of 128 bytes, the MN-major
//      layout wgrad_wgmma_kernel reads; pixels past the image are zero-filled and add nothing;
//   B: the 10 x 10 input halo of the NB channels, as conv3x3_halo_kernel loads it ([channel group][10 x 10 pixels][8 channels],
//      image borders and padding from TMA's zero fill).  Read MN-major, 8 consecutive pixels of a halo row are one 128-byte core
//      matrix: tap (dh, dw) starts (dh * 10 + dw) * 16 bytes in, the second 8 pixels of a k16 step (the next output row) lie one
//      halo row (LBO = 160 bytes) on, the next 8 channels one channel group (SBO = HALO_CG_BYTES) on.
// Warpgroup 0 accumulates taps 0-4 and warpgroup 1 taps 5-8 (9 x NB / 2 fp32 per thread would not fit one warpgroup), so both
// read every stage and its empty barrier counts all eight consumer warps.  A row block past the off-centre rows of a folded
// filter (rb >= rb_off) runs the centre tap alone, on warpgroup 0.  Each CTA adds its partial sums into dW once, at the end.
constexpr uint32_t WH_A_BYTES = WPIX * 128;  // the dy tile of a stage

__host__ __device__ constexpr uint32_t wgrad_halo_stage_bytes(int nb) {
  return (WH_A_BYTES + (uint32_t)(nb / 8) * HALO_CG_BYTES + 1023u) & ~1023u;
}

// One consumer warpgroup of wgrad3x3_halo_kernel: taps tap0 .. tap0 + NT - 1 of every stage (NT = 0: none, the warpgroup only
// frees the stages), then their partial sums into dW.  The tap count is a template parameter and the waits are unconditional so
// that no branch separates the wgmmas of the loop: ptxas serialises wgmmas on a divergent path.
template <int NB, int NT>
__device__ __forceinline__ void wgrad_halo_consume(const WParams& p, uint32_t ring, uint32_t bars, int t0, int t1, int tap0, int rb,
                                                   int ctile) {
  constexpr uint32_t stage_bytes = wgrad_halo_stage_bytes(NB);
  const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  auto full_bar = [&](int s) { return bars + 8u * s; };
  auto empty_bar = [&](int s) { return bars + 8u * (MAX_STAGES + s); };
  float acc[NT > 0 ? NT : 1][NB / 2];
  int stg = 0, prev = 0;
  uint32_t par = 0;
  for (int mt = t0; mt < t1; ++mt) {
    mbar_wait(full_bar(stg), par);
    if constexpr (NT > 0) {
      const uint32_t sa = ring + stg * stage_bytes, sx = sa + WH_A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const int tap = tap0 + t;
        const uint32_t sx_t = sx + (uint32_t)((tap / 3) * HALO_W + tap % 3) * 16u;
#pragma unroll
        for (int j = 0; j < WPIX / 16; ++j) {
          const uint64_t da = smem_desc(sa + (uint32_t)j * 16u * 128u, 128, WPIX * 128, 8 * 128);
          const uint64_t db = smem_desc_noswizzle(sx_t + (uint32_t)j * 2u * HALO_W * 16u, HALO_W * 16, HALO_CG_BYTES);
          mma_mn<NB>(acc[t], da, db, (mt != t0 || j != 0) ? 1u : 0u);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();  // the previous stage's MMAs are complete: its shared memory may be refilled
    }
    __syncwarp();
    if (lane == 0 && mt != t0) mbar_arrive(empty_bar(prev));
    prev = stg;
    if (++stg == p.stages) {
      stg = 0;
      par ^= 1;
    }
  }
  if constexpr (NT > 0) {
    wgmma_wait<0>();
#pragma unroll
    for (int t = 0; t < NT; ++t) fence_regs(acc[t]);
  }
  __syncwarp();
  if (lane == 0) mbar_arrive(empty_bar(prev));
  if constexpr (NT > 0) {
    const int row_len = 9 * p.cpad;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int ko = 64 * rb + wq * 16 + (lane >> 2) + 8 * h;
      if (ko < p.K) {
        float* drow = p.dw + (long long)ko * row_len + tap0 * p.cpad + ctile * NB + 2 * (lane & 3);
#pragma unroll
        for (int t = 0; t < NT; ++t) {
          if (ko >= wgrad_rows(p, tap0 + t)) continue;
#pragma unroll
          for (int j = 0; j < NB / 8; ++j)
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(drow + t * p.cpad + 8 * j), "f"(acc[t][4 * j + 2 * h]),
                         "f"(acc[t][4 * j + 2 * h + 1])
                         : "memory");
        }
      }
    }
  }
}

template <int NB>
__global__ void __launch_bounds__(NUM_THREADS, 1)
wgrad3x3_halo_kernel(const __grid_constant__ CUtensorMap map_dy, const __grid_constant__ CUtensorMap map_x, const WParams p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr uint32_t a_bytes = WH_A_BYTES, stage_bytes = wgrad_halo_stage_bytes(NB);
  const uint32_t ctrl = smem_base + p.stages * stage_bytes;
  auto full_bar = [&](int s) { return ctrl + 8u * s; };
  auto empty_bar = [&](int s) { return ctrl + 8u * (MAX_STAGES + s); };

  const int warp = threadIdx.x >> 5;
  // work item: tile range (slowest), then in-channel tile, then row block
  const int items = p.rb_all * p.n_ctiles;
  const int split = blockIdx.x / items, item = blockIdx.x - split * items;
  const int ctile = item / p.rb_all, rb = item - ctile * p.rb_all;
  const bool all_taps = rb < p.rb_off;
  const int t0 = split * p.tiles_per_cta, t1 = min(t0 + p.tiles_per_cta, p.tiles);

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);  // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    // ===================================================================================== TMA producer
    if (elect_one()) {
      const uint32_t tx = a_bytes + (NB / 8) * (HALO_H * HALO_W * 16);
      int stg = 0;
      uint32_t par = 1;  // the first pass through the ring is free
      for (int mt = t0; mt < t1; ++mt) {
        const int n_img = mt / p.halo_thw;
        const int rem = mt - n_img * p.halo_thw;
        const int th = rem / p.halo_tw, tw = rem - th * p.halo_tw;
        mbar_wait(empty_bar(stg), par);
        const uint32_t sa = smem_base + stg * stage_bytes;
        mbar_expect_tx(full_bar(stg), tx);
        tma_load_tiled_4d(sa, &map_dy, full_bar(stg), 64 * rb, tw * HALO_TILE, th * HALO_TILE, n_img);
        for (int cg = 0; cg < NB / 8; ++cg)
          tma_load_tiled_4d(sa + a_bytes + (uint32_t)cg * HALO_CG_BYTES, &map_x, full_bar(stg), ctile * NB + 8 * cg,
                            tw * HALO_TILE - 1, th * HALO_TILE - 1, n_img);
        if (++stg == p.stages) {
          stg = 0;
          par ^= 1;
        }
      }
    }
  } else if (warp >= 4) {
    // ===================================================================================== MMA + epilogue
    const int wg = (warp >> 2) - 1;
    const uint32_t ring = smem_base, bars = ctrl;  // full barriers, then the empty ones at + 8 MAX_STAGES
    if (!all_taps && wg == 0)
      wgrad_halo_consume<NB, 1>(p, ring, bars, t0, t1, CENTRE_TAP, rb, ctile);
    else if (!all_taps)
      wgrad_halo_consume<NB, 0>(p, ring, bars, t0, t1, 0, rb, ctile);
    else if (wg == 0)
      wgrad_halo_consume<NB, 5>(p, ring, bars, t0, t1, 0, rb, ctile);
    else
      wgrad_halo_consume<NB, 4>(p, ring, bars, t0, t1, 5, rb, ctile);
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_tiled = nullptr;
EncodeIm2colFn g_im2col = nullptr;
int g_num_sms = 0;
long long g_launches = 0;
long long g_halo_launches = 0;
long long g_wgrad_halo_launches = 0;
bool g_force_im2col = false;
bool g_wgrad_force_im2col = false;
long long launch_count() { return g_launches; }
long long halo_launch_count() { return g_halo_launches; }
long long wgrad_halo_launch_count() { return g_wgrad_halo_launches; }
void force_im2col(bool on) { g_force_im2col = on; }
void wgrad_force_im2col(bool on) { g_wgrad_force_im2col = on; }

int init_driver() {
  if (g_tiled && g_im2col) return SGB_OK;
  cudaDriverEntryPointQueryResult qres;
  void* fn = nullptr;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) {
    sgb_set_error("cuTensorMapEncodeTiled entry point not found");
    return SGB_E_CUDA;
  }
  g_tiled = (EncodeTiledFn)fn;
  fn = nullptr;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) {
    sgb_set_error("cuTensorMapEncodeIm2col entry point not found");
    return SGB_E_CUDA;
  }
  g_im2col = (EncodeIm2colFn)fn;
  int dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
  return SGB_OK;
}

int encode_tiled(CUtensorMap* map, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* byte_strides,
                 const cuuint32_t* box, CUtensorMapSwizzle swizzle, const char* what) {
  const cuuint32_t elem_strides[5] = {1, 1, 1, 1, 1};
  const CUresult r = g_tiled(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), dims, byte_strides, box,
                             elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_SUCCESS) return SGB_OK;
  char shape[256] = "";
  for (int i = 0, n = 0; i < rank && n < (int)sizeof(shape); ++i)
    n += snprintf(shape + n, sizeof(shape) - n, "%s%llu (box %u, stride %llu)", i ? ", " : "", (unsigned long long)dims[i],
                  (unsigned)box[i], i ? (unsigned long long)byte_strides[i - 1] : 2ull);
  sgb_set_error("cuTensorMapEncodeTiled(%s) failed with %d: dims %s", what, (int)r, shape);
  return SGB_E_CUDA;
}

namespace {

// 64 / 32 / 16 bf16 channels per row -> 128B / 64B / 32B swizzle
CUtensorMapSwizzle swizzle_for(int kc) {
  return kc == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (kc == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// The im2col map of an NHWC bf16 tensor (N x H x W x C, `pitch` elements per pixel) traversed at `stride`: each box is `pixels`
// consecutive output pixels x `channels` channels of one tap; lower / upper are the corners of the filter window ({w, h}).
int encode_im2col(CUtensorMap* map, const void* ptr, int N, int H, int W, int C, int pitch, int stride, const int (&lower)[2],
                  const int (&upper)[2], int channels, int pixels, const char* what) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t strides[3] = {(cuuint64_t)pitch * 2, (cuuint64_t)W * pitch * 2, (cuuint64_t)H * W * pitch * 2};
  const cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  const CUresult r = g_im2col(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, lower, upper,
                              (cuuint32_t)channels, (cuuint32_t)pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(channels),
                              CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_SUCCESS) return SGB_OK;
  sgb_set_error("cuTensorMapEncodeIm2col(%s) failed with %d (C=%d W=%d H=%d N=%d pitch=%d lower=%d,%d upper=%d,%d stride=%d box=%d)", what,
                (int)r, C, W, H, N, pitch, lower[0], lower[1], upper[0], upper[1], stride, channels);
  return SGB_E_CUDA;
}

// The input-halo map of the halo kernels: an NHWC bf16 tensor of `pitch` elements per pixel, read as {8 channels, 10, 10, 1}
// boxes, no swizzle; boxes reaching past the image or past C are zero-filled.
int encode_halo_map(CUtensorMap* map, const void* x, int N, int H, int W, int C, int pitch) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t strides[3] = {(cuuint64_t)pitch * 2, (cuuint64_t)W * pitch * 2, (cuuint64_t)H * W * pitch * 2};
  const cuuint32_t box[4] = {8, HALO_W, HALO_H, 1};
  return encode_tiled(map, x, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE, "halo");
}

// One implicit GEMM of the im2col / halo kernels: the R x S filter b (b_rows K-major rows of b_cols columns, b_cols_per_tap per
// tap) over the NHWC slice a at (stride, pad) onto a P x Q grid, the rows written to y.
struct Problem {
  // gathered tensor (NHWC bf16, channel slice): N x H x W x C with channel pitch a_pitch (elements)
  const void* a;
  int N, H, W, C, a_pitch;
  // B matrix: b_rows = GEMM N (output channels of this GEMM), b_cols = taps * b_cols_per_tap, K-major bf16
  const void* b;
  int b_rows, b_cols, b_cols_per_tap;
  int R, S, stride, pad, P, Q, flip;
  // optional explicit tap table (ntaps > 0): im2col offsets (dh, dw) and B column block of each tap
  int ntaps;
  int tap_dh[9], tap_dw[9], tap_b[9];
  // strided output rows (Params::out_mode)
  int out_mode, o_mul, oh_add, ow_add, outH, outW;
  void* y;
  int y_pitch, y_off;
  const float* scale;
  const float* shift;
  const void* residual;
  double* stats;
  int stats_repl, act;
  // 0, or SgbConvDesc::centre_from: fprop (flip 0) -- output channels from here on have zero off-centre taps; dgrad (flip 1) --
  // gathered channels from here on meet zero off-centre taps.  Only with R = S = 3, stride 1, pad 1 and no tap table.
  int centre_from;
};

bool supported(const Problem& q) {
  if (q.C % 16 != 0 || q.b_rows % 8 != 0) return false;
  if (!((q.R == 1 && q.S == 1) || (q.R == 3 && q.S == 3))) return false;
  if (q.stride != 1 && q.stride != 2) return false;
  if (q.a_pitch % 8 != 0 || q.y_pitch % 8 != 0 || q.y_off % 8 != 0) return false;
  if (((uintptr_t)q.a & 15) || ((uintptr_t)q.b & 15) || ((uintptr_t)q.y & 15)) return false;
  if ((long long)q.N * q.P * q.Q >= (1ll << 31)) return false;
  if (q.b_rows > 4096) return false;  // shared-memory statistics buffer
  return true;
}

// kernel variant of one N tile width + its register footprint (decides how many CTAs can share an SM)
template <class Fn>
struct Variant {
  int bn;
  Fn fn;
  int regs = 0;
  bool ready = false;
};
typedef void (*ConvFn)(const CUtensorMap, const CUtensorMap, const Params);
typedef void (*WgradFn)(const CUtensorMap, const CUtensorMap, const WParams);
template <bool SKIP>
Variant<ConvFn> g_conv[6] = {{16, conv_wgmma_kernel<16, SKIP>}, {32, conv_wgmma_kernel<32, SKIP>},
                             {48, conv_wgmma_kernel<48, SKIP>}, {64, conv_wgmma_kernel<64, SKIP>},
                             {96, conv_wgmma_kernel<96, SKIP>}, {128, conv_wgmma_kernel<128, SKIP>}};
template <bool SKIP>
Variant<ConvFn> g_halo[6] = {{16, conv3x3_halo_kernel<16, SKIP>}, {32, conv3x3_halo_kernel<32, SKIP>},
                             {48, conv3x3_halo_kernel<48, SKIP>}, {64, conv3x3_halo_kernel<64, SKIP>},
                             {96, conv3x3_halo_kernel<96, SKIP>}, {128, conv3x3_halo_kernel<128, SKIP>}};
Variant<WgradFn> g_wgrad[6] = {{16, wgrad_wgmma_kernel<16>}, {32, wgrad_wgmma_kernel<32>}, {48, wgrad_wgmma_kernel<48>},
                               {64, wgrad_wgmma_kernel<64>}, {96, wgrad_wgmma_kernel<96>}, {128, wgrad_wgmma_kernel<128>}};
Variant<WgradFn> g_wgrad_halo[3] = {{16, wgrad3x3_halo_kernel<16>}, {32, wgrad3x3_halo_kernel<32>}, {48, wgrad3x3_halo_kernel<48>}};

// The variant of tile width bn in `table`; its shared-memory limit is raised and its register count read on first use.
template <class Fn, int N>
int prepare(Variant<Fn> (&table)[N], int bn, const char* what, Variant<Fn>*& var) {
  for (auto& v : table)
    if (v.bn == bn) var = &v;
  if (var->ready) return SGB_OK;
  if (int rc = sgb_cuda_check(cudaFuncSetAttribute(var->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024), what)) return rc;
  cudaFuncAttributes fa{};
  if (int rc = sgb_cuda_check(cudaFuncGetAttributes(&fa, var->fn), what)) return rc;
  var->regs = fa.numRegs;
  var->ready = true;
  return SGB_OK;
}

// CTAs of NUM_THREADS threads of `regs` registers each that one SM's 64K registers hold, at most two
int max_ctas_per_sm(int regs) {
  const int ctas = 65536 / (((regs + 7) / 8) * 8 * NUM_THREADS);
  return ctas > 2 ? 2 : (ctas < 1 ? 1 : ctas);
}

// N tile: the narrowest variant that holds N in one tile, else the widest of 128 / 96 / 64 with the least padding
int pick_bn(int n) {
  for (int bn : {16, 32, 48, 64, 96, 128})
    if (n <= bn) return bn;
  int best = 128, best_waste = (n + 127) / 128 * 128 - n;
  for (int bn : {96, 64}) {
    const int waste = (n + bn - 1) / bn * bn - n;
    if (waste < best_waste) { best_waste = waste; best = bn; }
  }
  return best;
}

// Shared memory of conv3x3_halo_kernel: the resident filter slice, `stages` halo buffers, barriers and statistics partials.
size_t halo_smem(int C, int bn, int n, bool stats, int stages) {
  const size_t b_bytes = ((size_t)9 * C * bn * 2 + 1023) & ~(size_t)1023;
  const size_t a_stage = ((size_t)(C / 8) * HALO_CG_BYTES + 1023) & ~(size_t)1023;
  return 1024 + b_bytes + (size_t)stages * a_stage + HALO_CTRL_BYTES + (stats ? (size_t)(8 * 2 * bn + 4 * n) * 4 : 0);
}

// The 8 x 8 tiles of a P x Q map put at least 85 % of the MMA rows inside the image (160², 80², 56², 40²; not 28², 20², 14², 7²).
bool halo_tiles_fit(int P, int Q) {
  const long long covered = (long long)((P + 7) / 8) * 8 * ((Q + 7) / 8) * 8;
  return 20ll * P * Q >= 17 * covered;
}

// Shape rule of the halo kernel, from the per-shape timings of tools/time_conv_halo.py: a 3x3 / stride-1 / pad-1 "same"
// convolution with plain NHWC rows whose 8 x 8 tiles put at least 85 % of the MMA rows inside the image (160², 80², 56², 40²
// maps; not 28², 20², 14², 7²), with the filter slice and two halo buffers in one CTA's shared memory.  Returns its N tile:
// pick_bn's, else -- for at most 96 gathered channels -- a narrower one of at least 64 columns that pads N no more (each N tile
// reloads the halo; narrowed tiles over 128 channels lost to conv_wgmma_kernel); 0: the shape stays on conv_wgmma_kernel.
// The N tile does not change any output: each column is its own dot product.
int halo_bn(const Problem& q) {
  if (q.R != 3 || q.S != 3 || q.stride != 1 || q.pad != 1 || q.ntaps > 0 || q.out_mode != 0) return 0;
  if (q.P != q.H || q.Q != q.W) return 0;
  if (!halo_tiles_fit(q.P, q.Q)) return 0;
  const int n = q.b_rows, full = pick_bn(n);
  auto waste = [&](int bn) { return (n + bn - 1) / bn * bn - n; };
  for (int bn : {full, 96, 64})
    if (bn <= full && (bn == full || (q.C <= 96 && bn >= 64 && waste(bn) <= waste(full))) &&
        halo_smem(q.C, bn, n, q.stats != nullptr, 2) <= 227 * 1024)
      return bn;
  return 0;
}

int launch_halo(const Problem& q, const Params& p0, int bn, cudaStream_t st) {
  Params p = p0;
  p.n_tiles = (p.N + bn - 1) / bn;
  p.halo_tw = (q.Q + HALO_TILE - 1) / HALO_TILE;
  p.halo_thw = p.halo_tw * ((q.P + HALO_TILE - 1) / HALO_TILE);
  p.M = q.N * p.halo_thw;  // tiles
  // Of a folded filter the halo kernel skips only dgrad's zero taps (centre_c).  fprop runs every tap: a straddling N tile has
  // nothing to skip, and the grid gives every N tile the same number of CTAs, so those of a centre-only tile finish early and
  // idle -- skipping measured 1-4 % slower there (tools/time_zero_taps.py).
  p.centre_n = 0;
  Variant<ConvFn>* var = nullptr;
  if (int rc = prepare(p.centre_c > 0 ? g_halo<true> : g_halo<false>, bn, "conv3x3_halo_kernel", var)) return rc;
  int ctas_per_sm = max_ctas_per_sm(var->regs);
  int stages = 0;
  for (;; --ctas_per_sm) {
    const size_t budget = (ctas_per_sm == 1 ? 227u : 227u / ctas_per_sm - 1u) * 1024u;
    for (stages = HALO_MAX_STAGES; stages >= 2 && halo_smem(q.C, bn, p.N, p.stats != nullptr, stages) > budget; --stages) {
    }
    if (stages >= 2 || ctas_per_sm == 1) break;
  }
  if (stages < 2) { sgb_set_error("conv3x3_halo: tile does not fit shared memory"); return SGB_E_UNSUPPORTED; }
  p.stages = stages;
  const size_t smem = halo_smem(q.C, bn, p.N, p.stats != nullptr, stages);

  alignas(64) CUtensorMap map_a, map_b;
  if (int rc = encode_halo_map(&map_a, q.a, q.N, q.H, q.W, q.C, q.a_pitch)) return rc;
  const cuuint64_t b_dims[2] = {(cuuint64_t)q.b_cols, (cuuint64_t)q.b_rows}, b_strides[1] = {(cuuint64_t)q.b_cols * 2};
  const cuuint32_t b_box[2] = {16, (cuuint32_t)bn};
  if (int rc = encode_tiled(&map_b, q.b, 2, b_dims, b_strides, b_box, CU_TENSOR_MAP_SWIZZLE_32B, "halo B")) return rc;
  // every CTA serves one N tile: the grid is a multiple of n_tiles
  int per_nt = g_num_sms * ctas_per_sm / p.n_tiles;
  if (per_nt > p.M) per_nt = p.M;
  if (per_nt < 1) per_nt = 1;
  var->fn<<<per_nt * p.n_tiles, NUM_THREADS, smem, st>>>(map_a, map_b, p);
  ++g_launches;
  ++g_halo_launches;
  return sgb_cuda_check(cudaGetLastError(), "conv3x3_halo_kernel");
}

int launch(const Problem& q, cudaStream_t st) {
  if (int rc = init_driver()) return rc;
  Params p{};
  p.M = q.N * q.P * q.Q;
  p.N = q.b_rows;
  p.C = q.C;
  p.KC = q.C % 64 == 0 ? 64 : (q.C % 32 == 0 ? 32 : 16);
  // Few channels per k-iteration make the pipeline latency-bound (one mbarrier round trip per 4-8 KB of A): with 48 / 96 / 288
  // channels use 64-channel boxes anyway -- the channels past C are zero-filled by TMA's bounds check (the matching B columns
  // belong to the next tap or are out of bounds: finite x 0), so C = 48 runs 1 k-iteration per tap instead of 3 and C = 96 runs 2
  // instead of 3, at the price of some zero MMA work.
  if (p.KC < 64 && q.C > 32) p.KC = 64;
  const int bn = pick_bn(p.N);
  p.n_tiles = (p.N + bn - 1) / bn;
  p.P = q.P; p.Q = q.Q; p.stride = q.stride; p.pad = q.pad;
  if (q.ntaps > 0) {
    p.ntaps = q.ntaps;
    for (int t = 0; t < q.ntaps; ++t) { p.tap_dh[t] = (signed char)q.tap_dh[t]; p.tap_dw[t] = (signed char)q.tap_dw[t]; p.tap_b[t] = (signed char)q.tap_b[t]; }
  } else {
    p.ntaps = q.R * q.S;
    for (int t = 0; t < p.ntaps; ++t) {
      p.tap_dh[t] = (signed char)(t / q.S);
      p.tap_dw[t] = (signed char)(t % q.S);
      p.tap_b[t] = (signed char)(q.flip ? (p.ntaps - 1 - t) : t);
    }
  }
  if (p.ntaps > 9) return SGB_E_UNSUPPORTED;
  p.out_mode = q.out_mode; p.o_mul = q.o_mul; p.oh_add = q.oh_add; p.ow_add = q.ow_add; p.outH = q.outH; p.outW = q.outW;
  p.b_cols_per_tap = q.b_cols_per_tap;
  p.y = (bf16*)q.y; p.y_pitch = q.y_pitch; p.y_off = q.y_off;
  p.scale = q.scale; p.shift = q.shift; p.residual = (const bf16*)q.residual;
  p.stats = q.stats; p.stats_repl = q.stats_repl > 0 ? q.stats_repl : 1; p.act = q.act;
  if (q.centre_from > 0) {
    if (q.R != 3 || q.S != 3 || q.stride != 1 || q.pad != 1 || q.ntaps > 0 || q.centre_from % 16 != 0 ||
        q.centre_from >= (q.flip ? q.C : q.b_rows))
      return SGB_E_INVALID;
    (q.flip ? p.centre_c : p.centre_n) = q.centre_from;
  }
  if (!g_force_im2col)
    if (const int hbn = halo_bn(q)) return launch_halo(q, p, hbn, st);
  Variant<ConvFn>* var = nullptr;
  if (int rc = prepare(p.centre_n > 0 || p.centre_c > 0 ? g_conv<true> : g_conv<false>, bn, "conv_wgmma_kernel", var)) return rc;
  // Small tiles leave the pipeline latency-bound: co-resident CTAs overlap each other's loads, MMAs and epilogues.
  // Limits: registers (64K per SM) and shared memory (228 KB per SM, 227 KB per CTA).
  const uint32_t a_bytes = BLOCK_M * p.KC * 2, b_bytes = ((uint32_t)(bn * p.KC * 2) + 1023u) & ~1023u;
  const uint32_t stage_bytes = a_bytes + b_bytes;
  const uint32_t ctrl_bytes = CTRL_BAR_BYTES + (p.stats ? (uint32_t)(8 * 2 * bn + 2 * p.N) * 4u : 0u);
  int ctas_per_sm = max_ctas_per_sm(var->regs);
  int stages = 0;
  for (;; --ctas_per_sm) {
    const uint32_t budget = (ctas_per_sm == 1 ? 226u : 227u / ctas_per_sm - 1u) * 1024u;
    stages = budget > ctrl_bytes + 1024 ? (int)((budget - ctrl_bytes - 1024) / stage_bytes) : 0;
    if (stages > MAX_STAGES) stages = MAX_STAGES;
    if (stages >= 4 || ctas_per_sm == 1) break;
  }
  if (stages < 2) { sgb_set_error("conv_wgmma: tile does not fit shared memory"); return SGB_E_UNSUPPORTED; }
  p.stages = stages;
  const size_t smem = 1024 + (size_t)stages * stage_bytes + ctrl_bytes;

  alignas(64) CUtensorMap map_a, map_b;
  int lower[2] = {-q.pad, -q.pad}, upper[2] = {q.pad - (q.S - 1), q.pad - (q.R - 1)};
  if (q.ntaps > 0) {  // explicit tap table: base pixel = output-class pixel, no padding
    lower[0] = lower[1] = 0;
    upper[0] = q.Q - q.W;
    upper[1] = q.P - q.H;
  }
  if (int rc = encode_im2col(&map_a, q.a, q.N, q.H, q.W, q.C, q.a_pitch, q.stride, lower, upper, p.KC, BLOCK_M, "A")) return rc;
  const cuuint64_t b_dims[2] = {(cuuint64_t)q.b_cols, (cuuint64_t)q.b_rows}, b_strides[1] = {(cuuint64_t)q.b_cols * 2};
  const cuuint32_t b_box[2] = {(cuuint32_t)p.KC, (cuuint32_t)bn};
  if (int rc = encode_tiled(&map_b, q.b, 2, b_dims, b_strides, b_box, swizzle_for(p.KC), "B")) return rc;
  const int m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  int grid = m_tiles * p.n_tiles;
  if (grid > g_num_sms * ctas_per_sm) grid = g_num_sms * ctas_per_sm;
  var->fn<<<grid, NUM_THREADS, smem, st>>>(map_a, map_b, p);
  ++g_launches;
  return sgb_cuda_check(cudaGetLastError(), "conv_wgmma_kernel");
}

// One weight gradient of the wgrad kernels: dW [K][R][S][C] (fp32, accumulated into) of the R x S filter at (stride, pad) that
// maps the NHWC slice x onto the P x Q slice dy.
struct WgradProblem {
  const void* x;   // NHWC bf16 slice, N x H x W x C
  const void* dy;  // NHWC bf16 slice, N x P x Q x K
  int N, H, W, C, x_pitch;
  int K, y_pitch;
  int R, S, stride, pad, P, Q;
  float* dw;       // fp32 [K][R][S][C], accumulated into
  int centre_from; // 0, or (3x3 only) rows from here on need only their centre tap: their off-centre dw entries are not written
};

bool wgrad_supported(const WgradProblem& q) {
  if (q.C % 16 != 0 || q.K % 8 != 0) return false;
  if (!((q.R == 1 && q.S == 1) || (q.R == 3 && q.S == 3))) return false;
  if (q.pad != q.R / 2 || (q.stride != 1 && q.stride != 2)) return false;
  if (q.x_pitch % 8 != 0 || q.y_pitch % 8 != 0) return false;
  if (((uintptr_t)q.x & 15) || ((uintptr_t)q.dy & 15)) return false;
  if ((long long)q.N * q.P * q.Q >= (1ll << 31)) return false;
  return true;
}

// Shape rule of wgrad3x3_halo_kernel, from the per-shape timings of tools/time_conv_halo.py: the 3x3 / stride-1 / pad-1 "same"
// convolutions whose 8 x 8 tiles cover the map with little waste (halo_tiles_fit), where it measured 1.13-5.5x faster than
// wgrad_wgmma_kernel on every such shape of bench configurations 2-4; the smaller maps were not timed on it.  Returns its
// in-channel tile (32 channels, else 48, else 16: each tile reads dy once more, and 5 taps x NB / 2 accumulators per thread must
// fit the registers); 0: wgrad_wgmma_kernel serves the shape.
int wgrad_halo_nb(const WgradProblem& q) {
  if (q.R != 3 || q.S != 3 || q.stride != 1 || q.pad != 1 || q.P != q.H || q.Q != q.W) return 0;
  if (!halo_tiles_fit(q.P, q.Q)) return 0;
  return q.C % 32 == 0 ? 32 : (q.C % 48 == 0 ? 48 : 16);
}

int launch_wgrad_halo(const WgradProblem& q, const WParams& p0, int nb, cudaStream_t st) {
  WParams p = p0;
  p.n_ctiles = q.C / nb;
  p.halo_tw = (q.Q + HALO_TILE - 1) / HALO_TILE;
  p.halo_thw = p.halo_tw * ((q.P + HALO_TILE - 1) / HALO_TILE);
  p.tiles = q.N * p.halo_thw;
  Variant<WgradFn>* var = nullptr;
  if (int rc = prepare(g_wgrad_halo, nb, "wgrad3x3_halo_kernel", var)) return rc;
  const int ctas_per_sm = max_ctas_per_sm(var->regs);
  const uint32_t stage_bytes = wgrad_halo_stage_bytes(nb);
  const uint32_t budget = (ctas_per_sm == 1 ? 227u : 113u) * 1024u - 1024u - CTRL_BAR_BYTES;
  p.stages = (int)(budget / stage_bytes);
  if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
  const size_t smem = 1024 + (size_t)p.stages * stage_bytes + CTRL_BAR_BYTES;
  // tile ranges: one wave of CTAs over the (row block, in-channel tile) items
  const int items = p.rb_all * p.n_ctiles;
  int splits = g_num_sms * ctas_per_sm / items;
  if (splits < 1) splits = 1;
  p.tiles_per_cta = (p.tiles + splits - 1) / splits;
  splits = (p.tiles + p.tiles_per_cta - 1) / p.tiles_per_cta;

  alignas(64) CUtensorMap map_dy, map_x;
  const cuuint64_t dy_dims[4] = {(cuuint64_t)q.K, (cuuint64_t)q.Q, (cuuint64_t)q.P, (cuuint64_t)q.N};
  const cuuint64_t dy_strides[3] = {(cuuint64_t)q.y_pitch * 2, (cuuint64_t)q.Q * q.y_pitch * 2, (cuuint64_t)q.P * q.Q * q.y_pitch * 2};
  const cuuint32_t dy_box[4] = {64, HALO_TILE, HALO_TILE, 1};
  if (int rc = encode_tiled(&map_dy, q.dy, 4, dy_dims, dy_strides, dy_box, CU_TENSOR_MAP_SWIZZLE_128B, "dy tile")) return rc;
  if (int rc = encode_halo_map(&map_x, q.x, q.N, q.H, q.W, q.C, q.x_pitch)) return rc;
  var->fn<<<splits * items, NUM_THREADS, smem, st>>>(map_dy, map_x, p);
  ++g_launches;
  ++g_wgrad_halo_launches;
  return sgb_cuda_check(cudaGetLastError(), "wgrad3x3_halo_kernel");
}

int wgrad_launch(const WgradProblem& q, cudaStream_t st) {
  if (int rc = init_driver()) return rc;
  WParams p{};
  p.K = q.K; p.C = q.C; p.R = q.R; p.S = q.S; p.stride = q.stride; p.pad = q.pad; p.P = q.P; p.Q = q.Q;
  p.npix = q.N * q.P * q.Q;
  // in-channels per CTA: the widest variant that divides C; boxes as wide as the swizzle allows
  int nb = 16;
  for (int cand : {128, 96, 64, 48, 32})
    if (q.C % cand == 0) { nb = cand; break; }
  p.CB = nb % 64 == 0 ? 64 : (nb % 32 == 0 ? 32 : 16);
  p.n_ctiles = q.C / nb;
  if (q.centre_from != 0 && (q.R != 3 || q.S != 3 || q.stride != 1 || q.pad != 1 || q.centre_from < 0 || q.centre_from >= q.K ||
                             q.centre_from % 16 != 0))
    return SGB_E_INVALID;
  // the 64-row blocks that cover K (off the centre of a folded filter: centre_from), paired, with a shared odd last one
  p.rb_all = (q.K + 63) / 64;
  p.rb_off = q.centre_from > 0 ? (q.centre_from + 63) / 64 : p.rb_all;
  p.centre_from = q.centre_from;
  p.items = 0;
  for (int t = 0; t < q.R * q.S; ++t) p.items += (wgrad_row_blocks(p, t) + 1) / 2;
  p.cpad = q.C;
  p.dw = q.dw;
  if (!g_wgrad_force_im2col)
    if (const int nb = wgrad_halo_nb(q)) return launch_wgrad_halo(q, p, nb, st);
  Variant<WgradFn>* var = nullptr;
  if (int rc = prepare(g_wgrad, nb, "wgrad_wgmma_kernel", var)) return rc;
  const uint32_t stage_bytes = 2 * WPIX * 128 + (uint32_t)(nb / p.CB) * WPIX * p.CB * 2;
  int stages = (int)((200 * 1024 - CTRL_BAR_BYTES - 1024) / stage_bytes);
  if (stages > MAX_STAGES) stages = MAX_STAGES;
  // A CTA that shares one row block gives stage s to warpgroup s % 2 only when the ring has an even length.  With an odd one a
  // warpgroup would wait for phase n of a stage whose phase n - 1 (the other warpgroup's) may not have completed, and a parity wait
  // cannot tell the two apart.
  if (p.rb_all % 2 || p.rb_off % 2) stages &= ~1;
  if (stages < 2) return SGB_E_UNSUPPORTED;
  p.stages = stages;
  const size_t smem = 1024 + (size_t)stages * stage_bytes + CTRL_BAR_BYTES;
  // pixel splits: fill ~2 waves of SMs, keep at least 8 pipeline iterations per CTA
  const int base_ctas = p.items * p.n_ctiles;
  const int total_iters = (p.npix + WPIX - 1) / WPIX;
  int splits = (2 * g_num_sms + base_ctas - 1) / base_ctas;
  if (splits > total_iters / 8) splits = total_iters / 8;
  if (splits < 1) splits = 1;
  int iters_per = (total_iters + splits - 1) / splits;
  p.pix_per_cta = iters_per * WPIX;
  splits = (p.npix + p.pix_per_cta - 1) / p.pix_per_cta;

  alignas(64) CUtensorMap map_dy, map_x;
  const cuuint64_t dy_dims[2] = {(cuuint64_t)q.K, (cuuint64_t)p.npix}, dy_strides[1] = {(cuuint64_t)q.y_pitch * 2};
  const cuuint32_t dy_box[2] = {64, (cuuint32_t)WPIX};
  if (int rc = encode_tiled(&map_dy, q.dy, 2, dy_dims, dy_strides, dy_box, CU_TENSOR_MAP_SWIZZLE_128B, "dy")) return rc;
  const int lower[2] = {-q.pad, -q.pad}, upper[2] = {q.pad - (q.S - 1), q.pad - (q.R - 1)};
  if (int rc = encode_im2col(&map_x, q.x, q.N, q.H, q.W, q.C, q.x_pitch, q.stride, lower, upper, p.CB, WPIX, "x, wgrad")) return rc;
  const int grid = base_ctas * splits;
  var->fn<<<grid, NUM_THREADS, smem, st>>>(map_dy, map_x, p);
  ++g_launches;
  return sgb_cuda_check(cudaGetLastError(), "wgrad_wgmma_kernel");
}

// ------------------------------------------------------------------------------------------------ the ABI's calls as GEMMs
Problem gemm(const sgb_bf16* a, int N, int H, int W, int C, int a_pitch, const sgb_bf16* b, int b_rows, int b_cols_per_tap, int R,
             int S, int stride, int pad, int P, int Q, void* y, int y_pitch, int y_off) {
  Problem q{};
  q.a = a; q.N = N; q.H = H; q.W = W; q.C = C; q.a_pitch = a_pitch;
  q.b = b; q.b_rows = b_rows; q.b_cols = R * S * b_cols_per_tap; q.b_cols_per_tap = b_cols_per_tap;
  q.R = R; q.S = S; q.stride = stride; q.pad = pad; q.P = P; q.Q = Q;
  q.y = y; q.y_pitch = y_pitch; q.y_off = y_off;
  q.stats_repl = 1;
  return q;
}

// The GEMM's P x Q rows are output parity class (ph, pw) of an outH x outW image: row (n, j, i) is pixel (2 j + ph, 2 i + pw).
void parity_output(Problem& q, int ph, int pw, int outH, int outW) {
  q.out_mode = 1; q.o_mul = 2; q.oh_add = ph; q.ow_add = pw; q.outH = outH; q.outW = outW;
}

// The taps of a stride-2 convolution's filter that reach input-gradient parity class (ph, pw): tap r meets row h = 2 j + ph of
// the input when h + pad - r is even, through dy row j + (ph + pad - r) / 2 (columns alike).
void stride2_taps(Problem& q, int ph, int pw, int pad) {
  q.ntaps = 0;
  for (int r = 0; r < q.R; ++r) {
    if (((ph + pad - r) & 1) != 0) continue;
    for (int s = 0; s < q.S; ++s) {
      if (((pw + pad - s) & 1) != 0) continue;
      q.tap_dh[q.ntaps] = (ph + pad - r) / 2;
      q.tap_dw[q.ntaps] = (pw + pad - s) / 2;
      q.tap_b[q.ntaps] = r * q.S + s;
      ++q.ntaps;
    }
  }
}

// 2 x 2 / stride 2 / no padding over a dense x (the backward of ConvTranspose2d(2, 2), modules/sampling.py:72-73): the patches
// do not overlap, so x viewed as the image [N * H/2][2][W/2][2C] -- row pair, row parity, column pair, (column parity, channel)
// -- turns the layer into a 2 x 1 filter at stride 1 without padding, 2C channels per tap, whose KRSC rows [K][dh][(dw, c)] are
// those of the 2 x 2 filter.  Returns false when d is not such a call.
bool row_pairs(const SgbConvDesc& d, SgbConvDesc* pairs) {
  if (!(d.R == 2 && d.S == 2 && d.stride == 2 && d.pad == 0 && d.x_pitch == d.C && d.x_off == 0 && d.H % 2 == 0 && d.W % 2 == 0 &&
        d.P == d.H / 2 && d.Q == d.W / 2 && (2 * d.C) % 16 == 0 && d.K % 8 == 0 && d.y_pitch % 8 == 0 && d.y_off % 8 == 0 &&
        (long long)d.N * (d.H / 2) < (1ll << 31)))
    return false;
  *pairs = d;
  pairs->N = d.N * (d.H / 2); pairs->H = 2; pairs->W = d.W / 2; pairs->C = 2 * d.C; pairs->x_pitch = 2 * d.C;
  pairs->S = 1; pairs->stride = 1; pairs->P = 1; pairs->Q = d.W / 2;
  return true;
}

Problem fprop_problem(const SgbConvDesc& d, const sgb_bf16* x, const sgb_bf16* w, void* y, const SgbEpilogue* ep) {
  Problem q = gemm(x + d.x_off, d.N, d.H, d.W, d.C, d.x_pitch, w, d.K, d.C, d.R, d.S, d.stride, d.pad, d.P, d.Q, y, d.y_pitch, d.y_off);
  q.centre_from = d.centre_from;
  if (ep) {
    q.scale = ep->scale; q.shift = ep->shift; q.residual = ep->residual; q.stats = ep->stats;
    q.stats_repl = ep->stats_repl > 0 ? ep->stats_repl : 1; q.act = ep->act;
  }
  return q;
}

WgradProblem wgrad_problem(const SgbConvDesc& d, const sgb_bf16* x, const sgb_bf16* dy, float* dw) {
  WgradProblem q{};
  q.x = x + d.x_off; q.dy = dy + d.y_off;
  q.N = d.N; q.H = d.H; q.W = d.W; q.C = d.C; q.x_pitch = d.x_pitch;
  q.K = d.K; q.y_pitch = d.y_pitch;
  q.R = d.R; q.S = d.S; q.stride = d.stride; q.pad = d.pad; q.P = d.P; q.Q = d.Q;
  q.dw = dw;
  q.centre_from = d.centre_from;
  return q;
}

}  // namespace

int conv_fprop(const SgbConvDesc& d, const sgb_bf16* x, const sgb_bf16* w, void* y, const SgbEpilogue* ep, cudaStream_t st) {
  if (ep && ep->out_f32) return DECLINED;
  if (d.pad == d.R / 2) {
    const Problem q = fprop_problem(d, x, w, y, ep);
    if (supported(q)) return launch(q, st);
  }
  SgbConvDesc pairs;
  if (!row_pairs(d, &pairs)) return DECLINED;
  // the 2 x 1 filter as two explicit taps of a 1 x 1 one: rows 0 and 1 of the pair, B column blocks 0 and 1
  Problem q = fprop_problem(pairs, x, w, y, ep);
  q.R = 1;
  q.ntaps = 2;
  q.tap_dh[1] = 1;
  q.tap_b[1] = 1;
  return supported(q) ? launch(q, st) : SGB_E_UNSUPPORTED;
}

// The transposed convolution as four 1 x 1 GEMMs, one per output parity (dh, dw), each writing the output pixels
// (2h + dh, 2w + dw) through the strided-row epilogue the stride-2 input gradients use.  w_up rows are ordered (dh, dw, co).
int convt2x2_fprop(const SgbConvDesc& d, const sgb_bf16* x_small, const sgb_bf16* w_up, const float* bias, sgb_bf16* y_up,
                   cudaStream_t st) {
  if (d.K % 16 != 0 || d.C % 16 != 0) return DECLINED;
  for (int cls = 0; cls < 4; ++cls) {
    Problem q = gemm(x_small + d.y_off, d.N, d.P, d.Q, d.K, d.y_pitch, w_up + (size_t)cls * d.C * d.K, d.C, d.K, 1, 1, 1, 0, d.P,
                     d.Q, y_up, d.x_pitch, d.x_off);
    q.shift = bias;
    parity_output(q, cls >> 1, cls & 1, d.H, d.W);
    if (!supported(q)) return DECLINED;  // identical for the four classes: declines before any launch
    if (int rc = launch(q, st)) return rc;
  }
  return SGB_OK;
}

int conv_dgrad(const SgbConvDesc& d, const sgb_bf16* dy, const sgb_bf16* w_crsk, sgb_bf16* dx, int accumulate, cudaStream_t st) {
  const int Kp = ((d.K + 7) / 8) * 8;  // channels gathered per tap (w_crsk rows are padded with zeros to Kp)
  // dy gathered through an R x S filter at stride 1, against the CRSK rows, accumulated into dx or not
  auto dgrad_gemm = [&](int pad, int P, int Q) {
    Problem q = gemm(dy + d.y_off, d.N, d.P, d.Q, d.K, d.y_pitch, w_crsk, d.C, Kp, d.R, d.S, 1, pad, P, Q, dx, d.x_pitch, d.x_off);
    q.residual = accumulate ? dx : nullptr;
    return q;
  };
  if (d.stride == 1 && d.pad == d.R / 2 && d.K % 16 == 0) {
    // dgrad of a stride-1 "same" convolution == convolution of dy with the spatially flipped CRSK filter
    Problem q = dgrad_gemm(d.R - 1 - d.pad, d.H, d.W);
    q.flip = 1;
    q.centre_from = d.centre_from;
    if (supported(q)) return launch(q, st);
  }
  if (d.stride == 2 && d.K % 16 == 0 && d.R == 3 && d.S == 3 && d.pad == 1 && d.H == 2 * d.P && d.W == 2 * d.Q) {
    // stride-2 dgrad = 4 output-parity classes, each an exact stride-1 gather of dy with a subset of the taps
    for (int cls = 0; cls < 4; ++cls) {
      Problem q = dgrad_gemm(0, d.P, d.Q);
      parity_output(q, cls >> 1, cls & 1, d.H, d.W);
      stride2_taps(q, cls >> 1, cls & 1, d.pad);
      if (!supported(q)) return DECLINED;  // identical for the 4 classes: declines before any launch
      if (int rc = launch(q, st)) return rc;
    }
    return SGB_OK;
  }
  if (d.stride == 2 && d.K % 16 == 0 && d.R == 1 && d.S == 1 && d.pad == 0 && d.H == 2 * d.P && d.W == 2 * d.Q) {
    // 1x1 stride-2 dgrad: only the even/even input pixels receive a gradient.  With accumulate the other three parity
    // classes are untouched; otherwise they are zero-filled first.
    Problem q = dgrad_gemm(0, d.P, d.Q);
    parity_output(q, 0, 0, d.H, d.W);
    const bool dense = d.x_pitch == d.C && d.x_off == 0;
    if (supported(q) && (accumulate || dense)) {
      if (!accumulate) cudaMemsetAsync(dx, 0, (size_t)d.N * d.H * d.W * d.C * sizeof(sgb_bf16), st);
      return launch(q, st);
    }
  }
  return DECLINED;
}

int conv_wgrad(const SgbConvDesc& d, const sgb_bf16* x, const sgb_bf16* dy, float* dw, cudaStream_t st) {
  const WgradProblem q = wgrad_problem(d, x, dy, dw);
  if (wgrad_supported(q)) return wgrad_launch(q, st);
  SgbConvDesc pairs;
  if (row_pairs(d, &pairs)) return wgrad_launch(wgrad_problem(pairs, x, dy, dw), st);
  return DECLINED;
}

}  // namespace sm100

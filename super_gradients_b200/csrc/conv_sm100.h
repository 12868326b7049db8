// Interface between the C-ABI dispatch (conv_mma.cu) and the tcgen05 / TMA implicit-GEMM kernel (conv_sm100.cu).
#pragma once
#include <cuda_runtime.h>

namespace sm100 {

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
  // strided output rows (see conv_sm100.cu: Params::out_mode)
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

struct WgradProblem {
  const void* x;   // NHWC bf16 slice, N x H x W x C
  const void* dy;  // NHWC bf16 slice, N x P x Q x K
  int N, H, W, C, x_pitch;
  int K, y_pitch;
  int R, S, stride, pad, P, Q;
  float* dw;       // fp32 [K][R][S][C], accumulated into
  int centre_from; // 0, or (3x3 only) rows from here on need only their centre tap: their off-centre dw entries are not written
};

bool wgrad_supported(const WgradProblem& q);
int wgrad_launch(const WgradProblem& q, cudaStream_t st);
bool supported(const Problem& q);
int launch(const Problem& q, cudaStream_t st);
long long launch_count();       // every launch of the kernels of conv_sm100.cu
long long halo_launch_count();  // the conv3x3_halo_kernel launches among them
void force_im2col(bool on);     // test-only: 3x3 stride-1 convolutions skip the halo kernel
long long wgrad_halo_launch_count();  // the wgrad3x3_halo_kernel launches among them
void wgrad_force_im2col(bool on);     // test-only: 3x3 stride-1 weight gradients skip the halo kernel

}  // namespace sm100

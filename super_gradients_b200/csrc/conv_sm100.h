// The wgmma / TMA convolution engine (conv_sm100.cu) as the C-ABI entry points (conv.cu) see it: one call per operation on the
// ABI's own descriptor, which re-describes the call as the engine's GEMMs and launches them, returns an SGB_E_* code, or returns
// DECLINED when the shape is not one the engine serves.
#pragma once
#include <cuda_runtime.h>

#include "sgb200.h"

namespace sm100 {

constexpr int DECLINED = 1;  // not SGB_OK and not an SGB_E_* code: the mma.sync engine serves the call

int conv_fprop(const SgbConvDesc& d, const sgb_bf16* x, const sgb_bf16* w, void* y, const SgbEpilogue* ep, cudaStream_t st);
int convt2x2_fprop(const SgbConvDesc& d, const sgb_bf16* x_small, const sgb_bf16* w_up, const float* bias, sgb_bf16* y_up,
                   cudaStream_t st);
int conv_dgrad(const SgbConvDesc& d, const sgb_bf16* dy, const sgb_bf16* w_crsk, sgb_bf16* dx, int accumulate, cudaStream_t st);
int conv_wgrad(const SgbConvDesc& d, const sgb_bf16* x, const sgb_bf16* dy, float* dw, cudaStream_t st);

long long launch_count();       // every launch of the kernels of conv_sm100.cu
long long halo_launch_count();  // the conv3x3_halo_kernel launches among them
void force_im2col(bool on);     // test-only: 3x3 stride-1 convolutions skip the halo kernel
long long wgrad_halo_launch_count();  // the wgrad3x3_halo_kernel launches among them
void wgrad_force_im2col(bool on);     // test-only: 3x3 stride-1 weight gradients skip the halo kernel

}  // namespace sm100

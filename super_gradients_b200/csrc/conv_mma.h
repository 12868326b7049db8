// The mma.sync implicit-GEMM convolution engine (conv_mma.cu): serves every call the wgmma engine declines.
#pragma once
#include <cuda_runtime.h>

#include "sgb200.h"

namespace igemm {

int conv_fprop(const SgbConvDesc& d, const sgb_bf16* x, const sgb_bf16* w, void* y, const SgbEpilogue* ep, cudaStream_t st);
int convt2x2_fprop(const SgbConvDesc& d, const sgb_bf16* x_small, const sgb_bf16* w_up, const float* bias, sgb_bf16* y_up,
                   cudaStream_t st);
int conv_dgrad(const SgbConvDesc& d, const sgb_bf16* dy, const sgb_bf16* w_crsk, sgb_bf16* dx, int accumulate, cudaStream_t st);
int conv_wgrad(const SgbConvDesc& d, const sgb_bf16* x, const sgb_bf16* dy, float* dw, cudaStream_t st);

}  // namespace igemm

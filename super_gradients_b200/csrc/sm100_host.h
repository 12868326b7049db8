// Host-side state of the wgmma / TMA convolution kernels: the driver's tensor-map encoders (resolved through
// cudaGetDriverEntryPoint, so the library has no link-time dependency on libcuda), the SM count and the launch counter.
#pragma once

#include <cuda.h>

namespace sm100 {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
extern EncodeTiledFn g_tiled;
extern EncodeIm2colFn g_im2col;
extern int g_num_sms;
extern long long g_launches;

int init_driver();                          // SGB_OK or an error code (message in sgb_last_error)
CUtensorMapSwizzle swizzle_for(int kc);     // 64 / 32 / 16 bf16 channels per row -> 128B / 64B / 32B swizzle

}  // namespace sm100

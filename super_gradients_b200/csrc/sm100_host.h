// Host-side helpers of the wgmma / TMA kernels (defined in conv_sm100.cu): the driver's tensor-map encoders, resolved through
// cudaGetDriverEntryPoint so the library has no link-time dependency on libcuda, and the one tiled-map encoder every kernel uses.
#pragma once

#include <cuda.h>

namespace sm100 {

int init_driver();  // SGB_OK or an error code (message in sgb_last_error)

// A tiled TMA map of a bf16 tensor of `rank` dimensions, innermost first, with byte_strides[i] between consecutive indices of
// dimension i + 1, read in `box` boxes; no interleave, 128-byte L2 promotion, out-of-bounds elements zero-filled.  `what` names
// the map in the error message.
int encode_tiled(CUtensorMap* map, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* byte_strides,
                 const cuuint32_t* box, CUtensorMapSwizzle swizzle, const char* what);

}  // namespace sm100

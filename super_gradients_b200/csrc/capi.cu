// Error reporting + device probe of the C ABI.
#include <cstdarg>
#include <cstdio>

#include "common.cuh"
#include "conv_sm100.h"

static thread_local char g_err[512] = "";

void sgb_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int sgb_cuda_check(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return SGB_OK;
  sgb_set_error("%s: %s", what, cudaGetErrorString(e));
  return SGB_E_CUDA;
}

extern "C" const char* sgb_last_error(void) { return g_err; }
extern "C" int sgb_version(void) { return 100; }
extern "C" int sgb_check_device(void) {
  int dev = 0;
  if (int rc = sgb_cuda_check(cudaGetDevice(&dev), "cudaGetDevice")) return rc;
  cudaDeviceProp prop;
  if (int rc = sgb_cuda_check(cudaGetDeviceProperties(&prop, dev), "cudaGetDeviceProperties")) return rc;
  if (prop.major != 9) {
    sgb_set_error("libsgb200 is built for sm_90a only; device is sm_%d%d", prop.major, prop.minor);
    return SGB_E_ARCH;
  }
  return SGB_OK;
}

extern "C" int64_t sgb_sm100_launches(void) { return (int64_t)sm100::launch_count(); }
extern "C" int64_t sgb_conv_halo_launches(void) { return (int64_t)sm100::halo_launch_count(); }
extern "C" void sgb_conv_force_im2col(int on) { sm100::force_im2col(on != 0); }
extern "C" int64_t sgb_conv_wgrad_halo_launches(void) { return (int64_t)sm100::wgrad_halo_launch_count(); }
extern "C" void sgb_conv_wgrad_force_im2col(int on) { sm100::wgrad_force_im2col(on != 0); }

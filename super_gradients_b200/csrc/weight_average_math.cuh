// Arithmetic of the best-snapshot average (training/utils/weight_averaging_utils.py:89-95), host+device: the CUDA kernel in
// weight_average.cu runs it per element, and the CPU suite compiles this header with g++ (-ffp-contract=off) behind a serial driver.
//
// The reference's running mean over the occupied slots s_0 .. s_{k-1}:
//   a <- s_0;  for n = 1 .. k-1:  a <- (a * n + s_n) / (n + 1)
// is three float32 tensor ops per step, each rounded on its own.  nvcc contracts `a * n + s` into one FMA unless told otherwise, so
// the device side spells every op with its round-to-nearest intrinsic; the host side relies on -ffp-contract=off.
#pragma once
#include <stdint.h>

#ifndef SGB_HD
#ifdef __CUDACC__
#define SGB_HD __host__ __device__ __forceinline__
#else
#define SGB_HD static inline
#endif
#endif

namespace sgb_avg {

// one step of the running mean: (a * n + s) / (n + 1), every op rounded to float32
SGB_HD float step(float a, float s, int n) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(__fadd_rn(__fmul_rn(a, (float)n), s), (float)(n + 1));
#else
  const float an = a * (float)n;
  const float sum = an + s;
  return sum / (float)(n + 1);
#endif
}

// element i of the average of slots[0 .. k-1]
SGB_HD float average(const float* const* slots, int32_t k, int64_t i) {
  float a = slots[0][i];
  for (int n = 1; n < k; ++n) a = step(a, slots[n][i], n);
  return a;
}

}  // namespace sgb_avg

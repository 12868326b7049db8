// Shared device helpers for libsgb200 (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "sgb200.h"

typedef __nv_bfloat16 bf16;

void sgb_set_error(const char* fmt, ...);
int sgb_cuda_check(cudaError_t e, const char* what);
#define SGB_LAUNCH_CHECK(what)                                  \
  do {                                                          \
    int _rc = sgb_cuda_check(cudaGetLastError(), what);         \
    if (_rc) return _rc;                                        \
  } while (0)
#define SGB_REQUIRE(cond, msg)                                  \
  do {                                                          \
    if (!(cond)) {                                              \
      sgb_set_error("%s: requirement failed: %s", __func__, msg); \
      return SGB_E_INVALID;                                     \
    }                                                           \
  } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* gmem, bool pred) {
  int sz = pred ? 16 : 0;  // src-size 0 => 16 bytes of zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_addr), "l"(gmem), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3,
                                                  uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == SGB_ACT_RELU) return v > 0.f ? v : 0.f;
  if (act == SGB_ACT_SILU) return v / (1.f + __expf(-v));
  return v;
}
// derivative of the activation expressed through pre-activation value `pre`
__device__ __forceinline__ float act_grad(float pre, int act) {
  if (act == SGB_ACT_RELU) return pre > 0.f ? 1.f : 0.f;
  if (act == SGB_ACT_SILU) {
    float s = 1.f / (1.f + __expf(-pre));
    return s * (1.f + pre * (1.f - s));
  }
  return 1.f;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

static inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// CTA cap of the streaming per-channel kernels: 132 SMs x 6 CTAs
static inline int sgb_chan_grid_cap() { return 132 * 6; }

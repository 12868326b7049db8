// Box arithmetic of torchvision's CPU NMS (csrc/ops/cpu/nms_kernel.cpp) and of batched_nms's coordinate-offset trick
// (ops/boxes.py:_batched_nms_coordinate_trick), host+device: the per-image NMS (nms.cu), the sliding-window merge
// (sliding_window.cu) and the CPU suite's host build (tests/host_kernels/merge_nms_host.cpp) all evaluate these functions.
//
// Every operation is one fp32 rounding with no contraction (device: explicitly rounded intrinsics, host: built with
// -ffp-contract=off), and `ovr > iou_threshold` is compared in double, as the CPU kernel promotes it.
#pragma once
#include <math.h>
#include <stdint.h>

#ifndef SGB_HD
#ifdef __CUDACC__
#define SGB_HD __host__ __device__ __forceinline__
#else
#define SGB_HD static inline
#endif
#endif

namespace sgb_nms {

SGB_HD float add_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
SGB_HD float sub_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
SGB_HD float mul_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
SGB_HD float div_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

// areas = (x2 - x1) * (y2 - y1)
SGB_HD float area(float x1, float y1, float x2, float y2) { return mul_rn(sub_rn(x2, x1), sub_rn(y2, y1)); }

// offsets = idxs * (max_coordinate + 1); boxes_for_nms = boxes + offsets[:, None].  `step` is max_coordinate + 1.
SGB_HD float offset_step(float max_coordinate) { return add_rn(max_coordinate, 1.0f); }
SGB_HD float label_offset(int label, float step) { return mul_rn((float)label, step); }

// Maximum that propagates NaN, as torch's boxes.max() does (fmaxf drops it): a NaN coordinate makes max_coordinate, and with it
// every offset box, NaN, so that no IoU exceeds the threshold and nothing is suppressed.
SGB_HD float max_nan(float a, float b) { return (a > b || a != a) ? a : b; }

// Box i (kept, earlier in score order) suppresses box j: inter / (areas[i] + areas[j] - inter) > iou_threshold.
SGB_HD bool suppresses(float ix1, float iy1, float ix2, float iy2, float ia, float jx1, float jy1, float jx2, float jy2, float ja, double thr) {
  const float xx1 = fmaxf(ix1, jx1), yy1 = fmaxf(iy1, jy1);
  const float xx2 = fminf(ix2, jx2), yy2 = fminf(iy2, jy2);
  const float w = fmaxf(0.f, sub_rn(xx2, xx1)), h = fmaxf(0.f, sub_rn(yy2, yy1));
  const float inter = mul_rn(w, h);
  const float ovr = div_rn(inter, sub_rn(add_rn(ia, ja), inter));
  return (double)ovr > thr;
}

// Sort key of a candidate: ascending key = score descending, then list position ascending (torchvision's stable descending sort).
// -0.0 and +0.0 compare equal in that sort, so both map to the key of +0.0 and fall back to list position.
SGB_HD uint32_t score_key(float f) {
  uint32_t b;
#ifdef __CUDA_ARCH__
  b = __float_as_uint(f);
#else
  union {
    float f;
    uint32_t u;
  } u;
  u.f = f;
  b = u.u;
#endif
  if (b == 0x80000000u) b = 0u;
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
SGB_HD uint64_t sort_key(float score, uint32_t pos) { return ((uint64_t)(~score_key(score)) << 32) | pos; }

}  // namespace sgb_nms

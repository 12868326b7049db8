// Arithmetic of the row-wise classification decode (Accuracy / Top5 and the classification predict() decode), host+device: the
// CUDA kernel in classify.cu runs one warp per row over these functions, and the CPU suite compiles this header with g++ behind a
// serial driver that replays the same 32 lane states and the same butterfly merge.
//
// Ranking: value descending, then index ascending; NaN ranks above every number (torch.sort / torch.topk, and torch.argmax returns
// the first NaN).  The top-1 index is the element ranked first; the target t is in the top k when fewer than k elements rank above
// (x_t, t).  Softmax maximum: 1 / sum_j exp(x_j - max) with an online rescaled sum (one pass).
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

namespace sgb_cls {

// (a, ia) ranks before (b, ib)
SGB_HD bool before(float a, int ia, float b, int ib) {
  const bool na = a != a, nb = b != b;
  if (na || nb) return na && (!nb || ia < ib);
  return a > b || (a == b && ia < ib);
}

struct Lane {
  float best;    // value of the best-ranked element seen
  int best_i;    // its index (-1: none yet)
  int above;     // elements ranked above the target
  float m, s;    // running maximum and sum of exp(x - m)
};

SGB_HD Lane lane_init() {
  Lane l;
  l.best = 0.f;
  l.best_i = -1;
  l.above = 0;
  l.m = -INFINITY;
  l.s = 0.f;
  return l;
}

SGB_HD float exp_f(float x) {
#ifdef __CUDA_ARCH__
  return expf(x);
#else
  return ::expf(x);
#endif
}

// a * b + c with two roundings on host and device (nvcc would contract it into an FMA)
SGB_HD float mul_add(float a, float b, float c) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(__fmul_rn(a, b), c);
#else
  return a * b + c;
#endif
}

// element j with value x; (xt, t) is the target's value and index (t < 0: no target)
SGB_HD void lane_update(Lane& l, float x, int j, float xt, int t) {
  if (l.best_i < 0 || before(x, j, l.best, l.best_i)) {
    l.best = x;
    l.best_i = j;
  }
  if (t >= 0 && before(x, j, xt, t)) ++l.above;
  if (x > l.m) {
    l.s = mul_add(l.s, exp_f(l.m - x), 1.f);
    l.m = x;
  } else {
    l.s += exp_f(x - l.m);
  }
}

// commutative: the butterfly's two partners compute the same state
SGB_HD Lane lane_merge(const Lane& a, const Lane& b) {
  Lane r = a;
  if (b.best_i >= 0 && (a.best_i < 0 || before(b.best, b.best_i, a.best, a.best_i))) {
    r.best = b.best;
    r.best_i = b.best_i;
  }
  r.above = a.above + b.above;
  if (a.s == 0.f) {
    r.m = b.m;
    r.s = b.s;
  } else if (b.s != 0.f) {
    const float m = a.m > b.m ? a.m : b.m;
    r.m = m;
    r.s = mul_add(a.s, exp_f(a.m - m), mul_add(b.s, exp_f(b.m - m), 0.f));
  }
  return r;
}

}  // namespace sgb_cls

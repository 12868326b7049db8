// Arithmetic of the DetectionMetrics prediction / target matching (row (f)-N4), host+device like pose_loss_math.cuh: the CUDA
// kernel in detection_match.cu calls these per (prediction, threshold) and the CPU suite compiles this header with g++ behind a
// serial driver (tests/host_kernels/detection_match_host.cpp) to check it, bit for bit, against the reference's outputs.
//
// Reference (src/super_gradients/training/utils/detection_utils.py):
//   change_bbox_bounds_for_image_size_inplace :174-185   predictions clipped to the image
//   cxcywh2xyxy :725-735 (+ denormalisation :1269-1273)   targets -> pixel XYXY, in exactly this operation order
//   box_iou :257-276, crowd_ioa :797-812                  float32, (area1 + area2) - inter
//   get_top_k_idx_per_cls :1342-1359                      predictions used: non-zero score, rank < top_k inside their class
//   IoUMatching.compute_targets :902-960                  greedy loop over predictions (confidence order) x targets (IoU order)
//   IoUMatching.compute_crowd_targets :962-1005           crowd targets only switch predictions to "ignore"
//
// The greedy loop is restated per threshold j: a prediction takes the still-free same-class target of highest IoU (first one on
// ties, the order of the reference's stable descending sort) if that IoU is > thr[j]; thresholds never interact, so each one can
// run on its own warp.  Every float operation is a single IEEE round-to-nearest step (no FMA contraction on the device).
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

namespace sgb_match {

#ifdef __CUDA_ARCH__
SGB_HD float fadd(float a, float b) { return __fadd_rn(a, b); }
SGB_HD float fsub(float a, float b) { return __fsub_rn(a, b); }
SGB_HD float fmul(float a, float b) { return __fmul_rn(a, b); }
SGB_HD float fdiv(float a, float b) { return __fdiv_rn(a, b); }
#else
SGB_HD float fadd(float a, float b) { return a + b; }
SGB_HD float fsub(float a, float b) { return a - b; }
SGB_HD float fmul(float a, float b) { return a * b; }
SGB_HD float fdiv(float a, float b) { return a / b; }
#endif

struct Box {
  float x1, y1, x2, y2;
};

SGB_HD float clampf(float v, float lo, float hi) { return fminf(fmaxf(v, lo), hi); }

SGB_HD Box clip_box(Box b, float height, float width) {
  return Box{clampf(b.x1, 0.f, width), clampf(b.y1, 0.f, height), clampf(b.x2, 0.f, width), clampf(b.y2, 0.f, height)};
}

// (cx, cy, w, h) -> XYXY: y1 = cy - h * 0.5; x1 = cx - w * 0.5; y2 = h + y1; x2 = w + x1; then the optional scale to pixels
SGB_HD Box target_xyxy(float cx, float cy, float w, float h, bool denormalize, float height, float width) {
  Box b;
  b.y1 = fsub(cy, fmul(h, 0.5f));
  b.x1 = fsub(cx, fmul(w, 0.5f));
  b.y2 = fadd(h, b.y1);
  b.x2 = fadd(w, b.x1);
  if (denormalize) {
    b.x1 = fmul(b.x1, width);
    b.x2 = fmul(b.x2, width);
    b.y1 = fmul(b.y1, height);
    b.y2 = fmul(b.y2, height);
  }
  return b;
}

SGB_HD float area(Box b) { return fmul(fsub(b.x2, b.x1), fsub(b.y2, b.y1)); }

SGB_HD float intersection(Box a, Box b) {
  const float w = fmaxf(fsub(fminf(a.x2, b.x2), fmaxf(a.x1, b.x1)), 0.f);
  const float h = fmaxf(fsub(fminf(a.y2, b.y2), fmaxf(a.y1, b.y1)), 0.f);
  return fmul(w, h);
}

SGB_HD float iou(Box a, float area_a, Box b, float area_b) {
  const float inter = intersection(a, b);
  return fdiv(inter, fsub(fadd(area_a, area_b), inter));
}

SGB_HD float ioa(Box det, float det_area, Box crowd) { return fdiv(intersection(det, crowd), det_area); }

// confidence order inside a class and across the image: higher score first, equal scores by prediction index
SGB_HD bool before(float score_a, int a, float score_b, int b) { return score_a > score_b || (score_a == score_b && a < b); }

struct Best {
  float v;
  int t;
};

// The free same-class target of highest IoU > thr among targets first, first + step, ... (the kernel strides a warp's lanes
// over the targets and merges the lanes' results with better(); the host driver calls it with first = 0, step = 1).
SGB_HD Best best_free_target(Box p, float area_p, float cls_p, float thr, const Box* tbox, const float* tarea, const float* tcls,
                             const uint8_t* taken, int n_targets, int first, int step) {
  Best b{thr, -1};
  for (int t = first; t < n_targets; t += step) {
    if (tcls[t] != cls_p || taken[t]) continue;
    const float v = iou(p, area_p, tbox[t], tarea[t]);
    if (v > b.v) b = Best{v, t};  // NaN (two empty boxes) never matches; ascending t keeps the first of equal IoUs
  }
  return b;
}

SGB_HD Best better(Best a, Best b) {
  if (b.t < 0) return a;
  if (a.t < 0) return b;
  return (b.v > a.v || (b.v == a.v && b.t < a.t)) ? b : a;
}

// max over the same-class crowd targets of the intersection-over-detection-area, with torch.max's NaN propagation
SGB_HD float best_crowd_ioa(Box p, float area_p, float cls_p, const Box* cbox, const float* ccls, int n_crowd) {
  float best = 0.f;
  bool nan = false;
  for (int c = 0; c < n_crowd; ++c) {
    if (ccls[c] != cls_p) continue;
    const float v = ioa(p, area_p, cbox[c]);
    if (v != v) nan = true;
    else if (v > best) best = v;
  }
  return nan ? NAN : best;
}

// ---- DistanceMatching (detection_utils.py:1008-1118) with EuclideanDistance / ManhattanDistance (:1293-1340) ----
// The pair score is the distance between box centres, (x1 + x2) / 2 and (y1 + y2) / 2 of the clipped prediction and of the
// (denormalised) target; a different class is +inf.  Per prediction the reference visits the targets by stable ascending
// distance and takes, for threshold j, the first one still free at j with distance < thr[j] (strict) -- i.e. the nearest free
// target, lowest index on ties, if it is nearer than thr[j].  Crowd targets: min distance < thr[j] switches "ignore" on.
enum DistanceMetric { kEuclidean = 0, kManhattan = 1 };

struct Point {
  float x, y;
};

SGB_HD Point centre(Box b) { return Point{fdiv(fadd(b.x1, b.x2), 2.f), fdiv(fadd(b.y1, b.y2), 2.f)}; }

// sqrt(dx * dx + dy * dy): two rounded products, one rounded add, a correctly rounded sqrt (== torch's (diff**2).sum(2).sqrt());
// |dx| + |dy| for Manhattan
SGB_HD float centre_distance(int metric, Point a, Point b) {
  const float dx = fsub(a.x, b.x), dy = fsub(a.y, b.y);
  if (metric == kManhattan) return fadd(fabsf(dx), fabsf(dy));
#ifdef __CUDA_ARCH__
  return __fsqrt_rn(fadd(fmul(dx, dx), fmul(dy, dy)));
#else
  return sqrtf(fadd(fmul(dx, dx), fmul(dy, dy)));
#endif
}

// The free same-class target of smallest distance < thr among targets first, first + step, ... (lanes as best_free_target;
// merge with nearer()).  NaN distances never match, as NaN sorts last and fails `< thr` in the reference.
SGB_HD Best nearest_free_target(int metric, Point p, float cls_p, float thr, const Box* tbox, const float* tcls, const uint8_t* taken,
                                int n_targets, int first, int step) {
  Best b{thr, -1};
  for (int t = first; t < n_targets; t += step) {
    if (tcls[t] != cls_p || taken[t]) continue;
    const float v = centre_distance(metric, p, centre(tbox[t]));
    if (v < b.v) b = Best{v, t};  // ascending t keeps the first of equal distances (the stable sort's order)
  }
  return b;
}

SGB_HD Best nearer(Best a, Best b) {
  if (b.t < 0) return a;
  if (a.t < 0) return b;
  return (b.v < a.v || (b.v == a.v && b.t < a.t)) ? b : a;
}

// min over the same-class crowd targets of the centre distance (+inf when there is none), with torch.min's NaN propagation
SGB_HD float nearest_crowd_distance(int metric, Point p, float cls_p, const Box* cbox, const float* ccls, int n_crowd) {
  float best = INFINITY;
  bool nan = false;
  for (int c = 0; c < n_crowd; ++c) {
    if (ccls[c] != cls_p) continue;
    const float v = centre_distance(metric, p, centre(cbox[c]));
    if (v != v) nan = true;
    else if (v < best) best = v;
  }
  return nan ? NAN : best;
}

}  // namespace sgb_match

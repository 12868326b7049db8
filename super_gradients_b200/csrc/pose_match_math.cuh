// Arithmetic of the PoseEstimationMetrics prediction / target matching, host+device like detection_match_math.cuh: the CUDA kernel
// in pose_match.cu calls these per (prediction, target) pair and per threshold, and the CPU suite compiles this header with g++
// behind a serial driver (tests/host_kernels/pose_match_host.cpp) to check it against the reference's outputs.
//
// Reference (src/super_gradients/training/metrics/):
//   pose_estimation_metrics.py:264-292   ground truth: ignored = crowd or every joint at visibility 0; derived boxes and areas
//   pose_estimation_utils.py:8-32        compute_visible_bbox_xywh (restated with the numpy min / max semantics it was written for)
//   pose_estimation_utils.py:57-94       compute_oks: the float32 operation order of one (prediction, target) pair
//   pose_estimation_utils.py:190-194     top-k predictions by score
//   pose_estimation_utils.py:196-233     greedy loop over predictions (confidence order) x targets (OKS order)
//   pose_estimation_utils.py:237-256     ignored ("crowd") targets only switch predictions to "ignore"
//
// The greedy loop is restated per threshold j: a prediction takes the still-free regular target of highest OKS (lowest index on
// ties, the order of the reference's stable descending sort) if that OKS is > thr[0] and > thr[j] (the loop only visits pairs above
// thr[0]); thresholds never interact, so each one can run on its own warp.  Every float operation other than the exp / sum of the
// OKS is a single IEEE round-to-nearest step (no FMA contraction on the device).
#pragma once
#include <math.h>
#include <stdint.h>

#include "detection_match_math.cuh"

namespace sgb_pose_match {

using sgb_match::Best;
using sgb_match::fadd;
using sgb_match::fdiv;
using sgb_match::fmul;
using sgb_match::fsub;

// bits of the per-target flag byte
constexpr uint8_t FLAG_CROWD = 1;     // is_crowd
constexpr uint8_t FLAG_HAS_BOX = 2;   // the XYWH box is given (else derived from the visible joints)
constexpr uint8_t FLAG_HAS_AREA = 4;  // the area is given (else w * h of the box)

// torch.finfo(torch.float64).eps added to a float32 tensor: the sum is float32
constexpr float kAreaEps = 2.220446049250313e-16f;

SGB_HD bool isnan_(float v) { return v != v; }

// numpy's np.min / np.max propagate NaN
SGB_HD float np_min(float a, float b) { return (isnan_(a) || isnan_(b)) ? NAN : (b < a ? b : a); }
SGB_HD float np_max(float a, float b) { return (isnan_(a) || isnan_(b)) ? NAN : (b > a ? b : a); }

// torch.clamp_min(v, 0) keeps NaN
SGB_HD float clamp0(float v) { return v < 0.f ? 0.f : v; }

// vars = (sigmas * 2) ** 2 (pose_estimation_utils.py:58)
SGB_HD float oks_var(float sigma) {
  const float s2 = fmul(sigma, 2.f);
  return fmul(s2, s2);
}

// joints [J, 3] = (x, y, visibility): count of visibility > 0 (k1 of compute_oks, pose_estimation_utils.py:71)
SGB_HD int n_visible(const float* joints, int J) {
  int k = 0;
  for (int j = 0; j < J; ++j) k += joints[3 * j + 2] > 0.f ? 1 : 0;
  return k;
}

// gt_is_ignore = visibility.eq(0).all(1) | is_crowd (pose_estimation_metrics.py:280-281)
SGB_HD bool is_ignored(const float* joints, int J, uint8_t flags) {
  if (flags & FLAG_CROWD) return true;
  for (int j = 0; j < J; ++j)
    if (!(joints[3 * j + 2] == 0.f)) return false;
  return true;
}

// compute_visible_bbox_xywh (pose_estimation_utils.py:8-32) with numpy's where= / initial= semantics: minimum over the visible joints
// starting from 1e6 (a result of exactly 1e6 becomes 0), maximum starting from 0, w = x2 - x1, h = y2 - y1
SGB_HD void visible_box_xywh(const float* joints, int J, float* xywh) {
  const float init = 1000000.f;
  float x1 = init, y1 = init, x2 = 0.f, y2 = 0.f;
  for (int j = 0; j < J; ++j) {
    if (!(joints[3 * j + 2] > 0.f)) continue;
    x1 = np_min(x1, joints[3 * j]);
    y1 = np_min(y1, joints[3 * j + 1]);
    x2 = np_max(x2, joints[3 * j]);
    y2 = np_max(y2, joints[3 * j + 1]);
  }
  if (x1 == init) x1 = 0.f;
  if (y1 == init) y1 = 0.f;
  xywh[0] = x1;
  xywh[1] = y1;
  xywh[2] = fsub(x2, x1);
  xywh[3] = fsub(y2, y1);
}

// gt_areas = gt_bboxes[:, 2] * gt_bboxes[:, 3] when no area is given (pose_estimation_metrics.py:267-268)
SGB_HD float box_area(const float* xywh) { return fmul(xywh[2], xywh[3]); }

// OKS of one predicted pose (xy with stride `pstride` floats per joint) against one target (compute_oks,
// pose_estimation_utils.py:67-94): e = (dx^2 + dy^2) / vars / (area + eps) / 2 in float32, then the mean of exp(-e) over the visible
// joints (all J when none is visible, with dx / dy the distance to the doubled box).  exp and the sum run in double and are rounded
// to float once: torch's float32 exp and summation order are not reproducible bit for bit anyway.
SGB_HD float oks(const float* pxy, int pstride, const float* tj, const float* xywh, float area, int k1, const float* vars, int J) {
  const float a = fadd(area, kAreaEps);
  const float x0 = fsub(xywh[0], xywh[2]), x1 = fadd(xywh[0], fmul(xywh[2], 2.f));
  const float y0 = fsub(xywh[1], xywh[3]), y1 = fadd(xywh[1], fmul(xywh[3], 2.f));
  double sum = 0.0;
  for (int j = 0; j < J; ++j) {
    const float xd = pxy[j * pstride], yd = pxy[j * pstride + 1];
    float dx, dy;
    if (k1 > 0) {
      if (!(tj[3 * j + 2] > 0.f)) continue;
      dx = fsub(xd, tj[3 * j]);
      dy = fsub(yd, tj[3 * j + 1]);
    } else {
      dx = fadd(clamp0(fsub(x0, xd)), clamp0(fsub(xd, x1)));
      dy = fadd(clamp0(fsub(y0, yd)), clamp0(fsub(yd, y1)));
    }
    const float e = fdiv(fdiv(fdiv(fadd(fmul(dx, dx), fmul(dy, dy)), vars[j]), a), 2.f);
    sum += exp(-(double)e);
  }
  return (float)(sum / (double)(k1 > 0 ? k1 : J));
}

// torch.topk order: higher score first, NaN above everything, equal scores by prediction index (torch leaves that order unspecified)
SGB_HD bool before(float score_a, int a, float score_b, int b) {
  const bool na = isnan_(score_a), nb = isnan_(score_b);
  if (na || nb) return (na && nb) ? a < b : na;
  return score_a > score_b || (score_a == score_b && a < b);
}

// a pair qualifies when OKS > thr[0] and OKS > thr[j] (pose_estimation_utils.py:204, :211); NaN in either never qualifies
SGB_HD float qualify_floor(float thr0, float thrj) { return (isnan_(thr0) || isnan_(thrj)) ? NAN : (thrj > thr0 ? thrj : thr0); }

// The free regular target of highest OKS above `floor` among targets first, first + step, ... of one prediction's OKS row (the kernel
// strides a warp's lanes over the targets and merges the lanes' results with sgb_match::better(); the host driver calls it with
// first = 0, step = 1).  The reference's `is_matching_with_ignore` (pose_estimation_utils.py:219-222) is never true: it reads
// targets_ignored, which the metric builds as gt_is_ignore[~gt_is_ignore] (pose_estimation_metrics.py:287), i.e. all False -- ignored
// targets only enter through the crowd rule below.
SGB_HD Best best_free_target(const float* oks_row, float floor, const uint8_t* taken, int n_targets, int first, int step) {
  Best b{floor, -1};
  for (int t = first; t < n_targets; t += step) {
    if (taken[t]) continue;
    const float v = oks_row[t];
    if (v > b.v) b = Best{v, t};  // NaN never matches; ascending t keeps the first of equal OKS
  }
  return b;
}

// max over the ignored targets' OKS with torch.max's NaN propagation (pose_estimation_utils.py:250)
SGB_HD float best_crowd_oks(const float* oks_row, int n_crowd) {
  float best = -INFINITY;
  for (int c = 0; c < n_crowd; ++c) {
    const float v = oks_row[c];
    if (isnan_(v)) return NAN;
    if (v > best) best = v;
  }
  return best;
}

}  // namespace sgb_pose_match

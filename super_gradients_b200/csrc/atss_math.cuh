// Arithmetic of the ATSS assigner (row L2, the static assigner of PP-YOLOE recipes) on top of the box arithmetic it shares with
// the task-aligned assigners (tal_math.cuh), host+device like pose_loss_math.cuh: the kernels in atss.cu call these and the CPU
// suite compiles this header with g++ behind a serial driver (tests/host_kernels/atss_host.cpp) to check the assignment against
// the reference's recorded outputs.
//
// Reference: ATSSAssigner.forward, src/super_gradients/training/losses/ppyolo_loss.py:301-434, called by PPYoloELoss with
// topk = 9, force_gt_matching = False and pred_bboxes given (:810-820); helpers iou_similarity :38-60 (eps 1e-10),
// batch_iou_similarity :17-35 (eps 1e-9), bbox_center :233-240, check_points_inside_bboxes :178-211, compute_max_iou_anchor
// :165-175; PPYoloELoss._bbox_decode :1054-1061.
#pragma once
#include <math.h>
#include <stdint.h>

#include "tal_math.cuh"

namespace sgb_atss {

constexpr int kMaxLevels = 8;
constexpr int kMaxTopk = 16;

struct Levels {
  int n;
  int start[kMaxLevels + 1];  // start[n] = L
};

using sgb_tal::Box;
using sgb_tal::decode_box;
using sgb_tal::iou;
using sgb_tal::load_box;

SGB_HD float center_x(const Box& b) { return (b.x1 + b.x2) / 2.f; }
SGB_HD float center_y(const Box& b) { return (b.y1 + b.y2) / 2.f; }

// torch.norm(gt_center - anchor_center, p = 2)
SGB_HD float center_distance(const Box& g, const Box& a) {
  const float dx = center_x(g) - center_x(a), dy = center_y(g) - center_y(a);
  return sqrtf(dx * dx + dy * dy);
}

SGB_HD bool center_inside(const Box& a, const Box& g) { return sgb_tal::inside_gt(center_x(a), center_y(a), g); }

// mean + unbiased standard deviation of the candidates' IoUs (torch accumulates the variance in double)
SGB_HD float iou_threshold(const float* v, int n) {
  double s = 0.0;
  for (int i = 0; i < n; ++i) s += (double)v[i];
  const double mean = s / n;
  double q = 0.0;
  for (int i = 0; i < n; ++i) q += ((double)v[i] - mean) * ((double)v[i] - mean);
  const float sd = n > 1 ? (float)sqrt(q / (n - 1)) : NAN;  // torch.std of one element is NaN: nothing is selected
  return (float)mean + sd;
}

// an anchor claimed by several GTs goes to the GT (padded rows included: they are zero boxes) of highest IoU with the anchor
// box, first one on ties (compute_max_iou_anchor: argmax over the GT axis)
SGB_HD int argmax_iou_gt(const Box& a, const float* gt_boxes, int n_max) {
  float best = -1.f;
  int bg = 0;
  for (int g = 0; g < n_max; ++g) {
    const float v = iou(load_box(gt_boxes + g * 4), a, 1e-10f);
    if (v > best) {
      best = v;
      bg = g;
    }
  }
  return bg;
}

}  // namespace sgb_atss

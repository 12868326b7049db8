// Pose-specific arithmetic of YoloNASPoseLoss (row L7): OKS, the assigner's pair IoU, the keypoint terms of one anchor and the
// finalisation, written once as host+device inline functions on top of the task-aligned assigner and box-loss arithmetic shared
// with the detection losses (tal_math.cuh).  The CUDA kernels in pose_loss.cu call them per thread, and the CPU test-suite
// compiles this very header with g++ (tests/host_kernels/pose_loss_host.cpp) to check the arithmetic against the oracle without
// a GPU.
//
// Reference: src/super_gradients/training/losses/yolo_nas_pose_loss.py
//   batch_pose_oks :45-74, YoloNASPoseTaskAlignedAssigner.forward :77-244, YoloNASPoseLoss.forward :404-494,
//   _keypoint_loss :514-564, _bbox_loss :574-639, _df_loss :496-512, _focal_loss :663-682.
#pragma once
#include <math.h>
#include <stdint.h>

#include "sgb200.h"
#include "tal_math.cuh"

namespace sgb_pose {

using sgb_tal::Box;
using PBox = sgb_tal::Box;
using sgb_tal::cls_term;
using sgb_tal::inside_gt;
using sgb_tal::sigmoid_f;

// unnormalised partial sums of one anchor: cls, iou, dfl, pose_cls, pose_reg
struct AnchorSums {
  float cls, iou, dfl, pcls, preg;
};

// batch_pose_oks (:45-74): mean over the VISIBLE joints of exp(-d^2 / (2 sigma)^2 / (0.53 * box area + eps) / 2).
// gpose [J][3] = (x, y, visibility), ppose [J][2] in pixels.
SGB_HD float oks(const float* gpose, const float* ppose, const float* sigmas, int J, const Box& g) {
  const float area = (g.x2 - g.x1) * (g.y2 - g.y1) * 0.53f;
  float num = 0.f, nvis = 0.f;
  for (int j = 0; j < J; ++j) {
    if (!(gpose[3 * j + 2] > 0.f)) continue;
    float dx = gpose[3 * j] - ppose[2 * j], dy = gpose[3 * j + 1] - ppose[2 * j + 1];
    float s2 = 2.f * sigmas[j];
    float e = (dx * dx + dy * dy) / (s2 * s2) / (area + 1e-9f) / 2.f;
    num += expf(-e);
    nvis += 1.f;
  }
  return num / (nvis + 1e-9f);
}

// the "iou" of the assigner: box IoU, times the pose OKS when assigner_multiply_by_pose_oks (:140-147)
SGB_HD float pair_iou(const SgbPoseLossDesc& d, const Box& g, const float* gpose, const Box& p, const float* ppose,
                      const float* sigmas) {
  float iou = sgb_tal::iou(g, p, 1e-9f);
  if (d.multiply_by_oks) iou *= oks(gpose, ppose, sigmas, d.J, g);
  return iou;
}

SGB_HD float tal_metric(const SgbPoseLossDesc& d, float score, float iou) { return sgb_tal::tal_metric(d.alpha, d.beta, score, iou); }

// softmax-expectation decode of one anchor's 4 x nb DFL logits -> xyxy in pixels at out
SGB_HD void decode_box(const float* z, int nb, float apx, float apy, float s, float* out) {
  sgb_tal::store_box(out, sgb_tal::decode_box(z, nb, apx, apy, s));
}

// One anchor of the assigner after the per-gt top-k selection (:166-206): the shared multi-assignment rule with the pose pair
// IoU (box IoU, times OKS when multiply_by_oks) and the person score.  topk [B][n_max][topk] holds the selected anchor indices
// per gt (-1 = none).
SGB_HD void resolve_anchor(const SgbPoseLossDesc& d, int b, int l, const float* pbox, const float* cls, const float* pose,
                           const float* ap, const float* gtb, const float* gtp, const uint8_t* gtv, const float* sigmas,
                           const int* topk, int* ag_out, float* met_out, float* iou_out) {
  const int64_t i = (int64_t)b * d.L + l;
  const int g0 = b * d.n_max;
  const Box p = sgb_tal::load_box(pbox + i * 4);
  const float* pp = pose + i * d.J * 2;
  *ag_out = sgb_tal::resolve_anchor(
      l, ap[l * 2], ap[l * 2 + 1], d.n_max, d.topk, gtb + (int64_t)g0 * 4, gtv + g0, topk + (int64_t)g0 * d.topk, d.alpha, d.beta,
      [&](int g, const Box& gb) { return pair_iou(d, gb, gtp + (int64_t)(g0 + g) * d.J * 3, p, pp, sigmas); },
      [&](int) { return sigmoid_f(cls[i]); }, met_out, iou_out);
}

// assigned score of one anchor (:208-222) and whether it is a positive for the box / keypoint terms (crowd targets keep
// their assignment but contribute neither a classification target nor regression terms, :224-231 and _bbox_loss :597)
SGB_HD void finish_anchor(int ag, float met, float gt_max_metric, float gt_max_iou, bool crowd, int* pos_gt, float* score) {
  *pos_gt = -1;
  *score = 0.f;
  if (ag >= 0 && !crowd) {
    *pos_gt = ag;
    *score = sgb_tal::assigned_score(met, gt_max_metric, gt_max_iou);
  }
}

// All loss terms of one anchor and the FINAL gradients of
//   grad_scale * [w_cls*cls/norm + w_iou*iou/norm + w_dfl*dfl/norm + w_pose_cls*pose_cls + w_pose_reg*pose_reg]
// w.r.t. its person logit (always written) and, for a positive anchor (pos_gt >= 0), its DFL logits, keypoint coordinates
// and joint logits (callers pre-zero those buffers; non-positive anchors write nothing there).
//   inv_norm = grad_scale / max(sum assigned scores, 1);  inv_pos = grad_scale / max(number of positives, 1).
SGB_HD void anchor_loss(const SgbPoseLossDesc& d, int b, int l, const float* cls, const float* reg, const float* pose,
                        const float* plog, const float* ap, const float* st, const float* gtb, const float* gtp,
                        const float* sigmas, int pos_gt, float q, float inv_norm, float inv_pos, float* gcls, float* greg,
                        float* gpose, float* gplog, AnchorSums* acc) {
  const int64_t i = (int64_t)b * d.L + l;
  const int nb = d.reg_max + 1, J = d.J;
  {
    float lc, gc;
    cls_term(d.cls_type == 0, -1.f, cls[i], q, &lc, &gc);
    acc->cls += lc;
    if (gcls) gcls[i] = gc * d.w_cls * inv_norm;
  }
  if (pos_gt < 0) return;
  const int64_t bg = (int64_t)b * d.n_max + pos_gt;
  const float s = st[l];
  const float ax = ap[l * 2] / s, ay = ap[l * 2 + 1] / s;
  const float gx1 = gtb[bg * 4 + 0] / s, gy1 = gtb[bg * 4 + 1] / s, gx2 = gtb[bg * 4 + 2] / s, gy2 = gtb[bg * 4 + 3] / s;
  // ---- box: DFL expectation, IoU loss, DFL cross-entropy
  const float* z = reg + i * 4 * nb;
  float mx[4], se[4], dist[4];
  for (int sd = 0; sd < 4; ++sd) {
    float m = -INFINITY;
    for (int k = 0; k < nb; ++k) m = fmaxf(m, z[sd * nb + k]);
    float e_sum = 0.f, e_w = 0.f;
    for (int k = 0; k < nb; ++k) {
      float e = expf(z[sd * nb + k] - m);
      e_sum += e;
      e_w += e * (float)k;
    }
    mx[sd] = m;
    se[sd] = e_sum;
    dist[sd] = e_w / e_sum;
  }
  float liou, gb[4];
  sgb_tal::iou_loss_grad(d.iou_type, ax - dist[0], ay - dist[1], ax + dist[2], ay + dist[3], gx1, gy1, gx2, gy2, &liou, gb);
  const float tgt[4] = {ax - gx1, ay - gy1, gx2 - ax, gy2 - ay};
  const float sgn[4] = {-1.f, -1.f, 1.f, 1.f};  // x1 = ax - d0, y1 = ay - d1, x2 = ax + d2, y2 = ay + d3
  float ldfl = 0.f;
  for (int sd = 0; sd < 4; ++sd) {
    const auto [tl, wl, wr] = sgb_tal::dfl_target(tgt[sd], d.reg_max);
    for (int k = 0; k < nb; ++k) {
      const float p = expf(z[sd * nb + k] - mx[sd]) / se[sd];
      if (k == tl) ldfl -= logf(fmaxf(p, 1e-38f)) * wl;
      if (k == tl + 1) ldfl -= logf(fmaxf(p, 1e-38f)) * wr;
      if (greg) {
        const float gd = 0.25f * (p - (k == tl ? wl : 0.f) - (k == tl + 1 ? wr : 0.f));
        const float gi = gb[sd] * sgn[sd] * p * ((float)k - dist[sd]);
        greg[i * 4 * nb + sd * nb + k] = q * (d.w_dfl * gd + d.w_iou * gi) * inv_norm;
      }
    }
  }
  acc->iou += liou * q;
  acc->dfl += ldfl * 0.25f * q;
  // ---- keypoints: OKS-style regression on the visible joints + visibility classification on all joints
  const float* gp = gtp + bg * J * 3;
  const float area = (gtb[bg * 4 + 2] - gtb[bg * 4 + 0]) * (gtb[bg * 4 + 3] - gtb[bg * 4 + 1]) * 0.53f;  // pixels
  float nvis = 0.f;
  for (int j = 0; j < J; ++j) nvis += gp[3 * j + 2] > 0.f ? 1.f : 0.f;
  const float inv_vis = 1.f / (nvis + 1e-9f);
  const float kf = d.rescale_with_score ? q * inv_norm : inv_pos;  // factor of this anchor's keypoint terms in the total
  float reg_sum = 0.f, vis_sum = 0.f;
  for (int j = 0; j < J; ++j) {
    const float v = gp[3 * j + 2] > 0.f ? 1.f : 0.f;
    const float dx = pose[(i * J + j) * 2] - gp[3 * j], dy = pose[(i * J + j) * 2 + 1] - gp[3 * j + 1];
    const float s2 = 2.f * sigmas[j];
    const float c = 1.f / (s2 * s2) / (area + 1e-9f) / 2.f;
    const float ex = expf(-(dx * dx + dy * dy) * c);
    reg_sum += (1.f - ex) * v;
    if (gpose) {
      const float g = d.w_pose_reg * kf * ex * c * 2.f * v * inv_vis;
      gpose[(i * J + j) * 2] = g * dx;
      gpose[(i * J + j) * 2 + 1] = g * dy;
    }
    float lj, gj;
    cls_term(d.pose_cls_type == 1, 0.25f, plog[i * J + j], v, &lj, &gj);
    vis_sum += lj;
    if (gplog) gplog[i * J + j] = d.w_pose_cls * kf * gj / (float)J;
  }
  const float wgt = d.rescale_with_score ? q : 1.f;
  acc->preg += reg_sum * inv_vis * wgt;
  acc->pcls += vis_sum / (float)J * wgt;
}

// log_losses of the reference from the accumulated sums:
// sums = {cls, iou, dfl, sum assigned scores, pose_cls, pose_reg, number of positives, -}
SGB_HD void finalize(const SgbPoseLossDesc& d, const double* sums, float* out) {
  const double nrm = sums[3] < 1.0 ? 1.0 : sums[3];
  const double kden = d.rescale_with_score ? nrm : (sums[6] < 1.0 ? 1.0 : sums[6]);
  const float c = (float)(d.w_cls * sums[0] / nrm), i = (float)(d.w_iou * sums[1] / nrm), f = (float)(d.w_dfl * sums[2] / nrm);
  const float pc = (float)(d.w_pose_cls * sums[4] / kden), pr = (float)(d.w_pose_reg * sums[5] / kden);
  out[0] = c;
  out[1] = i;
  out[2] = f;
  out[3] = pc;
  out[4] = pr;
  out[5] = c + i + f + pc + pr;
}

}  // namespace sgb_pose

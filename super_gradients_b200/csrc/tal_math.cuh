// Arithmetic shared by the task-aligned assigners and box losses of PPYoloELoss (loss.cu), YoloNASPoseLoss (pose_loss.cu) and
// the ATSS assigner (atss.cu), host+device like the other *_math.cuh headers: the kernels call these per thread, and the CPU
// suite compiles this header with g++ behind the serial drivers of tests/host_kernels/ (pose_loss_host.cpp, atss_host.cpp).
// block_topk and fill_background are device / launch code and exist only under nvcc.
//
// Reference: src/super_gradients/training/losses/ppyolo_loss.py
//   batch_iou_similarity :17-35 (eps 1e-9), iou_similarity :38-60 (eps 1e-10), check_points_inside_bboxes :178-211,
//   TaskAlignedAssigner.forward :454-561, PPYoloELoss._bbox_decode :1054-1061, _df_loss :994-1006, GIoULoss :564-638,
//   _focal_loss :1069-1077;  CIoU: training/losses/functional.py:82-133.
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

namespace sgb_tal {

struct Box {
  float x1, y1, x2, y2;
};

SGB_HD Box load_box(const float* p) { return Box{p[0], p[1], p[2], p[3]}; }
SGB_HD void store_box(float* p, const Box& b) {
  p[0] = b.x1;
  p[1] = b.y1;
  p[2] = b.x2;
  p[3] = b.y2;
}

SGB_HD float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }
SGB_HD float softplus_f(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }  // = BCE-with-logits(x, 0)

// IoU of two xyxy boxes; the reference uses eps = 1e-9 in the assigners' batch form and 1e-10 in the ATSS candidate form
SGB_HD float iou(const Box& g, const Box& p, float eps) {
  const float ov = fmaxf(fminf(g.x2, p.x2) - fmaxf(g.x1, p.x1), 0.f) * fmaxf(fminf(g.y2, p.y2) - fmaxf(g.y1, p.y1), 0.f);
  const float a1 = fmaxf(g.x2 - g.x1, 0.f) * fmaxf(g.y2 - g.y1, 0.f);
  const float a2 = fmaxf(p.x2 - p.x1, 0.f) * fmaxf(p.y2 - p.y1, 0.f);
  return ov / (a1 + a2 - ov + eps);
}

// softmax-expectation decode of one anchor's 4 x nb DFL logits: distances in stride units around the anchor point, box in pixels
SGB_HD Box decode_box(const float* z, int nb, float apx, float apy, float s) {
  float d[4];
  for (int sd = 0; sd < 4; ++sd) {
    float mx = -INFINITY;
    for (int b = 0; b < nb; ++b) mx = fmaxf(mx, z[sd * nb + b]);
    float se = 0.f, sw = 0.f;
    for (int b = 0; b < nb; ++b) {
      const float e = expf(z[sd * nb + b] - mx);
      se += e;
      sw += e * (float)b;
    }
    d[sd] = sw / se;
  }
  const float ax = apx / s, ay = apy / s;
  return Box{(ax - d[0]) * s, (ay - d[1]) * s, (ax + d[2]) * s, (ay + d[3]) * s};
}

// alignment metric score^alpha * iou^beta
SGB_HD float tal_metric(float alpha, float beta, float score, float iou) {
  const float a = alpha == 1.f ? score : powf(score, alpha);
  return a * powf(iou, beta);
}

SGB_HD bool inside_gt(float ax, float ay, const Box& g) {  // check_points_inside_bboxes, eps = 1e-9
  return fminf(fminf(ax - g.x1, ay - g.y1), fminf(g.x2 - ax, g.y2 - ay)) > 1e-9f;
}

// One anchor after the per-GT top-k selection (ppyolo_loss.py:521-538): the valid GTs whose top-k list holds anchor l and whose
// box contains the anchor point (ax, ay) claim it.  One claim -> that GT; several -> the GT row of highest pair IoU over ALL rows
// (padded rows are zero boxes), first maximum wins.  gtb [n_max][4], gtv [n_max] and sel [n_max][topk] are the rows of the
// anchor's image.  pair_iou(g, box) is the IoU of GT row g with the anchor's prediction, score(g) its score for GT g's class.
// Returns the assigned GT (or -1) with the metric and IoU of that pair (0 when unassigned).
template <class PairIou, class Score>
SGB_HD int resolve_anchor(int l, float ax, float ay, int n_max, int topk, const float* gtb, const uint8_t* gtv, const int* sel,
                          float alpha, float beta, PairIou pair_iou, Score score, float* met, float* iou_out) {
  int npos = 0, first = -1, best_g = 0;
  float best_iou = -1.f;
  for (int g = 0; g < n_max; ++g) {
    const Box gb = load_box(gtb + g * 4);
    const float v = pair_iou(g, gb);
    if (v > best_iou) {
      best_iou = v;
      best_g = g;
    }
    if (!gtv[g]) continue;
    bool in_topk = false;
    for (int k = 0; k < topk; ++k) in_topk |= (sel[g * topk + k] == l);
    if (!in_topk || !inside_gt(ax, ay, gb)) continue;
    if (npos == 0) first = g;
    ++npos;
  }
  const int ag = npos == 1 ? first : (npos > 1 ? best_g : -1);
  *met = 0.f;
  *iou_out = 0.f;
  if (ag >= 0) {
    *iou_out = pair_iou(ag, load_box(gtb + ag * 4));
    *met = tal_metric(alpha, beta, score(ag), *iou_out);
  }
  return ag;
}

// assigned score of a positive anchor: its metric normalised by its GT's largest metric, times that GT's largest IoU (:553-558)
SGB_HD float assigned_score(float met, float gt_max_metric, float gt_max_iou) { return met / (gt_max_metric + 1e-9f) * gt_max_iou; }

// focal (gamma = 2, weight NOT detached) or plain BCE with logits against a soft / hard label q; alpha <= 0: no alpha_t
SGB_HD void cls_term(int focal, float alpha, float x, float q, float* loss, float* grad) {
  const float p = sigmoid_f(x);
  const float bce = softplus_f(x) - x * q;
  if (!focal) {
    *loss = bce;
    *grad = p - q;
    return;
  }
  const float dq = p - q;
  const float at = alpha > 0.f ? alpha * q + (1.f - alpha) * (1.f - q) : 1.f;
  *loss = at * dq * dq * bce;
  *grad = at * (2.f * dq * p * (1.f - p) * bce + dq * dq * dq);
}

// GIoU (iou_type 0) or CIoU (1) loss of a predicted box against a target, and its gradient w.r.t. (x1, y1, x2, y2)
SGB_HD void iou_loss_grad(int iou_type, float x1, float y1, float x2, float y2, float gx1, float gy1, float gx2, float gy2,
                          float* loss, float* gb) {
  const float eps = 1e-10f;
  const float ix1 = fmaxf(x1, gx1), iy1 = fmaxf(y1, gy1), ix2 = fminf(x2, gx2), iy2 = fminf(y2, gy2);
  const float wi = fmaxf(ix2 - ix1, 0.f), hi = fmaxf(iy2 - iy1, 0.f);
  const float ov = wi * hi;
  const float w1 = x2 - x1, h1 = y2 - y1, w2 = gx2 - gx1, h2 = gy2 - gy1;
  const float un = w1 * h1 + w2 * h2 - ov + eps;
  const float iou = ov / un;
  const bool pos = wi > 0.f && hi > 0.f;
  const float dov[4] = {(pos && x1 > gx1) ? -hi : 0.f, (pos && y1 > gy1) ? -wi : 0.f, (pos && x2 < gx2) ? hi : 0.f,
                        (pos && y2 < gy2) ? wi : 0.f};
  const float da1[4] = {-h1, -w1, h1, w1};
  const float cw = fmaxf(x2, gx2) - fminf(x1, gx1), chh = fmaxf(y2, gy2) - fminf(y1, gy1);
  if (iou_type == 0) {
    const float ac = cw * chh + eps;
    *loss = 1.f - (iou - (ac - un) / ac);
    const float dac[4] = {x1 < gx1 ? -chh : 0.f, y1 < gy1 ? -cw : 0.f, x2 > gx2 ? chh : 0.f, y2 > gy2 ? cw : 0.f};
    for (int k = 0; k < 4; ++k) {
      float dun = da1[k] - dov[k];
      float diou = (dov[k] * un - ov * dun) / (un * un);
      float dr = (dun * ac - un * dac[k]) / (ac * ac);
      gb[k] = -diou - dr;
    }
    return;
  }
  // (1 - iou) + rho2 / (cw^2 + ch^2 + eps) + v * alpha, alpha = v / max((1 - iou) + v, eps) detached
  const float c2 = cw * cw + chh * chh + eps;
  const float dxc = (x1 + x2) * 0.5f - (gx1 + gx2) * 0.5f, dyc = (y1 + y2) * 0.5f - (gy1 + gy2) * 0.5f;
  const float rho2 = dxc * dxc + dyc * dyc;
  const float k4pi2 = 4.f / (3.14159265358979323846f * 3.14159265358979323846f);
  const float at = atanf(w2 / h2) - atanf(w1 / h1);
  const float v = k4pi2 * at * at;
  const float alpha = v / fmaxf((1.f - iou) + v, eps);
  *loss = (1.f - iou) + rho2 / c2 + v * alpha;
  const float dcw[4] = {x1 < gx1 ? -1.f : 0.f, 0.f, x2 > gx2 ? 1.f : 0.f, 0.f};
  const float dch[4] = {0.f, y1 < gy1 ? -1.f : 0.f, 0.f, y2 > gy2 ? 1.f : 0.f};
  const float drho[4] = {dxc, dyc, dxc, dyc};  // d rho2 / d coord = 2 * d * 0.5
  const float den = w1 * w1 + h1 * h1;
  const float dat_w = -h1 / den, dat_h = w1 / den;  // d at / d w1, d at / d h1
  const float dw1[4] = {-1.f, 0.f, 1.f, 0.f}, dh1[4] = {0.f, -1.f, 0.f, 1.f};
  for (int k = 0; k < 4; ++k) {
    float dun = da1[k] - dov[k];
    float diou = (dov[k] * un - ov * dun) / (un * un);
    float dc2 = 2.f * cw * dcw[k] + 2.f * chh * dch[k];
    float dterm = (drho[k] * c2 - rho2 * dc2) / (c2 * c2);
    float dv = k4pi2 * 2.f * at * (dat_w * dw1[k] + dat_h * dh1[k]);
    gb[k] = -diou + dterm + alpha * dv;
  }
}

// DFL target of one side (_df_loss): the distance t, clipped to [0, reg_max - 0.01], splits between bins tl and tl + 1 with
// weights wl and wr
struct DflTarget {
  int tl;
  float wl, wr;
};
SGB_HD DflTarget dfl_target(float t, int reg_max) {
  const float tcl = fminf(fmaxf(t, 0.f), (float)reg_max - 0.01f);
  const int tl = (int)tcl;  // trunc == floor (non-negative)
  const float wl = (float)(tl + 1) - tcl;
  return DflTarget{tl, wl, 1.f - wl};
}

// assigner workspace, all [B][...]: pbox [L][4] f32 decoded boxes in pixels, topk [n][k] i32 selected anchors per GT (-1: none),
// gmax [n][2] i32 float bits of the largest metric / IoU per GT (atomicMax), apair [L][2] f32 metric and IoU of the assigned
// pair, agt [L] i32 assigned GT or -1
struct Ws {
  float* pbox;
  int* topk;
  int* gmax;
  float* apair;
  int* agt;
};
SGB_HD int64_t ws_floats(int B, int L, int n, int k) {
  return (int64_t)B * L * 4 + (int64_t)B * n * k + (int64_t)B * n * 2 + (int64_t)B * L * 2 + (int64_t)B * L;
}
SGB_HD Ws ws_carve(void* ws, int B, int L, int n, int k) {
  Ws w;
  float* p = reinterpret_cast<float*>(ws);
  w.pbox = p;
  p += (int64_t)B * L * 4;
  w.topk = reinterpret_cast<int*>(p);
  p += (int64_t)B * n * k;
  w.gmax = reinterpret_cast<int*>(p);
  p += (int64_t)B * n * 2;
  w.apair = p;
  p += (int64_t)B * L * 2;
  w.agt = reinterpret_cast<int*>(p);
  return w;
}

#ifdef __CUDACC__
// Block-wide iterative top-k of a shared-memory row v[0, n), 256 threads: each of k rounds takes the largest remaining value,
// ties to the lowest index (strict comparison within a thread, butterfly within each warp, then thread 0 merges the 8 warps),
// hands the index to take(round, index) on thread 0 and marks that entry -INFINITY so it is never taken again.  -INFINITY and
// NaN are never taken: a round with none left gets the index 0x7fffffff.
template <class Take>
__device__ __forceinline__ void block_topk(float* v, int n, int k, Take take) {
  __shared__ float sval[8];
  __shared__ int sidx[8];
  const int t = threadIdx.x;
  for (int r = 0; r < k; ++r) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int l = t; l < n; l += blockDim.x) {
      const float x = v[l];
      if (x > bv) {  // strict: keeps the lowest index within a thread
        bv = x;
        bi = l;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) {
        bv = ov;
        bi = oi;
      }
    }
    if ((t & 31) == 0) {
      sval[t >> 5] = bv;
      sidx[t >> 5] = bi;
    }
    __syncthreads();
    if (t == 0) {
      for (int q = 1; q < 8; ++q)
        if (sval[q] > bv || (sval[q] == bv && sidx[q] < bi)) {
          bv = sval[q];
          bi = sidx[q];
        }
      take(r, bi);
      if (bi < n) v[bi] = -INFINITY;
    }
    __syncthreads();
  }
}

// Every anchor is background (a batch without targets): label[i] = value, score[i] = 0 and, when box is given, a zero box.
// Defined in loss.cu.
int fill_background(int* label, int value, float* score, float* box, int64_t n, cudaStream_t st);
#endif

}  // namespace sgb_tal

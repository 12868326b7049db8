// DFL head decode, task-aligned assignment and the fused VFL + GIoU/CIoU + DFL loss (forward AND backward in one
// launch) for YOLO-NAS / PP-YOLOE.  HBM-bound: the logits [B, L, C + 4*(reg_max+1)] are read once and their
// gradient written once (SURVEY.md section 8d); everything the assigner needs per (gt, anchor) pair is recomputed
// in registers / shared memory instead of being materialised as the reference's [B, n, L] temporaries.
//
// Reference: src/super_gradients/training/losses/ppyolo_loss.py
//   TaskAlignedAssigner.forward :454-561, batch_iou_similarity :17-35, check_points_inside_bboxes :178-211,
//   gather_topk_anchors :214-230, compute_max_iou_anchor :165-175, PPYoloELoss._bbox_decode :1054-1061,
//   _varifocal_loss :1079-1084, _bbox_loss :1008-1052, GIoULoss :564-638, _df_loss :994-1006, forward :944-988;
//   CIoU: training/losses/functional.py:82-133;  decode: detection_models/yolo_nas/dfl_heads.py:199-245.
#include <math_constants.h>

#include "common.cuh"
#include "tal_math.cuh"

namespace {

using namespace sgb_tal;

constexpr int MAXBINS = 32;  // reg_max + 1 <= 32

// ------------------------------------------------------------------------------------------------ head decode
__global__ void dfl_decode_kernel(const bf16* __restrict__ reg, int reg_pitch, const bf16* __restrict__ cls,
                                  int cls_pitch, int N, int Hf, int Wf, int L, int abase, int ncls, int reg_max,
                                  float stride, float cell_off, float* pred_bboxes, float* pred_scores,
                                  float* cls_logits, float* reg_distri) {
  const int HW = Hf * Wf;
  const int nb = reg_max + 1;
  const int per = 4 + ncls;  // work items per anchor: 4 sides + ncls classes
  const int64_t total = (int64_t)N * HW * per;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int item = i % per;
    int64_t a = i / per;
    int hw = a % HW;
    int n = a / HW;
    int64_t row = (int64_t)n * L + abase + hw;
    if (item < 4) {
      const bf16* z = reg + ((int64_t)n * HW + hw) * reg_pitch + item * nb;
      float v[MAXBINS];
      float mx = -CUDART_INF_F;
#pragma unroll 1
      for (int b = 0; b < nb; ++b) {
        v[b] = __bfloat162float(z[b]);
        mx = fmaxf(mx, v[b]);
        if (reg_distri) reg_distri[row * (4 * nb) + item * nb + b] = v[b];
      }
      float se = 0.f, sw = 0.f;
#pragma unroll 1
      for (int b = 0; b < nb; ++b) {
        float e = expf(v[b] - mx);
        se += e;
        sw += e * (float)b;
      }
      float d = sw / se;
      float ax = (float)(hw % Wf) + cell_off, ay = (float)(hw / Wf) + cell_off;
      float c = (item & 1) ? ay : ax;
      float o = item < 2 ? (c - d) : (c + d);
      pred_bboxes[row * 4 + item] = o * stride;
    } else {
      int c = item - 4;
      float x = __bfloat162float(cls[((int64_t)n * HW + hw) * cls_pitch + c]);
      if (cls_logits) cls_logits[row * ncls + c] = x;
      pred_scores[row * ncls + c] = 1.f / (1.f + expf(-x));
    }
  }
}

// Tiled form of the decode: one CTA owns DT consecutive anchors of one image.  Their reg / cls rows are staged in shared memory with
// 16-byte loads (the rows of consecutive anchors are contiguous in NHWC), one thread per (anchor, box side) runs the softmax
// expectation over its bins from shared memory, and all threads then stream the fp32 copies out: the output rows of consecutive
// anchors are contiguous too, so every store instruction writes consecutive floats.  Same arithmetic per element as the kernel above
// (max, expf, sums in bin order), which served one (anchor, side) or one (anchor, class) per thread with 2-byte loads and a
// divergent 4-of-84 split: 240 us for the 80 x 80 level at batch 32, against 250 MB = 38 us at the HBM peak.
constexpr int DT = 64;
__global__ void __launch_bounds__(256) dfl_decode_tile_kernel(const bf16* __restrict__ reg, int reg_pitch, const bf16* __restrict__ cls, int cls_pitch,
                                                              int HW, int Wf, int L, int abase, int ncls, int nb, float stride, float cell_off,
                                                              float* __restrict__ pred_bboxes, float* __restrict__ pred_scores,
                                                              float* __restrict__ cls_logits, float* __restrict__ reg_distri) {
  extern __shared__ __align__(16) unsigned char dsm[];
  const int tiles = (HW + DT - 1) / DT;
  const int n = blockIdx.x / tiles, t0 = (blockIdx.x % tiles) * DT;
  const int na = min(DT, HW - t0);
  const int rc = 4 * nb;                       // reg channels used
  const int rv = (rc + 7) / 8, cv = (ncls + 7) / 8;  // 16-byte vectors per anchor row (the pitch covers the round-up: checked on the host)
  uint4* sreg = reinterpret_cast<uint4*>(dsm);  // [DT][rv]
  uint4* scls = sreg + DT * rv;                 // [DT][cv]
  const int64_t a0 = (int64_t)n * HW + t0;
  for (int i = threadIdx.x; i < na * rv; i += 256) {
    const int a = i / rv, v = i - a * rv;
    sreg[i] = *reinterpret_cast<const uint4*>(reg + (a0 + a) * reg_pitch + v * 8);
  }
  for (int i = threadIdx.x; i < na * cv; i += 256) {
    const int a = i / cv, v = i - a * cv;
    scls[i] = *reinterpret_cast<const uint4*>(cls + (a0 + a) * cls_pitch + v * 8);
  }
  __syncthreads();
  const bf16* breg = reinterpret_cast<const bf16*>(sreg);
  const bf16* bcls = reinterpret_cast<const bf16*>(scls);
  const int64_t row0 = (int64_t)n * L + abase + t0;
  // boxes: thread -> (anchor, side)
  for (int i = threadIdx.x; i < na * 4; i += 256) {
    const int a = i >> 2, side = i & 3;
    const bf16* z = breg + a * rv * 8 + side * nb;
    float mx = -CUDART_INF_F;
    for (int b = 0; b < nb; ++b) mx = fmaxf(mx, __bfloat162float(z[b]));
    float se = 0.f, sw = 0.f;
    for (int b = 0; b < nb; ++b) {
      const float e = expf(__bfloat162float(z[b]) - mx);
      se += e;
      sw += e * (float)b;
    }
    const float d = sw / se;
    const int hw = t0 + a;
    const float ax = (float)(hw % Wf) + cell_off, ay = (float)(hw / Wf) + cell_off;
    const float c = (side & 1) ? ay : ax;
    const float o = side < 2 ? (c - d) : (c + d);
    pred_bboxes[(row0 + a) * 4 + side] = o * stride;
  }
  if (reg_distri) {
    for (int i = threadIdx.x; i < na * rc; i += 256) {
      const int a = i / rc, c = i - a * rc;
      reg_distri[row0 * rc + i] = __bfloat162float(breg[a * rv * 8 + c]);
    }
  }
  for (int i = threadIdx.x; i < na * ncls; i += 256) {
    const int a = i / ncls, c = i - a * ncls;
    const float x = __bfloat162float(bcls[a * cv * 8 + c]);
    if (cls_logits) cls_logits[row0 * ncls + i] = x;
    pred_scores[row0 * ncls + i] = 1.f / (1.f + expf(-x));
  }
}

// Keypoint decode of one pyramid level (row L8: yolo_nas_pose_ndfl_heads.py:186-199): per anchor and joint
//   xy = (offset * multiplier + anchor_point_in_stride_units - compensation) * stride,  score = sigmoid(logit).
// pose: [N, HW, pose_pitch] bf16 with channel 2*j + {0: x, 1: y};  logit: [N, HW, logit_pitch] bf16, joint j at channel
// logit_off + j (the reference keeps the joint logits in the class head: channels 1..J of cls_pred).
__global__ void pose_keypoint_decode_kernel(const bf16* __restrict__ pose, int pose_pitch, const bf16* __restrict__ logit,
                                            int logit_pitch, int logit_off, int N, int Hf, int Wf, int L, int abase, int J,
                                            float stride, float cell_off, float mult, float comp, float* coords,
                                            float* scores, float* logits_out) {
  const int HW = Hf * Wf;
  const int64_t total = (int64_t)N * HW * J;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int j = i % J;
    const int64_t a = i / J;
    const int hw = a % HW;
    const int n = a / HW;
    const int64_t row = (int64_t)n * L + abase + hw;
    const bf16* pz = pose + ((int64_t)n * HW + hw) * pose_pitch + 2 * j;
    const float ax = (float)(hw % Wf) + cell_off, ay = (float)(hw / Wf) + cell_off;
    const float ox = __bfloat162float(pz[0]), oy = __bfloat162float(pz[1]);
    coords[(row * J + j) * 2 + 0] = (ox * mult + (ax - comp)) * stride;
    coords[(row * J + j) * 2 + 1] = (oy * mult + (ay - comp)) * stride;
    const float x = __bfloat162float(logit[((int64_t)n * HW + hw) * logit_pitch + logit_off + j]);
    if (logits_out) logits_out[row * J + j] = x;
    scores[row * J + j] = 1.f / (1.f + expf(-x));
  }
}

// 8 channels per thread (two 16-byte loads when the row length allows, one 16-byte store), 32-bit index arithmetic
__global__ void __launch_bounds__(256) head_grad_scatter_v8_kernel(const float* __restrict__ g, int gC, int HW, int L, int abase, bf16* __restrict__ dy,
                                                                    int pitch, int cv, uint32_t total) {
  for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < total; i += gridDim.x * 256u) {
    const uint32_t v = i % (uint32_t)cv, a = i / (uint32_t)cv;  // a = n * HW + hw
    const uint32_t n = a / (uint32_t)HW, hw = a - n * (uint32_t)HW;
    const float* src = g + ((size_t)n * L + abase + hw) * gC + v * 8;
    float f[8];
    const int c0 = (int)v * 8;
    if (c0 + 8 <= gC && (gC & 3) == 0) {
      const float4 lo = *reinterpret_cast<const float4*>(src), hi = *reinterpret_cast<const float4*>(src + 4);
      f[0] = lo.x; f[1] = lo.y; f[2] = lo.z; f[3] = lo.w; f[4] = hi.x; f[5] = hi.y; f[6] = hi.z; f[7] = hi.w;
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = c0 + e < gC ? src[e] : 0.f;
    }
    uint4 r;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
    for (int e = 0; e < 4; ++e) h[e] = __floats2bfloat162_rn(f[2 * e], f[2 * e + 1]);
    *reinterpret_cast<uint4*>(dy + (size_t)a * pitch + c0) = r;
  }
}

// gradient of the raw fp32 copies back into the per-level bf16 NHWC head outputs
__global__ void head_grad_scatter_kernel(const float* __restrict__ g, int gC, int N, int HW, int L, int abase,
                                         bf16* dy, int pitch, int cpad) {
  const int64_t total = (int64_t)N * HW * cpad;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int c = i % cpad;
    int64_t a = i / cpad;
    int hw = a % HW;
    int n = a / HW;
    float v = c < gC ? g[((int64_t)n * L + abase + hw) * gC + c] : 0.f;
    dy[((int64_t)n * HW + hw) * pitch + c] = __float2bfloat16_rn(v);
  }
}

// ------------------------------------------------------------------------------------------------ TAL
__global__ void tal_decode_kernel(SgbLossDesc d, const float* __restrict__ reg, const float* __restrict__ ap,
                                  const float* __restrict__ st, float* pbox) {
  const int nb = d.reg_max + 1;
  const int64_t total = (int64_t)d.B * d.L;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int l = i % d.L;
    store_box(pbox + i * 4, decode_box(reg + i * 4 * nb, nb, ap[l * 2], ap[l * 2 + 1], st[l]));
  }
}

// one CTA per (image, gt): metric over all anchors -> block-wide top-k
__global__ void __launch_bounds__(256) tal_topk_kernel(SgbLossDesc d, const float* __restrict__ cls,
                                                       const float* __restrict__ ap, const float* __restrict__ gtb,
                                                       const int* __restrict__ gtl, const uint8_t* __restrict__ gtv,
                                                       Ws w) {
  extern __shared__ float smet[];  // [L]
  const int bg = blockIdx.x;  // b * n_max + g
  const int b = bg / d.n_max;
  const int t = threadIdx.x;
  if (t < 2) w.gmax[bg * 2 + t] = 0;
  if (!gtv[bg]) {
    for (int j = t; j < d.topk; j += blockDim.x) w.topk[bg * d.topk + j] = -1;
    return;
  }
  const Box g = load_box(gtb + bg * 4);
  const int label = gtl[bg];
  for (int l = t; l < d.L; l += blockDim.x) {
    const float iou_gp = iou(g, load_box(w.pbox + ((int64_t)b * d.L + l) * 4), 1e-9f);
    const float score = sigmoid_f(cls[((int64_t)b * d.L + l) * d.ncls + label]);
    const float in_gt = inside_gt(ap[l * 2], ap[l * 2 + 1], g) ? 1.f : 0.f;
    smet[l] = tal_metric(d.alpha, d.beta, score, iou_gp) * in_gt;
  }
  __syncthreads();
  block_topk(smet, d.L, d.topk, [&](int k, int l) { w.topk[bg * d.topk + k] = l; });
}

// one thread per (image, anchor): positive mask, multi-assignment resolution, per-gt maxima
__global__ void tal_resolve_kernel(SgbLossDesc d, const float* __restrict__ cls, const float* __restrict__ ap,
                                   const float* __restrict__ gtb, const int* __restrict__ gtl,
                                   const uint8_t* __restrict__ gtv, Ws w) {
  const int64_t total = (int64_t)d.B * d.L;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int l = i % d.L, b = i / d.L, g0 = b * d.n_max;
    const Box p = load_box(w.pbox + i * 4);
    float met, iou_ag;
    const int ag = resolve_anchor(
        l, ap[l * 2], ap[l * 2 + 1], d.n_max, d.topk, gtb + g0 * 4, gtv + g0, w.topk + g0 * d.topk, d.alpha, d.beta,
        [&](int, const Box& gb) { return iou(gb, p, 1e-9f); }, [&](int g) { return sigmoid_f(cls[i * d.ncls + gtl[g0 + g]]); }, &met,
        &iou_ag);
    w.agt[i] = ag;
    w.apair[i * 2 + 0] = met;
    w.apair[i * 2 + 1] = iou_ag;
    if (ag >= 0) {  // metric and iou are non-negative: their float bit patterns order like ints
      atomicMax(&w.gmax[(g0 + ag) * 2 + 0], __float_as_int(met));
      atomicMax(&w.gmax[(g0 + ag) * 2 + 1], __float_as_int(iou_ag));
    }
  }
}

__global__ void tal_finish_kernel(SgbLossDesc d, const float* __restrict__ gtb, const int* __restrict__ gtl, Ws w,
                                  int* alabel, float* abox, float* ascore, double* sums) {
  const int64_t total = (int64_t)d.B * d.L;
  float local = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int b = i / d.L;
    int ag = w.agt[i];
    int bg = b * d.n_max + (ag >= 0 ? ag : 0);
    // the reference gathers gt 0's box for unassigned anchors (argmax of an all-zero column)
    store_box(abox + i * 4, load_box(gtb + bg * 4));
    float sc = 0.f;
    int lab = d.ncls;
    if (ag >= 0) {
      lab = gtl[bg];
      sc = assigned_score(w.apair[i * 2], __int_as_float(w.gmax[bg * 2 + 0]), __int_as_float(w.gmax[bg * 2 + 1]));
    }
    alabel[i] = lab;
    ascore[i] = sc;
    local += sc;
  }
  local = warp_sum(local);
  if ((threadIdx.x & 31) == 0 && local != 0.f) atomicAdd(&sums[3], (double)local);
}

// ------------------------------------------------------------------------------------------------ loss fwd + bwd
// one warp per anchor.
__global__ void __launch_bounds__(256) loss_kernel(SgbLossDesc d, const float* __restrict__ cls,
                                                   const float* __restrict__ reg, const float* __restrict__ ap,
                                                   const float* __restrict__ st, const int* __restrict__ alabel,
                                                   const float* __restrict__ abox, const float* __restrict__ ascore,
                                                   double* sums, float grad_scale, float* gcls, float* greg) {
  const int lane = threadIdx.x & 31;
  const int nb = d.reg_max + 1;
  const int64_t total = (int64_t)d.B * d.L;
  const int64_t warp0 = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  double nrm = sums[3];
  if (nrm < 1.0) nrm = 1.0;
  const float inv = grad_scale / (float)nrm;
  float acc_cls = 0.f, acc_iou = 0.f, acc_dfl = 0.f;
  for (int64_t i = warp0; i < total; i += nwarps) {
    const int l = i % d.L;
    const int lab = alabel[i];
    const float q = ascore[i];
    // ---- varifocal loss over classes (alpha = 0.75, gamma = 2)
    for (int c = lane; c < d.ncls; c += 32) {
      float x = cls[i * d.ncls + c];
      float p = 1.f / (1.f + expf(-x));
      float sp = fmaxf(x, 0.f) + log1pf(expf(-fabsf(x)));  // softplus(x) = BCE(x, 0)
      float loss, g;
      if (c == lab) {
        float bce = sp - x * q;
        loss = q * bce;
        g = q * (p - q);
      } else {
        float wgt = 0.75f * p * p;
        loss = wgt * sp;
        g = 0.75f * (2.f * p * p * (1.f - p) * sp + p * p * p);
      }
      acc_cls += loss;
      if (gcls) gcls[i * d.ncls + c] = g * d.w_cls * inv;
    }
    // ---- box terms (positives only)
    if (lab == d.ncls) {
      if (greg)
        for (int j = lane; j < 4 * nb; j += 32) greg[i * 4 * nb + j] = 0.f;
      continue;
    }
    const float s = st[l];
    const float ax = ap[l * 2] / s, ay = ap[l * 2 + 1] / s;
    const float gx1 = abox[i * 4 + 0] / s, gy1 = abox[i * 4 + 1] / s, gx2 = abox[i * 4 + 2] / s,
                gy2 = abox[i * 4 + 3] / s;
    float dist[4], prob = 0.f;  // lane b (< nb) keeps p_b of the side being processed; we need all 4 later
    float pside[4];
#pragma unroll
    for (int sd = 0; sd < 4; ++sd) {
      float z = lane < nb ? reg[i * 4 * nb + sd * nb + lane] : -CUDART_INF_F;
      float mx = z;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float e = lane < nb ? expf(z - mx) : 0.f;
      float se = warp_sum(e);
      prob = e / se;
      pside[sd] = prob;
      dist[sd] = warp_sum(prob * (float)lane);
    }
    float liou, gb[4];
    iou_loss_grad(d.iou_type, ax - dist[0], ay - dist[1], ax + dist[2], ay + dist[3], gx1, gy1, gx2, gy2, &liou, gb);
    // ---- DFL
    float tgt[4] = {ax - gx1, ay - gy1, gx2 - ax, gy2 - ay};
    float ldfl = 0.f;
    const float wq = q;  // bbox_weight = sum_c assigned_scores = q
    // d(box)/d(dist): x1 = ax - d0, y1 = ay - d1, x2 = ax + d2, y2 = ay + d3
    const float sgn[4] = {-1.f, -1.f, 1.f, 1.f};
#pragma unroll
    for (int sd = 0; sd < 4; ++sd) {
      const auto [tl, wl, wr] = dfl_target(tgt[sd], d.reg_max);
      float p = pside[sd];
      float lp = lane < nb ? logf(fmaxf(p, 1e-38f)) : 0.f;
      float ce = 0.f;
      if (lane == tl) ce = -lp * wl;
      if (lane == tl + 1) ce = -lp * wr;
      ldfl += warp_sum(ce);
      if (greg && lane < nb) {
        float gd = wq * 0.25f * (p - (lane == tl ? wl : 0.f) - (lane == tl + 1 ? wr : 0.f));
        float gi = wq * gb[sd] * sgn[sd] * p * ((float)lane - dist[sd]);
        greg[i * 4 * nb + sd * nb + lane] = (d.w_dfl * gd + d.w_iou * gi) * inv;
      }
    }
    if (lane == 0) {
      acc_iou += liou * wq;
      acc_dfl += ldfl * 0.25f * wq;
    }
  }
  acc_cls = warp_sum(acc_cls);
  __shared__ float sh[3][8];
  if (lane == 0) {
    sh[0][threadIdx.x >> 5] = acc_cls;
    sh[1][threadIdx.x >> 5] = acc_iou;
    sh[2][threadIdx.x >> 5] = acc_dfl;
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    float v = 0.f;
    for (int q = 0; q < (int)(blockDim.x >> 5); ++q) v += sh[threadIdx.x][q];
    atomicAdd(&sums[threadIdx.x], (double)v);
  }
}

__global__ void loss_finalize_kernel(SgbLossDesc d, const double* sums, float* out) {
  double nrm = sums[3] < 1.0 ? 1.0 : sums[3];
  float c = (float)(d.w_cls * sums[0] / nrm), i = (float)(d.w_iou * sums[1] / nrm), f = (float)(d.w_dfl * sums[2] / nrm);
  out[0] = c;
  out[1] = i;
  out[2] = f;
  out[3] = c + i + f;
}

int check_loss(const SgbLossDesc* d) {
  SGB_REQUIRE(d && d->B > 0 && d->L > 0 && d->ncls > 0, "bad desc");
  SGB_REQUIRE(d->reg_max + 1 <= MAXBINS, "reg_max + 1 must be <= 32");
  SGB_REQUIRE(d->n_max >= 0 && d->topk > 0 && d->topk <= 64, "n_max / topk");
  // tal_topk_kernel takes one anchor per round: with every anchor taken it would write past the metric row (torch.topk raises)
  SGB_REQUIRE(d->topk <= d->L, "topk must not exceed the number of anchors");
  return SGB_OK;
}

}  // namespace

namespace sgb_tal {

__global__ void fill_background_kernel(int* label, int value, float* score, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    label[i] = value;
    score[i] = 0.f;
  }
}

int fill_background(int* label, int value, float* score, float* box, int64_t n, cudaStream_t st) {
  if (box) cudaMemsetAsync(box, 0, n * 4 * sizeof(float), st);
  const int grid = (int)((n + 255) / 256 > 132 * 8 ? 132 * 8 : (n + 255) / 256);
  fill_background_kernel<<<grid, 256, 0, st>>>(label, value, score, n);
  SGB_LAUNCH_CHECK("fill_background_kernel");
  return SGB_OK;
}

}  // namespace sgb_tal

extern "C" int sgb_dfl_decode(const sgb_bf16* reg, int reg_pitch, const sgb_bf16* cls, int cls_pitch, int N, int Hf,
                              int Wf, int L, int anchor_base, int ncls, int reg_max, float stride, float cell_offset,
                              float* pred_bboxes, float* pred_scores, float* cls_logits, float* reg_distri,
                              void* stream) {
  SGB_REQUIRE(reg && cls && pred_bboxes && pred_scores, "null pointer");
  SGB_REQUIRE(reg_max + 1 <= MAXBINS, "reg_max + 1 must be <= 32");
  SGB_REQUIRE(anchor_base >= 0 && anchor_base + Hf * Wf <= L, "anchor range");
  {
    const int nb = reg_max + 1, rv = (4 * nb + 7) / 8, cv = (ncls + 7) / 8;
    const size_t smem = (size_t)DT * (rv + cv) * 16;
    const int64_t ctas = (int64_t)N * ((Hf * Wf + DT - 1) / DT);
    if (reg_pitch % 8 == 0 && cls_pitch % 8 == 0 && reg_pitch >= rv * 8 && cls_pitch >= cv * 8 && smem <= 48 * 1024 && ctas < (1ll << 31) &&
        ((uintptr_t)reg % 16 == 0) && ((uintptr_t)cls % 16 == 0)) {
      dfl_decode_tile_kernel<<<(int)ctas, 256, smem, (cudaStream_t)stream>>>((const bf16*)reg, reg_pitch, (const bf16*)cls, cls_pitch, Hf * Wf, Wf, L,
                                                                             anchor_base, ncls, nb, stride, cell_offset, pred_bboxes, pred_scores,
                                                                             cls_logits, reg_distri);
      SGB_LAUNCH_CHECK("dfl_decode_tile_kernel");
      return SGB_OK;
    }
  }
  int64_t total = (int64_t)N * Hf * Wf * (4 + ncls);
  int grid = (int)((total + 255) / 256 > 132 * 16 ? 132 * 16 : (total + 255) / 256);
  dfl_decode_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const bf16*)reg, reg_pitch, (const bf16*)cls, cls_pitch, N,
                                                            Hf, Wf, L, anchor_base, ncls, reg_max, stride, cell_offset,
                                                            pred_bboxes, pred_scores, cls_logits, reg_distri);
  SGB_LAUNCH_CHECK("dfl_decode_kernel");
  return SGB_OK;
}

extern "C" int sgb_pose_keypoint_decode(const sgb_bf16* pose, int pose_pitch, const sgb_bf16* logit, int logit_pitch,
                                        int logit_off, int N, int Hf, int Wf, int L, int anchor_base, int J, float stride,
                                        float cell_offset, float offset_multiplier, int compensate_grid_cell_offset,
                                        float* pose_coords, float* pose_scores, float* pose_logits, void* stream) {
  SGB_REQUIRE(pose && logit && pose_coords && pose_scores, "null pointer");
  SGB_REQUIRE(N > 0 && Hf > 0 && Wf > 0 && J > 0, "bad shape");
  SGB_REQUIRE(pose_pitch >= 2 * J && logit_pitch >= logit_off + J && logit_off >= 0, "channel range exceeds pitch");
  SGB_REQUIRE(anchor_base >= 0 && anchor_base + Hf * Wf <= L, "anchor range");
  int64_t total = (int64_t)N * Hf * Wf * J;
  int grid = (int)((total + 255) / 256 > 132 * 16 ? 132 * 16 : (total + 255) / 256);
  pose_keypoint_decode_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      (const bf16*)pose, pose_pitch, (const bf16*)logit, logit_pitch, logit_off, N, Hf, Wf, L, anchor_base, J, stride, cell_offset,
      offset_multiplier, compensate_grid_cell_offset ? cell_offset : 0.f, pose_coords, pose_scores, pose_logits);
  SGB_LAUNCH_CHECK("pose_keypoint_decode_kernel");
  return SGB_OK;
}

extern "C" int sgb_head_grad_scatter(const float* grad, int gC, int N, int HW, int L, int anchor_base, sgb_bf16* dy,
                                     int pitch, void* stream) {
  SGB_REQUIRE(grad && dy && pitch >= gC, "bad args");
  int cpad = ((gC + 7) / 8) * 8;
  if (cpad > pitch) cpad = pitch;
  if (pitch % 8 == 0 && cpad % 8 == 0 && (uintptr_t)dy % 16 == 0 && (uintptr_t)grad % 16 == 0 && (int64_t)N * HW * (cpad / 8) < (1ll << 31)) {
    const uint32_t tot = (uint32_t)((int64_t)N * HW * (cpad / 8));
    const int grid8 = (int)((tot + 255u) / 256u > 132u * 16u ? 132u * 16u : (tot + 255u) / 256u);
    head_grad_scatter_v8_kernel<<<grid8 < 1 ? 1 : grid8, 256, 0, (cudaStream_t)stream>>>(grad, gC, HW, L, anchor_base, (bf16*)dy, pitch, cpad / 8, tot);
    SGB_LAUNCH_CHECK("head_grad_scatter_v8_kernel");
    return SGB_OK;
  }
  int64_t total = (int64_t)N * HW * cpad;
  int grid = (int)((total + 255) / 256 > 132 * 16 ? 132 * 16 : (total + 255) / 256);
  head_grad_scatter_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(grad, gC, N, HW, L, anchor_base, (bf16*)dy, pitch,
                                                                   cpad);
  SGB_LAUNCH_CHECK("head_grad_scatter_kernel");
  return SGB_OK;
}

extern "C" int64_t sgb_tal_workspace_bytes(const SgbLossDesc* d) {
  if (!d) return 0;
  return ws_floats(d->B, d->L, d->n_max > 0 ? d->n_max : 1, d->topk) * 4 + 256;
}

extern "C" int sgb_tal_assign(const SgbLossDesc* d, const float* cls_logits, const float* reg_distri,
                              const float* anchor_points, const float* stride_tensor, const float* gt_boxes,
                              const int32_t* gt_labels, const uint8_t* gt_valid, int32_t* assigned_label,
                              float* assigned_box, float* assigned_score, double* sums, void* workspace,
                              int64_t workspace_bytes, void* stream) {
  if (int rc = check_loss(d)) return rc;
  // the top-k keeps one gt's metric row of all L anchors in shared memory
  const size_t smem = (size_t)d->L * sizeof(float);
  SGB_REQUIRE(d->n_max == 0 || smem <= 200 * 1024, "too many anchors for the shared-memory metric row");
  SGB_REQUIRE(cls_logits && reg_distri && anchor_points && stride_tensor && assigned_label && assigned_box &&
                  assigned_score && sums && workspace,
              "null pointer");
  SGB_REQUIRE(workspace_bytes >= sgb_tal_workspace_bytes(d), "workspace too small");
  SGB_REQUIRE(d->n_max > 0 ? (gt_boxes && gt_labels && gt_valid) : true, "gt pointers");
  cudaStream_t st = (cudaStream_t)stream;
  const int nmax = d->n_max > 0 ? d->n_max : 1;
  Ws w = ws_carve(workspace, d->B, d->L, nmax, d->topk);
  const int64_t BL = (int64_t)d->B * d->L;
  int grid = (int)((BL + 255) / 256 > 132 * 8 ? 132 * 8 : (BL + 255) / 256);
  tal_decode_kernel<<<grid, 256, 0, st>>>(*d, reg_distri, anchor_points, stride_tensor, w.pbox);
  SGB_LAUNCH_CHECK("tal_decode_kernel");
  if (d->n_max > 0) {
    // The opt-in above 48 KB counts the kernel's static shared memory too (the top-k's merge slots), so it is set
    // whatever the row size.  It is a per-device setting: set on every call, so every device
    // gets it, and always to the same cap, so concurrent callers never lower it under each other.
    if (int rc = sgb_cuda_check(cudaFuncSetAttribute(tal_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024),
                                "cudaFuncSetAttribute(tal_topk_kernel)"))
      return rc;
    tal_topk_kernel<<<d->B * d->n_max, 256, smem, st>>>(*d, cls_logits, anchor_points, gt_boxes, gt_labels, gt_valid,
                                                        w);
    SGB_LAUNCH_CHECK("tal_topk_kernel");
  }
  // negative batch: every anchor is background (ppyolo_loss.py:499-503)
  if (d->n_max == 0) return fill_background(assigned_label, d->ncls, assigned_score, assigned_box, BL, st);
  tal_resolve_kernel<<<grid, 256, 0, st>>>(*d, cls_logits, anchor_points, gt_boxes, gt_labels, gt_valid, w);
  SGB_LAUNCH_CHECK("tal_resolve_kernel");
  tal_finish_kernel<<<grid, 256, 0, st>>>(*d, gt_boxes, gt_labels, w, assigned_label, assigned_box, assigned_score,
                                          sums);
  SGB_LAUNCH_CHECK("tal_finish_kernel");
  return SGB_OK;
}

extern "C" int sgb_dfl_iou_loss_fwd_bwd(const SgbLossDesc* d, const float* cls_logits, const float* reg_distri,
                                        const float* anchor_points, const float* stride_tensor,
                                        const int32_t* assigned_label, const float* assigned_box,
                                        const float* assigned_score, double* sums, float grad_scale, float* grad_cls,
                                        float* grad_reg, void* stream) {
  if (int rc = check_loss(d)) return rc;
  SGB_REQUIRE(cls_logits && reg_distri && anchor_points && stride_tensor && assigned_label && assigned_box &&
                  assigned_score && sums,
              "null pointer");
  const int64_t BL = (int64_t)d->B * d->L;
  int64_t warps_per_cta = 8;
  int64_t want = (BL + warps_per_cta - 1) / warps_per_cta;
  int grid = (int)(want > 132 * 8 ? 132 * 8 : want);
  loss_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(*d, cls_logits, reg_distri, anchor_points, stride_tensor,
                                                      assigned_label, assigned_box, assigned_score, sums, grad_scale,
                                                      grad_cls, grad_reg);
  SGB_LAUNCH_CHECK("loss_kernel");
  return SGB_OK;
}

extern "C" int sgb_loss_finalize(const SgbLossDesc* d, const double* sums, float* loss_out, void* stream) {
  SGB_REQUIRE(d && sums && loss_out, "null pointer");
  loss_finalize_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(*d, sums, loss_out);
  SGB_LAUNCH_CHECK("loss_finalize_kernel");
  return SGB_OK;
}

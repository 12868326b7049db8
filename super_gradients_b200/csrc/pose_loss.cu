// YoloNASPoseLoss (row L7) on the GPU: OKS-aware task-aligned assigner with crowd handling, then ONE kernel that computes
// the five loss terms (person focal/BCE, GIoU/CIoU, DFL, joint-visibility BCE/focal, OKS keypoint regression) and their
// final gradients.  HBM / latency bound: B*L anchors, 1 + 4*(reg_max+1) + 3*J floats each, read once; only the few
// thousand positive anchors do more than the person-logit term.  The arithmetic lives in pose_loss_math.cuh and tal_math.cuh
// (shared with the detection losses and the CPU test harness); this file is the parallel schedule around it.
//
// Reference: src/super_gradients/training/losses/yolo_nas_pose_loss.py (see pose_loss_math.cuh for line numbers).
#include "common.cuh"
#include "pose_loss_math.cuh"

namespace {

using namespace sgb_pose;
using namespace sgb_tal;

constexpr int MAXBINS = 32;  // reg_max + 1 <= 32
constexpr int MAXJ = 64;

__global__ void pose_decode_kernel(SgbPoseLossDesc d, const float* __restrict__ reg, const float* __restrict__ ap,
                                   const float* __restrict__ st, float* pbox) {
  const int nb = d.reg_max + 1;
  const int64_t total = (int64_t)d.B * d.L;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int l = i % d.L;
    decode_box(reg + i * 4 * nb, nb, ap[l * 2], ap[l * 2 + 1], st[l], pbox + i * 4);
  }
}

// one CTA per (image, gt): metric of every anchor -> iterative top-k (ties: lowest anchor index, like the detection path)
__global__ void __launch_bounds__(256) pose_topk_kernel(SgbPoseLossDesc d, const float* __restrict__ cls,
                                                        const float* __restrict__ pose, const float* __restrict__ ap,
                                                        const float* __restrict__ gtb, const float* __restrict__ gtp,
                                                        const uint8_t* __restrict__ gtv, const float* __restrict__ sigmas,
                                                        Ws w) {
  extern __shared__ float smet[];  // [L]
  __shared__ float sgp[MAXJ * 3];
  __shared__ float ssig[MAXJ];
  const int bg = blockIdx.x;  // b * n_max + g
  const int b = bg / d.n_max;
  const int t = threadIdx.x;
  if (t < 2) w.gmax[bg * 2 + t] = 0;
  if (!gtv[bg]) {
    for (int j = t; j < d.topk; j += blockDim.x) w.topk[bg * d.topk + j] = -1;
    return;
  }
  for (int j = t; j < d.J * 3; j += blockDim.x) sgp[j] = gtp[(int64_t)bg * d.J * 3 + j];
  for (int j = t; j < d.J; j += blockDim.x) ssig[j] = sigmas[j];
  __syncthreads();
  const Box g = load_box(gtb + bg * 4);
  for (int l = t; l < d.L; l += blockDim.x) {
    const int64_t i = (int64_t)b * d.L + l;
    const float iou = pair_iou(d, g, sgp, load_box(w.pbox + i * 4), pose + i * d.J * 2, ssig);
    const float in_gt = inside_gt(ap[l * 2], ap[l * 2 + 1], g) ? 1.f : 0.f;
    smet[l] = tal_metric(d, sigmoid_f(cls[i]), iou) * in_gt;
  }
  __syncthreads();
  block_topk(smet, d.L, d.topk, [&](int k, int l) { w.topk[bg * d.topk + k] = l; });
}

__global__ void pose_resolve_kernel(SgbPoseLossDesc d, const float* __restrict__ cls, const float* __restrict__ pose,
                                    const float* __restrict__ ap, const float* __restrict__ gtb,
                                    const float* __restrict__ gtp, const uint8_t* __restrict__ gtv,
                                    const float* __restrict__ sigmas, Ws w) {
  const int64_t total = (int64_t)d.B * d.L;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int l = i % d.L, b = i / d.L;
    int ag;
    float met, iou;
    resolve_anchor(d, b, l, w.pbox, cls, pose, ap, gtb, gtp, gtv, sigmas, w.topk, &ag, &met, &iou);
    w.agt[i] = ag;
    w.apair[i * 2 + 0] = met;
    w.apair[i * 2 + 1] = iou;
    if (ag >= 0) {  // metric and iou are non-negative: their float bit patterns order like ints
      const int bg = b * d.n_max + ag;
      atomicMax(&w.gmax[bg * 2 + 0], __float_as_int(met));
      atomicMax(&w.gmax[bg * 2 + 1], __float_as_int(iou));
    }
  }
}

__global__ void pose_finish_kernel(SgbPoseLossDesc d, const uint8_t* __restrict__ gtc, Ws w, int* assigned_gt,
                                   float* assigned_score, double* sums) {
  const int64_t total = (int64_t)d.B * d.L;
  float lsum = 0.f, lpos = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int b = i / d.L;
    const int ag = w.agt[i];
    const int bg = b * d.n_max + (ag >= 0 ? ag : 0);
    int pos;
    float sc;
    finish_anchor(ag, w.apair[i * 2], __int_as_float(w.gmax[bg * 2 + 0]), __int_as_float(w.gmax[bg * 2 + 1]),
                  ag >= 0 && gtc[bg] != 0, &pos, &sc);
    assigned_gt[i] = pos;
    assigned_score[i] = sc;
    lsum += sc;
    lpos += pos >= 0 ? 1.f : 0.f;
  }
  lsum = warp_sum(lsum);
  lpos = warp_sum(lpos);
  if ((threadIdx.x & 31) == 0) {
    if (lsum != 0.f) atomicAdd(&sums[3], (double)lsum);
    if (lpos != 0.f) atomicAdd(&sums[6], (double)lpos);
  }
}

// one thread per anchor; block-reduced partial sums -> five fp64 atomics per CTA
__global__ void __launch_bounds__(256) pose_loss_kernel(SgbPoseLossDesc d, const float* __restrict__ cls,
                                                        const float* __restrict__ reg, const float* __restrict__ pose,
                                                        const float* __restrict__ plog, const float* __restrict__ ap,
                                                        const float* __restrict__ st, const float* __restrict__ gtb,
                                                        const float* __restrict__ gtp, const float* __restrict__ sigmas,
                                                        const int* __restrict__ assigned_gt,
                                                        const float* __restrict__ assigned_score, double* sums,
                                                        float grad_scale, float* gcls, float* greg, float* gpose,
                                                        float* gplog) {
  const int64_t total = (int64_t)d.B * d.L;
  double nrm = sums[3];
  if (nrm < 1.0) nrm = 1.0;
  double npos = sums[6];
  if (npos < 1.0) npos = 1.0;
  const float inv_norm = grad_scale / (float)nrm, inv_pos = grad_scale / (float)npos;
  AnchorSums acc{0.f, 0.f, 0.f, 0.f, 0.f};
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int l = i % d.L, b = i / d.L;
    anchor_loss(d, b, l, cls, reg, pose, plog, ap, st, gtb, gtp, sigmas, assigned_gt[i], assigned_score[i], inv_norm, inv_pos,
                gcls, greg, gpose, gplog, &acc);
  }
  float v[5] = {acc.cls, acc.iou, acc.dfl, acc.pcls, acc.preg};
  __shared__ float sh[5][8];
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    v[k] = warp_sum(v[k]);
    if ((threadIdx.x & 31) == 0) sh[k][threadIdx.x >> 5] = v[k];
  }
  __syncthreads();
  if (threadIdx.x < 5) {
    float s = 0.f;
    for (int q = 0; q < (int)(blockDim.x >> 5); ++q) s += sh[threadIdx.x][q];
    const int slot = threadIdx.x < 3 ? threadIdx.x : threadIdx.x + 1;  // sums[3] is the normaliser
    if (s != 0.f) atomicAdd(&sums[slot], (double)s);
  }
}

__global__ void pose_finalize_kernel(SgbPoseLossDesc d, const double* sums, float* out) { finalize(d, sums, out); }

int check_desc(const SgbPoseLossDesc* d) {
  SGB_REQUIRE(d && d->B > 0 && d->L > 0 && d->J > 0, "bad desc");
  SGB_REQUIRE(d->J <= MAXJ, "at most 64 joints");
  SGB_REQUIRE(d->reg_max + 1 <= MAXBINS, "reg_max + 1 must be <= 32");
  SGB_REQUIRE(d->n_max >= 0 && d->topk > 0 && d->topk <= 64, "n_max / topk");
  SGB_REQUIRE(d->topk <= d->L, "topk must not exceed the number of anchors");  // torch.topk raises there
  SGB_REQUIRE(d->iou_type == 0 || d->iou_type == 1, "iou_type");
  return SGB_OK;
}

}  // namespace

extern "C" int64_t sgb_pose_tal_workspace_bytes(const SgbPoseLossDesc* d) {
  if (!d) return 0;
  return ws_floats(d->B, d->L, d->n_max > 0 ? d->n_max : 1, d->topk) * 4 + 256;
}

extern "C" int sgb_pose_tal_assign(const SgbPoseLossDesc* d, const float* cls_logits, const float* reg_distri,
                                   const float* pose_coords, const float* anchor_points, const float* stride_tensor,
                                   const float* gt_boxes, const float* gt_poses, const uint8_t* gt_crowd,
                                   const uint8_t* gt_valid, const float* sigmas, int32_t* assigned_gt,
                                   float* assigned_score, double* sums, void* workspace, int64_t workspace_bytes,
                                   void* stream) {
  if (int rc = check_desc(d)) return rc;
  // the top-k keeps one gt's metric row of all L anchors in shared memory
  const size_t smem = (size_t)d->L * sizeof(float);
  SGB_REQUIRE(d->n_max == 0 || smem <= 200 * 1024, "too many anchors for the shared-memory metric row");
  SGB_REQUIRE(cls_logits && reg_distri && pose_coords && anchor_points && stride_tensor && sigmas && assigned_gt &&
                  assigned_score && sums && workspace,
              "null pointer");
  SGB_REQUIRE(workspace_bytes >= sgb_pose_tal_workspace_bytes(d), "workspace too small");
  SGB_REQUIRE(d->n_max > 0 ? (gt_boxes && gt_poses && gt_crowd && gt_valid) : true, "gt pointers");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t BL = (int64_t)d->B * d->L;
  const int grid = (int)((BL + 255) / 256 > 132 * 8 ? 132 * 8 : (BL + 255) / 256);
  // no targets in the batch: every anchor is background (:118-131)
  if (d->n_max == 0) return fill_background(assigned_gt, -1, assigned_score, nullptr, BL, st);
  Ws w = ws_carve(workspace, d->B, d->L, d->n_max, d->topk);
  pose_decode_kernel<<<grid, 256, 0, st>>>(*d, reg_distri, anchor_points, stride_tensor, w.pbox);
  SGB_LAUNCH_CHECK("pose_decode_kernel");
  // The opt-in above 48 KB counts the kernel's static shared memory too (its gt pose, sigmas and the top-k's merge
  // slots), so it is set whatever the row size.  It is a per-device setting: set on every call, so every device
  // gets it, and always to the same cap, so concurrent callers never lower it under each other.
  if (int rc = sgb_cuda_check(cudaFuncSetAttribute(pose_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024),
                              "cudaFuncSetAttribute(pose_topk_kernel)"))
    return rc;
  pose_topk_kernel<<<d->B * d->n_max, 256, smem, st>>>(*d, cls_logits, pose_coords, anchor_points, gt_boxes, gt_poses,
                                                       gt_valid, sigmas, w);
  SGB_LAUNCH_CHECK("pose_topk_kernel");
  pose_resolve_kernel<<<grid, 256, 0, st>>>(*d, cls_logits, pose_coords, anchor_points, gt_boxes, gt_poses, gt_valid,
                                            sigmas, w);
  SGB_LAUNCH_CHECK("pose_resolve_kernel");
  pose_finish_kernel<<<grid, 256, 0, st>>>(*d, gt_crowd, w, assigned_gt, assigned_score, sums);
  SGB_LAUNCH_CHECK("pose_finish_kernel");
  return SGB_OK;
}

extern "C" int sgb_pose_loss_fwd_bwd(const SgbPoseLossDesc* d, const float* cls_logits, const float* reg_distri,
                                     const float* pose_coords, const float* pose_logits, const float* anchor_points,
                                     const float* stride_tensor, const float* gt_boxes, const float* gt_poses,
                                     const float* sigmas, const int32_t* assigned_gt, const float* assigned_score,
                                     double* sums, float grad_scale, float* grad_cls, float* grad_reg, float* grad_pose,
                                     float* grad_pose_logits, void* stream) {
  if (int rc = check_desc(d)) return rc;
  SGB_REQUIRE(cls_logits && reg_distri && pose_coords && pose_logits && anchor_points && stride_tensor && sigmas &&
                  assigned_gt && assigned_score && sums,
              "null pointer");
  SGB_REQUIRE(d->n_max > 0 ? (gt_boxes && gt_poses) : true, "gt pointers");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t BL = (int64_t)d->B * d->L;
  // only positive anchors write box / keypoint gradients
  if (grad_reg) cudaMemsetAsync(grad_reg, 0, BL * 4 * (d->reg_max + 1) * sizeof(float), st);
  if (grad_pose) cudaMemsetAsync(grad_pose, 0, BL * d->J * 2 * sizeof(float), st);
  if (grad_pose_logits) cudaMemsetAsync(grad_pose_logits, 0, BL * d->J * sizeof(float), st);
  const int grid = (int)((BL + 255) / 256 > 132 * 8 ? 132 * 8 : (BL + 255) / 256);
  pose_loss_kernel<<<grid, 256, 0, st>>>(*d, cls_logits, reg_distri, pose_coords, pose_logits, anchor_points, stride_tensor,
                                         gt_boxes, gt_poses, sigmas, assigned_gt, assigned_score, sums, grad_scale, grad_cls,
                                         grad_reg, grad_pose, grad_pose_logits);
  SGB_LAUNCH_CHECK("pose_loss_kernel");
  return SGB_OK;
}

extern "C" int sgb_pose_loss_finalize(const SgbPoseLossDesc* d, const double* sums, float* loss_out, void* stream) {
  SGB_REQUIRE(d && sums && loss_out, "null pointer");
  pose_finalize_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(*d, sums, loss_out);
  SGB_LAUNCH_CHECK("pose_finalize_kernel");
  return SGB_OK;
}

// ATSS assigner (row L2's static variant: ppyolo_loss.py:301-434) with the outputs of sgb_tal_assign, so that the fused
// varifocal / IoU / DFL kernel (loss.cu) runs unchanged behind either assigner.  Two launches:
//   atss_candidates_kernel  one CTA per (image, gt): per pyramid level the topk anchors closest to the GT centre (negated distance
//                           row in shared memory, block-wide top-k, ties -> lowest index), IoU threshold = mean + std over the
//                           levels x topk candidates, positives counted / owned per anchor with atomics
//   atss_resolve_kernel     one thread per (image, anchor): 0 / 1 / several claiming GTs -> label, box, IoU(gt, predicted box)
// instead of the reference's [B, n, L] float tensors (IoU, distance, one-hot top-k, masks: ~10 x B*n*L*4 bytes each way).
// Algorithmic traffic: reg_distri read once (B*L*68*4 B) + anchors; everything else is per-GT shared-memory work.
// The arithmetic is in atss_math.cuh and tal_math.cuh (shared with the CPU test build).
#include "atss_math.cuh"
#include "common.cuh"

namespace {

using namespace sgb_tal;
using sgb_atss::Levels;

__global__ void __launch_bounds__(256) atss_candidates_kernel(SgbLossDesc d, Levels lv, const float* __restrict__ anchors,
                                                              const float* __restrict__ gtb, const uint8_t* __restrict__ gtv,
                                                              int* __restrict__ count, int* __restrict__ owner) {
  extern __shared__ float sdist[];  // negated distance row of one level: the nearest anchors are the largest entries
  __shared__ int cand[sgb_atss::kMaxLevels * sgb_atss::kMaxTopk];
  __shared__ float ciou[sgb_atss::kMaxLevels * sgb_atss::kMaxTopk];
  __shared__ float thr_s;
  const int bg = blockIdx.x, b = bg / d.n_max, g = bg - b * d.n_max, t = threadIdx.x;
  if (!gtv[bg]) return;
  const Box gt = load_box(gtb + (int64_t)bg * 4);
  for (int lvl = 0; lvl < lv.n; ++lvl) {
    const int base = lv.start[lvl], num = lv.start[lvl + 1] - base;
    for (int a = t; a < num; a += blockDim.x) sdist[a] = -sgb_atss::center_distance(gt, load_box(anchors + (int64_t)(base + a) * 4));
    __syncthreads();
    block_topk(sdist, num, d.topk, [&](int k, int a) { cand[lvl * d.topk + k] = base + a; });
  }
  const int K = lv.n * d.topk;
  if (t < K) ciou[t] = iou(gt, load_box(anchors + (int64_t)cand[t] * 4), 1e-10f);
  __syncthreads();
  if (t == 0) thr_s = sgb_atss::iou_threshold(ciou, K);
  __syncthreads();
  if (t < K && ciou[t] > thr_s && sgb_atss::center_inside(load_box(anchors + (int64_t)cand[t] * 4), gt)) {
    const int64_t i = (int64_t)b * d.L + cand[t];
    atomicAdd(&count[i], 1);
    atomicMin(&owner[i], g);
  }
}

__global__ void atss_resolve_kernel(SgbLossDesc d, const float* __restrict__ reg, const float* __restrict__ anchors,
                                    const float* __restrict__ ap, const float* __restrict__ st, const float* __restrict__ gtb,
                                    const int* __restrict__ gtl, const int* __restrict__ count, const int* __restrict__ owner,
                                    int* __restrict__ alabel, float* __restrict__ abox, float* __restrict__ ascore, double* sums) {
  const int64_t total = (int64_t)d.B * d.L;
  const int bins = d.reg_max + 1;
  float local = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int l = (int)(i % d.L), b = (int)(i / d.L);
    const float* gts = gtb + (int64_t)b * d.n_max * 4;
    const int c = count[i];
    int ag = -1;
    if (c == 1) ag = owner[i];
    else if (c > 1) ag = sgb_atss::argmax_iou_gt(load_box(anchors + (int64_t)l * 4), gts, d.n_max);
    // the reference gathers gt 0's box for unassigned anchors (argmax of an all-zero column)
    const Box gb = load_box(gts + (ag >= 0 ? ag : 0) * 4);
    store_box(abox + i * 4, gb);
    float sc = 0.f;
    int lab = d.ncls;
    if (ag >= 0) {
      lab = gtl[b * d.n_max + ag];
      sc = iou(gb, decode_box(reg + i * 4 * bins, bins, ap[l * 2], ap[l * 2 + 1], st[l]), 1e-9f);
    }
    alabel[i] = lab;
    ascore[i] = sc;
    local += sc;
  }
  local = warp_sum(local);
  if ((threadIdx.x & 31) == 0 && local != 0.f) atomicAdd(&sums[3], (double)local);
}

__global__ void atss_init_kernel(int* count, int* owner, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    count[i] = 0;
    owner[i] = 0x7fffffff;
  }
}

}  // namespace

extern "C" int64_t sgb_atss_workspace_bytes(const SgbLossDesc* d) {
  if (!d) return 0;
  return (int64_t)d->B * d->L * 2 * (int64_t)sizeof(int) + 256;
}

extern "C" int sgb_atss_assign(const SgbLossDesc* d, const float* reg_distri, const float* anchors, const float* anchor_points,
                               const float* stride_tensor, const int32_t* level_sizes, int32_t n_levels, const float* gt_boxes,
                               const int32_t* gt_labels, const uint8_t* gt_valid, int32_t* assigned_label, float* assigned_box,
                               float* assigned_score, double* sums, void* workspace, int64_t workspace_bytes, void* stream) {
  SGB_REQUIRE(d && reg_distri && anchors && anchor_points && stride_tensor && level_sizes && assigned_label && assigned_box &&
                  assigned_score && sums && workspace,
              "null pointer");
  SGB_REQUIRE(d->B > 0 && d->L > 0 && d->ncls > 0 && d->reg_max > 0 && d->n_max >= 0, "bad loss shape");
  SGB_REQUIRE(n_levels > 0 && n_levels <= sgb_atss::kMaxLevels, "1..8 pyramid levels");
  SGB_REQUIRE(d->topk > 0 && d->topk <= sgb_atss::kMaxTopk, "ATSS topk must be in 1..16");
  SGB_REQUIRE(workspace_bytes >= sgb_atss_workspace_bytes(d), "workspace too small");
  SGB_REQUIRE(d->n_max > 0 ? (gt_boxes && gt_labels && gt_valid) : true, "gt pointers");
  Levels lv;
  lv.n = n_levels;
  int acc = 0, widest = 0;
  for (int i = 0; i < n_levels; ++i) {
    // torch.topk raises when a level holds fewer than topk anchors (ppyolo_loss.py:291)
    SGB_REQUIRE(level_sizes[i] >= d->topk, "every pyramid level needs at least topk anchors");
    lv.start[i] = acc;
    acc += level_sizes[i];
    widest = level_sizes[i] > widest ? level_sizes[i] : widest;
  }
  lv.start[n_levels] = acc;
  SGB_REQUIRE(acc == d->L, "level sizes must add up to the number of anchors");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t BL = (int64_t)d->B * d->L;
  const int grid = (int)((BL + 255) / 256 > 132 * 8 ? 132 * 8 : (BL + 255) / 256);
  int* count = reinterpret_cast<int*>(workspace);
  int* owner = count + BL;
  atss_init_kernel<<<grid, 256, 0, st>>>(count, owner, BL);
  SGB_LAUNCH_CHECK("atss_init_kernel");
  if (d->n_max > 0) {
    const size_t smem = (size_t)widest * sizeof(float);
    SGB_REQUIRE(smem <= 200 * 1024, "pyramid level too large for the shared-memory distance row");
    if (smem > 48 * 1024) cudaFuncSetAttribute(atss_candidates_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    atss_candidates_kernel<<<d->B * d->n_max, 256, smem, st>>>(*d, lv, anchors, gt_boxes, gt_valid, count, owner);
    SGB_LAUNCH_CHECK("atss_candidates_kernel");
  }
  // negative batch (ppyolo_loss.py:352-357): every anchor is background, boxes and scores are zero
  if (d->n_max == 0) return fill_background(assigned_label, d->ncls, assigned_score, assigned_box, BL, st);
  atss_resolve_kernel<<<grid, 256, 0, st>>>(*d, reg_distri, anchors, anchor_points, stride_tensor, gt_boxes, gt_labels, count, owner,
                                            assigned_label, assigned_box, assigned_score, sums);
  SGB_LAUNCH_CHECK("atss_resolve_kernel");
  return SGB_OK;
}

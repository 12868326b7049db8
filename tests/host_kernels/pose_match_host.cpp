// Test infrastructure: serial HOST driver around super_gradients_b200/csrc/pose_match_math.cuh (the arithmetic of the CUDA pose
// matching kernel), compiled with g++ by tests/host_pose_match.py.  Same steps as pose_match_kernel, one image after the other,
// "lanes" collapsed to first = 0 / step = 1; same arguments as sgb_pose_keypoint_matching without the stream.
#include <math.h>

#include <vector>

#include "sgb200.h"
#include "pose_match_math.cuh"

namespace pm = sgb_pose_match;
using sgb_match::Best;

extern "C" int pose_match_host(const float* poses, const float* scores, const int32_t* pred_count, const float* gt_joints, const float* gt_boxes,
                               const float* gt_areas, const uint8_t* gt_flags, const int32_t* gt_count, const float* sigmas, const float* thresholds,
                               int32_t B, int32_t max_preds, int32_t max_targets, int32_t J, int32_t T, int32_t top_k, uint8_t* matched,
                               uint8_t* ignore, float* used_scores, int32_t* used_count, int32_t* n_targets, float* oks_out) {
  if (B <= 0 || max_preds <= 0 || max_targets <= 0 || J <= 0 || T <= 0 || T > SGB_MATCH_MAX_THRESHOLDS || top_k <= 0) return 1;
  const int K = top_k < max_preds ? top_k : max_preds;
  std::vector<float> vars(J);
  for (int j = 0; j < J; ++j) vars[j] = pm::oks_var(sigmas[j]);
  for (int b = 0; b < B; ++b) {
    const int P = pred_count[b] < 0 ? 0 : (pred_count[b] > max_preds ? max_preds : pred_count[b]);
    const int M = gt_count[b] < 0 ? 0 : (gt_count[b] > max_targets ? max_targets : gt_count[b]);
    const int n_used = P < K ? P : K;
    const float* sc = scores + (int64_t)b * max_preds;
    const float* tj = gt_joints + (int64_t)b * max_targets * J * 3;
    std::vector<float> box(4 * M), area(M);
    std::vector<int> k1(M), col;
    for (int t = 0; t < M; ++t) {
      const int64_t g = (int64_t)b * max_targets + t;
      if (gt_flags[g] & pm::FLAG_HAS_BOX) {
        for (int c = 0; c < 4; ++c) box[4 * t + c] = gt_boxes[g * 4 + c];
      } else {
        pm::visible_box_xywh(tj + t * J * 3, J, &box[4 * t]);
      }
      area[t] = (gt_flags[g] & pm::FLAG_HAS_AREA) ? gt_areas[g] : pm::box_area(&box[4 * t]);
      k1[t] = pm::n_visible(tj + t * J * 3, J);
    }
    std::vector<int> order(n_used);
    for (int i = 0; i < P; ++i) {
      int rank = 0;
      for (int j = 0; j < P; ++j) rank += pm::before(sc[j], j, sc[i], i) ? 1 : 0;
      if (rank < n_used) order[rank] = i;
    }
    for (int t = 0; t < M; ++t)
      if (!pm::is_ignored(tj + t * J * 3, J, gt_flags[(int64_t)b * max_targets + t])) col.push_back(t);
    const int n_reg = (int)col.size();
    for (int t = 0; t < M; ++t)
      if (pm::is_ignored(tj + t * J * 3, J, gt_flags[(int64_t)b * max_targets + t])) col.push_back(t);
    std::vector<float> oks((size_t)n_used * M);
    for (int k = 0; k < n_used; ++k)
      for (int c = 0; c < M; ++c) {
        const int t = col[c];
        const float* pxy = poses + ((int64_t)b * max_preds + order[k]) * J * 3;
        oks[(size_t)k * M + c] = pm::oks(pxy, 3, tj + t * J * 3, &box[4 * t], area[t], k1[t], vars.data(), J);
        if (oks_out) oks_out[((int64_t)b * K + k) * max_targets + t] = oks[(size_t)k * M + c];
      }
    uint8_t* mt = matched + (int64_t)b * K * T;
    uint8_t* ig = ignore + (int64_t)b * K * T;
    for (int i = 0; i < K * T; ++i) mt[i] = ig[i] = 0;
    for (int j = 0; j < T; ++j) {
      const float floor = pm::qualify_floor(thresholds[0], thresholds[j]);
      std::vector<uint8_t> taken(M > 0 ? M : 1, 0);
      for (int k = 0; k < n_used && n_reg > 0; ++k) {
        const Best best = pm::best_free_target(&oks[(size_t)k * M], floor, taken.data(), n_reg, 0, 1);
        if (best.t >= 0) {
          taken[best.t] = 1;
          mt[k * T + j] = 1;
        }
      }
    }
    for (int k = 0; k < n_used; ++k) {
      const float best = M > n_reg ? pm::best_crowd_oks(&oks[(size_t)k * M + n_reg], M - n_reg) : -INFINITY;
      for (int j = 0; j < T; ++j) ig[k * T + j] = best > thresholds[j] ? 1 : 0;
    }
    for (int k = 0; k < K; ++k) used_scores[(int64_t)b * K + k] = k < n_used ? sc[order[k]] : 0.f;
    used_count[b] = n_used;
    n_targets[b] = n_reg;
  }
  return 0;
}

// the lane-strided search + merge the kernel performs: 32 "lanes" merged in butterfly order
extern "C" int pose_best_free_target_lanes(const float* oks_row, float floor, const uint8_t* taken, int n_targets, float* out_v) {
  Best lane[32];
  for (int l = 0; l < 32; ++l) lane[l] = pm::best_free_target(oks_row, floor, taken, n_targets, l, 32);
  for (int o = 16; o > 0; o >>= 1) {
    Best next[32];
    for (int l = 0; l < 32; ++l) next[l] = sgb_match::better(lane[l], lane[l ^ o]);
    for (int l = 0; l < 32; ++l) lane[l] = next[l];
  }
  for (int l = 1; l < 32; ++l)
    if (lane[l].t != lane[0].t) return -2;  // every lane must agree after the butterfly
  *out_v = lane[0].v;
  return lane[0].t;
}

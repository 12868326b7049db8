// Test infrastructure: serial HOST driver around the distance matching of super_gradients_b200/csrc/detection_match_math.cuh
// (DetectionMetricsDistanceBased), compiled with g++ by tests/host_distance_match.py.  Same steps as
// detection_match_kernel<DistanceRule>, one image after the other, "lanes" collapsed to first = 0 / step = 1.
#include <vector>

#include "sgb200.h"
#include "detection_match_math.cuh"

using sgb_match::Best;
using sgb_match::Box;
using sgb_match::Point;

extern "C" int distance_match_host(const SgbMatchDesc* d, int metric, const float* preds, const int32_t* pred_count, const float* targets,
                                   const int32_t* target_count, const float* crowd, const int32_t* crowd_count, const float* thresholds,
                                   uint8_t* matched, uint8_t* ignore) {
  const int T = d->n_thresholds;
  for (int b = 0; b < d->B; ++b) {
    const int P = pred_count[b], M = target_count[b], C = d->max_crowd > 0 ? crowd_count[b] : 0;
    if (P < 0 || P > d->max_preds || M < 0 || M > d->max_targets || C < 0 || C > d->max_crowd) return 1;
    const float* pr = preds + (int64_t)b * d->max_preds * 6;
    uint8_t* mt = matched + (int64_t)b * d->max_preds * T;
    uint8_t* ig = ignore + (int64_t)b * d->max_preds * T;
    std::vector<Box> pbox(P), tbox(M), cbox(C);
    std::vector<float> pscore(P), pcls(P), tcls(M), ccls(C);
    for (int i = 0; i < P; ++i) {
      const float* r = pr + i * 6;
      pbox[i] = sgb_match::clip_box(Box{r[0], r[1], r[2], r[3]}, d->height, d->width);
      pscore[i] = r[4];
      pcls[i] = r[5];
    }
    for (int i = 0; i < M; ++i) {
      const float* r = targets + ((int64_t)b * d->max_targets + i) * 5;
      tbox[i] = sgb_match::target_xyxy(r[1], r[2], r[3], r[4], d->denormalize_targets != 0, d->height, d->width);
      tcls[i] = r[0];
    }
    for (int i = 0; i < C; ++i) {
      const float* r = crowd + ((int64_t)b * d->max_crowd + i) * 5;
      cbox[i] = sgb_match::target_xyxy(r[1], r[2], r[3], r[4], d->denormalize_targets != 0, d->height, d->width);
      ccls[i] = r[0];
    }
    std::vector<uint8_t> used(P);
    for (int i = 0; i < P; ++i) {
      int rank = 0;
      for (int j = 0; j < P; ++j) rank += (pcls[j] == pcls[i] && sgb_match::before(pscore[j], j, pscore[i], i)) ? 1 : 0;
      used[i] = (rank < d->top_k && pscore[i] != 0.f) ? 1 : 0;
    }
    std::vector<int> order(P);
    int n_used = 0;
    for (int i = 0; i < P; ++i) {
      if (used[i]) {
        int pos = 0;
        for (int j = 0; j < P; ++j) pos += (used[j] && sgb_match::before(pscore[j], j, pscore[i], i)) ? 1 : 0;
        order[pos] = i;
        ++n_used;
      }
      for (int j = 0; j < T; ++j) {
        mt[i * T + j] = 0;
        ig[i * T + j] = used[i] ? 0 : 1;
      }
    }
    for (int i = P * T; i < d->max_preds * T; ++i) mt[i] = ig[i] = 0;
    if (M > 0)
      for (int j = 0; j < T; ++j) {
        std::vector<uint8_t> taken(M, 0);
        for (int k = 0; k < n_used; ++k) {
          const int p = order[k];
          const Best best = sgb_match::nearest_free_target(metric, sgb_match::centre(pbox[p]), pcls[p], thresholds[j], tbox.data(), tcls.data(), taken.data(), M, 0, 1);
          if (best.t >= 0) {
            taken[best.t] = 1;
            mt[p * T + j] = 1;
          }
        }
      }
    if (C > 0)
      for (int k = 0; k < n_used; ++k) {
        const int p = order[k];
        const float best = sgb_match::nearest_crowd_distance(metric, sgb_match::centre(pbox[p]), pcls[p], cbox.data(), ccls.data(), C);
        for (int j = 0; j < T; ++j)
          if (best < thresholds[j]) ig[p * T + j] = 1;
      }
  }
  return 0;
}

// the lane-strided search + nearer() butterfly the kernel performs: 32 "lanes" merged in butterfly order
extern "C" int nearest_free_target_lanes(int metric, const float* pbox4, float cls_p, float thr, const float* tbox4, const float* tcls, const uint8_t* taken,
                                         int n_targets, float* out_v) {
  const Point p = sgb_match::centre(Box{pbox4[0], pbox4[1], pbox4[2], pbox4[3]});
  std::vector<Box> tb(n_targets);
  for (int t = 0; t < n_targets; ++t) tb[t] = Box{tbox4[4 * t], tbox4[4 * t + 1], tbox4[4 * t + 2], tbox4[4 * t + 3]};
  Best lane[32];
  for (int l = 0; l < 32; ++l) lane[l] = sgb_match::nearest_free_target(metric, p, cls_p, thr, tb.data(), tcls, taken, n_targets, l, 32);
  for (int o = 16; o > 0; o >>= 1) {
    Best next[32];
    for (int l = 0; l < 32; ++l) next[l] = sgb_match::nearer(lane[l], lane[l ^ o]);
    for (int l = 0; l < 32; ++l) lane[l] = next[l];
  }
  for (int l = 1; l < 32; ++l)
    if (lane[l].t != lane[0].t) return -2;  // every lane must agree after the butterfly
  *out_v = lane[0].v;
  return lane[0].t;
}

// Serial host build of the sliding-window merge NMS (super_gradients_b200/csrc/sliding_window.cu) over the product's arithmetic header
// nms_math.cuh: the same sort key, the same trick / per-class selection, and the same blocked greedy schedule (each block of NB
// candidates of a class tested against the class's kept list, then resolved within itself).  Built with -ffp-contract=off.
#include <algorithm>
#include <math.h>
#include <stdint.h>
#include <vector>

#include "nms_math.cuh"

static const int NB = 64;

// boxes [n, 4] (canvas pixels, list order), scores [n], labels [n] (integral) -> keep [n] list indices in output order; returns
// the number kept
extern "C" int merge_nms_host(const float* boxes, const float* scores, const int* labels, int n, double iou_thr, int64_t* keep) {
  if (n == 0) return 0;
  std::vector<uint64_t> keys(n);
  for (int j = 0; j < n; ++j) keys[j] = sgb_nms::sort_key(scores[j], (uint32_t)j);
  std::sort(keys.begin(), keys.end());
  const bool trick = 4 * (int64_t)n <= 4000;
  float m = -INFINITY;
  for (int j = 0; j < 4 * n; ++j) m = sgb_nms::max_nan(m, boxes[j]);
  const float step = sgb_nms::offset_step(m);
  std::vector<float> bx(4 * n), area(n);
  std::vector<int> lab(n), pos(n);
  for (int i = 0; i < n; ++i) {
    const int p = (int)(keys[i] & 0xffffffffu);
    pos[i] = p;
    lab[i] = labels[p];
    const float off = trick ? sgb_nms::label_offset(labels[p], step) : 0.f;
    for (int c = 0; c < 4; ++c) bx[4 * i + c] = trick ? sgb_nms::add_rn(boxes[4 * p + c], off) : boxes[4 * p + c];
    area[i] = sgb_nms::area(bx[4 * i], bx[4 * i + 1], bx[4 * i + 2], bx[4 * i + 3]);
  }
  std::vector<char> kept(n, 0);
  int lmax = 0;
  for (int i = 0; i < n; ++i) lmax = std::max(lmax, lab[i] + 1);
  for (int c = 0; c < (trick ? 1 : lmax); ++c) {
    std::vector<int> cand, klist;
    for (int i = 0; i < n; ++i)
      if (trick || lab[i] == c) cand.push_back(i);
    for (size_t s0 = 0; s0 < cand.size(); s0 += NB) {
      const int ns = (int)std::min<size_t>(NB, cand.size() - s0);
      uint64_t mask[NB] = {0};
      bool sup[NB] = {false};
      for (int r = 0; r < ns; ++r) {
        const float* b = &bx[4 * cand[s0 + r]];
        const float a = area[cand[s0 + r]];
        for (int k : klist)
          if (sgb_nms::suppresses(bx[4 * k], bx[4 * k + 1], bx[4 * k + 2], bx[4 * k + 3], area[k], b[0], b[1], b[2], b[3], a, iou_thr)) {
            sup[r] = true;
            break;
          }
        for (int q = r + 1; q < ns; ++q) {
          const float* e = &bx[4 * cand[s0 + q]];
          if (sgb_nms::suppresses(b[0], b[1], b[2], b[3], a, e[0], e[1], e[2], e[3], area[cand[s0 + q]], iou_thr)) mask[r] |= 1ull << q;
        }
      }
      uint64_t remv = 0;
      for (int r = 0; r < ns; ++r) {
        if (sup[r] || ((remv >> r) & 1ull)) continue;
        remv |= mask[r];
        klist.push_back(cand[s0 + r]);
        kept[cand[s0 + r]] = 1;
      }
    }
  }
  int nk = 0;
  for (int i = 0; i < n; ++i)
    if (kept[i]) keep[nk++] = pos[i];
  return nk;
}

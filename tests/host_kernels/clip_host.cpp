// Serial host driver around the clip_grad_norm arithmetic of super_gradients_b200/csrc/optim_math.cuh (compiled with g++
// -ffp-contract=off by tests/host_clip.py): sgb_clip_grad_norm as its two kernels compute it.  The per-chunk sums run serially in
// double, where the device reduces each chunk as a tree; both then add the chunk sums in double.
#include <stdint.h>

#include "optim_math.cuh"

using namespace sgb_optim;

extern "C" {

float clip_total_norm_host(double grad_sqsum) { return clip_total_norm(grad_sqsum); }

float clip_coef_host(float total, float max_norm) { return clip_coef(total, max_norm); }

// chunks[c] = {start, len, first chunk of its tensor, chunks of its tensor}; hp = two hp_len-wide rows
void clip_grad_norm_host(const float* g, const int64_t* chunks, int32_t nchunk, float* hp, int32_t hp_len, int32_t gs_col, float max_norm, double* partials,
                         float* norm_coef) {
  for (int32_t c = 0; c < nchunk; ++c) {
    double s = 0.0;
    for (int64_t i = chunks[4 * c]; i < chunks[4 * c] + chunks[4 * c + 1]; ++i) {
      const double x = mul(g[i], hp[gs_col]);
      s += x * x;
    }
    partials[c] = s;
  }
  double total = 0.0;
  for (int32_t c = 0; c < nchunk; ++c) total += partials[c];
  norm_coef[0] = clip_total_norm(total);
  norm_coef[1] = clip_coef(norm_coef[0], max_norm);
  clip_scale_rows(hp, hp_len, gs_col, norm_coef[1]);
}
}

// Serial host driver around super_gradients_b200/csrc/optim_math.cuh (compiled with g++ -ffp-contract=off by tests/host_optim.py):
// the flat-buffer optimizer steps exactly as the CUDA kernels compute each element.  The Lamb sums run serially in double per
// chunk of the chunk table, where the device reduces each chunk as a tree; both then add the chunk sums in double.
#include <stdint.h>

#include "optim_math.cuh"

using namespace sgb_optim;

extern "C" {

void adam_host(float* p, const float* g, float* m, float* v, int64_t n, const float* hp) {
  for (int64_t i = 0; i < n; ++i) adam(p[i], g[i], m[i], v[i], hp);
}

void rmsprop_host(float* p, const float* g, float* sa, float* buf, float* ga, int64_t n, const float* hp) {
  for (int64_t i = 0; i < n; ++i) rmsprop(p[i], g[i], sa[i], buf ? buf + i : nullptr, ga ? ga + i : nullptr, hp);
}

void rmsprop_tf_host(float* p, const float* g, float* sa, float* buf, float* ga, int64_t n, const float* hp) {
  for (int64_t i = 0; i < n; ++i) rmsprop_tf(p[i], g[i], sa[i], buf ? buf + i : nullptr, ga ? ga + i : nullptr, hp);
}

void lion_host(float* p, const float* g, float* m, int64_t n, const float* hp) {
  for (int64_t i = 0; i < n; ++i) lion(p[i], g[i], m[i], hp);
}

// chunks[c] = {start, len, first chunk of its tensor, chunks of its tensor}; hp = two LAMB_HP rows (row 1 from n_decay on)
void lamb_grad_sqnorm_host(const float* g, const int64_t* chunks, int32_t nchunk, const float* hp, double* partials) {
  for (int32_t c = 0; c < nchunk; ++c) {
    double s = 0.0;
    for (int64_t i = chunks[4 * c]; i < chunks[4 * c] + chunks[4 * c + 1]; ++i) {
      const double x = mul(g[i], hp[LAMB_GS]);
      s += x * x;
    }
    partials[c] = s;
  }
}

void lamb_step_host(float* p, const float* g, float* m, float* v, float* u, int64_t n_decay, const int64_t* chunks, int32_t nchunk,
                    const float* hp, double* partials) {
  double total = 0.0;
  for (int32_t c = 0; c < nchunk; ++c) total += partials[c];
  double* pu = partials + nchunk;
  for (int32_t c = 0; c < nchunk; ++c) {
    const int64_t a = chunks[4 * c], b = a + chunks[4 * c + 1];
    const float* row = hp + (a < n_decay ? 0 : LAMB_HP);
    const float clip = lamb_clip(total, row);
    double sp = 0.0, su = 0.0;
    for (int64_t i = a; i < b; ++i) {
      u[i] = lamb_update(p[i], g[i], m[i], v[i], clip, row);
      sp += (double)p[i] * p[i];
      su += (double)u[i] * u[i];
    }
    pu[2 * c] = sp;
    pu[2 * c + 1] = su;
  }
  for (int32_t c = 0; c < nchunk; ++c) {
    const int64_t a = chunks[4 * c], b = a + chunks[4 * c + 1];
    const float* row = hp + (a < n_decay ? 0 : LAMB_HP);
    double sp = 0.0, su = 0.0;
    for (int64_t k = chunks[4 * c + 2]; k < chunks[4 * c + 2] + chunks[4 * c + 3]; ++k) {
      sp += pu[2 * k];
      su += pu[2 * k + 1];
    }
    const float t = lamb_trust(sp, su, row);
    for (int64_t i = a; i < b; ++i) p[i] = lamb_apply(p[i], u[i], t, row);
  }
}
}

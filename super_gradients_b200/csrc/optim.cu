// SGD, AdamW, Adam, RMSprop, RMSpropTF, Lion and Lamb over the flat fp32 parameter / gradient buffers (training/flat_state.py),
// and the EMA update.  Hyper-parameters are read from DEVICE memory, one row per weight-decay range in the layouts of
// optim_math.cuh, so a CUDA-graph-captured step follows the host's schedule.  The per-element arithmetic of Adam, RMSprop,
// RMSpropTF, Lion and Lamb is optim_math.cuh's; sgd_kernel, adamw_kernel and ema_kernel spell theirs with plain operators, which
// nvcc contracts into FMAs (g * gs + wd * p is one).  The elementwise optimizers are one grid-stride pass per weight-decay range.
//
// Lamb needs a global gradient norm and per-tensor norms of p and of the update.  Every reduction runs over a chunk table
// (fused_optimizers.lamb_chunk_table: {start, len, first chunk of its tensor, chunks of its tensor}; a chunk lies inside one
// tensor), one CTA per chunk, in float64, in a fixed order (thread-strided partial sums, then a fixed shuffle / shared-memory
// tree), and without atomics, so two runs of one step are bit-identical:
//   1. grad_sqnorm_kernel   partials[c]             = sum over chunk c of (g * gs)^2
//   2. lamb_update_kernel   every CTA adds partials[0 .. nchunk) itself -> clip; m / v update -> update buffer;
//                           partials[nchunk + 2c .. +1] = sum over chunk c of p^2 and update^2
//   3. lamb_apply_kernel    every CTA adds its tensor's chunk sums -> trust ratio; p -= lr * trust * update
// clip_grad_norm runs grad_sqnorm_kernel over the same table with any optimizer's grad_scale column, then clip_finalize_kernel
// multiplies the coefficient into that column, before the optimizer's own launches.
#include "common.cuh"
#include "optim_math.cuh"

namespace {

using namespace sgb_optim;

constexpr int TPB = 256;

inline int grid_for(int64_t work, int per_cta = TPB * 4, int max_ctas = 132 * 8) {
  int64_t g = (work + per_cta - 1) / per_cta;
  if (g > max_ctas) g = max_ctas;
  if (g < 1) g = 1;
  return (int)g;
}

__global__ void sgd_kernel(float* p, const float* g, float* mom, int64_t n, const float* hp) {
  const float lr = hp[SGD_LR], mu = hp[SGD_MOMENTUM], wd = hp[SGD_WD], gs = hp[SGD_GS];
  const bool nesterov = hp[SGD_NESTEROV] != 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float gr = g[i] * gs + wd * p[i];
    float d = gr;
    if (mu != 0.f) {
      float b = mu * mom[i] + gr;
      mom[i] = b;
      d = nesterov ? gr + mu * b : b;
    }
    p[i] -= lr * d;
  }
}
__global__ void adamw_kernel(float* p, const float* g, float* m, float* v, int64_t n, const float* hp) {
  const float lr = hp[ADAMW_LR], b1 = hp[ADAMW_B1], b2 = hp[ADAMW_B2], eps = hp[ADAMW_EPS], wd = hp[ADAMW_WD], bc1 = hp[ADAMW_BC1], bc2 = hp[ADAMW_BC2],
              gs = hp[ADAMW_GS];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float gr = g[i] * gs;
    float pi = p[i] * (1.f - lr * wd);
    float mi = b1 * m[i] + (1.f - b1) * gr;
    float vi = b2 * v[i] + (1.f - b2) * gr * gr;
    m[i] = mi;
    v[i] = vi;
    float denom = sqrtf(vi) / sqrtf(bc2) + eps;
    p[i] = pi - (lr / bc1) * mi / denom;
  }
}
__global__ void ema_kernel(float* e, const float* p, int64_t n, const float* decay) {
  const float d = *decay;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    e[i] = e[i] * d + (1.f - d) * p[i];
}

__global__ void __launch_bounds__(TPB) adam_kernel(float* p, const float* g, float* m, float* v, int64_t n, const float* hp) {
  float h[ADAM_HP];
#pragma unroll
  for (int j = 0; j < ADAM_HP; ++j) h[j] = hp[j];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float pi = p[i], mi = m[i], vi = v[i];
    adam(pi, g[i], mi, vi, h);
    p[i] = pi;
    m[i] = mi;
    v[i] = vi;
  }
}

// TF: RMSpropTF when true, torch.optim.RMSprop otherwise; buf / ga may be null (no momentum / not centered)
template <bool TF>
__global__ void __launch_bounds__(TPB) rmsprop_kernel(float* p, const float* g, float* sa, float* buf, float* ga, int64_t n, const float* hp) {
  float h[RMS_HP];
#pragma unroll
  for (int j = 0; j < RMS_HP; ++j) h[j] = hp[j];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float pi = p[i], si = sa[i], bi = buf ? buf[i] : 0.f, gi = ga ? ga[i] : 0.f;
    if (TF) rmsprop_tf(pi, g[i], si, &bi, &gi, h);
    else rmsprop(pi, g[i], si, &bi, &gi, h);
    p[i] = pi;
    sa[i] = si;
    if (buf) buf[i] = bi;
    if (ga) ga[i] = gi;
  }
}

__global__ void __launch_bounds__(TPB) lion_kernel(float* p, const float* g, float* m, int64_t n, const float* hp) {
  float h[LION_HP];
#pragma unroll
  for (int j = 0; j < LION_HP; ++j) h[j] = hp[j];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float pi = p[i], mi = m[i];
    lion(pi, g[i], mi, h);
    p[i] = pi;
    m[i] = mi;
  }
}

// block-wide sum of two doubles in a fixed order; the result is valid in every thread
__device__ __forceinline__ double2 block_sum2(double a, double b) {
  __shared__ double2 part[TPB / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_down_sync(0xffffffffu, a, o);
    b += __shfl_down_sync(0xffffffffu, b, o);
  }
  const int w = threadIdx.x >> 5;
  __syncthreads();  // part[] may still be read by a previous call
  if ((threadIdx.x & 31) == 0) part[w] = make_double2(a, b);
  __syncthreads();
  double2 s = part[0];
#pragma unroll
  for (int k = 1; k < TPB / 32; ++k) {
    s.x += part[k].x;
    s.y += part[k].y;
  }
  return s;
}

// partials[c] = sum over chunk c of (g * *gs)^2; gs points at the grad_scale column of the optimizer's row 0 (Lamb's global norm
// and clip_grad_norm's total norm)
__global__ void __launch_bounds__(TPB) grad_sqnorm_kernel(const float* __restrict__ g, const int64_t* __restrict__ chunks, const float* __restrict__ gs_ptr,
                                                          double* __restrict__ partials) {
  const int64_t a = chunks[4 * blockIdx.x], b = a + chunks[4 * blockIdx.x + 1];
  const float gs = *gs_ptr;
  double s = 0.0;
  for (int64_t i = a + threadIdx.x; i < b; i += TPB) {
    const double x = mul(g[i], gs);
    s += x * x;
  }
  const double2 t = block_sum2(s, 0.0);
  if (threadIdx.x == 0) partials[blockIdx.x] = t.x;
}

// one CTA: adds partials[0 .. nchunk) in the order lamb_update_kernel uses -> total norm and clip coefficient (norm_coef[0], [1]);
// the coefficient is multiplied into the grad_scale column of both rows, so every optimizer kernel reads clipped gradients
__global__ void __launch_bounds__(TPB) clip_finalize_kernel(const double* __restrict__ partials, int32_t nchunk, float* __restrict__ hp, int32_t hp_len,
                                                            int32_t gs_col, float max_norm, float* __restrict__ norm_coef) {
  double s = 0.0;
  for (int c = threadIdx.x; c < nchunk; c += TPB) s += partials[c];
  const double total = block_sum2(s, 0.0).x;
  if (threadIdx.x == 0) {
    const float norm = clip_total_norm(total), coef = clip_coef(norm, max_norm);
    norm_coef[0] = norm;
    norm_coef[1] = coef;
    clip_scale_rows(hp, hp_len, gs_col, coef);
  }
}

__global__ void __launch_bounds__(TPB) lamb_update_kernel(const float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                                          float* __restrict__ u, int64_t n_decay, const int64_t* __restrict__ chunks, int32_t nchunk,
                                                          const float* __restrict__ hp, double* __restrict__ partials) {
  double s = 0.0;
  for (int c = threadIdx.x; c < nchunk; c += TPB) s += partials[c];
  const double total = block_sum2(s, 0.0).x;
  const int64_t a = chunks[4 * blockIdx.x], b = a + chunks[4 * blockIdx.x + 1];
  const float* row = hp + (a < n_decay ? 0 : LAMB_HP);
  float h[LAMB_HP];
#pragma unroll
  for (int j = 0; j < LAMB_HP; ++j) h[j] = row[j];
  const float clip = lamb_clip(total, h);
  double sp = 0.0, su = 0.0;
  for (int64_t i = a + threadIdx.x; i < b; i += TPB) {
    float mi = m[i], vi = v[i];
    const float pi = p[i];
    const float ui = lamb_update(pi, g[i], mi, vi, clip, h);
    m[i] = mi;
    v[i] = vi;
    u[i] = ui;
    sp += (double)pi * pi;
    su += (double)ui * ui;
  }
  const double2 t = block_sum2(sp, su);
  if (threadIdx.x == 0) {
    partials[nchunk + 2 * blockIdx.x] = t.x;
    partials[nchunk + 2 * blockIdx.x + 1] = t.y;
  }
}

__global__ void __launch_bounds__(TPB) lamb_apply_kernel(float* __restrict__ p, const float* __restrict__ u, int64_t n_decay, const int64_t* __restrict__ chunks,
                                                         int32_t nchunk, const float* __restrict__ hp, const double* __restrict__ partials) {
  const int64_t a = chunks[4 * blockIdx.x], b = a + chunks[4 * blockIdx.x + 1];
  const int64_t first = chunks[4 * blockIdx.x + 2], cnt = chunks[4 * blockIdx.x + 3];
  const double* pu = partials + nchunk;
  double sp = 0.0, su = 0.0;
  for (int64_t k = first + threadIdx.x; k < first + cnt; k += TPB) {
    sp += pu[2 * k];
    su += pu[2 * k + 1];
  }
  const double2 t = block_sum2(sp, su);
  const float* row = hp + (a < n_decay ? 0 : LAMB_HP);
  float h[LAMB_HP];
#pragma unroll
  for (int j = 0; j < LAMB_HP; ++j) h[j] = row[j];
  const float trust = lamb_trust(t.x, t.y, h);
  for (int64_t i = a + threadIdx.x; i < b; i += TPB) p[i] = lamb_apply(p[i], u[i], trust, h);
}

}  // namespace

// ================================================================================================== C ABI
extern "C" int sgb_sgd_step(float* p, const float* g, float* mom, int64_t n, const float* hp, void* stream) {
  SGB_REQUIRE(p && g && mom && hp, "null pointer");
  sgd_kernel<<<grid_for(n, TPB * 4), TPB, 0, (cudaStream_t)stream>>>(p, g, mom, n, hp);
  SGB_LAUNCH_CHECK("sgd_kernel");
  return SGB_OK;
}
extern "C" int sgb_adamw_step(float* p, const float* g, float* m, float* v, int64_t n, const float* hp, void* stream) {
  SGB_REQUIRE(p && g && m && v && hp, "null pointer");
  adamw_kernel<<<grid_for(n, TPB * 4), TPB, 0, (cudaStream_t)stream>>>(p, g, m, v, n, hp);
  SGB_LAUNCH_CHECK("adamw_kernel");
  return SGB_OK;
}
extern "C" int sgb_ema_update(float* ema, const float* p, int64_t n, const float* decay, void* stream) {
  SGB_REQUIRE(ema && p && decay, "null pointer");
  ema_kernel<<<grid_for(n, TPB * 4), TPB, 0, (cudaStream_t)stream>>>(ema, p, n, decay);
  SGB_LAUNCH_CHECK("ema_kernel");
  return SGB_OK;
}

extern "C" int sgb_adam_step(float* p, const float* g, float* m, float* v, int64_t n, const float* hp, void* stream) {
  SGB_REQUIRE(p && g && m && v && hp, "null pointer");
  SGB_REQUIRE(n >= 0, "n must be >= 0");
  if (n == 0) return SGB_OK;
  adam_kernel<<<grid_for(n), TPB, 0, (cudaStream_t)stream>>>(p, g, m, v, n, hp);
  SGB_LAUNCH_CHECK("adam_kernel");
  return SGB_OK;
}

extern "C" int sgb_rmsprop_step(float* p, const float* g, float* square_avg, float* momentum_buffer, float* grad_avg, int64_t n, const float* hp, void* stream) {
  SGB_REQUIRE(p && g && square_avg && hp, "null pointer");
  SGB_REQUIRE(n >= 0, "n must be >= 0");
  if (n == 0) return SGB_OK;
  rmsprop_kernel<false><<<grid_for(n), TPB, 0, (cudaStream_t)stream>>>(p, g, square_avg, momentum_buffer, grad_avg, n, hp);
  SGB_LAUNCH_CHECK("rmsprop_kernel");
  return SGB_OK;
}

extern "C" int sgb_rmsprop_tf_step(float* p, const float* g, float* square_avg, float* momentum_buffer, float* grad_avg, int64_t n, const float* hp, void* stream) {
  SGB_REQUIRE(p && g && square_avg && hp, "null pointer");
  SGB_REQUIRE(n >= 0, "n must be >= 0");
  if (n == 0) return SGB_OK;
  rmsprop_kernel<true><<<grid_for(n), TPB, 0, (cudaStream_t)stream>>>(p, g, square_avg, momentum_buffer, grad_avg, n, hp);
  SGB_LAUNCH_CHECK("rmsprop_tf_kernel");
  return SGB_OK;
}

extern "C" int sgb_lion_step(float* p, const float* g, float* m, int64_t n, const float* hp, void* stream) {
  SGB_REQUIRE(p && g && m && hp, "null pointer");
  SGB_REQUIRE(n >= 0, "n must be >= 0");
  if (n == 0) return SGB_OK;
  lion_kernel<<<grid_for(n), TPB, 0, (cudaStream_t)stream>>>(p, g, m, n, hp);
  SGB_LAUNCH_CHECK("lion_kernel");
  return SGB_OK;
}

extern "C" int sgb_lamb_grad_sqnorm(const float* g, const int64_t* chunks, int32_t nchunk, const float* hp, double* partials, void* stream) {
  SGB_REQUIRE(g && chunks && hp && partials, "null pointer");
  SGB_REQUIRE(nchunk >= 1, "nchunk must be >= 1");
  grad_sqnorm_kernel<<<nchunk, TPB, 0, (cudaStream_t)stream>>>(g, chunks, hp + LAMB_GS, partials);
  SGB_LAUNCH_CHECK("grad_sqnorm_kernel");
  return SGB_OK;
}

extern "C" int sgb_clip_grad_norm(const float* g, const int64_t* chunks, int32_t nchunk, float* hp, int32_t hp_len, int32_t gs_col, float max_norm, double* partials,
                                  float* norm_coef, void* stream) {
  SGB_REQUIRE(g && chunks && hp && partials && norm_coef, "null pointer");
  SGB_REQUIRE(nchunk >= 1, "nchunk must be >= 1");
  SGB_REQUIRE(gs_col >= 0 && gs_col < hp_len, "gs_col must index a column of the hp_len-wide rows");
  SGB_REQUIRE(max_norm > 0.f, "max_norm must be > 0");
  grad_sqnorm_kernel<<<nchunk, TPB, 0, (cudaStream_t)stream>>>(g, chunks, hp + gs_col, partials);
  SGB_LAUNCH_CHECK("grad_sqnorm_kernel");
  clip_finalize_kernel<<<1, TPB, 0, (cudaStream_t)stream>>>(partials, nchunk, hp, hp_len, gs_col, max_norm, norm_coef);
  SGB_LAUNCH_CHECK("clip_finalize_kernel");
  return SGB_OK;
}

extern "C" int sgb_lamb_step(float* p, const float* g, float* m, float* v, float* update, int64_t n_decay, const int64_t* chunks, int32_t nchunk, const float* hp,
                             double* partials, void* stream) {
  SGB_REQUIRE(p && g && m && v && update && chunks && hp && partials, "null pointer");
  SGB_REQUIRE(nchunk >= 1 && n_decay >= 0, "nchunk must be >= 1 and n_decay >= 0");
  lamb_update_kernel<<<nchunk, TPB, 0, (cudaStream_t)stream>>>(p, g, m, v, update, n_decay, chunks, nchunk, hp, partials);
  SGB_LAUNCH_CHECK("lamb_update_kernel");
  lamb_apply_kernel<<<nchunk, TPB, 0, (cudaStream_t)stream>>>(p, update, n_decay, chunks, nchunk, hp, partials);
  SGB_LAUNCH_CHECK("lamb_apply_kernel");
  return SGB_OK;
}

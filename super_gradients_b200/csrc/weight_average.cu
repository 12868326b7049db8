// Best-snapshot average of Trainer.train(average_best_models=True): one HBM-bound pass that reads every element of the k occupied
// snapshot slots once and writes the average once (k * n * 4 bytes read, n * 4 written).  The per-element arithmetic is
// weight_average_math.cuh.
#include "common.cuh"
#include "weight_average_math.cuh"

namespace {

constexpr int TPB = 256;

// float4 loads when out and every slot are 16-byte aligned (the slot pointers live in device memory, so each CTA checks them), the
// n % 4 tail and any misaligned call element by element
__global__ void __launch_bounds__(TPB) average_snapshots_kernel(const float* const* slots, int32_t k, int64_t n, float* __restrict__ out) {
  __shared__ const float* s[SGB_AVG_MAX_SLOTS];
  __shared__ int misaligned;
  if (threadIdx.x == 0) misaligned = (int)(reinterpret_cast<uintptr_t>(out) & 15);
  __syncthreads();
  for (int j = threadIdx.x; j < k; j += blockDim.x) {
    s[j] = slots[j];
    if (reinterpret_cast<uintptr_t>(s[j]) & 15) atomicOr(&misaligned, 1);
  }
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t done = 0;
  if (!misaligned) {
    const int64_t n4 = n >> 2;
    for (int64_t v = t; v < n4; v += stride) {
      float4 a = __ldcs(reinterpret_cast<const float4*>(s[0]) + v);
#pragma unroll 4
      for (int j = 1; j < k; ++j) {
        const float4 b = __ldcs(reinterpret_cast<const float4*>(s[j]) + v);
        a.x = sgb_avg::step(a.x, b.x, j);
        a.y = sgb_avg::step(a.y, b.y, j);
        a.z = sgb_avg::step(a.z, b.z, j);
        a.w = sgb_avg::step(a.w, b.w, j);
      }
      __stcs(reinterpret_cast<float4*>(out) + v, a);
    }
    done = n4 << 2;
  }
  for (int64_t i = done + t; i < n; i += stride) out[i] = sgb_avg::average(s, k, i);
}

}  // namespace

extern "C" int sgb_average_snapshots(const float* const* slots, int32_t k, int64_t n, float* out, void* stream) {
  SGB_REQUIRE(slots && out, "null pointer");
  SGB_REQUIRE(k >= 1 && k <= SGB_AVG_MAX_SLOTS, "k must be in [1, SGB_AVG_MAX_SLOTS]");
  SGB_REQUIRE(n >= 0, "n must be >= 0");
  if (n == 0) return SGB_OK;
  const int64_t work = (n + 3) / 4;
  const int grid = (int)(work < (int64_t)132 * 16 * TPB ? (work + TPB - 1) / TPB : 132 * 16);
  average_snapshots_kernel<<<grid, TPB, 0, (cudaStream_t)stream>>>(slots, k, n, out);
  SGB_LAUNCH_CHECK("average_snapshots_kernel");
  return SGB_OK;
}

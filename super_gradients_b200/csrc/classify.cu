// Row-wise classification decode: one warp per logits row, one pass over the row (arithmetic in classify_math.cuh).  Produces
// the top-1 index, top-k membership of the target and the softmax maximum; Accuracy / Top5 accumulate their counters on the
// device (no host synchronisation per batch) and predict() reads label + confidence of a whole batch with one copy.
#include "classify_math.cuh"
#include "common.cuh"

namespace {

constexpr int kWarps = 8;

struct Rows {
  int64_t N;
  int C, k;
  int64_t row_stride, target_stride;
  int logits_bf16, target_bf16;
};

__device__ __forceinline__ float load(const void* p, int bf, int64_t i) {
  return bf ? __bfloat162float(((const bf16*)p)[i]) : ((const float*)p)[i];
}

__device__ __forceinline__ sgb_cls::Lane shfl_lane(const sgb_cls::Lane& l, int o) {
  sgb_cls::Lane r;
  r.best = __shfl_xor_sync(0xffffffffu, l.best, o);
  r.best_i = __shfl_xor_sync(0xffffffffu, l.best_i, o);
  r.above = __shfl_xor_sync(0xffffffffu, l.above, o);
  r.m = __shfl_xor_sync(0xffffffffu, l.m, o);
  r.s = __shfl_xor_sync(0xffffffffu, l.s, o);
  return r;
}

__global__ void __launch_bounds__(kWarps * 32) classify_rows_kernel(const Rows d, const void* __restrict__ logits,
                                                                    const int64_t* __restrict__ target, const void* __restrict__ soft,
                                                                    unsigned long long* __restrict__ counters, int32_t* __restrict__ label,
                                                                    float* __restrict__ confidence) {
  __shared__ unsigned long long block_counts[4];
  if (threadIdx.x < 4) block_counts[threadIdx.x] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (row < d.N) {
    int64_t t = -1;
    if (target) {
      t = target[row];
    } else if (soft) {  // argmax of the soft-label row: the same ranking, first maximum
      float bv = 0.f;
      int bi = -1;
      for (int j = lane; j < d.C; j += 32) {
        const float x = load(soft, d.target_bf16, row * d.target_stride + j);
        if (bi < 0 || sgb_cls::before(x, j, bv, bi)) bv = x, bi = j;
      }
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (oi >= 0 && (bi < 0 || sgb_cls::before(ov, oi, bv, bi))) bv = ov, bi = oi;
      }
      t = bi;
    }
    const bool valid = t >= 0 && t < d.C;
    const int ti = valid ? (int)t : -1;
    const float xt = valid ? load(logits, d.logits_bf16, row * d.row_stride + ti) : 0.f;
    sgb_cls::Lane l = sgb_cls::lane_init();
    for (int j = lane; j < d.C; j += 32) sgb_cls::lane_update(l, load(logits, d.logits_bf16, row * d.row_stride + j), j, xt, ti);
    for (int o = 16; o > 0; o >>= 1) l = sgb_cls::lane_merge(l, shfl_lane(l, o));
    if (lane == 0) {
      if (label) label[row] = l.best_i;
      if (confidence) confidence[row] = 1.f / l.s;
      if (counters) {
        if (valid) {
          if (l.best_i == ti) atomicAdd(&block_counts[0], 1ull);
          if (l.above < d.k) atomicAdd(&block_counts[1], 1ull);
        } else {
          atomicAdd(&block_counts[3], 1ull);
        }
        atomicAdd(&block_counts[2], 1ull);
      }
    }
  }
  __syncthreads();
  if (counters && threadIdx.x < 4 && block_counts[threadIdx.x]) atomicAdd(&counters[threadIdx.x], block_counts[threadIdx.x]);
}

}  // namespace

extern "C" int sgb_classify_rows(const void* logits, int64_t N, int32_t C, int64_t row_stride, int32_t logits_bf16, const int64_t* target,
                                 const void* soft_target, int64_t target_stride, int32_t target_bf16, int32_t k, int64_t* counters,
                                 int32_t* label, float* confidence, void* stream) {
  SGB_REQUIRE(N >= 0, "N must be >= 0");
  if (N == 0) return SGB_OK;
  SGB_REQUIRE(logits, "null logits");
  SGB_REQUIRE(counters || label || confidence, "no output requested");
  SGB_REQUIRE(C >= 1 && row_stride >= C, "C must be >= 1 and the row stride >= C");
  if (counters) {
    SGB_REQUIRE((target != nullptr) != (soft_target != nullptr), "counters need exactly one of target / soft_target");
    SGB_REQUIRE(k >= 1 && k <= C, "k must be in [1, C]");
    SGB_REQUIRE(!soft_target || target_stride >= C, "soft-target row stride must be >= C");
  }
  const int64_t blocks = (N + kWarps - 1) / kWarps;
  SGB_REQUIRE(blocks <= 0x7fffffff, "too many rows");
  const Rows d = {N, C, k, row_stride, target_stride, logits_bf16 ? 1 : 0, target_bf16 ? 1 : 0};
  classify_rows_kernel<<<(unsigned)blocks, kWarps * 32, 0, (cudaStream_t)stream>>>(d, logits, counters ? target : nullptr, counters ? soft_target : nullptr,
                                                                                  (unsigned long long*)counters, label, confidence);
  SGB_LAUNCH_CHECK("classify_rows_kernel");
  return SGB_OK;
}

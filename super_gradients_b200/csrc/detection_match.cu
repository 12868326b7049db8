// DetectionMetrics matching (row (f)-N4): which NMS outputs are true positives / ignored, for every IoU threshold, one launch per
// validation batch instead of the reference's per-image Python loop over (prediction, target) pairs with a dozen small tensor ops
// per pair (detection_utils.py:937-958).  One CTA per image; its predictions, targets and crowd targets live in shared memory;
// warp j runs threshold j's greedy assignment (the thresholds never interact), lanes stride over the targets.
// DetectionMetricsDistanceBased (detection_utils.py:1008-1118) is the same kernel with another pair rule: the staging, the
// top-k-per-class selection and the prediction order are shared, only the score of a (prediction, target) pair differs.
// Latency-bound integer / compare work on a few KB per image -- no roofline to speak of; the point is removing ~1e4 launches and a
// device->host sync per validation batch.  The arithmetic is in detection_match_math.cuh (shared with the CPU test build).
#include "common.cuh"
#include "detection_match_math.cuh"

namespace {

using sgb_match::Best;
using sgb_match::Box;

struct Smem {
  Box* pbox;
  float *parea, *pscore, *pcls;
  int* order;       // used predictions in confidence order
  uint8_t* used;
  Box* tbox;
  float *tarea, *tcls;
  Box* cbox;
  float* ccls;
  uint8_t* taken;   // [n_thresholds][max_targets]
};

__host__ __device__ inline size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

__host__ __device__ inline size_t carve(const SgbMatchDesc& d, char* base, Smem* s) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += align16(bytes);
    return p;
  };
  Smem t;
  t.pbox = (Box*)take(sizeof(Box) * d.max_preds);
  t.parea = (float*)take(4 * (size_t)d.max_preds);
  t.pscore = (float*)take(4 * (size_t)d.max_preds);
  t.pcls = (float*)take(4 * (size_t)d.max_preds);
  t.order = (int*)take(4 * (size_t)d.max_preds);
  t.used = (uint8_t*)take((size_t)d.max_preds);
  t.tbox = (Box*)take(sizeof(Box) * d.max_targets);
  t.tarea = (float*)take(4 * (size_t)d.max_targets);
  t.tcls = (float*)take(4 * (size_t)d.max_targets);
  t.cbox = (Box*)take(sizeof(Box) * (d.max_crowd > 0 ? d.max_crowd : 1));
  t.ccls = (float*)take(4 * (size_t)(d.max_crowd > 0 ? d.max_crowd : 1));
  t.taken = (uint8_t*)take((size_t)d.n_thresholds * d.max_targets);
  if (s) *s = t;
  return off;
}

// The pair rule of the greedy assignment.  IoU: a higher score is closer, a pair matches when IoU > thr, a crowd target
// switches "ignore" on when IoA > thr; thresholds are read from device memory.
struct IouRule {
  const float* thresholds;
  __device__ float thr(int j) const { return thresholds[j]; }
  __device__ Best best_free(const Smem& s, int p, float thr, const uint8_t* taken, int M, int lane) const {
    return sgb_match::best_free_target(s.pbox[p], s.parea[p], s.pcls[p], thr, s.tbox, s.tarea, s.tcls, taken, M, lane, 32);
  }
  __device__ Best merge(Best a, Best b) const { return sgb_match::better(a, b); }
  __device__ float crowd(const Smem& s, int p, int C) const { return sgb_match::best_crowd_ioa(s.pbox[p], s.parea[p], s.pcls[p], s.cbox, s.ccls, C); }
  __device__ bool crowd_hits(float v, float thr) const { return v > thr; }
};

// Centre distance: a lower score is closer, a pair matches when distance < thr, a crowd target switches "ignore" on when the
// nearest same-class one is nearer than thr; the thresholds travel by value in the launch parameters (checked on the host).
template <int kMetric>
struct DistanceRule {
  float thresholds[SGB_MATCH_MAX_THRESHOLDS];
  __device__ float thr(int j) const { return thresholds[j]; }
  __device__ Best best_free(const Smem& s, int p, float thr, const uint8_t* taken, int M, int lane) const {
    return sgb_match::nearest_free_target(kMetric, sgb_match::centre(s.pbox[p]), s.pcls[p], thr, s.tbox, s.tcls, taken, M, lane, 32);
  }
  __device__ Best merge(Best a, Best b) const { return sgb_match::nearer(a, b); }
  __device__ float crowd(const Smem& s, int p, int C) const {
    return sgb_match::nearest_crowd_distance(kMetric, sgb_match::centre(s.pbox[p]), s.pcls[p], s.cbox, s.ccls, C);
  }
  __device__ bool crowd_hits(float v, float thr) const { return v < thr; }
};

template <class Rule>
__global__ void detection_match_kernel(const SgbMatchDesc d, const Rule rule, const float* __restrict__ preds, const int32_t* __restrict__ pred_count,
                                       const float* __restrict__ targets, const int32_t* __restrict__ target_count,
                                       const float* __restrict__ crowd, const int32_t* __restrict__ crowd_count,
                                       uint8_t* __restrict__ matched, uint8_t* __restrict__ ignore) {
  extern __shared__ __align__(16) char smem_raw[];
  __shared__ int n_used_s;
  Smem s;
  carve(d, smem_raw, &s);
  const int b = blockIdx.x, tid = threadIdx.x, nthr = blockDim.x, T = d.n_thresholds;
  const int P = min(max(pred_count[b], 0), d.max_preds);
  const int M = min(max(target_count[b], 0), d.max_targets);
  const int C = d.max_crowd > 0 ? min(max(crowd_count[b], 0), d.max_crowd) : 0;
  const float* pr = preds + (int64_t)b * d.max_preds * 6;
  uint8_t* mt = matched + (int64_t)b * d.max_preds * T;
  uint8_t* ig = ignore + (int64_t)b * d.max_preds * T;

  for (int i = tid; i < P; i += nthr) {
    const float* r = pr + i * 6;
    const Box bx = sgb_match::clip_box(Box{r[0], r[1], r[2], r[3]}, d.height, d.width);
    s.pbox[i] = bx;
    s.parea[i] = sgb_match::area(bx);
    s.pscore[i] = r[4];
    s.pcls[i] = r[5];
  }
  for (int i = tid; i < M; i += nthr) {
    const float* r = targets + ((int64_t)b * d.max_targets + i) * 5;
    const Box bx = sgb_match::target_xyxy(r[1], r[2], r[3], r[4], d.denormalize_targets != 0, d.height, d.width);
    s.tbox[i] = bx;
    s.tarea[i] = sgb_match::area(bx);
    s.tcls[i] = r[0];
  }
  for (int i = tid; i < C; i += nthr) {
    const float* r = crowd + ((int64_t)b * d.max_crowd + i) * 5;
    s.cbox[i] = sgb_match::target_xyxy(r[1], r[2], r[3], r[4], d.denormalize_targets != 0, d.height, d.width);
    s.ccls[i] = r[0];
  }
  for (int i = tid; i < T * d.max_targets; i += nthr) s.taken[i] = 0;
  if (tid == 0) n_used_s = 0;
  __syncthreads();

  // get_top_k_idx_per_cls: non-zero score and fewer than top_k same-class predictions ahead in confidence order
  for (int i = tid; i < P; i += nthr) {
    const float sc = s.pscore[i], cl = s.pcls[i];
    int rank = 0;
    for (int j = 0; j < P; ++j) rank += (s.pcls[j] == cl && sgb_match::before(s.pscore[j], j, sc, i)) ? 1 : 0;
    s.used[i] = (rank < d.top_k && sc != 0.f) ? 1 : 0;
  }
  __syncthreads();
  for (int i = tid; i < P; i += nthr) {
    const uint8_t u = s.used[i];
    if (u) {
      const float sc = s.pscore[i];
      int pos = 0;
      for (int j = 0; j < P; ++j) pos += (s.used[j] && sgb_match::before(s.pscore[j], j, sc, i)) ? 1 : 0;
      s.order[pos] = i;
      atomicAdd(&n_used_s, 1);
    }
    for (int j = 0; j < T; ++j) {
      mt[i * T + j] = 0;
      ig[i * T + j] = u ? 0 : 1;
    }
  }
  for (int i = P * T + tid; i < d.max_preds * T; i += nthr) {
    mt[i] = 0;
    ig[i] = 0;
  }
  __syncthreads();
  const int n_used = n_used_s;

  // IoUMatching / DistanceMatching.compute_targets: warp j owns threshold j
  const int warp = tid >> 5, lane = tid & 31, n_warps = nthr >> 5;
  if (M > 0) {
    for (int j = warp; j < T; j += n_warps) {
      const float thr = rule.thr(j);
      uint8_t* taken = s.taken + (size_t)j * d.max_targets;
      for (int k = 0; k < n_used; ++k) {
        const int p = s.order[k];
        Best best = rule.best_free(s, p, thr, taken, M, lane);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          Best other;
          other.v = __shfl_xor_sync(0xffffffffu, best.v, o);
          other.t = __shfl_xor_sync(0xffffffffu, best.t, o);
          best = rule.merge(best, other);
        }
        if (best.t >= 0 && lane == 0) {
          taken[best.t] = 1;
          mt[p * T + j] = 1;
        }
        __syncwarp();
      }
    }
  }
  __syncthreads();

  // IoUMatching / DistanceMatching.compute_crowd_targets
  if (C > 0) {
    for (int k = tid; k < n_used; k += nthr) {
      const int p = s.order[k];
      const float best = rule.crowd(s, p, C);
      for (int j = 0; j < T; ++j)
        if (rule.crowd_hits(best, rule.thr(j))) ig[p * T + j] = 1;
    }
  }
}

// The argument checks common to both entry points (errors carry the entry point's name); *bytes = dynamic shared memory.
#define MATCH_REQUIRE(cond, msg)                                  \
  do {                                                            \
    if (!(cond)) {                                                \
      sgb_set_error("%s: requirement failed: %s", entry, msg);    \
      return SGB_E_INVALID;                                       \
    }                                                             \
  } while (0)

static int check_match_args(const char* entry, const SgbMatchDesc* d, const float* preds, const int32_t* pred_count, const float* targets,
                            const int32_t* target_count, const float* crowd, const int32_t* crowd_count, const float* thresholds,
                            uint8_t* matched, uint8_t* ignore, size_t* bytes) {
  MATCH_REQUIRE(d && preds && pred_count && targets && target_count && thresholds && matched && ignore, "null pointer");
  MATCH_REQUIRE(d->B > 0 && d->max_preds > 0 && d->max_targets > 0 && d->max_crowd >= 0, "bad shape");
  MATCH_REQUIRE(d->n_thresholds > 0 && d->n_thresholds <= SGB_MATCH_MAX_THRESHOLDS, "1..32 thresholds");
  MATCH_REQUIRE(d->max_crowd == 0 || (crowd && crowd_count), "crowd targets missing");
  MATCH_REQUIRE(d->top_k > 0, "top_k");
  *bytes = carve(*d, nullptr, nullptr);
  MATCH_REQUIRE(*bytes <= 200 * 1024, "predictions + targets of one image exceed shared memory");
  return SGB_OK;
}
#undef MATCH_REQUIRE

template <class Rule>
static int launch_match(const SgbMatchDesc* d, const Rule& rule, size_t bytes, const float* preds, const int32_t* pred_count,
                        const float* targets, const int32_t* target_count, const float* crowd, const int32_t* crowd_count,
                        uint8_t* matched, uint8_t* ignore, void* stream) {
  if (bytes > 48 * 1024) cudaFuncSetAttribute(detection_match_kernel<Rule>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  int warps = d->n_thresholds < 4 ? 4 : d->n_thresholds;
  detection_match_kernel<Rule><<<d->B, warps * 32, bytes, (cudaStream_t)stream>>>(*d, rule, preds, pred_count, targets, target_count, crowd,
                                                                                  crowd_count, matched, ignore);
  SGB_LAUNCH_CHECK("detection_match_kernel");
  return SGB_OK;
}

template <int kMetric>
static int launch_distance(const SgbMatchDesc* d, const float* thresholds, size_t bytes, const float* preds, const int32_t* pred_count,
                           const float* targets, const int32_t* target_count, const float* crowd, const int32_t* crowd_count,
                           uint8_t* matched, uint8_t* ignore, void* stream) {
  DistanceRule<kMetric> rule{};
  for (int j = 0; j < d->n_thresholds; ++j) rule.thresholds[j] = thresholds[j];
  return launch_match(d, rule, bytes, preds, pred_count, targets, target_count, crowd, crowd_count, matched, ignore, stream);
}

}  // namespace

extern "C" int sgb_detection_matching(const SgbMatchDesc* d, const float* preds, const int32_t* pred_count, const float* targets,
                                      const int32_t* target_count, const float* crowd, const int32_t* crowd_count,
                                      const float* thresholds, uint8_t* matched, uint8_t* ignore, void* stream) {
  size_t bytes = 0;
  const int rc = check_match_args(__func__, d, preds, pred_count, targets, target_count, crowd, crowd_count, thresholds, matched, ignore, &bytes);
  if (rc != SGB_OK) return rc;
  return launch_match(d, IouRule{thresholds}, bytes, preds, pred_count, targets, target_count, crowd, crowd_count, matched, ignore, stream);
}

extern "C" int sgb_detection_distance_matching(const SgbMatchDesc* d, int32_t metric, const float* preds, const int32_t* pred_count,
                                               const float* targets, const int32_t* target_count, const float* crowd,
                                               const int32_t* crowd_count, const float* thresholds, uint8_t* matched, uint8_t* ignore,
                                               void* stream) {
  size_t bytes = 0;
  const int rc = check_match_args(__func__, d, preds, pred_count, targets, target_count, crowd, crowd_count, thresholds, matched, ignore, &bytes);
  if (rc != SGB_OK) return rc;
  SGB_REQUIRE(metric == SGB_DISTANCE_EUCLIDEAN || metric == SGB_DISTANCE_MANHATTAN, "distance metric: SGB_DISTANCE_EUCLIDEAN or SGB_DISTANCE_MANHATTAN");
  for (int j = 0; j < d->n_thresholds; ++j)  // host memory: read here and passed by value
    SGB_REQUIRE(std::isfinite(thresholds[j]) && thresholds[j] >= 0.f, "distance thresholds must be finite and >= 0");
  return metric == SGB_DISTANCE_EUCLIDEAN
             ? launch_distance<sgb_match::kEuclidean>(d, thresholds, bytes, preds, pred_count, targets, target_count, crowd, crowd_count, matched, ignore, stream)
             : launch_distance<sgb_match::kManhattan>(d, thresholds, bytes, preds, pred_count, targets, target_count, crowd, crowd_count, matched, ignore, stream);
}

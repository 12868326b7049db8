// PoseEstimationMetrics matching: which predicted poses are true positives / ignored, for every OKS threshold, one launch per
// validation batch instead of the reference's per-image Python loops (compute_oks visits every (target, prediction) pair with about
// ten tensor ops, compute_img_keypoint_matching then walks the sorted OKS matrix; pose_estimation_utils.py:67-94, :196-233).
// One CTA per image: its top-k predictions' poses, its targets (joints, boxes, areas) and the OKS matrix [used predictions x
// targets] live in shared memory; the OKS matrix is computed once by all threads, then warp j runs threshold j's greedy assignment
// (the thresholds never interact) with its lanes strided over the targets.  The arithmetic is in pose_match_math.cuh (shared with
// the CPU test build).
//
// Shared memory of one image, every term rounded up to 16 bytes (carve()):
//   4P (scores) + 4K (order) + 8KJ (predicted xy) + 4J (vars) + 4T (thresholds) + 4K (crowd best) + KT (matched)
//   + 12MJ (target joints) + 16M (boxes) + 4M (areas) + 4M (visible-joint counts) + 4M (column -> target) + 4KM (OKS) + TM (taken)
// with P = the prediction row pitch, K = min(top_k, P), M = the target row pitch, J joints and T thresholds.  At the pose recipe's
// settings (P = K = 30 kept predictions, J = 17, T = 10) that is 4896 bytes + 362 bytes per target: the 200 KB limit admits up to
// 552 targets in one image.  Larger working sets are refused (SGB_E_INVALID), never truncated.
#include "common.cuh"
#include "pose_match_math.cuh"

namespace {

using sgb_match::Best;
namespace pm = sgb_pose_match;

struct Dims {
  int P, M, J, T, K;  // pitches: predictions, targets, joints, thresholds, used predictions (min(top_k, P))
};

struct Smem {
  float* score;     // [P]
  int* order;       // [K] used predictions in confidence order
  float* pxy;       // [K][J][2] poses of the used predictions
  float* vars;      // [J]
  float* thr;       // [T]
  float* crowd;     // [K] best OKS over the ignored targets
  uint8_t* mflag;   // [K][T]
  float* tj;        // [M][J][3]
  float* tbox;      // [M][4] XYWH (given or derived)
  float* tarea;     // [M]
  int* tk1;         // [M] visible joints
  int* col;         // [M] OKS column -> target: regular targets first, then the ignored ones, each in target order
  float* oks;       // [K][M]
  uint8_t* taken;   // [T][M]
};

__host__ __device__ inline size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

__host__ __device__ inline size_t carve(const Dims& d, char* base, Smem* s) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += align16(bytes);
    return p;
  };
  const size_t P = d.P, M = d.M, J = d.J, T = d.T, K = d.K;
  Smem t;
  t.score = (float*)take(4 * P);
  t.order = (int*)take(4 * K);
  t.pxy = (float*)take(8 * K * J);
  t.vars = (float*)take(4 * J);
  t.thr = (float*)take(4 * T);
  t.crowd = (float*)take(4 * K);
  t.mflag = (uint8_t*)take(K * T);
  t.tj = (float*)take(12 * M * J);
  t.tbox = (float*)take(16 * M);
  t.tarea = (float*)take(4 * M);
  t.tk1 = (int*)take(4 * M);
  t.col = (int*)take(4 * M);
  t.oks = (float*)take(4 * K * M);
  t.taken = (uint8_t*)take(T * M);
  if (s) *s = t;
  return off;
}

__global__ void pose_match_kernel(const Dims d, const float* __restrict__ poses, const float* __restrict__ scores,
                                  const int32_t* __restrict__ pred_count, const float* __restrict__ gt_joints, const float* __restrict__ gt_boxes,
                                  const float* __restrict__ gt_areas, const uint8_t* __restrict__ gt_flags, const int32_t* __restrict__ gt_count,
                                  const float* __restrict__ sigmas, const float* __restrict__ thresholds, uint8_t* __restrict__ matched,
                                  uint8_t* __restrict__ ignore, float* __restrict__ used_scores, int32_t* __restrict__ used_count,
                                  int32_t* __restrict__ n_targets, float* __restrict__ oks_out) {
  extern __shared__ __align__(16) char smem_raw[];
  __shared__ int n_reg_s;
  Smem s;
  carve(d, smem_raw, &s);
  const int b = blockIdx.x, tid = threadIdx.x, nthr = blockDim.x;
  const int J = d.J, T = d.T;
  const int P = min(max(pred_count[b], 0), d.P);
  const int M = min(max(gt_count[b], 0), d.M);
  const int n_used = min(P, d.K);

  for (int i = tid; i < P; i += nthr) s.score[i] = scores[(int64_t)b * d.P + i];
  for (int j = tid; j < J; j += nthr) s.vars[j] = pm::oks_var(sigmas[j]);
  for (int j = tid; j < T; j += nthr) s.thr[j] = thresholds[j];
  for (int i = tid; i < d.K * T; i += nthr) s.mflag[i] = 0;
  for (int i = tid; i < T * M; i += nthr) s.taken[i] = 0;
  const float* gj = gt_joints + (int64_t)b * d.M * J * 3;
  for (int i = tid; i < M * J * 3; i += nthr) s.tj[i] = gj[i];
  __syncthreads();

  // ground truth (pose_estimation_metrics.py:264-292): derived boxes / areas, visible-joint counts
  for (int t = tid; t < M; t += nthr) {
    const int64_t g = (int64_t)b * d.M + t;
    const uint8_t f = gt_flags[g];
    const float* tj = s.tj + t * J * 3;
    float* bx = s.tbox + 4 * t;
    if (f & pm::FLAG_HAS_BOX) {
      for (int c = 0; c < 4; ++c) bx[c] = gt_boxes[g * 4 + c];
    } else {
      pm::visible_box_xywh(tj, J, bx);
    }
    s.tarea[t] = (f & pm::FLAG_HAS_AREA) ? gt_areas[g] : pm::box_area(bx);
    s.tk1[t] = pm::n_visible(tj, J);
  }
  // top-k by score (pose_estimation_utils.py:190-194), ranked among all P rows
  for (int i = tid; i < P; i += nthr) {
    const float sc = s.score[i];
    int rank = 0;
    for (int j = 0; j < P; ++j) rank += pm::before(s.score[j], j, sc, i) ? 1 : 0;
    if (rank < n_used) s.order[rank] = i;
  }
  // regular targets first, then the ignored ones (targets / crowd_targets of pose_estimation_metrics.py:283-292)
  if (tid == 0) {
    int n = 0;
    for (int t = 0; t < M; ++t)
      if (!pm::is_ignored(s.tj + t * J * 3, J, gt_flags[(int64_t)b * d.M + t])) s.col[n++] = t;
    n_reg_s = n;
    for (int t = 0; t < M; ++t)
      if (pm::is_ignored(s.tj + t * J * 3, J, gt_flags[(int64_t)b * d.M + t])) s.col[n++] = t;
  }
  __syncthreads();
  const int n_reg = n_reg_s;
  for (int i = tid; i < n_used * J; i += nthr) {
    const int k = i / J, j = i - k * J;
    const float* p = poses + (((int64_t)b * d.P + s.order[k]) * J + j) * 3;
    s.pxy[2 * i] = p[0];
    s.pxy[2 * i + 1] = p[1];
  }
  __syncthreads();

  // the OKS matrix, once: compute_oks (pose_estimation_utils.py:57-94)
  for (int i = tid; i < n_used * M; i += nthr) {
    const int k = i / M, c = i - k * M, t = s.col[c];
    const float v = pm::oks(s.pxy + k * J * 2, 2, s.tj + t * J * 3, s.tbox + 4 * t, s.tarea[t], s.tk1[t], s.vars, J);
    s.oks[i] = v;
    if (oks_out) oks_out[((int64_t)b * d.K + k) * d.M + t] = v;
  }
  __syncthreads();

  // greedy assignment (pose_estimation_utils.py:196-233): warp j owns threshold j
  const int warp = tid >> 5, lane = tid & 31, n_warps = nthr >> 5;
  if (n_reg > 0) {
    for (int j = warp; j < T; j += n_warps) {
      const float floor = pm::qualify_floor(s.thr[0], s.thr[j]);
      uint8_t* taken = s.taken + (size_t)j * M;
      for (int k = 0; k < n_used; ++k) {
        Best best = pm::best_free_target(s.oks + k * M, floor, taken, n_reg, lane, 32);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          Best other;
          other.v = __shfl_xor_sync(0xffffffffu, best.v, o);
          other.t = __shfl_xor_sync(0xffffffffu, best.t, o);
          best = sgb_match::better(best, other);
        }
        if (best.t >= 0 && lane == 0) {
          taken[best.t] = 1;
          s.mflag[k * T + j] = 1;
        }
        __syncwarp();
      }
    }
  }
  // crowd rule (pose_estimation_utils.py:237-256)
  for (int k = tid; k < n_used; k += nthr) s.crowd[k] = M > n_reg ? pm::best_crowd_oks(s.oks + k * M + n_reg, M - n_reg) : -INFINITY;
  __syncthreads();

  uint8_t* mt = matched + (int64_t)b * d.K * T;
  uint8_t* ig = ignore + (int64_t)b * d.K * T;
  for (int i = tid; i < d.K * T; i += nthr) {
    const int k = i / T, j = i - k * T;
    const bool u = k < n_used;
    mt[i] = u ? s.mflag[i] : 0;
    ig[i] = (u && s.crowd[k] > s.thr[j]) ? 1 : 0;
  }
  for (int k = tid; k < d.K; k += nthr) used_scores[(int64_t)b * d.K + k] = k < n_used ? s.score[s.order[k]] : 0.f;
  if (tid == 0) {
    used_count[b] = n_used;
    n_targets[b] = n_reg;
  }
}

}  // namespace

extern "C" int sgb_pose_keypoint_matching(const float* poses, const float* scores, const int32_t* pred_count, const float* gt_joints,
                                          const float* gt_boxes, const float* gt_areas, const uint8_t* gt_flags, const int32_t* gt_count,
                                          const float* sigmas, const float* thresholds, int32_t B, int32_t max_preds, int32_t max_targets,
                                          int32_t n_joints, int32_t n_thresholds, int32_t top_k, uint8_t* matched, uint8_t* ignore,
                                          float* used_scores, int32_t* used_count, int32_t* n_targets, float* oks_out, void* stream) {
  SGB_REQUIRE(poses && scores && pred_count && gt_joints && gt_boxes && gt_areas && gt_flags && gt_count && sigmas && thresholds, "null input");
  SGB_REQUIRE(matched && ignore && used_scores && used_count && n_targets, "null output");
  SGB_REQUIRE(B > 0 && max_preds > 0 && max_targets > 0 && n_joints > 0, "bad shape");
  SGB_REQUIRE(n_thresholds > 0 && n_thresholds <= SGB_MATCH_MAX_THRESHOLDS, "1..32 OKS thresholds");
  SGB_REQUIRE(top_k > 0, "top_k");
  const Dims d{max_preds, max_targets, n_joints, n_thresholds, top_k < max_preds ? top_k : max_preds};
  const size_t bytes = carve(d, nullptr, nullptr);
  SGB_REQUIRE(bytes <= 200 * 1024, "predictions + targets of one image exceed shared memory");
  if (bytes > 48 * 1024) cudaFuncSetAttribute(pose_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  const int warps = n_thresholds < 4 ? 4 : n_thresholds;
  pose_match_kernel<<<B, warps * 32, bytes, (cudaStream_t)stream>>>(d, poses, scores, pred_count, gt_joints, gt_boxes, gt_areas, gt_flags,
                                                                     gt_count, sigmas, thresholds, matched, ignore, used_scores, used_count,
                                                                     n_targets, oks_out);
  SGB_LAUNCH_CHECK("pose_match_kernel");
  return SGB_OK;
}

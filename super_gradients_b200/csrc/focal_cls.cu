// Focal classification term of PPYoloELoss (use_varifocal_loss=False; ppyolo_loss.py:1069-1077, call site :834-838), as a
// replacement pass AFTER the fused varifocal / IoU / DFL kernel: sums[0] := sum of the focal loss over [B, L, C] and grad_cls :=
// its final gradient (w_cls * grad_scale / normaliser folded in), so that the fused kernel -- measured and profiled with the
// varifocal term every YOLO-NAS / PP-YOLOE recipe uses -- stays byte-identical.  Elementwise and HBM-bound: reads the logits and
// the per-anchor label / score once, writes the gradient once (2 * 4 * B*L*C bytes).  The arithmetic (gamma = 2, weight not
// detached, optional alpha_t) is sgb_tal::cls_term of tal_math.cuh, shared with the pose loss and the CPU test build.
#include "common.cuh"
#include "tal_math.cuh"

namespace {

__global__ void __launch_bounds__(256) focal_cls_kernel(SgbLossDesc d, const float* __restrict__ cls, const int* __restrict__ alabel,
                                                        const float* __restrict__ ascore, double* sums, float grad_scale, float alpha,
                                                        float* __restrict__ gcls) {
  const int64_t total = (int64_t)d.B * d.L * d.ncls;
  double nrm = sums[3];
  if (nrm < 1.0) nrm = 1.0;
  const float inv = grad_scale / (float)nrm;
  float acc = 0.f;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / d.ncls;
    const int c = (int)(e - i * d.ncls);
    const float q = alabel[i] == c ? ascore[i] : 0.f;
    float loss, g;
    sgb_tal::cls_term(1, alpha, cls[e], q, &loss, &g);
    acc += loss;
    if (gcls) gcls[e] = g * d.w_cls * inv;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0 && acc != 0.f) atomicAdd(&sums[0], (double)acc);
}

}  // namespace

extern "C" int sgb_focal_cls_fwd_bwd(const SgbLossDesc* d, const float* cls_logits, const int32_t* assigned_label,
                                     const float* assigned_score, double* sums, float grad_scale, float alpha, float* grad_cls,
                                     void* stream) {
  SGB_REQUIRE(d && cls_logits && assigned_label && assigned_score && sums, "null pointer");
  SGB_REQUIRE(d->B > 0 && d->L > 0 && d->ncls > 0, "bad loss shape");
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(sums, 0, sizeof(double), st);  // drop the varifocal sum the fused kernel left in sums[0]
  const int64_t total = (int64_t)d->B * d->L * d->ncls;
  const int grid = (int)((total + 255) / 256 > 132 * 8 ? 132 * 8 : (total + 255) / 256);
  focal_cls_kernel<<<grid, 256, 0, st>>>(*d, cls_logits, assigned_label, assigned_score, sums, grad_scale, alpha, grad_cls);
  SGB_LAUNCH_CHECK("focal_cls_kernel");
  return SGB_OK;
}

// The convolution entry points of the C ABI: validate the call, offer it to the wgmma / TMA engine (conv_sm100.cu), and give the
// calls it declines to the mma.sync engine (conv_mma.cu), which serves any filter size, stride and channel slice.
#include "common.cuh"
#include "conv_mma.h"
#include "conv_sm100.h"

namespace {

int check_desc(const SgbConvDesc* d) {
  SGB_REQUIRE(d != nullptr, "desc is null");
  SGB_REQUIRE(d->N > 0 && d->H > 0 && d->W > 0 && d->C > 0 && d->K > 0 && d->R > 0 && d->S > 0, "positive dims");
  SGB_REQUIRE(d->stride >= 1 && d->pad >= 0, "stride/pad");
  SGB_REQUIRE(d->P == (d->H + 2 * d->pad - d->R) / d->stride + 1, "P inconsistent");
  SGB_REQUIRE(d->Q == (d->W + 2 * d->pad - d->S) / d->stride + 1, "Q inconsistent");
  SGB_REQUIRE(d->C % 8 == 0, "C must be a multiple of 8 (pad the channels)");
  SGB_REQUIRE(d->x_pitch % 8 == 0 && d->x_off % 8 == 0, "x pitch/offset must be multiples of 8");
  SGB_REQUIRE(d->x_pitch >= d->x_off + d->C, "x slice exceeds pitch");
  SGB_REQUIRE(d->y_pitch >= d->y_off + d->K, "y slice exceeds pitch");
  SGB_REQUIRE(d->centre_from == 0 || (d->R == 3 && d->S == 3 && d->stride == 1 && d->pad == 1 && d->centre_from > 0 &&
                                      d->centre_from < d->K && d->centre_from % 16 == 0),
              "centre_from needs a 3x3 / stride-1 / pad-1 convolution and 0 < centre_from < K, a multiple of 16");
  return SGB_OK;
}

}  // namespace

extern "C" int sgb_conv_fprop(const SgbConvDesc* d, const sgb_bf16* x, const sgb_bf16* w, void* y, const SgbEpilogue* ep,
                              void* stream) {
  if (int rc = check_desc(d)) return rc;
  SGB_REQUIRE(x && w && y, "null pointer");
  const int rc = sm100::conv_fprop(*d, x, w, y, ep, (cudaStream_t)stream);
  return rc != sm100::DECLINED ? rc : igemm::conv_fprop(*d, x, w, y, ep, (cudaStream_t)stream);
}

extern "C" int sgb_convt2x2_fprop(const SgbConvDesc* d, const sgb_bf16* x_small, const sgb_bf16* w_up, const float* bias,
                                  sgb_bf16* y_up, void* stream) {
  // d: equivalent conv (N,H,W,C)=upsampled -> (N,P,Q,K)=small with R=S=2, stride 2, pad 0
  if (int rc = check_desc(d)) return rc;
  SGB_REQUIRE(d->R == 2 && d->S == 2 && d->stride == 2 && d->pad == 0, "convt2x2 needs R=S=2, stride 2, pad 0");
  SGB_REQUIRE(d->K % 8 == 0 && d->y_pitch % 8 == 0 && d->y_off % 8 == 0, "small-side channels must be multiples of 8");
  const int rc = sm100::convt2x2_fprop(*d, x_small, w_up, bias, y_up, (cudaStream_t)stream);
  return rc != sm100::DECLINED ? rc : igemm::convt2x2_fprop(*d, x_small, w_up, bias, y_up, (cudaStream_t)stream);
}

extern "C" int sgb_conv_dgrad(const SgbConvDesc* d, const sgb_bf16* dy, const sgb_bf16* w_crsk, sgb_bf16* dx, int accumulate,
                              void* stream) {
  if (int rc = check_desc(d)) return rc;
  SGB_REQUIRE(dy && w_crsk && dx, "null pointer");
  SGB_REQUIRE(d->K % 8 == 0 || d->y_pitch - d->y_off >= ((d->K + 7) / 8) * 8, "dy channels must be padded to 8");
  SGB_REQUIRE(d->y_pitch % 8 == 0 && d->y_off % 8 == 0, "dy pitch/offset must be multiples of 8");
  SGB_REQUIRE(d->stride == 1 || d->stride == 2, "dgrad supports stride 1 or 2");
  const int rc = sm100::conv_dgrad(*d, dy, w_crsk, dx, accumulate, (cudaStream_t)stream);
  return rc != sm100::DECLINED ? rc : igemm::conv_dgrad(*d, dy, w_crsk, dx, accumulate, (cudaStream_t)stream);
}

extern "C" int sgb_conv_wgrad(const SgbConvDesc* d, const sgb_bf16* x, const sgb_bf16* dy, float* dw, void* stream) {
  if (int rc = check_desc(d)) return rc;
  SGB_REQUIRE(x && dy && dw, "null pointer");
  SGB_REQUIRE(d->y_pitch % 8 == 0 && d->y_off % 8 == 0, "dy pitch/offset must be multiples of 8");
  SGB_REQUIRE(d->K % 8 == 0 || d->y_pitch - d->y_off >= ((d->K + 7) / 8) * 8, "dy channels must be padded to 8");
  const int rc = sm100::conv_wgrad(*d, x, dy, dw, (cudaStream_t)stream);
  return rc != sm100::DECLINED ? rc : igemm::conv_wgrad(*d, x, dy, dw, (cudaStream_t)stream);
}

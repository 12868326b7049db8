// Test infrastructure: serial HOST drivers around super_gradients_b200/csrc/resample_math.cuh (the ImageNet pre-processing kernel's
// arithmetic) and classify_math.cuh (the row-wise classification decode), compiled with g++ by tests/host_classification.py.
#include <cstring>
#include <vector>

#include "classify_math.cuh"
#include "preprocess_math.cuh"
#include "resample_math.cuh"

static inline uint16_t f32_to_bf16_rn(float f) {  // round to nearest even, as __float2bfloat16_rn (no NaNs here)
  uint32_t u;
  std::memcpy(&u, &f, 4);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}

static inline float bf16_to_f32(uint16_t b) {
  uint32_t u = (uint32_t)b << 16;
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}

// table [batch][SGB_RS_FIELDS] as sgb_resample_crop_u8; out: bf16 bit patterns [batch][out_h][out_w][out_pitch]
extern "C" int resample_crop_host(const int64_t* table, const uint8_t* src, int batch, int C, int out_h, int out_w, int out_pitch, int reverse,
                                  double max_value, const float* mean, const float* std, uint16_t* out) {
  for (int b = 0; b < batch; ++b) {
    const int64_t* t = table + (int64_t)b * SGB_RS_FIELDS;
    const int h = (int)t[SGB_RS_H], w = (int)t[SGB_RS_W], pitch = (int)t[SGB_RS_PITCH], rh = (int)t[SGB_RS_RESIZED_H], rw = (int)t[SGB_RS_RESIZED_W];
    const int top = (int)t[SGB_RS_CROP_TOP], left = (int)t[SGB_RS_CROP_LEFT];
    const uint8_t* img = src + t[SGB_RS_OFFSET];
    const sgb_rs::Axis ax = sgb_rs::axis(w, rw), ay = sgb_rs::axis(h, rh);
    std::vector<int32_t> k(sgb_rs::max_taps(w, rw) + sgb_rs::max_taps(h, rh));
    // horizontal pass over every source row, crop columns only (uint8)
    std::vector<uint8_t> mid((size_t)h * out_w * C);
    for (int col = 0; col < out_w; ++col) {
      int xmin;
      const int n = sgb_rs::coeffs(ax, left + col, w, k.data(), xmin);
      for (int y = 0; y < h; ++y)
        for (int c = 0; c < C; ++c) {
          int32_t acc = 1 << (sgb_rs::kPrecisionBits - 1);
          for (int i = 0; i < n; ++i) acc += (int32_t)img[(int64_t)y * pitch + (xmin + i) * C + c] * k[i];
          mid[((size_t)y * out_w + col) * C + c] = sgb_rs::clip8(acc);
        }
    }
    for (int oy = 0; oy < out_h; ++oy) {
      int ymin;
      const int n = sgb_rs::coeffs(ay, top + oy, h, k.data(), ymin);
      for (int col = 0; col < out_w; ++col) {
        float v[4];
        for (int c = 0; c < C; ++c) {
          int32_t acc = 1 << (sgb_rs::kPrecisionBits - 1);
          for (int i = 0; i < n; ++i) acc += (int32_t)mid[((size_t)(ymin + i) * out_w + col) * C + c] * k[i];
          v[c] = (float)sgb_rs::clip8(acc);
        }
        uint16_t* o = out + (((int64_t)b * out_h + oy) * out_w + col) * out_pitch;
        for (int c = 0; c < out_pitch; ++c)
          o[c] = f32_to_bf16_rn(c < C ? sgb_prep::standardize(v[reverse ? C - 1 - c : c], max_value, mean != nullptr, mean ? mean[c] : 0.f, std ? std[c] : 1.f) : 0.f);
      }
    }
  }
  return 0;
}

// the 32 lane states of one warp per row and the kernel's butterfly merge; target: int64 [N] or NULL, soft: f32 [N][C] or NULL
extern "C" int classify_rows_host(const void* logits, int bf16, int64_t N, int C, const int64_t* target, const float* soft, int k, int64_t* counters,
                                  int32_t* label, float* confidence) {
  for (int64_t row = 0; row < N; ++row) {
    auto x_at = [&](int j) { return bf16 ? bf16_to_f32(((const uint16_t*)logits)[row * C + j]) : ((const float*)logits)[row * C + j]; };
    int64_t t = -1;
    if (target) {
      t = target[row];
    } else if (soft) {
      int bi = -1;
      for (int j = 0; j < C; ++j)
        if (bi < 0 || sgb_cls::before(soft[row * C + j], j, soft[row * C + bi], bi)) bi = j;
      t = bi;
    }
    const bool valid = t >= 0 && t < C;
    const int ti = valid ? (int)t : -1;
    const float xt = valid ? x_at(ti) : 0.f;
    sgb_cls::Lane lanes[32];
    for (int l = 0; l < 32; ++l) {
      lanes[l] = sgb_cls::lane_init();
      for (int j = l; j < C; j += 32) sgb_cls::lane_update(lanes[l], x_at(j), j, xt, ti);
    }
    for (int o = 16; o > 0; o >>= 1) {
      sgb_cls::Lane next[32];
      for (int l = 0; l < 32; ++l) next[l] = sgb_cls::lane_merge(lanes[l], lanes[l ^ o]);
      std::memcpy(lanes, next, sizeof(lanes));
    }
    if (label) label[row] = lanes[0].best_i;
    if (confidence) confidence[row] = 1.f / lanes[0].s;
    if (counters) {
      if (valid) {
        counters[0] += lanes[0].best_i == ti;
        counters[1] += lanes[0].above < k;
      } else {
        counters[3] += 1;
      }
      counters[2] += 1;
    }
  }
  return 0;
}

// Serial host driver around super_gradients_b200/csrc/weight_average_math.cuh (compiled with g++ -ffp-contract=off by
// tests/test_weight_averaging_cpu.py): the best-snapshot average exactly as the CUDA kernel computes each element.
#include <stdint.h>

#include "weight_average_math.cuh"

extern "C" {

// out[i] = average of slots[0 .. k-1] at element i, for i in [0, n)
void average_snapshots_host(const float* const* slots, int32_t k, int64_t n, float* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = sgb_avg::average(slots, k, i);
}
}

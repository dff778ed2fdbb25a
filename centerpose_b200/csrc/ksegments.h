// The fixed K segments of a batch-invariant plan (CP_PLAN_BATCH_INVARIANT, plan.cu select_kernels).  Host code only, in a
// header so that tests/host can compile and check it without a GPU.
#pragma once

namespace cp {

// G is the largest divisor of `slabs` with tiles1 x G <= 132, tiles1 being the (m, n) tiles of one image of one model:
// what splitk_factor picks at batch 1 on a 132-SM H100 (its workspace bound never binds there).  132 is a constant,
// never the device's SM count, so G depends on the layer's shape alone.
constexpr int kInvariantSMs = 132;
inline int fixed_ksegments(long long tiles1, int slabs) {
  int G = 1;
  for (int g = 2; g <= slabs; ++g)
    if (slabs % g == 0 && tiles1 * g <= kInvariantSMs) G = g;
  return G;
}

}  // namespace cp

// TEST INFRASTRUCTURE ONLY: compiles centerpose_b200/csrc/arena_pack.h (the liveness packer of the plan's activation
// arena, plan.cu) for the host so that tests/test_arena_pack_host.py can check it on random and real lifetime sets.
// Never loaded by the product.
#include <stdint.h>

#include <vector>

#include "../../centerpose_b200/csrc/arena_pack.h"

static std::vector<cp::ArenaAlloc> allocs(int n, const int64_t* floats, const int32_t* first, const int32_t* last) {
  std::vector<cp::ArenaAlloc> a(n);
  for (int i = 0; i < n; ++i) {
    a[i].floats = (size_t)floats[i];
    a[i].first = first[i];
    a[i].last = last[i];
  }
  return a;
}

extern "C" {

int64_t ap_align() { return (int64_t)cp::kArenaAlign; }

// arena_pack: offsets into off[n]; returns the arena size in floats
int64_t ap_pack(int n, const int64_t* floats, const int32_t* first, const int32_t* last, int64_t* off) {
  std::vector<size_t> o;
  const size_t arena = cp::arena_pack(allocs(n, floats, first, last), &o);
  for (int i = 0; i < n; ++i) off[i] = (int64_t)o[i];
  return (int64_t)arena;
}

int64_t ap_live_peak(int n, const int64_t* floats, const int32_t* first, const int32_t* last) {
  return (int64_t)cp::arena_live_peak(allocs(n, floats, first, last));
}

}  // extern "C"

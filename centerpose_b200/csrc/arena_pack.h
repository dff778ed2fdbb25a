// Liveness packing of a plan's activation arena (plan.cu).  Host code only, in a header so that tests/host can compile
// and check it without a GPU.
//
// Every allocation of the schedule is live over an inclusive range of op indices: from the op that first writes it to
// the op that last reads it.  Allocations whose ranges do not overlap may share memory.  pack() places the largest
// allocations first, each at the lowest offset that does not collide with an already placed allocation live at the same
// time.  Sizes are multiples of kArenaAlign floats, so every offset is too: kernel selection, tensor maps and split-K
// factors see the same alignment as in the bump-allocated arena.  The result depends on the input order only through
// the tie-break, so the same schedule always gets the same layout.
#pragma once
#include <stddef.h>

#include <algorithm>
#include <utility>
#include <vector>

namespace cp {

constexpr size_t kArenaAlign = 64;      // floats (256 bytes)

inline size_t arena_align(size_t floats) { return (floats + kArenaAlign - 1) / kArenaAlign * kArenaAlign; }

struct ArenaAlloc {
  size_t floats = 0;          // a multiple of kArenaAlign
  int first = -1, last = -1;  // inclusive op range over which it is live; first < 0: never touched (gets no memory)
};

inline bool arena_live_together(const ArenaAlloc& a, const ArenaAlloc& b) {
  return a.first >= 0 && b.first >= 0 && a.first <= b.last && b.first <= a.last;
}

// Offsets (floats) of the allocations in *off; returns the arena size in floats.  An allocation that is never touched
// or has no floats gets offset 0 and takes no memory.
inline size_t arena_pack(const std::vector<ArenaAlloc>& a, std::vector<size_t>* off) {
  const size_t n = a.size();
  off->assign(n, 0);
  std::vector<size_t> order;
  for (size_t i = 0; i < n; ++i)
    if (a[i].first >= 0 && a[i].floats) order.push_back(i);
  std::stable_sort(order.begin(), order.end(), [&](size_t x, size_t y) {
    if (a[x].floats != a[y].floats) return a[x].floats > a[y].floats;
    return a[x].first < a[y].first;
  });
  size_t arena = 0;
  std::vector<size_t> placed;
  std::vector<std::pair<size_t, size_t>> busy;      // [begin, end) of the placed allocations live together with this one
  for (size_t i : order) {
    busy.clear();
    for (size_t j : placed)
      if (arena_live_together(a[i], a[j])) busy.push_back({(*off)[j], (*off)[j] + a[j].floats});
    std::sort(busy.begin(), busy.end());
    size_t at = 0;
    for (const auto& b : busy) {
      if (at + a[i].floats <= b.first) break;
      at = std::max(at, b.second);
    }
    (*off)[i] = at;
    arena = std::max(arena, at + a[i].floats);
    placed.push_back(i);
  }
  return arena;
}

// The largest sum of the sizes of allocations live at one op: no packing can use less memory.
inline size_t arena_live_peak(const std::vector<ArenaAlloc>& a) {
  int ops = 0;
  for (const auto& x : a) ops = std::max(ops, x.last + 1);
  std::vector<size_t> live(ops + 1, 0);
  for (const auto& x : a)
    if (x.first >= 0)
      for (int t = x.first; t <= x.last; ++t) live[t] += x.floats;
  return *std::max_element(live.begin(), live.end());
}

}  // namespace cp

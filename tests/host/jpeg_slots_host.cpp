// centerpose_b200/csrc/jpeg_core.h compiled for the host: the slot capacity of a decoded size against what a parsed
// file needs (tests/test_mjpeg_graph_cpu.py).
#include <stdint.h>

#include "../../centerpose_b200/csrc/jpeg_core.h"

using namespace cp::jpeg;

extern "C" {

// out: comp, nseg, nsub, nblocks, nplane
void js_capacity(int out_h, int out_w, int64_t max_bytes, int words, int64_t* out) {
  SlotCap c = slot_capacity(out_h, out_w, max_bytes, words);
  const int64_t v[5] = {c.comp, c.nseg, c.nsub, c.nblocks, c.nplane};
  for (int k = 0; k < 5; ++k) out[k] = v[k];
}

// the need of a file as the workspace layouts size it; returns its cp_jpeg_refusal (0: out filled)
int js_need(const uint8_t* b, int64_t n, int words, int* hw, int64_t* out) {
  cp_jpeg_header h;
  int r = parse(b, n, &h);
  if (r != CP_JPEG_OK) return r;
  SlotCap c = frame_need(h, words);
  const int64_t v[5] = {c.comp, c.nseg, c.nsub, c.nblocks, c.nplane};
  for (int k = 0; k < 5; ++k) out[k] = v[k];
  hw[0] = h.out_h;
  hw[1] = h.out_w;
  return 0;
}

}  // extern "C"

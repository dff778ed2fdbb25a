// centerpose_b200/csrc/jpeg_core.h compiled for the host: the whole baseline decoder run sequentially (the restatement
// tests/test_jpeg_cpu.py pins against cv2.imdecode), and a simulation of the device's subsequence decode.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../centerpose_b200/csrc/jpeg_core.h"

using namespace cp::jpeg;

namespace {

struct Segment {
  std::vector<uint8_t> bytes;
};

// scan preparation: drops stuffed 0x00 bytes and fill bytes, cuts at RSTn and checks their numbering
int segments(const cp_jpeg_header& h, const uint8_t* b, std::vector<Segment>& segs) {
  int64_t nmcu = (int64_t)h.mcux * h.mcuy;
  int64_t nseg = h.restart_interval ? (nmcu + h.restart_interval - 1) / h.restart_interval : 1;
  segs.assign(nseg, Segment());
  int64_t s = 0;
  int err = 0;
  const int64_t n = h.scan_end - h.scan_begin;
  const uint8_t* r = b + h.scan_begin;
  for (int64_t i = 0; i < n; ++i) {
    uint8_t c = r[i], prev = i ? r[i - 1] : 0, next = i + 1 < n ? r[i + 1] : 0;
    if (c == 0xFF) {
      if (next == 0x00 && s < nseg) segs[s].bytes.push_back(c);
    } else if (prev == 0xFF) {
      if (c >= 0xD0 && c <= 0xD7) {
        if (s < nseg - 1 && c != 0xD0 + (s & 7)) err |= CP_JPEG_ERR_RESTART;
        ++s;
      }
    } else if (s < nseg) {
      segs[s].bytes.push_back(c);
    }
  }
  if (s < nseg - 1) err |= CP_JPEG_ERR_RESTART;
  return err;
}

int64_t seg_mcus(const cp_jpeg_header& h, int64_t s) {
  int64_t nmcu = (int64_t)h.mcux * h.mcuy;
  if (!h.restart_interval) return nmcu;
  int64_t a = s * h.restart_interval, e = a + h.restart_interval;
  return (e < nmcu ? e : nmcu) - a;
}

// coefficients of every block (decode order, natural order, DC predicted); words 0: the sequential decoder, else the
// subsequence decode at that many 32-bit words, rounds -> the synchronisation rounds of the slowest segment
int coefficients(const uint8_t* b, int64_t n, int words, std::vector<int16_t>& coef, int* rounds) {
  cp_jpeg_header h;
  if (parse(b, n, &h) != CP_JPEG_OK) return -1;
  std::vector<Segment> segs;
  int err = segments(h, b, segs);
  const int bpm = h.blocks_per_mcu;
  int64_t total = (int64_t)h.mcux * h.mcuy * bpm;
  coef.assign(total * 64, 0);
  std::vector<int32_t> diff(total, 0);
  if (rounds) *rounds = 0;
  int64_t base = 0;
  for (size_t si = 0; si < segs.size(); ++si) {
    const uint8_t* sb = segs[si].bytes.data();
    uint32_t nb = (uint32_t)segs[si].bytes.size(), bits = nb * 8;
    int nblocks = (int)(seg_mcus(h, si) * bpm);
    int16_t* c = coef.data() + base * 64;
    int32_t* d = diff.data() + base;
    if (words == 0) {
      err |= emit(h, sb, nb, State{0, 0, 0}, bits, 0, nblocks, true, c, d);
    } else {
      const uint32_t S = 32u * words;
      int nsub = bits ? (int)((bits + S - 1) / S) : 1;
      std::vector<uint64_t> st(nsub), nx(nsub);
      for (int j = 0; j < nsub; ++j) st[j] = pack(State{j * S, 0, 0});
      int r = 0;
      for (bool changed = true; changed;) {         // Jacobi rounds: every subsequence from its predecessor's exit
        ++r;
        changed = false;
        nx[0] = st[0];
        for (int j = 0; j + 1 < nsub; ++j) {
          int dcs;
          nx[j + 1] = pack(walk(h, sb, nb, unpack(st[j]), (j + 1) * S, dcs));
          changed |= nx[j + 1] != st[j + 1];
        }
        st.swap(nx);
      }
      if (rounds && r > *rounds) *rounds = r;
      int first = 0;
      for (int j = 0; j < nsub; ++j) {
        err |= emit(h, sb, nb, unpack(st[j]), (j + 1) * S, first, nblocks, j == nsub - 1, c, d);
        int dcs;
        walk(h, sb, nb, unpack(st[j]), (j + 1) * S, dcs);
        first += dcs;
      }
    }
    // DC prediction, reset at each restart, per component
    int32_t pred[3] = {0, 0, 0};
    for (int k = 0; k < nblocks; ++k) {
      int comp = block_component(h, k % bpm);
      pred[comp] += d[k];
      c[(int64_t)k * 64] = (int16_t)pred[comp];
    }
    base += nblocks;
  }
  return err;
}

}  // namespace

extern "C" {

int jh_header_size() { return (int)sizeof(cp_jpeg_header); }

int jh_parse(const uint8_t* b, int64_t n, cp_jpeg_header* h) { return parse(b, n, h); }

int64_t jh_blocks(const uint8_t* b, int64_t n) {
  cp_jpeg_header h;
  if (parse(b, n, &h) != CP_JPEG_OK) return -1;
  return (int64_t)h.mcux * h.mcuy * h.blocks_per_mcu;
}

int jh_coefficients(const uint8_t* b, int64_t n, int words, int16_t* out, int* rounds) {
  std::vector<int16_t> c;
  int err = coefficients(b, n, words, c, rounds);
  if (err >= 0) memcpy(out, c.data(), c.size() * sizeof(int16_t));
  return err;
}

// the decoded BGR image [out_h, out_w, 3]; returns cp_jpeg_error bits, or -1 for a refused header
int jh_decode(const uint8_t* b, int64_t n, uint8_t* out) {
  cp_jpeg_header h;
  if (parse(b, n, &h) != CP_JPEG_OK) return -1;
  std::vector<int16_t> coef;
  int err = coefficients(b, n, 0, coef, nullptr);
  std::vector<uint8_t> plane[3];
  const uint8_t* planes[3] = {nullptr, nullptr, nullptr};
  int ps[3] = {0, 0, 0};
  for (int c = 0; c < h.ncomp; ++c) {
    ps[c] = plane_w(h, c);
    plane[c].assign((size_t)ps[c] * plane_h(h, c), 0);
    planes[c] = plane[c].data();
  }
  int64_t total = (int64_t)h.mcux * h.mcuy * h.blocks_per_mcu;
  for (int64_t g = 0; g < total; ++g) {
    int x, y;
    int c = block_origin(h, g, x, y);
    idct_islow(coef.data() + g * 64, h.quant[c], plane[c].data() + (int64_t)y * ps[c] + x, ps[c]);
  }
  for (int oy = 0; oy < h.out_h; ++oy)
    for (int ox = 0; ox < h.out_w; ++ox) pixel(h, planes, ps, ox, oy, out + ((int64_t)oy * h.out_w + ox) * 3);
  return err;
}

}  // extern "C"

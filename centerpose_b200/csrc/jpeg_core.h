// Baseline JPEG decoding, written once as host / device code: the kernels of jpeg.cu call the per-symbol, per-block and
// per-pixel steps below, and tests/host compiles the same header with g++ to restate the whole decoder sequentially on
// the CPU and pin it against cv2.imdecode (libjpeg-turbo) bit for bit.
//
// What is restated, in libjpeg-turbo's terms:
//   jdmarker.c     the marker walk (SOF0/1, DQT 8/16-bit, DHT, DRI, SOS, APP0 JFIF, APP14 Adobe), and for a missing DHT
//                  the standard tables of T.81 Annex K.3 (jstdhuff.c), installed in slots 0 and 1 of each class;
//   jdapimin.c     the colour-space rule: JFIF or Adobe transform 1 is YCbCr, Adobe transform 0 or ids R G B is RGB,
//                  otherwise three components are YCbCr;
//   jdhuff.c       the derived tables (a lookahead table for short codes, maxcode / valoffset for long ones), the
//                  sequential symbol decode and HUFF_EXTEND, the DC predictor reset at each restart;
//   jidctint.c     jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2) ending in the post-IDCT range limit, saturating as
//                  libjpeg-turbo's SIMD IDCTs do (see range_limit);
//   jdsample.c     h2v1 / h2v2 / h1v2 "fancy" (triangle) up-sampling with its alternating biases, edge replication at
//                  the downsampled width and height, plain replication when the downsampled width is 2 or less, and
//                  box replication for 4:1:1 (int_upsample);
//   jdcolor.c      ycc_rgb_convert with its SCALEBITS 16 fixed-point tables;
//   OpenCV         the EXIF orientation (APP1 Exif, IFD0 tag 0x0112) applied by flips and transposes.
#pragma once
#include <stdint.h>
#include <string.h>

#include "../../include/centerpose_b200.h"

#if defined(__CUDACC__)
#define JPG_HD __host__ __device__ __forceinline__
#define JPG_UNROLL _Pragma("unroll")
#else
#define JPG_HD inline
#define JPG_UNROLL
#endif

namespace cp {
namespace jpeg {

// zig-zag index -> natural (row-major) index, T.81 Figure A.6 (jpeg_natural_order), one byte per entry, entry k in
// byte k % 8 of word k / 8
JPG_HD int natural_order(int k) {
  uint64_t w;
  switch (k >> 3) {
    case 0: w = 0x0a03020910080100ull; break;
    case 1: w = 0x05040b1219201811ull; break;
    case 2: w = 0x22293028211a130cull; break;
    case 3: w = 0x1c150e07060d141bull; break;
    case 4: w = 0x242b323938312a23ull; break;
    case 5: w = 0x332c251e170f161dull; break;
    case 6: w = 0x2e271f262d343b3aull; break;
    default: w = 0x3f3e372f363d3c35ull; break;
  }
  return (int)((w >> ((k & 7) * 8)) & 63);
}

// ---------------------------------------------------------------- the decoder state at a symbol boundary
// pos: bit position in the restart segment; blk: block within the MCU; k: zig-zag index of the next coefficient (0: the
// DC difference comes next).  The component, and so the DC or AC table, follows from blk.
struct State {
  uint32_t pos;
  int blk, k;
};
JPG_HD uint64_t pack(State s) { return ((uint64_t)s.pos << 16) | ((uint64_t)s.blk << 8) | (uint64_t)s.k; }
JPG_HD State unpack(uint64_t v) { return State{(uint32_t)(v >> 16), (int)((v >> 8) & 0xff), (int)(v & 0xff)}; }

JPG_HD int block_component(const cp_jpeg_header& h, int blk) {
  if (h.ncomp == 1) return 0;
  int ny = h.comp_h[0] * h.comp_v[0];
  return blk < ny ? 0 : 1 + (blk - ny);
}

// 32 bits of the segment from bit `pos`, zeros past its end (libjpeg fills a starved bit buffer with zeros)
JPG_HD uint32_t peek32(const uint8_t* seg, uint32_t nbytes, uint32_t pos) {
  uint32_t i = pos >> 3;
  uint64_t w = 0;
JPG_UNROLL
  for (int b = 0; b < 5; ++b) w = (w << 8) | (i + b < nbytes ? seg[i + b] : 0u);
  return (uint32_t)(w >> (8 - (pos & 7)));
}

JPG_HD int extend(int r, int s) { return s == 0 ? 0 : (r < (1 << (s - 1)) ? r + (int)(~0u << s) + 1 : r); }

// one Huffman code of `t` at the top of `bits`: (length << 8) | symbol, or 0 for a code in no table
JPG_HD int huff_decode(const cp_jpeg_huff& t, uint32_t bits) {
  int e = t.look[bits >> 23];
  if (e) return e;
  for (int l = 10; l <= 16; ++l) {
    int code = (int)(bits >> (32 - l));
    if (code <= t.maxcode[l]) return (l << 8) | t.vals[(code + t.valoffset[l]) & 0xff];
  }
  return 0;
}

// What one symbol did.  coef: natural index written (-1: none), value: its value (the DC difference for coef 0);
// dc: the symbol began a block; done: it ended one; err: a cp_jpeg_error bit.
struct Sym {
  int coef, value, err;
  bool dc, done;
};

// Decodes the symbol at s (a Huffman code and its extra bits) and returns the state after it.
JPG_HD State step(const cp_jpeg_header& h, const uint8_t* seg, uint32_t nbytes, State s, Sym& o) {
  o.coef = -1; o.value = 0; o.err = 0; o.dc = s.k == 0; o.done = false;
  int c = block_component(h, s.blk);
  uint32_t bits = peek32(seg, nbytes, s.pos);
  int e = huff_decode(s.k == 0 ? h.dc[c] : h.ac[c], bits);
  if (!e) {
    o.err = CP_JPEG_ERR_CODE;
    s.pos += 16;                  // no symbol here: skip on, so that a thread decoding from a guess still moves
    s.k = 0;
    return s;
  }
  int len = e >> 8, sym = e & 0xff;
  uint32_t rest = bits << len;
  if (s.k == 0) {
    int r = sym ? (int)(rest >> (32 - sym)) : 0;
    o.coef = 0; o.value = extend(r, sym);
    s.pos += len + sym;
    s.k = 1;
  } else {
    int run = sym >> 4, sz = sym & 15;
    s.pos += len + sz;
    if (sz) {
      s.k += run;
      if (s.k > 63) { o.err = CP_JPEG_ERR_RUN; s.k = 64; }
      else {
        o.coef = natural_order(s.k);
        o.value = extend((int)(rest >> (32 - sz)), sz);
        s.k += 1;
      }
    } else if (run == 15) {
      s.k += 16;
      if (s.k > 64) { o.err = CP_JPEG_ERR_RUN; s.k = 64; }
    } else {
      s.k = 64;                   // EOB
    }
  }
  if (s.k >= 64) {
    s.k = 0;
    o.done = true;
    if (++s.blk == h.blocks_per_mcu) s.blk = 0;
  }
  return s;
}

// ---------------------------------------------------------------- one subsequence of a restart segment
// The parallel decode cuts a segment of `nbytes` bytes into subsequences of S bits; the thread of subsequence j decodes
// the symbols that start in [its start state, (j + 1) S) and the segment, and its exit state is the start of j + 1.

// Walks from s to the exit state, counting the symbols that begin a block.
JPG_HD State walk(const cp_jpeg_header& h, const uint8_t* seg, uint32_t nbytes, State s, uint32_t stop, int& dcs) {
  const uint32_t bits = nbytes * 8u;
  dcs = 0;
  while (s.pos < stop && s.pos < bits) {
    Sym o;
    s = step(h, seg, nbytes, s, o);
    dcs += o.dc;
  }
  return s;
}

// The final pass over one subsequence that starts exact at s, with `first` blocks of the segment begun before it:
// writes the coefficients of the segment's blocks (natural order, coefficient 0 left for the DC predictor) and the DC
// differences, and returns cp_jpeg_error bits.  Symbols past the segment's `nblocks` blocks are ignored, as libjpeg
// ignores the bits after a segment's last MCU.  `last`: j is the segment's last subsequence, which also checks that the
// segment held all its blocks.
JPG_HD int emit(const cp_jpeg_header& h, const uint8_t* seg, uint32_t nbytes, State s, uint32_t stop, int first,
                int nblocks, bool last, int16_t* coef, int32_t* dcdiff) {
  const uint32_t bits = nbytes * 8u;
  int cur = s.k ? first - 1 : first;
  if (cur < 0) return CP_JPEG_ERR_CODE;          // mid-block with no block begun: only a corrupt stream gets here
  while (s.pos < stop && s.pos < bits && cur < nblocks) {
    Sym o;
    State n = step(h, seg, nbytes, s, o);
    if (o.err) return o.err;
    if (n.pos > bits) return CP_JPEG_ERR_SHORT;
    if (o.coef == 0) dcdiff[cur] = o.value;
    else if (o.coef > 0) coef[(int64_t)cur * 64 + o.coef] = (int16_t)o.value;
    cur += o.done;
    s = n;
  }
  return last && cur < nblocks ? CP_JPEG_ERR_SHORT : 0;
}

// ---------------------------------------------------------------- dequantisation and jpeg_idct_islow
enum { CONST_BITS = 13, PASS1_BITS = 2 };
#define JPG_FIX(x) ((int32_t)((x) * (1 << CONST_BITS) + 0.5))
JPG_HD int32_t descale(int32_t x, int n) { return (x + (1 << (n - 1))) >> n; }

// The post-IDCT range limit, x + CENTERJSAMPLE saturated to 0..255.  libjpeg-turbo's C IDCT indexes its range-limit
// table with x & RANGE_MASK (1023), which wraps for |x| >= 512; its SIMD IDCTs, which cv2 runs on x86-64, pack with
// signed saturation instead.  The tests pin the saturation against cv2 with DC-only blocks up to |x| = 1023.  Both
// agree for |x| < 512, which covers every stream an encoder writes from 8-bit samples.
JPG_HD uint8_t range_limit(int32_t x) { return (uint8_t)(x < -128 ? 0 : x > 127 ? 255 : x + 128); }

// coef: natural order, DC already predicted; q: the component's table (natural order); out: row stride `stride`
JPG_HD void idct_islow(const int16_t* coef, const int16_t* q, uint8_t* out, int stride) {
  int32_t ws[64];
  JPG_UNROLL
  for (int col = 0; col < 8; ++col) {
    const int16_t* in = coef + col;
    const int16_t* qt = q + col;
    if (!in[8] && !in[16] && !in[24] && !in[32] && !in[40] && !in[48] && !in[56]) {
      int32_t dc = ((int32_t)in[0] * qt[0]) * (1 << PASS1_BITS);
      for (int r = 0; r < 8; ++r) ws[r * 8 + col] = dc;
      continue;
    }
    int32_t z2 = (int32_t)in[16] * qt[16], z3 = (int32_t)in[48] * qt[48];
    int32_t z1 = (z2 + z3) * JPG_FIX(0.541196100);
    int32_t tmp2 = z1 + z3 * (-JPG_FIX(1.847759065));
    int32_t tmp3 = z1 + z2 * JPG_FIX(0.765366865);
    z2 = (int32_t)in[0] * qt[0]; z3 = (int32_t)in[32] * qt[32];
    int32_t tmp0 = (z2 + z3) * (1 << CONST_BITS), tmp1 = (z2 - z3) * (1 << CONST_BITS);
    int32_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    tmp0 = (int32_t)in[56] * qt[56]; tmp1 = (int32_t)in[40] * qt[40];
    tmp2 = (int32_t)in[24] * qt[24]; tmp3 = (int32_t)in[8] * qt[8];
    z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2; int32_t z4 = tmp1 + tmp3;
    int32_t z5 = (z3 + z4) * JPG_FIX(1.175875602);
    tmp0 *= JPG_FIX(0.298631336); tmp1 *= JPG_FIX(2.053119869);
    tmp2 *= JPG_FIX(3.072711026); tmp3 *= JPG_FIX(1.501321110);
    z1 *= -JPG_FIX(0.899976223); z2 *= -JPG_FIX(2.562915447);
    z3 *= -JPG_FIX(1.961570560); z4 *= -JPG_FIX(0.390180644);
    z3 += z5; z4 += z5;
    tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
    const int n = CONST_BITS - PASS1_BITS;
    ws[0 * 8 + col] = descale(tmp10 + tmp3, n); ws[7 * 8 + col] = descale(tmp10 - tmp3, n);
    ws[1 * 8 + col] = descale(tmp11 + tmp2, n); ws[6 * 8 + col] = descale(tmp11 - tmp2, n);
    ws[2 * 8 + col] = descale(tmp12 + tmp1, n); ws[5 * 8 + col] = descale(tmp12 - tmp1, n);
    ws[3 * 8 + col] = descale(tmp13 + tmp0, n); ws[4 * 8 + col] = descale(tmp13 - tmp0, n);
  }
  JPG_UNROLL
  for (int row = 0; row < 8; ++row) {
    const int32_t* w = ws + row * 8;
    uint8_t* o = out + row * stride;
    const int n = CONST_BITS + PASS1_BITS + 3;
    if (!w[1] && !w[2] && !w[3] && !w[4] && !w[5] && !w[6] && !w[7]) {
      uint8_t v = range_limit(descale(w[0], PASS1_BITS + 3));
      for (int c = 0; c < 8; ++c) o[c] = v;
      continue;
    }
    int32_t z2 = w[2], z3 = w[6];
    int32_t z1 = (z2 + z3) * JPG_FIX(0.541196100);
    int32_t tmp2 = z1 + z3 * (-JPG_FIX(1.847759065));
    int32_t tmp3 = z1 + z2 * JPG_FIX(0.765366865);
    int32_t tmp0 = (w[0] + w[4]) * (1 << CONST_BITS), tmp1 = (w[0] - w[4]) * (1 << CONST_BITS);
    int32_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    tmp0 = w[7]; tmp1 = w[5]; tmp2 = w[3]; tmp3 = w[1];
    z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2; int32_t z4 = tmp1 + tmp3;
    int32_t z5 = (z3 + z4) * JPG_FIX(1.175875602);
    tmp0 *= JPG_FIX(0.298631336); tmp1 *= JPG_FIX(2.053119869);
    tmp2 *= JPG_FIX(3.072711026); tmp3 *= JPG_FIX(1.501321110);
    z1 *= -JPG_FIX(0.899976223); z2 *= -JPG_FIX(2.562915447);
    z3 *= -JPG_FIX(1.961570560); z4 *= -JPG_FIX(0.390180644);
    z3 += z5; z4 += z5;
    tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
    o[0] = range_limit(descale(tmp10 + tmp3, n)); o[7] = range_limit(descale(tmp10 - tmp3, n));
    o[1] = range_limit(descale(tmp11 + tmp2, n)); o[6] = range_limit(descale(tmp11 - tmp2, n));
    o[2] = range_limit(descale(tmp12 + tmp1, n)); o[5] = range_limit(descale(tmp12 - tmp1, n));
    o[3] = range_limit(descale(tmp13 + tmp0, n)); o[4] = range_limit(descale(tmp13 - tmp0, n));
  }
}
#undef JPG_FIX

// ---------------------------------------------------------------- geometry of the component planes
// Component c's plane holds whole blocks: plane_w(c) x plane_h(c) bytes; its samples that are image content are the
// first ds_w(c) x ds_h(c) (libjpeg's downsampled_width / _height).
JPG_HD int plane_w(const cp_jpeg_header& h, int c) { return h.mcux * (h.ncomp == 1 ? 1 : h.comp_h[c]) * 8; }
JPG_HD int plane_h(const cp_jpeg_header& h, int c) { return h.mcuy * (h.ncomp == 1 ? 1 : h.comp_v[c]) * 8; }
JPG_HD int ds_w(const cp_jpeg_header& h, int c) { return (h.width * h.comp_h[c] + h.hmax - 1) / h.hmax; }
JPG_HD int ds_h(const cp_jpeg_header& h, int c) { return (h.height * h.comp_v[c] + h.vmax - 1) / h.vmax; }

// block g of the frame (in decode order) -> component and top-left sample in its plane
JPG_HD int block_origin(const cp_jpeg_header& h, int64_t g, int& x, int& y) {
  if (h.ncomp == 1) {
    x = (int)(g % h.mcux) * 8; y = (int)(g / h.mcux) * 8;
    return 0;
  }
  int64_t m = g / h.blocks_per_mcu;
  int r = (int)(g % h.blocks_per_mcu);
  int mx = (int)(m % h.mcux), my = (int)(m / h.mcux);
  int ny = h.comp_h[0] * h.comp_v[0];
  if (r < ny) {
    x = (mx * h.comp_h[0] + r % h.comp_h[0]) * 8; y = (my * h.comp_v[0] + r / h.comp_h[0]) * 8;
    return 0;
  }
  x = mx * 8; y = my * 8;
  return 1 + (r - ny);
}

// ---------------------------------------------------------------- up-sampling and colour, one output pixel
JPG_HD int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// the chroma sample at image pixel (x, y) of plane p (stride ps) as jdsample.c up-samples it
JPG_HD int chroma(const cp_jpeg_header& h, const uint8_t* p, int ps, int x, int y) {
  const int hx = h.hmax, vy = h.vmax;
  const int dw = ds_w(h, 1), dh = ds_h(h, 1);
  if (hx == 1 && vy == 1) return p[y * ps + x];
  if (hx == 4 || (dw <= 2 && hx == 2)) return p[(y / vy) * ps + x / hx];      // int_upsample, h2v1 / h2v2_upsample
  if (hx == 1) {                                                            // h1v2_fancy_upsample
    int r = y >> 1, nr = clampi((y & 1) ? r + 1 : r - 1, 0, dh - 1);
    return (3 * p[r * ps + x] + p[nr * ps + x] + ((y & 1) ? 2 : 1)) >> 2;
  }
  int i = x >> 1;
  if (vy == 1) {                                                            // h2v1_fancy_upsample
    const uint8_t* row = p + y * ps;
    if (!(x & 1)) return i == 0 ? row[0] : (3 * row[i] + row[i - 1] + 1) >> 2;
    return i == dw - 1 ? row[i] : (3 * row[i] + row[i + 1] + 2) >> 2;
  }
  int r = y >> 1, nr = clampi((y & 1) ? r + 1 : r - 1, 0, dh - 1);          // h2v2_fancy_upsample
  const uint8_t* r0 = p + r * ps;
  const uint8_t* r1 = p + nr * ps;
  int cs = 3 * r0[i] + r1[i];
  if (!(x & 1)) return i == 0 ? (cs * 4 + 8) >> 4 : (cs * 3 + 3 * r0[i - 1] + r1[i - 1] + 8) >> 4;
  return i == dw - 1 ? (cs * 4 + 7) >> 4 : (cs * 3 + 3 * r0[i + 1] + r1[i + 1] + 7) >> 4;
}

// jdcolor.c build_ycc_rgb_table: FIX(x) = x * 2^16 rounded, ONE_HALF = 2^15, an arithmetic right shift
#define JPG_CFIX(x) ((int32_t)((x) * 65536.0 + 0.5))
JPG_HD int cr_r(int cr) { return (JPG_CFIX(1.40200) * (cr - 128) + (1 << 15)) >> 16; }
JPG_HD int cb_b(int cb) { return (JPG_CFIX(1.77200) * (cb - 128) + (1 << 15)) >> 16; }
JPG_HD int cbcr_g(int cb, int cr) {
  return (-JPG_CFIX(0.34414) * (cb - 128) + (1 << 15) - JPG_CFIX(0.71414) * (cr - 128)) >> 16;
}
#undef JPG_CFIX

// the image pixel that lands at output (ox, oy) under EXIF orientation o (OpenCV's ExifTransform)
JPG_HD void oriented_source(const cp_jpeg_header& h, int ox, int oy, int& x, int& y) {
  const int W = h.width, H = h.height;
  switch (h.orientation) {
    case 2: x = W - 1 - ox; y = oy; break;
    case 3: x = W - 1 - ox; y = H - 1 - oy; break;
    case 4: x = ox; y = H - 1 - oy; break;
    case 5: x = oy; y = ox; break;
    case 6: x = oy; y = H - 1 - ox; break;
    case 7: x = W - 1 - oy; y = H - 1 - ox; break;
    case 8: x = W - 1 - oy; y = ox; break;
    default: x = ox; y = oy; break;
  }
}

// BGR of output pixel (ox, oy); planes[c] with strides ps[c]
JPG_HD void pixel(const cp_jpeg_header& h, const uint8_t* const* planes, const int* ps, int ox, int oy, uint8_t* bgr) {
  int x, y;
  oriented_source(h, ox, oy, x, y);
  int Y = planes[0][y * ps[0] + x];
  if (h.ncomp == 1) { bgr[0] = bgr[1] = bgr[2] = (uint8_t)Y; return; }
  int cb = chroma(h, planes[1], ps[1], x, y), cr = chroma(h, planes[2], ps[2], x, y);
  bgr[0] = (uint8_t)clampi(Y + cb_b(cb), 0, 255);
  bgr[1] = (uint8_t)clampi(Y + cbcr_g(cb, cr), 0, 255);
  bgr[2] = (uint8_t)clampi(Y + cr_r(cr), 0, 255);
}

// ---------------------------------------------------------------- the capacity of a slot of one decoded size
// Upper bounds on what one frame needs in the decode workspace, for every supported file that decodes to out_h x out_w
// (the coded frame in either orientation, any sampling, gray included, any restart interval) in at most max_bytes
// bytes, at `words` 32-bit words per subsequence: its compacted scan bytes, restart segments (at most one per MCU),
// subsequences, blocks and component-plane bytes.  A plane holds whole blocks, so the plane bytes are 64 per block.
struct SlotCap {
  int64_t comp, nseg, nsub, nblocks, nplane;
};

// What one parsed frame needs, in the same terms (jpeg.cu's workspace layouts size by it).
JPG_HD SlotCap frame_need(const cp_jpeg_header& h, int words) {
  const int64_t nraw = h.scan_end - h.scan_begin, nmcu = (int64_t)h.mcux * h.mcuy;
  SlotCap c{nraw + 8, h.restart_interval ? (nmcu + h.restart_interval - 1) / h.restart_interval : 1, 0,
            nmcu * h.blocks_per_mcu, 0};
  c.nsub = (nraw * 8 + 32 * words - 1) / (32 * words) + c.nseg;
  for (int k = 0; k < h.ncomp; ++k) c.nplane += (int64_t)plane_w(h, k) * plane_h(h, k);
  return c;
}

JPG_HD SlotCap slot_capacity(int out_h, int out_w, int64_t max_bytes, int words) {
  SlotCap c{max_bytes + 8, 0, 0, 0, 0};
  const int hs[6] = {1, 2, 1, 2, 4, 1}, vs[6] = {1, 1, 2, 2, 1, 1};      // luma 1x1 2x1 1x2 2x2 4x1, then gray
  for (int o = 0; o < 2; ++o) {
    const int64_t w = o ? out_h : out_w, h = o ? out_w : out_h;
    for (int k = 0; k < 6; ++k) {
      const int64_t nmcu = ((w + 8 * hs[k] - 1) / (8 * hs[k])) * ((h + 8 * vs[k] - 1) / (8 * vs[k]));
      const int64_t nb = k == 5 ? nmcu : nmcu * (hs[k] * vs[k] + 2);
      if (nmcu > c.nseg) c.nseg = nmcu;
      if (nb > c.nblocks) c.nblocks = nb;
    }
  }
  c.nsub = (max_bytes * 8 + 32 * words - 1) / (32 * words) + c.nseg;
  c.nplane = c.nblocks * 64;
  return c;
}

// ---------------------------------------------------------------- host: the header parser
// T.81 Annex K.3 (Tables K.3 - K.6), the tables libjpeg-turbo installs in slots 0 (luma) and 1 (chroma) of each class
// when a file defines none there (MJPEG).  bits[l] = number of codes of length l (1..16).
static const uint8_t kStdDcBits[2][17] = {{0, 0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0},
                                          {0, 0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}};
static const uint8_t kStdAcBits[2][17] = {{0, 0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
                                          {0, 0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
static const uint8_t kStdAcVals[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71,
     0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72,
     0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37,
     0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59,
     0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83,
     0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3,
     0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
     0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
     0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22,
     0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1,
     0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36,
     0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58,
     0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a,
     0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a,
     0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
     0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
     0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};

struct RawHuff {
  bool defined;
  uint8_t bits[17];
  uint8_t vals[256];
};

// jdhuff.c jpeg_make_d_derived_tbl with a 9-bit lookahead; false for a table libjpeg refuses
inline bool derive(const RawHuff& r, bool is_dc, cp_jpeg_huff& t) {
  memset(&t, 0, sizeof(t));
  int n = 0;
  for (int l = 1; l <= 16; ++l) n += r.bits[l];
  if (n > 256) return false;
  memcpy(t.vals, r.vals, n);
  int huffsize[257], huffcode[257], p = 0;
  for (int l = 1; l <= 16; ++l)
    for (int i = 0; i < r.bits[l]; ++i) huffsize[p++] = l;
  huffsize[p] = 0;
  int code = 0, si = huffsize[0];
  p = 0;
  while (huffsize[p]) {
    while (huffsize[p] == si) huffcode[p++] = code++;
    if (code >= (1 << si)) return false;          // a code set that overflows its length
    code <<= 1;
    ++si;
  }
  p = 0;
  for (int l = 1; l <= 16; ++l) {
    if (r.bits[l]) {
      t.valoffset[l] = p - huffcode[p];
      p += r.bits[l];
      t.maxcode[l] = huffcode[p - 1];
    } else {
      t.maxcode[l] = -1;
    }
  }
  t.maxcode[0] = -1;
  t.maxcode[17] = 0x7fffffff;
  p = 0;
  for (int l = 1; l <= 9; ++l)
    for (int i = 0; i < r.bits[l]; ++i, ++p) {
      int lo = huffcode[p] << (9 - l);
      for (int j = 0; j < (1 << (9 - l)); ++j) t.look[lo + j] = (uint16_t)((l << 8) | r.vals[p]);
    }
  if (is_dc)
    for (int i = 0; i < n; ++i)
      if (r.vals[i] > 15) return false;
  return true;
}

inline int refuse(cp_jpeg_header* h, int reason) {
  h->status = reason;
  return reason;
}

// EXIF orientation from an APP1 payload (after the marker length), 1 when absent or out of range
inline int exif_orientation(const uint8_t* p, int64_t n) {
  if (n < 14 || memcmp(p, "Exif\0\0", 6) != 0) return 0;
  const uint8_t* t = p + 6;
  int64_t tn = n - 6;
  bool le;
  if (t[0] == 'I' && t[1] == 'I') le = true;
  else if (t[0] == 'M' && t[1] == 'M') le = false;
  else return 0;
  auto u16 = [&](int64_t o) -> uint32_t { return le ? t[o] | t[o + 1] << 8 : t[o] << 8 | t[o + 1]; };
  auto u32 = [&](int64_t o) -> uint32_t {
    return le ? (uint32_t)t[o] | (uint32_t)t[o + 1] << 8 | (uint32_t)t[o + 2] << 16 | (uint32_t)t[o + 3] << 24
              : (uint32_t)t[o] << 24 | (uint32_t)t[o + 1] << 16 | (uint32_t)t[o + 2] << 8 | (uint32_t)t[o + 3];
  };
  if (u16(2) != 42) return 0;
  int64_t ifd = u32(4);
  if (ifd < 8 || ifd + 2 > tn) return 0;
  int cnt = (int)u16(ifd);
  for (int i = 0; i < cnt; ++i) {
    int64_t e = ifd + 2 + 12 * (int64_t)i;
    if (e + 12 > tn) break;
    if (u16(e) == 0x0112) {
      uint32_t v = u16(e + 8);
      return v >= 1 && v <= 8 ? (int)v : 1;
    }
  }
  return 0;
}

// The marker walk: fills *h and returns CP_JPEG_OK or the cp_jpeg_refusal.
inline int parse(const uint8_t* b, int64_t n, cp_jpeg_header* h) {
  memset(h, 0, sizeof(*h));
  h->orientation = 1;
  if (n < 2 || b[0] != 0xFF || b[1] != 0xD8) return refuse(h, CP_JPEG_NOT_JPEG);
  RawHuff huff[2][4];
  memset(huff, 0, sizeof(huff));
  uint16_t qt[4][64];
  bool qdef[4] = {false, false, false, false};
  bool sof = false, jfif = false, adobe = false, exif_seen = false;
  int adobe_transform = -1, cid[4] = {0, 0, 0, 0}, tq[4] = {0, 0, 0, 0};
  int64_t i = 2;
  for (;;) {
    // a marker: 0xFF, any number of fill bytes 0xFF, then the code
    if (i >= n || b[i] != 0xFF) return refuse(h, i >= n ? CP_JPEG_TRUNCATED : CP_JPEG_BAD_HEADER);
    while (i < n && b[i] == 0xFF) ++i;
    if (i >= n) return refuse(h, CP_JPEG_TRUNCATED);
    int m = b[i++];
    if (m == 0xD8 || m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;    // parameterless
    if (m == 0xD9) return refuse(h, CP_JPEG_TRUNCATED);                   // EOI before a scan
    if (i + 2 > n) return refuse(h, CP_JPEG_TRUNCATED);
    int64_t len = b[i] << 8 | b[i + 1];
    if (len < 2) return refuse(h, CP_JPEG_BAD_HEADER);
    if (i + len > n) return refuse(h, CP_JPEG_TRUNCATED);
    const uint8_t* p = b + i + 2;
    int64_t pn = len - 2;
    i += len;
    if (m >= 0xC0 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
      if (m == 0xC2 || m == 0xC6 || m == 0xCA || m == 0xCE) return refuse(h, CP_JPEG_PROGRESSIVE);
      if (m == 0xC3 || m == 0xC7 || m == 0xCB || m == 0xCF) return refuse(h, CP_JPEG_LOSSLESS);
      if (m >= 0xC9) return refuse(h, CP_JPEG_ARITHMETIC);
      if (m == 0xC5) return refuse(h, CP_JPEG_MULTI_SCAN);                // hierarchical
      if (sof || pn < 6) return refuse(h, CP_JPEG_BAD_HEADER);
      if (p[0] != 8) return refuse(h, CP_JPEG_PRECISION);
      h->height = p[1] << 8 | p[2];
      h->width = p[3] << 8 | p[4];
      h->ncomp = p[5];
      if (h->ncomp != 1 && h->ncomp != 3) return refuse(h, CP_JPEG_COMPONENTS);
      if (pn < 6 + 3 * h->ncomp) return refuse(h, CP_JPEG_BAD_HEADER);
      if (h->height == 0) return refuse(h, CP_JPEG_DNL);
      if (h->width == 0) return refuse(h, CP_JPEG_BAD_HEADER);
      // cv2.imread's limit; it also keeps every plane index (at most (W + 31) (H + 15) samples) inside int32
      if ((int64_t)h->width * h->height > ((int64_t)1 << 30)) return refuse(h, CP_JPEG_TOO_LARGE);
      for (int c = 0; c < h->ncomp; ++c) {
        cid[c] = p[6 + 3 * c];
        h->comp_h[c] = p[7 + 3 * c] >> 4;
        h->comp_v[c] = p[7 + 3 * c] & 15;
        tq[c] = p[8 + 3 * c];
        if (tq[c] > 3 || h->comp_h[c] < 1 || h->comp_v[c] < 1) return refuse(h, CP_JPEG_BAD_HEADER);
      }
      sof = true;
    } else if (m == 0xC4) {                                               // DHT
      while (pn > 0) {
        if (pn < 17) return refuse(h, CP_JPEG_BAD_TABLE);
        int tc = p[0] >> 4, th = p[0] & 15;
        if (tc > 1 || th > 3) return refuse(h, CP_JPEG_BAD_TABLE);
        RawHuff& r = huff[tc][th];
        r.bits[0] = 0;
        int cnt = 0;
        for (int l = 1; l <= 16; ++l) cnt += (r.bits[l] = p[l]);
        if (cnt > 256 || pn < 17 + cnt) return refuse(h, CP_JPEG_BAD_TABLE);
        memcpy(r.vals, p + 17, cnt);
        r.defined = true;
        p += 17 + cnt;
        pn -= 17 + cnt;
      }
    } else if (m == 0xCC) {
      return refuse(h, CP_JPEG_ARITHMETIC);                               // DAC
    } else if (m == 0xDB) {                                               // DQT
      while (pn > 0) {
        int pq = p[0] >> 4, t = p[0] & 15;
        int sz = pq ? 129 : 65;
        if (pq > 1 || t > 3 || pn < sz) return refuse(h, CP_JPEG_BAD_TABLE);
        for (int k = 0; k < 64; ++k) qt[t][natural_order(k)] = pq ? (uint16_t)(p[1 + 2 * k] << 8 | p[2 + 2 * k]) : p[1 + k];
        qdef[t] = true;
        p += sz;
        pn -= sz;
      }
    } else if (m == 0xDD) {                                               // DRI
      if (pn < 2) return refuse(h, CP_JPEG_BAD_HEADER);
      h->restart_interval = p[0] << 8 | p[1];
    } else if (m == 0xDC) {
      return refuse(h, CP_JPEG_DNL);
    } else if (m == 0xE0) {
      if (pn >= 14 && memcmp(p, "JFIF\0", 5) == 0) jfif = true;
    } else if (m == 0xE1) {
      if (!exif_seen) {
        int o = exif_orientation(p, pn);
        if (o) { h->orientation = o; exif_seen = true; }
      }
    } else if (m == 0xEE) {
      if (pn >= 12 && memcmp(p, "Adobe", 5) == 0) { adobe = true; adobe_transform = p[11]; }
    } else if (m == 0xDA) {                                               // SOS
      if (!sof) return refuse(h, CP_JPEG_BAD_HEADER);
      if (pn < 1) return refuse(h, CP_JPEG_BAD_HEADER);
      int ns = p[0];
      if (ns != h->ncomp) return refuse(h, CP_JPEG_MULTI_SCAN);
      if (pn < 4 + 2 * ns) return refuse(h, CP_JPEG_BAD_HEADER);
      int Ss = p[1 + 2 * ns], Se = p[2 + 2 * ns], AhAl = p[3 + 2 * ns];
      if (Ss != 0 || Se != 63 || AhAl != 0) return refuse(h, CP_JPEG_BAD_HEADER);
      // colour space (jdapimin.c default_decompress_parms)
      if (h->ncomp == 3) {
        bool rgb;
        if (jfif) rgb = false;
        else if (adobe) rgb = adobe_transform == 0;
        else rgb = cid[0] == 'R' && cid[1] == 'G' && cid[2] == 'B';
        if (rgb) return refuse(h, CP_JPEG_RGB);
      }
      // sampling
      if (h->ncomp == 1) {
        h->comp_h[0] = h->comp_v[0] = 1;
      } else {
        if (h->comp_h[1] != 1 || h->comp_v[1] != 1 || h->comp_h[2] != 1 || h->comp_v[2] != 1)
          return refuse(h, CP_JPEG_SAMPLING);
        int hy = h->comp_h[0], vy = h->comp_v[0];
        if (!((hy <= 2 && vy <= 2) || (hy == 4 && vy == 1))) return refuse(h, CP_JPEG_SAMPLING);
      }
      h->hmax = h->comp_h[0];
      h->vmax = h->comp_v[0];
      h->mcux = (h->width + 8 * h->hmax - 1) / (8 * h->hmax);
      h->mcuy = (h->height + 8 * h->vmax - 1) / (8 * h->vmax);
      h->blocks_per_mcu = h->ncomp == 1 ? 1 : h->hmax * h->vmax + 2;
      // tables: the scan's component order must be the frame's, each with its DC / AC table
      for (int s = 0; s < ns; ++s) {
        int id = p[1 + 2 * s], td = p[2 + 2 * s] >> 4, ta = p[2 + 2 * s] & 15;
        if (id != cid[s] || td > 3 || ta > 3) return refuse(h, CP_JPEG_MULTI_SCAN);
        if (!qdef[tq[s]]) return refuse(h, CP_JPEG_BAD_TABLE);
        for (int k = 0; k < 64; ++k) h->quant[s][k] = (int16_t)qt[tq[s]][k];
        RawHuff dc = huff[0][td], ac = huff[1][ta];
        if (!dc.defined && td < 2) {                                      // jstdhuff.c std_huff_tables
          memcpy(dc.bits, kStdDcBits[td], 17);
          for (int v = 0; v < 12; ++v) dc.vals[v] = (uint8_t)v;
          dc.defined = true;
        }
        if (!ac.defined && ta < 2) {
          memcpy(ac.bits, kStdAcBits[ta], 17);
          memcpy(ac.vals, kStdAcVals[ta], 162);
          ac.defined = true;
        }
        if (!dc.defined || !ac.defined) return refuse(h, CP_JPEG_BAD_TABLE);
        if (!derive(dc, true, h->dc[s]) || !derive(ac, false, h->ac[s])) return refuse(h, CP_JPEG_BAD_TABLE);
      }
      h->scan_begin = i;
      // the entropy-coded data runs to the first marker that is not RSTn (0xFF 0x00 is a stuffed 0xFF)
      int64_t e = i;
      for (;;) {
        const void* f = e < n ? memchr(b + e, 0xFF, (size_t)(n - e)) : nullptr;
        if (!f) { e = n; break; }
        e = (const uint8_t*)f - b;
        int64_t j = e + 1;
        while (j < n && b[j] == 0xFF) ++j;
        if (j >= n) { e = n; break; }
        if (b[j] == 0x00 || (b[j] >= 0xD0 && b[j] <= 0xD7)) { e = j + 1; continue; }
        if (b[j] == 0xDC) return refuse(h, CP_JPEG_DNL);
        if (b[j] == 0xDA) return refuse(h, CP_JPEG_MULTI_SCAN);
        break;
      }
      h->scan_end = e;
      bool swap = h->orientation >= 5;
      h->out_h = swap ? h->width : h->height;
      h->out_w = swap ? h->height : h->width;
      return refuse(h, CP_JPEG_OK);
    }
  }
}

}  // namespace jpeg
}  // namespace cp

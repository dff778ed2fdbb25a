// Stand-alone entry points next to the plan:
//   cp_dcn_v2_forward -- the `_ext.dcn_v2_forward` replacement (NCHW in / out), built from
//                        the same implicit-GEMM deformable kernel the plan uses
//                        (reference: DCNv2/src/cuda/dcn_v2_cuda.cu:42-172).
//   cp_preprocess     -- batched uint8 HWC frames -> normalised fp32 NCHW network input
//                        (reference: detectors/base_detector.py:91-148, fix_res branch); cp_preprocess_ragged does
//                        the same for frames of different sizes in one launch, and cp_preprocess_yuv420 for YUV 4:2:0
//                        frames (NV12 / I420, NV21 / YV12, each in limited or full range; the colour conversion of cv2.cvtColor fused into the warp's tap fetch), and
//                        cp_preprocess_formats for the camera formats (RGB24, RGBA, BGRA, YUYV, UYVY, gray and the
//                        Bayer mosaics), one per frame; cp_preprocess_resize_affine for a frame first resized by
//                        cv2.resize at a test scale (fused into the warp's tap fetch);
//                        cp_preprocess_slots_dev is the graph-safe form for one tracking step of a uniform batch, and
//                        cp_preprocess_slots_ragged_dev (over a cp_preprocess_frame_table) that of slots of mixed sizes,
//                        cp_preprocess_slots_rows_dev that of the live slots of a step with idle slots (a table may hold
//                        one format per frame: cp_preprocess_frame_table_formats, launched as CP_PIX_PER_FRAME);
//   cp_gather_rows_dev -- a row gather through a device map, the graph-safe reordering of per-slot rows.
#include <climits>
#include <cstring>
#include <type_traits>
#include <vector>

#include "common.cuh"

namespace cp {
namespace {

// cv2.warpAffine(src, M, dsize, flags=INTER_LINEAR) (BORDER_CONSTANT 0) for 8-bit 3-channel frames, restated bit for bit
// (OpenCV imgwarp.cpp WarpAffineInvoker + remapBilinear, third party: opencv-python >= 4.5.3.56, 4.13.0 in this image,
// checked by tests/test_preprocess_host.py against cv2 itself):
//   * M is inverted on the host exactly like cv::warpAffine does (cp_preprocess_affine below);
//   * AB_BITS = 10: X0 = cvRound((M[1] y + M[2]) * 1024) + 16, adelta[x] = cvRound(M[0] x * 1024) (cvRound = round
//     half to even), X = (X0 + adelta[x]) >> 5 -> integer source pixel X >> 5 and a 1/32-pixel fraction X & 31;
//   * the four bilinear weights are the integers (32 - fy)(32 - fx) * 32, ... (sum 32768, INTER_REMAP_COEF_BITS = 15);
//   * pixel = (sum of weight * source + 16384) >> 15, neighbours outside the image contribute the border value 0;
// followed by ((v / 255.) - mean) / std evaluated in double and rounded once to float32 like the numpy expression at
// base_detector.py:132.  `Minv` = the inverted 2 x 3 matrix (dst -> src).
struct WarpM {
  double m[6];
};

// The source position of output pixel (x, y) under the inverted matrix W in 1/32 pixels, warpAffine's coordinate
// generator.
__device__ __forceinline__ int2 affine_pos(const WarpM& W, int x, int y) {
  // unfused double arithmetic (the host code OpenCV runs here has no FMA contraction)
  const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(W.m[1], (double)y), W.m[2]), 1024.0)) + 16;
  const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(W.m[4], (double)y), W.m[5]), 1024.0)) + 16;
  const int ad = __double2int_rn(__dmul_rn(__dmul_rn(W.m[0], (double)x), 1024.0));
  const int bd = __double2int_rn(__dmul_rn(__dmul_rn(W.m[3], (double)x), 1024.0));
  return make_int2((X0 + ad) >> 5, (Y0 + bd) >> 5);
}

// The source position of a coordinate-map entry m = (map x, map y) in 1/32 pixels, cv2.remap's generator for float
// maps (imgwarp.cpp RemapInvoker, INTER_LINEAR): cvRound(m * INTER_TAB_SIZE) of the float32 product.  cvRound is the
// x86 conversion, whose result for NaN, +-inf and products beyond the int range is INT_MIN; that lands far outside the
// frame, so the pixel is the border value 0.  (__float2int_rn would give 0 for NaN and saturate the others, which
// samples inside the frame.)
__device__ __forceinline__ int cv_round32(float v) {
  const float p = __fmul_rn(v, 32.f);
  return p >= -2147483648.f && p < 2147483648.f ? __float2int_rn(p) : INT_MIN;
}
__device__ __forceinline__ int2 map_pos(float2 m) { return make_int2(cv_round32(m.x), cv_round32(m.y)); }

// one output pixel of a [sh, sw] frame whose source position is (X, Y) in 1/32 pixels (affine_pos or map_pos), all
// three channels.  The source pixels come from `px`: px.taps(iy, ix, in-frame flags) sees the 2 x 2 taps (iy, ix) ..
// (iy + 1, ix + 1) once, then px(k, yy, xx, c) is channel c (B, G, R) of in-frame tap k = 2 (yy - iy) + (xx - ix) as
// an integer 0..255.  Taps outside the frame are the border value 0 and are never fetched.  Channel c's value goes to
// out[c * plane], then to prev(c, value), the previous-frame write of the launch's mode (preprocess_kernel).
template <class Fetch, class Prev>
__device__ __forceinline__ void warp_walk(Fetch px, float* __restrict__ out, size_t plane, int sh, int sw, int2 pos,
                                          const float* mean, const float* stdv, Prev prev) {
  const int X = pos.x, Y = pos.y;
  int ix = X >> 5, iy = Y >> 5;
  // saturate_cast<short> of the integer coordinates (only matters for absurd scales; keeps the restatement exact)
  ix = max(-32768, min(32767, ix));
  iy = max(-32768, min(32767, iy));
  const int fx = X & 31, fy = Y & 31;
  const int w00 = (32 - fy) * (32 - fx) * 32, w01 = (32 - fy) * fx * 32, w10 = fy * (32 - fx) * 32, w11 = fy * fx * 32;
  const bool y0 = iy >= 0 && iy < sh, y1 = iy + 1 >= 0 && iy + 1 < sh;
  const bool x0 = ix >= 0 && ix < sw, x1 = ix + 1 >= 0 && ix + 1 < sw;
  px.taps(iy, ix, y0 && x0, y0 && x1, y1 && x0, y1 && x1);
  for (int c = 0; c < 3; ++c) {
    int v00 = 0, v01 = 0, v10 = 0, v11 = 0;
    if (y0) {
      if (x0) v00 = px(0, iy, ix, c);
      if (x1) v01 = px(1, iy, ix + 1, c);
    }
    if (y1) {
      if (x0) v10 = px(2, iy + 1, ix, c);
      if (x1) v11 = px(3, iy + 1, ix + 1, c);
    }
    int u8 = (v00 * w00 + v01 * w01 + v10 * w10 + v11 * w11 + (1 << 14)) >> 15;
    u8 = max(0, min(255, u8));
    const double r = ((double)u8 / 255.0 - (double)mean[c]) / (double)stdv[c];
    out[c * plane] = (float)r;
    prev(c, (float)r);
  }
}

// interleaved 8-bit pixels of kBytes (3 or 4) bytes with B, G and R at bytes kB, kG and kR: BGR <0, 1, 2>, RGB24 and
// RGBA <2, 1, 0>, BGRA <0, 1, 2> (cv2.cvtColor COLOR_RGB2BGR / COLOR_RGBA2BGR / COLOR_BGRA2BGR are these channel
// selects; alpha is never read).  Every channel is read where it is used.
template <int kBytes, int kB, int kG, int kR>
struct PackedFetch {
  const uint8_t* __restrict__ img;
  int sw;
  __device__ __forceinline__ void taps(int, int, bool, bool, bool, bool) {}
  __device__ __forceinline__ int operator()(int, int yy, int xx, int c) const {
    return img[((size_t)yy * sw + xx) * kBytes + (c == 0 ? kB : (c == 1 ? kG : kR))];
  }
};

// YUV frames converted per tap to the BGR that cv2.cvtColor gives, restated bit for bit (OpenCV color_yuv.simd.hpp,
// 8-bit: BT.601 limited range in 20-bit fixed point, no chroma interpolation; tests/yuv_ref.py and tests/yuv422_ref.py,
// pinned against cv2 on every (Y, U, V)):
//   y = max(Y - 16, 0) * 1220542 + 2^19, u = U - 128, v = V - 128
//   B = sat((y + 2116026 u) >> 20), G = sat((y - 852492 v - 409993 u) >> 20), R = sat((y + 1673527 v) >> 20)
// 4:2:0 (COLOR_YUV2BGR_NV12 / _I420) [3 sh / 2, sw] (sh, sw even): the Y plane [sh, sw] comes first; then NV12: U, V
// interleaved, row yy / 2, bytes (xx & ~1) and (xx | 1); I420: the U plane [sh/2, sw/2], then the V plane [sh/2, sw/2].
// kVFirst swaps the chroma: V, U interleaved (NV21, COLOR_YUV2BGR_NV21) or the V plane first (YV12, COLOR_YUV2BGR_YV12).
// kFull: full range (JFIF), with no cv2 4:2:0 code: the same 2x2 chroma, then cv2's COLOR_YCrCb2BGR in 14-bit fixed
// point (tests/phone_ref.py, pinned against cv2 on every (Y, Cr, Cb)):
//   B = sat(Y + ((29049 u + 2^13) >> 14)), G = sat(Y + ((-11698 v - 5636 u + 2^13) >> 14)), R = sat(Y + ((22987 v + 2^13) >> 14))
// Packed 4:2:2 (COLOR_YUV2BGR_YUYV / _UYVY) [sh, sw, 2] (sw even): the pixel pair (xx & ~1, xx | 1) of a row is 4 bytes,
// Y0 U Y1 V (YUYV) or U Y0 V Y1 (UYVY), one U, V for both pixels.  Every in-frame tap is read and converted once, before
// the first channel is written; taps outside stay BGR 0, warpAffine's border of the converted image.
template <int kLayout, bool kVFirst = false, bool kFull = false>
struct YuvFetch {
  const uint8_t* __restrict__ img;
  int sh, sw;
  int yv[4], u[4], v[4];      // per tap: max(Y - 16, 0) * 1220542 + 2^19 (kFull: Y), U - 128, V - 128
  __device__ __forceinline__ void taps(int iy, int ix, bool in00, bool in01, bool in10, bool in11) {
    const bool in[4] = {in00, in01, in10, in11};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      yv[k] = u[k] = v[k] = 0;
      if (!in[k]) continue;
      const int yy = iy + (k >> 1), xx = ix + (k & 1);
      int Y, U, V;
      if constexpr (kLayout == CP_PIX_NV12 || kLayout == CP_PIX_I420) {
        const uint8_t* __restrict__ chroma = img + (size_t)sh * sw;
        if constexpr (kLayout == CP_PIX_NV12) {
          const size_t o = (size_t)(yy >> 1) * sw + (xx & ~1);
          U = chroma[o + kVFirst];
          V = chroma[o + !kVFirst];
        } else {
          const size_t o = (size_t)(yy >> 1) * (sw >> 1) + (xx >> 1);
          if constexpr (kVFirst) {
            V = chroma[o];
            U = chroma[(size_t)(sh >> 1) * (sw >> 1) + o];
          } else {
            U = chroma[o];
            V = chroma[(size_t)(sh >> 1) * (sw >> 1) + o];
          }
        }
        Y = img[(size_t)yy * sw + xx];
      } else {
        constexpr int kY = kLayout == CP_PIX_YUYV422 ? 0 : 1, kU = 1 - kY;    // byte of Y0 and of U in a pair
        const uint8_t* __restrict__ pair = img + ((size_t)yy * sw + (xx & ~1)) * 2;
        Y = pair[kY + 2 * (xx & 1)];
        U = pair[kU];
        V = pair[kU + 2];
      }
      yv[k] = kFull ? Y : max(Y - 16, 0) * 1220542 + (1 << 19);
      u[k] = U - 128;
      v[k] = V - 128;
    }
  }
  __device__ __forceinline__ int operator()(int k, int, int, int c) const {
    if constexpr (kFull) {
      const int t = c == 0 ? 29049 * u[k] : (c == 1 ? -11698 * v[k] - 5636 * u[k] : 22987 * v[k]);
      return max(0, min(255, yv[k] + ((t + (1 << 13)) >> 14)));
    } else {
      const int t = c == 0 ? yv[k] + 2116026 * u[k]
                           : (c == 1 ? yv[k] - 852492 * v[k] - 409993 * u[k] : yv[k] + 1673527 * v[k]);
      return max(0, min(255, t >> 20));
    }
  }
};

// Bayer mosaics [sh, sw] (sh, sw >= 3) demosaiced per tap to the BGR that cv2.cvtColor's bilinear COLOR_Bayer??2BGR
// gives, restated bit for bit (tests/bayer_ref.py, pinned against cv2).  The four patterns are one fetch with a phase
// (py, px): pixel (y, x) of the frame's pattern is pixel (y + py, x + px) of R G / G B, so rggb is (0, 0), grbg (0, 1),
// gbrg (1, 0) and bggr (1, 1).  An interior pixel keeps its own channel and takes
//   at R or B: G = (N + S + W + E + 2) >> 2, the other chroma = (NW + NE + SW + SE + 2) >> 2;
//   at G: the chroma of its row's other sites = (W + E + 1) >> 1, that of its column's = (N + S + 1) >> 1;
// and an in-frame border pixel (y, x) takes the BGR of interior pixel (clamp(y, 1, sh - 2), clamp(x, 1, sw - 2)).
// The clamped 3 x 3 neighbourhoods of the four taps lie in one window of at most 4 x 4 bytes, read once; every in-frame
// tap is demosaiced from it before the first channel is written, taps outside stay BGR 0.
struct BayerFetch {
  const uint8_t* __restrict__ img;
  int sh, sw;
  int py, px;
  int b[4], g[4], r[4];
  __device__ __forceinline__ void taps(int iy, int ix, bool in00, bool in01, bool in10, bool in11) {
    const bool in[4] = {in00, in01, in10, in11};
#pragma unroll
    for (int k = 0; k < 4; ++k) b[k] = g[k] = r[k] = 0;
    if (!(in00 || in01 || in10 || in11)) return;
    // the clamped centres of the tap rows and columns; the window starts one row and column before the first
    const int cy0 = max(1, min(sh - 2, iy)), cy1 = max(1, min(sh - 2, iy + 1));
    const int cx0 = max(1, min(sw - 2, ix)), cx1 = max(1, min(sw - 2, ix + 1));
    const int r0 = cy0 - 1, c0 = cx0 - 1;
    // rows r0 .. r0 + 3, bytes c0 .. c0 + 3 (byte j of a word is column c0 + j); the fourth row and column are needed
    // only where they are in the frame, so their reads are clamped into it
    uint32_t win[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint8_t* __restrict__ row = img + (size_t)min(r0 + j, sh - 1) * sw + c0;
      win[j] = row[0] | (uint32_t)row[1] << 8 | (uint32_t)row[2] << 16 | (uint32_t)row[min(3, sw - 1 - c0)] << 24;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (!in[k]) continue;
      const int cy = k >> 1 ? cy1 : cy0, cx = k & 1 ? cx1 : cx0;
      const bool down = cy != cy0;                     // the neighbourhood's rows are window rows 1..3, else 0..2
      const int sh8 = 8 * (cx - c0 - 1);               // and its columns start at byte cx - c0 - 1
      const uint32_t N = (down ? win[1] : win[0]) >> sh8, C = (down ? win[2] : win[1]) >> sh8,
                     S = (down ? win[3] : win[2]) >> sh8;
      const int n_w = N & 255, n = N >> 8 & 255, n_e = N >> 16 & 255, w = C & 255, c = C >> 8 & 255, e = C >> 16 & 255,
                s_w = S & 255, s = S >> 8 & 255, s_e = S >> 16 & 255;
      const bool even_row = ((cy + py) & 1) == 0, chroma = ((cy + py + cx + px) & 1) == 0;
      // own: the chroma of the row's colour (R on an R G row), other: the other chroma
      const int own = chroma ? c : (w + e + 1) >> 1;
      const int other = chroma ? (n_w + n_e + s_w + s_e + 2) >> 2 : (n + s + 1) >> 1;
      g[k] = chroma ? (n + s + w + e + 2) >> 2 : c;
      r[k] = even_row ? own : other;
      b[k] = even_row ? other : own;
    }
  }
  __device__ __forceinline__ int operator()(int k, int, int, int c) const { return c == 0 ? b[k] : (c == 1 ? g[k] : r[k]); }
};
__device__ __forceinline__ BayerFetch bayer_fetch(const uint8_t* __restrict__ img, int sh, int sw, int format) {
  return BayerFetch{img, sh, sw, format == CP_PIX_BAYER_BGGR8 || format == CP_PIX_BAYER_GBRG8,
                    format == CP_PIX_BAYER_BGGR8 || format == CP_PIX_BAYER_GRBG8};
}

// A BGR frame [sh, sw] served as cv2.resize(frame, (rw, rh)) (INTER_LINEAR) gives it, restated bit for bit (OpenCV
// resize.cpp, INTER_RESIZE_COEF_BITS = 11; tests/resize_ref.py, pinned against cv2): the walk runs over the [rh, rw]
// resized image, and every in-frame tap is resized from its 2 x 2 source pixels once, before the first channel is
// written; taps outside stay BGR 0.  Per axis, with cv2's inverse scale (the host's 1 / (dst / src) in double),
// destination index d takes f = (float)((d + 0.5) scale - 0.5), s = floor(f), f -= s and the weights
// a0 = rne((1 - f) 2048), a1 = rne(f 2048) (float32 products).  Across, s < 0 or s >= sw - 1 puts s at the nearest
// column with weights (2048, 0), and S = src[s] a0 + src[s + 1] a1.  Down, f is kept and the rows s and s + 1 are each
// clamped into the frame (clamping f as across is off by one on the first and last rows of an upscale); the pixel is
// sat((((b0 (S0 >> 4)) >> 16) + ((b1 (S1 >> 4)) >> 16) + 2) >> 2), cv2's VResizeLinear<uchar>.
struct ResizeFetch {
  const uint8_t* __restrict__ img;
  int sh, sw;                          // the source frame
  double scale_x, scale_y;
  int bgr[4][3];
  // the first source index of destination index d on an axis of inverse scale `scale`, and its two weights
  static __device__ __forceinline__ int axis(int d, double scale, int& a0, int& a1) {
    // unfused double arithmetic, as in the host code
    float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
    const float s = floorf(f);
    f = __fsub_rn(f, s);
    a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
    a1 = __float2int_rn(__fmul_rn(f, 2048.f));
    return (int)s;
  }
  __device__ __forceinline__ void taps(int iy, int ix, bool in00, bool in01, bool in10, bool in11) {
    const bool in[4] = {in00, in01, in10, in11};
    int x0[2], x1[2], a0[2], a1[2], y0[2], y1[2], b0[2], b1[2];   // [j]: column ix + j, row iy + j
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      int s = axis(ix + j, scale_x, a0[j], a1[j]);
      if (s < 0 || s >= sw - 1) {
        s = s < 0 ? 0 : sw - 1;
        a0[j] = 2048;
        a1[j] = 0;
      }
      x0[j] = s * 3;
      x1[j] = min(s + 1, sw - 1) * 3;
      s = axis(iy + j, scale_y, b0[j], b1[j]);
      y0[j] = max(0, min(sh - 1, s));
      y1[j] = max(0, min(sh - 1, s + 1));
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      bgr[k][0] = bgr[k][1] = bgr[k][2] = 0;
      if (!in[k]) continue;
      const int j = k >> 1, i = k & 1;
      const uint8_t* __restrict__ r0 = img + (size_t)y0[j] * sw * 3;
      const uint8_t* __restrict__ r1 = img + (size_t)y1[j] * sw * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int S0 = r0[x0[i] + c] * a0[i] + r0[x1[i] + c] * a1[i];
        const int S1 = r1[x0[i] + c] * a0[i] + r1[x1[i] + c] * a1[i];
        bgr[k][c] = max(0, min(255, (((b0[j] * (S0 >> 4)) >> 16) + ((b1[j] * (S1 >> 4)) >> 16) + 2) >> 2));
      }
    }
  }
  __device__ __forceinline__ int operator()(int k, int, int, int c) const { return bgr[k][c]; }
};

// The eight 4:2:0 codes: NV12, I420, and 8 plus the bits 1 (planar), 2 (V first) and 4 (full range) for the others.
__host__ __device__ constexpr bool is_yuv420(int format) {
  return format == CP_PIX_NV12 || format == CP_PIX_I420 || (format >= CP_PIX_NV21 && format <= CP_PIX_YV12_FULL);
}

// The bytes of one sh x sw frame in a cp_pixel_format (0 for CP_PIX_PER_FRAME or an unknown value).
__host__ __device__ constexpr size_t frame_bytes(int format, size_t sh, size_t sw) {
  return is_yuv420(format)                                 ? sh * sw * 3 / 2
         : format == CP_PIX_BGR || format == CP_PIX_RGB24    ? sh * sw * 3
         : format == CP_PIX_RGBA || format == CP_PIX_BGRA    ? sh * sw * 4
         : format == CP_PIX_YUYV422 || format == CP_PIX_UYVY422 ? sh * sw * 2
         : format >= CP_PIX_GRAY && format <= CP_PIX_BAYER_GRBG8 ? sh * sw
                                                             : 0;
}

// the tap fetch of a frame at img in format kFormat
template <int kFormat>
__device__ __forceinline__ auto make_fetch(const uint8_t* __restrict__ img, int sh, int sw) {
  if constexpr (kFormat == CP_PIX_BGR || kFormat == CP_PIX_BGRA)
    return PackedFetch<kFormat == CP_PIX_BGR ? 3 : 4, 0, 1, 2>{img, sw};
  else if constexpr (kFormat == CP_PIX_RGB24 || kFormat == CP_PIX_RGBA)
    return PackedFetch<kFormat == CP_PIX_RGB24 ? 3 : 4, 2, 1, 0>{img, sw};
  else if constexpr (kFormat == CP_PIX_GRAY)
    return PackedFetch<1, 0, 0, 0>{img, sw};           // COLOR_GRAY2BGR: B = G = R = Y
  else if constexpr (kFormat >= CP_PIX_BAYER_RGGB8 && kFormat <= CP_PIX_BAYER_GRBG8)
    return bayer_fetch(img, sh, sw, kFormat);
  else if constexpr (is_yuv420(kFormat))
    return YuvFetch<kFormat & 1 ? CP_PIX_I420 : CP_PIX_NV12, (kFormat & 2) != 0, (kFormat & 4) != 0>{img, sh, sw};
  else
    return YuvFetch<kFormat>{img, sh, sw};
}

// per-frame parameters of a frame table
struct RaggedFrame {
  WarpM W;
  long long offset;     // bytes into the packed frame buffer
  int sh, sw;
};

// A table of per-frame formats (launched as CP_PIX_PER_FRAME) keeps frame b's cp_pixel_format in the top byte of its
// offset, so its entries are RaggedFrames of the same 64 bytes and a walk still reads one entry per output pixel.
constexpr int kFormatShift = 56;
constexpr long long kOffsetMask = (1ll << kFormatShift) - 1;
// A mapped frame (a table of cp_preprocess_frame_table_maps, launched with CP_PIX_REMAP) sets bit 6 of that byte, above
// every format, and keeps the device address of its coordinate map, float2 [dh, dw], in the bits of W.m[0]; the rest
// of W is unused.  Unmapped frames of the same table keep their affine.
constexpr long long kMappedFlag = 1ll << (kFormatShift + 6);
__device__ __forceinline__ const float2* frame_map(const RaggedFrame& f) {
  return reinterpret_cast<const float2*>(__double_as_longlong(f.W.m[0]));
}

// walk(fetch) with the tap fetch of frame f in the format of launch code kCode (a cp_pixel_format or CP_PIX_PER_FRAME,
// with or without CP_PIX_REMAP); CP_PIX_PER_FRAME: in the format its entry holds.  The format is uniform across a frame,
// so the branch costs a frame's threads nothing but the switch.  Only the CP_PIX_REMAP instances mask the mapped flag.
template <int kCode, class Walk>
__device__ __forceinline__ void frame_walk(const uint8_t* __restrict__ frames, const RaggedFrame& f, Walk walk) {
  constexpr bool kRemap = kCode & CP_PIX_REMAP;
  constexpr int kFormat = kCode & ~CP_PIX_REMAP;
  if constexpr (kFormat != CP_PIX_PER_FRAME) {
    walk(make_fetch<kFormat>(frames + (kRemap ? f.offset & kOffsetMask : f.offset), f.sh, f.sw));
  } else {
    const uint8_t* img = frames + (f.offset & kOffsetMask);
    const int format = kRemap ? (int)((f.offset & ~kMappedFlag) >> kFormatShift) : (int)(f.offset >> kFormatShift);
    switch (format) {
      case CP_PIX_NV12: walk(make_fetch<CP_PIX_NV12>(img, f.sh, f.sw)); break;
      case CP_PIX_I420: walk(make_fetch<CP_PIX_I420>(img, f.sh, f.sw)); break;
      case CP_PIX_NV21: walk(make_fetch<CP_PIX_NV21>(img, f.sh, f.sw)); break;
      case CP_PIX_YV12: walk(make_fetch<CP_PIX_YV12>(img, f.sh, f.sw)); break;
      case CP_PIX_NV12_FULL: walk(make_fetch<CP_PIX_NV12_FULL>(img, f.sh, f.sw)); break;
      case CP_PIX_I420_FULL: walk(make_fetch<CP_PIX_I420_FULL>(img, f.sh, f.sw)); break;
      case CP_PIX_NV21_FULL: walk(make_fetch<CP_PIX_NV21_FULL>(img, f.sh, f.sw)); break;
      case CP_PIX_YV12_FULL: walk(make_fetch<CP_PIX_YV12_FULL>(img, f.sh, f.sw)); break;
      case CP_PIX_BGR: walk(make_fetch<CP_PIX_BGR>(img, f.sh, f.sw)); break;
      case CP_PIX_RGB24: walk(make_fetch<CP_PIX_RGB24>(img, f.sh, f.sw)); break;
      case CP_PIX_RGBA: walk(make_fetch<CP_PIX_RGBA>(img, f.sh, f.sw)); break;
      case CP_PIX_BGRA: walk(make_fetch<CP_PIX_BGRA>(img, f.sh, f.sw)); break;
      case CP_PIX_YUYV422: walk(make_fetch<CP_PIX_YUYV422>(img, f.sh, f.sw)); break;
      case CP_PIX_UYVY422: walk(make_fetch<CP_PIX_UYVY422>(img, f.sh, f.sw)); break;
      case CP_PIX_GRAY: walk(make_fetch<CP_PIX_GRAY>(img, f.sh, f.sw)); break;
      case CP_PIX_BAYER_RGGB8:
      case CP_PIX_BAYER_BGGR8:
      case CP_PIX_BAYER_GBRG8:
      case CP_PIX_BAYER_GRBG8: walk(bayer_fetch(img, f.sh, f.sw, format)); break;   // one walk, the phase at run time
      default: break;                                  // no table the host builds holds another value
    }
  }
}

// The arguments of preprocess_kernel.  Every one is a kernel argument or device memory, so a captured launch replays
// unchanged.
struct PreprocessArgs {
  const uint8_t* frames;
  const RaggedFrame* fr;     // the table form: row n is slot s = rows ? rows[n] : n, its frame fr[s]
  const int* rows;
  WarpM W;                   // the uniform form: one sh x sw frame per row, frame n at byte n * frame_bytes
  int sh, sw;
  int B, dh, dw;
  float mean[3], stdv[3];
  const int* start;          // the previous frame (PrevMode): prev null: none; store null: the twin (start[s]: a slot
  float* store;              // beginning a video); else the exchange (the live rows name distinct slots)
  float* prev;
  float* out;
  int rh, rw;                // kResizeBgr: the size the frame is resized to, and cv2's inverse scales of the two axes
  double scale_x, scale_y;
};

// The launch code of cp_preprocess_resize_affine (internal, not a cp_pixel_format): the uniform form over BGR frames
// served through ResizeFetch, without previous frames.
constexpr int kResizeBgr = 256 | CP_PIX_BGR;

// The previous-frame writes of a launch (PreprocessArgs): none; the twin, prev[n] = the value where start[s] is set;
// the exchange, prev[n] = start[s] ? value : store[s], then store[s] = value.  The mode is a template parameter, so a
// launch without previous frames runs the walk alone and each mode keeps the registers it needs by itself.
enum PrevMode { kNoPrev, kTwin, kExchange };

// B rows of [3, dh, dw]: row n is frame n (uniform) or the frame of slot s through the table (kTable), in format
// kFormat (CP_PIX_PER_FRAME: each table entry's own).  Every thread is one output pixel of one row, grid-stride, and
// reads and writes only its own elements.  kFormat | CP_PIX_REMAP (table form only): a mapped entry takes its source
// position from its coordinate map at the output pixel, an unmapped one from its affine.  kResizeBgr (uniform form):
// frame n is BGR [a.sh, a.sw] and the walk runs over its resize to [a.rh, a.rw] (ResizeFetch).
template <int kFormat, bool kTable, PrevMode kMode>
__global__ void preprocess_kernel(const PreprocessArgs a) {
  static_assert(kTable || !(kFormat & CP_PIX_REMAP), "coordinate maps come through a frame table");
  const size_t plane = (size_t)a.dh * a.dw, total = (size_t)a.B * plane;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % a.dw);
    const size_t t = i / a.dw;
    const int y = (int)(t % a.dh);
    const int n = (int)(t / a.dh);
    int s = n;
    RaggedFrame f;
    if constexpr (kTable) {
      if (kMode == kExchange || a.rows) s = a.rows[n];      // the exchange is the rows form's only
      f = a.fr[s];
    } else if constexpr (kFormat == kResizeBgr) {
      f = RaggedFrame{a.W, (long long)n * a.sh * a.sw * 3, a.rh, a.rw};   // the walk's frame is the resized image
    } else {
      f = RaggedFrame{a.W, (long long)(n * frame_bytes(kFormat, a.sh, a.sw)), a.sh, a.sw};
    }
    const size_t px = (size_t)y * a.dw + x, o = (size_t)n * 3 * plane + px;
    const bool start = kMode != kNoPrev && a.start && a.start[s];
    float* prev = a.prev + o;
    float* store = a.store + (size_t)s * 3 * plane + px;
    // a mapped launch reads the map before the format switch; the others generate the affine position inside it
    int2 mapped{};
    if constexpr ((kFormat & CP_PIX_REMAP) != 0)
      mapped = f.offset & kMappedFlag ? map_pos(frame_map(f)[px]) : affine_pos(f.W, x, y);
    const auto walk = [&](auto fetch) {
      const int2 pos = [&] {
        if constexpr ((kFormat & CP_PIX_REMAP) != 0)
          return mapped;
        else
          return affine_pos(f.W, x, y);
      }();
      warp_walk(fetch, a.out + o, plane, f.sh, f.sw, pos, a.mean, a.stdv, [&](int c, float v) {
        if constexpr (kMode == kTwin) {
          if (start) prev[c * plane] = v;
        } else if constexpr (kMode == kExchange) {
          prev[c * plane] = start ? v : store[c * plane];
          store[c * plane] = v;
        }
      });
    };
    if constexpr (kFormat == kResizeBgr)
      walk(ResizeFetch{a.frames + f.offset, a.sh, a.sw, a.scale_x, a.scale_y});
    else
      frame_walk<kFormat>(a.frames, f, walk);
  }
}

// dst row i = src row map[i], or zeros where map[i] < 0; rows of `words` 32-bit words
__global__ void gather_rows_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, size_t words, int n,
                                  const int* __restrict__ map) {
  const size_t total = (size_t)n * words;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int r = map[i / words];
    dst[i] = r >= 0 ? src[(size_t)r * words + i % words] : 0u;
  }
}

// cv::warpAffine inverts the forward matrix like this (imgwarp.cpp), in double, before the fixed-point walk
WarpM invert_affine(const double* trans_input) {
  WarpM W;
  double* M = W.m;
  for (int i = 0; i < 6; ++i) M[i] = trans_input[i];
  double D = M[0] * M[4] - M[1] * M[3];
  D = D != 0 ? 1. / D : 0;
  const double A11 = M[4] * D, A22 = M[0] * D;
  M[0] = A11;
  M[1] *= -D;
  M[3] *= -D;
  M[4] = A22;
  const double b1 = -M[0] * M[2] - M[1] * M[5];
  const double b2 = -M[3] * M[2] - M[4] * M[5];
  M[2] = b1;
  M[5] = b2;
  return W;
}

// fix_res affine of base_detector.py:109-121 (c = frame centre, s = max side, rot 0) in closed form: the float32 control
// points of utils/image.py:35-68 give an isotropic scale a = dst_w / s.  (cv2.getAffineTransform solves the same three
// point pairs by LU; the two agree to <= 3e-14, which the fixed-point walk cannot see except on exact rounding ties.
// Callers that hold the reference's own `trans_input` pass it to cp_preprocess_affine.)
void fix_res_affine(int src_h, int src_w, int dst_h, int dst_w, double T[6]) {
  const float cx = (float)(src_w / 2.0), cy = (float)(src_h / 2.0);
  const float s = (float)(src_h > src_w ? src_h : src_w);
  const float src1y = cy + s * -0.5f;                               // float32 control points
  const float dst0x = (float)(dst_w * 0.5), dst0y = (float)(dst_h * 0.5);
  const float dst1y = dst0y + (float)(dst_w * -0.5);
  const double a = ((double)dst1y - (double)dst0y) / ((double)src1y - (double)cy);
  T[0] = a;
  T[1] = 0.0;
  T[2] = (double)dst0x - a * (double)cx;
  T[3] = 0.0;
  T[4] = a;
  T[5] = (double)dst0y - a * (double)cy;
}

int preprocess_blocks(size_t total) {
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  return blocks;
}

bool is_yuv422(int format) { return format == CP_PIX_YUYV422 || format == CP_PIX_UYVY422; }
bool is_bayer(int format) { return format >= CP_PIX_BAYER_RGGB8 && format <= CP_PIX_BAYER_GRBG8; }
bool known_format(int format) {
  return format == CP_PIX_BGR || is_yuv420(format) || format == CP_PIX_RGB24 || format == CP_PIX_RGBA ||
         format == CP_PIX_BGRA || is_yuv422(format) || format == CP_PIX_GRAY || is_bayer(format);
}

// a launch code of a frame table: a cp_pixel_format or CP_PIX_PER_FRAME, either with or without CP_PIX_REMAP
bool table_code(int code) {
  const int format = code & ~CP_PIX_REMAP;
  return code >= 0 && (known_format(format) || format == CP_PIX_PER_FRAME);
}

// f(std::integral_constant<int, format>) for a format chosen at run time (one of cp_pixel_format or
// CP_PIX_PER_FRAME), already checked
template <class F>
void with_base_format(int format, F f) {
  switch (format) {
    case CP_PIX_NV12: f(std::integral_constant<int, CP_PIX_NV12>{}); break;
    case CP_PIX_I420: f(std::integral_constant<int, CP_PIX_I420>{}); break;
    case CP_PIX_NV21: f(std::integral_constant<int, CP_PIX_NV21>{}); break;
    case CP_PIX_YV12: f(std::integral_constant<int, CP_PIX_YV12>{}); break;
    case CP_PIX_NV12_FULL: f(std::integral_constant<int, CP_PIX_NV12_FULL>{}); break;
    case CP_PIX_I420_FULL: f(std::integral_constant<int, CP_PIX_I420_FULL>{}); break;
    case CP_PIX_NV21_FULL: f(std::integral_constant<int, CP_PIX_NV21_FULL>{}); break;
    case CP_PIX_YV12_FULL: f(std::integral_constant<int, CP_PIX_YV12_FULL>{}); break;
    case CP_PIX_BGR: f(std::integral_constant<int, CP_PIX_BGR>{}); break;
    case CP_PIX_RGB24: f(std::integral_constant<int, CP_PIX_RGB24>{}); break;
    case CP_PIX_RGBA: f(std::integral_constant<int, CP_PIX_RGBA>{}); break;
    case CP_PIX_BGRA: f(std::integral_constant<int, CP_PIX_BGRA>{}); break;
    case CP_PIX_YUYV422: f(std::integral_constant<int, CP_PIX_YUYV422>{}); break;
    case CP_PIX_UYVY422: f(std::integral_constant<int, CP_PIX_UYVY422>{}); break;
    case CP_PIX_GRAY: f(std::integral_constant<int, CP_PIX_GRAY>{}); break;
    case CP_PIX_BAYER_RGGB8: f(std::integral_constant<int, CP_PIX_BAYER_RGGB8>{}); break;
    case CP_PIX_BAYER_BGGR8: f(std::integral_constant<int, CP_PIX_BAYER_BGGR8>{}); break;
    case CP_PIX_BAYER_GBRG8: f(std::integral_constant<int, CP_PIX_BAYER_GBRG8>{}); break;
    case CP_PIX_BAYER_GRBG8: f(std::integral_constant<int, CP_PIX_BAYER_GRBG8>{}); break;
    default: f(std::integral_constant<int, CP_PIX_PER_FRAME>{});
  }
}

// with_base_format for a launch code, already checked: a table code with CP_PIX_REMAP gives its own constant
template <class F>
void with_format(int code, F f) {
  if (code & CP_PIX_REMAP)
    with_base_format(code & ~CP_PIX_REMAP,
                     [&](auto k) { f(std::integral_constant<int, decltype(k)::value | CP_PIX_REMAP>{}); });
  else
    with_base_format(code, f);
}

// the arguments every form of preprocess_kernel takes; the entry points fill in the frame source and previous frame
PreprocessArgs preprocess_args(const uint8_t* frames, float* out, int B, int dh, int dw, const float mean[3],
                               const float stdv[3]) {
  PreprocessArgs a{};
  a.frames = frames;
  a.out = out;
  a.B = B;
  a.dh = dh;
  a.dw = dw;
  for (int c = 0; c < 3; ++c) {
    a.mean[c] = mean[c];
    a.stdv[c] = stdv[c];
  }
  return a;
}

// enqueues preprocess_kernel in `format`: the table form when a.fr is set (which may also be CP_PIX_PER_FRAME, carry
// CP_PIX_REMAP and take the store exchange, with rows), else the uniform form; the previous-frame mode is the one a's
// pointers select; kResizeBgr: its one instance, uniform without previous frames
int launch_preprocess(int format, const PreprocessArgs& a, cudaStream_t s) {
  const int blocks = preprocess_blocks((size_t)a.B * a.dh * a.dw);
  if (format == kResizeBgr && !a.fr && !a.prev) {
    preprocess_kernel<kResizeBgr, false, kNoPrev><<<blocks, 256, 0, s>>>(a);
    CP_LAUNCH_CHECK("preprocess_kernel");
    return CP_OK;
  }
  if (a.fr ? !table_code(format) || (a.store && !a.rows) : !known_format(format) || a.store)
    return fail(CP_ERR_INVALID, "preprocess_kernel: no instance for pixel format " + std::to_string(format) +
                                    (a.fr ? " over a frame table" : " over a uniform batch") +
                                    (a.store ? " with a store" : ""));
  const PrevMode mode = !a.prev ? kNoPrev : !a.store ? kTwin : kExchange;
  with_format(format, [&](auto k) {
    constexpr int kFormat = decltype(k)::value;
    if (a.fr) {
      if (mode == kNoPrev)
        preprocess_kernel<kFormat, true, kNoPrev><<<blocks, 256, 0, s>>>(a);
      else if (mode == kTwin)
        preprocess_kernel<kFormat, true, kTwin><<<blocks, 256, 0, s>>>(a);
      else
        preprocess_kernel<kFormat, true, kExchange><<<blocks, 256, 0, s>>>(a);
    } else if constexpr (kFormat != CP_PIX_PER_FRAME && !(kFormat & CP_PIX_REMAP)) {
      if (mode == kNoPrev)
        preprocess_kernel<kFormat, false, kNoPrev><<<blocks, 256, 0, s>>>(a);
      else
        preprocess_kernel<kFormat, false, kTwin><<<blocks, 256, 0, s>>>(a);
    }
  });
  CP_LAUNCH_CHECK("preprocess_kernel");
  return CP_OK;
}

// The per-frame parameters of a ragged batch, checked against the packed buffer before any work is enqueued.  Frame b
// is in `format` (a cp_pixel_format), or in formats[b] when `formats` (host int32 [B]) is given; then each entry's
// offset also carries the frame's format (kFormatShift), for a CP_PIX_PER_FRAME launch.  maps (host, B device
// pointers, or NULL): frame b with maps[b] set is a mapped entry (kMappedFlag), for a CP_PIX_REMAP launch.
int ragged_frames(const char* who, int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw, int B, int dst_h,
                  int dst_w, const double* trans_input, int format, const int32_t* formats, std::vector<RaggedFrame>& fr,
                  const float* const* maps = nullptr) {
  const std::string w0 = who;
  if ((formats || maps) && frames_bytes > kOffsetMask)
    return fail(CP_ERR_INVALID, w0 + ": a " + std::to_string(frames_bytes) + "-byte buffer is too large for per-frame "
                                "formats or maps");
  fr.resize(B);
  for (int b = 0; b < B; ++b) {
    const int h = src_hw[2 * b], w = src_hw[2 * b + 1];
    const int fmt = formats ? formats[b] : format;
    if (!known_format(fmt))
      return fail(CP_ERR_INVALID, w0 + ": frame " + std::to_string(b) + " has unknown pixel format " +
                                      std::to_string(fmt));
    const bool yuv = is_yuv420(fmt);
    if (h <= 0 || w <= 0 || (yuv && (h % 2 || w % 2)) || (is_yuv422(fmt) && w % 2) ||
        (is_bayer(fmt) && (h < 3 || w < 3)))
      return fail(CP_ERR_INVALID, w0 + ": frame " + std::to_string(b) + " has size " + std::to_string(h) + " x " +
                                      std::to_string(w) + (yuv ? " (YUV 4:2:0 needs even sizes)"
                                                           : is_yuv422(fmt) ? " (YUV 4:2:2 needs an even width)"
                                                           : is_bayer(fmt) ? " (a Bayer mosaic needs at least 3 x 3)" : ""));
    const int64_t bytes = (int64_t)frame_bytes(fmt, h, w);
    if (offsets[b] < 0 || offsets[b] > frames_bytes || bytes > frames_bytes - offsets[b])
      return fail(CP_ERR_INVALID, w0 + ": frame " + std::to_string(b) + " (" + std::to_string(h) + " x " +
                                      std::to_string(w) + " at byte " + std::to_string(offsets[b]) +
                                      ") lies outside the " + std::to_string(frames_bytes) + "-byte buffer");
    double T[6];
    if (trans_input) {
      for (int i = 0; i < 6; ++i) T[i] = trans_input[6 * b + i];
    } else {
      fix_res_affine(h, w, dst_h, dst_w, T);
    }
    fr[b].W = invert_affine(T);
    fr[b].offset = formats ? offsets[b] | (long long)fmt << kFormatShift : offsets[b];
    fr[b].sh = h;
    fr[b].sw = w;
    if (maps && maps[b]) {
      if ((uintptr_t)maps[b] % alignof(float2))
        return fail(CP_ERR_INVALID, w0 + ": the map of frame " + std::to_string(b) + " is not 8-byte aligned");
      const long long addr = (long long)(uintptr_t)maps[b];
      std::memcpy(&fr[b].W.m[0], &addr, sizeof addr);
      fr[b].offset |= kMappedFlag;
    }
  }
  return CP_OK;
}

// uploads the frame table `fr` (stream-ordered) and enqueues the table form of preprocess_kernel over it
int launch_ragged(const char* who, int format, const std::vector<RaggedFrame>& fr, PreprocessArgs a, cudaStream_t s) {
  RaggedFrame* dfr = nullptr;
  CP_CUDA_CHECK(cudaMallocAsync(&dfr, sizeof(RaggedFrame) * fr.size(), s));
  int rc;
  // a pageable source: the bytes are staged before cudaMemcpyAsync returns, so `fr` may go out of scope
  if (cudaMemcpyAsync(dfr, fr.data(), sizeof(RaggedFrame) * fr.size(), cudaMemcpyHostToDevice, s) != cudaSuccess) {
    rc = fail(CP_ERR_CUDA, std::string(who) + ": parameter upload");
  } else {
    a.fr = dfr;
    rc = launch_preprocess(format, a, s);
  }
  cudaFreeAsync(dfr, s);
  return rc;
}

// checks a frame table's frames (ragged_frames) and writes it to `table`
int upload_frame_table(const char* who, int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw, int format,
                       const int32_t* formats, int B, int dst_h, int dst_w, const double* trans_input, void* table,
                       void* stream_, const float* const* maps = nullptr) {
  std::vector<RaggedFrame> fr;
  int rc = ragged_frames(who, frames_bytes, offsets, src_hw, B, dst_h, dst_w, trans_input, format, formats, fr, maps);
  if (rc) return rc;
  // a build-time call: the copy is complete when it returns, so `fr` may go out of scope
  cudaStream_t s = (cudaStream_t)stream_;
  cudaError_t e = cudaMemcpyAsync(table, fr.data(), sizeof(RaggedFrame) * B, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return fail(CP_ERR_CUDA, std::string(who) + ": table upload: " + cudaGetErrorString(e));
  return CP_OK;
}

}  // namespace

int dcn_v2_backward_impl(const float* input, const float* weight, const float* offset, const float* mask,
                         const float* grad_output, float* grad_input, float* grad_offset, float* grad_mask,
                         float* grad_weight, float* grad_bias, int B, int C, int H, int W, int Co,
                         int32_t precision, cudaStream_t s);      // dcn_bwd.cu
}  // namespace cp

using namespace cp;

// cp_conv2d / cp_dcn_v2_forward_ex store unrounded outputs and fail when a tensor-core precision has no kernel for the shape
constexpr ConvPolicy kStandAlone{false, true, false, false};

extern "C" {

int cp_conv2d(const float* x, const float* weight, const float* bias, const float* residual, float* out, int32_t B,
              int32_t H, int32_t W, int32_t Cin, int32_t Cout, int32_t k, int32_t stride, int32_t pad, int32_t relu,
              int32_t precision, void* stream_) {
  if (!x || !weight || !out) return fail(CP_ERR_INVALID, "cp_conv2d: null argument");
  if (B <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || k <= 0 || stride <= 0 || pad < 0)
    return fail(CP_ERR_INVALID, "cp_conv2d: bad shape");
  if (Cin % 16 || Cout % 4) return fail(CP_ERR_INVALID, "cp_conv2d: Cin must be a multiple of 16 and Cout of 4");
  if (!known_precision(precision)) return fail(CP_ERR_INVALID, "unknown precision");
  int rc;
  cudaStream_t s = (cudaStream_t)stream_;
  const int CoPad = conv_cout_pad(Cout);
  const int K = k * k * Cin;
  float* scratch = nullptr;
  CP_CUDA_CHECK(cudaMallocAsync(&scratch, ((size_t)K * CoPad + CoPad) * sizeof(float), s));
  float* wp = scratch;
  float* bp = wp + (size_t)K * CoPad;
  do {
    if ((rc = launch_pack_conv_weight(weight, nullptr, wp, Cout, Cin, k, k, CoPad, K, CoPad, 0, s))) break;
    if ((rc = launch_pack_bias(bias, nullptr, nullptr, nullptr, nullptr, nullptr, bp, Cout, CoPad, 0.f, s))) break;
    IgemmParams p{};
    p.nsrc = 1;
    p.src[0] = x;
    p.srcC[0] = Cin;
    p.srcStride[0] = Cin;
    p.B = B;
    p.Hin = H;
    p.Win = W;
    p.Cin = Cin;
    p.kh = p.kw = k;
    p.stride = stride;
    p.pad = pad;
    p.Hout = (H + 2 * pad - k) / stride + 1;
    p.Wout = (W + 2 * pad - k) / stride + 1;
    p.Cout = Cout;
    p.CoutPad = CoPad;
    p.Kpad = K;
    p.wgt = wp;
    p.bias = bp;
    p.residual = residual;
    p.resStride = Cout;
    p.relu = relu;
    p.out = out;
    p.outStride = Cout;
    p.mode = IGEMM_NHWC_VEC;
    rc = run_conv(p, precision, kStandAlone, s);
  } while (0);
  cudaFreeAsync(scratch, s);
  return rc;
}

int cp_dcn_v2_backward(const float* input, const float* weight, const float* offset, const float* mask,
                       const float* grad_output, float* grad_input, float* grad_offset, float* grad_mask,
                       float* grad_weight, float* grad_bias, int32_t B, int32_t C, int32_t H, int32_t W, int32_t Co,
                       int32_t precision, void* stream_) {
  if (!known_precision(precision)) return fail(CP_ERR_INVALID, "unknown precision");
  if (!input || !weight || !offset || !mask || !grad_output || !grad_input || !grad_offset || !grad_mask || !grad_weight ||
      !grad_bias)
    return fail(CP_ERR_INVALID, "cp_dcn_v2_backward: null argument");
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || Co <= 0) return fail(CP_ERR_INVALID, "cp_dcn_v2_backward: bad shape");
  return dcn_v2_backward_impl(input, weight, offset, mask, grad_output, grad_input, grad_offset, grad_mask, grad_weight,
                              grad_bias, B, C, H, W, Co, precision, (cudaStream_t)stream_);
}

int cp_dcn_v2_forward(const float* input, const float* weight, const float* bias, const float* offset,
                      const float* mask, float* output, int32_t B, int32_t C, int32_t H, int32_t W, int32_t Co,
                      void* stream_) {
  return cp_dcn_v2_forward_ex(input, weight, bias, offset, mask, output, B, C, H, W, Co, CP_PREC_FP32, stream_);
}

int cp_dcn_v2_forward_ex(const float* input, const float* weight, const float* bias, const float* offset,
                         const float* mask, float* output, int32_t B, int32_t C, int32_t H, int32_t W, int32_t Co,
                         int32_t precision, void* stream_) {
  if (!known_precision(precision)) return fail(CP_ERR_INVALID, "unknown precision");
  if (!input || !weight || !bias || !offset || !mask || !output)
    return fail(CP_ERR_INVALID, "cp_dcn_v2_forward: null argument");
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || Co <= 0) return fail(CP_ERR_INVALID, "cp_dcn_v2_forward: bad shape");
  cudaStream_t s = (cudaStream_t)stream_;
  // zero channels pad C to a whole K block of dcn_tma (16) and, in bf16, to the 32-channel span of a gather thread
  const int Cp = round_up(C, precision == CP_PREC_BF16 ? 32 : 16);
  const int CoPad = conv_cout_pad(Co);
  const size_t npix = (size_t)B * H * W;
  const size_t n_x = npix * Cp, n_om = npix * 32, n_w = (size_t)9 * Cp * CoPad, n_b = CoPad;
  float* scratch = nullptr;
  CP_CUDA_CHECK(cudaMallocAsync(&scratch, (n_x + n_om + n_w + n_b) * sizeof(float), s));
  float* x = scratch;
  float* om = x + n_x;
  float* wp = om + n_om;
  float* bp = wp + n_w;
  int rc = CP_OK;
  do {
    if (Cp != C && cudaMemsetAsync(x, 0, n_x * sizeof(float), s) != cudaSuccess) {
      rc = fail(CP_ERR_CUDA, "cp_dcn_v2_forward: memset");
      break;
    }
    if ((rc = launch_nchw_to_nhwc(input, x, B, C, H, W, Cp, 0, s))) break;
    if ((rc = launch_nchw_to_nhwc(offset, om, B, 18, H, W, 32, 0, s))) break;
    if ((rc = launch_nchw_to_nhwc(mask, om, B, 9, H, W, 32, 18, s))) break;
    if ((rc = launch_pack_conv_weight(weight, nullptr, wp, Co, C, 3, 3, CoPad, 9 * Cp, CoPad, 0, s, Cp))) break;
    if ((rc = launch_pack_bias(bias, nullptr, nullptr, nullptr, nullptr, nullptr, bp, Co, CoPad, 0.f, s))) break;
    IgemmParams p{};
    p.nsrc = 1;
    p.src[0] = x;
    p.srcC[0] = Cp;
    p.srcStride[0] = Cp;
    p.B = B;
    p.Hin = p.Hout = H;
    p.Win = p.Wout = W;
    p.Cin = Cp;
    p.Cout = Co;
    p.CoutPad = CoPad;
    p.kh = p.kw = 3;
    p.stride = 1;
    p.pad = 1;
    p.Kpad = 9 * Cp;
    p.wgt = wp;
    p.bias = bp;
    p.out = output;
    p.out_nchw = 1;
    p.offmask = om;
    p.omStride = 32;
    p.mask_is_logit = 0;
    p.mode = IGEMM_DCN;
    rc = run_conv(p, precision, kStandAlone, s);
  } while (0);
  cudaFreeAsync(scratch, s);
  return rc;
}

int cp_preprocess_affine(const uint8_t* frames, float* out, int32_t B, int32_t src_h, int32_t src_w, int32_t dst_h,
                         int32_t dst_w, const double trans_input[6], const float mean[3], const float stdv[3], void* stream_) {
  if (!frames || !out || !mean || !stdv || !trans_input) return fail(CP_ERR_INVALID, "cp_preprocess: null argument");
  if (B <= 0 || src_h <= 0 || src_w <= 0 || dst_h <= 0 || dst_w <= 0)
    return fail(CP_ERR_INVALID, "cp_preprocess: bad shape");
  PreprocessArgs a = preprocess_args(frames, out, B, dst_h, dst_w, mean, stdv);
  a.W = invert_affine(trans_input);
  a.sh = src_h;
  a.sw = src_w;
  return launch_preprocess(CP_PIX_BGR, a, (cudaStream_t)stream_);
}

int cp_preprocess_resize_affine(const uint8_t* frames, float* out, int32_t B, int32_t src_h, int32_t src_w, int32_t rs_h,
                                int32_t rs_w, int32_t dst_h, int32_t dst_w, const double trans_input[6],
                                const float mean[3], const float stdv[3], void* stream_) {
  if (!frames || !out || !mean || !stdv || !trans_input)
    return fail(CP_ERR_INVALID, "cp_preprocess_resize_affine: null argument");
  if (B <= 0 || src_h <= 0 || src_w <= 0 || rs_h <= 0 || rs_w <= 0 || dst_h <= 0 || dst_w <= 0)
    return fail(CP_ERR_INVALID, "cp_preprocess_resize_affine: bad shape (B " + std::to_string(B) + ", frame " +
                                    std::to_string(src_h) + " x " + std::to_string(src_w) + ", resized " +
                                    std::to_string(rs_h) + " x " + std::to_string(rs_w) + ", output " +
                                    std::to_string(dst_h) + " x " + std::to_string(dst_w) + ")");
  // cv2.resize copies a frame of the same size
  if (rs_h == src_h && rs_w == src_w)
    return cp_preprocess_affine(frames, out, B, src_h, src_w, dst_h, dst_w, trans_input, mean, stdv, stream_);
  PreprocessArgs a = preprocess_args(frames, out, B, dst_h, dst_w, mean, stdv);
  a.W = invert_affine(trans_input);
  a.sh = src_h;
  a.sw = src_w;
  a.rh = rs_h;
  a.rw = rs_w;
  // cv2's inverse scales: 1 / inv_scale with inv_scale = dst / src, in double
  a.scale_x = 1. / ((double)rs_w / src_w);
  a.scale_y = 1. / ((double)rs_h / src_h);
  return launch_preprocess(kResizeBgr, a, (cudaStream_t)stream_);
}

// the fix_res affine of the frame size (fix_res_affine above)
int cp_preprocess(const uint8_t* frames, float* out, int32_t B, int32_t src_h, int32_t src_w, int32_t dst_h,
                  int32_t dst_w, const float mean[3], const float stdv[3], void* stream_) {
  if (src_h <= 0 || src_w <= 0 || dst_h <= 0 || dst_w <= 0) return fail(CP_ERR_INVALID, "cp_preprocess: bad shape");
  double T[6];
  fix_res_affine(src_h, src_w, dst_h, dst_w, T);
  return cp_preprocess_affine(frames, out, B, src_h, src_w, dst_h, dst_w, T, mean, stdv, stream_);
}

int cp_preprocess_ragged(const uint8_t* frames, int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw,
                         float* out, int32_t B, int32_t dst_h, int32_t dst_w, const double* trans_input,
                         const float mean[3], const float stdv[3], void* stream_) {
  if (!frames || !offsets || !src_hw || !out || !mean || !stdv) return fail(CP_ERR_INVALID, "cp_preprocess_ragged: null argument");
  if (B <= 0 || dst_h <= 0 || dst_w <= 0 || frames_bytes <= 0) return fail(CP_ERR_INVALID, "cp_preprocess_ragged: bad shape");
  std::vector<RaggedFrame> fr;
  int rc = ragged_frames("cp_preprocess_ragged", frames_bytes, offsets, src_hw, B, dst_h, dst_w, trans_input, CP_PIX_BGR,
                         nullptr, fr);
  if (rc) return rc;
  return launch_ragged("cp_preprocess_ragged", CP_PIX_BGR, fr, preprocess_args(frames, out, B, dst_h, dst_w, mean, stdv),
                       (cudaStream_t)stream_);
}

int cp_preprocess_yuv420(const uint8_t* frames, int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw,
                         int32_t format, float* out, int32_t B, int32_t dst_h, int32_t dst_w, const double* trans_input,
                         const float mean[3], const float stdv[3], void* stream_) {
  if (!frames || !offsets || !src_hw || !out || !mean || !stdv) return fail(CP_ERR_INVALID, "cp_preprocess_yuv420: null argument");
  if (B <= 0 || dst_h <= 0 || dst_w <= 0 || frames_bytes <= 0) return fail(CP_ERR_INVALID, "cp_preprocess_yuv420: bad shape");
  if (!is_yuv420(format))
    return fail(CP_ERR_INVALID, "cp_preprocess_yuv420: unknown pixel format " + std::to_string(format));
  std::vector<RaggedFrame> fr;
  int rc = ragged_frames("cp_preprocess_yuv420", frames_bytes, offsets, src_hw, B, dst_h, dst_w, trans_input, format,
                         nullptr, fr);
  if (rc) return rc;
  return launch_ragged("cp_preprocess_yuv420", format, fr, preprocess_args(frames, out, B, dst_h, dst_w, mean, stdv),
                       (cudaStream_t)stream_);
}

int cp_preprocess_formats(const uint8_t* frames, int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw,
                          const int32_t* formats, float* out, int32_t B, int32_t dst_h, int32_t dst_w,
                          const double* trans_input, const float mean[3], const float stdv[3], void* stream_) {
  if (!frames || !offsets || !src_hw || !formats || !out || !mean || !stdv)
    return fail(CP_ERR_INVALID, "cp_preprocess_formats: null argument");
  if (B <= 0 || dst_h <= 0 || dst_w <= 0 || frames_bytes <= 0) return fail(CP_ERR_INVALID, "cp_preprocess_formats: bad shape");
  int format = formats[0];
  for (int b = 1; b < B; ++b)
    if (formats[b] != format) format = CP_PIX_PER_FRAME;
  std::vector<RaggedFrame> fr;
  int rc = ragged_frames("cp_preprocess_formats", frames_bytes, offsets, src_hw, B, dst_h, dst_w, trans_input, format,
                         format == CP_PIX_PER_FRAME ? formats : nullptr, fr);
  if (rc) return rc;
  return launch_ragged("cp_preprocess_formats", format, fr, preprocess_args(frames, out, B, dst_h, dst_w, mean, stdv),
                       (cudaStream_t)stream_);
}

int cp_preprocess_remap(const uint8_t* frames, int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw,
                        const int32_t* formats, const float* const* maps, float* out, int32_t B, int32_t dst_h,
                        int32_t dst_w, const double* trans_input, const float mean[3], const float stdv[3],
                        void* stream_) {
  if (!frames || !offsets || !src_hw || !formats || !maps || !out || !mean || !stdv)
    return fail(CP_ERR_INVALID, "cp_preprocess_remap: null argument");
  if (B <= 0 || dst_h <= 0 || dst_w <= 0 || frames_bytes <= 0) return fail(CP_ERR_INVALID, "cp_preprocess_remap: bad shape");
  int format = formats[0];
  for (int b = 1; b < B; ++b)
    if (formats[b] != format) format = CP_PIX_PER_FRAME;
  std::vector<RaggedFrame> fr;
  int rc = ragged_frames("cp_preprocess_remap", frames_bytes, offsets, src_hw, B, dst_h, dst_w, trans_input, format,
                         format == CP_PIX_PER_FRAME ? formats : nullptr, fr, maps);
  if (rc) return rc;
  return launch_ragged("cp_preprocess_remap", format | CP_PIX_REMAP, fr,
                       preprocess_args(frames, out, B, dst_h, dst_w, mean, stdv), (cudaStream_t)stream_);
}

int cp_preprocess_slots_dev(const uint8_t* frames, int32_t format, int32_t B, int32_t src_h, int32_t src_w,
                            int32_t dst_h, int32_t dst_w, const double* trans_input, const float mean[3],
                            const float stdv[3], const int32_t* start, float* out, float* prev, void* stream_) {
  if (!frames || !out || !mean || !stdv) return fail(CP_ERR_INVALID, "cp_preprocess_slots_dev: null argument");
  if (!start != !prev) return fail(CP_ERR_INVALID, "cp_preprocess_slots_dev: start and prev go together");
  if (!known_format(format))
    return fail(CP_ERR_INVALID, "cp_preprocess_slots_dev: unknown pixel format " + std::to_string(format));
  if (B <= 0 || src_h <= 0 || src_w <= 0 || dst_h <= 0 || dst_w <= 0)
    return fail(CP_ERR_INVALID, "cp_preprocess_slots_dev: bad shape");
  if (is_yuv420(format) && (src_h % 2 || src_w % 2))
    return fail(CP_ERR_INVALID, "cp_preprocess_slots_dev: YUV 4:2:0 frames need an even size, got " +
                                    std::to_string(src_h) + " x " + std::to_string(src_w));
  if (is_yuv422(format) && src_w % 2)
    return fail(CP_ERR_INVALID, "cp_preprocess_slots_dev: YUV 4:2:2 frames need an even width, got " +
                                    std::to_string(src_h) + " x " + std::to_string(src_w));
  if (is_bayer(format) && (src_h < 3 || src_w < 3))
    return fail(CP_ERR_INVALID, "cp_preprocess_slots_dev: Bayer mosaics need at least 3 x 3, got " +
                                    std::to_string(src_h) + " x " + std::to_string(src_w));
  double T[6];
  if (trans_input)
    for (int i = 0; i < 6; ++i) T[i] = trans_input[i];
  else
    fix_res_affine(src_h, src_w, dst_h, dst_w, T);
  PreprocessArgs a = preprocess_args(frames, out, B, dst_h, dst_w, mean, stdv);
  a.W = invert_affine(T);
  a.sh = src_h;
  a.sw = src_w;
  a.start = start;
  a.prev = prev;
  return launch_preprocess(format, a, (cudaStream_t)stream_);
}

int64_t cp_preprocess_frame_table_bytes(int32_t B) {
  if (B <= 0) return fail(CP_ERR_INVALID, "cp_preprocess_frame_table_bytes: B must be > 0, got " + std::to_string(B));
  return (int64_t)sizeof(RaggedFrame) * B;
}

int cp_preprocess_frame_table(int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw, int32_t format,
                              int32_t B, int32_t dst_h, int32_t dst_w, const double* trans_input, void* table,
                              void* stream_) {
  if (!offsets || !src_hw || !table) return fail(CP_ERR_INVALID, "cp_preprocess_frame_table: null argument");
  if (B <= 0 || dst_h <= 0 || dst_w <= 0 || frames_bytes <= 0)
    return fail(CP_ERR_INVALID, "cp_preprocess_frame_table: bad shape");
  if (!known_format(format))
    return fail(CP_ERR_INVALID, "cp_preprocess_frame_table: unknown pixel format " + std::to_string(format));
  return upload_frame_table("cp_preprocess_frame_table", frames_bytes, offsets, src_hw, format, nullptr, B, dst_h, dst_w,
                            trans_input, table, stream_);
}

int cp_preprocess_frame_table_formats(int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw,
                                      const int32_t* formats, int32_t B, int32_t dst_h, int32_t dst_w,
                                      const double* trans_input, void* table, void* stream_) {
  if (!offsets || !src_hw || !formats || !table) return fail(CP_ERR_INVALID, "cp_preprocess_frame_table_formats: null argument");
  if (B <= 0 || dst_h <= 0 || dst_w <= 0 || frames_bytes <= 0)
    return fail(CP_ERR_INVALID, "cp_preprocess_frame_table_formats: bad shape");
  return upload_frame_table("cp_preprocess_frame_table_formats", frames_bytes, offsets, src_hw, CP_PIX_PER_FRAME, formats,
                            B, dst_h, dst_w, trans_input, table, stream_);
}

int cp_preprocess_frame_table_maps(int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw, int32_t format,
                                   const int32_t* formats, const float* const* maps, int32_t B, int32_t dst_h,
                                   int32_t dst_w, const double* trans_input, void* table, void* stream_) {
  if (!offsets || !src_hw || !maps || !table) return fail(CP_ERR_INVALID, "cp_preprocess_frame_table_maps: null argument");
  if (B <= 0 || dst_h <= 0 || dst_w <= 0 || frames_bytes <= 0)
    return fail(CP_ERR_INVALID, "cp_preprocess_frame_table_maps: bad shape");
  if (format == CP_PIX_PER_FRAME ? !formats : !known_format(format) || formats)
    return fail(CP_ERR_INVALID, "cp_preprocess_frame_table_maps: format " + std::to_string(format) +
                                    (formats ? " with per-frame formats (they take CP_PIX_PER_FRAME)"
                                             : " (a cp_pixel_format, or CP_PIX_PER_FRAME with per-frame formats)"));
  return upload_frame_table("cp_preprocess_frame_table_maps", frames_bytes, offsets, src_hw, format, formats, B, dst_h,
                            dst_w, trans_input, table, stream_, maps);
}

int cp_preprocess_slots_ragged_dev(const uint8_t* frames, const void* table, int32_t format, int32_t B, int32_t dst_h,
                                   int32_t dst_w, const float mean[3], const float stdv[3], const int32_t* start,
                                   float* out, float* prev, void* stream_) {
  if (!frames || !table || !out || !mean || !stdv)
    return fail(CP_ERR_INVALID, "cp_preprocess_slots_ragged_dev: null argument");
  if (!start != !prev) return fail(CP_ERR_INVALID, "cp_preprocess_slots_ragged_dev: start and prev go together");
  if (!table_code(format))
    return fail(CP_ERR_INVALID, "cp_preprocess_slots_ragged_dev: unknown pixel format " + std::to_string(format));
  if (B <= 0 || dst_h <= 0 || dst_w <= 0) return fail(CP_ERR_INVALID, "cp_preprocess_slots_ragged_dev: bad shape");
  PreprocessArgs a = preprocess_args(frames, out, B, dst_h, dst_w, mean, stdv);
  a.fr = (const RaggedFrame*)table;
  a.start = start;
  a.prev = prev;
  return launch_preprocess(format, a, (cudaStream_t)stream_);
}

int cp_preprocess_slots_rows_dev(const uint8_t* frames, const void* table, int32_t format, const int32_t* rows, int32_t B,
                                 int32_t dst_h, int32_t dst_w, const float mean[3], const float stdv[3],
                                 const int32_t* start, float* store, float* out, float* prev, void* stream_) {
  if (!frames || !table || !rows || !out || !mean || !stdv)
    return fail(CP_ERR_INVALID, "cp_preprocess_slots_rows_dev: null argument");
  if (!store != !prev) return fail(CP_ERR_INVALID, "cp_preprocess_slots_rows_dev: store and prev go together");
  if (!table_code(format))
    return fail(CP_ERR_INVALID, "cp_preprocess_slots_rows_dev: unknown pixel format " + std::to_string(format));
  if (B <= 0 || dst_h <= 0 || dst_w <= 0) return fail(CP_ERR_INVALID, "cp_preprocess_slots_rows_dev: bad shape");
  PreprocessArgs a = preprocess_args(frames, out, B, dst_h, dst_w, mean, stdv);
  a.fr = (const RaggedFrame*)table;
  a.rows = rows;
  a.start = start;
  a.store = store;
  a.prev = prev;
  return launch_preprocess(format, a, (cudaStream_t)stream_);
}

int cp_gather_rows_dev(const void* src, void* dst, int64_t row_bytes, int32_t n, const int32_t* map, void* stream_) {
  if (!src || !dst || !map) return fail(CP_ERR_INVALID, "cp_gather_rows_dev: null argument");
  if (n <= 0 || row_bytes <= 0 || row_bytes % 4)
    return fail(CP_ERR_INVALID, "cp_gather_rows_dev: bad shape (n " + std::to_string(n) + ", row_bytes " +
                                    std::to_string(row_bytes) + ": rows are a positive multiple of 4 bytes)");
  const size_t words = (size_t)row_bytes / 4;
  gather_rows_kernel<<<preprocess_blocks(words * n), 256, 0, (cudaStream_t)stream_>>>(
      (const uint32_t*)src, (uint32_t*)dst, words, n, map);
  CP_LAUNCH_CHECK("gather_rows_kernel");
  return CP_OK;
}

}  // extern "C"

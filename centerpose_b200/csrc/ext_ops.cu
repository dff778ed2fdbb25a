// Stand-alone entry points next to the plan:
//   cp_dcn_v2_forward -- the `_ext.dcn_v2_forward` replacement (NCHW in / out), built from
//                        the same implicit-GEMM deformable kernel the plan uses
//                        (reference: DCNv2/src/cuda/dcn_v2_cuda.cu:42-172).
//   cp_preprocess     -- batched uint8 HWC frames -> normalised fp32 NCHW network input
//                        (reference: detectors/base_detector.py:91-148, fix_res branch); cp_preprocess_ragged does
//                        the same for frames of different sizes in one launch, and cp_preprocess_yuv420 for NV12 / I420
//                        frames (the colour conversion of cv2.cvtColor fused into the warp's tap fetch);
//                        cp_preprocess_slots_dev is the graph-safe form for one tracking step of a uniform batch, and
//                        cp_preprocess_slots_ragged_dev (over a cp_preprocess_frame_table) that of slots of mixed sizes.
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

// one output pixel (x, y) of a [sh, sw] frame under the inverted matrix W, all three channels.  The source pixels come
// from `px`: px.taps(iy, ix, in-frame flags) sees the 2 x 2 taps (iy, ix) .. (iy + 1, ix + 1) once, then px(k, yy, xx, c)
// is channel c (B, G, R) of in-frame tap k = 2 (yy - iy) + (xx - ix) as an integer 0..255.  Taps outside the frame are
// the border value 0 and are never fetched.  kTwin: the same values also go to `twin` when it is not null (a tracking
// slot's previous-frame input at the start of its video); without it the walk compiles as it always has.
template <class Fetch, bool kTwin = false>
__device__ __forceinline__ void warp_walk(Fetch px, float* __restrict__ out, size_t plane, int sh, int sw, int x,
                                          int y, const WarpM& W, const float* mean, const float* stdv,
                                          float* __restrict__ twin = nullptr) {
  // unfused double arithmetic (the host code OpenCV runs here has no FMA contraction)
  const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(W.m[1], (double)y), W.m[2]), 1024.0)) + 16;
  const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(W.m[4], (double)y), W.m[5]), 1024.0)) + 16;
  const int ad = __double2int_rn(__dmul_rn(__dmul_rn(W.m[0], (double)x), 1024.0));
  const int bd = __double2int_rn(__dmul_rn(__dmul_rn(W.m[3], (double)x), 1024.0));
  const int X = (X0 + ad) >> 5, Y = (Y0 + bd) >> 5;
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
    if (kTwin && twin) twin[c * plane] = (float)r;
  }
}

// interleaved 8-bit BGR [sh, sw, 3]: every channel is read where it is used
struct BgrFetch {
  const uint8_t* __restrict__ img;
  int sw;
  __device__ __forceinline__ void taps(int, int, bool, bool, bool, bool) {}
  __device__ __forceinline__ int operator()(int, int yy, int xx, int c) const {
    return img[((size_t)yy * sw + xx) * 3 + c];
  }
};

__device__ __forceinline__ void warp_pixel(const uint8_t* __restrict__ img, float* __restrict__ out, size_t plane, int sh,
                                           int sw, int x, int y, const WarpM& W, const float* mean, const float* stdv) {
  warp_walk(BgrFetch{img, sw}, out, plane, sh, sw, x, y, W, mean, stdv);
}

// YUV 4:2:0 [3 sh / 2, sw] (sh, sw even) converted per tap to the BGR that cv2.cvtColor(COLOR_YUV2BGR_NV12 / _I420)
// gives, restated bit for bit (OpenCV color_yuv.simd.hpp, yuv42x_to_rgb8 for 8-bit: BT.601 limited range in 20-bit
// fixed point, no chroma interpolation; tests/yuv_ref.py yuv420_to_bgr, pinned against cv2 on every (Y, U, V)):
//   y = max(Y - 16, 0) * 1220542 + 2^19, u = U - 128, v = V - 128
//   B = sat((y + 2116026 u) >> 20), G = sat((y - 852492 v - 409993 u) >> 20), R = sat((y + 1673527 v) >> 20)
// The Y plane [sh, sw] comes first; then NV12: U, V interleaved, row yy / 2, bytes (xx & ~1) and (xx | 1); I420: the U
// plane [sh/2, sw/2], then the V plane [sh/2, sw/2].  Only in-frame taps are converted: warpAffine's border 0 is BGR 0.
template <int kFormat>
struct Yuv420Fetch {
  const uint8_t* __restrict__ img;
  int sh, sw;
  int yv[4], u[4], v[4];      // per tap: max(Y - 16, 0) * 1220542 + 2^19, U - 128, V - 128
  // every in-frame tap is read and converted once, before the first channel is written
  __device__ __forceinline__ void taps(int iy, int ix, bool in00, bool in01, bool in10, bool in11) {
    const bool in[4] = {in00, in01, in10, in11};
    const uint8_t* __restrict__ chroma = img + (size_t)sh * sw;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      yv[k] = u[k] = v[k] = 0;
      if (!in[k]) continue;
      const int yy = iy + (k >> 1), xx = ix + (k & 1);
      int U, V;
      if (kFormat == CP_PIX_NV12) {
        const size_t o = (size_t)(yy >> 1) * sw + (xx & ~1);
        U = chroma[o];
        V = chroma[o + 1];
      } else {
        const size_t o = (size_t)(yy >> 1) * (sw >> 1) + (xx >> 1);
        U = chroma[o];
        V = chroma[(size_t)(sh >> 1) * (sw >> 1) + o];
      }
      yv[k] = max((int)img[(size_t)yy * sw + xx] - 16, 0) * 1220542 + (1 << 19);
      u[k] = U - 128;
      v[k] = V - 128;
    }
  }
  __device__ __forceinline__ int operator()(int k, int, int, int c) const {
    const int t = c == 0 ? yv[k] + 2116026 * u[k]
                         : (c == 1 ? yv[k] - 852492 * v[k] - 409993 * u[k] : yv[k] + 1673527 * v[k]);
    return max(0, min(255, t >> 20));
  }
};

__global__ void preprocess_kernel(const uint8_t* __restrict__ frames, float* __restrict__ out, int B, int sh,
                                  int sw, int dh, int dw, const WarpM W, float m0, float m1, float m2, float s0, float s1,
                                  float s2) {
  size_t total = (size_t)B * dh * dw;
  const float mean[3] = {m0, m1, m2};
  const float stdv[3] = {s0, s1, s2};
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % dw);
    const size_t t = i / dw;
    const int y = (int)(t % dh);
    const int n = (int)(t / dh);
    warp_pixel(frames + (size_t)n * sh * sw * 3, out + (((size_t)n * 3) * dh + y) * dw + x, (size_t)dh * dw, sh, sw, x, y,
               W, mean, stdv);
  }
}

// per-frame parameters of the ragged launch
struct RaggedFrame {
  WarpM W;
  long long offset;     // bytes into the packed frame buffer
  int sh, sw;
};

__global__ void preprocess_ragged_kernel(const uint8_t* __restrict__ frames, const RaggedFrame* __restrict__ fr,
                                         float* __restrict__ out, int B, int dh, int dw, float m0, float m1, float m2,
                                         float s0, float s1, float s2) {
  size_t total = (size_t)B * dh * dw;
  const float mean[3] = {m0, m1, m2};
  const float stdv[3] = {s0, s1, s2};
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % dw);
    const size_t t = i / dw;
    const int y = (int)(t % dh);
    const int n = (int)(t / dh);
    const RaggedFrame f = fr[n];
    warp_pixel(frames + f.offset, out + (((size_t)n * 3) * dh + y) * dw + x, (size_t)dh * dw, f.sh, f.sw, x, y, f.W, mean,
               stdv);
  }
}

// the ragged launch on YUV 4:2:0 frames (kFormat: cp_pixel_format): the same walk with the tap fetch converting to BGR
template <int kFormat>
__global__ void preprocess_yuv420_kernel(const uint8_t* __restrict__ frames, const RaggedFrame* __restrict__ fr,
                                         float* __restrict__ out, int B, int dh, int dw, float m0, float m1, float m2,
                                         float s0, float s1, float s2) {
  size_t total = (size_t)B * dh * dw;
  const float mean[3] = {m0, m1, m2};
  const float stdv[3] = {s0, s1, s2};
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % dw);
    const size_t t = i / dw;
    const int y = (int)(t % dh);
    const int n = (int)(t / dh);
    const RaggedFrame f = fr[n];
    warp_walk(Yuv420Fetch<kFormat>{frames + f.offset, f.sh, f.sw}, out + (((size_t)n * 3) * dh + y) * dw + x,
              (size_t)dh * dw, f.sh, f.sw, x, y, f.W, mean, stdv);
  }
}

// The frames of one tracking step: B slots of one size, format (cp_pixel_format) and affine, frame n at byte n * bytes.
// Every parameter is a kernel argument or device memory, so a captured launch replays unchanged.  A slot whose start[n]
// is set begins a video with this frame, which is then also its previous frame: the walk writes it to prev[n] as well.
template <int kFormat>
__global__ void preprocess_slots_kernel(const uint8_t* __restrict__ frames, float* __restrict__ out,
                                        float* __restrict__ prev, const int* __restrict__ start, int B, int sh, int sw,
                                        int dh, int dw, const WarpM W, float m0, float m1, float m2, float s0, float s1,
                                        float s2) {
  const size_t total = (size_t)B * dh * dw, plane = (size_t)dh * dw;
  const size_t bytes = kFormat == CP_PIX_BGR ? (size_t)sh * sw * 3 : (size_t)sh * sw * 3 / 2;
  const float mean[3] = {m0, m1, m2};
  const float stdv[3] = {s0, s1, s2};
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % dw);
    const size_t t = i / dw;
    const int y = (int)(t % dh);
    const int n = (int)(t / dh);
    const size_t o = (((size_t)n * 3) * dh + y) * dw + x;
    float* twin = start && start[n] ? prev + o : nullptr;
    const uint8_t* img = frames + n * bytes;
    if constexpr (kFormat == CP_PIX_BGR)
      warp_walk<BgrFetch, true>(BgrFetch{img, sw}, out + o, plane, sh, sw, x, y, W, mean, stdv, twin);
    else
      warp_walk<Yuv420Fetch<kFormat>, true>(Yuv420Fetch<kFormat>{img, sh, sw}, out + o, plane, sh, sw, x, y, W, mean,
                                            stdv, twin);
  }
}

// The frames of one tracking step when the slots differ in size: the ragged walk of preprocess_ragged_kernel /
// preprocess_yuv420_kernel over a frame table `fr` in device memory (built once, cp_preprocess_frame_table), with the
// start-flag twin write of preprocess_slots_kernel.  Nothing is read from the host, so a captured launch replays unchanged.
template <int kFormat>
__global__ void preprocess_slots_ragged_kernel(const uint8_t* __restrict__ frames, const RaggedFrame* __restrict__ fr,
                                               float* __restrict__ out, float* __restrict__ prev,
                                               const int* __restrict__ start, int B, int dh, int dw, float m0, float m1,
                                               float m2, float s0, float s1, float s2) {
  const size_t total = (size_t)B * dh * dw, plane = (size_t)dh * dw;
  const float mean[3] = {m0, m1, m2};
  const float stdv[3] = {s0, s1, s2};
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % dw);
    const size_t t = i / dw;
    const int y = (int)(t % dh);
    const int n = (int)(t / dh);
    const size_t o = (((size_t)n * 3) * dh + y) * dw + x;
    float* twin = start && start[n] ? prev + o : nullptr;
    const RaggedFrame f = fr[n];
    if constexpr (kFormat == CP_PIX_BGR)
      warp_walk<BgrFetch, true>(BgrFetch{frames + f.offset, f.sw}, out + o, plane, f.sh, f.sw, x, y, f.W, mean, stdv,
                                twin);
    else
      warp_walk<Yuv420Fetch<kFormat>, true>(Yuv420Fetch<kFormat>{frames + f.offset, f.sh, f.sw}, out + o, plane, f.sh,
                                            f.sw, x, y, f.W, mean, stdv, twin);
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

// The per-frame parameters of a ragged batch, checked against the packed buffer before any work is enqueued.  `yuv`:
// the frames are YUV 4:2:0 (even sizes, h * w * 3 / 2 bytes each), else BGR (h * w * 3 bytes).
int ragged_frames(const char* who, int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw, int B, int dst_h,
                  int dst_w, const double* trans_input, bool yuv, std::vector<RaggedFrame>& fr) {
  const std::string w0 = who;
  fr.resize(B);
  for (int b = 0; b < B; ++b) {
    const int h = src_hw[2 * b], w = src_hw[2 * b + 1];
    if (h <= 0 || w <= 0 || (yuv && (h % 2 || w % 2)))
      return fail(CP_ERR_INVALID, w0 + ": frame " + std::to_string(b) + " has size " + std::to_string(h) + " x " +
                                      std::to_string(w) + (yuv ? " (YUV 4:2:0 needs even sizes)" : ""));
    const int64_t bytes = yuv ? (int64_t)h * w * 3 / 2 : (int64_t)h * w * 3;
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
    fr[b].offset = offsets[b];
    fr[b].sh = h;
    fr[b].sw = w;
  }
  return CP_OK;
}

// uploads the per-frame parameters (stream-ordered) and enqueues launch(device parameters)
template <class Launch>
int launch_ragged(const char* who, const char* kernel, const std::vector<RaggedFrame>& fr, cudaStream_t s,
                  Launch launch) {
  const int B = (int)fr.size();
  RaggedFrame* dfr = nullptr;
  CP_CUDA_CHECK(cudaMallocAsync(&dfr, sizeof(RaggedFrame) * B, s));
  int rc = CP_OK;
  // a pageable source: the bytes are staged before cudaMemcpyAsync returns, so `fr` may go out of scope
  if (cudaMemcpyAsync(dfr, fr.data(), sizeof(RaggedFrame) * B, cudaMemcpyHostToDevice, s) != cudaSuccess) {
    rc = fail(CP_ERR_CUDA, std::string(who) + ": parameter upload");
  } else {
    launch(dfr);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess)
      rc = fail(CP_ERR_CUDA, std::string(kernel) + ": " + cudaGetErrorString(e));
    else
      ++g_launch_counter;
  }
  cudaFreeAsync(dfr, s);
  return rc;
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
  const int Cp = round_up(C, 16);
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
  const WarpM W = invert_affine(trans_input);
  preprocess_kernel<<<preprocess_blocks((size_t)B * dst_h * dst_w), 256, 0, (cudaStream_t)stream_>>>(
      frames, out, B, src_h, src_w, dst_h, dst_w, W, mean[0], mean[1], mean[2], stdv[0], stdv[1], stdv[2]);
  CP_LAUNCH_CHECK("preprocess_kernel");
  return CP_OK;
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
  int rc = ragged_frames("cp_preprocess_ragged", frames_bytes, offsets, src_hw, B, dst_h, dst_w, trans_input, false, fr);
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream_;
  return launch_ragged("cp_preprocess_ragged", "preprocess_ragged_kernel", fr, s, [&](const RaggedFrame* dfr) {
    preprocess_ragged_kernel<<<preprocess_blocks((size_t)B * dst_h * dst_w), 256, 0, s>>>(
        frames, dfr, out, B, dst_h, dst_w, mean[0], mean[1], mean[2], stdv[0], stdv[1], stdv[2]);
  });
}

int cp_preprocess_yuv420(const uint8_t* frames, int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw,
                         int32_t format, float* out, int32_t B, int32_t dst_h, int32_t dst_w, const double* trans_input,
                         const float mean[3], const float stdv[3], void* stream_) {
  if (!frames || !offsets || !src_hw || !out || !mean || !stdv) return fail(CP_ERR_INVALID, "cp_preprocess_yuv420: null argument");
  if (B <= 0 || dst_h <= 0 || dst_w <= 0 || frames_bytes <= 0) return fail(CP_ERR_INVALID, "cp_preprocess_yuv420: bad shape");
  if (format != CP_PIX_NV12 && format != CP_PIX_I420)
    return fail(CP_ERR_INVALID, "cp_preprocess_yuv420: unknown pixel format " + std::to_string(format));
  std::vector<RaggedFrame> fr;
  int rc = ragged_frames("cp_preprocess_yuv420", frames_bytes, offsets, src_hw, B, dst_h, dst_w, trans_input, true, fr);
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream_;
  return launch_ragged("cp_preprocess_yuv420", "preprocess_yuv420_kernel", fr, s, [&](const RaggedFrame* dfr) {
    const int blocks = preprocess_blocks((size_t)B * dst_h * dst_w);
    if (format == CP_PIX_NV12)
      preprocess_yuv420_kernel<CP_PIX_NV12><<<blocks, 256, 0, s>>>(frames, dfr, out, B, dst_h, dst_w, mean[0], mean[1],
                                                                    mean[2], stdv[0], stdv[1], stdv[2]);
    else
      preprocess_yuv420_kernel<CP_PIX_I420><<<blocks, 256, 0, s>>>(frames, dfr, out, B, dst_h, dst_w, mean[0], mean[1],
                                                                    mean[2], stdv[0], stdv[1], stdv[2]);
  });
}

int cp_preprocess_slots_dev(const uint8_t* frames, int32_t format, int32_t B, int32_t src_h, int32_t src_w,
                            int32_t dst_h, int32_t dst_w, const double* trans_input, const float mean[3],
                            const float stdv[3], const int32_t* start, float* out, float* prev, void* stream_) {
  if (!frames || !out || !mean || !stdv) return fail(CP_ERR_INVALID, "cp_preprocess_slots_dev: null argument");
  if (!start != !prev) return fail(CP_ERR_INVALID, "cp_preprocess_slots_dev: start and prev go together");
  if (format != CP_PIX_BGR && format != CP_PIX_NV12 && format != CP_PIX_I420)
    return fail(CP_ERR_INVALID, "cp_preprocess_slots_dev: unknown pixel format " + std::to_string(format));
  if (B <= 0 || src_h <= 0 || src_w <= 0 || dst_h <= 0 || dst_w <= 0)
    return fail(CP_ERR_INVALID, "cp_preprocess_slots_dev: bad shape");
  if (format != CP_PIX_BGR && (src_h % 2 || src_w % 2))
    return fail(CP_ERR_INVALID, "cp_preprocess_slots_dev: YUV 4:2:0 frames need an even size, got " +
                                    std::to_string(src_h) + " x " + std::to_string(src_w));
  double T[6];
  if (trans_input)
    for (int i = 0; i < 6; ++i) T[i] = trans_input[i];
  else
    fix_res_affine(src_h, src_w, dst_h, dst_w, T);
  const WarpM W = invert_affine(T);
  const int blocks = preprocess_blocks((size_t)B * dst_h * dst_w);
  cudaStream_t s = (cudaStream_t)stream_;
  auto launch = [&](auto kernel) {
    kernel<<<blocks, 256, 0, s>>>(frames, out, prev, start, B, src_h, src_w, dst_h, dst_w, W, mean[0], mean[1], mean[2],
                                  stdv[0], stdv[1], stdv[2]);
  };
  if (format == CP_PIX_BGR)
    launch(preprocess_slots_kernel<CP_PIX_BGR>);
  else if (format == CP_PIX_NV12)
    launch(preprocess_slots_kernel<CP_PIX_NV12>);
  else
    launch(preprocess_slots_kernel<CP_PIX_I420>);
  CP_LAUNCH_CHECK("preprocess_slots_kernel");
  return CP_OK;
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
  if (format != CP_PIX_BGR && format != CP_PIX_NV12 && format != CP_PIX_I420)
    return fail(CP_ERR_INVALID, "cp_preprocess_frame_table: unknown pixel format " + std::to_string(format));
  std::vector<RaggedFrame> fr;
  int rc = ragged_frames("cp_preprocess_frame_table", frames_bytes, offsets, src_hw, B, dst_h, dst_w, trans_input,
                         format != CP_PIX_BGR, fr);
  if (rc) return rc;
  // a build-time call: the copy is complete when it returns, so `fr` may go out of scope
  cudaStream_t s = (cudaStream_t)stream_;
  cudaError_t e = cudaMemcpyAsync(table, fr.data(), sizeof(RaggedFrame) * B, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess)
    return fail(CP_ERR_CUDA, std::string("cp_preprocess_frame_table: table upload: ") + cudaGetErrorString(e));
  return CP_OK;
}

int cp_preprocess_slots_ragged_dev(const uint8_t* frames, const void* table, int32_t format, int32_t B, int32_t dst_h,
                                   int32_t dst_w, const float mean[3], const float stdv[3], const int32_t* start,
                                   float* out, float* prev, void* stream_) {
  if (!frames || !table || !out || !mean || !stdv)
    return fail(CP_ERR_INVALID, "cp_preprocess_slots_ragged_dev: null argument");
  if (!start != !prev) return fail(CP_ERR_INVALID, "cp_preprocess_slots_ragged_dev: start and prev go together");
  if (format != CP_PIX_BGR && format != CP_PIX_NV12 && format != CP_PIX_I420)
    return fail(CP_ERR_INVALID, "cp_preprocess_slots_ragged_dev: unknown pixel format " + std::to_string(format));
  if (B <= 0 || dst_h <= 0 || dst_w <= 0) return fail(CP_ERR_INVALID, "cp_preprocess_slots_ragged_dev: bad shape");
  const RaggedFrame* fr = (const RaggedFrame*)table;
  const int blocks = preprocess_blocks((size_t)B * dst_h * dst_w);
  cudaStream_t s = (cudaStream_t)stream_;
  auto launch = [&](auto kernel) {
    kernel<<<blocks, 256, 0, s>>>(frames, fr, out, prev, start, B, dst_h, dst_w, mean[0], mean[1], mean[2], stdv[0],
                                  stdv[1], stdv[2]);
  };
  if (format == CP_PIX_BGR)
    launch(preprocess_slots_ragged_kernel<CP_PIX_BGR>);
  else if (format == CP_PIX_NV12)
    launch(preprocess_slots_ragged_kernel<CP_PIX_NV12>);
  else
    launch(preprocess_slots_ragged_kernel<CP_PIX_I420>);
  CP_LAUNCH_CHECK("preprocess_slots_ragged_kernel");
  return CP_OK;
}

}  // extern "C"

// 7x7 stride-1 pad-3 stem convolutions (pose_dla_dcn.py:234-238, 253-271): NCHW fp32 input with 1 / 3 / 8
// channels -> 16 channels NHWC, folded BatchNorm + ReLU, optional "+ previous stem" after the ReLU
// (tracking stems, :313-318).  Direct convolution: K = 49*Cin is too small and too ragged for a GEMM tile and
// the layer is bound by its 64 B/pixel output write, so the input halo tile and the folded weights live in
// shared memory and every thread owns 4 pixels x 16 output channels in registers.
// The ResNet stems (msra_resnet.py:116-118, 126-147) are the same convolution at stride 2 with 64 outputs
// (stem_conv7s2_kernel): there four threads share a pixel quadruple, one per 16-channel group.
#include "common.cuh"

namespace cp {
namespace {

constexpr int ST_TX = 16, ST_TY = 16;    // threads
constexpr int ST_PX = 4;                 // pixels per thread along x (strided by ST_TX -> conflict-free smem reads)
constexpr int ST_W = ST_TX * ST_PX;      // 64-wide, 16-high output tile
constexpr int ST_HALO_W = ST_W + 6, ST_HALO_H = ST_TY + 6;

__global__ void __launch_bounds__(ST_TX* ST_TY)
    stem_conv7_kernel(const float* __restrict__ in, const float* __restrict__ wgt, const float* __restrict__ bias,
                      const float* __restrict__ residual, float* __restrict__ out, int B, int Cin, int H, int W,
                      int relu, int ipm, long long wstride, int in_ipm) {
  extern __shared__ __align__(16) float sm[];
  float* ws = sm;                                        // [(ky*7+kx)*Cin + c][16]   (16-byte aligned)
  float* tile = sm + 49 * Cin * 16;                      // [Cin][ST_HALO_H][ST_HALO_W]
  const int tid = threadIdx.y * ST_TX + threadIdx.x;
  const int n = blockIdx.z;
  const int x0 = blockIdx.x * ST_W, y0 = blockIdx.y * ST_TY;
  const int nw = 49 * Cin * 16;
  // image n runs model n / ipm (IgemmParams::ipm) on input image n % in_ipm: in_ipm = ipm when every model reads the same
  // frames, the launch's whole batch when each model has its own input (IgemmParams::nchw_per_model)
  wgt += (size_t)(n / ipm) * wstride;
  bias += (size_t)(n / ipm) * wstride;
  const int n_in = n % in_ipm;
  if (tid == 0) griddep_launch_dependents();      // PDL (common.cuh): weights are constants, the image is not
  for (int i = tid; i < nw; i += ST_TX * ST_TY) ws[i] = __ldg(wgt + i);
  griddep_wait();
  const int nt = Cin * ST_HALO_H * ST_HALO_W;
  for (int i = tid; i < nt; i += ST_TX * ST_TY) {
    int xx = i % ST_HALO_W;
    int t = i / ST_HALO_W;
    int yy = t % ST_HALO_H;
    int c = t / ST_HALO_H;
    int gy = y0 + yy - 3, gx = x0 + xx - 3;
    float v = 0.f;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = __ldg(in + (((size_t)n_in * Cin + c) * H + gy) * W + gx);
    tile[i] = v;
  }
  __syncthreads();

  float acc[ST_PX][16];
#pragma unroll
  for (int i = 0; i < ST_PX; ++i)
#pragma unroll
    for (int o = 0; o < 16; ++o) acc[i][o] = 0.f;

  for (int c = 0; c < Cin; ++c) {
    for (int ky = 0; ky < 7; ++ky) {
      const float* trow = tile + (c * ST_HALO_H + threadIdx.y + ky) * ST_HALO_W + threadIdx.x;
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        const float4* wp = reinterpret_cast<const float4*>(ws + ((ky * 7 + kx) * Cin + c) * 16);
        const float4 w0 = wp[0], w1 = wp[1], w2 = wp[2], w3 = wp[3];
#pragma unroll
        for (int i = 0; i < ST_PX; ++i) {
          const float v = trow[kx + i * ST_TX];
          acc[i][0] = fmaf(v, w0.x, acc[i][0]);
          acc[i][1] = fmaf(v, w0.y, acc[i][1]);
          acc[i][2] = fmaf(v, w0.z, acc[i][2]);
          acc[i][3] = fmaf(v, w0.w, acc[i][3]);
          acc[i][4] = fmaf(v, w1.x, acc[i][4]);
          acc[i][5] = fmaf(v, w1.y, acc[i][5]);
          acc[i][6] = fmaf(v, w1.z, acc[i][6]);
          acc[i][7] = fmaf(v, w1.w, acc[i][7]);
          acc[i][8] = fmaf(v, w2.x, acc[i][8]);
          acc[i][9] = fmaf(v, w2.y, acc[i][9]);
          acc[i][10] = fmaf(v, w2.z, acc[i][10]);
          acc[i][11] = fmaf(v, w2.w, acc[i][11]);
          acc[i][12] = fmaf(v, w3.x, acc[i][12]);
          acc[i][13] = fmaf(v, w3.y, acc[i][13]);
          acc[i][14] = fmaf(v, w3.z, acc[i][14]);
          acc[i][15] = fmaf(v, w3.w, acc[i][15]);
        }
      }
    }
  }
  float b[16];
#pragma unroll
  for (int o = 0; o < 16; ++o) b[o] = __ldg(bias + o);
  const int gy = y0 + threadIdx.y;
  if (gy >= H) return;
#pragma unroll
  for (int i = 0; i < ST_PX; ++i) {
    const int gx = x0 + threadIdx.x + i * ST_TX;
    if (gx >= W) continue;
    const size_t pix = ((size_t)n * H + gy) * W + gx;
    float v[16];
#pragma unroll
    for (int o = 0; o < 16; ++o) {
      v[o] = acc[i][o] + b[o];
      if (relu) v[o] = fmaxf(v[o], 0.f);
    }
    if (residual) {
      const float4* r = reinterpret_cast<const float4*>(residual + pix * 16);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float4 rv = __ldg(r + q);
        v[q * 4 + 0] += rv.x;
        v[q * 4 + 1] += rv.y;
        v[q * 4 + 2] += rv.z;
        v[q * 4 + 3] += rv.w;
      }
    }
    float4* o4 = reinterpret_cast<float4*>(out + pix * 16);
#pragma unroll
    for (int q = 0; q < 4; ++q) o4[q] = make_float4(v[q * 4], v[q * 4 + 1], v[q * 4 + 2], v[q * 4 + 3]);
  }
}


// ------------------------------------------------------------------------------------------------------------------
// 3x3 stride-1 pad-1 convolution, 16 -> 16 channels, NHWC fp32 in and out (DLA level0 at full resolution,
// pose_dla_dcn.py:239-240 + _make_conv_level).  K = 144 is too small for a tensor-core tile to pay for itself at 8.4 M
// positions (it ran at half the speed of the generic FFMA implicit GEMM on the tensor-core gather kernel); a direct
// convolution with the halo tile transposed into channel planes in shared memory runs at the FFMA rate instead.
constexpr int C3_TX = 16, C3_TY = 16, C3_PX = 4;
constexpr int C3_W = C3_TX * C3_PX;                              // 64 x 16 output pixels per CTA
constexpr int C3_HW = C3_W + 2, C3_HH = C3_TY + 2;
constexpr int C3_PLANE = C3_HH * C3_HW + 1;                       // odd plane pitch: the NHWC -> planes transpose spreads banks

__global__ void __launch_bounds__(C3_TX* C3_TY, 2)
    conv3_c16_kernel(const float* __restrict__ in, int inStride, const float* __restrict__ wgt, const float* __restrict__ bias,
                     float* __restrict__ out, int outStride, int B, int H, int W, int relu, int ipm, long long wstride) {
  extern __shared__ __align__(16) float sm[];
  float* ws = sm;                                  // [(ky*3+kx)*16 + c][16]
  float* tile = sm + 9 * 16 * 16;                  // [16 planes][C3_PLANE]
  const int tid = threadIdx.y * C3_TX + threadIdx.x;
  const int n = blockIdx.z;
  const int x0 = blockIdx.x * C3_W, y0 = blockIdx.y * C3_TY;
  wgt += (size_t)(n / ipm) * wstride;      // model n / ipm (IgemmParams::ipm)
  bias += (size_t)(n / ipm) * wstride;
  if (tid == 0) griddep_launch_dependents();      // PDL (common.cuh)
  for (int i = tid; i < 9 * 16 * 16; i += C3_TX * C3_TY) ws[i] = __ldg(wgt + i);
  griddep_wait();
  for (int i = tid; i < C3_HH * C3_HW * 4; i += C3_TX * C3_TY) {
    const int q = i & 3, pix = i >> 2;
    const int xx = pix % C3_HW, yy = pix / C3_HW;
    const int gy = y0 + yy - 1, gx = x0 + xx - 1;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (gy >= 0 && gy < H && gx >= 0 && gx < W)
      v = __ldg(reinterpret_cast<const float4*>(in + (((size_t)n * H + gy) * W + gx) * inStride) + q);
    float* t = tile + (q * 4) * C3_PLANE + yy * C3_HW + xx;
    t[0] = v.x;
    t[C3_PLANE] = v.y;
    t[2 * C3_PLANE] = v.z;
    t[3 * C3_PLANE] = v.w;
  }
  __syncthreads();

  float acc[C3_PX][16];
#pragma unroll
  for (int i = 0; i < C3_PX; ++i)
#pragma unroll
    for (int o = 0; o < 16; ++o) acc[i][o] = 0.f;

  for (int c = 0; c < 16; ++c) {
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const float* trow = tile + c * C3_PLANE + (threadIdx.y + ky) * C3_HW + threadIdx.x;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const float4* wp = reinterpret_cast<const float4*>(ws + ((ky * 3 + kx) * 16 + c) * 16);
        const float4 w0 = wp[0], w1 = wp[1], w2 = wp[2], w3 = wp[3];
#pragma unroll
        for (int i = 0; i < C3_PX; ++i) {
          const float v = trow[kx + i * C3_TX];
          acc[i][0] = fmaf(v, w0.x, acc[i][0]);
          acc[i][1] = fmaf(v, w0.y, acc[i][1]);
          acc[i][2] = fmaf(v, w0.z, acc[i][2]);
          acc[i][3] = fmaf(v, w0.w, acc[i][3]);
          acc[i][4] = fmaf(v, w1.x, acc[i][4]);
          acc[i][5] = fmaf(v, w1.y, acc[i][5]);
          acc[i][6] = fmaf(v, w1.z, acc[i][6]);
          acc[i][7] = fmaf(v, w1.w, acc[i][7]);
          acc[i][8] = fmaf(v, w2.x, acc[i][8]);
          acc[i][9] = fmaf(v, w2.y, acc[i][9]);
          acc[i][10] = fmaf(v, w2.z, acc[i][10]);
          acc[i][11] = fmaf(v, w2.w, acc[i][11]);
          acc[i][12] = fmaf(v, w3.x, acc[i][12]);
          acc[i][13] = fmaf(v, w3.y, acc[i][13]);
          acc[i][14] = fmaf(v, w3.z, acc[i][14]);
          acc[i][15] = fmaf(v, w3.w, acc[i][15]);
        }
      }
    }
  }
  float b[16];
#pragma unroll
  for (int o = 0; o < 16; ++o) b[o] = __ldg(bias + o);
  const int gy = y0 + threadIdx.y;
  if (gy >= H) return;
#pragma unroll
  for (int i = 0; i < C3_PX; ++i) {
    const int gx = x0 + threadIdx.x + i * C3_TX;
    if (gx >= W) continue;
    float4* o4 = reinterpret_cast<float4*>(out + (((size_t)n * H + gy) * W + gx) * outStride);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float4 r;
      r.x = acc[i][q * 4 + 0] + b[q * 4 + 0];
      r.y = acc[i][q * 4 + 1] + b[q * 4 + 1];
      r.z = acc[i][q * 4 + 2] + b[q * 4 + 2];
      r.w = acc[i][q * 4 + 3] + b[q * 4 + 3];
      if (relu) {
        r.x = fmaxf(r.x, 0.f);
        r.y = fmaxf(r.y, 0.f);
        r.z = fmaxf(r.z, 0.f);
        r.w = fmaxf(r.w, 0.f);
      }
      o4[q] = r;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// 7x7 stride-2 pad-3 stem, NCHW fp32 input with 1 / 3 / 8 channels -> 64 channels NHWC, folded BatchNorm + ReLU
// (msra_resnet.py:116-118, 237-239; pre_* stems :126-147).  A CTA makes a 64 x 4 output tile; thread (tx, ty, g) owns
// pixels x0 + tx + 16 i (i < 4) of row y0 + ty and channels [16 g, 16 g + 16).  The threads of a warp share g, so the
// weight reads are broadcasts; the input halo is (2 * 64 + 5) x (2 * 4 + 5) per channel.
constexpr int S2_TX = 16, S2_TY = 4, S2_G = 4, S2_PX = 4;
constexpr int S2_W = S2_TX * S2_PX;
constexpr int S2_HALO_W = 2 * S2_W + 5, S2_HALO_H = 2 * S2_TY + 5;

__global__ void __launch_bounds__(S2_TX* S2_TY* S2_G)
    stem_conv7s2_kernel(const float* __restrict__ in, const float* __restrict__ wgt, const float* __restrict__ bias,
                        float* __restrict__ out, int Cin, int H, int W, int Ho, int Wo, int relu, int ipm,
                        long long wstride, int in_ipm) {
  extern __shared__ __align__(16) float sm[];
  float* ws = sm;                                        // [(ky*7+kx)*Cin + c][64]
  float* tile = sm + 49 * Cin * 64;                      // [Cin][S2_HALO_H][S2_HALO_W]
  const int tx = threadIdx.x, ty = threadIdx.y, g = threadIdx.z;
  const int tid = (g * S2_TY + ty) * S2_TX + tx;
  constexpr int NT = S2_TX * S2_TY * S2_G;
  const int n = blockIdx.z;
  const int x0 = blockIdx.x * S2_W, y0 = blockIdx.y * S2_TY;
  const int nw = 49 * Cin * 64;
  // image n runs model n / ipm on input image n % in_ipm (as stem_conv7_kernel)
  wgt += (size_t)(n / ipm) * wstride;
  bias += (size_t)(n / ipm) * wstride;
  const int n_in = n % in_ipm;
  if (tid == 0) griddep_launch_dependents();      // PDL (common.cuh): weights are constants, the image is not
  for (int i = tid; i < nw; i += NT) ws[i] = __ldg(wgt + i);
  griddep_wait();
  const int nt = Cin * S2_HALO_H * S2_HALO_W;
  for (int i = tid; i < nt; i += NT) {
    const int xx = i % S2_HALO_W;
    const int t = i / S2_HALO_W;
    const int yy = t % S2_HALO_H;
    const int c = t / S2_HALO_H;
    const int gy = 2 * y0 + yy - 3, gx = 2 * x0 + xx - 3;
    float v = 0.f;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = __ldg(in + (((size_t)n_in * Cin + c) * H + gy) * W + gx);
    tile[i] = v;
  }
  __syncthreads();

  float acc[S2_PX][16];
#pragma unroll
  for (int i = 0; i < S2_PX; ++i)
#pragma unroll
    for (int o = 0; o < 16; ++o) acc[i][o] = 0.f;

  for (int c = 0; c < Cin; ++c) {
    for (int ky = 0; ky < 7; ++ky) {
      const float* trow = tile + (c * S2_HALO_H + 2 * ty + ky) * S2_HALO_W + 2 * tx;
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        const float4* wp = reinterpret_cast<const float4*>(ws + ((ky * 7 + kx) * Cin + c) * 64 + g * 16);
        const float4 w0 = wp[0], w1 = wp[1], w2 = wp[2], w3 = wp[3];
#pragma unroll
        for (int i = 0; i < S2_PX; ++i) {
          const float v = trow[kx + 2 * S2_TX * i];
          acc[i][0] = fmaf(v, w0.x, acc[i][0]);
          acc[i][1] = fmaf(v, w0.y, acc[i][1]);
          acc[i][2] = fmaf(v, w0.z, acc[i][2]);
          acc[i][3] = fmaf(v, w0.w, acc[i][3]);
          acc[i][4] = fmaf(v, w1.x, acc[i][4]);
          acc[i][5] = fmaf(v, w1.y, acc[i][5]);
          acc[i][6] = fmaf(v, w1.z, acc[i][6]);
          acc[i][7] = fmaf(v, w1.w, acc[i][7]);
          acc[i][8] = fmaf(v, w2.x, acc[i][8]);
          acc[i][9] = fmaf(v, w2.y, acc[i][9]);
          acc[i][10] = fmaf(v, w2.z, acc[i][10]);
          acc[i][11] = fmaf(v, w2.w, acc[i][11]);
          acc[i][12] = fmaf(v, w3.x, acc[i][12]);
          acc[i][13] = fmaf(v, w3.y, acc[i][13]);
          acc[i][14] = fmaf(v, w3.z, acc[i][14]);
          acc[i][15] = fmaf(v, w3.w, acc[i][15]);
        }
      }
    }
  }
  float b[16];
#pragma unroll
  for (int o = 0; o < 16; ++o) b[o] = __ldg(bias + g * 16 + o);
  const int gy = y0 + ty;
  if (gy >= Ho) return;
#pragma unroll
  for (int i = 0; i < S2_PX; ++i) {
    const int gx = x0 + tx + i * S2_TX;
    if (gx >= Wo) continue;
    float4* o4 = reinterpret_cast<float4*>(out + (((size_t)n * Ho + gy) * Wo + gx) * 64 + g * 16);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float4 r;
      r.x = acc[i][q * 4 + 0] + b[q * 4 + 0];
      r.y = acc[i][q * 4 + 1] + b[q * 4 + 1];
      r.z = acc[i][q * 4 + 2] + b[q * 4 + 2];
      r.w = acc[i][q * 4 + 3] + b[q * 4 + 3];
      if (relu) {
        r.x = fmaxf(r.x, 0.f);
        r.y = fmaxf(r.y, 0.f);
        r.z = fmaxf(r.z, 0.f);
        r.w = fmaxf(r.w, 0.f);
      }
      o4[q] = r;
    }
  }
}

// the ResNet stem: stride 2, 64 outputs, no residual (the tracking stems are summed after their max-pools)
bool stem_s2_supported(const IgemmParams& p) {
  return p.mode == IGEMM_NCHW_SCALAR && p.kh == 7 && p.kw == 7 && p.stride == 2 && p.pad == 3 && p.Cout == 64 &&
         p.CoutPad == 64 && p.Cin <= 8 && !p.out_nchw && p.outStride == 64 && !p.residual;
}

int launch_stem_conv_s2(const IgemmParams& p, cudaStream_t s) {
  const size_t smem = ((size_t)p.Cin * S2_HALO_H * S2_HALO_W + (size_t)49 * p.Cin * 64) * sizeof(float);
  static PerDevice<size_t> configured;
  if (smem > 48 * 1024 && smem > configured.here()) {
    CP_CUDA_CHECK(cudaFuncSetAttribute(stem_conv7s2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured.here() = smem;
  }
  dim3 grid((p.Wout + S2_W - 1) / S2_W, (p.Hout + S2_TY - 1) / S2_TY, p.B);
  dim3 block(S2_TX, S2_TY, S2_G);
  CP_CUDA_CHECK(launch_kernel(stem_conv7s2_kernel, grid, block, smem, s, p.src[0], p.wgt, p.bias, p.out, p.Cin, p.Hin,
                              p.Win, p.Hout, p.Wout, p.relu, model_ipm(p), p.wstride,
                              (p.nchw_per_model & 1u) ? p.B : model_ipm(p)));
  CP_LAUNCH_CHECK("stem_conv7s2_kernel");
  return CP_OK;
}

}  // namespace

bool conv3_c16_supported(const IgemmParams& p) {
  return p.mode == IGEMM_NHWC_VEC && p.nsrc == 1 && p.kh == 3 && p.kw == 3 && p.stride == 1 && p.pad == 1 && p.Cin == 16 &&
         p.Cout == 16 && p.CoutPad == 16 && !p.out_nchw && !p.residual && p.srcStride[0] % 4 == 0 && p.outStride % 4 == 0;
}

int launch_conv3_c16(const IgemmParams& p, cudaStream_t s) {
  if (!conv3_c16_supported(p)) return fail(CP_ERR_INVALID, "conv3_c16: unsupported shape");
  const size_t smem = ((size_t)9 * 16 * 16 + (size_t)16 * C3_PLANE) * sizeof(float);
  static PerDevice<bool> configured;
  if (!configured.here()) {
    CP_CUDA_CHECK(cudaFuncSetAttribute(conv3_c16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured.here() = true;
  }
  dim3 grid((p.Win + C3_W - 1) / C3_W, (p.Hin + C3_TY - 1) / C3_TY, p.B);
  dim3 block(C3_TX, C3_TY);
  CP_CUDA_CHECK(launch_kernel(conv3_c16_kernel, grid, block, smem, s, p.src[0], p.srcStride[0], p.wgt, p.bias, p.out, p.outStride,
                              p.B, p.Hin, p.Win, p.relu, model_ipm(p), p.wstride));
  CP_LAUNCH_CHECK("conv3_c16_kernel");
  return CP_OK;
}

bool stem_supported(const IgemmParams& p) {
  if (stem_s2_supported(p)) return true;
  return p.mode == IGEMM_NCHW_SCALAR && p.kh == 7 && p.kw == 7 && p.stride == 1 && p.pad == 3 && p.Cout == 16 &&
         p.CoutPad == 16 && p.Cin <= 8 && !p.out_nchw && p.outStride == 16 &&
         (!p.residual || (p.res_after_relu && p.resStride == 16));
}

int launch_stem_conv(const IgemmParams& p, cudaStream_t s) {
  if (!stem_supported(p)) return fail(CP_ERR_INVALID, "stem_conv: unsupported shape");
  if (stem_s2_supported(p)) return launch_stem_conv_s2(p, s);
  const size_t smem = ((size_t)p.Cin * ST_HALO_H * ST_HALO_W + (size_t)49 * p.Cin * 16) * sizeof(float);
  static PerDevice<size_t> configured;
  if (smem > 48 * 1024 && smem > configured.here()) {
    CP_CUDA_CHECK(cudaFuncSetAttribute(stem_conv7_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured.here() = smem;
  }
  dim3 grid((p.Win + ST_W - 1) / ST_W, (p.Hin + ST_TY - 1) / ST_TY, p.B);
  dim3 block(ST_TX, ST_TY);
  CP_CUDA_CHECK(launch_kernel(stem_conv7_kernel, grid, block, smem, s, p.src[0], p.wgt, p.bias, p.residual, p.out, p.B, p.Cin,
                              p.Hin, p.Win, p.relu, model_ipm(p), p.wstride,
                              (p.nchw_per_model & 1u) ? p.B : model_ipm(p)));
  CP_LAUNCH_CHECK("stem_conv7_kernel");
  return CP_OK;
}

}  // namespace cp

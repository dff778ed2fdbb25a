// Memory-bound helper kernels: 2x2 max-pool, depthwise transposed-conv
// up-sampling fused with the skip add, weight / BatchNorm packing, layout
// changes, GroupNorm+ReLU and the convGRU gate.  All NHWC fp32, float4 along C.
#include "common.cuh"

namespace cp {
namespace {

constexpr int TPB = 256;

inline int blocks_for(size_t n) {
  size_t b = (n + TPB - 1) / TPB;
  const size_t cap = 132 * 32;  // grid-stride beyond this
  return (int)(b < cap ? (b ? b : 1) : cap);
}

// ---- MaxPool2d(2, 2)  (pose_dla_dcn.py:203) ---------------------------------
__global__ void maxpool2_kernel(const float4* __restrict__ in, float4* __restrict__ out, int B, int H,
                                int W, int C4) {
  griddep_launch_dependents();      // PDL (common.cuh)
  griddep_wait();
  const int Ho = H / 2, Wo = W / 2;
  size_t total = (size_t)B * Ho * Wo * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int c = i % C4;
    size_t t = i / C4;
    int ox = t % Wo;
    t /= Wo;
    int oy = t % Ho;
    int n = t / Ho;
    const float4* p = in + ((size_t)(n * H + 2 * oy) * W + 2 * ox) * C4 + c;
    float4 a = __ldg(p), b = __ldg(p + C4), d = __ldg(p + (size_t)W * C4), e = __ldg(p + (size_t)W * C4 + C4);
    float4 r;
    r.x = fmaxf(fmaxf(a.x, b.x), fmaxf(d.x, e.x));
    r.y = fmaxf(fmaxf(a.y, b.y), fmaxf(d.y, e.y));
    r.z = fmaxf(fmaxf(a.z, b.z), fmaxf(d.z, e.z));
    r.w = fmaxf(fmaxf(a.w, b.w), fmaxf(d.w, e.w));
    out[i] = r;
  }
}

// ---- MaxPool2d(3, 2, 1) (msra_resnet.py:120, 132, 139, 147) [+ residual: the tracking stems' sum, :242-247] ----
// The -inf padding never wins: every window holds its centre (2 oy, 2 ox).  The sum is residual + pool, the order of
// `x = x + self.pre_img_layer(pre_img)`.
__global__ void maxpool3s2_kernel(const float4* __restrict__ in, const float4* __restrict__ res, float4* __restrict__ out,
                                  int B, int H, int W, int C4) {
  griddep_launch_dependents();      // PDL (common.cuh)
  griddep_wait();
  const int Ho = H / 2, Wo = W / 2;
  const size_t total = (size_t)B * Ho * Wo * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = i % C4;
    size_t t = i / C4;
    const int ox = t % Wo;
    t /= Wo;
    const int oy = t % Ho;
    const int n = t / Ho;
    float4 r = __ldg(in + ((size_t)(n * H + 2 * oy) * W + 2 * ox) * C4 + c);
    for (int dy = -1; dy <= 1; ++dy) {
      const int iy = 2 * oy + dy;
      if (iy < 0 || iy >= H) continue;
      for (int dx = -1; dx <= 1; ++dx) {
        const int ix = 2 * ox + dx;
        if (ix < 0 || ix >= W) continue;
        const float4 v = __ldg(in + ((size_t)(n * H + iy) * W + ix) * C4 + c);
        r.x = fmaxf(r.x, v.x);
        r.y = fmaxf(r.y, v.y);
        r.z = fmaxf(r.z, v.z);
        r.w = fmaxf(r.w, v.w);
      }
    }
    if (res) {
      const float4 a = __ldg(res + i);
      r.x = a.x + r.x;
      r.y = a.y + r.y;
      r.z = a.z + r.z;
      r.w = a.w + r.w;
    }
    out[i] = r;
  }
}

// ---- depthwise ConvTranspose2d(C, C, 2f, stride f, pad f/2, groups C) + skip add
//      (pose_dla_dcn.py:402-405, :415-417).  Every output pixel receives exactly
//      2 x 2 taps; weights are packed [ky][kx][C].
// IDX = unsigned for every shape the network uses (< 2^32 float4 elements): the three divisions of the index decode are
// then 32-bit (the 64-bit ones were ~100 instructions per 16 bytes moved and held the kernel at half the HBM rate).
template <typename IDX, bool MULTI>
__global__ void upsample_add_kernel(const float4* __restrict__ in, const float4* __restrict__ w,
                                    const float4* __restrict__ skip, float4* __restrict__ out, int B,
                                    int Hin, int Win, int C4, int f, int ipm, long long wstride4) {
  griddep_launch_dependents();      // PDL (common.cuh)
  griddep_wait();
  const IDX Ho = (IDX)(Hin * f), Wo = (IDX)(Win * f), C4u = (IDX)C4;
  const int k = 2 * f, pad = f / 2;
  const IDX total = (IDX)B * Ho * Wo * C4u;
  for (IDX i = (IDX)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (IDX)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4u);
    IDX t = i / C4u;
    const int ox = (int)(t % Wo);
    t /= Wo;
    const int oy = (int)(t % Ho);
    const int n = (int)(t / Ho);
    float4 acc = skip ? __ldg(skip + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 up = make_float4(0.f, 0.f, 0.f, 0.f);
    int iy_hi = (oy + pad) / f, ky_lo = (oy + pad) - iy_hi * f;
    int ix_hi = (ox + pad) / f, kx_lo = (ox + pad) - ix_hi * f;
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      int iy = iy_hi - a, ky = ky_lo + a * f;
      if (iy < 0 || iy >= Hin || ky >= k) continue;
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        int ix = ix_hi - b, kx = kx_lo + b * f;
        if (ix < 0 || ix >= Win || kx >= k) continue;
        float4 v = __ldg(in + ((size_t)(n * Hin + iy) * Win + ix) * C4 + c);
        float4 ww = __ldg(w + (MULTI ? (size_t)(n / ipm) * wstride4 : 0) + (size_t)(ky * k + kx) * C4 + c);
        up.x = fmaf(v.x, ww.x, up.x);
        up.y = fmaf(v.y, ww.y, up.y);
        up.z = fmaf(v.z, ww.z, up.z);
        up.w = fmaf(v.w, ww.w, up.w);
      }
    }
    acc.x += up.x; acc.y += up.y; acc.z += up.z; acc.w += up.w;
    out[i] = acc;
  }
}

// ---- weight packing ----------------------------------------------------------
// OIHW -> [k = (ky*kw + kx)*Cin + ci][CoutPad], multiplied by the folded BN scale.
__global__ void pack_conv_weight_kernel(const float* __restrict__ w, const float* __restrict__ scale,
                                        float* __restrict__ out, int Cout, int Cin, int kh, int kw,
                                        int CoutPad, int Kpad, int ld, int colOff, int CinPad) {
  size_t total = (size_t)Kpad * CoutPad;
  const int K = kh * kw * CinPad;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int co = i % CoutPad;
    int k = i / CoutPad;
    float v = 0.f;
    if (co < Cout && k < K) {
      int ci = k % CinPad;
      int tap = k / CinPad;
      if (ci < Cin) {
        v = w[((size_t)co * Cin + ci) * kh * kw + tap];
        if (scale) v *= scale[co];
      }
    }
    out[(size_t)k * ld + colOff + co] = v;
  }
}

// ConvTranspose2d [Cin][Cout][4][4] -> phase p = py * 2 + px: [k = (2a + b) * Cin + ci][CoutPad] holds
// w[ci][co][ky(py, a)][kx(px, b)] * scale[co] (IGEMM_DECONV, common.cuh); rows K..Kpad and columns Cout.. are zero.
__global__ void pack_deconv_weight_kernel(const float* __restrict__ w, const float* __restrict__ scale, float* __restrict__ out,
                                          int Cin, int Cout, int CoutPad, int Kpad) {
  const size_t total = (size_t)4 * Kpad * CoutPad;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int co = i % CoutPad;
    const size_t r = i / CoutPad;
    const int k = r % Kpad, ph = r / Kpad;
    float v = 0.f;
    if (co < Cout && k < 4 * Cin) {
      const int ci = k % Cin, tap = k / Cin;
      const int ky = deconv_ky(ph >> 1, tap >> 1), kx = deconv_ky(ph & 1, tap & 1);
      v = w[(((size_t)ci * Cout + co) * 4 + ky) * 4 + kx];
      if (scale) v *= scale[co];
    }
    out[i] = v;
  }
}

// scale = gamma / sqrt(var + eps);  bias = (conv_bias - mean) * scale + beta
// (BatchNorm2d eval folding; any pointer may be null: no BN -> scale 1, bias = conv_bias)
__global__ void pack_bias_kernel(const float* conv_bias, const float* g, const float* b, const float* mean,
                                 const float* var, float* scale_out, float* bias_out, int C, int CPad,
                                 float eps) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= CPad) return;
  float sc = 1.f, bi = 0.f;
  if (i < C) {
    float cb = conv_bias ? conv_bias[i] : 0.f;
    if (g) {
      sc = g[i] / sqrtf(var[i] + eps);
      bi = (cb - mean[i]) * sc + b[i];
    } else {
      bi = cb;
    }
  } else {
    sc = 0.f;
  }
  if (scale_out) scale_out[i] = sc;
  bias_out[i] = bi;
}

// ConvTranspose weight [C,1,k,k] -> [ky][kx][C]
__global__ void pack_up_weight_kernel(const float* __restrict__ w, float* __restrict__ out, int C, int k) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C * k * k) return;
  int c = i % C;
  int t = i / C;
  out[i] = w[(size_t)c * k * k + t];
}

__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int C, int H,
                                    int W, int outStride, int chanOffset) {
  size_t total = (size_t)B * C * H * W;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int c = i % C;
    size_t pix = i / C;   // (n, y, x) flattened
    size_t hw = (size_t)H * W;
    int n = pix / hw;
    size_t r = pix - (size_t)n * hw;
    out[pix * outStride + chanOffset + c] = __ldg(in + ((size_t)n * C + c) * hw + r);
  }
}

__global__ void nhwc_to_nchw_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int C, int H,
                                    int W, int inStride) {
  size_t hw = (size_t)H * W;
  size_t total = (size_t)B * C * hw;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    size_t r = i % hw;
    size_t t = i / hw;
    int c = t % C;
    int n = t / C;
    out[i] = __ldg(in + ((size_t)n * hw + r) * inStride + c);
  }
}

// ---- GroupNorm(groups, C) + ReLU over an NHWC channel slice (GN.py:4-9) -------
// pass 1: per (sample, block, group) partial sum / sum-of-squares in double, each added in a fixed order so that the
// statistics -- and the normalised output -- are bit-reproducible from run to run
__global__ void gn_stats_kernel(const float* __restrict__ x, int HW, int C, int stride, int chanOffset,
                                int groups, double* __restrict__ partial) {
  // grid: (kGnBlocks, B); each block reduces a slab of pixels for all groups
  const int n = blockIdx.y;
  const int cpg = C / groups;
  __shared__ double sh_s[TPB], sh_q[TPB];
  const int pix_per_block = (HW + gridDim.x - 1) / gridDim.x;
  const int p0 = blockIdx.x * pix_per_block;
  const int p1 = min(HW, p0 + pix_per_block);
  // thread t owns channel t % C and strides over pixels with the other C-lanes
  const int c = threadIdx.x % C;
  const int lane = threadIdx.x / C;
  const int nl = blockDim.x / C;
  double s = 0.0, q = 0.0;
  for (int pidx = p0 + lane; pidx < p1; pidx += nl) {
    float v = __ldg(x + ((size_t)n * HW + pidx) * stride + chanOffset + c);
    s += v;
    q += (double)v * v;
  }
  sh_s[threadIdx.x] = s;
  sh_q[threadIdx.x] = q;
  __syncthreads();
  if (threadIdx.x < groups) {
    const int g = threadIdx.x;
    double ss = 0.0, qq = 0.0;
    for (int l = 0; l < nl; ++l)
      for (int cc = g * cpg; cc < (g + 1) * cpg; ++cc) {
        ss += sh_s[l * C + cc];
        qq += sh_q[l * C + cc];
      }
    double* dst = partial + (((size_t)n * gridDim.x + blockIdx.x) * groups + g) * 2;
    dst[0] = ss;
    dst[1] = qq;
  }
}

// pass 2: the partials of every (sample, group) added in block order
__global__ void gn_stats_finish_kernel(const double* __restrict__ partial, int nblocks, int groups,
                                       double* __restrict__ stats) {
  const int n = blockIdx.x;
  for (int i = threadIdx.x; i < groups * 2; i += blockDim.x) {
    double t = 0.0;
    for (int b = 0; b < nblocks; ++b) t += partial[((size_t)n * nblocks + b) * groups * 2 + i];
    stats[(size_t)n * groups * 2 + i] = t;
  }
}

template <bool MULTI>
__global__ void gn_apply_relu_kernel(float* __restrict__ x, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, int B, int HW, int C, int stride,
                                     int chanOffset, int groups, float eps, const double* __restrict__ stats, int ipm,
                                     long long wstride) {
  const int cpg = C / groups;
  size_t total = (size_t)B * HW * C;
  const double cnt = (double)HW * cpg;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int c = i % C;
    size_t pix = i / C;
    int n = pix / HW;
    int g = c / cpg;
    double s = stats[((size_t)n * groups + g) * 2], q = stats[((size_t)n * groups + g) * 2 + 1];
    double mean = s / cnt;
    double var = q / cnt - mean * mean;
    if (var < 0) var = 0;
    float rstd = (float)(1.0 / sqrt(var + (double)eps));
    float* p = x + pix * stride + chanOffset + c;
    const size_t wo = MULTI ? (size_t)(n / ipm) * wstride : 0;      // model n / ipm's gamma and beta
    float v = (*p - (float)mean) * rstd * __ldg(gamma + wo + c) + __ldg(beta + wo + c);
    *p = fmaxf(v, 0.f);
  }
}

// ---- convGRU gate (convGRU.py:32-39) ----------------------------------------
// xi: [M, 3C] = (Wir x + b, Wiz x + b, Win x + b);  hh: [M, 3C] = (Whr h, Whz h, Whn h) or null (h = 0)
__global__ void gru_gates_kernel(const float* __restrict__ xi, const float* __restrict__ hh,
                                 const float* __restrict__ hprev, float* __restrict__ hout, size_t M, int C) {
  size_t total = M * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int c = i % C;
    size_t m = i / C;
    const float* xr = xi + m * 3 * C;
    float hr = 0.f, hz = 0.f, hn = 0.f, h = 0.f;
    if (hh) {
      const float* hp = hh + m * 3 * C;
      hr = hp[c];
      hz = hp[C + c];
      hn = hp[2 * C + c];
      h = hprev[i];
    }
    float r = 1.f / (1.f + expf(-(xr[c] + hr)));
    float z = 1.f / (1.f + expf(-(xr[C + c] + hz)));
    float nn = tanhf(xr[2 * C + c] + r * hn);
    hout[i] = (1.f - z) * nn + z * h;
  }
}

}  // namespace

int launch_maxpool2(const float* in, float* out, int B, int H, int W, int C, cudaStream_t s) {
  if (C % 4 || H % 2 || W % 2) return fail(CP_ERR_INVALID, "maxpool2: C%4, H%2, W%2");
  size_t total = (size_t)B * (H / 2) * (W / 2) * (C / 4);
  CP_CUDA_CHECK(launch_kernel(maxpool2_kernel, dim3(blocks_for(total)), dim3(TPB), 0, s, (const float4*)in, (float4*)out, B, H, W,
                              C / 4));
  CP_LAUNCH_CHECK("maxpool2_kernel");
  return CP_OK;
}

int launch_maxpool3s2(const float* in, const float* res, float* out, int B, int H, int W, int C, cudaStream_t s) {
  if (C % 4 || H % 2 || W % 2) return fail(CP_ERR_INVALID, "maxpool3s2: C%4, H%2, W%2");
  size_t total = (size_t)B * (H / 2) * (W / 2) * (C / 4);
  CP_CUDA_CHECK(launch_kernel(maxpool3s2_kernel, dim3(blocks_for(total)), dim3(TPB), 0, s, (const float4*)in,
                              (const float4*)res, (float4*)out, B, H, W, C / 4));
  CP_LAUNCH_CHECK("maxpool3s2_kernel");
  return CP_OK;
}

int launch_pack_deconv_weight(const float* w, const float* scale, float* out, int Cin, int Cout, int CoutPad, int Kpad,
                              cudaStream_t s) {
  const size_t total = (size_t)4 * Kpad * CoutPad;
  pack_deconv_weight_kernel<<<blocks_for(total), TPB, 0, s>>>(w, scale, out, Cin, Cout, CoutPad, Kpad);
  CP_LAUNCH_CHECK("pack_deconv_weight_kernel");
  return CP_OK;
}

int launch_upsample_add(const float* in, const float* w, const float* skip, float* out, int B, int Hin,
                        int Win, int C, int f, cudaStream_t s, int ipm, long long wstride) {
  if (C % 4) return fail(CP_ERR_INVALID, "upsample: C%4");
  if (ipm <= 0) ipm = B;
  if (wstride % 4) return fail(CP_ERR_INVALID, "upsample: model weight stride % 4");
  size_t total = (size_t)B * Hin * f * Win * f * (C / 4);
  if (total < (1ull << 31))
    CP_CUDA_CHECK(launch_kernel(ipm < B ? upsample_add_kernel<unsigned, true> : upsample_add_kernel<unsigned, false>, dim3(blocks_for(total)), dim3(TPB), 0, s, (const float4*)in,
                                (const float4*)w, (const float4*)skip, (float4*)out, B, Hin, Win, C / 4, f, ipm, wstride / 4));
  else
    CP_CUDA_CHECK(launch_kernel(ipm < B ? upsample_add_kernel<size_t, true> : upsample_add_kernel<size_t, false>, dim3(blocks_for(total)), dim3(TPB), 0, s, (const float4*)in,
                                (const float4*)w, (const float4*)skip, (float4*)out, B, Hin, Win, C / 4, f, ipm, wstride / 4));
  CP_LAUNCH_CHECK("upsample_add_kernel");
  return CP_OK;
}

int launch_pack_conv_weight(const float* w, const float* scale, float* out, int Cout, int Cin, int kh,
                            int kw, int CoutPad, int Kpad, int ld, int colOff, cudaStream_t s, int CinPad) {
  size_t total = (size_t)Kpad * CoutPad;
  pack_conv_weight_kernel<<<blocks_for(total), TPB, 0, s>>>(w, scale, out, Cout, Cin, kh, kw, CoutPad, Kpad,
                                                            ld, colOff, CinPad > 0 ? CinPad : Cin);
  CP_LAUNCH_CHECK("pack_conv_weight_kernel");
  return CP_OK;
}

int launch_pack_bias(const float* conv_bias, const float* g, const float* b, const float* mean,
                     const float* var, float* scale_out, float* bias_out, int C, int CPad, float eps,
                     cudaStream_t s) {
  pack_bias_kernel<<<(CPad + TPB - 1) / TPB, TPB, 0, s>>>(conv_bias, g, b, mean, var, scale_out, bias_out, C,
                                                          CPad, eps);
  CP_LAUNCH_CHECK("pack_bias_kernel");
  return CP_OK;
}

int launch_pack_up_weight(const float* w, float* out, int C, int k, cudaStream_t s) {
  int total = C * k * k;
  pack_up_weight_kernel<<<(total + TPB - 1) / TPB, TPB, 0, s>>>(w, out, C, k);
  CP_LAUNCH_CHECK("pack_up_weight_kernel");
  return CP_OK;
}

int launch_nchw_to_nhwc(const float* in, float* out, int B, int C, int H, int W, int outStride,
                        int chanOffset, cudaStream_t s) {
  size_t total = (size_t)B * C * H * W;
  nchw_to_nhwc_kernel<<<blocks_for(total), TPB, 0, s>>>(in, out, B, C, H, W, outStride, chanOffset);
  CP_LAUNCH_CHECK("nchw_to_nhwc_kernel");
  return CP_OK;
}

int launch_nhwc_to_nchw(const float* in, float* out, int B, int C, int H, int W, int inStride, cudaStream_t s) {
  size_t total = (size_t)B * C * H * W;
  nhwc_to_nchw_kernel<<<blocks_for(total), TPB, 0, s>>>(in, out, B, C, H, W, inStride);
  CP_LAUNCH_CHECK("nhwc_to_nchw_kernel");
  return CP_OK;
}

int launch_group_norm_relu(float* x, const float* gamma, const float* beta, int B, int HW, int C, int stride,
                           int chanOffset, int groups, float eps, double* ws, cudaStream_t s, int ipm, long long wstride) {
  if (C > 256 || 256 % C != 0) return fail(CP_ERR_INVALID, "group_norm: C must divide 256");
  if (groups <= 0 || groups > kGnMaxGroups || C % groups) return fail(CP_ERR_INVALID, "group_norm: bad group count");
  double* stats = ws;                                   // [B][groups][2]
  double* partial = ws + (size_t)B * kGnMaxGroups * 2;   // [B][kGnBlocks][groups][2]
  dim3 grid(kGnBlocks, B);
  gn_stats_kernel<<<grid, TPB, 0, s>>>(x, HW, C, stride, chanOffset, groups, partial);
  CP_LAUNCH_CHECK("gn_stats_kernel");
  gn_stats_finish_kernel<<<B, 64, 0, s>>>(partial, kGnBlocks, groups, stats);
  CP_LAUNCH_CHECK("gn_stats_finish_kernel");
  size_t total = (size_t)B * HW * C;
  if (ipm <= 0) ipm = B;
  // several models in the launch: the model-indexed instantiation
  (ipm < B ? gn_apply_relu_kernel<true> : gn_apply_relu_kernel<false>)<<<blocks_for(total), TPB, 0, s>>>(
      x, gamma, beta, B, HW, C, stride, chanOffset, groups, eps, stats, ipm, wstride);
  CP_LAUNCH_CHECK("gn_apply_relu_kernel");
  return CP_OK;
}

int launch_gru_gates(const float* xi, const float* hh, const float* hprev, float* hout, int M, int C,
                     int first_step, cudaStream_t s) {
  size_t total = (size_t)M * C;
  gru_gates_kernel<<<blocks_for(total), TPB, 0, s>>>(xi, first_step ? nullptr : hh, hprev, hout, (size_t)M, C);
  CP_LAUNCH_CHECK("gru_gates_kernel");
  return CP_OK;
}

}  // namespace cp

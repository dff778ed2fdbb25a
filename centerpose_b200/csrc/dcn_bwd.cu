// DCNv2 backward (SURVEY.md row f-4): gradients of the modulated deformable 3x3 convolution (stride 1, pad 1,
// dilation 1, one deformable group) w.r.t. input, offset, mask, weight and bias.
// Reference semantics: dcn_v2_cuda.cu:206-335 (per image: GEMM -> col2im_coord -> col2im -> im2col -> GEMM -> GEMV)
// with the kernels of dcn_v2_im2col_cuda.cu:197-330 (CPU twins: dcn_v2_im2col_cpu.cpp:58-125, 198-329).
//
// Here the whole batch is one pass over NHWC buffers and the column matrix is touched exactly twice:
//   1. gcol[m][tap * Cp + c] = sum_o W[o][c][tap] * gout[m][o]      -- a 1x1 convolution Co -> 9 Cp over the output
//      gradient, run by the forward convolution kernels (cp::run_conv: FFMA or wgmma, like cp_conv2d)
//   2. dcn_bwd_sample_kernel, one warp per (position, tap), lanes over channels: reads its gcol slice, re-samples the
//      four bilinear corners of the input, accumulates grad_mask / grad_offset (warp reduction, written NCHW), scatters
//      grad_input with vector atomics (NHWC) and OVERWRITES the gcol slice with the forward column value
//      (mask * sampled input) -- the im2col of step 4 of the reference for free
//   3. dcn_bwd_wgrad_kernel: grad_weight / grad_bias = columns^T x gout, a TN GEMM whose reduction runs over the
//      B H W positions; split over position ranges, partial sums added in split order by dcn_bwd_wgrad_finish
//      (deterministic; the reference accumulates image by image through BLAS)
// grad_input uses float atomics like the reference's CUDA col2im (dcn_v2_im2col_cuda.cu:252): its summation order is not
// fixed; everything else is deterministic.
#include "common.cuh"

namespace cp {
namespace {

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float dot4(const float4& a, const float4& b) {
  return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
}

// weights of the 1x1 "transposed" convolution: wp[o][tap * Cp + c] = W[o][c][tap], zero padded to [CoP][NPad]
__global__ void dcn_bwd_pack_w_kernel(const float* __restrict__ w, float* __restrict__ wp, int Co, int C, int CoP, int Cp,
                                      int NPad) {
  const size_t total = (size_t)CoP * NPad;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = (int)(i % NPad), o = (int)(i / NPad);
    const int tap = q / Cp, c = q - tap * Cp;
    float v = 0.f;
    if (o < Co && tap < 9 && c < C) v = __ldg(w + ((size_t)o * C + c) * 9 + tap);
    wp[i] = v;
  }
}

struct SampleArgs {
  const float* x;      // [M][Cp] NHWC input
  const float* om;     // [M][32]: 18 offsets (dy, dx per tap) + 9 masks
  float* gcol;         // [M][ld] in: d(out)/d(column); out: the forward column
  float* gin;          // [M][Cp] NHWC, zeroed
  float* goff;         // [B][18][H][W]
  float* gmask;        // [B][9][H][W]
  int B, H, W, Cp, ld;
};

__global__ void __launch_bounds__(256) dcn_bwd_sample_kernel(const SampleArgs a) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long M = (long long)a.B * a.H * a.W;
  if (warp >= M * 9) return;
  const long long pix = warp / 9;
  const int tap = (int)(warp - pix * 9);
  const int ky = tap / 3, kx = tap - ky * 3;
  const int HW = a.H * a.W;
  const int b = (int)(pix / HW), p = (int)(pix - (long long)b * HW);
  const int oy = p / a.W, ox = p - oy * a.W;
  const float* om = a.om + pix * 32;
  const float off_h = __ldg(om + 2 * tap), off_w = __ldg(om + 2 * tap + 1), mk = __ldg(om + 18 + tap);
  const float h_im = (float)(oy - 1 + ky) + off_h, w_im = (float)(ox - 1 + kx) + off_w;
  // dcn_v2_im2col_cpu.cpp:160 / :62 / :88 / :303: one test decides whether the sample contributes anything
  const bool inside = h_im > -1.f && w_im > -1.f && h_im < (float)a.H && w_im < (float)a.W;
  float* gc = a.gcol + pix * a.ld + tap * a.Cp;
  float mval = 0.f, gh = 0.f, gw = 0.f;
  if (!inside) {
    for (int c0 = lane * 4; c0 < a.Cp; c0 += 128) *reinterpret_cast<float4*>(gc + c0) = make_float4(0.f, 0.f, 0.f, 0.f);
  } else {
    const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
    const int h_high = h_low + 1, w_high = w_low + 1;
    const float lh = h_im - (float)h_low, lw = w_im - (float)w_low;
    const float hh = 1.f - lh, hw = 1.f - lw;
    const bool t_ok = h_low >= 0, b_ok = h_high <= a.H - 1, l_ok = w_low >= 0, r_ok = w_high <= a.W - 1;
    // forward interpolation weights (dmcn_im2col_bilinear, :27-56)
    const float w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;
    // gradient weights of the four corners as dmcn_get_gradient_weight writes them (:58-82)
    const float gA = (float)(h_low + 1) - h_im, gB = (h_im + 1.f) - (float)h_high;
    const float gC = (float)(w_low + 1) - w_im, gD = (w_im + 1.f) - (float)w_high;
    const float q1 = gA * gC, q2 = gA * gD, q3 = gB * gC, q4 = gB * gD;
    // coordinate weights (dmcn_get_coordinate_weight, :84-125)
    const float cw_l = (float)(w_low + 1) - w_im, cw_r = w_im - (float)w_low;     // bp_dir 0 (d / d h)
    const float ch_t = (float)(h_low + 1) - h_im, ch_b = h_im - (float)h_low;     // bp_dir 1 (d / d w)
    const size_t img = (size_t)b * HW;
    const float* x1 = a.x + (img + (size_t)(t_ok ? h_low : 0) * a.W + (l_ok ? w_low : 0)) * a.Cp;
    const float* x2 = a.x + (img + (size_t)(t_ok ? h_low : 0) * a.W + (r_ok ? w_high : 0)) * a.Cp;
    const float* x3 = a.x + (img + (size_t)(b_ok ? h_high : 0) * a.W + (l_ok ? w_low : 0)) * a.Cp;
    const float* x4 = a.x + (img + (size_t)(b_ok ? h_high : 0) * a.W + (r_ok ? w_high : 0)) * a.Cp;
    float* g1 = a.gin + (x1 - a.x);
    float* g2 = a.gin + (x2 - a.x);
    float* g3 = a.gin + (x3 - a.x);
    float* g4 = a.gin + (x4 - a.x);
    const bool ok1 = t_ok && l_ok, ok2 = t_ok && r_ok, ok3 = b_ok && l_ok, ok4 = b_ok && r_ok;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int c0 = lane * 4; c0 < a.Cp; c0 += 128) {
      const float4 g = *reinterpret_cast<const float4*>(gc + c0);
      const float4 v1 = ok1 ? ld4(x1 + c0) : z, v2 = ok2 ? ld4(x2 + c0) : z;
      const float4 v3 = ok3 ? ld4(x3 + c0) : z, v4 = ok4 ? ld4(x4 + c0) : z;
      float4 val;
      val.x = w1 * v1.x + w2 * v2.x + w3 * v3.x + w4 * v4.x;
      val.y = w1 * v1.y + w2 * v2.y + w3 * v3.y + w4 * v4.y;
      val.z = w1 * v1.z + w2 * v2.z + w3 * v3.z + w4 * v4.z;
      val.w = w1 * v1.w + w2 * v2.w + w3 * v3.w + w4 * v4.w;
      mval += dot4(g, val);
      // d(sample) / d(h): -(w_low + 1 - w) x[t,l] - (w - w_low) x[t,r] + (w_low + 1 - w) x[b,l] + (w - w_low) x[b,r]
      float4 dh, dw;
      dh.x = ((-cw_l * v1.x + -cw_r * v2.x) + cw_l * v3.x) + cw_r * v4.x;
      dh.y = ((-cw_l * v1.y + -cw_r * v2.y) + cw_l * v3.y) + cw_r * v4.y;
      dh.z = ((-cw_l * v1.z + -cw_r * v2.z) + cw_l * v3.z) + cw_r * v4.z;
      dh.w = ((-cw_l * v1.w + -cw_r * v2.w) + cw_l * v3.w) + cw_r * v4.w;
      dw.x = ((-ch_t * v1.x + ch_t * v2.x) + -ch_b * v3.x) + ch_b * v4.x;
      dw.y = ((-ch_t * v1.y + ch_t * v2.y) + -ch_b * v3.y) + ch_b * v4.y;
      dw.z = ((-ch_t * v1.z + ch_t * v2.z) + -ch_b * v3.z) + ch_b * v4.z;
      dw.w = ((-ch_t * v1.w + ch_t * v2.w) + -ch_b * v3.w) + ch_b * v4.w;
      gh += (dh.x * g.x) * mk + (dh.y * g.y) * mk + (dh.z * g.z) * mk + (dh.w * g.w) * mk;
      gw += (dw.x * g.x) * mk + (dw.y * g.y) * mk + (dw.z * g.z) * mk + (dw.w * g.w) * mk;
      // col2im (:198-257): cur_top_grad = column gradient * mask, spread over the in-image corners
      const float4 top = make_float4(g.x * mk, g.y * mk, g.z * mk, g.w * mk);
      if (ok1) atomicAdd(reinterpret_cast<float4*>(g1 + c0), make_float4(q1 * top.x, q1 * top.y, q1 * top.z, q1 * top.w));
      if (ok2) atomicAdd(reinterpret_cast<float4*>(g2 + c0), make_float4(q2 * top.x, q2 * top.y, q2 * top.z, q2 * top.w));
      if (ok3) atomicAdd(reinterpret_cast<float4*>(g3 + c0), make_float4(q3 * top.x, q3 * top.y, q3 * top.z, q3 * top.w));
      if (ok4) atomicAdd(reinterpret_cast<float4*>(g4 + c0), make_float4(q4 * top.x, q4 * top.y, q4 * top.z, q4 * top.w));
      // the forward column (im2col, :127-195): val * mask
      *reinterpret_cast<float4*>(gc + c0) = make_float4(val.x * mk, val.y * mk, val.z * mk, val.w * mk);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mval += __shfl_xor_sync(0xffffffffu, mval, o);
    gh += __shfl_xor_sync(0xffffffffu, gh, o);
    gw += __shfl_xor_sync(0xffffffffu, gw, o);
  }
  if (lane == 0) {
    a.goff[((size_t)b * 18 + 2 * tap) * HW + p] = gh;
    a.goff[((size_t)b * 18 + 2 * tap + 1) * HW + p] = gw;
    a.gmask[((size_t)b * 9 + tap) * HW + p] = mval;
  }
}

// part[s][q][o] = sum over the positions of split s of col[m][q] * gout[m][o]; row q == N is the bias row (col == 1).
// 64 x 64 tile, 256 threads, 4 x 4 per thread, 16 positions per shared-memory step.
constexpr int WG_T = 64, WG_K = 16;
__global__ void __launch_bounds__(256) dcn_bwd_wgrad_kernel(const float* __restrict__ col, int ld, const float* __restrict__ go,
                                                           int CoP, long long M, int N, long long rows_per_split,
                                                           float* __restrict__ part) {
  __shared__ __align__(16) float As[WG_K][WG_T], Bs[WG_K][WG_T];
  const int q0 = blockIdx.x * WG_T, o0 = blockIdx.y * WG_T, s = blockIdx.z;
  const long long m0 = (long long)s * rows_per_split, m1 = min(M, m0 + rows_per_split);
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int lr = tid >> 4, lc = (tid & 15) * 4;          // loader: row 0..15, 4 consecutive columns
  float acc[4][4] = {};
  for (long long m = m0; m < m1; m += WG_K) {
    const long long mr = m + lr;
    float4 av = make_float4(0.f, 0.f, 0.f, 0.f), bv = av;
    if (mr < m1) {
      const int q = q0 + lc;
      if (q + 3 < N) {
        av = ld4(col + mr * ld + q);
      } else {
        float t[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) t[j] = (q + j < N) ? __ldg(col + mr * ld + q + j) : ((q + j == N) ? 1.f : 0.f);
        av = make_float4(t[0], t[1], t[2], t[3]);
      }
      if (o0 + lc < CoP) bv = ld4(go + mr * CoP + o0 + lc);
    }
    *reinterpret_cast<float4*>(&As[lr][lc]) = av;
    *reinterpret_cast<float4*>(&Bs[lr][lc]) = bv;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < WG_K; ++k) {
      const float4 a4 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b4 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float aa[4] = {a4.x, a4.y, a4.z, a4.w}, bb[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(aa[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* dst = part + (size_t)s * (N + 1) * CoP;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = q0 + ty * 4 + i;
    if (q > N) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int o = o0 + tx * 4 + j;
      if (o < CoP) dst[(size_t)q * CoP + o] = acc[i][j];
    }
  }
}

// grad_weight[o][c][tap] = sum_s part[s][tap * Cp + c][o];  grad_bias[o] = sum_s part[s][N][o]
__global__ void dcn_bwd_wgrad_finish(const float* __restrict__ part, int S, int N, int CoP, int Cp, int C, int Co,
                                     float* __restrict__ gw, float* __restrict__ gb) {
  const size_t total = (size_t)(N + 1) * Co;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int o = (int)(i % Co), q = (int)(i / Co);
    float v = 0.f;
    for (int s = 0; s < S; ++s) v += __ldg(part + ((size_t)s * (N + 1) + q) * CoP + o);
    if (q == N) {
      gb[o] = v;
    } else {
      const int tap = q / Cp, c = q - tap * Cp;
      if (c < C) gw[((size_t)o * C + c) * 9 + tap] = v;
    }
  }
}

}  // namespace

// shapes the tensor-core kernels do not take (a few channels) run on the FFMA kernel: same result class, fp32
constexpr ConvPolicy kColumnGemm{false, true, false, true};

int dcn_v2_backward_impl(const float* input, const float* weight, const float* offset, const float* mask,
                         const float* grad_output, float* grad_input, float* grad_offset, float* grad_mask,
                         float* grad_weight, float* grad_bias, int B, int C, int H, int W, int Co,
                         int32_t precision, cudaStream_t s) {
  const int Cp = round_up(C, 16), CoP = round_up(Co, 16);
  const int N = 9 * Cp, NPad = round_up(N, 64);
  const long long M = (long long)B * H * W;
  // split the position range of the weight-gradient GEMM so that the grid fills the SMs a few times over
  int num_sms = 0;
  if (int rc = device_sm_count(&num_sms)) return rc;
  const int tiles = ((N + 1 + WG_T - 1) / WG_T) * ((CoP + WG_T - 1) / WG_T);
  int S = (4 * num_sms + tiles - 1) / tiles;
  const long long max_s = (M + 255) / 256;
  if (S > max_s) S = (int)max_s;
  if (S < 1) S = 1;
  long long rps = ((M + S - 1) / S + WG_K - 1) / WG_K * WG_K;
  S = (int)((M + rps - 1) / rps);
  const size_t n_x = (size_t)M * Cp, n_go = (size_t)M * CoP, n_om = (size_t)M * 32, n_col = (size_t)M * N;
  const size_t n_wp = (size_t)CoP * NPad, n_part = (size_t)S * (N + 1) * CoP;
  float* scratch = nullptr;
  CP_CUDA_CHECK(cudaMallocAsync(&scratch, (2 * n_x + n_go + n_om + n_col + n_wp + NPad + n_part) * sizeof(float), s));
  float* x = scratch;
  float* gin = x + n_x;
  float* go = gin + n_x;
  float* om = go + n_go;
  float* gcol = om + n_om;
  float* wp = gcol + n_col;
  float* bz = wp + n_wp;
  float* part = bz + NPad;
  int rc = CP_OK;
  do {
    if (cudaMemsetAsync(x, 0, (2 * n_x + n_go) * sizeof(float), s) != cudaSuccess ||
        cudaMemsetAsync(bz, 0, NPad * sizeof(float), s) != cudaSuccess) {
      rc = fail(CP_ERR_CUDA, "cp_dcn_v2_backward: memset");
      break;
    }
    if ((rc = launch_nchw_to_nhwc(input, x, B, C, H, W, Cp, 0, s))) break;
    if ((rc = launch_nchw_to_nhwc(grad_output, go, B, Co, H, W, CoP, 0, s))) break;
    if ((rc = launch_nchw_to_nhwc(offset, om, B, 18, H, W, 32, 0, s))) break;
    if ((rc = launch_nchw_to_nhwc(mask, om, B, 9, H, W, 32, 18, s))) break;
    {
      const size_t total = n_wp;
      int blocks = (int)((total + 255) / 256);
      if (blocks > 132 * 8) blocks = 132 * 8;
      dcn_bwd_pack_w_kernel<<<blocks, 256, 0, s>>>(weight, wp, Co, C, CoP, Cp, NPad);
      CP_LAUNCH_CHECK("dcn_bwd_pack_w_kernel");
    }
    // 1. column gradients: 1x1 convolution CoP -> N over the output gradient
    IgemmParams p{};
    p.nsrc = 1;
    p.src[0] = go;
    p.srcC[0] = CoP;
    p.srcStride[0] = CoP;
    p.B = B;
    p.Hin = p.Hout = H;
    p.Win = p.Wout = W;
    p.Cin = CoP;
    p.kh = p.kw = 1;
    p.stride = 1;
    p.pad = 0;
    p.Cout = N;
    p.CoutPad = NPad;
    p.Kpad = CoP;
    p.wgt = wp;
    p.bias = bz;
    p.out = gcol;
    p.outStride = N;
    p.mode = IGEMM_NHWC_VEC;
    if ((rc = run_conv(p, precision, kColumnGemm, s))) break;
    // 2. sampling pass
    SampleArgs a;
    a.x = x;
    a.om = om;
    a.gcol = gcol;
    a.gin = gin;
    a.goff = grad_offset;
    a.gmask = grad_mask;
    a.B = B;
    a.H = H;
    a.W = W;
    a.Cp = Cp;
    a.ld = N;
    const long long warps = M * 9;
    dcn_bwd_sample_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, s>>>(a);
    CP_LAUNCH_CHECK("dcn_bwd_sample_kernel");
    if ((rc = launch_nhwc_to_nchw(gin, grad_input, B, C, H, W, Cp, s))) break;
    // 3. weight / bias gradients
    dim3 grid((N + 1 + WG_T - 1) / WG_T, (CoP + WG_T - 1) / WG_T, S);
    dcn_bwd_wgrad_kernel<<<grid, 256, 0, s>>>(gcol, N, go, CoP, M, N, rps, part);
    CP_LAUNCH_CHECK("dcn_bwd_wgrad_kernel");
    {
      const size_t total = (size_t)(N + 1) * Co;
      int blocks = (int)((total + 255) / 256);
      if (blocks > 132 * 8) blocks = 132 * 8;
      dcn_bwd_wgrad_finish<<<blocks, 256, 0, s>>>(part, S, N, CoP, Cp, C, Co, grad_weight, grad_bias);
      CP_LAUNCH_CHECK("dcn_bwd_wgrad_finish");
    }
  } while (0);
  cudaFreeAsync(scratch, s);
  return rc;
}

}  // namespace cp

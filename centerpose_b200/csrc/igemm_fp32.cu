// fp32 implicit-GEMM convolution on CUDA cores -- the parity-mode kernel.
//
// One kernel family covers every dense contraction of the CenterPose network:
//   * 3x3 / 1x1 convolutions over NHWC activations, with channel concatenation
//     of up to four sources (DLA Root nodes, pose_dla_dcn.py:160-168),
//   * the 7x7 stems reading the user's NCHW input directly
//     (pose_dla_dcn.py:234-238, 253-271),
//   * the dense 4x4 stride-2 transposed convolutions of the ResNet up-sampling (msra_resnet.py:208-233), as four
//     sub-pixel phase GEMMs over the input (IGEMM_DECONV, common.cuh; the phase is blockIdx.z),
//   * the DCNv2 modulated deformable 3x3 convolution: the A tile is produced by
//     bilinear sampling at offset positions and multiplied by the mask, exactly
//     the arithmetic of dcn_v2_im2col_cuda.cu:25-54,125-195, but the
//     `columns[B, 9C, HW]` matrix is never written to HBM.
// Epilogue: + folded bias, optional residual (before or after ReLU), ReLU,
// NHWC or NCHW store.
//
// Tiling: BM = 128 output pixels x BN in {16, 32, 64} channels x BK = 16,
// 256 threads, each thread an 8 x (BN/16) register tile, double-buffered
// shared memory with register prefetch of the next K tile.
#include "common.cuh"

namespace cp {

namespace {

constexpr int BM = 128;
constexpr int BK = 16;
constexpr int NT = 256;
constexpr int APAD = 4;

struct RowCtx {
  int n, oy, ox;   // decoded output pixel
  bool valid;
};

// per-(row, tap) deformable sampling state
struct DcnTap {
  float w1, w2, w3, w4, mask;
  int o1, o2, o3, o4;  // pixel offsets (in pixels, not floats) of the 4 corners, clamped in-bounds
};


// MULTI: the launch holds several models (IgemmParams::ipm); otherwise the code is that of one model
template <int BN, int MODE, bool MULTI>
__global__ void __launch_bounds__(NT, 2) igemm_fp32_kernel(const IgemmParams p) {
  constexpr int TN = BN / 16;
  __shared__ __align__(16) float As[2][BK][BM + APAD];
  __shared__ __align__(16) float Bs[2][BK][BN];
  griddep_launch_dependents();      // PDL (common.cuh)
  griddep_wait();

  const int tid = threadIdx.x;
  const int tx = tid & 15;
  const int ty = tid >> 4;
  // the GEMM rows: output pixels, or for IGEMM_DECONV the input pixels of phase blockIdx.z = py * 2 + px
  constexpr bool DECONV = MODE == IGEMM_DECONV;
  const int Hg = DECONV ? p.Hin : p.Hout, Wg = DECONV ? p.Win : p.Wout;
  const int py = blockIdx.z >> 1, px = blockIdx.z & 1;
  // row blocks are cut per model (IgemmParams::ipm); rows from M on belong to the next model
  const int Mm = MULTI ? p.ipm * Hg * Wg : 0;
  const int bpm = MULTI ? (Mm + BM - 1) / BM : 1;
  const int model = MULTI ? blockIdx.x / bpm : 0;
  const int M = MULTI ? (model + 1) * Mm : p.B * Hg * Wg;
  const int m0 = MULTI ? model * Mm + (blockIdx.x - model * bpm) * BM : blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const float* const wgt = (MULTI ? p.wgt + (size_t)model * p.wstride : p.wgt) + (size_t)blockIdx.z * p.Kpad * p.CoutPad;
  // NCHW sources are the models' shared input frames, unless each model has its own (IgemmParams::nchw_per_model)
  const int n_shared = (MULTI && !(p.nchw_per_model & 1u)) ? model * p.ipm : 0;

  // ---- A-load assignment: this thread fills k-quad `kq` of rows r0 and r0+64
  const int kq = tid & 3;
  const int r0 = tid >> 2;
  RowCtx row[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    int m = m0 + r0 + i * 64;
    row[i].valid = m < M;
    int mm = row[i].valid ? m : 0;
    row[i].ox = mm % Wg;
    int t = mm / Wg;
    row[i].oy = t % Hg;
    row[i].n = t / Hg;
  }

  const int ktiles = p.Kpad / BK;
  const int chunks_per_tap = (MODE == IGEMM_NCHW_SCALAR) ? 1 : p.Cin / BK;

  float4 a_reg[2];
  float4 b_reg;
  DcnTap dt[2];

  auto load_tile = [&](int kt) {
    // ---------------- B tile
    if (tid < BK * BN / 4) {
      int k = tid / (BN / 4);
      int n4 = tid % (BN / 4);
      b_reg = __ldg(reinterpret_cast<const float4*>(wgt + (size_t)(kt * BK + k) * p.CoutPad + n0 + n4 * 4));
    }
    // ---------------- A tile
    if (MODE == IGEMM_NCHW_SCALAR) {
      const int K = p.kh * p.kw * p.Cin;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          int k = kt * BK + kq * 4 + j;
          float x = 0.f;
          if (row[i].valid && k < K) {
            int c = k % p.Cin;
            int tap = k / p.Cin;
            int ky = tap / p.kw, kx = tap % p.kw;
            int iy = row[i].oy * p.stride - p.pad + ky;
            int ix = row[i].ox * p.stride - p.pad + kx;
            if (iy >= 0 && iy < p.Hin && ix >= 0 && ix < p.Win)
              x = __ldg(p.src[0] + (((size_t)(row[i].n - n_shared) * p.Cin + c) * p.Hin + iy) * p.Win + ix);
          }
          v[j] = x;
        }
        a_reg[i] = make_float4(v[0], v[1], v[2], v[3]);
      }
    } else if (DECONV) {
      const int tap = kt / chunks_per_tap;
      const int c0 = (kt - tap * chunks_per_tap) * BK;
      const int dy = deconv_dy(py, tap >> 1), dx = deconv_dy(px, tap & 1);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int iy = row[i].oy + dy, ix = row[i].ox + dx;
        const bool ok = row[i].valid && iy >= 0 && iy < p.Hin && ix >= 0 && ix < p.Win;
        a_reg[i] = ok ? __ldg(reinterpret_cast<const float4*>(
                            p.src[0] + ((size_t)(row[i].n * p.Hin + iy) * p.Win + ix) * p.srcStride[0] + c0 + kq * 4))
                      : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    } else if (MODE == IGEMM_NHWC_VEC) {
      int tap = kt / chunks_per_tap;
      int c0 = (kt - tap * chunks_per_tap) * BK;
      int ky = tap / p.kw, kx = tap - ky * p.kw;
      // locate the source that owns channel c0 (uniform over the CTA)
      int s = 0, cbase = 0;
      while (s + 1 < p.nsrc && c0 >= cbase + p.srcC[s]) { cbase += p.srcC[s]; ++s; }
      const float* sp = p.src[s];
      const int sstride = p.srcStride[s];
      const int cl = c0 - cbase + kq * 4;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        int iy = row[i].oy * p.stride - p.pad + ky;
        int ix = row[i].ox * p.stride - p.pad + kx;
        bool ok = row[i].valid && iy >= 0 && iy < p.Hin && ix >= 0 && ix < p.Win;
        a_reg[i] = ok ? __ldg(reinterpret_cast<const float4*>(
                            sp + ((size_t)(row[i].n * p.Hin + iy) * p.Win + ix) * sstride + cl))
                      : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    } else {  // IGEMM_DCN
      int tap = kt / chunks_per_tap;
      int c0 = (kt - tap * chunks_per_tap) * BK;
      if (c0 == 0) {
        int ky = tap / 3, kx = tap - ky * 3;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          DcnTap d;
          d.w1 = d.w2 = d.w3 = d.w4 = 0.f;
          d.mask = 0.f;
          d.o1 = d.o2 = d.o3 = d.o4 = 0;
          if (row[i].valid) {
            const float* om = p.offmask +
                              ((size_t)(row[i].n * p.Hout + row[i].oy) * p.Wout + row[i].ox) * p.omStride;
            float dy = __ldg(om + 2 * tap);
            float dx = __ldg(om + 2 * tap + 1);
            float mk = __ldg(om + 18 + tap);
            if (p.mask_is_logit) mk = 1.0f / (1.0f + expf(-mk));
            float h_im = (float)(row[i].oy - 1 + ky) + dy;
            float w_im = (float)(row[i].ox - 1 + kx) + dx;
            const int H = p.Hin, W = p.Win;
            if (h_im > -1.f && w_im > -1.f && h_im < (float)H && w_im < (float)W) {
              int h_low = (int)floorf(h_im);
              int w_low = (int)floorf(w_im);
              int h_high = h_low + 1, w_high = w_low + 1;
              float lh = h_im - (float)h_low, lw = w_im - (float)w_low;
              float hh = 1.f - lh, hw = 1.f - lw;
              bool t_ok = h_low >= 0, b_ok = h_high <= H - 1;
              bool l_ok = w_low >= 0, r_ok = w_high <= W - 1;
              int hl = t_ok ? h_low : 0, hhh = b_ok ? h_high : H - 1;
              int wl = l_ok ? w_low : 0, whh = r_ok ? w_high : W - 1;
              d.w1 = (t_ok && l_ok) ? hh * hw : 0.f;
              d.w2 = (t_ok && r_ok) ? hh * lw : 0.f;
              d.w3 = (b_ok && l_ok) ? lh * hw : 0.f;
              d.w4 = (b_ok && r_ok) ? lh * lw : 0.f;
              d.o1 = hl * W + wl;
              d.o2 = hl * W + whh;
              d.o3 = hhh * W + wl;
              d.o4 = hhh * W + whh;
              d.mask = mk;
            }
          }
          dt[i] = d;
        }
      }
      const int sstride = p.srcStride[0];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float* base = p.src[0] + (size_t)row[i].n * p.Hin * p.Win * sstride + c0 + kq * 4;
        float4 v1 = __ldg(reinterpret_cast<const float4*>(base + (size_t)dt[i].o1 * sstride));
        float4 v2 = __ldg(reinterpret_cast<const float4*>(base + (size_t)dt[i].o2 * sstride));
        float4 v3 = __ldg(reinterpret_cast<const float4*>(base + (size_t)dt[i].o3 * sstride));
        float4 v4 = __ldg(reinterpret_cast<const float4*>(base + (size_t)dt[i].o4 * sstride));
        float4 r;
        r.x = (dt[i].w1 * v1.x + dt[i].w2 * v2.x + dt[i].w3 * v3.x + dt[i].w4 * v4.x) * dt[i].mask;
        r.y = (dt[i].w1 * v1.y + dt[i].w2 * v2.y + dt[i].w3 * v3.y + dt[i].w4 * v4.y) * dt[i].mask;
        r.z = (dt[i].w1 * v1.z + dt[i].w2 * v2.z + dt[i].w3 * v3.z + dt[i].w4 * v4.z) * dt[i].mask;
        r.w = (dt[i].w1 * v1.w + dt[i].w2 * v2.w + dt[i].w3 * v3.w + dt[i].w4 * v4.w) * dt[i].mask;
        a_reg[i] = r;
      }
    }
  };

  auto store_tile = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      int r = r0 + i * 64;
      As[buf][kq * 4 + 0][r] = a_reg[i].x;
      As[buf][kq * 4 + 1][r] = a_reg[i].y;
      As[buf][kq * 4 + 2][r] = a_reg[i].z;
      As[buf][kq * 4 + 3][r] = a_reg[i].w;
    }
    if (tid < BK * BN / 4) {
      int k = tid / (BN / 4);
      int n4 = tid % (BN / 4);
      *reinterpret_cast<float4*>(&Bs[buf][k][n4 * 4]) = b_reg;
    }
  };

  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  load_tile(0);
  store_tile(0);
  __syncthreads();

  for (int kt = 0; kt < ktiles; ++kt) {
    const int cur = kt & 1;
    if (kt + 1 < ktiles) load_tile(kt + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[8], b[TN];
      float4 a0 = *reinterpret_cast<const float4*>(&As[cur][k][ty * 8]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[cur][k][ty * 8 + 4]);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w;
      a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
      if (TN == 4) {
        float4 bv = *reinterpret_cast<const float4*>(&Bs[cur][k][tx * 4]);
        b[0] = bv.x; b[1 % TN] = bv.y; b[2 % TN] = bv.z; b[3 % TN] = bv.w;
      } else if (TN == 2) {
        float2 bv = *reinterpret_cast<const float2*>(&Bs[cur][k][tx * 2]);
        b[0] = bv.x; b[1 % TN] = bv.y;
      } else {
        b[0] = Bs[cur][k][tx];
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < ktiles) {
      store_tile(cur ^ 1);
      __syncthreads();
    }
  }

  // ---------------- epilogue
  float bias[TN];
#pragma unroll
  for (int j = 0; j < TN; ++j) bias[j] = __ldg((MULTI ? p.bias + (size_t)model * p.wstride : p.bias) + n0 + tx * TN + j);

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int m = m0 + ty * 8 + i;
    if (m >= M) continue;
    if (DECONV) {      // input pixel (n, y, x) of phase (py, px) -> output pixel (n, 2y + py, 2x + px)
      const int x = m % Wg, t = m / Wg;
      m = ((t / Hg) * p.Hout + 2 * (t % Hg) + py) * p.Wout + 2 * x + px;
    }
    float v[TN];
#pragma unroll
    for (int j = 0; j < TN; ++j) v[j] = acc[i][j] + bias[j];
    const int nbase = n0 + tx * TN;
    if (p.residual && !p.res_after_relu) {
#pragma unroll
      for (int j = 0; j < TN; ++j)
        if (nbase + j < p.Cout) v[j] += __ldg(p.residual + (size_t)m * p.resStride + nbase + j);
    }
    if (p.relu) {
#pragma unroll
      for (int j = 0; j < TN; ++j) v[j] = fmaxf(v[j], 0.f);
    }
    if (p.residual && p.res_after_relu) {
#pragma unroll
      for (int j = 0; j < TN; ++j)
        if (nbase + j < p.Cout) v[j] += __ldg(p.residual + (size_t)m * p.resStride + nbase + j);
    }
    if (p.out_nchw) {
      int ox = m % p.Wout;
      int t = m / p.Wout;
      int oy = t % p.Hout;
      int n = t / p.Hout;
#pragma unroll
      for (int j = 0; j < TN; ++j)
        if (nbase + j < p.Cout)
          p.out[(((size_t)n * p.Cout + nbase + j) * p.Hout + oy) * p.Wout + ox] = v[j];
    } else {
      float* o = p.out + (size_t)m * p.outStride + nbase;
      if (TN == 4 && nbase + 3 < p.Cout) {
        *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1 % TN], v[2 % TN], v[3 % TN]);
      } else {
#pragma unroll
        for (int j = 0; j < TN; ++j)
          if (nbase + j < p.Cout) o[j] = v[j];
      }
    }
  }
}

template <int BN, bool MULTI>
int launch_bn_models(const IgemmParams& p, dim3 grid, cudaStream_t stream) {
  switch (p.mode) {
    case IGEMM_NCHW_SCALAR: CP_CUDA_CHECK(launch_kernel(igemm_fp32_kernel<BN, IGEMM_NCHW_SCALAR, MULTI>, grid, dim3(NT), 0, stream, p)); break;
    case IGEMM_NHWC_VEC: CP_CUDA_CHECK(launch_kernel(igemm_fp32_kernel<BN, IGEMM_NHWC_VEC, MULTI>, grid, dim3(NT), 0, stream, p)); break;
    case IGEMM_DCN: CP_CUDA_CHECK(launch_kernel(igemm_fp32_kernel<BN, IGEMM_DCN, MULTI>, grid, dim3(NT), 0, stream, p)); break;
    case IGEMM_DECONV: CP_CUDA_CHECK(launch_kernel(igemm_fp32_kernel<BN, IGEMM_DECONV, MULTI>, grid, dim3(NT), 0, stream, p)); break;
    default: return fail(CP_ERR_INVALID, "igemm: bad mode");
  }
  CP_LAUNCH_CHECK("igemm_fp32_kernel");
  return CP_OK;
}

template <int BN>
int launch_bn(const IgemmParams& p0, cudaStream_t stream) {
  IgemmParams p = p0;
  p.ipm = model_ipm(p0);
  const bool deconv = p.mode == IGEMM_DECONV;
  const int Mm = p.ipm * (deconv ? p.Hin * p.Win : p.Hout * p.Wout);
  dim3 grid((Mm + BM - 1) / BM * (p.B / p.ipm), p.CoutPad / BN, deconv ? 4 : 1);
  // several models in the launch: the model-indexed instantiations; one model runs the one-model code unchanged
  return p.B > p.ipm ? launch_bn_models<BN, true>(p, grid, stream) : launch_bn_models<BN, false>(p, grid, stream);
}

}  // namespace

int launch_igemm_fp32(const IgemmParams& p, cudaStream_t stream) {
  if (p.Kpad % BK != 0) return fail(CP_ERR_INVALID, "igemm: Kpad must be a multiple of 16");
  if (p.B % model_ipm(p)) return fail(CP_ERR_INVALID, "igemm: batch is not a whole number of models");
  if (p.mode != IGEMM_NCHW_SCALAR) {
    if (p.Cin % BK != 0) return fail(CP_ERR_INVALID, "igemm: Cin must be a multiple of 16 for NHWC modes");
    for (int s = 0; s < p.nsrc; ++s)
      if (p.srcC[s] % BK != 0 || p.srcStride[s] % 4 != 0)
        return fail(CP_ERR_INVALID, "igemm: source channels must be a multiple of 16");
    if (p.Kpad != p.kh * p.kw * p.Cin) return fail(CP_ERR_INVALID, "igemm: Kpad mismatch");
  }
  if (p.mode == IGEMM_DCN && (p.kh != 3 || p.kw != 3 || p.stride != 1 || p.pad != 1 || p.nsrc != 1))
    return fail(CP_ERR_INVALID, "igemm: DCN supports 3x3 stride 1 pad 1 only");
  if (p.mode == IGEMM_DECONV &&
      (p.kh != 2 || p.kw != 2 || p.nsrc != 1 || p.out_nchw || p.Hout != 2 * p.Hin || p.Wout != 2 * p.Win))
    return fail(CP_ERR_INVALID, "igemm: transposed conv needs one NHWC source, 2x2 phase taps and an NHWC 2x output");
  if (!p.out_nchw && (p.outStride % 4 != 0)) return fail(CP_ERR_INVALID, "igemm: outStride % 4");
  if (p.CoutPad % 64 == 0) return launch_bn<64>(p, stream);
  if (p.CoutPad % 32 == 0) return launch_bn<32>(p, stream);
  if (p.CoutPad % 16 == 0) return launch_bn<16>(p, stream);
  return fail(CP_ERR_INVALID, "igemm: CoutPad must be a multiple of 16");
}

}  // namespace cp

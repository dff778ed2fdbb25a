// wgmma (Hopper warpgroup MMA) implicit-GEMM convolution for sm_90a.
//
//   D[m, n] = sum_k A[m, k] * W[n, k]      m = output pixel, n = output channel, k = (tap, ci)
//
// Same contract as igemm_fp32.cu (IgemmParams: NHWC fp32 activations, channel-concatenated
// sources, DCNv2 deformable gather, the sub-pixel phases of the 4x4 stride-2 transposed conv with the phase in
// blockIdx.y, fused bias / residual / ReLU epilogue) but the contraction
// runs on the tensor cores:
//   * warps 0-7 (two threads per tile row) GATHER the A tile -- plain im2col rows or the
//     bilinear deformable samples of dcn_v2_im2col_cuda.cu:125-195 -- convert it and write it
//     straight into shared memory in the canonical K-major SWIZZLE_128B layout the wgmma
//     descriptor expects (a data-dependent gather cannot come from TMA); thread 0 also streams
//     the weight tile of the stage, pre-swizzled at load time, with one cp.async.bulk;
//   * warpgroups 2 and 3 each multiply 64 rows of the tile (wgmma m64nBN) into register
//     accumulators and run the epilogue.
// Precisions:
//   PREC_BF16   bf16 operands, fp32 accumulate                                  (fast mode)
//   PREC_TF32X3 tf32, 3-term split  a_hi*b_hi + a_lo*b_hi + a_hi*b_lo           (fp32-equivalent mode; the gather
//               writes fp32 A tiles, the consumers split them into hi / lo in registers: mma_kblock_x3)
// Every mbarrier wait carries a clock64 watchdog that traps instead of hanging the GPU.
#include "common.cuh"
#include "umma_common.cuh"

namespace cp {
namespace {

constexpr int UM_BM = 128;
constexpr int UM_PROD_WARPS = 8;            // A-gather warps: two threads per tile row, 4 chunks each
constexpr int UM_THREADS = (UM_PROD_WARPS + 8) * 32;       // + two consumer warpgroups
constexpr uint32_t ROW_BYTES = 128;        // one K block = 128 bytes per row (64 bf16 / 32 tf32)
constexpr uint32_t A_TILE_BYTES = UM_BM * ROW_BYTES;

using namespace umma;

struct UmmaSmem {   // control block at the head of dynamic smem (the tiles follow, 1024-byte aligned)
  unsigned long long full[8];
  unsigned long long empty[8];
};

template <int PREC>
struct PrecTraits;
template <>
struct PrecTraits<0> {   // bf16
  static constexpr int kElems = 64, kChunkCh = 8, kTilesB = 1;
};
template <>
struct PrecTraits<1> {   // tf32 x 3
  static constexpr int kElems = 32, kChunkCh = 4, kTilesB = 2;     // hi + lo weight tiles
};

// ------------------------------------------------------------------ the kernel
// MULTI: the launch holds several models (IgemmParams::ipm); otherwise the code is that of one model
template <int PREC, int MODE, int BN, bool MULTI>
__global__ void __launch_bounds__(UM_THREADS, 1) igemm_umma_kernel(const IgemmParams p, const int STAGES, const int NACC) {
  using T = PrecTraits<PREC>;
  extern __shared__ __align__(1024) unsigned char smem[];
  UmmaSmem* ctl = reinterpret_cast<UmmaSmem*>(smem);
  if (threadIdx.x == 0) griddep_launch_dependents();      // PDL (common.cuh)
  const uint32_t tiles0 = (smem_u32(smem) + 512u + 1023u) & ~1023u;   // first tile, 1024-aligned
  const uint32_t b_tile_bytes = (uint32_t)BN * ROW_BYTES * T::kTilesB; // hi (+ lo) weight tiles of one stage
  const uint32_t stage_bytes = A_TILE_BYTES + b_tile_bytes;

  const int tid = threadIdx.x, warp = tid >> 5;
  // 1-D grid, n tile fastest: the CTAs that share an A row block run back to back and hit it in L2
  // (gridDim.y would overflow at 65535 row blocks: B = 32 at 512 x 512 has 65536).  Row blocks are cut per model
  // (IgemmParams::ipm) so that a block never mixes two models' weights; rows from M on belong to the next model.
  // The GEMM rows are output pixels, or for IGEMM_DECONV the input pixels of phase blockIdx.y = py * 2 + px, whose
  // weight tiles follow the previous phases' (common.cuh).
  constexpr bool DECONV = MODE == IGEMM_DECONV;
  const int Hg = DECONV ? p.Hin : p.Hout, Wg = DECONV ? p.Win : p.Wout;
  const int py = blockIdx.y >> 1, px = blockIdx.y & 1;
  const int n_tiles = p.CoutPad / BN;
  const int n_tile = blockIdx.x % n_tiles;
  const int Mm = MULTI ? p.ipm * Hg * Wg : 0;
  const int bpm = MULTI ? (Mm + UM_BM - 1) / UM_BM : 1;
  const int model = MULTI ? (blockIdx.x / n_tiles) / bpm : 0;
  const int m0 = MULTI ? model * Mm + ((blockIdx.x / n_tiles) - model * bpm) * UM_BM : (blockIdx.x / n_tiles) * UM_BM;
  const int M = MULTI ? (model + 1) * Mm : p.B * Hg * Wg;
  const int K = p.kh * p.kw * p.Cin;
  const int KB = (K + T::kElems - 1) / T::kElems;

  // one ring of (A tile, weight tile) stages; full: every gather thread + the weight copy's expect_tx arrival, empty:
  // one arrival per consumer warpgroup
  Ring ring{ctl->full, ctl->empty, STAGES};
  if (tid == 0) {
    ring_init(ring, UM_PROD_WARPS * 32 + 1, 2);
    fence_mbar_init();
  }
  __syncthreads();
  griddep_wait();      // PDL: the prologue above is private to the CTA; activations are read from here on

  if (warp < UM_PROD_WARPS) {
    // =========================== A producers: two threads per tile row, four 16-byte chunks each ===============
    {
      const unsigned char* wsrc =
          reinterpret_cast<const unsigned char*>(p.wgt_umma) + (size_t)model * p.tstride +
          ((size_t)blockIdx.y * n_tiles + n_tile) * KB * b_tile_bytes;
      const int r = tid >> 1;
      const int qbase = (tid & 1) * 4;
      const int m = m0 + r;
      const bool valid = m < M;
      int ox = 0, oy = 0, n = 0;
      if (valid) {
        ox = m % Wg;
        int t = m / Wg;
        oy = t % Hg;
        n = t / Hg;
      }
      const uint32_t row_off = (uint32_t)(r >> 3) * 1024u + (uint32_t)(r & 7) * 128u;
      const uint32_t sw = (uint32_t)(r & 7);
      // DCN sampling state of the current tap
      float w1 = 0, w2 = 0, w3 = 0, w4 = 0, mk = 0;
      int o1 = 0, o2 = 0, o3 = 0, o4 = 0;
      int cur_tap = -1;
      constexpr int F4 = T::kChunkCh / 4;     // float4 loads per chunk (2 for bf16, 1 for tf32)

      for (int kb = 0; kb < KB; ++kb) {
        // ---- issue every global load of this thread's 4 chunks first (memory-level parallelism) ...
        float4 ld[4][MODE == IGEMM_DCN ? 4 * F4 : F4];
        bool live[4];
#pragma unroll
        for (int qi = 0; qi < 4; ++qi) {
          const int k0 = kb * T::kElems + (qbase + qi) * T::kChunkCh;
          live[qi] = false;
#pragma unroll
          for (int j = 0; j < (MODE == IGEMM_DCN ? 4 * F4 : F4); ++j) ld[qi][j] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (valid && k0 < K) {
            const int tap = k0 / p.Cin;
            const int c = k0 - tap * p.Cin;
            if (MODE == IGEMM_DCN) {
              if (tap != cur_tap) {
                cur_tap = tap;
                const int ky = tap / 3, kx = tap - ky * 3;
                const float* om = p.offmask + ((size_t)(n * p.Hout + oy) * p.Wout + ox) * p.omStride;
                const float dy = __ldg(om + 2 * tap), dx = __ldg(om + 2 * tap + 1);
                float mm = __ldg(om + 18 + tap);
                if (p.mask_is_logit) mm = 1.0f / (1.0f + expf(-mm));
                const float h_im = (float)(oy - 1 + ky) + dy, w_im = (float)(ox - 1 + kx) + dx;
                const int H = p.Hin, W = p.Win;
                w1 = w2 = w3 = w4 = 0.f;
                mk = 0.f;
                o1 = o2 = o3 = o4 = 0;
                if (h_im > -1.f && w_im > -1.f && h_im < (float)H && w_im < (float)W) {
                  const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
                  const int h_high = h_low + 1, w_high = w_low + 1;
                  const float lh = h_im - (float)h_low, lw = w_im - (float)w_low;
                  const float hh = 1.f - lh, hw = 1.f - lw;
                  const bool t_ok = h_low >= 0, b_ok = h_high <= H - 1, l_ok = w_low >= 0, r_ok = w_high <= W - 1;
                  const int hl = t_ok ? h_low : 0, hb = b_ok ? h_high : H - 1;
                  const int wl = l_ok ? w_low : 0, wr = r_ok ? w_high : W - 1;
                  w1 = (t_ok && l_ok) ? hh * hw : 0.f;
                  w2 = (t_ok && r_ok) ? hh * lw : 0.f;
                  w3 = (b_ok && l_ok) ? lh * hw : 0.f;
                  w4 = (b_ok && r_ok) ? lh * lw : 0.f;
                  o1 = hl * W + wl;
                  o2 = hl * W + wr;
                  o3 = hb * W + wl;
                  o4 = hb * W + wr;
                  mk = mm;
                }
              }
              live[qi] = true;
              const int ss = p.srcStride[0];
              const float* base = p.src[0] + (size_t)n * p.Hin * p.Win * ss + c;
#pragma unroll
              for (int h4 = 0; h4 < F4; ++h4) {
                ld[qi][0 * F4 + h4] = __ldg(reinterpret_cast<const float4*>(base + (size_t)o1 * ss) + h4);
                ld[qi][1 * F4 + h4] = __ldg(reinterpret_cast<const float4*>(base + (size_t)o2 * ss) + h4);
                ld[qi][2 * F4 + h4] = __ldg(reinterpret_cast<const float4*>(base + (size_t)o3 * ss) + h4);
                ld[qi][3 * F4 + h4] = __ldg(reinterpret_cast<const float4*>(base + (size_t)o4 * ss) + h4);
              }
            } else {
              const int ky = tap / p.kw, kx = tap - ky * p.kw;
              const int iy = DECONV ? oy + deconv_dy(py, ky) : oy * p.stride - p.pad + ky;
              const int ix = DECONV ? ox + deconv_dy(px, kx) : ox * p.stride - p.pad + kx;
              if (iy >= 0 && iy < p.Hin && ix >= 0 && ix < p.Win) {
                int s = 0, cb = 0;
                while (s + 1 < p.nsrc && c >= cb + p.srcC[s]) {
                  cb += p.srcC[s];
                  ++s;
                }
                const float* sp = p.src[s] + ((size_t)(n * p.Hin + iy) * p.Win + ix) * p.srcStride[s] + (c - cb);
#pragma unroll
                for (int h4 = 0; h4 < F4; ++h4) ld[qi][h4] = __ldg(reinterpret_cast<const float4*>(sp) + h4);
              }
            }
          }
        }
        // ---- ... then wait for the stage, convert and store into the swizzled K-major tile
        ring.wait_empty();
        if (tid == 0) {
          ring.arrive_full_tx(b_tile_bytes);
          bulk_g2s(tiles0 + (uint32_t)ring.stage * stage_bytes + A_TILE_BYTES, wsrc + (size_t)kb * b_tile_bytes, b_tile_bytes,
                   ring.full_bar());
        }
        const uint32_t a_dst = tiles0 + (uint32_t)ring.stage * stage_bytes + row_off;
#pragma unroll
        for (int qi = 0; qi < 4; ++qi) {
          float v[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = 0.f;
          if (MODE == IGEMM_DCN) {
            if (live[qi]) {
#pragma unroll
              for (int h4 = 0; h4 < F4; ++h4) {
                const float4 c1 = ld[qi][0 * F4 + h4], c2 = ld[qi][1 * F4 + h4], c3 = ld[qi][2 * F4 + h4],
                             c4 = ld[qi][3 * F4 + h4];
                // w1..w4 / mk belong to the tap of the LAST chunk decoded above: the chunks of one thread share a
                // tap because umma_supported requires Cin to be a multiple of the thread's 4-chunk span
                v[h4 * 4 + 0] = (w1 * c1.x + w2 * c2.x + w3 * c3.x + w4 * c4.x) * mk;
                v[h4 * 4 + 1] = (w1 * c1.y + w2 * c2.y + w3 * c3.y + w4 * c4.y) * mk;
                v[h4 * 4 + 2] = (w1 * c1.z + w2 * c2.z + w3 * c3.z + w4 * c4.z) * mk;
                v[h4 * 4 + 3] = (w1 * c1.w + w2 * c2.w + w3 * c3.w + w4 * c4.w) * mk;
              }
            }
          } else {
#pragma unroll
            for (int h4 = 0; h4 < F4; ++h4) {
              v[h4 * 4 + 0] = ld[qi][h4].x;
              v[h4 * 4 + 1] = ld[qi][h4].y;
              v[h4 * 4 + 2] = ld[qi][h4].z;
              v[h4 * 4 + 3] = ld[qi][h4].w;
            }
          }
          const uint32_t coff = ((uint32_t)(qbase + qi) ^ sw) << 4;
          if (PREC == 0)
            st_shared_v4(a_dst + coff, pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]),
                         pack_bf16x2(v[6], v[7]));
          else
            st_shared_v4f(a_dst + coff, v[0], v[1], v[2], v[3]);
        }
        fence_proxy_async_smem();
        ring.arrive_full();
        ring.advance();
      }
    }

  } else {
    // =========================== consumers: warpgroup c multiplies rows [64 c, 64 c + 64) of the tile ============
    const int c = (warp - UM_PROD_WARPS) >> 2, wt = tid & 127;
    constexpr bool X3 = PREC == 1;
    float acc[BN / 2];
    float sums[X3 ? BN / 2 : 1];
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
#pragma unroll
    for (int j = 0; j < (X3 ? BN / 2 : 1); ++j) sums[j] = 0.f;
    int gk = 0;                              // tf32x3: K block inside its accumulation group
    for (int kb = 0; kb < KB; ++kb) {
      ring.wait_full();
      const uint32_t a_tile = tiles0 + (uint32_t)ring.stage * stage_bytes + (uint32_t)c * 64u * ROW_BYTES;
      const uint64_t db = make_desc(tiles0 + (uint32_t)ring.stage * stage_bytes + A_TILE_BYTES, 32);
      // tf32x3: NACC K blocks are chained in the accumulator, then added into round-to-nearest fp32 sums
      if (X3)
        mma_kblock_x3<BN, 4>(acc, a_tile, wt, db, ((uint32_t)BN * ROW_BYTES) >> 4, gk == 0);
      else
        mma_kblock<BN, false, true, 4>(acc, make_desc(a_tile, 32), db, 0, 0, kb == 0);
      if (wt == 0) ring.arrive_empty();
      ring.advance();
      if (X3) {
        if (gk == NACC - 1 || kb == KB - 1) {
#pragma unroll
          for (int j = 0; j < (X3 ? BN / 2 : 1); ++j) sums[j] += acc[X3 ? j : 0];
          gk = 0;
        } else {
          ++gk;
        }
      }
    }
    const float* bias = MULTI ? p.bias + (size_t)model * p.wstride : p.bias;
    EpiParams ep = epi_params(p, false);
    ep.bias = bias;
    const int col_end = min(p.Cout, (n_tile + 1) * BN);
    float* dstage = reinterpret_cast<float*>(smem + (tiles0 - smem_u32(smem)) + (size_t)STAGES * stage_bytes) +
                    (size_t)c * (DRAIN_STAGE_BYTES / 4);
    auto fn = [&](int r, int cb, float (&v)[16]) {
      int m = m0 + c * 64 + r;
      const bool valid = m < M;
      int ox = 0, oy = 0, n = 0;
      if (valid) {
        ox = m % Wg;
        const int t = m / Wg;
        oy = t % Hg;
        n = t / Hg;
        if (DECONV) {      // input pixel (n, y, x) of phase (py, px) -> output pixel (n, 2y + py, 2x + px)
          oy = 2 * oy + py;
          ox = 2 * ox + px;
          m = (n * p.Hout + oy) * p.Wout + ox;
        }
      }
      if (cb < BN) epilogue_row<16>(ep, v, valid, m, n, oy, ox, n_tile * BN + cb, col_end);
    };
    if constexpr (X3)
      drain_rows<BN>(sums, dstage, wt, 1 + c, fn);
    else
      drain_rows<BN>(acc, dstage, wt, 1 + c, fn);
  }
}

// ------------------------------------------------------------------ weight tiling
// src: fp32 [Ksrc][ld] (k-major rows, BN-folded, the matrix the fp32 kernel consumes);
// dst: for n_tile, for kb: [hi tile | lo tile] (tf32x3) or one bf16 tile, BN rows x 128 bytes in the SWIZZLE_128B
// K-major image.
template <int PREC>
__global__ void pack_umma_weight_kernel(const float* __restrict__ src, int ld, int K, int Cout, int BN, int n_tiles,
                                        int KB, unsigned char* __restrict__ dst) {
  using T = PrecTraits<PREC>;
  const size_t total = (size_t)n_tiles * KB * BN * 8;   // one thread per 16-byte chunk
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = i & 7;
    size_t t = i >> 3;
    const int nr = t % BN;
    t /= BN;
    const int kb = t % KB;
    const int nt = t / KB;
    const int n = nt * BN + nr;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = kb * T::kElems + q * T::kChunkCh + j;
      v[j] = (j < T::kChunkCh && k < K && n < Cout) ? src[(size_t)k * ld + n] : 0.f;
    }
    const size_t tile = ((size_t)nt * KB + kb) * (size_t)BN * ROW_BYTES * T::kTilesB;
    const size_t off = (size_t)(nr >> 3) * 1024 + (size_t)(nr & 7) * 128 + (size_t)((q ^ (nr & 7)) << 4);
    if (PREC == 0) {
      uint4 w;
      w.x = pack_bf16x2(v[0], v[1]);
      w.y = pack_bf16x2(v[2], v[3]);
      w.z = pack_bf16x2(v[4], v[5]);
      w.w = pack_bf16x2(v[6], v[7]);
      *reinterpret_cast<uint4*>(dst + tile + off) = w;
    } else {
      float h[4], l[4];
      for (int j = 0; j < 4; ++j) {
        h[j] = tf32_round(v[j]);
        l[j] = tf32_round(v[j] - h[j]);
      }
      *reinterpret_cast<float4*>(dst + tile + off) = make_float4(h[0], h[1], h[2], h[3]);
      *reinterpret_cast<float4*>(dst + tile + (size_t)BN * ROW_BYTES + off) = make_float4(l[0], l[1], l[2], l[3]);
    }
  }
}

}  // namespace

// ---- host side -----------------------------------------------------------------------------------------------
// The N tile is the wgmma N of one consumer warpgroup; its accumulator takes BN / 2 registers per thread (tf32x3: twice
// that with the promoted sums) out of the 128 a thread of this 512-thread kernel has.
int umma_tile_n(int CoutPad, int prec) { return wgmma_tile_n(CoutPad, prec == 1 ? 64 : 128); }

bool umma_supported(const IgemmParams& p, int prec) {
  if (p.mode != IGEMM_NHWC_VEC && p.mode != IGEMM_DCN && p.mode != IGEMM_DECONV) return false;
  if (p.mode == IGEMM_DECONV &&
      (p.kh != 2 || p.kw != 2 || p.nsrc != 1 || p.out_nchw || p.Hout != 2 * p.Hin || p.Wout != 2 * p.Win))
    return false;
  const int ch = prec == 0 ? 8 : 4;
  if (p.Cin % ch) return false;
  // DCN: a gather thread blends its four chunks with the sampling weights of one tap, so they must not straddle two
  if (p.mode == IGEMM_DCN && p.Cin % (4 * ch)) return false;
  for (int s = 0; s < p.nsrc; ++s)
    if (p.srcC[s] % ch || p.srcStride[s] % 4) return false;
  return umma_tile_n(p.CoutPad, prec) != 0;
}

size_t umma_weight_bytes(int Kreal, int CoutPad, int prec) {
  const int elems = prec == 0 ? 64 : 32;
  const int KB = (Kreal + elems - 1) / elems;
  const int bn = umma_tile_n(CoutPad, prec);
  return (size_t)(CoutPad / bn) * KB * bn * ROW_BYTES * (prec == 0 ? 1 : 2);
}

int launch_pack_umma_weight(const float* src, int ld, int Kreal, int Cout, int CoutPad, int prec, void* dst,
                            cudaStream_t s) {
  const int elems = prec == 0 ? 64 : 32;
  const int KB = (Kreal + elems - 1) / elems;
  const int bn = umma_tile_n(CoutPad, prec);
  const int nt = CoutPad / bn;
  size_t total = (size_t)nt * KB * bn * 8;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 32) blocks = 132 * 32;
  if (prec == 0)
    pack_umma_weight_kernel<0><<<blocks, 256, 0, s>>>(src, ld, Kreal, Cout, bn, nt, KB, (unsigned char*)dst);
  else
    pack_umma_weight_kernel<1><<<blocks, 256, 0, s>>>(src, ld, Kreal, Cout, bn, nt, KB, (unsigned char*)dst);
  CP_LAUNCH_CHECK("pack_umma_weight_kernel");
  return CP_OK;
}

template <int PREC, int BN, bool MULTI>
static int launch_igemm_umma_bn(const IgemmParams& p, int stages, size_t smem, int nacc, cudaStream_t stream,
                                LaunchInfo* info) {
  const auto kern = (p.mode == IGEMM_DCN)      ? smem_kernel<igemm_umma_kernel<PREC, IGEMM_DCN, BN, MULTI>>()
                    : (p.mode == IGEMM_DECONV) ? smem_kernel<igemm_umma_kernel<PREC, IGEMM_DECONV, BN, MULTI>>()
                                               : smem_kernel<igemm_umma_kernel<PREC, IGEMM_NHWC_VEC, BN, MULTI>>();
  if (int rc = kern.opt_in()) return rc;
  IgemmParams q = p;
  q.ipm = model_ipm(p);
  const bool deconv = p.mode == IGEMM_DECONV;
  const int Mm = q.ipm * (deconv ? p.Hin * p.Win : p.Hout * p.Wout);
  dim3 grid((unsigned)((size_t)(p.CoutPad / BN) * ((Mm + UM_BM - 1) / UM_BM) * (p.B / q.ipm)), deconv ? 4 : 1);
  CP_CUDA_CHECK(launch_kernel(kern.fn, grid, dim3(UM_THREADS), smem, stream, q, stages, nacc));
  CP_LAUNCH_CHECK("igemm_umma_kernel");
  if (info) {
    info->BN = BN;
    info->ksplit = 1;
    info->grid = (long long)grid.x * grid.y;
  }
  return CP_OK;
}

template <bool MULTI>
static int launch_igemm_umma_prec(const IgemmParams& p, int prec, int bn, int stages, size_t smem, int nacc,
                                  cudaStream_t stream, LaunchInfo* info) {
  if (prec == 0) {
    switch (bn) {
      case 16: return launch_igemm_umma_bn<0, 16, MULTI>(p, stages, smem, nacc, stream, info);
      case 32: return launch_igemm_umma_bn<0, 32, MULTI>(p, stages, smem, nacc, stream, info);
      case 64: return launch_igemm_umma_bn<0, 64, MULTI>(p, stages, smem, nacc, stream, info);
      default: return launch_igemm_umma_bn<0, 128, MULTI>(p, stages, smem, nacc, stream, info);
    }
  }
  switch (bn) {
    case 16: return launch_igemm_umma_bn<1, 16, MULTI>(p, stages, smem, nacc, stream, info);
    case 32: return launch_igemm_umma_bn<1, 32, MULTI>(p, stages, smem, nacc, stream, info);
    default: return launch_igemm_umma_bn<1, 64, MULTI>(p, stages, smem, nacc, stream, info);
  }
}

int launch_igemm_umma(const IgemmParams& p, int prec, cudaStream_t stream, LaunchInfo* info) {
  if (!umma_supported(p, prec)) return fail(CP_ERR_INVALID, "igemm_umma: unsupported shape");
  if (!p.wgt_umma) return fail(CP_ERR_INVALID, "igemm_umma: weight tiles missing");
  if (p.B % model_ipm(p)) return fail(CP_ERR_INVALID, "igemm_umma: batch is not a whole number of models");
  const int bn = umma_tile_n(p.CoutPad, prec);
  const size_t stage_bytes = (size_t)A_TILE_BYTES + (size_t)bn * ROW_BYTES * (prec == 0 ? 1 : 2);
  const size_t fixed = 512 + 1024 + 2 * (size_t)DRAIN_STAGE_BYTES;     // control block, alignment, epilogue staging
  int stages = (int)((224 * 1024 - fixed) / stage_bytes);
  if (stages > 6) stages = 6;
  // deformable gather: neighbouring rows / taps sample overlapping 2x2 neighbourhoods (each input pixel is touched by
  // up to 36 samples); a small pipeline leaves most of the shared memory / L1 for those re-reads
  if (p.mode == IGEMM_DCN && stages > 2) stages = 2;
  if (stages < 2) return fail(CP_ERR_INVALID, "igemm_umma: tile does not fit shared memory");
  const size_t smem = fixed + stages * stage_bytes;
  // tf32x3: K blocks (12 MMAs each) chained in the accumulator before they are added into the fp32 sums
  const int nacc = prec == 1 ? kX3GroupBlocks : 1;
  // several models in the launch: the model-indexed instantiations; one model runs the one-model code unchanged
  if (p.B > model_ipm(p)) return launch_igemm_umma_prec<true>(p, prec, bn, stages, smem, nacc, stream, info);
  return launch_igemm_umma_prec<false>(p, prec, bn, stages, smem, nacc, stream, info);
}

}  // namespace cp

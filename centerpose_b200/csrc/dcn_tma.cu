// TMA-staged DCNv2 (modulated deformable 3x3 convolution, stride 1, pad 1, dilation 1, one deformable group)
// on wgmma, tf32 operands.  Reference semantics: dcn_v2_im2col_cuda.cu:125-195 (bilinear sampling with per-corner
// bounds, modulation mask) followed by the GEMM of dcn_v2_cuda.cu:105-160, + folded BatchNorm + ReLU
// (pose_dla_dcn.py:363-379 DeformConv).
//
// Why a second deformable kernel: the gather kernel (igemm_umma.cu) fetches the four bilinear corners of every
// (position, tap, channel chunk) from global memory; each input pixel is re-fetched ~36 times through L1/L2 and the
// producers sit on load latency.  Learned
// offsets are small, so here the rows a tile can reach are STAGED ONCE in shared memory by TMA and the corners are
// gathered from shared memory:
//
//   tile    = an 8 x 16 patch of output positions of one image (128 positions = 128 GEMM rows)
//   slab    = 16 channels x 32 columns x 24 rows around it (halo 8 in x and y, zero-filled outside the image),
//             64 bytes per position in TMA SWIZZLE_64B order (conflict-free 16-byte gathers); double buffered
//   K order = slab-major, tap-minor (the weight tiles of conv_tma.cu with 16-channel slabs are reused unchanged)
//   samples with a corner outside the slab (|offset| > ~7 px) are fetched from global memory instead - slow path,
//   same arithmetic, so the result never depends on how large the offsets are.
//
//   warp 0        : TMA producer for slabs
//   warp 1        : weight-tile producer (cp.async.bulk, pre-swizzled tiles)
//   warps 4-7     : consumer of tile rows [0, 64) (wgmma into registers + epilogue); thread i also writes the sampling
//                   records (one 16-byte record per tap) of position i of the NEXT tile
//   warps 8-11    : gather, one thread per position: 4 corners x 16 channels from the slab -> bilinear blend * mask ->
//                   A tile in the SWIZZLE_64B K-major layout (tf32-rounded; fp32 in x3, where the consumers split it
//                   into hi / lo in registers), AH A stages
//   warps 12-15   : consumer of tile rows [64, 128)
#include <cuda.h>

#include "common.cuh"
#include "umma_common.cuh"

namespace cp {
namespace {

using namespace umma;

constexpr int DT_BM = 128;
constexpr int DT_THREADS = 512;     // 4 control + 4 gather + 8 consumer warps
constexpr int DT_CS = 16;            // channels per slab = one K block of 64-byte rows
constexpr int DT_PH = 8, DT_PW = 16;  // output patch (rows x columns) = 128 positions
constexpr int DT_HALO = 8;           // slab margin around the patch, both directions
constexpr int DT_SH = DT_PH + 2 * DT_HALO, DT_SW = DT_PW + 2 * DT_HALO;     // slab rows x columns (24 x 32)
constexpr uint32_t DT_SLAB_BYTES = DT_SH * DT_SW * DT_CS * 4;               // 49152
constexpr uint32_t DT_COEF_BYTES = DT_BM * 9 * 16;

struct DcnTmaParams {
  CUtensorMap amap;
  const float* src;
  int srcStride;
  const float* offmask;
  int omStride, mask_is_logit;
  int B, H, W, Cin, Cout, CoutPad, BN;
  int tiles_x, tiles_per_image;      // patches per image row / per image
  long long total_tiles;             // m tiles x n tiles (n fastest)
  int SB;
  int group;                         // x3: K blocks (16 channels) per accumulation group
  int AH;                            // A stages (1 or 2)
  const float* bias;
  const float* residual;
  int resStride, relu, res_after_relu;
  float* out;
  int outStride, out_nchw, round_tf32;
  const unsigned char* wtiles;
  // split-K (small maps: fewer tiles than SMs): tile = (m, n) tile * ksplit + split; a split walks `sps` slabs, stores its
  // partial sums to `part` ([mn tile][split][BN / 4][128 rows] float4) and dcn_tma_splitk_finish runs the epilogue
  int ksplit, sps;
  float* part;
  int ipm;                           // models (IgemmParams::ipm): image n takes model n / ipm's bias and weight tiles
  long long wstride, tstride;
};

struct DcnCtl {
  unsigned long long s_full[2], s_empty[2];
  unsigned long long a_full[2], a_empty[2];
  unsigned long long c_full[2], c_empty[2];
  unsigned long long b_full[8], b_empty[8];
};

// record bits: [0,14) slab position of the clamped top-left corner (in-slab) or (row << 7 | col) in the image
// (global path);  14: right corner is +1 column;  15: bottom corner is +1 row;  16-19: corner weights alive;
// 20: all corners inside the slab;  21: sample inside the image
constexpr int RB_DX = 14, RB_DY = 15, RB_W = 16, RB_SLAB = 20, RB_LIVE = 21;

// Sampling records of one output position (all 9 taps) -> shared memory.  dcn_v2_im2col_cuda.cu:160-195: the sample
// (h_im, w_im) is used only when it lies in (-1, H) x (-1, W); every corner carries its own bounds test.
__device__ __forceinline__ void coef_row(const DcnTmaParams& p, const float* __restrict__ om, int oy, int ox, int ys,
                                         int xs, uint32_t dst) {
  float o[27];
#pragma unroll
  for (int j = 0; j < 27; ++j) o[j] = __ldg(om + j);
  const int H = p.H, W = p.W;
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    const int ky = tap / 3, kx = tap - ky * 3;
    float mm = o[18 + tap];
    if (p.mask_is_logit) mm = 1.0f / (1.0f + expf(-mm));
    const float h_im = (float)(oy - 1 + ky) + o[2 * tap], w_im = (float)(ox - 1 + kx) + o[2 * tap + 1];
    float lh = 0.f, lw = 0.f, mk = 0.f;
    uint32_t pk = 0;
    if (h_im > -1.f && w_im > -1.f && h_im < (float)H && w_im < (float)W) {
      const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
      lh = h_im - (float)h_low;
      lw = w_im - (float)w_low;
      const bool t_ok = h_low >= 0, b_ok = h_low + 1 <= H - 1, l_ok = w_low >= 0, r_ok = w_low + 1 <= W - 1;
      const int hl = t_ok ? h_low : 0, hb = b_ok ? h_low + 1 : H - 1;
      const int wl = l_ok ? w_low : 0, wr = r_ok ? w_low + 1 : W - 1;
      const bool in_slab = (hl >= ys) && (hb < ys + DT_SH) && (wl >= xs) && (wr < xs + DT_SW);
      pk = in_slab ? (uint32_t)((hl - ys) * DT_SW + (wl - xs)) : (uint32_t)((hl << 7) | wl);
      pk |= (uint32_t)(wr - wl) << RB_DX;
      pk |= (uint32_t)(hb - hl) << RB_DY;
      pk |= (uint32_t)((t_ok && l_ok) ? 1 : 0) << (RB_W + 0);
      pk |= (uint32_t)((t_ok && r_ok) ? 1 : 0) << (RB_W + 1);
      pk |= (uint32_t)((b_ok && l_ok) ? 1 : 0) << (RB_W + 2);
      pk |= (uint32_t)((b_ok && r_ok) ? 1 : 0) << (RB_W + 3);
      pk |= (uint32_t)(in_slab ? 1 : 0) << RB_SLAB;
      pk |= 1u << RB_LIVE;
      mk = mm;
    }
    st_shared_v4(dst + (uint32_t)tap * 16u, __float_as_uint(lh), __float_as_uint(lw), __float_as_uint(mk), pk);
  }
}

// MULTI: the launch holds several models (DcnTmaParams::ipm); otherwise the code is that of one model.
// FOLD (batch-invariant plans): one CTA per (m, n) tile sums the ksplit K segments of `sps` slabs back to back, each
// exactly as a split-K CTA of that segment does (x3: accumulation groups start at the segment's first K block; tf32:
// the segment's first wgmma starts a fresh accumulator), and adds them in segment order into a running total,
// ((0 + seg 0) + seg 1) + ..., as splitk_finish adds the parked partial sums: the same bits on either path.
template <bool X3, int BN, bool MULTI, bool FOLD>
__global__ void __launch_bounds__(DT_THREADS, 1) dcn_tma_kernel(const __grid_constant__ DcnTmaParams p) {
  extern __shared__ __align__(1024) unsigned char smem[];
  DcnCtl* ctl = reinterpret_cast<DcnCtl*>(smem);
  if (threadIdx.x == 0) griddep_launch_dependents();      // PDL (common.cuh)
  const uint32_t sbase = smem_u32(smem);
  const uint32_t coef0 = sbase + 1024u;
  const uint32_t slabs0 = (coef0 + 2u * DT_COEF_BYTES + 1023u) & ~1023u;
  const uint32_t a_stage = 8192u;                              // A tile of 128 rows x 64 bytes
  const uint32_t atiles0 = slabs0 + 2u * DT_SLAB_BYTES;
  const uint32_t btile_bytes = (uint32_t)BN * 64u * (X3 ? 2u : 1u);
  const uint32_t btiles0 = atiles0 + (uint32_t)p.AH * a_stage;
  const uint32_t drain0 = btiles0 + (uint32_t)p.SB * btile_bytes;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_tiles = p.CoutPad / BN;
  const int nslab = FOLD ? p.sps * p.ksplit : p.sps;  // slabs one tile walks (all of them unless split-K)
  const int KB = nslab * 9;
  const int KB_all = (p.Cin / DT_CS) * 9;
  const int KS_SPLIT = FOLD ? 1 : p.ksplit;
  const long long total_tiles = p.total_tiles;

  if (tid == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(smem_u32(&ctl->s_full[s]), 1);
      mbar_init(smem_u32(&ctl->s_empty[s]), 4);             // one arrival per gather warp
      mbar_init(smem_u32(&ctl->c_full[s]), 4);              // one arrival per record-writing warp (4-7)
      mbar_init(smem_u32(&ctl->c_empty[s]), 4);
    }
    for (int s = 0; s < p.AH; ++s) {
      mbar_init(smem_u32(&ctl->a_full[s]), 4);              // written by the four gather warps
      mbar_init(smem_u32(&ctl->a_empty[s]), 2);             // released by both consumer warpgroups
    }
    for (int s = 0; s < p.SB; ++s) {
      mbar_init(smem_u32(&ctl->b_full[s]), 1);
      mbar_init(smem_u32(&ctl->b_empty[s]), 2);
    }
    fence_mbar_init();
  }
  __syncthreads();
  // PDL: the weight producer (warp 1) reads per-plan constants and runs ahead; every other role waits for the previous
  // launch (the offset / mask convolution whose output the records are built from) before it touches global memory
  if (warp != 1) griddep_wait();

  if (warp < 4) {
    // the control warpgroup hands registers to the consumers (a 64 x BN accumulator + the x3 running sums)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0) {
      // ===================== slabs via TMA =====================
      if (lane == 0) {
        int stage = 0;
        uint32_t phase = 0;
        for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
          const long long m_tile = (tile / KS_SPLIT) / n_tiles;
          const int s0 = (int)(tile % KS_SPLIT) * nslab;
          const int img = (int)(m_tile / p.tiles_per_image);
          const int pt = (int)(m_tile - (long long)img * p.tiles_per_image);
          const int y0 = (pt / p.tiles_x) * DT_PH, x0 = (pt % p.tiles_x) * DT_PW;
          for (int s = 0; s < nslab; ++s) {
            mbar_wait(smem_u32(&ctl->s_empty[stage]), phase ^ 1u);
            const uint32_t bar = smem_u32(&ctl->s_full[stage]);
            mbar_arrive_expect_tx(bar, DT_SLAB_BYTES);
            tma_load_4d(slabs0 + (uint32_t)stage * DT_SLAB_BYTES, &p.amap, (s0 + s) * DT_CS, x0 - DT_HALO, y0 - DT_HALO, img,
                        bar);
            if (++stage == 2) {
              stage = 0;
              phase ^= 1u;
            }
          }
        }
      }
      __syncwarp();
    } else if (warp == 1) {
      // ===================== weight tiles =====================
      if (lane == 0) {
        int stage = 0;
        uint32_t phase = 0;
        for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
          const int n_tile = (int)((tile / KS_SPLIT) % n_tiles);
          const int model = MULTI ? (int)((tile / KS_SPLIT) / n_tiles / p.tiles_per_image) / p.ipm : 0;
          const unsigned char* wsrc = p.wtiles + (size_t)model * p.tstride +
                                      ((size_t)n_tile * KB_all + (size_t)(tile % KS_SPLIT) * KB) * btile_bytes;
          for (int kb = 0; kb < KB; ++kb) {
            mbar_wait(smem_u32(&ctl->b_empty[stage]), phase ^ 1u);
            const uint32_t bar = smem_u32(&ctl->b_full[stage]);
            mbar_arrive_expect_tx(bar, btile_bytes);
            bulk_g2s(btiles0 + (uint32_t)stage * btile_bytes, wsrc + (size_t)kb * btile_bytes, btile_bytes, bar);
            if (++stage == p.SB) {
              stage = 0;
              phase ^= 1u;
            }
          }
        }
      }
      __syncwarp();
    }
  } else if (warp >= 8 && warp < 12) {
    // 128 x 40 + 128 x 120 + 256 x 176 = 64 K registers: the consumers also hold the hi / lo A fragments of a K block
    asm volatile("setmaxnreg.dec.sync.aligned.u32 120;");
    // ===================== gather: thread = one position of the tile; the record of a (position, tap) is decoded once
    // for all 16 channels and a stage is synchronised once per K block =====================
    const int gt = tid - 256;
    const int row = gt & 127;
    const uint32_t a_row = atiles0 + (uint32_t)(row >> 3) * 512u + (uint32_t)(row & 7) * 64u;
    const uint32_t asw = (uint32_t)(row >> 1) & 3u;
    int ss = 0, cb = 0;
    uint32_t ps = 0, pc = 0;
    uint32_t cnt = 0;                      // K blocks produced; stage = cnt % AH
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const long long m_tile = (tile / KS_SPLIT) / n_tiles;
      const int s0 = (int)(tile % KS_SPLIT) * nslab;
      const int img = (int)(m_tile / p.tiles_per_image);
      mbar_wait(smem_u32(&ctl->c_full[cb]), pc);
      const uint32_t crow = coef0 + (uint32_t)cb * DT_COEF_BYTES + (uint32_t)row * 144u;
      const float* gimg = p.src + (size_t)img * p.H * p.W * p.srcStride;
      int cur = -1;
      uint32_t slab = 0;
      float4 rec_next = ld_shared_v4f(crow);      // tap 0: the first K block
      for (int kb = 0; kb < KB; ++kb) {
        const int s = kb / 9;
        if (s != cur) {
          if (cur >= 0) {                     // done with the previous slab
            __syncwarp();
            if (lane == 0) mbar_arrive(smem_u32(&ctl->s_empty[ss]));
            if (++ss == 2) {
              ss = 0;
              ps ^= 1u;
            }
          }
          mbar_wait(smem_u32(&ctl->s_full[ss]), ps);
          slab = slabs0 + (uint32_t)ss * DT_SLAB_BYTES;
          cur = s;
        }
        const float4 rec = rec_next;
        {                                   // the record of the next K block: its latency hides behind this gather
          const int kn = kb + 1;
          const int tn = kn - (kn / 9) * 9;
          rec_next = ld_shared_v4f(crow + (uint32_t)(kn < KB ? tn : 0) * 16u);
        }
        const uint32_t pk = __float_as_uint(rec.w);
        float4 v[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) v[c] = make_float4(0.f, 0.f, 0.f, 0.f);
        if ((pk >> RB_LIVE) & 1u) {
          const float lh = rec.x, lw = rec.y, mk = rec.z;
          const float hh = 1.f - lh, hw = 1.f - lw;
          const float w1 = ((pk >> (RB_W + 0)) & 1u) ? hh * hw * mk : 0.f;
          const float w2 = ((pk >> (RB_W + 1)) & 1u) ? hh * lw * mk : 0.f;
          const float w3 = ((pk >> (RB_W + 2)) & 1u) ? lh * hw * mk : 0.f;
          const float w4 = ((pk >> (RB_W + 3)) & 1u) ? lh * lw * mk : 0.f;
          if ((pk >> RB_SLAB) & 1u) {
            // slab rows are 64 bytes in TMA SWIZZLE_64B order: 16-byte chunk c of position q sits at c ^ ((q >> 1) & 3)
            const uint32_t q1 = pk & 0x3FFFu, q2 = q1 + ((pk >> RB_DX) & 1u);
            const uint32_t q3 = q1 + ((pk >> RB_DY) & 1u) * (uint32_t)DT_SW, q4 = q3 + ((pk >> RB_DX) & 1u);
            // chunk c of position q: slab + 64 q + ((c ^ s) << 4) == (slab + 64 q + (s << 4)) ^ (c << 4)  (64-byte aligned rows)
            const uint32_t b1 = slab + q1 * 64u + ((q1 << 3) & 0x30u), b2 = slab + q2 * 64u + ((q2 << 3) & 0x30u);
            const uint32_t b3 = slab + q3 * 64u + ((q3 << 3) & 0x30u), b4 = slab + q4 * 64u + ((q4 << 3) & 0x30u);
            // all sixteen 16-byte loads are issued before the first blend (ld_shared_v4f is volatile: source order is kept),
            // so their latencies overlap instead of being paid one after the other by this warp
            float4 c1[4], c2[4], c3[4], c4[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              c1[c] = ld_shared_v4f(b1 ^ ((uint32_t)c << 4));
              c2[c] = ld_shared_v4f(b2 ^ ((uint32_t)c << 4));
            }
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              c3[c] = ld_shared_v4f(b3 ^ ((uint32_t)c << 4));
              c4[c] = ld_shared_v4f(b4 ^ ((uint32_t)c << 4));
            }
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              v[c].x = w1 * c1[c].x + w2 * c2[c].x + w3 * c3[c].x + w4 * c4[c].x;
              v[c].y = w1 * c1[c].y + w2 * c2[c].y + w3 * c3[c].y + w4 * c4[c].y;
              v[c].z = w1 * c1[c].z + w2 * c2[c].z + w3 * c3[c].z + w4 * c4[c].z;
              v[c].w = w1 * c1[c].w + w2 * c2[c].w + w3 * c3[c].w + w4 * c4[c].w;
            }
          } else {      // corner rows outside the staged slab: same arithmetic from global memory
            const int hl = (int)((pk >> 7) & 127u), wl = (int)(pk & 127u);
            const float* g = gimg + ((size_t)hl * p.W + wl) * p.srcStride + (s0 + s) * DT_CS;
            const size_t dx = (size_t)((pk >> RB_DX) & 1u) * p.srcStride;
            const size_t dy = (size_t)((pk >> RB_DY) & 1u) * p.W * p.srcStride;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const float4 c1 = __ldg(reinterpret_cast<const float4*>(g) + c);
              const float4 c2 = __ldg(reinterpret_cast<const float4*>(g + dx) + c);
              const float4 c3 = __ldg(reinterpret_cast<const float4*>(g + dy) + c);
              const float4 c4 = __ldg(reinterpret_cast<const float4*>(g + dy + dx) + c);
              v[c].x = w1 * c1.x + w2 * c2.x + w3 * c3.x + w4 * c4.x;
              v[c].y = w1 * c1.y + w2 * c2.y + w3 * c3.y + w4 * c4.y;
              v[c].z = w1 * c1.z + w2 * c2.z + w3 * c3.z + w4 * c4.z;
              v[c].w = w1 * c1.w + w2 * c2.w + w3 * c3.w + w4 * c4.w;
            }
          }
        }
        const int sa = (int)(cnt & (uint32_t)(p.AH - 1));          // barrier index == tile slot
        const uint32_t a_dst = a_row + (uint32_t)sa * a_stage + (asw << 4);      // chunk c -> a_dst ^ (c << 4)
        mbar_wait(smem_u32(&ctl->a_empty[sa]), ((cnt >> (p.AH - 1)) & 1u) ^ 1u);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const uint32_t off = (uint32_t)c << 4;
          if (X3)
            st_shared_v4f(a_dst ^ off, v[c].x, v[c].y, v[c].z, v[c].w);
          else
            st_shared_v4f(a_dst ^ off, tf32_round(v[c].x), tf32_round(v[c].y), tf32_round(v[c].z), tf32_round(v[c].w));
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&ctl->a_full[sa]));
        ++cnt;
      }
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(smem_u32(&ctl->s_empty[ss]));       // last slab of the tile
        mbar_arrive(smem_u32(&ctl->c_empty[cb]));
      }
      if (++ss == 2) {
        ss = 0;
        ps ^= 1u;
      }
      if (++cb == 2) {
        cb = 0;
        pc ^= 1u;
      }
    }
  } else {
    // ===================== consumers: warpgroup c multiplies rows [64 c, 64 c + 64) of every tile =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 176;");
    const int c = warp >= 12 ? 1 : 0, wt = tid & 127;
    float* dstage = reinterpret_cast<float*>(smem + (drain0 - sbase)) + (size_t)c * (DRAIN_STAGE_BYTES / 4);
    EpiParams ep;
    ep.bias = p.bias;
    ep.residual = p.residual;
    ep.resStride = p.resStride;
    ep.relu = p.relu;
    ep.res_after_relu = p.res_after_relu;
    ep.round_tf32 = p.round_tf32;
    ep.out = p.out;
    ep.outStride = p.outStride;
    ep.out_nchw = p.out_nchw;
    ep.Cout = p.Cout;
    ep.CoutPad = p.CoutPad;
    ep.H = p.H;
    ep.W = p.W;
    // Warpgroup 0 is idle while the gather runs, and its thread i == position i: it also prepares the sampling records
    // of the NEXT tile (double-buffered), so the gather warps never wait for them.
    int cb = 0;
    uint32_t pc = 0;
    auto make_records = [&](long long t) {
      const long long mt = (t / KS_SPLIT) / n_tiles;
      const int im = (int)(mt / p.tiles_per_image);
      const int pt = (int)(mt - (long long)im * p.tiles_per_image);
      const int y0 = (pt / p.tiles_x) * DT_PH, x0 = (pt % p.tiles_x) * DT_PW;
      const int oy = y0 + (wt >> 4), ox = x0 + (wt & 15);
      mbar_wait(smem_u32(&ctl->c_empty[cb]), pc ^ 1u);
      coef_row(p, p.offmask + ((size_t)((size_t)im * p.H + oy) * p.W + ox) * p.omStride, oy, ox, y0 - DT_HALO, x0 - DT_HALO,
               coef0 + (uint32_t)cb * DT_COEF_BYTES + (uint32_t)wt * 144u);
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&ctl->c_full[cb]));
      if (++cb == 2) {
        cb = 0;
        pc ^= 1u;
      }
    };
    if (c == 0 && (long long)blockIdx.x < total_tiles) make_records(blockIdx.x);
    const uint32_t bar_a_full = smem_u32(&ctl->a_full[0]), bar_a_empty = smem_u32(&ctl->a_empty[0]);
    const uint32_t bar_b_full = smem_u32(&ctl->b_full[0]), bar_b_empty = smem_u32(&ctl->b_empty[0]);
    int sb = 0;
    uint32_t pb = 0, cnt = 0;
    float acc[BN / 2];
    float sums[X3 ? BN / 2 : 1];
    float tot[FOLD ? BN / 2 : 1];      // fold: the running total of the finished K segments
    const int KB_seg = FOLD ? p.sps * 9 : KB;
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      if (c == 0 && tile + gridDim.x < total_tiles) make_records(tile + gridDim.x);
#pragma unroll
      for (int j = 0; j < (X3 ? BN / 2 : 1); ++j) sums[j] = 0.f;
      if constexpr (FOLD) {
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) tot[j] = 0.f;
      }
      int gk = 0;
      int kseg = 0;                    // fold: K blocks done in the current segment
      for (int kbi = 0; kbi < KB; ++kbi, ++cnt) {
        const bool seg_end = FOLD ? kseg == KB_seg - 1 : kbi == KB - 1;
        const uint32_t sa = cnt & (uint32_t)(p.AH - 1);
        mbar_wait(bar_a_full + 8u * sa, (cnt >> (p.AH - 1)) & 1u);
        mbar_wait(bar_b_full + 8u * (uint32_t)sb, pb);
        const uint32_t a_tile = atiles0 + sa * a_stage + (uint32_t)c * 64u * 64u;
        const uint64_t db = make_desc(btiles0 + (uint32_t)sb * btile_bytes, DT_CS);
        if (X3)
          mma_kblock_x3<BN, 2>(acc, a_tile, wt, db, ((uint32_t)BN * 64u) >> 4, gk == 0);
        else
          mma_kblock<BN, false, false, 2>(acc, make_desc(a_tile, DT_CS), db, 0, 0, FOLD ? kseg == 0 : kbi == 0);
        if (wt == 0) {
          mbar_arrive(bar_a_empty + 8u * sa);
          mbar_arrive(bar_b_empty + 8u * (uint32_t)sb);
        }
        if (++sb == p.SB) {
          sb = 0;
          pb ^= 1u;
        }
        if (X3) {
          // two-level accumulation (see conv_tma.cu): every finished group is added, with round-to-nearest, into sums
          if (gk == p.group - 1 || seg_end) {
#pragma unroll
            for (int j = 0; j < (X3 ? BN / 2 : 1); ++j) sums[j] += acc[X3 ? j : 0];
            gk = 0;
          } else {
            ++gk;
          }
        }
        if constexpr (FOLD) {
          // the segment is done: add it to the total; the next one starts from zero, as its split-K CTA would
          if (seg_end) {
#pragma unroll
            for (int j = 0; j < BN / 2; ++j) {
              if (X3) {
                tot[j] += sums[X3 ? j : 0];
                sums[X3 ? j : 0] = 0.f;
              } else {
                tot[j] += acc[j];
              }
            }
          }
          kseg = seg_end ? 0 : kseg + 1;
        }
      }
      const int n_tile = (int)((tile / KS_SPLIT) % n_tiles);
      const long long m_tile = (tile / KS_SPLIT) / n_tiles;
      const int n = (int)(m_tile / p.tiles_per_image);
      const int pt = (int)(m_tile - (long long)n * p.tiles_per_image);
      const int col_end = min(p.Cout, (n_tile + 1) * BN);
      if (MULTI) ep.bias = p.bias + (size_t)(n / p.ipm) * p.wstride;
      auto fn = [&](int r, int cb0, float (&v)[16]) {
        if (cb0 >= BN) return;
        const int i = c * 64 + r;
        if (KS_SPLIT > 1) {
          // split-K: the finished columns of this position go to the workspace instead of through the epilogue
          float4* part_row = reinterpret_cast<float4*>(p.part) + ((size_t)tile * (BN >> 2) + (cb0 >> 2)) * 128 + i;
#pragma unroll
          for (int q = 0; q < 4; ++q) __stcg(part_row + (size_t)q * 128, make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]));
        } else {
          const int oy = (pt / p.tiles_x) * DT_PH + (i >> 4), ox = (pt % p.tiles_x) * DT_PW + (i & 15);
          const int m = (n * p.H + oy) * p.W + ox;
          epilogue_row<16>(ep, v, true, m, n, oy, ox, n_tile * BN + cb0, col_end);
        }
      };
      if constexpr (FOLD)
        drain_rows<BN>(tot, dstage, wt, 1 + c, fn);
      else if constexpr (X3)
        drain_rows<BN>(sums, dstage, wt, 1 + c, fn);
      else
        drain_rows<BN>(acc, dstage, wt, 1 + c, fn);
    }
  }
}

// split-K, second half (splitk_finish, umma_common.cuh): tile row i -> position i of the 8 x 16 patch
template <bool MULTI>
__global__ void __launch_bounds__(256) dcn_tma_splitk_finish(const __grid_constant__ DcnTmaParams p, long long mn_tiles) {
  splitk_finish<MULTI>(p, DT_BM, mn_tiles, [&](long long mn, int i, int* n, int* oy, int* ox) {
    const long long m_tile = mn / (p.CoutPad / p.BN);
    *n = (int)(m_tile / p.tiles_per_image);
    const int pt = (int)(m_tile - (long long)*n * p.tiles_per_image);
    *oy = (pt / p.tiles_x) * DT_PH + (i >> 4);
    *ox = (pt % p.tiles_x) * DT_PW + (i & 15);
    return true;
  });
}

}  // namespace

// wgmma N of the consumer warpgroups (x3: the accumulator and the running sums, BN / 2 registers each)
int dcn_tma_tile_n(int CoutPad, int) { return wgmma_tile_n(CoutPad, 128); }

bool dcn_tma_supported(const IgemmParams& p, int x3) {
  if (p.mode != IGEMM_DCN || p.nsrc != 1) return false;
  if (p.kh != 3 || p.kw != 3 || p.stride != 1 || p.pad != 1) return false;
  if (p.Cin % DT_CS || p.srcStride[0] % 4) return false;
  const int W = p.Win, H = p.Hin;
  if (W > 128 || H > 128 || (W % DT_PW) || (H % DT_PH)) return false;     // records pack image coordinates in 7 bits
  return dcn_tma_tile_n(p.CoutPad, x3) != 0;
}

long long dcn_tma_image_tiles(const IgemmParams& p, int BN) {
  return (long long)(p.Win / DT_PW) * (p.Hin / DT_PH) * (p.CoutPad / BN);
}

int dcn_tma_encode(const IgemmParams& p, int Bmax, void* map_out) {
  return tma_encode_nhwc_box(p.src[0], p.srcC[0], p.Win, p.Hin, Bmax, p.srcStride[0], DT_CS, DT_SW, DT_SH, 1, map_out);
}

// The instance of one launch (null: no such N tile).  FOLD: the K segments folded in one CTA per tile.
using DcnTmaKernel = void (*)(DcnTmaParams);
template <bool FOLD>
static DcnTmaKernel dcn_tma_kernel_for(int BN, bool x3, bool multi) {
  switch (BN) {
    case 16: return multi ? (x3 ? dcn_tma_kernel<true, 16, true, FOLD> : dcn_tma_kernel<false, 16, true, FOLD>)
                          : (x3 ? dcn_tma_kernel<true, 16, false, FOLD> : dcn_tma_kernel<false, 16, false, FOLD>);
    case 32: return multi ? (x3 ? dcn_tma_kernel<true, 32, true, FOLD> : dcn_tma_kernel<false, 32, true, FOLD>)
                          : (x3 ? dcn_tma_kernel<true, 32, false, FOLD> : dcn_tma_kernel<false, 32, false, FOLD>);
    case 64: return multi ? (x3 ? dcn_tma_kernel<true, 64, true, FOLD> : dcn_tma_kernel<false, 64, true, FOLD>)
                          : (x3 ? dcn_tma_kernel<true, 64, false, FOLD> : dcn_tma_kernel<false, 64, false, FOLD>);
    case 128: return multi ? (x3 ? dcn_tma_kernel<true, 128, true, FOLD> : dcn_tma_kernel<false, 128, true, FOLD>)
                           : (x3 ? dcn_tma_kernel<true, 128, false, FOLD> : dcn_tma_kernel<false, 128, false, FOLD>);
    default: return nullptr;
  }
}

int launch_dcn_tma(const IgemmParams& p, const void* map, const ConvKernel& k, cudaStream_t stream, LaunchInfo* info) {
  const bool x3 = k.x3;
  if (!p.wgt_umma) return fail(CP_ERR_INVALID, "dcn_tma: weight tiles missing");
  if (!dcn_tma_supported(p, x3)) return fail(CP_ERR_INVALID, "dcn_tma: unsupported shape");
  DcnTmaParams q;
  memset(&q, 0, sizeof(q));
  memcpy(&q.amap, map, sizeof(CUtensorMap));
  q.src = p.src[0];
  q.srcStride = p.srcStride[0];
  q.offmask = p.offmask;
  q.omStride = p.omStride;
  q.mask_is_logit = p.mask_is_logit;
  q.B = p.B;
  q.H = p.Hin;
  q.W = p.Win;
  q.Cin = p.Cin;
  q.Cout = p.Cout;
  q.CoutPad = p.CoutPad;
  q.BN = k.BN;
  q.tiles_x = p.Win / DT_PW;
  q.tiles_per_image = q.tiles_x * (p.Hin / DT_PH);
  const long long mn = (long long)q.tiles_per_image * p.B * (p.CoutPad / q.BN);
  const uint32_t a_stage = 8192u;
  q.group = kX3GroupBlocks * 2;      // 16-channel K blocks: same MMA count per group as conv_tma.cu
  const uint32_t btile = (uint32_t)q.BN * 64u * (x3 ? 2u : 1u);
  const size_t budget = 226 * 1024;
  // two A stages where >= 3 weight stages still fit, else one
  q.AH = 2;
  size_t fixed = 1024 + 2 * (size_t)DT_COEF_BYTES + 1024 + 2 * (size_t)DT_SLAB_BYTES + (size_t)q.AH * a_stage +
                 2 * (size_t)DRAIN_STAGE_BYTES;
  if (fixed + 3 * (size_t)btile > budget) {
    q.AH = 1;
    fixed -= a_stage;
  }
  if (fixed + 2 * (size_t)btile > budget) return fail(CP_ERR_INVALID, "dcn_tma: tile does not fit shared memory");
  q.SB = (int)((budget - fixed) / btile);
  if (q.SB > 8) q.SB = 8;
  q.bias = p.bias;
  q.residual = p.residual;
  q.resStride = p.resStride;
  q.relu = p.relu;
  q.res_after_relu = p.res_after_relu;
  q.out = p.out;
  q.outStride = p.outStride;
  q.out_nchw = p.out_nchw;
  q.round_tf32 = k.round_out;
  q.wtiles = (const unsigned char*)p.wgt_umma;
  q.ipm = model_ipm(p);
  q.wstride = p.wstride;
  q.tstride = p.tstride;
  const bool multi = p.B > q.ipm;      // several models: the model-indexed instantiations
  const size_t smem = fixed + (size_t)q.SB * btile;
  int num_sms = 0;
  if (int rc = device_sm_count(&num_sms)) return rc;
  // split-K: at batch 1 the 512 -> 256 DCN at 16 x 16 is 4 tiles of 288 K blocks; deal slab ranges to idle SMs.
  // Batch-invariant plans fix the segments by the layer's shape (k.ksegments) and split them only when their partial sums
  // fit the workspace; otherwise one CTA per tile folds them (the FOLD instances of dcn_tma_kernel), with the same bits.
  const int nslab = p.Cin / DT_CS;
  const size_t tile_floats = (size_t)DT_BM * q.BN;
  bool fold = false;
  q.part = p.splitk_ws;
  if (k.ksegments > 0) {
    if (nslab % k.ksegments) return fail(CP_ERR_INVALID, "dcn_tma: K segments do not fit the launch");
    q.ksplit = k.ksegments;
    fold = q.ksplit > 1 && (size_t)mn * q.ksplit * tile_floats > p.splitk_ws_floats;
  } else {
    q.ksplit = splitk_factor(mn, nslab, num_sms, tile_floats, p.splitk_ws_floats);
  }
  q.sps = nslab / q.ksplit;
  q.total_tiles = fold ? mn : mn * q.ksplit;
  const DcnTmaKernel kern = fold ? dcn_tma_kernel_for<true>(q.BN, x3, multi) : dcn_tma_kernel_for<false>(q.BN, x3, multi);
  if (!kern) return fail(CP_ERR_INVALID, "dcn_tma: unsupported N tile");
  static PerDevice<bool, 32> configured;
  const int slot = (fold ? 16 : 0) + (multi ? 8 : 0) + (x3 ? 4 : 0) + (q.BN == 128 ? 3 : (q.BN == 64 ? 2 : (q.BN == 32 ? 1 : 0)));
  if (!configured.here(slot)) {
    CP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    configured.here(slot) = true;
  }
  const unsigned grid = (unsigned)(q.total_tiles < num_sms ? q.total_tiles : num_sms);
  CP_CUDA_CHECK(launch_kernel(kern, dim3(grid), dim3(DT_THREADS), smem, stream, q));
  CP_LAUNCH_CHECK("dcn_tma_kernel");
  if (info) {
    info->BN = q.BN;
    info->ksplit = q.ksplit;
    info->grid = grid;
    info->path = q.ksplit == 1 ? CP_KPATH_ONE : (fold ? CP_KPATH_FOLD : CP_KPATH_SPLIT);
  }
  if (q.ksplit > 1 && !fold) {
    const long long threads = mn * (q.BN / 4) * DT_BM;
    CP_CUDA_CHECK(launch_kernel(multi ? dcn_tma_splitk_finish<true> : dcn_tma_splitk_finish<false>, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, stream, q, mn));
    CP_LAUNCH_CHECK("dcn_tma_splitk_finish");
  }
  return CP_OK;
}

}  // namespace cp

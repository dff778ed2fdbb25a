// TMA-fed wgmma convolution ("shifted-window" implicit GEMM) for stride-1 1x1 / 3x3 convolutions
// over NHWC fp32 activations, tf32 operands.
//
// Idea: pad the image by one pixel and flatten it to a 1-D sequence of positions with pitch Wt = W + 2.
// A 3x3 tap (ky, kx) is then a CONSTANT offset (ky-1)*Wt + (kx-1) in that sequence, so the A operand of
// tap (ky,kx) for 128 consecutive output positions is simply the same shared-memory slab read from a
// different start row.  One TMA tiled load (box = 32 channels x Wt columns x BOXH rows, out-of-bounds
// elements zero-filled = the convolution padding) brings a [positions][32 ch] slab of 128-byte rows in
// SWIZZLE_128B layout; nine wgmma descriptors with different start addresses contract it against nine
// weight tiles.  Outputs computed at the two pad columns of every row are discarded (W/Wt efficiency).
// The im2col matrix never exists anywhere and no thread touches activation data before the epilogue.
//
//   warp 0 : TMA producer for activation slabs            (ring of SA stages)
//   warp 1 : weight-tile producer, cp.async.bulk          (ring of SB stages, tiles pre-swizzled at load time)
//   warpgroups 1, 2 : consumers, rows [0, 64) / [64, 128) of the tile: wgmma into registers + epilogue
//   warpgroup 3 (x3 only) : hi / lo splitters of the activation slabs
//   warpgroup 4 (x3 with the fused per-head 1x1 only) : the 1x1, from a ring of relu(conv + bias) chunks the
//                           consumers fill, so it runs under the next tile's MMAs
// Reference semantics: nn.Conv2d(k, stride 1, padding k//2) + folded BatchNorm + residual + ReLU
// (pose_dla_dcn.py:37-62, 153-168, 496-505).
#include <cuda.h>

#include "common.cuh"
#include "umma_common.cuh"

namespace cp {
namespace {

constexpr int TM_BM = 128;
constexpr int TM_THREADS = 384;       // control warpgroup + two consumer warpgroups
constexpr int TM_THREADS_X3 = 512;    // + the splitter warpgroup
constexpr int TM_THREADS_X3F = 640;   // + the fused 1x1 warpgroup
// x3 fused 1x1: a hidden-ring slot holds relu(conv + bias) of one tile's 128 rows x 32 columns; the 1x1 weights of
// one N tile (BN = 128 hidden channels x 16 outputs) are staged next to the ring
constexpr uint32_t TM_HSLOT_BYTES = 128u * 32u * 4u;
constexpr uint32_t TM_W1_BYTES = 128u * 16u * 4u;

struct TmaConvParams {
  CUtensorMap amap[4];
  int nsrc;
  int srcC[4];
  int B, H, W, Cin, Cout, CoutPad, BN;
  int k;              // 1 or 3
  int tile_m;         // output positions per tile (128)
  int Wt, boxh;       // padded pitch and slab rows (k == 3)
  int tiles_per_image;
  long long total_tiles;                // m tiles x n tiles (n fastest), x split-K factor
  long long m_tiles;                    // number of 128-position tiles
  uint32_t slab_bytes, slab_stride;   // TMA transaction bytes, 1024-aligned stage stride
  int SA, SB;
  const float* bias;
  const float* residual;
  int resStride, relu, res_after_relu;
  float* out;
  int outStride, out_nchw;
  int round_tf32;     // round the stored outputs to tf32 (consumers feed them to the tf32 MMAs untouched)
  int cslab;          // channels per slab: 32 (128-byte rows, SWIZZLE_128B) or 16 (64-byte rows, SWIZZLE_64B; Cin = 16 layers)
  int x3;             // 3-term split (fp32-equivalent): hi/lo slabs + hi/lo weight tiles, BN <= 128
  int group;          // x3: K blocks per accumulation group (promoted into the fp32 sums after each group)
  const unsigned char* wtiles;
  // split-K (x3, not fused): the K loop of a tile is dealt to `ksplit` CTAs (slab-aligned ranges of `sps` slabs); every
  // CTA stores its promoted partial sums and conv_tma_splitk_finish adds them in split order (deterministic) and runs
  // the epilogue.  ksplit == 1: off.  Tile index = (m, n) tile * ksplit + split.
  int ksplit, sps;
  float* part;          // [mn tiles][ksplit][BN / 4][tile_m] float4
  // fused per-head 1x1 (see IgemmParams): tph = N tiles per head, processed back to back by the same CTA
  int fuse, tph;
  const float* fuse_w[16];
  const float* fuse_b[16];
  float* fuse_out[16];
  int fuse_cout[16];
  // models (IgemmParams::ipm): image n is model n / ipm's.  The 1x1 position tiles are cut per model (tiles_per_model
  // of them over its ipm images) so that no tile mixes two models' weights.
  int ipm;
  long long wstride, tstride, tiles_per_model;
  int RS;             // x3 fused 1x1: slots of the hidden ring (1 or 2)
};

using namespace umma;

struct TmaCtl {
  unsigned long long a_full[4], a_empty[4], a_split[4];
  unsigned long long b_full[8], b_empty[8];
  unsigned long long h_full[2], h_empty[2];     // x3 fused 1x1: hidden ring
};
static_assert(sizeof(TmaCtl) <= 512, "control block");

// Tile geometry of one 128-position output tile.
struct TileGeo {
  int n_tile, img, g0, r_lo, model;
  long long pos0;
};
// MULTI: the launch holds several models (TmaConvParams::ipm); otherwise model is 0 and the code is that of one model.
template <bool MULTI>
__device__ __forceinline__ TileGeo decode_tile(const TmaConvParams& p, long long ct, int n_tiles) {
  TileGeo g;
  g.n_tile = (int)(ct % n_tiles);
  const long long m_tile = ct / n_tiles;
  g.img = 0;
  g.g0 = 0;
  g.r_lo = 0;
  g.pos0 = 0;
  g.model = 0;
  if (p.k == 3) {
    g.img = (int)(m_tile / p.tiles_per_image);
    g.g0 = (int)(m_tile - (long long)g.img * p.tiles_per_image) * p.tile_m;
    const int t = g.g0 - 1;
    g.r_lo = (t >= 0) ? t / p.Wt : -((-t + p.Wt - 1) / p.Wt);      // floor((g0 - 1) / Wt)
    if (MULTI) g.model = g.img / p.ipm;
  } else if (MULTI) {
    g.model = (int)(m_tile / p.tiles_per_model);
    g.pos0 = (long long)g.model * p.ipm * p.H * p.W + (m_tile - g.model * p.tiles_per_model) * p.tile_m;
  } else {
    g.pos0 = m_tile * p.tile_m;
  }
  return g;
}

// output position i of a tile -> (valid, image, row, column, flat NHWC index)
template <bool MULTI>
__device__ __forceinline__ bool tile_position(const TmaConvParams& p, const TileGeo& g, int i, int* n, int* oy, int* ox, int* m) {
  bool valid;
  if (p.k == 3) {
    const int gg = g.g0 + i;
    *oy = gg / p.Wt;
    const int xp = gg - *oy * p.Wt;
    *ox = xp - 1;
    *n = g.img;
    valid = (*oy < p.H) && (xp >= 1) && (xp <= p.W);
  } else {
    const long long pix = g.pos0 + i;
    // rows past the model's images belong to the next model
    valid = pix < (MULTI ? (long long)(g.model + 1) * p.ipm : (long long)p.B) * p.H * p.W;
    const long long pp = valid ? pix : 0;
    *ox = (int)(pp % p.W);
    const long long t = pp / p.W;
    *oy = (int)(t % p.H);
    *n = (int)(t / p.H);
  }
  *m = (int)(((size_t)*n * p.H + *oy) * p.W + *ox);
  return valid;
}

// PERSISTENT kernel: gridDim.x = min(#tiles, #SMs); CTA c processes tiles c, c + gridDim.x, ...  Every role keeps its
// pipeline state across tiles, so the TMA / split of tile i+1 overlap the epilogue of tile i and the fixed cost of a CTA
// (barrier init, descriptor fetch, pipeline fill) is paid once per SM instead of per tile.
//
// FOLD (x3, not fused; batch-invariant plans): one CTA per (m, n) tile sums the ksplit K segments of `sps` slabs back to
// back, each exactly as a split-K CTA of that segment does (its accumulation groups start at the segment's first K
// block), and adds them in segment order into a running total, ((0 + seg 0) + seg 1) + ..., which is what
// splitk_finish computes from the parked partial sums: a tile's outputs are the same bits on either path.
template <bool X3, bool FUSE, int BN, bool MULTI, bool FOLD>
__global__ void __launch_bounds__(X3 ? (FUSE ? TM_THREADS_X3F : TM_THREADS_X3) : TM_THREADS, 1)
    conv_tma_kernel(const __grid_constant__ TmaConvParams p) {
  // x3 fused: the per-head 1x1 runs in its own warpgroup (warps 16 - 19) behind the hidden ring
  constexpr bool EPI = X3 && FUSE;
  // setmaxnreg per role; the counts of the five (x3 fused) or four (x3) warpgroups add up to at most what the launch
  // gives 640 (96 each) or 512 (128 each) threads.  Counts above the launch's are taken with .inc, below it with .dec.
  constexpr int REG_CTL = EPI ? 32 : 40, REG_SPLIT = EPI ? 40 : 48, REG_EPI = 104, REG_CONS = EPI ? 152 : 208;
  extern __shared__ __align__(1024) unsigned char smem[];
  TmaCtl* ctl = reinterpret_cast<TmaCtl*>(smem);
  if (threadIdx.x == 0) griddep_launch_dependents();      // PDL (common.cuh): the next launch may take this SM when we retire
  const uint32_t slabs0 = (smem_u32(smem) + 512u + 1023u) & ~1023u;
  const uint32_t rowb = (uint32_t)p.cslab * 4u;                               // bytes per position row
  const uint32_t btile_bytes = (uint32_t)BN * rowb * (X3 ? 2u : 1u);          // hi (+ lo) weight tile
  const uint32_t a_stage = p.slab_stride * (X3 ? 2u : 1u);                    // hi (+ lo) slab
  const uint32_t btiles0 = slabs0 + (uint32_t)p.SA * a_stage;
  const uint32_t drain0 = btiles0 + (uint32_t)p.SB * btile_bytes;             // epilogue staging, one per consumer warpgroup

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_tiles = p.CoutPad / BN;
  const int taps = p.k * p.k;
  const int KS_SPLIT = FOLD ? 1 : p.ksplit;        // split-K factor (1 = off)
  const int sps = FOLD ? p.sps * p.ksplit : p.sps; // slabs per split (fold: every slab of the tile)
  const int KB = sps * taps;                       // K blocks THIS CTA runs per tile
  const int KB_all = (p.Cin / p.cslab) * taps;     // K blocks of the whole contraction (weight-tile addressing)
  const long long total_tiles = p.total_tiles;
  // Tile order of this CTA: units of `tph` consecutive tiles (same positions, the N tiles of one head when the 1x1 is
  // fused; tph = 1 otherwise), units strided over the CTAs.
  const long long tph = FUSE ? p.tph : 1;
  auto tile_at = [&](long long it) { return ((long long)blockIdx.x + (it / tph) * gridDim.x) * tph + (it % tph); };

  if (tid == 0) {
    for (int s = 0; s < p.SA; ++s) {
      mbar_init(smem_u32(&ctl->a_full[s]), 1);
      mbar_init(smem_u32(&ctl->a_empty[s]), 2);     // one arrival per consumer warpgroup
      mbar_init(smem_u32(&ctl->a_split[s]), 128);
    }
    for (int s = 0; s < p.SB; ++s) {
      mbar_init(smem_u32(&ctl->b_full[s]), 1);
      mbar_init(smem_u32(&ctl->b_empty[s]), 2);
    }
    if constexpr (EPI) {
      for (int s = 0; s < p.RS; ++s) {
        mbar_init(smem_u32(&ctl->h_full[s]), 256);     // every consumer thread
        mbar_init(smem_u32(&ctl->h_empty[s]), 128);    // every 1x1 thread
      }
    }
    fence_mbar_init();
  }
  __syncthreads();
  // PDL: everything above touched shared memory only.  The weight producer (warp 1) reads per-plan constants and runs
  // ahead; every other role waits here for the previous launch of the stream to finish before it reads an activation
  // (TMA slabs, residuals) or writes one.
  if (warp != 1) griddep_wait();

  // x3: 512 threads leave 128 registers per thread, but a consumer thread carries a 64 x BN accumulator AND the promoted
  // sums.  The control and splitter warpgroups hand registers to the consumers with setmaxnreg; the role code sits
  // inside the branch that executed it so that ptxas allocates per branch.
  if (warp < 4) {
    if (X3) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REG_CTL));
    if (warp == 0) {
      // ===================== activation slabs via TMA =====================
      if (lane == 0) {
        int stage = 0;
        uint32_t phase = 0;
        for (long long it = 0, tile = tile_at(0); tile < total_tiles; tile = tile_at(++it)) {
          const TileGeo g = decode_tile<MULTI>(p, tile / KS_SPLIT, n_tiles);
          const int s_begin = (int)(tile % KS_SPLIT) * sps;
          for (int s = s_begin; s < s_begin + sps; ++s) {
            int src = 0, cb = 0;
            while (src + 1 < p.nsrc && s * p.cslab >= cb + p.srcC[src]) {
              cb += p.srcC[src];
              ++src;
            }
            mbar_wait(smem_u32(&ctl->a_empty[stage]), phase ^ 1u);
            const uint32_t bar = smem_u32(&ctl->a_full[stage]);
            mbar_arrive_expect_tx(bar, p.slab_bytes);
            const uint32_t dst = slabs0 + (uint32_t)stage * a_stage;
            if (p.k == 3)
              tma_load_4d(dst, &p.amap[src], s * p.cslab - cb, -1, g.r_lo - 1, g.img, bar);
            else
              tma_load_2d(dst, &p.amap[src], s * p.cslab - cb, (int)g.pos0, bar);
            if (++stage == p.SA) {
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
        for (long long it = 0, tile = tile_at(0); tile < total_tiles; tile = tile_at(++it)) {
          const unsigned char* wsrc;
          if constexpr (MULTI) {
            const TileGeo g = decode_tile<MULTI>(p, tile / KS_SPLIT, n_tiles);
            wsrc = p.wtiles + (size_t)g.model * p.tstride +
                   ((size_t)g.n_tile * KB_all + (size_t)(tile % KS_SPLIT) * KB) * btile_bytes;
          } else {
            const int n_tile = (int)((tile / KS_SPLIT) % n_tiles);
            wsrc = p.wtiles + ((size_t)n_tile * KB_all + (size_t)(tile % KS_SPLIT) * KB) * btile_bytes;
          }
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
  } else if (EPI && warp >= 16) {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REG_EPI));
    // ===================== fused per-head 1x1 (x3): hidden ring -> head outputs =====================
    // Thread (rg, hh, og) accumulates rows rg + 32 i (i < 4) x outputs 8 og .. 8 og + 7 over hidden channels
    // c0 + 16 hh .. + 15 of every 32-column chunk, in increasing order and across the head's tph N tiles: each
    // (row, output) sees the products and order of a thread per row and half.
    const int wt = tid - 512, rg = wt >> 2, hh = (wt >> 1) & 1, og = wt & 1;
    // the hidden ring, then the staged 1x1 weights, take the place of the consumers' staging buffers
    const float* hring = reinterpret_cast<const float*>(smem + (drain0 - smem_u32(smem)));
    float4* w1 = reinterpret_cast<float4*>(smem + (drain0 - smem_u32(smem)) + (size_t)p.RS * TM_HSLOT_BYTES);
    const uint32_t bar_h_full = smem_u32(&ctl->h_full[0]), bar_h_empty = smem_u32(&ctl->h_empty[0]);
    auto at = [&](int r, int col) { return r * 32 + ((((col >> 2) ^ r) & 7) << 2) + (col & 3); };
    // the tile's 1x1 weights as float4 (hidden k, outputs 4 q .. 4 q + 3) at (4 k + q) ^ (k & 16 ? 4 : 0): rows k and
    // k ^ 1 trade places in the upper half of every 32, so the two hidden halves of a warp read different banks
    auto stage_w1 = [&](long long tile) {
      const TileGeo g = decode_tile<MULTI>(p, tile, n_tiles);
      const int head = g.n_tile / p.tph, part = g.n_tile - head * p.tph;
      const float4* src = reinterpret_cast<const float4*>(p.fuse_w[head] + (MULTI ? (size_t)g.model * p.wstride : 0)) +
                          (size_t)part * BN * 4;
      for (int i = wt; i < BN * 4; i += 128) w1[i ^ (((i >> 2) & 16) ? 4 : 0)] = __ldg(src + i);
    };
    int rs = 0;
    uint32_t rp = 0;
    float acc2[32];
    long long it = 0, tile = tile_at(0);
    if (tile < total_tiles) stage_w1(tile);
    wg_bar_sync(3);
    while (tile < total_tiles) {
      const TileGeo g = decode_tile<MULTI>(p, tile, n_tiles);
      const int head = g.n_tile / p.tph, part = g.n_tile - head * p.tph;
      if (part == 0) {
#pragma unroll
        for (int j = 0; j < 32; ++j) acc2[j] = 0.f;
      }
#pragma unroll 1
      for (int c0 = 0; c0 < BN; c0 += 32) {
        mbar_wait(bar_h_full + 8u * (uint32_t)rs, rp);
        const float* hs = hring + (size_t)rs * (TM_HSLOT_BYTES / 4);
#pragma unroll
        for (int m4 = 0; m4 < 4; ++m4) {
          const int k0 = 16 * hh + 4 * m4;          // hidden channels c0 + k0 .. + 3
          float4 hv[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) hv[i] = *reinterpret_cast<const float4*>(hs + at(rg + 32 * i, k0));
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const int wi = (((c0 + k0 + kk) << 2) + 2 * og) ^ (hh << 2);
            const float4 wa = w1[wi], wb = w1[wi + 1];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float h = kk == 0 ? hv[i].x : kk == 1 ? hv[i].y : kk == 2 ? hv[i].z : hv[i].w;
              acc2[8 * i + 0] = fmaf(h, wa.x, acc2[8 * i + 0]);
              acc2[8 * i + 1] = fmaf(h, wa.y, acc2[8 * i + 1]);
              acc2[8 * i + 2] = fmaf(h, wa.z, acc2[8 * i + 2]);
              acc2[8 * i + 3] = fmaf(h, wa.w, acc2[8 * i + 3]);
              acc2[8 * i + 4] = fmaf(h, wb.x, acc2[8 * i + 4]);
              acc2[8 * i + 5] = fmaf(h, wb.y, acc2[8 * i + 5]);
              acc2[8 * i + 6] = fmaf(h, wb.z, acc2[8 * i + 6]);
              acc2[8 * i + 7] = fmaf(h, wb.w, acc2[8 * i + 7]);
            }
          }
        }
        mbar_arrive(bar_h_empty + 8u * (uint32_t)rs);
        if (++rs == p.RS) {
          rs = 0;
          rp ^= 1u;
        }
      }
      if (part == p.tph - 1) {
        // the two hidden halves of a (row, output) are in lanes that differ in bit 1
#pragma unroll
        for (int j = 0; j < 32; ++j) acc2[j] += __shfl_xor_sync(0xffffffffu, acc2[j], 2);
        if (hh == 0) {
          const int co = p.fuse_cout[head] - 8 * og;          // outputs of this thread: min(8, co)
          const float* b2 = p.fuse_b[head] + (MULTI ? (size_t)g.model * p.wstride : 0) + 8 * og;
          float bo[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) bo[u] = u < co ? __ldg(b2 + u) : 0.f;
          const size_t plane = (size_t)p.H * p.W;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            int n1, oy1, ox1, m1;
            if (!tile_position<MULTI>(p, g, rg + 32 * i, &n1, &oy1, &ox1, &m1)) continue;
            float* o = p.fuse_out[head] + ((size_t)n1 * p.fuse_cout[head] * p.H + oy1) * p.W + ox1 + 8 * og * plane;
#pragma unroll
            for (int u = 0; u < 8; ++u)
              if (u < co) o[u * plane] = acc2[8 * i + u] + bo[u];
          }
        }
      }
      tile = tile_at(++it);
      wg_bar_sync(3);              // every thread is done with this tile's weights
      if (tile < total_tiles) stage_w1(tile);
      wg_bar_sync(3);
    }
  } else if (X3 && warp >= 12) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REG_SPLIT));
    // ===================== hi / lo splitters (x3): slab -> tf32-exact hi (in place) + lo slab =====================
    const int st = tid - 384;
    int stage = 0;
    uint32_t phase = 0;
    const uint32_t nchunk = p.slab_bytes >> 4;
    for (long long it = 0, tile = tile_at(0); tile < total_tiles; tile = tile_at(++it)) {
      for (int s = 0; s < sps; ++s) {
        mbar_wait(smem_u32(&ctl->a_full[stage]), phase);
        const uint32_t hi = slabs0 + (uint32_t)stage * a_stage;
        const uint32_t lo = hi + p.slab_stride;
        for (uint32_t c0 = st; c0 < nchunk; c0 += 128 * 4) {
          float4 v[4];
#pragma unroll
          for (int u = 0; u < 4; ++u)                       // 4 independent loads in flight per thread
            if (c0 + u * 128 < nchunk) v[u] = ld_shared_v4f(hi + ((c0 + u * 128) << 4));
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            if (c0 + u * 128 < nchunk) {
              float4 h, l;
              h.x = tf32_round(v[u].x); l.x = tf32_round(v[u].x - h.x);
              h.y = tf32_round(v[u].y); l.y = tf32_round(v[u].y - h.y);
              h.z = tf32_round(v[u].z); l.z = tf32_round(v[u].z - h.z);
              h.w = tf32_round(v[u].w); l.w = tf32_round(v[u].w - h.w);
              st_shared_v4f(hi + ((c0 + u * 128) << 4), h.x, h.y, h.z, h.w);
              st_shared_v4f(lo + ((c0 + u * 128) << 4), l.x, l.y, l.z, l.w);
            }
          }
        }
        fence_proxy_async_smem();
        mbar_arrive(smem_u32(&ctl->a_split[stage]));
        if (++stage == p.SA) {
          stage = 0;
          phase ^= 1u;
        }
      }
    }
  } else {
    if (X3) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REG_CONS));
    // ===================== consumers: warpgroup c multiplies rows [64 c, 64 c + 64) of every tile =====================
    const int c = (warp - 4) >> 2, wt = tid & 127;
    float* dstage = reinterpret_cast<float*>(smem + (drain0 - smem_u32(smem))) + (size_t)c * (DRAIN_STAGE_BYTES / 4);
    const uint32_t bar_a = smem_u32(X3 ? &ctl->a_split[0] : &ctl->a_full[0]);
    const uint32_t bar_a_empty = smem_u32(&ctl->a_empty[0]);
    const uint32_t bar_b_full = smem_u32(&ctl->b_full[0]), bar_b_empty = smem_u32(&ctl->b_empty[0]);
    const uint32_t a_lo_u = p.slab_stride >> 4, b_lo_u = ((uint32_t)BN * rowb) >> 4;
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
    int sa = 0, sb = 0;
    uint32_t pa = 0, pb = 0;
    float acc[BN / 2];
    float sums[X3 ? BN / 2 : 1];
    float tot[FOLD ? BN / 2 : 1];        // fold: the running total of the finished K segments
    float acc2[FUSE ? 16 : 1];           // fused 1x1: partial outputs (this thread's half of the hidden channels) of its row
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
#pragma unroll
    for (int j = 0; j < (FUSE ? 16 : 1); ++j) acc2[j] = 0.f;
    for (long long it = 0, tile = tile_at(0); tile < total_tiles; tile = tile_at(++it)) {
      const TileGeo g = decode_tile<MULTI>(p, tile / KS_SPLIT, n_tiles);
      // A row of tap (ky, kx) for tile row 64 c: start of the slab + (g0 - 1 - r_lo Wt) + ky Wt + kx + 64 c
      const uint32_t row0 = (p.k == 3 ? (uint32_t)(g.g0 - 1 - g.r_lo * p.Wt) : 0u) + (uint32_t)c * 64u;
#pragma unroll
      for (int j = 0; j < (X3 ? BN / 2 : 1); ++j) sums[j] = 0.f;
      if constexpr (FOLD) {
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) tot[j] = 0.f;
      }
      // x3: the K blocks of an accumulation group chain on one accumulator, so each stays in flight until the next one of
      // its group is queued behind it, and the group's last is waited for before the promotion; the wgmmas and their
      // order are those of a wait after every K block.  With one slab stage the next slab's TMA needs the stage back at
      // once, so there (and in tf32, where there is no group) every K block is waited for.
      const int group = X3 ? p.group : 1;
      const bool overlap = X3 && p.SA > 1;
      int tap = 0;
      // retire the K block before position (sb, sa, tap): its weight stage, and its slab stage when it was a slab's last tap
      auto release_prev = [&]() {
        if (wt == 0) {
          mbar_arrive(bar_b_empty + 8u * (uint32_t)(sb == 0 ? p.SB - 1 : sb - 1));
          if (tap == 0) mbar_arrive(bar_a_empty + 8u * (uint32_t)(sa == 0 ? p.SA - 1 : sa - 1));
        }
      };
      const int KB_seg = FOLD ? p.sps * taps : KB;       // K blocks of one segment
      for (int seg = 0; seg < (FOLD ? p.ksplit : 1); ++seg) {
        for (int kb0 = 0; kb0 < KB_seg; kb0 += group) {
          const int n_kb = min(group, KB_seg - kb0);
          for (int i = 0; i < n_kb; ++i) {
            if (tap == 0) mbar_wait(bar_a + 8u * (uint32_t)sa, pa);
            const int ky = tap / 3, kx = tap - ky * 3;
            const uint32_t arow = row0 + (p.k == 3 ? (uint32_t)(ky * p.Wt + kx) : 0u);
            mbar_wait(bar_b_full + 8u * (uint32_t)sb, pb);
            const uint64_t da = make_desc(slabs0 + (uint32_t)sa * a_stage + arow * rowb, p.cslab);
            const uint64_t db = make_desc(btiles0 + (uint32_t)sb * btile_bytes, p.cslab);
            const bool fresh = X3 ? i == 0 : kb0 == 0;
            if (p.cslab == 32)
              mma_kblock_issue<BN, X3, false, 4>(acc, da, db, a_lo_u, b_lo_u, fresh);
            else
              mma_kblock_issue<BN, X3, false, 2>(acc, da, db, a_lo_u, b_lo_u, fresh);
            if (overlap && i > 0) {
              wg_wait<1>();
              release_prev();
            }
            if (++sb == p.SB) {
              sb = 0;
              pb ^= 1u;
            }
            if (++tap == taps) {
              tap = 0;
              if (++sa == p.SA) {
                sa = 0;
                pa ^= 1u;
              }
            }
            if (!overlap) {
              wg_wait<0>();
              release_prev();
            }
          }
          wg_wait<0>();
          if (overlap) release_prev();
          // two-level accumulation: the tensor core sums `group` K blocks, every finished group is added into fp32
          // registers with round-to-nearest
#pragma unroll
          for (int j = 0; j < (X3 ? BN / 2 : 1); ++j)
            if (X3) sums[j] += acc[X3 ? j : 0];
        }
        if constexpr (FOLD) {
          // the segment is done: add it to the total and start the next one from zero, as its split-K CTA would
#pragma unroll
          for (int j = 0; j < BN / 2; ++j) {
            tot[j] += sums[j];
            sums[j] = 0.f;
          }
        }
      }
      // x3: the next tile's first wgmma overwrites the accumulator, so it is dead through the epilogue; saying so frees
      // its registers there for the drain and the fused 1x1 (ptxas then spills less, DESIGN §4)
      if (X3) {
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
      }
      if constexpr (EPI) {
        // relu(conv + bias) of this warpgroup's 64 rows goes to the hidden ring, 32 columns per slot, 16-byte groups
        // XOR-swizzled by row & 7 (conflict-free float4 reads); the 1x1 warpgroup takes it from there
        const int fr0 = (wt >> 5) * 16 + ((wt & 31) >> 2), fcq = (wt & 3) * 2;     // accumulator fragment (drain_rows)
        const float* b1 = p.bias + (MULTI ? (size_t)g.model * p.wstride : 0) + (size_t)g.n_tile * BN;
        float* hring = reinterpret_cast<float*>(smem + (drain0 - smem_u32(smem)));        // hidden ring
        const uint32_t bar_h_full = smem_u32(&ctl->h_full[0]), bar_h_empty = smem_u32(&ctl->h_empty[0]);
        auto at = [&](int r, int col) { return r * 32 + ((((col >> 2) ^ r) & 7) << 2) + (col & 3); };
#pragma unroll
        for (int c0 = 0; c0 < BN; c0 += 32) {
          const uint32_t chunk = (uint32_t)it * (BN / 32) + c0 / 32;       // chunks so far: ring slot and phase
          const uint32_t rs = chunk % p.RS, rp = (chunk / p.RS) & 1u;
          mbar_wait(bar_h_empty + 8u * rs, rp ^ 1u);
          float* hs = hring + (size_t)rs * (TM_HSLOT_BYTES / 4) + c * 64 * 32;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            if (j * 8 >= c0 && j * 8 < c0 + 32) {
              const int col = j * 8 - c0 + fcq;
              const float bx = __ldg(b1 + c0 + col), by = __ldg(b1 + c0 + col + 1);
              hs[at(fr0, col)] = fmaxf(sums[X3 ? 4 * j : 0] + bx, 0.f);
              hs[at(fr0, col + 1)] = fmaxf(sums[X3 ? 4 * j + 1 : 0] + by, 0.f);
              hs[at(fr0 + 8, col)] = fmaxf(sums[X3 ? 4 * j + 2 : 0] + bx, 0.f);
              hs[at(fr0 + 8, col + 1)] = fmaxf(sums[X3 ? 4 * j + 3 : 0] + by, 0.f);
            }
          }
          mbar_arrive(bar_h_full + 8u * rs);
        }
        continue;
      }
      // ---- epilogue: rows of this warpgroup, 32 columns at a time through shared memory (drain_rows)
      const int r_me = wt >> 1;
      int n, oy, ox, m;
      const bool valid = tile_position<MULTI>(p, g, c * 64 + r_me, &n, &oy, &ox, &m);
      const int col_end = min(p.Cout, (g.n_tile + 1) * BN);
      const int head = FUSE ? g.n_tile / p.tph : 0, part = FUSE ? g.n_tile - head * p.tph : 0;
      const size_t wofs = MULTI ? (size_t)g.model * p.wstride : 0;      // this tile's model's biases and fused 1x1 weights
      if (MULTI) ep.bias = p.bias + wofs;
      if (FUSE && part == 0) {
#pragma unroll
        for (int j = 0; j < (FUSE ? 16 : 1); ++j) acc2[j] = 0.f;
      }
      auto fn = [&](int r, int cb, float (&v)[16]) {
        if (cb >= BN) return;
        if (!FUSE && KS_SPLIT > 1) {
          // split-K: park the partial sums of this K range, [mn tile][split][float4 column group][row];
          // conv_tma_splitk_finish adds the ranges in split order (a fixed summation order) and runs the epilogue
          const long long mn = tile / KS_SPLIT;
          const int ks = (int)(tile % KS_SPLIT);
          float4* mine = reinterpret_cast<float4*>(p.part) + (((size_t)mn * KS_SPLIT + ks) * (BN >> 2) + (cb >> 2)) * p.tile_m +
                         c * 64 + r;
#pragma unroll
          for (int q = 0; q < 4; ++q) __stcg(mine + (size_t)q * p.tile_m, make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]));
        } else if (FUSE) {
          // hidden = relu(conv3x3 + bias) never leaves the SM: multiply it with this head's 1x1 weights right here
          const float* b1 = p.bias + wofs + (size_t)g.n_tile * BN + cb;
          const float4* w2 = reinterpret_cast<const float4*>(p.fuse_w[head] + wofs) + ((size_t)part * BN + cb) * 4;
#pragma unroll
          for (int q = 0; q < 16; ++q) {
            const float h = fmaxf(v[q] + __ldg(b1 + q), 0.f);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const float4 w = __ldg(w2 + q * 4 + u);
              acc2[FUSE ? 4 * u + 0 : 0] = fmaf(h, w.x, acc2[FUSE ? 4 * u + 0 : 0]);
              acc2[FUSE ? 4 * u + 1 : 0] = fmaf(h, w.y, acc2[FUSE ? 4 * u + 1 : 0]);
              acc2[FUSE ? 4 * u + 2 : 0] = fmaf(h, w.z, acc2[FUSE ? 4 * u + 2 : 0]);
              acc2[FUSE ? 4 * u + 3 : 0] = fmaf(h, w.w, acc2[FUSE ? 4 * u + 3 : 0]);
            }
          }
        } else {
          epilogue_row<16>(ep, v, valid, m, n, oy, ox, g.n_tile * BN + cb, col_end);
        }
      };
      if constexpr (FOLD)
        drain_rows<BN>(tot, dstage, wt, 1 + c, fn);
      else if constexpr (X3)
        drain_rows<BN>(sums, dstage, wt, 1 + c, fn);
      else
        drain_rows<BN>(acc, dstage, wt, 1 + c, fn);
      if (FUSE && part == p.tph - 1) {
        // the two threads of a row (lanes 2 r, 2 r + 1) each hold half of the hidden channels
#pragma unroll
        for (int j = 0; j < (FUSE ? 16 : 1); ++j) acc2[j] += __shfl_xor_sync(0xffffffffu, acc2[j], 1);
        if ((wt & 1) == 0 && valid) {
          const int co = p.fuse_cout[head];
          float* o = p.fuse_out[head] + ((size_t)n * co * p.H + oy) * p.W + ox;
          const size_t plane = (size_t)p.H * p.W;
#pragma unroll
          for (int j = 0; j < 16; ++j)
            if (j < co) o[j * plane] = acc2[FUSE ? j : 0] + __ldg(p.fuse_b[head] + wofs + j);
        }
      }
    }
  }
}

// weight tiles for the slab-major K order:  kb = slab * taps + tap,  element j of the row = channel slab*32 + j
__global__ void pack_tma_weight_kernel(const float* __restrict__ src, int ld, int Cin, int taps, int Cout, int BN, int n_tiles,
                                       int round_tf32, int x3, int cslab, unsigned char* __restrict__ dst) {
  const int KB = (Cin / cslab) * taps;
  const int cpr = cslab / 4;                 // 16-byte chunks per row: 8 or 4
  const size_t rowb = (size_t)cslab * 4;
  const size_t total = (size_t)n_tiles * KB * BN * cpr;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = i % cpr;
    size_t t = i / cpr;
    const int nr = t % BN;
    t /= BN;
    const int kb = t % KB;
    const int nt = t / KB;
    const int n = nt * BN + nr;
    const int slab = kb / taps, tap = kb - slab * taps;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = tap * Cin + slab * cslab + q * 4 + j;
      float x = (n < Cout) ? src[(size_t)k * ld + n] : 0.f;
      v[j] = round_tf32 ? tf32_round(x) : x;
    }
    const size_t tile = ((size_t)nt * KB + kb) * (size_t)BN * rowb * (x3 ? 2 : 1);
    // SWIZZLE_128B: chunk ^= row & 7 (address bits [7,10));  SWIZZLE_64B: chunk ^= (row >> 1) & 3 (bits [7,9))
    const int sw = cslab == 32 ? (nr & 7) : ((nr >> 1) & 3);
    const size_t off = (size_t)nr * rowb + (size_t)((q ^ sw) << 4);
    *reinterpret_cast<float4*>(dst + tile + off) = make_float4(v[0], v[1], v[2], v[3]);
    if (x3) {     // lo tile = residual of the tf32 rounding (round_tf32 is always set together with x3)
      float l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k = tap * Cin + slab * cslab + q * 4 + j;
        const float x = (n < Cout) ? src[(size_t)k * ld + n] : 0.f;
        l[j] = tf32_round(x - v[j]);
      }
      *reinterpret_cast<float4*>(dst + tile + (size_t)BN * rowb + off) = make_float4(l[0], l[1], l[2], l[3]);
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

}  // namespace

// split-K, second half (splitk_finish, umma_common.cuh): tile row i -> output position
template <bool MULTI>
__global__ void __launch_bounds__(256) conv_tma_splitk_finish(const __grid_constant__ TmaConvParams p, long long mn_tiles) {
  splitk_finish<MULTI>(p, p.tile_m, mn_tiles, [&](long long mn, int i, int* n, int* oy, int* ox) {
    int m;
    return tile_position<MULTI>(p, decode_tile<MULTI>(p, mn, p.CoutPad / p.BN), i, n, oy, ox, &m);
  });
}

// ---------------------------------------------------------------------------------------------------- host side
// Channels per activation slab.  32 (128-byte rows) by default; 16 (64-byte rows, SWIZZLE_64B) when Cin is not a
// multiple of 32, or when the 3-term split (hi + lo slabs) could not be double-buffered with 32-channel slabs.
static int tma_boxh(int Wt) { return (TM_BM + 1 + 2 * Wt + Wt - 1) / Wt + 1; }

// Shared memory for the slab and weight-tile rings: 227 KB less the control block, alignment, slack and the two
// epilogue staging buffers.
constexpr size_t TM_BUDGET = 222 * 1024 - 2 * (size_t)DRAIN_STAGE_BYTES;
// x3 fused 1x1: the hidden ring and the staged 1x1 weights take the place of the two staging buffers
static size_t tma_epi_bytes(int rs) { return (size_t)rs * TM_HSLOT_BYTES + TM_W1_BYTES; }

// Stage counts of the slab ring (SA), the weight-tile ring (SB) and, x3 with the fused 1x1 (epi), the hidden ring (RS).
// Two hidden slots where two slab stages and three weight stages still fit next to them, else one.
static int tma_smem_layout(uint32_t a_stage, uint32_t btile, int k, bool epi, int* SA, int* SB, int* RS, size_t* smem) {
  size_t fixed = 2 * (size_t)DRAIN_STAGE_BYTES;
  *RS = 0;
  if (epi) {
    *RS = 2 * (size_t)a_stage + 3 * (size_t)btile <= 222 * 1024 - tma_epi_bytes(2) ? 2 : 1;
    fixed = tma_epi_bytes(*RS);
  }
  const size_t budget = 222 * 1024 - fixed;
  int sa = 2;
  if ((size_t)sa * a_stage + 2 * (size_t)btile > budget) sa = 1;
  if ((size_t)sa * a_stage + 2 * (size_t)btile > budget) return fail(CP_ERR_INVALID, "conv_tma: slab does not fit shared memory");
  int sb = (int)((budget - (size_t)sa * a_stage) / btile);
  if (sb > 8) sb = 8;
  if (sb < 2) return fail(CP_ERR_INVALID, "conv_tma: tile does not fit shared memory");
  if (k == 1 && sa < 4) {
    // 1x1: slabs are small (16 KB); use up to 4 stages of them
    int s4 = (int)((budget - (size_t)sb * btile) / a_stage);
    if (s4 > 4) s4 = 4;
    if (s4 > sa) sa = s4;
  }
  *SA = sa;
  *SB = sb;
  *smem = 512 + 2048 + (size_t)sa * a_stage + (size_t)sb * btile + fixed;
  return CP_OK;
}

int tma_cslab(const IgemmParams& p, int x3) {
  if (p.Cin % 32) return 16;
  if (!x3 || p.kh != 3) return 32;
  const int Wt = p.Win + 2;
  const int boxh = tma_boxh(Wt);
  const size_t slab32 = ((size_t)boxh * Wt * 128 + 1023) / 1024 * 1024;
  const int bn = tma_tile_n(p.CoutPad, x3);
  const size_t need = 2 * (2 * slab32) + 2 * ((size_t)bn * 128 * 2);
  return need > TM_BUDGET ? 16 : 32;
}

// wgmma N of the consumer warpgroups: the accumulator takes BN / 2 registers per thread (x3: twice that with the sums);
// N = 256 would spill
int tma_tile_n(int CoutPad, int) { return wgmma_tile_n(CoutPad, 128); }

bool tma_conv_supported(const IgemmParams& p, int x3) {
  if (p.mode != IGEMM_NHWC_VEC) return false;
  if (!((p.kh == 1 && p.kw == 1 && p.pad == 0) || (p.kh == 3 && p.kw == 3 && p.pad == 1))) return false;
  if (p.stride != 1) return false;
  const int cs = tma_cslab(p, x3);
  if (p.Cin % cs) return false;
  for (int s = 0; s < p.nsrc; ++s)
    if (p.srcC[s] % cs || p.srcStride[s] % 4) return false;
  if (p.kh == 3 && p.Win + 2 > 256) return false;
  const int bn = tma_tile_n(p.CoutPad, x3);
  if (bn == 0) return false;
  // one single-buffered slab stage (+ its lo copy in x3) and two weight tiles must fit shared memory
  const size_t slab = p.kh == 3 ? (size_t)tma_boxh(p.Win + 2) * (p.Win + 2) * cs * 4 : (size_t)TM_BM * cs * 4;
  const size_t a_stage = ((slab + 1023) / 1024 * 1024) * (x3 ? 2 : 1);
  const size_t btile = (size_t)bn * cs * 4 * (x3 ? 2 : 1);
  // a shape question only (cp_plan_memory answers it without a driver); tma_encode_nhwc_box reports a missing encoder
  return a_stage + 2 * btile <= TM_BUDGET;
}

long long conv_tma_image_tiles(const IgemmParams& p, int BN) {
  const long long positions = p.kh == 3 ? (long long)p.Hin * (p.Win + 2) : (long long)p.Hin * p.Win;
  return (positions + TM_BM - 1) / TM_BM * (p.CoutPad / BN);
}

size_t tma_weight_bytes(int Cin, int taps, int CoutPad, int x3) {
  return (size_t)CoutPad * Cin * taps * 4 * (x3 ? 2 : 1);
}

// The tiles are tf32-rounded: both TMA kernels feed them to the tf32 MMAs as they are.
int launch_pack_tma_weight(const float* src, int ld, int Cin, int taps, int Cout, int CoutPad, int x3, int cs, int bn,
                           void* dst, cudaStream_t s) {
  const int nt = CoutPad / bn;
  size_t total = (size_t)nt * (Cin / cs) * taps * bn * (cs / 4);
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 32) blocks = 132 * 32;
  pack_tma_weight_kernel<<<blocks, 256, 0, s>>>(src, ld, Cin, taps, Cout, bn, nt, 1, x3, cs, (unsigned char*)dst);
  CP_LAUNCH_CHECK("pack_tma_weight_kernel");
  return CP_OK;
}

// One 4-D fp32 NHWC tensor map {C, W, H, B} with box {boxC, boxW, boxH, 1}, un-swizzled or SWIZZLE_64B (dcn_tma.cu slabs).
int tma_encode_nhwc_box(const float* base, int C, int W, int H, int B, int strideFloats, int boxC, int boxW, int boxH,
                        int swizzle64, void* map_out) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return fail(CP_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)strideFloats * 4, (cuuint64_t)W * strideFloats * 4, (cuuint64_t)H * W * strideFloats * 4};
  cuuint32_t box[4] = {(cuuint32_t)boxC, (cuuint32_t)boxW, (cuuint32_t)boxH, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(reinterpret_cast<CUtensorMap*>(map_out), CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)base, dims, strides, box,
                   es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(CP_ERR_CUDA, "cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
  return CP_OK;
}

// Encodes the tensor maps of the op's sources into `maps_out` (4 x 128 bytes, host memory, reusable across launches).
int tma_conv_encode(const IgemmParams& p, int Bmax, int cs, void* maps_out) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return fail(CP_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  CUtensorMap* maps = reinterpret_cast<CUtensorMap*>(maps_out);
  const int Wt = p.Win + 2;
  const int boxh = tma_boxh(Wt);
  const CUtensorMapSwizzle swz = cs == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  for (int s = 0; s < p.nsrc; ++s) {
    CUresult r;
    if (p.kh == 3) {
      cuuint64_t dims[4] = {(cuuint64_t)p.srcC[s], (cuuint64_t)p.Win, (cuuint64_t)p.Hin, (cuuint64_t)Bmax};
      cuuint64_t strides[3] = {(cuuint64_t)p.srcStride[s] * 4, (cuuint64_t)p.Win * p.srcStride[s] * 4,
                               (cuuint64_t)p.Hin * p.Win * p.srcStride[s] * 4};
      cuuint32_t box[4] = {(cuuint32_t)cs, (cuuint32_t)Wt, (cuuint32_t)boxh, 1};
      cuuint32_t es[4] = {1, 1, 1, 1};
      r = enc(&maps[s], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)p.src[s], dims, strides, box, es,
              CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    } else {
      cuuint64_t dims[2] = {(cuuint64_t)p.srcC[s], (cuuint64_t)Bmax * p.Hin * p.Win};
      cuuint64_t strides[1] = {(cuuint64_t)p.srcStride[s] * 4};
      cuuint32_t box[2] = {(cuuint32_t)cs, (cuuint32_t)TM_BM};
      cuuint32_t es[2] = {1, 1};
      r = enc(&maps[s], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)p.src[s], dims, strides, box, es,
              CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (r != CUDA_SUCCESS) return fail(CP_ERR_CUDA, "cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
  }
  return CP_OK;
}

// FOLD (x3, not fused only): the K segments folded in one CTA per tile (batch-invariant plans)
template <bool X3, bool FUSE, bool MULTI, bool FOLD = false>
static int launch_conv_tma_kernel(const TmaConvParams& q, const cudaLaunchConfig_t& cfg0) {
  void (*kern)(TmaConvParams) = nullptr;
  switch (q.BN) {
    case 16: kern = conv_tma_kernel<X3, FUSE, 16, MULTI, FOLD>; break;
    case 32: kern = conv_tma_kernel<X3, FUSE, 32, MULTI, FOLD>; break;
    case 64: kern = conv_tma_kernel<X3, FUSE, 64, MULTI, FOLD>; break;
    case 128: kern = conv_tma_kernel<X3, FUSE, 128, MULTI, FOLD>; break;
    default: return fail(CP_ERR_INVALID, "conv_tma: unsupported N tile");
  }
  static PerDevice<bool, 4> configured;
  const int slot = q.BN == 128 ? 3 : (q.BN == 64 ? 2 : (q.BN == 32 ? 1 : 0));
  if (!configured.here(slot)) {
    CP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    configured.here(slot) = true;
  }
  cudaLaunchConfig_t cfg = cfg0;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = g_pdl ? 1 : 0;
  CP_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, q));
  CP_LAUNCH_CHECK("conv_tma_kernel");
  return CP_OK;
}

int launch_conv_tma(const IgemmParams& p, const void* maps, const ConvKernel& k, cudaStream_t stream, LaunchInfo* info) {
  if (!p.wgt_umma) return fail(CP_ERR_INVALID, "conv_tma: weight tiles missing");
  if (p.B % model_ipm(p)) return fail(CP_ERR_INVALID, "conv_tma: batch is not a whole number of models");
  const bool x3 = k.x3;
  TmaConvParams q;
  memset(&q, 0, sizeof(q));
  memcpy(q.amap, maps, sizeof(CUtensorMap) * 4);
  q.nsrc = p.nsrc;
  for (int s = 0; s < 4; ++s) q.srcC[s] = p.srcC[s];
  q.B = p.B;
  q.H = p.Hin;
  q.W = p.Win;
  q.Cin = p.Cin;
  q.Cout = p.Cout;
  q.CoutPad = p.CoutPad;
  q.BN = k.BN;
  q.x3 = x3;
  q.cslab = k.cslab;
  q.group = kX3GroupBlocks * (32 / q.cslab);       // same number of MMAs per accumulation group
  q.k = p.kh;
  q.Wt = p.Win + 2;
  q.tile_m = TM_BM;
  q.boxh = tma_boxh(q.Wt);
  q.ipm = model_ipm(p);
  q.wstride = p.wstride;
  q.tstride = p.tstride;
  size_t m_tiles;
  if (q.k == 3) {
    q.tiles_per_image = (p.Hin * q.Wt + q.tile_m - 1) / q.tile_m;
    m_tiles = (size_t)q.tiles_per_image * p.B;
    q.slab_bytes = (uint32_t)q.boxh * q.Wt * (uint32_t)q.cslab * 4u;
  } else {
    q.tiles_per_image = 0;
    q.tiles_per_model = ((long long)q.ipm * p.Hin * p.Win + q.tile_m - 1) / q.tile_m;
    m_tiles = (size_t)q.tiles_per_model * (p.B / q.ipm);
    q.slab_bytes = (uint32_t)q.tile_m * (uint32_t)q.cslab * 4u;
  }
  q.slab_stride = (q.slab_bytes + 1023u) & ~1023u;
  const uint32_t btile = (uint32_t)q.BN * (uint32_t)q.cslab * 4u * (x3 ? 2u : 1u);
  const uint32_t a_stage = q.slab_stride * (x3 ? 2u : 1u);
  size_t smem = 0;
  if (int rc = tma_smem_layout(a_stage, btile, q.k, x3 && p.fuse_n > 0, &q.SA, &q.SB, &q.RS, &smem)) return rc;
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
  if (p.fuse_n > 0) {
    if (p.fuse_hidden % q.BN || p.CoutPad != p.fuse_n * p.fuse_hidden || !p.relu || p.residual || (x3 && q.BN != 128))
      return fail(CP_ERR_INVALID, "conv_tma: fused 1x1 needs relu, no residual and head_conv a multiple of the N tile");
    q.fuse = 1;
    q.tph = p.fuse_hidden / q.BN;
    for (int h = 0; h < p.fuse_n; ++h) {
      q.fuse_w[h] = p.fuse_w[h];
      q.fuse_b[h] = p.fuse_b[h];
      q.fuse_out[h] = p.fuse_out[h];
      q.fuse_cout[h] = p.fuse_cout[h];
    }
  }
  q.m_tiles = (long long)m_tiles;
  q.part = p.splitk_ws;
  const long long mn = (long long)m_tiles * (p.CoutPad / q.BN);
  const int nslab = q.Cin / q.cslab;
  int num_sms = 0;
  if (int rc = device_sm_count(&num_sms)) return rc;
  // split-K (tf32x3, plain epilogue): small feature maps give a persistent kernel fewer tiles than SMs while every tile
  // walks a long serial K loop (level5 at batch 1: 16 tiles x 144 K blocks).  Deal slab-aligned K ranges to more CTAs.
  // Batch-invariant plans fix the segments by the layer's shape (k.ksegments) and split them only when their partial sums
  // fit the workspace; otherwise one CTA per tile folds them (the FOLD instances of conv_tma_kernel), with the same bits.
  const size_t tile_floats = (size_t)q.tile_m * q.BN;
  bool fold = false;
  if (k.ksegments > 0) {
    if (nslab % k.ksegments || (k.ksegments > 1 && (!x3 || q.fuse)))
      return fail(CP_ERR_INVALID, "conv_tma: K segments do not fit the launch");
    q.ksplit = k.ksegments;
    fold = q.ksplit > 1 && (size_t)mn * q.ksplit * tile_floats > p.splitk_ws_floats;
  } else {
    q.ksplit = x3 && !q.fuse ? splitk_factor(mn, nslab, num_sms, tile_floats, p.splitk_ws_floats) : 1;
  }
  q.sps = nslab / q.ksplit;
  q.total_tiles = fold ? mn : mn * q.ksplit;
  if (q.total_tiles >= (1ll << 31)) return fail(CP_ERR_INVALID, "conv_tma: too many tiles");
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)(q.total_tiles < num_sms ? q.total_tiles : num_sms));
  cfg.blockDim = dim3(x3 ? (q.fuse ? TM_THREADS_X3F : TM_THREADS_X3) : TM_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  // several models in the launch: the model-indexed instantiations; one model runs the one-model code unchanged
  const bool multi = p.B > q.ipm;
  int rc;
  if (fold)
    rc = multi ? launch_conv_tma_kernel<true, false, true, true>(q, cfg) : launch_conv_tma_kernel<true, false, false, true>(q, cfg);
  else if (multi)
    rc = x3 ? (q.fuse ? launch_conv_tma_kernel<true, true, true>(q, cfg) : launch_conv_tma_kernel<true, false, true>(q, cfg))
            : (q.fuse ? launch_conv_tma_kernel<false, true, true>(q, cfg) : launch_conv_tma_kernel<false, false, true>(q, cfg));
  else
    rc = x3 ? (q.fuse ? launch_conv_tma_kernel<true, true, false>(q, cfg) : launch_conv_tma_kernel<true, false, false>(q, cfg))
            : (q.fuse ? launch_conv_tma_kernel<false, true, false>(q, cfg) : launch_conv_tma_kernel<false, false, false>(q, cfg));
  if (rc) return rc;
  if (info) {
    info->BN = q.BN;
    info->ksplit = q.ksplit;
    info->grid = cfg.gridDim.x;
    info->path = q.ksplit == 1 ? CP_KPATH_ONE : (fold ? CP_KPATH_FOLD : CP_KPATH_SPLIT);
  }
  if (q.ksplit > 1 && !fold) {
    const long long threads = mn * (q.BN / 4) * q.tile_m;
    CP_CUDA_CHECK(launch_kernel(multi ? conv_tma_splitk_finish<true> : conv_tma_splitk_finish<false>,
                                dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, stream, q, mn));
    CP_LAUNCH_CHECK("conv_tma_splitk_finish");
  }
  return CP_OK;
}

}  // namespace cp

// Heat-map decode, keypoint-to-centre grouping, output-map -> image affine,
// score filter + Gaussian soft-NMS and per-object PnP, entirely on the GPU.
//
// Two kernels per batch:
//   peaks_topk_kernel   one CTA per (image, heat-map channel): sigmoid, 3x3
//                       equality NMS and an exact top-K (radix select + bitonic
//                       sort) in shared memory -- each map is read from HBM once.
//                       Maps over TOPK_SMEM_CELLS cells (keep_res / fix_short
//                       inputs of ~800 x 600 and up) keep the NMS-ed map in the
//                       workspace instead; the selection is the same.
//   group_pose_kernel   one CTA per image: gathers at the K centres, K x K
//                       nearest-peak match per joint, the decode.py gates, the
//                       post_process.py affine, soft-NMS and the PnP solve
//                       (pose_core.h), writing the fixed-shape pose records.
//
// Reference semantics reproduced (paths relative to /root/reference/src/lib):
//   detectors/object_pose.py:136-138  sigmoid;  models/decode.py:17-23 _nms;
//   :40-68 _topk / _topk_channel;  :72-375 object_pose_decode(Inference=True);
//   utils/post_process.py:12-68;  utils/image.py:23-74 (rot = 0);
//   detectors/object_pose.py:184-197 merge_outputs, :27-124 soft_nms_nvidia;
//   detectors/base_detector.py:548-566 point assembly;  utils/pnp/*.
// The seven-gate test at decode.py:183-188 follows the pinned torch==1.1.0
// semantics (uint8 adds, `== 7` means all gates hold) -- see DESIGN.md.
#include "common.cuh"
#include "pose_core.h"
#include "pnp_warp.cuh"

namespace cp {
namespace {

constexpr float SENT = -10000.0f;
constexpr int TOPK_THREADS = 1024;
constexpr int KM = CP_MAX_K;
// cells of a heat map whose sigmoid and NMS-ed copies both fit the kernel's shared memory (200 KB of 8 bytes per cell)
constexpr size_t TOPK_SMEM_CELLS = 200 * 1024 / 8;

__host__ __device__ __forceinline__ bool topk_staged(size_t hw) { return hw <= TOPK_SMEM_CELLS; }

__device__ __forceinline__ float sigmoid_acc(float x) { return 1.0f / (1.0f + expf(-x)); }

// ---------------------------------------------------------------------------
// kernel 1: per-channel sigmoid + NMS + top-K
// STAGED: the sigmoid map (raw) and the NMS-ed map (nv) live in shared memory (topk_staged).  Otherwise the NMS reads
// the map from global memory, recomputing the sigmoid of each neighbour, and nv is this channel's slice of nv_ws
// ([B][C_hm + J][HW] floats of the workspace); the values and the selection are the same.
// ---------------------------------------------------------------------------
template <bool STAGED>
__global__ void __launch_bounds__(TOPK_THREADS, 1)
peaks_topk_kernel(const float* __restrict__ hm, const float* __restrict__ hm_hp, int C_hm, int J, int H, int W,
                  int K, int apply_sigmoid, float* __restrict__ peak_val, int* __restrict__ peak_idx,
                  float* __restrict__ nv_ws) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int HW = H * W;
  float* raw = reinterpret_cast<float*>(smem_raw);
  __shared__ unsigned int hist[256];
  __shared__ unsigned int s_prefix, s_need, s_cnt;
  __shared__ int warp_tot[TOPK_THREADS / 32];
  __shared__ unsigned long long keys[KM];

  const int ch = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int CH = C_hm + J;
  const float* src = (ch < C_hm) ? hm + ((size_t)b * C_hm + ch) * HW : hm_hp + ((size_t)b * J + (ch - C_hm)) * HW;

  // apply_sigmoid: 0 = both maps are probabilities already, 1 = both are logits, 2 = only hm is a logit
  // (opt.mse_loss: the reference skips the hm_hp sigmoid, object_pose.py:136-138)
  const bool sig = (ch < C_hm) ? (apply_sigmoid != 0) : (apply_sigmoid == 1);
  float* nv = STAGED ? raw + HW : nv_ws + ((size_t)b * CH + ch) * HW;
  auto heat = [&](int i) -> float {
    if (STAGED) return raw[i];
    const float v = __ldg(src + i);
    return sig ? sigmoid_acc(v) : v;
  };
  if (STAGED) {
    for (int i = tid; i < HW; i += TOPK_THREADS) {
      float v = __ldg(src + i);
      raw[i] = sig ? sigmoid_acc(v) : v;
    }
    __syncthreads();
  }
  // 3x3 max-pool (stride 1, -inf padding) equality NMS: keep = (hmax == heat)
  for (int i = tid; i < HW; i += TOPK_THREADS) {
    int y = i / W, x = i - y * W;
    float v = heat(i);
    float m = v;
    for (int dy = -1; dy <= 1; ++dy) {
      int yy = y + dy;
      if (yy < 0 || yy >= H) continue;
      for (int dx = -1; dx <= 1; ++dx) {
        int xx = x + dx;
        if (xx < 0 || xx >= W) continue;
        m = fmaxf(m, heat(yy * W + xx));
      }
    }
    nv[i] = (m == v) ? v + 0.0f : 0.0f;      // heat * keep; -0 is canonicalised (torch.topk compares it equal to +0)
  }
  if (tid == 0) {
    s_prefix = 0;
    s_need = K;
    s_cnt = 0;
  }
  __syncthreads();

  // radix select of the K-th largest value on order-preserving keys: positive floats get the sign bit set, negative
  // floats are bit-inverted, so the unsigned order of the keys is the float order for raw (un-sigmoided, possibly
  // negative) maps too
  auto ord = [](float f) -> unsigned int {
    const unsigned int b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
  };
  auto unord = [](unsigned int k) -> float { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); };
  unsigned int mask = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += TOPK_THREADS) hist[i] = 0;
    __syncthreads();
    const unsigned int prefix = s_prefix;
    for (int i = tid; i < HW; i += TOPK_THREADS) {
      unsigned int bits = ord(nv[i]);
      if ((bits & mask) == prefix) atomicAdd(&hist[(bits >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      unsigned int need = s_need, cum = 0;
      int d = 255;
      for (; d > 0; --d) {
        if (cum + hist[d] >= need) break;
        cum += hist[d];
      }
      s_need = need - cum;
      s_prefix = prefix | ((unsigned int)d << shift);
    }
    mask |= 255u << shift;
    __syncthreads();
  }
  const unsigned int T = s_prefix;      // bit pattern of the K-th largest value
  const unsigned int need = s_need;     // how many elements equal to T are selected (lowest indices first)
  const unsigned int n_gt = K - need;

  for (int i = tid; i < KM; i += TOPK_THREADS) keys[i] = 0ull;
  __syncthreads();
  // strictly greater: unordered compaction
  for (int i = tid; i < HW; i += TOPK_THREADS) {
    unsigned int bits = ord(nv[i]);
    if (bits > T) {
      unsigned int pos = atomicAdd(&s_cnt, 1u);
      keys[pos] = ((unsigned long long)bits << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned int)i);
    }
  }
  // ties: ordered by index -> contiguous chunk per thread + block scan
  const int per = (HW + TOPK_THREADS - 1) / TOPK_THREADS;
  const int i0 = tid * per, i1 = min(HW, i0 + per);
  int mine = 0;
  for (int i = i0; i < i1; ++i) mine += (ord(nv[i]) == T);
  int incl = mine;
  const int lane = tid & 31, wid = tid >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    int v = warp_tot[lane];
    int s = v;
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += t;
    }
    warp_tot[lane] = s - v;  // exclusive
  }
  __syncthreads();
  int rank = warp_tot[wid] + incl - mine;
  for (int i = i0; i < i1 && rank < (int)need; ++i) {
    if (ord(nv[i]) == T) {
      keys[n_gt + rank] = ((unsigned long long)T << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned int)i);
      ++rank;
    }
  }
  __syncthreads();
  // bitonic sort of KM keys, descending (value desc, index asc)
  for (int k2 = 2; k2 <= KM; k2 <<= 1) {
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      if (tid < KM) {
        int ixj = tid ^ j;
        if (ixj > tid) {
          unsigned long long a = keys[tid], c = keys[ixj];
          bool desc = ((tid & k2) == 0);
          if ((a < c) == desc) {
            keys[tid] = c;
            keys[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  if (tid < K) {
    unsigned long long kk = keys[tid];
    peak_val[((size_t)b * CH + ch) * K + tid] = unord((unsigned int)(kk >> 32));
    peak_idx[((size_t)b * CH + ch) * K + tid] = (int)(0xFFFFFFFFu - (unsigned int)(kk & 0xFFFFFFFFull));
  }
}

// ---------------------------------------------------------------------------
// kernel 2: grouping + post-process + soft-NMS + PnP
// ---------------------------------------------------------------------------
struct GroupArgs {
  cp_decode_params prm;
  cp_heads h;
  const double* meta;
  const float* peak_val;
  const int* peak_idx;
  float* dets;    // [B,K,CP_DETS_RECORD] (user buffer or workspace)
  float* poses;   // [B,K,CP_POSE_RECORD]
  int* n_valid;
  // several models' heads in one launch (cp_infer_multi): image b is frame b % ipm of model b / ipm, which decodes
  // with that model's visible_thresh and balance; the meta rows are the frames'
  int ipm;
  int visible_thresh[CP_MAX_MODELS];
  float balance[CP_MAX_MODELS];
};

__device__ __forceinline__ float gatherf(const float* base, int b, int C, int c, int HW, int ind) {
  return __ldg(base + ((size_t)b * C + c) * HW + ind);
}

// python slice start:stop on a length-n axis
__device__ __forceinline__ void py_slice(int start, int stop, int n, int* s0, int* s1) {
  if (start < 0) start += n;
  if (stop < 0) stop += n;
  start = max(0, min(start, n));
  stop = max(0, min(stop, n));
  *s0 = start;
  *s1 = max(start, stop);
}

__global__ void __launch_bounds__(256, 1) group_pose_kernel(const GroupArgs a) {
  const cp_decode_params& P = a.prm;
  const int b = blockIdx.x, tid = threadIdx.x, NT = blockDim.x;
  const int K = P.K, J = P.num_joints, H = P.out_h, W = P.out_w, HW = H * W;
  const int CH = P.num_classes + J;
  const float th = 0.1f;

  __shared__ float c_score[KM];
  __shared__ float c_bbox[KM][4];
  __shared__ float c_disp[KM][16];
  __shared__ float hmx[8][KM], hmy[8][KM], hms[8][KM];
  __shared__ double nb_bbox[KM][4];
  __shared__ double nb_score[KM];
  __shared__ int nb_perm[KM];
  __shared__ int c_src[KM];       // candidate k of the image = entry (c_src / K, c_src % K) of the per-class top-K lists
  __shared__ int s_n0, s_n1;

  float* dets = a.dets + (size_t)b * K * CP_DETS_RECORD;
  float* poses = a.poses + (size_t)b * K * CP_POSE_RECORD;
  const double* meta = a.meta + (size_t)(b % a.ipm) * CP_META_DOUBLES;
  const int model = b / a.ipm;

  // ---------------- decode.py:52-68 _topk: the K best of the num_classes x K per-class candidates.  Every per-class list
  // is sorted (value descending, index ascending), so the rank of a candidate in the merged order (value descending,
  // flat index class * K + k ascending) is a sum of binary searches; ranks are distinct, the first K fill c_src.
  if (P.num_classes == 1) {
    for (int k = tid; k < K; k += NT) c_src[k] = k;
  } else {
    const float* pv = a.peak_val + (size_t)b * CH * K;
    for (int f = tid; f < P.num_classes * K; f += NT) {
      const int c = f / K, kk = f - c * K;
      const float v = pv[f];
      int rank = 0;
      for (int c2 = 0; c2 < P.num_classes; ++c2) {
        const float* l = pv + (size_t)c2 * K;
        int lo = 0, hi = K;                   // number of entries of list c2 that are > v
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (l[mid] > v) lo = mid + 1; else hi = mid;
        }
        rank += lo;
        if (c2 < c) {                         // equal values of an earlier class come first
          int lo2 = lo, hi2 = K;
          while (lo2 < hi2) {
            const int mid = (lo2 + hi2) >> 1;
            if (l[mid] >= v) lo2 = mid + 1; else hi2 = mid;
          }
          rank += lo2 - lo;
        } else if (c2 == c) {
          rank += kk - lo;                    // equal values of the own class with a lower index
        }
      }
      if (rank < K) c_src[rank] = f;
    }
  }
  __syncthreads();
  // ---------------- phase A: centres (decode.py:83-109, 304-345)
  for (int k = tid; k < K; k += NT) {
    const int src = c_src[k];
    const int ind = a.peak_idx[(size_t)b * CH * K + src];
    const float score = a.peak_val[(size_t)b * CH * K + src];
    const float xs = (float)(ind % W), ys = (float)(ind / W);
    float* d = dets + (size_t)k * CP_DETS_RECORD;
    c_score[k] = score;
    for (int j = 0; j < 2 * J; ++j) {
      float v = gatherf(a.h.hps, b, 2 * J, j, HW, ind) + ((j & 1) ? ys : xs);
      c_disp[k][j] = v;
      d[CP_D_KPS_DISP_MEAN + j] = v;
    }
    float cx, cy;
    if (a.h.reg) {
      cx = xs + gatherf(a.h.reg, b, 2, 0, HW, ind);
      cy = ys + gatherf(a.h.reg, b, 2, 1, HW, ind);
    } else {
      cx = xs + 0.5f;
      cy = ys + 0.5f;
    }
    float w = gatherf(a.h.wh, b, 2, 0, HW, ind), hgt = gatherf(a.h.wh, b, 2, 1, HW, ind);
    float bb[4] = {cx - w / 2.0f, cy - hgt / 2.0f, cx + w / 2.0f, cy + hgt / 2.0f};
    for (int t = 0; t < 4; ++t) {
      c_bbox[k][t] = bb[t];
      d[CP_D_BBOX + t] = bb[t];
    }
    d[CP_D_SCORE] = score;
    d[CP_D_CLS] = (float)(src / K);
    d[CP_D_IND] = (float)ind;
    for (int t = 0; t < 3; ++t) {
      d[CP_D_OBJ_SCALE + t] = a.h.scale ? gatherf(a.h.scale, b, 3, t, HW, ind) : 0.0f;
      d[CP_D_OBJ_SCALE_UNC + t] =
          a.h.scale_uncertainty ? sqrtf(expf(gatherf(a.h.scale_uncertainty, b, 3, t, HW, ind))) : 0.0f;
    }
    for (int t = 0; t < 2; ++t) d[CP_D_TRACKING + t] = a.h.tracking ? gatherf(a.h.tracking, b, 2, t, HW, ind) : 0.0f;
    for (int t = 0; t < 2 * J; ++t) {
      d[CP_D_TRACKING_HP + t] = a.h.tracking_hp ? gatherf(a.h.tracking_hp, b, 2 * J, t, HW, ind) : 0.0f;
      d[CP_D_KPS_DISP_STD + t] =
          a.h.hps_uncertainty ? sqrtf(expf(gatherf(a.h.hps_uncertainty, b, 2 * J, t, HW, ind))) * a.balance[model] : 0.0f;
    }
  }
  // ---------------- phase B: per-joint heat-map peaks (decode.py:129-144)
  for (int i = tid; i < J * K; i += NT) {
    const int j = i / K, m = i - j * K;
    const int ind = a.peak_idx[((size_t)b * CH + P.num_classes + j) * K + m];
    float s = a.peak_val[((size_t)b * CH + P.num_classes + j) * K + m];
    float x = (float)(ind % W), y = (float)(ind / W);
    if (a.h.hp_offset) {
      x += gatherf(a.h.hp_offset, b, 2, 0, HW, ind);
      y += gatherf(a.h.hp_offset, b, 2, 1, HW, ind);
    } else {
      x += 0.5f;
      y += 0.5f;
    }
    if (!(s > th)) {
      s = -1.0f;
      x = SENT;
      y = SENT;
    }
    hmx[j][m] = x;
    hmy[j][m] = y;
    hms[j][m] = s;
  }
  __syncthreads();

  // ---------------- phase C: nearest peak per (centre, joint) and the gates (decode.py:147-252)
  for (int i = tid; i < K * J; i += NT) {
    const int k = i / J, j = i - k * J;
    const float rx = c_disp[k][2 * j], ry = c_disp[k][2 * j + 1];
    float best = INFINITY;
    int bi = 0;
    for (int m = 0; m < K; ++m) {
      float dx = rx - hmx[j][m], dy = ry - hmy[j][m];
      float dd = sqrtf(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
      if (dd < best) {
        best = dd;
        bi = m;
      }
    }
    const float sx = hmx[j][bi], sy = hmy[j][bi], ss = hms[j][bi];
    const float l = c_bbox[k][0], t = c_bbox[k][1], r = c_bbox[k][2], bt = c_bbox[k][3];
    const float size = fmaxf(bt - t, r - l);
    const bool bad = (sx < l) || (sx > r) || (sy < t) || (sy > bt) || (ss < th) || (best > __fmul_rn(size, 0.3f));
    float kx = rx, ky = ry;
    if (P.rep_mode == 4) {
      kx = sx;
      ky = sy;
    } else if (P.rep_mode != 3 && !bad) {
      kx = sx;
      ky = sy;
    }
    float* d = dets + (size_t)k * CP_DETS_RECORD;
    d[CP_D_KPS + 2 * j] = kx;
    d[CP_D_KPS + 2 * j + 1] = ky;
    const bool ok2 = (sx > __fmul_rn(0.8f, l)) && (sx < __fmul_rn(1.2f, r)) && (sy > __fmul_rn(0.8f, t)) &&
                     (sy < __fmul_rn(1.2f, bt)) && (ss > th) && (best < __fmul_rn(size, 0.5f)) && (c_score[k] > th) &&
                     !P.modern_bool_semantics;      // torch >= 1.2: `mask_2 == 7` on a bool sum is never true
    float mean_x = SENT, mean_y = SENT, std_x = SENT, std_y = SENT, height = SENT;
    if ((P.rep_mode == 1 || P.rep_mode == 2) && ok2 && !(sx == SENT || sy == SENT)) {
      const float* hp = a.h.hm_hp + ((size_t)b * J + j) * HW;
      if (P.use_moments) {
        const int ran = 5;
        int r0, r1, q0, q1;
        py_slice((int)sy, (int)(sy + (float)(2 * ran + 1)), H + 2 * ran, &r0, &r1);
        py_slice((int)sx, (int)(sx + (float)(2 * ran + 1)), W + 2 * ran, &q0, &q1);
        const int nr = r1 - r0, nc = q1 - q0;
        double win[121];
        for (int rr = 0; rr < nr; ++rr)
          for (int cc = 0; cc < nc; ++cc) {
            int yy = r0 + rr - ran, xx = q0 + cc - ran;
            double v = 0.0;
            if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
              float raw = __ldg(hp + yy * W + xx);
              v = (double)(P.apply_sigmoid == 1 ? sigmoid_acc(raw) : raw);
            }
            win[rr * nc + cc] = v;
          }
        double hh, mx, my, wx, wy;
        if (pose::moments(win, nr, nc, &hh, &mx, &my, &wx, &wy)) {
          if (wx == 0.0) wx = 1e-10;   // least_squares(max_nfev=1) returns a strictly feasible start point
          if (wy == 0.0) wy = 1e-10;
          mean_x = (float)((double)sx + mx - (double)ran);
          mean_y = (float)((double)sy + my - (double)ran);
          std_x = (float)wx;
          std_y = (float)wy;
          height = (float)hh;
        }
      } else {
        int iy = (int)sy, ix = (int)sx;
        if (iy < 0) iy += H;
        if (ix < 0) ix += W;
        if (iy >= 0 && iy < H && ix >= 0 && ix < W) {   // the reference raises IndexError outside
          float raw = __ldg(hp + iy * W + ix);
          height = P.apply_sigmoid == 1 ? sigmoid_acc(raw) : raw;
          mean_x = sx;
          mean_y = sy;
          std_x = 1.0f;
          std_y = 1.0f;
        }
      }
    }
    d[CP_D_KPS_HM_MEAN + 2 * j] = mean_x;
    d[CP_D_KPS_HM_MEAN + 2 * j + 1] = mean_y;
    d[CP_D_KPS_HM_STD + 2 * j] = std_x;
    d[CP_D_KPS_HM_STD + 2 * j + 1] = std_y;
    d[CP_D_KPS_HM_HEIGHT + j] = height;
  }
  __syncthreads();

  // ---------------- output-map -> image affine (image.py:35-68 with rot = 0, float32 control points)
  const float cxf = (float)meta[0], cyf = (float)meta[1], swf = (float)meta[2];
  const float dwf = (float)W, dhf = (float)H;
  const float d0x = dwf * 0.5f, d0y = dhf * 0.5f;
  const float d1y = d0y + dwf * -0.5f;
  const float s1y = cyf + swf * -0.5f;
  const double aff = ((double)cyf - (double)s1y) / ((double)d0y - (double)d1y);
  const double tx = (double)cxf - aff * (double)d0x, ty = (double)cyf - aff * (double)d0y;
  const float ratio = (float)(meta[2] / (double)max(W, H));   // s / max(w, h), rounded once to float32
  const double img_w = meta[3], img_h = meta[4];
  // multi-scale testing (object_pose.py:171-177): the image-space coordinates of a scale != 1 pass are divided by the
  // scale as float32 values, `(np.array(v, np.float32) / scale).tolist()`, before merge_outputs / the PnP see them
  const float tsc = P.test_scale > 0.0f ? P.test_scale : 1.0f;      // 0 (a zero-initialised struct) means 1
  const bool rescale = tsc != 1.0f;
  auto unscale = [&](double v) -> double { return rescale ? (double)__fdiv_rn((float)v, tsc) : v; };

  // ---------------- phase D: score filter (object_pose.py:188-191); scores are sorted descending
  if (tid == 0) {
    int n0 = 0;
    while (n0 < K && c_score[n0] > P.vis_thresh) ++n0;
    s_n0 = n0;
  }
  __syncthreads();
  const int n0 = s_n0;
  for (int i = tid; i < n0; i += NT) {
    for (int p = 0; p < 2; ++p) {
      float x = c_bbox[i][2 * p], y = c_bbox[i][2 * p + 1];
      if (x == SENT && y == SENT) {
        nb_bbox[i][2 * p] = unscale(-10000.0);
        nb_bbox[i][2 * p + 1] = unscale(-10000.0);
      } else {
        nb_bbox[i][2 * p] = unscale(aff * (double)x + tx);
        nb_bbox[i][2 * p + 1] = unscale(aff * (double)y + ty);
      }
    }
    nb_score[i] = (double)c_score[i];
    nb_perm[i] = i;
  }
  __syncthreads();
  // ---------------- phase E: Gaussian soft-NMS (sequential by definition)
  if (tid == 0) {
    int n1 = n0;
    if ((P.nms || P.num_scales > 1) && n0 > 0) n1 = pose::soft_nms(&nb_bbox[0][0], nb_score, nb_perm, n0, (double)P.vis_thresh);
    s_n1 = n1;
    a.n_valid[b] = n1;
  }
  __syncthreads();
  const int n1 = s_n1;

  // ---------------- phase F: records, one thread per surviving detection
  for (int i = tid; i < n1; i += NT) {
    const int k = nb_perm[i];
    const float* d = dets + (size_t)k * CP_DETS_RECORD;
    float* o = poses + (size_t)i * CP_POSE_RECORD;
    o[CP_P_SCORE] = (float)nb_score[i];
    o[CP_P_CLS] = d[CP_D_CLS];
    o[CP_P_SRC_INDEX] = (float)k;
    for (int t = 0; t < 4; ++t) o[CP_P_BBOX + t] = (float)nb_bbox[i][t];
    if (!rescale) {
      o[CP_P_CT] = (float)((nb_bbox[i][0] + nb_bbox[i][2]) / 2.0);
      o[CP_P_CT + 1] = (float)((nb_bbox[i][1] + nb_bbox[i][3]) / 2.0);
    } else {      // post_process.py:40 computes `ct` from the bbox BEFORE object_pose.py:171-177 divides the bbox
      double ub[4];
      for (int p = 0; p < 2; ++p) {
        const float x = c_bbox[k][2 * p], y = c_bbox[k][2 * p + 1];
        const bool sent = (x == SENT && y == SENT);
        ub[2 * p] = sent ? -10000.0 : aff * (double)x + tx;
        ub[2 * p + 1] = sent ? -10000.0 : aff * (double)y + ty;
      }
      o[CP_P_CT] = (float)((ub[0] + ub[2]) / 2.0);
      o[CP_P_CT + 1] = (float)((ub[1] + ub[3]) / 2.0);
    }
    double kps[16], dmean[16], hmean[16];
    for (int j = 0; j < J; ++j) {
      const int offs[3] = {CP_D_KPS, CP_D_KPS_DISP_MEAN, CP_D_KPS_HM_MEAN};
      double* dst[3] = {kps, dmean, hmean};
      for (int q = 0; q < 3; ++q) {
        float x = d[offs[q] + 2 * j], y = d[offs[q] + 2 * j + 1];
        if (x == SENT && y == SENT) {
          dst[q][2 * j] = unscale(-10000.0);
          dst[q][2 * j + 1] = unscale(-10000.0);
        } else {
          dst[q][2 * j] = unscale(aff * (double)x + tx);
          dst[q][2 * j + 1] = unscale(aff * (double)y + ty);
        }
      }
    }
    for (int t = 0; t < 2 * J; ++t) {
      o[CP_P_KPS + t] = (float)kps[t];
      o[CP_P_KPS_DISP_MEAN + t] = (float)dmean[t];
      o[CP_P_KPS_HM_MEAN + t] = (float)hmean[t];
      o[CP_P_KPS_HM_STD + t] = __fmul_rn(__fmul_rn(d[CP_D_KPS_HM_STD + t], ratio), 0.32f);
      o[CP_P_KPS_DISP_STD + t] = __fmul_rn(__fmul_rn(d[CP_D_KPS_DISP_STD + t], ratio), 0.32f);
      o[CP_P_TRACKING_HP + t] = __fmul_rn(d[CP_D_TRACKING_HP + t], ratio);
      if (rescale) {
        o[CP_P_KPS_DISP_STD + t] = __fdiv_rn(o[CP_P_KPS_DISP_STD + t], tsc);
        o[CP_P_TRACKING_HP + t] = __fdiv_rn(o[CP_P_TRACKING_HP + t], tsc);
      }
    }
    for (int t = 0; t < J; ++t) o[CP_P_KPS_HM_HEIGHT + t] = d[CP_D_KPS_HM_HEIGHT + t];
    for (int t = 0; t < 3; ++t) {
      o[CP_P_OBJ_SCALE + t] = d[CP_D_OBJ_SCALE + t];
      o[CP_P_OBJ_SCALE_UNC + t] = d[CP_D_OBJ_SCALE_UNC + t];
    }
    for (int t = 0; t < 2; ++t) {
      o[CP_P_TRACKING + t] = __fmul_rn(d[CP_D_TRACKING + t], ratio);
      if (rescale) o[CP_P_TRACKING + t] = __fdiv_rn(o[CP_P_TRACKING + t], tsc);
    }
  }
  // ---------------- phase G: PnP, one WARP per surviving detection
  {
    extern __shared__ double pnp_scratch[];
    const int warp = tid >> 5, lane = tid & 31, NW = NT >> 5;
    double* sm = pnp_scratch + warp * PNP_SCRATCH;
    double* pts = sm + 288;
    for (int i = warp; i < n1; i += NW) {
      const int k = nb_perm[i];
      const float* d = dets + (size_t)k * CP_DETS_RECORD;
      float* o = poses + (size_t)i * CP_POSE_RECORD;
      pose::PnPOut po;
      po.status = CP_PNP_NOT_RUN;
      po.n_pts = 0;
      if (P.use_pnp) {
        const int n_in = (P.rep_mode == 1) ? 16 : 8;
        __syncwarp();
        if (lane < n_in) {
          // rep_mode 1: point 2j = displacement mean of joint j, point 2j+1 = heat-map mean; else point j = kps[j]
          const int j = (P.rep_mode == 1) ? (lane >> 1) : lane;
          const int off = (P.rep_mode == 1) ? ((lane & 1) ? CP_D_KPS_HM_MEAN : CP_D_KPS_DISP_MEAN) : CP_D_KPS;
          const float x = d[off + 2 * j], y = d[off + 2 * j + 1];
          double X0 = -10000.0, Y0 = -10000.0;
          if (!(x == SENT && y == SENT)) {
            X0 = aff * (double)x + tx;
            Y0 = aff * (double)y + ty;
          }
          pts[2 * lane] = unscale(X0);
          pts[2 * lane + 1] = unscale(Y0);
        }
        __syncwarp();
        float sc[3] = {d[CP_D_OBJ_SCALE], d[CP_D_OBJ_SCALE + 1], d[CP_D_OBJ_SCALE + 2]};
        solve_and_shell_warp(pts, n_in, sc, meta + 5, img_w, img_h, a.visible_thresh[model], P.opencv_return, &po, sm, lane);
      }
      if (lane == 0) {
        o[CP_P_STATUS] = (float)po.status;
        o[CP_P_NPTS] = (float)po.n_pts;
        const bool has_pose = (po.status == CP_PNP_OK || po.status == CP_PNP_INVISIBLE);
        const bool has_proj = has_pose || po.status == CP_PNP_BEHIND;
        for (int t = 0; t < 3; ++t) o[CP_P_LOCATION + t] = has_pose ? (float)po.loc[t] : 0.0f;
        for (int t = 0; t < 4; ++t) o[CP_P_QUAT + t] = has_pose ? (float)po.quat[t] : 0.0f;
        o[CP_P_REPROJ] = has_proj ? (float)po.reproj : 0.0f;
        for (int t = 0; t < 16; ++t) o[CP_P_PROJ_CUBOID + t] = has_proj ? (float)po.proj[t] : 0.0f;
        for (int t = 0; t < 27; ++t) o[CP_P_KPS_3D_CAM + t] = has_pose ? (float)po.kps3d[t] : 0.0f;
        for (int t = 0; t < 18; ++t) o[CP_P_KPS_PNP + t] = has_pose ? (float)po.kpspnp[t] : 0.0f;
      }
      __syncwarp();
    }
  }
  // zero the unused slots so the all-gathered tensor is deterministic
  for (int i = n1 * CP_POSE_RECORD + tid; i < K * CP_POSE_RECORD; i += NT) poses[i] = 0.0f;
}

struct WsLayout {
  size_t peak_val, peak_idx, dets, nv, total;
};

WsLayout ws_layout(const cp_decode_params* p) {
  WsLayout w;
  size_t n = (size_t)p->batch * (p->num_classes + p->num_joints) * p->K;
  size_t off = 0;
  w.peak_val = off;
  off += (n * sizeof(float) + 255) / 256 * 256;
  w.peak_idx = off;
  off += (n * sizeof(int) + 255) / 256 * 256;
  w.dets = off;
  off += ((size_t)p->batch * p->K * CP_DETS_RECORD * sizeof(float) + 255) / 256 * 256;
  w.nv = off;        // the NMS-ed maps of peaks_topk_kernel when they do not fit its shared memory
  const size_t hw = (size_t)p->out_h * p->out_w;
  if (!topk_staged(hw)) off += ((size_t)p->batch * (p->num_classes + p->num_joints) * hw * sizeof(float) + 255) / 256 * 256;
  w.total = off;
  return w;
}

int validate(const cp_decode_params* p) {
  if (!p) return fail(CP_ERR_INVALID, "decode: null params");
  if (p->batch <= 0 || p->out_h <= 0 || p->out_w <= 0) return fail(CP_ERR_INVALID, "decode: bad shape");
  if (p->num_classes < 1 || p->num_classes > CP_MAX_CLASSES)
    return fail(CP_ERR_INVALID, "decode: num_classes must be in 1..CP_MAX_CLASSES");
  if (!(p->test_scale >= 0.0f)) return fail(CP_ERR_INVALID, "decode: test_scale must be > 0 (0 or 1: single-scale testing)");
  if (p->num_joints != 8) return fail(CP_ERR_INVALID, "decode: num_joints must be 8");
  if (p->K <= 0 || p->K > CP_MAX_K) return fail(CP_ERR_INVALID, "decode: K must be in 1..128");
  if ((size_t)p->out_h * p->out_w < (size_t)p->K) return fail(CP_ERR_INVALID, "decode: map smaller than K");
  if ((size_t)p->out_h * p->out_w >= (1u << 30)) return fail(CP_ERR_INVALID, "decode: head map too large");
  if (p->rep_mode == 2)
    return fail(CP_ERR_INVALID, "decode: rep_mode 2 (random GMM sampling, base_detector.py:568-650) is not supported");
  if (p->rep_mode < 0 || p->rep_mode > 4) return fail(CP_ERR_INVALID, "decode: rep_mode must be 0, 1, 3 or 4");
  return CP_OK;
}

}  // namespace
}  // namespace cp

using namespace cp;

extern "C" {

size_t cp_decode_workspace_bytes(const cp_decode_params* prm) {
  if (validate(prm)) return 0;
  return ws_layout(prm).total;
}

int cp_decode_pnp(const cp_decode_params* prm, const cp_heads* heads, const double* meta, float* dets, float* poses,
                  int32_t* n_valid, void* workspace, size_t workspace_bytes, void* stream_) {
  return cp::decode_pnp_models(prm, 1, heads, meta, dets, poses, n_valid, workspace, workspace_bytes, stream_);
}

}  // extern "C"

namespace cp {

// prm[0 .. models): prm[0].batch = models x frames; prm[m] gives model m its visible_thresh and balance
int decode_pnp_models(const cp_decode_params* prm, int models, const cp_heads* heads, const double* meta, float* dets,
                      float* poses, int32_t* n_valid, void* workspace, size_t workspace_bytes, void* stream_) {
  int rc = validate(prm);
  if (rc) return rc;
  if (models < 1 || models > CP_MAX_MODELS || prm->batch % models)
    return fail(CP_ERR_INVALID, "cp_decode_pnp: batch is not a whole number of models");
  if (!heads || !meta || !poses || !n_valid || !workspace) return fail(CP_ERR_INVALID, "cp_decode_pnp: null argument");
  if (!heads->hm || !heads->wh || !heads->hps || !heads->hm_hp)
    return fail(CP_ERR_INVALID, "cp_decode_pnp: hm, wh, hps and hm_hp heads are required");
  if (prm->use_pnp && !heads->scale) return fail(CP_ERR_INVALID, "cp_decode_pnp: PnP needs the scale head");
  WsLayout w = ws_layout(prm);
  if (workspace_bytes < w.total) return fail(CP_ERR_INVALID, "cp_decode_pnp: workspace too small");
  cudaStream_t s = (cudaStream_t)stream_;
  char* ws = (char*)workspace;
  float* peak_val = (float*)(ws + w.peak_val);
  int* peak_idx = (int*)(ws + w.peak_idx);
  float* dets_buf = dets ? dets : (float*)(ws + w.dets);

  const int HW = prm->out_h * prm->out_w;
  dim3 g1(prm->num_classes + prm->num_joints, prm->batch);
  if (topk_staged(HW)) {
    const size_t smem = (size_t)HW * 2 * sizeof(float);
    static cp::PerDevice<size_t> configured;
    if (smem > configured.here()) {
      CP_CUDA_CHECK(cudaFuncSetAttribute(peaks_topk_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      configured.here() = smem;
    }
    peaks_topk_kernel<true><<<g1, TOPK_THREADS, smem, s>>>(heads->hm, heads->hm_hp, prm->num_classes, prm->num_joints,
                                                           prm->out_h, prm->out_w, prm->K, prm->apply_sigmoid, peak_val,
                                                           peak_idx, nullptr);
  } else {
    peaks_topk_kernel<false><<<g1, TOPK_THREADS, 0, s>>>(heads->hm, heads->hm_hp, prm->num_classes, prm->num_joints,
                                                         prm->out_h, prm->out_w, prm->K, prm->apply_sigmoid, peak_val,
                                                         peak_idx, (float*)(ws + w.nv));
  }
  CP_LAUNCH_CHECK("peaks_topk_kernel");
  GroupArgs ga;
  ga.prm = *prm;
  ga.h = *heads;
  ga.meta = meta;
  ga.peak_val = peak_val;
  ga.peak_idx = peak_idx;
  ga.dets = dets_buf;
  ga.poses = poses;
  ga.n_valid = n_valid;
  ga.ipm = prm->batch / models;
  for (int m = 0; m < models; ++m) {
    ga.visible_thresh[m] = prm[m].visible_thresh;
    ga.balance[m] = prm[m].balance;
  }
  static cp::PerDevice<bool> pose_configured;
  if (!pose_configured.here()) {      // static (~29 KB) + dynamic (20 KB) shared memory crosses the 48 KB default
    CP_CUDA_CHECK(cudaFuncSetAttribute(group_pose_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    pose_configured.here() = true;
  }
  group_pose_kernel<<<prm->batch, 256, 8 * PNP_SCRATCH * sizeof(double), s>>>(ga);
  CP_LAUNCH_CHECK("group_pose_kernel");
  return CP_OK;
}

}  // namespace cp

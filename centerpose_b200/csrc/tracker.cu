// CenterPoseTrack state on the device: Tracker.step (association, 32-state Kalman filter per object as eight 4-state
// filters, scale pool, second PnP with the filtered keypoints) and the rendering of the previous-frame heat maps.
// The logic is track_core.h (host-tested against the unmodified reference tracker, tests/test_track_core_host.py); this
// file is its parallel orchestration: one CTA per video stream.
//
// Reference (relative to /root/reference/src/lib): utils/tracker.py:15-302, detectors/base_detector.py:150-388
// (_get_additional_inputs), :502-544 (gaussian_fusion), :660-665 (tracker.step in run()).
#include <string.h>

#include <new>

#include "common.cuh"
#include "pnp_warp.cuh"
#include "track_core.h"

using namespace cp;
using namespace cp::track;

namespace cp {
namespace {
// The per-category settings of a tracker of several categories (cp_tracker_create_multi): stream s belongs to category
// s / S and uses its visible_thresh (second PnP) and conf_border (keypoint-confidence gain).  Passed by value to the
// step and render kernels; a one-category tracker has one row.
struct CatCfg {
  int S;                                   // streams per category
  int visible_thresh[CP_MAX_MODELS];
  double conf_lo[CP_MAX_MODELS], conf_hi[CP_MAX_MODELS];
};
}  // namespace
}  // namespace cp

struct cp_tracker {
  cp_tracker_config cfg;                    // cfg.streams: every category's streams (models x streams per category)
  CatCfg cat;
  Slot* slots[2] = {nullptr, nullptr};      // [streams][max_tracks], ping-pong: slots[cur[s]] = current tracks of s
  int* n_tracks[2] = {nullptr, nullptr};    // [streams]
  int* cur = nullptr;                       // [streams] current buffer of each stream, flipped by the step kernel
  int* id_count = nullptr;                  // [streams]
  int* modes = nullptr;                     // [streams] render modes of the latest cp_tracker_render_ex
  int* ids = nullptr;                       // [streams] stream map of the latest _ex call (batch row -> stream)
  void* plan = nullptr;                     // hungarian: [streams][max_tracks] Entry of the association kernel
  int* plan_n = nullptr;                    // hungarian: [streams]
};

namespace cp {
namespace {

constexpr int TRK_THREADS = 256;
constexpr int TRK_MAXK = CP_MAX_K;

struct StepArgs {
  Cfg cfg;
  CatCfg cat;
  int opencv_return, T, K;
  const float* poses;       // [B, K, 192]
  const int* n_valid;       // [B]
  const double* meta;       // [B, 16]
  Slot* slots0;             // [streams, T] the two buffers of the track state
  Slot* slots1;
  int* n0;                  // [streams]
  int* n1;
  int* cur;                 // [streams] which buffer is current
  const int* ids;           // [B] tracker stream of each batch row, or nullptr: the identity
  int* id_count;            // [streams]
  float* tracks_out;        // [B, T, 320]
  int* n_out;               // [B]
  Entry* plan;              // hungarian: [B, T] entries written by tracker_assoc_kernel, else nullptr
  int* plan_n;              // hungarian: [B]
};

// the Dijkstra scan of lsa_solve spread over the CTA: thread t relaxes column remaining[t] (nc <= CP_MAX_K <=
// TRK_THREADS) and the serial scan's choice becomes a reduction over (value, key): the smaller value wins, equal values
// go to the larger key, key = 256 + t for an unassigned column (the last one of the scan wins) and 255 - t otherwise
// (the first one wins), so the same column is picked as by the left-to-right scan of lsa_solve.
// the state a batch row reads and writes: row b is tracker stream s = ids[b]; its current tracks are buffer cur[s]
struct StreamState {
  int s, c;
  const Slot* old;
  Slot* nxt;
  int* new_n;
  int M;
};

__device__ __forceinline__ StreamState stream_state(const StepArgs& a, int b) {
  StreamState st;
  st.s = a.ids ? a.ids[b] : b;
  st.c = a.cur[st.s];
  const size_t off = (size_t)st.s * a.T;
  st.old = (st.c ? a.slots1 : a.slots0) + off;
  st.nxt = (st.c ? a.slots0 : a.slots1) + off;
  st.M = (st.c ? a.n1 : a.n0)[st.s];
  st.new_n = (st.c ? a.n0 : a.n1) + st.s;
  return st;
}

struct LsaSync {
  double val[TRK_THREADS / 32];
  int key[TRK_THREADS / 32];
  double minVal;
  int i, sink, nrem;
};
static_assert(CP_MAX_K <= TRK_THREADS && CP_MAX_K < 256, "one column per thread, keys below 256");

__device__ __forceinline__ void lsa_pick(double& best, int& key, double ob, int ok) {
  if (ob < best || (ob == best && ok > key)) {
    best = ob;
    key = ok;
  }
}

__device__ void lsa_solve_cta(const LsaCost& cost, int nr, int nc, LsaWork* w, LsaSync* sy) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, NW = TRK_THREADS / 32;
  if (tid == 0) lsa_init(w, nr, nc);
  for (int cur = 0; cur < nr; ++cur) {
    __syncthreads();
    for (int t = tid; t < nc; t += TRK_THREADS) {
      w->remaining[t] = nc - t - 1;
      w->SC[t] = 0;
      w->spc[t] = INFINITY;
    }
    for (int t = tid; t < nr; t += TRK_THREADS) w->SR[t] = 0;
    if (tid == 0) {
      sy->i = cur;
      sy->sink = -1;
      sy->nrem = nc;
      sy->minVal = 0.0;
    }
    __syncthreads();
    while (true) {
      const int i = sy->i, nrem = sy->nrem;
      const double minVal = sy->minVal;
      double best = INFINITY;
      int key = -1;
      if (tid < nrem) {
        const int j = w->remaining[tid];
        const double r = minVal + cost(i, j) - w->u[i] - w->v[j];
        double sp = w->spc[j];
        if (r < sp) {
          w->path[j] = i;
          w->spc[j] = r;
          sp = r;
        }
        best = sp;
        key = w->row4col[j] == -1 ? 256 + tid : 255 - tid;
      }
      for (int o = 16; o > 0; o >>= 1) lsa_pick(best, key, __shfl_down_sync(0xffffffffu, best, o), __shfl_down_sync(0xffffffffu, key, o));
      if (lane == 0) {
        sy->val[warp] = best;
        sy->key[warp] = key;
      }
      __syncthreads();
      if (tid == 0) {
        for (int q = 1; q < NW; ++q) lsa_pick(best, key, sy->val[q], sy->key[q]);
        const int index = key >= 256 ? key - 256 : 255 - key;
        const int j = w->remaining[index];
        w->SR[i] = 1;
        sy->minVal = best;
        if (w->row4col[j] == -1)
          sy->sink = j;
        else
          sy->i = w->row4col[j];
        w->SC[j] = 1;
        w->remaining[index] = w->remaining[nrem - 1];
        sy->nrem = nrem - 1;
      }
      __syncthreads();
      if (sy->sink >= 0) break;
    }
    // lsa_finish_row: potentials in parallel, the augmentation (a few steps) on thread 0
    const double minVal = sy->minVal;
    for (int t = tid; t < nr; t += TRK_THREADS)
      if (w->SR[t] && t != cur) w->u[t] += minVal - w->spc[w->col4row[t]];
    for (int t = tid; t < nc; t += TRK_THREADS)
      if (w->SC[t]) w->v[t] -= minVal - w->spc[t];
    __syncthreads();
    if (tid == 0) {
      w->u[cur] += minVal;
      int j = sy->sink;
      while (true) {
        const int i = w->path[j];
        w->row4col[j] = i;
        const int t = w->col4row[i];
        w->col4row[i] = j;
        j = t;
        if (i == cur) break;
      }
    }
  }
  __syncthreads();
}

// Steps 0-1 with the optimal assignment, one CTA per stream: staging and the order of `ret` on thread 0, the solver on
// the CTA.  A kernel of its own so that the step kernel's register allocation stays as it is; the step kernel then
// reads the entries from a.plan.
__global__ void __launch_bounds__(TRK_THREADS, 1) tracker_assoc_kernel(const StepArgs a) {
  const int b = blockIdx.x, tid = threadIdx.x;
  __shared__ int det_idx[TRK_MAXK];
  __shared__ float fbuf[3 * 2 * TRK_MAXK];
  __shared__ int ibuf[4 * TRK_MAXK];
  __shared__ LsaWork lsa;
  __shared__ LsaSync sync;
  __shared__ int s_N;
  const float* poses = a.poses + (size_t)b * a.K * CP_POSE_RECORD;
  const StreamState st = stream_state(a, b);
  const Slot* old = st.old;
  const int M = st.M;
  int nv = a.n_valid[b];
  if (nv > a.K) nv = a.K;
  if (nv < 0) nv = 0;
  if (tid == 0) s_N = plan_stage(a.cfg, poses, nv, old, M, det_idx, fbuf, ibuf);
  __syncthreads();
  const int N = s_N;
  const LsaCost v = plan_cost(fbuf, ibuf, N, M);
  if (N > 0 && M > 0) lsa_solve_cta(v, v.transpose ? M : N, v.transpose ? N : M, &lsa, &sync);
  if (tid == 0) {
    int* match_of_det = ibuf + N + M;
    int* det_of_trk = match_of_det + N;
    lsa_pairs(v, N, M, &lsa, match_of_det, det_of_trk);
    int idc = a.id_count[st.s];
    a.plan_n[b] = plan_entries(a.cfg, poses, det_idx, N, old, M, match_of_det, det_of_trk, &idc, a.plan + (size_t)b * a.T, a.T);
    a.id_count[st.s] = idc;
  }
}

__global__ void __launch_bounds__(TRK_THREADS, 1) tracker_step_kernel(const StepArgs a) {
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, NW = TRK_THREADS / 32;
  __shared__ Entry entries[TRK_MAXK];
  __shared__ int det_idx[TRK_MAXK];
  __shared__ float fbuf[3 * 2 * TRK_MAXK];
  __shared__ int ibuf[4 * TRK_MAXK];
  __shared__ unsigned char taken[TRK_MAXK];
  __shared__ int s_n, s_vis;
  __shared__ double s_conf[2];
  __shared__ double pnp_sm[(TRK_THREADS / 32) * PNP_SCRATCH];

  const float* poses = a.poses + (size_t)b * a.K * CP_POSE_RECORD;
  // every thread reads cur[s] here, before the first barrier; thread 0 flips it at the end
  const StreamState st = stream_state(a, b);
  const Slot* old = st.old;
  Slot* nxt = st.nxt;
  const int M = st.M;
  int nv = a.n_valid[b];
  if (nv > a.K) nv = a.K;
  if (nv < 0) nv = 0;

  if (tid == 0) {      // this stream's category settings (CatCfg), read back from shared memory where they are used
    const int cat = st.s / a.cat.S;
    s_vis = a.cat.visible_thresh[cat];
    s_conf[0] = a.cat.conf_lo[cat];
    s_conf[1] = a.cat.conf_hi[cat];
  }
  if (a.plan) {
    const int n = a.plan_n[b];
    for (int e = tid; e < n; e += TRK_THREADS) entries[e] = a.plan[(size_t)b * a.T + e];
    if (tid == 0) s_n = n;
  } else if (tid == 0) {
    // Steps 0-1 and the order of `ret` (serial, a few hundred operations)
    int idc = a.id_count[st.s];
    s_n = plan_step(a.cfg, poses, nv, old, M, &idc, entries, a.T, det_idx, fbuf, ibuf, taken);
    a.id_count[st.s] = idc;
  }
  __syncthreads();
  const int n = s_n;
  // Steps 2-4: one thread per entry (gaussian_fusion, eight 4-state predict/update, scale pool)
  for (int e = tid; e < n; e += TRK_THREADS) {
    const Entry en = entries[e];
    if (en.kind == ENTRY_MATCHED)
      entry_matched(a.cfg, &nxt[e], &old[en.trk], poses + (size_t)en.det * CP_POSE_RECORD);
    else if (en.kind == ENTRY_NEW)
      entry_new(a.cfg, &nxt[e], poses + (size_t)en.det * CP_POSE_RECORD, en.id);
    else
      entry_lost(&nxt[e], &old[en.trk]);
  }
  __syncthreads();
  // Steps 5-6: read-out + second PnP, one WARP per entry (every lane computes the identical read-out)
  const double* meta = a.meta + (size_t)b * CP_META_DOUBLES;
  double* sm = pnp_sm + warp * PNP_SCRATCH;
  for (int e = warp; e < n; e += NW) {
    double mean[16], sd[16], conf_avg, sc[3], su[3];
    Cfg ccfg = a.cfg;
    ccfg.conf_lo = s_conf[0];
    ccfg.conf_hi = s_conf[1];
    entry_readout(ccfg, &nxt[e], mean, sd, &conf_avg, sc, su);
    pose::PnPOut po;
    po.status = CP_PNP_NOT_RUN;
    po.n_pts = 0;
    int in_boxes = 0;
    if (a.cfg.use_pnp && (a.cfg.kalman || a.cfg.scale_pool)) {
      double V[24];
      if (a.cfg.scale_pool)
        pose::cuboid_vertices_d(sc, V);
      else
        pose::cuboid_vertices(nxt[e].rec + CP_P_OBJ_SCALE, V);
      __syncwarp();
      // the category's visibility gate is applied after the solve rather than inside it: the same status, and the
      // shared solve keeps the register allocation of a one-category step
      solve_and_shell_warp_v(mean, 8, V, meta + 5, meta[3], meta[4], 0, a.opencv_return, &po, sm, lane);
      if (po.status == CP_PNP_OK && pose::pnp_gate_invisible(po.kpspnp, s_vis)) po.status = CP_PNP_INVISIBLE;
      in_boxes = (po.status == CP_PNP_OK && conf_avg > 0.25) ? 1 : 0;
    } else {
      in_boxes = ((int)nxt[e].rec[CP_P_STATUS] == CP_PNP_OK && nxt[e].age == 1) ? 1 : 0;
    }
    __syncwarp();
    if (lane == 0) {
      slot_store_pose(&nxt[e], po);
      slot_store_pnp_kf(&nxt[e], po);
      write_track_record(&nxt[e], mean, sd, conf_avg, sc, su, &po, in_boxes,
                         a.tracks_out + ((size_t)b * a.T + e) * CP_TRACK_RECORD);
    }
    __syncwarp();
  }
  // unused output rows are zeroed so the tensor is deterministic
  float* tail = a.tracks_out + ((size_t)b * a.T + n) * CP_TRACK_RECORD;
  for (int i = tid; i < (a.T - n) * CP_TRACK_RECORD; i += TRK_THREADS) tail[i] = 0.f;
  if (tid == 0) {
    *st.new_n = n;
    a.n_out[b] = n;
    a.cur[st.s] = st.c ^ 1;
  }
}

__global__ void tracker_reset_kernel(int* n0, int* n1, int* id_count, int streams, int index) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < streams && (index < 0 || i == index)) {
    n0[i] = 0;
    n1[i] = 0;
    id_count[i] = 0;
  }
}

// init_track with meta['pre_dets'] (tracker.py:21-48), one CTA per stream; seeds go into the current slots
// (row b seeds stream ids[b], or b when ids is nullptr)
__global__ void __launch_bounds__(128) tracker_seed_kernel(const Cfg cfg, int T, const float* seeds, const int* n_seeds,
                                                            int S, Slot* slots0, Slot* slots1, int* n0, int* n1,
                                                            const int* cur, const int* ids, int* id_count) {
  const int b = blockIdx.x;
  int ns = n_seeds[b];
  if (ns < 0) return;
  if (ns > S) ns = S;
  const int s = ids ? ids[b] : b, c = cur[s];
  Slot* slots = (c ? slots1 : slots0) + (size_t)s * T;
  int* n_tracks = (c ? n1 : n0) + s;
  __shared__ int keep[TRK_MAXK];
  __shared__ int s_n;
  const float* sb = seeds + (size_t)b * S * CP_SEED_RECORD;
  if (threadIdx.x == 0) {
    int n = 0;
    for (int k = 0; k < ns; ++k)
      if ((double)sb[(size_t)k * CP_SEED_RECORD + CP_P_SCORE] > cfg.new_thresh) keep[n++] = k;
    s_n = n;
    *n_tracks = n;
    id_count[s] = n;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < s_n; t += blockDim.x)
    entry_seed(cfg, &slots[t], sb + (size_t)keep[t] * CP_SEED_RECORD, t + 1);
}

// ---- previous-frame heat maps ----------------------------------------------------------------------------------------
struct RenderArgs {
  Cfg cfg;
  CatCfg cat;
  int T, inp_h, inp_w, render_hm_mode, render_hmhp_mode;
  double pre_thresh;
  const Slot* slots0;      // [streams, T]
  const Slot* slots1;
  const int* n0;           // [streams]
  const int* n1;
  const int* cur;          // [streams]
  const int* ids;          // [B] tracker stream of image b, or nullptr: the identity
  const double* meta;      // [B,16]: [3] original width, [4] original height
  const double* trans;     // [B,6]
  float* pre_hm;           // [B,1,h,w]
  float* pre_hm_hp;        // [B,8,h,w]
  const int* modes;        // [B] cp_render_mode, or nullptr: all CP_RENDER_TRACKS
};

struct Patch {
  int x, y, r, live;
  double k;
};

// np.dot(t, [x, y, 1]) with a float32 point and the float64 2 x 3 matrix (utils/image.py:71-74)
__device__ __forceinline__ void affine_pt(const double* t, float x, float y, double* ox, double* oy) {
  *ox = t[0] * (double)x + t[1] * (double)y + t[2] * 1.0;
  *oy = t[3] * (double)x + t[4] * (double)y + t[5] * 1.0;
}

// one CTA per (track, stream): thread 0 derives the nine patches exactly like base_detector.py:213-315, all threads draw
__global__ void __launch_bounds__(256) tracker_render_kernel(const RenderArgs a) {
  const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int rmode = a.modes ? a.modes[b] : CP_RENDER_TRACKS;
  const int sid = a.ids ? a.ids[b] : b, c = a.cur[sid];
  if (t >= (c ? a.n1 : a.n0)[sid] || rmode == CP_RENDER_EMPTY) return;
  const bool gt = rmode == CP_RENDER_GT;
  const double conf_lo = a.cat.conf_lo[sid / a.cat.S], conf_hi = a.cat.conf_hi[sid / a.cat.S];      // CatCfg
  __shared__ Patch pt[9];
  if (tid == 0) {
    for (int i = 0; i < 9; ++i) pt[i].live = 0;
    const Slot& s = (c ? a.slots1 : a.slots0)[(size_t)sid * a.T + t];
    const float* r = s.rec;
    const double* tr = a.trans + (size_t)b * 6;
    const double ori_w = a.meta[(size_t)b * CP_META_DOUBLES + 3], ori_h = a.meta[(size_t)b * CP_META_DOUBLES + 4];
    if (gt || !((double)r[CP_P_SCORE] < a.pre_thresh)) {
      // _trans_bbox (base_detector.py:79-89): float32 box, transformed corners rounded back to float32, clipped
      double x0, y0, x1, y1;
      affine_pt(tr, r[CP_P_BBOX], r[CP_P_BBOX + 1], &x0, &y0);
      affine_pt(tr, r[CP_P_BBOX + 2], r[CP_P_BBOX + 3], &x1, &y1);
      float bx0 = (float)x0, by0 = (float)y0, bx1 = (float)x1, by1 = (float)y1;
      const float wm = (float)(a.inp_w - 1), hm = (float)(a.inp_h - 1);
      bx0 = fminf(fmaxf(bx0, 0.f), wm);
      bx1 = fminf(fmaxf(bx1, 0.f), wm);
      by0 = fminf(fmaxf(by0, 0.f), hm);
      by1 = fminf(fmaxf(by1, 0.f), hm);
      const float h = __fsub_rn(by1, by0), w = __fsub_rn(bx1, bx0);
      if (h > 0.f && w > 0.f) {
        double rad = gaussian_radius(ceil((double)h), ceil((double)w));
        int radius = (int)rad;
        if (radius < 0) radius = 0;
        const float cx = __fadd_rn(bx0, bx1) / 2.0f, cy = __fadd_rn(by0, by1) / 2.0f;
        pt[0].x = (int)cx;
        pt[0].y = (int)cy;
        pt[0].r = radius;
        pt[0].k = (a.render_hm_mode == 1 && !gt) ? (double)r[CP_P_SCORE] : 1.0;
        pt[0].live = 1;
        if (gt) {
          // base_detector.py:166-209: kps_gt[1:] in image pixels, int64 truncation, affine, truncation again; every point
          // is drawn with heat 1 wherever it lands (draw_umich_gaussian's slicing clips it, see the draw loop below)
          for (int j = 0; j < 8 && s.has_gt; ++j) {
            const double px = (double)s.kps_gt[2 * (j + 1)] * ori_w, py = (double)s.kps_gt[2 * (j + 1) + 1] * ori_h;
            const long long ix = (long long)px, iy = (long long)py;
            double ax, ay;
            affine_pt(tr, (float)ix, (float)iy, &ax, &ay);
            Patch& q = pt[1 + j];
            q.x = (int)(long long)ax;
            q.y = (int)(long long)ay;
            q.r = radius;
            q.k = 1.0;
            q.live = 1;
          }
        } else {
          // keypoints: normalised 9-point sets, entry 0 is the centre (base_detector.py:238-251)
          double px[8], py[8];
          bool have = true;
          const int mode = a.render_hmhp_mode;
          if (mode == 0 || mode == 1) {       // kps_ori: the detection's own keypoints, normalised
            for (int j = 0; j < 8; ++j) {
              px[j] = ((double)r[CP_P_KPS + 2 * j] / ori_w) * ori_w;
              py[j] = ((double)r[CP_P_KPS + 2 * j + 1] / ori_h) * ori_h;
            }
          } else if (a.cfg.kalman || a.cfg.scale_pool) {
            // kps_pnp_kf when the filtered PnP returned a tuple.  The reference's fall-back (kps_mean_kf[1:]: seven PIXEL
            // coordinates multiplied by the image size) can never land inside the image: nothing is drawn
            have = s.has_pnp_kf != 0;
            for (int j = 0; j < 8 && have; ++j) {
              px[j] = (double)s.kps_pnp_kf[2 * (j + 1)] * ori_w;
              py[j] = (double)s.kps_pnp_kf[2 * (j + 1) + 1] * ori_h;
            }
          } else {
            // 'kps_pnp' of the first PnP, or zeros when that failed (base_detector.py:248-253)
            const bool pose = ((int)r[CP_P_STATUS] == CP_PNP_OK || (int)r[CP_P_STATUS] == CP_PNP_INVISIBLE);
            for (int j = 0; j < 8; ++j) {
              px[j] = pose ? (double)r[CP_P_KPS_PNP + 2 * (j + 1)] * ori_w : 0.0;
              py[j] = pose ? (double)r[CP_P_KPS_PNP + 2 * (j + 1) + 1] * ori_h : 0.0;
            }
          }
          if (have) {
            for (int j = 0; j < 8; ++j) {
              Patch& q = pt[1 + j];
              q.live = 0;
              // COCO-style visibility, int64 truncation, affine of the truncated point, truncation again
              const bool outside = px[j] >= ori_w || px[j] < 0 || py[j] < 0 || py[j] >= ori_h;
              if (outside) continue;
              const long long ix = (long long)px[j], iy = (long long)py[j];
              double ax, ay;
              affine_pt(tr, (float)ix, (float)iy, &ax, &ay);
              const long long jx = (long long)ax, jy = (long long)ay;
              if (!(jx >= 0 && jx < a.inp_w && jy >= 0 && jy < a.inp_h)) continue;
              double k = 1.0;
              if (mode == 0 || mode == 2) {
                const double rd = a.cfg.hps_uncertainty ? s.fus_std[2 * j] : (double)r[CP_P_KPS_HM_STD + 2 * j];
                if (!((int)rd > 0)) continue;                   // radius_detector[j, 0] > 0 (int32 truncation)
                if (a.cfg.kalman && s.has_kf) {
                  const double std_c = sqrt(s.f.P[j][0] + s.f.P[j][5]);
                  k = 1.0 - pow(exp(log(0.15) / (conf_lo - conf_hi)), std_c - conf_hi);
                  if (k < 0.0) k = 0.0;
                } else if (a.cfg.hps_uncertainty) {
                  const double std_c = sqrt(s.fus_std[2 * j] + s.fus_std[2 * j + 1]);
                  k = 1.0 - pow(exp(log(0.15) / (conf_lo - conf_hi)), std_c - conf_hi);
                  if (k < 0.0) k = 0.0;
                } else {
                  k = (double)r[CP_P_KPS_HM_HEIGHT + j];
                }
              }
              q.x = (int)jx;
              q.y = (int)jy;
              q.r = radius;
              q.k = k;
              q.live = 1;
            }
          }
        }
      }
    }
  }
  __syncthreads();
  const size_t plane = (size_t)a.inp_h * a.inp_w;
  for (int i = 0; i < 9; ++i) {
    if (!(pt[i].live & 1)) continue;
    const Patch q = pt[i];
    float* map = (i == 0) ? a.pre_hm + (size_t)b * plane : a.pre_hm_hp + ((size_t)b * 8 + (i - 1)) * plane;
    // draw_umich_gaussian (utils/image.py:135-150): the patch clipped to the map, np.maximum compositing.  A centre left
    // of / above the map gives left / top < 0 and numpy's slices then keep exactly the part of the patch inside the map
    // (nothing once x < -r); a centre right of / below it gives right / bottom <= 0, the same.
    const int left = min(q.x, q.r), right = min(a.inp_w - q.x, q.r + 1);
    const int top = min(q.y, q.r), bottom = min(a.inp_h - q.y, q.r + 1);
    const int pw = left + right, ph = top + bottom;
    if (pw <= 0 || ph <= 0) continue;
    for (int e = tid; e < pw * ph; e += blockDim.x) {
      const int dy = e / pw - top, dx = e % pw - left;
      const float v = umich_value(dx, dy, q.r, q.k);
      // values are >= 0: the unsigned order of the bit patterns is the float order
      atomicMax(reinterpret_cast<unsigned int*>(map + (size_t)(q.y + dy) * a.inp_w + (q.x + dx)), __float_as_uint(v));
    }
  }
}

Cfg make_cfg(const cp_tracker_config& c) {
  Cfg g;
  g.kalman = c.kalman;
  g.scale_pool = c.scale_pool;
  g.use_pnp = c.use_pnp;
  g.hps_uncertainty = c.hps_uncertainty;
  g.max_age = c.max_age;
  g.new_thresh = (double)c.new_thresh;
  g.R = (double)c.R;
  g.conf_lo = (double)c.conf_lo;
  g.conf_hi = (double)c.conf_hi;
  g.hungarian = c.hungarian;
  return g;
}

}  // namespace
}  // namespace cp

extern "C" {

int cp_tracker_create(const cp_tracker_config* cfg, cp_tracker** out) { return cp_tracker_create_multi(cfg, 1, out); }

int cp_tracker_create_multi(const cp_tracker_config* cfgs, int32_t models, cp_tracker** out) {
  if (!cfgs || !out) return fail(CP_ERR_INVALID, "cp_tracker_create: null argument");
  if (models < 1 || models > CP_MAX_MODELS)
    return fail(CP_ERR_INVALID, "cp_tracker_create_multi: models must be in 1..CP_MAX_MODELS");
  const cp_tracker_config* cfg = cfgs;
  if (cfg->streams <= 0 || cfg->max_tracks <= 0 || cfg->max_tracks > CP_MAX_K)
    return fail(CP_ERR_INVALID, "cp_tracker_create: streams must be > 0 and max_tracks in 1..128");
  if ((long long)cfg->streams * models > (1 << 30))
    return fail(CP_ERR_INVALID, "cp_tracker_create_multi: too many streams");
  for (int m = 0; m < models; ++m) {
    if (cfgs[m].conf_lo == cfgs[m].conf_hi)
      return fail(CP_ERR_INVALID, "cp_tracker_create: conf_border needs two distinct values");
    cp_tracker_config a = cfgs[0], b = cfgs[m];
    a.visible_thresh = b.visible_thresh = 0;      // the per-category settings (opt.c)
    a.conf_lo = b.conf_lo = a.conf_hi = b.conf_hi = 0.f;
    if (memcmp(&a, &b, sizeof(a)))
      return fail(CP_ERR_INVALID, "cp_tracker_create_multi: the configs of category " + std::to_string(m) +
                                      " and category 0 differ in more than visible_thresh, conf_lo and conf_hi");
  }
  cp_tracker* t = new (std::nothrow) cp_tracker();
  if (!t) return fail(CP_ERR_INVALID, "cp_tracker_create: out of host memory");
  t->cfg = *cfg;
  t->cfg.streams = cfg->streams * models;
  t->cat.S = cfg->streams;
  for (int m = 0; m < models; ++m) {
    t->cat.visible_thresh[m] = cfgs[m].visible_thresh;
    t->cat.conf_lo[m] = (double)cfgs[m].conf_lo;
    t->cat.conf_hi[m] = (double)cfgs[m].conf_hi;
  }
  cfg = &t->cfg;
  struct DeviceGuard {
    int prev = -1;
    ~DeviceGuard() {
      if (prev >= 0) cudaSetDevice(prev);
    }
  } guard;
  cudaError_t e = cudaGetDevice(&guard.prev);
  if (e == cudaSuccess) e = cudaSetDevice(cfg->device);
  const size_t ns = (size_t)cfg->streams * cfg->max_tracks;
  for (int i = 0; i < 2 && e == cudaSuccess; ++i) {
    e = cudaMalloc(&t->slots[i], ns * sizeof(Slot));
    if (e == cudaSuccess) e = cudaMalloc(&t->n_tracks[i], sizeof(int) * cfg->streams);
    if (e == cudaSuccess) e = cudaMemset(t->n_tracks[i], 0, sizeof(int) * cfg->streams);
  }
  if (e == cudaSuccess) e = cudaMalloc(&t->id_count, sizeof(int) * cfg->streams);
  if (e == cudaSuccess) e = cudaMemset(t->id_count, 0, sizeof(int) * cfg->streams);
  if (e == cudaSuccess) e = cudaMalloc(&t->modes, sizeof(int) * cfg->streams);
  if (e == cudaSuccess) e = cudaMalloc(&t->ids, sizeof(int) * cfg->streams);
  if (e == cudaSuccess) e = cudaMalloc(&t->cur, sizeof(int) * cfg->streams);
  if (e == cudaSuccess) e = cudaMemset(t->cur, 0, sizeof(int) * cfg->streams);
  if (e == cudaSuccess && cfg->hungarian) e = cudaMalloc(&t->plan, ns * sizeof(Entry));
  if (e == cudaSuccess && cfg->hungarian) e = cudaMalloc(&t->plan_n, sizeof(int) * cfg->streams);
  if (e != cudaSuccess) {
    cp_tracker_destroy(t);
    return fail(CP_ERR_CUDA, std::string("cp_tracker_create: ") + cudaGetErrorString(e));
  }
  *out = t;
  return CP_OK;
}

int cp_tracker_destroy(cp_tracker* t) {
  if (!t) return CP_OK;
  for (int i = 0; i < 2; ++i) {
    if (t->slots[i]) cudaFree(t->slots[i]);
    if (t->n_tracks[i]) cudaFree(t->n_tracks[i]);
  }
  if (t->id_count) cudaFree(t->id_count);
  if (t->modes) cudaFree(t->modes);
  if (t->ids) cudaFree(t->ids);
  if (t->cur) cudaFree(t->cur);
  if (t->plan) cudaFree(t->plan);
  if (t->plan_n) cudaFree(t->plan_n);
  delete t;
  return CP_OK;
}

int cp_tracker_reset(cp_tracker* t, int32_t index, void* stream) {
  if (!t) return fail(CP_ERR_INVALID, "cp_tracker_reset: null tracker");
  if (index >= t->cfg.streams) return fail(CP_ERR_INVALID, "cp_tracker_reset: stream index out of range");
  tracker_reset_kernel<<<(t->cfg.streams + 127) / 128, 128, 0, (cudaStream_t)stream>>>(t->n_tracks[0], t->n_tracks[1],
                                                                                         t->id_count, t->cfg.streams, index);
  CP_LAUNCH_CHECK("tracker_reset_kernel");
  return CP_OK;
}

}  // extern "C"

namespace {

// A stream map of `batch` rows: every id in 0..streams-1 and none twice.  The range's lower end and duplicates are
// checked before the tracker is looked at, so a bad map is reported even with a null handle.
int check_stream_ids(const cp_tracker* t, int32_t batch, const int32_t* ids, const char* fn) {
  if (!ids || batch <= 0) return CP_OK;
  for (int i = 0; i < batch; ++i) {
    if (ids[i] < 0) return fail(CP_ERR_INVALID, std::string(fn) + ": stream id " + std::to_string(ids[i]) + " out of range");
    for (int j = 0; j < i; ++j)
      if (ids[j] == ids[i]) return fail(CP_ERR_INVALID, std::string(fn) + ": duplicate stream id " + std::to_string(ids[i]));
  }
  if (!t) return CP_OK;
  for (int i = 0; i < batch; ++i)
    if (ids[i] >= t->cfg.streams)
      return fail(CP_ERR_INVALID, std::string(fn) + ": stream id " + std::to_string(ids[i]) + " out of range 0.." +
                                      std::to_string(t->cfg.streams - 1));
  return CP_OK;
}

// the validated host map -> the tracker's device copy (stream-ordered behind the kernels that read the previous map)
int upload_stream_ids(cp_tracker* t, int32_t batch, const int32_t* ids, cudaStream_t s, const int** dev) {
  *dev = nullptr;
  if (!ids) return CP_OK;
  CP_CUDA_CHECK(cudaMemcpyAsync(t->ids, ids, sizeof(int32_t) * batch, cudaMemcpyHostToDevice, s));
  *dev = t->ids;
  return CP_OK;
}

}  // namespace

extern "C" {

int cp_tracker_step(cp_tracker* t, int32_t batch, const float* poses, const int32_t* n_valid, int32_t K, const double* meta,
                    float* tracks_out, int32_t* n_tracks, void* stream) {
  return cp_tracker_step_ex(t, batch, nullptr, poses, n_valid, K, meta, tracks_out, n_tracks, stream);
}

int cp_tracker_step_ex(cp_tracker* t, int32_t batch, const int32_t* stream_ids, const float* poses, const int32_t* n_valid,
                       int32_t K, const double* meta, float* tracks_out, int32_t* n_tracks, void* stream) {
  if (int rc = check_stream_ids(t, batch, stream_ids, "cp_tracker_step")) return rc;
  if (!t || !poses || !n_valid || !meta || !tracks_out || !n_tracks) return fail(CP_ERR_INVALID, "cp_tracker_step: null argument");
  if (batch <= 0 || batch > t->cfg.streams) return fail(CP_ERR_INVALID, "cp_tracker_step: batch exceeds the tracker's streams");
  if (K <= 0 || K > CP_MAX_K) return fail(CP_ERR_INVALID, "cp_tracker_step: K must be in 1..128");
  cudaStream_t s = (cudaStream_t)stream;
  StepArgs a;
  if (int rc = upload_stream_ids(t, batch, stream_ids, s, &a.ids)) return rc;
  a.cfg = make_cfg(t->cfg);
  a.cat = t->cat;
  a.opencv_return = t->cfg.opencv_return;
  a.T = t->cfg.max_tracks;
  a.K = K;
  a.poses = poses;
  a.n_valid = n_valid;
  a.meta = meta;
  a.slots0 = t->slots[0];
  a.slots1 = t->slots[1];
  a.n0 = t->n_tracks[0];
  a.n1 = t->n_tracks[1];
  a.cur = t->cur;
  a.id_count = t->id_count;
  a.tracks_out = tracks_out;
  a.n_out = n_tracks;
  a.plan = t->cfg.hungarian ? static_cast<Entry*>(t->plan) : nullptr;
  a.plan_n = t->cfg.hungarian ? t->plan_n : nullptr;
  if (a.plan) {
    tracker_assoc_kernel<<<batch, TRK_THREADS, 0, s>>>(a);
    CP_LAUNCH_CHECK("tracker_assoc_kernel");
  }
  tracker_step_kernel<<<batch, TRK_THREADS, 0, s>>>(a);     // flips cur[] of the streams it steps, and only those
  CP_LAUNCH_CHECK("tracker_step_kernel");
  return CP_OK;
}

int cp_tracker_render(cp_tracker* t, int32_t batch, const double* meta, const double* trans_input, int32_t inp_h,
                      int32_t inp_w, float* pre_hm, float* pre_hm_hp, void* stream) {
  return cp_tracker_render_ex2(t, batch, nullptr, meta, trans_input, inp_h, inp_w, nullptr, pre_hm, pre_hm_hp, stream);
}

int cp_tracker_render_ex(cp_tracker* t, int32_t batch, const double* meta, const double* trans_input, int32_t inp_h,
                         int32_t inp_w, const int32_t* modes, float* pre_hm, float* pre_hm_hp, void* stream) {
  return cp_tracker_render_ex2(t, batch, nullptr, meta, trans_input, inp_h, inp_w, modes, pre_hm, pre_hm_hp, stream);
}

int cp_tracker_render_ex2(cp_tracker* t, int32_t batch, const int32_t* stream_ids, const double* meta,
                          const double* trans_input, int32_t inp_h, int32_t inp_w, const int32_t* modes, float* pre_hm,
                          float* pre_hm_hp, void* stream) {
  bool any_mode = false;
  for (int b = 0; modes && b < batch; ++b) {
    if (modes[b] < CP_RENDER_TRACKS || modes[b] > CP_RENDER_EMPTY)
      return fail(CP_ERR_INVALID, "cp_tracker_render_ex: unknown render mode " + std::to_string(modes[b]) + " (0, 1 or 2)");
    any_mode = any_mode || modes[b] != CP_RENDER_TRACKS;
  }
  if (int rc = check_stream_ids(t, batch, stream_ids, "cp_tracker_render")) return rc;
  if (!t || !meta || !trans_input || !pre_hm || !pre_hm_hp) return fail(CP_ERR_INVALID, "cp_tracker_render: null argument");
  if (batch <= 0 || batch > t->cfg.streams || inp_h <= 0 || inp_w <= 0) return fail(CP_ERR_INVALID, "cp_tracker_render: bad shape");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t plane = (size_t)inp_h * inp_w;
  RenderArgs a;
  if (int rc = upload_stream_ids(t, batch, stream_ids, s, &a.ids)) return rc;
  CP_CUDA_CHECK(cudaMemsetAsync(pre_hm, 0, sizeof(float) * plane * batch, s));
  CP_CUDA_CHECK(cudaMemsetAsync(pre_hm_hp, 0, sizeof(float) * plane * 8 * batch, s));
  if (any_mode) CP_CUDA_CHECK(cudaMemcpyAsync(t->modes, modes, sizeof(int32_t) * batch, cudaMemcpyHostToDevice, s));
  a.cfg = make_cfg(t->cfg);
  a.cat = t->cat;
  a.T = t->cfg.max_tracks;
  a.inp_h = inp_h;
  a.inp_w = inp_w;
  a.render_hm_mode = t->cfg.render_hm_mode;
  a.render_hmhp_mode = t->cfg.render_hmhp_mode;
  a.pre_thresh = (double)t->cfg.pre_thresh;
  a.slots0 = t->slots[0];
  a.slots1 = t->slots[1];
  a.n0 = t->n_tracks[0];
  a.n1 = t->n_tracks[1];
  a.cur = t->cur;
  a.meta = meta;
  a.trans = trans_input;
  a.pre_hm = pre_hm;
  a.pre_hm_hp = pre_hm_hp;
  a.modes = any_mode ? t->modes : nullptr;
  dim3 grid(t->cfg.max_tracks, batch);
  tracker_render_kernel<<<grid, 256, 0, s>>>(a);
  CP_LAUNCH_CHECK("tracker_render_kernel");
  return CP_OK;
}

int cp_tracker_seed(cp_tracker* t, int32_t batch, const float* seeds, const int32_t* n_seeds, int32_t S, void* stream) {
  return cp_tracker_seed_ex(t, batch, nullptr, seeds, n_seeds, S, stream);
}

int cp_tracker_seed_ex(cp_tracker* t, int32_t batch, const int32_t* stream_ids, const float* seeds, const int32_t* n_seeds,
                       int32_t S, void* stream) {
  if (S < 0 || S > CP_MAX_K) return fail(CP_ERR_INVALID, "cp_tracker_seed: S must be in 0..128");
  if (int rc = check_stream_ids(t, batch, stream_ids, "cp_tracker_seed")) return rc;
  if (!t || !n_seeds || (S > 0 && !seeds)) return fail(CP_ERR_INVALID, "cp_tracker_seed: null argument");
  if (batch <= 0 || batch > t->cfg.streams) return fail(CP_ERR_INVALID, "cp_tracker_seed: batch exceeds the tracker's streams");
  if (S > t->cfg.max_tracks)
    return fail(CP_ERR_INVALID, "cp_tracker_seed: S = " + std::to_string(S) + " seeds exceed max_tracks = " +
                                    std::to_string(t->cfg.max_tracks));
  cudaStream_t s = (cudaStream_t)stream;
  const int* ids = nullptr;
  if (int rc = upload_stream_ids(t, batch, stream_ids, s, &ids)) return rc;
  tracker_seed_kernel<<<batch, 128, 0, s>>>(make_cfg(t->cfg), t->cfg.max_tracks, seeds, n_seeds, S, t->slots[0],
                                            t->slots[1], t->n_tracks[0], t->n_tracks[1], t->cur, ids, t->id_count);
  CP_LAUNCH_CHECK("tracker_seed_kernel");
  return CP_OK;
}

}  // extern "C"

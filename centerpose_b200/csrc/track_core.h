// CenterPoseTrack post-network state (SURVEY.md row f-2 / a-T), written once as __host__ __device__ code: the CUDA
// tracker kernel (tracker.cu) calls it, and tests/host compiles the same header with g++ to check it on the CPU against
// tests/golden/tracker_seq.json (the UNMODIFIED reference tracker on a seeded sequence).
//
// Reference behaviour reproduced (paths relative to /root/reference/src/lib):
//   detectors/base_detector.py:502-544   gaussian_fusion (product of the displacement and heat-map Gaussians)
//   utils/tracker.py:55-84               init_kf: 32-state constant-velocity filter = 8 keypoints x (x, y, vx, vy)
//   utils/tracker.py:86-101              update_kf (measurement = fused keypoints + the negated tracking_hp offsets)
//   utils/tracker.py:103-116             update_scale_pool (inverse-variance fusion of the scale history)
//   utils/tracker.py:21-48               init_track with meta['pre_dets'] (ground-truth seeding)
//   utils/tracker.py:118-236             step: association (greedy :304-314 or optimal :154-177), matched / new / lost
//                                        tracks
//   utils/tracker.py:238-262             filter read-out, keypoint confidence from the filter covariance
//   utils/image.py:102-150               gaussian_radius / gaussian2D / draw_umich_gaussian (previous-frame heat maps)
// filterpy.kalman.KalmanFilter (third party, requirements.txt: filterpy>=1.4.5): predict x = F x, P = F P F^T + Q with
// Q = I; update in Joseph form P = (I - K H) P (I - K H)^T + K R K^T, H = I.
//
// Structure used here: F couples x with vx and y with vy only, H = I, Q = I, R and the initial P are diagonal, so the
// 32 x 32 covariance stays block diagonal with one 4 x 4 block per keypoint for ever; the filter is eight independent
// 4-state filters (the 32 x 32 inverse of the reference factorises into the same eight 4 x 4 inverses).
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/centerpose_b200.h"
#include "pose_core.h"

namespace cp {
namespace track {

struct Cfg {
  int kalman, scale_pool, use_pnp, hps_uncertainty, max_age;
  double new_thresh, R, conf_lo, conf_hi;      // opt.new_thresh, opt.R, opt.conf_border[opt.c]
  int hungarian;                               // opt.hungarian
};

// per-track filter state that is not part of the fp32 pose record
struct Filter {
  double x[32];          // keypoint i: x[4i] = u, x[4i+1] = v, x[4i+2] = du, x[4i+3] = dv
  double P[8][16];       // 4 x 4 covariance block of keypoint i, row-major
  double sp_w[3];        // scale pool: running sum of unc^-2
  double sp_m[3];        //             running sum of unc^-2 * scale
};

// ---- gaussian_fusion (base_detector.py:505-535); heat-map entries < 0 are the -10000 sentinels -----------------------
CP_HD void gaussian_fusion(const float* disp_mean, const float* disp_std, const float* hm_mean, const float* hm_std,
                           int hps_uncertainty, double* mean, double* std) {
  for (int i = 0; i < 16; ++i) {
    const double dm = disp_mean[i], ds = disp_std[i], hm = hm_mean[i], hs = hm_std[i];
    if (hps_uncertainty) {
      if (hm < 0 || hs < 0) {
        std[i] = ds;
        mean[i] = dm;
      } else {
        const double wd = 1.0 / (ds * ds), wh = 1.0 / (hs * hs);
        const double s = 1.0 / sqrt(wd + wh);
        std[i] = s;
        mean[i] = s * s * (wd * dm + wh * hm);
      }
    } else {
      if (hm < 0 || hs < 0) {
        std[i] = 20.0;
        mean[i] = dm;
      } else {
        const double s = hs / sqrt(2.0);
        const double wh = 1.0 / (hs * hs);
        std[i] = s;
        mean[i] = s * s * (wh * dm + wh * hm);
      }
    }
  }
}

// ---- 4 x 4 helpers ----------------------------------------------------------------------------------------------------
CP_HD void mat4_mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double s = 0.0;
      for (int k = 0; k < 4; ++k) s += A[i * 4 + k] * B[k * 4 + j];
      C[i * 4 + j] = s;
    }
}
CP_HD void mat4_mul_bt(const double* A, const double* B, double* C) {      // C = A B^T
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double s = 0.0;
      for (int k = 0; k < 4; ++k) s += A[i * 4 + k] * B[j * 4 + k];
      C[i * 4 + j] = s;
    }
}
// Gauss-Jordan with partial pivoting (numpy.linalg.inv = LU with partial pivoting; on a block-diagonal matrix the pivot
// search never leaves the block)
CP_HDN bool mat4_inv(const double* A, double* Inv) {
  double M[4][8];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      M[i][j] = A[i * 4 + j];
      M[i][4 + j] = (i == j) ? 1.0 : 0.0;
    }
  for (int c = 0; c < 4; ++c) {
    int piv = c;
    double best = fabs(M[c][c]);
    for (int r = c + 1; r < 4; ++r)
      if (fabs(M[r][c]) > best) {
        best = fabs(M[r][c]);
        piv = r;
      }
    if (best == 0.0) return false;
    if (piv != c)
      for (int j = 0; j < 8; ++j) {
        const double t = M[c][j];
        M[c][j] = M[piv][j];
        M[piv][j] = t;
      }
    const double inv = 1.0 / M[c][c];
    for (int j = 0; j < 8; ++j) M[c][j] *= inv;
    for (int r = 0; r < 4; ++r) {
      if (r == c) continue;
      const double f = M[r][c];
      if (f != 0.0)
        for (int j = 0; j < 8; ++j) M[r][j] -= f * M[c][j];
    }
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) Inv[i * 4 + j] = M[i][4 + j];
  return true;
}

// ---- the filter, one keypoint (4 states) at a time ----------------------------------------------------------------------
// tracker.py:55-84: R = diag(std_x^2, std_y^2, opt.R, opt.R), P = R; x = (mean_x, mean_y, -tracking_hp_x, -tracking_hp_y)
CP_HD void kf_init_kp(Filter* f, int i, const double* fus_mean, const double* fus_std, const float* tracking_hp, double Rv) {
  double* P = f->P[i];
  for (int e = 0; e < 16; ++e) P[e] = 0.0;
  P[0] = fus_std[2 * i] * fus_std[2 * i];
  P[5] = fus_std[2 * i + 1] * fus_std[2 * i + 1];
  P[10] = Rv;
  P[15] = Rv;
  f->x[4 * i] = fus_mean[2 * i];
  f->x[4 * i + 1] = fus_mean[2 * i + 1];
  f->x[4 * i + 2] = -(double)tracking_hp[2 * i];
  f->x[4 * i + 3] = -(double)tracking_hp[2 * i + 1];
}

// predict (F = [[1,0,1,0],[0,1,0,1],[0,0,1,0],[0,0,0,1]], Q = I) followed by update_kf (tracker.py:86-101) with the new
// observation; Joseph-form covariance update
CP_HDN void kf_predict_update_kp(Filter* f, int i, const double* fus_mean, const double* fus_std, const float* tracking_hp,
                                 double Rv) {
  const double F[16] = {1, 0, 1, 0, 0, 1, 0, 1, 0, 0, 1, 0, 0, 0, 0, 1};
  double* x = f->x + 4 * i;
  double* P = f->P[i];
  // predict
  const double xp[4] = {x[0] + x[2], x[1] + x[3], x[2], x[3]};
  double FP[16], Pp[16];
  mat4_mul(F, P, FP);
  mat4_mul_bt(FP, F, Pp);
  for (int d = 0; d < 4; ++d) Pp[d * 5] += 1.0;
  // update
  const double z[4] = {fus_mean[2 * i], fus_mean[2 * i + 1], -(double)tracking_hp[2 * i], -(double)tracking_hp[2 * i + 1]};
  const double Rd[4] = {fus_std[2 * i] * fus_std[2 * i], fus_std[2 * i + 1] * fus_std[2 * i + 1], Rv, Rv};
  double S[16], Si[16], K[16];
  for (int e = 0; e < 16; ++e) S[e] = Pp[e];
  for (int d = 0; d < 4; ++d) S[d * 5] += Rd[d];
  if (!mat4_inv(S, Si)) {
    for (int d = 0; d < 4; ++d) x[d] = xp[d];
    for (int e = 0; e < 16; ++e) P[e] = Pp[e];
    return;
  }
  mat4_mul(Pp, Si, K);
  double y[4];
  for (int d = 0; d < 4; ++d) y[d] = z[d] - xp[d];
  for (int d = 0; d < 4; ++d) x[d] = xp[d] + K[d * 4] * y[0] + K[d * 4 + 1] * y[1] + K[d * 4 + 2] * y[2] + K[d * 4 + 3] * y[3];
  double IK[16], T[16], J[16], KR[16], KRK[16];
  for (int e = 0; e < 16; ++e) IK[e] = -K[e];
  for (int d = 0; d < 4; ++d) IK[d * 5] += 1.0;
  mat4_mul(IK, Pp, T);
  mat4_mul_bt(T, IK, J);
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) KR[r * 4 + c] = K[r * 4 + c] * Rd[c];
  mat4_mul_bt(KR, K, KRK);
  for (int e = 0; e < 16; ++e) P[e] = J[e] + KRK[e];
}

// tracker.py:249-260: std of a keypoint from the filter covariance -> confidence; < 0.15 blanks the keypoint for the PnP
CP_HD double kp_confidence(double pxx, double pyy, double lo, double hi) {
  const double std_c = sqrt(pxx + pyy);
  const double c = 1.0 - pow(exp(log(0.15) / (lo - hi)), std_c - hi);
  return c > 0.0 ? c : 0.0;
}

// ---- association (tracker.py:128-153 + greedy_assignment :304-314); float32 arithmetic like the reference's arrays ------
#if defined(__CUDA_ARCH__)
#define CP_FSUB(a, b) __fsub_rn(a, b)
#define CP_FMUL(a, b) __fmul_rn(a, b)
#define CP_FADD(a, b) __fadd_rn(a, b)
#else
CP_HD float cp_f_noinline_sub(volatile float a, volatile float b) { return a - b; }
CP_HD float cp_f_noinline_mul(volatile float a, volatile float b) { return a * b; }
CP_HD float cp_f_noinline_add(volatile float a, volatile float b) { return a + b; }
#define CP_FSUB(a, b) cp_f_noinline_sub(a, b)
#define CP_FMUL(a, b) cp_f_noinline_mul(a, b)
#define CP_FADD(a, b) cp_f_noinline_add(a, b)
#endif

// dist[i][j] of tracker.py:146-152: float32 squared distance, + 1e18 (float64) where the pair is invalid
CP_HD double pair_cost(const float* det_c, const float* det_size, const int* det_cls, const float* trk_c,
                       const float* trk_size, const int* trk_cls, int i, int j) {
  const float dx = CP_FSUB(trk_c[2 * j], det_c[2 * i]), dy = CP_FSUB(trk_c[2 * j + 1], det_c[2 * i + 1]);
  const float d = CP_FADD(CP_FMUL(dx, dx), CP_FMUL(dy, dy));
  const bool invalid = (d > trk_size[j]) || (d > det_size[i]) || (det_cls[i] != trk_cls[j]);
  return (double)d + (invalid ? 1e18 : 0.0);
}

// the Hungarian branch clips the matrix first (tracker.py:156: dist[dist > 1e18] = 1e18)
CP_HD double clipped_cost(const float* det_c, const float* det_size, const int* det_cls, const float* trk_c,
                          const float* trk_size, const int* trk_cls, int i, int j) {
  const double d = pair_cost(det_c, det_size, det_cls, trk_c, trk_size, trk_cls, i, j);
  return d > 1e18 ? 1e18 : d;
}

// det_c: N x 2 (ct + tracking, float32), det_size / det_cls: N;  trk_c: M x 2, trk_size / trk_cls: M
// match_of_det[i] = matched track or -1;  det_of_trk[j] = matched detection or -1.  `taken` is M bytes of scratch.
CP_HDN void greedy_associate(const float* det_c, const float* det_size, const int* det_cls, int N, const float* trk_c,
                             const float* trk_size, const int* trk_cls, int M, int* match_of_det, int* det_of_trk,
                             unsigned char* taken) {
  for (int j = 0; j < M; ++j) {
    taken[j] = 0;
    det_of_trk[j] = -1;
  }
  for (int i = 0; i < N; ++i) {
    match_of_det[i] = -1;
    int best = -1;
    double bd = 0.0;
    for (int j = 0; j < M; ++j) {
      double dd = pair_cost(det_c, det_size, det_cls, trk_c, trk_size, trk_cls, i, j);
      if (taken[j]) dd = 1e18;              // column already assigned (dist[:, j] = 1e18)
      if (best < 0 || dd < bd) {            // argmin keeps the FIRST minimum
        best = j;
        bd = dd;
      }
    }
    if (best >= 0 && bd < 1e16) {
      taken[best] = 1;
      match_of_det[i] = best;
      det_of_trk[best] = i;
    }
  }
}

// ---- optimal association (tracker.py:154-177, opt.hungarian) --------------------------------------------------------
// The reference calls sklearn 0.22's linear_assignment; the oracle stands in for it with
// scipy.optimize.linear_sum_assignment, and this is scipy's solver (shortest augmenting paths with potentials, Crouse
// 2016), restated so that the same pairs come out, ties included: fp64 potentials u / v, one Dijkstra search per row,
// columns scanned in the order of a `remaining` list that starts reversed and shrinks by swap-with-last, and the scan's
// tie rule "the first minimum, unless a later equal one is an unassigned column".  Rows are the smaller side (scipy
// transposes a tall matrix).  The matrix is never stored: the cost functor recomputes entries.
struct LsaWork {
  double u[CP_MAX_K], v[CP_MAX_K], spc[CP_MAX_K];      // row / column potentials, shortest path cost per column
  int path[CP_MAX_K], col4row[CP_MAX_K], row4col[CP_MAX_K], remaining[CP_MAX_K];
  unsigned char SR[CP_MAX_K], SC[CP_MAX_K];
};

// the rows x cols view of the clipped N x M dist matrix
struct LsaCost {
  const float *det_c, *det_size, *trk_c, *trk_size;
  const int *det_cls, *trk_cls;
  int transpose;             // rows = tracks (N > M)
  CP_HD double operator()(int r, int c) const {
    return transpose ? clipped_cost(det_c, det_size, det_cls, trk_c, trk_size, trk_cls, c, r)
                     : clipped_cost(det_c, det_size, det_cls, trk_c, trk_size, trk_cls, r, c);
  }
};

CP_HD void lsa_init(LsaWork* w, int nr, int nc) {
  for (int i = 0; i < nr; ++i) {
    w->u[i] = 0.0;
    w->col4row[i] = -1;
  }
  for (int j = 0; j < nc; ++j) {
    w->v[j] = 0.0;
    w->row4col[j] = -1;
    w->path[j] = -1;
  }
}

CP_HD void lsa_begin_row(LsaWork* w, int nr, int nc) {
  for (int it = 0; it < nc; ++it) w->remaining[it] = nc - it - 1;
  for (int i = 0; i < nr; ++i) w->SR[i] = 0;
  for (int j = 0; j < nc; ++j) {
    w->SC[j] = 0;
    w->spc[j] = INFINITY;
  }
}

// after the search of row `cur` reached `sink`: update the potentials, then augment along `path`
CP_HD void lsa_finish_row(LsaWork* w, int nr, int nc, int cur, int sink, double minVal) {
  w->u[cur] += minVal;
  for (int i = 0; i < nr; ++i)
    if (w->SR[i] && i != cur) w->u[i] += minVal - w->spc[w->col4row[i]];
  for (int j = 0; j < nc; ++j)
    if (w->SC[j]) w->v[j] -= minVal - w->spc[j];
  int j = sink;
  while (true) {
    const int i = w->path[j];
    w->row4col[j] = i;
    const int t = w->col4row[i];
    w->col4row[i] = j;
    j = t;
    if (i == cur) break;
  }
}

// serial solver (nr <= nc <= CP_MAX_K): col4row[r] = the column of row r.  Returns false on an infeasible matrix (an
// infinite cost; never the case for dist, whose entries are at most 1e18)
template <class Cost>
CP_HDN bool lsa_solve(const Cost& cost, int nr, int nc, LsaWork* w) {
  lsa_init(w, nr, nc);
  for (int cur = 0; cur < nr; ++cur) {
    lsa_begin_row(w, nr, nc);
    int nrem = nc, i = cur, sink = -1;
    double minVal = 0.0;
    while (sink < 0) {
      int index = -1;
      double lowest = INFINITY;
      w->SR[i] = 1;
      for (int it = 0; it < nrem; ++it) {
        const int j = w->remaining[it];
        const double r = minVal + cost(i, j) - w->u[i] - w->v[j];
        if (r < w->spc[j]) {
          w->path[j] = i;
          w->spc[j] = r;
        }
        if (w->spc[j] < lowest || (w->spc[j] == lowest && w->row4col[j] == -1)) {
          lowest = w->spc[j];
          index = it;
        }
      }
      minVal = lowest;
      if (index < 0 || minVal == INFINITY) return false;
      const int j = w->remaining[index];
      if (w->row4col[j] == -1)
        sink = j;
      else
        i = w->row4col[j];
      w->SC[j] = 1;
      w->remaining[index] = w->remaining[--nrem];
    }
    lsa_finish_row(w, nr, nc, cur, sink, minVal);
  }
  return true;
}

// scipy's pairs and the post-filter of tracker.py:166-177 (a pair costing more than 1e16 is dropped).
// match_of_det[i] = j for a kept pair, -2 - j for a dropped one, -1 when unassigned; det_of_trk[j] likewise.
CP_HD void lsa_pairs(const LsaCost& cost, int N, int M, const LsaWork* w, int* match_of_det, int* det_of_trk) {
  for (int i = 0; i < N; ++i) match_of_det[i] = -1;
  for (int j = 0; j < M; ++j) det_of_trk[j] = -1;
  if (N == 0 || M == 0) return;
  const int nr = cost.transpose ? M : N;
  for (int r = 0; r < nr; ++r) {
    const int c = w->col4row[r];
    if (c < 0) continue;
    const int i = cost.transpose ? c : r, j = cost.transpose ? r : c;
    const bool drop = cost(r, c) > 1e16;
    match_of_det[i] = drop ? -2 - j : j;
    det_of_trk[j] = drop ? -2 - i : i;
  }
}

// ---- one track ------------------------------------------------------------------------------------------------------
struct Slot {
  float rec[CP_POSE_RECORD];     // the detection the track carries (cp_pose_field layout, image pixels)
  int id, age, active, has_kf;
  int has_pnp_kf;                // the second PnP of the latest step returned a tuple ('kps_pnp_kf' in the track dict)
  float kps_pnp_kf[18];          // its 9 normalised projected points (centre first)
  double fus_mean[16], fus_std[16];
  Filter f;
  int has_gt;                    // seeded from a dict with 'kps_gt' (drawn by the ground-truth render)
  float kps_gt[18];              // its 9 normalised points (centre first)
};

CP_HD void slot_fusion(const Cfg& c, Slot* s) {
  gaussian_fusion(s->rec + CP_P_KPS_DISP_MEAN, s->rec + CP_P_KPS_DISP_STD, s->rec + CP_P_KPS_HM_MEAN, s->rec + CP_P_KPS_HM_STD,
                  c.hps_uncertainty, s->fus_mean, s->fus_std);
}

// tracker.py:103-116 as running sums (the reference re-adds the whole history in the same order every frame)
CP_HD void scale_pool_add(Slot* s, bool first) {
  for (int k = 0; k < 3; ++k) {
    const double u = (double)s->rec[CP_P_OBJ_SCALE_UNC + k];
    const double w = 1.0 / (u * u);
    s->f.sp_w[k] = (first ? 0.0 : s->f.sp_w[k]) + w;
    s->f.sp_m[k] = (first ? 0.0 : s->f.sp_m[k]) + w * (double)s->rec[CP_P_OBJ_SCALE + k];
  }
}

// Step 2 (tracker.py:167-186): detection `rec` continues track `old`
CP_HDN void entry_matched(const Cfg& c, Slot* dst, const Slot* old, const float* rec) {
  for (int i = 0; i < CP_POSE_RECORD; ++i) dst->rec[i] = rec[i];
  dst->id = old->id;
  dst->age = 1;
  dst->active = old->active + 1;
  dst->has_kf = old->has_kf;
  dst->has_pnp_kf = 0;
  dst->has_gt = 0;
  dst->f = old->f;
  slot_fusion(c, dst);
  if (c.kalman) {
    for (int i = 0; i < 8; ++i) kf_predict_update_kp(&dst->f, i, dst->fus_mean, dst->fus_std, dst->rec + CP_P_TRACKING_HP, c.R);
    dst->has_kf = 1;
  }
  if (c.scale_pool) scale_pool_add(dst, false);
}

// Step 3 (tracker.py:188-204): an unmatched detection above new_thresh starts a track
CP_HDN void entry_new(const Cfg& c, Slot* dst, const float* rec, int id) {
  for (int i = 0; i < CP_POSE_RECORD; ++i) dst->rec[i] = rec[i];
  dst->id = id;
  dst->age = 1;
  dst->active = 1;
  dst->has_kf = 0;
  dst->has_pnp_kf = 0;
  dst->has_gt = 0;
  slot_fusion(c, dst);
  for (int i = 0; i < 32; ++i) dst->f.x[i] = 0.0;
  for (int i = 0; i < 8; ++i)
    for (int e = 0; e < 16; ++e) dst->f.P[i][e] = 0.0;
  for (int k = 0; k < 3; ++k) dst->f.sp_w[k] = dst->f.sp_m[k] = 0.0;
  if (c.kalman) {
    for (int i = 0; i < 8; ++i) kf_init_kp(&dst->f, i, dst->fus_mean, dst->fus_std, dst->rec + CP_P_TRACKING_HP, c.R);
    dst->has_kf = 1;
  }
  if (c.scale_pool) scale_pool_add(dst, true);
}

// init_track (tracker.py:31-49): one dict of meta['pre_dets'] (cp_seed_field layout) starts track `id`.  The filter
// starts from the dict's own kps_fusion_mean / kps_fusion_std, which are not re-derived through gaussian_fusion.
CP_HDN void entry_seed(const Cfg& c, Slot* dst, const float* seed, int id) {
  for (int i = 0; i < CP_POSE_RECORD; ++i) dst->rec[i] = seed[i];
  if (seed[CP_S_HAS_CT] == 0.f) {
    dst->rec[CP_P_CT] = (float)(((double)seed[CP_P_BBOX] + (double)seed[CP_P_BBOX + 2]) / 2);
    dst->rec[CP_P_CT + 1] = (float)(((double)seed[CP_P_BBOX + 1] + (double)seed[CP_P_BBOX + 3]) / 2);
  }
  dst->id = id;
  dst->age = 1;
  dst->active = 1;
  dst->has_kf = 0;
  dst->has_pnp_kf = seed[CP_S_HAS_KPS_PNP_KF] != 0.f ? 1 : 0;
  for (int t = 0; t < 18; ++t) dst->kps_pnp_kf[t] = dst->has_pnp_kf ? seed[CP_S_KPS_PNP_KF + t] : 0.f;
  dst->has_gt = seed[CP_S_HAS_KPS_GT] != 0.f ? 1 : 0;
  for (int t = 0; t < 18; ++t) dst->kps_gt[t] = seed[CP_S_KPS_GT + t];
  for (int i = 0; i < 16; ++i) {
    dst->fus_mean[i] = (double)seed[CP_S_KPS_FUSION_MEAN + i];
    dst->fus_std[i] = (double)seed[CP_S_KPS_FUSION_STD + i];
  }
  for (int i = 0; i < 32; ++i) dst->f.x[i] = 0.0;
  for (int i = 0; i < 8; ++i)
    for (int e = 0; e < 16; ++e) dst->f.P[i][e] = 0.0;
  for (int k = 0; k < 3; ++k) dst->f.sp_w[k] = dst->f.sp_m[k] = 0.0;
  if (c.kalman) {
    for (int i = 0; i < 8; ++i) kf_init_kp(&dst->f, i, dst->fus_mean, dst->fus_std, dst->rec + CP_P_TRACKING_HP, c.R);
    dst->has_kf = 1;
  }
  if (c.scale_pool) scale_pool_add(dst, true);
}

// Step 4 (tracker.py:206-236): a track without a detection is kept, unmoved, while age < max_age
CP_HD void entry_lost(Slot* dst, const Slot* old) {
  *dst = *old;
  dst->age = old->age + 1;
  dst->active = 0;
}

// Step 5 (tracker.py:238-270): filter read-out.  kps_mean_kf gets the -10000 sentinel where the confidence is < 0.15
// (in the returned copy only -- the state keeps the estimate); conf_avg = sum(conf) / 8 (0 without the filter).
CP_HDN void entry_readout(const Cfg& c, const Slot* s, double* kps_mean_kf /*16*/, double* kps_std_kf /*16*/, double* conf_avg,
                          double* scale_new /*3*/, double* scale_unc /*3*/) {
  double csum = 0.0;
  for (int i = 0; i < 8; ++i) {
    if (c.kalman) {
      const double pxx = s->f.P[i][0], pyy = s->f.P[i][5];
      kps_mean_kf[2 * i] = s->f.x[4 * i];
      kps_mean_kf[2 * i + 1] = s->f.x[4 * i + 1];
      kps_std_kf[2 * i] = sqrt(pxx);
      kps_std_kf[2 * i + 1] = sqrt(pyy);
      const double conf = kp_confidence(pxx, pyy, c.conf_lo, c.conf_hi);
      csum += conf;
      if (conf < 0.15) kps_mean_kf[2 * i] = kps_mean_kf[2 * i + 1] = -10000.0;
    } else {
      kps_mean_kf[2 * i] = (double)s->rec[CP_P_KPS + 2 * i];
      kps_mean_kf[2 * i + 1] = (double)s->rec[CP_P_KPS + 2 * i + 1];
      kps_std_kf[2 * i] = kps_std_kf[2 * i + 1] = 0.0;
    }
  }
  *conf_avg = csum / 8.0;
  for (int k = 0; k < 3; ++k) {
    if (c.scale_pool) {
      const double sd = 1.0 / sqrt(s->f.sp_w[k]);
      scale_unc[k] = sd;
      scale_new[k] = s->f.sp_m[k] * (sd * sd);
    } else {
      scale_new[k] = (double)s->rec[CP_P_OBJ_SCALE + k];
      scale_unc[k] = (double)s->rec[CP_P_OBJ_SCALE_UNC + k];
    }
  }
}

// The second PnP wrote a pose: pnp_shell mutates the track dict (cuboid_pnp_shell.py:27-54), so the record's pose fields
// now hold the filtered result
CP_HD void slot_store_pose(Slot* s, const pose::PnPOut& po) {
  if (po.status != CP_PNP_OK && po.status != CP_PNP_INVISIBLE) return;
  float* o = s->rec;
  o[CP_P_STATUS] = (float)po.status;
  o[CP_P_NPTS] = (float)po.n_pts;
  for (int t = 0; t < 3; ++t) o[CP_P_LOCATION + t] = (float)po.loc[t];
  for (int t = 0; t < 4; ++t) o[CP_P_QUAT + t] = (float)po.quat[t];
  o[CP_P_REPROJ] = (float)po.reproj;
  for (int t = 0; t < 16; ++t) o[CP_P_PROJ_CUBOID + t] = (float)po.proj[t];
  for (int t = 0; t < 27; ++t) o[CP_P_KPS_3D_CAM + t] = (float)po.kps3d[t];
  for (int t = 0; t < 18; ++t) o[CP_P_KPS_PNP + t] = (float)po.kpspnp[t];
}

// tracker.py:283-286: ret[idx]['kps_pnp_kf'] exists when the filtered PnP returned a tuple.  A matched / new track is a
// fresh dict (no stale key); a lost track keeps its dict, and re-solving the unchanged state gives the same answer.
CP_HD void slot_store_pnp_kf(Slot* s, const pose::PnPOut& po) {
  s->has_pnp_kf = (po.status == CP_PNP_OK) ? 1 : 0;
  for (int t = 0; t < 18; ++t) s->kps_pnp_kf[t] = s->has_pnp_kf ? (float)po.kpspnp[t] : 0.f;
}

// one output row (cp_track_field layout)
CP_HDN void write_track_record(const Slot* s, const double* kps_mean_kf, const double* kps_std_kf, double conf_avg,
                               const double* scale_new, const double* scale_unc, const pose::PnPOut* po, int in_boxes,
                               float* o /*CP_TRACK_RECORD*/) {
  for (int i = 0; i < CP_POSE_RECORD; ++i) o[i] = s->rec[i];
  for (int i = CP_POSE_RECORD; i < CP_TRACK_RECORD; ++i) o[i] = 0.f;
  o[CP_T_ID] = (float)s->id;
  o[CP_T_AGE] = (float)s->age;
  o[CP_T_ACTIVE] = (float)s->active;
  o[CP_T_IN_BOXES] = (float)in_boxes;
  o[CP_T_PNP2_STATUS] = (float)(po ? po->status : CP_PNP_NOT_RUN);
  o[CP_T_CONF_AVG] = (float)conf_avg;
  for (int i = 0; i < 16; ++i) {
    o[CP_T_KPS_FUSION_MEAN + i] = (float)s->fus_mean[i];
    o[CP_T_KPS_FUSION_STD + i] = (float)s->fus_std[i];
    o[CP_T_KPS_MEAN_KF + i] = (float)kps_mean_kf[i];
    o[CP_T_KPS_STD_KF + i] = (float)kps_std_kf[i];
  }
  for (int k = 0; k < 3; ++k) {
    o[CP_T_OBJ_SCALE_KF + k] = (float)scale_new[k];
    o[CP_T_OBJ_SCALE_UNC_KF + k] = (float)scale_unc[k];
  }
  if (po && po->status == CP_PNP_OK) {
    for (int t = 0; t < 18; ++t) o[CP_T_KPS_PNP_KF + t] = (float)po->kpspnp[t];
    for (int t = 0; t < 27; ++t) o[CP_T_KPS_3D_CAM_KF + t] = (float)po->kps3d[t];
  }
}

// ---- Steps 0-4 as a plan (serial; tiny): which detections enter, who continues which track, the order of `ret` -----------
enum { ENTRY_MATCHED = 0, ENTRY_NEW = 1, ENTRY_LOST = 2 };
struct Entry {
  int kind, det, trk, id;
};

// Step 0 (tracker.py:121-130) and the arrays of Step 1: with PnP on and at least one solved box, only the solved
// detections are tracked.  Scratch: det_idx[K], fbuf[3 * (K + M)] floats, ibuf[2 * K + 2 * M] ints.  Returns N.
CP_HDN int plan_stage(const Cfg& c, const float* poses, int n_valid, const Slot* old, int M, int* det_idx, float* fbuf,
                      int* ibuf) {
  int N = 0;
  bool any_box = false;
  if (c.use_pnp)
    for (int i = 0; i < n_valid; ++i) any_box = any_box || ((int)poses[(size_t)i * CP_POSE_RECORD + CP_P_STATUS] == CP_PNP_OK);
  for (int i = 0; i < n_valid; ++i)
    if (!any_box || (int)poses[(size_t)i * CP_POSE_RECORD + CP_P_STATUS] == CP_PNP_OK) det_idx[N++] = i;
  float* det_c = fbuf;
  float* det_size = det_c + 2 * N;
  float* trk_c = det_size + N;
  float* trk_size = trk_c + 2 * M;
  int* det_cls = ibuf;
  int* trk_cls = det_cls + N;
  for (int i = 0; i < N; ++i) {
    const float* r = poses + (size_t)det_idx[i] * CP_POSE_RECORD;
    det_c[2 * i] = (float)((double)r[CP_P_CT] + (double)r[CP_P_TRACKING]);
    det_c[2 * i + 1] = (float)((double)r[CP_P_CT + 1] + (double)r[CP_P_TRACKING + 1]);
    det_size[i] = (float)(((double)r[CP_P_BBOX + 2] - (double)r[CP_P_BBOX]) * ((double)r[CP_P_BBOX + 3] - (double)r[CP_P_BBOX + 1]));
    det_cls[i] = (int)r[CP_P_CLS];
  }
  for (int j = 0; j < M; ++j) {
    const float* r = old[j].rec;
    trk_c[2 * j] = r[CP_P_CT];
    trk_c[2 * j + 1] = r[CP_P_CT + 1];
    trk_size[j] = (float)(((double)r[CP_P_BBOX + 2] - (double)r[CP_P_BBOX]) * ((double)r[CP_P_BBOX + 3] - (double)r[CP_P_BBOX + 1]));
    trk_cls[j] = (int)r[CP_P_CLS];
  }
  return N;
}

// the staged arrays of plan_stage as the solver's cost view
CP_HD LsaCost plan_cost(const float* fbuf, const int* ibuf, int N, int M) {
  LsaCost v;
  v.det_c = fbuf;
  v.det_size = fbuf + 2 * N;
  v.trk_c = v.det_size + N;
  v.trk_size = v.trk_c + 2 * M;
  v.det_cls = ibuf;
  v.trk_cls = ibuf + N;
  v.transpose = N > M;
  return v;
}

// Steps 2-4 as a list: matched pairs in row order; then new tracks over unmatched_dets = the unassigned detections in
// order followed by those of dropped pairs (in row order); then lost tracks over unmatched_tracks, built the same way.
// Without dropped pairs (greedy) this is the plain row / column order.  *id_count advances for every new track.
CP_HDN int plan_entries(const Cfg& c, const float* poses, const int* det_idx, int N, const Slot* old, int M,
                        const int* match_of_det, const int* det_of_trk, int* id_count, Entry* entries, int max_entries) {
  int n = 0;
  for (int i = 0; i < N && n < max_entries; ++i)
    if (match_of_det[i] >= 0) entries[n++] = Entry{ENTRY_MATCHED, det_idx[i], match_of_det[i], 0};
  for (int pass = 0; pass < 2; ++pass)
    for (int i = 0; i < N && n < max_entries; ++i)
      if ((pass == 0 ? match_of_det[i] == -1 : match_of_det[i] < -1) &&
          (double)poses[(size_t)det_idx[i] * CP_POSE_RECORD + CP_P_SCORE] > c.new_thresh) {
        *id_count += 1;
        entries[n++] = Entry{ENTRY_NEW, det_idx[i], -1, *id_count};
      }
  for (int j = 0; j < M && n < max_entries; ++j)
    if (det_of_trk[j] == -1 && old[j].age < c.max_age) entries[n++] = Entry{ENTRY_LOST, -1, j, 0};
  for (int i = 0; i < N && n < max_entries; ++i)
    if (match_of_det[i] < -1 && old[-2 - match_of_det[i]].age < c.max_age)
      entries[n++] = Entry{ENTRY_LOST, -1, -2 - match_of_det[i], 0};
  return n;
}

// poses: n_valid records of this frame; old: M tracks.  Scratch: det_idx[K], fbuf[3 * (K + M)] floats, ibuf[2 * K + 2 * M]
// ints, taken[M], and with c.hungarian the solver's `lsa`.  Returns the number of entries written (<= max_entries);
// *id_count is advanced for every new track.
CP_HDN int plan_step(const Cfg& c, const float* poses, int n_valid, const Slot* old, int M, int* id_count, Entry* entries,
                     int max_entries, int* det_idx, float* fbuf, int* ibuf, unsigned char* taken, LsaWork* lsa = nullptr) {
  const int N = plan_stage(c, poses, n_valid, old, M, det_idx, fbuf, ibuf);
  const LsaCost v = plan_cost(fbuf, ibuf, N, M);
  int* match_of_det = ibuf + N + M;
  int* det_of_trk = match_of_det + N;
  if (c.hungarian) {
    if (N > 0 && M > 0) lsa_solve(v, v.transpose ? M : N, v.transpose ? N : M, lsa);
    lsa_pairs(v, N, M, lsa, match_of_det, det_of_trk);
  } else {
    greedy_associate(v.det_c, v.det_size, v.det_cls, N, v.trk_c, v.trk_size, v.trk_cls, M, match_of_det, det_of_trk, taken);
  }
  return plan_entries(c, poses, det_idx, N, old, M, match_of_det, det_of_trk, id_count, entries, max_entries);
}

// ---- previous-frame heat maps (base_detector.py:150-388) -----------------------------------------------------------------
// utils/image.py:102-122
CP_HD double gaussian_radius(double height, double width) {
  const double mo = 0.7;
  const double b1 = height + width, c1 = width * height * (1 - mo) / (1 + mo);
  const double r1 = (b1 + sqrt(b1 * b1 - 4 * c1)) / 2;
  const double b2 = 2 * (height + width), c2 = (1 - mo) * width * height;
  const double r2 = (b2 + sqrt(b2 * b2 - 16 * c2)) / 2;
  const double a3 = 4 * mo, b3 = -2 * mo * (height + width), c3 = (mo - 1) * width * height;
  const double r3 = (b3 + sqrt(b3 * b3 - 4 * a3 * c3)) / 2;
  double r = r1 < r2 ? r1 : r2;
  return r < r3 ? r : r3;
}

// value of draw_umich_gaussian's patch at offset (dx, dy) from the centre, radius r, scaled by k, as the float32 that
// np.maximum(..., out=float32 map) stores
CP_HD float umich_value(int dx, int dy, int r, double k) {
  const double diameter = 2.0 * r + 1.0;
  const double sigma = diameter / 6.0;
  double h = exp(-((double)dx * dx + (double)dy * dy) / (2.0 * sigma * sigma));
  if (h < 2.220446049250313e-16) h = 0.0;          // h[h < eps * h.max()] = 0, h.max() = 1 at the centre
  return (float)(h * k);
}

}  // namespace track
}  // namespace cp

// TEST INFRASTRUCTURE ONLY: the host build of centerpose_b200/csrc/track_core.h for the ground-truth seeding and the
// optimal (hungarian) association, checked on the CPU against tests/golden/tracker_seq_{gt_first,gt_every,hungarian}.json
// and against scipy.optimize.linear_sum_assignment.  The step below is the serial statement of tracker_assoc_kernel +
// tracker_step_kernel, the seeding that of tracker_seed_kernel.  Never loaded by the product.
#include <vector>

#include "../../centerpose_b200/csrc/track_core.h"

using namespace cp;
using namespace cp::track;

struct GtHostTracker {
  Cfg cfg;
  int visible_thresh, opencv_return, max_tracks;
  int id_count = 0;
  std::vector<Slot> tracks;
  LsaWork lsa;
};

// a dense row-major matrix as the solver's cost view
struct MatCost {
  const double* c;
  int nc;
  double operator()(int r, int k) const { return c[(size_t)r * nc + k]; }
};

struct MatCostT {
  const double* c;
  int nc;
  double operator()(int r, int k) const { return c[(size_t)k * nc + r]; }
};

extern "C" {

void* gth_create(int kalman, int scale_pool, int use_pnp, int hps_uncertainty, int max_age, double new_thresh, double R,
                 double conf_lo, double conf_hi, int hungarian, int visible_thresh, int opencv_return, int max_tracks) {
  GtHostTracker* t = new GtHostTracker();
  t->cfg = Cfg{kalman, scale_pool, use_pnp, hps_uncertainty, max_age, new_thresh, R, conf_lo, conf_hi, hungarian};
  t->visible_thresh = visible_thresh;
  t->opencv_return = opencv_return;
  t->max_tracks = max_tracks;
  return t;
}
void gth_destroy(void* h) { delete (GtHostTracker*)h; }

// init_track with meta['pre_dets']: seeds [n][CP_SEED_RECORD]; returns the number of tracks
int gth_seed(void* h, const float* seeds, int n) {
  GtHostTracker* t = (GtHostTracker*)h;
  t->tracks.clear();
  t->id_count = 0;
  for (int k = 0; k < n; ++k) {
    const float* s = seeds + (size_t)k * CP_SEED_RECORD;
    if ((double)s[CP_P_SCORE] > t->cfg.new_thresh) {
      Slot sl;
      entry_seed(t->cfg, &sl, s, ++t->id_count);
      t->tracks.push_back(sl);
    }
  }
  return (int)t->tracks.size();
}

// Tracker.step for one video stream; out: [max_tracks][CP_TRACK_RECORD]; returns the number of tracks
int gth_step(void* h, const float* poses, int n_valid, const double* cam, double width, double height, float* out) {
  GtHostTracker* t = (GtHostTracker*)h;
  const int M = (int)t->tracks.size(), K = n_valid;
  std::vector<Entry> entries(t->max_tracks);
  std::vector<int> det_idx(K + 1), ibuf(2 * K + 2 * M + 4);
  std::vector<float> fbuf(3 * (K + M) + 4);
  std::vector<unsigned char> taken(M + 1);
  const int n = plan_step(t->cfg, poses, n_valid, t->tracks.data(), M, &t->id_count, entries.data(), t->max_tracks,
                          det_idx.data(), fbuf.data(), ibuf.data(), taken.data(), &t->lsa);
  std::vector<Slot> next(n);
  for (int e = 0; e < n; ++e) {
    const Entry& en = entries[e];
    if (en.kind == ENTRY_MATCHED)
      entry_matched(t->cfg, &next[e], &t->tracks[en.trk], poses + (size_t)en.det * CP_POSE_RECORD);
    else if (en.kind == ENTRY_NEW)
      entry_new(t->cfg, &next[e], poses + (size_t)en.det * CP_POSE_RECORD, en.id);
    else
      entry_lost(&next[e], &t->tracks[en.trk]);
  }
  for (int e = 0; e < n; ++e) {
    double mean[16], sd[16], conf_avg, sc[3], su[3];
    entry_readout(t->cfg, &next[e], mean, sd, &conf_avg, sc, su);
    pose::PnPOut po;
    po.status = CP_PNP_NOT_RUN;
    po.n_pts = 0;
    int in_boxes = 0;
    if (t->cfg.use_pnp && (t->cfg.kalman || t->cfg.scale_pool)) {
      double V[24];
      if (t->cfg.scale_pool)
        pose::cuboid_vertices_d(sc, V);
      else
        pose::cuboid_vertices(next[e].rec + CP_P_OBJ_SCALE, V);
      pose::solve_and_shell_v(mean, 8, V, cam, width, height, t->visible_thresh, t->opencv_return, &po);
      slot_store_pose(&next[e], po);
      slot_store_pnp_kf(&next[e], po);
      in_boxes = (po.status == CP_PNP_OK && conf_avg > 0.25) ? 1 : 0;
    } else {
      in_boxes = ((int)next[e].rec[CP_P_STATUS] == CP_PNP_OK && next[e].age == 1) ? 1 : 0;
    }
    write_track_record(&next[e], mean, sd, conf_avg, sc, su, &po, in_boxes, out + (size_t)e * CP_TRACK_RECORD);
  }
  t->tracks.swap(next);
  return n;
}

// the solver core on a dense nr x nc matrix, returned like scipy: min(nr, nc) pairs sorted by row.  Returns the number
// of pairs, or -1 when the solver reports an infeasible matrix.
int gth_lsa(const double* cost, int nr, int nc, int* rows, int* cols) {
  static LsaWork w;
  if (nr == 0 || nc == 0) return 0;
  if (nr > CP_MAX_K || nc > CP_MAX_K) return -1;
  if (nr <= nc) {
    if (!lsa_solve(MatCost{cost, nc}, nr, nc, &w)) return -1;
    for (int r = 0; r < nr; ++r) {
      rows[r] = r;
      cols[r] = w.col4row[r];
    }
    return nr;
  }
  // tall: solve the transpose (rows = the original columns), then list the pairs by original row
  if (!lsa_solve(MatCostT{cost, nc}, nc, nr, &w)) return -1;
  int n = 0;
  std::vector<int> col_of_row(nr, -1);
  for (int k = 0; k < nc; ++k) col_of_row[w.col4row[k]] = k;
  for (int r = 0; r < nr; ++r)
    if (col_of_row[r] >= 0) {
      rows[n] = r;
      cols[n] = col_of_row[r];
      ++n;
    }
  return n;
}
}

// CPU test harness for the host state machine of the estimator (xivo_b200/csrc/estimator.h +
// estimator_host.cpp.inc + tracker_host.cpp.inc): compiled with g++ (no nvcc, no GPU) into a small shared object that
// tests/test_host_logic.py and tests/test_host_twin.py drive through ctypes.  Test infrastructure only — nothing here is
// linked into libxivo_b200.so.  No kernel is emulated: the callers supply what the device phases compute (the twin tests
// take it from the oracle), and the entry points run the host decisions in between — configuration, message heap, clocks,
// gravity initialisation, the nominal-state Runge-Kutta chain, the filter's update steps and the image tracker.
#include <chrono>
#include <cstring>
#include <string>

#include "../../xivo_b200/csrc/estimator.h"
#include "../../xivo_b200/csrc/homography.h"

namespace xb {
struct HostScope {  // the library's version also feeds the profiler; timing is irrelevant here
  explicit HostScope(const char*) {}
};
}  // namespace xb

#include "../../xivo_b200/csrc/estimator_host.cpp.inc"
#include "../../xivo_b200/csrc/tracker_host.cpp.inc"

namespace {
std::string g_err;
}

extern "C" {
const char* hh_error() { return g_err.c_str(); }

void* hh_create(const char* cfg_json, int G, int F, int tracker_only) {
  try {
    return new xb::Estimator(xb::Json::parse(cfg_json), xb::EkfLayout{G, F}, tracker_only != 0);
  } catch (const std::exception& e) {
    g_err = e.what();
    return nullptr;
  }
}
void hh_destroy(void* h) { delete static_cast<xb::Estimator*>(h); }

void hh_inertial(void* h, unsigned long long ts, const double* gyro, const double* accel) { static_cast<xb::Estimator*>(h)->inertial_internal(ts, gyro, accel); }
int hh_visual_begin(void* h, unsigned long long ts, int type) { return static_cast<xb::Estimator*>(h)->visual_begin(ts, type) ? 1 : 0; }
int hh_sticky_error(void* h) { return static_cast<xb::Estimator*>(h)->error; }

// Rsb(9) Tsb(3) Vsb(3) bg(3) ba(3) Rbc(9) Tbc(3) Rsg(9) = 42 doubles
void hh_motion(void* h, double* out) {
  const xb::MotionX& X = static_cast<xb::Estimator*>(h)->X;
  memcpy(out, X.Rsb.m, 72); memcpy(out + 9, X.Tsb.v, 24); memcpy(out + 12, X.Vsb.v, 24); memcpy(out + 15, X.bg.v, 24);
  memcpy(out + 18, X.ba.v, 24); memcpy(out + 21, X.Rbc.m, 72); memcpy(out + 30, X.Tbc.v, 24); memcpy(out + 33, X.Rsg.m, 72);
}
// flags: gravity_initialized, vision_initialized, imu_counter, vision_counter
void hh_flags(void* h, int* out) {
  auto* e = static_cast<xb::Estimator*>(h);
  out[0] = e->gravity_initialized; out[1] = e->vision_initialized; out[2] = e->imu_counter; out[3] = e->vision_counter;
}
unsigned long long hh_curr_time(void* h) { return static_cast<xb::Estimator*>(h)->curr_time; }
// pending Runge-Kutta stage records (16 doubles each: R(9), gyro-bg(3), accel-ba(3), h); returns the count, clears the queue
int hh_take_stages(void* h, double* out, int max_records) {
  auto* e = static_cast<xb::Estimator*>(h);
  static_assert(sizeof(xb::ImuStage) == 16 * sizeof(double), "ImuStage layout");
  const int n = (int)e->stages.size();
  if (n <= max_records && n) memcpy(out, e->stages.data(), sizeof(xb::ImuStage) * (size_t)n);
  e->stages.clear();
  return n;
}
void hh_initial_pmm(void* h, double* out529) { memcpy(out529, static_cast<xb::Estimator*>(h)->Pmm, 529 * 8); }
void hh_camera(void* h, double* out11) {
  const xb::CameraParams& c = static_cast<xb::Estimator*>(h)->cam;
  const double v[11] = {(double)c.model, (double)c.rows, (double)c.cols, c.fx, c.fy, c.cx, c.cy, c.k0, c.k1, c.k2, c.k3};
  memcpy(out11, v, sizeof(v));
}

// message heap: push (ts, type) and pop in execution order (MaintainBuffer, estimator.cpp:923-941)
void hh_push(void* h, unsigned long long ts, int type) {
  xb::Msg m;
  m.ts = ts; m.type = type;
  static_cast<xb::Estimator*>(h)->push(std::move(m));
}
int hh_pop(void* h, unsigned long long* ts, int* type) {
  xb::Msg m;
  if (!static_cast<xb::Estimator*>(h)->pop_ready(&m)) return 0;
  *ts = m.ts; *type = m.type;
  return 1;
}

// ---- the visual path with the device phases supplied by the caller (tests/test_host_twin.py feeds the oracle's values) ----
void hh_init_with_sim_depths(void* h) { static_cast<xb::Estimator*>(h)->sim_initialize_depths = true; }
// Batch::process_visual up to the sub-filter launch (estimator.cu): returns -1 when the message does not proceed, else the
// number of features queued for Feature::SubfilterUpdate
int hh_pcw_begin(void* h, unsigned long long ts, int n, const int* ids, const double* xp_depth) {
  auto* e = static_cast<xb::Estimator*>(h);
  if (!e->visual_begin(ts, 3) || e->error) return -1;
  e->predict_features();
  std::vector<int> vi(ids, ids + n);
  std::vector<double> vx(xp_depth, xp_depth + 3 * (size_t)n);
  for (int k = 0; k < n; ++k) e->ids_to_depths.insert({vi[k], vx[3 * k + 2]});
  e->tracker_update_pointcloud(vi, vx);
  e->stages.clear();  // the covariance side of Propagate is the device's
  e->update_step_pre();
  return (int)e->subfilter_list.size();
}
void hh_subfilter_ids(void* h, int* out) {
  auto* e = static_cast<xb::Estimator*>(h);
  for (size_t i = 0; i < e->subfilter_list.size(); ++i) out[i] = e->subfilter_list[i]->id;
}
// homography.h on its own: the mask of cv::findHomography(pts0, pts1, method, thresh, mask, max_iters, confidence); returns ok
int hh_homography_mask(const float* p0, const float* p1, int n, int method, double thresh, int max_iters, double confidence, unsigned char* mask) {
  std::vector<uint8_t> m;
  const bool ok = xb::homography::find_homography_mask(p0, p1, n, method, thresh, max_iters, confidence, m);
  memcpy(mask, m.data(), (size_t)n);
  return ok ? 1 : 0;
}
// the sub-filter's input states (after Feature::Triangulate where it ran): n x x(3), plus tri_ok flags
void hh_subfilter_inputs(void* h, double* x3, int* tri_ok) {
  auto* e = static_cast<xb::Estimator*>(h);
  for (size_t i = 0; i < e->subfilter_list.size(); ++i) {
    memcpy(x3 + 3 * i, e->subfilter_list[i]->x, 24);
    tri_ok[i] = e->subfilter_list[i]->tri_ok;
  }
}
// local state x(3) and own covariance P(9) of the features of list `which` (0 = instate_features, 1 = in_update, 2 = tracks)
int hh_feature_states(void* h, int which, int* ids, double* x3, double* P9, int max_n) {
  auto* e = static_cast<xb::Estimator*>(h);
  const std::vector<xb::Feature*>& v = which == 0 ? e->instate_features : which == 1 ? e->in_update : e->tracks;
  int n = 0;
  for (xb::Feature* f : v) {
    if (n < max_n) { ids[n] = f->id; memcpy(x3 + 3 * n, f->x, 24); memcpy(P9 + 9 * n, f->P, 72); }
    ++n;
  }
  return n;
}
void hh_depth_refine_counts(void* h, int* ok_failed) {
  auto* e = static_cast<xb::Estimator*>(h);
  ok_failed[0] = e->num_depth_refined; ok_failed[1] = e->num_depth_refine_failed;
}
void hh_triangulation_counts(void* h, int* good_bad) {
  auto* e = static_cast<xb::Estimator*>(h);
  good_bad[0] = e->num_good_triangulations; good_bad[1] = e->num_bad_triangulations;
}
// triangulate.h on its own: method index as in xb::TriMethod, g01 = [R(9) | T(3)]; returns 1 and x_out(3) on success
int hh_triangulate(int method, const double* R9, const double* T3, const double* xc0, const double* xc1, double zmin, double zmax,
                   double max_theta, double beta, double* x_out) {
  xb::TriOptions o;
  o.method = static_cast<xb::TriMethod>(method);
  o.zmin = zmin; o.zmax = zmax; o.max_theta_thresh = max_theta; o.beta_thresh = beta;
  xb::SE3h g;
  memcpy(g.R.m, R9, 72); memcpy(g.T.v, T3, 24);
  return xb::triangulate_feature_state(o, g, xc0, xc1, x_out) ? 1 : 0;
}
// out13: n x {x(3), P(9), outlier_counter}; returns the number of in-state features (the Jacobian / gate batch)
int hh_after_subfilter(void* h, const double* out13) {
  auto* e = static_cast<xb::Estimator*>(h);
  static_assert(sizeof(xb::SubfilterOut) == 13 * sizeof(double), "SubfilterOut layout");
  e->update_step_after_subfilter(reinterpret_cast<const xb::SubfilterOut*>(out13));
  e->edits.clear();  // applied to P by cov_edit_kernel in the product
  return (int)e->instate_features.size();
}
int hh_after_gate(void* h, const double* mh) {
  auto* e = static_cast<xb::Estimator*>(h);
  e->update_step_after_gate(mh);
  e->edits.clear();
  return (int)e->in_update.size();
}
// ---- 1-point RANSAC: the gate with the covariance diagonal of this frame; -1 = the two RANSAC device phases are pending
static std::vector<xb::Feature*> g_table_order;  // index space of the device feature table (instate_features before the gate)
int hh_after_gate_diag(void* h, const double* mh, const double* diag) {
  auto* e = static_cast<xb::Estimator*>(h);
  g_table_order = e->instate_features;
  e->update_step_after_gate(mh, diag);
  e->edits.clear();
  return e->ransac.active ? -1 : (int)e->in_update.size();
}
// ids of the device table order; low / high innovation ids; the rows the temporary update zeroes as (first, count) pairs
int hh_ransac_info(void* h, int* table_ids, int* low_ids, int* n_low, int* high_ids, int* n_high, int* zero_pairs, int* n_zero) {
  auto* e = static_cast<xb::Estimator*>(h);
  for (size_t i = 0; i < g_table_order.size(); ++i) table_ids[i] = g_table_order[i]->id;
  *n_low = *n_high = 0;
  for (size_t i = 0; i < e->ransac.mh_inliers.size(); ++i) {
    if (e->ransac.low[i]) low_ids[(*n_low)++] = e->ransac.mh_inliers[i]->id;
    else high_ids[(*n_high)++] = e->ransac.mh_inliers[i]->id;
  }
  *n_zero = (int)e->ransac.zero_edits.size();
  for (int i = 0; i < *n_zero; ++i) { zero_pairs[2 * i] = e->ransac.zero_edits[i].a; zero_pairs[2 * i + 1] = e->ransac.zero_edits[i].n; }
  return (int)g_table_order.size();
}
void hh_ransac_temp(void* h, const double* err) { static_cast<xb::Estimator*>(h)->ransac_after_temp_update(err); }
int hh_ransac_finish(void* h, const double* mh_table) {
  auto* e = static_cast<xb::Estimator*>(h);
  e->ransac_finish(mh_table, g_table_order);
  e->edits.clear();
  return (int)e->in_update.size();
}
int hh_ransac_rejected(void* h) { return static_cast<xb::Estimator*>(h)->num_oneptransac_rejected; }
void hh_after_update(void* h, const double* err, const double* Pmm, const double* diag, int had_update) {
  auto* e = static_cast<xb::Estimator*>(h);
  e->update_step_after_update(err, Pmm, diag, had_update != 0);
  e->edits.clear();
}
// which: 0 = instate_features, 1 = in_update, 2 = tracks.  Per feature: id, sind, ref group sind, FeatureStatus, TrackStatus
int hh_features(void* h, int which, int* out5, int max_n) {
  auto* e = static_cast<xb::Estimator*>(h);
  const std::vector<xb::Feature*>& v = which == 0 ? e->instate_features : which == 1 ? e->in_update : e->tracks;
  int n = 0;
  for (xb::Feature* f : v) {
    if (n < max_n) {
      int* o = out5 + 5 * n;
      o[0] = f->id; o[1] = f->sind; o[2] = f->ref ? f->ref->sind : -2; o[3] = (int)f->status; o[4] = (int)f->tstatus;
    }
    ++n;
  }
  return n;
}
// in-state groups: id, sind, GroupStatus; returns count; gauge group id in *gauge
int hh_groups(void* h, int* out3, int max_n, int* gauge) {
  auto* e = static_cast<xb::Estimator*>(h);
  *gauge = e->gauge_group;
  int n = 0;
  for (auto& kv : e->graph.groups) {
    xb::Group* g = kv.second;
    if (!g->instate()) continue;
    if (n < max_n) { out3[3 * n] = g->id; out3[3 * n + 1] = g->sind; out3[3 * n + 2] = (int)g->status; }
    ++n;
  }
  return n;
}
// read-back tables (estimator_accessors.cpp) from a host copy of P; flat rows of doubles:
// feature: id, sind, ref group id, Xs(3), Xc(3), xc(3), pred(2), meas(2), cov(6) = 22;  group: id, sind, pose(7), cov(36) = 45
int hh_feature_rows(void* h, const double* P, int n_output, double* out22, int max_rows) {
  const auto rows = static_cast<xb::Estimator*>(h)->instate_feature_rows(P, n_output);
  for (size_t i = 0; i < rows.size() && (int)i < max_rows; ++i) {
    double* o = out22 + 22 * i;
    o[0] = rows[i].id; o[1] = rows[i].sind; o[2] = rows[i].ref_group_id;
    memcpy(o + 3, rows[i].Xs, 24); memcpy(o + 6, rows[i].Xc, 24); memcpy(o + 9, rows[i].xc, 24);
    memcpy(o + 12, rows[i].pred, 16); memcpy(o + 14, rows[i].meas, 16); memcpy(o + 16, rows[i].cov, 48);
  }
  return (int)rows.size();
}
int hh_group_rows(void* h, const double* P, double* out45, int max_rows) {
  const auto rows = static_cast<xb::Estimator*>(h)->instate_group_rows(P);
  for (size_t i = 0; i < rows.size() && (int)i < max_rows; ++i) {
    double* o = out45 + 45 * i;
    o[0] = rows[i].id; o[1] = rows[i].sind;
    memcpy(o + 2, rows[i].pose, 56); memcpy(o + 9, rows[i].cov, 288);
  }
  return (int)rows.size();
}
int hh_just_dropped(void* h, int* out, int max_n) {
  auto* e = static_cast<xb::Estimator*>(h);
  for (size_t i = 0; i < e->just_dropped_ids.size() && (int)i < max_n; ++i) out[i] = e->just_dropped_ids[i];
  return (int)e->just_dropped_ids.size();
}
const char* hh_error_msg(void* h) { return static_cast<xb::Estimator*>(h)->error_msg.c_str(); }

// tracker mask (tracker.cpp:471-488, :760-774)
void hh_mask_init(void* h, int rows, int cols) {
  auto* e = static_cast<xb::Estimator*>(h);
  e->tracker_set_geometry(rows, cols, true);
  e->reset_mask();
}
void hh_mask_reset(void* h) { static_cast<xb::Estimator*>(h)->reset_mask(); }
void hh_mask_out(void* h, double x, double y) { static_cast<xb::Estimator*>(h)->mask_out(x, y); }
int hh_mask_valid(void* h, double x, double y) { return static_cast<xb::Estimator*>(h)->mask_valid(x, y) ? 1 : 0; }
void hh_mask_dump(void* h, unsigned char* out) {
  auto* e = static_cast<xb::Estimator*>(h);
  for (int y = 0; y < e->rows; ++y)
    for (int x = 0; x < e->cols; ++x) out[(size_t)y * e->cols + x] = e->mask_bit(x, y) ? 255 : 0;
}

// ---- image tracker (tracker_host.cpp.inc) with the device phases supplied by the caller; keypoints packed as launch_fast_detect writes them
static std::vector<std::array<int, 3>> matches_of(const int* m3, int nm) {
  std::vector<std::array<int, 3>> m((size_t)nm);
  for (int i = 0; i < nm; ++i) m[i] = {m3[3 * i], m3[3 * i + 1], m3[3 * i + 2]};
  return m;
}
void hh_tracker_geometry(void* h, int rows, int cols) { static_cast<xb::Estimator*>(h)->tracker_set_geometry(rows, cols, true); }
int hh_tracker_lk_begin(void* h, float* p0, float* p1, int max_pts) { return static_cast<xb::Estimator*>(h)->tracker_lk_begin(p0, p1, max_pts); }
int hh_tracker_lk_accept(void* h, const float* p0, const float* p1, unsigned char* lkst, const unsigned char* desc, const unsigned char* valid) {
  return static_cast<xb::Estimator*>(h)->tracker_lk_accept(p0, p1, lkst, desc, valid);
}
int hh_tracker_detect_budget(void* h) { return static_cast<xb::Estimator*>(h)->detect_budget; }
void hh_tracker_detect_select(void* h, const unsigned* kps, int n) { static_cast<xb::Estimator*>(h)->tracker_detect_select(kps, n); }
int hh_tracker_order_keypoints(void* h, const unsigned* kps, int n, int use_mask, float* kpxy) {
  return static_cast<xb::Estimator*>(h)->tracker_order_keypoints(kps, n, use_mask != 0, kpxy);
}
// descriptors of the query features (32 bytes each); returns their count
int hh_tracker_queries(void* h, unsigned char* out, int max_n) {
  auto* e = static_cast<xb::Estimator*>(h);
  for (size_t i = 0; i < e->query_feats.size() && (int)i < max_n; ++i) memcpy(out + 32 * i, e->query_feats[i]->descriptor, 32);
  return (int)e->query_feats.size();
}
void hh_tracker_detect_select_desc(void* h, const unsigned char* desc, const int* m3, int nm) {
  static_cast<xb::Estimator*>(h)->tracker_detect_select_desc(desc, matches_of(m3, nm));
}
void hh_tracker_lk_finish(void* h) { static_cast<xb::Estimator*>(h)->tracker_lk_finish(); }
int hh_tracker_match_begin(void* h, const unsigned* kps, int n, float* kpxy) { return static_cast<xb::Estimator*>(h)->tracker_match_begin(kps, n, kpxy); }
void hh_tracker_match_finish(void* h, const unsigned char* desc, const int* m3, int nm) {
  static_cast<xb::Estimator*>(h)->tracker_match_finish(desc, matches_of(m3, nm));
}
void hh_tracker_only_finish(void* h) { static_cast<xb::Estimator*>(h)->tracker_only_finish(); }
// per track: id, TrackStatus, last pixel (x, y); returns the track count
int hh_tracks(void* h, int* ids, int* status, double* xy, int max_n) {
  auto* e = static_cast<xb::Estimator*>(h);
  int n = 0;
  for (xb::Feature* f : e->tracks) {
    if (n < max_n) { ids[n] = f->id; status[n] = (int)f->tstatus; xy[2 * n] = f->xp()[0]; xy[2 * n + 1] = f->xp()[1]; }
    ++n;
  }
  return n;
}
// the descriptor of every track (32 bytes each); returns the track count
int hh_track_descriptors(void* h, unsigned char* out, int max_n) {
  auto* e = static_cast<xb::Estimator*>(h);
  for (size_t i = 0; i < e->tracks.size() && (int)i < max_n; ++i) memcpy(out + 32 * i, e->tracks[i]->descriptor, 32);
  return (int)e->tracks.size();
}
// num_failed_to_track, num_outliers_rejected, num_new_detections
void hh_tracker_counts(void* h, int* out3) {
  auto* e = static_cast<xb::Estimator*>(h);
  out3[0] = e->num_failed_to_track; out3[1] = e->num_outliers_rejected; out3[2] = e->num_new_detections;
}
}

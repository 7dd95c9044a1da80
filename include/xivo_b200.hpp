// xivo_b200.hpp — header-only C++ facade over the C ABI (xivo_b200.h, xivo_b200_estimator.h) with the
// reference's class surface for the hot path: xivo::Estimator mirrors the public methods of
// src/estimator.h:131-231 that the per-frame loop and pybind11/pyxivo.cpp:332-398 use, xivo::Tracker the
// read side of src/tracker.h:25-54.  Differences forced by the boundary (SURVEY.md §8b):
//   * images are POD views (rows, cols, channels, tightly packed uint8) instead of cv::Mat;
//   * vectors / matrices are std::array / std::vector<double> (row-major) instead of Eigen types —
//     an Eigen user maps them with Eigen::Map<const Matrix<double, R, C, RowMajor>>;
//   * kMaxGroup / kMaxFeature are constructor arguments (compile-time macros in src/core.h:92-105);
//   * errors the reference raises with LOG(FATAL) / throw surface as xivo::Error (std::runtime_error);
//   * any number of estimators may live in one process (the reference's are singletons, src/factory.cpp:18-22).
#ifndef XIVO_B200_HPP_
#define XIVO_B200_HPP_

#include <algorithm>
#include <array>
#include <chrono>
#include <cstdint>
#include <fstream>
#include <iterator>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "xivo_b200_estimator.h"

namespace xivo {

using timestamp_t = std::chrono::nanoseconds;  // src/core.h: timestamp_t
using Vec2 = std::array<double, 2>;
using Vec3 = std::array<double, 3>;
using Mat3 = std::array<double, 9>;   // row-major
using Mat34 = std::array<double, 12>;  // row-major [R | T]: the SE3 accessors gsb / gbc / gsc

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& what) : std::runtime_error(what), code(c) {}
};

struct ImageView {  // stands in for const cv::Mat&: 8UC1 or 8UC3, continuous
  const uint8_t* data;
  int rows, cols, channels;
};

class Estimator;
using EstimatorPtr = std::shared_ptr<Estimator>;

class Estimator {
 public:
  // CreateSystem(cfg) / CreateSystemTrackerOnly(cfg) (src/factory.cpp:17-122); cfg_json is the config text.
  Estimator(const std::string& cfg_json, int max_groups, int max_features, bool tracker_only = false, int device = 0) {
    if (int rc = xivo_ctx_create(device, &ctx_)) throw Error(rc, xivo_last_error());
    if (int rc = xivo_batch_create(ctx_, cfg_json.c_str(), 1, max_groups, max_features, tracker_only ? 1 : 0, &b_)) {
      const std::string msg = xivo_last_error();
      xivo_ctx_destroy(ctx_);
      throw Error(rc, msg);
    }
    tracker_only_ = tracker_only;
  }
  static EstimatorPtr Create(const std::string& cfg_json, int max_groups = 15, int max_features = 30) {
    return std::make_shared<Estimator>(cfg_json, max_groups, max_features);
  }
  static EstimatorPtr CreateFromFile(const std::string& path, int max_groups = 15, int max_features = 30, bool tracker_only = false) {
    std::ifstream f(path);
    if (!f) throw Error(XIVO_ERR_ARG, "cannot open " + path);
    std::string text((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    return std::make_shared<Estimator>(text, max_groups, max_features, tracker_only);
  }
  ~Estimator() {
    if (b_) xivo_batch_destroy(b_);
    if (ctx_) xivo_ctx_destroy(ctx_);
  }
  Estimator(const Estimator&) = delete;
  Estimator& operator=(const Estimator&) = delete;

  // ---- ingest (src/estimator.h:131-143)
  void InertialMeas(const timestamp_t& ts, const Vec3& gyro, const Vec3& accel) {
    const uint64_t t = (uint64_t)ts.count();
    check(xivo_batch_inertial_meas(b_, &t, gyro.data(), accel.data()));
  }
  void VisualMeas(const timestamp_t& ts, const ImageView& img) { visual(ts, img, 0); }
  void VisualMeasTrackerOnly(const timestamp_t& ts, const ImageView& img) { visual(ts, img, 1); }
  // cv::imread(path) + VisualMeas, the overloads of the reference's binding (pybind11/pyxivo.cpp:338-341) and its vio app
  // (src/app/vio.cpp:72): the PNG file is decoded on the device into the frame ring like IMREAD_COLOR (xivo_batch_visual_meas_png, BGR)
  void VisualMeas(const timestamp_t& ts, const std::string& path) { visual_png(ts, path, 0); }
  void VisualMeasTrackerOnly(const timestamp_t& ts, const std::string& path) { visual_png(ts, path, 1); }
  // xp_and_depths: n x 3 row-major (x, y, depth), as MatX3 rows in the reference
  void VisualMeasPointCloud(const timestamp_t& ts, const std::vector<int>& feature_ids, const std::vector<double>& xp_and_depths) {
    pointcloud(ts, feature_ids, xp_and_depths, 0);
  }
  void VisualMeasPointCloudTrackerOnly(const timestamp_t& ts, const std::vector<int>& feature_ids,
                                       const std::vector<double>& xp_and_depths) {
    pointcloud(ts, feature_ids, xp_and_depths, 1);
  }

  // ---- accessors (src/estimator.h:153-231)
  Mat34 gsb() const { Mat34 g; check(xivo_get_gsb(b_, 0, g.data())); return g; }
  Mat34 gbc() const { Mat34 g; check(xivo_get_gbc(b_, 0, g.data())); return g; }
  Mat34 gsc() const { Mat34 g; check(xivo_get_gsc(b_, 0, g.data())); return g; }
  timestamp_t ts() const { uint64_t t = 0; check(xivo_get_time_ns(b_, 0, &t)); return timestamp_t((int64_t)t); }
  int state_dim() const { return xivo_batch_state_dim(b_); }  // kFullSize
  std::vector<double> P() const {  // N x N row-major (symmetric)
    const int n = state_dim();
    std::vector<double> p((size_t)n * n);
    check(xivo_get_P(b_, 0, p.data()));
    return p;
  }
  std::array<double, 81> Pstate() const { std::array<double, 81> p; check(xivo_get_Pstate(b_, 0, p.data())); return p; }
  Vec3 Vsb() const { return motion().v; }
  Vec3 bg() const { return motion().bg; }
  Vec3 ba() const { return motion().ba; }
  Mat3 Rsg() const { return motion().rsg; }
  bool MeasurementUpdateInitialized() const { return counters()[8] != 0; }
  bool VisionInitialized() const { return counters()[9] != 0; }
  int gauge_group() const { return counters()[2]; }
  int num_instate_features() const { return counters()[0]; }
  int num_instate_groups() const { return counters()[1]; }
  int num_mh_rejected() const { return counters()[3]; }
  int num_tracker_failed_to_track() const { return counters()[4]; }
  int num_tracker_new_detections() const { return counters()[5]; }
  void InitWithSimDepths() { check(xivo_init_with_sim_depths(b_)); }

  // Per-feature accessors, both overloads of src/estimator_accessors.cpp (row-major flat vectors instead of Eigen MatX*).
  // No argument: the features of the last update.  (int n_output): every in-state feature sorted by the norm of its covariance
  // block; like the reference the result has max(count, n_output) rows of which the first min(count, n_output) are filled
  // (the rest is uninitialised there and zero here).
  std::vector<int> InstateFeatureIDs() const { return feature_table(-1).ids; }
  std::vector<int> InstateFeatureIDs(int n) const { return pad(feature_table(n).ids, 1, n); }
  std::vector<int> InstateFeatureSinds() const { return feature_table(-1).sinds; }
  std::vector<int> InstateFeatureSinds(int n) const { return pad(feature_table(n).sinds, 1, n); }
  std::vector<int> InstateFeatureRefGroups() const { return feature_table(-1).refs; }
  std::vector<int> InstateFeatureRefGroups(int n) const { return pad(feature_table(n).refs, 1, n); }
  std::vector<double> InstateFeaturePositions() const { return feature_table(-1).Xs; }  // n x 3
  std::vector<double> InstateFeaturePositions(int n) const { return pad(feature_table(n).Xs, 3, n); }
  std::vector<double> InstateFeatureXc() const { return feature_table(-1).Xc; }  // n x 3
  std::vector<double> InstateFeatureXc(int n) const { return pad(feature_table(n).Xc, 3, n); }
  std::vector<double> InstateFeaturexc() const { return feature_table(-1).xc; }  // n x 3
  std::vector<double> InstateFeaturexc(int n) const { return pad(feature_table(n).xc, 3, n); }
  std::vector<double> InstateFeaturePreds() const { return feature_table(-1).pred; }  // n x 2
  std::vector<double> InstateFeaturePreds(int n) const { return pad(feature_table(n).pred, 2, n); }
  std::vector<double> InstateFeatureMeas() const { return feature_table(-1).meas; }  // n x 2
  std::vector<double> InstateFeatureMeas(int n) const { return pad(feature_table(n).meas, 2, n); }
  std::vector<double> InstateFeatureCovs() const { return feature_table(-1).cov; }  // n x 6: (0,0) (0,1) (0,2) (1,1) (1,2) (2,2)
  std::vector<double> InstateFeatureCovs(int n) const { return pad(feature_table(n).cov, 6, n); }
  std::vector<int> InstateGroupIDs() const { return group_table().ids; }
  std::vector<int> InstateGroupSinds() const { return group_table().sinds; }
  std::vector<double> InstateGroupPoses() const { return group_table().pose; }  // n x 7: qx qy qz qw Tx Ty Tz (MatX7)
  // n x 21 exactly as the reference fills it: its column counter restarts in every row of the 6x6 block, so columns 0..5 end
  // up as cov(5,5) cov(4,5) cov(3,5) cov(2,5) cov(1,5) cov(0,5) and columns 6..20 are never written (zero here).
  std::vector<double> InstateGroupCovs() const {
    const GroupTable g = group_table();
    const size_t n = g.ids.size();
    std::vector<double> out(21 * n, 0.0);
    for (size_t i = 0; i < n; ++i)
      for (int ii = 0; ii < 6; ++ii)
        for (int jj = ii, cnt = 0; jj < 6; ++jj, ++cnt) out[21 * i + cnt] = g.cov[36 * i + 6 * ii + jj];
    return out;
  }
  std::vector<double> InstateGroupCovBlocks() const { return group_table().cov; }  // n x 36: the full blocks (not in the reference)
  std::vector<int> JustDroppedFeatureIDs() const {
    std::vector<int> ids(kMaxTracks);
    int n = 0;
    check(xivo_get_just_dropped(b_, 0, ids.data(), kMaxTracks, &n));
    ids.resize(std::min(n, kMaxTracks));
    return ids;
  }
  double td() const { double t = 0; check(xivo_get_calibration(b_, 0, nullptr, nullptr, &t, nullptr, nullptr)); return t; }
  Mat3 Ca() const { Mat3 m; check(xivo_get_calibration(b_, 0, m.data(), nullptr, nullptr, nullptr, nullptr)); return m; }
  Mat3 Cg() const { Mat3 m; check(xivo_get_calibration(b_, 0, nullptr, m.data(), nullptr, nullptr, nullptr)); return m; }
  std::array<double, 9> CameraIntrinsics() const {  // fx fy cx cy k0 k1 k2 k3 0 (pybind11/pyxivo.cpp:285-287)
    std::array<double, 9> v;
    check(xivo_get_calibration(b_, 0, nullptr, nullptr, nullptr, v.data(), nullptr));
    return v;
  }
  int CameraDistortionType() const { int t = 0; check(xivo_get_calibration(b_, 0, nullptr, nullptr, nullptr, nullptr, &t)); return t; }
  void ScaleInitVelocity(double scale) { check(xivo_scale_init_velocity(b_, 0, scale)); }
  int num_tracker_outlier_rejected() const { return tracker_counters()[0]; }
  int num_oneptransac_rejected() const { return tracker_counters()[3]; }
  bool UsingLoopClosure() const { return false; }  // USE_MAPPER is off in the reference's default build
  void CloseLoop() {}

  // tracked_features_no_descriptor(): (id, last pixel position) per live track
  std::vector<std::tuple<int, Vec2>> tracked_features_no_descriptor() const {
    std::vector<int> ids(kMaxTracks), st(kMaxTracks);
    std::vector<double> xy(2 * kMaxTracks);
    int n = 0;
    check(xivo_get_tracked_features(b_, 0, ids.data(), xy.data(), st.data(), kMaxTracks, &n));
    std::vector<std::tuple<int, Vec2>> out;
    out.reserve(n);
    for (int i = 0; i < n; ++i) out.emplace_back(ids[i], Vec2{xy[2 * i], xy[2 * i + 1]});
    return out;
  }

  // tracked_features(): (id, last pixel position, descriptor) like estimator.h:198 -- the descriptor is the feature's 32 BRIEF bytes
  // (empty when the tracker extracts none; the reference hands out the cv::Mat row)
  std::vector<std::tuple<int, Vec2, std::vector<uint8_t>>> tracked_features() const {
    const auto base = tracked_features_no_descriptor();
    std::vector<uint8_t> desc(32 * (size_t)kMaxTracks), has(kMaxTracks);
    int n = 0;
    check(xivo_get_tracked_descriptors(b_, 0, desc.data(), has.data(), kMaxTracks, &n));
    std::vector<std::tuple<int, Vec2, std::vector<uint8_t>>> out;
    out.reserve(base.size());
    for (size_t i = 0; i < base.size(); ++i)
      out.emplace_back(std::get<0>(base[i]), std::get<1>(base[i]),
                       (int)i < n && has[i] ? std::vector<uint8_t>(desc.begin() + 32 * i, desc.begin() + 32 * (i + 1)) : std::vector<uint8_t>());
    return out;
  }

  xivo_batch* handle() { return b_; }

 private:
  static constexpr int kMaxTracks = 4096;
  struct Motion { Vec3 v, bg, ba; Mat3 rsg; };
  struct Features { std::vector<int> ids, sinds, refs; std::vector<double> Xs, x; };
  struct Groups { std::vector<int> ids, sinds; std::vector<double> gsb; };
  struct FeatureTable { std::vector<int> ids, sinds, refs; std::vector<double> Xs, Xc, xc, pred, meas, cov; };
  struct GroupTable { std::vector<int> ids, sinds; std::vector<double> pose, cov; };

  void check(int rc) const {
    if (rc) throw Error(rc, xivo_last_error());
  }
  void visual(const timestamp_t& ts, const ImageView& img, int tracker_only) {
    const uint64_t t = (uint64_t)ts.count();
    const uint8_t* p = img.data;
    check(xivo_batch_visual_meas(b_, &t, &p, img.rows, img.cols, img.channels, tracker_only));
  }
  void visual_png(const timestamp_t& ts, const std::string& path, int tracker_only) {
    std::ifstream f(path, std::ios::binary);
    if (!f) throw Error(XIVO_ERR_ARG, "cannot open " + path);
    const std::vector<uint8_t> bytes((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    const uint64_t t = (uint64_t)ts.count();
    const uint8_t* src = bytes.data();
    const size_t n = bytes.size();
    if (int rc = xivo_batch_visual_meas_png(b_, &t, &src, &n, 3, tracker_only)) throw Error(rc, path + ": " + xivo_last_error());
  }
  void pointcloud(const timestamp_t& ts, const std::vector<int>& ids, const std::vector<double>& xpd, int tracker_only) {
    if (xpd.size() != 3 * ids.size()) throw Error(XIVO_ERR_ARG, "xp_and_depths must be n x 3");
    const uint64_t t = (uint64_t)ts.count();
    const int n = (int)ids.size();
    const int* pi = ids.data();
    const double* px = xpd.data();
    check(xivo_batch_visual_meas_pointcloud(b_, &t, &n, &pi, &px, tracker_only));
  }
  Motion motion() const {
    Motion m;
    check(xivo_get_motion(b_, 0, m.v.data(), m.bg.data(), m.ba.data(), m.rsg.data()));
    return m;
  }
  std::array<int, XIVO_NUM_COUNTERS> counters() const {
    std::array<int, XIVO_NUM_COUNTERS> c;
    check(xivo_get_counters(b_, 0, c.data()));
    return c;
  }
  Features instate_features() const {
    const int cap = state_dim();
    Features f;
    f.ids.resize(cap); f.sinds.resize(cap); f.refs.resize(cap); f.Xs.resize(3 * (size_t)cap); f.x.resize(3 * (size_t)cap);
    int n = 0;
    check(xivo_get_instate_features(b_, 0, f.ids.data(), f.sinds.data(), f.refs.data(), f.Xs.data(), f.x.data(), cap, &n));
    f.ids.resize(n); f.sinds.resize(n); f.refs.resize(n); f.Xs.resize(3 * (size_t)n); f.x.resize(3 * (size_t)n);
    return f;
  }
  FeatureTable feature_table(int n_output) const {
    const int cap = state_dim();
    FeatureTable t;
    t.ids.resize(cap); t.sinds.resize(cap); t.refs.resize(cap);
    t.Xs.resize(3 * (size_t)cap); t.Xc.resize(3 * (size_t)cap); t.xc.resize(3 * (size_t)cap);
    t.pred.resize(2 * (size_t)cap); t.meas.resize(2 * (size_t)cap); t.cov.resize(6 * (size_t)cap);
    int n = 0;
    check(xivo_get_instate_feature_table(b_, 0, n_output, t.ids.data(), t.sinds.data(), t.refs.data(), t.Xs.data(), t.Xc.data(), t.xc.data(),
                                         t.pred.data(), t.meas.data(), t.cov.data(), cap, &n));
    t.ids.resize(n); t.sinds.resize(n); t.refs.resize(n);
    t.Xs.resize(3 * (size_t)n); t.Xc.resize(3 * (size_t)n); t.xc.resize(3 * (size_t)n);
    t.pred.resize(2 * (size_t)n); t.meas.resize(2 * (size_t)n); t.cov.resize(6 * (size_t)n);
    return t;
  }
  // rows of the (int n_output) overloads: max(number of in-state features, n_output)
  template <typename T>
  std::vector<T> pad(std::vector<T> v, int width, int n_output) const {
    int count = 0;
    check(xivo_get_instate_feature_table(b_, 0, 1 << 20, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, &count));
    v.resize((size_t)width * std::max(count, n_output), T(0));
    return v;
  }
  GroupTable group_table() const {
    const int cap = state_dim();
    GroupTable g;
    g.ids.resize(cap); g.sinds.resize(cap); g.pose.resize(7 * (size_t)cap); g.cov.resize(36 * (size_t)cap);
    int n = 0;
    check(xivo_get_instate_group_table(b_, 0, g.ids.data(), g.sinds.data(), g.pose.data(), g.cov.data(), cap, &n));
    g.ids.resize(n); g.sinds.resize(n); g.pose.resize(7 * (size_t)n); g.cov.resize(36 * (size_t)n);
    return g;
  }
  std::array<int, 4> tracker_counters() const {
    std::array<int, 4> c;
    check(xivo_get_tracker_counters(b_, 0, c.data()));
    return c;
  }
  Groups instate_groups() const {
    const int cap = state_dim();
    Groups g;
    g.ids.resize(cap); g.sinds.resize(cap); g.gsb.resize(12 * (size_t)cap);
    int n = 0;
    check(xivo_get_instate_groups(b_, 0, g.ids.data(), g.sinds.data(), g.gsb.data(), cap, &n));
    g.ids.resize(n); g.sinds.resize(n); g.gsb.resize(12 * (size_t)n);
    return g;
  }

  xivo_ctx* ctx_ = nullptr;
  xivo_batch* b_ = nullptr;
  bool tracker_only_ = false;
};

// One handle of n independent sequences, each fed its own messages per call (xivo_batch_feed / xivo_batch_feed_png): recorded
// sequences with different start times, lengths, IMU rates and dropped frames run side by side, every one of them bit-identical to an
// Estimator fed the same messages one at a time.  Getters take the sequence index.  With IsolateFailures(true) a failed sequence does
// not end the run: Feed / FeedPng return false when sequences failed during the call, Failed() lists them with their messages, and
// their getters throw until ResetSequence brings them back.
class Batch {
 public:
  // What one sequence receives in one Feed / FeedPng call: its IMU samples in order, then at most one frame.
  struct Input {
    std::vector<uint64_t> imu_ts;
    std::vector<Vec3> gyro, accel;
    bool has_frame = false;
    uint64_t frame_ts = 0;
    ImageView image{nullptr, 0, 0, 0};  // Feed
    std::vector<uint8_t> png;            // FeedPng: the PNG file's bytes
  };

  Batch(const std::string& cfg_json, int n_seq, int max_groups, int max_features, bool tracker_only = false, int device = 0) {
    if (int rc = xivo_ctx_create(device, &ctx_)) throw Error(rc, xivo_last_error());
    if (int rc = xivo_batch_create(ctx_, cfg_json.c_str(), n_seq, max_groups, max_features, tracker_only ? 1 : 0, &b_)) {
      const std::string msg = xivo_last_error();
      xivo_ctx_destroy(ctx_);
      throw Error(rc, msg);
    }
    n_ = n_seq;
  }
  ~Batch() {
    if (b_) xivo_batch_destroy(b_);
    if (ctx_) xivo_ctx_destroy(ctx_);
  }
  Batch(const Batch&) = delete;
  Batch& operator=(const Batch&) = delete;
  int size() const { return n_; }

  // Failure isolation (xivo_batch_isolate_failures); turning it off is refused while a sequence is failed
  void IsolateFailures(bool on) { check(xivo_batch_isolate_failures(b_, on ? 1 : 0)); }
  struct Status { int code = 0; std::string msg; };
  // {0, ""} while sequence `seq` runs, else its error code and message
  Status SequenceStatus(int seq) const {
    Status st;
    char buf[1024];
    check(xivo_batch_sequence_status(b_, seq, &st.code, buf, sizeof(buf)));
    if (st.code) st.msg = buf;
    return st;
  }
  // every failed sequence with its status
  std::map<int, Status> Failed() const {
    std::map<int, Status> out;
    for (int s = 0; s < n_; ++s) {
      Status st = SequenceStatus(s);
      if (st.code) out[s] = st;
    }
    return out;
  }

  // in[s] for every sequence s; the frames are image views of one geometry.  false: sequences failed during the call (isolating handle)
  bool Feed(const std::vector<Input>& in, bool tracker_only = false) {
    Flat f = flatten(in);
    std::vector<const uint8_t*> imgs(n_, nullptr);
    int rows = 0, cols = 0, ch = 0;
    for (int s = 0; s < n_; ++s)
      if (in[s].has_frame) {
        imgs[s] = in[s].image.data;
        rows = in[s].image.rows; cols = in[s].image.cols; ch = in[s].image.channels;
      }
    return message(xivo_batch_feed(b_, f.n_imu.data(), f.ts.data(), f.gyro.data(), f.accel.data(), f.frame_ts.data(), imgs.data(), rows, cols, ch, 0,
                                   tracker_only ? 1 : 0));
  }
  // the same with PNG frames (Input::png), decoded on the device like cv::imread (channels = 3: BGR)
  bool FeedPng(const std::vector<Input>& in, int channels = 3, bool tracker_only = false) {
    Flat f = flatten(in);
    std::vector<const uint8_t*> png(n_, nullptr);
    std::vector<size_t> bytes(n_, 0);
    for (int s = 0; s < n_; ++s)
      if (in[s].has_frame) { png[s] = in[s].png.data(); bytes[s] = in[s].png.size(); }
    return message(xivo_batch_feed_png(b_, f.n_imu.data(), f.ts.data(), f.gyro.data(), f.accel.data(), f.frame_ts.data(), png.data(), bytes.data(),
                                       channels, tracker_only ? 1 : 0));
  }
  // sequence `seq` starts over, with the handle's config (cfg_json empty) or a compatible one of its own (xivo_batch_reset_sequence)
  void ResetSequence(int seq, const std::string& cfg_json = std::string()) {
    check(xivo_batch_reset_sequence(b_, seq, cfg_json.empty() ? nullptr : cfg_json.c_str()));
  }

  Mat34 gsb(int seq) const { Mat34 g; check(xivo_get_gsb(b_, seq, g.data())); return g; }
  timestamp_t ts(int seq) const { uint64_t t = 0; check(xivo_get_time_ns(b_, seq, &t)); return timestamp_t((int64_t)t); }
  int num_instate_features(int seq) const { return counters(seq)[0]; }
  int num_instate_groups(int seq) const { return counters(seq)[1]; }
  xivo_batch* handle() { return b_; }

 private:
  struct Flat { std::vector<int> n_imu; std::vector<uint64_t> ts, frame_ts; std::vector<double> gyro, accel; };
  Flat flatten(const std::vector<Input>& in) const {
    if ((int)in.size() != n_) throw Error(XIVO_ERR_ARG, "Batch: expected one Input per sequence");
    Flat f;
    f.n_imu.resize(n_);
    f.frame_ts.assign(n_, 0);
    for (int s = 0; s < n_; ++s) {
      const Input& x = in[s];
      if (x.gyro.size() != x.imu_ts.size() || x.accel.size() != x.imu_ts.size())
        throw Error(XIVO_ERR_ARG, "Batch: sequence " + std::to_string(s) + ": IMU stamps, gyro and accel differ in length");
      f.n_imu[s] = (int)x.imu_ts.size();
      f.ts.insert(f.ts.end(), x.imu_ts.begin(), x.imu_ts.end());
      for (size_t k = 0; k < x.imu_ts.size(); ++k) {
        f.gyro.insert(f.gyro.end(), x.gyro[k].begin(), x.gyro[k].end());
        f.accel.insert(f.accel.end(), x.accel[k].begin(), x.accel[k].end());
      }
      if (x.has_frame) f.frame_ts[s] = x.frame_ts;
    }
    return f;
  }
  void check(int rc) const {
    if (rc) throw Error(rc, xivo_last_error());
  }
  bool message(int rc) const {
    if (rc == XIVO_SEQ_FAILED) return false;
    check(rc);
    return true;
  }
  std::array<int, XIVO_NUM_COUNTERS> counters(int seq) const {
    std::array<int, XIVO_NUM_COUNTERS> c;
    check(xivo_get_counters(b_, seq, c.data()));
    return c;
  }
  xivo_ctx* ctx_ = nullptr;
  xivo_batch* b_ = nullptr;
  int n_ = 0;
};

// Kernel-level Tracker facade: the OpenCV calls of Tracker::DetectLK / UpdateLK (src/tracker.cpp:224, :476-528) on
// caller-owned images.  The stateful tracker (feature list, mask, redetection) lives inside xivo::Estimator, as it does
// behind Estimator::VisualMeas in the reference.
class Tracker {
 public:
  explicit Tracker(int device = 0) {
    if (int rc = xivo_ctx_create(device, &ctx_)) throw Error(rc, xivo_last_error());
  }
  ~Tracker() { if (ctx_) xivo_ctx_destroy(ctx_); }
  Tracker(const Tracker&) = delete;
  Tracker& operator=(const Tracker&) = delete;

  // ---- the stateful surface of src/tracker.h:25-54: Tracker::Create(cfg), Update(img), UpdatePointCloud(ids, xps), features_, counters.
  // cfg_json is a full or tracker-only estimator config (camera_cfg + tracker_cfg, cfg/tumvi_tracker_only_cam0.json); the tracker runs
  // inside a tracker-only estimator (CreateSystemTrackerOnly) with the message reorder buffer switched off, so that every Update takes
  // effect immediately as Tracker::Update does.  Frames are stamped 1 ms apart (the tracker itself never looks at time).
  static std::shared_ptr<Tracker> Create(const std::string& cfg_json, int device = 0) {
    auto t = std::make_shared<Tracker>(device);
    std::string cfg = cfg_json;
    const size_t close = cfg.rfind('}');
    if (close == std::string::npos) throw Error(XIVO_ERR_ARG, "Tracker::Create: not a JSON object");
    cfg.insert(close, ", \"message_buffer_size\": 0");  // a repeated key: the last one wins in the parser
    t->session_ = std::make_shared<Estimator>(cfg, 15, 30, /*tracker_only=*/true, device);
    return t;
  }
  void Update(const ImageView& img) { UpdateLK(img); }
  void UpdateLK(const ImageView& img) { session().VisualMeasTrackerOnly(next_stamp(), img); }
  // xps: n x 2 row-major pixel positions (MatX2 rows in the reference)
  void UpdatePointCloud(const std::vector<int>& feature_ids, const std::vector<double>& xps) {
    std::vector<double> xpd(3 * feature_ids.size(), 1.0);
    for (size_t i = 0; i < feature_ids.size(); ++i) { xpd[3 * i] = xps.at(2 * i); xpd[3 * i + 1] = xps.at(2 * i + 1); }
    session().VisualMeasPointCloudTrackerOnly(next_stamp(), feature_ids, xpd);
  }
  // features_: (id, last pixel position) of every live track, in the tracker's list order
  std::vector<std::tuple<int, Vec2>> features() { return session().tracked_features_no_descriptor(); }
  int num_rejected_outliers() { return session().num_tracker_outlier_rejected(); }
  int num_failed_to_track() { return session().num_tracker_failed_to_track(); }
  int num_new_detections() { return session().num_tracker_new_detections(); }

  struct KeyPoints { std::vector<int> xy; std::vector<int> response; int total = 0; };
  // cv::FastFeatureDetector::detect (TYPE_9_16): raster-ordered keypoints, integer scores
  KeyPoints Detect(const ImageView& img, int threshold, bool nonmax = true, int max_kp = 1 << 16) const {
    KeyPoints k;
    k.xy.resize(2 * (size_t)max_kp); k.response.resize(max_kp);
    if (int rc = xivo_fast_detect(ctx_, img.data, img.rows, img.cols, img.channels, threshold, nonmax ? 1 : 0, k.xy.data(), k.response.data(), max_kp, &k.total))
      throw Error(rc, xivo_last_error());
    const int n = k.total < max_kp ? k.total : max_kp;
    k.xy.resize(2 * (size_t)n); k.response.resize(n);
    return k;
  }
  struct Flow { std::vector<float> pts1; std::vector<uint8_t> status; std::vector<float> err; };
  // cv::calcOpticalFlowPyrLK with OPTFLOW_USE_INITIAL_FLOW semantics when `guess` is given (src/tracker.cpp:526-528)
  Flow TrackLK(const ImageView& prev, const ImageView& next, const std::vector<float>& pts0, const std::vector<float>* guess = nullptr, int win = 15,
               int max_level = 5, int max_iter = 30, double eps = 0.01) const {
    const int n = (int)(pts0.size() / 2);
    Flow f;
    f.pts1 = guess ? *guess : pts0;
    f.status.resize(n); f.err.resize(n);
    if (int rc = xivo_lk_track(ctx_, prev.data, next.data, prev.rows, prev.cols, prev.channels, pts0.data(), f.pts1.data(), f.status.data(), f.err.data(), n,
                               win, max_level, max_iter, eps, guess ? 1 : 0, 1e-4))
      throw Error(rc, xivo_last_error());
    return f;
  }

 private:
  Estimator& session() {
    if (!session_) throw Error(XIVO_ERR_STATE, "stateful Tracker calls need Tracker::Create(cfg)");
    return *session_;
  }
  timestamp_t next_stamp() { return timestamp_t((stamp_ += 1000000)); }
  xivo_ctx* ctx_ = nullptr;
  std::shared_ptr<Estimator> session_;
  int64_t stamp_ = 0;
};

}  // namespace xivo
#endif

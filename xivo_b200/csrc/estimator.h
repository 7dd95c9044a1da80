// Host state machine of the estimator: the reference's Estimator / Tracker / Graph /
// MemoryManager control flow restated around the CUDA kernels.  One `Estimator` per
// independent sequence; a `Batch` advances B of them in lock-step so that every kernel launch
// and every host<->device synchronisation is shared by all sequences.
//
// Reference files followed (relative to /root/reference): src/estimator.cpp, src/manager.cpp,
// src/update.cpp, src/tracker.cpp, src/graph.cpp, src/graphbase.cpp, src/mm.cpp, src/group.h,
// src/feature.cpp, src/options.cpp, src/princedormand.cpp, src/rk4.cpp, src/core.h.
//
// Determinism note (DESIGN.md "documented deviations"): wherever the reference's result depends
// on std::unordered_map iteration order, heap addresses or an unstable std::sort, this
// implementation (and the oracle) use: ascending id for graph iteration, pool-slot order for
// MakePtrVectorUnique, std::stable_sort for candidate ranking.
#pragma once
#include <array>
#include <cstdint>
#include <list>
#include <map>
#include <memory>
#include <algorithm>
#include <set>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "hostmath.h"
#include "json.h"
#include "kernels.h"
#include "triangulate.h"

namespace xb {

enum class TrackStatus : int { CREATED = 0, TRACKED = 1, DROPPED = 2 };
enum class FeatureStatus : int { CREATED = 0, INITIALIZING = 1, READY = 2, INSTATE = 3, REJECTED_BY_FILTER = 4, REJECTED_BY_TRACKER = 5, NULLREFED = 6, GAUGE = 7 };
enum class GroupStatus : int { CREATED = 0, INSTATE = 1, FLOATING = 2, GAUGE = 3 };

// sorted-vector set of ids (the adjacency lists of the visibility graph; ascending = the iteration
// order of the ordered containers they replace)
inline void ids_insert(std::vector<int>& v, int id) {
  if (v.empty() || v.back() < id) { v.push_back(id); return; }
  auto it = std::lower_bound(v.begin(), v.end(), id);
  if (it == v.end() || *it != id) v.insert(it, id);
}
inline void ids_erase(std::vector<int>& v, int id) {
  auto it = std::lower_bound(v.begin(), v.end(), id);
  if (it != v.end() && *it == id) v.erase(it);
}

struct Group {
  int id = -1, sind = -1, birth = 0, slot = -1;  // birth: Estimator::step_counter when the group entered the graph (lifetime = step_counter - birth)
  GroupStatus status = GroupStatus::CREATED;
  M3 Rsb = m3_eye();
  V3 Tsb{{0, 0, 0}};
  // GroupAdj (the features seen from this group) is not stored: a feature is seen by every group created while it lives (one group per
  // frame, every live feature is TRACKED or new in it: manager.cpp:569-627), so "g saw f" <=> f.first_gid <= g.id <= f.last_gid -- see Feature.
  std::set<int> gauge;   // ids of its gauge features (Graph::gauge_features_)
  int n_owned = 0;       // features of the graph whose ref is this group ("does the group own any feature it saw", manager.cpp:288-296, without a scan)
  bool instate() const { return status == GroupStatus::INSTATE || status == GroupStatus::GAUGE; }
  SE3h gsb() const { return SE3h{Rsb, Tsb}; }
  void reset(int new_id) {  // Group::Create/Reset; keeps the slot and the containers' capacity
    id = new_id; sind = -1; birth = 0;
    status = GroupStatus::CREATED;
    Rsb = m3_eye(); Tsb = V3{{0, 0, 0}};
    gauge.clear(); n_owned = 0;
  }
};

struct alignas(64) Feature {
  // Layout: with hundreds of sequences per GPU every per-frame loop over the features starts cache-cold, so what those loops read sits in
  // the first two cache lines (ids / status / owner / id range | local state, prediction, last pixel), the sub-filter's 3 x 3 covariance and
  // the cached world position in the next two, and what only detection, read-back or the optional paths touch comes last.
  // ---- line 0
  int id = -1, sind = -1, birth = 0, slot = -1, init_counter = 0;  // birth: as for Group
  FeatureStatus status = FeatureStatus::CREATED;
  TrackStatus tstatus = TrackStatus::CREATED;
  int track_len = 0;
  Group* ref = nullptr;
  // FeatureAdj keys (the groups that saw this feature) as an id range: every group created between the feature's first and latest frame saw
  // it, groups that were removed since simply no longer exist in Graph::groups.  The per-frame association then costs two stores instead of
  // a sorted insert into a per-feature heap vector and a per-group one (cold: one cache miss each for ~130 features per frame), and removing
  // a group touches no feature.
  int first_gid = -1, last_gid = -1;
  double outlier_counter = 0;
  bool tri_ok = false, has_descriptor = false;
  float response = 0.f;
  // ---- line 1
  alignas(64) double x[3] = {0, 0, 2.0};
  double pred[2] = {-1, -1};
  // Track: only front() (two-view triangulation), back() and the length are ever read on this path (the full
  // history feeds the OOS update, out of scope).
  std::array<double, 2> last_xp{{0, 0}};
  // ---- lines 2, 3
  alignas(64) double P[9] = {0};
  V3 Xs{{0, 0, 0}};
  std::array<double, 2> first_xp{{0, 0}};
  // ---- cold
  // descriptor path (Feature::descriptor(), Feature::keypoint(), feature.h:50-56): the BRIEF-32 bytes set at detection (replaced every frame
  // when `differential`) and the pixel of the keypoint the feature was created from
  uint8_t descriptor[32] = {0};
  float kp0[2] = {0, 0};
  // FeatureAdj itself (graphbase.h:49-51: unordered_map<group id, pixel at the time the group first saw the feature>), kept only when
  // use_depth_opt needs it: Graph::GetObservationsOf walks it in ITERATION order (graphbase.cpp:146-152) and RefineDepth's two_view
  // mode picks the first and the last element of that walk, so it is the same container with the same insert / erase history.
  std::unordered_map<int, std::array<double, 2>> obs;
  bool instate() const { return status == FeatureStatus::INSTATE || status == FeatureStatus::GAUGE; }
  const std::array<double, 2>& xp() const { return last_xp; }
  void observe(double u, double v) {
    last_xp = {u, v};
    if (track_len++ == 0) first_xp = last_xp;
  }
  void reset(int new_id, double u, double v) {  // Feature::Create/Reset (feature.cpp:43-91); keeps slot + capacity
    id = new_id; sind = -1; birth = 0; init_counter = 0;
    status = FeatureStatus::CREATED; tstatus = TrackStatus::CREATED;
    ref = nullptr;
    x[0] = u; x[1] = v; x[2] = 2.0;
    for (double& p : P) p = 0;
    pred[0] = pred[1] = -1;
    outlier_counter = 0; tri_ok = false; response = 0.f;
    has_descriptor = false; kp0[0] = (float)u; kp0[1] = (float)v;
    track_len = 0; first_gid = last_gid = -1;
    std::unordered_map<int, std::array<double, 2>>().swap(obs);  // a fresh map (bucket count and all), as `feature_adj_[fid]` is
    Xs = V3{{0, 0, 0}};
    observe(u, v);
  }
  double z() const { return std::exp(x[2]); }
  double score() const { return -P[8]; }
};
// The per-frame loops walk ~130 features that were last touched a whole round of other sequences ago: ask for the lines of the feature
// `ahead` positions further down the list while the current one is processed (lines = 2: ids + local state, 4: + sub-filter covariance).
inline void prefetch_feature(const Feature* f, int lines) {
  const char* p = reinterpret_cast<const char*>(f);
  for (int k = 0; k < lines; ++k) __builtin_prefetch(p + 64 * k, 1, 1);
}
template <class Vec>
inline void prefetch_ahead(const Vec& v, size_t i, int lines, size_t ahead = 6) {
  if (i + ahead < v.size()) prefetch_feature(v[i + ahead], lines);
}

// One row of the reference's per-feature read-back accessors (src/estimator_accessors.cpp; pybind11/pyxivo.cpp:357-374).
struct FeatureRow {
  int id, sind, ref_group_id;
  double Xs[3];    // InstateFeaturePositions: the cached Feature::Xs_ (last Feature::Xs(gbc) evaluation)
  double Xc[3];    // InstateFeatureXc: unproject_logz(x)
  double xc[3];    // InstateFeaturexc: the local state x = [x/z, y/z, log z]
  double pred[2];  // InstateFeaturePreds: last Feature::Predict pixel
  double meas[2];  // InstateFeatureMeas: last observation
  double cov[6];   // InstateFeatureCovs: P block (0,0) (0,1) (0,2) (1,1) (1,2) (2,2)
};
// One row of InstateGroupIDs / Sinds / Poses / Covs.
struct GroupRow {
  int id, sind;
  double pose[7];   // qx qy qz qw Tx Ty Tz (Eigen::Quaternion(Rsb) as in estimator_accessors.cpp InstateGroupPoses)
  double cov[36];   // the 6x6 block of P, row-major
};

// CircBufWithHash of src/mm.cpp:35-121 (USE_MAPPER off).
template <typename T>
class Pool {
 public:
  void init(int n) {
    items_.clear();
    items_.resize(n);  // contiguous, never resized afterwards: pointers into it stay valid
    for (int i = 0; i < n; ++i) items_[i].slot = i;
    initialized_.assign(n, false);
    active_.assign(n, false);
    n_init_ = 0;
    search_ = 0;
  }
  T* get() {  // returns nullptr when full (reference: LOG(FATAL))
    const int n = (int)items_.size();
    if (n_init_ < n) {
      for (;;) {
        if (!initialized_[search_]) {
          initialized_[search_] = active_[search_] = true;
          ++n_init_;
          T* r = &items_[search_];
          search_ = (search_ + 1) % n;
          return r;
        }
        search_ = (search_ + 1) % n;
      }
    }
    const int start = search_;
    do {
      if (!active_[search_]) {
        active_[search_] = true;
        T* r = &items_[search_];
        search_ = (search_ + 1) % n;
        return r;
      }
      search_ = (search_ + 1) % n;
    } while (search_ != start);
    return nullptr;
  }
  void deactivate(T* t) { active_[t->slot] = false; }
  void destroy(T* t) {
    if (initialized_[t->slot]) --n_init_;
    active_[t->slot] = false;
    initialized_[t->slot] = false;
  }

 private:
  std::vector<T> items_;
  std::vector<char> initialized_, active_;
  int n_init_ = 0, search_ = 0;
};

// id -> object map as a sorted vector (ids are handed out in increasing order, so insertion is a
// push_back); iteration is ascending by id like the ordered maps of the reference's graph.
template <typename T>
struct FlatMap {
  using value_type = std::pair<int, T*>;
  std::vector<value_type> v;
  typename std::vector<value_type>::iterator begin() { return v.begin(); }
  typename std::vector<value_type>::iterator end() { return v.end(); }
  typename std::vector<value_type>::const_iterator begin() const { return v.begin(); }
  typename std::vector<value_type>::const_iterator end() const { return v.end(); }
  size_t size() const { return v.size(); }
  typename std::vector<value_type>::iterator find(int id) {
    auto it = std::lower_bound(v.begin(), v.end(), id, [](const value_type& a, int k) { return a.first < k; });
    return it != v.end() && it->first == id ? it : v.end();
  }
  typename std::vector<value_type>::const_iterator find(int id) const {
    auto it = std::lower_bound(v.begin(), v.end(), id, [](const value_type& a, int k) { return a.first < k; });
    return it != v.end() && it->first == id ? it : v.end();
  }
  size_t count(int id) const { return find(id) != v.end(); }
  T* at(int id) const {
    auto it = find(id);
    if (it == v.end()) throw std::out_of_range("FlatMap::at");
    return it->second;
  }
  void put(int id, T* p) {
    if (v.empty() || v.back().first < id) { v.emplace_back(id, p); return; }
    auto it = std::lower_bound(v.begin(), v.end(), id, [](const value_type& a, int k) { return a.first < k; });
    if (it != v.end() && it->first == id) it->second = p;
    else v.insert(it, value_type(id, p));
  }
  void erase(int id) {
    auto it = find(id);
    if (it != v.end()) v.erase(it);
  }
};

// Visibility graph (src/graph.cpp, src/graphbase.cpp): id-ordered object maps; the adjacency lists live
// in the objects themselves (Feature::adj, Group::adj, Group::gauge).
// Allocator of the two hash maps below: their list nodes (24 bytes each, allocated and freed one at a time as features come and go) are
// carved from chunks owned by the map, with a free list, instead of one malloc block each.  The container's algorithm -- and with it the
// iteration order the decisions depend on -- is untouched; what changes is that the ~130 nodes a per-frame walk chases lie in a few
// dozen cache lines instead of one line each (with 512 sequences per GPU every phase starts cache-cold: tests/cpp/host_perf.cpp).
struct NodeArena {
  std::vector<std::unique_ptr<unsigned char[]>> chunks;
  void* free_list = nullptr;
  size_t block = 0, used = 0, cap = 0;
  void* get(size_t bytes) {
    if (!block) block = (bytes + 15) & ~(size_t)15;
    if (free_list) { void* p = free_list; free_list = *static_cast<void**>(p); return p; }
    if (used + block > cap) { cap = block * 256; used = 0; chunks.emplace_back(new unsigned char[cap]); }
    void* p = chunks.back().get() + used;
    used += block;
    return p;
  }
  void put(void* p) { *static_cast<void**>(p) = free_list; free_list = p; }
};
template <typename T>
struct ArenaAlloc {
  using value_type = T;
  std::shared_ptr<NodeArena> arena;
  ArenaAlloc() : arena(std::make_shared<NodeArena>()) {}
  template <typename U>
  ArenaAlloc(const ArenaAlloc<U>& o) : arena(o.arena) {}
  T* allocate(size_t n) {
    // single objects of one size (the list nodes) come from the arena; arrays (the bucket table) and anything else from the heap
    if (n == 1 && sizeof(T) >= sizeof(void*) && (!arena->block || arena->block == ((sizeof(T) + 15) & ~(size_t)15))) return static_cast<T*>(arena->get(sizeof(T)));
    return static_cast<T*>(::operator new(n * sizeof(T)));
  }
  void deallocate(T* p, size_t n) {
    if (n == 1 && sizeof(T) >= sizeof(void*) && arena->block == ((sizeof(T) + 15) & ~(size_t)15)) arena->put(p);
    else ::operator delete(p);
  }
  template <typename U>
  bool operator==(const ArenaAlloc<U>& o) const { return arena == o.arena; }
  template <typename U>
  bool operator!=(const ArenaAlloc<U>& o) const { return arena != o.arena; }
};
template <typename P>
using IdHashMap = std::unordered_map<int, P, std::hash<int>, std::equal_to<int>, ArenaAlloc<std::pair<const int, P>>>;

struct Graph {
  FlatMap<Feature> features;
  FlatMap<Group> groups;
  // The reference keeps its objects in std::unordered_map<int, Ptr> (graphbase.h:49-51) and three decisions read them in
  // ITERATION order (GraphBase::GetFeaturesIf / GetGroupsIf, graphbase.cpp:124-146): the gauge-feature candidates
  // (graph.cpp:291), the group candidates and their features in AddGroupOfFeatures (manager.cpp:479-497) and the unsorted
  // "median" of AdaptInitialDepth (manager.cpp:257-266).  That order is a property of libstdc++'s hash table, so the same
  // container type is kept here with the same insert / erase history and used for exactly those reads; everything else uses
  // the id-sorted maps above.  (oracle/estimator_oracle.py does the same through oracle/stdumap.cpp; tests/test_reference_pin.py
  // checks the result against the reference's own estimator.)
  IdHashMap<Feature*> um_features;
  IdHashMap<Group*> um_groups;
  bool keep_observations = false;  // maintain Feature::obs (use_depth_opt)
  const int* step = nullptr;       // the owning estimator's step counter: objects entering the graph are stamped with it
  template <typename Pred>
  std::vector<Feature*> features_std(Pred p) const {
    std::vector<Feature*> out;
    for (const auto& kv : um_features)
      if (p(kv.second)) out.push_back(kv.second);
    return out;
  }
  template <typename Pred>
  std::vector<Group*> groups_std(Pred p) const {
    std::vector<Group*> out;
    for (const auto& kv : um_groups)
      if (p(kv.second)) out.push_back(kv.second);
    return out;
  }
  void add_feature(Feature* f);
  void add_group(Group* g);
  void remove_feature(Feature* f);
  void remove_group(Group* g);
  void add_group_to_feature(Group* g, Feature* f);
  void add_feature_to_group(Feature* f, Group* g);
  bool has_feature(int fid) const { return features.count(fid) != 0; }
  template <typename Pred>
  std::vector<Feature*> features_if(Pred p) const {
    std::vector<Feature*> out;
    for (auto& kv : features)
      if (p(kv.second)) out.push_back(kv.second);
    return out;
  }
  template <typename Pred>
  std::vector<Group*> groups_if(Pred p) const {
    std::vector<Group*> out;
    for (auto& kv : groups)
      if (p(kv.second)) out.push_back(kv.second);
    return out;
  }
  Group* find_new_owner(Feature* f) const;
};

struct TrackerCfg {
  int mask_size = 15, margin = 16, num_features_min = 120, num_features_max = 150, max_pixel_displacement = 64;
  int win_size = 15, max_level = 4, max_iter = 15;
  double eps = 0.01;
  int fast_threshold = 5;
  bool fast_nonmax = true, normalize = false;
  // descriptor path (tracker.cpp:176-217): BRIEF-32 per track and frame, descriptor check, rescue of dropped tracks, MATCH tracker
  bool extract_descriptor = false, differential = true, match_dropped_tracks = false, match_tracker = false;
  int descriptor_distance_thresh = -1;
  // tracker-level outlier rejection by homography (tracker.cpp:131-150): method = cv::RANSAC (8) or cv::LMEDS (4)
  bool do_outlier_rejection = false;
  int outlier_method = 8, outlier_max_iters = 2000;
  double outlier_reproj_thresh = 3.0, outlier_confidence = 0.995;
};

struct EstimatorCfg {
  bool simulation = false;
  std::string integration_method = "unspecified";
  bool clamp_signals = false;
  double max_accel[3] = {0, 0, 0}, max_gyro[3] = {0, 0, 0};
  double sub_Rtri = 3.5 * 3.5, sub_mh = 5.991;
  int sub_ready_steps = 5;
  // Feature::RefineDepth on in-state candidates (estimator.cpp:143-155; depth_opt.damping is parsed by the reference and never used)
  bool use_depth_opt = false, depth_two_view = false, depth_use_hessian = false;
  int depth_max_iters = 5;
  double depth_eps = 1e-4, depth_max_res_norm = 2.0;
  bool triangulate_pre_subfilter = false;  // Feature::Triangulate on a feature's second observation (manager.cpp:229-231)
  TriOptions tri;
  double adapt_weight = 0.99;
  int adapt_min_lifetime = 5;
  int remove_outlier_counter = 10, group_degrees_fixed = 4, max_group_lifetime = 1;
  M3 Ca = m3_eye(), Cg = m3_eye();
  V3 g{{0, 0, -9.8}};
  double Qmodel[529] = {0}, Qimu[144] = {0};
  double R = 1, Roos = 1;
  double init_z = 1, init_std_x = 1, init_std_y = 1, init_std_z = 1, min_z = 0.05, max_z = 5;
  double init_std_x_badtri = 0, init_std_y_badtri = 0, init_std_z_badtri = 0;  // jsoncpp: a missing number reads as 0 (estimator.cpp:356-358)
  bool use_MH_gating = true;
  bool use_1pt_RANSAC = false;
  double ransac_thresh = 5.0, ransac_prob = 0.95, ransac_chi2 = 5.89;
  int min_inliers = 5;
  double MH_thresh = 5.991, MH_mult = 1.1;
  double owner_change_cov_factor = 1.5;
  int strict_criteria_timesteps = 5, num_gauge_xy_features = 3;
  double collinear_thresh = 1e-3, max_subfilter_outlier = 0.01;
  int gravity_init_counter = 20;
  double pd_stepsize = 0.002, rk4_stepsize = 0.002;
  int max_features_mem = 256, max_groups_mem = 128;
  int message_buffer_size = 10;
  bool cov_update_tf32x3 = false;  // "covariance_update": "tf32x3" (ekf_tc_kernels.cu)
};

struct MotionX {
  M3 Rsb = m3_eye(), Rbc = m3_eye(), Rsg = m3_eye();
  V3 Tsb{{0, 0, 0}}, Vsb{{0, 0, 0}}, bg{{0, 0, 0}}, ba{{0, 0, 0}}, Tbc{{0, 0, 0}};
  int counter = 0;
  double td = 0;  // camera-IMU time offset X.td (estimator.cpp:245); constant: USE_ONLINE_TEMPORAL_CALIB is off in the reference build
};

struct Msg {
  uint64_t ts = 0;
  int type = 0;  // 0 inertial, 1 visual image, 2 visual tracker-only, 3 point cloud, 4 point cloud tracker-only
  double gyro[3] = {0, 0, 0}, accel[3] = {0, 0, 0};
  int img_slot = -1;
  std::vector<int> ids;
  std::vector<double> xp_depth;
  uint64_t seqno = 0;
};

class Batch;

class Estimator {
 public:
  Estimator(const Json& cfg, EkfLayout lay, bool tracker_only);
  // ---- message heap (src/estimator.cpp:923-1046)
  void push(Msg&& m);
  bool pop_ready(Msg* out);
  // ---- inertial path (src/estimator.cpp:475-592)
  void inertial_internal(uint64_t ts, const double* gyro, const double* accel);
  // ---- visual path, split at the device phases
  bool visual_begin(uint64_t ts, int type);  // false -> message dropped / vision not initialised
  void predict_features();
  void tracker_update_pointcloud(const std::vector<int>& ids, const std::vector<double>& xp_depth);
  void update_step_pre();                                                // lifetimes, ProcessTracks pass 1
  void update_step_after_subfilter(const SubfilterOut* out);            // ProcessTracks pass 2, SelectAndAddNewFeatures
  void update_step_after_gate(const double* mh, const double* diag_after_edits = nullptr);  // OutlierRejection .. in_current_ekf_update_ (returns early with ransac.active set)
  void ransac_after_temp_update(const double* err);                     // AbsorbError of the low-innovation update (motion state only)
  bool ransac_begin(const double* diag_after_edits);
  void ransac_finish(const double* mh_at_temp_state, const std::vector<Feature*>& table_order);  // rescue / reject, RestoreState, then the tail of update_step_after_gate
  void update_step_after_gate_finish();
  void update_step_after_update(const double* err, const double* Pmm, const double* diagP, bool had_update);
  void tracker_only_finish();
  // ---- image tracker (tracker_host.cpp.inc: src/tracker.cpp), split at the device phases.  Arrays are the sequence's own rows of the
  // read-back tables; keypoints are packed as launch_fast_detect writes them.
  void tracker_set_geometry(int rows, int cols, bool host_mask);  // host_mask: the mask bitmap exists only on the host-decision path
  // UpdateLK up to the LK launch: writes p0 / p1 (max_pts rows) and returns the frame's kind
  enum { kTrkOverflow = -1, kTrkFirst = 1, kTrkLK = 2, kTrkEmpty = 3 };  // (values as track_accept_kernel reads them)
  int tracker_lk_begin(float* p0, float* p1, int max_pts);
  // UpdateLK's descriptor check, accept loop and homography rejection (desc / desc_valid: BRIEF at p1, null without descriptors);
  // returns the detection budget
  int tracker_lk_accept(const float* p0, const float* p1, uint8_t* lkst, const uint8_t* desc, const uint8_t* desc_valid);
  // DetectLK's greedy pick: without descriptors from the detected keypoints; with descriptors from sorted_kp (tracker_order_keypoints),
  // their descriptors and the cross-checked (query, keypoint, distance) matches of query_feats
  void tracker_detect_select(const unsigned* kps, int n);
  void tracker_detect_select_desc(const uint8_t* desc, const std::vector<std::array<int, 3>>& matches);
  void tracker_lk_finish();
  // keypoints in the order DetectLK / UpdateMatch walk them, into sorted_kp and kpxy (x, y per keypoint); returns their count
  int tracker_order_keypoints(const unsigned* kps, int n, bool use_mask, float* kpxy);
  // UpdateLK with the decisions made on the device: the accept kernel's keep flags, the select kernel's picks
  void tracker_replay(int kind, const float* p1, const uint8_t* keep, int need, const unsigned* picks, int npicks);
  // UpdateMatch: keypoint order and query list before the device phase, the matches applied after it
  int tracker_match_begin(const unsigned* kps, int n, float* kpxy);
  void tracker_match_finish(const uint8_t* desc, const std::vector<std::array<int, 3>>& matches);

  // helpers used by Batch
  EkfLayout lay;
  EstimatorCfg c;
  TrackerCfg tc;
  CameraParams cam;
  bool tracker_only = false;
  MotionX X;
  double Pmm[529];  // host mirror of the motion block of P
  double Phi[529];  // pending strip transition (product of per-substep F)
  bool prop_pending = false;
  // Runge-Kutta records whose covariance algebra has not run on the device yet: one per stage (the default), or, with
  // compact_records (set by Batch, whose kernel rebuilds the intermediate stages), one per sub-step
  std::vector<ImuStage> stages;
  std::vector<ImuStep> steps;
  bool compact_records = false;
  int stages_per_step = 7;  // 7 = Prince-Dormand, 4 = RK4
  int pending_stages() const { return (int)stages.size() + (int)steps.size() * stages_per_step; }
  // the queue must be flushed to the device before it can overflow (one Propagate call adds <= ~256 stages)
  bool needs_state_now() const { return pending_stages() > kMaxStages - 320; }
  std::vector<EditOp> edits;  // pending covariance edits, in order
  std::vector<double> diagP;  // last downloaded diagonal of P
  std::vector<char> gsel, fsel;
  std::vector<Group*> gslot;  // the group in state slot s (null = free): the per-frame tables walk G slots instead of every live group
  Graph graph;
  Pool<Feature> fpool;
  Pool<Group> gpool;
  std::vector<Feature*> tracks;  // Tracker::features_ (a list in the reference; order is what matters)
  std::vector<Feature*> instate_features, new_features, inliers, in_update, subfilter_list;
  std::vector<Group*> instate_groups, needs_new_gauge;
  // Estimator::affected_groups_ is a std::unordered_set<GroupPtr> (estimator.h:364): its few elements sit in distinct buckets, where libstdc++
  // links every new node at the head of the list, so DiscardAffectedGroups meets them in REVERSE insertion order (exact for two groups;
  // pinned on the reference by tests/test_reference_pin.py::ransac_two_groups_89, where the order decides which group adopts whose features)
  struct OrderedIds {
    std::vector<int> v;
    void insert(int id) { if (std::find(v.begin(), v.end(), id) == v.end()) v.push_back(id); }
    bool empty() const { return v.empty(); }
    void clear() { v.clear(); }
  } affected_groups;
  // ---- filter-level 1-point RANSAC (Estimator::OnePointRANSAC, update.cpp:213-393; call site manager.cpp:642-656) ----
  // Host decisions around two extra device phases: (1) a temporary update with the low-innovation features on a covariance whose
  // high-innovation rows are zeroed, (2) Jacobians + Mahalanobis distances of the high-innovation features at the temporarily absorbed state.
  struct Ransac {
    bool active = false;                 // this frame needs the two device phases
    std::vector<Feature*> mh_inliers;    // the MH inliers that are still in the state (input order = output order)
    std::vector<char> low;               // per mh_inlier: |xp - Predict| < 1pt_RANSAC_thresh
    std::vector<EditOp> zero_edits;      // rows / columns zeroed before the temporary update
    MotionX X0;                          // BackupState
    // what the Jacobians of the survivors are recomputed from at the end of OnePointRANSAC (update.cpp:381-385), in the index space of the
    // device feature table: a survivor whose owner changed in the DiscardAffectedGroups that precedes the RANSAC (manager.cpp:645) is
    // re-linearised about its NEW reference group and re-expressed state here -- unlike in frames without RANSAC, where J_ stays as
    // ComputeInstateJacobians left it
    std::vector<char> jalive;
    std::vector<double> jx;              // 3 per table entry
    std::vector<int> jref, jsind;
  } ransac;
  int num_oneptransac_rejected = 0;
  bool in_ransac_destroy = false;        // RemoveFeatureFromState inside OnePointRANSAC precedes RestoreState: its zeroing of P_ does not survive
  std::vector<int> just_dropped_ids;
  std::map<int, double> ids_to_depths;
  bool sim_initialize_depths = false;
  int gauge_group = -1;
  int step_counter = 0;  // update steps so far (UpdateStep, manager.cpp:18-46): the clock of Feature::lifetime_ / Group::lifetime_
  int feature_counter = 10000, group_counter = 0;
  // tracker bookkeeping (src/tracker.h)
  bool tracker_initialized = false;
  // Tracker::mask_ as a bitmap: bit (y, x) set = free pixel; one row = mask_stride 64-bit words
  std::vector<uint64_t> mask;
  int mask_stride = 0;
  bool mask_bit(int x, int y) const { return (mask[(size_t)y * mask_stride + (x >> 6)] >> (x & 63)) & 1; }
  void mask_fill_row(int y, int x0, int x1, bool v);  // [x0, x1] inclusive
  int mask_half = -1;  // MaskOut's function-local static (tracker.cpp:763)
  int rows = 0, cols = 0;
  int num_failed_to_track = 0, num_new_detections = 0, num_mh_rejected = 0;
  int num_outliers_rejected = 0;  // Tracker::num_outliers_rejected_ (keeps its last value when OutlierRejection returns early, tracker.cpp:598, :713-715)
  std::vector<unsigned> sorted_kp;      // this frame's detected keypoints in selection order (tracker_order_keypoints)
  std::vector<Feature*> query_feats;    // the features whose descriptors are matched against sorted_kp
  int detect_budget = 0;                // DetectLK's num_to_add of this frame (0: no detection)
  bool check_homography = false;        // DetectLK's check_homography: this frame's outlier rejection ran
  int num_depth_refined = 0, num_depth_refine_failed = 0;
  int num_good_triangulations = 0, num_bad_triangulations = 0;  // Feature::num_good/bad_triangulations_ (feature.cpp:730-748)
  // time / imu (src/estimator.cpp)
  bool gravity_initialized = false, vision_initialized = false, meas_update_initialized = false;
  int gravity_init_counter = 0, imu_counter = 0, vision_counter = 0;
  std::vector<V3> gravity_init_buf;
  uint64_t last_imu_time = 0, curr_imu_time = 0, last_vision_time = 0, curr_vision_time = 0, last_time = 0, curr_time = 0;
  V3 last_accel{{0, 0, 0}}, curr_accel{{0, 0, 0}}, last_gyro{{0, 0, 0}}, curr_gyro{{0, 0, 0}}, slope_accel{{0, 0, 0}}, slope_gyro{{0, 0, 0}};
  int error = 0;  // sticky error code (reference: throw / LOG(FATAL))
  std::string error_msg;

  SE3h gsb() const { return SE3h{X.Rsb, X.Tsb}; }
  SE3h gbc() const { return SE3h{X.Rbc, X.Tbc}; }
  Feature* create_feature(double x, double y);
  void destroy_feature(Feature* f) { fpool.destroy(f); }
  void deactivate_feature(Feature* f) { fpool.deactivate(f); }
  // mask helpers (tracker.cpp:760-774)
  void reset_mask();
  void mask_out(double x, double y);
  bool mask_valid(double x, double y) const;
  Feature* track_keypoint(unsigned k, const uint8_t* desc);           // a detected keypoint becomes a new track (desc: its descriptor or null)
  bool match_passes(const Feature* f, unsigned k, int dist) const;    // CheckDescriptorDistance + displacement of a cross-checked match

 private:
  std::vector<Msg> buf_;
  bool buf_initialized_ = false;
  uint64_t seqno_ = 0;
  bool good_timestamp(uint64_t now) const;
  void update_system_clock(uint64_t now);
  bool initialize_gravity();
  void propagate(bool visual_meas);
  void compose_motion(MotionX& Xs, const V3& V, const V3& gyro, const V3& accel, double dt) const;
  static void compose_motion_core(M3& Rsb, V3& Tsb, V3& Vsb, const V3& V, const V3& gc, const V3& ac, const V3& g_s, double dt);
  static V3 stage_velocity(const M3& Rsb, const V3& Vsb, const V3& ac, const V3& g_s, double dt);
  void record_stage(const M3& Rsb, const V3& gc, const V3& ac, double h_enc);
  void nominal_step(bool pd, const V3& gyro0, const V3& accel0, double h, bool closes_call);
  void integrate_nominal(const V3& gyro0, const V3& accel0, double dt);
  void state_plus(const double* dX);
  // state slots
  void add_group_to_state(Group* g);
  void add_feature_to_state(Feature* f);
  void remove_group_from_state(Group* g);
  void remove_feature_from_state(Feature* f);
  void fix_feature_xy(Feature* f);
  // manager.cpp
  void select_and_add_new_features();
  void add_features_within_groups();
  void zero_gauge_xy_add_features();
  void add_group_of_features(int free_group_slots);
  void discard_affected_groups();
  void find_new_gauge_features();
  std::vector<Feature*> graph_find_new_gauge_features(Group* g);
  void destroy_features(const std::vector<Feature*>& v);
  void destroy_and_untrack(const std::vector<Feature*>& v);
  void discard_features(const std::vector<Feature*>& v);
  void discard_group(Group* g);
  void adapt_initial_depth();
  void enforce_max_group_lifetime();
  void switch_ref_group();
  bool candidate(const Feature* f, bool strict) const;
  V3 feature_Xc(const Feature* f, M3* J = nullptr) const;
  V3 feature_Xs(Feature* f, M3* J = nullptr) const;
  bool change_owner(Feature* f, Group* nref);
  void feature_initialize(Feature* f, double z0, double sx, double sy, double sz);
  void triangulate_feature(Feature* f);
  bool refine_depth(Feature* f);

 public:
  // read-back tables (estimator_accessors.cpp); P = host copy of the N x N covariance, row-major
  std::vector<FeatureRow> instate_feature_rows(const double* P, int n_output) const;
  std::vector<GroupRow> instate_group_rows(const double* P) const;
};

// The first setting that one batch handle needs to be the same for every sequence and that differs between the two estimators,
// as its config key ("tracker_cfg.KLT.win_size"), or "" when a sequence configured like `b` may join a handle configured like `a`.
std::string batch_incompatibility(const Estimator& a, const Estimator& b);

// cv::BFMatcher's cross-checked matches (knnMatch with compactResult, in query order) as (query, keypoint, distance), from the nearest
// keypoint of every query (best_t / best_t_dist) and the nearest query of every keypoint (best_q)
void cross_checked(int nq, const int* best_t, const int* best_t_dist, const int* best_q, std::vector<std::array<int, 3>>* out);

}  // namespace xb

// CPU harness for the compact Runge-Kutta records (one ImuStep per sub-step, what Batch streams to imu_cov_propagate): compiled with g++
// (no nvcc, no GPU) for tests/test_compact_records.py, which runs the same IMU stream through an estimator that writes one record per
// stage and one that writes one per sub-step and compares their nominal states and, stage by stage, the records.
#include <cstring>
#include <string>

#include "../../xivo_b200/csrc/estimator.h"
#include "../../xivo_b200/csrc/homography.h"

namespace xb {
struct HostScope {
  explicit HostScope(const char*) {}
};
}  // namespace xb

#include "../../xivo_b200/csrc/estimator_host.cpp.inc"

extern "C" {
void* cr_create(const char* cfg_json, int compact) {
  try {
    auto* e = new xb::Estimator(xb::Json::parse(cfg_json), xb::EkfLayout{4, 14}, false);
    e->compact_records = compact != 0;
    return e;
  } catch (const std::exception&) {
    return nullptr;
  }
}
void cr_destroy(void* h) { delete static_cast<xb::Estimator*>(h); }
void cr_inertial(void* h, unsigned long long ts, const double* gyro, const double* accel) { static_cast<xb::Estimator*>(h)->inertial_internal(ts, gyro, accel); }
int cr_visual_begin(void* h, unsigned long long ts) { return static_cast<xb::Estimator*>(h)->visual_begin(ts, 3) ? 1 : 0; }
int cr_pending_stages(void* h) { return static_cast<xb::Estimator*>(h)->pending_stages(); }
int cr_needs_state_now(void* h) { return static_cast<xb::Estimator*>(h)->needs_state_now() ? 1 : 0; }
// Rsb(9) Tsb(3) Vsb(3)
void cr_motion(void* h, double* out15) {
  const xb::MotionX& X = static_cast<xb::Estimator*>(h)->X;
  memcpy(out15, X.Rsb.m, 72); memcpy(out15 + 9, X.Tsb.v, 24); memcpy(out15 + 12, X.Vsb.v, 24);
}
// the pending records as per-stage records (16 doubles: R(9), gyro-bg(3), accel-ba(3), h on the first stage of a sub-step, else 0);
// compact records are expanded by imu_stage_from_step, the function the kernel uses.  Returns the stage count and clears the queue.
int cr_take_stages(void* h, double* out, int max_records) {
  auto* e = static_cast<xb::Estimator*>(h);
  const int n = e->pending_stages();
  if (n > max_records) return -1;
  if (!e->compact_records) {
    if (n) memcpy(out, e->stages.data(), sizeof(xb::ImuStage) * (size_t)n);
  } else {
    const int nst = e->stages_per_step;
    for (size_t k = 0; k < e->steps.size(); ++k)
      for (int s = 0; s < nst; ++s) {
        xb::M3 R;
        xb::V3 gc, ac;
        xb::imu_stage_from_step(e->steps[k], s, nst == 7, &R, &gc, &ac);
        double* o = out + 16 * (k * nst + s);
        memcpy(o, R.m, 72); memcpy(o + 9, gc.v, 24); memcpy(o + 12, ac.v, 24);
        o[15] = s == 0 ? e->steps[k].h : 0.0;
      }
  }
  e->stages.clear();
  e->steps.clear();
  return n;
}
}

// CPU test harness for the batch-wide setting check of xivo_batch_reset_sequence (batch_incompatibility in
// xivo_b200/csrc/estimator_host.cpp.inc): compiled with g++ (no nvcc, no GPU) into a small shared object that
// tests/test_batch_reset_logic.py drives through ctypes.  Test infrastructure only — nothing here is linked into libxivo_b200.so.
#include <cstring>
#include <string>

#include "../../xivo_b200/csrc/estimator.h"
#include "../../xivo_b200/csrc/homography.h"

namespace xb {
struct HostScope {  // the library's version also feeds the profiler
  explicit HostScope(const char*) {}
};
}  // namespace xb

#include "../../xivo_b200/csrc/estimator_host.cpp.inc"

namespace {
std::string g_err;
}

extern "C" {
const char* rh_error() { return g_err.c_str(); }

// 1: the two configs may share a handle; 0: they may not, `key` (capacity cap) holds the first batch-wide key that differs;
// -1: a config was refused by the parser (rh_error)
int rh_incompatibility(const char* handle_cfg, int G, int F, int tracker_only, const char* seq_cfg, int G2, int F2, int tracker_only2, char* key, int cap) {
  try {
    const xb::Estimator a(xb::Json::parse(handle_cfg), xb::EkfLayout{G, F}, tracker_only != 0);
    const xb::Estimator b(xb::Json::parse(seq_cfg), xb::EkfLayout{G2, F2}, tracker_only2 != 0);
    const std::string k = xb::batch_incompatibility(a, b);
    snprintf(key, cap, "%s", k.c_str());
    return k.empty() ? 1 : 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}
}
